"""Bundle adjustment model (reference: README.md:163-198 sparse example, examples/module/ba).

    forward(observations, camera_indices, point_indices) = project(points[pidx], poses[cidx]) - observations      (M, 2)
    project(p, T) = -(T p)[:2] / (T p)[2]

Both `poses` (C, 7) SE3 and `points_3d` (P, 3) are parameters.  `forward` is ordinary LieTensor code (generic dense
route / the reference run it as is); `pp.optim.LM(..., solver=PCG(), sparse=True)` recognises the type and solves the
step with the point blocks eliminated (Schur complement) and a matrix-free PCG on the cameras
(optim/structured.py:BAProblem)."""
from torch import nn

from ..autograd.function import psjac
from ..lietensor.lietensor import Parameter


class BundleAdjustment(nn.Module):
    def __init__(self, poses, points_3d):
        super().__init__()
        self.poses = Parameter(poses, sjac=True)
        self.points_3d = Parameter(points_3d, sjac=True)

    @staticmethod
    @psjac
    def project(points, poses):
        pts = poses.Act(points)
        return -pts[..., :2] / pts[..., 2].unsqueeze(-1)

    def forward(self, observations, camera_indices, point_indices):
        poses = self.poses[camera_indices]
        points = self.points_3d[point_indices]
        return BundleAdjustment.project(points, poses) - observations


class BALBundleAdjustment(nn.Module):
    """Bundle adjustment of a BAL ("Bundle Adjustment in the Large") problem: the model of the reference's
    examples/module/ba/bundle_adjustment.py `Reproj(K, C, P)`.

        y = T_c p_j,   n = -y[:2] / y[2],   r = f (1 + k1 |n|^2 + k2 |n|^4) n - z                      (M, 2)

    Parameters, in the reference's order: `intrinsics` (C, 3) = (f, k1, k2) per camera, `poses` (C, 7) SE3 and
    `points_3d` (P, 3).  `BALBundleAdjustment(d["intrinsics"], d["cameras"], d["points"])` takes the output of
    `pp.utils.read_bal` as it is.  `forward` is ordinary LieTensor code; on CUDA, `pp.optim.LM(..., solver=PCG(),
    sparse=True)` recognises the type and solves each step with the points eliminated (Schur complement) and a
    matrix-free PCG over the 9 unknowns (pose, f, k1, k2) of every camera (optim/structured.py:BALProblem)."""

    def __init__(self, intrinsics, poses, points_3d):
        super().__init__()
        self.intrinsics = Parameter(intrinsics, sjac=True)
        self.poses = Parameter(poses, sjac=True)
        self.points_3d = Parameter(points_3d, sjac=True)

    @staticmethod
    @psjac
    def project(intrinsics, poses, points):
        y = poses.Act(points)
        n = -y[..., :2] / y[..., [2]]
        rho = n.square().sum(dim=-1, keepdim=True)
        f, k1, k2 = intrinsics[..., :1], intrinsics[..., 1:2], intrinsics[..., 2:3]
        return f * (1 + k1 * rho + k2 * rho.square()) * n

    def forward(self, observations, camera_indices, point_indices):
        return BALBundleAdjustment.project(self.intrinsics[camera_indices], self.poses[camera_indices],
                                           self.points_3d[point_indices]) - observations
