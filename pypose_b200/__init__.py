"""pypose_b200 — an H100-native implementation of PyPose's data-parallel core.

`import pypose_b200 as pp` exposes the hot-path surface of pypose v0.9.5 (LieTensor op family,
pp.optim LM/GN inner loop, IMU preintegration scan) with every numeric operator implemented as a
hand-written sm_90a CUDA kernel behind a C-ABI library (include/b200pose.h).  There is no CPU
fallback: operators on CPU tensors raise.
"""
import torch

from ._version import __version__
from . import _C
from .lietensor import LieTensor, Parameter, SO3, so3, SE3, se3, Sim3, sim3, RxSO3, rxso3
from .lietensor import randn_like, randn_SE3, randn_SO3, randn_so3, randn_se3
from .lietensor import randn_Sim3, randn_sim3, randn_RxSO3, randn_rxso3
from .lietensor import identity_like, identity_SO3, identity_so3, identity_SE3, identity_se3
from .lietensor import identity_Sim3, identity_sim3, identity_RxSO3, identity_rxso3
from .lietensor import add, add_, mul, Exp, Log, Inv, Mul, Retr, Act, Adj, AdjT, Jinvp, Jr
from .lietensor import SO3_type, so3_type, SE3_type, se3_type
from .lietensor import Sim3_type, sim3_type, RxSO3_type, rxso3_type
from .lietensor import tensor, translation, rotation, scale, matrix, euler, vec2skew, quat2unit
from .lietensor import mat2SO3, mat2SE3, mat2Sim3, mat2RxSO3, from_matrix, euler2SO3
from .lietensor.lietensor import retain_ltype
from . import func
from .function import *
from .basics import *
from . import autograd
from . import module
from .module.loss import geodesic_loss
from . import optim
from . import testing
from . import utils
from . import metric
from . import sparse
from .sparse import bsr_bsc_matmul
