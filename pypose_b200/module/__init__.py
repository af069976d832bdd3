from .reproj import PoseReproj, TwoPoseReproj
from .pgo import PoseGraph
from .ba import BundleAdjustment, BALBundleAdjustment
from .imu_preintegrator import IMUPreintegrator
from .loss import GeodesicLoss, geodesic_loss
from .pnp import EPnP
from .icp import ICP
from .dynamics import System, LTI, LTV, NLS, toBTN, runsys
from .lqr import LQR
from .mpc import MPC
