"""bio_ik_b200 — H100-native bio2 / bio2_memetic population loop of TAMS-Group/bio_ik.

Host-side mirror of the reference interface (Goal classes, Problem, IKSolver) over
the C ABI of libbioik_b200.so (include/bioik_b200.h).  All compute runs in
hand-written sm_90a CUDA kernels; there is no CPU fallback.
"""
from . import _abi, goals, model, problem, robots  # noqa: F401
from .goals import *  # noqa: F401,F403
from .model import JointModelGroup, Link, RobotModel  # noqa: F401
from .problem import Problem  # noqa: F401
