"""poseidon_b200 — a Blackwell-native distributed CNN training engine with the capabilities
of petuum/poseidon (PMLS-Caffe): Caffe prototxt / caffemodel / solverstate compatible,
distributed wait-free backprop + sufficient-factor broadcasting re-imagined as fused
sm_90a CUDA kernels over NVLink / NVSwitch.  See SURVEY.md / DESIGN.md.
"""
__version__ = "0.1.0"

from . import proto  # noqa: F401
from .layers import NetContext  # noqa: F401
from .net.net import Net  # noqa: F401
from .parallel.context import RankContext, init_rank_context  # noqa: F401
from .solver.solver import (AdaGradSolver, NesterovSolver, SGDSolver, Solver,  # noqa: F401
                            get_solver)
from .engine import CaffeEngine  # noqa: F401,E402
