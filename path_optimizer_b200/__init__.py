"""path_optimizer_b200: H100-native batched path-QP solver behind the OsqpSolver boundary of
LiJiangnanBit/path_optimizer.  See DESIGN.md / INTEGRATION.md."""
from .abi import BOUNDS_DTYPE, FORMULATIONS, STATE_DTYPE, Params, Stats  # noqa: F401
