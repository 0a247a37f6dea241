"""fplll_b200 — GPU-native (H100) fp64 Gram-Schmidt / LLL inner loop and BKZ enumeration behind fplll's API.

Host-side mirror of the reference classes (same method names, argument meaning and error behaviour):
  MatGSO          <- fplll/gso.h:33 MatGSO<Z_NR<long>, FP_NR<double>>
  lll_reduction   <- fplll/wrapper.h:136 (the <long,double> stage)
All compute happens in hand-written sm_90a kernels behind the C-ABI of include/*.h.
"""
from ._lib import B200Error  # noqa: F401
from .gso import MatGSO, lll_reduction, GSO_DEFAULT, GSO_ROW_EXPO, GSO_OP_FORCE_LONG, GSO_TRANSFORM  # noqa: F401
from .gso import OP_ROW_ADDMUL, OP_MOVE_ROW, OP_ROW_SWAP, OP_ROW_OP_END, OP_NEGATE  # noqa: F401
from .gso import RED_SUCCESS, RED_GSO_FAILURE, RED_BABAI_FAILURE, RED_LLL_FAILURE  # noqa: F401
from .bkz import BKZParam, bkz_reduction, load_strategies  # noqa: F401
from .bkz import BKZ_DEFAULT, BKZ_VERBOSE, BKZ_NO_LLL, BKZ_MAX_LOOPS, BKZ_AUTO_ABORT, BKZ_GH_BND, BKZ_SHRINK_RADIUS  # noqa: F401
from .bkz import BKZ_MAX_TIME, BKZ_BOUNDED_LLL, BKZ_SD_VARIANT, BKZ_SLD_RED  # noqa: F401
from .householder import MatHouseholder, hlll_reduction  # noqa: F401
from .enumeration import enumerate_svp  # noqa: F401
from .io import read_matrix, write_matrix, load_strategies_json, GSODump  # noqa: F401
