"""Drop-in shim: scripts written for Refefer/Dampr (`from dampr import Dampr, setup_logging`,
`from dampr.inputs import ...`, `from dampr.utils import filter_by_count`) run unmodified on the
device engine. Everything lives in dampr_b200."""
from dampr_b200 import *  # noqa: F401,F403
from dampr_b200 import settings, setup_logging, Dampr, PMap, PReduce, PJoin, ARReduce, BlockMapper, BlockReducer, Dataset  # noqa: F401
