"""dampr_b200 — H100-native map / shuffle / reduce engine behind the Dampr DSL.

Same public names as the reference package (dampr/__init__.py:14-33) so that
``from dampr_b200 import Dampr`` (or the ``dampr`` shim package) is a drop-in for
``from dampr import Dampr``.
"""
import logging

from . import settings
from .dsl import Dampr, PMap, PReduce, PJoin, ARReduce, ValueEmitter
from .operators import BlockMapper, BlockReducer
from .datasets import Dataset, Chunker

__all__ = ["Dampr", "PMap", "PReduce", "PJoin", "ARReduce", "BlockMapper", "BlockReducer", "Dataset",
           "Chunker", "settings", "setup_logging"]


def setup_logging(debug=False):
    """Convenience function for enabling logging (dampr/__init__.py:27-33)."""
    logging.basicConfig(level=logging.DEBUG if debug else logging.INFO,
                        format="%(asctime)s %(levelname)s %(message)s")
