"""openrec.tf2.recommenders surface (reference: openrec/tf2/recommenders/__init__.py:1-5)."""
from .bpr import BPR
from .wrmf import WRMF
from .gmf import GMF
from .ucml import UCML
from .retriever import Retriever

__all__ = ["BPR", "WRMF", "GMF", "UCML", "Retriever"]
try:  # DLRM needs the MLP / interaction kernels
    from .dlrm import DLRM  # noqa: F401
    __all__.append("DLRM")
except ImportError:  # pragma: no cover
    pass


def __getattr__(name):   # row-sharded BPR / UCML / GMF / WRMF / DLRM (torch.distributed): imported on demand
    if name in ("ShardedBPR", "ShardedUCML"):
        from . import sharded
        return getattr(sharded, name)
    if name in ("ShardedGMF", "ShardedWRMF"):
        from . import sharded_pointwise
        return getattr(sharded_pointwise, name)
    if name == "ShardedDLRM":
        from .sharded_dlrm import ShardedDLRM
        return ShardedDLRM
    raise AttributeError(name)
