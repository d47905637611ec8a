"""oktopk_b200 -- Hopper-native (H100) sparse-gradient allreduce training library.

Public API (parity with the reference's ``distributed_optimizer`` / ``compression`` /
``allreducer`` modules, SURVEY A.3)::

    import oktopk_b200 as okt
    okt.init()                                             # torchrun env -> process group
    opt = okt.DistributedOptimizer(torch.optim.SGD(model.parameters(), lr=0.1, momentum=0.9),
                                   named_parameters=model.named_parameters(),
                                   compression=okt.compressors['oktopk'], is_sparse=True, density=0.001)
    opt.zero_grad(); loss.backward(); opt.step()
"""
from .config import LossScale, OkTopkConfig, preset  # noqa: F401
from .compression import compressors, NoneCompressor, TopKCompressor, GaussianCompressor  # noqa: F401
from .parallel.world import init, world, rank, size, shutdown  # noqa: F401
from .parallel.state import SparseState  # noqa: F401

__version__ = "0.1.0"


def __getattr__(name):
    # heavier modules are imported lazily so that `import oktopk_b200` stays cheap
    if name in ("DistributedOptimizer", "BertAdam", "Lamb", "broadcast_parameters"):
        from . import optimizer as _o
        return getattr(_o, name)
    if name in ("optimizer", "models", "train", "utils", "ops", "parallel", "compression", "config"):
        import importlib
        return importlib.import_module("." + name, __name__)
    if name == "AllReducer":
        from .parallel.allreducer import AllReducer
        return AllReducer
    raise AttributeError(name)
