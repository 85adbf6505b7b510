"""horovod_b200 — a Hopper-native (H100) data-parallel collective library with Horovod's capabilities.

`import horovod_b200.torch as hvd` gives the reference's PyTorch API
(horovod/torch/__init__.py): init/rank/size, async named collectives,
DistributedOptimizer, broadcast helpers, process sets, elastic.
"""
__version__ = "0.1.0"


def run(*args, **kwargs):
    """Programmatic launcher, see horovod_b200.runner.run (reference horovod/runner/__init__.py:95)."""
    from horovod_b200.runner import run as _run
    return _run(*args, **kwargs)
