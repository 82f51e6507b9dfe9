"""b200ocl -- H100-native replay-step engine behind the plugin surface of
RaptorMai/online-continual-learning (agents/*, utils/buffer/*, utils/name_match.py).

Host side is Python/PyTorch (device memory, streams, torch.distributed); all
arithmetic on the path runs in hand-written sm_90a CUDA behind the C ABI declared
in include/b200ocl.h (libb200ocl.so, loaded with ctypes).  There is no CPU or
library fallback: every op raises if the CUDA library is missing.
"""
__version__ = '0.1.0'


def install(reference_name_match=None, extra=()):
    """Patch the reference registries in place (see registry.install); `extra` names opt-in agents, e.g. ('EWC',)."""
    from . import registry
    return registry.install(reference_name_match, extra=extra)
