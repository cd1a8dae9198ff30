"""hpc — H100 (sm_90a) build of the HPC-Ops quantized-inference hot path.

Same Python-over-torch API as the reference package: every public function of the in-scope modules
is re-exported at package level and the same operators are reachable as `torch.ops.hpc.*`
(reference hpc/__init__.py does the same for its modules). Underneath is a torch-free C-ABI library
(`_C.so`, see include/hpc_b200.h) of hand-written sm_90a kernels, bound with ctypes.
"""
import importlib as _importlib

from . import _ffi  # loads _C.so; raises if the extension has not been built (no fallback)
from . import _ops as _ops_mod

# in-scope modules of the reference package, in import order
_MODULES = ("attention", "group_gemm", "fuse_moe", "act", "gemm", "multicast_handle", "communicator",
            "allreduce", "rope", "sampler", "stem", "normalization")

__all__ = []
for _name in _MODULES:
    _mod = _importlib.import_module(f"{__name__}.{_name}")
    for _attr, _obj in vars(_mod).items():
        if _attr.startswith("_") or not callable(_obj):
            continue
        if getattr(_obj, "__module__", _mod.__name__) != _mod.__name__:
            continue  # re-export what the module defines, not what it imports (Tensor, Optional, ...)
        globals()[_attr] = _obj
        __all__.append(_attr)

__version__ = _ffi.lib.hpc_version().decode()
__built_json__ = _ffi.lib.hpc_built_json().decode()

# torch.ops.hpc.version() / built_json(), as registered by reference src/C/version.cc:14
_ops_mod.define("version() -> str")
_ops_mod.impl("version", lambda: __version__, "CompositeExplicitAutograd")
_ops_mod.define("built_json() -> str")
_ops_mod.impl("built_json", lambda: __built_json__, "CompositeExplicitAutograd")
