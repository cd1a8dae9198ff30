"""ctypes binding of the C-ABI library (include/hpc_b200.h).

The library is the product: if `_C.so` is missing or a launcher reports an error this module
raises — there is no CPU or PyTorch fallback anywhere in `hpc`.
"""
import ctypes
import re
from pathlib import Path

import torch

_pkg_dir = Path(__file__).parent

_so_files = list(_pkg_dir.glob("_C*.so"))
if len(_so_files) != 1:
    raise ImportError(
        f"hpc (H100 build): expected exactly one _C*.so next to {__file__}, found "
        f"{len(_so_files)}. Build it with `python hpc-ops_b200/build.py` (needs nvcc, sm_90a)."
    )

_HEADER = Path(__file__).resolve().parents[2] / "include" / "hpc_b200.h"

# The C types include/hpc_b200.h may use. Anything else is an error, not a guess: a ctypes c_int
# slot silently truncates a 64-bit stride or a pointer.
_PARAM_TYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "uint64_t": ctypes.c_uint64,
                "float": ctypes.c_float, "double": ctypes.c_double,
                "cudaStream_t": ctypes.c_void_p}
_RETURN_TYPES = {"int": ctypes.c_int, "int64_t": ctypes.c_int64, "const char*": ctypes.c_char_p}
_PROTOTYPE = re.compile(r"^[ \t]*([A-Za-z_][\w \t*]*?)\s*\b(hpc_\w+)\s*\(([^()]*)\)\s*;", re.M)


def _param_type(fn: str, param: str):
    if "*" in param:
        return ctypes.c_void_p
    m = re.fullmatch(r"(\w+(?: \w+)*) \w+", param)
    typ = m.group(1) if m else param
    if typ not in _PARAM_TYPES:
        raise ImportError(f"hpc_b200.h: {fn} has a parameter of type {typ!r}, which has no ctypes "
                          f"binding (allowed: pointers, {', '.join(_PARAM_TYPES)})")
    return _PARAM_TYPES[typ]


def prototypes(header_text: str) -> dict:
    """{name: (restype, argtypes)} for every `RET hpc_name(PARAMS);` in a C header's text."""
    text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", header_text, flags=re.S)
    protos = {}
    for ret, name, params in _PROTOTYPE.findall(text):
        ret = re.sub(r" ?\*", "*", " ".join(ret.split()))
        if ret not in _RETURN_TYPES:
            raise ImportError(f"hpc_b200.h: {name} returns {ret!r}, which has no ctypes binding "
                              f"(allowed: {', '.join(_RETURN_TYPES)})")
        params = " ".join(params.split())
        argtypes = [] if params == "void" else [_param_type(name, p.strip())
                                                for p in params.split(",")]
        protos[name] = (_RETURN_TYPES[ret], argtypes)
    return protos


def bind(lib, header_text: str | None = None):
    """Set restype and argtypes of every function include/hpc_b200.h (or `header_text`) declares
    and `lib` exports, and return `lib`. A declared function the library lacks (one built from an
    older commit, e.g. for an A/B timing) stays unbound and fails at its first call."""
    if header_text is None:
        header_text = _HEADER.read_text()
    for name, (restype, argtypes) in prototypes(header_text).items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            continue
        fn.restype, fn.argtypes = restype, argtypes
    return lib


lib = bind(ctypes.CDLL(str(_so_files[0])))


def check(rc: int, what: str = ""):
    """Turn a launcher status into the RuntimeError the reference raises via TORCH_CHECK."""
    if rc != 0:
        msg = lib.hpc_last_error().decode("utf-8", "replace")
        raise RuntimeError(f"hpc {what} failed (code {rc}): {msg}")


def require(cond: bool, msg: str):
    """Reject an argument the way a launcher would: RuntimeError, as the reference's TORCH_CHECK."""
    if not cond:
        raise RuntimeError(msg)


def ptr(t):
    """Raw data pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_of(t) -> int:
    """cudaStream_t of torch's current stream on the tensor's device."""
    return torch.cuda.current_stream(t.device).cuda_stream


_sm_count_cache = {}


def sm_count(device=None) -> int:
    dev = torch.cuda.current_device() if device is None else torch.device(device).index
    if dev is None:
        dev = torch.cuda.current_device()
    if dev not in _sm_count_cache:
        _sm_count_cache[dev] = torch.cuda.get_device_properties(dev).multi_processor_count
    return _sm_count_cache[dev]
