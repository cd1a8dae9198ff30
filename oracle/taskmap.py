"""ORACLE (test infrastructure): ctypes front-end of oracle/taskmap.c and oracle/_ref."""
import ctypes
import subprocess
from pathlib import Path

import numpy as np

_DIR = Path(__file__).resolve().parent
_ARGS = [ctypes.c_void_p] + [ctypes.c_int] * 7


def _build():
    so = _DIR / "_build" / "liboracle.so"
    if not so.exists() or so.stat().st_mtime < (_DIR / "taskmap.c").stat().st_mtime:
        subprocess.run(["make", "-C", str(_DIR), "_build/liboracle.so"], check=True,
                       capture_output=True)
    return so


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(str(_build()))
        _lib.oracle_taskmap_bytes.restype = ctypes.c_int64
        _lib.oracle_taskmap_bytes.argtypes = _ARGS
        _lib.oracle_assign_attention_decode_task.restype = ctypes.c_int
        _lib.oracle_assign_attention_decode_task.argtypes = _ARGS + [ctypes.c_void_p, ctypes.c_int64]
    return _lib


def ref_lib():
    """The real reference scheduler compiled from /root/reference, or None if not built."""
    global _ref
    if _ref is None:
        so = _DIR / "_ref" / "libref_taskmap.so"
        if not so.exists():
            return None
        try:
            _ref = ctypes.CDLL(str(so))
        except OSError:
            return None
        _ref.ref_assign_attention_decode_task.restype = ctypes.c_int64
        _ref.ref_assign_attention_decode_task.argtypes = _ARGS + [ctypes.c_void_p, ctypes.c_int64]
    return _ref


def _prep(lens):
    lens = np.ascontiguousarray(np.asarray(lens, dtype=np.int32))
    return lens, lens.ctypes.data_as(ctypes.c_void_p)


def assign(lens, num_total_ctas, num_head_kv, num_seq_q, tilen, new_kv_included, min_process_len):
    """Packed host task map (int32 [rows, 12]) from the C restatement."""
    lens, p = _prep(lens)
    a = (p, num_total_ctas, len(lens), num_head_kv, num_seq_q, tilen, int(new_kv_included),
         min_process_len)
    nbytes = lib().oracle_taskmap_bytes(*a)
    out = np.zeros(nbytes // 4, dtype=np.int32)
    rc = lib().oracle_assign_attention_decode_task(*a, out.ctypes.data_as(ctypes.c_void_p), nbytes)
    assert rc == 0
    return out.reshape(-1, 12)


def assign_ref(lens, num_total_ctas, num_head_kv, num_seq_q, tilen, new_kv_included,
               min_process_len):
    """Same, from the real reference code (oracle/_ref). Returns None when unavailable."""
    r = ref_lib()
    if r is None:
        return None
    lens, p = _prep(lens)
    a = (p, num_total_ctas, len(lens), num_head_kv, num_seq_q, tilen, int(new_kv_included),
         min_process_len)
    nbytes = r.ref_assign_attention_decode_task(*a, None, 0)
    out = np.zeros(nbytes // 4, dtype=np.int32)
    r.ref_assign_attention_decode_task(*a, out.ctypes.data_as(ctypes.c_void_p), nbytes)
    return out.reshape(-1, 12)


def pair_chunks(lens, num_total_ctas, num_head_kv, num_seq_q, min_process_len,
                new_kv_included=True):
    """Split-k chunks of every (request, kv head) pair of the decode schedule: {(b, h): [(first
    key, keys), ...]} in chunk order. lens as the decode call receives them."""
    tm = assign(lens, num_total_ctas, num_head_kv, num_seq_q, 128, new_kv_included,
                min_process_len)
    rows = tm[1:1 + int(tm[0, 0]) * int(tm[0, 1])]
    out = {}
    for h, b, c, st, n in rows[:, :5].tolist():
        if h >= 0 and b >= 0:
            out.setdefault((b, h), []).append((c, st, n))
    return {k: [(st, n) for _, st, n in sorted(v)] for k, v in out.items()}
