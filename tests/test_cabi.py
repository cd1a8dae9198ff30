"""The C-ABI library loads and exports every symbol include/hpc_b200.h declares, and `hpc._ffi`
binds each one from the header with the right ctypes types (no GPU needed)."""
import ctypes
import re
from pathlib import Path

import pytest

REPO = Path(__file__).resolve().parents[1]


def declared_symbols():
    text = (REPO / "include" / "hpc_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(hpc_[a-z0-9_]+)\s*\(", text)))


def test_header_declares_entry_points():
    syms = declared_symbols()
    for must in ("hpc_attention_decode_fp8_async", "hpc_assign_attention_decode_task_sync",
                 "hpc_assign_attention_decode_task_async", "hpc_last_error"):
        assert must in syms


def test_library_exports_all_declared(lib_path):
    lib = ctypes.CDLL(str(lib_path))
    missing = [s for s in declared_symbols() if not hasattr(lib, s)]
    assert not missing, f"symbols declared in include/hpc_b200.h but not exported: {missing}"


def test_version_and_error_strings(lib_path, hpc):
    lib = hpc._ffi.bind(ctypes.CDLL(str(lib_path)))
    assert b"b200" in lib.hpc_version()
    assert b"sm_90a" in lib.hpc_built_json()
    assert lib.hpc_last_error() is not None


def test_python_package_imports_and_mirrors_reference_names(hpc):
    for name in ("attention_decode_fp8", "get_attention_decode_task_workspace",
                 "assign_attention_decode_task", "print_attention_decode_task", "QuantType"):
        assert hasattr(hpc, name), name
    assert hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR.value == 1
    import torch

    assert hasattr(torch.ops.hpc, "attention_decode_fp8")
    assert hasattr(torch.ops.hpc, "assign_attention_decode_task")


def test_launcher_rejects_bad_arguments_without_gpu(lib_path, hpc):
    """Argument validation happens before any CUDA call: unsupported shapes fail loudly."""
    lib = hpc._ffi.bind(ctypes.CDLL(str(lib_path)))
    rc = lib.hpc_assign_attention_decode_task_async(None, None, 148, 5000, 8, 1, 128, 1, 64, None)
    assert rc == 1 and b"batch" in lib.hpc_last_error()
    rc = lib.hpc_assign_attention_decode_task_async(None, None, 148, 4, 8, 1, 96, 1, 64, None)
    assert rc == 1 and b"tilen" in lib.hpc_last_error()


def test_every_declared_function_binds_from_the_header(lib_path, hpc):
    """Each prototype in include/hpc_b200.h parses, and each exported one gets one argtype per
    declared parameter."""
    protos = hpc._ffi.prototypes((REPO / "include" / "hpc_b200.h").read_text())
    assert sorted(protos) == declared_symbols()
    lib = hpc._ffi.bind(ctypes.CDLL(str(lib_path)))
    for name, (restype, argtypes) in protos.items():
        fn = getattr(lib, name)
        assert fn.restype is restype and fn.argtypes == argtypes, name
    assert len(lib.hpc_attention_decode_fp8_async.argtypes) == 38
    assert lib.hpc_last_error.argtypes == [] and lib.hpc_last_error.restype is ctypes.c_char_p


SYNTHETIC_HEADER = """
/* a comment with hpc_commented(int x); inside */
int64_t hpc_sizes(const int* lens, int n,   // trailing comment
                  int64_t stride, uint64_t seed, float scale, double eps,
                  void** table, cudaStream_t stream);
const char* hpc_name(void);
int hpc_missing(int x);
"""


def test_header_types_map_to_ctypes(hpc):
    c = ctypes
    protos = hpc._ffi.prototypes(SYNTHETIC_HEADER)
    assert protos == {
        "hpc_sizes": (c.c_int64, [c.c_void_p, c.c_int, c.c_int64, c.c_uint64, c.c_float,
                                  c.c_double, c.c_void_p, c.c_void_p]),
        "hpc_name": (c.c_char_p, []),
        "hpc_missing": (c.c_int, [c.c_int]),
    }

    class FakeLib:  # exports hpc_sizes and hpc_name only, like a library built before hpc_missing
        hpc_sizes = type("Fn", (), {})()
        hpc_name = type("Fn", (), {})()

    lib = hpc._ffi.bind(FakeLib(), SYNTHETIC_HEADER)
    assert lib.hpc_sizes.argtypes == protos["hpc_sizes"][1]
    assert lib.hpc_name.restype is c.c_char_p and lib.hpc_name.argtypes == []
    assert not hasattr(lib, "hpc_missing")


@pytest.mark.parametrize("decl", ["int hpc_bad(void* p, size_t n);", "int hpc_bad(unsigned n);",
                                  "void hpc_bad(int n);", "int hpc_bad(int n[4]);"])
def test_unknown_header_type_fails_import(hpc, decl):
    with pytest.raises(ImportError, match="hpc_bad"):
        hpc._ffi.prototypes(SYNTHETIC_HEADER + decl)
