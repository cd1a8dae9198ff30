"""Bound probe of the FP8 decode kernel at C2: is it limited by the loads or by the warpgroup?

    python tools/decode_fp8_probe.py --build-only            # compile the two probe libraries
    python tools/decode_fp8_probe.py [--reps 5] [--iters 300] # time them next to hpc/_C.so (GPU)
    python tools/decode_fp8_probe.py --no-build --out DIR --normal LIB  # probes built earlier,
                                                                        # next to another build

csrc/decode_attn_fp8.cu is compiled a second time with HPC_DECODE_FP8_PROBE set (the library build
never sets it), each variant into its own shared library under build/probe/:
  producer  the warpgroup waits for each K/V stage and frees it at once, without any math: the time
            the TMA stream alone takes, i.e. the ceiling of this access pattern on the card
  consumer  the producer signals each stage without loading it (the ring is zeroed once): the time
            the warpgroup's per-tile path alone takes
Each is timed like `tools/decode_fp8_ab.py --parts sweep` times
hpc_attention_decode_fp8_partial_async (CUDA events over back-to-back launches), alternating with
the normal kernel of hpc/_C.so; medians are printed as one JSON line with the card they were
measured on. The kernel is HBM-bound when consumer < normal and normal is close to producer.
"""
import argparse
import ctypes
import json
import shutil
import statistics
import subprocess
import sys
from pathlib import Path

REPO = Path(__file__).resolve().parents[1]
PKG = REPO / "hpc-ops_b200"
VARIANTS = {"producer": 1, "consumer": 2}


def build(csrc: Path, out: Path, force: bool = False):
    sys.path.insert(0, str(PKG))
    import build as libbuild  # hpc-ops_b200/build.py: the product's nvcc flags

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    out.mkdir(parents=True, exist_ok=True)
    deps = [csrc / "decode_attn_fp8.cu", *csrc.glob("*.cuh"), *csrc.glob("*.h")]
    newest = max(p.stat().st_mtime for p in deps)
    host = out / "host_utils.o"
    if force or not host.exists() or host.stat().st_mtime < newest:
        subprocess.run([nvcc, *libbuild.NVCC_FLAGS, "-c", str(csrc / "host_utils.cu"), "-o", str(host)],
                       check=True)
    libs = {}
    for name, val in VARIANTS.items():
        so = out / f"decode_fp8_{name}.so"
        if force or not so.exists() or so.stat().st_mtime < newest:
            obj = out / f"decode_fp8_{name}.o"
            subprocess.run([nvcc, *libbuild.NVCC_FLAGS, f"-DHPC_DECODE_FP8_PROBE={val}", "-c",
                            str(csrc / "decode_attn_fp8.cu"), "-o", str(obj)], check=True)
            subprocess.run([nvcc, "-shared", "-o", str(so), str(obj), str(host), "-gencode",
                            "arch=compute_90a,code=sm_90a", "-lcudart"], check=True)
        libs[name] = so
    return libs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--csrc", default=str(PKG / "csrc"), help="sources to build the probes from")
    ap.add_argument("--out", default=str(REPO / "build" / "probe"))
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--no-build", action="store_true", help="time the libraries already in --out")
    ap.add_argument("--normal", default=None, help="library of the normal kernel (default hpc/_C.so)")
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=300)
    a = ap.parse_args()
    if a.no_build:
        libs = {k: Path(a.out) / f"decode_fp8_{k}.so" for k in VARIANTS}
    else:
        libs = build(Path(a.csrc), Path(a.out), a.force)
    if a.build_only:
        print(json.dumps({k: str(v) for k, v in libs.items()}))
        return

    sys.path.insert(0, str(REPO))
    sys.path.insert(0, str(PKG))
    import torch

    import hpc
    from hpc import _ffi
    from hpc import attention as hatt
    from synth.decode import make_decode_fp8_inputs
    from timing import card, time_eager

    B, Sq, Hkv, Hq, S, MPL = 64, 1, 8, 32, 8192, 64  # C2
    d = make_decode_fp8_inputs(B, Sq, [S] * B, Hkv, Hq, seed=41, device="cuda")
    kc, vc = d["kvcache"][:, 0], d["kvcache"][:, 1]
    tm = hpc.get_attention_decode_task_workspace(B, S, Hkv, MPL)
    hpc.assign_attention_decode_task(d["kv_lens_total"], tm, Hkv, Sq, True, MPL)
    out = torch.empty((B * Sq, Hq, 128), dtype=torch.bfloat16, device="cuda")
    _, args, keep = hatt._decode_fp8_prepare(d["q"], kc, vc, d["block_ids"], d["kv_lens_total"],
                                             d["q_scale"], d["k_scale"], d["v_scale"], Sq - 1, True,
                                             1, True, tm, None, out)
    fns = {"normal": _ffi.lib.hpc_attention_decode_fp8_partial_async}
    if a.normal:
        libs = {"normal": Path(a.normal), **libs}
    for name, so in libs.items():
        fns[name] = _ffi.bind(ctypes.CDLL(str(so))).hpc_attention_decode_fp8_partial_async
    for fn in fns.values():
        _ffi.check(fn(*args))
    runs = {k: [] for k in fns}
    for _ in range(a.reps):
        for k, fn in fns.items():
            runs[k].append(time_eager(lambda: fn(*args), a.iters, warm=10))
    alg = B * Hkv * S * 2 * 128  # K and V bytes of the step
    res = {"card": card(), "shape": "C2", "iters": a.iters}
    for k, v in runs.items():
        med = statistics.median(v)
        res[k] = {"ms_median": med, "ms_min": min(v), "ms_max": max(v), "tb_s": alg / med / 1e9}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
