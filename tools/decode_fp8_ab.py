"""A/B of two builds of the library on the FP8 decode path: same outputs bit for bit, and timings.

    python tools/decode_fp8_ab.py --base build/baseline/_C.so [--new hpc-ops_b200/hpc/_C.so]
                                  [--reps 5] [--steps 1000] [--parts outputs,bench,sweep] [--out DIR]

Each library gets its own copy of the tree (in a temporary directory) with that library as
hpc/_C.so; everything that compares outputs runs there in a subprocess of its own:
  * outputs: hpc.attention_decode_fp8 over rows 4..32 (MTP 1-4 at group 4 and 8), both quant types,
    NHD and HND caches (NHD at rows <= 16 takes the rotated walk); np.array_equal
  * C2: `bench.py --no-extra` alternated between the builds `--reps` times each (step time, kernel
    time, tokens/s); the first run of each also dumps its output, compared bit for bit
  * sweep: kernel time of hpc_attention_decode_fp8_partial_async at C2 (B 64, Hq 32, Hkv 8, 8192
    tokens each) on NHD and HND caches, both libraries loaded side by side in one process,
    alternated. With `--parts sweep --base hpc-ops_b200/hpc/_C.so` both arms are the current
    build: its NHD and HND kernel times.
One JSON document goes to stdout and to DIR/decode_fp8_ab_<parts>.json.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
from pathlib import Path

from timing import card, time_eager

REPO = Path(__file__).resolve().parents[1]
PKG = REPO / "hpc-ops_b200"

# (num_head_q, num_head_kv, num_seq_q): rows = group * num_seq_q = 4, 8, 12, 16, 24, 32
SHAPES = [(32, 8, 1), (32, 8, 2), (32, 8, 3), (64, 8, 2), (64, 8, 3), (64, 8, 4)]


def worker(out_dir: Path):
    """Runs inside one arm's tree: writes every case's output as float32 .npy."""
    sys.path.insert(0, str(REPO))
    sys.path.insert(0, str(PKG))
    import numpy as np
    import torch

    import hpc
    from synth.decode import make_decode_fp8_inputs, make_decode_fp8_kpt_inputs

    out_dir.mkdir(parents=True, exist_ok=True)
    B = 8
    lens = [1000 + 397 * i for i in range(B)]
    for quant in (1, 0):
        for layout in ("NHD", "HND"):
            for hq, hkv, sq in SHAPES:
                make = make_decode_fp8_inputs if quant == 1 else make_decode_fp8_kpt_inputs
                d = make(B, sq, lens, hkv, hq, seed=23, layout=layout, device="cuda")
                kc, vc = (d["kvcache"][:, 0], d["kvcache"][:, 1]) if quant == 1 else (d["kcache"], d["vcache"])
                qt = (hpc.QuantType.QPERTOKEN_PERHEAD_KPERTENSOR_VPERTENSOR if quant == 1 else
                      hpc.QuantType.QPERTOKEN_PERHEAD_KPERTOKEN_PERHEAD_VPERHEAD)
                tm = hpc.get_attention_decode_task_workspace(B, max(lens), hkv, 256)
                hpc.assign_attention_decode_task(d["kv_lens_total"], tm, hkv, sq, True, 256)
                y = hpc.attention_decode_fp8(d["q"], kc, vc, d["block_ids"], d["kv_lens_total"],
                                             d["q_scale"], d["k_scale"], d["v_scale"], mtp=sq - 1,
                                             new_kv_included=True, quant_type=qt, task_map=tm)
                torch.cuda.synchronize()
                np.save(out_dir / f"q{quant}_{layout}_r{hq // hkv * sq}.npy", y.float().cpu().numpy())
                del d


def make_arm(tmp: Path, name: str, so: Path) -> Path:
    dst = tmp / name
    shutil.copytree(REPO, dst, symlinks=True,
                    ignore=shutil.ignore_patterns(".git", "build", "__pycache__",
                                                  "bench_outputs", "*.o", "_C*.so"))
    shutil.copy2(so, dst / "hpc-ops_b200" / "hpc" / "_C.so")
    return dst


def last_json(text: str):
    for line in reversed(text.strip().splitlines()):
        if line.startswith("{"):
            return json.loads(line)
    raise RuntimeError("no JSON line in:\n" + text[-2000:])


def compare_dirs(a: Path, b: Path):
    import numpy as np

    res = {}
    for f in sorted(a.glob("*.npy")):
        x, y = np.load(f), np.load(b / f.name)
        res[f.stem] = bool(x.shape == y.shape and np.array_equal(x, y))
    return res


def sweep(base_so: Path, iters: int, reps: int):
    """Kernel time at C2 on NHD and HND caches, both libraries in this process, alternated."""
    import ctypes

    sys.path.insert(0, str(REPO))
    sys.path.insert(0, str(PKG))
    import torch

    import hpc
    from hpc import _ffi
    from hpc import attention as hatt
    from synth import decode as sd

    base = _ffi.bind(ctypes.CDLL(str(base_so)))
    fns = {"base": base.hpc_attention_decode_fp8_partial_async,
           "new": _ffi.lib.hpc_attention_decode_fp8_partial_async}
    B, Sq, Hkv, Hq, S, MPL = 64, 1, 8, 32, 8192, 64

    rows = []
    for layout in ("NHD", "HND"):
        d = sd.make_decode_fp8_inputs(B, Sq, [S] * B, Hkv, Hq, seed=41, layout=layout, device="cuda")
        kc, vc = d["kvcache"][:, 0], d["kvcache"][:, 1]
        tm = hpc.get_attention_decode_task_workspace(B, S, Hkv, MPL)
        hpc.assign_attention_decode_task(d["kv_lens_total"], tm, Hkv, Sq, True, MPL)
        out = torch.empty((B * Sq, Hq, 128), dtype=torch.bfloat16, device="cuda")
        _, args, keep = hatt._decode_fp8_prepare(d["q"], kc, vc, d["block_ids"], d["kv_lens_total"],
                                                 d["q_scale"], d["k_scale"], d["v_scale"], Sq - 1,
                                                 True, 1, True, tm, None, out)
        for fn in fns.values():
            _ffi.check(fn(*args))
        t = {k: [] for k in fns}
        for _ in range(reps):
            for k, fn in fns.items():
                t[k].append(time_eager(lambda: fn(*args), iters, warm=5))
        r = {"layout": layout}
        for k, v in t.items():
            r[k + "_ms"] = statistics.median(v)
            r[k + "_spread"] = [min(v), max(v)]
        r["new_over_base"] = r["new_ms"] / r["base_ms"]
        rows.append(r)
        print(json.dumps(r), file=sys.stderr)
        del d, keep
        torch.cuda.empty_cache()
    return rows


def summarize(runs):
    keys = {"ms_per_step": lambda j: j["ms_per_step"], "kernel_ms": lambda j: j["roofline"]["kernel_ms"],
            "value": lambda j: j["value"], "roofline_frac": lambda j: j["roofline"]["frac"]}
    return {k: {"median": statistics.median([f(j) for j in runs]), "min": min(f(j) for j in runs),
                "max": max(f(j) for j in runs)} for k, f in keys.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worker", metavar="DIR", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--base", default=str(REPO / "build" / "baseline" / "_C.so"))
    ap.add_argument("--new", default=str(PKG / "hpc" / "_C.so"))
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--sweep-iters", type=int, default=200)
    ap.add_argument("--parts", default="outputs,bench,sweep")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    parts = set(a.parts.split(","))
    if a.worker:
        worker(Path(a.worker))
        return

    res = {"card": card()}
    with tempfile.TemporaryDirectory() as td:
        tmp = Path(td)
        arms = {"base": make_arm(tmp, "base", Path(a.base)), "new": make_arm(tmp, "new", Path(a.new))}
        env = dict(os.environ, PYTHONDONTWRITEBYTECODE="1")
        for name, tree in (arms.items() if "outputs" in parts else ()):
            r = subprocess.run([sys.executable, str(tree / "tools" / "decode_fp8_ab.py"), "--worker",
                                str(tmp / f"out_{name}")], cwd=tree, env=env, capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError(f"{name} worker failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
        if "outputs" in parts:
            eq = compare_dirs(tmp / "out_base", tmp / "out_new")
            res["outputs_equal"] = bool(eq) and all(eq.values())
            res["outputs"] = eq

        runs = {"base": [], "new": []}
        for i in range(a.reps if "bench" in parts else 0):
            for name, tree in arms.items():
                cmd = [sys.executable, "bench.py", "--gpus", "1", "--no-extra", "--steps", str(a.steps),
                       "--warmup", str(a.warmup)]
                if i == 0:
                    cmd += ["--dump-outputs", str(tmp / f"c2_{name}")]
                r = subprocess.run(cmd, cwd=tree, env=env, capture_output=True, text=True)
                if r.returncode != 0:
                    raise RuntimeError(f"{name} bench failed:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}")
                j = last_json(r.stdout)
                runs[name].append(j)
                print(json.dumps({"arm": name, "ms_per_step": j["ms_per_step"],
                                  "kernel_ms": j["roofline"]["kernel_ms"], "value": j["value"],
                                  "clocks": j.get("clocks")}), file=sys.stderr)
        if "bench" in parts:
            res["c2_output_equal"] = compare_dirs(tmp / "c2_base", tmp / "c2_new")
            res["c2"] = {k: summarize(v) for k, v in runs.items()}
            res["c2_runs"] = {k: [{"ms_per_step": j["ms_per_step"], "kernel_ms": j["roofline"]["kernel_ms"],
                                   "value": j["value"], "clocks": j.get("clocks")} for j in v]
                              for k, v in runs.items()}
    if "sweep" in parts:
        res["sweep"] = sweep(Path(a.base), a.sweep_iters, 3)
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        Path(a.out).mkdir(parents=True, exist_ok=True)
        (Path(a.out) / f"decode_fp8_ab_{'_'.join(sorted(parts))}.json").write_text(text)


if __name__ == "__main__":
    main()
