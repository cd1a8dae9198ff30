"""Generate the Stem KV-prep fixtures tests/golden/stem_kvprep_*.npz from the REFERENCE's own code,
the way tests/golden/make_golden.py does for the other ops (and with its helpers).

Run in the build container only (needs /root/reference; the GPU box never runs this):
    python tests/golden/make_golden_stem.py

The reference keeps its KV-prep ground truth as pure-torch functions in its test file
(`_gather_per_token_kscale`, `_kv_prep_reference`); they are AST-extracted and executed unmodified
on CPU. They take a per-token kscale; a per-tensor kscale is passed as that scale at every token
(and vscale[0] for every head), which is what per-tensor scaling means.
"""
import ast
import math
import sys
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
from make_golden import OUT, REF, _bf16_bits, _TorchCPU  # noqa: E402

from synth import stem as ss  # noqa: E402  (make_golden put the repository on sys.path)

SRC = REF / "tests/test_stem_qkpertoken_perhead_vperhead.py"


def _extract():
    src = SRC.read_text()
    ns = {"torch": _TorchCPU(), "math": math, "STEM_BLOCK_SIZE": 128, "STEM_STRIDE": 16,
          "LAMBDA_MAG": 0.3}
    for node in ast.parse(src).body:
        if isinstance(node, ast.FunctionDef) and node.name in ("_gather_per_token_kscale",
                                                               "_kv_prep_reference"):
            exec(compile(ast.get_source_segment(src, node), str(SRC), "exec"), ns)
    return ns["_kv_prep_reference"]


def case(tag, kv_lens, hkv, page, quant, seed):
    fn = _extract()
    d = ss.make_inputs([1] * len(kv_lens), kv_lens, hkv, hkv, page, "nhd", quant, seed=seed)
    nb = d["kcache"].shape[0]
    if quant == 1:
        ks_tok = torch.full((nb, page // 32, hkv, 32), float(d["kscale"][0]))
        vs = torch.full((hkv,), float(d["vscale"][0]))
    else:
        ks_tok, vs = d["kscale"], d["vscale"]
    kflat, vbias = fn(d["kcache"], d["vcache"], ks_tok, vs, d["kv_indices"], d["kv_seq_lens"], page)
    np.savez_compressed(
        OUT / f"stem_kvprep_{tag}.npz", kcache=d["kcache"].view(torch.uint8).numpy(),
        vcache=d["vcache"].view(torch.uint8).numpy(), kscale=d["kscale"].numpy(),
        vscale=d["vscale"].numpy(), kv_indices=d["kv_indices"].numpy(),
        kv_seq_lens=d["kv_seq_lens"].numpy(), kflat=_bf16_bits(kflat), vbias=vbias.numpy(),
        meta=np.array([page, quant]))
    print("wrote stem_kvprep", tag, tuple(kflat.shape))


if __name__ == "__main__":
    case("q0_p32", [300, 515, 77], 2, 32, 0, 61)
    case("q1_p64", [640, 129, 1], 1, 64, 1, 62)
    case("q0_p64", [200, 33], 2, 64, 0, 63)
