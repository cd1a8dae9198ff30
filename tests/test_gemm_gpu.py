"""GPU parity tests of the BF16 x FP32 route GEMM at the reference's tolerances (grid of reference
tests/test_gemm_bf16xfp32.py:14-45). The per-element fp64 checks at every split are in
tests/test_gemm_exact_gpu.py."""
import pytest
import torch

from oracle import gemm as og

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m", [1, 6, 16, 64, 144, 416, 1024, 4096, 12303])
@pytest.mark.parametrize("n", [192, 512, 1024, 2048])
@pytest.mark.parametrize("use_fp32_output", [True, False])
@pytest.mark.parametrize("use_split_flag", [True, False])
def test_gemm_bf16xfp32(hpc, m, n, use_fp32_output, use_split_flag):
    k = 4096
    x, w, w_high, w_low, scale = og.make_inputs(m, n, k, device="cuda")
    split_flag = hpc.get_gemm_bf16xfp32_workspace(n) if use_split_flag else None
    my = hpc.gemm_bf16xfp32(x, w_high, w_low, scale, use_fp32_output, True, split_flag)
    if use_split_flag:
        assert (split_flag == 0).all()
    gt = og.gemm_fp32(x, w)
    assert my.dtype == (torch.float32 if use_fp32_output else torch.bfloat16)
    assert torch.allclose(gt, my.float(), rtol=0.08, atol=0.01), (gt - my.float()).abs().max()
    if use_fp32_output:
        exact = og.gemm_split_exact(x, w_high, w_low, scale)
        rel = (my.double() - exact).norm() / exact.norm()
        assert rel < 1e-5, rel


@pytest.mark.parametrize("m,n,k", [(37, 64, 512), (300, 320, 1000 // 8 * 8), (129, 384, 4096)])
def test_gemm_bf16xfp32_odd_shapes_no_splitk(hpc, m, n, k):
    x, w, w_high, w_low, scale = og.make_inputs(m, n, k, device="cuda")
    for splitk in (False, True):
        my = hpc.gemm_bf16xfp32(x, w_high, w_low, scale, True, splitk)
        exact = og.gemm_split_exact(x, w_high, w_low, scale)
        rel = (my.double() - exact).norm() / exact.norm()
        assert rel < 1e-5, (m, n, k, splitk, rel)


def test_gemm_rejects_bad_shapes(hpc):
    x, w, w_high, w_low, scale = og.make_inputs(8, 64, 64, device="cuda")
    with pytest.raises(RuntimeError):
        hpc.gemm_bf16xfp32(x, w_high[:40], w_low[:40], scale)
    with pytest.raises(RuntimeError):
        hpc.gemm_bf16xfp32(x.float(), w_high, w_low, scale)
