"""Every epilogue instance of the tensor-core GEMM: activation (none / ReLU / tanh) x output kind (fp32, split fp16,
both) for both tile widths, against an fp64 matmul.  The activation and the output kind are template parameters of
cn_gemm_tc_kernel and gemm_tc picks the instance, so each pair is its own kernel; the rollout launches only some of
them, the rest are reached through cn_internal_gemm_tc_ex."""
import pytest
import torch

from tests.test_gpu_gemm_tc import C_GEMM, _c, _gemm, _operands, _ref, _split_ok

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("out", ["f32", "f16", "both"])
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("bn", [64, 256])
def test_gemm_tc_epilogue_instance(bn, act, out):
    """Rows of a partial last tile, a window that cuts through a tile: fp32 within the componentwise bound, and the
    split output exactly the (hi, lo) split of what the fp32 output holds."""
    M, N, K = 300, 2 * bn, 128
    act_lo, act_hi = 40, N - 24
    A, W, b = _operands(M, N, K, 7 * bn + 3 * act + len(out))
    Cout = torch.full((M, N), float("nan"), device="cuda") if out != "f16" else None
    hi = torch.zeros((M, N), dtype=torch.float16, device="cuda") if out != "f32" else None
    lo = torch.zeros_like(hi) if hi is not None else None
    _gemm(A, W, b, M, N, K, act, bn, out=Cout, split=(hi, lo) if hi is not None else None, ldh=N if hi is not None else 0,
          act_lo=act_lo, act_hi=act_hi)
    ref, scale, win = _ref(A, W, b, act, act_lo, act_hi)
    if Cout is not None:
        c = _c(Cout, ref, scale, act, win)
        assert c <= C_GEMM, c
        if hi is not None:
            assert _split_ok(hi, lo, Cout)
    else:
        s = hi.double() + lo.double()
        floor = 2.0 ** -22 * ref.abs() + 2.0 ** -25 + (1e-6 * win.double() if act == 2 else 0.0)
        excess = ((s - ref).abs() - floor).clamp_min(0)
        assert float((excess / scale.clamp_min(1e-300)).max()) <= C_GEMM
