"""The TMA-store epilogue of the BN = 256 tensor-core GEMM instances (cn_gemm_tc.cuh, tc_epilogue_tma).

Each consumer warp group stages its output in a few shared-memory boxes that TMA stores; a box is rewritten only after
TMA has read it.  At M = 300 (test_gpu_gemm_tc_epilogue_kinds.py) every CTA runs one tile; here the row count gives
every CTA three or more tiles, so the staging buffers are reused across tiles, for all nine activation x output-kind
instances.  An output TMA cannot store (unaligned base or row pitch) is refused before anything is launched."""
import pytest
import torch

from tests.test_gpu_gemm_tc import _check_epilogue_instance, _gemm, _lib, _operands

pytestmark = pytest.mark.gpu


def _rows_for_three_tiles_per_cta(N):
    """a row count whose 128 x 256 tiles number at least 3 per SM, the last row tile partial"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    row_tiles = -(-3 * sms // (N // 256))
    return row_tiles * 128 - 37


@pytest.mark.parametrize("out", ["f32", "f16", "both"])
@pytest.mark.parametrize("act", [0, 1, 2])
def test_gemm_tc_bn256_staging_reused_across_tiles(act, out):
    N = 512
    _check_epilogue_instance(_rows_for_three_tiles_per_cta(N), N, 128, act, 256, out, 900 + 3 * act + len(out))


@pytest.mark.parametrize("case", ["f32_base", "f16_base", "f16_pitch"])
def test_gemm_tc_bn256_unaligned_output_refused(case):
    """fp32 output 4 bytes off a 16-byte boundary, split output 2 bytes off, split output with a row pitch of
    (N + 4) fp16 = 520 bytes: an error, and the output buffers keep their sentinel (nothing was launched)."""
    lib, _capi = _lib()
    M, N, K = 300, 256, 128
    A, W, b = _operands(M, N, K, 5)
    out, split, ldh = None, None, 0
    if case == "f32_base":
        buf = torch.full((M * N + 4,), float("nan"), device="cuda")
        out = buf[1:1 + M * N].view(M, N)
    else:
        pitch = N + 4 if case == "f16_pitch" else N + 8
        col0 = 0 if case == "f16_pitch" else 1
        hb = torch.full((M, pitch), float("nan"), dtype=torch.float16, device="cuda")
        lb = hb.clone()
        split, ldh = (hb[:, col0:], lb[:, col0:]), pitch
    with pytest.raises(RuntimeError, match="16-byte"):
        _gemm(A, W, b, M, N, K, 0, 256, out=out, split=split, ldh=ldh)
    torch.cuda.synchronize()
    if out is not None:
        assert torch.isnan(buf).all()
    else:
        assert torch.isnan(split[0]).all() and torch.isnan(split[1]).all()
