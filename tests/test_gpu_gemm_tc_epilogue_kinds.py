"""Every epilogue instance of the tensor-core GEMM: activation (none / ReLU / tanh) x output kind (fp32, split fp16,
both) for both tile widths, against an fp64 matmul.  The activation and the output kind are template parameters of
cn_gemm_tc_kernel and gemm_tc picks the instance, so each pair is its own kernel; the rollout launches only some of
them, the rest are reached through cn_internal_gemm_tc_ex."""
import pytest

from tests.test_gpu_gemm_tc import _check_epilogue_instance

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("out", ["f32", "f16", "both"])
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("bn", [64, 256])
def test_gemm_tc_epilogue_instance(bn, act, out):
    """Rows of a partial last tile (M = 300), a window that cuts through a tile (_check_epilogue_instance)."""
    _check_epilogue_instance(300, 2 * bn, 128, act, bn, out, 7 * bn + 3 * act + len(out))
