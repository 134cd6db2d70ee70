"""GPU test of the wgmma / TMA GEMM (3xFP16 error-compensated) against an fp64 matmul, through the internal hooks
cn_internal_gemm_tc and cn_internal_gemm_tc_ex (the epilogue and operand variants the rollout uses: device-side row
range, column-view A operands, split fp16 outputs at a column offset, activation windows), and of the whole policy
forward in gemm_mode=1.  _check_epilogue_instance is the shared check of the per-instance epilogue tests
(test_gpu_gemm_tc_epilogue_kinds.py, test_gpu_gemm_tc_tma_store.py).

Error bound, per element:  |C - C_fp64| <= C_GEMM * (|A| @ |W|^T + |b|)  (+ C_TANH absolute after a tanh), so small
operands cannot hide an error.  C_GEMM is 3x the worst value measured on an H100 80GB HBM3 (400 W power limit) over
this file (pytest -s prints the measured values)."""
import ctypes as C

import pytest
import torch

from tests.policy_stages import nearest_split

pytestmark = pytest.mark.gpu

C_GEMM = 3e-6           # componentwise bound of the 3xFP16 wgmma GEMM (measured worst 9.9e-7)
C_TANH = 1e-6          # absolute allowance of the tanh epilogue (fast_tanh: ~2e-7)
F16_NAN = 0x7E00


def _lib():
    from crowdnav_prediction_attngraph_b200 import _capi
    lib = _capi.load_library()
    lib.cn_internal_gemm_tc.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int,
                                        C.c_int]
    lib.cn_internal_gemm_tc_ex.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                           C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_int, C.c_int, C.c_int]
    return lib, _capi


def _gemm(A, W, b, M, N, K, act, bn, out=None, m=None, m0=None, a_col0=0, a_pitch=0, split=None, ldh=0, act_lo=0,
          act_hi=0):
    """out: fp32 [M, N] or None; split: (hi, lo) fp16 tensors already offset to the output column; m / m0: ints kept
    on the device (row count / first row)."""
    lib, _capi = _lib()
    dm = torch.tensor([m], dtype=torch.int32, device="cuda") if m is not None else None
    dm0 = torch.tensor([m0], dtype=torch.int32, device="cuda") if m0 is not None else None
    p = lambda t: t.data_ptr() if t is not None else None
    _capi.check(lib, lib.cn_internal_gemm_tc_ex(p(A), p(W), p(b), p(out), M, N, K, act, bn, p(dm), p(dm0), a_col0,
                                                a_pitch, p(split[0]) if split else None, p(split[1]) if split else None,
                                                ldh, act_lo, act_hi), "cn_internal_gemm_tc_ex")
    torch.cuda.synchronize()


def _ref(A, W, b, act, act_lo=0, act_hi=1 << 30):
    A64, W64 = A.double(), W.double()
    y = A64 @ W64.T
    s = A64.abs() @ W64.abs().T
    if b is not None:
        y, s = y + b.double(), s + b.double().abs()
    cols = torch.arange(y.shape[1], device=y.device)
    win = (cols >= act_lo) & (cols < act_hi)
    if act == 1:
        y = torch.where(win, y.clamp_min(0), y)
    elif act == 2:
        y = torch.where(win, torch.tanh(y), y)
    return y, s, win


def _c(got, ref, scale, act, win=None):
    """measured componentwise constant: max (|err| - tanh allowance) / scale"""
    floor = torch.zeros_like(ref)
    if act == 2:
        floor = floor + (C_TANH if win is None else C_TANH * win.double())
    excess = ((got.double() - ref).abs() - floor).clamp_min(0)
    if torch.isnan(got).any():
        return float("inf")
    return float((excess / scale.clamp_min(1e-300)).max())


def _operands(M, N, K, seed, sa=2.0, sw=0.05):
    g = torch.Generator().manual_seed(seed)
    A = (torch.randn(M, K, generator=g) * sa).cuda()
    A[:, ::7] = 0                                     # post-ReLU-like zeros
    W = (torch.randn(N, K, generator=g) * sw).cuda()
    b = torch.randn(N, generator=g).cuda()
    return A, W, b


@pytest.mark.parametrize("M,N,K,act,bn", [(128, 256, 64, 0, 256), (256, 256, 128, 0, 256), (300, 512, 128, 1, 256),
                                          (4096, 1536, 512, 0, 256), (1000, 256, 512, 1, 256),
                                          (128, 64, 64, 0, 64), (4096, 384, 128, 0, 64), (300, 128, 256, 1, 64),
                                          (4096, 512, 256, 2, 64), (777, 256, 320, 0, 64)])
def test_gemm_tc_matches_fp64(M, N, K, act, bn):
    """The plain hook (whole rows, fp32 output): within 3e-6 of max(1, max |pre-activation|) over the matrix, and
    within the componentwise bound element by element."""
    lib, _capi = _lib()
    A, W, b = _operands(M, N, K, M + N + K)
    Cout = torch.full((M, N), float("nan"), device="cuda")
    _capi.check(lib, lib.cn_internal_gemm_tc(A.data_ptr(), W.data_ptr(), b.data_ptr(), Cout.data_ptr(), M, N, K, act, bn),
                "cn_internal_gemm_tc")
    torch.cuda.synchronize()
    ref, scale, _ = _ref(A, W, b, act)
    pre_max = (A.double() @ W.double().T + b.double()).abs().max().item()   # magnitude of the accumulated products
    err = (Cout.double() - ref).abs().max().item()
    assert err < 3e-6 * max(1.0, pre_max), (err, pre_max)
    c = _c(Cout, ref, scale, act)
    print("\nGEMM-C M=%d N=%d K=%d act=%d bn=%d c=%.3g" % (M, N, K, act, bn, c))
    assert c <= C_GEMM, c


@pytest.mark.parametrize("bn", [64, 256])
@pytest.mark.parametrize("m0,m", [(None, 517), (200, 517), (128, 640), (300, 301), (0, 0)])
def test_gemm_tc_device_row_range(bn, m0, m):
    """Rows [m0, m) are computed; tiles wholly past m and the rows before m0 are never touched (NaN sentinel kept).
    Rows of the last partial tile past m may be written: the kernel stores rows up to the extent M by design."""
    M, N, K = 1000, 2 * bn, 256
    A, W, b = _operands(M, N, K, 11 + bn)
    Cout = torch.full((M, N), float("nan"), device="cuda")
    _gemm(A, W, b, M, N, K, 1, bn, out=Cout, m=m, m0=m0)
    lo = m0 or 0
    if m > lo:
        ref, scale, _ = _ref(A[lo:m], W, b, 1)
        assert _c(Cout[lo:m], ref, scale, 1) <= C_GEMM
    tile_end = lo + -(-(m - lo) // 128) * 128 if m > lo else lo
    assert torch.isnan(Cout[:lo]).all() and torch.isnan(Cout[tile_end:]).all()


def _split_ok(hi, lo, v):
    """hi is the fp16 nearest to hi + lo, and (hi, lo) is exactly the split of the fp32 value v"""
    vv = v.float().clamp(-65504, 65504)
    h2 = vv.half()
    return nearest_split(hi, lo) and torch.equal(hi, h2) and torch.equal(lo, (vv - h2.float()).half())


@pytest.mark.parametrize("bn,N,K,act,act_lo,act_hi", [
    (64, 128, 256, 1, 0, 64),          # the rollout's [enc | te] GEMM: ReLU on whole tiles [0, 64)
    (64, 128, 256, 1, 32, 96),         # windows cutting through tiles
    (64, 192, 128, 2, 10, 150),
    (256, 512, 128, 1, 100, 300),
    (256, 512, 256, 2, 0, 257),
])
def test_gemm_tc_act_window_and_split_output(bn, N, K, act, act_lo, act_hi):
    """fp32 and split output together (as the [enc | te] GEMM writes them), the activation on [act_lo, act_hi) only."""
    M = 300
    A, W, b = _operands(M, N, K, bn + N + act_lo)
    Cout = torch.full((M, N), float("nan"), device="cuda")
    hi = torch.full((M, N), 0, dtype=torch.float16, device="cuda")
    lo = torch.full((M, N), 0, dtype=torch.float16, device="cuda")
    _gemm(A, W, b, M, N, K, act, bn, out=Cout, split=(hi, lo), ldh=N, act_lo=act_lo, act_hi=act_hi)
    ref, scale, win = _ref(A, W, b, act, act_lo, act_hi)
    c = _c(Cout, ref, scale, act, win)
    print("\nGEMM-C window bn=%d [%d,%d) act=%d c=%.3g" % (bn, act_lo, act_hi, act, c))
    assert c <= C_GEMM, c
    assert _split_ok(hi, lo, Cout)


@pytest.mark.parametrize("bn,N,K,a_col0,a_pitch,col0,ldh", [
    (64, 256, 64, 64, 128, 0, 256),    # u = W_s^T te: A = columns 64..127 of [enc | te]
    (64, 64, 256, 0, 256, 64, 128),    # edge embedding into columns 64..127 of the GRU input, split only
    (64, 256, 256, 256, 512, 0, 256),  # critic.2: A = columns 256..511 of [actor.0 | critic.0]
    (256, 256, 128, 64, 256, 256, 512),
])
def test_gemm_tc_column_view_and_split_offset(bn, N, K, a_col0, a_pitch, col0, ldh):
    """A read as a column view (pitch != K); split-only output written into a column offset of a wider matrix: the
    columns outside [col0, col0 + N) keep their sentinel."""
    M = 333
    g = torch.Generator().manual_seed(N + K + a_col0)
    Af = (torch.randn(M, a_pitch, generator=g) * 2).cuda()
    W = (torch.randn(N, K, generator=g) * 0.05).cuda()
    b = torch.randn(N, generator=g).cuda()
    sent = torch.full((M, ldh), F16_NAN, dtype=torch.int16, device="cuda").view(torch.float16)
    hi, lo = sent.clone(), sent.clone()
    _gemm(Af, W, b, M, N, K, 1, bn, out=None, a_col0=a_col0, a_pitch=a_pitch,
          split=(hi[:, col0:], lo[:, col0:]), ldh=ldh)
    ref, scale, _ = _ref(Af[:, a_col0:a_col0 + K], W, b, 1)
    h, l_ = hi[:, col0:col0 + N], lo[:, col0:col0 + N]
    s = h.double() + l_.double()
    assert nearest_split(h, l_)                                               # hi = fp16 nearest to hi + lo
    excess = ((s - ref).abs() - 2.0 ** -22 * ref.abs() - 2.0 ** -25).clamp_min(0)
    c = float((excess / scale.clamp_min(1e-300)).max())
    print("\nGEMM-C view bn=%d K=%d col0=%d c=%.3g" % (bn, K, a_col0, c))
    assert c <= C_GEMM, c
    for t in (hi, lo):
        outside = torch.cat([t[:, :col0], t[:, col0 + N:]], 1).view(torch.int16)
        assert (outside == F16_NAN).all()


@pytest.mark.parametrize("bn", [64, 256])
@pytest.mark.parametrize("extra", ["sms-1", "sms", "sms+1", "2sms+1"])
def test_gemm_tc_persistent_tile_counts(bn, extra):
    """Tile counts around the SM count: CTAs walk 1, 2 or 3 tiles and the 2-stage (BN = 256) / 4-stage (BN = 64)
    operand rings wrap across tiles (K = 512: 8 k-blocks per tile)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    tiles = dict({"sms-1": sms - 1, "sms": sms, "sms+1": sms + 1, "2sms+1": 2 * sms + 1})[extra]
    N, K = bn, 512
    M = tiles * 128 - 5                                # last tile partial
    A, W, b = _operands(M, N, K, tiles + bn)
    Cout = torch.full((M, N), float("nan"), device="cuda")
    _gemm(A, W, b, M, N, K, 0, bn, out=Cout)
    ref, scale, _ = _ref(A, W, b, 0)
    c = _c(Cout, ref, scale, 0)
    assert c <= C_GEMM, (tiles, c)


def _check_epilogue_instance(M, N, K, act, bn, out, seed):
    """One activation x output-kind instance (out: "f32", "f16" or "both"), activation window [40, N - 24) cutting
    through a tile: fp32 within the componentwise bound, and the split output exactly the (hi, lo) split of what the
    fp32 output holds (split alone: hi + lo within the bound after the split's own rounding)."""
    act_lo, act_hi = 40, N - 24
    A, W, b = _operands(M, N, K, seed)
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
        floor = 2.0 ** -22 * ref.abs() + 2.0 ** -25 + (C_TANH * win.double() if act == 2 else 0.0)
        excess = ((s - ref).abs() - floor).clamp_min(0)
        assert float((excess / scale.clamp_min(1e-300)).max()) <= C_GEMM


# row magnitudes of A from which the split keeps fp32-equivalent accuracy with the fixed 2^6 weight scale
# (below it the lo piece of A goes subnormal in fp16 and the relative error grows as 2^-25 / |a|)
SWEEP_A_MIN = 2.0 ** -6


def test_gemm_tc_magnitude_sweep():
    """A ~ randn * 2^-12 .. 2^12, W ~ randn * 2^-9 .. 2^3 (K = 512): the componentwise constant stays within C_GEMM
    where |A| >= SWEEP_A_MIN; below it the numbers are reported, not asserted (with torch's fp32 GEMM beside them)."""
    M, N, K = 256, 256, 512
    rows = []
    bad = []
    for ea in range(-12, 13, 3):
        for ew in range(-9, 4, 3):
            g = torch.Generator().manual_seed(1000 + 31 * ea + ew)
            A = (torch.randn(M, K, generator=g) * 2.0 ** ea).cuda()
            W = (torch.randn(N, K, generator=g) * 2.0 ** ew).cuda()
            Cout = torch.full((M, N), float("nan"), device="cuda")
            _gemm(A, W, None, M, N, K, 0, 256, out=Cout)
            ref, scale, _ = _ref(A, W, None, 0)
            c = _c(Cout, ref, scale, 0)
            c32 = _c(A @ W.T, ref, scale, 0)
            rows.append((ea, ew, c, c32))
            if 2.0 ** ea >= SWEEP_A_MIN and not c <= C_GEMM:
                bad.append((ea, ew, c))
    print("\nGEMM-SWEEP  log2|A| log2|W|  c(3xFP16)  c(torch fp32)")
    for ea, ew, c, c32 in rows:
        print("GEMM-SWEEP  %7d %7d  %9.3g  %9.3g%s" % (ea, ew, c, c32, "" if 2.0 ** ea >= SWEEP_A_MIN else "  (reported)"))
    assert not bad, bad


@pytest.mark.parametrize("name,H", [("policy_h20", 20), ("policy_h50", 50)])
def test_cuda_policy_tensor_core_mode_matches_reference_golden(name, H):
    from oracle.policy_ref import PolicyRef
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy
    from tests.policy_fixture import load_policy_golden, synth_state_dict
    import numpy as np
    g, obs, h, masks = load_policy_golden(name)
    sd = synth_state_dict(PolicyRef(12).state_dict())
    pol = CudaPolicy(h.shape[0], H, 12, device="cuda:0", gemm_mode=1)
    pol.load_state_dict(sd)
    dobs = {k: v.cuda() for k, v in obs.items()}
    value, action, logp, h1, mean = pol.act(dobs, h.cuda(), masks.cuda(), deterministic=True, return_mean=True)
    np.testing.assert_allclose(mean.cpu().numpy(), g["synth_mean"], rtol=0, atol=1e-4)
    np.testing.assert_allclose(value.cpu().numpy(), g["synth_value"], rtol=0, atol=1e-4)
    np.testing.assert_allclose(h1.cpu().numpy(), g["synth_h"], rtol=0, atol=1e-4)
