"""Stage-by-stage GPU check of the DS-RNN rollout forward (cn_dsrnn_act, base='srnn') against the fp64 stage reference of
tests/dsrnn_stages.py, and of its edge-GRU GEMM (the TC_OUT_GRU instance of cn_gemm_tc_kernel, whose epilogue computes
the whole GRU cell) on its own through cn_internal_gemm_tc_gru.

Every stage's output, read back through cn_internal_dsrnn_buffer, is compared with fp64 arithmetic applied to the
engine's OWN input to that stage, so a ReLU or mask flip upstream can neither hide nor inflate a stage's error, and the
whole forward is compared with the oracle (oracle/dsrnn_ref.py in float64) at the end.  The bounds scale with the
stage's own operands:

  linear stages        |err| <= c * (|X| @ |W|^T + |b|)  per element        (+ C_TANH absolute after a tanh)
  edge GRU             |err| <= c * (S_z / 2 + S_in + S_hn + |gh_n| S_r / 4) + C_GATE, from the pre-activation scales
                       S_r, S_z, S_in, S_hn of each unit (tests/dsrnn_stages.py, edge_gru)
  edge attention       |err| <= c * max |s_j| of the environment
  node GRU             |err| <= c absolute
  split (hi, lo) pair  hi is the fp16 nearest to hi + lo, and hi + lo may differ from the stage value by the split's
                       own 2^-22 relative + 2^-25 absolute on top of the stage bound

The constants below are at least 3x the worst values measured on an H100 80GB HBM3 (700 W power limit) over every case
of this file; the comment beside each gives that worst value, and each test prints its measured constants beside their
bounds (pytest -s).
"""
import ctypes as C

import pytest
import torch

from oracle.dsrnn_ref import DsrnnRef
from tests.dsrnn_fixture import dsrnn_state_dict
from tests.dsrnn_stages import DsrnnStages, buffer_info, edge_gru, edge_rows, interleave_gru, read
from tests.policy_stages import Buf
from tests.test_gpu_policy_stages import C_TANH, Checker, _split16

pytestmark = pytest.mark.gpu
DEV = "cuda:0"

# c of the componentwise bounds; the comment gives the worst value measured over this file.  The tanh epilogues carry
# test_gpu_policy_stages.C_TANH (1e-6 absolute).
C_ENC = 5e-7              # 1.6e-7  edge and node encoders on the CUDA cores (fp32 fmaf, K <= 16)
C_TC = dict(te=2.5e-6,    # 8.0e-7  wgmma 3xFP16 GEMMs (truncating fp32 accumulation inside the tensor core)
            u=1.5e-6,     # 4.9e-7
            emb=2.5e-6,   # 8.2e-7
            gi=4.5e-6,    # 1.4e-6
            gh=2e-6,      # 5.6e-7
            ac1=5e-7, a2=5e-7, c2=5e-7)   # 0, 1.4e-7, 1.5e-7 beyond C_TANH
C_HEAD = 1.5e-7           # 4.3e-8  value / mean heads on the CUDA cores
C_EDGE = 8e-7             # 2.4e-7  edge GRU (cn_dsrnn_act and the epilogue alone), of its scale, beyond C_GATE
C_GATE = 1e-6             # 0       absolute allowance of the fp32 gate math (expf, tanhf) of a GRU cell: no error
                          #         was left beyond C_EDGE * scale ("*_gate" in the printed constants)
C_ATTN = 1.2e-6           # 3.7e-7  edge attention, of max |s_j| (H = 128: temperature 16)
C_GRU = 7e-7              # 2.2e-7  node GRU, absolute
E2E = 1e-4                # 1.2e-5  value / mean / node and edge state against DsrnnRef.double(), absolute; value: of
                          #         max(1, |value|)
ROWS = 16384              # rows per chunk of the fp64 edge-GRU reference (its gate tensors are [rows, 1024])

CASES = {   # name: (N, H, W, edge state in)
    "n1": (1, 1, 2, "random"),              # one row in a 128-row tile
    "tail129": (43, 3, 16, "random"),       # N H = 129: a one-row last tile; the largest W
    "ragged": (300, 20, 12, "random"),      # partial last tile; some zero masks
    "h128": (3, 128, 12, "random"),         # temperature 16; four score registers per lane
    "zero_state": (64, 20, 2, "none"),      # edge_h_in None, against explicit zeros
    "bench": (4096, 20, 2, "random"),       # tools/bench_dsrnn.py's shape: many tiles per CTA of the persistent GEMM
    "n4096_h50": (4096, 50, 12, "random"),  # a large crowd
}


class _Chk(Checker):
    """Checker that also keeps each stage's bound, to print it beside the measured constant"""

    def __init__(self, tag):
        super(_Chk, self).__init__(tag)
        self.bound = {}

    def _note(self, name, cm, c):
        self.bound[name] = c
        super(_Chk, self)._note(name, cm, c)

    def raw(self, name, err):
        """largest absolute error of a stage (recorded, not asserted: it sizes the absolute allowances)"""
        self.worst[name] = max(self.worst.get(name, 0.0), float(err))

    def report(self):
        print("\nSTAGE-C %s %s" % (self.tag, " ".join(
            "%s=%.3g/%s" % (k, v, "%.3g" % self.bound[k] if k in self.bound else "-") for k, v in sorted(self.worst.items()))))


def _gru_stage(chk, name, got, A, h, B, bias):
    """the edge GRU on row chunks of its engine inputs A (hi + lo) and h (fp32 m h); got: the engine's h' [M, 256]"""
    for r0 in range(0, A.shape[0], ROWS):
        ref, scale = edge_gru(A[r0:r0 + ROWS], h[r0:r0 + ROWS], B, bias)
        g = got[r0:r0 + ROWS]
        assert bool(torch.isfinite(g).all()), "%s: %s is not finite" % (chk.tag, name)
        # the absolute part of the error that C_EDGE * scale leaves (what C_GATE has to cover)
        chk.raw(name + "_gate", ((g.double() - ref).abs() - C_EDGE * scale).max())
        chk.stage(name, g, ref, scale, C_EDGE, C_GATE)


def _inputs(N, H, W, edge, gen):
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=gen) * 3, temporal_edges=torch.randn(N, 1, 2, generator=gen),
               spatial_edges=torch.randn(N, H, W, generator=gen) * 4)
    h = torch.randn(N, 1, 128, generator=gen) * 0.5
    he = torch.randn(N, H + 1, 256, generator=gen) * 0.5 if edge == "random" else None
    masks = (torch.rand(N, 1, generator=gen) > 0.2).float()
    masks[0] = 1.0
    return obs, h, he, masks


@pytest.mark.parametrize("case", list(CASES))
def test_dsrnn_stages_match_fp64(case):
    """One act call; every stage against fp64 on the engine's own inputs, the outputs against DsrnnRef.double()."""
    from crowdnav_prediction_attngraph_b200.policy import CudaDsrnn
    N, H, W, edge = CASES[case]
    NH = N * H
    oracle = DsrnnRef(W)
    sd = dsrnn_state_dict(oracle.state_dict())
    sd["dist.fc_mean.bias"] = torch.tensor([0.3, -0.2])
    sd["base.critic_linear.bias"] = torch.tensor([0.7])
    oracle.load_state_dict(sd)
    oracle = oracle.double().to(DEV)
    eng = CudaDsrnn(N, H, W, device=DEV)
    eng.load_state_dict(sd)
    sref = DsrnnStages(sd, H, W, device=DEV)
    chk = _Chk(case)
    gen = torch.Generator().manual_seed(17 * N + H)
    obs, h, he, masks = _inputs(N, H, W, edge, gen)
    cu = lambda t: None if t is None else t.to(DEV)
    v, a, lp, h1, he1, mean = eng.act({k: cu(x) for k, x in obs.items()}, cu(h), cu(he), cu(masks), deterministic=True,
                                      return_mean=True)
    torch.cuda.synchronize()
    outs = dict(value=v.clone(), mean=mean.clone(), h1=h1.reshape(N, 128).clone(), he1=he1.clone())
    f = lambda t: t.to(DEV, torch.float64)
    m = masks.to(DEV).reshape(N)
    he_in = torch.zeros(N * (H + 1), 256, device=DEV) if he is None else he.to(DEV).reshape(-1, 256)
    # 1. edge GRU A operands [ReLU(encoder_linear x) | m h]: the encoder against fp64, the state half a split of m h
    At, As = read(eng, "At"), read(eng, "As")
    for side, A, x, rows in (("temporal", At, obs["temporal_edges"].reshape(N, 2), edge_rows(he_in, m, 1, H + 1, 0)),
                             ("spatial", As, obs["spatial_edges"].reshape(NH, W), edge_rows(he_in, m, H, H + 1, 1))):
        chk.stage(side + "_enc", Buf(A.val[:, :64], A.hi[:, :64], A.lo[:, :64]), *sref.edge_emb(side, f(x)), C_ENC)
        hm = rows.double()
        chk.stage(side + "_pack_h", Buf(A.val[:, 64:], A.hi[:, 64:], A.lo[:, 64:]), hm, torch.ones_like(hm), 0.0)
        # 2. the edge GRUs, straight into the edge state: temporal row 0, spatial rows 1..H of every environment
        got = he1[:, 0] if side == "temporal" else he1[:, 1:].reshape(NH, 256)
        _gru_stage(chk, side + "_gru", got, A.val, hm, *sref.edge[side][2:])
    del As
    # 3. [h_t' | wv]: h_t' is the split of edge-state row 0; te, u
    HW = read(eng, "HW")
    chk.split_of("HW_ht", Buf(None, HW.hi[:, :256], HW.lo[:, :256]), he1[:, 0])
    te, Te = read(eng, "te"), read(eng, "Te")
    chk.stage("te", te, *sref.te(HW.val[:, :256]), C_TC["te"])
    chk.split_of("Te", Te, te.raw)
    u = read(eng, "u")
    chk.stage("u", u, *sref.u(Te.val), C_TC["u"])
    # 4. edge attention over the engine's spatial states, with its u and fp32 te; wv's split in columns 256..511
    wv = read(eng, "wv")
    wv_ref, smax = sref.edge_attention(he1[:, 1:].double(), u.val, te.val)
    chk.stage("edge_attn", wv, wv_ref, smax[:, None].expand_as(wv_ref), C_ATTN)
    chk.split_of("HW_wv", Buf(None, HW.hi[:, 256:], HW.lo[:, 256:]), wv.raw)
    # 5. node GRU input [enc | emb], h0 = h m (exact), gi, gh, the cell
    T1 = read(eng, "T1")
    chk.stage("enc", Buf(T1.val[:, :64], T1.hi[:, :64], T1.lo[:, :64]), *sref.enc(f(obs["robot_node"]).reshape(N, 7)),
              C_ENC)
    chk.stage("emb", Buf(T1.val[:, 64:], T1.hi[:, 64:], T1.lo[:, 64:]), *sref.emb(HW.val), C_TC["emb"])
    h0, H0 = read(eng, "h0"), read(eng, "H0")
    assert torch.equal(h0.raw, h.to(DEV).reshape(N, 128) * m[:, None])
    chk.split_of("H0", H0, h0.raw)
    gi, gh = read(eng, "gi"), read(eng, "gh")
    chk.stage("gi", gi, *sref.gi(T1.val), C_TC["gi"])
    chk.stage("gh", gh, *sref.gh(H0.val), C_TC["gh"])
    h1_ref = sref.gru(gi.val, gh.val, h0.val)[0]
    chk.stage("node_gru", outs["h1"], h1_ref, torch.ones_like(h1_ref), C_GRU)
    H1 = read(eng, "H1")
    chk.split_of("H1", H1, outs["h1"])
    # 6. actor / critic and the heads
    Ac1 = read(eng, "Ac1")
    chk.stage("ac1", Ac1, *sref.ac1(H1.val), C_TC["ac1"], C_TANH)
    a2, c2 = read(eng, "a2"), read(eng, "c2")
    chk.stage("a2", a2, *sref.a2(Ac1.val[:, :256]), C_TC["a2"], C_TANH)
    chk.stage("c2", c2, *sref.c2(Ac1.val[:, 256:]), C_TC["c2"], C_TANH)
    chk.stage("value", outs["value"], *sref.value(c2.val), C_HEAD)
    chk.stage("mean", outs["mean"], *sref.mean(a2.val), C_HEAD)
    # 7. the whole forward against the oracle
    with torch.no_grad():
        rv, rm, rh, rhe = oracle({k: f(x) for k, x in obs.items()}, f(h), he_in.reshape(N, H + 1, 256).double(),
                                 f(masks))
    for name, want in (("value", rv), ("mean", rm), ("h1", rh.reshape(N, 128)), ("he1", rhe)):
        scale = max(1.0, float(want.abs().max())) if name == "value" else 1.0
        err = float((outs[name].double() - want).abs().max()) / scale
        chk.raw("e2e_" + name, err)
        assert err < E2E, (case, name, err)
    if he is None:
        # a null edge state runs exactly as explicit zeros
        again = eng.act({k: cu(x) for k, x in obs.items()}, cu(h), torch.zeros(N, H + 1, 256, device=DEV), cu(masks),
                        deterministic=True, return_mean=True)
        for name, x in zip(("value", "h1", "he1", "mean"), (again[0], again[3], again[4], again[5])):
            assert torch.equal(x.reshape(outs[name].shape), outs[name]), name
    chk.report()
    eng.close()


def test_dsrnn_buffer_hook_rejects_unknown_names():
    from crowdnav_prediction_attngraph_b200.policy import CudaDsrnn
    eng = CudaDsrnn(4, 3, 2, device=DEV)
    with pytest.raises(RuntimeError, match="unknown buffer 'nope'"):
        buffer_info(eng, "nope")
    assert buffer_info(eng, "As")[2:] == (12, 320, 320, 1)
    eng.close()


# ---- the GRU epilogue on its own ------------------------------------------------------------------------------------
F32_NAN = 0x7FC00000
F16_NAN = 0x7E00


def _gru_hook():
    from crowdnav_prediction_attngraph_b200 import _capi
    lib = _capi.load_library()
    fn = lib.cn_internal_gemm_tc_gru
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p] * 6 + [C.c_int] * 4 + [C.c_void_p, C.c_void_p, C.c_int]
    return lib, fn, _capi


def _gru_call(A, B, bias, h_in, mask, h_out, M, group, pitch, off, oh=None, ol=None, ldh=0):
    lib, fn, _capi = _gru_hook()
    p = lambda t: None if t is None else t.data_ptr()
    _capi.check(lib, fn(p(A), p(B), p(bias), p(h_in), p(mask), p(h_out), M, group, pitch, off, p(oh), p(ol), ldh),
                "cn_internal_gemm_tc_gru")
    torch.cuda.synchronize()


LAYOUTS = {   # name: (group, pitch, off) of the engine's two edge GRUs at H humans
    "temporal_h1": (1, 2, 0), "spatial_h1": (1, 2, 1),
    "temporal_h20": (1, 21, 0), "spatial_h20": (20, 21, 1),
    "temporal_h128": (1, 129, 0), "spatial_h128": (128, 129, 1),
}
VARIANTS = {   # name: (previous state, split output, pre-activation amplitude)
    "state_split": (True, True, 1.0),
    "null_state": (False, True, 1.0),
    "sat30": (True, False, 30.0),        # sigmoid and tanh saturate
}
GRU_CASES = [(M, lay, var) for M in (1, 127, 128, 129, 300) for lay in LAYOUTS for var in VARIANTS] + \
            [(81920, lay, var) for lay in ("temporal_h20", "spatial_h20") for var in VARIANTS]


def _gru_operands(M, group, pitch, off, with_h, amp, seed):
    g = torch.Generator().manual_seed(seed)
    E = -(-M // group)                                     # environments (the last one may be partial)
    wih, whh = torch.randn(768, 64, generator=g) * 0.0625, torch.randn(768, 256, generator=g) * 0.0625
    bih, bhh = torch.randn(768, generator=g) * 0.3, torch.randn(768, generator=g) * 0.3
    B, bias = interleave_gru(wih.double(), whh.double(), bih.double(), bhh.double())
    B, bias = (B * amp).float().to(DEV), (bias * amp).float().to(DEV)
    masks = (torch.rand(E, generator=g) > 0.25).float().to(DEV)
    masks[0] = 1.0
    he = (torch.randn(E * pitch, 256, generator=g) * 0.6).to(DEV) if with_h else None
    hm = edge_rows(he, masks, group, pitch, off)[:M] if with_h else torch.zeros(M, 256, device=DEV)
    x = (torch.randn(M, 64, generator=g) * 1.5).clamp_min(0).to(DEV)
    return torch.cat([x, hm], 1).contiguous(), B, bias, he, masks, hm, E


@pytest.mark.parametrize("M,layout,variant", GRU_CASES)
def test_gru_epilogue_matches_fp64(M, layout, variant):
    """h' of every GEMM row in its state row against fp64 fed the same split A and fp32 m h; every state row outside
    the row mapping (and every split column past 256) bit for bit untouched; nothing NaN or Inf."""
    group, pitch, off = LAYOUTS[layout]
    with_h, split, amp = VARIANTS[variant]
    A, B, bias, he, masks, hm, E = _gru_operands(M, group, pitch, off, with_h, amp, M + pitch + 7 * off)
    h_out = torch.full((E * pitch, 256), float("nan"), device=DEV)
    oh = ol = None
    if split:
        oh = torch.full((M, 512), F16_NAN, dtype=torch.int16, device=DEV).view(torch.float16)
        ol = oh.clone()
    _gru_call(A, B, bias, he, masks, h_out, M, group, pitch, off, oh, ol, 512 if split else 0)
    r = torch.arange(M, device=DEV)
    rows = (r // group) * pitch + off + r % group
    chk = _Chk("gru/%d/%s/%s" % (M, layout, variant))
    ahi, alo = _split16(A)
    _gru_stage(chk, "gru", h_out[rows], ahi.double() + alo.double(), hm.double(), B.double(), bias.double())
    untouched = torch.ones(E * pitch, dtype=torch.bool, device=DEV)
    untouched[rows] = False
    assert bool((h_out[untouched].view(torch.int32) == F32_NAN).all()), "state rows outside the row mapping written"
    if split:
        chk.split_of("split", Buf(None, oh[:, :256].float(), ol[:, :256].float()), h_out[rows])
        for t in (oh, ol):
            assert bool((t[:, 256:].view(torch.int16) == F16_NAN).all()), "split columns past 256 written"
    chk.report()


def test_gru_hook_rejects_bad_arguments():
    """every bad argument is refused with a named error before anything is launched"""
    M, group, pitch, off = 4, 2, 3, 1
    A, B, bias, he, masks, _, E = _gru_operands(M, group, pitch, off, True, 1.0, 1)
    h_out = torch.full((E * pitch, 256), float("nan"), device=DEV)
    oh = torch.zeros(M, 512, dtype=torch.float16, device=DEV)
    bad = [dict(M=0), dict(group=0), dict(off=2), dict(pitch=2), dict(off=-1), dict(mask=None), dict(h_out=None),
           dict(A=None), dict(bias=None), dict(ol=None), dict(ldh=128), dict(ldh=257)]
    for kw in bad:
        a = dict(A=A, B=B, bias=bias, h_in=he, mask=masks, h_out=h_out, M=M, group=group, pitch=pitch, off=off, oh=oh,
                 ol=oh.clone(), ldh=512)
        a.update(kw)
        with pytest.raises(RuntimeError, match="cn_internal_gemm_tc_gru: need"):
            _gru_call(**a)
    assert bool(torch.isnan(h_out).all())
