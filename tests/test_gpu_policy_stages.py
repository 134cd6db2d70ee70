"""Stage-by-stage GPU check of the rollout policy forward (cn_policy_act) against the fp64 stage reference of
tests/policy_stages.py, for every kernel variant and the edge shapes.

Every stage's output, read back through cn_internal_policy_buffer, is compared with fp64 arithmetic applied to the
engine's OWN input to that stage, so the error of each kernel is measured on its own (a ReLU mask flip can then move a
value only by rounding noise), and the whole forward is compared with the fp64 oracle at the end.  The bounds scale with
the stage's own operands, so small magnitudes cannot hide an error:

  linear stages        |err| <= c * (|X| @ |W|^T + |b|)  per element        (+ C_TANH absolute after a tanh)
  human-human attn.    |err| <= c * max |V| of the row's environment and head
  robot-human attn.    |err| <= c * max |s_j| of the environment
  GRU                  |err| <= c absolute
  split (hi, lo) pair  hi == fp16_rn(hi + lo), and hi + lo may differ from the stage value by the split's own
                       2^-22 relative + 2^-25 absolute on top of the stage bound
                       (hi == fp16_rn(hi + lo) up to ties: lo may round to exactly half an ulp of hi)

The constants below are at least 3x the worst values measured on an H100 80GB HBM3 (400 W power limit) over all
variants and shapes of this file.  Each test prints its measured constants (pytest -s).
"""
import pytest
import torch

from tests.policy_stages import Buf, StagedRef, buffer_info, nearest_split, read_buffer

pytestmark = pytest.mark.gpu

# c of the componentwise bounds; the comment gives the worst value measured over all variants and shapes of this file.
# "tc": wgmma 3xFP16 GEMMs (truncating fp32 accumulation inside the tensor core); "f32": fp32 CUDA-core GEMM
# (gemm_mode 0) and the CUDA-core stages of both modes (e1, rs, value, mean).  After a tanh the C_TANH allowance
# absorbed every error measured, so those stages carry the GEMM-wide constant.
C_TC = dict(e2=2e-6,     # 6.7e-7
            qkv=5e-6,    # 1.5e-6
            sout=3e-6,   # 8.3e-7
            t1=3e-6,     # 8.7e-7
            u=2e-6,      # 5.1e-7
            emb=2e-6,    # 5.8e-7
            gi=4e-6,     # 1.0e-6
            gh=4e-6,     # 1.2e-6
            ac1=3e-6, a2=3e-6, c2=3e-6)    # 0, 1.2e-7, 9.1e-8 beyond C_TANH
C_F32 = dict(e1=1e-6,    # 3.1e-7
             e2=2e-6,    # 4.3e-7
             qkv=2e-6,   # 5.2e-7
             sout=2e-6,  # 4.6e-7
             rs=1e-6,    # 2.4e-7
             t1=1e-6,    # 2.9e-7
             u=2e-6,     # 3.8e-7
             emb=1e-6,   # 2.7e-7
             gi=2e-6,    # 6.1e-7
             gh=2e-6,    # 5.3e-7
             ac1=1e-6, a2=1e-6, c2=1e-6,   # 0 beyond C_TANH
             value=2e-7,  # 4.4e-8
             mean=2e-7)   # 5.7e-8
C_HH = dict(f32=2e-6,    # 5.5e-7  human-human attention, of max |V|
            tc=2e-6,     # 3.4e-7
            fused=1.5e-5)  # 4.3e-6: includes the error of its own QKV projection (Q and K enter the scores)
C_HR = 2e-6              # 6.0e-7  robot-human attention, of max |s_j|
C_GRU = 1e-6             # 3.1e-7  GRU cell, absolute
C_TANH = 1e-6            # absolute allowance of a tanh epilogue (fast_tanh / tanhf: ~2e-7)
C_FOLD = 2.0 ** -24      # folded weights: fp64 sum rounded once to fp32
E2E = 1e-4                                # action mean / h1 against PolicyRef.double(), absolute; value: of max(1, |value|)

SHAPES = {   # name: (N, H, Win, pattern of n)
    "n1": (1, 1, 12, "one"),
    "h128": (3, 128, 12, [128, 1, 128]),
    "mc_lt_128": (5, 20, 12, "random"),
    "mc_1280": (64, 20, 12, "full"),
    "varnum": (70, 5, 2, "random"),
    "clamp": (300, 20, 12, "clamp"),
    "n4096_h20": (4096, 20, 12, "half1"),
    "n4096_h50": (4096, 50, 12, "half1"),
    "n4096_h100": (4096, 100, 12, "half1"),
    "n8192": (8192, 20, 12, "random"),
    "n8193": (8193, 20, 12, "random"),
}
VARIANTS = {   # name: (gemm_mode, environment read by cn_policy_create)
    "f32": (0, {}),
    "tc": (1, {}),
    "attn_r2": (1, {"CN_ATTN_R": "2"}),
    "attn_r4": (1, {"CN_ATTN_R": "4"}),
    "fused": (1, {"CN_FUSE_QKV": "1"}),
    "chunks": (1, {"CN_QKV_CHUNKS": "2"}),
}
_ALL = [s for s in SHAPES if s not in ("n8192", "n8193")]
_SOME = ["h128", "mc_lt_128", "clamp", "n4096_h20", "n4096_h100"]
CASES = [(v, s) for v in ("f32", "tc") for s in _ALL] + [("fused", s) for s in SHAPES] + \
        [(v, s) for v in ("attn_r2", "attn_r4", "chunks") for s in _SOME]


def _env(monkeypatch, env):
    for k in ("CN_ATTN_R", "CN_FUSE_QKV", "CN_QKV_CHUNKS", "CN_PDL"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)


def _inputs(N, H, Win, pattern, gen, it):
    if pattern == "one":
        n = torch.ones(N, 1)
    elif isinstance(pattern, list):
        n = torch.tensor(pattern, dtype=torch.float32)[:, None]
    elif pattern == "full":
        n = torch.full((N, 1), float(H))
    else:
        n = torch.randint(1, H + 1, (N, 1), generator=gen).float()
        if pattern == "clamp":                 # outside [1, H]: the engine clamps (0 -> 1, H + 3 -> H)
            n[::7] = 0.0
            n[3::11] = H + 3.0
        if pattern == "half1" and it == 1:
            n[: N // 2] = 1.0                  # half of the batch sees one human: many tiny segments
    ncl = n.clamp(1, H)
    sp = torch.randn(N, H, Win, generator=gen) * 3
    sp[torch.arange(H)[None, :] >= ncl] = 15.0
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=gen) * 3, temporal_edges=torch.randn(N, 1, 2, generator=gen),
               spatial_edges=sp, detected_human_num=n)
    masks = (torch.rand(N, 1, generator=gen) > 0.1).float()
    return obs, masks


def _split16(v):
    """the engine's fp32 -> (hi, lo) fp16 split of fp32 values, as float32 tensors"""
    v = v.float().clamp(-65504.0, 65504.0)
    hi = v.half().float()
    return hi, (v - hi).half().float()


class Checker(object):
    def __init__(self, tag):
        self.tag, self.worst = tag, {}

    def _note(self, name, cm, c):
        self.worst[name] = max(self.worst.get(name, 0.0), cm)
        assert cm <= c, "%s: stage %s error is %.3g of its scale, bound %.3g" % (self.tag, name, cm, c)

    def split(self, name, b):
        """hi is the fp16 nearest to hi + lo, |lo| <= ulp(hi) / 2 (hi + lo itself is checked by the stage).  This is
        hi == fp16_rn(hi + lo) up to ties: lo = fp16_rn(v - hi) may round up to exactly half an ulp."""
        assert nearest_split(b.hi, b.lo), "%s: %s hi is not the fp16 nearest to hi + lo" % (self.tag, name)

    def split_of(self, name, b, f32):
        """the split pair is exactly the split of the fp32 value the same kernel stored"""
        hi, lo = _split16(f32)
        assert torch.equal(b.hi, hi) and torch.equal(b.lo, lo), "%s: %s split != split of its fp32 copy" % (self.tag, name)

    def stage(self, name, got, ref, scale, c, absolute=0.0):
        g = got.val if isinstance(got, Buf) else got.double()
        floor = torch.full_like(ref, absolute)
        if isinstance(got, Buf) and got.split:
            self.split(name, got)
            floor = floor + 2.0 ** -22 * ref.abs() + 2.0 ** -25
        excess = ((g - ref).abs() - floor).clamp_min(0)
        r = excess / scale.clamp_min(1e-300)
        cm = float(r.max()) if r.numel() else 0.0
        if r.numel() and torch.isnan(g).any():
            cm = float("inf")
        self._note(name, cm, c)


def _check_call(chk, sref, pol, mode, fused, obs, h, masks, outs, first):
    """every stage of one cn_policy_act call against the fp64 stage reference on the engine's inputs"""
    tc = mode == 1
    dev = "cuda"
    f = lambda t: t.to(dev, torch.float64)
    N, H = pol.N, pol.H
    torch.cuda.synchronize()
    n, row_start, row_env = sref.layout(obs["detected_human_num"])
    Mc = int(row_start[-1])
    B = lambda name, rows=None: read_buffer(pol, name, rows)
    # 0. compaction
    assert torch.equal(B("row_start").val, row_start) and int(B("mc").val[0]) == Mc
    assert torch.equal(B("row_env", Mc).val, row_env)
    CL = C_TC if tc else C_F32
    # folded weights (cn_fold_mm_kernel / cn_fold_mv_kernel), once per handle
    if first:
        for name, ref in (("Wqkv", sref.Wqkv), ("bqkv", sref.bqkv), ("Wos", sref.Wos), ("bos", sref.bos),
                          ("Woac", sref.Woac), ("boac", sref.boac)):
            got = B(name).val.reshape(ref.shape)
            assert float(((got - ref).abs() - C_FOLD * ref.abs()).max()) <= 1e-12 * float(ref.abs().max()), name
    # 1. human-human branch
    e1 = B("e1", Mc)
    chk.stage("e1", e1, *sref.embed1(f(obs["spatial_edges"]), row_start, row_env), C_F32["e1"])
    e2 = B("e2", Mc)
    chk.stage("e2", e2, *sref.embed2(e1.val), CL["e2"])
    if fused:
        with pytest.raises(RuntimeError, match="never written"):
            buffer_info(pol, "qkv")
        qkv_in = sref.qkv(e2.val)[0]
        c_hh = C_HH["fused"]
    else:
        qkv = B("qkv", Mc)
        chk.stage("qkv", qkv, *sref.qkv(e2.val), CL["qkv"])
        qkv_in = qkv.val
        c_hh = C_HH["tc" if tc else "f32"]
    ao = B("ao", Mc)
    chk.stage("hh_attn", ao, *sref.hh_attention(qkv_in, n, row_start, row_env), c_hh)
    del qkv_in
    sout = B("sout", Mc)
    chk.stage("sout", sout, *sref.outproj(ao.val), CL["sout"])
    # 2. robot branch: rs -> [enc | te] -> u
    rs = B("rs")
    chk.stage("rs", rs, *sref.robot(StagedRef.robot_input(f(obs["robot_node"]), f(obs["temporal_edges"]))), C_F32["rs"])
    t1 = B("t1")
    ref_t1, sc_t1 = sref.enc_te(rs.val)
    if tc:
        t1f = B("t1.f32")                      # [enc | te]: emb overwrote only the split pair's te half
        chk.stage("t1", t1f, ref_t1, sc_t1, CL["t1"])
        chk.split_of("t1", Buf(None, t1.hi[:, :64], t1.lo[:, :64]), t1f.raw[:, :64])
        te_hr = t1f.val[:, 64:]                # the robot-human attention reads the fp32 te
        hi, lo = _split16(t1f.raw[:, 64:])
        te_u = hi.double() + lo.double()      # the u GEMM read the split te
    else:
        chk.stage("t1", t1.val[:, :64], ref_t1[:, :64], sc_t1[:, :64], CL["t1"])
        te_hr = te_u = ref_t1[:, 64:]          # emb overwrote te: recomputed from this stage's own input (rs)
    u = B("u")
    chk.stage("u", u, *sref.u(te_u), CL["u"])
    # 3. robot-human attention, edge embedding, GRU
    wv = B("wv")
    wv_ref, _, smax = sref.hr_attention(sout.val, u.val, te_hr, n, row_start)
    chk.stage("hr_attn", wv, wv_ref, smax[:, None].expand_as(wv_ref), C_HR)
    if tc:
        wvf = B("wv.f32")
        chk.stage("hr_attn", wvf, wv_ref, smax[:, None].expand_as(wv_ref), C_HR)
        chk.split_of("wv", wv, wvf.raw)
    emb_ref, emb_sc = sref.emb(wv.val)
    if tc:
        chk.stage("emb", Buf(t1.val[:, 64:], t1.hi[:, 64:], t1.lo[:, 64:]), emb_ref, emb_sc, CL["emb"])
    else:
        chk.stage("emb", t1.val[:, 64:], emb_ref, emb_sc, CL["emb"])
    gi = B("gi")
    chk.stage("gi", gi, *sref.gi(t1.val), CL["gi"])
    h0 = B("h0")
    h0_ref = (h.reshape(N, 128).float() * masks.reshape(N, 1).float()).cuda()   # fp32 product, exact here
    h0f = B("h0.f32") if tc else h0
    assert torch.equal(h0f.raw, h0_ref)
    if tc:
        chk.split_of("h0", h0, h0f.raw)
    gh = B("gh")
    chk.stage("gh", gh, *sref.gh(h0.val), CL["gh"])
    h1_ref = sref.gru(gi.val, gh.val, h0f.val)[0]
    h_out = outs["h_out"].reshape(N, 128)
    chk.stage("gru", h_out, h1_ref, torch.ones_like(h1_ref), C_GRU)
    if tc:
        h1 = B("h1")
        chk.split_of("h1", h1, h_out)
        h1_in = h1.val
    else:
        h1_in = h_out.double()
    # 4. heads
    ac1 = B("ac1")
    chk.stage("ac1", ac1, *sref.ac1(h1_in), CL["ac1"], C_TANH)
    a2, c2 = B("a2"), B("c2")
    chk.stage("a2", a2, *sref.a2(ac1.val[:, :256]), CL["a2"], C_TANH)
    chk.stage("c2", c2, *sref.c2(ac1.val[:, 256:]), CL["c2"], C_TANH)
    chk.stage("value", outs["value"], *sref.value(c2.val), C_F32["value"])
    chk.stage("mean", outs["mean"], *sref.mean(a2.val), C_F32["mean"])


def _run(pol, obs, h, masks):
    value, action, logp, h1, mean = pol.act({k: v.cuda() for k, v in obs.items()}, h.cuda(), masks.cuda(),
                                            deterministic=True, return_mean=True)
    torch.cuda.synchronize()
    return dict(value=value.clone(), mean=mean.clone(), h_out=h1.clone())


@pytest.mark.parametrize("variant,shape", CASES)
def test_policy_stages_match_fp64(variant, shape, monkeypatch):
    """Three consecutive act calls per handle (workspace, operand rings and the hidden state carry over); every
    stage of every call against fp64 on the engine's own inputs, the outputs against PolicyRef.double()."""
    from oracle.policy_ref import PolicyRef
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy, make_reference_like_state_dict
    N, H, Win, pattern = SHAPES[shape]
    mode, env = VARIANTS[variant]
    _env(monkeypatch, env)
    seed = 17 * N + H
    sd = make_reference_like_state_dict(Win, seed=seed)
    sd["dist.fc_mean.bias"] = torch.tensor([0.3, -0.2])
    sd["base.critic_linear.bias"] = torch.tensor([0.7])
    pol = CudaPolicy(N, H, Win, device="cuda:0", gemm_mode=mode)
    pol.load_state_dict(sd)
    fused = variant == "fused" and N <= 8192
    if variant == "fused" and N > 8192:        # above QA_MAX_ENVS the two-kernel path runs instead
        buffer_info(pol, "qkv")
    sref = StagedRef(sd, H, device="cuda")
    oracle = PolicyRef(Win)
    oracle.load_state_dict(sd)
    oracle = oracle.double().cuda()
    chk = Checker("%s/%s" % (variant, shape))
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(N, 1, 128, generator=gen) * 0.5
    for it in range(3):
        obs, masks = _inputs(N, H, Win, pattern, gen, it)
        outs = _run(pol, obs, h, masks)
        _check_call(chk, sref, pol, mode, fused, obs, h, masks, outs, it == 0)
        dobs = {k: v.cuda().double() for k, v in obs.items()}
        dobs["detected_human_num"] = dobs["detected_human_num"].clamp(1, H)     # the oracle itself does not clamp
        with torch.no_grad():
            rv, rm, rh = oracle(dobs, h.cuda().double(), masks.cuda().double())
        for name, got, want in (("value", outs["value"], rv), ("mean", outs["mean"], rm),
                                ("h1", outs["h_out"].reshape(N, 128), rh.reshape(N, 128))):
            scale = max(1.0, float(want.abs().max())) if name == "value" else 1.0     # |value| reaches ~20
            err = float((got.double() - want).abs().max()) / scale
            chk.worst["e2e_" + name] = max(chk.worst.get("e2e_" + name, 0.0), err)
            assert err < E2E, (chk.tag, it, name, err)
        if pattern == "clamp":
            # n = 0 runs exactly as n = 1, and n > H exactly as n = H
            again = _run(pol, dict(obs, detected_human_num=obs["detected_human_num"].clamp(1, H)), h, masks)
            for k in again:
                assert torch.equal(again[k], outs[k]), k
        h = outs["h_out"].cpu()                # the engine's own state feeds the next call
    print("\nSTAGE-C %s %s" % (chk.tag, " ".join("%s=%.3g" % kv for kv in sorted(chk.worst.items()))))
    pol.close()


_PDL_BUFFERS = ["row_start", "row_env", "mc", "e1", "e2", "qkv", "ao", "sout", "rs", "t1", "u", "wv", "h0", "gi", "gh",
                "h1", "ac1", "a2", "c2"]


@pytest.mark.parametrize("fused", ["0", "1"])
def test_policy_pdl_off_is_bit_identical(fused, monkeypatch):
    """CN_PDL=0 launches the same kernels without programmatic dependent launch: every buffer and output must be
    bit-identical to the default (gemm_mode 1, with and without the fused QKV-attention kernel)."""
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy, make_reference_like_state_dict
    N, H, Win = 4096, 50, 12
    sd = make_reference_like_state_dict(Win, seed=77)
    pols = []
    for pdl in ("1", "0"):
        _env(monkeypatch, {"CN_FUSE_QKV": fused, "CN_PDL": pdl})
        p = CudaPolicy(N, H, Win, device="cuda:0", gemm_mode=1)
        p.load_state_dict(sd)
        pols.append(p)
    gen = torch.Generator().manual_seed(5)
    h = torch.randn(N, 1, 128, generator=gen) * 0.5
    names = [b for b in _PDL_BUFFERS if not (fused == "1" and b == "qkv")]
    for it in range(3):
        obs, masks = _inputs(N, H, Win, "half1", gen, it)
        outs = [_run(p, obs, h, masks) for p in pols]
        for k in outs[0]:
            assert torch.equal(outs[0][k], outs[1][k]), (it, k)
        Mc = int(read_buffer(pols[0], "mc", device="cpu").val[0])
        for name in names:
            rows = Mc if name in ("row_env", "e1", "e2", "qkv", "ao", "sout") else None
            a, b = (read_buffer(p, name, rows, device="cpu") for p in pols)
            if a.split:
                assert torch.equal(a.hi, b.hi) and torch.equal(a.lo, b.lo), (it, name)
            else:
                assert torch.equal(a.raw, b.raw), (it, name)
        h = outs[0]["h_out"].cpu()
    for p in pols:
        p.close()


def test_policy_buffer_hook_rejects_unknown_names():
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy
    pol = CudaPolicy(4, 3, 12, device="cuda:0", gemm_mode=0)
    with pytest.raises(RuntimeError, match="unknown buffer 'nope'"):
        buffer_info(pol, "nope")
    with pytest.raises(RuntimeError, match="gemm_mode 1 only"):
        buffer_info(pol, "h1")
    with pytest.raises(RuntimeError, match="finalize"):
        buffer_info(pol, "Wqkv")
    pol.close()
