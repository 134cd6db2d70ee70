"""Stage-by-stage GPU check of the GST predictor step (cn_gst_step) against the fp64 stage reference of
tests/gst_stages.py, from one environment to 4096.

Each check replays the same seeded history from cn_gst_reset and stops the last step right after one stage
(cn_internal_gst_stop_after), then reads the workspace back (cn_internal_gst_buffer).  Every stage's output is
compared with fp64 arithmetic applied to the engine's OWN input to that stage, so each kernel is measured on its own:

  compaction           bit for bit against numpy (masks, inputs, counts, prefix sums, maps, the ring)
  linear stages        |err| <= c * (|X| @ |W|^T + |b|)  per element
  LayerNorm            |err| <= c * (|gamma| * (max_j scale_j / sigma + |z|) + |beta|)  (GstStages.layer_norm)
  attention            |err| <= c * max |V| over the group's live rows and the head
  LSTM cell            |err| <= c absolute
  h2p                  linear bound, then the running sum and the world position exactly in fp32
  split (hi, lo) pair  hi is the fp16 nearest to hi + lo, and hi + lo may differ from the stage value by the split's
                       own 2^-22 relative + 2^-25 absolute on top of the stage bound
  final kernel         exact on the engine's pred: copied positions, pred - robot, penalty, reward; rows sorted by
                       distance with equal keys in index order (keys within one ulp may swap: x*x + y*y may contract)

and the step's output against the chained fp64 reference.  The shapes drive the loops the small fixtures never reach:
scans with several elements per thread, grid-stride row kernels past their first pass, hundreds of GEMM row tiles.

The constants are at least 3x the worst values measured on an H100 80GB HBM3 (700 W power limit) over all shapes of
this file; each test prints its measured constants (pytest -s).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests.gst_stages import (Buf, GstStages, Ring, T, compaction, declare, final_rows, penalty, random_history,
                              read_buffer, sort_keys, split16)
from tests.policy_stages import nearest_split

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

# c of the bounds; the comment gives the worst value measured over all shapes of this file
C_LIN = dict(qkv=4e-6,    # 1.1e-6
             out=3e-6,    # 8.5e-7
             ffn1=2e-6,   # 6.0e-7
             ffn2=4e-6,   # 1.1e-6
             gx=3e-6,     # 8.4e-7
             gh=3e-6,     # 9.1e-7
             h2p=8e-7)    # 2.4e-7
C_LN = dict(embed=5e-7,   # 1.4e-7
            norm1=2e-7)   # 5.9e-8
C_ATTN = 1.5e-5          # 4.4e-6
C_CELL = 4e-6            # 1.3e-6
E2E = 1.5e-5             # 4.4e-6  final spatial_edges against the chained fp64 reference, of max(1, |value|)
NEAR_THR = 1e-6          # predicted points this close to the collision distance may fall on either side of it
SENTINEL = 12345.0
GUARD = 256              # floats after the N * H * 2(P + 1) output that the step must not touch

SHAPES = {   # name: (N, H, P, visibility per frame)
    "n1_h1": (1, 1, 5, 1.0),
    "n3_h128_all": (3, 128, 5, 1.0),
    "n64_h128": (64, 128, 5, 0.15),
    "n300_h33": (300, 33, 5, 0.5),
    "p1": (50, 20, 1, 0.5),
    "p3": (50, 20, 3, 0.5),
    "n1025_h5": (1025, 5, 5, 0.5),
    "n4096_h20": (4096, 20, 5, 0.5),
    "n4096_h100": (4096, 100, 5, 0.5),
}


def _passes(sms):
    """rows one pass of the grid-stride kernels covers: rows_grid = 4 * SMs CTAs of 256 threads"""
    threads = 4 * sms * 256
    return dict(warp_rows=threads // 32, elem_rows=threads // 64, h2p_rows=threads // 2)


def _assert_coverage(shape, comp, sms):
    """the shape drives the code paths it is in this file for"""
    N, H, P, _ = SHAPES[shape]
    R0, D = (int(x) for x in comp["counts"])
    gc = comp["gcount"]
    p = _passes(sms)
    if shape == "n1_h1":
        assert (gc == H).all()                                   # 8-thread attention CTAs without masked keys
    elif shape == "n3_h128_all":
        assert gc.max() == 128                                   # 1024 threads, 96 KB of shared memory
    elif shape == "n64_h128":
        assert 0 < np.median(gc) < 32 and gc.max() == 128 and (gc == 0).any()
    elif shape == "n300_h33":
        assert N * T > 1024                                      # group scan: two elements per thread
        assert comp["rowm"].reshape(N, T, H)[:, :, 32].any()     # the 33rd human: a second chunk of one
    elif shape in ("p1", "p3"):
        assert P < 5
    elif shape == "n1025_h5":
        assert N > 1024                                          # estart scan: two elements per thread
    elif shape == "n4096_h20":
        assert R0 > p["warp_rows"] and D > p["elem_rows"]        # embed / res_ln, res / cell past their first pass
        assert R0 // 128 >= 200                                  # hundreds of 128-row GEMM tiles
    elif shape == "n4096_h100":
        assert D > p["h2p_rows"]                                 # h2p past its first pass
    return dict(R0=R0, D=D, **p)


class _Handle(object):
    def __init__(self, N, H, P, params):
        from crowdnav_prediction_attngraph_b200 import _capi
        self.capi, self.lib = _capi, _capi.load_library()
        declare(self.lib)
        self.h = C.c_void_p()
        _capi.check(self.lib, self.lib.cn_gst_create(N, H, P, 0.3, 0.3, -20.0, 0, C.byref(self.h)), "create")
        for k, a in params.items():
            a = np.ascontiguousarray(a, dtype=np.float32)
            _capi.check(self.lib, self.lib.cn_gst_set_param(self.h, k.encode(), a.ctypes.data, a.size), k)
        _capi.check(self.lib, self.lib.cn_gst_finalize(self.h), "finalize")
        self.N, self.H, self.P, self.W = N, H, P, 2 * (P + 1)
        self.out = torch.full((N * H * self.W + GUARD,), SENTINEL, device="cuda")
        self.pen = torch.zeros(N, device="cuda")

    def run(self, hist, steps, stop=None, reward=None):
        """cn_gst_reset, then `steps` steps of the history; the last stops after `stop` (None: the whole step) and
        adds its penalty to `reward` (returned)"""
        chk = self.capi.check
        chk(self.lib, self.lib.cn_gst_reset(self.h, None), "reset")
        rw = None
        for s in range(steps):
            robot, sp2, vis = hist[s]
            last = s == steps - 1
            if last and stop:
                chk(self.lib, self.lib.cn_internal_gst_stop_after(self.h, stop.encode()), "stop_after(%s)" % stop)
            if last and reward is not None:
                rw = reward.clone()
            chk(self.lib, self.lib.cn_gst_step(self.h, robot.data_ptr(), sp2.data_ptr(), vis.data_ptr(),
                                               rw.data_ptr() if rw is not None else None, self.pen.data_ptr(),
                                               self.out.data_ptr(), None), "step %d" % s)
        torch.cuda.synchronize()
        return rw

    def buf(self, name, rows=None, device="cuda"):
        return read_buffer(self.lib, self.h, name, rows, device)

    def rows(self):
        return self.out[:self.N * self.H * self.W].reshape(self.N, self.H, self.W).cpu().numpy()

    def close(self):
        self.lib.cn_gst_destroy(self.h)


class Checker(object):
    def __init__(self, tag):
        self.tag, self.worst = tag, {}

    def note(self, name, v, c):
        self.worst[name] = max(self.worst.get(name, 0.0), v)
        assert v <= c, "%s: %s is %.3g, bound %.3g" % (self.tag, name, v, c)

    def split_of(self, name, b, f32):
        """the split pair is exactly the split of the fp32 value the same kernel computed"""
        hi, lo = split16(f32)
        assert torch.equal(b.hi, hi) and torch.equal(b.lo, lo), "%s: %s split != split of its fp32 value" % (self.tag, name)

    def stage(self, name, got, ref, scale, c):
        g = got.val if isinstance(got, Buf) else got.double()
        floor = torch.zeros_like(ref)
        if isinstance(got, Buf) and got.split:
            assert nearest_split(got.hi, got.lo), "%s: %s hi is not the fp16 nearest to hi + lo" % (self.tag, name)
            floor = floor + 2.0 ** -22 * ref.abs() + 2.0 ** -25
        assert g.shape == ref.shape, (self.tag, name, g.shape, ref.shape)
        if g.numel() == 0:
            return
        assert not torch.isnan(g).any(), "%s: %s has NaN" % (self.tag, name)
        excess = ((g - ref).abs() - floor).clamp_min(0)
        self.note(name, float((excess / scale.clamp_min(1e-300)).max()), c)


def _upload(hist_np):
    return [(torch.from_numpy(r).cuda(), torch.from_numpy(s).cuda(), torch.from_numpy(v).cuda()) for r, s, v in hist_np]


def _params():
    return dict(np.load(os.path.join(GOLD, "gst_params.npz")))


def _check_compaction(k, comp, ring, N, H):
    def eq(name, ref, rows=None):
        got = k.buf(name, rows, device="cpu").raw.numpy().reshape(np.shape(ref))
        assert np.array_equal(got, ref), name
    R0, D = (int(x) for x in comp["counts"])
    eq("rowm", comp["rowm"])
    eq("inp", comp["inp"])
    eq("fp", comp["fp"])
    eq("pos_last", comp["pos_last"])
    for name in ("gcount", "gstart", "ecount", "estart", "cidx"):
        eq(name, comp[name].astype(np.int32))
    eq("crow", comp["crow"].astype(np.int32), R0)
    eq("drow", comp["drow"].astype(np.int32), D)
    assert k.buf("counts", device="cpu").raw.numpy()[:2].tolist() == [R0, D]
    eq("ring_pos", ring.pos.reshape(-1, 2))
    eq("ring_mask", ring.mask.reshape(-1))


def _engine_order(out, expected, sp2):
    """Which human each output row holds: the float32 key order (stable), and where the engine's rows differ from it
    (keys within one ulp), the matching human of lowest index.  Asserts the rows are those of a permutation that sorts
    by distance with equal positions in index order.  Returns (perm [N,H], number of envs with a near-tie swap)."""
    N, H, _ = out.shape
    key = sort_keys(sp2)
    perm = np.argsort(key, 1, kind="stable")
    bad = ~(out == np.take_along_axis(expected, perm[..., None], 1)).all(-1)
    swapped = np.flatnonzero(bad.any(1))
    for e in swapped:
        used = np.zeros(H, bool)
        for r in range(H):
            cand = np.flatnonzero(~used & (expected[e] == out[e, r]).all(-1))
            assert cand.size, "env %d row %d is no human's row" % (e, r)
            perm[e, r] = cand[0]
            used[cand[0]] = True
    assert (np.sort(perm, 1) == np.arange(H)).all()
    ks = np.take_along_axis(key, perm, 1)
    assert (np.maximum.accumulate(ks, 1) - ks <= np.spacing(ks)).all(), "rows not sorted by distance"
    pos = np.take_along_axis(sp2, perm[..., None], 1)
    same = (pos[:, 1:] == pos[:, :-1]).all(-1)
    assert (perm[:, 1:] > perm[:, :-1])[same].all(), "equal positions not in index order"
    return perm, len(swapped)


def _check_final(chk, k, st, comp, hist_np, S, reward_in, rw, stats):
    N, H, P = k.N, k.H, k.P
    robot, sp2, _ = hist_np[S - 1]
    fp = comp["fp"].reshape(N, H)
    pred = k.buf("pred", device="cpu").raw.numpy().reshape(N, H, T, 2)
    thr = float(np.float32(0.6))
    pen_ref, dist, counted = penalty(robot, fp, pred, P, thr)
    near = ((np.abs(dist - thr) < NEAR_THR) & counted).any((1, 2))
    pen = k.pen.cpu().numpy()
    assert np.array_equal(pen[~near], pen_ref[~near].astype(np.float32))
    want_rw = (reward_in.cpu().numpy() + pen_ref.astype(np.float32)).astype(np.float32)
    assert np.array_equal(rw.cpu().numpy()[~near], want_rw[~near])
    stats["near_thr_envs"] = stats.get("near_thr_envs", 0) + int(near.sum())
    stats["penalised_envs"] = stats.get("penalised_envs", 0) + int((pen < 0).sum())
    if P < T:                        # points k >= P are predicted but add no penalty
        pen_all = penalty(robot, fp, pred, T, thr)[0]
        only_late = (pen_all != pen_ref) & ~near
        stats["late_only_envs"] = stats.get("late_only_envs", 0) + int(only_late.sum())
    out = k.rows()
    guard = k.out[N * H * k.W:].cpu()
    assert (guard == SENTINEL).all(), "the step wrote past its 2(P+1)-wide rows"
    expected = final_rows(robot, sp2, fp, pred, P)
    assert expected.dtype == np.float32
    perm, swaps = _engine_order(out, expected, sp2)
    stats["tie_swaps"] = stats.get("tie_swaps", 0) + swaps
    assert np.array_equal(out, np.take_along_axis(expected, perm[..., None], 1))
    # end to end: the chained fp64 reference from the same compaction
    pc = np.zeros((N * H, T, 2))
    pc[comp["drow"]] = st.chain(comp).cpu().numpy()
    pc = pc.reshape(N, H, T, 2)
    ref = np.take_along_axis(final_rows(robot.astype(np.float64), sp2.astype(np.float64), fp, pc, P), perm[..., None], 1)
    chk.note("e2e", float((np.abs(out - ref) / np.maximum(1.0, np.abs(ref))).max()), E2E)
    pen_c, dist_c, _ = penalty(robot.astype(np.float64), fp, pc, P, thr)
    amb = ((np.abs(dist_c - thr) < 10 * E2E) & counted).any((1, 2)) | near
    assert np.array_equal(pen[~amb], pen_c[~amb].astype(np.float32))


def _check_encoder(chk, k, st, inp, start, rows):
    """at stop "obs.out" / "decK.out": embedding, QKV, attention and out-projection on their own inputs; returns the
    fp32 X0 and O the residual adds"""
    X0, tX = k.buf("X0", rows), k.buf("tX", rows)
    chk.stage("embed", X0, *st.embed(inp), C_LN["embed"])
    chk.split_of("embed", tX, X0.raw)
    qkv = k.buf("QKV", rows)
    chk.stage("qkv", qkv, *st.qkv(tX.val), C_LIN["qkv"])
    tA = k.buf("tA", rows)
    chk.stage("attn", tA, *st.attention(qkv.val, start), C_ATTN)
    del qkv
    O = k.buf("O", rows)
    chk.stage("out", O, *st.outproj(tA.val), C_LIN["out"])
    return X0.raw, O.raw


def _check_encoder_tail(chk, k, st, rows, X0, O):
    X1 = k.buf("X1", rows)
    assert torch.equal(X1.raw, X0 + O), "X1 != X0 + O in fp32"
    tY = k.buf("tY", rows)
    chk.stage("norm1", tY, *st.norm1(X1.val), C_LN["norm1"])
    tF = k.buf("tF", rows)
    chk.stage("ffn1", tF, *st.ffn1(tY.val), C_LIN["ffn1"])
    O2 = k.buf("O", rows)
    chk.stage("ffn2", O2, *st.ffn2(tF.val), C_LIN["ffn2"])
    tXS = k.buf("tXS", rows)
    chk.split_of("res", tXS, X1.raw + O2.raw)
    GX = k.buf("GX", rows)
    chk.stage("gx", GX, *st.gx(tXS.val), C_LIN["gx"])
    return GX.val


def _check_cell(chk, k, st, D, gx, gh, c_prev):
    h, c, hd = k.buf("h32", D), k.buf("c32", D), k.buf("tHd", D)
    h_ref, c_ref = st.cell(gx, gh, c_prev)
    one = torch.ones_like(h_ref)
    chk.stage("cell", h, h_ref, one, C_CELL)
    chk.stage("cell", c, c_ref, one, C_CELL)
    chk.split_of("cell", hd, h.raw)


def _check_h2p(chk, k, st, comp, D, tt, mu_prev):
    h, xin, mu = k.buf("h32", D), k.buf("xin", D), k.buf("mu_cum", D)
    chk.stage("h2p", xin, *st.h2p(h.val), C_LIN["h2p"])
    want = xin.raw if tt == 0 else mu_prev + xin.raw
    assert torch.equal(mu.raw, want), "mu_cum is not the fp32 running sum"
    drow = torch.as_tensor(comp["drow"], device="cuda")
    pred = k.buf("pred").raw[drow, 2 * tt:2 * tt + 2]
    pos_last = k.buf("pos_last").raw[drow]
    assert torch.equal(pred, mu.raw + pos_last), "pred != mu_cum + pos_last in fp32"
    return mu.raw


def _check_step(chk, k, st, hist, hist_np, S, comp, ring, stats):
    N, H = k.N, k.H
    R0, D = (int(x) for x in comp["counts"])
    reward_in = torch.from_numpy(np.random.RandomState(S).normal(0, 3, N).astype(np.float32)).cuda()
    k.run(hist, S)
    _check_compaction(k, comp, ring, N, H)
    # observation encoder
    k.run(hist, S, "obs.out")
    X0, O = _check_encoder(chk, k, st, comp["inp"][comp["crow"]], comp["gstart"], R0)
    k.run(hist, S, "obs.gx")
    GX = _check_encoder_tail(chk, k, st, R0, X0, O)
    # LSTM over the observed frames
    hd_prev = c_prev = None
    for t in range(T):
        k.run(hist, S, "lstm%d" % t)
        gx = st.lstm_gx(GX, comp["cidx"], comp["drow"], t)
        if t == 0:
            gh, cp = st.bhh.expand(D, 256), torch.zeros(D, 64, dtype=torch.float64, device="cuda")
        else:
            GH = k.buf("GH", D)
            chk.stage("gh", GH, *st.gh(hd_prev.val), C_LIN["gh"])
            gh, cp = GH.val, c_prev.val
        _check_cell(chk, k, st, D, gx, gh, cp)
        hd_prev, c_prev = k.buf("tHd", D), k.buf("c32", D)
    del GX
    # decoding
    k.run(hist, S, "dec0.h2p")
    _check_h2p(chk, k, st, comp, D, 0, None)
    for tt in range(1, T):
        pre = "dec%d." % tt
        k.run(hist, S, pre + "out")
        xin, mu_prev = k.buf("xin", D), k.buf("mu_cum", D).raw
        hd_prev, c_prev = k.buf("tHd", D), k.buf("c32", D)
        X0, O = _check_encoder(chk, k, st, xin.raw, comp["estart"], D)
        k.run(hist, S, pre + "cell")
        GXd = _check_encoder_tail(chk, k, st, D, X0, O)
        GH = k.buf("GH", D)
        chk.stage("gh", GH, *st.gh(hd_prev.val), C_LIN["gh"])
        _check_cell(chk, k, st, D, GXd, GH.val, c_prev.val)
        k.run(hist, S, pre + "h2p")
        _check_h2p(chk, k, st, comp, D, tt, mu_prev)
    # the wrapper's tail on the engine's predictions, and the output end to end (after the stages, so that an
    # arithmetic error is reported by the stage that made it)
    rw = k.run(hist, S, reward=reward_in)
    _check_final(chk, k, st, comp, hist_np, S, reward_in, rw, stats)


@pytest.mark.parametrize("shape", list(SHAPES))
def test_gst_stages_match_fp64(shape):
    """At step 5 (the first full history) and step 7 (the ring has wrapped): compaction bit for bit, every stage
    against fp64 on the engine's own inputs, the final kernel exactly on the engine's predictions, the output against
    the chained fp64 reference."""
    N, H, P, vis_p = SHAPES[shape]
    params = _params()
    hist_np = random_history(N, H, 7, vis_p, 1000 + 7 * N + H + P)
    hist = _upload(hist_np)
    st = GstStages(params, H, device="cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    k = _Handle(N, H, P, params)
    chk = Checker(shape)
    stats = {}
    ring = Ring(N, H)
    for S in range(1, 8):
        pos, m = ring.step(*hist_np[S - 1])
        if S in (5, 7):
            comp = compaction(pos, m)
            cov = _assert_coverage(shape, comp, sms)
            chk.tag = "%s/step%d" % (shape, S)
            _check_step(chk, k, st, hist, hist_np, S, comp, ring, stats)
            print("\nCOVER %s step %d %s" % (shape, S, " ".join("%s=%s" % kv for kv in sorted(cov.items()))))
    if P < T:
        assert stats["late_only_envs"] > 0, "no env had a collision at k >= P only: the P < 5 penalty was not exercised"
    print("\nSTAGE-C %s %s" % (shape, " ".join("%s=%.3g" % kv for kv in sorted(chk.worst.items()))))
    print("FINAL %s %s" % (shape, " ".join("%s=%d" % kv for kv in sorted(stats.items()))))
    k.close()
    torch.cuda.empty_cache()


def _full_run(hist_np, lo, hi, H, steps=7):
    """one handle over envs [lo, hi) of the history; (pred, spatial_edges, penalty) after `steps` steps"""
    k = _Handle(hi - lo, H, 5, _params())
    hist = _upload([(r[lo:hi], s[lo:hi], v[lo:hi]) for r, s, v in hist_np])
    k.run(hist, steps)
    res = (k.buf("pred", device="cpu").raw.reshape(hi - lo, -1), torch.from_numpy(k.rows()), k.pen.cpu())
    k.close()
    return res


def test_gst_bit_identical_across_shards_pdl_and_runs(monkeypatch):
    """N = 4096, H = 20: two handles of 2048 environments, and of 1 + 4095, equal one handle of 4096; CN_PDL=0 equals
    the default; two runs of the same step are equal."""
    N, H = 4096, 20
    hist_np = random_history(N, H, 7, 0.5, 4242)
    monkeypatch.delenv("CN_PDL", raising=False)
    whole = _full_run(hist_np, 0, N, H)
    for cut in (2048, 1):
        parts = [_full_run(hist_np, 0, cut, H), _full_run(hist_np, cut, N, H)]
        for i, name in enumerate(("pred", "spatial_edges", "penalty")):
            assert torch.equal(torch.cat([parts[0][i], parts[1][i]]), whole[i]), (cut, name)
    monkeypatch.setenv("CN_PDL", "0")                 # read by cn_gst_create
    nopdl = _full_run(hist_np, 0, N, H)
    monkeypatch.delenv("CN_PDL")
    for a, b in zip(whole, nopdl):
        assert torch.equal(a, b)
    k = _Handle(N, H, 5, _params())
    hist = _upload(hist_np)
    runs = []
    for _ in range(2):
        k.run(hist, 7)
        runs.append((k.buf("pred", device="cpu").raw.clone(), torch.from_numpy(k.rows()), k.pen.cpu()))
    k.close()
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_gst_stage_hook_rejects_unknown_names():
    k = _Handle(2, 3, 5, _params())
    with pytest.raises(RuntimeError, match="unknown buffer 'nope'"):
        k.buf("nope")
    with pytest.raises(RuntimeError, match="unknown stage 'obs.nope'"):
        k.capi.check(k.lib, k.lib.cn_internal_gst_stop_after(k.h, b"obs.nope"), "stop_after")
    k.close()
