"""CPU: pins the GST predictor's stage reference (tests/gst_stages.py, used stage by stage by test_gpu_gst_stages.py)
against the padded fp32 oracle (oracle/gst_ref.py), the reference fixtures and the wrapper oracle, including the edge
inputs the compact layout treats specially: one human, nobody visible, everybody visible in all five frames."""
import os

import numpy as np
import pytest
import torch

from oracle.gst_ref import PretextWrapperRef, gst_forward, load_params
from tests.gst_stages import GstStages, Ring, compaction, final_rows, penalty, random_history, sort_keys

GOLD = os.path.join(os.path.dirname(__file__), "golden")
PARAMS = os.path.join(GOLD, "gst_params.npz")
FIXTURE_ATOL = 5e-5         # the GPU tests' tolerance on predicted positions (test_gpu_gst.py)
ORACLE_ATOL = 2e-5          # fp32 noise of the padded oracle after five recursive decoding steps


def _params():
    return dict(np.load(PARAMS))


def _frames(in_traj, in_mask):
    """fixture / oracle layout [N,H,5,2], [N,H,5(,1)] -> frames [5,N,H,2], [5,N,H]"""
    m = np.asarray(in_mask, np.float32).reshape(in_traj.shape[:3])
    return np.ascontiguousarray(in_traj.transpose(2, 0, 1, 3), np.float32), np.ascontiguousarray(m.transpose(2, 0, 1))


def _chain(in_traj, in_mask):
    N, H = in_traj.shape[:2]
    comp = compaction(*_frames(in_traj, in_mask))
    pred = GstStages(_params(), H).chain(comp).numpy()
    full = np.full((N * H, 5, 2), np.nan)
    full[comp["drow"]] = pred
    return comp, full.reshape(N, H, 5, 2)


def _oracle(in_traj, in_mask):
    out, mask = gst_forward(load_params(PARAMS), in_traj, np.asarray(in_mask, np.float32).reshape(in_traj.shape[:3] + (1,)))
    return out[..., :2].double().numpy(), mask[..., 0].numpy()


def _assert_matches_oracle(in_traj, in_mask):
    comp, pred = _chain(in_traj, in_mask)
    ref, fp = _oracle(in_traj, in_mask)
    N, H = fp.shape
    assert np.array_equal(comp["fp"].reshape(N, H), fp)
    ok = fp > 0
    assert np.isfinite(pred[ok]).all()
    np.testing.assert_allclose(pred[ok], ref[ok], rtol=0, atol=ORACLE_ATOL)
    return comp


@pytest.mark.parametrize("name", ["gst_io.npz", "gst_io_h13.npz", "gst_io_h128.npz"])
def test_chain_matches_fixture_and_oracle(name):
    g = np.load(os.path.join(GOLD, name))
    _, pred = _chain(g["in_traj"], g["in_mask"])
    ok = g["out_mask"][:, :, 0] > 0
    np.testing.assert_allclose(pred[ok], g["out_traj"][:, :, :, :2][ok], rtol=0, atol=FIXTURE_ATOL)
    _assert_matches_oracle(g["in_traj"], g["in_mask"])


def _walk(N, H, vis, seed):
    rng = np.random.RandomState(seed)
    traj = (rng.uniform(-5, 5, (N, H, 1, 2)) + np.cumsum(rng.normal(0, 0.2, (N, H, 5, 2)), 2)).astype(np.float32)
    return traj, vis


@pytest.mark.parametrize("N,H", [(4, 1), (3, 7), (2, 33)])
@pytest.mark.parametrize("pattern", ["random", "nobody", "everybody"])
def test_chain_matches_oracle_edge_inputs(N, H, pattern):
    rng = np.random.RandomState(N * 100 + H)
    vis = {"random": rng.rand(N, H, 5) < 0.6, "nobody": np.zeros((N, H, 5), bool),
           "everybody": np.ones((N, H, 5), bool)}[pattern]
    traj, vis = _walk(N, H, vis, N + H)
    comp = _assert_matches_oracle(traj, vis)
    if pattern == "nobody":
        assert comp["counts"].tolist() == [0, 0]
    if pattern == "everybody":
        assert comp["counts"].tolist() == [N * H * 5, N * H]
        assert (comp["gcount"] == H).all()                     # no masked keys anywhere


def test_attention_masked_term_equals_padded_softmax():
    """The explicit (H - n) * exp(q . b_k - max) term equals the padded soft-max over all H keys of mha.py."""
    H = 9
    st = GstStages(_params(), H)
    rng = np.random.RandomState(3)
    n = np.array([0, 1, 4, 9, 2])
    start = np.concatenate([[0], np.cumsum(n)])
    qkv = torch.tensor(rng.normal(0, 1.5, (start[-1], 192)))
    got, vmax = st.attention(qkv, start)
    for g in range(len(n)):
        rows = qkv[start[g]:start[g + 1]]
        pad = st.bin.expand(H, 192).clone()                    # a masked row's Q|K|V is the bias
        pad[:n[g]] = rows
        q = pad[:, :64].reshape(H, 8, 8).transpose(0, 1) * 8 ** -0.5
        k = pad[:, 64:128].reshape(H, 8, 8).transpose(0, 1)
        v = pad[:, 128:].reshape(H, 8, 8).transpose(0, 1)
        w = torch.softmax(q @ k.transpose(-1, -2), -1)
        mask = (torch.arange(H) < n[g]).double()
        w = w * mask
        w = w / (w.sum(-1, keepdim=True) + 1e-10)
        ref = (w @ v).transpose(0, 1).reshape(H, 64)[:n[g]]
        assert torch.allclose(got[start[g]:start[g + 1]], ref, rtol=0, atol=1e-13)
        if n[g]:
            assert torch.equal(vmax[start[g]], v[:, :n[g]].abs().amax(dim=(1, 2)).repeat_interleave(8))


def test_ring_compaction_and_tail_match_wrapper_oracle():
    """Ring + compaction + chain + final_rows / penalty over 7 wrapper steps equal PretextWrapperRef.process (the
    frames the ring hands over, the penalty and the distance-sorted spatial_edges rows)."""
    N, H, P = 16, 6, 5
    w = PretextWrapperRef(load_params(PARAMS), N, H)
    ring = Ring(N, H)
    st = GstStages(_params(), H)
    hits = 0
    for s, (robot, sp2, vis) in enumerate(random_history(N, H, 7, 0.7, 11)):
        pos, m = ring.step(robot, sp2, vis)
        sp = np.tile(sp2, (1, 1, 6))                           # the raw observation repeats the position
        O = dict(robot_node=robot.reshape(N, 1, 7), spatial_edges=sp, visible_masks=vis.astype(bool),
                 temporal_edges=np.zeros((N, 1, 2), np.float32), detected_human_num=np.ones((N, 1), np.float32))
        obs, _, pen_ref = w.process(O)
        assert np.array_equal(np.stack(w.traj), pos) and np.array_equal(np.stack(w.mask)[..., 0], m)
        comp = compaction(pos, m)
        pred = np.zeros((N * H, 5, 2))
        pred[comp["drow"]] = st.chain(comp).numpy()
        fp = comp["fp"].reshape(N, H)
        pen, dist, counted = penalty(robot.astype(np.float64), fp, pred.reshape(N, H, 5, 2), P, 0.6)
        near = (np.abs(dist - 0.6) < 1e-4) & counted
        keep = ~near.any((1, 2))
        np.testing.assert_array_equal(pen[keep], pen_ref[keep])
        hits += int((pen < 0).sum())
        rows = final_rows(robot.astype(np.float64), sp2.astype(np.float64), fp, pred.reshape(N, H, 5, 2), P)
        order = np.argsort(sort_keys(sp2), 1, kind="stable")
        rows = np.take_along_axis(rows, order[..., None], 1)
        np.testing.assert_allclose(rows, obs["spatial_edges"], rtol=0, atol=ORACLE_ATOL, err_msg="step %d" % s)
    assert hits > 0                                            # the penalty path ran
