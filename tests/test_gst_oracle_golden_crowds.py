"""Pins oracle/gst_ref.py (GST predictor + VecPretextNormalize processing, BASELINE config 3) on crowds other than the
shipped 20 humans -- 13 and 128 humans in the predictor, 10 + 3, 50 and 100 humans behind the wrapper -- against vectors
recorded from the UNMODIFIED reference (tools/make_golden_gst.py, opt-in modes).  Tolerances as in
test_gst_oracle_golden.py."""
import os

import numpy as np
import pytest

from oracle.gst_ref import PretextWrapperRef, gst_forward, load_params

GOLD = os.path.join(os.path.dirname(__file__), "golden")
IO = ["gst_io_h13.npz", "gst_io_h128.npz"]
ROLLOUTS = ["gst_rollout_h10_range3.npz", "gst_rollout_h50.npz", "gst_rollout_h100_x2.npz"]
KEYS = ("robot_node", "temporal_edges", "spatial_edges", "detected_human_num", "visible_masks")


@pytest.mark.parametrize("name", IO)
def test_gst_forward_matches_reference(name):
    p = load_params(os.path.join(GOLD, "gst_params.npz"))
    g = np.load(os.path.join(GOLD, name))
    out, mask = gst_forward(p, g["in_traj"], g["in_mask"].astype(np.float32))
    assert np.array_equal(mask.numpy(), g["out_mask"])
    np.testing.assert_allclose(out.numpy(), g["out_traj"], rtol=0, atol=2e-5)


@pytest.mark.parametrize("name", ROLLOUTS)
def test_wrapper_processing_matches_reference(name):
    p = load_params(os.path.join(GOLD, "gst_params.npz"))
    g = np.load(os.path.join(GOLD, name))
    meta = eval(str(g["meta"][0]))
    T1, N, H = g["raw_spatial_edges"].shape[:3]
    assert H == meta["human_num"] + meta["human_num_range"]          # rows = VecPretextNormalize.max_human_num
    w = PretextWrapperRef(p, N, H)
    for t in range(T1):
        O = {k: g["raw_" + k][t] for k in KEYS}
        rews = g["reward_env"][t - 1] if t > 0 else None
        obs, r, pen = w.process(O, rews)
        np.testing.assert_allclose(obs["spatial_edges"], g["fin_spatial_edges"][t], rtol=0, atol=2e-4, err_msg="t=%d" % t)
        if t > 0:
            np.testing.assert_allclose(r.reshape(N), g["reward"][t - 1], rtol=0, atol=1e-6)


def test_fixtures_cover_the_crowds():
    """The fixtures hold what the GPU tests rely on: (env, frame) groups wider than one and than three warps."""
    m = np.load(os.path.join(GOLD, "gst_io_h128.npz"))["in_mask"][..., 0]
    assert m.sum(1).max() > 96                                         # a frame with more than three warps of rows
    v = np.load(os.path.join(GOLD, "gst_rollout_h50.npz"))["raw_visible_masks"]
    assert v.sum(-1).max() > 32
