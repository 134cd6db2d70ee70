"""GPU: BASELINE config 3 (row a16) -- the GST predictor + VecPretextNormalize step (cn_gst_step) against vectors recorded
from the unmodified reference (tools/make_golden_gst.py) and against the oracle in lock-step."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


class _Gst(object):
    def __init__(self, N, H):
        from crowdnav_prediction_attngraph_b200 import _capi
        self.capi, self.lib = _capi, _capi.load_library()
        self.h = C.c_void_p()
        _capi.check(self.lib, self.lib.cn_gst_create(N, H, 5, 0.3, 0.3, -20.0, 0, C.byref(self.h)), "create")
        p = np.load(os.path.join(GOLD, "gst_params.npz"))
        for k in p.files:
            a = np.ascontiguousarray(p[k], dtype=np.float32)
            _capi.check(self.lib, self.lib.cn_gst_set_param(self.h, k.encode(), a.ctypes.data, a.size), k)
        _capi.check(self.lib, self.lib.cn_gst_finalize(self.h), "finalize")
        _capi.check(self.lib, self.lib.cn_gst_reset(self.h, None), "reset")
        self.N, self.H = N, H
        self.out = torch.zeros(N, H, 12, device="cuda")
        self.pen = torch.zeros(N, device="cuda")

    def step(self, robot, sp2, vis, reward=None):
        r = torch.tensor(robot, dtype=torch.float32, device="cuda").contiguous()
        s = torch.tensor(sp2, dtype=torch.float32, device="cuda").contiguous()
        v = torch.tensor(vis, dtype=torch.uint8, device="cuda").contiguous()
        rw = None if reward is None else torch.tensor(reward, dtype=torch.float32, device="cuda").contiguous()
        self.capi.check(self.lib, self.lib.cn_gst_step(self.h, r.data_ptr(), s.data_ptr(), v.data_ptr(),
                                                        rw.data_ptr() if rw is not None else None, self.pen.data_ptr(),
                                                        self.out.data_ptr(), None), "step")
        torch.cuda.synchronize()
        return self.out.cpu().numpy(), self.pen.cpu().numpy(), None if rw is None else rw.cpu().numpy()

    def close(self):
        self.lib.cn_gst_destroy(self.h)


def _unsort(sp2, rows):
    """rows are sorted by the float32 norm of the current relative position (ties by index): undo it."""
    key = np.sqrt((sp2.astype(np.float32) ** 2).sum(-1, dtype=np.float32))
    out = np.zeros_like(rows)
    for n in range(sp2.shape[0]):
        order = np.argsort(key[n], kind="stable")
        out[n, order] = rows[n]
    return out


def test_gst_kernel_matches_reference_predictor():
    g = np.load(os.path.join(GOLD, "gst_io.npz"))
    N, H = g["in_traj"].shape[:2]
    k = _Gst(N, H)
    robot = np.zeros((N, 7), np.float32)
    for t in range(5):
        rows, pen, _ = k.step(robot, g["in_traj"][:, :, t], g["in_mask"][:, :, t, 0])
    rows = _unsort(g["in_traj"][:, :, 4], rows)
    ok = g["out_mask"][:, :, 0] > 0
    pred = rows[:, :, 2:].reshape(N, H, 5, 2)
    np.testing.assert_allclose(pred[ok], g["out_traj"][:, :, :, :2][ok], rtol=0, atol=5e-5)
    # humans that are not predicted keep the tiled current position
    cur = np.tile(g["in_traj"][:, :, 4], (1, 1, 5)).reshape(N, H, 5, 2)
    np.testing.assert_allclose(pred[~ok], cur[~ok], rtol=0, atol=0)
    k.close()


def test_pretext_kernel_matches_reference_wrapper_rollout():
    g = np.load(os.path.join(GOLD, "gst_rollout.npz"))
    T1, N, H = g["raw_spatial_edges"].shape[:3]
    k = _Gst(N, H)
    for t in range(T1):
        raw_sp = g["raw_spatial_edges"][t][:, :, :2]
        rew = g["reward_env"][t - 1].astype(np.float32) if t > 0 else None
        rows, pen, rw = k.step(g["raw_robot_node"][t].reshape(N, 7), raw_sp, g["raw_visible_masks"][t], rew)
        np.testing.assert_allclose(rows, g["fin_spatial_edges"][t], rtol=0, atol=3e-4, err_msg="t=%d" % t)
        if t > 0:
            np.testing.assert_allclose(rw, g["reward"][t - 1], rtol=0, atol=1e-5)
    k.close()


def test_config3_vec_env_matches_oracle_lockstep():
    from crowdnav_prediction_attngraph_b200.vec_env import CudaPretextVecEnv
    from oracle.crowd_env import EnvConfig, OracleVecEnv
    from oracle.gst_ref import PretextWrapperRef, load_params
    N, H, T = 4, 20, 60
    params = dict(np.load(os.path.join(GOLD, "gst_params.npz")))
    env = CudaPretextVecEnv(params, num_envs=N, human_num=H, seed=31, device="cuda:0")
    orc = OracleVecEnv(EnvConfig(human_num=H, predict_method="none", sort_humans=False), N, seed=31)
    w = PretextWrapperRef(load_params(os.path.join(GOLD, "gst_params.npz")), N, H)

    def raw(o):
        d = dict(o)
        d["spatial_edges"] = np.tile(o["spatial_edges"], (1, 1, 6))
        return d

    obs = env.reset()
    ref, _, _ = w.process(raw(orc.reset()))
    rng = np.random.RandomState(2)
    for t in range(T):
        np.testing.assert_allclose(obs["spatial_edges"].cpu().numpy(), ref["spatial_edges"], rtol=0, atol=5e-4, err_msg="t=%d" % t)
        assert np.array_equal(obs["detected_human_num"].cpu().numpy().reshape(N), ref["detected_human_num"].reshape(N))
        a = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
        obs, rew, done, infos = env.step(torch.from_numpy(a).cuda())
        o2, r2, d2, _ = orc.step(a)
        ref, r2p, _ = w.process(raw(o2), r2)
        assert np.array_equal(done, d2)
        np.testing.assert_allclose(rew.numpy().reshape(N), r2p.reshape(N), rtol=0, atol=1e-4)
    env.close()
