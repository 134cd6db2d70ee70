"""GPU: BASELINE config 3's GST predictor + VecPretextNormalize step (cn_gst_step) at crowds other than the shipped 20
humans: every predictor group size up to 128 humans, humans joining and leaving (human_num_range), the dense 100-human
crowd.  Against vectors recorded from the unmodified reference (tools/make_golden_gst.py, opt-in modes) with the
tolerances of test_gpu_gst.py, and against the oracle in lock-step."""
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from tests.test_gpu_gst import _Gst, _unsort

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
X2 = dict(circle_radius=2 * 6 * 2 ** 0.5, arena_size=12.0)       # BASELINE config 5's crowd: circle and arena x2


@pytest.mark.parametrize("name", ["gst_io_h13.npz", "gst_io_h128.npz"])
def test_gst_kernel_matches_reference_predictor(name):
    g = np.load(os.path.join(GOLD, name))
    N, H = g["in_traj"].shape[:2]
    k = _Gst(N, H)
    robot = np.zeros((N, 7), np.float32)
    for t in range(5):
        rows, pen, _ = k.step(robot, g["in_traj"][:, :, t], g["in_mask"][:, :, t, 0])
    rows = _unsort(g["in_traj"][:, :, 4], rows)
    ok = g["out_mask"][:, :, 0] > 0
    pred = rows[:, :, 2:].reshape(N, H, 5, 2)
    np.testing.assert_allclose(pred[ok], g["out_traj"][:, :, :, :2][ok], rtol=0, atol=5e-5)
    cur = np.tile(g["in_traj"][:, :, 4], (1, 1, 5)).reshape(N, H, 5, 2)
    np.testing.assert_allclose(pred[~ok], cur[~ok], rtol=0, atol=0)
    k.close()


@pytest.mark.parametrize("name", ["gst_rollout_h10_range3.npz", "gst_rollout_h50.npz", "gst_rollout_h100_x2.npz"])
def test_pretext_kernel_matches_reference_wrapper_rollout(name):
    g = np.load(os.path.join(GOLD, name))
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


LOCKSTEP = {
    # name: (envs, human_num, human_num_range, steps, phase, extra config)
    "h10_range3": (3, 10, 3, 60, "train", {}),
    "h50": (2, 50, 0, 40, "train", {}),
    "h100_x2": (2, 100, 0, 30, "train", X2),
    "h50_test_1env": (1, 50, 0, 40, "test", {}),
}


@pytest.mark.parametrize("case", sorted(LOCKSTEP))
def test_vec_env_matches_oracle_lockstep(case):
    from crowdnav_prediction_attngraph_b200.vec_env import CudaPretextVecEnv
    from oracle.crowd_env import EnvConfig, OracleVecEnv
    from oracle.gst_ref import PretextWrapperRef, load_params
    N, H, rng_h, T, phase, kw = LOCKSTEP[case]
    params = dict(np.load(os.path.join(GOLD, "gst_params.npz")))
    env = CudaPretextVecEnv(params, num_envs=N, nenv_total=N, human_num=H, human_num_range=rng_h, seed=31, device="cuda:0",
                            phase=2 if phase == "test" else 0, **kw)
    assert env.human_num == H + rng_h
    orc = OracleVecEnv(EnvConfig(human_num=H, human_num_range=rng_h, predict_method="none", sort_humans=False, **kw), N,
                       seed=31, phase=phase)
    w = PretextWrapperRef(load_params(os.path.join(GOLD, "gst_params.npz")), N, H + rng_h)

    def raw(o):
        d = dict(o)
        d["spatial_edges"] = np.tile(o["spatial_edges"], (1, 1, 6))
        return d

    obs = env.reset()
    ref, _, _ = w.process(raw(orc.reset()))
    rng = np.random.RandomState(2)
    seen = 0
    for t in range(T):
        np.testing.assert_allclose(obs["spatial_edges"].cpu().numpy(), ref["spatial_edges"], rtol=0, atol=5e-4, err_msg="t=%d" % t)
        assert np.array_equal(obs["detected_human_num"].cpu().numpy().reshape(N), ref["detected_human_num"].reshape(N))
        seen = max(seen, int(ref["detected_human_num"].max()))
        a = rng.uniform(-1, 1, (N, 2)).astype(np.float32)
        obs, rew, done, infos = env.step(torch.from_numpy(a).cuda())
        o2, r2, d2, _ = orc.step(a)
        ref, r2p, _ = w.process(raw(o2), r2)
        assert np.array_equal(done, d2)
        np.testing.assert_allclose(rew.numpy().reshape(N), r2p.reshape(N), rtol=0, atol=1e-4)
    assert seen > 0
    env.close()


def _reference_like_config(model_dir, human_num):
    """The fields make_vec_envs and Policy read, with the values of the reference's crowd_nav/configs/config.py for the
    GST-wrapper model (robot.policy 'selfAttn_merge_srnn', sim.predict_method 'inferred', env.use_wrapper)."""
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics="holonomic"),
        robot=ns(visible=False, policy="selfAttn_merge_srnn", radius=0.3, v_pref=1, FOV=2, sensor_range=5),
        humans=ns(policy="orca", radius=0.3, v_pref=1, FOV=2., random_goal_changing=True, end_goal_changing=True,
                  goal_change_chance=0.5),
        sim=ns(predict_method="inferred", human_num=human_num, human_num_range=0, predict_steps=5,
               circle_radius=6 * np.sqrt(2), arena_size=6),
        env=ns(randomize_attributes=True, time_step=0.25, time_limit=50, val_size=100, test_size=500, use_wrapper=True),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25), args=ns(sort_humans=True),
        pred=ns(model_dir=model_dir))


def test_compat_make_vec_envs_gst_h50_stepped_by_policy(tmp_path):
    """The reference-facing path: rl.networks.envs.make_vec_envs('CrowdSimPredRealGST-v0', ...) of the alias packages
    loads the predictor from config.pred.model_dir/checkpoint/epoch_100.pt, as the reference's wrapper does, and
    rl.networks.model.Policy steps it at 50 humans."""
    from crowdnav_prediction_attngraph_b200.compat.rl.networks.envs import make_vec_envs
    from crowdnav_prediction_attngraph_b200.compat.rl.networks.model import Policy
    os.makedirs(tmp_path / "checkpoint")
    p = np.load(os.path.join(GOLD, "gst_params.npz"))
    torch.save({"model_state_dict": {k: torch.tensor(p[k]) for k in p.files}}, str(tmp_path / "checkpoint" / "epoch_100.pt"))
    N, H = 4, 50
    cfg = _reference_like_config(str(tmp_path), H)
    envs = make_vec_envs("CrowdSimPredRealGST-v0", 425, N, 0.99, None, "cuda:0", False, config=cfg)
    assert envs.observation_space.spaces["spatial_edges"].shape == (H, 12)

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, 30, 2
    torch.manual_seed(0)
    policy = Policy(envs.observation_space.spaces, envs.action_space, base_kwargs=Args(), base="selfAttn_merge_srnn").to("cuda:0")
    obs = envs.reset()
    h = {"human_node_rnn": torch.zeros(N, 1, 128, device="cuda:0")}
    masks = torch.ones(N, 1, device="cuda:0")
    for _ in range(5):
        with torch.no_grad():
            value, action, logp, h = policy.act(obs, h, masks)
        obs, rew, done, infos = envs.step(action)
        assert obs["spatial_edges"].shape == (N, H, 12) and torch.isfinite(obs["spatial_edges"]).all()
        assert np.isfinite(np.asarray(rew)).all() and len(infos) == N
        masks = torch.tensor([[0.0] if d else [1.0] for d in done], device="cuda:0")
    envs.close()


def test_gst_create_accepts_up_to_128_humans():
    from crowdnav_prediction_attngraph_b200 import _capi
    lib = _capi.load_library()
    for H in (1, 5, 33, 128):
        h = C.c_void_p()
        _capi.check(lib, lib.cn_gst_create(2, H, 5, 0.3, 0.3, -20.0, 0, C.byref(h)), "create H=%d" % H)
        lib.cn_gst_destroy(h)
    h = C.c_void_p()
    assert lib.cn_gst_create(2, 129, 5, 0.3, 0.3, -20.0, 0, C.byref(h)) != 0
    assert not h.value
    assert b"human_num <= 128" in lib.cn_last_error()
