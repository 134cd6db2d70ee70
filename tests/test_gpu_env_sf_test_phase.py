"""GPU: social-force humans (humans.policy = 'social_force') in phase 'test' in the CUDA step kernel, whose ground-truth
look-ahead runs SOCIAL_FORCE.predict on the humans only, fp64 (cn_sf_lookahead).

  * golden replay against the unmodified reference (tools/make_golden.py) with the default settings, without the side
    stream, and with every rejection-sampling search sent to the CTA-scope event kernel (CN_DEFER_TRIES=1);
  * over 220 steps through episode ends, at 20, 50 and 100 humans (the three MAXH instantiations of the step kernel)
    and at 128 slots with the robot visible, environments picked by rank offset match the host build step for step;
  * the batched evaluation equals the sequential protocol, for a network policy and the two robot baselines;
  * the 500-case evaluation of the ORCA and social-force robots among social-force humans reproduces the recorded
    reference run (tests/golden/eval_baselines_sf_humans.npz, tools/make_golden_eval_baselines.py --humans social_force);
  * the reference's test.py flow (make_vec_envs with one environment, then evaluate) runs all 500 cases."""
import os
import types

import numpy as np
import pytest
import torch

from tests.golden_util import replay
from tests.harness_util import HarnessEnv
from tests.robot_policy_util import replay_robot
from tests.test_env_harness_sf_test_phase import SF_TEST_CASES, SF_TEST_ROBOT_CASES, load_sf_test_case
from tests.test_gpu_env_robot_visible import _np_obs, _policy, _step_fn

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

VARIANTS = [dict(), dict(CN_NO_SIDE_STREAM="1"), dict(CN_DEFER_TRIES="1")]


def _engine(**over):
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    return CudaCrowdVecEnv(device="cuda:0", **over)


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: ",".join("%s=%s" % kv for kv in v.items()) or "default")
@pytest.mark.parametrize("name", SF_TEST_CASES + SF_TEST_ROBOT_CASES)
def test_cuda_sf_test_phase_matches_reference_golden(name, variant, monkeypatch):
    for k, v in variant.items():
        monkeypatch.setenv(k, v)
    g, case, over = load_sf_test_case(name)
    env = _engine(**over)
    check = replay_robot if "robot_policy" in case else replay
    bad = check(g, case, lambda: _np_obs(env.reset()), _step_fn(env), env.get_state)
    env.close()
    assert not bad, bad[:5]


SF_TEST = dict(const_vel=0, human_policy=1, phase=2, randomize_attributes=1, random_goal_changing=1)


def _lockstep_vs_harness(N, T, offsets, tol=1e-9, **over):
    """CUDA engine of N environments vs the host build run as single-environment shards at the given rank offsets;
    environments whose spawn search overflowed (the reference would spin there) are excluded.  Done, info, the live
    count, line counts and visibility are exact, reward and Danger.min_dist within 1e-5 / 1e-6, positions within `tol`.
    The humans' fp32 velocities are held to 10 * tol plus one fp32 ulp rather than bit for bit: they narrow the fp64
    social-force velocity, whose push terms call exp() and whose FOV test calls atan2 / cos / sin / acos, and CUDA's fp64
    versions and glibc's differ in the last bit now and then (the difference replay_robot allows for the social-force
    robot).  Those last bits stay in the fp64 state and grow slowly through the crowd's interactions.  Measured on an
    H100: the first difference at 50 humans was t = 216, env 1023, one fp32 ulp of last_hvy; at 128 slots t = 178,
    env 42, last_hvx 4.473029e-06 against 4.473012e-06 (a velocity near zero, 1.7e-11 apart), with done, info, reward
    and positions agreeing; in that dense crowd the positions then drifted to 1.09e-9 apart at t = 186 (`tol` there).
    Returns (compared environment-steps, velocities that were not bit for bit equal)."""
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    env = CudaCrowdVecEnv(device="cuda:0", num_envs=N, nenv_total=N, **over)
    hs = [HarnessEnv(num_envs=1, nenv_total=N, rank_offset=r, **over) for r in offsets]
    H = env.human_num
    env.reset()
    for h in hs:
        h.reset()
    rng = np.random.RandomState(8)
    compared = ulp = 0
    for t in range(T):
        a = rng.uniform(-1.2, 1.2, (N, 2)).astype(np.float32)
        _, rew, done, info = env.step_device(torch.from_numpy(a).cuda())
        rew, done, info = rew.cpu().numpy(), done.cpu().numpy(), info.cpu().numpy()
        aux = env._out["info_aux"].cpu().numpy()
        st = {k: env.get_state(k) for k in ("hpx", "hpy", "rpx", "rpy", "last_hvx", "last_hvy", "orca_nlines", "vis",
                                             "hn", "spawn_overflow")}
        for h, e in zip(hs, offsets):
            _, out = h.step(a[e:e + 1])
            if st["spawn_overflow"][e] or h.get("spawn_overflow")[0]:
                continue
            compared += 1
            assert (done[e], info[e]) == (out["done"][0], out["info"][0]), (t, e)
            assert abs(rew[e] - out["reward"][0]) <= 1e-5, (t, e)
            assert abs(aux[e] - out["info_aux"][0]) <= 1e-6, (t, e)
            assert st["hn"][e] == h.get("hn")[0], (t, e)
            sl = slice(e * H, (e + 1) * H)
            for k in ("orca_nlines", "vis"):
                assert np.array_equal(st[k][sl], h.get(k)), (k, t, e)
            for k in ("last_hvx", "last_hvy"):
                x, y = st[k][sl], h.get(k)
                d = x != y
                assert np.array_equal(np.isnan(x), np.isnan(y)), (k, t, e)
                d &= ~np.isnan(y)
                assert np.all(np.abs(x[d] - y[d]) <= 10 * tol + np.spacing(np.abs(y[d]))), (k, t, e, x[d], y[d])
                ulp += int(d.sum())
            for k in ("hpx", "hpy"):
                np.testing.assert_allclose(st[k][sl], h.get(k), rtol=0, atol=tol, err_msg="%s t=%d e=%d" % (k, t, e))
            for k in ("rpx", "rpy"):
                assert abs(st[k][e] - h.get(k)[0]) <= tol, (k, t, e)
    env.close()
    print("compared", compared, "velocities not bit for bit equal", ulp)
    return compared, ulp


def test_sf_test_phase_h20_matches_host_build():
    n, _ = _lockstep_vs_harness(4096, 220, [0, 1, 517, 1024, 2047, 2048, 3333, 4095], human_num=20, **SF_TEST)
    assert n >= 1700


def test_sf_test_phase_h50_matches_host_build():
    n, _ = _lockstep_vs_harness(1024, 220, [0, 5, 300, 511, 512, 800, 1023], human_num=50,
                                circle_radius=1.5 * 6 * 2 ** 0.5, arena_size=9.0, **SF_TEST)
    assert n >= 1500


def test_sf_test_phase_h100_matches_host_build():
    n, _ = _lockstep_vs_harness(1024, 220, [0, 3, 999, 400, 1023], human_num=100, circle_radius=2 * 6 * 2 ** 0.5,
                                arena_size=12.0, **SF_TEST)
    assert n >= 1000


def test_sf_test_phase_128_slots_robot_visible_matches_host_build():
    # 128 humans in a crowd this dense amplify the last-bit exp() differences (see _lockstep_vs_harness): 1.09e-9 at
    # t = 186 on an H100; 1e-6 still separates them from any difference in the arithmetic, which shows at 1e-2 and up
    n, _ = _lockstep_vs_harness(64, 220, [0, 21, 42, 63], tol=1e-6, human_num=128, robot_visible=1,
                                circle_radius=3 * 6 * 2 ** 0.5, arena_size=18.0, **SF_TEST)
    assert n >= 800


def test_sf_test_phase_humans_joining_and_leaving_matches_host_build():
    n, _ = _lockstep_vs_harness(512, 220, [0, 7, 255, 511], human_num=18, human_num_range=4, **SF_TEST)
    assert n >= 800


@pytest.mark.parametrize("robot_policy,robot_visible", [(0, 0), (0, 1), (1, 0), (2, 0)])
def test_batched_evaluation_equals_sequential_with_sf_humans(robot_policy, robot_visible):
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    dev = torch.device("cuda:0")
    test_size = 9
    d = _capi.default_config_dict(num_envs=1, nenv_total=1, seed=425, human_num=20, const_vel=0, phase=2,
                                  test_size=test_size, human_policy=1, robot_policy=robot_policy,
                                  robot_visible=robot_visible, time_limit=30.0)
    pol = _policy(dev) if robot_policy == 0 else None
    env = _engine(cfg=d)
    seq = evaluate(pol, env, 1, dev, test_size, None, None, None)
    env.close()
    bat = evaluate_batched(pol, None, "CrowdSimVarNum-v0", 425, test_size, dev, cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    assert seq["case_code"] == bat["case_code"]
    assert seq["case_nav_time"] == bat["case_nav_time"]
    assert seq["case_path_len"] == pytest.approx(bat["case_path_len"], rel=0, abs=1e-12)
    for k in ("intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k


@pytest.mark.parametrize("name,robot_policy", [("ORCA_no_rand", 1), ("SF_no_rand", 2)])
def test_500_case_baseline_evaluation_among_sf_humans_reproduces_reference_run(name, robot_policy):
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate_batched
    g = np.load(os.path.join(GOLD, "eval_baselines_sf_humans.npz"))
    d = _capi.default_config_dict(num_envs=500, nenv_total=1, seed=425, human_num=20, const_vel=0, phase=2,
                                  test_size=500, human_policy=1, robot_policy=robot_policy)
    out = evaluate_batched(None, None, "CrowdSimVarNum-v0", 425, 500, torch.device("cuda:0"), cfg_dict=d)
    assert np.array_equal(out["case_code"], g[name + "_code"])
    assert np.array_equal(out["case_nav_time"], g[name + "_nav_time"])
    np.testing.assert_allclose(out["case_path_len"], g[name + "_path_len"], rtol=0, atol=1e-4)
    assert np.array_equal(out["case_too_close"], g[name + "_too_close"])
    mins = np.concatenate([np.asarray(m, np.float64) for m in out["case_min_dist"]] or [np.zeros(0)])
    np.testing.assert_allclose(mins, g[name + "_min_dist"], rtol=0, atol=1e-6)
    assert (g[name + "_too_close"] > 0).any()           # the 'future' danger zone fired


def _reference_config():
    """The fields make_vec_envs reads from crowd_nav/configs/config.py, at its defaults, with social-force humans."""
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics="holonomic"),
        robot=ns(visible=False, policy="selfAttn_merge_srnn", radius=0.3, v_pref=1, FOV=2, sensor_range=5),
        humans=ns(policy="social_force", radius=0.3, v_pref=1, FOV=2., random_goal_changing=False,
                  end_goal_changing=True, goal_change_chance=0.5),
        sim=ns(predict_method="none", human_num=20, human_num_range=0, predict_steps=5, circle_radius=6 * np.sqrt(2),
               arena_size=6),
        env=ns(randomize_attributes=False, time_step=0.25, time_limit=50, val_size=100, test_size=500),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25), args=ns(sort_humans=True))


def test_reference_test_py_flow_with_sf_humans_runs_500_cases():
    """test.py: make_vec_envs(num_processes=1) -> phase 'test' (rl/networks/envs.py:55-58), then evaluate() over
    test_size cases; the batched evaluation of the same configuration reports the same cases."""
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    from crowdnav_prediction_attngraph_b200.vec_env import make_vec_envs
    dev = torch.device("cuda:0")
    config = _reference_config()
    envs = make_vec_envs("CrowdSimVarNum-v0", 425, 1, 0.99, None, dev, allow_early_resets=True, config=config)
    assert (envs.cfgd["human_policy"], envs.cfgd["phase"]) == (1, 2)
    pol = _policy(dev)
    seq = evaluate(pol, envs, 1, dev, 500, None, config, None)
    envs.close()
    assert len(seq["case_code"]) == 500
    assert abs(seq["success_rate"] + seq["collision_rate"] + seq["timeout_rate"] - 1.0) < 1e-12
    bat = evaluate_batched(pol, None, "CrowdSimVarNum-v0", 425, 500, dev, cfg_dict=dict(envs.cfgd))
    assert seq["case_code"] == bat["case_code"]
    assert seq["case_nav_time"] == bat["case_nav_time"]
