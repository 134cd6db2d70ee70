"""GPU: robot.visible = True (cn_config.robot_visible) in the CUDA step kernel.

  * golden replay against the unmodified reference (tools/make_golden.py) with the default settings, the pre-solve
    forced off and on, and every rejection-sampling search sent to the CTA-scope event kernel (CN_DEFER_TRIES=1);
  * the pre-solve (humans' solve of the next step on the side stream, reading the robot's final state) equals the
    in-step solve bit for bit over 260 randomised steps through episode ends;
  * at full size (4096 x 20), at the config-5 shape (100 humans, circle and arena x2) and at 128 human slots (127
    humans plus the robot: 128 ORCA lines per human), environments picked by rank offset match the host build of the
    step logic step for step;
  * the GST wrapper's environments equal a plain unsorted CrowdSimVarNum-v0 engine driven by the same actions;
  * the batched evaluation equals the sequential protocol, for a network policy and for the ORCA / social-force robot
    baselines among humans that see the robot."""
import os

import numpy as np
import pytest
import torch

from tests.golden_util import replay
from tests.harness_util import HarnessEnv
from tests.robot_policy_util import replay_robot
from tests.test_env_harness_robot_visible import VIS_CASES, VIS_ROBOT_CASES, load_vis_case

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

VARIANTS = [dict(), dict(CN_PRESOLVE="0"), dict(CN_PRESOLVE="1"), dict(CN_DEFER_TRIES="1")]


def _engine(**over):
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    return CudaCrowdVecEnv(device="cuda:0", **over)


def _np_obs(obs):
    return {k: v.cpu().numpy() for k, v in obs.items()}


def _step_fn(env):
    def step(a):
        obs, rew, done, info = env.step_device(torch.from_numpy(np.ascontiguousarray(a)).cuda())
        out = dict(reward=rew.cpu().numpy(), done=done.cpu().numpy(), info=info.cpu().numpy(),
                   info_aux=env._out["info_aux"].cpu().numpy())
        return _np_obs(obs), out
    return step


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: ",".join("%s=%s" % kv for kv in v.items()) or "default")
@pytest.mark.parametrize("name", VIS_CASES + VIS_ROBOT_CASES)
def test_cuda_robot_visible_matches_reference_golden(name, variant, monkeypatch):
    for k, v in variant.items():
        monkeypatch.setenv(k, v)
    g, case, over = load_vis_case(name)
    env = _engine(**over)
    check = replay_robot if "robot_policy" in case else replay
    bad = check(g, case, lambda: _np_obs(env.reset()), _step_fn(env), env.get_state)
    env.close()
    assert not bad, bad[:5]


STATE = ("hpx", "hpy", "hvx", "hvy", "hgx", "hgy", "rpx", "rpy", "vis", "sim_exists", "last_hvx", "last_hvy",
         "orca_nlines", "orca_fail", "mt_pos", "hn")


def test_presolve_equals_in_step_solve_with_robot_visible(monkeypatch):
    N, H, T = 256, 20, 260
    over = dict(num_envs=N, human_num=H, seed=3, const_vel=0, robot_visible=1, randomize_attributes=1,
                random_goal_changing=1)
    envs = []
    for ps in ("1", "0"):
        monkeypatch.setenv("CN_PRESOLVE", ps)
        envs.append(_engine(**over))
    on, off = envs
    o1, o0 = _np_obs(on.reset()), _np_obs(off.reset())
    rng = np.random.RandomState(4)
    ends = 0
    for t in range(T):
        for k in o1:
            assert np.array_equal(o1[k], o0[k]), (k, t)
        a = torch.from_numpy(rng.uniform(-1.2, 1.2, (N, 2)).astype(np.float32)).cuda()
        r1, r0 = on.step_device(a), off.step_device(a)
        for x, y in zip(r1[1:], r0[1:]):
            assert torch.equal(x, y), t
        ends += int(r1[2].sum())
        o1, o0 = _np_obs(r1[0]), _np_obs(r0[0])
        for k in STATE:
            assert np.array_equal(on.get_state(k), off.get_state(k)), (k, t)
    assert ends > 50          # the comparison crossed many episode installs
    on.close(); off.close()


def _lockstep_vs_harness(N, T, offsets, tol=1e-9, **over):
    """CUDA engine of N environments vs the host build run as single-environment shards at the given rank offsets;
    environments whose spawn search overflowed (the reference would spin there) are excluded."""
    env = _engine(num_envs=N, nenv_total=N, **over)
    hs = [HarnessEnv(num_envs=1, nenv_total=N, rank_offset=r, **over) for r in offsets]
    idx = np.array(offsets)
    H = env.human_num
    env.reset()
    for h in hs:
        h.reset()
    rng = np.random.RandomState(8)
    compared = 0
    for t in range(T):
        a = rng.uniform(-1.2, 1.2, (N, 2)).astype(np.float32)
        _, rew, done, info = env.step_device(torch.from_numpy(a).cuda())
        rew, done, info = rew.cpu().numpy(), done.cpu().numpy(), info.cpu().numpy()
        st = {k: env.get_state(k) for k in ("hpx", "hpy", "rpx", "rpy", "last_hvx", "last_hvy", "orca_nlines", "vis",
                                             "spawn_overflow")}
        for j, (h, e) in enumerate(zip(hs, idx)):
            _, out = h.step(a[e:e + 1])
            if st["spawn_overflow"][e] or h.get("spawn_overflow")[0]:
                continue
            compared += 1
            assert (done[e], info[e]) == (out["done"][0], out["info"][0]), (t, e)
            assert abs(rew[e] - out["reward"][0]) <= 1e-5, (t, e)
            sl = slice(e * H, (e + 1) * H)
            for k in ("last_hvx", "last_hvy", "orca_nlines", "vis"):
                assert np.array_equal(st[k][sl], h.get(k)), (k, t, e)
            for k in ("hpx", "hpy"):
                np.testing.assert_allclose(st[k][sl], h.get(k), rtol=0, atol=tol, err_msg="%s t=%d e=%d" % (k, t, e))
            for k in ("rpx", "rpy"):
                assert abs(st[k][e] - h.get(k)[0]) <= tol, (k, t, e)
    env.close()
    return compared


def test_full_size_robot_visible_matches_host_build():
    n = _lockstep_vs_harness(4096, 100, [0, 1, 517, 1024, 2047, 2048, 3333, 4095], human_num=20, const_vel=0,
                             robot_visible=1, randomize_attributes=1, random_goal_changing=1)
    assert n >= 700


def test_config5_shape_robot_visible_matches_host_build():
    n = _lockstep_vs_harness(4096, 100, [0, 3, 999, 1500, 2222, 3000, 4001, 4095], human_num=100, const_vel=0,
                             robot_visible=1, circle_radius=2 * 6 * 2 ** 0.5, arena_size=12.0)
    assert n >= 400


def test_128_slots_robot_visible_matches_host_build():
    """127 other humans plus the robot: up to 128 ORCA lines per human (the shared-memory line store plus its
    overflow rows, and linearProgram3 over all of them)."""
    n = _lockstep_vs_harness(64, 30, [0, 21, 42, 63], human_num=128, const_vel=0, robot_visible=1,
                             circle_radius=3 * 6 * 2 ** 0.5, arena_size=18.0)
    assert n >= 60


def test_gst_wrapper_env_state_equals_plain_unsorted_varnum_engine():
    from crowdnav_prediction_attngraph_b200.vec_env import CudaPretextVecEnv
    N, H, T = 64, 20, 120
    params = dict(np.load(os.path.join(GOLD, "gst_params.npz")))
    over = dict(num_envs=N, human_num=H, seed=31, robot_visible=1, randomize_attributes=1, random_goal_changing=1)
    gst = CudaPretextVecEnv(params, device="cuda:0", **over)
    plain = _engine(const_vel=0, sort_humans=0, **over)
    assert gst.cfgd["robot_visible"] == 1
    gst.reset()
    plain.reset()
    rng = np.random.RandomState(6)
    for t in range(T):
        a = torch.from_numpy(rng.uniform(-1, 1, (N, 2)).astype(np.float32)).cuda()
        _, _, d1, i1 = gst.step_device(a)
        o2, _, d2, i2 = plain.step_device(a)
        assert torch.equal(d1, d2) and torch.equal(i1, i2), t
        for k in STATE:
            assert np.array_equal(gst.get_state(k), plain.get_state(k)), (k, t)
    gst.close(); plain.close()


def _policy(dev):
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    from crowdnav_prediction_attngraph_b200.policy import Policy, make_reference_like_state_dict

    class Args(object):
        num_processes, seq_length, num_mini_batch = 1, 30, 2
    spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((20, 2)),
              'detected_human_num': Box((1,))}
    pol = Policy(spaces, Box((2,)), base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    pol.load_state_dict(make_reference_like_state_dict(2, seed=5), strict=False)
    return pol


@pytest.mark.parametrize("robot_policy,randomize", [(0, 0), (0, 1), (1, 0), (1, 1), (2, 0)])
def test_batched_evaluation_equals_sequential_with_robot_visible(robot_policy, randomize):
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    dev = torch.device("cuda:0")
    test_size = 9
    d = _capi.default_config_dict(num_envs=1, nenv_total=1, seed=425, human_num=20, const_vel=0, phase=2,
                                  test_size=test_size, robot_policy=robot_policy, robot_visible=1,
                                  randomize_attributes=randomize, random_goal_changing=randomize, time_limit=30.0)
    pol = _policy(dev) if robot_policy == 0 else None
    env = _engine(cfg=d)
    seq = evaluate(pol, env, 1, dev, test_size, None, None, None)
    env.close()
    bat = evaluate_batched(pol, None, "CrowdSimVarNum-v0", 425, test_size, dev, cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    for k in ("success_rate", "collision_rate", "timeout_rate", "collision_cases", "timeout_cases"):
        assert seq[k] == bat[k], k
    for k in ("intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k


def test_robot_visible_is_refused_for_crowdsimpred():
    from crowdnav_prediction_attngraph_b200 import _capi
    with pytest.raises(RuntimeError, match="CrowdSimVarNum-v0"):
        _engine(num_envs=4, const_vel=1, robot_visible=1)
    with pytest.raises(RuntimeError, match="robot_visible 2"):
        _engine(num_envs=4, const_vel=0, robot_visible=2)
    assert _capi.default_config_dict()["robot_visible"] == 0
