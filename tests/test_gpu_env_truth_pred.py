"""GPU: CrowdSimPred-v0 with sim.predict_method = 'truth' in the CUDA step kernel (the TRUTH instantiations of
cn_env_step_kernel): every observation runs the ground-truth look-ahead and observes its kept rows.

  * golden replay against the unmodified reference (tools/make_golden.py) with the default settings, without the side
    stream, and with every rejection-sampling search sent to the CTA-scope event kernel (CN_DEFER_TRIES=1), including
    the future-collision penalty the next step's reward reads against the trajectory the reference stored;
  * over 220 steps through episode ends, environments picked by rank offset match the host build
    (tests/cpu_harness/truth_harness.cpp) step for step: 4096 x 20 humans, 50 and 100 humans (the three MAXH
    instantiations), 128 slots with the robot visible, humans joining and leaving, phase 'test', social-force humans;
  * the batched evaluation equals the sequential protocol;
  * a device-resident rollout of the attention-graph policy and one PPO.update give finite results;
  * a reference Config builds through make_vec_envs, steps and evaluates; the ORCA robot on CrowdSimPred-v0 is refused."""
import types

import numpy as np
import pytest
import torch

from tests.golden_util import replay
from tests.test_env_harness_truth_pred import (TRUTH_CASES, FinishedEpisodeDiagnosticsMasked, TruthHarnessEnv,
                                               future_penalty, load_truth_case, recorded_trajectories)
from tests.test_gpu_env_robot_visible import _np_obs, _step_fn

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

VARIANTS = [dict(), dict(CN_NO_SIDE_STREAM="1"), dict(CN_DEFER_TRIES="1")]


def _engine(**over):
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    return CudaCrowdVecEnv(device="cuda:0", **over)


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: ",".join("%s=%s" % kv for kv in v.items()) or "default")
@pytest.mark.parametrize("name", TRUTH_CASES)
def test_cuda_truth_matches_reference_golden(name, variant, monkeypatch):
    for k, v in variant.items():
        monkeypatch.setenv(k, v)
    g, case, over = load_truth_case(name)
    env = _engine(**over)
    trajs = recorded_trajectories(g)
    pen_bad, t_box = [], [0]

    def check_pen(t):
        if t in trajs:
            rob = np.stack([env.get_state("rpx"), env.get_state("rpy")], -1)
            pen = env.get_state("fut_pen")
            for k in range(env.num_envs):
                want = future_penalty(trajs[t][k], rob[k])
                if abs(pen[k] - want) > 1e-9:
                    pen_bad.append((t, k, pen[k], want))

    def reset():
        ob = _np_obs(env.reset())
        check_pen(0)
        return ob

    step = _step_fn(env)

    def step_checked(a):
        out = step(a)
        t_box[0] += 1
        check_pen(t_box[0])
        return out

    bad = replay(FinishedEpisodeDiagnosticsMasked(g), case, reset, step_checked, env.get_state)
    env.close()
    assert not bad, bad[:5]
    assert not pen_bad, pen_bad[:5]


TRUTH = dict(const_vel=2, randomize_attributes=1, random_goal_changing=1)


def _lockstep_vs_harness(N, T, offsets, tol=1e-9, **over):
    """CUDA engine of N environments vs the host build run as single-environment shards at the given rank offsets;
    environments whose spawn search overflowed (the reference would spin there) are excluded.  Done, info, the live
    count, line counts, visibility and simulator existence are exact, reward and Danger.min_dist within 1e-5 / 1e-6,
    observations within 1e-5 (fp32 of fp64 differences), the stored future penalty and positions within `tol`.  ORCA
    velocities are bit for bit; social-force ones within 10 * tol plus one fp32 ulp (CUDA's fp64 exp / atan2 and
    glibc's differ in the last bit now and then, see tests/test_gpu_env_sf_test_phase.py).  Returns the compared
    environment-steps."""
    env = _engine(num_envs=N, nenv_total=N, **over)
    hs = [TruthHarnessEnv(num_envs=1, nenv_total=N, rank_offset=r, **over) for r in offsets]
    H = env.human_num
    sf = over.get("human_policy", 0) == 1
    ob = _np_obs(env.reset())
    hob = [h.reset() for h in hs]
    rng = np.random.RandomState(8)
    compared = 0
    for t in range(T + 1):
        st = {k: env.get_state(k) for k in ("hpx", "hpy", "rpx", "rpy", "last_hvx", "last_hvy", "orca_nlines", "vis",
                                             "hn", "sim_exists", "fut_pen", "spawn_overflow")}
        for h, e, ho in zip(hs, offsets, hob):
            if st["spawn_overflow"][e] or h.get("spawn_overflow")[0]:
                continue
            compared += 1
            for k in ob:
                np.testing.assert_allclose(ob[k][e], ho[k][0], rtol=0, atol=1e-5, err_msg="obs %s t=%d e=%d" % (k, t, e))
            assert st["hn"][e] == h.get("hn")[0], (t, e)
            sl = slice(e * H, (e + 1) * H)
            for k in ("orca_nlines", "vis", "sim_exists"):
                assert np.array_equal(st[k][sl], h.get(k)), (k, t, e)
            for k in ("last_hvx", "last_hvy"):
                x, y = st[k][sl], h.get(k)
                if sf:
                    assert np.all(np.abs(x - y) <= 10 * tol + np.spacing(np.abs(y))), (k, t, e)
                else:
                    assert np.array_equal(x, y), (k, t, e)
            for k in ("hpx", "hpy"):
                np.testing.assert_allclose(st[k][sl], h.get(k), rtol=0, atol=tol, err_msg="%s t=%d e=%d" % (k, t, e))
            for k in ("rpx", "rpy", "fut_pen"):
                assert abs(st[k][e] - h.get(k)[0]) <= tol, (k, t, e)
        if t == T:
            break
        a = rng.uniform(-1.2, 1.2, (N, 2)).astype(np.float32)
        o, rew, done, info = env.step_device(torch.from_numpy(a).to(DEV))
        ob = _np_obs(o)
        rew, done, info = rew.cpu().numpy(), done.cpu().numpy(), info.cpu().numpy()
        aux = env._out["info_aux"].cpu().numpy()
        for j, (h, e) in enumerate(zip(hs, offsets)):
            hob[j], out = h.step(a[e:e + 1])
            if st["spawn_overflow"][e] or h.get("spawn_overflow")[0]:
                continue
            assert (done[e], info[e]) == (out["done"][0], out["info"][0]), (t, e)
            assert abs(rew[e] - out["reward"][0]) <= 1e-5, (t, e)
            assert abs(aux[e] - out["info_aux"][0]) <= 1e-6, (t, e)
    env.close()
    return compared


def test_truth_h20_4096_envs_matches_host_build():
    n = _lockstep_vs_harness(4096, 220, [0, 1, 517, 1024, 2047, 2048, 3333, 4095], human_num=20, **TRUTH)
    assert n >= 1700


def test_truth_h50_matches_host_build():
    n = _lockstep_vs_harness(1024, 220, [0, 5, 300, 511, 512, 800, 1023], human_num=50,
                             circle_radius=1.5 * 6 * 2 ** 0.5, arena_size=9.0, **TRUTH)
    assert n >= 1500


def test_truth_h100_matches_host_build():
    n = _lockstep_vs_harness(1024, 220, [0, 3, 999, 400, 1023], human_num=100, circle_radius=2 * 6 * 2 ** 0.5,
                             arena_size=12.0, **TRUTH)
    assert n >= 1000


def test_truth_128_slots_robot_visible_matches_host_build():
    """127 other humans plus the robot in the real solve, 127 in the look-ahead's: every simulator is re-created twice
    per step, and up to 128 ORCA lines per human (shared-memory line store plus overflow rows)."""
    n = _lockstep_vs_harness(64, 220, [0, 21, 42, 63], human_num=128, robot_visible=1,
                             circle_radius=3 * 6 * 2 ** 0.5, arena_size=18.0, **TRUTH)
    assert n >= 800


def test_truth_humans_joining_and_leaving_matches_host_build():
    n = _lockstep_vs_harness(512, 220, [0, 7, 255, 511], human_num=18, human_num_range=4, **TRUTH)
    assert n >= 800


def test_truth_test_phase_robot_visible_matches_host_build():
    n = _lockstep_vs_harness(1024, 220, [0, 9, 512, 1023], human_num=20, phase=2, robot_visible=1, **TRUTH)
    assert n >= 800


def test_truth_sf_humans_matches_host_build():
    for phase in (0, 2):
        n = _lockstep_vs_harness(2048, 220, [0, 33, 1024, 2047], human_num=20, human_policy=1, phase=phase, **TRUTH)
        assert n >= 800


def test_presolve_stays_off_for_truth(monkeypatch):
    """CN_PRESOLVE=1 forces the side-stream pre-solve for 'const_vel'; 'truth' never runs it (its observation look-ahead
    creates simulators the pre-solve's provisional marks do not cover), so forcing it changes nothing."""
    over = dict(num_envs=256, human_num=20, seed=3, **TRUTH)
    envs = []
    for ps in ("1", "0"):
        monkeypatch.setenv("CN_PRESOLVE", ps)
        envs.append(_engine(**over))
    on, off = envs
    on.reset(); off.reset()
    rng = np.random.RandomState(4)
    for t in range(60):
        a = torch.from_numpy(rng.uniform(-1.2, 1.2, (256, 2)).astype(np.float32)).to(DEV)
        r1, r0 = on.step_device(a), off.step_device(a)
        for k in r1[0]:
            assert torch.equal(r1[0][k], r0[0][k]), (k, t)
        for x, y in zip(r1[1:], r0[1:]):
            assert torch.equal(x, y), t
    on.close(); off.close()


def _policy(dev, H=20, W=12):
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    from crowdnav_prediction_attngraph_b200.policy import Policy, make_reference_like_state_dict

    class Args(object):
        num_processes, seq_length, num_mini_batch = 1, 30, 2
    spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
              'detected_human_num': Box((1,))}
    pol = Policy(spaces, Box((2,)), base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    pol.load_state_dict(make_reference_like_state_dict(W, seed=5), strict=False)
    return pol


@pytest.mark.parametrize("robot_visible,human_policy", [(0, 0), (1, 0), (0, 1)])
def test_batched_evaluation_equals_sequential_with_truth(robot_visible, human_policy):
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    test_size = 9
    d = _capi.default_config_dict(num_envs=1, nenv_total=1, seed=425, human_num=20, const_vel=2, phase=2,
                                  test_size=test_size, robot_visible=robot_visible, human_policy=human_policy,
                                  randomize_attributes=1, random_goal_changing=1, time_limit=30.0)
    pol = _policy(DEV)
    env = _engine(cfg=d)
    seq = evaluate(pol, env, 1, DEV, test_size, None, None, None)
    env.close()
    bat = evaluate_batched(pol, None, "CrowdSimPred-v0", 425, test_size, DEV, cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    assert seq["case_code"] == bat["case_code"]
    assert seq["case_nav_time"] == bat["case_nav_time"]
    for k in ("intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k


def test_device_resident_rollout_and_ppo_update_with_truth():
    """train.py's loop on the device-resident path (act -> step -> insert without host round trips) for two
    rollouts of 30 steps, then one PPO.update: finite losses, the weights move, and the rollout crossed episode ends."""
    from crowdnav_prediction_attngraph_b200 import ppo
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    N, T = 256, 30
    env = _engine(num_envs=N, human_num=20, seed=425, **TRUTH)

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, T, 2
    torch.manual_seed(425)
    pol = Policy(env.observation_space.spaces, env.action_space, base_kwargs=Args(), base='selfAttn_merge_srnn').to(DEV)
    ro = RolloutStorage(T, N, env.observation_space.spaces, env.action_space, 128, 256, device=DEV)
    obs = env.reset()
    for k in ro.obs:
        ro.obs[k][0].copy_(obs[k])
    eng = pol._engine(N, DEV)
    ends = 0
    for i in range(2 * T):
        ro.rollout_step_zero_copy(eng, env)
        ends += int((ro.masks[ro.step if ro.step else T] == 0).sum())
        if ro.step == 0 and i < T:
            ro.after_update()
    assert ends > 0
    assert torch.isfinite(ro.rewards).all() and torch.isfinite(ro.obs['spatial_edges']).all()
    assert (ro.obs['spatial_edges'][..., 2:] != 15).any()          # observed future rows
    with torch.no_grad():
        o = {k: ro.obs[k][-1] for k in ro.obs}
        hx = {k: ro.recurrent_hidden_states[k][-1] for k in ro.recurrent_hidden_states}
        nv = pol.get_value(o, hx, ro.masks[-1]).detach()
    ro.compute_returns(nv, True, 0.99, 0.95, False)
    agent = ppo.PPO(pol, 0.2, 2, 2, 0.5, 0.01, lr=4e-5, eps=1e-5, max_grad_norm=0.5)
    w0 = pol.base.spatial_linear[0].weight.detach().clone()
    losses = agent.update(ro)
    assert np.isfinite(losses).all()
    assert not torch.equal(w0, pol.base.spatial_linear[0].weight.detach())
    env.close()


def _reference_config(**kw):
    """The fields make_vec_envs reads from crowd_nav/configs/config.py, at its defaults, with 'truth' predictions."""
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics="holonomic"),
        robot=ns(visible=kw.get("visible", False), policy=kw.get("policy", "selfAttn_merge_srnn"), radius=0.3, v_pref=1,
                 FOV=2, sensor_range=5),
        humans=ns(policy="orca", radius=0.3, v_pref=1, FOV=2., random_goal_changing=True, end_goal_changing=True,
                  goal_change_chance=0.5),
        sim=ns(predict_method="truth", human_num=20, human_num_range=0, predict_steps=5, circle_radius=6 * np.sqrt(2),
               arena_size=6),
        env=ns(randomize_attributes=True, time_step=0.25, time_limit=50, val_size=100, test_size=500),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25), args=ns(sort_humans=True))


def test_reference_config_builds_steps_and_evaluates_through_make_vec_envs():
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    from crowdnav_prediction_attngraph_b200.vec_env import make_vec_envs
    config = _reference_config()
    envs = make_vec_envs("CrowdSimPred-v0", 425, 16, 0.99, None, DEV, allow_early_resets=True, config=config)
    assert (envs.cfgd["const_vel"], envs.cfgd["phase"]) == (2, 0)
    assert envs.observation_space['spatial_edges'].shape == (20, 12)
    obs = envs.reset()
    for _ in range(30):
        obs, rew, done, infos = envs.step(torch.zeros(16, 2, device=DEV))
    assert np.isfinite(rew.numpy()).all() and len(infos) == 16
    envs.close()
    pol = _policy(DEV)
    one = make_vec_envs("CrowdSimPred-v0", 425, 1, 0.99, None, DEV, allow_early_resets=True, config=config)
    assert (one.cfgd["const_vel"], one.cfgd["phase"]) == (2, 2)
    seq = evaluate(pol, one, 1, DEV, 12, None, config, None)
    one.close()
    bat = evaluate_batched(pol, config, "CrowdSimPred-v0", 425, 12, DEV)
    assert seq["case_code"] == bat["case_code"]
    with pytest.raises(NotImplementedError):
        make_vec_envs("CrowdSimPred-v0", 425, 16, 0.99, None, DEV, allow_early_resets=True,
                      config=_reference_config(policy="orca"))


def test_cn_env_create_refusals_with_truth():
    with pytest.raises(RuntimeError, match="ORCA / social-force robot"):
        _engine(num_envs=4, const_vel=2, robot_policy=1)
    with pytest.raises(RuntimeError, match="const_vel 3"):
        _engine(num_envs=4, const_vel=3)
    env = _engine(num_envs=4, const_vel=2, robot_visible=1)
    env.close()
