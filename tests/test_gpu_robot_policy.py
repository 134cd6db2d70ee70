"""GPU: the ORCA and social-force robot policies (cn_config.robot_policy 1 / 2) in the CUDA step kernel.

  * golden replay against the unmodified reference (tools/make_golden.py), with the pre-solve on and off, without the
    side stream, and with every rejection-sampling search sent to the CTA-scope event kernel (CN_DEFER_TRIES=1);
  * batched evaluation equals the sequential protocol for both baselines, with randomised attributes too (the
    frozen robot simulator is handed from case 0 to every parallel case);
  * the full 500-case evaluation of the shipped baselines ORCA_no_rand / SF_no_rand reproduces the recorded reference
    run (tests/golden/eval_baselines.npz, tools/make_golden_eval_baselines.py) and the figures of the shipped test logs
    (tests/golden/shipped_baseline_logs.json)."""
import json
import os

import numpy as np
import pytest
import torch

from tests.robot_policy_util import ROBOT_CASES, load_robot_case, replay_robot

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

VARIANTS = [dict(), dict(CN_PRESOLVE="0"), dict(CN_PRESOLVE="1"), dict(CN_NO_SIDE_STREAM="1")]


def _replay(name, monkeypatch, env_vars):
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    for k, v in env_vars.items():
        monkeypatch.setenv(k, v)
    g, case, over = load_robot_case(name)
    env = CudaCrowdVecEnv(device="cuda:0", **over)

    def step(a):
        obs, rew, done, info = env.step_device(torch.from_numpy(a).cuda())
        out = dict(reward=rew.cpu().numpy(), done=done.cpu().numpy(), info=info.cpu().numpy(),
                   info_aux=env._out["info_aux"].cpu().numpy())
        return {k: v.cpu().numpy() for k, v in obs.items()}, out

    bad = replay_robot(g, case, lambda: {k: v.cpu().numpy() for k, v in env.reset().items()}, step, env.get_state)
    env.close()
    return bad


@pytest.mark.parametrize("variant", VARIANTS, ids=lambda v: ",".join("%s=%s" % kv for kv in v.items()) or "default")
@pytest.mark.parametrize("name", ROBOT_CASES)
def test_cuda_robot_policy_matches_reference_golden(name, variant, monkeypatch):
    bad = _replay(name, monkeypatch, variant)
    assert not bad, bad[:5]


@pytest.mark.parametrize("name", [c for c in ROBOT_CASES if c.endswith("_rand")])
def test_cuda_robot_policy_heavy_event_path_matches_reference_golden(name, monkeypatch):
    bad = _replay(name, monkeypatch, dict(CN_DEFER_TRIES="1"))
    assert not bad, bad[:5]


def _baseline_cfg(robot_policy, **over):
    """trained_models/ORCA_no_rand and SF_no_rand: CrowdSimVarNum-v0, 20 ORCA humans, phase 'test', seed 425."""
    from crowdnav_prediction_attngraph_b200 import _capi
    d = dict(num_envs=1, nenv_total=1, seed=425, human_num=20, const_vel=0, phase=2, test_size=500,
             robot_policy=robot_policy)
    d.update(over)
    return _capi.default_config_dict(**d)


@pytest.mark.parametrize("robot_policy,randomize", [(1, 0), (2, 0), (1, 1), (2, 1)])
def test_batched_evaluation_equals_sequential_for_robot_baselines(robot_policy, randomize):
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    dev = torch.device("cuda:0")
    test_size = 20
    d = _baseline_cfg(robot_policy, test_size=test_size, randomize_attributes=randomize,
                      random_goal_changing=randomize)
    env = CudaCrowdVecEnv(device=dev, cfg=d)
    seq = evaluate(None, env, 1, dev, test_size, None, None, None)
    if robot_policy == 1:
        nd_seq = env.get_state("rsim_nd")[0]
    env.close()
    bat = evaluate_batched(None, None, "CrowdSimVarNum-v0", 425, test_size, dev, cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    assert seq["case_code"] == bat["case_code"]
    assert seq["case_nav_time"] == bat["case_nav_time"]
    assert seq["case_path_len"] == pytest.approx(bat["case_path_len"], rel=0, abs=1e-12)
    for k in ("intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k
    if robot_policy == 1 and randomize:
        # the sequential run froze neighborDist at case 0 and kept it for all 20 cases
        assert nd_seq != pytest.approx(10.0)


def _fixture():
    g = np.load(os.path.join(GOLD, "eval_baselines.npz"))
    with open(os.path.join(GOLD, "shipped_baseline_logs.json")) as f:
        logs = json.load(f)
    return g, logs


@pytest.mark.parametrize("name,robot_policy", [("ORCA_no_rand", 1), ("SF_no_rand", 2)])
def test_500_case_baseline_evaluation_reproduces_reference_run(name, robot_policy):
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate_batched
    g, logs = _fixture()
    d = _baseline_cfg(robot_policy, num_envs=500)
    out = evaluate_batched(None, None, "CrowdSimVarNum-v0", 425, 500, torch.device("cuda:0"), cfg_dict=d)
    code = g[name + "_code"]
    assert np.array_equal(out["case_code"], code)
    assert np.array_equal(out["case_nav_time"], g[name + "_nav_time"])
    np.testing.assert_allclose(out["case_path_len"], g[name + "_path_len"], rtol=0, atol=1e-4)
    assert np.array_equal(out["case_too_close"], g[name + "_too_close"])
    mins = np.concatenate([np.asarray(m, np.float64) for m in out["case_min_dist"]] or [np.zeros(0)])
    np.testing.assert_allclose(mins, g[name + "_min_dist"], rtol=0, atol=1e-6)
    # the figures the reference logs, at the log's rounding (2 decimals), against the recorded reference run
    ref_ratio = float(np.mean(g[name + "_too_close"] / g[name + "_steps"] * 100))
    ref_min = float(np.mean(g[name + "_min_dist"]))
    assert round(out["intrusion_ratio"], 2) == round(ref_ratio, 2)
    assert round(out["min_intrusion_dist"], 2) == round(ref_min, 2)
    # ... and against the shipped log, at the agreement DESIGN.md §3.8 records
    log = logs[name]
    for k in log["matching_keys"]:
        assert round(out[k], 2) == log[k], k
    if log["cases_match"]:
        assert out["collision_cases"] == log["collision_cases"]
        assert out["timeout_cases"] == log["timeout_cases"]
