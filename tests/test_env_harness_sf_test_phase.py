"""Social-force humans (humans.policy = 'social_force') in phase 'test' on the CPU: the host build of the step kernel's
logic with the social-force look-ahead (tests/cpu_harness/env_harness.cpp) and the oracle (oracle/crowd_env.py)
against goldens recorded from the unmodified reference (tools/make_golden.py).  In phase 'test' the step runs the
ground-truth look-ahead calc_human_future_traj('truth') with SOCIAL_FORCE.predict on the humans only, fp64, and its
kept rows feed the 'future' danger zone and, on CrowdSimPred-v0, the future-collision penalty.  Also the config mapping:
one environment gives phase 'test' with social-force humans."""
import types

import numpy as np
import pytest

from oracle.crowd_env import CrowdEnvOracle, EnvConfig
from tests.golden_util import load_env_case, replay
from tests.harness_util import HarnessEnv
from tests.robot_oracle import RobotPolicyOracle
from tests.robot_policy_util import ROBOT_POLICY, replay_robot

# CrowdSimVarNum-v0 (8 randomised humans, goal changes), CrowdSimPred-v0 (10 randomised humans: future penalty and
# 'future' danger zone together), the first with robot.visible (the real solve sees the robot, the look-ahead does
# not), humans joining / leaving (the look-ahead over the live count)
SF_TEST_CASES = ["env_varnum_h8_sf_test_rand", "env_pred_h10_sf_test_rand", "env_varnum_h8_sf_test_vis_rand",
                 "env_varnum_h6_range2_sf_test"]
# the ORCA and the social-force robot among 20 social-force humans
SF_TEST_ROBOT_CASES = ["env_varnum_h20_test_sf_humans_orca_robot", "env_varnum_h20_test_sf_humans_sf_robot"]


def load_sf_test_case(name):
    g, case, over = load_env_case(name)
    over["robot_visible"] = int(case.get("robot_visible", False))
    if "robot_policy" in case:
        over["robot_policy"] = ROBOT_POLICY[case["robot_policy"]]
    return g, case, over


@pytest.mark.parametrize("name", SF_TEST_CASES + SF_TEST_ROBOT_CASES)
def test_fixture_is_sf_test_phase_with_episode_ends_and_danger(name):
    g, case, over = load_sf_test_case(name)
    assert (over["human_policy"], over["phase"]) == (1, 2)
    assert g["done"].sum() >= 1
    assert (g["info"] == 4).sum() >= 5                  # Danger steps from the 'future' danger zone


@pytest.mark.parametrize("name", SF_TEST_CASES)
def test_kernel_logic_host_build_sf_test_phase_matches_reference_golden(name):
    g, case, over = load_sf_test_case(name)
    env = HarnessEnv(**over)
    bad = replay(g, case, env.reset, env.step, env.get)
    assert not bad, bad[:5]


@pytest.mark.parametrize("name", SF_TEST_ROBOT_CASES)
def test_kernel_logic_host_build_sf_test_phase_robot_matches_reference_golden(name):
    g, case, over = load_sf_test_case(name)
    env = HarnessEnv(**over)
    bad = replay_robot(g, case, env.reset, env.step, env.get)
    assert not bad, bad[:5]


@pytest.mark.parametrize("name", [n for n in SF_TEST_CASES if "vis" not in n] + SF_TEST_ROBOT_CASES)
def test_oracle_sf_test_phase_matches_reference_golden(name):
    """EnvConfig takes no robot.visible, so the robot-visible fixture is left to the host build."""
    g, case, _ = load_sf_test_case(name)
    cfg = EnvConfig(human_num=case["human_num"], human_num_range=case.get("human_num_range", 0),
                    human_policy="social_force", predict_method=case["predict_method"],
                    randomize_attributes=case["randomize"], random_goal_changing=case["goal_changing"])
    T, N = g["actions"].shape[:2]
    obs_keys = [k[3:] for k in g.files if k.startswith("ob_")]
    for k in range(N):
        if "robot_policy" in case:
            env = RobotPolicyOracle(cfg, case["seed"] + k, case["nenv"], "test", case["robot_policy"])
        else:
            env = CrowdEnvOracle(cfg, case["seed"] + k, case["nenv"], "test")
        ob = env.reset()
        for t in range(T + 1):
            n = int(g["st_count"][t, k])
            st = env.get_state()
            assert len(st["hpx"]) == n, (name, k, t)
            for key in ("hpx", "hpy", "hvx", "hvy", "hgx", "hgy", "hrad", "hvpref"):
                np.testing.assert_allclose(st[key], g["st_" + key][t, k][:n], rtol=0, atol=1e-9,
                                           err_msg="%s t=%d" % (key, t))
            np.testing.assert_allclose(st["belief"], g["st_belief"][t, k][:n], rtol=0, atol=1e-9)
            assert np.array_equal(st["vis"], g["st_vis"][t, k][:n])
            for key in obs_keys:
                ref = g["ob_" + key][t, k]
                if ref.dtype == bool:
                    assert np.array_equal(ob[key], ref), (key, t)
                else:
                    np.testing.assert_allclose(ob[key], ref, rtol=0, atol=1e-6, err_msg="%s t=%d" % (key, t))
            if t == T:
                break
            ob, rew, done, info = env.worker_step(g["actions"][t, k].copy())
            assert bool(done) == bool(g["done"][t, k]) and info["info"] == g["info"][t, k], (name, k, t)
            np.testing.assert_allclose(rew, g["reward"][t, k], rtol=0, atol=1e-9)
            np.testing.assert_allclose(info["min_danger"], g["min_danger"][t, k], rtol=0, atol=1e-9)


def _reference_like_config(**kw):
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics="holonomic"),
        robot=ns(visible=kw.get("visible", False), policy=kw.get("policy", "selfAttn_merge_srnn"), radius=0.3, v_pref=1,
                 FOV=2, sensor_range=5),
        humans=ns(policy="social_force", radius=0.3, v_pref=1, FOV=2., random_goal_changing=False,
                  end_goal_changing=True, goal_change_chance=0.5),
        sim=ns(predict_method=kw.get("predict_method", "none"), human_num=20, human_num_range=0, predict_steps=5,
               circle_radius=6 * np.sqrt(2), arena_size=6),
        env=ns(randomize_attributes=False, time_step=0.25, time_limit=50, val_size=100, test_size=500),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25), args=ns(sort_humans=True))


@pytest.mark.parametrize("env_name,kw", [("CrowdSimVarNum-v0", {}), ("CrowdSimPred-v0", dict(predict_method="const_vel")),
                                         ("CrowdSimVarNum-v0", dict(visible=True)),
                                         ("CrowdSimVarNum-v0", dict(policy="orca")),
                                         ("CrowdSimVarNum-v0", dict(policy="social_force"))])
def test_config_maps_one_env_with_sf_humans_to_test_phase(env_name, kw):
    """rl/networks/envs.py:55-58 (the reference's test.py): one environment runs phase 'test'."""
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    d = config_dict_from_reference(_reference_like_config(**kw), 1, 425, env_name)
    assert (d["human_policy"], d["phase"]) == (1, 2)
    assert config_dict_from_reference(_reference_like_config(**kw), 4, 425, env_name)["phase"] == 0
