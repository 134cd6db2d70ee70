"""The ORCA and social-force robot policies (cn_config.robot_policy 1 / 2) on the CPU: the oracle and the host build of
the step kernel's logic against golden vectors recorded from the unmodified reference (tools/make_golden.py), and the
mapping of the reference Config onto cn_config."""
import copy
import types

import numpy as np
import pytest

from oracle.crowd_env import EnvConfig
from tests.harness_util import HarnessEnv
from tests.robot_oracle import RobotPolicyOracle
from tests.robot_policy_util import ROBOT_CASES, load_robot_case, replay_robot
from tests.test_oracle_golden import check_state


@pytest.mark.parametrize("name", ROBOT_CASES)
def test_oracle_robot_policy_matches_reference_golden(name):
    g, case, _ = load_robot_case(name)
    cfg = EnvConfig(human_num=case["human_num"], predict_method=case["predict_method"],
                    randomize_attributes=case["randomize"], random_goal_changing=case["goal_changing"])
    T, N = g["actions"].shape[:2]
    obs_keys = [k[3:] for k in g.files if k.startswith("ob_")]
    for k in range(N):
        env = RobotPolicyOracle(cfg, case["seed"] + k, case["nenv"], case.get("phase", "train"), case["robot_policy"])
        env.reset()
        for t in range(T):
            ob, rew, done, info = env.worker_step(g["actions"][t, k].copy())
            assert bool(done) == bool(g["done"][t, k]) and info["info"] == g["info"][t, k], (name, k, t)
            np.testing.assert_allclose(rew, g["reward"][t, k], rtol=0, atol=1e-9)
            np.testing.assert_allclose(info["min_danger"], g["min_danger"][t, k], rtol=0, atol=1e-9)
            rv = np.array(env.last_robot_action, dtype=np.float64)
            if case["robot_policy"] == "orca":
                assert np.array_equal(rv.astype(np.float32), g["robot_vel"][t, k].astype(np.float32)), (name, k, t)
            else:
                assert np.array_equal(rv, g["robot_vel"][t, k]), (name, k, t)          # fp64, bit for bit
            ha = np.asarray(env.last_sim_actions, dtype=np.float32)
            ok = ~np.isnan(g["human_actions"][t, k][:, 0])
            assert np.array_equal(ha[ok], g["human_actions"][t, k][ok]), (name, k, t)
            for key in obs_keys:
                if g["ob_" + key].dtype == bool:
                    assert np.array_equal(ob[key], g["ob_" + key][t + 1, k]), (key, t)
                else:
                    np.testing.assert_allclose(ob[key], g["ob_" + key][t + 1, k], rtol=0, atol=1e-6, err_msg=key)
            check_state(env.get_state(), g, t + 1, k)


@pytest.mark.parametrize("name", ROBOT_CASES)
def test_kernel_logic_host_build_robot_policy_matches_reference_golden(name):
    g, case, over = load_robot_case(name)
    env = HarnessEnv(**over)
    bad = replay_robot(g, case, env.reset, env.step, env.get)
    assert not bad, bad[:5]


def _reference_like_config(robot_policy, human_num_range=0):
    """The fields config_dict_from_reference reads, with the shipped baselines' values."""
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics="holonomic"),
        robot=ns(visible=False, policy=robot_policy, radius=0.3, v_pref=1, FOV=2, sensor_range=5),
        humans=ns(policy="orca", radius=0.3, v_pref=1, FOV=2., random_goal_changing=False, end_goal_changing=True,
                  goal_change_chance=0.5),
        sim=ns(predict_method="none", human_num=20, human_num_range=human_num_range, predict_steps=5,
               circle_radius=6 * np.sqrt(2), arena_size=6),
        env=ns(randomize_attributes=False, time_step=0.25, time_limit=50, val_size=100, test_size=500),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25), args=ns(sort_humans=True))


@pytest.mark.parametrize("policy,code", [("orca", 1), ("social_force", 2), ("selfAttn_merge_srnn", 0), ("srnn", 0)])
def test_config_maps_robot_policy(policy, code):
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    d = config_dict_from_reference(_reference_like_config(policy), 1, 425, "CrowdSimVarNum-v0")
    assert d["robot_policy"] == code


@pytest.mark.parametrize("policy", ["orca", "social_force"])
def test_config_rejects_uncovered_robot_policy_settings(policy):
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference, make_vec_envs
    cfg = _reference_like_config(policy)
    pred = copy.deepcopy(cfg)
    pred.sim.predict_method = "const_vel"
    with pytest.raises(NotImplementedError, match="CrowdSimPred-v0"):
        config_dict_from_reference(pred, 1, 425, "CrowdSimPred-v0")
    with pytest.raises(NotImplementedError, match="human_num_range"):
        config_dict_from_reference(_reference_like_config(policy, human_num_range=2), 1, 425, "CrowdSimVarNum-v0")
    with pytest.raises(NotImplementedError, match="GST wrapper"):
        make_vec_envs("CrowdSimVarNum-v0", 425, 1, 0.99, None, "cuda:0", False, config=cfg, pretext_wrapper=True,
                      gst_params={})
    # the network policy keeps all three
    net = _reference_like_config("selfAttn_merge_srnn", human_num_range=2)
    assert config_dict_from_reference(net, 1, 425, "CrowdSimVarNum-v0")["robot_policy"] == 0
