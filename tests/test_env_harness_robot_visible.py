"""robot.visible = True (the humans' ORCA / social-force solves see the robot) in the host build of the step kernel's
logic (tests/cpu_harness/env_harness.cpp), replayed against goldens recorded from the unmodified reference (tools/make_golden.py):
bit-exact done / info / ORCA velocities / line counts / failure index / sim_exists, fp64 state within 1e-9.  Also the
config mapping of robot.visible."""
import copy
import types

import numpy as np
import pytest

from tests.golden_util import load_env_case, replay
from tests.harness_util import HarnessEnv
from tests.robot_policy_util import ROBOT_POLICY, replay_robot

# train (config-1 shape; randomised with goal changes, episode ends crossed), test phase (simulators rebuilt on every
# agent-count change), humans joining / leaving (the robot's index follows the live count), social-force humans,
# humans.FOV = 1 (the dummy robot at (7, 7) occurs)
VIS_CASES = ["env_varnum_h5_vis", "env_varnum_h20_vis_rand", "env_varnum_h20_test_vis_rand", "env_varnum_h6_range2_vis",
             "env_varnum_h8_sf_vis", "env_varnum_h10_vis_fov1"]
# the ORCA robot among humans that see it
VIS_ROBOT_CASES = ["env_varnum_h10_orca_robot_vis_rand"]


def load_vis_case(name):
    g, case, over = load_env_case(name)
    over["robot_visible"] = int(case["robot_visible"])
    if "human_fov" in case:
        over["human_fov"] = float(case["human_fov"])
    if "robot_policy" in case:
        over["robot_policy"] = ROBOT_POLICY[case["robot_policy"]]
    return g, case, over


@pytest.mark.parametrize("name", VIS_CASES)
def test_kernel_logic_host_build_robot_visible_matches_reference_golden(name):
    g, case, over = load_vis_case(name)
    env = HarnessEnv(**over)
    bad = replay(g, case, env.reset, env.step, env.get)
    assert not bad, bad[:5]


@pytest.mark.parametrize("name", VIS_ROBOT_CASES)
def test_kernel_logic_host_build_robot_visible_orca_robot_matches_reference_golden(name):
    g, case, over = load_vis_case(name)
    env = HarnessEnv(**over)
    bad = replay_robot(g, case, env.reset, env.step, env.get)
    assert not bad, bad[:5]


def test_fov1_golden_contains_dummy_robot_encounters():
    """The FOV = 1 recording is only a test of the dummy robot if some human has the robot behind it while it is within
    neighborDist: count such (step, env, human) triples from the recorded state."""
    g, case, _ = load_vis_case("env_varnum_h10_vis_fov1")
    rob, px, py = g["st_robot"][:-1], g["st_hpx"][:-1], g["st_hpy"][:-1]
    vx, vy = g["st_hvx"][:-1], g["st_hvy"][:-1]
    th = np.arctan2(vy, vx)
    dx, dy = rob[..., 0:1] - px, rob[..., 1:2] - py
    c = (np.cos(th) * dx + np.sin(th) * dy) / np.hypot(dx, dy)
    behind = np.arccos(np.clip(c, -1, 1)) > np.pi * case["human_fov"] / 2
    assert int(np.nansum(behind & ~np.isnan(px))) > 100


def _reference_like_config(visible=True, **kw):
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics=kw.get("kinematics", "holonomic")),
        robot=ns(visible=visible, policy=kw.get("policy", "selfAttn_merge_srnn"), radius=0.3, v_pref=1, FOV=2,
                 sensor_range=5),
        humans=ns(policy="orca", radius=0.3, v_pref=1, FOV=2., random_goal_changing=False, end_goal_changing=True,
                  goal_change_chance=0.5),
        sim=ns(predict_method=kw.get("predict_method", "none"), human_num=20, human_num_range=0, predict_steps=5,
               circle_radius=6 * np.sqrt(2), arena_size=6),
        env=ns(randomize_attributes=False, time_step=0.25, time_limit=50, val_size=100, test_size=500),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25), args=ns(sort_humans=True))


def test_config_maps_robot_visible():
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    assert config_dict_from_reference(_reference_like_config(True), 4, 425, "CrowdSimVarNum-v0")["robot_visible"] == 1
    assert config_dict_from_reference(_reference_like_config(False), 4, 425, "CrowdSimVarNum-v0")["robot_visible"] == 0
    # the GST wrapper path (make_vec_envs(pretext_wrapper=True)) snapshots the config as CrowdSimVarNum-v0, unsorted
    d = config_dict_from_reference(_reference_like_config(True), 4, 425, "CrowdSimVarNum-v0", allow_unsorted=True)
    assert d["robot_visible"] == 1
    # the ORCA robot among humans that see it
    d = config_dict_from_reference(_reference_like_config(True, policy="orca"), 1, 425, "CrowdSimVarNum-v0")
    assert (d["robot_visible"], d["robot_policy"]) == (1, 1)


def test_config_rejects_uncovered_robot_visible_settings():
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    pred = _reference_like_config(True, predict_method="const_vel")
    with pytest.raises(NotImplementedError, match=r"CrowdSimPred-v0.*\(H \+ 1, 2\)"):
        config_dict_from_reference(pred, 4, 425, "CrowdSimPred-v0")
    invisible = copy.deepcopy(pred)
    invisible.robot.visible = False
    assert config_dict_from_reference(invisible, 4, 425, "CrowdSimPred-v0")["robot_visible"] == 0
    with pytest.raises(NotImplementedError, match="holonomic"):
        config_dict_from_reference(_reference_like_config(True, kinematics="unicycle"), 4, 425, "CrowdSimVarNum-v0")


def test_config_struct_carries_robot_visible_beside_robot_policy():
    """robot_policy and robot_visible share the 4 bytes robot_policy had: an int32 store of robot_policy (little-endian)
    reads back as (robot_policy, robot_visible = 0), and the struct keeps its size."""
    import ctypes as C
    from crowdnav_prediction_attngraph_b200 import _capi
    cfg = _capi.config_from_dict(_capi.default_config_dict(robot_policy=2, robot_visible=1))
    assert (cfg.robot_policy, cfg.robot_visible) == (2, 1)
    assert _capi.CnConfig.robot_visible.offset == _capi.CnConfig.robot_policy.offset + 2
    C.c_int32.from_buffer(cfg, _capi.CnConfig.robot_policy.offset).value = 1
    assert (cfg.robot_policy, cfg.robot_visible) == (1, 0)
