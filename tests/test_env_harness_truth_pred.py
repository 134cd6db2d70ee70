"""CrowdSimPred-v0 with sim.predict_method = 'truth' on the CPU: the host build of the step kernel's logic with the
observation look-ahead (tests/cpu_harness/truth_harness.cpp) and the oracle (tests/truth_oracle.py) against goldens
recorded from the unmodified reference (tools/make_golden.py).  Every observation, the first of an episode included,
runs calc_human_future_traj('truth'): buffer_len nested solves of the live humans from their true state, the kept rows
of the humans the robot sees as observation columns and as the trajectory the next step's reward penalises.  The
look-ahead is often the call that creates a human's rvo2 simulator (after a reset, a join / leave, with robot.visible on
every step), freezing every human's true radius.  Also the config mapping and the configurations still refused."""
import ctypes as C
import os
import subprocess
import types

import numpy as np
import pytest

from crowdnav_prediction_attngraph_b200 import _capi
from oracle.crowd_env import EnvConfig
from tests import harness_util
from tests.golden_util import GOLD, load_env_case, replay
from tests.harness_util import HarnessEnv
from tests.robot_policy_util import ROBOT_SRC
from tests.test_env_harness_robot_visible import VIS_SRC
from tests.test_env_harness_sf_test_phase import SF_SRC
from tests.truth_oracle import TruthPredOracle

# phase 'train' (the next step's reward reads the observed trajectory) and 'test' (two look-aheads per step), ORCA and
# social-force humans, randomised humans with goal changes, humans joining / leaving, robot.visible (humans.FOV = 1.0 in
# the train-phase case, so that the dummy robot occurs)
TRUTH_CASES = ["env_pred_h20_truth", "env_pred_h10_truth_rand", "env_pred_h10_truth_test_rand", "env_pred_h6_range3_truth",
               "env_pred_h10_truth_vis_rand", "env_pred_h10_truth_test_vis_rand", "env_pred_h8_sf_truth_rand",
               "env_pred_h8_sf_truth_test_rand"]

TRUTH_SO = os.path.join(harness_util.HERE, "_build_truth_harness.so")
TRUTH_SRC = os.path.join(harness_util.HERE, "cpu_harness", "truth_harness.cpp")
STATE_DTYPES = dict(harness_util.STATE_DTYPES, hwx="f8", hwy="f8", sim_n="u1")


def _build_truth_harness():
    core = harness_util.CORE
    deps = [TRUTH_SRC, SF_SRC, VIS_SRC, ROBOT_SRC, harness_util.SRC] + \
        [os.path.join(core, f) for f in os.listdir(core) if f.endswith(".cuh")]
    if os.path.exists(TRUTH_SO) and all(os.path.getmtime(TRUTH_SO) >= os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", TRUTH_SO, TRUTH_SRC])


class TruthHarnessEnv(HarnessEnv):
    """HarnessEnv of CrowdSimPred-v0 / 'truth' (robot.visible as vis_harness_create takes it): the same buffers, with
    truth_harness_reset / truth_harness_step (the observation look-ahead) as reset and step."""

    def __init__(self, **cfg_over):
        cfg_over.setdefault("const_vel", 2)
        super().__init__(**cfg_over)
        self.lib.harness_destroy(self.h)
        self.h = None
        _build_truth_harness()
        old, lib = self.lib, C.CDLL(TRUTH_SO)
        for name in ("harness_destroy", "harness_state_bytes", "harness_state_copy"):
            f, o = getattr(lib, name), getattr(old, name)
            f.argtypes, f.restype = o.argtypes, o.restype
        lib.truth_harness_create.restype = C.c_void_p
        lib.truth_harness_create.argtypes = [C.POINTER(_capi.CnConfig)]
        lib.truth_harness_reset.restype = C.c_int
        lib.truth_harness_reset.argtypes = old.harness_reset.argtypes
        lib.truth_harness_step.restype = C.c_int
        lib.truth_harness_step.argtypes = old.harness_step.argtypes
        self.lib = lib
        self.h = lib.truth_harness_create(C.byref(self.cfg))

    def reset(self):
        assert self.lib.truth_harness_reset(self.h, C.byref(self.obp)) == 0
        return self._obs()

    def step(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.float32)
        assert self.lib.truth_harness_step(self.h, a.ctypes.data, C.byref(self.obp), C.byref(self.outp)) == 0
        return self._obs(), {k: v.copy() for k, v in self.out.items()}

    def get(self, name):
        nbytes = self.lib.harness_state_bytes(self.h, name.encode())
        assert nbytes, name
        arr = np.zeros(nbytes // np.dtype(STATE_DTYPES[name]).itemsize, STATE_DTYPES[name])
        assert self.lib.harness_state_copy(self.h, name.encode(), arr.ctypes.data, nbytes, 0) == 0
        return arr


def load_truth_case(name):
    g, case, over = load_env_case(name)
    assert case["predict_method"] == "truth"
    over["const_vel"] = 2
    over["robot_visible"] = int(case.get("robot_visible", False))
    if "human_fov" in case:
        over["human_fov"] = float(case["human_fov"])
    return g, case, over


class FinishedEpisodeDiagnosticsMasked(object):
    """A fixture whose per-human solver diagnostics are masked (NaN, which replay() skips) on the steps that end an
    episode.  The reference records them before its auto-reset, i.e. from the observation look-ahead its step() runs on
    the FINISHED episode, whose observation the vector env then discards; the engine installs the next episode in the
    same launch and runs the look-ahead of the observation it returns instead."""

    def __init__(self, g):
        self._g, self.files = g, g.files
        ha = np.array(g["human_actions"])
        ha[g["done"]] = np.nan
        self._ha = ha

    def __getitem__(self, k):
        return self._ha if k == "human_actions" else self._g[k]


def recorded_trajectories(g):
    """{step: [N, P + 1, H, 4] trajectory the reference stored at that observation} (the steps it was recorded at)."""
    traj = g["st_traj"]
    if traj.ndim < 5:                   # human_num_range > 0: the fixture keeps no trajectory
        return {}
    steps = g["st_traj_step"] if "st_traj_step" in g.files else np.arange(traj.shape[0])
    return {int(t): traj[i] for i, t in enumerate(steps)}


def future_penalty(traj, robot_xy, collision_penalty=-20.0, threshold=0.6):
    """CrowdSimPred.calc_reward's penalty (crowd_sim_pred.py:216-233) of one stored trajectory [P + 1, H, 4]."""
    P = traj.shape[0] - 1
    idx = np.linalg.norm(traj[1:, :, :2] - robot_xy, axis=-1) < threshold
    return float(np.min(idx * (collision_penalty / 2. ** np.arange(2, P + 2).reshape((P, 1)))))


@pytest.mark.parametrize("name", TRUTH_CASES)
def test_fixture_is_truth_with_episode_ends_and_danger(name):
    g, case, over = load_truth_case(name)
    assert os.path.getsize(os.path.join(GOLD, name + ".npz")) < 1 << 20
    assert g["done"].sum() >= 1
    assert (g["info"] == 4).sum() >= 5
    assert g["ob_spatial_edges"].shape[-1] == 2 * (_capi.default_config_dict()["predict_steps"] + 1)


@pytest.mark.parametrize("name", [n for n in TRUTH_CASES if "range" not in n])
def test_fixture_observation_is_the_stored_truth_trajectory(name):
    """The reference's observation rows of the humans it sees are its stored trajectory minus the robot's position,
    distance-sorted: columns 2.. are the look-ahead's kept rows, not a constant-velocity extrapolation."""
    g, case, _ = load_truth_case(name)
    trajs = recorded_trajectories(g)
    assert trajs
    for t, traj in trajs.items():
        for k in range(traj.shape[0]):
            vis = g["st_vis"][t, k]
            rel = np.transpose(traj[k][:, vis, :2], (1, 0, 2)) - g["st_robot"][t, k][:2]
            rows = rel.reshape(int(vis.sum()), 2 * traj.shape[1]).astype(np.float32)
            rows = rows[np.argsort(np.linalg.norm(rel[:, 0].astype(np.float64), axis=-1), kind="stable")]
            np.testing.assert_array_equal(g["ob_spatial_edges"][t, k][:len(rows)], rows, err_msg="t=%d k=%d" % (t, k))


@pytest.mark.parametrize("name", TRUTH_CASES)
def test_kernel_logic_host_build_truth_matches_reference_golden(name):
    """done, info, collisions, the ORCA velocities / line counts of every simulator's LAST solve (the observation
    look-ahead's) and simulator existence bit for bit; observations, rewards and state at the replay's tolerances; the
    future-collision penalty the next reward reads, against the trajectory the reference stored."""
    g, case, over = load_truth_case(name)
    env = TruthHarnessEnv(**over)
    trajs = recorded_trajectories(g)
    pen_bad, t_box = [], [0]

    def check_pen(t):
        if t in trajs:
            rob = np.stack([env.get("rpx"), env.get("rpy")], -1)
            for k in range(env.N):
                want = future_penalty(trajs[t][k], rob[k])
                if abs(env.get("fut_pen")[k] - want) > 1e-9:
                    pen_bad.append((t, k, env.get("fut_pen")[k], want))

    def reset():
        ob = env.reset()
        check_pen(0)
        return ob

    def step(a):
        out = env.step(a)
        t_box[0] += 1
        check_pen(t_box[0])
        return out

    bad = replay(FinishedEpisodeDiagnosticsMasked(g), case, reset, step, env.get)
    assert not bad, bad[:5]
    assert not pen_bad, pen_bad[:5]


@pytest.mark.parametrize("name", [n for n in TRUTH_CASES if "vis" not in n])
def test_oracle_truth_matches_reference_golden(name):
    """EnvConfig takes no robot.visible, so the robot-visible fixtures are left to the host build."""
    g, case, _ = load_truth_case(name)
    cfg = EnvConfig(human_num=case["human_num"], human_num_range=case.get("human_num_range", 0),
                    human_policy=case.get("human_policy", "orca"), predict_method="const_vel",
                    randomize_attributes=case["randomize"], random_goal_changing=case["goal_changing"])
    T, N = g["actions"].shape[:2]
    obs_keys = [k[3:] for k in g.files if k.startswith("ob_")]
    trajs = recorded_trajectories(g)
    for k in range(N):
        env = TruthPredOracle(cfg, case["seed"] + k, case["nenv"], case.get("phase", "train"))
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
            assert np.array_equal(st["sim_exists"], g["st_sim_exists"][t, k][:n]), (name, k, t)
            if t in trajs:
                np.testing.assert_allclose(st["traj"], trajs[t][k], rtol=0, atol=1e-9, err_msg="traj t=%d" % t)
            for key in obs_keys:
                np.testing.assert_allclose(ob[key], g["ob_" + key][t, k], rtol=0, atol=1e-6, err_msg="%s t=%d" % (key, t))
            if t == T:
                break
            ob, rew, done, info = env.worker_step(g["actions"][t, k].copy())
            assert bool(done) == bool(g["done"][t, k]) and info["info"] == g["info"][t, k], (name, k, t)
            np.testing.assert_allclose(rew, g["reward"][t, k], rtol=0, atol=1e-9)
            np.testing.assert_allclose(info["min_danger"], g["min_danger"][t, k], rtol=0, atol=1e-9)
            if case.get("human_policy", "orca") == "orca" and not done:     # done: the next episode's reset solved last
                ok = ~np.isnan(g["human_actions"][t, k][:len(env.last_sim_actions), 0])
                ha = np.asarray(env.last_sim_actions, dtype=np.float32)
                assert np.array_equal(ha[ok], g["human_actions"][t, k][:len(ha)][ok]), (name, k, t)


def test_reset_creates_every_simulator_under_truth_only():
    """The reference after reset(): under 'truth' the observation look-ahead has created every human's simulator,
    under 'const_vel' none exists yet."""
    g, _, _ = load_truth_case("env_pred_h20_truth")
    assert g["st_sim_exists"][0].all()
    c = np.load(os.path.join(GOLD, "env_pred_h20.npz"))
    assert not c["st_sim_exists"][0].any()


def _reference_like_config(**kw):
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics="holonomic"),
        robot=ns(visible=kw.get("visible", False), policy=kw.get("policy", "selfAttn_merge_srnn"), radius=0.3, v_pref=1,
                 FOV=2, sensor_range=5),
        humans=ns(policy=kw.get("humans", "orca"), radius=0.3, v_pref=1, FOV=2., random_goal_changing=False,
                  end_goal_changing=True, goal_change_chance=0.5),
        sim=ns(predict_method=kw.get("predict_method", "truth"), human_num=20, human_num_range=0, predict_steps=5,
               circle_radius=6 * np.sqrt(2), arena_size=6),
        env=ns(randomize_attributes=False, time_step=0.25, time_limit=50, val_size=100, test_size=500),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25), args=ns(sort_humans=True))


@pytest.mark.parametrize("kw", [{}, dict(visible=True), dict(humans="social_force"),
                                dict(humans="social_force", visible=True)])
def test_config_maps_truth_to_const_vel_2(kw):
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    for n, phase in ((16, 0), (1, 2)):
        d = config_dict_from_reference(_reference_like_config(**kw), n, 425, "CrowdSimPred-v0")
        assert (d["const_vel"], d["phase"], d["robot_policy"]) == (2, phase, 0)
        assert d["robot_visible"] == int(kw.get("visible", False))
        assert d["human_policy"] == (1 if kw.get("humans") == "social_force" else 0)
    d = config_dict_from_reference(_reference_like_config(predict_method="const_vel"), 16, 425, "CrowdSimPred-v0")
    assert d["const_vel"] == 1


@pytest.mark.parametrize("kw,env_name", [
    (dict(predict_method="const_vel", visible=True), "CrowdSimPred-v0"),     # the reference raises on its first reset
    (dict(policy="orca"), "CrowdSimPred-v0"),                                # the ORCA / social-force robot
    (dict(policy="social_force"), "CrowdSimPred-v0"),
    (dict(predict_method="inferred"), "CrowdSimPred-v0"),
    (dict(), "CrowdSimVarNumCollect-v0"),
])
def test_config_still_refuses(kw, env_name):
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    with pytest.raises(NotImplementedError):
        config_dict_from_reference(_reference_like_config(**kw), 16, 425, env_name)


def test_truth_behind_the_gst_wrapper_is_refused():
    import torch
    from crowdnav_prediction_attngraph_b200.vec_env import make_vec_envs
    for env_name, wrap in (("CrowdSimPredRealGST-v0", False), ("CrowdSimPred-v0", True)):
        with pytest.raises(NotImplementedError):
            make_vec_envs(env_name, 425, 4, 0.99, None, torch.device("cpu"), False, config=_reference_like_config(),
                          pretext_wrapper=wrap, gst_params={})


def test_cn_env_create_refuses_unknown_prediction_mode():
    lib = _capi.load_library()
    cfg = _capi.config_from_dict(_capi.default_config_dict(const_vel=3))
    h = C.c_void_p()
    assert lib.cn_env_create(C.byref(cfg), C.byref(h)) != 0
    assert b"const_vel 3 unsupported" in lib.cn_last_error()
