#!/usr/bin/env python
"""Generate golden vectors from the UNMODIFIED reference (runs only in the build container).

Imports the reference package from $CROWDNAV_REFERENCE_ROOT behind the stand-ins in oracle/shims
(gym / baselines / matplotlib stubs and the `rvo2` module backed by oracle/rvo2_ref.cpp),
steps `CrowdSimPred-v0` / `CrowdSimVarNum-v0` exactly as rl/networks/shmem_vec_env.py's
worker does (step; reset on done), and records per-step observations, rewards, dones, info
codes, human ORCA velocities and the full persistent state.  Output: tests/golden/env_*.npz.

    python tools/make_golden.py            # writes all fixtures
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
from reference_root import reference_root  # noqa: E402
REF = reference_root()
sys.path.insert(0, REF)
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

INFO_CODE = {"Nothing": 0, "Timeout": 1, "Collision": 2, "ReachGoal": 3, "Danger": 4}

# Step counts keep every fixture under 1 MB and still reach a ReachGoal episode end in the 20-human train and test
# recordings (env 0, steps 171 and 173); traj_every = k stores the human trajectory buffers (a third of a recording) only
# at every k-th step.  tools/make_golden_policy.py and make_golden_update.py record the longer env_pred_h20 rollout
# they cut their inputs from themselves (run_case with steps=LONG_H20_STEPS).
LONG_H20_STEPS = 260
CASES = {
    # BASELINE config 2 semantics (SURVEY.md §8d C2), small N
    "env_pred_h20": dict(env_name="CrowdSimPred-v0", human_num=20, predict_method="const_vel",
                         randomize=False, goal_changing=False, nenv=4, steps=175, seed=425, traj_every=4),
    # BASELINE config 4 semantics (randomised ORCA humans + goal changing), small N / H
    "env_pred_h20_rand": dict(env_name="CrowdSimPred-v0", human_num=20, predict_method="const_vel",
                              randomize=True, goal_changing=True, nenv=3, steps=180, seed=425),
    "env_pred_h50_rand": dict(env_name="CrowdSimPred-v0", human_num=50, predict_method="const_vel",
                              randomize=True, goal_changing=True, nenv=2, steps=70, seed=7),
    # BASELINE config 1 (CrowdSimVarNum-v0, predict_method none, 5 humans, 4 envs)
    "env_varnum_h5": dict(env_name="CrowdSimVarNum-v0", human_num=5, predict_method="none",
                          randomize=False, goal_changing=False, nenv=4, steps=260, seed=425),
    # phase='test' (SURVEY.md §8f row 1): ground-truth ORCA look-ahead before the reward, 'future' danger zone,
    # test seeds (offset 1000, case_size = env.test_size)
    "env_pred_h20_test": dict(env_name="CrowdSimPred-v0", human_num=20, predict_method="const_vel",
                              randomize=False, goal_changing=False, nenv=3, steps=175, seed=425, phase="test"),
    "env_varnum_h5_test": dict(env_name="CrowdSimVarNum-v0", human_num=5, predict_method="none",
                               randomize=False, goal_changing=False, nenv=2, steps=160, seed=425, phase="test"),
    # sim.human_num_range > 0 (SURVEY 8f row 4): humans join / leave every 5 s; per-human arrays are padded to
    # human_num + range with NaN, `st_count` holds the live count
    "env_varnum_h5_range2": dict(env_name="CrowdSimVarNum-v0", human_num=5, predict_method="none", human_num_range=2,
                                 randomize=False, goal_changing=False, nenv=3, steps=200, seed=425),
    "env_pred_h6_range3": dict(env_name="CrowdSimPred-v0", human_num=6, predict_method="const_vel", human_num_range=3,
                               randomize=True, goal_changing=True, nenv=2, steps=200, seed=9),
    # humans.policy = 'social_force' (SURVEY 8f row 4)
    "env_pred_h8_sf": dict(env_name="CrowdSimPred-v0", human_num=8, predict_method="const_vel", human_policy="social_force",
                           randomize=True, goal_changing=True, nenv=2, steps=160, seed=21),
    "env_pred_h10_test_rand": dict(env_name="CrowdSimPred-v0", human_num=10, predict_method="const_vel",
                                   randomize=True, goal_changing=True, nenv=2, steps=200, seed=11, phase="test"),
    # robot.policy = 'orca' / 'social_force' (the paper's baselines, trained_models/ORCA_no_rand and SF_no_rand): the
    # robot is driven inside env.step, the scripted action is passed and ignored; robot_vel records its velocity after
    # every step.  The randomised train-phase cases cross episode ends, which keep the robot's frozen rvo2 simulator.
    "env_varnum_h20_test_orca_robot": dict(env_name="CrowdSimVarNum-v0", human_num=20, predict_method="none",
                                           robot_policy="orca", randomize=False, goal_changing=False, nenv=2, steps=120,
                                           seed=425, phase="test"),
    "env_varnum_h10_orca_robot_rand": dict(env_name="CrowdSimVarNum-v0", human_num=10, predict_method="none",
                                           robot_policy="orca", randomize=True, goal_changing=True, nenv=2, steps=200,
                                           seed=31),
    "env_varnum_h20_test_sf_robot": dict(env_name="CrowdSimVarNum-v0", human_num=20, predict_method="none",
                                         robot_policy="social_force", randomize=False, goal_changing=False, nenv=2,
                                         steps=120, seed=425, phase="test"),
    "env_varnum_h10_sf_robot_rand": dict(env_name="CrowdSimVarNum-v0", human_num=10, predict_method="none",
                                         robot_policy="social_force", randomize=True, goal_changing=True, nenv=2,
                                         steps=200, seed=31),
    # robot.visible = True (crowd_sim.py:695-699): every human's ORCA / social-force solve gets the robot (or, outside
    # the human's FOV, the dummy robot at (7, 7) with config.robot.radius) as its last agent.  The test-phase case
    # rebuilds each simulator twice per step (hn + 1 agents in get_human_actions, hn in the look-ahead); the range
    # case moves the robot's index with the live count; humans.FOV = 1.0 makes the dummy robot actually occur.
    "env_varnum_h5_vis": dict(env_name="CrowdSimVarNum-v0", human_num=5, predict_method="none", robot_visible=True,
                              randomize=False, goal_changing=False, nenv=4, steps=200, seed=425),
    "env_varnum_h20_vis_rand": dict(env_name="CrowdSimVarNum-v0", human_num=20, predict_method="none",
                                    robot_visible=True, randomize=True, goal_changing=True, nenv=3, steps=180, seed=425),
    "env_varnum_h20_test_vis_rand": dict(env_name="CrowdSimVarNum-v0", human_num=20, predict_method="none",
                                         robot_visible=True, randomize=True, goal_changing=True, nenv=2, steps=120,
                                         seed=11, phase="test"),
    "env_varnum_h6_range2_vis": dict(env_name="CrowdSimVarNum-v0", human_num=6, predict_method="none", human_num_range=2,
                                     robot_visible=True, randomize=True, goal_changing=True, nenv=3, steps=200, seed=9),
    "env_varnum_h8_sf_vis": dict(env_name="CrowdSimVarNum-v0", human_num=8, predict_method="none",
                                 human_policy="social_force", robot_visible=True, randomize=True, goal_changing=True,
                                 nenv=2, steps=160, seed=21),
    "env_varnum_h10_orca_robot_vis_rand": dict(env_name="CrowdSimVarNum-v0", human_num=10, predict_method="none",
                                               robot_policy="orca", robot_visible=True, randomize=True,
                                               goal_changing=True, nenv=2, steps=200, seed=31),
    "env_varnum_h10_vis_fov1": dict(env_name="CrowdSimVarNum-v0", human_num=10, predict_method="none",
                                    robot_visible=True, human_fov=1.0, randomize=True, goal_changing=True, nenv=3,
                                    steps=200, seed=17),
}


def action_script(rng, k, t, ob, mode):
    """Deterministic-but-varied robot actions: goal seeking + noise / idle / random."""
    rn = ob["robot_node"] if not isinstance(ob["robot_node"], list) else np.array(ob["robot_node"], dtype=np.float64)
    rn = np.asarray(rn, dtype=np.float64).reshape(-1)
    to_goal = np.array([rn[3] - rn[0], rn[4] - rn[1]])
    d = np.linalg.norm(to_goal) + 1e-9
    m = mode[k % len(mode)]
    if m == "goal":
        a = to_goal / d * 1.2 + rng.normal(0, 0.3, 2)      # sometimes > v_pref: exercises clipping
    elif m == "idle":
        a = rng.normal(0, 0.02, 2)
    else:
        a = rng.uniform(-1.2, 1.2, 2)
    return a.astype(np.float32)


def build_reference_env(case, rank):
    import gym
    import crowd_sim  # noqa: F401  registers ids
    from crowd_nav.configs.config import Config
    cfg = Config()
    cfg.sim.human_num = case["human_num"]
    cfg.sim.human_num_range = case.get("human_num_range", 0)
    cfg.humans.policy = case.get("human_policy", "orca")
    cfg.robot.policy = case.get("robot_policy", "selfAttn_merge_srnn")
    cfg.sim.predict_method = case["predict_method"]
    cfg.env.use_wrapper = False
    cfg.env.randomize_attributes = case["randomize"]
    cfg.humans.random_goal_changing = case["goal_changing"]
    cfg.orca.neighbor_dist = 10
    cfg.robot.visible = case.get("robot_visible", False)
    if "human_fov" in case:
        cfg.humans.FOV = case["human_fov"]
    env = gym.make(case["env_name"])
    env.configure(cfg)
    env.thisSeed = case["seed"] + rank
    env.nenv = case["nenv"]
    env.phase = case.get("phase", "train")
    return env, cfg


def _pad(a, n, fill=np.nan):
    a = np.asarray(a)
    if a.shape[0] == n:
        return a
    out = np.full((n,) + a.shape[1:], fill, dtype=a.dtype if a.dtype != bool else bool)
    out[:a.shape[0]] = a
    return out


def ref_state(env, cfg):
    H = env.human_num
    Hmax = cfg.sim.human_num + cfg.sim.human_num_range
    f = lambda name: _pad(np.array([float(getattr(h, name)) for h in env.humans], dtype=np.float64), Hmax)
    r = env.robot
    traj = getattr(env, "human_future_traj", None)
    if cfg.sim.predict_method == "none" or cfg.sim.human_num_range > 0:
        traj = None       # VarNum keeps no prediction (the test-phase look-ahead buffer is internal)
    return dict(
        robot=np.array([r.px, r.py, r.vx, r.vy, r.gx, r.gy], dtype=np.float64),
        hpx=f("px"), hpy=f("py"), hvx=f("vx"), hvy=f("vy"), hgx=f("gx"), hgy=f("gy"),
        hrad=f("radius"), hvpref=f("v_pref"),
        belief=_pad(np.array(env.last_human_states, dtype=np.float64).reshape(H, 5), Hmax),
        count=int(H),
        traj=np.zeros((0,)) if traj is None else np.array(traj, dtype=np.float64),
        vis=_pad(np.array(env.human_visibility, dtype=bool), Hmax, False),
        global_time=float(env.global_time), potential=float(env.potential),
        nd_global=float(cfg.orca.neighbor_dist),
        sim_exists=_pad(np.array([getattr(h.policy, "sim", None) is not None for h in env.humans], dtype=bool), Hmax, False),
    )


def ob_to_f32(ob, H, W):
    out = dict(
        robot_node=np.asarray(ob["robot_node"], dtype=np.float32).reshape(1, 7),
        temporal_edges=np.asarray(ob["temporal_edges"], dtype=np.float32).reshape(1, 2),
        spatial_edges=np.asarray(ob["spatial_edges"], dtype=np.float32).reshape(H, W),
        detected_human_num=np.asarray(ob["detected_human_num"], dtype=np.float32).reshape(1),
    )
    if "visible_masks" in ob:
        out["visible_masks"] = np.asarray(ob["visible_masks"], dtype=bool).reshape(H)
    return out


def run_case(name, case):
    sys.argv = ["x", "--no-cuda", "--env-name", case["env_name"]]
    import rvo2
    rvo2.ONLY_AGENT0 = False          # the genuine full doStep of every per-human simulator
    H = case["human_num"] + case.get("human_num_range", 0)          # array width = max_human_num
    W = 12 if case["predict_method"] == "const_vel" else 2
    N, T = case["nenv"], case["steps"]
    mode = ["goal", "goal", "rand", "idle"]
    rec = dict(actions=np.zeros((T, N, 2), np.float32), reward=np.zeros((T, N)), done=np.zeros((T, N), bool),
               info=np.zeros((T, N), np.int32), min_danger=np.zeros((T, N)),
               human_actions=np.zeros((T, N, H, 2), np.float32),
               orca_nlines=np.zeros((T, N, H), np.int32), orca_fail=np.zeros((T, N, H), np.int32),
               robot_vel=np.zeros((T, N, 2)))
    obs_keys = ["robot_node", "temporal_edges", "spatial_edges", "detected_human_num"] + \
               (["visible_masks"] if W == 2 else [])
    state_keys = ["robot", "hpx", "hpy", "hvx", "hvy", "hgx", "hgy", "hrad", "hvpref", "belief", "traj",
                  "vis", "global_time", "potential", "nd_global", "sim_exists", "count"]
    obs_rec = {k: [[None] * N for _ in range(T + 1)] for k in obs_keys}
    st_rec = {k: [[None] * N for _ in range(T + 1)] for k in state_keys}
    for k in range(N):
        env, cfg = build_reference_env(case, k)
        rng = np.random.RandomState(1000 + k)
        ob = env.reset()
        o32 = ob_to_f32(ob, H, W)
        for key in obs_keys:
            obs_rec[key][0][k] = o32[key]
        st = ref_state(env, cfg)
        for key in state_keys:
            st_rec[key][0][k] = st[key]
        for t in range(T):
            a = action_script(rng, k, t, ob, mode)
            rec["actions"][t, k] = a
            # human ORCA velocities are read back from the env after the step
            ob, rew, done, info = env.step(a.copy())
            rec["reward"][t, k] = rew
            rec["done"][t, k] = done
            rec["info"][t, k] = INFO_CODE[type(info["info"]).__name__]
            rec["min_danger"][t, k] = getattr(info["info"], "min_dist", 0.0)
            rec["robot_vel"][t, k] = env.robot.vx, env.robot.vy
            # velocities/diagnostics of the step just taken (before a possible respawn zeroes them
            # we read the sims, which always hold the solved velocity of agent 0)
            rec["human_actions"][t, k, len(env.humans):] = np.nan
            rec["orca_nlines"][t, k, len(env.humans):] = -1
            rec["orca_fail"][t, k, len(env.humans):] = -2
            for i, h in enumerate(env.humans):
                sim = getattr(h.policy, "sim", None)
                if sim is not None:
                    rec["human_actions"][t, k, i] = sim.getAgentVelocity(0)
                    rec["orca_nlines"][t, k, i] = sim._numLines(0)
                    rec["orca_fail"][t, k, i] = sim._lineFail(0)
                else:       # respawned this step: velocity no longer observable
                    rec["human_actions"][t, k, i] = np.nan
                    rec["orca_nlines"][t, k, i] = -1
                    rec["orca_fail"][t, k, i] = -2
            if done:
                ob = env.reset()
            o32 = ob_to_f32(ob, H, W)
            for key in obs_keys:
                obs_rec[key][t + 1][k] = o32[key]
            st = ref_state(env, cfg)
            for key in state_keys:
                st_rec[key][t + 1][k] = st[key]
        print(name, "env", k, "episodes:", int(rec["done"][:, k].sum()),
              "infos:", np.bincount(rec["info"][:, k], minlength=5).tolist())
    out = dict(rec)
    for key in obs_keys:
        out["ob_" + key] = np.array(obs_rec[key])
    for key in state_keys:
        out["st_" + key] = np.array(st_rec[key])
    out["meta"] = np.array([repr(case)])
    return out


if __name__ == "__main__":
    only = sys.argv[1:]
    for name, case in CASES.items():
        if only and name not in only:
            continue
        out = run_case(name, case)
        if case.get("traj_every", 1) > 1:
            out["st_traj_step"] = np.arange(0, case["steps"] + 1, case["traj_every"], dtype=np.int32)
            out["st_traj"] = out["st_traj"][out["st_traj_step"]]
        path = os.path.join(REPO, "tests", "golden", name + ".npz")
        np.savez_compressed(path, **out)
        print("wrote", path, os.path.getsize(path) // 1024, "KiB")
