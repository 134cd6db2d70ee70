#!/usr/bin/env python
"""Golden vectors of the data-collection environment CrowdSimVarNumCollect-v0, recorded from the UNMODIFIED reference.

Runs the reference behind the stand-ins in oracle/shims like tools/make_golden.py (CROWDNAV_REFERENCE_ROOT) and steps
each environment with the zero action collect_data.py passes.  Per step it stores pred_info (float32, as the vec env
buffers hold it), the info code, done, the robot's position / velocity / goal, the humans' state, human_pred_id and
max_human_id.  It also runs collect_data.py's own collectData with np.random seeded and a small tot_steps in a
temporary directory and stores the text files it writes.  Output: tests/golden/collect_*.npz.

    CROWDNAV_REFERENCE_ROOT=... python tools/make_golden_collect.py
"""
import os
import sys
import tempfile

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
sys.path.insert(0, os.path.join(REPO, "tools"))
from reference_root import reference_root  # noqa: E402
REF = reference_root()
sys.path.insert(0, REF)
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402

INFO_CODE = {"Nothing": 0, "Timeout": 1, "Collision": 2, "ReachGoal": 3, "Danger": 4}

# the reference's default config (20 randomised ORCA humans with goal changes) and robot.policy 'orca' unless stated;
# seed 2**31 + 5 exercises the upper half of collect_data.py's np.random.randint(0, 2**32 - 1) seeds.  There is no
# phase-'test' case: the reference raises there on the first step (CrowdSimVarNum.step runs the ground-truth look-ahead,
# whose calc_human_future_traj reads self.human_visibility, crowd_sim_var_num.py:225, which the collect environment's
# generate_ob never sets), so collect_data.py with data.render (one environment, phase 'test') cannot run.
CASES = {
    "collect_h20_train": dict(human_num=20, nenv=3, steps=300, seed=2 ** 31 + 5, phase="train", robot_policy="orca"),
    "collect_h8_sf_humans": dict(human_num=8, nenv=2, steps=250, seed=21, phase="train", robot_policy="orca",
                                 human_policy="social_force"),
    "collect_h10_sf_robot": dict(human_num=10, nenv=2, steps=300, seed=31, phase="train", robot_policy="social_force"),
}
# collect_data.py itself: np.random.seed(FILES_SEED) before collectData, data.tot_steps frames, num_processes envs
FILES = dict(np_seed=7, tot_steps=60, num_processes=2)


def _config(case):
    from crowd_nav.configs.config import Config
    cfg = Config()
    cfg.sim.human_num = case["human_num"]
    cfg.humans.policy = case.get("human_policy", "orca")
    cfg.robot.policy = case["robot_policy"]
    cfg.sim.predict_method = "none"
    cfg.env.use_wrapper = False
    return cfg


def run_case(name, case):
    sys.argv = ["x", "--no-cuda", "--env-name", "CrowdSimVarNumCollect-v0"]
    import gym
    import rvo2
    import crowd_sim  # noqa: F401  registers the ids
    rvo2.ONLY_AGENT0 = False
    H, N, T = case["human_num"], case["nenv"], case["steps"]
    rec = {k: [] for k in ("pred_info", "info", "done", "robot", "hpx", "hpy", "hvx", "hvy", "hgx", "hgy", "hrad", "hvpref",
                           "pred_id", "max_id")}
    per_env = []
    for k in range(N):
        cfg = _config(case)
        env = gym.make("CrowdSimVarNumCollect-v0")
        env.configure(cfg)
        env.thisSeed = case["seed"] + k
        env.nenv = N
        env.phase = case["phase"]
        r = {key: [] for key in rec}

        def snap(ob, info, done):
            r["pred_info"].append(np.asarray(ob["pred_info"], dtype=np.float32))
            r["info"].append(info)
            r["done"].append(done)
            ro = env.robot
            r["robot"].append([ro.px, ro.py, ro.vx, ro.vy, ro.gx, ro.gy])
            for key, attr in (("hpx", "px"), ("hpy", "py"), ("hvx", "vx"), ("hvy", "vy"), ("hgx", "gx"), ("hgy", "gy"),
                              ("hrad", "radius"), ("hvpref", "v_pref")):
                r[key].append([float(getattr(h, attr)) for h in env.humans])
            r["pred_id"].append(np.array(env.human_pred_id, dtype=np.int64, copy=True))
            r["max_id"].append(int(env.max_human_id))

        ob = env.reset()
        snap(ob, 0, False)
        for _ in range(T):
            ob, _, done, info = env.step(np.zeros(2))
            snap(ob, INFO_CODE[type(info["info"]).__name__], bool(done))
        per_env.append(r)
        infos = np.array(r["info"][1:])
        print(name, "env", k, "ReachGoal", int((infos == 3).sum()), "Collision", int((infos == 2).sum()),
              "max id", r["max_id"][-1])
    out = {}
    for key in rec:
        dt = {"pred_info": np.float32, "info": np.int32, "done": bool, "pred_id": np.int32, "max_id": np.int32}.get(key, np.float64)
        out[key] = np.stack([np.asarray(r[key], dtype=dt) for r in per_env], axis=1)      # [T + 1, N, ...]
    out["meta"] = np.array([repr(case)])
    return out


def goal_branches(g):
    """(median-branch count, uniform-branch count) of the ReachGoal goal draws in a recording."""
    med = uni = 0
    T1, N = g["info"].shape
    for k in range(N):
        for t in range(1, T1):
            if g["info"][t, k] != 3:
                continue
            goal = g["robot"][t, k, 4:6]
            m = np.median(np.stack([g["hpx"][t - 1, k], g["hpy"][t - 1, k]], -1), axis=0)
            if np.array_equal(goal, m):
                med += 1
            else:
                uni += 1
    return med, uni


def run_files():
    """collect_data.py's collectData (unmodified) on a small tot_steps; returns {relative path: text}."""
    sys.argv = ["x", "--no-cuda"]
    import torch
    import rvo2
    rvo2.ONLY_AGENT0 = False
    import collect_data
    from crowd_nav.configs.config import Config
    cfg = Config()
    tmp = tempfile.mkdtemp()
    cfg.data.tot_steps = FILES["tot_steps"]
    cfg.data.num_processes = FILES["num_processes"]
    cfg.data.data_save_dir = tmp
    np.random.seed(FILES["np_seed"])
    seed = np.random.RandomState(FILES["np_seed"]).randint(0, np.iinfo(np.uint32).max)
    collect_data.collectData(torch.device("cpu"), True, cfg)
    files = {}
    for root, _, names in os.walk(tmp):
        for n in sorted(names):
            p = os.path.join(root, n)
            files[os.path.relpath(p, tmp)] = open(p).read()
    return int(seed), files


if __name__ == "__main__":
    only = sys.argv[1:]
    totals = np.zeros(3, np.int64)
    # collect_data.py first: the reference's Config keeps its sections as class attributes, so the per-case settings
    # below would leak into the Config collectData builds
    if not only or "files" in only:
        seed, files = run_files()
        names = sorted(files)
        path = os.path.join(REPO, "tests", "golden", "collect_files.npz")
        np.savez_compressed(path, names=np.array(names), texts=np.array([files[n] for n in names]),
                            meta=np.array([repr(dict(FILES, seed=seed))]))
        print("collect_data.py seed", seed, "files", names, "wrote", path, os.path.getsize(path) // 1024, "KiB")
    for name, case in CASES.items():
        if only and name not in only:
            continue
        out = run_case(name, case)
        med, uni = goal_branches(out)
        totals += [med, uni, int((out["info"] == 2).sum())]
        print(name, "goal draws: median", med, "uniform", uni)
        path = os.path.join(REPO, "tests", "golden", name + ".npz")
        np.savez_compressed(path, **out)
        print("wrote", path, os.path.getsize(path) // 1024, "KiB")
    print("totals: ReachGoal median", totals[0], "uniform", totals[1], "Collision", totals[2])
