#!/usr/bin/env python
"""Record what the UNMODIFIED reference produces for the full rl/evaluation.py test protocol of the two shipped robot
baselines, trained_models/ORCA_no_rand and SF_no_rand (CrowdSimVarNum-v0, 20 humans, seed 425, test_size 500, the robot
driven by ORCA / social force inside env.step, zero actions passed).  Runs only in the build container: the reference
is imported from $CROWDNAV_REFERENCE_ROOT behind oracle/shims (rvo2 -> oracle/rvo2_ref.cpp).

Per case: outcome code, nav time, path length, too-close frame count, the min-distance list, steps.  The cases are
split over processes.  Each process seeds episode k as the sequential protocol does: case_counter 2k mod test_size
(the loop's explicit reset and the vec env's auto-reset at done both advance it), and the auto-reset episode's first
robot position ends the path (rl/evaluation.py:96-97).  The robot's rvo2 simulator is created once per process, as in
the reference; without randomised attributes its frozen parameters are the configured constants, so the split does
not change them.  Output: tests/golden/eval_baselines.npz.

--humans social_force runs the same protocol among social-force humans (humans.policy = 'social_force', whose phase
'test' look-ahead runs SOCIAL_FORCE.predict) and writes tests/golden/eval_baselines_sf_humans.npz; the default, orca,
writes eval_baselines.npz as before.

    python tools/make_golden_eval_baselines.py [--procs 8] [--humans orca|social_force]
"""
import argparse
import multiprocessing as mp
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
from reference_root import reference_root  # noqa: E402
REF = reference_root()

import numpy as np  # noqa: E402

BASELINES = {"ORCA_no_rand": "orca", "SF_no_rand": "social_force"}
SEED, TEST_SIZE, HUMANS = 425, 500, 20
INFO_CODE = {"Timeout": 1, "Collision": 2, "ReachGoal": 3}


def run_block(args):
    policy, humans, lo, hi = args
    sys.path.insert(0, REF)
    sys.argv = ["x", "--no-cuda", "--env-name", "CrowdSimVarNum-v0"]
    import gym
    import crowd_sim  # noqa: F401
    from crowd_nav.configs.config import Config
    from crowd_sim.envs.utils.info import Danger
    cfg = Config()
    cfg.robot.policy = policy
    cfg.humans.policy = humans
    cfg.sim.human_num = HUMANS
    cfg.sim.predict_method = "none"
    cfg.env.randomize_attributes = False
    cfg.humans.random_goal_changing = False
    cfg.env.use_wrapper = False
    env = gym.make("CrowdSimVarNum-v0")
    env.configure(cfg)
    env.thisSeed, env.nenv, env.phase = SEED, 1, "test"
    out = []
    for k in range(lo, hi):
        env.case_counter["test"] = (2 * k) % TEST_SIZE
        ob = env.reset()
        last = np.asarray(ob["robot_node"], np.float32).reshape(-1)[:2]
        path, close, mins, steps, t_begin = 0.0, 0, [], 0, 0.0
        while True:
            steps += 1
            t_begin = env.global_time
            ob, rew, done, info = env.step(np.zeros(2, np.float32))
            if done:
                ob = env.reset()                    # the vec env's auto-reset: its robot position ends the path
            pos = np.asarray(ob["robot_node"], np.float32).reshape(-1)[:2]
            path = path + float(np.linalg.norm(pos - last))      # float32 norm, float64 sum (the engine's evaluate)
            last = pos
            if isinstance(info["info"], Danger):
                close += 1
                mins.append(float(info["info"].min_dist))
            if done:
                break
        code = INFO_CODE[type(info["info"]).__name__]
        out.append((k, code, cfg.env.time_limit if code == 1 else float(t_begin), float(path), close, mins, steps))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=8)
    ap.add_argument("--humans", choices=("orca", "social_force"), default="orca")
    a = ap.parse_args()
    rec = {}
    with mp.get_context("spawn").Pool(a.procs) as pool:
        for name, policy in BASELINES.items():
            edges = np.linspace(0, TEST_SIZE, 4 * a.procs + 1).astype(int)
            rows = [r for block in pool.map(run_block, [(policy, a.humans, lo, hi) for lo, hi in zip(edges[:-1], edges[1:])])
                    for r in block]
            rows.sort()
            rec[name + "_code"] = np.array([r[1] for r in rows], np.int32)
            rec[name + "_nav_time"] = np.array([r[2] for r in rows])
            rec[name + "_path_len"] = np.array([r[3] for r in rows])
            rec[name + "_too_close"] = np.array([r[4] for r in rows], np.int32)
            rec[name + "_steps"] = np.array([r[6] for r in rows], np.int32)
            rec[name + "_min_dist_count"] = np.array([len(r[5]) for r in rows], np.int32)
            rec[name + "_min_dist"] = np.array([x for r in rows for x in r[5]])
            codes = rec[name + "_code"]
            print(name, "success %.2f collision %.2f timeout %.2f" % tuple(np.mean(codes == c) for c in (3, 2, 1)))
    fname = "eval_baselines.npz" if a.humans == "orca" else "eval_baselines_sf_humans.npz"
    path = os.path.join(REPO, "tests", "golden", fname)
    np.savez_compressed(path, **rec)
    print("wrote", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    main()
