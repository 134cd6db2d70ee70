"""Cost of social-force humans in phase 'test' (the ground-truth look-ahead runs SOCIAL_FORCE.predict, cn_sf_lookahead)
against ORCA humans in phase 'test' (the look-ahead runs nested ORCA solves), CrowdSimVarNum-v0.

1. Environment step: for N in (500, 4096) and H in (20, 50, 100) (the circle and arena scaled by 1.5 / 2 at 50 / 100
   humans so that the spawn search finds room), ORCA and social-force engines alternate, each fresh with the same seed,
   stepped by step_device with one fixed random action per environment.  Per run: the mean wall time per step (CUDA
   events over --steps steps after --warmup) and, in a separate profiled window, the median over --steps steps of the
   engine's own stage times (cn_env_stage_ms: step kernel, side-stream event kernels, ORCA pre-solve).
2. Evaluation: the wall time of the 500-case evaluate_batched of the social-force robot among ORCA and among social-force
   humans (20 humans, seed 425), one untimed run first.

One JSON line per run, then one summary line with the card's name and power limit.

    python tools/bench_sf_test_phase.py [--steps 200] [--warmup 40] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

SCALE = {20: 1.0, 50: 1.5, 100: 2.0}
HUMANS = {0: "orca", 1: "social_force"}


def card():
    import torch
    out = dict(name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                                     "-i", "0"], text=True).strip()
        out["nvidia_smi"] = q
    except (OSError, subprocess.CalledProcessError) as e:
        out["nvidia_smi"] = "unavailable: %s" % e
    return out


def measure_step(N, H, human_policy, steps, warmup):
    import ctypes as C

    import numpy as np
    import torch
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    dev = torch.device("cuda", 0)
    s = SCALE[H]
    env = CudaCrowdVecEnv(num_envs=N, nenv_total=N, seed=425, human_num=H, const_vel=0, phase=2, test_size=500,
                          human_policy=human_policy, circle_radius=s * 6 * 2 ** 0.5, arena_size=s * 6.0, device=dev)
    act = torch.from_numpy(np.random.RandomState(3).uniform(-1.2, 1.2, (N, 2)).astype(np.float32)).to(dev)
    env.reset()
    for _ in range(warmup):
        env.step_device(act)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        env.step_device(act)
    e1.record()
    torch.cuda.synchronize()
    wall = e0.elapsed_time(e1) / steps
    env.lib.cn_env_profile(env._h, 1)
    rows = []
    for _ in range(steps):
        env.step_device(act)
        buf = (C.c_float * 3)()
        _capi.check(env.lib, env.lib.cn_env_stage_ms(env._h, buf), "cn_env_stage_ms")
        rows.append(list(buf))
    env.lib.cn_env_profile(env._h, 0)
    med = np.median(np.array(rows), axis=0)
    overflow = int(env.get_state("spawn_overflow").sum())
    env.close()
    torch.cuda.empty_cache()
    return dict(kind="step", envs=N, humans=H, human_policy=HUMANS[human_policy], wall_ms_per_step=round(wall, 4),
                median_ms=dict(step_kernel=round(float(med[0]), 4), event_kernels_side=round(float(med[1]), 4),
                               presolve_side=round(float(med[2]), 4)),
                spawn_overflow_envs=overflow)


def measure_eval(human_policy):
    import torch
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate_batched
    dev = torch.device("cuda", 0)
    d = _capi.default_config_dict(num_envs=500, nenv_total=1, seed=425, human_num=20, const_vel=0, phase=2,
                                  test_size=500, human_policy=human_policy, robot_policy=2)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = evaluate_batched(None, None, "CrowdSimVarNum-v0", 425, 500, dev, cfg_dict=d)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return dict(kind="eval500_sf_robot", human_policy=HUMANS[human_policy], wall_s=round(wall, 3),
                env_steps=int(sum(out["episode_steps"])), success_rate=out["success_rate"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_sf_test_phase.py measures on a CUDA device; none is available")
    runs = []
    for N in (500, 4096):
        for H in (20, 50, 100):
            for _ in range(a.reps):
                for hp in (0, 1):
                    r = measure_step(N, H, hp, a.steps, a.warmup)
                    print(json.dumps(r), flush=True)
                    runs.append(r)
    measure_eval(1)                                   # warm-up: module load, allocator
    for _ in range(a.reps):
        for hp in (0, 1):
            r = measure_eval(hp)
            print(json.dumps(r), flush=True)
            runs.append(r)
    summary = dict(card=card(), steps=a.steps, warmup=a.warmup, reps=a.reps)
    for r in runs:
        if r["kind"] == "step":
            key = "N%d_H%d_%s" % (r["envs"], r["humans"], r["human_policy"])
            summary.setdefault(key + "_step_kernel_ms", []).append(r["median_ms"]["step_kernel"])
            summary.setdefault(key + "_wall_ms", []).append(r["wall_ms_per_step"])
        else:
            summary.setdefault("eval500_sf_robot_%s_humans_s" % r["human_policy"], []).append(r["wall_s"])
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
