"""Cost of CrowdSimPred-v0 with sim.predict_method = 'truth' against 'const_vel'.

With 'truth' every observation runs the ground-truth look-ahead: predict_steps * pred_interval nested ORCA solves of the
humans, so a phase-'train' step runs 1 + 5 solves instead of 1 (and phase 'test' 1 + 5 + 5 instead of 1 + 5); the
side-stream ORCA pre-solve is off for 'truth'.

1. Environment step: step_device with one fixed random action per environment; the mean wall time per step (CUDA
   events over --steps steps after --warmup) and, in a separate profiled window, the median step-kernel time
   (cn_env_stage_ms).
2. Device-resident rollout: the attention-graph policy's act, the step and the storage insert without host round trips
   (RolloutStorage.rollout_step_zero_copy, as bench.py's headline number), --steps steps after --warmup.

Sizes: 4096 environments x 20 humans and 2048 x 50 (circle and arena x 1.5), phase 'train', the reference's default
attributes; and 4096 x 20 in phase 'test' for the step.  The two methods alternate, each on a fresh engine with the same
seed.  One JSON line per run, then one summary line (env-steps/s) with the card's name, power limit and clocks.

    python tools/bench_truth_pred.py [--steps 200] [--warmup 60] [--reps 2]
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

METHODS = {1: "const_vel", 2: "truth"}
SIZES = [(4096, 20, 0), (2048, 50, 0), (4096, 20, 2)]          # (N, H, phase)
SCALE = {20: 1.0, 50: 1.5}


def card():
    import torch
    out = dict(name=torch.cuda.get_device_name(0))
    try:
        out["nvidia_smi"] = subprocess.check_output(
            ["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader", "-i", "0"],
            text=True).strip()
    except (OSError, subprocess.CalledProcessError) as e:
        out["nvidia_smi"] = "unavailable: %s" % e
    return out


def _env(N, H, phase, method):
    import torch
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    s = SCALE[H]
    return CudaCrowdVecEnv(num_envs=N, nenv_total=N, seed=425, human_num=H, const_vel=method, phase=phase,
                           circle_radius=s * 6 * 2 ** 0.5, arena_size=s * 6.0, device=torch.device("cuda", 0))


def measure_step(N, H, phase, method, steps, warmup):
    import ctypes as C

    import numpy as np
    import torch
    from crowdnav_prediction_attngraph_b200 import _capi
    env = _env(N, H, phase, method)
    act = torch.from_numpy(np.random.RandomState(3).uniform(-1.2, 1.2, (N, 2)).astype(np.float32)).to(env.device)
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
        rows.append(buf[0])
    env.lib.cn_env_profile(env._h, 0)
    overflow = int(env.get_state("spawn_overflow").sum())
    env.close()
    torch.cuda.empty_cache()
    return dict(kind="step", envs=N, humans=H, phase="test" if phase == 2 else "train", method=METHODS[method],
                wall_ms_per_step=round(wall, 4), step_kernel_median_ms=round(float(np.median(rows)), 4),
                env_steps_per_s=round(N / wall * 1000.0), spawn_overflow_envs=overflow)


def measure_rollout(N, H, method, steps, warmup):
    import torch
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    env = _env(N, H, 0, method)
    dev = env.device
    T = 30

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, T, 2
    torch.manual_seed(425)
    policy = Policy(env.observation_space.spaces, env.action_space, base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    ro = RolloutStorage(T, N, env.observation_space.spaces, env.action_space, 128, 256, device=dev)
    obs = env.reset()
    for k in ro.obs:
        ro.obs[k][0].copy_(obs[k])
    eng = policy._engine(N, dev)

    def step():
        ro.rollout_step_zero_copy(eng, env)
        if ro.step == 0:
            ro.after_update()
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    env.close()
    del eng, policy, ro, env
    torch.cuda.empty_cache()
    return dict(kind="rollout", envs=N, humans=H, phase="train", method=METHODS[method], ms_per_step=round(ms, 4),
                env_steps_per_s=round(N / ms * 1000.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=60)
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_truth_pred.py measures on a CUDA device; none is available")
    runs = []
    for _ in range(a.reps):
        for N, H, phase in SIZES:
            for m in (1, 2):
                runs.append(measure_step(N, H, phase, m, a.steps, a.warmup))
                print(json.dumps(runs[-1]), flush=True)
        for N, H, phase in SIZES:
            if phase == 0:
                for m in (1, 2):
                    runs.append(measure_rollout(N, H, m, a.steps, a.warmup))
                    print(json.dumps(runs[-1]), flush=True)
    summary = dict(card=card(), steps=a.steps, warmup=a.warmup, reps=a.reps)
    for r in runs:
        key = "%s_N%d_H%d_%s_%s_env_steps_per_s" % (r["kind"], r["envs"], r["humans"], r["phase"], r["method"])
        summary.setdefault(key, []).append(r["env_steps_per_s"])
        if r["kind"] == "step":
            summary.setdefault(key.replace("env_steps_per_s", "kernel_ms"), []).append(r["step_kernel_median_ms"])
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
