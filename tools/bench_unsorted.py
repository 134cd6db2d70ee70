#!/usr/bin/env python
"""Cost of the policy on unsorted humans (args.sort_humans = False, cn_policy_config.visible_masks) against the sorted
policy, on the GPU.

  * `act`: N = 4096 at H = 20 / 50 / 100, a sorted and a visible_masks handle of the same weights, alternating in one
    process.  Both see the same number of rows per environment (the masked handle's mask holds as many visible slots
    as detected_human_num, spread over the slots), so the difference is the mask compaction and the slot gather.
    Device time per call (CUDA events over `--steps` calls) and the median of every stage (mask_rows is the
    compaction of the masked handle).
  * the device-resident rollout (policy act + environment step into RolloutStorage) on CrowdSimVarNum-v0 at N = 4096,
    H = 20, with sort_humans = True and False.

One JSON line per measurement, then the card's name, power limit and clocks.

    python tools/bench_unsorted.py [--steps 200] [--warmup 20] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)


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


def act_inputs(N, H, seed=3):
    import torch
    g = torch.Generator().manual_seed(seed)
    n = torch.randint(1, H + 1, (N, 1), generator=g)
    # the same count of visible slots, at random places
    key = torch.rand(N, H, generator=g)
    rank = key.argsort(1).argsort(1)
    vis = rank < n
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=g), temporal_edges=torch.randn(N, 1, 2, generator=g),
               spatial_edges=torch.randn(N, H, 12, generator=g), detected_human_num=n.float(), visible_masks=vis)
    obs = {k: v.cuda() for k, v in obs.items()}
    return obs, torch.randn(N, 1, 128, generator=g).cuda() * 0.5, torch.ones(N, 1).cuda()


def measure_act(N, H, steps, warmup, reps):
    import numpy as np
    import torch
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy, make_reference_like_state_dict
    sd = make_reference_like_state_dict(12, seed=1)
    obs, h, masks = act_inputs(N, H)
    pols = {vm: CudaPolicy(N, H, 12, device="cuda:0", visible_masks=vm) for vm in (False, True)}
    for p in pols.values():
        p.load_state_dict(sd)
    times = {vm: [] for vm in pols}
    stages = {vm: {} for vm in pols}
    for _ in range(reps):
        for vm, p in pols.items():
            for _ in range(warmup):
                p.act(obs, h, masks, deterministic=True)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                p.act(obs, h, masks, deterministic=True)
            e1.record()
            torch.cuda.synchronize()
            times[vm].append(e0.elapsed_time(e1) / steps)
            p.profile(True)
            for _ in range(min(steps, 50)):
                p.act(obs, h, masks, deterministic=True)
                for k, v in p.stage_ms().items():
                    stages[vm].setdefault(k, []).append(v)
            p.profile(False)
    rows = {vm: p.lib.cn_policy_last_rows(p._h) for vm, p in pols.items()}
    assert rows[False] == rows[True], rows
    out = []
    for vm in pols:
        out.append(dict(kind="act", envs=N, humans=H, handle="visible_masks" if vm else "sorted", rows=rows[vm],
                        ms_per_call=[round(t, 4) for t in times[vm]], ms_per_call_min=round(min(times[vm]), 4),
                        stage_median_ms={k: round(float(np.median(v)), 4) for k, v in stages[vm].items()}))
    for p in pols.values():
        p.close()
    torch.cuda.empty_cache()
    return out


def measure_rollout(N, H, sort_humans, steps, warmup):
    import types

    import torch
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    env = CudaCrowdVecEnv(num_envs=N, nenv_total=N, seed=425, human_num=H, const_vel=0, sort_humans=int(sort_humans),
                          randomize_attributes=1, random_goal_changing=1, device=torch.device("cuda", 0))
    dev = env.device
    T = 30
    args = types.SimpleNamespace(num_processes=N, seq_length=T, num_mini_batch=2, sort_humans=sort_humans)
    torch.manual_seed(425)
    policy = Policy(env.observation_space.spaces, env.action_space, base_kwargs=args, base='selfAttn_merge_srnn').to(dev)
    ro = RolloutStorage(T, N, env.observation_space.spaces, env.action_space, 128, 256, device=dev)
    obs = env.reset()
    for k in ro.obs:
        ro.obs[k][0].copy_(obs[k])
    eng = policy._engine(N, dev)
    assert eng.visible_masks == (not sort_humans)

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
    return dict(kind="rollout", env="CrowdSimVarNum-v0", envs=N, humans=H, sort_humans=sort_humans,
                ms_per_step=round(ms, 4), env_steps_per_s=round(N / ms * 1000.0))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--humans", type=int, nargs="*", default=[20, 50, 100])
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_unsorted.py needs a CUDA device")
    for H in a.humans:
        for r in measure_act(4096, H, a.steps, a.warmup, a.reps):
            print(json.dumps(r), flush=True)
    for rep in range(2):
        for sort_humans in (True, False):
            print(json.dumps(measure_rollout(4096, 20, sort_humans, a.steps, a.warmup)), flush=True)
    print(json.dumps(dict(kind="card", **card())), flush=True)


if __name__ == "__main__":
    main()
