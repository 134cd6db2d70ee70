"""Cost of robot.visible = True (the humans' solves take the robot as one more agent) at 4096 environments x 20 humans,
for CrowdSimVarNum-v0 and for the GST configuration (CrowdSimPredRealGST-v0 + VecPretextNormalize, BASELINE config 3).

Visible and invisible runs alternate inside one call (--reps rounds of invisible, visible), each on a fresh engine with
the same seed.  Per run: the rollout step (policy act + environment step, CUDA events over --steps steps after --warmup)
and the environment step alone (the engine's step_device with the last actions; for the GST configuration the wrapper's
step, i.e. environment + predictor), then a profiled window with the env launches' times, the humans whose solve needed
linearProgram3 and the human rows the policy computed.  One JSON line per run, then one summary line with the card's name
and power limit.

    python tools/bench_robot_visible.py [--steps 200] [--warmup 40] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

N, H = 4096, 20


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


def measure(kind, visible, steps, warmup):
    import numpy as np
    import torch
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv, CudaPretextVecEnv
    from crowdnav_prediction_attngraph_b200.policy import Policy
    dev = torch.device("cuda", 0)
    kw = dict(num_envs=N, nenv_total=N, seed=425, human_num=H, robot_visible=int(visible), device=dev)
    if kind == "gst":
        params = dict(np.load(os.path.join(REPO, "tests", "golden", "gst_params.npz")))
        env = CudaPretextVecEnv(params, **kw)
    else:
        env = CudaCrowdVecEnv(const_vel=0, **kw)

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, 30, 2
    torch.manual_seed(425)
    policy = Policy(env.observation_space.spaces, env.action_space, base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    eng = policy._engine(N, dev)
    obs = env.reset()
    h = torch.zeros(N, 1, 128, device=dev)
    masks = torch.ones(N, 1, device=dev)
    action = None

    def step(obs, h, masks):
        value, action, logp, h2 = eng.act(obs, h, masks)
        obs, rew, done, info = env.step_device(action)
        return obs, h2, (1.0 - done.float()).unsqueeze(1), action

    for _ in range(warmup):
        obs, h, masks, action = step(obs, h, masks)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        obs, h, masks, action = step(obs, h, masks)
    e1.record()
    torch.cuda.synchronize()
    ms_rollout = e0.elapsed_time(e1) / steps
    act = action.clone()
    for _ in range(10):
        env.step_device(act)
    torch.cuda.synchronize()
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record()
    for _ in range(steps):
        env.step_device(act)
    f1.record()
    torch.cuda.synchronize()
    ms_env = f0.elapsed_time(f1) / steps
    # where the rollout step goes (a separate window: profile mode serialises the side streams' joins): the env
    # launches' CUDA-event times, the humans whose ORCA solve fell through to linearProgram3 and the human rows the
    # policy computes (it compacts the rows of humans the robot sees)
    import ctypes as C
    from crowdnav_prediction_attngraph_b200 import _capi
    core = env.env if kind == "gst" else env
    lib = core.lib
    lib.cn_env_profile(core._h, 1)
    eng.lib.cn_policy_profile(eng._h, 1)
    ns = eng.lib.cn_policy_stage_count()
    names = [eng.lib.cn_policy_stage_name(i).decode() for i in range(ns)]
    reps, stage, lp3, rows, pstage = 20, [0.0] * 3, 0.0, 0.0, [0.0] * ns
    for _ in range(reps):
        obs, h, masks, action = step(obs, h, masks)
        pbuf = (C.c_float * ns)()
        _capi.check(eng.lib, eng.lib.cn_policy_stage_ms(eng._h, pbuf, ns), "cn_policy_stage_ms")
        pstage = [s + b / reps for s, b in zip(pstage, pbuf)]
        buf = (C.c_float * 3)()
        _capi.check(lib, lib.cn_env_stage_ms(core._h, buf), "cn_env_stage_ms")
        stage = [s + b / reps for s, b in zip(stage, buf)]
        lp3 += float(core.get_state("lp_cost").sum()) / reps
        rows += float(eng.lib.cn_policy_last_rows(eng._h)) / reps
    lib.cn_env_profile(core._h, 0)
    eng.lib.cn_policy_profile(eng._h, 0)
    overflow = int(env.get_state("spawn_overflow").sum())
    env.close()
    del eng, policy, env
    torch.cuda.empty_cache()
    return dict(config=kind, robot_visible=int(visible), envs=N, humans=H, rollout_ms_per_step=ms_rollout,
                env_ms_per_step=ms_env,
                profiled_ms=dict(env_step_kernel=stage[0], env_event_kernels_side=stage[1], env_presolve_side=stage[2],
                                 policy_total=sum(pstage), **{"policy_" + n: round(v, 4) for n, v in zip(names, pstage)}),
                lp3_humans_per_step=lp3, policy_human_rows_per_step=rows, spawn_overflow_envs=overflow)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--configs", default="varnum,gst")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_robot_visible.py measures on a CUDA device; none is available")
    runs = []
    for kind in a.configs.split(","):
        for _ in range(a.reps):
            for visible in (False, True):
                r = measure(kind, visible, a.steps, a.warmup)
                print(json.dumps(r), flush=True)
                runs.append(r)
    summary = dict(card=card(), steps=a.steps, warmup=a.warmup, reps=a.reps)
    for kind in a.configs.split(","):
        for key in ("rollout_ms_per_step", "env_ms_per_step", "env_step_kernel", "env_presolve_side", "policy_total",
                    "lp3_humans_per_step", "policy_human_rows_per_step"):
            for v in (0, 1):
                xs = [r["profiled_ms"][key] if key in r["profiled_ms"] else r[key]
                      for r in runs if r["config"] == kind and r["robot_visible"] == v]
                summary["%s_%s_%s" % (kind, key, "visible" if v else "invisible")] = [round(x, 4) for x in xs]
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
