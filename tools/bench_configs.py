"""Informational device-rollout timings of BASELINE configs other than the bench line (bench.py times
configs[1]).  Same zero-copy rollout step as bench.py `value`; CUDA events; one JSON line per config.

    python tools/bench_configs.py [--steps 60] [--warmup 20] [--configs c2,c4]
"""
import argparse
import json
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

CONFIGS = {
    # name: (env kwargs, envs per GPU)
    "c2": (dict(human_num=20), 4096),
    "c4": (dict(human_num=50, randomize_attributes=1, random_goal_changing=1, goal_change_chance=0.5), 2048),
    "c2_h50": (dict(human_num=50), 4096),
    # BASELINE config 5 as bench.py runs it (circle and arena x2, see bench.py EXTRA_CONFIGS)
    "c5": (dict(human_num=100, circle_radius=2 * 6 * 2 ** 0.5, arena_size=12.0), 4096),
    "c1_varnum": (dict(human_num=5, const_vel=0), 4096),
    # BASELINE config 3: CrowdSimPredRealGST-v0 + VecPretextNormalize (GST predictor), H = 20, N = 4096
    "c3": (dict(human_num=20), 4096),
    # config 3 at config 4's and config 5's crowds (c3_h100: circle and arena x2, as c5)
    "c3_h50": (dict(human_num=50), 4096),
    "c3_h100": (dict(human_num=100, circle_radius=2 * 6 * 2 ** 0.5, arena_size=12.0), 4096),
}


def run(name, steps, warmup):
    import torch
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    kw, N = CONFIGS[name]
    dev = torch.device("cuda", 0)
    if name.startswith("c3"):
        return run_c3(name, kw, N, dev, steps, warmup)
    env = CudaCrowdVecEnv(num_envs=N, nenv_total=N, rank_offset=0, seed=425, device=dev, **kw)

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, 30, 2
    torch.manual_seed(425)
    policy = Policy(env.observation_space.spaces, env.action_space, base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    rollouts = RolloutStorage(30, N, env.observation_space.spaces, env.action_space, 128, 256, device=dev)
    obs = env.reset()
    for k in rollouts.obs:
        rollouts.obs[k][0].copy_(obs[k])
    eng = policy._engine(N, dev)

    def device_step():
        rollouts.rollout_step_zero_copy(eng, env)
        if rollouts.step == 0:
            rollouts.after_update()

    for _ in range(warmup):
        device_step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        device_step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    # env-only share: time the env step alone with the last actions
    act = rollouts.actions[rollouts.step - 1 if rollouts.step else 0]
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    f0.record()
    for _ in range(steps):
        env.step_device(act)
    f1.record()
    torch.cuda.synchronize()
    ms_env = f0.elapsed_time(f1) / steps
    # per-stage timing (CUDA events inside the library; profile mode serialises the side streams' joins)
    import ctypes as C
    from crowdnav_prediction_attngraph_b200 import _capi
    lib = eng.lib
    lib.cn_policy_profile(eng._h, 1)
    lib.cn_env_profile(env._h, 1)
    ns = lib.cn_policy_stage_count()
    names = [lib.cn_policy_stage_name(i).decode() for i in range(ns)]
    acc, est, reps = [0.0] * ns, [0.0] * 3, 5
    for _ in range(reps):
        s = rollouts.step
        o = {k: rollouts.obs[k][s] for k in rollouts.obs}
        value, action, logp, h_new = eng.act(o, rollouts.recurrent_hidden_states['human_node_rnn'][s], rollouts.masks[s])
        buf = (C.c_float * ns)()
        _capi.check(lib, lib.cn_policy_stage_ms(eng._h, buf, ns), "stage_ms")
        nobs, rew, done, info = env.step_device(action)
        ebuf = (C.c_float * 3)()
        _capi.check(lib, lib.cn_env_stage_ms(env._h, ebuf), "env_stage_ms")
        for i in range(ns):
            acc[i] += buf[i] / reps
        for i in range(3):
            est[i] += ebuf[i] / reps
        rollouts.insert(nobs, {'human_node_rnn': h_new}, action, logp, value, rew, (1.0 - done.float()).unsqueeze(1))
    stages = {"env_step_kernel": est[0], "env_event_kernels_side": est[1], "env_presolve_side": est[2]}
    stages.update({n: round(v, 4) for n, v in zip(names, acc)})
    overflow = int(env.get_state("spawn_overflow").sum())
    print(json.dumps({"config": name, "stages_ms": stages, "env_kwargs": kw, "envs": N, "ms_per_step": ms, "env_steps_per_s": N / ms * 1e3,
                      "env_only_ms_per_step": ms_env, "valid_human_rows": int(eng.lib.cn_policy_last_rows(eng._h)),
                      "spawn_overflow_envs": overflow, "defer_ctl": [int(x) for x in env.get_state("defer_ctl")]}))
    del eng, policy, env


def run_c3(name, kw, N, dev, steps, warmup):
    import numpy as np
    import torch
    from crowdnav_prediction_attngraph_b200.vec_env import CudaPretextVecEnv
    from crowdnav_prediction_attngraph_b200.policy import Policy
    params = dict(np.load(os.path.join(REPO, "tests", "golden", "gst_params.npz")))
    free0 = torch.cuda.mem_get_info(dev)[0]        # the engine's workspaces are cudaMalloc'd outside torch's allocator
    env = CudaPretextVecEnv(params, num_envs=N, nenv_total=N, rank_offset=0, seed=425, device=dev, **kw)

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, 30, 2
    torch.manual_seed(425)
    policy = Policy(env.observation_space.spaces, env.action_space, base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    eng = policy._engine(N, dev)
    obs = env.reset()
    h = torch.zeros(N, 1, 128, device=dev)
    masks = torch.ones(N, 1, device=dev)

    def step(obs, h, masks):
        value, action, logp, h2 = eng.act(obs, h, masks)
        obs, rew, done, info = env.step_device(action)
        return obs, h2, (1.0 - done.float()).unsqueeze(1)

    for _ in range(warmup):
        obs, h, masks = step(obs, h, masks)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        obs, h, masks = step(obs, h, masks)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    raw = env.env.reset()
    f0.record()
    for _ in range(20):
        env._process(raw, None)
    f1.record()
    torch.cuda.synchronize()
    print(json.dumps({"config": name, "env_kwargs": kw, "envs": N, "ms_per_step": ms, "env_steps_per_s": N / ms * 1e3,
                      "gst_pretext_kernel_ms": f0.elapsed_time(f1) / 20,
                      "valid_human_rows": int(eng.lib.cn_policy_last_rows(eng._h)),
                      "device_mem_gb": (free0 - torch.cuda.mem_get_info(dev)[0]) / 2 ** 30}))
    env.close()
    del eng, policy, env


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--configs", default="c2,c4")
    a = ap.parse_args()
    for c in a.configs.split(","):
        run(c, a.steps, a.warmup)
