#!/usr/bin/env python
"""Benchmark of the DS-RNN policy (base='srnn') on CrowdSimVarNum-v0 (W = 2), default N = 4096, H = 20.

Prints, from one run on one GPU: the card name and power limit; the per-stage times of cn_dsrnn_act (CUDA events,
median over --profile-calls calls) and the edge GRU's achieved TFLOP/s (shape-derived FLOPs of the three fp16 products of
its 3xFP16 GEMM: 3 x 2 M 1024 320, against the 989 TFLOP/s dense fp16 data-sheet figure); the engine's act time
alternated with the reference's own SRNN module (rl.networks.model.Policy(base='srnn').act with args.env_type =
'crowd_sim', default torch settings, on the same card and inputs) when tools/stage_reference.py has staged the
unmodified reference under baseline/_ref (or $CROWDNAV_REFERENCE_ROOT names a checkout), else the same forward in
PyTorch eager from oracle/dsrnn_ref.py; "compared_with" names which one was timed; the device-resident rollout step
(act + env step into the rollout storage) in env-steps/s; and one PPO update (PyTorch, cuDNN GRUs).
Writes nothing to the repository."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name(0)


def reference_srnn(N, H, dev):
    """The unmodified reference's DS-RNN Policy (behind oracle/shims), or None when no reference is staged."""
    for root in (os.path.join(REPO, "baseline", "_ref"), os.environ.get("CROWDNAV_REFERENCE_ROOT", "")):
        if root and os.path.isfile(os.path.join(root, "rl", "networks", "srnn_model.py")):
            break
    else:
        return None
    sys.path[:0] = [os.path.join(REPO, "oracle", "shims"), root]
    import numpy as np
    import gym
    from arguments import get_args
    from rl.networks.model import Policy
    argv = sys.argv
    sys.argv = ["x", "--env-name", "CrowdSimVarNum-v0", "--num-processes", str(N)]
    try:
        args = get_args()
    finally:
        sys.argv = argv
    args.env_type = 'crowd_sim'      # arguments.py never defines it and SRNN.__init__ reads it (DESIGN.md 3.11)
    sp = {"robot_node": gym.spaces.Box(-np.inf, np.inf, (1, 7)), "temporal_edges": gym.spaces.Box(-np.inf, np.inf, (1, 2)),
          "spatial_edges": gym.spaces.Box(-np.inf, np.inf, (H, 2)),
          "detected_human_num": gym.spaces.Box(-np.inf, np.inf, (1,))}
    act = gym.spaces.Box(-np.inf * np.ones(2), np.inf * np.ones(2), dtype=np.float32)
    return Policy(sp, act, base_kwargs=args, base='srnn').to(dev)


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--humans", type=int, default=20)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--profile-calls", type=int, default=11)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dsrnn needs a CUDA device"
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200 import ppo
    from oracle.dsrnn_ref import DsrnnRef

    class Args(object):
        num_processes, seq_length, num_mini_batch = a.envs, a.steps, 2
        human_node_rnn_size, human_human_edge_rnn_size = 128, 256
    N, H, dev = a.envs, a.humans, torch.device("cuda:0")
    res = {"card": card(), "N": N, "H": H}
    torch.manual_seed(0)
    env = CudaCrowdVecEnv(num_envs=N, human_num=H, seed=425, device=dev, const_vel=0)
    sp = env.observation_space.spaces
    pol = Policy(sp, env.action_space, base='srnn', base_kwargs=Args()).to(dev)
    obs = env.reset()
    obs = {k: v for k, v in obs.items() if k in ("robot_node", "temporal_edges", "spatial_edges", "detected_human_num")}
    h = torch.randn(N, 1, 128, device=dev) * 0.5
    he = torch.randn(N, H + 1, 256, device=dev) * 0.5
    masks = torch.ones(N, 1, device=dev)
    eng = pol._engine(N, dev)
    run_eng = lambda: eng.act(obs, h, he, masks)                               # noqa: E731
    ref, kind = reference_srnn(N, H, dev), "reference rl.networks.model.Policy(base='srnn'), env_type 'crowd_sim'"
    if ref is None:
        ref, kind = DsrnnRef(2).to(dev), "oracle/dsrnn_ref.py (PyTorch eager restatement; no staged reference)"
    ref.load_state_dict(pol.state_dict())
    res["compared_with"] = kind

    def ref_forward():
        if isinstance(ref, DsrnnRef):
            v_, m_, _, e_ = ref(obs, h, he, masks)
            return v_, m_, e_
        v_, feat, hx = ref.base(obs, {'human_node_rnn': h, 'human_human_edge_rnn': he}, masks, infer=True)
        return v_, ref.dist.fc_mean(feat), hx['human_human_edge_rnn']

    def run_ref():
        with torch.no_grad():
            if isinstance(ref, DsrnnRef):
                ref(obs, h, he, masks)
            else:
                ref.act(obs, {'human_node_rnn': h, 'human_human_edge_rnn': he}, masks)
    run_eng(); run_ref(); torch.cuda.synchronize()
    with torch.no_grad():
        v_ref, m_ref, e_ref = ref_forward()
    v, _, _, _, e, m = eng.act(obs, h, he, masks, deterministic=True, return_mean=True)
    res["max_abs_err_vs_compared"] = {"value": float((v - v_ref).abs().max()), "mean": float((m - m_ref).abs().max()),
                                      "edge": float((e - e_ref).abs().max())}
    t_eng, t_ref = [], []
    for _ in range(a.rounds):                       # alternated, so both see the same card state
        t_eng.append(timed(run_eng, a.reps))
        t_ref.append(timed(run_ref, a.reps))
    res["act_ms_engine"], res["act_ms_compared"] = min(t_eng), min(t_ref)
    res["act_ms_engine_all"], res["act_ms_compared_all"] = t_eng, t_ref
    eng.profile(True)
    samples = []
    for _ in range(a.profile_calls):
        run_eng()
        samples.append(eng.stage_ms())
    eng.profile(False)
    stages = {k: statistics.median(s_[k] for s_ in samples) for k in samples[0]}
    res["stage_ms_median_of"] = a.profile_calls
    res["stage_ms"] = stages
    flop = 3 * 2.0 * (N * H) * 1024 * 320
    res["spatial_edge_gru_tflops"] = flop / (stages["spatial_edge_gru"] * 1e-3) / 1e12
    res["spatial_edge_gru_share_of_989"] = res["spatial_edge_gru_tflops"] / 989.0
    # device-resident rollout step into the storage + one PPO update
    T = a.steps
    st = RolloutStorage(T, N, sp, env.action_space, 128, 256, device=dev)
    o = env.reset()
    for k in st.obs:
        st.obs[k][0].copy_(o[k])
    st.rollout_step_zero_copy(eng, env)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(T - 1):
        st.rollout_step_zero_copy(eng, env)
    torch.cuda.synchronize()
    res["rollout_env_steps_per_s"] = N * (T - 1) / (time.perf_counter() - t0)
    with torch.no_grad():
        nv = pol.get_value({k: st.obs[k][-1] for k in st.obs}, {k: st.recurrent_hidden_states[k][-1]
                                                                 for k in st.recurrent_hidden_states}, st.masks[-1])
    st.compute_returns(nv, True, 0.99, 0.95, False)
    agent = ppo.PPO(pol, 0.2, 1, 2, 0.5, 0.0, lr=4e-5, eps=1e-5, max_grad_norm=0.5)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    agent.update(st)
    torch.cuda.synchronize()
    res["ppo_update_s_1_epoch_2_minibatches"] = time.perf_counter() - t0
    res["peak_mem_gb"] = torch.cuda.max_memory_allocated() / 1e9
    env.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
