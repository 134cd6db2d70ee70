"""Per-stage GPU times of the rollout policy forward (cn_policy_act) on its own, without the environment.

bench.py's breakdown_ms times the stages while the environment's pre-solve runs on its side stream, so those numbers
include contention for SMs.  This script calls cn_policy_act alone at N = 4096, H = 20 with a bench-like distribution
of detected humans (mean about 4.2), takes the stage times from cn_policy_profile / cn_policy_stage_ms and prints the
median over the timed calls.  It also prints, computed from the shapes, the rows, output tiles, L2 -> shared-memory
operand bytes and issued FLOPs of the three BN = 256 GEMMs (embed2, qkv, outproj), with the card name and power limit.

--no-self-attn times the network without human-human attention (the reference's use_self_attn = False) instead: its
stages, the whole act (CUDA events around cn_policy_act alone, profiling off) and the device-resident rollout rate of
CrowdSimPred-v0 (env step + act into the rollout storage, as bench.py's value rate, at --humans).

    python tools/policy_stage_times.py [--envs 4096] [--humans 20] [--reps 300] [--warmup 30] [--seed 0] [--no-self-attn]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402

from crowdnav_prediction_attngraph_b200.policy import CudaPolicy, make_reference_like_state_dict  # noqa: E402

BM = 128            # output tile rows of cn_gemm_tc_kernel
BN = 256            # output tile columns of the per-human GEMMs
# (name, stage, K, N) of the per-human 3xFP16 GEMMs
GEMMS = [("embed2", "embed2_gemm", 128, 512), ("qkv", "qkv_gemm", 512, 1536), ("outproj", "outproj_spatial_gemm", 512, 256)]
GEMMS_NSA = [("spatial2", "spatial_linear2", 128, 256)]      # no_self_attn: its only per-human tensor-core GEMM


def gemm_counts(rows, K, N):
    """Output tiles, operand bytes moved from L2 into shared memory and issued tensor-core FLOPs of one launch.
    Each k-element of a 128 x 256 tile loads A (hi, lo) for 128 rows and B (hi, lo) for 256 rows, 2 bytes each.
    Issued FLOPs count the three fp16 products (hi.hi, hi.lo, lo.hi) over whole 128-row tiles."""
    row_tiles = -(-rows // BM)
    col_tiles = N // BN
    a_bytes = row_tiles * col_tiles * K * BM * 2 * 2
    b_bytes = row_tiles * col_tiles * K * BN * 2 * 2
    return dict(row_tiles=row_tiles, tiles=row_tiles * col_tiles, l2_smem_MB=(a_bytes + b_bytes) / 1e6,
                issued_GFLOP=3 * 2.0 * row_tiles * BM * N * K / 1e9, alg_GFLOP=2.0 * rows * N * K / 1e9)


def card():
    out = dict(name=torch.cuda.get_device_name(0))
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        out["power_limit"], out["clocks_max_sm"] = [s.strip() for s in q.split(",")]
    except Exception as e:  # the timing does not depend on it; say why it is missing
        out["power_limit"] = "unavailable (%s)" % e
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--humans", type=int, default=20)
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--no-self-attn", action="store_true", help="the network without human-human attention")
    ap.add_argument("--rollout-steps", type=int, default=300, help="timed steps of the rollout rate (--no-self-attn)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("policy_stage_times.py needs a CUDA device")
    N, H, Win = a.envs, a.humans, 12
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(a.seed)
    # detected humans per environment: Binomial(H, 0.21) clamped to >= 1 (mean about 4.2 at H = 20, as in the bench)
    n = (torch.rand(N, H, generator=g) < 0.21).sum(1, keepdim=True).float().clamp_min(1)
    sp = torch.randn(N, H, Win, generator=g) * 3
    sp[torch.arange(H)[None, :] >= n] = 15.0
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=g) * 3, temporal_edges=torch.randn(N, 1, 2, generator=g),
               spatial_edges=sp, detected_human_num=n)
    obs = {k: v.to(dev) for k, v in obs.items()}
    h = (torch.randn(N, 1, 128, generator=g) * 0.5).to(dev)
    masks = torch.ones(N, 1, device=dev)
    noise = torch.randn(N, 2, generator=g).to(dev)

    self_attn = not a.no_self_attn
    pol = CudaPolicy(N, H, Win, device=dev, self_attn=self_attn)
    pol.load_state_dict(make_reference_like_state_dict(input_size=Win, seed=0, self_attn=self_attn))
    lib = pol.lib
    ns = lib.cn_policy_stage_count()
    names = [lib.cn_policy_handle_stage_name(pol._h, i).decode() for i in range(ns)]
    names = [k for k in names if k]
    ns = len(names)
    lib.cn_policy_profile(pol._h, 1)
    buf = (C.c_float * ns)()
    samples = {k: [] for k in names}
    totals = []
    for i in range(a.warmup + a.reps):
        pol.act(obs, h, masks, noise=noise)
        rc = lib.cn_policy_stage_ms(pol._h, buf, ns)          # synchronises on the last stage's event
        if rc:
            raise SystemExit("cn_policy_stage_ms failed")
        if i >= a.warmup:
            for k, v in zip(names, buf):
                samples[k].append(v)
            totals.append(sum(buf))
    lib.cn_policy_profile(pol._h, 0)
    rows = int(lib.cn_policy_last_rows(pol._h))
    med = {k: statistics.median(v) for k, v in samples.items()}

    info = card()
    print("card: %s, power limit %s, max SM clock %s" % (info["name"], info.get("power_limit"), info.get("clocks_max_sm")))
    print("N = %d, H = %d, compacted rows Mc = %d (mean detected humans %.3f), %d timed calls after %d warm-up"
          % (N, H, rows, rows / N, a.reps, a.warmup))
    print("%-22s %9s %9s %9s" % ("stage", "median", "min", "max"))
    for k in names:
        print("%-22s %9.4f %9.4f %9.4f" % (k, med[k], min(samples[k]), max(samples[k])))
    print("%-22s %9.4f" % ("sum of stages", statistics.median(totals)))
    print("%-8s %6s %6s %6s %12s %10s %8s %12s %12s" % ("gemm", "K", "N", "tiles", "L2->smem MB", "issued GF", "alg GF",
                                                        "issued TF/s", "L2->smem TB/s"))
    shapes = {}
    for name, stage, K, Ncol in (GEMMS if self_attn else GEMMS_NSA):
        c = gemm_counts(rows, K, Ncol)
        shapes[name] = dict(K=K, N=Ncol, tiles=c["tiles"], l2_smem_MB=round(c["l2_smem_MB"], 1),
                            issued_GFLOP=round(c["issued_GFLOP"], 2), alg_GFLOP=round(c["alg_GFLOP"], 2))
        print("%-8s %6d %6d %6d %12.1f %10.2f %8.2f %12.1f %12.2f" % (
            name, K, Ncol, c["tiles"], c["l2_smem_MB"], c["issued_GFLOP"], c["alg_GFLOP"], c["issued_GFLOP"] / med[stage],
            c["l2_smem_MB"] / 1e3 / med[stage]))
    extra = {}
    if not self_attn:
        extra["act_ms"] = round(whole_act_ms(pol, obs, h, masks, noise, a.warmup, a.reps), 5)
        extra["rollout"] = rollout_rate(N, H, dev, a.warmup, a.rollout_steps)
        print("whole act (profiling off): %.4f ms median" % extra["act_ms"])
        print("device-resident rollout, CrowdSimPred-v0, N = %d, H = %d: %.3f M env-steps/s (%.4f ms per step)"
              % (N, H, extra["rollout"]["env_steps_per_s"] / 1e6, extra["rollout"]["ms_per_step"]))
    print(json.dumps(dict(card=info, N=N, H=H, self_attn=self_attn, rows=rows, reps=a.reps,
                          median_ms={k: round(v, 5) for k, v in med.items()},
                          sum_median_ms=round(statistics.median(totals), 5), gemms=shapes, **extra)))


def whole_act_ms(pol, obs, h, masks, noise, warmup, reps):
    """Median of CUDA-event times around single act calls (profiling off)."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for i in range(warmup + reps):
        e0.record()
        pol.act(obs, h, masks, noise=noise)
        e1.record()
        e1.synchronize()
        if i >= warmup:
            out.append(e0.elapsed_time(e1))
    return statistics.median(out)


def rollout_rate(N, H, dev, warmup, steps):
    """env step + act of the use_self_attn = False policy into the rollout storage, everything on the device
    (RolloutStorage.rollout_step_zero_copy, as bench.py's value rate); env-steps/s over `steps` timed steps."""
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    T = 30
    env = CudaCrowdVecEnv(num_envs=N, seed=425, human_num=H, device=dev)

    class Args(object):
        num_processes, seq_length, num_mini_batch, use_self_attn = N, T, 2, False
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
    for _ in range(warmup + 400):           # burn-in: episodes desynchronise, as bench.py's --burn-in
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / steps
    env.close()
    return dict(env_steps_per_s=round(N / ms * 1e3, 1), ms_per_step=round(ms, 5), steps=steps)


if __name__ == "__main__":
    main()
