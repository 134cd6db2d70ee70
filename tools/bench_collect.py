#!/usr/bin/env python
"""Throughput of the data-collection path (CrowdSimVarNumCollect-v0 + the device recorder); prints one JSON line.

  collect_env_steps_per_s   collect step of N = 4096 environments x 20 humans, device-resident, zero actions
  recorded_rows_per_s       the same loop with every observation appended to the recorder and flushed per chunk
                            (rows copied to the host per second; text writing excluded)
  dataset_40k_*             collect_dataset of collect_data.py's default dataset: data.num_processes = 5
                            environments x data.tot_steps = 40 000 frames, files written, end to end; the text writer's
                            own time (overlapped with the device work) reported separately

    python tools/bench_collect.py [--envs 4096] [--steps 200] [--frames 40000] [--dataset-envs 5]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

import torch  # noqa: E402


def power_limit_w():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return float(out.splitlines()[0])
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--chunk", type=int, default=25)
    ap.add_argument("--frames", type=int, default=40000)
    ap.add_argument("--dataset-envs", type=int, default=5)
    a = ap.parse_args()
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.collect import CudaCollectVecEnv, Recorder, collect_dataset, \
        reference_default_config
    dev = torch.device("cuda:0")
    N, H = a.envs, 20
    d = _capi.default_config_dict(num_envs=N, nenv_total=N, human_num=H, const_vel=0, sort_humans=0,
                                  randomize_attributes=1, random_goal_changing=1, robot_policy=1, seed=425)
    env = CudaCollectVecEnv(device=dev, cfg=d)
    zero = torch.zeros(N, 2, device=dev)
    pi = env.reset_device()
    for _ in range(a.warmup):
        pi = env.step_device(zero)[0]
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        pi = env.step_device(zero)[0]
    e1.record()
    torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / a.steps
    # with the recorder: append every observation, flush every `chunk` frames (host copy included, no text)
    rec = Recorder(N, H, a.chunk, dev)
    rows = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        rec.append(pi)
        if rec.pending() == a.chunk:
            rows += len(rec.flush()[0])
        pi = env.step_device(zero)[0]
    if rec.pending():
        rows += len(rec.flush()[0])
    torch.cuda.synchronize()
    rec_s = time.perf_counter() - t0
    rec.close()
    env.close()
    with tempfile.TemporaryDirectory() as tmp:
        st = collect_dataset(reference_default_config(), a.dataset_envs, a.frames, tmp, 425, True)
        size = sum(os.path.getsize(os.path.join(r, f)) for r, _, fs in os.walk(tmp) for f in fs)
    print(json.dumps(dict(
        gpu=torch.cuda.get_device_name(0), power_limit_w=power_limit_w(), envs=N, humans=H,
        collect_step_ms=round(step_ms, 4), collect_env_steps_per_s=round(N / step_ms * 1e3),
        recorded_rows_per_s=round(rows / rec_s), recorded_env_steps_per_s=round(N * a.steps / rec_s),
        dataset_40k_envs=a.dataset_envs, dataset_40k_frames=a.frames, dataset_40k_rows=st["rows"],
        dataset_40k_bytes=size, dataset_40k_total_s=round(st["total_s"], 3), dataset_40k_device_s=round(st["device_s"], 3),
        dataset_40k_write_s=round(st["write_s"], 3),
        text_rows_per_s=round(st["rows"] / st["write_s"]) if st["write_s"] > 0 else None)))


if __name__ == "__main__":
    main()
