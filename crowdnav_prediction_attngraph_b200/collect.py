"""Data collection on the engine: CrowdSimVarNumCollect-v0 and collect_data.py's dataset writer.

`CudaCollectVecEnv` is what make_vec_envs('CrowdSimVarNumCollect-v0', ...) returns: N collect environments on one GPU
whose observation is {'pred_info': [N, H, 4]} (frame, prediction id, px, py; inf for humans the robot does not see).
With wrap_pytorch=False (what collect_data.py asks for) reset / step return numpy arrays like ShmemVecEnv, with
wrap_pytorch=True device tensors.

`collect_dataset` writes the per-environment text files collect_data.py writes, byte for byte, without a host round trip
per step: a device recorder (cn_recorder_*) keeps a chunk of observations on the GPU, compacts their visible rows and
copies them to the host once per chunk; a writer thread formats and writes chunk k while the GPU steps chunk k + 1.

    python -m crowdnav_prediction_attngraph_b200.collect --num-envs 4096 --frames 40000 --out datasets/orca_20humans
"""
import argparse
import copy
import ctypes as C
import os
import threading
import time
import types

import numpy as np
import torch

from . import _capi
from .vec_env import COLLECT_ENV, LazyInfos, _trace, config_dict_from_reference

_STATE_DT = dict(rpx="f8", rpy="f8", rgx="f8", rgy="f8", rvx="f4", rvy="f4", hpx="f8", hpy="f8", hgx="f8", hgy="f8",
                 hrad="f8", hvpref="f8", hvx="f4", hvy="f4", vis="u1", step_count="i4", case_counter="u4", mt="u4",
                 mt_pos="i4", pred_id="i4", max_id="i4", rgoal_due="u1", rgoal_med="f8", rwx="f8", rwy="f8", evt="u1")


class CudaCollectVecEnv(object):
    """N CrowdSimVarNumCollect-v0 environments resident on one GPU (crowd_sim_var_num_collect.py)."""

    def __init__(self, device=None, cfg=None, wrap_pytorch=False, **cfg_over):
        self.lib = _capi.load_library()
        self.device = torch.device(device if device is not None else "cuda:0")
        if self.device.type != "cuda":
            raise RuntimeError("CudaCollectVecEnv needs a CUDA device (no CPU fallback)")
        d = dict(cfg) if cfg is not None else _capi.default_config_dict(const_vel=0, sort_humans=0)
        d.update(cfg_over)
        d["device"] = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.cfgd = d
        self.wrap_pytorch = wrap_pytorch
        self._cfg = _capi.config_from_dict(d)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            _capi.check(self.lib, self.lib.cn_env_create_collect(C.byref(self._cfg), C.byref(self._h)),
                        "cn_env_create_collect")
        self.closed = False
        N, H = d["num_envs"], d["human_num"]
        self.num_envs, self.human_num = N, H
        dev = self.device
        self._pi = [torch.zeros(N, H, 4, device=dev) for _ in range(2)]      # double-buffered observation
        self._flip = 0
        layout = [("ep_ret", torch.float64), ("reward", torch.float32), ("info", torch.int32),
                  ("info_aux", torch.float32), ("ep_len", torch.int32), ("done", torch.uint8)]
        self._out = {k: torch.zeros(N, dtype=dt, device=dev) for k, dt in layout}
        self._outp = _capi.CnStepPtrs(*[self._out[k].data_ptr() if k in self._out else None
                                        for k, _ in _capi.CnStepPtrs._fields_])
        self._t_start = time.time()
        _trace("engine CudaCollectVecEnv N=%d (of %d, offset %d) H=%d robot_policy=%d device=%s" % (
            N, d["nenv_total"], d["rank_offset"], H, d["robot_policy"], dev))

    def _stream(self):
        return _capi.raw_stream(self.device.index or 0)

    # ------------------------------------------------------------------ device-resident surface
    def reset_device(self):
        self._flip ^= 1
        pi = self._pi[self._flip]
        _capi.check(self.lib, self.lib.cn_env_reset_collect(self._h, C.c_void_p(pi.data_ptr()), self._stream()),
                    "cn_env_reset_collect")
        return pi

    def step_device(self, actions):
        """(pred_info [N,H,4], reward [N] f32, done [N] u8, info [N] i32) as device tensors, valid for one more step."""
        if not torch.is_tensor(actions):
            actions = torch.as_tensor(np.asarray(actions, dtype=np.float32))
        if actions.dtype != torch.float32 or not actions.is_cuda or not actions.is_contiguous():
            actions = actions.to(self.device, torch.float32).contiguous()
        assert actions.shape == (self.num_envs, 2)
        self._flip ^= 1
        pi = self._pi[self._flip]
        rc = self.lib.cn_env_step_collect(self._h, C.c_void_p(actions.data_ptr()), C.c_void_p(pi.data_ptr()),
                                          C.byref(self._outp), self._stream())
        if rc:
            _capi.check(self.lib, rc, "cn_env_step_collect")
        self._last_actions = actions            # keep the (possibly converted) actions alive until the step ran
        return pi, self._out["reward"], self._out["done"], self._out["info"]

    # ------------------------------------------------------------------ VecEnv surface
    def _wrap(self, pi):
        return {"pred_info": pi if self.wrap_pytorch else pi.cpu().numpy()}

    def reset(self):
        return self._wrap(self.reset_device())

    def step(self, actions):
        pi, rew, done, info = self.step_device(actions)
        o = {k: v.cpu().numpy() for k, v in self._out.items()}
        dn = o["done"].astype(bool)
        infos = LazyInfos(o["info"], o["info_aux"], dn, o["ep_ret"], o["ep_len"], self._t_start)
        reward = torch.from_numpy(o["reward"]).unsqueeze(1) if self.wrap_pytorch else o["reward"]
        return self._wrap(pi), reward, dn, infos

    def render(self, mode="human"):
        raise NotImplementedError("rendering is outside the engine's scope")

    def get_state(self, name):
        nbytes = self.lib.cn_env_state_bytes(self._h, name.encode())
        if not nbytes:
            raise KeyError(name)
        arr = np.zeros(nbytes // np.dtype(_STATE_DT[name]).itemsize, _STATE_DT[name])
        _capi.check(self.lib, self.lib.cn_env_state_copy(self._h, name.encode(), arr.ctypes.data, nbytes, 0),
                    "cn_env_state_copy")
        return arr

    def launch_count(self):
        return int(self.lib.cn_env_launch_count(self._h))

    def close(self):
        if not self.closed and self._h:
            self.lib.cn_env_destroy(self._h)
            self.closed = True

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def unwrapped(self):
        return self


class Recorder(object):
    """Device chunk of pred_info observations; flush() returns (rows [n,4] float32, rows per environment [N] int64)
    in collect_data.py's order: environment, then frame, then human index."""

    def __init__(self, num_envs, human_num, chunk_frames, device):
        self.lib = _capi.load_library()
        self.device = torch.device(device)
        self.N, self.H, self.C = num_envs, human_num, chunk_frames
        self._h = C.c_void_p()
        _capi.check(self.lib, self.lib.cn_recorder_create(num_envs, human_num, chunk_frames, self.device.index or 0,
                                                          C.byref(self._h)), "cn_recorder_create")

    def append(self, pred_info):
        assert pred_info.is_cuda and pred_info.is_contiguous() and pred_info.shape == (self.N, self.H, 4)
        _capi.check(self.lib, self.lib.cn_recorder_append(self._h, C.c_void_p(pred_info.data_ptr()),
                                                          _capi.raw_stream(self.device.index or 0)), "cn_recorder_append")

    def pending(self):
        return int(self.lib.cn_recorder_pending(self._h))

    def flush(self):
        rows = np.empty((self.N * self.H * max(self.pending(), 1), 4), np.float32)
        counts = np.zeros(self.N, np.int64)
        n = C.c_int64(0)
        _capi.check(self.lib, self.lib.cn_recorder_flush(self._h, rows.ctypes.data, counts.ctypes.data, C.byref(n),
                                                         _capi.raw_stream(self.device.index or 0)), "cn_recorder_flush")
        return rows[:n.value], counts

    def close(self):
        if self._h:
            self.lib.cn_recorder_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def write_rows_txt(directory, rows, env_rows, env_base=0, append=False):
    """<directory>/<env_base + e>.txt for every environment e: its rows (consecutive in `rows`) as collect_data.py
    writes them.  The C writer releases the GIL, so a thread can run it while the GPU steps on."""
    lib = _capi.load_library()
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    env_rows = np.ascontiguousarray(env_rows, dtype=np.int64)
    _capi.check(lib, lib.cn_write_rows_txt(directory.encode(), rows.ctypes.data, env_rows.ctypes.data, len(env_rows),
                                           env_base, 1 if append else 0), "cn_write_rows_txt")


def format_rows(rows):
    """The text collect_data.py writes for float32 rows [n, 4]."""
    lib = _capi.load_library()
    rows = np.ascontiguousarray(rows, dtype=np.float32).reshape(-1, 4)
    n = lib.cn_format_rows(rows.ctypes.data, len(rows), None, 0)
    buf = C.create_string_buffer(int(n))
    lib.cn_format_rows(rows.ctypes.data, len(rows), buf, n)
    return buf.raw[:n].decode()


def collect_dataset(config, num_envs, frames, out_dir, seed, train_data, device="cuda:0", chunk_frames=None):
    """collect_data.py's collectData on the engine: robot.policy 'orca', `num_envs` environments (phase 'train', seeds
    seed + i), zero actions, every pred_interval-th observation from the reset one on, `frames` observations per
    environment, files <out_dir>/{train|test}/<i>.txt.  Returns timings: device_s (stepping and recording),
    write_s (text formatting and writing, overlapped with the device work), total_s, rows, steps."""
    if getattr(getattr(config, "data", None), "render", False):
        raise NotImplementedError("rendering is outside the engine's scope (config.data.render only selects one "
                                  "environment in collect_data.py)")
    config = copy.deepcopy(config)
    config.robot.policy = "orca"                                  # collect_data.py:15
    device = torch.device(device)
    d = config_dict_from_reference(config, num_envs, seed, COLLECT_ENV, device_index=device.index or 0)
    env = CudaCollectVecEnv(device=device, cfg=d)
    N, H = env.num_envs, env.human_num
    pred_interval = int(config.data.pred_timestep // config.env.time_step)
    if chunk_frames is None:
        chunk_frames = max(1, min(frames, (1 << 21) // (N * H)))   # ~32 MB of rows per chunk
    rec = Recorder(N, H, chunk_frames, device)
    path = os.path.join(out_dir, "train" if train_data else "test")
    os.makedirs(path, exist_ok=True)
    zero = torch.zeros(N, 2, device=device)
    write_s = [0.0]
    pending = [None]

    def write(rows, counts, append):
        t = time.perf_counter()
        write_rows_txt(path, rows, counts, 0, append)
        write_s[0] += time.perf_counter() - t

    def hand_off(rows, counts, append):
        if pending[0] is not None:
            pending[0].join()
        th = threading.Thread(target=write, args=(rows, counts, append))
        th.start()
        pending[0] = th

    t0 = time.perf_counter()
    rows_total, first, steps = 0, True, 0
    with torch.cuda.device(device):
        obs = env.reset_device()
        for step in range((frames - 1) * pred_interval + 1):
            if step % pred_interval == 0:
                rec.append(obs)
                if rec.pending() == chunk_frames:
                    rows, counts = rec.flush()
                    rows_total += len(rows)
                    hand_off(rows, counts, not first)
                    first = False
            if step == (frames - 1) * pred_interval:
                break
            obs = env.step_device(zero)[0]
            steps += 1
        if rec.pending():
            rows, counts = rec.flush()
            rows_total += len(rows)
            hand_off(rows, counts, not first)
        torch.cuda.synchronize(device)
    t_dev = time.perf_counter() - t0
    if pending[0] is not None:
        pending[0].join()
    total = time.perf_counter() - t0
    rec.close()
    env.close()
    return dict(device_s=t_dev, write_s=write_s[0], total_s=total, rows=rows_total, steps=steps, num_envs=N,
                frames=frames)


def reference_default_config(human_num=20):
    """The fields collect_dataset reads, with the reference's crowd_nav/configs/config.py defaults."""
    ns = types.SimpleNamespace
    return ns(
        action_space=ns(kinematics="holonomic"),
        robot=ns(visible=False, policy="orca", radius=0.3, v_pref=1, FOV=2, sensor_range=5),
        humans=ns(policy="orca", radius=0.3, v_pref=1, FOV=2., random_goal_changing=True, end_goal_changing=True,
                  goal_change_chance=0.5),
        sim=ns(predict_method="none", human_num=human_num, human_num_range=0, predict_steps=5,
               circle_radius=6 * np.sqrt(2), arena_size=6),
        env=ns(randomize_attributes=True, time_step=0.25, time_limit=50, val_size=100, test_size=500),
        reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
        orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5),
        sf=ns(A=2., B=1, KI=1), data=ns(pred_timestep=0.25, render=False), args=ns(sort_humans=True))


def main(argv=None):
    ap = argparse.ArgumentParser(description="Write a GST training dataset (collect_data.py's files) on the GPU.")
    ap.add_argument("--num-envs", type=int, default=5)
    ap.add_argument("--frames", type=int, default=40000, help="observations per environment (config.data.tot_steps)")
    ap.add_argument("--out", required=True, help="config.data.data_save_dir")
    ap.add_argument("--seed", type=int, default=None, help="default: np.random.randint(0, 2**32 - 1), as collect_data.py")
    ap.add_argument("--human-num", type=int, default=20)
    ap.add_argument("--test-data", action="store_true", help="write <out>/test instead of <out>/train")
    ap.add_argument("--device", default="cuda:0")
    a = ap.parse_args(argv)
    seed = a.seed if a.seed is not None else int(np.random.randint(0, np.iinfo(np.uint32).max))
    r = collect_dataset(reference_default_config(a.human_num), a.num_envs, a.frames, a.out, seed, not a.test_data,
                        device=a.device)
    print("seed %d: %d environments x %d frames, %d rows; device %.2f s, writing %.2f s (overlapped), total %.2f s" % (
        seed, r["num_envs"], r["frames"], r["rows"], r["device_s"], r["write_s"], r["total_s"]))


if __name__ == "__main__":
    main()
