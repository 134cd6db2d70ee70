"""Host-side mirror of the reference's vec-env surface over the CUDA engine.

`CudaCrowdVecEnv` keeps the contract of the wrapped `VecPyTorch(ShmemVecEnv(...))` object that
`make_vec_envs` returns in the reference (rl/networks/envs.py:97-140, 193-224;
rl/networks/shmem_vec_env.py:62-80): `reset()` -> dict of device tensors with leading dim N;
`step(action_tensor)` -> (obs dict on device, reward CPU float32 [N,1], done np.bool_[N],
infos sequence of dicts {'info': obj[, 'episode': {'r','l'}]}).  All N environments live in
HBM and one kernel launch advances them; there are no worker processes, pipes or pickles.

A zero-host-round-trip variant (`step_device`) returns reward/done/info as device tensors for the
device-resident rollout loop.
"""
import ctypes as C
import os
import time
from collections import OrderedDict

import numpy as np
import torch

from . import _capi

# crowd_sim/envs/utils/info.py equivalents (same __str__), index = CN_INFO_* code
class Nothing(object):
    def __str__(self):
        return ''


class Timeout(object):
    def __str__(self):
        return 'Timeout'


class Collision(object):
    def __str__(self):
        return 'Collision'


class ReachGoal(object):
    def __str__(self):
        return 'Reaching goal'


class Danger(object):
    def __init__(self, min_dist=0.0):
        self.min_dist = min_dist

    def __str__(self):
        return 'Too close'


_INFO_CLASSES = (Nothing, Timeout, Collision, ReachGoal, Danger)


def _trace(msg):
    """CROWDNAV_B200_TRACE=1: one stderr line per engine object (the drop-in tests look for it)."""
    if os.environ.get("CROWDNAV_B200_TRACE", "0") == "1":
        import sys
        sys.stderr.write("crowdnav_b200: %s\n" % msg)


class _Space(object):
    """Minimal Box-like descriptor (shape, dtype) — gym is not a dependency of the engine."""

    def __init__(self, shape, dtype=np.float32):
        self.shape = tuple(shape)
        self.dtype = np.dtype(dtype)
        self.low = -np.inf
        self.high = np.inf


class _DictSpace(object):
    def __init__(self, spaces):
        self.spaces = OrderedDict(sorted(spaces.items()))

    def __getitem__(self, k):
        return self.spaces[k]


class Box(_Space):
    pass


# robot.policy -> cn_config.robot_policy (0: the caller's action)
ROBOT_POLICIES = {"orca": 1, "social_force": 2}


def config_dict_from_reference(config, num_envs, seed, env_name, nenv_total=None, rank_offset=0, device_index=0,
                               phase=None, allow_unsorted=False):
    """Snapshot a reference `Config` object (crowd_nav/configs/config.py) into the flat cn_config.
    phase None follows rl/networks/envs.py:55-58: one environment -> 'test', more -> 'train'."""
    if phase is None:
        phase = "test" if (nenv_total or num_envs) == 1 else "train"
    if phase not in ("train", "test"):
        raise NotImplementedError("phase %r: the engine covers 'train' and 'test'" % (phase,))
    if config.action_space.kinematics != "holonomic":
        raise NotImplementedError("engine covers the holonomic robot")
    if config.humans.policy not in ("orca", "social_force"):
        raise NotImplementedError("humans.policy %r: the engine covers 'orca' and 'social_force'" % (config.humans.policy,))
    if env_name == "CrowdSimPred-v0":
        if config.sim.predict_method != "const_vel":
            raise NotImplementedError("CrowdSimPred-v0 is covered for predict_method='const_vel'")
        const_vel = 1
    elif env_name == "CrowdSimVarNum-v0":
        const_vel = 0
    else:
        raise NotImplementedError("env id %r is not covered by the CUDA engine" % env_name)
    robot_visible = bool(config.robot.visible)
    if robot_visible and const_vel:
        raise NotImplementedError(
            "robot.visible=True on CrowdSimPred-v0 is not covered: the reference cannot run it (calc_human_future_traj("
            "'const_vel') assigns prev_human_pos[:, 2:4], shape (H, 2), into an (H + 1, 2) slice, crowd_sim_var_num.py:"
            "155,174, and raises on the first reset)")
    # robot.policy 'orca' / 'social_force': the robot is driven inside env.step and the caller's action is ignored
    # (crowd_sim_var_num.py:371-377); any other name (a network policy) takes the caller's action
    robot_policy = ROBOT_POLICIES.get(getattr(config.robot, "policy", None), 0)
    if robot_policy:
        if const_vel:
            raise NotImplementedError(
                "robot.policy %r on CrowdSimPred-v0 is not covered: its ORCA branch (crowd_sim_pred.py:105-116) feeds the "
                "robot the ground-truth future trajectories ((predict_steps + 1) * human_num agents) and its "
                "social-force branch calls clip_action on a policy that has none" % (config.robot.policy,))
        if int(config.sim.human_num_range) > 0:
            raise NotImplementedError("robot.policy %r with sim.human_num_range > 0 is not covered (the robot's rvo2 "
                                      "simulator would be rebuilt as humans join and leave)" % (config.robot.policy,))
    sort_humans = getattr(getattr(config, "args", None), "sort_humans", True)
    if not sort_humans and not allow_unsorted:
        # the policy mirror masks attention with detected_human_num, which is only valid for distance-sorted rows
        # (selfAttn_srnn_temp_node.py:398-404 uses visible_masks otherwise); the GST wrapper sorts on its own
        raise NotImplementedError("args.sort_humans=False is covered only behind the GST wrapper (pretext_wrapper=True)")
    return _capi.default_config_dict(
        num_envs=num_envs, nenv_total=nenv_total or num_envs, rank_offset=rank_offset, seed=seed,
        human_num=config.sim.human_num, human_num_range=int(config.sim.human_num_range),
        predict_steps=config.sim.predict_steps, const_vel=const_vel,
        randomize_attributes=int(bool(config.env.randomize_attributes)),
        random_goal_changing=int(bool(config.humans.random_goal_changing)),
        end_goal_changing=int(bool(config.humans.end_goal_changing)), sort_humans=int(bool(sort_humans)),
        device=device_index, time_step=float(config.env.time_step), time_limit=float(config.env.time_limit),
        pred_timestep=float(config.data.pred_timestep), circle_radius=float(config.sim.circle_radius),
        arena_size=float(config.sim.arena_size), discomfort_dist=float(config.reward.discomfort_dist),
        discomfort_penalty_factor=float(config.reward.discomfort_penalty_factor),
        success_reward=float(config.reward.success_reward), collision_penalty=float(config.reward.collision_penalty),
        human_radius=float(config.humans.radius), human_v_pref=float(config.humans.v_pref),
        human_fov=float(config.humans.FOV), robot_radius=float(config.robot.radius),
        robot_v_pref=float(config.robot.v_pref), robot_fov=float(config.robot.FOV),
        sensor_range=float(config.robot.sensor_range), goal_change_chance=float(config.humans.goal_change_chance),
        orca_neighbor_dist=float(config.orca.neighbor_dist), orca_safety_space=float(config.orca.safety_space),
        orca_time_horizon=float(config.orca.time_horizon),
        human_policy=1 if config.humans.policy == "social_force" else 0, robot_policy=robot_policy,
        robot_visible=int(robot_visible),
        sf_A=float(config.sf.A), sf_B=float(config.sf.B), sf_KI=float(config.sf.KI),
        phase=2 if phase == "test" else 0, val_size=int(getattr(config.env, "val_size", 100)),
        test_size=int(getattr(config.env, "test_size", 500)))


class LazyInfos(object):
    """Sequence of per-env info dicts, materialised on access (train.py:180-189 iterates it)."""

    def __init__(self, info_codes, aux, done, ep_ret, ep_len, t_start=None):
        self._codes, self._aux, self._done, self._ret, self._len = info_codes, aux, done, ep_ret, ep_len
        self._t = round(time.time() - t_start, 6) if t_start is not None else 0.0     # Monitor's 't': seconds since creation

    def __len__(self):
        return len(self._codes)

    def __getitem__(self, i):
        code = int(self._codes[i])
        obj = Danger(float(self._aux[i])) if code == 4 else _INFO_CLASSES[code]()
        d = {'info': obj}
        if self._done[i]:
            d['episode'] = {'r': round(float(self._ret[i]), 6), 'l': int(self._len[i]), 't': self._t}
        return d

    def __iter__(self):
        for i in range(len(self)):
            yield self[i]


class _BaseEnvView(object):
    """What rl/evaluation.py:42-50,75 reaches through `eval_envs.venv.envs[0].env`: the raw environment's
    `time_limit`, `global_time` (simulation time of environment 0) and the writable `episode_k`."""

    def __init__(self, venv):
        self._venv = venv
        self.episode_k = 0

    @property
    def time_limit(self):
        return self._venv.cfgd["time_limit"]

    @property
    def global_time(self):
        return float(self._venv.get_state("step_count")[0]) * float(self._venv.cfgd["time_step"])


class _MonitorView(object):
    def __init__(self, venv):
        self.env = _BaseEnvView(venv)


class _VenvView(object):
    """Stands for the wrapped `DummyVecEnv` / `ShmemVecEnv` the reference's VecPyTorch holds in `.venv`."""

    def __init__(self, venv):
        self._venv = venv
        self.envs = [_MonitorView(venv)]
        self.num_envs = venv.num_envs

    @property
    def unwrapped(self):
        return self

    def __getattr__(self, name):           # VecEnvWrapper.__getattr__ passthrough (rl/vec_env/vec_env.py:194-197)
        return getattr(self._venv, name)


class CudaCrowdVecEnv(object):
    """N crowd-navigation environments resident on one GPU (one shard of the job)."""

    def __init__(self, num_envs=None, device=None, cfg=None, **cfg_over):
        self.lib = _capi.load_library()
        self.device = torch.device(device if device is not None else "cuda:0")
        if self.device.type != "cuda":
            raise RuntimeError("CudaCrowdVecEnv needs a CUDA device (no CPU fallback)")
        d = dict(cfg) if cfg is not None else _capi.default_config_dict()
        if num_envs is not None:
            d["num_envs"] = num_envs
            if cfg is None and "nenv_total" not in cfg_over:
                d["nenv_total"] = num_envs
        d.update(cfg_over)
        d["device"] = self.device.index if self.device.index is not None else torch.cuda.current_device()
        self.cfgd = d
        self._cfg = _capi.config_from_dict(d)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):       # the C entry point calls cudaSetDevice: keep the caller's current device
            _capi.check(self.lib, self.lib.cn_env_create(C.byref(self._cfg), C.byref(self._h)), "cn_env_create")
        N, H = d["num_envs"], d["human_num"] + d["human_num_range"]          # rows = max_human_num
        W = 2 * (d["predict_steps"] + 1) if d["const_vel"] else 2
        self.num_envs, self.human_num, self.row_width = N, H, W
        spaces = {
            'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
            'detected_human_num': Box((1,)),
        }
        if not d["const_vel"]:
            spaces['visible_masks'] = Box((H,), np.bool_)
        self.observation_space = _DictSpace(spaces)
        self.action_space = Box((2,))
        dev = self.device
        # double-buffered observation tensors so a returned dict stays valid for one more step
        self._obs_bufs = [self._alloc_obs(dev) for _ in range(2)]
        self._flip = 0
        # per-step results live in ONE packed device buffer (and one pinned host mirror) so that the
        # reference-facing step() needs a single D2H copy: [ep_ret f64 | reward f32 | info i32 | info_aux f32 |
        # ep_len i32 | done u8]
        layout = [("ep_ret", torch.float64), ("reward", torch.float32), ("info", torch.int32),
                  ("info_aux", torch.float32), ("ep_len", torch.int32), ("done", torch.uint8)]
        total = sum(N * torch.empty(0, dtype=dt).element_size() for _, dt in layout)
        self._out_packed = torch.zeros(total, dtype=torch.uint8, device=dev)
        self._host_packed = torch.zeros(total, dtype=torch.uint8).pin_memory()
        self._out, self._host, off = {}, {}, 0
        for k, dt in layout:
            nb = N * torch.empty(0, dtype=dt).element_size()
            self._out[k] = self._out_packed[off:off + nb].view(dt)
            self._host[k] = self._host_packed[off:off + nb].view(dt)
            off += nb
        self._outp = _capi.CnStepPtrs(*[self._out[k].data_ptr() if k in self._out else None
                                        for k, _ in _capi.CnStepPtrs._fields_])
        self._host_np = self._host_packed.numpy()
        self._np_layout, off = {}, 0            # field -> (byte offset, byte length, numpy dtype) inside the packed buffer
        for k, dt in layout:
            nb = N * torch.empty(0, dtype=dt).element_size()
            self._np_layout[k] = (off, off + nb, self._host[k].numpy().dtype)
            off += nb
        self._t_start = time.time()
        self.closed = False
        _trace("engine CudaCrowdVecEnv N=%d (of %d, offset %d) H=%d const_vel=%d phase=%d device=%s gst=0" % (
            N, d["nenv_total"], d["rank_offset"], H, d["const_vel"], d["phase"], self.device))

    def _alloc_obs(self, dev):
        N, H, W = self.num_envs, self.human_num, self.row_width
        t = OrderedDict(robot_node=torch.zeros(N, 1, 7, device=dev), temporal_edges=torch.zeros(N, 1, 2, device=dev),
                        spatial_edges=torch.zeros(N, H, W, device=dev), detected_human_num=torch.zeros(N, 1, device=dev))
        if not self.cfgd["const_vel"]:
            t['visible_masks'] = torch.zeros(N, H, dtype=torch.bool, device=dev)
        ptrs = _capi.CnObsPtrs(*[t[k].data_ptr() if k in t else None for k, _ in _capi.CnObsPtrs._fields_])
        return t, ptrs

    def _stream(self):
        return _capi.raw_stream(self.device.index or 0)

    # ------------------------------------------------------------------ VecEnv surface
    def reset(self):
        self._flip ^= 1
        obs, ptrs = self._obs_bufs[self._flip]
        _capi.check(self.lib, self.lib.cn_env_reset(self._h, C.byref(ptrs), self._stream()), "cn_env_reset")
        return dict(obs)

    def step_device(self, actions, obs_out=None, reward_out=None, not_done_out=None):
        """Device-resident step: returns (obs, reward[N] f32, done[N] u8, info[N] i32) as device tensors
        (views of internal buffers, valid until the next step).

        Zero-copy rollout: `obs_out` (dict of contiguous float32 device tensors shaped like the
        observation), `reward_out` ([N] or [N,1]) and `not_done_out` ([N] or [N,1], receives 1 - done)
        let the kernel write straight into the rollout storage slot instead of internal buffers."""
        if actions.dtype != torch.float32 or not actions.is_cuda or not actions.is_contiguous():
            actions = actions.to(self.device, torch.float32).contiguous()
        assert actions.shape == (self.num_envs, 2)
        if obs_out is None:
            self._flip ^= 1
            obs, ptrs = self._obs_bufs[self._flip]
        else:
            obs = obs_out
            for k, t in obs.items():
                assert t.is_cuda and t.is_contiguous(), k
            ptrs = _capi.CnObsPtrs(*[obs[k].data_ptr() if k in obs else None for k, _ in _capi.CnObsPtrs._fields_])
        outp, reward = self._outp, self._out["reward"]
        if reward_out is not None or not_done_out is not None:
            vals = {k: self._out[k].data_ptr() for k in self._out}
            if reward_out is not None:
                assert reward_out.is_cuda and reward_out.is_contiguous() and reward_out.numel() == self.num_envs \
                    and reward_out.dtype == torch.float32
                vals["reward"] = reward_out.data_ptr()
                reward = reward_out
            if not_done_out is not None:
                assert not_done_out.is_cuda and not_done_out.is_contiguous() and not_done_out.numel() == self.num_envs \
                    and not_done_out.dtype == torch.float32      # the kernel stores float 0.0 / 1.0
                vals["not_done"] = not_done_out.data_ptr()
            outp = _capi.CnStepPtrs(*[vals.get(k) for k, _ in _capi.CnStepPtrs._fields_])
        # the C entry points restore the caller's current device themselves (CnDeviceGuard): no context manager here
        rc = self.lib.cn_env_step(self._h, C.c_void_p(actions.data_ptr()), C.byref(ptrs), C.byref(outp), self._stream())
        if rc:
            _capi.check(self.lib, rc, "cn_env_step")
        return dict(obs), reward, self._out["done"], self._out["info"]

    def step_async(self, actions):
        self._pending = self.step_device(actions)

    def _fetch(self):
        """Packed step outputs (reward, done, info, episode stats: 25 B/env) -> pinned host buffer, then wait."""
        hp, dp = self._host_packed, self._out_packed
        rc = self.lib.cn_fetch_sync(C.c_void_p(hp.data_ptr()), C.c_void_p(dp.data_ptr()), dp.numel() * dp.element_size(),
                                    self.device.index or 0, self._stream())
        if rc:
            _capi.check(self.lib, rc, "cn_fetch_sync")

    def step_wait(self):
        obs, _, _, _ = self._pending
        return (obs,) + self._host_results()

    def _host_results(self):
        """(reward CPU [N,1], done np.bool_[N], lazy infos) from ONE snapshot of the pinned mirror (the mirror is
        overwritten by the next step; the snapshot belongs to the caller)."""
        self._fetch()
        snap = self._host_np.copy()
        f = {k: snap[a:b].view(dt) for k, (a, b, dt) in self._np_layout.items()}
        done = f["done"].view(np.bool_)
        infos = LazyInfos(f["info"], f["info_aux"], done, f["ep_ret"], f["ep_len"], self._t_start)
        return torch.from_numpy(f["reward"]).unsqueeze(1), done, infos

    def step(self, actions):
        self.step_async(actions)
        return self.step_wait()

    def talk2Env(self, data):
        return np.ones(self.num_envs, dtype=bool)

    def render(self, mode='human'):
        """Rendering is out of scope (SURVEY.md §2.1 row 1): a no-op with one warning, so that the reference's
        test.py (whose --visualize defaults to True) still runs."""
        if not getattr(self, "_render_warned", False):
            self._render_warned = True
            import warnings
            warnings.warn("crowdnav_b200: render() is a no-op (rendering is outside the engine's scope)")
        return None

    @property
    def venv(self):
        v = self.__dict__.get("_venv_view")
        if v is None:
            v = self.__dict__["_venv_view"] = _VenvView(self)
        return v

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

    # ------------------------------------------------------------------ parity-test access
    _DT = dict(rpx="f8", rpy="f8", rgx="f8", rgy="f8", rvx="f4", rvy="f4", potential="f8", fut_pen="f8",
               nd_global="f8", ep_ret="f8", ep_len="i4", step_count="i4", case_counter="u4", seed_off="i4",
               hpx="f8", hpy="f8", hgx="f8", hgy="f8", hrad="f8", hvpref="f8", hvx="f4", hvy="f4",
               bpx="f8", bpy="f8", bvx="f8", bvy="f8", brad="f8", vis="u1", sim_exists="u1",
               sim_nd="f4", sim_rself="f4", sim_vmax="f4", sim_rother="f4", mt="u4", mt_pos="i4",
               last_hvx="f4", last_hvy="f4", orca_nlines="i4", orca_fail="i4", evt="u1", spawn_overflow="u1",
               defer_ctl="i4", defer_list="i4", lp_cost="i4", hn="i4", prep_hn="i4", hwx="f8", hwy="f8",
               rwx="f8", rwy="f8", rsim_exists="u1", rsim_nd="f4", rsim_rother="f4")

    def get_state(self, name):
        nbytes = self.lib.cn_env_state_bytes(self._h, name.encode())
        if not nbytes:
            raise KeyError(name)
        arr = np.zeros(nbytes // np.dtype(self._DT[name]).itemsize, self._DT[name])
        _capi.check(self.lib, self.lib.cn_env_state_copy(self._h, name.encode(), arr.ctypes.data, nbytes, 0),
                    "cn_env_state_copy")
        return arr

    def set_state(self, name, arr):
        arr = np.ascontiguousarray(arr, dtype=self._DT[name])
        _capi.check(self.lib, self.lib.cn_env_state_copy(self._h, name.encode(), arr.ctypes.data, arr.nbytes, 1),
                    "cn_env_state_copy")

    def launch_count(self):
        return int(self.lib.cn_env_launch_count(self._h))


def make_vec_envs(env_name, seed, num_processes, gamma, log_dir, device, allow_early_resets,
                  num_frame_stack=None, config=None, ax=None, test_case=-1, wrap_pytorch=True,
                  pretext_wrapper=False, nenv_total=None, rank_offset=0, phase=None, gst_params=None):
    """Same signature as rl/networks/envs.py:97-140.  Returns the CUDA vec env (already 'VecPyTorch').
    Like the reference (envs.py:55-58) a single environment runs in phase 'test', several in 'train';
    `phase=` overrides (batched evaluation)."""
    device = torch.device(device)
    if pretext_wrapper or env_name == "CrowdSimPredRealGST-v0":
        if gst_params is None:
            raise ValueError("CrowdSimPredRealGST-v0 / pretext_wrapper=True needs gst_params= (the predictor checkpoint's "
                             "model_state_dict, config.pred.model_dir/checkpoint/epoch_100.pt)")
        d = config_dict_from_reference(config, num_processes, seed, "CrowdSimVarNum-v0", nenv_total=nenv_total,
                                       rank_offset=rank_offset, device_index=device.index if device.index is not None else 0,
                                       phase=phase, allow_unsorted=True)
        return CudaPretextVecEnv(gst_params, device=device, cfg=d)
    d = config_dict_from_reference(config, num_processes, seed, env_name, nenv_total=nenv_total,
                                   rank_offset=rank_offset,
                                   device_index=device.index if device.index is not None else 0, phase=phase)
    return CudaCrowdVecEnv(device=device, cfg=d)


class CudaPretextVecEnv(object):
    """`VecPretextNormalize(ShmemVecEnv([CrowdSimPredRealGST-v0 ...]))` on one GPU (BASELINE config 3, SURVEY row a16).

    The environments run in the engine's CrowdSimVarNum-v0 mode without sorting (that IS the raw RealGST
    observation, crowd_sim_pred_real_gst.py:73-88); one chain of kernels per step keeps the wrapper's 5-frame
    trajectory / mask buffers, runs the GST predictor, adds the future-collision penalty to the reward, writes the
    predicted relative positions into the 2(P+1)-wide spatial_edges and sorts the rows by distance
    (rl/vec_env/vec_pretext_normalize.py:112-191).  Like the reference, the buffers are NOT cleared when a
    single environment finishes an episode.  `gst_params`: dict name -> array with the predictor checkpoint's
    model_state_dict (e.g. np.load('tests/golden/gst_params.npz'))."""

    def __init__(self, gst_params, num_envs=None, device=None, cfg=None, **cfg_over):
        over = dict(cfg_over)
        d = dict(cfg) if cfg is not None else None
        if d is not None:
            d.update(const_vel=0, sort_humans=0)
        else:
            over.update(const_vel=0, sort_humans=0)
        if (d if d is not None else over).get("robot_policy", 0):
            raise NotImplementedError("the ORCA / social-force robot is not covered behind the GST wrapper "
                                      "(VecPretextNormalize): the reference's baselines run without it")
        self.env = CudaCrowdVecEnv(num_envs=num_envs, device=device, cfg=d, **over)
        e = self.env
        self.lib, self.device, self.cfgd = e.lib, e.device, e.cfgd
        self.num_envs, self.human_num = e.num_envs, e.human_num
        self.P = int(self.cfgd["predict_steps"])
        N, H, W = self.num_envs, self.human_num, 2 * (self.P + 1)
        self.row_width = W
        spaces = dict(e.observation_space.spaces)
        spaces['spatial_edges'] = Box((H, W))
        self.observation_space = _DictSpace(spaces)
        self.action_space = e.action_space
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):       # cn_gst_* call cudaSetDevice: keep the caller's current device
            _capi.check(self.lib, self.lib.cn_gst_create(N, H, self.P, float(self.cfgd["robot_radius"]),
                                                         float(self.cfgd["human_radius"]), float(self.cfgd["collision_penalty"]),
                                                         self.device.index or 0, C.byref(self._h)), "cn_gst_create")
            for k, v in gst_params.items():
                arr = np.ascontiguousarray(v.detach().cpu().numpy() if hasattr(v, "detach") else v, dtype=np.float32)
                _capi.check(self.lib, self.lib.cn_gst_set_param(self._h, k.encode(), arr.ctypes.data, arr.size),
                            "cn_gst_set_param(%s)" % k)
            _capi.check(self.lib, self.lib.cn_gst_finalize(self._h), "cn_gst_finalize")
        _trace("engine CudaPretextVecEnv N=%d H=%d P=%d device=%s gst=1" % (N, H, self.P, self.device))
        self._sp = [torch.zeros(N, H, W, device=self.device) for _ in range(2)]
        self._pen = torch.zeros(N, device=self.device)
        self._flip = 0
        self.closed = False

    def _stream(self):
        return _capi.raw_stream(self.device.index or 0)

    def _process(self, obs, reward):
        self._flip ^= 1
        sp = self._sp[self._flip]
        vm = obs['visible_masks']
        _capi.check(self.lib, self.lib.cn_gst_step(
            self._h, C.c_void_p(obs['robot_node'].data_ptr()), C.c_void_p(obs['spatial_edges'].data_ptr()),
            C.c_void_p(vm.data_ptr()), C.c_void_p(reward.data_ptr()) if reward is not None else None,
            C.c_void_p(self._pen.data_ptr()), C.c_void_p(sp.data_ptr()), self._stream()), "cn_gst_step")
        out = dict(obs)
        out['spatial_edges'] = sp
        out['visible_masks'] = vm.bool() if vm.dtype != torch.bool else vm
        return out

    def reset(self):
        with torch.cuda.device(self.device):
            _capi.check(self.lib, self.lib.cn_gst_reset(self._h, self._stream()), "cn_gst_reset")
        return self._process(self.env.reset(), None)

    def step_device(self, actions):
        """Device-resident step: (obs, reward [N] incl. the prediction penalty, done [N] u8, info [N] i32)."""
        obs, reward, done, info = self.env.step_device(actions)
        return self._process(obs, reward), reward, done, info

    def step(self, actions):
        obs, reward, done, info = self.step_device(actions)
        e = self.env
        return (obs,) + e._host_results()

    def talk2Env(self, data):
        return np.ones(self.num_envs, dtype=bool)

    def render(self, mode='human'):
        return self.env.render(mode)

    @property
    def venv(self):
        return self.env.venv

    @property
    def unwrapped(self):
        return self

    def get_state(self, name):
        return self.env.get_state(name)

    def set_state(self, name, arr):
        return self.env.set_state(name, arr)

    def launch_count(self):
        return self.env.launch_count() + int(self.lib.cn_gst_launch_count(self._h))

    def close(self):
        if not self.closed:
            self.lib.cn_gst_destroy(self._h)
            self.env.close()
            self.closed = True

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
