"""Test helper: drives the HOST build of the step-kernel logic (tests/cpu_harness/env_harness.cpp) through the
same struct layouts as the C ABI.  Test infrastructure only."""
import ctypes as C
import os
import subprocess

import numpy as np

from crowdnav_prediction_attngraph_b200 import _capi

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "_build_env_harness.so")
SRC = os.path.join(HERE, "cpu_harness", "env_harness.cpp")
CORE = os.path.join(HERE, "..", "crowdnav_prediction_attngraph_b200", "csrc")

STATE_DTYPES = dict(
    rpx="f8", rpy="f8", rgx="f8", rgy="f8", rvx="f4", rvy="f4", potential="f8", fut_pen="f8", nd_global="f8",
    ep_ret="f8", ep_len="i4", step_count="i4", case_counter="u4", seed_off="i4",
    hpx="f8", hpy="f8", hgx="f8", hgy="f8", hrad="f8", hvpref="f8", hvx="f4", hvy="f4",
    bpx="f8", bpy="f8", bvx="f8", bvy="f8", brad="f8", vis="u1", sim_exists="u1",
    sim_nd="f4", sim_rself="f4", sim_vmax="f4", sim_rother="f4", mt="u4", mt_pos="i4",
    last_hvx="f4", last_hvy="f4", orca_nlines="i4", orca_fail="i4", evt="u1", spawn_overflow="u1", hn="i4", prep_hn="i4",
    sim_n="u1", hwx="f8", hwy="f8",
    rwx="f8", rwy="f8", rsim_exists="u1", rsim_nd="f4", rsim_rother="f4",
    pred_id="i4", max_id="i4", rgoal_due="u1", rgoal_med="f8")


def build():
    deps = [SRC] + [os.path.join(CORE, f) for f in os.listdir(CORE) if f.endswith(".cuh")]
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", SO, SRC])


class HarnessEnv(object):
    """N environments stepped by the host build of the kernel logic, configured like cn_env_create (robot policy,
    robot.visible, social-force humans, phase 'test', 'truth' observations).  collect=True: the collect environment
    (cn_env_create_collect), whose reset() / step() return pred_info instead of the observation dict."""

    def __init__(self, collect=False, **cfg_over):
        build()
        self.lib = C.CDLL(SO)
        self.lib.harness_create.restype = C.c_void_p
        self.lib.harness_create.argtypes = [C.POINTER(_capi.CnConfig), C.c_int]
        self.lib.harness_destroy.argtypes = [C.c_void_p]
        self.lib.harness_reset.argtypes = [C.c_void_p, C.POINTER(_capi.CnObsPtrs), C.c_void_p]
        self.lib.harness_step.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(_capi.CnObsPtrs),
                                          C.POINTER(_capi.CnStepPtrs), C.c_void_p]
        self.lib.harness_state_bytes.restype = C.c_size_t
        self.lib.harness_state_bytes.argtypes = [C.c_void_p, C.c_char_p]
        self.lib.harness_state_copy.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_size_t, C.c_int]
        self.cfgd = _capi.default_config_dict(**cfg_over)
        self.cfg = _capi.config_from_dict(self.cfgd)
        self.collect = collect
        self.h = self.lib.harness_create(C.byref(self.cfg), int(collect))
        N, H = self.cfgd["num_envs"], self.cfgd["human_num"] + self.cfgd["human_num_range"]
        W = 2 * (self.cfgd["predict_steps"] + 1) if self.cfgd["const_vel"] else 2
        self.N, self.H, self.W = N, H, W
        if collect:
            self.pred_info = np.zeros((N, H, 4), np.float32)
            self.obp, self.pip = None, self.pred_info.ctypes.data
        else:
            self.ob = dict(robot_node=np.zeros((N, 1, 7), np.float32), temporal_edges=np.zeros((N, 1, 2), np.float32),
                           spatial_edges=np.zeros((N, H, W), np.float32), detected_human_num=np.zeros((N, 1), np.float32))
            if not self.cfgd["const_vel"]:
                self.ob["visible_masks"] = np.zeros((N, H), np.uint8)
            self.obp = C.pointer(_capi.CnObsPtrs(*[self.ob[k].ctypes.data if k in self.ob else None
                                                   for k, _ in _capi.CnObsPtrs._fields_]))
            self.pip = None
        self.out = dict(reward=np.zeros(N, np.float32), done=np.zeros(N, np.uint8), info=np.zeros(N, np.int32),
                        info_aux=np.zeros(N, np.float32), ep_ret=np.zeros(N, np.float64), ep_len=np.zeros(N, np.int32))
        self.outp = _capi.CnStepPtrs(*[self.out[k].ctypes.data if k in self.out else None
                                       for k, _ in _capi.CnStepPtrs._fields_])

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.harness_destroy(self.h)
            self.h = None

    def _obs(self):
        if self.collect:
            return self.pred_info.copy()
        o = {k: v.copy() for k, v in self.ob.items()}
        if "visible_masks" in o:
            o["visible_masks"] = o["visible_masks"].astype(bool)
        return o

    def reset(self):
        self.lib.harness_reset(self.h, self.obp, self.pip)
        return self._obs()

    def step(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.float32)
        self.lib.harness_step(self.h, a.ctypes.data, self.obp, C.byref(self.outp), self.pip)
        return self._obs(), {k: v.copy() for k, v in self.out.items()}

    def get(self, name):
        nbytes = self.lib.harness_state_bytes(self.h, name.encode())
        assert nbytes, name
        arr = np.zeros(nbytes // np.dtype(STATE_DTYPES[name]).itemsize, STATE_DTYPES[name])
        assert self.lib.harness_state_copy(self.h, name.encode(), arr.ctypes.data, nbytes, 0) == 0
        return arr

    def set(self, name, arr):
        arr = np.ascontiguousarray(arr, dtype=STATE_DTYPES[name])
        assert self.lib.harness_state_copy(self.h, name.encode(), arr.ctypes.data, arr.nbytes, 1) == 0
