"""Shared pieces of the data-collection tests (CrowdSimVarNumCollect-v0): the golden cases recorded by
tools/make_golden_collect.py, their engine configuration, a replay through any engine with reset() / step(actions) /
get(name), and the host build of the collect step (tests/cpu_harness/collect_harness.cpp)."""
import ast
import ctypes as C
import os
import subprocess

import numpy as np

from crowdnav_prediction_attngraph_b200 import _capi
from tests import harness_util
from tests.golden_util import GOLD
from tests.harness_util import HarnessEnv

COLLECT_CASES = ["collect_h20_train", "collect_h8_sf_humans", "collect_h10_sf_robot"]
COLLECT_SO = os.path.join(harness_util.HERE, "_build_collect_harness.so")
COLLECT_SRC = os.path.join(harness_util.HERE, "cpu_harness", "collect_harness.cpp")
STATE_DTYPES = dict(harness_util.STATE_DTYPES, rwx="f8", rwy="f8", rsim_exists="u1", rsim_nd="f4", rsim_rother="f4",
                    pred_id="i4", max_id="i4", rgoal_due="u1", rgoal_med="f8")


def load_collect_case(name):
    """(golden arrays, case dict, cn_config overrides) of a collect fixture: the reference's default config."""
    g = np.load(os.path.join(GOLD, name + ".npz"))
    case = ast.literal_eval(str(g["meta"][0]))
    over = dict(num_envs=case["nenv"], nenv_total=case["nenv"], seed=to_int32(case["seed"]), human_num=case["human_num"],
                const_vel=0, randomize_attributes=1, random_goal_changing=1, sort_humans=0,
                phase=2 if case["phase"] == "test" else 0,
                human_policy=1 if case.get("human_policy", "orca") == "social_force" else 0,
                robot_policy={"orca": 1, "social_force": 2}[case["robot_policy"]])
    return g, case, over


def to_int32(seed):
    """cn_config.seed carries seeds in [2**31, 2**32) as the same 32 bits."""
    return seed - 2 ** 32 if seed >= 2 ** 31 else seed


def replay_collect(g, reset_fn, step_fn, get_fn, pos_tol=1e-9):
    """Mismatch strings (empty = parity): pred_info, ids, info and done bit for bit, fp64 state within pos_tol."""
    T1, N, H = g["pred_id"].shape
    bad = []
    zeros = np.zeros((N, 2), np.float32)
    for t in range(T1):
        if t == 0:
            pi = reset_fn()
            out = None
        else:
            pi, out = step_fn(zeros)
        msg = []
        if not np.array_equal(pi.view(np.uint32), g["pred_info"][t].view(np.uint32)):
            msg.append("pred_info")
        if out is not None:
            if not np.array_equal(out["info"], g["info"][t]):
                msg.append("info")
            if not np.array_equal(out["done"].astype(bool), g["done"][t]):
                msg.append("done")
            if np.any(out["reward"] != 0):
                msg.append("reward")
        if not np.array_equal(get_fn("pred_id").reshape(N, H), g["pred_id"][t]):
            msg.append("pred_id")
        if not np.array_equal(get_fn("max_id"), g["max_id"][t]):
            msg.append("max_id")
        rob = np.stack([get_fn(k) for k in ("rpx", "rpy", "rgx", "rgy")], -1)
        if np.abs(rob - g["robot"][t][:, [0, 1, 4, 5]]).max() > pos_tol:
            msg.append("robot")
        for k in ("hpx", "hpy", "hgx", "hgy", "hrad", "hvpref"):
            if np.abs(get_fn(k).reshape(N, H) - g[k][t]).max() > pos_tol:
                msg.append(k)
        if msg:
            bad.append("t=%d: %s" % (t, ",".join(msg)))
    return bad


def _build():
    core = harness_util.CORE
    deps = [COLLECT_SRC, harness_util.SRC, os.path.join(harness_util.HERE, "cpu_harness", "robot_harness.cpp")] + \
        [os.path.join(core, f) for f in os.listdir(core) if f.endswith(".cuh")]
    if os.path.exists(COLLECT_SO) and all(os.path.getmtime(COLLECT_SO) >= os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", COLLECT_SO,
                           COLLECT_SRC])


class CollectHarnessEnv(HarnessEnv):
    """N collect environments stepped by the host build of the kernel logic; reset() / step() return pred_info."""

    def __init__(self, **cfg_over):
        super().__init__(**cfg_over)
        self.lib.harness_destroy(self.h)
        self.h = None
        _build()
        old, lib = self.lib, C.CDLL(COLLECT_SO)
        for name in ("harness_destroy", "harness_state_bytes", "harness_state_copy"):
            f, o = getattr(lib, name), getattr(old, name)
            f.argtypes, f.restype = o.argtypes, o.restype
        lib.collect_harness_create.restype = C.c_void_p
        lib.collect_harness_create.argtypes = [C.POINTER(_capi.CnConfig)]
        lib.collect_harness_reset.argtypes = [C.c_void_p, C.c_void_p]
        lib.collect_harness_step.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(_capi.CnStepPtrs)]
        self.lib = lib
        self.h = lib.collect_harness_create(C.byref(self.cfg))
        self.pred_info = np.zeros((self.N, self.H, 4), np.float32)

    def reset(self):
        self.lib.collect_harness_reset(self.h, self.pred_info.ctypes.data)
        return self.pred_info.copy()

    def step(self, actions):
        a = np.ascontiguousarray(actions, dtype=np.float32)
        self.lib.collect_harness_step(self.h, a.ctypes.data, self.pred_info.ctypes.data, C.byref(self.outp))
        return self.pred_info.copy(), {k: v.copy() for k, v in self.out.items()}

    def get(self, name):
        nbytes = self.lib.harness_state_bytes(self.h, name.encode())
        assert nbytes, name
        arr = np.zeros(nbytes // np.dtype(STATE_DTYPES[name]).itemsize, STATE_DTYPES[name])
        assert self.lib.harness_state_copy(self.h, name.encode(), arr.ctypes.data, nbytes, 0) == 0
        return arr
