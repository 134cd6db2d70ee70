"""Shared pieces of the robot-policy tests (robot.policy 'orca' / 'social_force'): the golden cases, a replay of
them through any engine with reset() / step(actions) / get(name) that also checks the robot's velocity, and the host
build of the step kernel's logic with the robot's policy (tests/cpu_harness/robot_harness.cpp)."""
import ctypes as C
import os
import subprocess

import numpy as np

from crowdnav_prediction_attngraph_b200 import _capi
from tests import harness_util
from tests.golden_util import load_env_case, replay
from tests.harness_util import HarnessEnv

ROBOT_SO = os.path.join(harness_util.HERE, "_build_robot_harness.so")
ROBOT_SRC = os.path.join(harness_util.HERE, "cpu_harness", "robot_harness.cpp")
STATE_DTYPES = dict(harness_util.STATE_DTYPES, rwx="f8", rwy="f8", rsim_exists="u1", rsim_nd="f4", rsim_rother="f4")


def _build_robot_harness():
    core = harness_util.CORE
    deps = [ROBOT_SRC, harness_util.SRC] + [os.path.join(core, f) for f in os.listdir(core) if f.endswith(".cuh")]
    if os.path.exists(ROBOT_SO) and all(os.path.getmtime(ROBOT_SO) >= os.path.getmtime(d) for d in deps):
        return
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", ROBOT_SO, ROBOT_SRC])


class RobotHarnessEnv(HarnessEnv):
    """HarnessEnv whose environments run cn_config.robot_policy (robot_harness_create): same buffers and entry points,
    plus the robot's state fields."""

    def __init__(self, **cfg_over):
        super().__init__(**cfg_over)
        self.lib.harness_destroy(self.h)
        self.h = None
        _build_robot_harness()
        old, lib = self.lib, C.CDLL(ROBOT_SO)
        for name in ("harness_destroy", "harness_reset", "harness_step", "harness_state_bytes", "harness_state_copy"):
            f, o = getattr(lib, name), getattr(old, name)
            f.argtypes, f.restype = o.argtypes, o.restype
        lib.robot_harness_create.restype = C.c_void_p
        lib.robot_harness_create.argtypes = [C.POINTER(_capi.CnConfig)]
        self.lib = lib
        self.h = lib.robot_harness_create(C.byref(self.cfg))

    def get(self, name):
        nbytes = self.lib.harness_state_bytes(self.h, name.encode())
        assert nbytes, name
        arr = np.zeros(nbytes // np.dtype(STATE_DTYPES[name]).itemsize, STATE_DTYPES[name])
        assert self.lib.harness_state_copy(self.h, name.encode(), arr.ctypes.data, nbytes, 0) == 0
        return arr

ROBOT_CASES = ["env_varnum_h20_test_orca_robot", "env_varnum_h10_orca_robot_rand",
               "env_varnum_h20_test_sf_robot", "env_varnum_h10_sf_robot_rand"]
ROBOT_POLICY = {"orca": 1, "social_force": 2}


def load_robot_case(name):
    g, case, over = load_env_case(name)
    over["robot_policy"] = ROBOT_POLICY[case["robot_policy"]]
    return g, case, over


def replay_robot(g, case, reset_fn, step_fn, get_fn):
    """replay() plus the robot's velocity after every step that did not end the episode (an ending step installs
    the next episode, whose robot stands still): the fp32 velocity bit for bit, and for social force the fp64
    velocity the next step integrates to 1e-12.  That one is not bit for bit: its push terms call exp(), and the C / CUDA
    exp() and numpy's differ in the last bit now and then (5e-15 measured over these goldens).  State positions are held to
    1e-9 by replay()."""
    bad = []
    t_box = [0]
    sf = case["robot_policy"] == "social_force"

    def step(actions):
        t = t_box[0]
        t_box[0] += 1
        ob, out = step_fn(actions)
        live = ~out["done"].astype(bool)
        ref = g["robot_vel"][t]
        v32 = np.stack([get_fn("rvx"), get_fn("rvy")], -1)
        if not np.array_equal(v32[live], ref[live].astype(np.float32)):
            bad.append("t=%d: robot velocity (fp32)" % t)
        if sf:
            v64 = np.stack([get_fn("rwx"), get_fn("rwy")], -1)
            if np.abs(v64[live] - ref[live]).max(initial=0.0) > 1e-12:
                bad.append("t=%d: robot velocity (fp64)" % t)
        return ob, out

    return replay(g, case, reset_fn, step, get_fn) + bad
