"""Shared pieces of the robot-policy tests (robot.policy 'orca' / 'social_force'): the golden cases, a replay of
them through any engine with reset() / step(actions) / get(name) that also checks the robot's velocity."""
import numpy as np

from tests.golden_util import load_env_case, replay

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
