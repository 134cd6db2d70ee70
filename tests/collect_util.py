"""Shared pieces of the data-collection tests (CrowdSimVarNumCollect-v0): the golden cases recorded by
tools/make_golden_collect.py, their engine configuration, a replay through any engine with reset() / step(actions) /
get(name)."""
import ast
import os

import numpy as np

from tests.golden_util import GOLD

COLLECT_CASES = ["collect_h20_train", "collect_h8_sf_humans", "collect_h10_sf_robot"]


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
