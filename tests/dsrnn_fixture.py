"""Shared helpers for the DS-RNN policy tests: the synthetic weights of tools/make_golden_dsrnn.py and its fixtures."""
import os

import numpy as np
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
OBS_KEYS = ["robot_node", "temporal_edges", "spatial_edges", "detected_human_num"]
ACT_CASES = {"varnum_h5": (5, 2), "varnum_h20": (20, 2), "pred_h20": (20, 12)}     # tag: (H, W)
UNUSED = ("base.humanNodeRNN.edge_embed.", "base.human_node_final_linear.", "base.spatial_linear.")


def dsrnn_state_dict(template):
    """make_golden_policy.param_fill with the scales of tests/golden/dsrnn_param_scales.npz (sorted keys, seed + index,
    N(0,1) * scale)."""
    sc = np.load(os.path.join(GOLD, "dsrnn_param_scales.npz"))
    seed = int(sc["seed"])
    keys = [str(k) for k in sc["keys"]]
    out = {}
    for i, (k, s) in enumerate(zip(keys, sc["scales"])):
        g = torch.Generator().manual_seed(seed + i)
        out[k] = torch.randn(tuple(template[k].shape), generator=g) * float(s)
    assert set(out) == set(template), set(out) ^ set(template)
    return out


def reference_shapes():
    """{key: shape string} of the reference SRNN's state_dict (W = 2), recorded with the fixtures."""
    sc = np.load(os.path.join(GOLD, "dsrnn_param_scales.npz"))
    return {str(k): str(s) for k, s in zip(sc["keys"], sc["shapes"])}


def act_case(tag):
    g = np.load(os.path.join(GOLD, "dsrnn_act.npz"))
    obs = {k: torch.from_numpy(g[tag + "_ob_" + k]) for k in OBS_KEYS}
    ins = {k: torch.from_numpy(g[tag + "_" + k]) for k in ("h", "he", "masks")}
    outs = {k: g[tag + "_" + k] for k in ("value", "mean", "h1", "he1")}
    return obs, ins, outs


def recurrent_case():
    return np.load(os.path.join(GOLD, "dsrnn_recurrent.npz"))


class Args(object):
    def __init__(self, **kw):
        self.num_processes, self.seq_length, self.num_mini_batch = 4, 30, 2
        self.human_node_rnn_size, self.human_human_edge_rnn_size = 128, 256
        self.__dict__.update(kw)


def spaces(H, W):
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    return ({'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
             'detected_human_num': Box((1,))}, Box((2,)))
