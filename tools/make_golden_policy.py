#!/usr/bin/env python
"""Golden vectors for the policy forward, generated from the UNMODIFIED reference module
(rl.networks.model.Policy, base selfAttn_merge_srnn) in the build container.

Weights are a deterministic synthetic fill (param_fill below) whose per-tensor scale follows the
shipped checkpoint trained_models/GST_predictor_rand/checkpoints/41665.pt, so fixtures stay
small (no 10 MB weight file in git); inputs are observations recorded in tests/golden/env_*.npz.
A second fixture stores the outputs of the shipped checkpoint itself on the same inputs
(only compared in this container, where the checkpoint exists).

--no-self-attn writes only the fixtures of the reference's ablation without human-human attention
(args.use_self_attn = False set on the argument namespace): policy_nsa_h20 (W = 12, env_pred_h20),
policy_nsa_h50 (W = 12, env_pred_h50_rand) and policy_nsa_varnum (W = 2, CrowdSimVarNum-v0,
env_varnum_h20_vis_rand).  Weights: tests/policy_no_self_attn_ref.synth_state_dict_nsa (the fill above for every key
shared with the full network; spatial_linear.0 / .2 from the reference's orthogonal initialiser with seeded
generators).  Each file also holds the reference module's state_dict keys and shapes.

--unsorted writes the fixtures of args.sort_humans = False (unsorted_fixtures below): policy_unsorted_{full,nsa}_
{varnum,h20,h50}.

    CROWDNAV_REFERENCE_ROOT=<reference checkout> python tools/make_golden_policy.py [--no-self-attn | --unsorted]
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
from reference_root import reference_root  # noqa: E402
REF = reference_root()
sys.path.insert(0, REF)
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402
import torch  # noqa: E402

CKPT = os.path.join(REF, "trained_models", "GST_predictor_rand", "checkpoints", "41665.pt")


def param_fill(state_dict, seed, scales):
    """Deterministic fill: keys in sorted order, torch.manual_seed(seed + index), N(0,1) * scale."""
    out = {}
    for i, k in enumerate(sorted(state_dict.keys())):
        g = torch.Generator().manual_seed(seed + i)
        out[k] = torch.randn(state_dict[k].shape, generator=g) * float(scales[k])
    return out


def build_reference_policy(env_name, H, W, nenv, use_self_attn=True):
    sys.argv = ["x", "--no-cuda", "--env-name", env_name, "--num-processes", str(nenv)]
    import gym
    from arguments import get_args
    from rl.networks.model import Policy
    args = get_args()
    args.use_self_attn = use_self_attn
    obs_space = {"robot_node": gym.spaces.Box(-np.inf, np.inf, (1, 7)),
                 "temporal_edges": gym.spaces.Box(-np.inf, np.inf, (1, 2)),
                 "spatial_edges": gym.spaces.Box(-np.inf, np.inf, (H, W)),
                 "detected_human_num": gym.spaces.Box(-np.inf, np.inf, (1,))}
    act_space = gym.spaces.Box(-np.inf * np.ones(2), np.inf * np.ones(2), dtype=np.float32)
    return Policy(obs_space, act_space, base_kwargs=args, base="selfAttn_merge_srnn")


def main():
    sd_ck = torch.load(CKPT, map_location="cpu")
    scales = {k: float(v.float().std()) if v.numel() > 1 else 1.0 for k, v in sd_ck.items()}
    scales = {k: (s if s > 0 else 0.05) for k, s in scales.items()}
    # output heads boosted so the synthetic policy reaches the checkpoint's output magnitudes
    # (|value| ~ 20, |mean| ~ 10): keeps the absolute 1e-4 tolerance test meaningful
    scales["base.critic_linear.weight"] *= 12.0
    scales["dist.fc_mean.weight"] *= 8.0
    np.savez(os.path.join(REPO, "tests", "golden", "policy_param_scales.npz"),
             keys=np.array(sorted(scales.keys())), scales=np.array([scales[k] for k in sorted(scales.keys())]),
             shapes=np.array([str(tuple(sd_ck[k].shape)) for k in sorted(scales.keys())]))
    for name, env_file, H, W in [("policy_h20", "env_pred_h20", 20, 12), ("policy_h50", "env_pred_h50_rand", 50, 12)]:
        g = long_h20_recording() if env_file == "env_pred_h20" else np.load(os.path.join(REPO, "tests", "golden", env_file + ".npz"))
        T, N = g["actions"].shape[:2]
        B = 64
        idx = np.random.RandomState(0).choice((T + 1) * N, B, replace=False)
        take = lambda k: torch.from_numpy(g["ob_" + k].reshape((T + 1) * N, *g["ob_" + k].shape[2:])[idx].astype(np.float32))
        obs = {k: take(k) for k in ["robot_node", "temporal_edges", "spatial_edges", "detected_human_num"]}
        gen = torch.Generator().manual_seed(123)
        h = torch.randn(B, 1, 128, generator=gen) * 0.5
        masks = (torch.rand(B, 1, generator=gen) > 0.1).float()
        pol = build_reference_policy("CrowdSimPred-v0", H, W, B)
        out = {}
        for tag, sd in [("synth", param_fill(sd_ck, 1000, scales)), ("ckpt", sd_ck)]:
            pol.load_state_dict(sd)
            rnn = {"human_node_rnn": h.clone(), "human_human_edge_rnn": torch.zeros(B, H + 1, 256)}
            with torch.no_grad():
                value, feat, hx = pol.base({k: v.clone() for k, v in obs.items()}, rnn, masks.clone(), infer=True)
                mean = pol.dist.fc_mean(feat)
            out[tag + "_value"] = value.numpy()
            out[tag + "_mean"] = mean.numpy()
            out[tag + "_h"] = hx["human_node_rnn"].numpy()
            print(name, tag, "value range", float(value.min()), float(value.max()), "mean abs max", float(mean.abs().max()))
        np.savez_compressed(os.path.join(REPO, "tests", "golden", name + ".npz"),
                            h=h.numpy(), masks=masks.numpy(), **{"ob_" + k: v.numpy() for k, v in obs.items()}, **out)



def no_self_attn_fixtures():
    sys.path.insert(0, os.path.join(REPO, "tests"))
    from tests.policy_no_self_attn_ref import synth_state_dict_nsa
    for name, env_name, env_file, H, W in [("policy_nsa_h20", "CrowdSimPred-v0", "env_pred_h20", 20, 12),
                                           ("policy_nsa_h50", "CrowdSimPred-v0", "env_pred_h50_rand", 50, 12),
                                           ("policy_nsa_varnum", "CrowdSimVarNum-v0", "env_varnum_h20_vis_rand", 20, 2)]:
        g = long_h20_recording() if env_file == "env_pred_h20" else np.load(os.path.join(REPO, "tests", "golden", env_file + ".npz"))
        T, N = g["actions"].shape[:2]
        B = 64
        idx = np.random.RandomState(0).choice((T + 1) * N, B, replace=False)
        take = lambda k: torch.from_numpy(g["ob_" + k].reshape((T + 1) * N, *g["ob_" + k].shape[2:])[idx].astype(np.float32))
        obs = {k: take(k) for k in ["robot_node", "temporal_edges", "spatial_edges", "detected_human_num"]}
        gen = torch.Generator().manual_seed(123)
        h = torch.randn(B, 1, 128, generator=gen) * 0.5
        masks = (torch.rand(B, 1, generator=gen) > 0.1).float()
        pol = build_reference_policy(env_name, H, W, B, use_self_attn=False)
        sd = pol.state_dict()
        pol.load_state_dict(synth_state_dict_nsa(sd))
        rnn = {"human_node_rnn": h.clone(), "human_human_edge_rnn": torch.zeros(B, H + 1, 256)}
        with torch.no_grad():
            value, feat, hx = pol.base({k: v.clone() for k, v in obs.items()}, rnn, masks.clone(), infer=True)
            mean = pol.dist.fc_mean(feat)
        keys = sorted(sd.keys())
        print(name, "value range", float(value.min()), float(value.max()), "mean abs max", float(mean.abs().max()),
              "detected", float(obs["detected_human_num"].mean()))
        np.savez_compressed(os.path.join(REPO, "tests", "golden", name + ".npz"),
                            h=h.numpy(), masks=masks.numpy(), **{"ob_" + k: v.numpy() for k, v in obs.items()},
                            synth_value=value.numpy(), synth_mean=mean.numpy(), synth_h=hx["human_node_rnn"].numpy(),
                            sd_keys=np.array(keys), sd_shapes=np.array([str(tuple(sd[k].shape)) for k in keys]))


def unsorted_fixtures():
    """args.sort_humans = False: both attentions masked with inputs['visible_masks'] (selfAttn_srnn_temp_node.py:375-383)
    instead of the detected_human_num prefix, for the full network (synthetic fill) and the use_self_attn = False
    ablation.  W = 2: 64 observations of the env_varnum_h20_unsorted_rand rollout (CrowdSimVarNum-v0 with sort_humans =
    False), eight of them with every mask cleared (the reference's dummy_human_mask).  W = 12: the GST wrapper's outputs
    (rows sorted by distance, masks in id order) of gst_rollout (H = 20) and gst_rollout_h50."""
    sys.path.insert(0, os.path.join(REPO, "tests"))
    from tests.policy_fixture import synth_state_dict
    from tests.policy_no_self_attn_ref import synth_state_dict_nsa
    keys = ["robot_node", "temporal_edges", "spatial_edges", "detected_human_num", "visible_masks"]
    for src, prefix, H, W in [("env_varnum_h20_unsorted_rand", "ob_", 20, 2), ("gst_rollout", "fin_", 20, 12),
                              ("gst_rollout_h50", "fin_", 50, 12)]:
        g = np.load(os.path.join(REPO, "tests", "golden", src + ".npz"))
        T1, N = g[prefix + "robot_node"].shape[:2]
        B = 64
        idx = np.random.RandomState(0).choice(T1 * N, B, replace=False)
        obs = {k: torch.from_numpy(g[prefix + k].reshape(T1 * N, *g[prefix + k].shape[2:])[idx]) for k in keys}
        obs = {k: v if k == "visible_masks" else v.float() for k, v in obs.items()}
        if W == 2:
            obs["visible_masks"][::8] = False
        gen = torch.Generator().manual_seed(123)
        h = torch.randn(B, 1, 128, generator=gen) * 0.5
        masks = (torch.rand(B, 1, generator=gen) > 0.1).float()
        env_name = "CrowdSimVarNum-v0" if W == 2 else "CrowdSimPred-v0"
        for net, use_sa in [("full", True), ("nsa", False)]:
            pol = build_reference_policy(env_name, H, W, B, use_self_attn=use_sa)
            pol.base.args.sort_humans = False
            sd = pol.state_dict()
            pol.load_state_dict(synth_state_dict(sd) if use_sa else synth_state_dict_nsa(sd))
            rnn = {"human_node_rnn": h.clone(), "human_human_edge_rnn": torch.zeros(B, H + 1, 256)}
            with torch.no_grad():
                value, feat, hx = pol.base({k: v.clone() for k, v in obs.items()}, rnn, masks.clone(), infer=True)
                mean = pol.dist.fc_mean(feat)
            name = "policy_unsorted_%s_%s" % (net, "varnum" if W == 2 else "h%d" % H)
            vis = obs["visible_masks"].numpy()
            print(name, "value range", float(value.min()), float(value.max()), "visible", float(vis.sum(1).mean()),
                  "none visible", int((vis.sum(1) == 0).sum()),
                  "non-prefix", int(sum(not vis[i, :vis[i].sum()].all() for i in range(B))))
            np.savez_compressed(os.path.join(REPO, "tests", "golden", name + ".npz"),
                                h=h.numpy(), masks=masks.numpy(), **{"ob_" + k: v.numpy() for k, v in obs.items()},
                                synth_value=value.numpy(), synth_mean=mean.numpy(), synth_h=hx["human_node_rnn"].numpy())


def long_h20_recording():
    """The 260-step env_pred_h20 rollout of the reference (the committed fixture keeps only its first steps)."""
    import make_golden
    return make_golden.run_case("env_pred_h20", dict(make_golden.CASES["env_pred_h20"], steps=make_golden.LONG_H20_STEPS))

if __name__ == "__main__":
    if "--unsorted" in sys.argv[1:]:
        unsorted_fixtures()
    else:
        no_self_attn_fixtures() if "--no-self-attn" in sys.argv[1:] else main()
