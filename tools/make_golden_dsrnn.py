#!/usr/bin/env python
"""Golden vectors for the DS-RNN policy forward (base = 'srnn'), generated from the UNMODIFIED reference module
(rl.networks.model.Policy -> rl/networks/srnn_model.py SRNN) on the CPU (--no-cuda).

As shipped the reference cannot build this model: SRNN.__init__ reads args.env_type (srnn_model.py:378), which
arguments.py never defines.  The script sets args.env_type = 'crowd_sim', the only value whose robot_linear input
width (7) matches the simulator's robot_node.

Weights are a seeded synthetic fill (make_golden_policy.param_fill) with per-tensor scales taken from the reference's
own initialisation (zero-initialised biases get 0.05) and the output heads boosted as in make_golden_policy.py; the
scales go to tests/golden/dsrnn_param_scales.npz, no weights are committed.  Inputs are observations recorded in
tests/golden/env_*.npz; hidden states come from a seeded torch generator and some masks are zero.

  dsrnn_act.npz        single steps: W = 2 at H = 5 and 20 (env_varnum_*), W = 12 at H = 20 (env_pred_h20)
  dsrnn_recurrent.npz  30 steps of env_varnum_h5 that feed the model its own states, with a done mid-way

`python tools/make_golden_dsrnn.py update` writes the PPO-update fixtures instead, in the manner of
make_golden_update.py: a recorded rollout [T = 30, N = 8] cut from env_varnum_h5 (windows with episodes ending
mid-rollout), teacher-forced through the reference SRNN from a seeded non-zero initial node and edge state, inserted
into the reference RolloutStorage; compute_returns (GAE), the first minibatch of recurrent_generator under a fixed
seed through evaluate_actions (outputs, final states, per-tensor gradient norms of a fixed scalar), ONE PPO.update
(losses, per-tensor sums / abs-sums / leading entries) and the update's change of up to 512 seeded entries of every
parameter tensor:

  dsrnn_update_t30_n8.npz, dsrnn_update_t30_n8_entries.npz
"""
import os
import sys

TOOLS = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(TOOLS)
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
sys.path.insert(0, TOOLS)
from reference_root import reference_root  # noqa: E402
REF = reference_root()
sys.path.insert(0, REF)
sys.path.insert(0, REPO)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from make_golden_policy import param_fill  # noqa: E402

GOLD = os.path.join(REPO, "tests", "golden")
SEED = 2000
OBS_KEYS = ["robot_node", "temporal_edges", "spatial_edges", "detected_human_num"]
# (fixture tag, recorded observations, H, W, env name)
ACT_CASES = [("varnum_h5", "env_varnum_h5", 5, 2, "CrowdSimVarNum-v0"),
             ("varnum_h20", "env_varnum_h20_vis_rand", 20, 2, "CrowdSimVarNum-v0"),
             ("pred_h20", "env_pred_h20", 20, 12, "CrowdSimPred-v0")]


def build_reference_srnn(env_name, H, W, nenv):
    sys.argv = ["x", "--no-cuda", "--env-name", env_name, "--num-processes", str(nenv)]
    import gym
    from arguments import get_args
    from rl.networks.model import Policy
    args = get_args()
    args.env_type = 'crowd_sim'
    obs_space = {"robot_node": gym.spaces.Box(-np.inf, np.inf, (1, 7)),
                 "temporal_edges": gym.spaces.Box(-np.inf, np.inf, (1, 2)),
                 "spatial_edges": gym.spaces.Box(-np.inf, np.inf, (H, W)),
                 "detected_human_num": gym.spaces.Box(-np.inf, np.inf, (1,))}
    act_space = gym.spaces.Box(-np.inf * np.ones(2), np.inf * np.ones(2), dtype=np.float32)
    return Policy(obs_space, act_space, base_kwargs=args, base="srnn")


def scales_of(sd):
    sc = {}
    for k, v in sd.items():
        s = float(v.float().std()) if v.numel() > 1 else 0.0
        sc[k] = s if s > 0 else 0.05
    sc["base.critic_linear.weight"] *= 12.0
    sc["dist.fc_mean.weight"] *= 8.0
    return sc


def step(pol, obs, h, he, masks):
    rnn = {"human_node_rnn": h.clone(), "human_human_edge_rnn": he.clone()}
    with torch.no_grad():
        value, feat, hx = pol.base({k: v.clone() for k, v in obs.items()}, rnn, masks.clone(), infer=True)
        mean = pol.dist.fc_mean(feat)
    return value, mean, hx["human_node_rnn"], hx["human_human_edge_rnn"]


def main():
    torch.manual_seed(0)
    ref_sd = build_reference_srnn("CrowdSimVarNum-v0", 5, 2, 1).state_dict()
    scales = scales_of(ref_sd)
    keys = sorted(scales)
    np.savez(os.path.join(GOLD, "dsrnn_param_scales.npz"), keys=np.array(keys),
             scales=np.array([scales[k] for k in keys]), seed=SEED,
             shapes=np.array([str(tuple(ref_sd[k].shape)) for k in keys]))
    out = {}
    B = 8
    for tag, env_file, H, W, env_name in ACT_CASES:
        g = np.load(os.path.join(GOLD, env_file + ".npz"))
        T1, N = g["ob_robot_node"].shape[:2]
        idx = np.random.RandomState(1).choice(T1 * N, B, replace=False)
        obs = {k: torch.from_numpy(g["ob_" + k].reshape(T1 * N, *g["ob_" + k].shape[2:])[idx].astype(np.float32))
               for k in OBS_KEYS}
        gen = torch.Generator().manual_seed(7)
        h = torch.randn(B, 1, 128, generator=gen) * 0.5
        he = torch.randn(B, H + 1, 256, generator=gen) * 0.5
        masks = (torch.rand(B, 1, generator=gen) > 0.25).float()
        masks[0] = 0.0
        pol = build_reference_srnn(env_name, H, W, B)
        sd = pol.state_dict()
        pol.load_state_dict(param_fill(sd, SEED, scales))
        value, mean, h1, he1 = step(pol, obs, h, he, masks)
        out.update({tag + "_ob_" + k: v.numpy() for k, v in obs.items()})
        out.update({tag + "_h": h.numpy(), tag + "_he": he.numpy(), tag + "_masks": masks.numpy(),
                    tag + "_value": value.numpy(), tag + "_mean": mean.numpy(), tag + "_h1": h1.numpy(),
                    tag + "_he1": he1.numpy()})
        print(tag, "value", float(value.abs().max()), "mean", float(mean.abs().max()), "edge", float(he1.abs().max()))
    np.savez_compressed(os.path.join(GOLD, "dsrnn_act.npz"), **out)

    # 30-step recurrent run on a recorded rollout: the model's own states are fed back, done in env 1 at step 12
    g = np.load(os.path.join(GOLD, "env_varnum_h5.npz"))
    T, H = 30, 5
    N = g["ob_robot_node"].shape[1]
    pol = build_reference_srnn("CrowdSimVarNum-v0", H, 2, N)
    pol.load_state_dict(param_fill(pol.state_dict(), SEED, scales))
    masks = np.ones((T, N, 1), np.float32)
    masks[0] = 0.0
    masks[12, 1] = 0.0
    h, he = torch.zeros(N, 1, 128), torch.zeros(N, H + 1, 256)
    vals, means, hs = [], [], []
    for t in range(T):
        obs = {k: torch.from_numpy(g["ob_" + k][t].astype(np.float32)) for k in OBS_KEYS}
        value, mean, h, he = step(pol, obs, h, he, torch.from_numpy(masks[t]))
        vals.append(value.numpy()); means.append(mean.numpy()); hs.append(h.numpy())
    np.savez_compressed(os.path.join(GOLD, "dsrnn_recurrent.npz"), masks=masks, value=np.stack(vals),
                        mean=np.stack(means), h=np.stack(hs), he_final=he.numpy(),
                        **{"ob_" + k: g["ob_" + k][:T].astype(np.float32) for k in OBS_KEYS})
    print("recurrent: value", float(np.abs(np.stack(vals)).max()))


UT, UN, UH = 30, 8, 5
HYPER = dict(clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01,
             lr=4e-5, eps=1e-5, max_grad_norm=0.5)
SEED_GEN = 777


def cut_rollout(g):
    """8 (environment, start) windows of the recording, each with an episode end at step 11, spaced >= 8 apart"""
    cols = []
    for e in range(g["done"].shape[1]):
        for d in np.nonzero(g["done"][:, e])[0]:
            s = int(d) - 11
            if s >= 0 and s + UT < g["done"].shape[0] and all(e != e2 or abs(s - s2) >= 8 for e2, s2 in cols):
                cols.append((e, s))
    cols = cols[:UN]
    assert len(cols) == UN, cols
    ob = {k: np.stack([g["ob_" + k][s:s + UT + 1, e] for e, s in cols], 1).astype(np.float32) for k in OBS_KEYS}
    act = np.stack([g["actions"][s:s + UT, e] for e, s in cols], 1).astype(np.float32)
    rew = np.stack([g["reward"][s:s + UT, e] for e, s in cols], 1).astype(np.float32)
    done = np.stack([g["done"][s:s + UT, e] for e, s in cols], 1)
    return ob, act, rew, done


def update_main():
    import gym
    from rl.networks.storage import RolloutStorage
    from rl.ppo import PPO
    sc = np.load(os.path.join(GOLD, "dsrnn_param_scales.npz"))
    scales = {str(k): float(v) for k, v in zip(sc["keys"], sc["scales"])}
    ob, act, rew, done = cut_rollout(np.load(os.path.join(GOLD, "env_varnum_h5.npz")))
    pol = build_reference_srnn("CrowdSimVarNum-v0", UH, 2, UN)
    pol.base.nminibatch, pol.base.seq_length = HYPER["num_mini_batch"], UT
    pol.load_state_dict(param_fill(pol.state_dict(), SEED, scales))
    pre = {k: v.clone() for k, v in pol.state_dict().items()}
    spaces = {"robot_node": gym.spaces.Box(-np.inf, np.inf, (1, 7)), "temporal_edges": gym.spaces.Box(-np.inf, np.inf, (1, 2)),
              "spatial_edges": gym.spaces.Box(-np.inf, np.inf, (UH, 2)),
              "detected_human_num": gym.spaces.Box(-np.inf, np.inf, (1,))}
    act_space = gym.spaces.Box(-np.inf * np.ones(2), np.inf * np.ones(2), dtype=np.float32)
    ro = RolloutStorage(UT, UN, spaces, act_space, 128, 256)
    gen = torch.Generator().manual_seed(11)
    ro.recurrent_hidden_states['human_node_rnn'][0].copy_(torch.randn(UN, 1, 128, generator=gen) * 0.5)
    ro.recurrent_hidden_states['human_human_edge_rnn'][0].copy_(torch.randn(UN, UH + 1, 256, generator=gen) * 0.5)
    for k in ro.obs:
        ro.obs[k][0].copy_(torch.from_numpy(ob[k][0]))
    for t in range(UT):
        with torch.no_grad():
            o = {k: ro.obs[k][t] for k in ro.obs}
            hx = {k: ro.recurrent_hidden_states[k][t] for k in ro.recurrent_hidden_states}
            value, feat, hx2 = pol.base(o, hx, ro.masks[t], infer=True)
            a = torch.from_numpy(act[t])
            logp = pol.dist(feat).log_probs(a)
        masks = torch.from_numpy(1.0 - done[t].astype(np.float32)).unsqueeze(1)
        ro.insert({k: torch.from_numpy(ob[k][t + 1]) for k in ro.obs}, hx2, a, logp, value,
                  torch.from_numpy(rew[t]).unsqueeze(1), masks, torch.ones(UN, 1))
    with torch.no_grad():
        o = {k: ro.obs[k][-1] for k in ro.obs}
        hx = {k: ro.recurrent_hidden_states[k][-1] for k in ro.recurrent_hidden_states}
        nv = pol.get_value(o, hx, ro.masks[-1]).detach()
    ro.compute_returns(nv, True, 0.99, 0.95, False)
    out = {"ob_" + k: v for k, v in ob.items()}
    hs = ro.recurrent_hidden_states
    out.update(actions=act, rewards=rew, done=done, value_preds=ro.value_preds.numpy().copy(),
               action_log_probs=ro.action_log_probs.numpy().copy(), returns=ro.returns.numpy().copy(),
               hidden=hs['human_node_rnn'].numpy().copy(), edge0=hs['human_human_edge_rnn'][0].numpy().copy(),
               masks=ro.masks.numpy().copy())
    adv = ro.returns[:-1] - ro.value_preds[:-1]
    adv = (adv - adv.mean()) / (adv.std() + 1e-5)
    torch.manual_seed(SEED_GEN)
    obs_b, hxs_b, act_b, vpred_b, ret_b, masks_b, old_lp_b, adv_b = next(iter(ro.recurrent_generator(adv, HYPER["num_mini_batch"])))
    out.update(mb_adv=adv_b.numpy().copy(), mb_actions=act_b.numpy().copy(), mb_masks=masks_b.numpy().copy(),
               mb_spatial_edges=obs_b["spatial_edges"].numpy().copy(), mb_h0=hxs_b["human_node_rnn"].numpy().copy(),
               mb_edge0=hxs_b["human_human_edge_rnn"].numpy().copy())
    values, lp, ent, hx = pol.evaluate_actions(obs_b, hxs_b, masks_b, act_b)
    out.update(mb_values=values.detach().numpy().copy(), mb_logp=lp.detach().numpy().copy(),
               mb_entropy=np.float64(ent.item()), mb_h_final=hx["human_node_rnn"].detach().numpy().copy(),
               mb_edge_final=hx["human_human_edge_rnn"].detach().numpy().copy())
    pol.zero_grad()
    (values.mean() + lp.mean() + ent).backward()
    gn = {k: float(p.grad.norm()) if p.grad is not None else -1.0 for k, p in pol.named_parameters()}
    out["grad_keys"] = np.array(sorted(gn))
    out["grad_norms"] = np.array([gn[k] for k in sorted(gn)])
    pol.zero_grad()
    agent = PPO(pol, **HYPER)
    torch.manual_seed(SEED_GEN + 1)
    out["losses"] = np.array(agent.update(ro), dtype=np.float64)
    sd = pol.state_dict()
    keys = sorted(sd)
    out["param_keys"] = np.array(keys)
    out["param_sum"] = np.array([float(sd[k].double().sum()) for k in keys])
    out["param_abs"] = np.array([float(sd[k].double().abs().sum()) for k in keys])
    out["param_head"] = np.stack([np.resize(sd[k].reshape(-1)[:4].double().numpy(), 4) for k in keys])
    np.savez_compressed(os.path.join(GOLD, "dsrnn_update_t30_n8.npz"), **out)
    rng = np.random.default_rng(2024)
    idx, off, delta = [], [0], []
    for k in keys:
        n = sd[k].numel()
        i = np.sort(rng.choice(n, min(n, 512), replace=False))
        idx.append(i.astype(np.int32))
        delta.append((sd[k].double() - pre[k].double()).reshape(-1).numpy()[i].astype(np.float32))
        off.append(off[-1] + len(i))
    np.savez_compressed(os.path.join(GOLD, "dsrnn_update_t30_n8_entries.npz"), keys=np.array(keys),
                        idx=np.concatenate(idx), off=np.array(off, dtype=np.int64), delta=np.concatenate(delta))
    print("update: losses", out["losses"], "dones per env", done.sum(0), "minibatch mask zeros",
          int((masks_b == 0).sum()), "unused grads", [k for k in keys if gn.get(k, 0) < 0])


if __name__ == "__main__":
    if sys.argv[1:] == ["update"]:
        update_main()
    else:
        main()
