#!/usr/bin/env python
"""Golden vectors for the PPO UPDATE path (SURVEY row a22/a23), generated from the UNMODIFIED reference
(rl.networks.model.Policy.evaluate_actions, rl.networks.storage.RolloutStorage, rl.ppo.PPO) in the build
container behind oracle/shims.

A recorded rollout [T=30, N=8] is cut from the 260-step env_pred_h20 recording (two 30-step windows of its 4
environments, chosen so that episodes end mid-rollout), teacher-forced through the reference policy
(synthetic weights = tests/policy_fixture.synth_state_dict) to get value / log-prob / hidden state, inserted
into the reference RolloutStorage, then: compute_returns (GAE), recurrent_generator under a fixed torch seed,
evaluate_actions on the first minibatch and ONE PPO.update (2 epochs x 2 minibatches, entropy_coef != 0 so the
entropy term is pinned).  Stored: the rollout inputs, returns, the minibatch outputs, the three losses and, per
parameter tensor, its sum / abs-sum / first 4 entries after the update.  A second file, update_t30_n8_entries.npz,
holds the update's change of up to 512 seeded entries of EVERY parameter tensor (the full 10 MB of weights do not
fit a fixture), compared entry by entry by tests/test_update_parity_reference.py.

--no-self-attn records the same two files for the reference's ablation without human-human attention
(args.use_self_attn = False; weights tests/policy_no_self_attn_ref.synth_state_dict_nsa):
update_nsa_t30_n8.npz and update_nsa_t30_n8_entries.npz.

--unsorted records the same two files for args.sort_humans = False (both attentions masked with visible_masks), on a
rollout of CrowdSimVarNum-v0 with unsorted observations (W = 2): four 30-step windows of each of the two environments
of tests/golden/env_varnum_h20_unsorted_rand.npz, every observation key, visible_masks included, through the reference
storage.  Weights: the full network's synthetic fill.  update_unsorted_t30_n8.npz and update_unsorted_t30_n8_entries.npz.

    CROWDNAV_REFERENCE_ROOT=<reference checkout> python tools/make_golden_update.py [--no-self-attn | --unsorted]
"""
import os
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
from reference_root import reference_root  # noqa: E402
sys.path.insert(0, reference_root())
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

T, N, H, W = 30, 8, 20, 12
WINDOWS = None      # filled by pick_windows
HYPER = dict(clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01,
             lr=4e-5, eps=1e-5, max_grad_norm=0.5)
SEED_GEN = 777
USE_SELF_ATTN = "--no-self-attn" not in sys.argv[1:]
UNSORTED = "--unsorted" in sys.argv[1:]
if UNSORTED:
    W = 2
OBS_KEYS = ["robot_node", "temporal_edges", "spatial_edges", "detected_human_num"] + (["visible_masks"] if UNSORTED else [])


def synth(template):
    if USE_SELF_ATTN:
        from policy_fixture import synth_state_dict
        return synth_state_dict(template)
    from policy_no_self_attn_ref import synth_state_dict_nsa
    return synth_state_dict_nsa(template)


def pick_windows(done, per_env=2):
    """`per_env` window starts per source env such that every window holds at least one episode end in steps 3..26"""
    starts = []
    for e in range(done.shape[1]):
        idx = np.nonzero(done[:, e])[0]
        got = []
        for d in idx:
            s = int(d) - 11
            if s >= 0 and s + T < done.shape[0] and all(abs(s - g) >= 8 for g in got):
                got.append(s)
            if len(got) == per_env:
                break
        assert len(got) == per_env, (e, idx)
        starts.append(got)
    return starts


def cut_rollout(g):
    ne = g["done"].shape[1]                                       # 4 source envs (env_pred_h20) or 2 (unsorted VarNum)
    starts = pick_windows(g["done"], N // ne)
    cols = [(e, s) for e in range(ne) for s in starts[e]]         # 8 (source env, start) pairs
    ob = {}
    for k in OBS_KEYS:
        ob[k] = np.stack([g["ob_" + k][s:s + T + 1, e] for e, s in cols], 1).astype(np.float32)
    act = np.stack([g["actions"][s:s + T, e] for e, s in cols], 1).astype(np.float32)
    rew = np.stack([g["reward"][s:s + T, e] for e, s in cols], 1).astype(np.float32)
    done = np.stack([g["done"][s:s + T, e] for e, s in cols], 1)
    return ob, act, rew, done


def reference_objects():
    from make_golden_policy import build_reference_policy
    argv = sys.argv
    pol = build_reference_policy("CrowdSimVarNum-v0" if UNSORTED else "CrowdSimPred-v0", H, W, N,
                                 use_self_attn=USE_SELF_ATTN)
    sys.argv = argv
    if UNSORTED:
        pol.base.args.sort_humans = False
    pol.base.nminibatch = HYPER["num_mini_batch"]
    pol.base.seq_length = T
    pol.load_state_dict(synth(pol.state_dict()))
    return pol


def fill_storage(pol, storage_cls, ob, act, rew, done, spaces, act_space):
    """train.py:152-191 with the recorded actions instead of sampled ones."""
    ro = storage_cls(T, N, spaces, act_space, 128, 256)
    for k in ro.obs:
        ro.obs[k][0].copy_(torch.from_numpy(ob[k][0]))
    for t in range(T):
        with torch.no_grad():
            o = {k: ro.obs[k][t] for k in ro.obs}
            hx = {k: ro.recurrent_hidden_states[k][t] for k in ro.recurrent_hidden_states}
            value, feat, hx2 = pol.base(o, hx, ro.masks[t], infer=True)
            dist = pol.dist(feat)
            a = torch.from_numpy(act[t])
            logp = dist.log_probs(a)
        masks = torch.from_numpy(1.0 - done[t].astype(np.float32)).unsqueeze(1)
        ro.insert({k: torch.from_numpy(ob[k][t + 1]) for k in ro.obs}, hx2, a, logp, value,
                  torch.from_numpy(rew[t]).unsqueeze(1), masks, torch.ones(N, 1))
    with torch.no_grad():
        o = {k: ro.obs[k][-1] for k in ro.obs}
        hx = {k: ro.recurrent_hidden_states[k][-1] for k in ro.recurrent_hidden_states}
        nv = pol.get_value(o, hx, ro.masks[-1]).detach()
    ro.compute_returns(nv, True, 0.99, 0.95, False)
    return ro


def spaces_for_reference():
    import gym
    sp = {"robot_node": gym.spaces.Box(-np.inf, np.inf, (1, 7)), "temporal_edges": gym.spaces.Box(-np.inf, np.inf, (1, 2)),
          "spatial_edges": gym.spaces.Box(-np.inf, np.inf, (H, W)), "detected_human_num": gym.spaces.Box(-np.inf, np.inf, (1,))}
    if UNSORTED:
        sp["visible_masks"] = gym.spaces.Box(-np.inf, np.inf, (H,))
    return sp, gym.spaces.Box(-np.inf * np.ones(2), np.inf * np.ones(2), dtype=np.float32)


def run_reference():
    """Everything the fixture stores, computed by the unmodified reference.  Returns (dict of arrays, policy)."""
    from rl.networks.storage import RolloutStorage
    from rl.ppo import PPO
    from make_golden_policy import long_h20_recording
    src = np.load(os.path.join(REPO, "tests", "golden", "env_varnum_h20_unsorted_rand.npz")) if UNSORTED \
        else long_h20_recording()
    ob, act, rew, done = cut_rollout(src)
    pol = reference_objects()
    spaces, act_space = spaces_for_reference()
    ro = fill_storage(pol, RolloutStorage, ob, act, rew, done, spaces, act_space)
    out = {"ob_" + k: v for k, v in ob.items()}
    out.update(actions=act, rewards=rew, done=done, value_preds=ro.value_preds.numpy().copy(),
               action_log_probs=ro.action_log_probs.numpy().copy(), returns=ro.returns.numpy().copy(),
               hidden=ro.recurrent_hidden_states['human_node_rnn'].numpy().copy(), masks=ro.masks.numpy().copy())
    adv = ro.returns[:-1] - ro.value_preds[:-1]
    adv = (adv - adv.mean()) / (adv.std() + 1e-5)
    torch.manual_seed(SEED_GEN)
    sample = next(iter(ro.recurrent_generator(adv, HYPER["num_mini_batch"])))
    obs_b, hxs_b, act_b, vpred_b, ret_b, masks_b, old_lp_b, adv_b = sample
    out.update(mb_adv=adv_b.numpy().copy(), mb_actions=act_b.numpy().copy(), mb_masks=masks_b.numpy().copy(),
               mb_spatial_edges=obs_b["spatial_edges"].numpy().copy(), mb_h0=hxs_b["human_node_rnn"].numpy().copy())
    values, lp, ent, hx = pol.evaluate_actions(obs_b, hxs_b, masks_b, act_b)
    out.update(mb_values=values.detach().numpy().copy(), mb_logp=lp.detach().numpy().copy(), mb_entropy=np.float64(ent.item()),
               mb_h_final=hx["human_node_rnn"].detach().numpy().copy())
    # gradient of a fixed scalar through evaluate_actions (no optimiser involved)
    pol.zero_grad()
    (values.mean() + lp.mean() + ent).backward()
    gn = {k: float(p.grad.norm()) if p.grad is not None else -1.0 for k, p in pol.named_parameters()}
    out["grad_keys"] = np.array(sorted(gn.keys()))
    out["grad_norms"] = np.array([gn[k] for k in sorted(gn.keys())])
    pol.zero_grad()
    agent = PPO(pol, **HYPER)
    torch.manual_seed(SEED_GEN + 1)
    vl, al, de = agent.update(ro)
    out.update(losses=np.array([vl, al, de], dtype=np.float64))
    sd = pol.state_dict()
    keys = sorted(sd.keys())
    out["param_keys"] = np.array(keys)
    out["param_sum"] = np.array([float(sd[k].double().sum()) for k in keys])
    out["param_abs"] = np.array([float(sd[k].double().abs().sum()) for k in keys])
    out["param_head"] = np.stack([np.resize(sd[k].reshape(-1)[:4].double().numpy(), 4) for k in keys])
    return out, pol


ENTRIES_PER_TENSOR = 512


def sample_entries(pol):
    """Seeded sample of the update's parameter change: up to ENTRIES_PER_TENSOR flat indices of every tensor (sorted
    keys), the entries' change from the synthetic initial weights."""
    sd = pol.state_dict()
    pre = synth(sd)
    rng = np.random.default_rng(2024)
    keys, idx, off, delta = sorted(sd.keys()), [], [0], []
    for k in keys:
        n = sd[k].numel()
        i = np.sort(rng.choice(n, min(n, ENTRIES_PER_TENSOR), replace=False))
        d = (sd[k].double() - pre[k].double()).reshape(-1).numpy()[i]
        idx.append(i.astype(np.int32))
        delta.append(d.astype(np.float32))
        off.append(off[-1] + len(i))
    return dict(keys=np.array(keys), idx=np.concatenate(idx), off=np.array(off, dtype=np.int64), delta=np.concatenate(delta))


if __name__ == "__main__":
    out, ref_pol = run_reference()
    tag = "update_unsorted_t30_n8" if UNSORTED else ("update_t30_n8" if USE_SELF_ATTN else "update_nsa_t30_n8")
    p = os.path.join(REPO, "tests", "golden", tag + ".npz")
    np.savez_compressed(p, **out)
    np.savez_compressed(os.path.join(REPO, "tests", "golden", tag + "_entries.npz"), **sample_entries(ref_pol))
    print("wrote", p, os.path.getsize(p), "bytes; losses", out["losses"], "entropy", out["mb_entropy"],
          "dones per env", out["done"].sum(0))
