"""The PPO update path with args.sort_humans = False against the UNMODIFIED reference, as
tests/test_update_parity_reference.py does for the sorted network.

Fixture tests/golden/update_unsorted_t30_n8.npz (tools/make_golden_update.py --unsorted): a recorded CrowdSimVarNum-v0
rollout [T=30, N=8] with unsorted observations and episodes ending mid-rollout, teacher-forced through the reference
policy with sort_humans = False, the reference storage's GAE and recurrent_generator (visible_masks travels with every
minibatch), evaluate_actions on the first minibatch and ONE PPO.update.  update_unsorted_t30_n8_entries.npz holds the
update's change of up to 512 seeded entries of every parameter tensor, compared entry by entry within 1e-6."""
import os
import types

import numpy as np
import torch

from tests.policy_fixture import synth_state_dict

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
T, N, H, W = 30, 8, 20, 2
HYPER = dict(clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01,
             lr=4e-5, eps=1e-5, max_grad_norm=0.5)
SEED_GEN = 777


def _fixture():
    return np.load(os.path.join(GOLD, "update_unsorted_t30_n8.npz"))


def _mirror_policy():
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
              'detected_human_num': Box((1,)), 'visible_masks': Box((H,), np.bool_)}
    args = types.SimpleNamespace(num_processes=N, seq_length=T, num_mini_batch=2, sort_humans=False)
    pol = Policy(spaces, Box((2,)), base='selfAttn_merge_srnn', base_kwargs=args)
    pol.load_state_dict(synth_state_dict(pol.state_dict()))
    return pol, spaces


def _mirror_storage(g, spaces):
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    ro = RolloutStorage(T, N, spaces, Box((2,)), 128, 256)
    assert ro.obs['visible_masks'].dtype == torch.bool
    for k in ro.obs:
        ro.obs[k][0].copy_(torch.from_numpy(g["ob_" + k][0]))
    for t in range(T):
        masks = torch.from_numpy(1.0 - g["done"][t].astype(np.float32)).unsqueeze(1)
        ro.insert({k: torch.from_numpy(g["ob_" + k][t + 1]) for k in ro.obs},
                  {'human_node_rnn': torch.from_numpy(g["hidden"][t + 1])}, torch.from_numpy(g["actions"][t]),
                  torch.from_numpy(g["action_log_probs"][t]), torch.from_numpy(g["value_preds"][t]),
                  torch.from_numpy(g["rewards"][t]).unsqueeze(1), masks, torch.ones(N, 1))
    return ro


def _close(a, b, rel):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(1.0, float(np.abs(b).max()))
    return float(np.abs(a - b).max()) <= rel * scale, float(np.abs(a - b).max()), scale


def test_rollout_has_non_prefix_masks():
    v = _fixture()["ob_visible_masks"].reshape(-1, H) > 0.5
    cnt = v.sum(1)
    assert sum(not v[i, :cnt[i]].all() for i in range(len(v))) > 50


def test_evaluate_actions_matches_reference():
    g = _fixture()
    pol, spaces = _mirror_policy()
    ro = _mirror_storage(g, spaces)
    ro.returns.copy_(torch.from_numpy(g["returns"]))
    adv = ro.returns[:-1] - ro.value_preds[:-1]
    adv = (adv - adv.mean()) / (adv.std() + 1e-5)
    torch.manual_seed(SEED_GEN)
    obs_b, hxs_b, act_b, vpred_b, ret_b, masks_b, old_lp_b, adv_b = next(iter(ro.recurrent_generator(adv, 2)))
    assert np.array_equal(obs_b["spatial_edges"].numpy(), g["mb_spatial_edges"])     # same permutation, same order
    assert float(masks_b.min()) == 0.0
    for packed in (True, False):
        pol.pack_valid_rows = packed
        values, lp, ent, hx = pol.evaluate_actions(obs_b, hxs_b, masks_b, act_b)
        for name, a, b in (("values", values, g["mb_values"]), ("logp", lp, g["mb_logp"]),
                           ("h_final", hx["human_node_rnn"], g["mb_h_final"])):
            ok, err, sc = _close(a.detach().numpy(), b, 1e-6)
            assert ok, (packed, name, err, sc)
        assert abs(float(ent.detach()) - float(g["mb_entropy"])) <= 1e-6
        pol.zero_grad()
        (values.mean() + lp.mean() + ent).backward()
        gn = {k: float(p.grad.norm()) if p.grad is not None else -1.0 for k, p in pol.named_parameters()}
        for k, ref in zip(g["grad_keys"], g["grad_norms"]):
            k = str(k)
            assert (gn[k] < 0) == (ref < 0), k
            assert abs(gn[k] - ref) <= 2e-4 * max(1.0, abs(ref)), (packed, k, gn[k], ref)


def test_ppo_update_matches_reference():
    from crowdnav_prediction_attngraph_b200.ppo import PPO
    g = _fixture()
    e = np.load(os.path.join(GOLD, "update_unsorted_t30_n8_entries.npz"))
    pol, spaces = _mirror_policy()
    ro = _mirror_storage(g, spaces)
    ro.compute_returns(torch.from_numpy(g["value_preds"][-1]), True, 0.99, 0.95, False)
    ok, err, sc = _close(ro.returns.numpy(), g["returns"], 1e-6)
    assert ok, (err, sc)
    agent = PPO(pol, **HYPER)
    torch.manual_seed(SEED_GEN + 1)
    losses = agent.update(ro)
    for a, b, name in zip(losses, g["losses"], ("value_loss", "action_loss", "dist_entropy")):
        assert abs(a - b) <= 1e-5 * max(1.0, abs(b)), (name, a, b)
    sd = pol.state_dict()
    pre = synth_state_dict(sd)
    for i, k in enumerate(g["param_keys"]):
        k = str(k)
        s, ab = float(sd[k].double().sum()), float(sd[k].double().abs().sum())
        assert abs(s - g["param_sum"][i]) <= 1e-6 * max(1.0, g["param_abs"][i]), (k, s, g["param_sum"][i])
    assert sorted(sd.keys()) == [str(k) for k in e["keys"]]
    for i, k in enumerate(e["keys"]):
        k = str(k)
        lo, hi = int(e["off"][i]), int(e["off"][i + 1])
        d_ref = e["delta"][lo:hi].astype(np.float64)
        d_own = (sd[k] - pre[k]).double().reshape(-1).numpy()[e["idx"][lo:hi]]
        err = float(np.abs(d_ref - d_own).max())
        assert err <= 1e-6, (k, err, float(np.abs(d_ref).max()))
