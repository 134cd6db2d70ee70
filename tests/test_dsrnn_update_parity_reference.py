"""DS-RNN (base='srnn') PPO update path against the UNMODIFIED reference, as tests/test_update_parity_reference.py does
for the attention-graph policy.

Fixture tests/golden/dsrnn_update_t30_n8.npz (tools/make_golden_dsrnn.py update): a recorded CrowdSimVarNum-v0 rollout
[T=30, N=8, H=5] with an episode end in every environment, teacher-forced through the reference SRNN from a seeded
non-zero initial node and edge state; compute_returns, the first minibatch of recurrent_generator through
evaluate_actions, and one PPO.update.  The mirror's storage is filled through its own insert() (the edge state given
to insert switches it to a real edge buffer; only slot 0 reaches the update), on CPU.  Same tolerances as the
attention-graph update test; the six tensors the forward never reads get no gradient and stay unchanged."""
import os

import numpy as np
import torch

from tests.dsrnn_fixture import UNUSED, Args, dsrnn_state_dict, spaces

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
T, N, H = 30, 8, 5
HYPER = dict(clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01,
             lr=4e-5, eps=1e-5, max_grad_norm=0.5)
SEED_GEN = 777


def _fixture():
    return np.load(os.path.join(GOLD, "dsrnn_update_t30_n8.npz"))


def _mirror_policy():
    from crowdnav_prediction_attngraph_b200.policy import Policy
    sp, act = spaces(H, 2)
    pol = Policy(sp, act, base='srnn', base_kwargs=Args(num_processes=N, seq_length=T, num_mini_batch=2))
    pol.load_state_dict(dsrnn_state_dict(pol.state_dict()))
    return pol, sp, act


def _mirror_storage(g, sp, act):
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    ro = RolloutStorage(T, N, sp, act, 128, 256)
    for k in ro.obs:
        ro.obs[k][0].copy_(torch.from_numpy(g["ob_" + k][0]))
    edge = torch.from_numpy(g["edge0"])
    for t in range(T):
        masks = torch.from_numpy(1.0 - g["done"][t].astype(np.float32)).unsqueeze(1)
        ro.insert({k: torch.from_numpy(g["ob_" + k][t + 1]) for k in ro.obs},
                  {'human_node_rnn': torch.from_numpy(g["hidden"][t + 1]), 'human_human_edge_rnn': edge},
                  torch.from_numpy(g["actions"][t]), torch.from_numpy(g["action_log_probs"][t]),
                  torch.from_numpy(g["value_preds"][t]), torch.from_numpy(g["rewards"][t]).unsqueeze(1), masks,
                  torch.ones(N, 1))
    hs = ro.recurrent_hidden_states
    assert hs['human_human_edge_rnn'].stride()[0] != 0
    hs['human_node_rnn'][0].copy_(torch.from_numpy(g["hidden"][0]))
    hs['human_human_edge_rnn'][0].copy_(edge)
    return ro


def _close(a, b, rel):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    scale = max(1.0, float(np.abs(b).max()))
    return float(np.abs(a - b).max()) <= rel * scale, float(np.abs(a - b).max()), scale


def test_dsrnn_evaluate_actions_matches_reference():
    g = _fixture()
    pol, sp, act = _mirror_policy()
    ro = _mirror_storage(g, sp, act)
    assert np.array_equal(ro.masks.numpy(), g["masks"])
    ro.returns.copy_(torch.from_numpy(g["returns"]))
    adv = ro.returns[:-1] - ro.value_preds[:-1]
    adv = (adv - adv.mean()) / (adv.std() + 1e-5)
    torch.manual_seed(SEED_GEN)
    obs_b, hxs_b, act_b, vpred_b, ret_b, masks_b, old_lp_b, adv_b = next(iter(ro.recurrent_generator(adv, 2)))
    assert float(masks_b.min()) == 0.0                     # episode ends inside the minibatch (GRU segments)
    assert np.array_equal(obs_b["spatial_edges"].numpy(), g["mb_spatial_edges"])
    assert np.array_equal(hxs_b["human_node_rnn"].numpy(), g["mb_h0"])
    assert np.array_equal(hxs_b["human_human_edge_rnn"].numpy(), g["mb_edge0"])     # the gathered edge states
    values, lp, ent, hx = pol.evaluate_actions(obs_b, hxs_b, masks_b, act_b)
    for name, a, b in (("values", values, g["mb_values"]), ("logp", lp, g["mb_logp"]),
                       ("h_final", hx["human_node_rnn"], g["mb_h_final"]),
                       ("edge_final", hx["human_human_edge_rnn"], g["mb_edge_final"])):
        ok, err, sc = _close(a.detach().numpy(), b, 1e-5)
        assert ok, (name, err, sc)
    assert abs(float(ent.detach()) - float(g["mb_entropy"])) <= 1e-6
    pol.zero_grad()
    (values.mean() + lp.mean() + ent).backward()
    gn = {k: float(p.grad.norm()) if p.grad is not None else -1.0 for k, p in pol.named_parameters()}
    for k, ref in zip(g["grad_keys"], g["grad_norms"]):
        k = str(k)
        assert (gn[k] < 0) == (ref < 0) == k.startswith(UNUSED), k
        assert abs(gn[k] - ref) <= 2e-4 * max(1.0, abs(ref)), (k, gn[k], ref)


def _mirror_update(g):
    from crowdnav_prediction_attngraph_b200.ppo import PPO
    pol, sp, act = _mirror_policy()
    ro = _mirror_storage(g, sp, act)
    ro.compute_returns(torch.from_numpy(g["value_preds"][-1]), True, 0.99, 0.95, False)
    ok, err, sc = _close(ro.returns.numpy(), g["returns"], 1e-6)
    assert ok, (err, sc)
    agent = PPO(pol, **HYPER)
    torch.manual_seed(SEED_GEN + 1)
    return pol, agent.update(ro)


def test_dsrnn_ppo_update_matches_reference():
    g = _fixture()
    e = np.load(os.path.join(GOLD, "dsrnn_update_t30_n8_entries.npz"))
    pol, losses = _mirror_update(g)
    for a, b, name in zip(losses, g["losses"], ("value_loss", "action_loss", "dist_entropy")):
        assert abs(a - b) <= 1e-5 * max(1.0, abs(b)), (name, a, b)
    sd = pol.state_dict()
    pre = dsrnn_state_dict(sd)
    assert sorted(sd) == [str(k) for k in g["param_keys"]] == [str(k) for k in e["keys"]]
    for i, k in enumerate(g["param_keys"]):
        k = str(k)
        s, ab = float(sd[k].double().sum()), float(sd[k].double().abs().sum())
        assert abs(s - g["param_sum"][i]) <= 1e-6 * max(1.0, g["param_abs"][i]), (k, s, g["param_sum"][i])
        assert abs(ab - g["param_abs"][i]) <= 1e-6 * max(1.0, g["param_abs"][i]), k
        head = np.resize(sd[k].reshape(-1)[:4].double().numpy(), 4)
        assert np.abs(head - g["param_head"][i]).max() <= 2e-6, (k, head, g["param_head"][i])
        # the six tensors the forward never reads stay exactly as loaded; every other one is trained except
        # spatial_edge_layer's bias, which shifts all H attention scores of an environment equally (the soft-max is
        # invariant: zero gradient up to rounding, no change in the reference either)
        if k.startswith(UNUSED):
            assert torch.equal(sd[k], pre[k]), k
        elif k != "base.attn.spatial_edge_layer.0.bias":
            assert not torch.equal(sd[k], pre[k]), k
        lo, hi = int(e["off"][i]), int(e["off"][i + 1])
        d_own = (sd[k] - pre[k]).double().reshape(-1).numpy()[e["idx"][lo:hi]]
        err = float(np.abs(e["delta"][lo:hi].astype(np.float64) - d_own).max())
        assert err <= 1e-6, (k, err)
