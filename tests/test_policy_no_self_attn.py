"""The policy without human-human attention (the reference's args.use_self_attn = False) on the CPU: the oracle and the
engine's module tree against fixtures of the UNMODIFIED reference (tools/make_golden_policy.py --no-self-attn,
tools/make_golden_update.py --no-self-attn), the PyTorch update path against one reference PPO.update, and the argument
checks of Policy."""
import os

import numpy as np
import pytest
import torch

from tests.policy_fixture import load_policy_golden
from tests.policy_no_self_attn_ref import PolicyRefNoSelfAttn, synth_state_dict_nsa

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FIXTURES = {"policy_nsa_h20": (20, 12), "policy_nsa_h50": (50, 12), "policy_nsa_varnum": (20, 2)}


def _spaces(H, W):
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    return {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
            'detected_human_num': Box((1,))}


def _args(**kw):
    class Args(object):
        num_processes, seq_length, num_mini_batch = 8, 30, 2
    a = Args()
    for k, v in kw.items():
        setattr(a, k, v)
    return a


def _policy(H, W, base='selfAttn_merge_srnn', **kw):
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    return Policy(_spaces(H, W), Box((2,)), base=base, base_kwargs=_args(**kw))


def _tree(module):
    return {k: tuple(v.shape) for k, v in module.state_dict().items()}


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_oracle_matches_reference(name):
    g, obs, h, masks = load_policy_golden(name)
    ref = PolicyRefNoSelfAttn(FIXTURES[name][1])
    ref.load_state_dict(synth_state_dict_nsa(ref.state_dict()))
    with torch.no_grad():
        v, m, h1 = ref(obs, h, masks)
    np.testing.assert_allclose(v.numpy(), g["synth_value"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(m.numpy(), g["synth_mean"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(h1.numpy(), g["synth_h"], rtol=0, atol=2e-5)


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_state_dict_keys_and_shapes_equal_reference(name):
    """Checkpoints interchange both ways: the engine's keys and shapes are the reference module's, and no
    spatial_attn.* key exists."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    g = np.load(os.path.join(GOLD, name + ".npz"))
    recorded = {str(k): str(s) for k, s in zip(g["sd_keys"], g["sd_shapes"])}
    H, W = FIXTURES[name]
    pol = _policy(H, W, use_self_attn=False)
    assert {k: str(s) for k, s in _tree(pol).items()} == recorded
    assert {k: str(tuple(v.shape)) for k, v in make_reference_like_state_dict(W, self_attn=False).items()} == recorded
    assert not any(k.startswith("base.spatial_attn.") for k in recorded)
    # a reference-made state dict loads strictly into the engine, and the engine's loads into the oracle
    sd = synth_state_dict_nsa(pol.state_dict())
    pol.load_state_dict(sd)
    ref = PolicyRefNoSelfAttn(W)
    ref.load_state_dict(pol.state_dict())
    # the full network's state dict does not load into the ablation
    with pytest.raises(RuntimeError):
        pol.load_state_dict(_policy(H, W).state_dict())


def test_initialisers_are_the_reference_ones():
    """spatial_linear of the ablation: orthogonal weights with gain sqrt(2) and zero biases (init_ in the reference)."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    sd = make_reference_like_state_dict(12, seed=3, self_attn=False)
    for i, (rows, cols) in ((0, (128, 12)), (2, (256, 128))):
        w = sd["base.spatial_linear.%d.weight" % i].double()
        assert tuple(w.shape) == (rows, cols)
        gram = w.T @ w if rows > cols else w @ w.T
        assert torch.allclose(gram, 2.0 * torch.eye(min(rows, cols), dtype=torch.float64), atol=1e-5)
        assert not sd["base.spatial_linear.%d.bias" % i].any()


def test_use_hr_attn_changes_nothing():
    for use_self_attn in (True, False):
        a = _tree(_policy(20, 12, use_self_attn=use_self_attn, use_hr_attn=True))
        b = _tree(_policy(20, 12, use_self_attn=use_self_attn, use_hr_attn=False))
        assert a == b


def test_missing_use_self_attn_means_true():
    assert _tree(_policy(20, 12)) == _tree(_policy(20, 12, use_self_attn=True))
    assert any(k.startswith("base.spatial_attn.") for k in _tree(_policy(20, 12)))


def test_srnn_ignores_use_self_attn():
    a = _policy(20, 2, base='srnn', use_self_attn=False)
    b = _policy(20, 2, base='srnn', use_self_attn=True)
    assert _tree(a) == _tree(b) and a.self_attn and b.self_attn


WIDTHS = [("human_node_rnn_size", 128), ("human_human_edge_rnn_size", 256), ("human_node_output_size", 256),
          ("human_node_embedding_size", 64), ("human_human_edge_embedding_size", 64), ("attention_size", 64)]


@pytest.mark.parametrize("base", ['selfAttn_merge_srnn', 'srnn'])
@pytest.mark.parametrize("name,width", WIDTHS)
def test_unsupported_width_is_refused(base, name, width):
    W = 2 if base == 'srnn' else 12
    _policy(20, W, base=base, **{name: width})                       # the engine's own width is accepted
    if base == 'selfAttn_merge_srnn' and name == "human_human_edge_embedding_size":
        _policy(20, W, base=base, **{name: 2 * width})               # its module never reads it
        return
    with pytest.raises(NotImplementedError, match="%s = %d" % (name, 2 * width)):
        _policy(20, W, base=base, **{name: 2 * width})


# ---- the PPO update against the reference's (update_nsa_t30_n8*.npz); as tests/test_update_parity_reference.py ------
T, N, H = 30, 8, 20
HYPER = dict(clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01,
             lr=4e-5, eps=1e-5, max_grad_norm=0.5)
SEED_GEN = 777


def _update_fixture():
    return np.load(os.path.join(GOLD, "update_nsa_t30_n8.npz"))


def _mirror():
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    pol = Policy(_spaces(H, 12), Box((2,)), base='selfAttn_merge_srnn', base_kwargs=_args(num_processes=N, seq_length=T,
                                                                                          use_self_attn=False))
    pol.load_state_dict(synth_state_dict_nsa(pol.state_dict()))
    return pol


def _storage(g):
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    ro = RolloutStorage(T, N, _spaces(H, 12), Box((2,)), 128, 256)
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
    return float(np.abs(a - b).max()) <= rel * max(1.0, float(np.abs(b).max()))


def test_evaluate_actions_matches_reference():
    g = _update_fixture()
    pol = _mirror()
    ro = _storage(g)
    ro.returns.copy_(torch.from_numpy(g["returns"]))
    adv = ro.returns[:-1] - ro.value_preds[:-1]
    adv = (adv - adv.mean()) / (adv.std() + 1e-5)
    torch.manual_seed(SEED_GEN)
    obs_b, hxs_b, act_b, _, _, masks_b, _, _ = next(iter(ro.recurrent_generator(adv, 2)))
    assert np.array_equal(obs_b["spatial_edges"].numpy(), g["mb_spatial_edges"])
    assert float(masks_b.min()) == 0.0
    for packed in (True, False):
        pol.pack_valid_rows = packed
        values, lp, ent, hx = pol.evaluate_actions(obs_b, hxs_b, masks_b, act_b)
        for name, a, b in (("values", values, g["mb_values"]), ("logp", lp, g["mb_logp"]),
                           ("h_final", hx["human_node_rnn"], g["mb_h_final"])):
            assert _close(a.detach().numpy(), b, 1e-5), (packed, name)
        assert abs(float(ent.detach()) - float(g["mb_entropy"])) <= 1e-6
        pol.zero_grad()
        (values.mean() + lp.mean() + ent).backward()
        gn = {k: float(p.grad.norm()) if p.grad is not None else -1.0 for k, p in pol.named_parameters()}
        assert sorted(gn) == [str(k) for k in g["grad_keys"]]
        for k, ref in zip(g["grad_keys"], g["grad_norms"]):
            k = str(k)
            assert (gn[k] < 0) == (ref < 0), k
            assert abs(gn[k] - ref) <= 2e-4 * max(1.0, abs(ref)), (packed, k, gn[k], ref)


def test_ppo_update_matches_reference():
    from crowdnav_prediction_attngraph_b200.ppo import PPO
    g = _update_fixture()
    e = np.load(os.path.join(GOLD, "update_nsa_t30_n8_entries.npz"))
    pol = _mirror()
    ro = _storage(g)
    ro.compute_returns(torch.from_numpy(g["value_preds"][-1]), True, 0.99, 0.95, False)
    agent = PPO(pol, **HYPER)
    torch.manual_seed(SEED_GEN + 1)
    losses = agent.update(ro)
    for a, b, name in zip(losses, g["losses"], ("value_loss", "action_loss", "dist_entropy")):
        assert abs(a - b) <= 1e-5 * max(1.0, abs(b)), (name, a, b)
    sd = pol.state_dict()
    pre = synth_state_dict_nsa(sd)
    assert sorted(sd.keys()) == [str(k) for k in g["param_keys"]] == [str(k) for k in e["keys"]]
    for i, k in enumerate(g["param_keys"]):
        k = str(k)
        assert abs(float(sd[k].double().sum()) - g["param_sum"][i]) <= 1e-6 * max(1.0, g["param_abs"][i]), k
        head = np.resize(sd[k].reshape(-1)[:4].double().numpy(), 4)
        assert np.abs(head - g["param_head"][i]).max() <= 2e-6, k
        lo, hi = int(e["off"][i]), int(e["off"][i + 1])
        d_own = (sd[k] - pre[k]).double().reshape(-1).numpy()[e["idx"][lo:hi]]
        assert np.abs(e["delta"][lo:hi].astype(np.float64) - d_own).max() <= 1e-6, k
    assert all(bool((sd[k] != pre[k]).any()) for k in sd if k.startswith("base.spatial_linear."))
