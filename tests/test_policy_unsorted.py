"""The policy on unsorted humans (the reference's args.sort_humans = False) on the CPU: the masked oracles against
fixtures of the UNMODIFIED reference (tools/make_golden_policy.py --unsorted), the PyTorch update path of Policy against
the oracle, the host build of the environment step against the unsorted CrowdSimVarNum-v0 recordings, and the
configuration gates."""
import os
import types

import numpy as np
import pytest
import torch

from tests.policy_fixture import synth_state_dict
from tests.policy_no_self_attn_ref import synth_state_dict_nsa
from tests.policy_unsorted_ref import PolicyRefNoSelfAttnUnsorted, PolicyRefUnsorted, mask_layout, visible_valid

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
# fixture -> (H, W)
FIXTURES = {"policy_unsorted_%s_%s" % (net, src): hw for net in ("full", "nsa")
            for src, hw in (("varnum", (20, 2)), ("h20", (20, 12)), ("h50", (50, 12)))}
ENV_FIXTURES = ["env_varnum_h20_unsorted_rand", "env_varnum_h6_range2_unsorted"]


def load_unsorted_golden(name):
    g = np.load(os.path.join(GOLD, name + ".npz"))
    obs = {k: torch.from_numpy(g["ob_" + k]) for k in ["robot_node", "temporal_edges", "spatial_edges",
                                                       "detected_human_num", "visible_masks"]}
    return g, obs, torch.from_numpy(g["h"]), torch.from_numpy(g["masks"])


def oracle_for(name):
    W = FIXTURES[name][1]
    if "_nsa_" in name:
        ref = PolicyRefNoSelfAttnUnsorted(W)
        ref.load_state_dict(synth_state_dict_nsa(ref.state_dict()))
    else:
        ref = PolicyRefUnsorted(W)
        ref.load_state_dict(synth_state_dict(ref.state_dict()))
    return ref


def _spaces(H, W):
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    return {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
            'detected_human_num': Box((1,)), 'visible_masks': Box((H,), np.bool_)}


def _policy(H, W, base='selfAttn_merge_srnn', **kw):
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    a = types.SimpleNamespace(num_processes=8, seq_length=30, num_mini_batch=2, **kw)
    return Policy(_spaces(H, W), Box((2,)), base=base, base_kwargs=a)


def test_fixtures_cover_non_prefix_and_empty_masks():
    for name in FIXTURES:
        vis = np.load(os.path.join(GOLD, name + ".npz"))["ob_visible_masks"]
        cnt = vis.sum(1)
        assert sum(not vis[i, :cnt[i]].all() for i in range(len(vis))) >= 32, name
        if name.endswith("varnum"):
            assert (cnt == 0).sum() >= 4, name


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_oracle_matches_reference(name):
    g, obs, h, masks = load_unsorted_golden(name)
    ref = oracle_for(name)
    with torch.no_grad():
        v, m, h1 = ref(obs, h, masks)
    np.testing.assert_allclose(v.numpy(), g["synth_value"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(m.numpy(), g["synth_mean"], rtol=0, atol=2e-5)
    np.testing.assert_allclose(h1.numpy(), g["synth_h"], rtol=0, atol=2e-5)


@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_prefix_oracle_differs_from_reference(name):
    """The fixtures pin the mask: the detected_human_num prefix gives other outputs on the same inputs."""
    from oracle.policy_ref import PolicyRef
    from tests.policy_no_self_attn_ref import PolicyRefNoSelfAttn
    g, obs, h, masks = load_unsorted_golden(name)
    W = FIXTURES[name][1]
    ref = PolicyRefNoSelfAttn(W) if "_nsa_" in name else PolicyRef(W)
    ref.load_state_dict(oracle_for(name).state_dict())
    with torch.no_grad():
        v = ref(obs, h, masks)[0]
    assert np.abs(v.numpy() - g["synth_value"]).max() > 1e-3


@pytest.mark.parametrize("name", sorted(FIXTURES))
@pytest.mark.parametrize("pack", [True, False])
def test_evaluate_actions_matches_reference(name, pack):
    """Policy.evaluate_actions (the PyTorch update path, T = 1) on the fixture's inputs within 1e-4 of the reference's
    outputs, in fp64 against the fp64 oracle within 1e-9; both with and without the packed valid rows."""
    g, obs, h, masks = load_unsorted_golden(name)
    H, W = FIXTURES[name]
    pol = _policy(H, W, sort_humans=False, use_self_attn="_nsa_" not in name)
    pol.load_state_dict(oracle_for(name).state_dict(), strict=False)
    pol.pack_valid_rows = pack
    act = torch.from_numpy(g["synth_mean"]) + 0.3
    with torch.no_grad():
        value, logp, ent, hx = pol.evaluate_actions(obs, {'human_node_rnn': h}, masks, act)
    np.testing.assert_allclose(value.numpy(), g["synth_value"], rtol=0, atol=1e-4)
    np.testing.assert_allclose(hx['human_node_rnn'].numpy(), g["synth_h"], rtol=0, atol=1e-5)
    pol64, ref64 = pol.double(), oracle_for(name).double()
    obs64 = {k: v if k == "visible_masks" else v.double() for k, v in obs.items()}
    with torch.no_grad():
        v64, _, _, hx64 = pol64.evaluate_actions(obs64, {'human_node_rnn': h.double()}, masks.double(), act.double())
        rv, rm, rh = ref64(obs64, h.double(), masks.double())
    np.testing.assert_allclose(v64.numpy(), rv.numpy(), rtol=0, atol=1e-9)
    np.testing.assert_allclose(hx64['human_node_rnn'].numpy(), rh.numpy(), rtol=0, atol=1e-9)


def test_update_gradients_ignore_masked_slots():
    """A masked slot cannot reach any output or gradient: changing its spatial edges changes nothing."""
    name = "policy_unsorted_full_varnum"
    g, obs, h, masks = load_unsorted_golden(name)
    pol = _policy(20, 2, sort_humans=False)
    pol.load_state_dict(oracle_for(name).state_dict(), strict=False)
    valid = visible_valid(obs["visible_masks"], 20)
    act = torch.from_numpy(g["synth_mean"]) + 0.3

    def grads(sp):
        pol.zero_grad()
        o = dict(obs, spatial_edges=sp)
        value, logp, ent, _ = pol.evaluate_actions(o, {'human_node_rnn': h}, masks, act)
        (value.sum() + logp.sum() + ent).backward()
        return value.detach(), {k: p.grad.clone() for k, p in pol.named_parameters() if p.grad is not None}
    v0, g0 = grads(obs["spatial_edges"])
    sp = obs["spatial_edges"].clone()
    sp[~valid] += 5.0
    v1, g1 = grads(sp)
    assert torch.equal(v0, v1)
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k


def test_mask_layout_takes_visible_slots_in_order():
    vis = torch.tensor([[0, 1, 0, 1], [0, 0, 0, 0], [1, 1, 1, 1], [0, 0, 1, 0]], dtype=torch.bool)
    n, row_start, row_env, row_slot = mask_layout(vis, 4)
    assert n.tolist() == [2, 1, 4, 1] and row_start.tolist() == [0, 2, 3, 7, 8]
    assert row_env.tolist() == [0, 0, 1, 2, 2, 2, 2, 3] and row_slot.tolist() == [1, 3, 0, 0, 1, 2, 3, 2]


def _ref_config(env_sort=False):
    ns = types.SimpleNamespace
    return ns(sim=ns(human_num=20, human_num_range=0, predict_steps=5, predict_method="none", circle_radius=6 * 2 ** 0.5,
                     arena_size=6),
              action_space=ns(kinematics="holonomic"), humans=ns(policy="orca", radius=0.3, v_pref=1, FOV=2.0,
                                                                random_goal_changing=False, goal_change_chance=0.5,
                                                                end_goal_changing=True),
              robot=ns(visible=False, radius=0.3, v_pref=1, FOV=2, sensor_range=5),
              env=ns(randomize_attributes=False, time_step=0.25, time_limit=50, val_size=100, test_size=500),
              data=ns(pred_timestep=0.25),
              reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
              orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5), sf=ns(A=2.0, B=1.0, KI=1.0),
              args=ns(sort_humans=env_sort))


def test_config_gates():
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    c = _ref_config()
    d = config_dict_from_reference(c, 8, 425, "CrowdSimVarNum-v0")
    assert d["sort_humans"] == 0 and d["const_vel"] == 0
    assert config_dict_from_reference(c, 8, 425, "CrowdSimVarNum-v0", allow_unsorted=True) == d
    c.sim.predict_method = "const_vel"
    with pytest.raises(NotImplementedError, match="KeyError"):
        config_dict_from_reference(c, 8, 425, "CrowdSimPred-v0")
    c.args.sort_humans = True
    assert config_dict_from_reference(c, 8, 425, "CrowdSimPred-v0")["sort_humans"] == 1


def test_policy_reads_sort_humans():
    assert _policy(20, 2, sort_humans=False).sort_humans is False
    assert _policy(20, 2).sort_humans is True                   # missing: True, as the reference's :376-377
    assert _policy(20, 2, sort_humans=True, use_self_attn=False).sort_humans is True
    # the DS-RNN never reads it and runs densely
    assert _policy(20, 2, base='srnn', sort_humans=False).sort_humans is True


@pytest.mark.parametrize("name", ENV_FIXTURES)
def test_host_build_matches_unsorted_reference_rollout(name):
    from tests.golden_util import load_env_case, replay
    from tests.harness_util import HarnessEnv
    g, case, over = load_env_case(name)
    assert case["sort_humans"] is False
    env = HarnessEnv(sort_humans=0, **over)
    bad = replay(g, case, env.reset, env.step, env.get)
    assert not bad, bad[:5]


def test_unsorted_rollouts_have_non_prefix_masks():
    """The recordings exercise what the prefix cannot express: visible slots after an invisible one."""
    for name in ENV_FIXTURES:
        vis = np.load(os.path.join(GOLD, name + ".npz"))["ob_visible_masks"]
        v = vis.reshape(-1, vis.shape[-1])
        cnt = v.sum(1)
        assert sum(not v[i, :cnt[i]].all() for i in range(len(v))) > 50, name
