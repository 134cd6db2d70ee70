"""DS-RNN policy (base='srnn') on the CPU: oracle/dsrnn_ref.py and the Policy mirror's PyTorch update path against
outputs of the UNMODIFIED reference module (tools/make_golden_dsrnn.py), the mirror's state_dict, the env_type check,
and the rollout storage's edge state."""
import numpy as np
import pytest
import torch

from oracle.dsrnn_ref import DsrnnRef
from tests.dsrnn_fixture import ACT_CASES, UNUSED, Args, act_case, dsrnn_state_dict, recurrent_case, reference_shapes, spaces

TOL = 2e-5


def _oracle(W):
    ref = DsrnnRef(W)
    ref.load_state_dict(dsrnn_state_dict(ref.state_dict()))
    return ref


@pytest.mark.parametrize("tag", sorted(ACT_CASES))
def test_oracle_matches_reference_single_step(tag):
    H, W = ACT_CASES[tag]
    obs, ins, outs = act_case(tag)
    with torch.no_grad():
        v, m, h1, he1 = _oracle(W)(obs, ins["h"], ins["he"], ins["masks"])
    for got, key in ((v, "value"), (m, "mean"), (h1, "h1"), (he1, "he1")):
        np.testing.assert_allclose(got.numpy(), outs[key], rtol=0, atol=TOL, err_msg=key)


def test_oracle_matches_reference_recurrent():
    g = recurrent_case()
    T, N = g["masks"].shape[:2]
    H = g["ob_spatial_edges"].shape[2]
    ref = _oracle(2)
    h, he = torch.zeros(N, 1, 128), torch.zeros(N, H + 1, 256)
    for t in range(T):
        obs = {k[3:]: torch.from_numpy(g[k][t]) for k in g.files if k.startswith("ob_")}
        with torch.no_grad():
            v, m, h, he = ref(obs, h, he, torch.from_numpy(g["masks"][t]))
        np.testing.assert_allclose(v.numpy(), g["value"][t], rtol=0, atol=TOL)
        np.testing.assert_allclose(m.numpy(), g["mean"][t], rtol=0, atol=TOL)
        np.testing.assert_allclose(h.numpy(), g["h"][t], rtol=0, atol=TOL)
    np.testing.assert_allclose(he.numpy(), g["he_final"], rtol=0, atol=TOL)


def _mirror(H, W, **kw):
    from crowdnav_prediction_attngraph_b200.policy import Policy
    sp, act = spaces(H, W)
    return Policy(sp, act, base='srnn', base_kwargs=Args(**kw))


def test_mirror_state_dict_is_the_reference_one():
    pol = _mirror(5, 2)
    sd = pol.state_dict()
    assert {k: str(tuple(v.shape)) for k, v in sd.items()} == reference_shapes()
    assert sum(v.numel() for v in sd.values()) == 973989
    b = pol.base
    assert (b.nenv, b.human_num, b.human_node_rnn_size, b.human_human_edge_rnn_size, b.output_size) == (4, 5, 128, 256, 256)
    # a reference-trained checkpoint loads (and the oracle's keys are the same)
    pol.load_state_dict(dsrnn_state_dict(sd))
    assert set(DsrnnRef(2).state_dict()) == set(sd)


@pytest.mark.parametrize("env_type", ["ros", "crowd_sim_pred"])
def test_mirror_refuses_other_env_type(env_type):
    with pytest.raises(NotImplementedError):
        _mirror(5, 2, env_type=env_type)
    _mirror(5, 2, env_type='crowd_sim')


def test_mirror_evaluate_actions_matches_reference_recurrent_run():
    """evaluate_actions over the 30-step recorded run (training-mode GRU segments cut at the done) gives the values
    and action log-probs of the reference's step-by-step rollout, and its final states; gradients reach every
    parameter except the six the forward never reads."""
    g = recurrent_case()
    T, N = g["masks"].shape[:2]
    H = g["ob_spatial_edges"].shape[2]
    pol = _mirror(H, 2, num_processes=N)
    pol.load_state_dict(dsrnn_state_dict(pol.state_dict()))
    inp = {k[3:]: torch.from_numpy(g[k]).reshape(T * N, *g[k].shape[2:]) for k in g.files if k.startswith("ob_")}
    act = torch.from_numpy(g["mean"]).reshape(T * N, 2) + 0.1
    hxs = {'human_node_rnn': torch.zeros(N, 1, 128),
           'human_human_edge_rnn': torch.zeros(1, 1, 1).expand(N, H + 1, 256)}
    v, lp, ent, out = pol.evaluate_actions(inp, hxs, torch.from_numpy(g["masks"]).reshape(T * N, 1), act)
    np.testing.assert_allclose(v.detach().numpy(), g["value"].reshape(T * N, 1), rtol=0, atol=TOL)
    std = pol.dist.logstd._bias.detach().exp().reshape(1, 2)
    ref_lp = torch.distributions.Normal(torch.from_numpy(g["mean"]).reshape(T * N, 2), std).log_prob(act).sum(-1, keepdim=True)
    np.testing.assert_allclose(lp.detach().numpy(), ref_lp.numpy(), rtol=0, atol=1e-4)
    np.testing.assert_allclose(out['human_node_rnn'].detach().numpy(), g["h"][-1], rtol=0, atol=TOL)
    np.testing.assert_allclose(out['human_human_edge_rnn'].detach().numpy(), g["he_final"], rtol=0, atol=TOL)
    (v.sum() + lp.sum() + ent).backward()
    for k, p in pol.named_parameters():
        assert (p.grad is None) == k.startswith(UNUSED), k


def test_storage_keeps_zero_edge_for_attention_graph_and_gathers_dsrnn_edges():
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    H, T, N = 5, 3, 4
    sp, act = spaces(H, 2)

    def insert(st, edge):
        obs = {k: torch.randn(N, *v.shape) for k, v in sp.items()}
        st.insert(obs, {'human_node_rnn': torch.randn(N, 1, 128), 'human_human_edge_rnn': edge}, torch.randn(N, 2),
                  torch.randn(N, 1), torch.randn(N, 1), torch.randn(N, 1), torch.ones(N, 1), torch.ones(N, 1))

    st = RolloutStorage(T, N, sp, act, 128, 256)
    for _ in range(T):
        insert(st, torch.zeros(1, 1, 1).expand(N, H + 1, 256))
    e = st.recurrent_hidden_states['human_human_edge_rnn']
    assert e.stride() == (0, 0, 0, 0) and e.shape == (T + 1, N, H + 1, 256)
    st = RolloutStorage(T, N, sp, act, 128, 256)
    edges = [torch.randn(N, H + 1, 256) for _ in range(T)]
    for ed in edges:
        insert(st, ed)
    e = st.recurrent_hidden_states['human_human_edge_rnn']
    assert e.stride()[0] != 0
    for t in range(T):
        assert torch.equal(e[t + 1], edges[t])
    st.after_update()
    assert torch.equal(e[0], edges[-1])
    gen = torch.Generator().manual_seed(3)
    perm = torch.randperm(N, generator=torch.Generator().manual_seed(3))
    batches = list(st.recurrent_generator(torch.zeros(T, N, 1), 2, generator=gen))
    for i, b in enumerate(batches):
        ind = perm[2 * i:2 * i + 2]
        assert torch.equal(b[1]['human_human_edge_rnn'], edges[-1].index_select(0, ind))
