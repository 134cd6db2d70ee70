"""CPU check of the stage-local fp64 policy reference (tests/policy_stages.py): chained on its own values it must be
the oracle forward (oracle/policy_ref.py in float64), so the GPU stage tests compare against the right function."""
import pytest
import torch

from tests.policy_stages import StagedRef


def _obs(N, H, Win, seed, n):
    gen = torch.Generator().manual_seed(seed)
    sp = torch.randn(N, H, Win, generator=gen, dtype=torch.float64) * 3
    sp[torch.arange(H)[None, :] >= n] = 15.0
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=gen, dtype=torch.float64) * 3,
               temporal_edges=torch.randn(N, 1, 2, generator=gen, dtype=torch.float64),
               spatial_edges=sp, detected_human_num=n.double())
    h = torch.randn(N, 1, 128, generator=gen, dtype=torch.float64)
    masks = (torch.rand(N, 1, generator=gen) > 0.2).double()
    return obs, h, masks


@pytest.mark.parametrize("H", [1, 5, 20, 128])
@pytest.mark.parametrize("Win", [2, 12])
def test_staged_reference_chain_equals_oracle_fp64(H, Win):
    from oracle.policy_ref import PolicyRef
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    N = 7
    gen = torch.Generator().manual_seed(H * 100 + Win)
    n = torch.randint(1, H + 1, (N, 1), generator=gen)
    n[0], n[-1] = H, 1                                     # ragged, with both ends of [1, H]
    sd = make_reference_like_state_dict(Win, seed=H + Win)
    sd["dist.fc_mean.bias"] = torch.tensor([0.3, -0.2])   # non-zero biases where the initialiser sets zeros
    sd["base.critic_linear.bias"] = torch.tensor([0.7])
    ref = PolicyRef(Win)
    ref.load_state_dict(sd)
    ref = ref.double()
    obs, h, masks = _obs(N, H, Win, H + 7 * Win, n)
    with torch.no_grad():
        rv, rm, rh = ref(obs, h, masks)
    st = StagedRef(sd, H).chain(obs, h, masks)
    assert int(st["row_start"][-1]) == int(n.sum())
    for got, want in ((st["value"], rv), (st["mean"], rm), (st["h1"], rh.reshape(N, 128))):
        assert float((got - want).abs().max()) < 1e-10


def test_staged_reference_clamps_detected_human_num():
    """cn_row_offsets_kernel clamps detected_human_num to [1, H] (0 -> 1 as the reference environment does, H + 3 -> H);
    the oracle does not clamp and gives NaN for 0, so the clamp is pinned here on the staged reference alone."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    N, H, Win = 4, 6, 12
    sd = make_reference_like_state_dict(Win, seed=5)
    sref = StagedRef(sd, H)
    n_raw = torch.tensor([[0.0], [H + 3.0], [2.7], [-1.0]])
    n_eff = torch.tensor([[1.0], [float(H)], [2.0], [1.0]])
    obs, h, masks = _obs(N, H, Win, 3, n_eff)
    a = sref.chain(obs, h, masks)
    b = sref.chain(dict(obs, detected_human_num=n_raw.double()), h, masks)
    assert a["n"].tolist() == [1, H, 2, 1]
    for k in ("value", "mean", "h1", "wv"):
        assert torch.equal(a[k], b[k]), k
