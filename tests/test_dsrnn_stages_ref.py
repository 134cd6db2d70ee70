"""CPU check of the stage-local fp64 DS-RNN reference (tests/dsrnn_stages.py): chained on its own values it must be the
oracle forward (oracle/dsrnn_ref.py in float64), and its interleaved edge-GRU operand must compute torch.nn.GRU's cell,
so the GPU stage tests compare against the right function."""
import pytest
import torch

from oracle.dsrnn_ref import DsrnnRef, gru_step
from tests.dsrnn_fixture import dsrnn_state_dict
from tests.dsrnn_stages import DsrnnStages, edge_gru, interleave_gru

F64 = torch.float64


@pytest.mark.parametrize("H", [1, 5, 20, 128])
@pytest.mark.parametrize("W", [2, 12, 16])
def test_staged_reference_chain_equals_oracle_fp64(H, W):
    N = 5
    ref = DsrnnRef(W)
    sd = dsrnn_state_dict(ref.state_dict())
    sd["dist.fc_mean.bias"] = torch.tensor([0.3, -0.2])        # head biases well away from zero
    sd["base.critic_linear.bias"] = torch.tensor([0.7])
    ref.load_state_dict(sd)
    ref = ref.double()
    g = torch.Generator().manual_seed(H * 100 + W)
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=g, dtype=F64) * 3,
               temporal_edges=torch.randn(N, 1, 2, generator=g, dtype=F64),
               spatial_edges=torch.randn(N, H, W, generator=g, dtype=F64) * 4,
               detected_human_num=torch.full((N, 1), float(H), dtype=F64))
    h = torch.randn(N, 1, 128, generator=g, dtype=F64) * 0.5
    he = torch.randn(N, H + 1, 256, generator=g, dtype=F64) * 0.5
    masks = torch.tensor([[1.0], [0.0], [1.0], [1.0], [0.0]], dtype=F64)
    st = DsrnnStages(sd, H, W)
    for edge in (he, None):
        with torch.no_grad():
            rv, rm, rh, rhe = ref(obs, h, torch.zeros_like(he) if edge is None else edge, masks)
        o = st.chain(obs, h, edge, masks)
        for name, got, want in (("value", o["value"], rv), ("mean", o["mean"], rm), ("h1", o["h1"], rh.reshape(N, 128)),
                                ("he1", o["he1"], rhe)):
            err = float((got - want).abs().max())
            assert err < 1e-10, (name, err)


def test_interleaved_edge_gru_equals_gru_step_fp64():
    """h' through the interleaved B [1024, 320] and bias [1024] (the layout the engine's GRU epilogue reads) equals
    torch.nn.GRU's cell, with every bias non-zero so that a bias in the wrong gate block shows."""
    g = torch.Generator().manual_seed(3)
    gru = torch.nn.GRU(64, 256).double()
    with torch.no_grad():
        for prm in gru.parameters():
            prm.copy_(torch.randn(prm.shape, generator=g, dtype=F64) * 0.1)
    M = 37
    x = torch.randn(M, 64, generator=g, dtype=F64).clamp_min(0)
    h = torch.randn(M, 256, generator=g, dtype=F64) * 0.7
    B, bias = interleave_gru(gru.weight_ih_l0.detach(), gru.weight_hh_l0.detach(), gru.bias_ih_l0.detach(),
                             gru.bias_hh_l0.detach())
    assert B.shape == (1024, 320) and bias.shape == (1024,)
    got, scale = edge_gru(torch.cat([x, h], 1), h, B, bias)
    with torch.no_grad():
        want = gru_step(gru, x, h)
    assert float((got - want).abs().max()) < 1e-12
    assert bool((scale > 0).all())
