"""ORACLE — TEST INFRASTRUCTURE ONLY.  Plain PyTorch fp32 restatement of the reference's DS-RNN policy forward
(base = 'srnn') on the rollout path (infer=True), layer for layer and UNFOLDED, following

  rl/networks/srnn_model.py:326-468  SRNN.forward (robot_linear, edge / node RNNs, heads)
  rl/networks/srnn_model.py:177-218  HumanHumanEdgeRNN (encoder_linear + ReLU, GRU 64 -> 256)
  rl/networks/srnn_model.py:256-323  EdgeAttention (one head, temperature H / sqrt(64), no mask)
  rl/networks/srnn_model.py:112-174  HumanNodeRNN (encoder_linear + ReLU, edge_attention_embed + ReLU, GRU, output_linear)
  rl/networks/distributions.py:76-95 DiagGaussian

State-dict keys and shapes are the reference's, so its checkpoints load.  Pinned against the unmodified reference
module: tools/make_golden_dsrnn.py -> tests/golden/dsrnn_*.npz (tests/test_dsrnn_oracle_golden.py).
"""
import torch
import torch.nn as nn


class _AddBias(nn.Module):
    def __init__(self, n):
        super().__init__()
        self._bias = nn.Parameter(torch.zeros(n, 1))


class _EdgeRNN(nn.Module):
    def __init__(self, input_size):
        super().__init__()
        self.gru = nn.GRU(64, 256)
        self.encoder_linear = nn.Linear(input_size, 64)


class _NodeRNN(nn.Module):
    def __init__(self):
        super().__init__()
        self.gru = nn.GRU(128, 128)
        self.encoder_linear = nn.Linear(3, 64)
        self.edge_embed = nn.Linear(256, 64)
        self.edge_attention_embed = nn.Linear(512, 64)
        self.output_linear = nn.Linear(128, 256)


class _EdgeAttn(nn.Module):
    def __init__(self):
        super().__init__()
        self.temporal_edge_layer = nn.ModuleList([nn.Linear(256, 64)])
        self.spatial_edge_layer = nn.ModuleList([nn.Linear(256, 64)])


class _Base(nn.Module):
    def __init__(self, input_size):
        super().__init__()
        self.humanNodeRNN = _NodeRNN()
        self.humanhumanEdgeRNN_spatial = _EdgeRNN(input_size)
        self.humanhumanEdgeRNN_temporal = _EdgeRNN(2)
        self.attn = _EdgeAttn()
        self.actor = nn.Sequential(nn.Linear(256, 256), nn.Tanh(), nn.Linear(256, 256), nn.Tanh())
        self.critic = nn.Sequential(nn.Linear(256, 256), nn.Tanh(), nn.Linear(256, 256), nn.Tanh())
        self.critic_linear = nn.Linear(256, 1)
        self.robot_linear = nn.Linear(7, 3)
        self.human_node_final_linear = nn.Linear(256, 2)     # never read by the forward
        self.spatial_linear = nn.Linear(input_size, 2)       # never read by the forward


def gru_step(gru, x, h):
    """One step of torch.nn.GRU (gate order r, z, n), written out."""
    gi = x @ gru.weight_ih_l0.t() + gru.bias_ih_l0
    gh = h @ gru.weight_hh_l0.t() + gru.bias_hh_l0
    ir, iz, inn = gi.chunk(3, -1)
    hr, hz, hn = gh.chunk(3, -1)
    r = torch.sigmoid(ir + hr)
    z = torch.sigmoid(iz + hz)
    n = torch.tanh(inn + r * hn)
    return (1 - z) * n + z * h


class DsrnnRef(nn.Module):
    def __init__(self, input_size):
        super().__init__()
        self.base = _Base(input_size)
        dist = nn.Module()
        dist.fc_mean = nn.Linear(256, 2)
        dist.logstd = _AddBias(2)
        self.dist = dist

    def forward(self, obs, h_node, h_edge, masks):
        """obs: dict [N,1,7] / [N,1,2] / [N,H,W]; h_node [N,1,128]; h_edge [N,H+1,256]; masks [N,1].
        Returns value [N,1], action mean [N,2], new node state [N,1,128], new edge state [N,H+1,256]."""
        b = self.base
        N, H = obs['spatial_edges'].shape[:2]
        m = masks.reshape(N, 1)
        he = h_edge * m[:, :, None]
        # temporal edge RNN: one row per environment
        et = b.humanhumanEdgeRNN_temporal
        xt = torch.relu(et.encoder_linear(obs['temporal_edges'].reshape(N, 2)))
        ht = gru_step(et.gru, xt, he[:, 0])
        # spatial edge RNN: one row per (environment, human slot), all H slots
        es = b.humanhumanEdgeRNN_spatial
        xs = torch.relu(es.encoder_linear(obs['spatial_edges'].reshape(N * H, -1)))
        hs = gru_step(es.gru, xs, he[:, 1:].reshape(N * H, 256)).reshape(N, H, 256)
        # edge attention: dot product of the embedded temporal and spatial states, soft-max over the H slots
        te = b.attn.temporal_edge_layer[0](ht)
        se = b.attn.spatial_edge_layer[0](hs)
        score = (te[:, None, :] * se).sum(-1) * (H / 8.0)
        p = torch.softmax(score, dim=-1)
        wv = (p[:, :, None] * hs).sum(1)
        # node RNN
        nr = b.humanNodeRNN
        enc = torch.relu(nr.encoder_linear(b.robot_linear(obs['robot_node'].reshape(N, 7))))
        emb = torch.relu(nr.edge_attention_embed(torch.cat([ht, wv], -1)))
        hn = gru_step(nr.gru, torch.cat([enc, emb], -1), h_node.reshape(N, 128) * m)
        x = nr.output_linear(hn)
        value = b.critic_linear(b.critic(x))
        mean = self.dist.fc_mean(b.actor(x))
        return value, mean, hn.reshape(N, 1, 128), torch.cat([ht[:, None], hs], 1)
