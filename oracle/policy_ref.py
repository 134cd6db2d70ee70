"""ORACLE — TEST INFRASTRUCTURE ONLY.  Plain PyTorch fp32 restatement of the reference policy
forward on the rollout path (infer=True), layer for layer and UNFOLDED, following

  rl/networks/selfAttn_srnn_temp_node.py:360-449  selfAttn_merge_SRNN.forward
  rl/networks/selfAttn_srnn_temp_node.py:63-91    SpatialEdgeSelfAttn (+ create_attn_mask :49-60)
  rl/networks/selfAttn_srnn_temp_node.py:145-223  EdgeAttention_M
  rl/networks/selfAttn_srnn_temp_node.py:262-285  EndRNN;  rl/networks/srnn_model.py:35-47 GRU step
  rl/networks/distributions.py:76-95              DiagGaussian

State-dict keys and shapes are the reference's (SURVEY.md §2.3), so shipped checkpoints load.
Pinned against the unmodified reference module: tools/make_golden_policy.py ->
tests/golden/policy_*.npz (tests/test_policy_ref_golden.py).
"""
import numpy as np
import torch
import torch.nn as nn


class _AddBias(nn.Module):
    def __init__(self, n):
        super().__init__()
        self._bias = nn.Parameter(torch.zeros(n, 1))


class _SpatialAttn(nn.Module):
    def __init__(self, input_size):
        super().__init__()
        self.embedding_layer = nn.Sequential(nn.Linear(input_size, 128), nn.ReLU(), nn.Linear(128, 512), nn.ReLU())
        self.q_linear = nn.Linear(512, 512)
        self.v_linear = nn.Linear(512, 512)
        self.k_linear = nn.Linear(512, 512)
        self.multihead_attn = nn.MultiheadAttention(512, 8)


class _HRAttn(nn.Module):
    def __init__(self):
        super().__init__()
        self.temporal_edge_layer = nn.ModuleList([nn.Linear(256, 64)])
        self.spatial_edge_layer = nn.ModuleList([nn.Linear(256, 64)])


class _EndRNN(nn.Module):
    def __init__(self):
        super().__init__()
        self.gru = nn.GRU(128, 128)
        self.encoder_linear = nn.Linear(256, 64)
        self.edge_attention_embed = nn.Linear(256, 64)
        self.output_linear = nn.Linear(128, 256)


class _Base(nn.Module):
    def __init__(self, input_size):
        super().__init__()
        self.humanNodeRNN = _EndRNN()
        self.attn = _HRAttn()
        self.actor = nn.Sequential(nn.Linear(256, 256), nn.Tanh(), nn.Linear(256, 256), nn.Tanh())
        self.critic = nn.Sequential(nn.Linear(256, 256), nn.Tanh(), nn.Linear(256, 256), nn.Tanh())
        self.critic_linear = nn.Linear(256, 1)
        self.robot_linear = nn.Sequential(nn.Linear(9, 256), nn.ReLU())
        self.human_node_final_linear = nn.Linear(256, 2)     # unused in forward, kept for load_state_dict
        self.spatial_attn = _SpatialAttn(input_size)
        self.spatial_linear = nn.Sequential(nn.Linear(512, 256), nn.ReLU())


class _Dist(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc_mean = nn.Linear(256, 2)
        self.logstd = _AddBias(2)


class PolicyRef(nn.Module):
    """forward(obs, h [N,1,128], masks [N,1]) -> (value [N,1], action_mean [N,2], h_new [N,1,128])."""

    def __init__(self, input_size=12):
        super().__init__()
        self.base = _Base(input_size)
        self.dist = _Dist()

    @staticmethod
    def _len_mask(n, H):
        # create_attn_mask: first n entries valid
        return torch.arange(H, device=n.device)[None, :] < n[:, None]

    def forward(self, obs, h, masks):
        b = self.base
        dt = b.robot_linear[0].weight.dtype                              # float32, or float64 after .double()
        sp = obs["spatial_edges"].to(dt)
        N, H, _ = sp.shape
        n = obs["detected_human_num"].reshape(N).to(torch.int64)
        valid = self._len_mask(n, H)                                     # [N,H]
        robot_states = b.robot_linear(torch.cat([obs["temporal_edges"].reshape(N, 2),
                                                 obs["robot_node"].reshape(N, 7)], -1).to(dt))   # [N,256]
        # human-human self attention (sequence-first MultiheadAttention with key_padding_mask)
        sa = b.spatial_attn
        emb = sa.embedding_layer(sp).transpose(0, 1)                     # [H,N,512]
        q, k, v = sa.q_linear(emb), sa.k_linear(emb), sa.v_linear(emb)
        z, _ = sa.multihead_attn(q, k, v, key_padding_mask=torch.logical_not(valid))
        z = z.transpose(0, 1)                                            # [N,H,512]
        hs = b.spatial_linear(z)                                         # [N,H,256]
        # robot-human attention
        te = b.attn.temporal_edge_layer[0](robot_states)                 # [N,64]
        se = b.attn.spatial_edge_layer[0](hs)                            # [N,H,64]
        attn = (te[:, None, :] * se).sum(-1) * (H / np.sqrt(64))
        attn = attn.masked_fill(valid == 0, -1e9)
        attn = torch.softmax(attn, dim=-1)
        weighted = torch.bmm(hs.permute(0, 2, 1), attn.unsqueeze(-1)).squeeze(-1)   # [N,256]
        # node GRU
        r = b.humanNodeRNN
        enc = torch.relu(r.encoder_linear(robot_states))
        edg = torch.relu(r.edge_attention_embed(weighted))
        x = torch.cat([enc, edg], -1).unsqueeze(0)                       # [1,N,128]
        h0 = (h.reshape(N, 128) * masks.reshape(N, 1)).to(dt).unsqueeze(0)
        y, h1 = r.gru(x, h0)
        out = r.output_linear(y[0])                                      # [N,256]
        value = b.critic_linear(b.critic(out))
        mean = self.dist.fc_mean(b.actor(out))
        return value, mean, h1[0].reshape(N, 1, 128)

    def logstd(self):
        return self.dist.logstd._bias.reshape(-1)
