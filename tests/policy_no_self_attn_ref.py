"""Test references of the policy without human-human attention (the reference's use_self_attn = False,
rl/networks/selfAttn_srnn_temp_node.py:340-345 and :402-416): spatial_linear = Linear(W, 128), ReLU, Linear(128, 256),
ReLU applied to the spatial edges, then the same robot-human attention, node GRU and heads as the full network.

  * `PolicyRefNoSelfAttn`: plain PyTorch restatement of the forward (infer=True), unfolded, with the reference's
    state_dict keys.  Pinned against the unmodified reference by tests/golden/policy_nsa_*.npz
    (tools/make_golden_policy.py --no-self-attn).
  * `synth_state_dict_nsa`: the fixtures' synthetic weights.
  * `StagedRefNoSelfAttn`: the fp64 stage reference of tests/policy_stages.py with the two spatial_linear layers in
    place of the human-human stages, for the engine's compacted rows.
"""
import numpy as np
import torch
import torch.nn as nn

from oracle.policy_ref import PolicyRef
from tests.policy_fixture import synth_state_dict
from tests.policy_stages import StagedRef

SPATIAL_LINEAR = "base.spatial_linear."


def synth_state_dict_nsa(template, seed=1000, layer_seed=2024):
    """Synthetic weights of the network without human-human attention.  Every key it shares with the full network gets
    synth_state_dict's value (the same tensor as in the full network's fixtures).  spatial_linear.0 [128, W] and
    spatial_linear.2 [256, 128] have no counterpart in the shipped checkpoint: their weights come from the reference's
    own initialiser (orthogonal, gain sqrt(2)) and their biases are N(0, 0.1^2), both from torch.Generator(layer_seed
    + i) for the i-th of the four tensors in sorted key order.  (The reference initialises those biases to zero; non-zero
    biases keep the bias path under test.)"""
    out = synth_state_dict({k: v for k, v in template.items() if not k.startswith(SPATIAL_LINEAR)}, seed)
    keys = sorted(k for k in template if k.startswith(SPATIAL_LINEAR))
    assert len(keys) == 4, keys
    for i, k in enumerate(keys):
        g = torch.Generator().manual_seed(layer_seed + i)
        t = torch.empty(tuple(template[k].shape))
        if k.endswith("weight"):
            nn.init.orthogonal_(t, gain=float(np.sqrt(2)), generator=g)
        else:
            t = torch.randn(t.shape, generator=g) * 0.1
        out[k] = t
    return out


class PolicyRefNoSelfAttn(PolicyRef):
    """forward(obs, h [N,1,128], masks [N,1]) -> (value [N,1], action_mean [N,2], h_new [N,1,128])."""

    def __init__(self, input_size=12):
        super().__init__(input_size)
        del self.base.spatial_attn
        self.base.spatial_linear = nn.Sequential(nn.Linear(input_size, 128), nn.ReLU(), nn.Linear(128, 256), nn.ReLU())

    def forward(self, obs, h, masks):
        b = self.base
        dt = b.robot_linear[0].weight.dtype
        sp = obs["spatial_edges"].to(dt)
        N, H, _ = sp.shape
        n = obs["detected_human_num"].reshape(N).to(torch.int64)
        valid = self._len_mask(n, H)
        robot_states = b.robot_linear(torch.cat([obs["temporal_edges"].reshape(N, 2),
                                                 obs["robot_node"].reshape(N, 7)], -1).to(dt))
        hs = b.spatial_linear(sp)                                        # [N,H,256]: no human-human attention
        te = b.attn.temporal_edge_layer[0](robot_states)
        se = b.attn.spatial_edge_layer[0](hs)
        attn = (te[:, None, :] * se).sum(-1) * (H / np.sqrt(64))
        attn = torch.softmax(attn.masked_fill(valid == 0, -1e9), dim=-1)
        weighted = torch.bmm(hs.permute(0, 2, 1), attn.unsqueeze(-1)).squeeze(-1)
        r = b.humanNodeRNN
        x = torch.cat([torch.relu(r.encoder_linear(robot_states)), torch.relu(r.edge_attention_embed(weighted))], -1)
        h0 = (h.reshape(N, 128) * masks.reshape(N, 1)).to(dt).unsqueeze(0)
        y, h1 = r.gru(x.unsqueeze(0), h0)
        out = r.output_linear(y[0])
        return b.critic_linear(b.critic(out)), self.dist.fc_mean(b.actor(out)), h1[0].reshape(N, 1, 128)


class StagedRefNoSelfAttn(StagedRef):
    """StagedRef of the network without human-human attention: `spatial1` (spatial_linear.0 + ReLU on the compacted
    rows, the engine's "e1") and `spatial2` (spatial_linear.2 + ReLU, the engine's "sout"); every later stage is
    StagedRef's."""

    def __init__(self, sd, H, device="cpu"):
        from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
        win = sd["base.spatial_linear.0.weight"].shape[1]
        # StagedRef folds the human-human weights in its constructor: give it stand-ins, then drop what it made of them
        full = make_reference_like_state_dict(win, seed=0)
        full.update({k: v for k, v in sd.items() if not k.startswith("base.spatial_linear.")})
        super().__init__(full, H, device)
        del self.W1, self.b1, self.W2, self.b2, self.Wqkv, self.bqkv, self.Wos, self.bos
        g = lambda k: sd[k].detach().to(device, torch.float64)
        self.L1, self.bl1 = g("base.spatial_linear.0.weight"), g("base.spatial_linear.0.bias")
        self.L2, self.bl2 = g("base.spatial_linear.2.weight"), g("base.spatial_linear.2.bias")

    def spatial1(self, spatial, row_start, row_env):
        e, j = row_env, self.human_index(row_start, row_env)
        y, s = self.lin(spatial.to(self.dev, torch.float64)[e, j], self.L1, self.bl1)
        return y.clamp_min(0), s

    def spatial2(self, e1):
        y, s = self.lin(e1, self.L2, self.bl2)
        return y.clamp_min(0), s

    def chain(self, obs, h, masks):
        f = lambda t: t.to(self.dev, torch.float64)
        N = obs["spatial_edges"].shape[0]
        n, row_start, row_env = self.layout(obs["detected_human_num"])
        o = dict(n=n, row_start=row_start, row_env=row_env)
        o["e1"] = self.spatial1(f(obs["spatial_edges"]), row_start, row_env)[0]
        o["sout"] = self.spatial2(o["e1"])[0]
        o["rs"] = self.robot(self.robot_input(f(obs["robot_node"]), f(obs["temporal_edges"])))[0]
        o["t1"] = self.enc_te(o["rs"])[0]
        te = o["t1"][:, 64:]
        o["u"] = self.u(te)[0]
        o["wv"] = self.hr_attention(o["sout"], o["u"], te, n, row_start)[0]
        o["emb"] = self.emb(o["wv"])[0]
        o["h0"] = f(h).reshape(N, 128) * f(masks).reshape(N, 1)
        o["gi"] = self.gi(torch.cat([o["t1"][:, :64], o["emb"]], 1))[0]
        o["gh"] = self.gh(o["h0"])[0]
        o["h1"] = self.gru(o["gi"], o["gh"], o["h0"])[0]
        o["ac1"] = self.ac1(o["h1"])[0]
        o["a2"] = self.a2(o["ac1"][:, :256])[0]
        o["c2"] = self.c2(o["ac1"][:, 256:])[0]
        o["value"] = self.value(o["c2"])[0]
        o["mean"] = self.mean(o["a2"])[0]
        return o
