"""Stage-local fp64 reference of the DS-RNN rollout forward (cn_dsrnn_act, base='srnn'), in plain torch.

Every stage is a function of its own inputs, so a test can feed it the CUDA engine's input to that stage (read back
through the internal hook cn_internal_dsrnn_buffer, see `read`) and compare the engine's output of that stage alone.
Chained on its own values (`DsrnnStages.chain`) it is the whole forward, which pins it against oracle/dsrnn_ref.py.
It uses the engine's layout and folds (csrc/cn_dsrnn.cu), done here in fp64 from the unfolded state dict:

  * humanNodeRNN.encoder_linear o robot_linear -> one 7 -> 64 layer (Wrob, brob);
  * [actor.0 ; critic.0] o humanNodeRNN.output_linear -> one 128 -> 512 layer (Woac, boac);
  * the attention score te . (W_s s + b_s) = u . s + b_s . te with u = W_s^T te;
  * each edge GRU is one GEMM [x_emb (64) | m h (256)] @ B^T + bias with B [1024, 320] and bias [1024] interleaved as
    `interleave_gru` builds them: column 256 t + 64 q + j holds gate q (r, z, gi_n, gh_n) of hidden unit 64 t + j.

Linear stages also return |X| @ |W|^T + |b|, the scale of a componentwise error bound; the edge GRU returns the
scale of its own bound (see `edge_gru`).
"""
import torch

from tests import policy_stages
from tests.policy_stages import StagedRef, _w

F64 = torch.float64
EDGE = 256
HOOK = "cn_internal_dsrnn_buffer"


def interleave_gru(wih, whh, bih, bhh):
    """B operand [1024, 320] and bias [1024] of the edge-GRU GEMM from torch.nn.GRU(64, 256)'s weight_ih_l0 [768, 64],
    weight_hh_l0 [768, 256], bias_ih_l0, bias_hh_l0 (gate blocks r, z, n).  Column tile t (256 columns) holds, for hidden
    units 64 t .. 64 t + 63:  r: [W_ir | W_hr], b_ir + b_hr;  z: [W_iz | W_hz], b_iz + b_hz;  gi_n: [W_in | 0], b_in;
    gh_n: [0 | W_hn], b_hn."""
    wr, wz, wn = wih.reshape(3, EDGE, 64)
    hr, hz, hn = whh.reshape(3, EDGE, EDGE)
    bir, biz, bin_ = bih.reshape(3, EDGE)
    bhr, bhz, bhn = bhh.reshape(3, EDGE)
    z64, z256 = torch.zeros_like(wr), torch.zeros_like(hr)
    B = torch.stack([torch.cat([wr, hr], 1), torch.cat([wz, hz], 1), torch.cat([wn, z256], 1),
                     torch.cat([z64, hn], 1)])                                  # [q, unit, 320]
    bias = torch.stack([bir + bhr, biz + bhz, bin_, bhn])                        # [q, unit]
    B = B.reshape(4, 4, 64, 64 + EDGE).transpose(0, 1).reshape(4 * EDGE, 64 + EDGE)
    bias = bias.reshape(4, 4, 64).transpose(0, 1).reshape(4 * EDGE)
    return B, bias


def gates(P):
    """interleaved GEMM columns [M, 1024] -> (r, z, gi_n, gh_n) blocks [M, 256], unit order"""
    P = P.reshape(P.shape[0], 4, 4, 64)
    return [P[:, :, q].reshape(P.shape[0], EDGE) for q in range(4)]


def edge_gru(A, h, B, bias):
    """One edge-GRU step as the engine runs it: pre-activations A @ B^T + bias of the interleaved operand (A = [x | m h],
    [M, 320]), h' = (1 - z) n + z h with n = tanh(gi_n + r gh_n); `h` [M, 256] is the previous state the z h term reads.
    Returns h' and the scale of its error bound from the four pre-activation scales S_r, S_z, S_in, S_hn of each unit:
      |dh'| <= c (S_z / 2 + S_in + S_hn + |gh_n| S_r / 4)
    since sigmoid' <= 1/4, tanh' <= 1, r <= 1 and |n - h| <= 2 (plus an absolute allowance for the fp32 gate math)."""
    pr, pz, pin, phn = gates(A @ B.T + bias)
    sr, sz, sin, shn = gates(A.abs() @ B.abs().T + bias.abs())
    r, z = torch.sigmoid(pr), torch.sigmoid(pz)
    n = torch.tanh(pin + r * phn)
    return (1 - z) * n + z * h, 0.5 * sz + sin + shn + 0.25 * phn.abs() * sr


def edge_rows(he, masks, group, pitch, off):
    """[M, 256] previous states m * h of the edge-GRU rows: GEMM row r reads state row (r / group) * pitch + off +
    r % group of `he` [E * pitch, 256] times masks[r / group] (fp32 product, as the engine)."""
    E = masks.numel()
    rows = (torch.arange(E, device=he.device)[:, None] * pitch + off + torch.arange(group, device=he.device)).reshape(-1)
    return he[rows] * masks.reshape(E).repeat_interleave(group)[:, None]


class DsrnnStages(object):
    def __init__(self, sd, H, W, device="cpu"):
        d = device
        self.H, self.W, self.dev = H, W, d
        g = lambda k: _w(sd, k, d)
        self.edge = {}
        for side in ("spatial", "temporal"):
            p = "base.humanhumanEdgeRNN_%s." % side
            B, bias = interleave_gru(g(p + "gru.weight_ih_l0"), g(p + "gru.weight_hh_l0"), g(p + "gru.bias_ih_l0"),
                                     g(p + "gru.bias_hh_l0"))
            self.edge[side] = (g(p + "encoder_linear.weight"), g(p + "encoder_linear.bias"), B, bias)
        self.Wt, self.bt = g("base.attn.temporal_edge_layer.0.weight"), g("base.attn.temporal_edge_layer.0.bias")
        self.Ws, self.bs = g("base.attn.spatial_edge_layer.0.weight"), g("base.attn.spatial_edge_layer.0.bias")
        r = "base.humanNodeRNN."
        we, wr = g(r + "encoder_linear.weight"), g("base.robot_linear.weight")
        self.Wrob, self.brob = we @ wr, we @ g("base.robot_linear.bias") + g(r + "encoder_linear.bias")
        self.Wa, self.ba = g(r + "edge_attention_embed.weight"), g(r + "edge_attention_embed.bias")
        self.Wih, self.bih = g(r + "gru.weight_ih_l0"), g(r + "gru.bias_ih_l0")
        self.Whh, self.bhh = g(r + "gru.weight_hh_l0"), g(r + "gru.bias_hh_l0")
        wo, bo = g(r + "output_linear.weight"), g(r + "output_linear.bias")
        wac = torch.cat([g("base.actor.0.weight"), g("base.critic.0.weight")])
        bac = torch.cat([g("base.actor.0.bias"), g("base.critic.0.bias")])
        self.Woac, self.boac = wac @ wo, wac @ bo + bac
        self.Wa2, self.ba2 = g("base.actor.2.weight"), g("base.actor.2.bias")
        self.Wc2, self.bc2 = g("base.critic.2.weight"), g("base.critic.2.bias")
        self.wcl, self.bcl = g("base.critic_linear.weight"), g("base.critic_linear.bias")
        self.Wm, self.bm = g("dist.fc_mean.weight"), g("dist.fc_mean.bias")

    lin = staticmethod(StagedRef.lin)

    # ---- stages ------------------------------------------------------------------------------------------------
    def edge_emb(self, side, x):
        """columns 0..63 of an edge GRU's A operand: ReLU(encoder_linear x), x [M, W] (spatial) or [N, 2] (temporal)"""
        We, be = self.edge[side][:2]
        y, s = self.lin(x, We, be)
        return y.clamp_min(0), s

    def edge_gru(self, side, A, h):
        B, bias = self.edge[side][2:]
        return edge_gru(A, h, B, bias)

    def te(self, ht):
        return self.lin(ht, self.Wt, self.bt)

    def u(self, te):
        return te @ self.Ws, te.abs() @ self.Ws.abs()

    def edge_attention(self, hs, u, te):
        """soft-max over the H spatial states hs [N, H, 256] of (u . s_j + b_s . te) * H / 8, weighted sum of s_j (no
        mask).  Returns wv [N, 256] and the largest |s_j| of the environment [N]."""
        sc = ((hs @ u[:, :, None])[..., 0] + (te @ self.bs)[:, None]) * (self.H / 8.0)
        p = torch.softmax(sc, -1)
        return (p[:, None, :] @ hs)[:, 0], hs.abs().amax(dim=(1, 2))

    def enc(self, robot):
        """columns 0..63 of the node GRU's input: ReLU(encoder_linear(robot_linear robot_node))"""
        y, s = self.lin(robot, self.Wrob, self.brob)
        return y.clamp_min(0), s

    def emb(self, hw):
        """columns 64..127 of the node GRU's input: ReLU(edge_attention_embed [h_t' | wv])"""
        y, s = self.lin(hw, self.Wa, self.ba)
        return y.clamp_min(0), s

    def gi(self, t1):
        return self.lin(t1, self.Wih, self.bih)

    def gh(self, h0):
        return self.lin(h0, self.Whh, self.bhh)

    gru = staticmethod(StagedRef.gru)

    def ac1(self, h1):
        y, s = self.lin(h1, self.Woac, self.boac)
        return torch.tanh(y), s

    def a2(self, a1):
        y, s = self.lin(a1, self.Wa2, self.ba2)
        return torch.tanh(y), s

    def c2(self, c1):
        y, s = self.lin(c1, self.Wc2, self.bc2)
        return torch.tanh(y), s

    def value(self, c2):
        return self.lin(c2, self.wcl, self.bcl)

    def mean(self, a2):
        return self.lin(a2, self.Wm, self.bm)

    # ---- the whole forward on its own values ---------------------------------------------------------------------
    def chain(self, obs, h, he, masks):
        """obs as DsrnnRef; h [N, 1, 128]; he [N, H + 1, 256] or None (zero state); masks [N, 1]"""
        f = lambda t: t.to(self.dev, F64)
        N, H = obs["spatial_edges"].shape[:2]
        m = f(masks).reshape(N)
        he = torch.zeros(N * (H + 1), EDGE, dtype=F64, device=self.dev) if he is None else f(he).reshape(-1, EDGE)
        o = {}
        xt = self.edge_emb("temporal", f(obs["temporal_edges"]).reshape(N, 2))[0]
        ht_in = edge_rows(he, m, 1, H + 1, 0)
        o["At"] = torch.cat([xt, ht_in], 1)
        o["ht"] = self.edge_gru("temporal", o["At"], ht_in)[0]
        xs = self.edge_emb("spatial", f(obs["spatial_edges"]).reshape(N * H, -1))[0]
        hs_in = edge_rows(he, m, H, H + 1, 1)
        o["As"] = torch.cat([xs, hs_in], 1)
        o["hs"] = self.edge_gru("spatial", o["As"], hs_in)[0].reshape(N, H, EDGE)
        o["te"] = self.te(o["ht"])[0]
        o["u"] = self.u(o["te"])[0]
        o["wv"] = self.edge_attention(o["hs"], o["u"], o["te"])[0]
        o["HW"] = torch.cat([o["ht"], o["wv"]], 1)
        o["T1"] = torch.cat([self.enc(f(obs["robot_node"]).reshape(N, 7))[0], self.emb(o["HW"])[0]], 1)
        o["h0"] = f(h).reshape(N, 128) * m[:, None]
        o["gi"] = self.gi(o["T1"])[0]
        o["gh"] = self.gh(o["h0"])[0]
        o["h1"] = self.gru(o["gi"], o["gh"], o["h0"])[0]
        o["Ac1"] = self.ac1(o["h1"])[0]
        o["a2"] = self.a2(o["Ac1"][:, :256])[0]
        o["c2"] = self.c2(o["Ac1"][:, 256:])[0]
        o["value"] = self.value(o["c2"])[0]
        o["mean"] = self.mean(o["a2"])[0]
        o["he1"] = torch.cat([o["ht"][:, None], o["hs"]], 1)
        return o


# ---- read-back of the CUDA engine's workspace (GPU only) -------------------------------------------------------------
class _HookLib(object):
    """The engine library with cn_internal_dsrnn_buffer in cn_internal_policy_buffer's place (the two hooks have the
    same signature and kind codes), so policy_stages' read-back helpers serve the DS-RNN handle unchanged."""

    def __init__(self, lib):
        self._lib = lib
        self.cn_internal_policy_buffer = getattr(lib, HOOK)
        self._stage_hook_declared = False        # policy_stages._declare sets the hook's ctypes prototype once

    def __getattr__(self, name):
        return getattr(self._lib, name)


class _HookView(object):
    """A policy.CudaDsrnn handle as policy_stages.buffer_info / read_buffer see it"""

    def __init__(self, eng):
        self._h, self.device, self.lib = eng._h, eng.device, _HookLib(eng.lib)


def buffer_info(eng, name):
    """(ptr, ptr_lo, rows, cols, ld, kind) of a workspace buffer of the DS-RNN handle `eng` (policy.CudaDsrnn);
    raises with the library's message"""
    return policy_stages.buffer_info(_HookView(eng), name)


def read(eng, name, device="cuda"):
    """a workspace buffer of the DS-RNN handle `eng` after the stream is idle, as a policy_stages.Buf"""
    return policy_stages.read_buffer(_HookView(eng), name, device=device)
