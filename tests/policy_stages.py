"""Stage-local fp64 reference of the rollout policy forward (cn_policy_act), in plain torch.

Every stage is a function of its own inputs, so a test can feed it the CUDA engine's input to that stage (read back
through the internal hook cn_internal_policy_buffer, see `read_buffer`) and compare the engine's output of that stage
alone.  Chained on its own values (`StagedRef.chain`) it is the whole forward, which pins it against
oracle/policy_ref.py.  It uses the engine's layout and folds:

  * per-human stages run on the compacted rows: row_start[e] = sum_{e' < e} n_e', row r belongs to environment
    row_env[r] and is its human j = r - row_start[e]; n_e = detected_human_num clamped to [1, H] (the reference
    environment reports at least one human, crowd_sim_pred.py maps 0 to 1);
  * q/k/v_linear o in_proj -> Wqkv, out_proj o spatial_linear -> Wos, [actor.0; critic.0] o output_linear -> Woac,
    folded here in fp64 from the unfolded state dict;
  * the robot-human score te . (W_s s + b_s) = u . s + b_s . te with u = W_s^T te.

Linear stages also return |X| @ |W|^T + |b|, the scale of a componentwise error bound.
"""
import ctypes as C

import torch

F64 = torch.float64


def _w(sd, key, dev):
    return sd[key].detach().to(dev, F64)


class StagedRef(object):
    def __init__(self, sd, H, device="cpu"):
        d = device
        self.H, self.dev = H, d
        g = lambda k: _w(sd, k, d)
        p = "base.spatial_attn."
        self.W1, self.b1 = g(p + "embedding_layer.0.weight"), g(p + "embedding_layer.0.bias")
        self.W2, self.b2 = g(p + "embedding_layer.2.weight"), g(p + "embedding_layer.2.bias")
        win, bin_ = g(p + "multihead_attn.in_proj_weight"), g(p + "multihead_attn.in_proj_bias")
        ws, bs = [], []
        for i, s in enumerate("qkv"):
            wl, bl = g(p + s + "_linear.weight"), g(p + s + "_linear.bias")
            wi, bi = win[512 * i:512 * (i + 1)], bin_[512 * i:512 * (i + 1)]
            ws.append(wi @ wl)
            bs.append(wi @ bl + bi)
        self.Wqkv, self.bqkv = torch.cat(ws), torch.cat(bs)
        wout, bout = g(p + "multihead_attn.out_proj.weight"), g(p + "multihead_attn.out_proj.bias")
        wsl, bsl = g("base.spatial_linear.0.weight"), g("base.spatial_linear.0.bias")
        self.Wos, self.bos = wsl @ wout, wsl @ bout + bsl
        self.Wr, self.br = g("base.robot_linear.0.weight"), g("base.robot_linear.0.bias")
        self.Wt, self.bt = g("base.attn.temporal_edge_layer.0.weight"), g("base.attn.temporal_edge_layer.0.bias")
        self.Ws, self.bs = g("base.attn.spatial_edge_layer.0.weight"), g("base.attn.spatial_edge_layer.0.bias")
        r = "base.humanNodeRNN."
        self.We, self.be = g(r + "encoder_linear.weight"), g(r + "encoder_linear.bias")
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

    # ---- layout ------------------------------------------------------------------------------------------------
    def layout(self, detected):
        """detected_human_num [N] or [N,1] -> (n [N] int64, row_start [N+1], row_env [Mc]).  Truncation toward zero,
        then the [1, H] clamp, as cn_row_offsets_kernel does."""
        n = detected.reshape(-1).to(self.dev, torch.float32).trunc().to(torch.int64).clamp(1, self.H)
        row_start = torch.zeros(n.numel() + 1, dtype=torch.int64, device=self.dev)
        row_start[1:] = torch.cumsum(n, 0)
        row_env = torch.repeat_interleave(torch.arange(n.numel(), device=self.dev), n)
        return n, row_start, row_env

    @staticmethod
    def human_index(row_start, row_env):
        return torch.arange(row_env.numel(), device=row_env.device) - row_start[row_env]

    # ---- stages ------------------------------------------------------------------------------------------------
    @staticmethod
    def lin(x, W, b=None):
        y = x @ W.T
        s = x.abs() @ W.abs().T
        if b is not None:
            y, s = y + b, s + b.abs()
        return y, s

    def embed1(self, spatial, row_start, row_env):
        e, j = row_env, self.human_index(row_start, row_env)
        x = spatial.to(self.dev, F64)[e, j]
        y, s = self.lin(x, self.W1, self.b1)
        return y.clamp_min(0), s

    def embed2(self, e1):
        y, s = self.lin(e1, self.W2, self.b2)
        return y.clamp_min(0), s

    def qkv(self, e2):
        return self.lin(e2, self.Wqkv, self.bqkv)

    def _pad(self, rows, n, row_start):
        """compacted rows [Mc, C] -> [N, H, C] (zeros past n_e) and the validity mask [N, H]"""
        N, H = n.numel(), self.H
        valid = torch.arange(H, device=self.dev)[None, :] < n[:, None]
        idx = (row_start[:N, None] + torch.arange(H, device=self.dev)[None, :]).clamp_max(max(rows.shape[0] - 1, 0))
        out = rows[idx] * valid[..., None]
        return out, valid

    def hh_attention(self, qkv, n, row_start, row_env):
        """Multi-head (8 x 64) soft-max attention of every row over the rows of its environment.  Returns the output
        [Mc, 512] and, per element, the largest |V| of the row's environment in that head (bound scale)."""
        pad, valid = self._pad(qkv, n, row_start)
        N, H = n.numel(), self.H
        q = pad[..., :512].reshape(N, H, 8, 64).transpose(1, 2) * 0.125
        k = pad[..., 512:1024].reshape(N, H, 8, 64).transpose(1, 2)
        v = pad[..., 1024:].reshape(N, H, 8, 64).transpose(1, 2)                 # [N, 8, H, 64]
        sc = q @ k.transpose(-1, -2)
        sc = sc.masked_fill(~valid[:, None, None, :], float("-inf"))
        o = torch.softmax(sc, -1) @ v                                            # [N, 8, H, 64]
        vmax = v.abs().amax(dim=(2, 3))                                          # [N, 8]
        j = self.human_index(row_start, row_env)
        ao = o.transpose(1, 2).reshape(N, H, 512)[row_env, j]
        vm = vmax[row_env].repeat_interleave(64, dim=1)
        return ao, vm

    def outproj(self, ao):
        y, s = self.lin(ao, self.Wos, self.bos)
        return y.clamp_min(0), s

    @staticmethod
    def robot_input(robot_node, temporal_edges):
        N = robot_node.shape[0]
        return torch.cat([temporal_edges.reshape(N, 2), robot_node.reshape(N, 7)], -1)

    def robot(self, xr):
        y, s = self.lin(xr.to(self.dev, F64), self.Wr, self.br)
        return y.clamp_min(0), s

    def enc_te(self, rs):
        """[enc | te] = [relu(encoder_linear rs) | temporal_edge_layer rs]"""
        y, s = self.lin(rs, torch.cat([self.We, self.Wt]), torch.cat([self.be, self.bt]))
        y = torch.cat([y[:, :64].clamp_min(0), y[:, 64:]], 1)
        return y, s

    def u(self, te):
        return te @ self.Ws, te.abs() @ self.Ws.abs()

    def hr_attention(self, sout, u, te, n, row_start):
        """Robot-human attention: soft-max over the n_e valid humans of (u . s_j + b_s . te) * H / 8, weighted sum
        of s_j.  Returns wv [N, 256], the weights [N, H] (0 past n_e) and the largest |s_j| of the environment."""
        pad, valid = self._pad(sout, n, row_start)                               # [N, H, 256]
        sc = ((pad @ u[:, :, None])[..., 0] + (te @ self.bs)[:, None]) * (self.H / 8.0)
        sc = sc.masked_fill(~valid, float("-inf"))
        p = torch.softmax(sc, -1)
        wv = (p[:, None, :] @ pad)[:, 0]
        smax = pad.abs().amax(dim=(1, 2))
        return wv, p, smax

    def emb(self, wv):
        y, s = self.lin(wv, self.Wa, self.ba)
        return y.clamp_min(0), s

    def gi(self, x):
        return self.lin(x, self.Wih, self.bih)

    def gh(self, h0):
        return self.lin(h0, self.Whh, self.bhh)

    @staticmethod
    def gru(gi, gh, h0):
        """PyTorch GRU cell (gates r, z, n); returns h1 and the gates [r | z | n]"""
        r = torch.sigmoid(gi[:, :128] + gh[:, :128])
        z = torch.sigmoid(gi[:, 128:256] + gh[:, 128:256])
        nn_ = torch.tanh(gi[:, 256:] + r * gh[:, 256:])
        return (1 - z) * nn_ + z * h0, torch.cat([r, z, nn_], 1)

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
    def chain(self, obs, h, masks):
        f = lambda t: t.to(self.dev, F64)
        N = obs["spatial_edges"].shape[0]
        n, row_start, row_env = self.layout(obs["detected_human_num"])
        o = dict(n=n, row_start=row_start, row_env=row_env)
        o["e1"] = self.embed1(f(obs["spatial_edges"]), row_start, row_env)[0]
        o["e2"] = self.embed2(o["e1"])[0]
        o["qkv"] = self.qkv(o["e2"])[0]
        o["ao"] = self.hh_attention(o["qkv"], n, row_start, row_env)[0]
        o["sout"] = self.outproj(o["ao"])[0]
        o["rs"] = self.robot(self.robot_input(f(obs["robot_node"]), f(obs["temporal_edges"])))[0]
        o["t1"] = self.enc_te(o["rs"])[0]                                        # [enc | te]
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


def nearest_split(hi, lo):
    """True where every (hi, lo) fp16 pair (any float dtype holding fp16 values) has hi = the fp16 nearest to hi + lo,
    i.e. |lo| <= ulp(hi) / 2 -- what a round-to-nearest split hi = rn(v), lo = rn(v - hi) gives.  (hi == rn(hi + lo)
    itself can fail at a tie: lo may round up to exactly half an ulp.)"""
    h = hi.double().abs().clamp_min(2.0 ** -14)
    half_ulp = torch.ldexp(torch.ones_like(h), torch.frexp(h).exponent - 12)   # exact; subnormals as exponent -14
    return bool((lo.double().abs() <= half_ulp).all())


# ---- read-back of the CUDA engine's workspace (GPU only) -------------------------------------------------------------
class Buf(object):
    """One workspace buffer: `val` (float64: fp32 value, or hi + lo of a split pair, exactly), `hi` / `lo` (float32
    copies of the fp16 pieces of a split pair, else None) and `raw` (the fp32 / int32 data)."""

    def __init__(self, val, hi=None, lo=None, raw=None):
        self.val, self.hi, self.lo, self.raw = val, hi, lo, raw

    @property
    def split(self):
        return self.hi is not None


def _declare(lib):
    if getattr(lib, "_stage_hook_declared", False):
        return
    lib.cn_internal_policy_buffer.restype = C.c_int
    lib.cn_internal_policy_buffer.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                              C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                              C.POINTER(C.c_int)]
    lib._stage_hook_declared = True


def buffer_info(pol, name):
    """(ptr, ptr_lo, rows, cols, ld, kind) of a named workspace buffer; raises with the library's message"""
    from crowdnav_prediction_attngraph_b200 import _capi
    lib = pol.lib
    _declare(lib)
    p, pl = C.c_void_p(), C.c_void_p()
    rows, cols, ld, kind = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    _capi.check(lib, lib.cn_internal_policy_buffer(pol._h, name.encode(), C.byref(p), C.byref(pl), C.byref(rows),
                                                   C.byref(cols), C.byref(ld), C.byref(kind)),
                "cn_internal_policy_buffer(%s)" % name)
    return p.value, pl.value, rows.value, cols.value, ld.value, kind.value


def _fetch(pol, ptr, nbytes, dtype, shape):
    from crowdnav_prediction_attngraph_b200 import _capi
    out = torch.empty(shape, dtype=dtype)
    dev = pol.device.index or 0
    _capi.check(pol.lib, pol.lib.cn_fetch_sync(C.c_void_p(out.data_ptr()), C.c_void_p(ptr), nbytes, dev,
                                               _capi.raw_stream(dev)), "cn_fetch_sync")
    return out


def read_buffer(pol, name, rows=None, device="cuda"):
    """Copy a workspace buffer back after the stream is idle (only the first `rows` rows, e.g. Mc of [M, C])."""
    ptr, plo, r, c, ld, kind = buffer_info(pol, name)
    r = r if rows is None else min(rows, r)
    if kind == 2:
        v = _fetch(pol, ptr, r * 4, torch.int32, (r,)).to(device)
        return Buf(v.long(), raw=v)
    if kind == 0:
        v = _fetch(pol, ptr, r * ld * 4, torch.float32, (r, ld))[:, :c].to(device)
        return Buf(v.double(), raw=v)
    hi = _fetch(pol, ptr, r * ld * 2, torch.float16, (r, ld))[:, :c].to(device).float()
    lo = _fetch(pol, plo, r * ld * 2, torch.float16, (r, ld))[:, :c].to(device).float()
    return Buf(hi.double() + lo.double(), hi=hi, lo=lo)
