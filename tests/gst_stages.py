"""Stage-local fp64 reference of the GST predictor step (cn_gst_step), in plain torch and numpy.

Every stage is a function of its own inputs, so a test can feed it the CUDA engine's input to that stage (read back
through the internal hook cn_internal_gst_buffer, see `read_buffer`) and compare the engine's output of that stage
alone.  Chained on its own values (`GstStages.chain`) it is the whole predictor, which pins it against
oracle/gst_ref.py.  It uses the engine's compact layout (csrc/cn_gst.cu, "Compact rows"):

  * observation rows r = (e * 5 + t) * H + n with row mask m[t-1] * m[4] (frame 0: m[0]) are live; the live rows are
    compacted in row order, group g = e * 5 + t owns compact rows [gstart[g], gstart[g + 1]), cidx[r] is the compact
    row of r (-1 when masked), crow[c] its source row;
  * decode rows are the humans with fp = m[3] * m[4], compacted in env order: env e owns [estart[e], estart[e + 1]),
    drow[d] = e * H + n;
  * in the attention the H - n masked neighbours of a group share the key b_k, so they enter the soft-max denominator
    as ONE term (H - n) * exp(q . b_k - max) (mha.py:236-242 takes the soft-max over all H keys, then masks and
    renormalises with + 1e-10).

`compaction` restates the integer / float32 bookkeeping in numpy, operation for operation, so the engine's maps can be
compared bit for bit.  Linear stages also return |X| @ |W|^T + |b|, the scale of a componentwise error bound;
LayerNorm returns its own scale (see `layer_norm`), the attention the largest |V| of the group and head.
"""
import ctypes as C

import numpy as np
import torch

F64 = torch.float64
T = 5
INVALID = np.float32(-999.0)
PRE = "gumbel_social_transformer."
ENC = PRE + "node_encoder_layers.0."
LN_EPS = 1e-5


# ---- compaction (numpy, bit for bit) -------------------------------------------------------------------------------
def frames_from_ring(ring_pos, ring_mask, newest, robot, sp2, vis):
    """The five frames one cn_gst_step sees: frames 0..3 from the ring slots (newest + 1 + t) % 5 (ring_pos [5,N,H,2],
    ring_mask [5,N,H] as they were BEFORE the step; `newest` = the slot the step writes), frame 4 = robot + sp2 (float32)
    and vis.  Returns pos [5,N,H,2] float32, m [5,N,H] float32."""
    cur = (robot[:, None, :2].astype(np.float32) + sp2.astype(np.float32)).astype(np.float32)
    pos = [ring_pos[(newest + 1 + t) % T] for t in range(T - 1)] + [cur]
    m = [ring_mask[(newest + 1 + t) % T].astype(np.float32) for t in range(T - 1)] + [(vis != 0).astype(np.float32)]
    return np.stack(pos).astype(np.float32), np.stack(m).astype(np.float32)


class Ring(object):
    """VecPretextNormalize's traj / mask buffers as the engine keeps them: a 5-slot ring, reset to -999 / 0."""

    def __init__(self, N, H):
        self.pos = np.full((T, N, H, 2), INVALID, np.float32)
        self.mask = np.zeros((T, N, H), np.uint8)
        self.newest = T - 1

    def step(self, robot, sp2, vis):
        """advance by one observation; returns the five frames (pos, m) the step sees"""
        self.newest = (self.newest + 1) % T
        pos, m = frames_from_ring(self.pos, self.mask, self.newest, robot, sp2, vis)
        self.pos[self.newest] = pos[T - 1]
        self.mask[self.newest] = vis != 0
        return pos, m


def compaction(pos, m):
    """gtc_prep / gtc_scan / gtc_index on frames pos [5,N,H,2], m [5,N,H] (float32).  Returns a dict of the engine's
    buffers: rowm [R], inp [R,2], gcount, gstart, ecount, estart, counts (2), cidx, crow, drow, fp [N*H], pos_last."""
    _, N, H = m.shape
    one = np.float32(1.0)
    mrel = np.empty_like(m)
    mrel[0] = m[0]
    mrel[1:] = m[:-1] * m[-1:]                       # interface.forward:77-78 (sic): m[t-1] * m[4]
    d = np.zeros_like(pos)
    d[1:] = pos[1:] - pos[:-1]
    mr = mrel[..., None]
    inp = INVALID * (one - mr) + d * mr               # exact: mr is 0 or 1
    rowm = mrel.transpose(1, 0, 2).reshape(-1)        # [N,5,H] row order
    inp = inp.transpose(1, 0, 2, 3).reshape(-1, 2)
    gcount = mrel.transpose(1, 0, 2).sum(-1).reshape(-1).astype(np.int64)
    fp = mrel[T - 1].reshape(-1)
    ecount = mrel[T - 1].sum(-1).astype(np.int64)
    gstart = np.concatenate([[0], np.cumsum(gcount)])
    estart = np.concatenate([[0], np.cumsum(ecount)])
    live = rowm != 0
    cidx = np.where(live, np.cumsum(live) - 1, -1)
    return dict(rowm=rowm, inp=inp, gcount=gcount, gstart=gstart, ecount=ecount, estart=estart,
                counts=np.array([gstart[-1], estart[-1]]), cidx=cidx, crow=np.flatnonzero(live), drow=np.flatnonzero(fp),
                fp=fp, pos_last=pos[T - 1].reshape(-1, 2), mrel=mrel)


KIND_NONE, KIND_ALL, KIND_APPROACH, KIND_DUP, KIND_AT_ROBOT = 3, 5, 1, 2, 4     # env e has kind e % 8


def random_history(N, H, steps, vis_p, seed):
    """Seeded observations of `steps` wrapper steps: lists of robot [N,7], sp2 [N,H,2] float32 and vis [N,H] uint8.
    Humans random-walk ~0.25 m per frame with occasional jumps of several metres (an episode reset does not clear the
    wrapper's buffers) and are visible independently per frame with probability vis_p, except by env kind (e % 8):
    KIND_NONE nobody visible, KIND_ALL everybody visible, KIND_APPROACH humans 2, 4, 6 walk straight at a still robot at
    0.25 m per frame (their later predicted points come within the collision distance first), KIND_DUP human 1 stands
    exactly where human 0 stands, KIND_AT_ROBOT human 3 (or the last) stands at the robot (distance key 0)."""
    rng = np.random.RandomState(seed)
    kind = np.arange(N) % 8
    rob = rng.uniform(-4, 4, (N, 2))
    hum = rob[:, None] + rng.uniform(-6, 6, (N, H, 2))
    app = [n for n in (2, 4, 6) if n < H]
    ang = rng.uniform(0, 2 * np.pi, (N, len(app)))
    d0 = rng.uniform(1.4, 3.4, (N, len(app)))
    out = []
    for s in range(steps):
        still = kind == KIND_APPROACH
        rob = rob + np.where(still[:, None], 0.0, rng.normal(0, 0.1, (N, 2)))
        hum = hum + rng.normal(0, 0.25 / np.sqrt(2), (N, H, 2))
        jump = rng.rand(N, H) < 0.03
        hum = hum + jump[..., None] * rng.uniform(-8, 8, (N, H, 2))
        vis = rng.rand(N, H) < vis_p
        vis[kind == KIND_NONE] = False
        vis[kind == KIND_ALL] = True
        sp2 = (hum - rob[:, None]).astype(np.float32)
        for i, n in enumerate(app):
            d = d0[still, i] - 0.25 * s
            sp2[still, n] = np.stack([d * np.cos(ang[still, i]), d * np.sin(ang[still, i])], -1)
            vis[still, n] = True
        if H > 1:
            sp2[kind == KIND_DUP, 1] = sp2[kind == KIND_DUP, 0]
        sp2[kind == KIND_AT_ROBOT, min(3, H - 1)] = 0.0
        robot = np.concatenate([rob, rng.normal(0, 1, (N, 5))], 1).astype(np.float32)
        out.append((robot, sp2, vis.astype(np.uint8)))
    return out


def split16(v):
    """the engine's fp32 -> (hi, lo) fp16 split (gt_split_store), as float32 tensors"""
    v = v.float().clamp(-65504.0, 65504.0)
    hi = v.half().float()
    return hi, (v - hi).half().float()


# ---- arithmetic stages (fp64) ---------------------------------------------------------------------------------------
class GstStages(object):
    def __init__(self, params, H, device="cpu"):
        g = lambda k: torch.as_tensor(np.asarray(params[k]), dtype=F64, device=device)
        self.H, self.dev = H, device
        self.We, self.be = g(PRE + "node_embedding.weight"), g(PRE + "node_embedding.bias")
        self.g0, self.b0 = g(ENC + "norm_node.weight"), g(ENC + "norm_node.bias")
        self.Win, self.bin = g(ENC + "self_attn.in_proj_weight"), g(ENC + "self_attn.in_proj_bias")
        self.Wout, self.bout = g(ENC + "self_attn.out_proj.weight"), g(ENC + "self_attn.out_proj.bias")
        self.g1, self.b1n = g(ENC + "norm1_node.weight"), g(ENC + "norm1_node.bias")
        self.W1, self.b1 = g(ENC + "linear1.weight"), g(ENC + "linear1.bias")
        self.W2, self.b2 = g(ENC + "linear2.weight"), g(ENC + "linear2.bias")
        self.Wih, self.bih = g("lstm.weight_ih_l0"), g("lstm.bias_ih_l0")
        self.Whh, self.bhh = g("lstm.weight_hh_l0"), g("lstm.bias_hh_l0")
        self.Wp, self.bp = g("hidden2pos.weight")[:2], g("hidden2pos.bias")[:2]    # the mean only (sampling=False)

    def t(self, x):
        return torch.as_tensor(x).to(self.dev, F64)

    @staticmethod
    def lin(x, W, b=None):
        y, s = x @ W.T, x.abs() @ W.abs().T
        if b is not None:
            y, s = y + b, s + b.abs()
        return y, s

    @staticmethod
    def layer_norm(pre, pre_scale, gamma, beta):
        """LayerNorm (eps 1e-5) of rows `pre` [M,64].  Scale of the bound, per element:
        |gamma| * (max_j pre_scale_j / sigma + |z|) + |beta| -- an error of u * pre_scale in the input (or in the mean)
        moves z by u * pre_scale / sigma, the normalisation itself by u * |z|."""
        mean = pre.mean(-1, keepdim=True)
        sigma = ((pre - mean) ** 2).mean(-1, keepdim=True).add(LN_EPS).sqrt()
        z = (pre - mean) / sigma
        kappa = pre_scale.amax(-1, keepdim=True) / sigma
        return z * gamma + beta, gamma.abs() * (kappa + z.abs()) + beta.abs()

    def embed(self, inp):
        """node embedding + norm_node of the compact rows' input [M,2] -> X0 [M,64] (gtc_embed_kernel)"""
        pre, s = self.lin(self.t(inp), self.We, self.be)
        return self.layer_norm(pre, s, self.g0, self.b0)

    def qkv(self, x):
        return self.lin(x, self.Win, self.bin)

    def attention(self, qkv, start, chunk_bytes=1 << 28):
        """Per group g (compact rows [start[g], start[g+1])), 8 heads of width 8: soft-max over the group's live rows
        and the H - n masked neighbours with the common key b_k, masked and renormalised with + 1e-10.  Returns the
        output [M,64] and, per element, the largest |V| over the group's live rows in that head."""
        H, dev = self.H, qkv.device
        start = torch.as_tensor(np.asarray(start), dtype=torch.int64, device=dev)
        M = qkv.shape[0]
        out = torch.zeros(M, 64, dtype=F64, device=dev)
        vmax = torch.zeros(M, 64, dtype=F64, device=dev)
        ng = start[1:] - start[:-1]
        groups = torch.nonzero(ng > 0)[:, 0]
        if groups.numel() == 0:
            return out, vmax
        L = int(ng.max())
        bk = self.bin[64:128].reshape(8, 8)
        B = max(1, chunk_bytes // (64 * 8 * L * L))
        ar = torch.arange(L, device=dev)
        for i in range(0, groups.numel(), B):
            gs = groups[i:i + B]
            n = ng[gs]
            valid = ar[None, :] < n[:, None]                                      # [b, L]
            idx = (start[gs][:, None] + ar[None, :]).clamp_max(M - 1)
            x = qkv[idx].reshape(len(gs), L, 3, 8, 8)
            q = x[:, :, 0] * 8.0 ** -0.5                                          # [b, L, head, 8]
            k, v = x[:, :, 1], x[:, :, 2]
            s = torch.einsum("blhd,bmhd->bhlm", q, k)
            sm = torch.einsum("blhd,hd->bhl", q, bk)                              # score of every masked key
            nmask = (H - n).to(F64)[:, None, None]
            s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
            mx = s.amax(-1)
            mx = torch.where(nmask > 0, torch.maximum(mx, sm), mx)
            e = torch.exp(s - mx[..., None])
            den = e.sum(-1) + nmask * torch.exp(sm - mx)                          # (H - n) * exp(q . b_k - max)
            p = e / den[..., None]
            o = torch.einsum("bhlm,bmhd->blhd", p, v) / (p.sum(-1).permute(0, 2, 1)[..., None] + 1e-10)
            vm = (v.abs() * valid[:, :, None, None]).amax(dim=(1, 3))              # [b, head]
            rows = idx[valid]
            out[rows] = o.reshape(len(gs), L, 64)[valid]
            vmax[rows] = vm[:, None, :, None].expand(-1, L, 8, 8).reshape(len(gs), L, 64)[valid]
        return out, vmax

    def outproj(self, a):
        return self.lin(a, self.Wout, self.bout)

    def norm1(self, x1):
        """norm1_node of the residual X1 = X0 + O (the engine's fp32 X1 is the exact input)"""
        return self.layer_norm(x1, x1.abs(), self.g1, self.b1n)

    def ffn1(self, y):
        z, s = self.lin(y, self.W1, self.b1)
        return z.clamp_min(0), s

    def ffn2(self, f):
        return self.lin(f, self.W2, self.b2)

    def gx(self, xs):
        return self.lin(xs, self.Wih, self.bih)

    def gh(self, h):
        return self.lin(h, self.Whh, self.bhh)

    def lstm_gx(self, GX, cidx, drow, t):
        """gate input of the decode rows in observed frame t: GX of the row's compact observation row, or b_ih when
        that frame of the human is masked (its encoder input is 0)"""
        drow = torch.as_tensor(np.asarray(drow), dtype=torch.int64, device=GX.device)
        cidx = torch.as_tensor(np.asarray(cidx), dtype=torch.int64, device=GX.device)
        e, n = drow // self.H, drow % self.H
        c = cidx[(e * T + t) * self.H + n]
        out = self.bih.to(GX.device).expand(drow.numel(), 256).clone()
        live = c >= 0
        out[live] = GX[c[live]]
        return out

    @staticmethod
    def cell(gx, gh, c_prev):
        """LSTM cell, gates (i, f, g, o); returns h, c"""
        a = gx + gh
        i, f, gg, o = torch.sigmoid(a[:, :64]), torch.sigmoid(a[:, 64:128]), torch.tanh(a[:, 128:192]), torch.sigmoid(a[:, 192:])
        c = f * c_prev + i * gg
        return o * torch.tanh(c), c

    def h2p(self, h):
        return self.lin(h, self.Wp, self.bp)

    def encoder(self, X0, start):
        """one encoder pass on its own values: X0 [M,64] -> dict of every stage's output"""
        o = dict(X0=X0)
        o["QKV"] = self.qkv(X0)[0]
        o["A"] = self.attention(o["QKV"], start)[0]
        o["O"] = self.outproj(o["A"])[0]
        o["X1"] = X0 + o["O"]
        o["Y"] = self.norm1(o["X1"])[0]
        o["F"] = self.ffn1(o["Y"])[0]
        o["O2"] = self.ffn2(o["F"])[0]
        o["XS"] = o["X1"] + o["O2"]
        o["GX"] = self.gx(o["XS"])[0]
        return o

    def chain(self, comp):
        """the whole predictor on its own values from the compaction `comp`; returns pred [Rd_live, 5, 2] (world
        positions of the decode rows drow) and the last stage values"""
        X0 = self.embed(comp["inp"][comp["crow"]])[0]
        GX = self.encoder(X0, comp["gstart"])["GX"]
        D = len(comp["drow"])
        h = torch.zeros(D, 64, dtype=F64, device=self.dev)
        c = torch.zeros_like(h)
        for t in range(T):
            gh = self.bhh.expand(D, 256) if t == 0 else self.gh(h)[0]
            h, c = self.cell(self.lstm_gx(GX, comp["cidx"], comp["drow"], t), gh, c)
        pos_last = self.t(comp["pos_last"][comp["drow"]])
        mu = torch.zeros(D, 2, dtype=F64, device=self.dev)
        pred = []
        xin = None
        for tt in range(T):
            if tt > 0:
                enc = self.encoder(self.embed(xin)[0], comp["estart"])
                h, c = self.cell(enc["GX"], self.gh(h)[0], c)
            xin = self.h2p(h)[0]
            mu = mu + xin
            pred.append(mu + pos_last)
        return torch.stack(pred, 1)


# ---- the wrapper's tail (gt_final_kernel) ---------------------------------------------------------------------------
def final_rows(robot, sp2, fp, pred, P):
    """Unsorted spatial_edges rows [N,H,2(P+1)]: the current relative position, then pred - robot for k < P where fp,
    else the current relative position again.  robot [N,>=2], sp2 [N,H,2], fp [N,H], pred [N,H,5,2] (numpy; the
    arithmetic is the dtype's)."""
    N, H = fp.shape
    rel = pred[:, :, :P] - robot[:, None, None, :2]
    cur = np.broadcast_to(sp2[:, :, None, :], rel.shape)
    body = np.where((fp != 0)[:, :, None, None], rel, cur).reshape(N, H, 2 * P)
    return np.concatenate([sp2, body], -1)


def penalty(robot, fp, pred, P, thr, collision_penalty=-20.0):
    """future-collision penalty: min over predicted points k < P of humans with fp = 1 that lie closer than thr of
    collision_penalty / 2^(k + 2), else 0.  Distances in float64 of the operands' (pred - robot) differences.
    Returns (penalty [N] float64, distance [N,H,P] float64, counted [N,H,P] bool)."""
    rel = (pred[:, :, :P] - robot[:, None, None, :2]).astype(np.float64)
    dist = np.sqrt((rel ** 2).sum(-1))
    counted = (fp != 0)[:, :, None] & np.ones_like(dist, dtype=bool)
    coll = (dist < thr) & counted
    coef = collision_penalty / 2.0 ** np.arange(2, P + 2)
    pen = np.where(coll, coef[None, None, :], 0.0).reshape(len(fp), -1).min(1)
    return pen, dist, counted


def sort_keys(sp2):
    """float32 distance keys of the current relative positions (x*x + y*y without contraction)"""
    s = sp2.astype(np.float32)
    return np.sqrt(s[..., 0] * s[..., 0] + s[..., 1] * s[..., 1])


# ---- read-back of the CUDA engine's workspace (GPU only) -------------------------------------------------------------
class Buf(object):
    """One workspace buffer: `val` (float64: fp32 value, or hi + lo of a split pair, exactly), `hi` / `lo` (float32
    copies of the fp16 pieces of a split pair, else None) and `raw` (the fp32 / int32 / uint8 data)."""

    def __init__(self, val, hi=None, lo=None, raw=None):
        self.val, self.hi, self.lo, self.raw = val, hi, lo, raw

    @property
    def split(self):
        return self.hi is not None


def declare(lib):
    if getattr(lib, "_gst_stage_hook_declared", False):
        return
    lib.cn_internal_gst_buffer.restype = C.c_int
    lib.cn_internal_gst_buffer.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                           C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int),
                                           C.POINTER(C.c_int)]
    lib.cn_internal_gst_stop_after.restype = C.c_int
    lib.cn_internal_gst_stop_after.argtypes = [C.c_void_p, C.c_char_p]
    lib._gst_stage_hook_declared = True


def buffer_info(lib, h, name):
    """(ptr, ptr_lo, rows, cols, ld, kind) of a named workspace buffer; raises with the library's message"""
    from crowdnav_prediction_attngraph_b200 import _capi
    declare(lib)
    p, pl = C.c_void_p(), C.c_void_p()
    rows, cols, ld, kind = C.c_int(), C.c_int(), C.c_int(), C.c_int()
    _capi.check(lib, lib.cn_internal_gst_buffer(h, name.encode(), C.byref(p), C.byref(pl), C.byref(rows), C.byref(cols),
                                                C.byref(ld), C.byref(kind)), "cn_internal_gst_buffer(%s)" % name)
    return p.value, pl.value, rows.value, cols.value, ld.value, kind.value


def _fetch(lib, ptr, nbytes, dtype, shape):
    from crowdnav_prediction_attngraph_b200 import _capi
    out = torch.empty(shape, dtype=dtype)
    if nbytes:
        _capi.check(lib, lib.cn_fetch_sync(C.c_void_p(out.data_ptr()), C.c_void_p(ptr), nbytes, 0, _capi.raw_stream(0)),
                    "cn_fetch_sync")
    return out


def read_buffer(lib, h, name, rows=None, device="cuda"):
    """Copy a workspace buffer back after the stream is idle (only the first `rows` rows, e.g. the live rows)."""
    ptr, plo, r, c, ld, kind = buffer_info(lib, h, name)
    r = r if rows is None else min(int(rows), r)
    if kind == 2:
        v = _fetch(lib, ptr, r * 4, torch.int32, (r,)).to(device)
        return Buf(v.long(), raw=v)
    if kind == 3:
        v = _fetch(lib, ptr, r, torch.uint8, (r,)).to(device)
        return Buf(v.long(), raw=v)
    if kind == 0:
        v = _fetch(lib, ptr, r * ld * 4, torch.float32, (r, ld))[:, :c].to(device)
        return Buf(v.double(), raw=v)
    hi = _fetch(lib, ptr, r * ld * 2, torch.float16, (r, ld))[:, :c].to(device).float()
    lo = _fetch(lib, plo, r * ld * 2, torch.float16, (r, ld))[:, :c].to(device).float()
    return Buf(hi.double() + lo.double(), hi=hi, lo=lo)
