"""Host-side mirror of the reference policy surface over the CUDA kernels.

`Policy` keeps the entry points train.py / test.py call on rl.networks.model.Policy
(rl/networks/model.py:14-90): `act`, `get_value`, `evaluate_actions`, `state_dict` with the
reference's keys and shapes (SURVEY.md §2.3) so checkpoints interchange both ways.

  * act / get_value (rollout, infer=True)  -> ONE call into the C ABI (cn_policy_act): the fused
    sm_90a forward; no torch ops on the hot path except drawing the Gaussian noise.
  * evaluate_actions (PPO update)          -> PyTorch on device (north_star: the clipped-loss
    minibatch update stays in PyTorch), written here for [T, N] batches with done-mask GRU resets.
"""
import ctypes as C
import math
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _capi

HIDDEN = 128
NOISE_BLOCK = 32          # rollout steps of action noise drawn per generator call (CudaPolicy.act)


class _AddBias(nn.Module):
    def __init__(self, n):
        super().__init__()
        self._bias = nn.Parameter(torch.zeros(n, 1))


def _ortho(m, gain=1.0):
    nn.init.orthogonal_(m.weight.data, gain=gain)
    nn.init.constant_(m.bias.data, 0)
    return m


class _Params(nn.Module):
    """Parameter container with the reference's module tree (names drive the state_dict keys).  self_attn=False is the
    reference's use_self_attn = False (selfAttn_srnn_temp_node.py:340-345): no spatial_attn, and spatial_linear =
    Linear(input_size, 128), ReLU, Linear(128, 256), ReLU with the orthogonal sqrt(2) init."""

    def __init__(self, input_size, self_attn=True):
        super().__init__()
        g = math.sqrt(2)
        base = nn.Module()
        rnn = nn.Module()
        rnn.gru = nn.GRU(128, HIDDEN)
        for name, prm in rnn.gru.named_parameters():          # srnn_model.py:27-31
            if 'bias' in name:
                nn.init.constant_(prm, 0)
            else:
                nn.init.orthogonal_(prm)
        rnn.encoder_linear = nn.Linear(256, 64)
        rnn.edge_attention_embed = nn.Linear(256, 64)
        rnn.output_linear = nn.Linear(HIDDEN, 256)
        base.humanNodeRNN = rnn
        att = nn.Module()
        att.temporal_edge_layer = nn.ModuleList([nn.Linear(256, 64)])
        att.spatial_edge_layer = nn.ModuleList([nn.Linear(256, 64)])
        base.attn = att
        base.actor = nn.Sequential(_ortho(nn.Linear(256, 256), g), nn.Tanh(), _ortho(nn.Linear(256, 256), g), nn.Tanh())
        base.critic = nn.Sequential(_ortho(nn.Linear(256, 256), g), nn.Tanh(), _ortho(nn.Linear(256, 256), g), nn.Tanh())
        base.critic_linear = _ortho(nn.Linear(256, 1), g)
        base.robot_linear = nn.Sequential(_ortho(nn.Linear(9, 256), g), nn.ReLU())
        base.human_node_final_linear = _ortho(nn.Linear(256, 2), g)   # unused by forward (reference :338)
        if self_attn:
            sa = nn.Module()
            sa.embedding_layer = nn.Sequential(nn.Linear(input_size, 128), nn.ReLU(), nn.Linear(128, 512), nn.ReLU())
            sa.q_linear = nn.Linear(512, 512)
            sa.v_linear = nn.Linear(512, 512)
            sa.k_linear = nn.Linear(512, 512)
            sa.multihead_attn = nn.MultiheadAttention(512, 8)
            base.spatial_attn = sa
            base.spatial_linear = nn.Sequential(_ortho(nn.Linear(512, 256), g), nn.ReLU())
        else:
            base.spatial_linear = nn.Sequential(_ortho(nn.Linear(input_size, 128), g), nn.ReLU(),
                                                _ortho(nn.Linear(128, 256), g), nn.ReLU())
        self.base = base
        dist = nn.Module()
        dist.fc_mean = _ortho(nn.Linear(256, 2))
        dist.logstd = _AddBias(2)
        self.dist = dist


def make_reference_like_state_dict(input_size=12, seed=0, self_attn=True):
    """Random-init parameters with the reference's initialisers (orthogonal where it uses them); self_attn=False: the
    use_self_attn = False network."""
    gen_state = torch.random.get_rng_state()
    torch.manual_seed(seed)
    sd = {k: v.detach().clone() for k, v in _Params(input_size, self_attn).state_dict().items()}
    torch.random.set_rng_state(gen_state)
    return sd


class CudaPolicy(object):
    """Thin handle on cn_policy: upload a reference state_dict, run the rollout forward.  self_attn=False runs the
    reference's use_self_attn = False network (cn_policy_config.no_self_attn).  visible_masks=True is the reference's
    sort_humans = False: act() masks the attention with obs['visible_masks'] (cn_policy_config.visible_masks)."""

    def __init__(self, num_envs, human_num, input_size=12, device="cuda:0", gemm_mode=1, self_attn=True,
                 visible_masks=False):
        self._setup(num_envs, human_num, input_size, device)
        self.self_attn = bool(self_attn)
        self.visible_masks = bool(visible_masks)
        cfg = _capi.CnPolicyConfig(num_envs, human_num, input_size,
                                   self.device.index if self.device.index is not None else 0, gemm_mode,
                                   0 if self.self_attn else 1, 1 if self.visible_masks else 0)
        self._h = C.c_void_p()
        _capi.check(self.lib, self.lib.cn_policy_create(C.byref(cfg), C.byref(self._h)), "cn_policy_create")

    def _setup(self, num_envs, human_num, input_size, device, **extra_outputs):
        """What every engine handle holds: the library, the device (CUDA only), the sizes, the two output buffers that
        act() alternates between (value, action, log_prob, h_out, mean and `extra_outputs` {name: shape}) and the noise
        generator state."""
        self.lib = _capi.load_library()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("%s needs a CUDA device (no CPU fallback)" % type(self).__name__)
        self.N, self.H, self.Win = num_envs, human_num, input_size
        N = num_envs
        shapes = dict(value=(N, 1), action=(N, 2), log_prob=(N, 1), h_out=(N, 1, HIDDEN), mean=(N, 2), **extra_outputs)
        self._bufs = [{k: torch.zeros(*shp, device=self.device) for k, shp in shapes.items()} for _ in range(2)]
        self._flip = 0
        self._gen = None

    def _stream(self):
        return _capi.raw_stream(self.device.index or 0)

    def load_state_dict(self, sd):
        for k, v in sd.items():
            if k.startswith("base.human_node_final_linear"):
                continue      # unused by the forward (reference selfAttn_srnn_temp_node.py:338)
            arr = v.detach().to("cpu", torch.float32).contiguous().numpy()
            _capi.check(self.lib, self.lib.cn_policy_set_param(self._h, k.encode(), arr.ctypes.data, arr.size),
                        "cn_policy_set_param(%s)" % k)
        with torch.cuda.device(self.device):
            _capi.check(self.lib, self.lib.cn_policy_finalize(self._h, self._stream()), "cn_policy_finalize")

    def _outputs(self, out, keys=("value", "action", "log_prob", "h_out")):
        """The next of the two internal output buffers, with the entries of `out` (caller memory) in their place."""
        self._flip ^= 1
        b = self._bufs[self._flip]
        if out is not None:
            b = dict(b)
            for k in keys:
                if k in out:
                    assert out[k].is_cuda and out[k].is_contiguous() and out[k].dtype == torch.float32, k
                    b[k] = out[k]
        return b

    def _inputs(self, **args):
        f32, dev = torch.float32, self.device
        for k, t in args.items():
            if t.dtype is not f32 or not t.is_contiguous() or t.device != dev:
                args[k] = t.to(dev, f32).contiguous()
        return args

    def _noise(self, deterministic, noise):
        """Standard normal action noise [N, 2] for this step (None when deterministic)."""
        N = self.N
        if not deterministic and noise is None:
            # torch.normal(mean, std) == randn * std + mean.  Data-parallel replicas are seeded alike by train.py
            # (identical initial weights): give every rank its own noise stream so their actions decorrelate.
            if self._gen is None and torch.distributed.is_available() and torch.distributed.is_initialized() \
                    and torch.distributed.get_world_size() > 1:
                self._gen = torch.Generator(device=self.device)
                self._gen.manual_seed(torch.initial_seed() + 7919 * torch.distributed.get_rank())
            # one generator call serves NOISE_BLOCK steps (a torch.randn launch costs ~10 us of host time per step)
            # The block is dropped when the generator was re-seeded or used by anyone else in between, so
            # torch.manual_seed(s) followed by act() still restarts the noise sequence.
            g = self._gen if self._gen is not None else torch.cuda.default_generators[self.device.index or 0]
            nb = self.__dict__.get("_noise_block")
            if nb is None or self._noise_i >= nb.shape[0] or self._noise_state != (g.initial_seed(), g.get_offset()):
                nb = self._noise_block = torch.randn(NOISE_BLOCK, N, 2, device=self.device, generator=self._gen)
                self._noise_i = 0
                self._noise_state = (g.initial_seed(), g.get_offset())
            noise = nb[self._noise_i]
            self._noise_i += 1
        return noise

    def act(self, obs, h, masks, deterministic=False, return_mean=False, noise=None, out=None):
        """obs: dict of device tensors; h: [N,1,128]; masks: [N,1].  Returns value, action, log_prob, h_new
        (views of internal double buffers: valid until the call after next).  `out` (optional dict with
        contiguous float32 device tensors value/action/log_prob/h_out) makes the kernels write straight
        into caller memory, e.g. the rollout-storage slot (zero-copy rollout)."""
        b = self._outputs(out)
        noise = self._noise(deterministic, noise)
        args = self._inputs(robot_node=obs["robot_node"], temporal_edges=obs["temporal_edges"],
                            spatial_edges=obs["spatial_edges"], detected_human_num=obs["detected_human_num"],
                            h_in=h, masks=masks)
        vm = None
        if self.visible_masks:
            vm = obs["visible_masks"]           # one byte per slot, as the environment writes it
            if vm.dtype not in (torch.bool, torch.uint8) or not vm.is_contiguous() or vm.device != self.device:
                vm = vm.to(self.device, torch.bool).contiguous()
            args["visible_masks"] = vm
        ptrs = _capi.CnActPtrs(
            args["robot_node"].data_ptr(), args["temporal_edges"].data_ptr(), args["spatial_edges"].data_ptr(),
            args["detected_human_num"].data_ptr(), args["h_in"].data_ptr(), args["masks"].data_ptr(),
            None if deterministic else noise.data_ptr(), b["value"].data_ptr(), b["action"].data_ptr(),
            b["log_prob"].data_ptr(), b["h_out"].data_ptr(), b["mean"].data_ptr(),
            None if vm is None else vm.data_ptr())
        rc = self.lib.cn_policy_act(self._h, C.byref(ptrs), self._stream())     # restores the caller's device itself
        if rc:
            _capi.check(self.lib, rc, "cn_policy_act")
        self._keep = (args, noise)      # keep inputs alive until the kernels are enqueued behind the next call
        if return_mean:
            return b["value"], b["action"], b["log_prob"], b["h_out"], b["mean"]
        return b["value"], b["action"], b["log_prob"], b["h_out"]

    def launch_count(self):
        return int(self.lib.cn_policy_launch_count(self._h))

    def profile(self, enable=True):
        _capi.check(self.lib, self.lib.cn_policy_profile(self._h, int(enable)), "cn_policy_profile")

    def stage_ms(self):
        """{stage: ms} of the last act, under this handle's own stage names (profiling must have been enabled with
        profile(True) before it)."""
        n = self.lib.cn_policy_handle_stage_count(self._h)
        out = (C.c_float * n)()
        _capi.check(self.lib, self.lib.cn_policy_stage_ms(self._h, out, n), "cn_policy_stage_ms")
        names = [self.lib.cn_policy_handle_stage_name(self._h, i).decode() for i in range(n)]
        return {k: float(out[i]) for i, k in enumerate(names) if k}

    def close(self):
        if self._h:
            self.lib.cn_policy_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


EDGE = 256                # human_human_edge_rnn_size
DSRNN_UNUSED = ("base.humanNodeRNN.edge_embed.", "base.human_node_final_linear.", "base.spatial_linear.")


def _is_zero_view(t):
    """An expanded scalar (every stride 0): the all-zero edge state the rollout storage keeps for a policy without
    a recurrent edge state.  The kernels take it as a NULL pointer, so it is never materialised."""
    return t is None or (t.dim() > 0 and all(s == 0 for s in t.stride()))


class CudaDsrnn(CudaPolicy):
    """Thin handle on cn_dsrnn (the DS-RNN forward); noise and output buffers as CudaPolicy."""

    def __init__(self, num_envs, human_num, input_size=2, device="cuda:0"):
        self._setup(num_envs, human_num, input_size, device, edge_h_out=(num_envs, human_num + 1, EDGE))
        cfg = _capi.CnDsrnnConfig(num_envs, human_num, input_size, self.device.index if self.device.index is not None else 0)
        self._h = C.c_void_p()
        _capi.check(self.lib, self.lib.cn_dsrnn_create(C.byref(cfg), C.byref(self._h)), "cn_dsrnn_create")

    def load_state_dict(self, sd):
        for k, v in sd.items():
            if k.startswith(DSRNN_UNUSED):
                continue
            arr = v.detach().to("cpu", torch.float32).contiguous().numpy()
            _capi.check(self.lib, self.lib.cn_dsrnn_set_param(self._h, k.encode(), arr.ctypes.data, arr.size),
                        "cn_dsrnn_set_param(%s)" % k)
        with torch.cuda.device(self.device):
            _capi.check(self.lib, self.lib.cn_dsrnn_finalize(self._h, self._stream()), "cn_dsrnn_finalize")

    def act(self, obs, h, edge_h, masks, deterministic=False, return_mean=False, noise=None, out=None):
        """As CudaPolicy.act, plus the edge state: edge_h [N,H+1,256] (None or an expanded zero: zero state) in,
        edge_h_out out (also an `out` key).  Returns value, action, log_prob, h_new, edge_h_new (, mean)."""
        b = self._outputs(out, ("value", "action", "log_prob", "h_out", "edge_h_out"))
        noise = self._noise(deterministic, noise)
        args = self._inputs(robot_node=obs["robot_node"], temporal_edges=obs["temporal_edges"],
                            spatial_edges=obs["spatial_edges"], h_in=h, masks=masks)
        if not _is_zero_view(edge_h):
            args.update(self._inputs(edge_h_in=edge_h))
        eh = args.get("edge_h_in")
        ptrs = _capi.CnDsrnnActPtrs(
            args["robot_node"].data_ptr(), args["temporal_edges"].data_ptr(), args["spatial_edges"].data_ptr(),
            args["h_in"].data_ptr(), None if eh is None else eh.data_ptr(), args["masks"].data_ptr(),
            None if deterministic else noise.data_ptr(), b["value"].data_ptr(), b["action"].data_ptr(),
            b["log_prob"].data_ptr(), b["h_out"].data_ptr(), b["edge_h_out"].data_ptr(), b["mean"].data_ptr())
        rc = self.lib.cn_dsrnn_act(self._h, C.byref(ptrs), self._stream())
        if rc:
            _capi.check(self.lib, rc, "cn_dsrnn_act")
        self._keep = (args, noise)
        res = (b["value"], b["action"], b["log_prob"], b["h_out"], b["edge_h_out"])
        return res + (b["mean"],) if return_mean else res

    def launch_count(self):
        return int(self.lib.cn_dsrnn_launch_count(self._h))

    def stage_ms(self):
        """{stage: ms} of the last act (profiling must have been enabled with profile(True) before it)."""
        n = self.lib.cn_dsrnn_stage_count()
        out = (C.c_float * n)()
        _capi.check(self.lib, self.lib.cn_dsrnn_stage_ms(self._h, out, n), "cn_dsrnn_stage_ms")
        return {self.lib.cn_dsrnn_stage_name(i).decode(): float(out[i]) for i in range(n)}

    def profile(self, enable=True):
        _capi.check(self.lib, self.lib.cn_dsrnn_profile(self._h, int(enable)), "cn_dsrnn_profile")

    def close(self):
        if self._h:
            self.lib.cn_dsrnn_destroy(self._h)
            self._h = None


class _SrnnParams(nn.Module):
    """Parameter container with the reference SRNN's module tree (srnn_model.py:326-387) and initialisers."""

    def __init__(self, input_size):
        super().__init__()
        g = math.sqrt(2)

        def gru(i, h):
            m = nn.GRU(i, h)
            for name, prm in m.named_parameters():                 # srnn_model.py:26-30
                if 'bias' in name:
                    nn.init.constant_(prm, 0)
                else:
                    nn.init.orthogonal_(prm)
            return m

        def edge_rnn(w):
            e = nn.Module()
            e.gru = gru(64, EDGE)
            e.encoder_linear = nn.Linear(w, 64)
            return e
        base = nn.Module()
        node = nn.Module()
        node.gru = gru(128, HIDDEN)
        node.encoder_linear = nn.Linear(3, 64)
        node.edge_embed = nn.Linear(EDGE, 64)                      # unused by the forward
        node.edge_attention_embed = nn.Linear(2 * EDGE, 64)
        node.output_linear = nn.Linear(HIDDEN, 256)
        base.humanNodeRNN = node
        base.humanhumanEdgeRNN_spatial = edge_rnn(input_size)
        base.humanhumanEdgeRNN_temporal = edge_rnn(2)
        att = nn.Module()
        att.temporal_edge_layer = nn.ModuleList([nn.Linear(EDGE, 64)])
        att.spatial_edge_layer = nn.ModuleList([nn.Linear(EDGE, 64)])
        base.attn = att
        base.actor = nn.Sequential(_ortho(nn.Linear(256, 256), g), nn.Tanh(), _ortho(nn.Linear(256, 256), g), nn.Tanh())
        base.critic = nn.Sequential(_ortho(nn.Linear(256, 256), g), nn.Tanh(), _ortho(nn.Linear(256, 256), g), nn.Tanh())
        base.critic_linear = _ortho(nn.Linear(256, 1), g)
        base.robot_linear = _ortho(nn.Linear(7, 3), g)
        base.human_node_final_linear = _ortho(nn.Linear(256, 2), g)   # unused by the forward
        base.spatial_linear = _ortho(nn.Linear(input_size, 2), g)     # unused by the forward
        self.base = base
        dist = nn.Module()
        dist.fc_mean = _ortho(nn.Linear(256, 2))
        dist.logstd = _AddBias(2)
        self.dist = dist


def _gru_masked(gru, x, h, masks, rep):
    """RNNBase._forward_gru (srnn_model.py:50-103) over [T, B, in] with done masks [T, n] (B = n * rep rows): the
    sequence is cut where any mask is 0, and each segment starts from h * mask.  Returns outputs [T, B, hid], h."""
    T = x.shape[0]
    cuts = [0] + [t + 1 for t in (masks[1:] == 0).any(-1).nonzero().flatten().tolist()] + [T]
    outs = []
    for a, b in zip(cuts[:-1], cuts[1:]):
        h = h * masks[a].repeat_interleave(rep)[:, None]
        y, h1 = gru(x[a:b], h[None])
        h = h1[0]
        outs.append(y)
    return torch.cat(outs, 0), h


def _hh_attention(q, k, v, valid):
    """softmax(q k^T / 8 + key mask) v for [B, 8, H, 64] tensors with H <= ~20 keys.  Written as two batched
    matmuls: at this shape the fused 'memory efficient' SDPA kernels (64 x 64 tiles for a 20-key sequence) cost
    3x the explicit form in forward + backward (CN_SDPA=1 switches back)."""
    if os.environ.get("CN_SDPA", "0") == "1":
        return F.scaled_dot_product_attention(q, k, v, attn_mask=valid[:, None, None, :])
    s = torch.matmul(q, k.transpose(-1, -2)) * 0.125
    s = s.masked_fill(~valid[:, None, None, :], float("-inf"))
    return torch.matmul(torch.softmax(s, dim=-1), v)


# The widths every kernel has fixed, by the argument that sets them in the reference's arguments.py, and which base's
# module reads it: selfAttn_merge_SRNN's EndRNN / EdgeAttention_M never read human_human_edge_embedding_size (its node
# GRU is RNNBase(edge=False)); SRNN's edge RNNs do.
WIDTHS = (("human_node_rnn_size", HIDDEN, ("selfAttn_merge_srnn", "srnn")),
          ("human_human_edge_rnn_size", 256, ("selfAttn_merge_srnn", "srnn")),
          ("human_node_output_size", 256, ("selfAttn_merge_srnn", "srnn")),
          ("human_node_embedding_size", 64, ("selfAttn_merge_srnn", "srnn")),
          ("human_human_edge_embedding_size", 64, ("srnn",)),
          ("attention_size", 64, ("selfAttn_merge_srnn", "srnn")))


def check_widths(args, base):
    """Refuse an argument file whose network widths differ from the ones the kernels are built for."""
    if args is None:
        return
    for name, width, bases in WIDTHS:
        v = getattr(args, name, width)
        if base in bases and int(v) != width:
            raise NotImplementedError("%s = %r: the engine's %s network is built for %s = %d only"
                                      % (name, v, base, name, width))


class Policy(nn.Module):
    """Drop-in for rl.networks.model.Policy(obs_space.spaces, action_space, base_kwargs=args, base=...).

    args.use_self_attn = False (selfAttn_merge_srnn only; True when absent) is the reference's ablation without
    human-human attention.  args.sort_humans = False (selfAttn_merge_srnn only; True when absent) masks both
    attentions with inputs['visible_masks'] instead of the detected_human_num prefix (selfAttn_srnn_temp_node.py:
    375-383).  args.use_hr_attn is accepted and changes nothing: the reference never reads it."""

    def __init__(self, obs_shape, action_space, base=None, base_kwargs=None):
        super().__init__()
        if base not in (None, 'selfAttn_merge_srnn', 'srnn'):
            raise NotImplementedError("base=%r: the engine runs 'selfAttn_merge_srnn' and 'srnn'" % (base,))
        args = base_kwargs
        self.dsrnn = base == 'srnn'
        if self.dsrnn:
            # The reference reads args.env_type (srnn_model.py:378), which arguments.py never defines; 'crowd_sim' is
            # the only value whose robot_linear input width (7) matches robot_node, so a missing env_type means it.
            env_type = getattr(args, 'env_type', 'crowd_sim') if args is not None else 'crowd_sim'
            if env_type != 'crowd_sim':
                raise NotImplementedError("base='srnn' runs env_type 'crowd_sim' only (got %r)" % (env_type,))
        check_widths(args, 'srnn' if self.dsrnn else 'selfAttn_merge_srnn')
        # the reference's SRNN ignores use_self_attn (srnn_model.py); older argument files lack it (True)
        self.self_attn = self.dsrnn or bool(getattr(args, 'use_self_attn', True))
        # the SRNN never reads sort_humans either; older argument files lack it (True, :376-377)
        self.sort_humans = self.dsrnn or bool(getattr(args, 'sort_humans', True))
        sp = obs_shape['spatial_edges'].shape
        self.human_num, self.input_size = int(sp[0]), int(sp[1])
        self.nenv = int(getattr(args, 'num_processes', 1)) if args is not None else 1
        self.seq_length = int(getattr(args, 'seq_length', 30)) if args is not None else 30
        self.nminibatch = int(getattr(args, 'num_mini_batch', 2)) if args is not None else 2
        p = _SrnnParams(self.input_size) if self.dsrnn else _Params(self.input_size, self.self_attn)
        self.base = p.base
        # attributes the reference's callers read / write on `actor_critic.base` (test.py:148, rl/evaluation.py:15-21)
        self.base.nenv = self.nenv
        self.base.human_num = self.human_num
        self.base.seq_length, self.base.nminibatch = self.seq_length, self.nminibatch
        self.base.human_node_rnn_size = int(getattr(args, 'human_node_rnn_size', HIDDEN)) if args is not None else HIDDEN
        self.base.human_human_edge_rnn_size = int(getattr(args, 'human_human_edge_rnn_size', 256)) if args is not None else 256
        self.base.output_size = 256
        self.dist = p.dist
        self.srnn = True
        self._cuda = None
        self._cuda_version = -1

    is_recurrent = True

    @property
    def recurrent_hidden_state_size(self):
        return HIDDEN

    # ------------------------------------------------------------------ CUDA rollout path
    def _engine(self, N, device):
        if self._cuda is None or self._cuda.N != N or self._cuda.device != device:
            if self.dsrnn:
                self._cuda = CudaDsrnn(N, self.human_num, self.input_size, device=device)
            else:
                self._cuda = CudaPolicy(N, self.human_num, self.input_size, device=device,
                                        gemm_mode=int(os.environ.get("CN_GEMM_MODE", "1")), self_attn=self.self_attn,
                                        visible_masks=not self.sort_humans)
            self._cuda_version = -1
        # parameter objects are fixed after construction: walk the module tree once, then only read the
        # version counters (the tree walk alone cost ~0.1 ms of host time per act)
        plist = self.__dict__.get("_plist")
        if plist is None:
            plist = self.__dict__["_plist"] = list(self.parameters())
        v = 0
        for p in plist:
            v += p._version
        # .to() / .data swaps replace storage without bumping the version: they move every parameter, watch the two ends
        ver = (v, plist[0].data_ptr(), plist[-1].data_ptr())
        if ver != self._cuda_version:                       # parameters changed (optimizer step / load_state_dict)
            self._cuda.load_state_dict(self.state_dict())
            self._cuda_version = ver
        return self._cuda

    def act(self, inputs, rnn_hxs, masks, deterministic=False):
        sp = inputs['spatial_edges']
        eng = self._engine(sp.shape[0], sp.device)
        if self.dsrnn:
            value, action, logp, h_new, e_new = eng.act(inputs, rnn_hxs['human_node_rnn'],
                                                        rnn_hxs.get('human_human_edge_rnn'), masks,
                                                        deterministic=deterministic)
            return value, action, logp, {'human_node_rnn': h_new, 'human_human_edge_rnn': e_new}
        value, action, logp, h_new = eng.act(inputs, rnn_hxs['human_node_rnn'], masks, deterministic=deterministic)
        z = self.__dict__.get("_zero_edge")
        if z is None or z.device != sp.device or z.shape[0] != sp.shape[0]:
            # all-zeros in the reference (selfAttn_srnn_temp_node.py:390-395): stride-0 view, no 2.7 GB buffer
            z = self.__dict__["_zero_edge"] = torch.zeros(1, 1, 1, device=sp.device).expand(sp.shape[0], self.human_num + 1, 256)
        out_hxs = {'human_node_rnn': h_new, 'human_human_edge_rnn': z}
        return value, action, logp, out_hxs

    def get_value(self, inputs, rnn_hxs, masks):
        sp = inputs['spatial_edges']
        eng = self._engine(sp.shape[0], sp.device)
        if self.dsrnn:
            return eng.act(inputs, rnn_hxs['human_node_rnn'], rnn_hxs.get('human_human_edge_rnn'), masks,
                           deterministic=True)[0]
        value, _, _, _ = eng.act(inputs, rnn_hxs['human_node_rnn'], masks, deterministic=True)
        return value

    # ------------------------------------------------------------------ PyTorch update path
    def _features(self, inputs, h0, masks, T, N):
        b = self.base
        H = self.human_num
        dt = b.robot_linear[0].weight.dtype            # fp32; fp64 when a test runs the module in double as its reference
        sp = inputs['spatial_edges'].reshape(T * N, H, -1).to(dt)
        if self.sort_humans:
            n = inputs['detected_human_num'].reshape(T * N).long().clamp(1, H)
            valid = torch.arange(H, device=sp.device)[None, :] < n[:, None]
        else:
            # visible_masks, and slot 0 alone for a sample that sees nobody (dummy_human_mask, :351-358, :382-383)
            valid = inputs['visible_masks'].reshape(T * N, H).bool().clone()
            valid[:, 0] |= ~valid.any(1)
            n = valid.sum(1)
        rs = b.robot_linear(torch.cat([inputs['temporal_edges'].reshape(T * N, 2),
                                       inputs['robot_node'].reshape(T * N, 7)], -1).to(dt))
        B = T * N
        use_tc = sp.is_cuda and dt == torch.float32 and getattr(self, "update_kernels", os.environ.get("CN_UPDATE_KERNELS", "1") == "1")
        if use_tc:
            from . import update_ops as uo

        def pad(x):
            out = x.new_zeros(B, H, x.shape[-1])
            out[valid] = x
            return out

        def compact_layout():
            row_start = torch.zeros(B + 1, dtype=torch.int32, device=sp.device)
            row_start[1:] = torch.cumsum(n, 0)
            return row_start, torch.repeat_interleave(torch.arange(B, device=sp.device, dtype=torch.int32), n)
        if not self.self_attn:
            # use_self_attn = False: spatial_linear straight on the spatial edges (selfAttn_srnn_temp_node.py:408-410)
            sl = b.spatial_linear
            hs_c = row_env = None
            if not getattr(self, "pack_valid_rows", True):
                hs = sl(sp)
            elif use_tc:
                e1 = torch.relu(F.linear(sp[valid], sl[0].weight, sl[0].bias))       # K = W <= 12: torch
                hs_c = uo.linear_tc(e1, sl[2].weight, sl[2].bias, 1)                  # [Mc, 256], compact
                hs = None
                row_env = compact_layout()[1]
            else:
                hs = pad(sl(sp[valid]))
        else:
            hs, hs_c, row_env = self._hh_features(sp, n, valid, B, use_tc, pad, compact_layout)
        return self._tail(rs, hs, hs_c, row_env, valid, h0, masks, T, N)

    def _hh_features(self, sp, n, valid, B, use_tc, pad, compact_layout):
        """Human-human attention then spatial_linear: hs [B, H, 256] (padded rows zero), or with the update kernels
        (hs = None) the compact hs_c [Mc, 256] and its row_env."""
        b = self.base
        H = self.human_num
        sa = b.spatial_attn
        mha = sa.multihead_attn
        wq, wk, wv = mha.in_proj_weight.chunk(3, 0)
        bq, bk, bv = mha.in_proj_bias.chunk(3, 0)
        if use_tc:
            from . import update_ops as uo
        hs_c = row_env = None

        def heads(x):
            return x.reshape(B, H, 8, 64).transpose(1, 2)
        amask = valid[:, None, None, :]
        if getattr(self, "pack_valid_rows", True):
            # Same compaction as the rollout kernels: rows j >= detected_human_num are keys masked by
            # key_padding_mask and queries whose outputs get weight exactly 0 in the robot-human soft-max
            # (masked_fill(-1e9)), so they contribute neither to the outputs nor to any gradient.  The per-row
            # layers (98 % of the FLOPs) run on the valid rows only; the tiny H x H attention runs padded.
            sp_p = sp[valid]                                             # [Mc, W]
            # update kernels (SURVEY §8f row 3): the three 128/512-wide per-row layers forward + backward on the wgmma
            # 3xFP16 GEMM and the attention core over compacted rows; plain torch ops on CPU or with CN_UPDATE_KERNELS=0
            if use_tc:
                e1 = torch.relu(F.linear(sp_p, sa.embedding_layer[0].weight, sa.embedding_layer[0].bias))   # K = 12: torch
                e = uo.linear_tc(e1, sa.embedding_layer[2].weight, sa.embedding_layer[2].bias, 1)
            else:
                e = sa.embedding_layer(sp_p)
            # The same exact folds as the rollout engine, written so that autograd sees them: in_proj o q/k/v_linear
            # is ONE 512 -> 1536 projection whose weight is the (differentiable) product of the two parameter
            # matrices, and out_proj o spatial_linear one 512 -> 256 projection: the per-row GEMMs of forward AND
            # backward shrink 2x, the parameter gradients flow back through the small 512^3 products.
            wl = torch.cat([sa.q_linear.weight, sa.k_linear.weight, sa.v_linear.weight], 0).reshape(3, 512, 512)
            bl = torch.stack([sa.q_linear.bias, sa.k_linear.bias, sa.v_linear.bias], 0)
            win = mha.in_proj_weight.reshape(3, 512, 512)
            w_qkv = torch.bmm(win, wl).reshape(1536, 512)
            b_qkv = (torch.bmm(win, bl.unsqueeze(-1)).squeeze(-1) + mha.in_proj_bias.reshape(3, 512)).reshape(1536)
            sl = b.spatial_linear[0]
            w_os = sl.weight @ mha.out_proj.weight
            b_os = sl.weight @ mha.out_proj.bias + sl.bias
            if use_tc:
                qkv = uo.linear_tc(e, w_qkv, b_qkv, 0)
                row_start, row_env = compact_layout()
                o = uo.hh_attention_rows(qkv, row_start, row_env)
                hs_c = uo.linear_tc(o, w_os, b_os, 1)          # [Mc, 256]: stays compact through the robot-human attention
                hs = None
            else:
                qkv = F.linear(e, w_qkv, b_qkv)
                q, k, v = [heads(pad(t)) for t in qkv.chunk(3, -1)]
                o = _hh_attention(q, k, v, valid)
                o = o.transpose(1, 2).reshape(B, H, 512)[valid]
                hs = pad(torch.relu(F.linear(o, w_os, b_os)))
        else:
            e = sa.embedding_layer(sp)
            q = heads(F.linear(sa.q_linear(e), wq, bq))
            k = heads(F.linear(sa.k_linear(e), wk, bk))
            v = heads(F.linear(sa.v_linear(e), wv, bv))
            o = F.scaled_dot_product_attention(q, k, v, attn_mask=amask)
            o = mha.out_proj(o.transpose(1, 2).reshape(B, H, 512))
            hs = b.spatial_linear(o)
        return hs, hs_c, row_env

    def _tail(self, rs, hs, hs_c, row_env, valid, h0, masks, T, N):
        """Robot-human attention, node GRU, actor / critic over the per-human features hs [B, H, 256], or the compact
        hs_c [Mc, 256] with its row_env (update kernels)."""
        b = self.base
        H = self.human_num
        B = T * N
        tc_rows = hs is None                       # update kernels: per-sample layers on the tensor cores as well
        if tc_rows:
            from . import update_ops as uo

            def lin(x, layer, act=0):
                return uo.linear_tc(x, layer.weight, layer.bias, act)
        else:
            def lin(x, layer, act=0):
                y = F.linear(x, layer.weight, layer.bias)
                return torch.relu(y) if act else y
        te = lin(rs, b.attn.temporal_edge_layer[0])
        if tc_rows:
            # robot-human attention over the compact rows: scores of the valid humans, soft-max per sample on a padded
            # [B, H] score table only, weighted sum by index_add (the padded [B, H, 256] feature tensor never exists)
            renv = row_env.long()
            se_c = lin(hs_c, b.attn.spatial_edge_layer[0])
            sc_c = (te.index_select(0, renv) * se_c).sum(-1) * (H / 8.0)
            scores = sc_c.new_full((B, H), -1e9)
            scores[valid] = sc_c
            att_c = torch.softmax(scores, dim=-1)[valid]
            wvv = hs_c.new_zeros(B, hs_c.shape[-1]).index_add_(0, renv, hs_c * att_c.unsqueeze(-1))
        else:
            se = b.attn.spatial_edge_layer[0](hs)
            att = (te[:, None, :] * se).sum(-1) * (H / 8.0)
            att = torch.softmax(att.masked_fill(~valid, -1e9), dim=-1)
            wvv = torch.bmm(hs.transpose(1, 2), att.unsqueeze(-1)).squeeze(-1)
        r = b.humanNodeRNN
        x = torch.cat([lin(rs, r.encoder_linear, 1), lin(wvv, r.edge_attention_embed, 1)], -1)
        g = r.gru
        h = h0.reshape(N, HIDDEN)
        m = masks.reshape(T, N, 1)
        if tc_rows:
            gi_all = uo.linear_tc(x, g.weight_ih_l0, g.bias_ih_l0, 0).reshape(T, N, 3 * HIDDEN)
        else:
            gi_all = F.linear(x.reshape(T, N, 128), g.weight_ih_l0, g.bias_ih_l0)
        if tc_rows:
            hseq = uo.gru_sequence(gi_all, h, m.reshape(T, N), g.weight_hh_l0, g.bias_hh_l0)    # one launch for the T steps
            h = hseq[-1]
        else:
            outs = []
            for t in range(T):
                h = h * m[t]
                gh = F.linear(h, g.weight_hh_l0, g.bias_hh_l0)
                ir, iz, inn = gi_all[t].chunk(3, -1)
                hr, hz, hn = gh.chunk(3, -1)
                rg = torch.sigmoid(ir + hr)
                zg = torch.sigmoid(iz + hz)
                ng = torch.tanh(inn + rg * hn)
                h = (1 - zg) * ng + zg * h
                outs.append(h)
            hseq = torch.stack(outs, 0)
        y = lin(hseq.reshape(T * N, HIDDEN), r.output_linear)
        hc = torch.tanh(lin(torch.tanh(lin(y, b.critic[0])), b.critic[2]))
        ha = torch.tanh(lin(torch.tanh(lin(y, b.actor[0])), b.actor[2]))
        return b.critic_linear(hc), ha, h.reshape(N, 1, HIDDEN)

    def _features_dsrnn(self, inputs, hxs, masks, T, N):
        """SRNN.forward with infer=False (srnn_model.py:389-468) over a [T, N] minibatch: PyTorch ops (cuDNN GRUs on
        a CUDA device).  hxs: node state [N,1,128] and edge state [N,H+1,256] (an expanded zero is fine)."""
        b = self.base
        H = self.human_num
        m = masks.reshape(T, N)
        he = hxs['human_human_edge_rnn'].reshape(N, H + 1, EDGE)
        et, es = b.humanhumanEdgeRNN_temporal, b.humanhumanEdgeRNN_spatial
        xt = torch.relu(et.encoder_linear(inputs['temporal_edges'].reshape(T, N, 2)))
        ht, ht_last = _gru_masked(et.gru, xt, he[:, 0], m, 1)                          # [T, N, 256]
        xs = torch.relu(es.encoder_linear(inputs['spatial_edges'].reshape(T, N * H, -1)))
        hs, hs_last = _gru_masked(es.gru, xs, he[:, 1:].reshape(N * H, EDGE), m, H)   # [T, N H, 256]
        hs = hs.reshape(T, N, H, EDGE)
        te = b.attn.temporal_edge_layer[0](ht)
        se = b.attn.spatial_edge_layer[0](hs)
        p = torch.softmax((te[:, :, None, :] * se).sum(-1) * (H / 8.0), dim=-1)
        wv = torch.matmul(p[:, :, None, :], hs).squeeze(2)                             # [T, N, 256]
        nr = b.humanNodeRNN
        enc = torch.relu(nr.encoder_linear(b.robot_linear(inputs['robot_node'].reshape(T, N, 7))))
        emb = torch.relu(nr.edge_attention_embed(torch.cat([ht, wv], -1)))
        hn, hn_last = _gru_masked(nr.gru, torch.cat([enc, emb], -1), hxs['human_node_rnn'].reshape(N, HIDDEN), m, 1)
        x = nr.output_linear(hn).reshape(T * N, 256)
        edge = torch.cat([ht_last[:, None], hs_last.reshape(N, H, EDGE)], 1)
        return b.critic_linear(b.critic(x)), b.actor(x), {'human_node_rnn': hn_last.reshape(N, 1, HIDDEN),
                                                         'human_human_edge_rnn': edge}

    def evaluate_actions(self, inputs, rnn_hxs, masks, action):
        """inputs flattened [T*N, ...] (storage.py recurrent_generator), rnn_hxs['human_node_rnn'] [N,1,128]
        (DS-RNN: and rnn_hxs['human_human_edge_rnn'] [N,H+1,256])."""
        h0 = rnn_hxs['human_node_rnn']
        N = h0.shape[0]
        T = inputs['spatial_edges'].shape[0] // N
        if self.dsrnn:
            value, feat, hxs = self._features_dsrnn(inputs, rnn_hxs, masks, T, N)
        else:
            value, feat, h = self._features(inputs, h0, masks, T, N)
            hxs = {'human_node_rnn': h}
        mean = self.dist.fc_mean(feat)
        logstd = self.dist.logstd._bias.t().view(1, -1).expand_as(mean)
        dist = torch.distributions.Normal(mean, logstd.exp())
        logp = dist.log_prob(action).sum(-1, keepdim=True)
        # the reference's FixedNormal defines `entrop` (typo, distributions.py:42), so model.py:88 reaches
        # torch's Normal.entropy() -> [B, 2] and .mean() averages over BOTH action dimensions
        entropy = dist.entropy().mean()
        return value, logp, entropy, hxs
