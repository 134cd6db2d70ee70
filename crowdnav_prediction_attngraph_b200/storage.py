"""Device-resident rollout buffer with the reference's RolloutStorage surface
(rl/networks/storage.py:13-253): obs{} / recurrent_hidden_states{} / masks / insert /
compute_returns (GAE) / after_update / recurrent_generator — everything stays on the GPU.

Differences that do not change results: tensors are created directly on `device`; the
`human_human_edge_rnn` hidden state (2.7 GB at N=4096, H=20 in the reference, storage.py:34) starts as a
stride-0 expanded zero, which is all the attention-graph policy ever stores there; the first `insert` of a
real edge state (the DS-RNN policy, base='srnn') replaces it with a [T+1, N, H+1, 256] buffer;
`recurrent_generator` gathers minibatches with one index_select per tensor instead of a Python loop over
environments (storage.py:208-223)."""

import torch

from .policy import CudaDsrnn, _is_zero_view


class RolloutStorage(object):
    def __init__(self, num_steps, num_processes, obs_shape, action_space, human_node_rnn_size,
                 human_human_edge_rnn_size, device="cpu"):
        T, N = num_steps, num_processes
        dev = torch.device(device)
        self.device = dev
        self.obs = {}
        for key in obs_shape:
            shp = tuple(obs_shape[key].shape)
            dt = torch.bool if str(getattr(obs_shape[key], "dtype", "float32")) == "bool" else torch.float32
            self.obs[key] = torch.zeros(T + 1, N, *shp, dtype=dt, device=dev)
        self.human_num = obs_shape['spatial_edges'].shape[0]
        self.recurrent_hidden_states = {
            'human_node_rnn': torch.zeros(T + 1, N, 1, human_node_rnn_size, device=dev),
            'human_human_edge_rnn': torch.zeros(1, 1, 1, 1, device=dev).expand(
                T + 1, N, self.human_num + 1, human_human_edge_rnn_size),
        }
        self.rewards = torch.zeros(T, N, 1, device=dev)
        self.value_preds = torch.zeros(T + 1, N, 1, device=dev)
        self.returns = torch.zeros(T + 1, N, 1, device=dev)
        self.action_log_probs = torch.zeros(T, N, 1, device=dev)
        self.actions = torch.zeros(T, N, action_space.shape[0], device=dev)
        self.masks = torch.ones(T + 1, N, 1, device=dev)
        self.bad_masks = torch.ones(T + 1, N, 1, device=dev)
        self.num_steps = T
        self.step = 0

    def to(self, device):
        dev = torch.device(device)
        if dev == self.device:
            return
        for key in self.obs:
            self.obs[key] = self.obs[key].to(dev)
        hn = self.recurrent_hidden_states
        hn['human_node_rnn'] = hn['human_node_rnn'].to(dev)
        e = hn['human_human_edge_rnn']
        hn['human_human_edge_rnn'] = e.to(dev) if self._edge_real() else torch.zeros(1, 1, 1, 1, device=dev).expand(*e.shape)
        for name in ("rewards", "value_preds", "returns", "action_log_probs", "actions", "masks", "bad_masks"):
            setattr(self, name, getattr(self, name).to(dev))
        self.device = dev

    def _edge_real(self):
        return self.recurrent_hidden_states['human_human_edge_rnn'].stride()[0] != 0

    def _edge_materialise(self):
        """Switch to a real (zero-filled) edge-state buffer; called the first time a recurrent edge state arrives."""
        if self._edge_real():
            return
        e = self.recurrent_hidden_states['human_human_edge_rnn']
        self.recurrent_hidden_states['human_human_edge_rnn'] = torch.zeros(*e.shape, device=self.device)
        self.__dict__.pop("_slots", None)

    def _dsts(self, s):
        dst = [self.obs[key][s + 1] for key in self.obs]
        dst += [self.recurrent_hidden_states['human_node_rnn'][s + 1], self.actions[s], self.action_log_probs[s],
                self.value_preds[s], self.rewards[s], self.masks[s + 1], self.bad_masks[s + 1]]
        if self._edge_real():
            dst.append(self.recurrent_hidden_states['human_human_edge_rnn'][s + 1])
        return dst

    def _slot_table(self):
        """Per step index: the destination tensors of insert() with their device pointers and byte sizes, built once per
        device (the storage tensors are never reallocated except by .to() and the switch to a real edge state, which
        drop the table)."""
        return [[(d, d.data_ptr(), d.numel() * d.element_size()) for d in self._dsts(s)] for s in range(self.num_steps)]

    def insert(self, obs, recurrent_hidden_states, actions, action_log_probs, value_preds, rewards, masks, bad_masks=None):
        """rl/networks/storage.py:70-86.  Every source that the GPU can read directly -- device tensors (observations,
        hidden state, action, log-prob, value) and PINNED host tensors (reward / masks built by the caller from `done`)
        -- is copied by ONE cn_copy_segments launch instead of twelve torch copy_ calls; pageable host tensors (what the
        reference's train.py builds) take the usual H2D copy_."""
        s = self.step
        edge = recurrent_hidden_states.get('human_human_edge_rnn')
        if not _is_zero_view(edge):
            self._edge_materialise()
        srcs = [obs[key] for key in self.obs]
        srcs += [recurrent_hidden_states['human_node_rnn'], actions, action_log_probs, value_preds, rewards, masks, bad_masks]
        if self._edge_real():
            srcs.append(edge)
        if self.device.type != "cuda":
            for dst, src in zip(self._dsts(s), srcs):
                if src is not None:
                    dst.copy_(src.reshape(dst.shape) if src.numel() == dst.numel() else src)
            self.step = (s + 1) % self.num_steps
            return
        d = self.__dict__
        segs = d.get("_segs")
        if segs is None:
            from . import _capi
            self._capi, self._lib = _capi, _capi.load_library()
            segs = self._segs = (_capi.CnCopySeg * 16)()
        tab = d.get("_slots")
        if tab is None or d.get("_slots_key") != self.rewards.data_ptr():
            tab = self._slots = self._slot_table()
            self._slots_key = self.rewards.data_ptr()
        dev, n = self.device, 0
        for (dst, dptr, nbytes), src in zip(tab[s], srcs):
            if src is None:
                continue
            if (n < 16 and src.dtype is dst.dtype and src.numel() * src.element_size() == nbytes and src.is_contiguous()
                    and (src.device == dev if src.is_cuda else src.is_pinned())):
                sptr = src.data_ptr()
                if sptr != dptr:
                    g = segs[n]
                    g.dst, g.src, g.bytes = dptr, sptr, nbytes
                    n += 1
            else:
                dst.copy_(src.reshape(dst.shape) if src.numel() == dst.numel() else src, non_blocking=True)
        if n:
            rc = self._lib.cn_copy_segments(segs, n, dev.index or 0, self._capi.raw_stream(dev.index or 0))
            if rc:
                self._capi.check(self._lib, rc, "cn_copy_segments")
        self.step = (s + 1) % self.num_steps

    def rollout_step_zero_copy(self, engine, env, deterministic=False):
        """One device-resident rollout step with NO copies: the policy kernels write value / action /
        log-prob / hidden state and the env kernels write observation / reward / mask straight into
        this storage's slots (equivalent to act -> envs.step -> insert of train.py:152-191)."""
        s = self.step
        o = {k: v[s] for k, v in self.obs.items()}
        hn = self.recurrent_hidden_states['human_node_rnn']
        out = dict(value=self.value_preds[s], action=self.actions[s], log_prob=self.action_log_probs[s], h_out=hn[s + 1])
        if isinstance(engine, CudaDsrnn):
            # the DS-RNN engine carries the edge state: its kernels write slot s + 1 of a real buffer
            self._edge_materialise()
            he = self.recurrent_hidden_states['human_human_edge_rnn']
            out["edge_h_out"] = he[s + 1]
            engine.act(o, hn[s], he[s], self.masks[s], deterministic=deterministic, out=out)
        else:
            engine.act(o, hn[s], self.masks[s], deterministic=deterministic, out=out)
        env.step_device(self.actions[s], obs_out={k: v[s + 1] for k, v in self.obs.items()},
                        reward_out=self.rewards[s], not_done_out=self.masks[s + 1])
        self.step = (s + 1) % self.num_steps

    def after_update(self):
        for key in self.obs:
            self.obs[key][0].copy_(self.obs[key][-1])
        self.recurrent_hidden_states['human_node_rnn'][0].copy_(self.recurrent_hidden_states['human_node_rnn'][-1])
        if self._edge_real():
            self.recurrent_hidden_states['human_human_edge_rnn'][0].copy_(self.recurrent_hidden_states['human_human_edge_rnn'][-1])
        self.masks[0].copy_(self.masks[-1])
        self.bad_masks[0].copy_(self.bad_masks[-1])

    def compute_returns(self, next_value, use_gae, gamma, gae_lambda, use_proper_time_limits=True):
        T = self.rewards.size(0)
        if use_gae:
            self.value_preds[-1] = next_value
            gae = torch.zeros_like(self.value_preds[0])
            for step in reversed(range(T)):
                delta = self.rewards[step] + gamma * self.value_preds[step + 1] * self.masks[step + 1] - self.value_preds[step]
                gae = delta + gamma * gae_lambda * self.masks[step + 1] * gae
                if use_proper_time_limits:
                    gae = gae * self.bad_masks[step + 1]
                self.returns[step] = gae + self.value_preds[step]
        else:
            self.returns[-1] = next_value
            for step in reversed(range(T)):
                r = self.returns[step + 1] * gamma * self.masks[step + 1] + self.rewards[step]
                if use_proper_time_limits:
                    r = r * self.bad_masks[step + 1] + (1 - self.bad_masks[step + 1]) * self.value_preds[step]
                self.returns[step] = r

    def recurrent_generator(self, advantages, num_mini_batch, generator=None):
        T, N = self.num_steps, self.rewards.size(1)
        assert N >= num_mini_batch
        per = N // num_mini_batch
        perm = torch.randperm(N, generator=generator).to(self.device)
        for start in range(0, per * num_mini_batch, per):
            ind = perm[start:start + per]
            flat = lambda x: x.index_select(1, ind).reshape(T * per, *x.shape[2:])
            obs_batch = {k: flat(v[:-1]) for k, v in self.obs.items()}
            he = self.recurrent_hidden_states['human_human_edge_rnn']
            hxs = {'human_node_rnn': self.recurrent_hidden_states['human_node_rnn'][0].index_select(0, ind),
                   'human_human_edge_rnn': he[0].index_select(0, ind) if self._edge_real() else he[0, :per]}
            yield (obs_batch, hxs, flat(self.actions), flat(self.value_preds[:-1]), flat(self.returns[:-1]),
                   flat(self.masks[:-1]), flat(self.action_log_probs), flat(advantages))
