"""Test references of the policy on unsorted humans (the reference's args.sort_humans = False,
rl/networks/selfAttn_srnn_temp_node.py:375-383): both attentions are masked with inputs['visible_masks'] (slot order,
any pattern) instead of the detected_human_num prefix, and a sample with no visible human keeps slot 0 only
(dummy_human_mask, :351-358).

  * `visible_valid`: that mask, [N, H] bool.
  * `PolicyRefUnsorted` / `PolicyRefNoSelfAttnUnsorted`: the plain PyTorch forwards of oracle/policy_ref.py and
    tests/policy_no_self_attn_ref.py with this mask.  Pinned against the unmodified reference by
    tests/golden/policy_unsorted_*.npz (tools/make_golden_policy.py --unsorted).
  * `StagedRefUnsorted` / `StagedRefNoSelfAttnUnsorted`: the fp64 stage references over the engine's compacted rows,
    with the rows chosen by the mask; row r holds slot row_slot[r].
"""
import torch

from oracle.policy_ref import PolicyRef
from tests.policy_no_self_attn_ref import PolicyRefNoSelfAttn, StagedRefNoSelfAttn
from tests.policy_stages import StagedRef


def visible_valid(vis, H):
    valid = torch.as_tensor(vis).reshape(-1, H).bool().clone()
    valid[:, 0] |= ~valid.any(1)
    return valid


def mask_layout(vis, H, dev="cpu"):
    """(n [N], row_start [N+1], row_env [Mc], row_slot [Mc]) of the visible-mask compaction, int64"""
    valid = visible_valid(vis, H).to(dev)
    n = valid.sum(1)
    row_start = torch.zeros(n.numel() + 1, dtype=torch.int64, device=dev)
    row_start[1:] = torch.cumsum(n, 0)
    nz = valid.nonzero()                       # row-major: environments in order, slots ascending
    return n, row_start, nz[:, 0], nz[:, 1]


class _MaskedForward(object):
    """forward(obs, h, masks) of the base class with the visible mask in place of the prefix mask"""

    def forward(self, obs, h, masks):
        self._valid = visible_valid(obs["visible_masks"], obs["spatial_edges"].shape[1])
        return super().forward(obs, h, masks)

    def _len_mask(self, n, H):
        return self._valid.to(n.device)


class PolicyRefUnsorted(_MaskedForward, PolicyRef):
    pass


class PolicyRefNoSelfAttnUnsorted(_MaskedForward, PolicyRefNoSelfAttn):
    pass


class _MaskedStages(object):
    """chain(obs, h, masks) of the base class over the visible-mask layout; o['row_slot'] is the slot of every row"""

    def chain(self, obs, h, masks):
        self._vis = obs["visible_masks"]
        o = super().chain(obs, h, masks)
        o["row_slot"] = self.row_slot
        return o

    def layout(self, detected):
        n, row_start, row_env, self.row_slot = mask_layout(self._vis, self.H, self.dev)
        return n, row_start, row_env

    def gather(self, spatial, row_env):
        return spatial.to(self.dev, torch.float64)[row_env, self.row_slot]


class StagedRefUnsorted(_MaskedStages, StagedRef):
    def embed1(self, spatial, row_start, row_env):
        y, s = self.lin(self.gather(spatial, row_env), self.W1, self.b1)
        return y.clamp_min(0), s


class StagedRefNoSelfAttnUnsorted(_MaskedStages, StagedRefNoSelfAttn):
    def spatial1(self, spatial, row_start, row_env):
        y, s = self.lin(self.gather(spatial, row_env), self.L1, self.bl1)
        return y.clamp_min(0), s
