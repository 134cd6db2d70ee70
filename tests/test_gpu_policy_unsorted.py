"""GPU: the policy on unsorted humans (the reference's args.sort_humans = False, cn_policy_config.visible_masks).

  * cn_policy_act against the reference's own outputs (tests/golden/policy_unsorted_*.npz), both networks, both GEMM
    modes;
  * a mask equal to the detected_human_num prefix gives outputs bitwise equal to a sorted handle's;
  * every stage against fp64 on the engine's own inputs (the checks of tests/test_gpu_policy_stages.py and
    tests/test_gpu_policy_no_self_attn.py over the visible-mask layout) at N = 4096, H = 20 / 50 / 128, with random
    masks that include all-false and all-true rows, and cn_policy_last_rows;
  * CN_PDL=0 gives bit-identical outputs under CN_ATTN_R=2 and CN_FUSE_QKV=1, CN_ATTN_R=2 the default's bits;
  * evaluate_actions with the update kernels on and off; a rollout on CrowdSimVarNum-v0 with sort_humans = False
    followed by a PPO.update; the environment against the unsorted recordings; the batched evaluation against the
    sequential one; the GST wrapper's outputs (sorted rows, id-ordered masks) through the masked handle, recorded and
    live (make_vec_envs(pretext_wrapper=True) driven by Policy.act)."""
import types

import numpy as np
import pytest
import torch

from tests.policy_stages import read_buffer
from tests.policy_unsorted_ref import (PolicyRefNoSelfAttnUnsorted, PolicyRefUnsorted, StagedRefNoSelfAttnUnsorted,
                                      StagedRefUnsorted, mask_layout)
from tests.test_gpu_policy_stages import E2E, Checker, _env, _run
from tests.test_policy_unsorted import FIXTURES, load_unsorted_golden, oracle_for

pytestmark = pytest.mark.gpu


def _handle(N, H, Win, sd, mode=1, self_attn=True, visible_masks=True):
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy
    pol = CudaPolicy(N, H, Win, device="cuda:0", gemm_mode=mode, self_attn=self_attn, visible_masks=visible_masks)
    pol.load_state_dict(sd)
    return pol


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("name", sorted(FIXTURES))
def test_act_matches_reference_fixture(name, mode):
    g, obs, h, masks = load_unsorted_golden(name)
    N, H, Win = obs["spatial_edges"].shape
    pol = _handle(N, H, Win, oracle_for(name).state_dict(), mode, self_attn="_nsa_" not in name)
    out = _run(pol, obs, h, masks)
    for k, want in (("value", g["synth_value"]), ("mean", g["synth_mean"]), ("h_out", g["synth_h"])):
        err = float((out[k].cpu().double() - torch.from_numpy(want).double()).abs().max())
        assert err < 1e-4, (name, mode, k, err)
    n = mask_layout(obs["visible_masks"], H)[0]
    assert pol.lib.cn_policy_last_rows(pol._h) == int(n.sum())
    pol.close()


def test_missing_mask_pointer_is_a_named_error():
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    pol = _handle(4, 5, 2, make_reference_like_state_dict(2))
    obs = dict(robot_node=torch.zeros(4, 1, 7), temporal_edges=torch.zeros(4, 1, 2), spatial_edges=torch.zeros(4, 5, 2),
               detected_human_num=torch.ones(4, 1))
    with pytest.raises(KeyError):
        pol.act({k: v.cuda() for k, v in obs.items()}, torch.zeros(4, 1, 128).cuda(), torch.ones(4, 1).cuda())
    import ctypes as C
    from crowdnav_prediction_attngraph_b200 import _capi
    t = {k: v.cuda() for k, v in obs.items()}
    o = torch.zeros(4, 256).cuda()
    ptrs = _capi.CnActPtrs(t["robot_node"].data_ptr(), t["temporal_edges"].data_ptr(), t["spatial_edges"].data_ptr(),
                           t["detected_human_num"].data_ptr(), o.data_ptr(), o.data_ptr(), None, o.data_ptr(),
                           o.data_ptr(), o.data_ptr(), o.data_ptr(), o.data_ptr(), None)
    assert pol.lib.cn_policy_act(pol._h, C.byref(ptrs), _capi.raw_stream(0)) != 0
    assert b"visible_masks is NULL" in pol.lib.cn_last_error()
    pol.close()


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("self_attn", [True, False])
@pytest.mark.parametrize("N,H", [(4096, 20), (300, 50)])
def test_prefix_mask_is_bitwise_the_sorted_handle(N, H, self_attn, mode):
    """The only change is the row selection: with the prefix as the mask, every output bit is the sorted handle's."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    sd = make_reference_like_state_dict(12, seed=5, self_attn=self_attn)
    gen = torch.Generator().manual_seed(N + H)
    n = torch.randint(0, H + 1, (N, 1), generator=gen).float()
    vis = torch.arange(H)[None, :] < n
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=gen) * 3, temporal_edges=torch.randn(N, 1, 2, generator=gen),
               spatial_edges=torch.randn(N, H, 12, generator=gen) * 3, detected_human_num=n, visible_masks=vis)
    h = torch.randn(N, 1, 128, generator=gen) * 0.5
    masks = (torch.rand(N, 1, generator=gen) > 0.1).float()
    outs = []
    for vm in (False, True):
        pol = _handle(N, H, 12, sd, mode, self_attn, visible_masks=vm)
        outs.append(_run(pol, obs, h, masks))
        outs[-1]["rows"] = pol.lib.cn_policy_last_rows(pol._h)
        pol.close()
    assert outs[0]["rows"] == outs[1]["rows"] == int(n.clamp(1, H).sum())
    for k in ("value", "mean", "h_out"):
        assert torch.equal(outs[0][k], outs[1][k]), k


def _mask_inputs(N, H, Win, gen):
    p = torch.rand(N, 1, generator=gen)
    vis = torch.rand(N, H, generator=gen) < p
    vis[::9] = False                       # nobody visible: slot 0 only
    vis[4::9] = True                       # everybody visible
    sp = torch.randn(N, H, Win, generator=gen) * 3
    sp[~vis] = 15.0
    obs = dict(robot_node=torch.randn(N, 1, 7, generator=gen) * 3, temporal_edges=torch.randn(N, 1, 2, generator=gen),
               spatial_edges=sp, detected_human_num=torch.randint(0, H + 1, (N, 1), generator=gen).float(),
               visible_masks=vis)
    masks = (torch.rand(N, 1, generator=gen) > 0.1).float()
    return obs, masks


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("self_attn", [True, False])
@pytest.mark.parametrize("H", [20, 50, 128])
def test_stages_match_fp64(H, self_attn, mode, monkeypatch):
    """Three consecutive act calls per handle at N = 4096; every stage against fp64 on the engine's own inputs, the
    row layout (row_start, row_env, row_slot, mc, cn_policy_last_rows) exactly, the outputs against the masked oracle
    in fp64."""
    from tests.test_gpu_policy_no_self_attn import _check_call as check_nsa
    from tests.test_gpu_policy_stages import _check_call as check_full
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    N, Win = 4096, 12
    _env(monkeypatch, {})
    seed = 31 * H + (0 if self_attn else 1)
    sd = make_reference_like_state_dict(Win, seed=seed, self_attn=self_attn)
    sd["dist.fc_mean.bias"] = torch.tensor([0.3, -0.2])
    sd["base.critic_linear.bias"] = torch.tensor([0.7])
    pol = _handle(N, H, Win, sd, mode, self_attn)
    sref = (StagedRefUnsorted if self_attn else StagedRefNoSelfAttnUnsorted)(sd, H, device="cuda")
    oracle = PolicyRefUnsorted(Win) if self_attn else PolicyRefNoSelfAttnUnsorted(Win)
    oracle.load_state_dict(sd)
    oracle = oracle.double().cuda()
    chk = Checker("unsorted/%d/%s/%d" % (mode, "full" if self_attn else "nsa", H))
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(N, 1, 128, generator=gen) * 0.5
    for it in range(3):
        obs, masks = _mask_inputs(N, H, Win, gen)
        outs = _run(pol, obs, h, masks)
        sref._vis = obs["visible_masks"]
        if self_attn:
            check_full(chk, sref, pol, mode, False, obs, h, masks, outs, it == 0)
        else:
            check_nsa(chk, sref, pol, mode, obs, h, masks, outs)
        n, row_start, row_env, row_slot = mask_layout(obs["visible_masks"], H, "cuda")
        Mc = int(row_start[-1])
        assert torch.equal(read_buffer(pol, "row_slot", Mc).val, row_slot)
        assert pol.lib.cn_policy_last_rows(pol._h) == Mc
        dobs = {k: v.cuda() if k == "visible_masks" else v.cuda().double() for k, v in obs.items()}
        with torch.no_grad():
            rv, rm, rh = oracle(dobs, h.cuda().double(), masks.cuda().double())
        for name, got, want in (("value", outs["value"], rv), ("mean", outs["mean"], rm),
                                ("h1", outs["h_out"].reshape(N, 128), rh.reshape(N, 128))):
            scale = max(1.0, float(want.abs().max())) if name == "value" else 1.0
            err = float((got.double() - want).abs().max()) / scale
            assert err < E2E, (chk.tag, it, name, err)
        h = outs["h_out"].cpu()
    print("\nSTAGE-C %s %s" % (chk.tag, " ".join("%s=%.3g" % kv for kv in sorted(chk.worst.items()))))
    pol.close()


@pytest.mark.parametrize("env", [{}, {"CN_ATTN_R": "2"}, {"CN_FUSE_QKV": "1"}])
def test_switches(env, monkeypatch):
    """Under each attention switch: CN_PDL=0 is bit-identical, a prefix mask is bit-identical to the sorted handle, and
    the outputs are the default's (CN_ATTN_R=2: bit for bit; CN_FUSE_QKV=1, a kernel of its own: within 1e-5)."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    N, H = 2048, 50
    sd = make_reference_like_state_dict(12, seed=3)
    obs, masks = _mask_inputs(N, H, 12, torch.Generator().manual_seed(9))
    h = torch.randn(N, 1, 128, generator=torch.Generator().manual_seed(10)) * 0.5

    def run(e, o=obs, vm=True):
        _env(monkeypatch, e)
        pol = _handle(N, H, 12, sd, visible_masks=vm)
        out = _run(pol, o, h, masks)
        pol.close()
        return out
    default, base, pdl_off = run({}), run(env), run(dict(env, CN_PDL="0"))
    cnt = obs["visible_masks"].sum(1, keepdim=True)
    prefix_obs = dict(obs, detected_human_num=cnt.float(), visible_masks=torch.arange(H)[None, :] < cnt)
    prefix, sorted_ = run(env, prefix_obs), run(env, prefix_obs, vm=False)
    for k in base:
        assert torch.equal(base[k], pdl_off[k]), (env, k)
        assert torch.equal(prefix[k], sorted_[k]), (env, k)
        if "CN_FUSE_QKV" in env:
            err = float((base[k] - default[k]).abs().max()) / max(1.0, float(default[k].abs().max()))
            assert err < 1e-5, (k, err)
        else:
            assert torch.equal(base[k], default[k]), (env, k)


def _args(**kw):
    a = dict(num_processes=8, seq_length=30, num_mini_batch=2, sort_humans=False)
    a.update(kw)
    return types.SimpleNamespace(**a)


def _spaces(H, W):
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    return {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
            'detected_human_num': Box((1,)), 'visible_masks': Box((H,), np.bool_)}


@pytest.mark.parametrize("self_attn", [True, False])
def test_evaluate_actions_update_kernels_on_and_off(self_attn):
    """The update path with the tensor-core update kernels against plain torch on the device and against fp64."""
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    T, N, H, W = 30, 8, 20, 12
    gen = torch.Generator().manual_seed(4)
    obs, _ = _mask_inputs(T * N, H, W, gen)
    masks = (torch.rand(T * N, 1, generator=gen) > 0.05).float()
    act = torch.randn(T * N, 2, generator=gen)
    h0 = torch.randn(N, 1, 128, generator=gen) * 0.5
    pol = Policy(_spaces(H, W), Box((2,)), base='selfAttn_merge_srnn', base_kwargs=_args(use_self_attn=self_attn)).cuda()
    d = {k: v.cuda() for k, v in obs.items()}
    res = {}
    for uk in (True, False):
        pol.update_kernels = uk
        pol.zero_grad()
        v, lp, ent, hx = pol.evaluate_actions(d, {'human_node_rnn': h0.cuda()}, masks.cuda(), act.cuda())
        (v.mean() + lp.mean() + ent).backward()
        res[uk] = (v.detach(), lp.detach(), hx['human_node_rnn'].detach(),
                   {k: p.grad.clone() for k, p in pol.named_parameters() if p.grad is not None})
    import copy
    p64 = copy.deepcopy(pol).double()
    p64.update_kernels = False
    d64 = {k: v if k == "visible_masks" else v.double() for k, v in d.items()}
    with torch.no_grad():
        v64, lp64, _, hx64 = p64.evaluate_actions(d64, {'human_node_rnn': h0.cuda().double()}, masks.cuda().double(),
                                                  act.cuda().double())
    for uk in (True, False):
        v, lp, hh, _ = res[uk]
        assert float((v.double() - v64).abs().max()) < 1e-3 * max(1.0, float(v64.abs().max())), uk
        assert float((hh.double() - hx64['human_node_rnn']).abs().max()) < 1e-4, uk
    for k, g in res[False][3].items():
        gk = res[True][3][k]
        assert float((gk - g).abs().max()) <= 1e-3 * max(1e-3, float(g.abs().max())), k


def _varnum_config(H=20, rng=0):
    ns = types.SimpleNamespace
    return ns(sim=ns(human_num=H, human_num_range=rng, predict_steps=5, predict_method="none",
                     circle_radius=6 * 2 ** 0.5, arena_size=6),
              action_space=ns(kinematics="holonomic"), humans=ns(policy="orca", radius=0.3, v_pref=1, FOV=2.0,
                                                                random_goal_changing=True, goal_change_chance=0.5,
                                                                end_goal_changing=True),
              robot=ns(visible=False, radius=0.3, v_pref=1, FOV=2, sensor_range=5, policy="selfAttn_merge_srnn"),
              env=ns(randomize_attributes=True, time_step=0.25, time_limit=50, val_size=100, test_size=500),
              data=ns(pred_timestep=0.25),
              reward=ns(discomfort_dist=0.25, discomfort_penalty_factor=10, success_reward=10, collision_penalty=-20),
              orca=ns(neighbor_dist=10, safety_space=0.15, time_horizon=5), sf=ns(A=2.0, B=1.0, KI=1.0),
              args=ns(sort_humans=False))


def test_rollout_then_ppo_update_on_varnum():
    """A device-resident rollout of CrowdSimVarNum-v0 with sort_humans = False into RolloutStorage, every act masked by
    the environment's visible_masks, then one PPO.update; the masked handle's values match the update path's."""
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.ppo import PPO
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200.vec_env import make_vec_envs
    T, N = 30, 16
    env = make_vec_envs("CrowdSimVarNum-v0", 7, N, 0.99, None, "cuda:0", False, config=_varnum_config())
    assert env.cfgd["sort_humans"] == 0
    torch.manual_seed(0)
    pol = Policy(env.observation_space.spaces, env.action_space, base='selfAttn_merge_srnn',
                 base_kwargs=_args(num_processes=N)).cuda()
    ro = RolloutStorage(T, N, env.observation_space.spaces, env.action_space, 128, 256, device="cuda")
    obs = env.reset()
    for k in ro.obs:
        ro.obs[k][0].copy_(obs[k])
    non_prefix = 0
    for t in range(T):
        with torch.no_grad():
            o = {k: ro.obs[k][t] for k in ro.obs}
            hx = {k: ro.recurrent_hidden_states[k][t] for k in ro.recurrent_hidden_states}
            value, action, logp, hx2 = pol.act(o, hx, ro.masks[t])
        vis = o["visible_masks"]
        cnt = vis.sum(1, keepdim=True)
        non_prefix += int((vis != (torch.arange(vis.shape[1], device=vis.device)[None] < cnt)).any(1).sum())
        obs, rew, done, infos = env.step(action)
        m = torch.from_numpy(1.0 - done.astype(np.float32)).unsqueeze(1).cuda()
        ro.insert(obs, hx2, action, logp, value, rew.cuda(), m, torch.ones(N, 1, device="cuda"))
    assert non_prefix > 0
    with torch.no_grad():
        nv = pol.get_value({k: ro.obs[k][-1] for k in ro.obs},
                           {k: ro.recurrent_hidden_states[k][-1] for k in ro.recurrent_hidden_states}, ro.masks[-1])
    ro.compute_returns(nv, True, 0.99, 0.95, False)
    # the rollout's values and log-probs are what evaluate_actions computes on the same inputs
    adv = ro.returns[:-1] - ro.value_preds[:-1]
    batch = next(iter(ro.recurrent_generator(adv, 1)))
    obs_b, hxs_b, act_b, vpred_b, _, masks_b, old_lp_b, _ = batch
    with torch.no_grad():
        v, lp, _, _ = pol.evaluate_actions(obs_b, hxs_b, masks_b, act_b)
    assert float((v - vpred_b).abs().max()) < 2e-3 * max(1.0, float(vpred_b.abs().max()))
    assert float((lp - old_lp_b).abs().max()) < 2e-3
    agent = PPO(pol, clip_param=0.2, ppo_epoch=2, num_mini_batch=2, value_loss_coef=0.5, entropy_coef=0.01, lr=4e-5,
                eps=1e-5, max_grad_norm=0.5)
    before = {k: p.detach().clone() for k, p in pol.named_parameters()}
    losses = agent.update(ro)
    assert all(np.isfinite(x) for x in losses)
    assert any(not torch.equal(before[k], p) for k, p in pol.named_parameters())
    env.close()


@pytest.mark.parametrize("name", ["env_varnum_h20_unsorted_rand", "env_varnum_h6_range2_unsorted"])
def test_env_matches_unsorted_reference_rollout(name):
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    from tests.golden_util import load_env_case, replay
    g, case, over = load_env_case(name)
    env = CudaCrowdVecEnv(device="cuda:0", sort_humans=0, **over)
    np_obs = lambda obs: {k: v.cpu().numpy() for k, v in obs.items()}

    def step(a):
        obs, rew, done, info = env.step_device(torch.from_numpy(a).cuda())
        out = dict(reward=rew.cpu().numpy(), done=done.cpu().numpy(), info=info.cpu().numpy(),
                   info_aux=env._out["info_aux"].cpu().numpy())
        return np_obs(obs), out

    bad = replay(g, case, lambda: np_obs(env.reset()), step, env.get_state, pos_tol=1e-9)
    assert not bad, bad[:5]
    env.close()


def test_batched_evaluation_equals_sequential_protocol():
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    from crowdnav_prediction_attngraph_b200.policy import Policy, make_reference_like_state_dict
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    test_size = 5
    d = _capi.default_config_dict(num_envs=1, nenv_total=1, seed=19, human_num=20, phase=2, test_size=test_size,
                                  time_limit=20.0, const_vel=0, sort_humans=0)
    env = CudaCrowdVecEnv(device="cuda:0", cfg=d)
    pol = Policy(env.observation_space.spaces, env.action_space, base='selfAttn_merge_srnn',
                 base_kwargs=_args(num_processes=1)).cuda()
    pol.load_state_dict(make_reference_like_state_dict(2, seed=5))
    seq = evaluate(pol, env, 1, torch.device("cuda:0"), test_size, None, None, None)
    env.close()
    bat = evaluate_batched(pol, None, "CrowdSimVarNum-v0", 19, test_size, torch.device("cuda:0"), cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    for k in ("success_rate", "collision_rate", "timeout_rate", "collision_cases", "timeout_cases"):
        assert seq[k] == bat[k], k
    for k in ("avg_nav_time", "path_length", "intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k


def test_gst_wrapper_outputs_through_masked_handle():
    """The GST wrapper's observation (rows sorted by distance, masks in id order) masks by id: the engine's handle on
    the recorded wrapper outputs equals the reference's module (policy_unsorted_full_h50), and differs from the
    detected_human_num prefix."""
    name = "policy_unsorted_full_h50"
    g, obs, h, masks = load_unsorted_golden(name)
    N, H, Win = obs["spatial_edges"].shape
    sd = oracle_for(name).state_dict()
    pol = _handle(N, H, Win, sd)
    out = _run(pol, obs, h, masks)
    pol.close()
    assert float((out["value"].cpu().double() - torch.from_numpy(g["synth_value"]).double()).abs().max()) < 1e-4
    pol = _handle(N, H, Win, sd, visible_masks=False)
    prefix = _run(pol, obs, h, masks)
    pol.close()
    assert float((prefix["value"] - out["value"]).abs().max()) > 1e-3


def test_gst_wrapper_end_to_end_act():
    """make_vec_envs(..., pretext_wrapper=True) with args.sort_humans = False driven by Policy.act: on the wrapper's live
    observations (rows sorted by distance, masks in id order) every step's value, action mean and hidden state equal
    the masked oracle in fp64, and the observations hold masks that are not the detected_human_num prefix."""
    import os
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.vec_env import make_vec_envs
    from oracle.policy_ref import PolicyRef
    N, steps = 64, 25
    params = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gst_params.npz")))
    env = make_vec_envs("CrowdSimPredRealGST-v0", 11, N, 0.99, None, "cuda:0", False, config=_varnum_config(),
                        pretext_wrapper=True, gst_params=params)
    torch.manual_seed(3)
    pol = Policy(env.observation_space.spaces, env.action_space, base='selfAttn_merge_srnn',
                 base_kwargs=_args(num_processes=N)).cuda()
    H, Win = env.observation_space.spaces['spatial_edges'].shape
    ref, ref_prefix = PolicyRefUnsorted(Win), PolicyRef(Win)
    keep = {k: v for k, v in pol.state_dict().items() if k in ref.state_dict()}
    ref.load_state_dict(keep)
    ref_prefix.load_state_dict(keep)
    ref, ref_prefix = ref.double().cuda(), ref_prefix.double().cuda()
    obs = env.reset()
    hx = {'human_node_rnn': torch.zeros(N, 1, 128, device="cuda"),
          'human_human_edge_rnn': torch.zeros(N, H + 1, 256, device="cuda")}
    masks = torch.zeros(N, 1, device="cuda")
    non_prefix, prefix_gap = 0, 0.0
    for t in range(steps):
        dobs = {k: v if k == "visible_masks" else v.double() for k, v in obs.items()}
        with torch.no_grad():
            rv, rm, rh = ref(dobs, hx['human_node_rnn'].double(), masks.double())
            pv = ref_prefix(dict(dobs, detected_human_num=dobs["detected_human_num"].clamp(1, H)),
                            hx['human_node_rnn'].double(), masks.double())[0]
            value, action, _, hx = pol.act(obs, hx, masks, deterministic=True)
        assert float((value.double() - rv).abs().max()) < 1e-4 * max(1.0, float(rv.abs().max())), t
        assert float((action.double() - rm).abs().max()) < 1e-4, t
        assert float((hx['human_node_rnn'].double() - rh).abs().max()) < 1e-4, t
        prefix_gap = max(prefix_gap, float((pv - rv).abs().max()))
        vis = obs["visible_masks"]
        cnt = vis.sum(1, keepdim=True)
        non_prefix += int((vis != (torch.arange(H, device=vis.device)[None] < cnt)).any(1).sum())
        obs, _, done, _ = env.step(action)
        masks = torch.from_numpy(1.0 - done.astype(np.float32)).unsqueeze(1).cuda()
    assert non_prefix > 0
    assert prefix_gap > 1e-3
    env.close()
