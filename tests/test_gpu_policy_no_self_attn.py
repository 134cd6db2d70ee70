"""GPU: the policy without human-human attention (the reference's use_self_attn = False, cn_policy_config.no_self_attn).

  * cn_policy_act against the reference's own outputs (tests/golden/policy_nsa_*.npz) in both GEMM modes;
  * every stage against fp64 on the engine's own inputs (the bounds and helpers of tests/test_gpu_policy_stages.py:
    layer 1 carries the CUDA-core embed1 constant, layer 2 the constant of the other K = 128 per-human GEMM, embed2),
    three consecutive calls per handle, at the edge shapes;
  * CN_PDL=0, CN_FUSE_QKV=1 and CN_ATTN_R=2 give bit-identical results;
  * the update path with and without the update kernels against fp64, a rollout into RolloutStorage followed by a
    PPO.update, the batched evaluation, and a checkpoint round trip."""
import copy
import io

import numpy as np
import pytest
import torch

from tests.policy_fixture import load_policy_golden
from tests.policy_no_self_attn_ref import PolicyRefNoSelfAttn, StagedRefNoSelfAttn, synth_state_dict_nsa
from tests.policy_stages import Buf, buffer_info, read_buffer
from tests.test_gpu_policy_stages import C_F32, C_GRU, C_HR, C_TANH, C_TC, E2E, Checker, _env, _inputs, _run, _split16

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _handle(N, H, Win, sd, mode=1):
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy
    pol = CudaPolicy(N, H, Win, device="cuda:0", gemm_mode=mode, self_attn=False)
    pol.load_state_dict(sd)
    return pol


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("name,Win", [("policy_nsa_h20", 12), ("policy_nsa_h50", 12), ("policy_nsa_varnum", 2)])
def test_act_matches_reference_fixture(name, Win, mode):
    g, obs, h, masks = load_policy_golden(name)
    sd = synth_state_dict_nsa(PolicyRefNoSelfAttn(Win).state_dict())
    N, H = obs["spatial_edges"].shape[:2]
    pol = _handle(N, H, Win, sd, mode)
    out = _run(pol, obs, h, masks)
    for k, want in (("value", g["synth_value"]), ("mean", g["synth_mean"]), ("h_out", g["synth_h"])):
        err = float((out[k].cpu().double() - torch.from_numpy(want).double()).abs().max())
        assert err < 1e-4, (name, mode, k, err)
    pol.close()


SHAPES = {   # name: (N, H, Win, pattern of n), as tests/test_gpu_policy_stages.py
    "n1": (1, 1, 12, "one"),
    "h128": (3, 128, 12, [128, 1, 128]),
    "varnum": (70, 5, 2, "random"),
    "clamp": (300, 20, 12, "clamp"),
    "n4096_h20": (4096, 20, 12, "half1"),
    "n4096_h50": (4096, 50, 12, "half1"),
    "n4096_h100": (4096, 100, 12, "half1"),
}


def _check_call(chk, sref, pol, mode, obs, h, masks, outs):
    tc = mode == 1
    f = lambda t: t.to("cuda", torch.float64)
    N = pol.N
    torch.cuda.synchronize()
    n, row_start, row_env = sref.layout(obs["detected_human_num"])
    Mc = int(row_start[-1])
    B = lambda name, rows=None: read_buffer(pol, name, rows)
    assert torch.equal(B("row_start").val, row_start) and int(B("mc").val[0]) == Mc
    assert torch.equal(B("row_env", Mc).val, row_env)
    CL = C_TC if tc else C_F32
    for name in ("e2", "qkv", "ao", "Wqkv", "Wos"):
        with pytest.raises(RuntimeError, match="does not exist"):
            buffer_info(pol, name)
    e1 = B("e1", Mc)
    chk.stage("spatial1", e1, *sref.spatial1(f(obs["spatial_edges"]), row_start, row_env), C_F32["e1"])
    sout = B("sout", Mc)
    chk.stage("spatial2", sout, *sref.spatial2(e1.val), CL["e2"])
    rs = B("rs")
    chk.stage("rs", rs, *sref.robot(sref.robot_input(f(obs["robot_node"]), f(obs["temporal_edges"]))), C_F32["rs"])
    t1 = B("t1")
    ref_t1, sc_t1 = sref.enc_te(rs.val)
    if tc:
        t1f = B("t1.f32")
        chk.stage("t1", t1f, ref_t1, sc_t1, CL["t1"])
        te_hr = t1f.val[:, 64:]
        hi, lo = _split16(t1f.raw[:, 64:])
        te_u = hi.double() + lo.double()
    else:
        chk.stage("t1", t1.val[:, :64], ref_t1[:, :64], sc_t1[:, :64], CL["t1"])
        te_hr = te_u = ref_t1[:, 64:]
    u = B("u")
    chk.stage("u", u, *sref.u(te_u), CL["u"])
    wv = B("wv")
    wv_ref, _, smax = sref.hr_attention(sout.val, u.val, te_hr, n, row_start)
    chk.stage("hr_attn", wv, wv_ref, smax[:, None].expand_as(wv_ref), C_HR)
    emb_ref, emb_sc = sref.emb(wv.val)
    if tc:
        chk.stage("emb", Buf(t1.val[:, 64:], t1.hi[:, 64:], t1.lo[:, 64:]), emb_ref, emb_sc, CL["emb"])
    else:
        chk.stage("emb", t1.val[:, 64:], emb_ref, emb_sc, CL["emb"])
    gi = B("gi")
    chk.stage("gi", gi, *sref.gi(t1.val), CL["gi"])
    h0 = B("h0")
    h0f = B("h0.f32") if tc else h0
    assert torch.equal(h0f.raw, (h.reshape(N, 128).float() * masks.reshape(N, 1).float()).cuda())
    gh = B("gh")
    chk.stage("gh", gh, *sref.gh(h0.val), CL["gh"])
    h_out = outs["h_out"].reshape(N, 128)
    chk.stage("gru", h_out, sref.gru(gi.val, gh.val, h0f.val)[0], torch.ones(N, 128, device="cuda", dtype=torch.float64),
              C_GRU)
    h1_in = B("h1").val if tc else h_out.double()
    ac1 = B("ac1")
    chk.stage("ac1", ac1, *sref.ac1(h1_in), CL["ac1"], C_TANH)
    a2, c2 = B("a2"), B("c2")
    chk.stage("a2", a2, *sref.a2(ac1.val[:, :256]), CL["a2"], C_TANH)
    chk.stage("c2", c2, *sref.c2(ac1.val[:, 256:]), CL["c2"], C_TANH)
    chk.stage("value", outs["value"], *sref.value(c2.val), C_F32["value"])
    chk.stage("mean", outs["mean"], *sref.mean(a2.val), C_F32["mean"])


@pytest.mark.parametrize("mode", [1, 0])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_stages_match_fp64(shape, mode, monkeypatch):
    """Three consecutive act calls per handle; every stage against fp64 on the engine's own inputs, the outputs against
    PolicyRefNoSelfAttn in fp64."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    N, H, Win, pattern = SHAPES[shape]
    _env(monkeypatch, {})
    seed = 17 * N + H
    sd = make_reference_like_state_dict(Win, seed=seed, self_attn=False)
    sd["dist.fc_mean.bias"] = torch.tensor([0.3, -0.2])
    sd["base.critic_linear.bias"] = torch.tensor([0.7])
    sd["base.spatial_linear.0.bias"] = torch.linspace(-0.3, 0.3, 128)
    sd["base.spatial_linear.2.bias"] = torch.linspace(-0.2, 0.2, 256)
    pol = _handle(N, H, Win, sd, mode)
    sref = StagedRefNoSelfAttn(sd, H, device="cuda")
    oracle = PolicyRefNoSelfAttn(Win)
    oracle.load_state_dict(sd)
    oracle = oracle.double().cuda()
    chk = Checker("nsa/%d/%s" % (mode, shape))
    gen = torch.Generator().manual_seed(seed)
    h = torch.randn(N, 1, 128, generator=gen) * 0.5
    for it in range(3):
        obs, masks = _inputs(N, H, Win, pattern, gen, it)
        outs = _run(pol, obs, h, masks)
        _check_call(chk, sref, pol, mode, obs, h, masks, outs)
        dobs = {k: v.cuda().double() for k, v in obs.items()}
        dobs["detected_human_num"] = dobs["detected_human_num"].clamp(1, H)
        with torch.no_grad():
            rv, rm, rh = oracle(dobs, h.cuda().double(), masks.cuda().double())
        for name, got, want in (("value", outs["value"], rv), ("mean", outs["mean"], rm),
                                ("h1", outs["h_out"].reshape(N, 128), rh.reshape(N, 128))):
            scale = max(1.0, float(want.abs().max())) if name == "value" else 1.0
            err = float((got.double() - want).abs().max()) / scale
            chk.worst["e2e_" + name] = max(chk.worst.get("e2e_" + name, 0.0), err)
            assert err < E2E, (chk.tag, it, name, err)
        if pattern == "clamp":
            again = _run(pol, dict(obs, detected_human_num=obs["detected_human_num"].clamp(1, H)), h, masks)
            for k in again:
                assert torch.equal(again[k], outs[k]), k
        h = outs["h_out"].cpu()
    print("\nSTAGE-C %s %s" % (chk.tag, " ".join("%s=%.3g" % kv for kv in sorted(chk.worst.items()))))
    pol.close()


_BUFFERS = ["row_start", "row_env", "mc", "e1", "sout", "rs", "t1", "u", "wv", "h0", "gi", "gh", "h1", "ac1", "a2", "c2"]


def test_pdl_off_and_attention_switches_are_bit_identical(monkeypatch):
    """CN_PDL=0 launches the same kernels without programmatic dependent launch, and the human-human attention
    switches (CN_FUSE_QKV=1, CN_ATTN_R=2, CN_QKV_CHUNKS=2) have nothing to act on: every buffer and output of each is
    bit-identical to the default."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    N, H, Win = 4096, 50, 12
    sd = make_reference_like_state_dict(Win, seed=77, self_attn=False)
    pols = []
    for env in ({}, {"CN_PDL": "0"}, {"CN_FUSE_QKV": "1"}, {"CN_ATTN_R": "2"}, {"CN_QKV_CHUNKS": "2"}):
        _env(monkeypatch, env)
        pols.append(_handle(N, H, Win, sd))
    gen = torch.Generator().manual_seed(5)
    h = torch.randn(N, 1, 128, generator=gen) * 0.5
    for it in range(3):
        obs, masks = _inputs(N, H, Win, "half1", gen, it)
        outs = [_run(p, obs, h, masks) for p in pols]
        Mc = int(read_buffer(pols[0], "mc", device="cpu").val[0])
        for i in range(1, len(pols)):
            for k in outs[0]:
                assert torch.equal(outs[0][k], outs[i][k]), (i, it, k)
            for name in _BUFFERS:
                rows = Mc if name in ("row_env", "e1", "sout") else None
                a, b = (read_buffer(p, name, rows, device="cpu") for p in (pols[0], pols[i]))
                if a.split:
                    assert torch.equal(a.hi, b.hi) and torch.equal(a.lo, b.lo), (i, it, name)
                else:
                    assert torch.equal(a.raw, b.raw), (i, it, name)
        h = outs[0]["h_out"].cpu()
    for p in pols:
        p.close()


def test_missing_key_is_named_and_stages_are_the_ablations():
    from crowdnav_prediction_attngraph_b200.policy import CudaPolicy, make_reference_like_state_dict
    sd = make_reference_like_state_dict(12, seed=1, self_attn=False)
    pol = CudaPolicy(4, 3, 12, device="cuda:0", self_attn=False)
    with pytest.raises(RuntimeError, match="base.spatial_linear.2.weight"):
        pol.load_state_dict({k: v for k, v in sd.items() if k != "base.spatial_linear.2.weight"})
    full = make_reference_like_state_dict(12, seed=1)
    with pytest.raises(RuntimeError, match="base.spatial_linear.0.weight' has 131072 elements, expected 1536"):
        pol.load_state_dict(full)
    pol.load_state_dict(sd)
    pol.profile(True)
    obs, masks = _inputs(4, 3, 12, "random", torch.Generator().manual_seed(0), 0)
    _run(pol, obs, torch.zeros(4, 1, 128), masks)
    ms = pol.stage_ms()
    assert list(ms) == ["pack_inputs", "spatial_linear0", "spatial_linear2", "robot_branch_join", "hr_attention", "gru",
                        "actor_critic_heads"]
    assert all(v >= 0 for v in ms.values())
    pol.close()


def _policy(N, H=20, W=12, **kw):
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.vec_env import Box

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, 30, 2
        use_self_attn = False
    a = Args()
    for k, v in kw.items():
        setattr(a, k, v)
    spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
              'detected_human_num': Box((1,))}
    return Policy(spaces, Box((2,)), base_kwargs=a, base='selfAttn_merge_srnn')


def test_evaluate_actions_kernels_on_equals_off():
    """As tests/test_gpu_update_kernels.py: one minibatch [T=30, N=48] with the update kernels, with plain torch ops and
    in fp64; the kernel path must be as close to fp64 as torch's fp32 path."""
    T, N, H = 30, 48, 20
    torch.manual_seed(3)
    pol = _policy(N, H).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(11)
    B = T * N
    obs = {'robot_node': torch.randn(B, 1, 7, device=DEV, generator=g), 'temporal_edges': torch.randn(B, 1, 2, device=DEV, generator=g),
           'spatial_edges': torch.randn(B, H, 12, device=DEV, generator=g) * 3,
           'detected_human_num': torch.randint(1, H + 1, (B, 1), device=DEV, generator=g).float()}
    hx = torch.randn(N, 1, 128, device=DEV, generator=g) * 0.3
    masks = (torch.rand(B, 1, device=DEV, generator=g) > 0.05).float()
    act = torch.randn(B, 2, device=DEV, generator=g)
    res = {}
    for tag, module, on in (("tc", pol, True), ("torch32", pol, False), ("fp64", copy.deepcopy(pol).double(), False)):
        module.update_kernels = on
        module.zero_grad()
        dt = torch.float64 if tag == "fp64" else torch.float32
        v, lp, ent, _ = module.evaluate_actions(obs, {'human_node_rnn': hx.to(dt)}, masks.to(dt), act.to(dt))
        (0.5 * v.pow(2).mean() - lp.mean() + 0.01 * ent).backward()
        res[tag] = (v.detach().double(), lp.detach().double(), float(ent.detach()),
                    {k: p.grad.double().clone() for k, p in module.named_parameters() if p.grad is not None})
    assert torch.allclose(res["tc"][0], res["fp64"][0], rtol=1e-5, atol=1e-5)
    assert torch.allclose(res["tc"][1], res["fp64"][1], rtol=1e-5, atol=1e-5)
    assert abs(res["tc"][2] - res["fp64"][2]) <= 1e-6
    assert any(k.startswith("base.spatial_linear.2") for k in res["tc"][3])
    report = []
    for k, g64 in res["fp64"][3].items():
        n64 = float(g64.norm())
        if n64 < 1e-12:
            continue
        d_tc64 = float((res["tc"][3][k] - g64).norm()) / n64
        d_3264 = float((res["torch32"][3][k] - g64).norm()) / n64
        d_tc32 = float((res["tc"][3][k] - res["torch32"][3][k]).norm()) / n64
        report.append((d_tc64, d_3264, d_tc32, k))
    report.sort(reverse=True)
    print("relative L2 gradient distances (kernels-fp64, torch32-fp64, kernels-torch32), worst five:", report[:5])
    for d_tc64, d_3264, d_tc32, k in report:
        assert d_tc64 <= max(3 * d_3264, 5e-4), (k, d_tc64, d_3264)
        assert d_tc32 <= max(3 * d_3264, 5e-4), (k, d_tc32, d_3264)


def test_rollout_then_ppo_update():
    """train.py's loop shape with the ablation: act into RolloutStorage, GAE, one PPO.update, and the engine picks up
    the new weights (act == evaluate_actions afterwards)."""
    from crowdnav_prediction_attngraph_b200 import ppo
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    N, steps = 32, 8
    torch.manual_seed(425)
    envs = CudaCrowdVecEnv(num_envs=N, human_num=20, seed=425, device=DEV)
    pol = _policy(N, seq_length=steps).to(DEV)
    pol.seq_length = steps
    ro = RolloutStorage(steps, N, envs.observation_space.spaces, envs.action_space, 128, 256, device=DEV)
    agent = ppo.PPO(pol, 0.2, 2, 2, 0.5, 0.01, lr=4e-5, eps=1e-5, max_grad_norm=0.5)
    obs = envs.reset()
    for k in ro.obs:
        ro.obs[k][0].copy_(obs[k])
    w0 = pol.base.spatial_linear[0].weight.detach().clone()
    for step in range(steps):
        with torch.no_grad():
            o = {k: ro.obs[k][step] for k in ro.obs}
            hx = {k: ro.recurrent_hidden_states[k][step] for k in ro.recurrent_hidden_states}
            value, action, logp, hx2 = pol.act(o, hx, ro.masks[step])
        obs, reward, done, infos = envs.step(action)
        masks = torch.FloatTensor([[0.0] if d else [1.0] for d in done])
        ro.insert(obs, hx2, action, logp, value, reward, masks, torch.ones(N, 1))
    with torch.no_grad():
        o = {k: ro.obs[k][-1] for k in ro.obs}
        hx = {k: ro.recurrent_hidden_states[k][-1] for k in ro.recurrent_hidden_states}
        nv = pol.get_value(o, hx, ro.masks[-1]).detach()
    ro.compute_returns(nv, True, 0.99, 0.95, False)
    losses = agent.update(ro)
    assert np.isfinite(losses).all()
    assert not torch.equal(w0, pol.base.spatial_linear[0].weight.detach())
    with torch.no_grad():
        o = {k: ro.obs[k][0] for k in ro.obs}
        hx = {k: ro.recurrent_hidden_states[k][0] for k in ro.recurrent_hidden_states}
        value, action, logp, _ = pol.act(o, hx, ro.masks[0])
        pol.seq_length = 1
        v2, lp2, _, _ = pol.evaluate_actions(o, hx, ro.masks[0], action)
    assert (value - v2).abs().max() < 2e-4 and (logp - lp2).abs().max() < 2e-4
    envs.close()


def test_batched_evaluation_equals_sequential_protocol():
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    test_size = 5
    d = _capi.default_config_dict(num_envs=1, nenv_total=1, seed=19, human_num=20, phase=2, test_size=test_size,
                                  time_limit=20.0)
    pol = _policy(1).to(DEV)
    pol.load_state_dict(make_reference_like_state_dict(12, seed=5, self_attn=False))
    env = CudaCrowdVecEnv(device=DEV, cfg=d)
    seq = evaluate(pol, env, 1, DEV, test_size, None, None, None)
    env.close()
    bat = evaluate_batched(pol, None, "CrowdSimPred-v0", 19, test_size, DEV, cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    for k in ("success_rate", "collision_rate", "timeout_rate", "collision_cases", "timeout_cases"):
        assert seq[k] == bat[k], k
    for k in ("avg_nav_time", "path_length", "intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k


def test_checkpoint_round_trip():
    """A checkpoint saved by the engine loads into a fresh ablation Policy and gives the same act outputs."""
    from crowdnav_prediction_attngraph_b200.policy import make_reference_like_state_dict
    N, H = 64, 20
    a = _policy(N).to(DEV)
    a.load_state_dict(make_reference_like_state_dict(12, seed=9, self_attn=False))
    buf = io.BytesIO()
    torch.save(a.state_dict(), buf)
    buf.seek(0)
    b = _policy(N).to(DEV)
    b.load_state_dict(torch.load(buf, map_location="cpu", weights_only=True))
    obs, masks = _inputs(N, H, 12, "random", torch.Generator().manual_seed(2), 0)
    obs = {k: v.to(DEV) for k, v in obs.items()}
    hx = {'human_node_rnn': torch.randn(N, 1, 128, device=DEV) * 0.5}
    with torch.no_grad():
        ra = [t.clone() for t in a.act(obs, hx, masks.to(DEV), deterministic=True)[:3]]
        rb = [t.clone() for t in b.act(obs, hx, masks.to(DEV), deterministic=True)[:3]]
    for x, y in zip(ra, rb):
        assert torch.equal(x, y)
