"""GPU: the DS-RNN policy forward (cn_dsrnn, base='srnn') against the unmodified reference's outputs
(tools/make_golden_dsrnn.py) and the fp32 oracle (oracle/dsrnn_ref.py), its zero edge state, sampling, one training
iteration of the train.py contract, and the batched evaluation."""
import numpy as np
import pytest
import torch

from oracle.dsrnn_ref import DsrnnRef
from tests.dsrnn_fixture import ACT_CASES, OBS_KEYS, UNUSED, Args, act_case, dsrnn_state_dict, recurrent_case, spaces

pytestmark = pytest.mark.gpu
TOL = 1e-4
DEV = "cuda:0"


def _engine(N, H, W):
    from crowdnav_prediction_attngraph_b200.policy import CudaDsrnn
    eng = CudaDsrnn(N, H, W, device=DEV)
    ref = DsrnnRef(W)
    sd = dsrnn_state_dict(ref.state_dict())
    ref.load_state_dict(sd)
    eng.load_state_dict(sd)
    return eng, ref


def _cuda(d):
    return {k: v.to(DEV) for k, v in d.items()}


def _check(got, want, what):
    for g, w, name in zip(got, want, ("value", "mean", "node state", "edge state")):
        err = float(np.abs(g.detach().cpu().numpy() - np.asarray(w)).max())
        assert err <= TOL, "%s %s: max abs error %.3g" % (what, name, err)


@pytest.mark.parametrize("tag", sorted(ACT_CASES))
def test_act_matches_reference_fixture(tag):
    H, W = ACT_CASES[tag]
    obs, ins, outs = act_case(tag)
    eng, _ = _engine(obs["spatial_edges"].shape[0], H, W)
    v, a, lp, h1, he1, m = eng.act(_cuda(obs), ins["h"].to(DEV), ins["he"].to(DEV), ins["masks"].to(DEV),
                                   deterministic=True, return_mean=True)
    _check((v, m, h1, he1), (outs["value"], outs["mean"], outs["h1"], outs["he1"]), tag)
    assert torch.equal(a, m)


@pytest.mark.parametrize("W", [2, 12])
@pytest.mark.parametrize("H", [5, 20, 50])
def test_act_matches_oracle_ragged_n(H, W):
    N = 300                                   # not a multiple of the 128-row tiles
    g = torch.Generator().manual_seed(H * 100 + W)
    obs = {"robot_node": torch.randn(N, 1, 7, generator=g) * 3, "temporal_edges": torch.randn(N, 1, 2, generator=g),
           "spatial_edges": torch.randn(N, H, W, generator=g) * 4,
           "detected_human_num": torch.randint(1, H + 1, (N, 1), generator=g).float()}
    h = torch.randn(N, 1, 128, generator=g) * 0.5
    he = torch.randn(N, H + 1, 256, generator=g) * 0.5
    masks = (torch.rand(N, 1, generator=g) > 0.2).float()
    eng, ref = _engine(N, H, W)
    with torch.no_grad():
        want = ref(obs, h, he, masks)
    v, a, lp, h1, he1, m = eng.act(_cuda(obs), h.to(DEV), he.to(DEV), masks.to(DEV), deterministic=True,
                                   return_mean=True)
    _check((v, m, h1, he1), [x.numpy() for x in want], "H=%d W=%d" % (H, W))


def test_recurrent_run_feeds_back_its_own_states():
    g = recurrent_case()
    T, N = g["masks"].shape[:2]
    H = g["ob_spatial_edges"].shape[2]
    eng, _ = _engine(N, H, 2)
    h = torch.zeros(N, 1, 128, device=DEV)
    he = None
    for t in range(T):
        obs = {k: torch.from_numpy(g["ob_" + k][t]).to(DEV) for k in OBS_KEYS}
        v, a, lp, h, he, m = eng.act(obs, h, he, torch.from_numpy(g["masks"][t]).to(DEV), deterministic=True,
                                     return_mean=True)
        last = t == T - 1
        _check((v, m, h) + ((he,) if last else ()), (g["value"][t], g["mean"][t], g["h"][t], g["he_final"]),
               "step %d" % t)


def test_zero_edge_state_null_equals_explicit_zeros():
    obs, ins, _ = act_case("varnum_h20")
    N = obs["spatial_edges"].shape[0]
    eng, _ = _engine(N, 20, 2)
    outs = []
    for edge in (None, torch.zeros(1, 1, 1, device=DEV).expand(N, 21, 256), torch.zeros(N, 21, 256, device=DEV)):
        r = eng.act(_cuda(obs), ins["h"].to(DEV), edge, ins["masks"].to(DEV), deterministic=True, return_mean=True)
        outs.append([x.clone() for x in r])
    for o in outs[1:]:
        for x, y in zip(outs[0], o):
            assert torch.equal(x, y)


def test_sampled_actions_follow_mean_plus_std_noise():
    obs, ins, _ = act_case("pred_h20")
    N = obs["spatial_edges"].shape[0]
    eng, ref = _engine(N, 20, 12)
    noise = torch.randn(N, 2, device=DEV)
    v, a, lp, h1, he1, m = eng.act(_cuda(obs), ins["h"].to(DEV), ins["he"].to(DEV), ins["masks"].to(DEV),
                                   noise=noise, return_mean=True)
    std = ref.dist.logstd._bias.detach().reshape(1, 2).exp().to(DEV)
    assert torch.allclose(a, noise * std + m, rtol=0, atol=1e-5)
    want_lp = torch.distributions.Normal(m, std).log_prob(a).sum(-1, keepdim=True)
    assert torch.allclose(lp, want_lp, atol=1e-5)


class _TrainArgs(Args):
    def __init__(self):
        super().__init__(num_processes=64, seq_length=8, num_mini_batch=2)
        self.num_steps, self.clip_param, self.ppo_epoch, self.value_loss_coef, self.entropy_coef = 8, 0.2, 2, 0.5, 0.0
        self.lr, self.eps, self.max_grad_norm, self.gamma, self.gae_lambda = 4e-5, 1e-5, 0.5, 0.99, 0.95


def test_train_iteration_varnum():
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.storage import RolloutStorage
    from crowdnav_prediction_attngraph_b200 import ppo
    a = _TrainArgs()
    dev = torch.device(DEV)
    torch.manual_seed(425)
    envs = CudaCrowdVecEnv(num_envs=a.num_processes, human_num=20, seed=425, device=dev, const_vel=0)
    pol = Policy(envs.observation_space.spaces, envs.action_space, base_kwargs=a, base='srnn').to(dev)
    st = RolloutStorage(a.num_steps, a.num_processes, envs.observation_space.spaces, envs.action_space, 128, 256, device=dev)
    agent = ppo.PPO(pol, a.clip_param, a.ppo_epoch, a.num_mini_batch, a.value_loss_coef, a.entropy_coef,
                    lr=a.lr, eps=a.eps, max_grad_norm=a.max_grad_norm)
    obs = envs.reset()
    for k in st.obs:
        st.obs[k][0].copy_(obs[k])
    unused = {k: p.detach().clone() for k, p in pol.named_parameters() if k.startswith(UNUSED)}
    assert len(unused) == 6
    acted = []
    for step in range(a.num_steps):
        with torch.no_grad():
            o = {k: st.obs[k][step] for k in st.obs}
            hx = {k: st.recurrent_hidden_states[k][step] for k in st.recurrent_hidden_states}
            value, action, logp, hx2 = pol.act(o, hx, st.masks[step])
        acted.append(hx2['human_human_edge_rnn'].clone())
        obs, reward, done, infos = envs.step(action)
        masks = torch.FloatTensor([[0.0] if d else [1.0] for d in done])
        st.insert(obs, hx2, action, logp, value, reward, masks, torch.ones(a.num_processes, 1))
    for step in range(a.num_steps):
        assert torch.equal(st.recurrent_hidden_states['human_human_edge_rnn'][step + 1], acted[step])
    with torch.no_grad():
        o = {k: st.obs[k][-1] for k in st.obs}
        hx = {k: st.recurrent_hidden_states[k][-1] for k in st.recurrent_hidden_states}
        next_value = pol.get_value(o, hx, st.masks[-1]).detach()
    st.compute_returns(next_value, True, a.gamma, a.gae_lambda, False)
    losses = agent.update(st)
    st.after_update()
    assert np.isfinite(losses).all()
    for k, p in pol.named_parameters():
        if k in unused:
            assert torch.equal(p.detach(), unused[k]), k
    envs.close()


def test_batched_evaluation_equals_sequential_for_dsrnn():
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    from crowdnav_prediction_attngraph_b200.policy import Policy
    dev = torch.device(DEV)
    test_size = 5
    d = _capi.default_config_dict(num_envs=1, nenv_total=1, seed=19, human_num=20, phase=2, test_size=test_size,
                                  time_limit=20.0, const_vel=0)
    sp, act = spaces(20, 2)
    pol = Policy(sp, act, base='srnn', base_kwargs=Args(num_processes=1))
    pol.load_state_dict(dsrnn_state_dict(pol.state_dict()))
    pol = pol.to(dev)
    env = CudaCrowdVecEnv(device=dev, cfg=d)
    seq = evaluate(pol, env, 1, dev, test_size, None, None, None)
    env.close()
    bat = evaluate_batched(pol, None, "CrowdSimVarNum-v0", 19, test_size, dev, cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    for k in ("success_rate", "collision_rate", "timeout_rate", "collision_cases", "timeout_cases"):
        assert seq[k] == bat[k], k
    for k in ("avg_nav_time", "path_length", "intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k
