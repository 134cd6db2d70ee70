"""The data-collection environment CrowdSimVarNumCollect-v0 on the GPU: the engine replays the reference goldens bit for
bit through the C ABI (with and without the side stream / pre-solve), collect_dataset writes the files the unmodified
collect_data.py wrote, and at N = 4096 the run is deterministic, shard invariant, hands out unique ids and records
exactly the rows a host-side filter of every observation keeps."""
import os

import numpy as np
import pytest
import torch

from tests.collect_util import COLLECT_CASES, load_collect_case, replay_collect
from tests.golden_util import GOLD

pytestmark = pytest.mark.gpu


def _env(**over):
    from crowdnav_prediction_attngraph_b200.collect import CudaCollectVecEnv
    from crowdnav_prediction_attngraph_b200 import _capi
    d = _capi.default_config_dict(const_vel=0, sort_humans=0)
    d.update(over)
    return CudaCollectVecEnv(device="cuda:0", cfg=d)


@pytest.mark.parametrize("variant", ["default", "presolve0", "presolve1", "no_side_stream"])
@pytest.mark.parametrize("name", COLLECT_CASES)
def test_engine_collect_matches_reference_golden(name, variant, monkeypatch):
    if variant == "presolve0":
        monkeypatch.setenv("CN_PRESOLVE", "0")
    elif variant == "presolve1":
        monkeypatch.setenv("CN_PRESOLVE", "1")
    elif variant == "no_side_stream":
        monkeypatch.setenv("CN_NO_SIDE_STREAM", "1")
    g, case, over = load_collect_case(name)
    env = _env(**over)

    def step(a):
        pi, _, _, _ = env.step_device(torch.as_tensor(a, device="cuda:0"))
        o = {k: v.cpu().numpy() for k, v in env._out.items()}
        return pi.cpu().numpy(), o

    bad = replay_collect(g, lambda: env.reset_device().cpu().numpy(), step, env.get_state)
    env.close()
    assert not bad, bad[:5]


def test_collect_dataset_writes_collect_data_files(tmp_path):
    import ast
    from crowdnav_prediction_attngraph_b200.collect import collect_dataset, reference_default_config
    f = np.load(os.path.join(GOLD, "collect_files.npz"))
    meta = ast.literal_eval(str(f["meta"][0]))
    stats = collect_dataset(reference_default_config(), meta["num_processes"], meta["tot_steps"], str(tmp_path),
                            meta["seed"], True, chunk_frames=7)          # several chunks, the last one partial
    assert stats["rows"] > 0
    for rel, text in zip(f["names"], f["texts"]):
        assert (tmp_path / str(rel)).read_text() == str(text), rel


def _run(N, T, **over):
    env = _env(num_envs=N, human_num=20, randomize_attributes=1, random_goal_changing=1, robot_policy=1, **over)
    zero = torch.zeros(N, 2, device="cuda:0")
    pis, ids, maxes = [env.reset_device().clone()], [torch.as_tensor(env.get_state("pred_id")).view(N, 20)], []
    maxes.append(env.get_state("max_id").copy())
    for _ in range(T):
        pis.append(env.step_device(zero)[0].clone())
        ids.append(torch.as_tensor(env.get_state("pred_id")).view(N, 20))
        maxes.append(env.get_state("max_id").copy())
    env.close()
    return torch.stack(pis).cpu().numpy(), torch.stack(ids).numpy(), np.stack(maxes)


def test_collect_n4096_deterministic_shard_invariant_unique_ids():
    N, T = 4096, 60
    a_pi, a_id, a_max = _run(N, T, seed=7)
    b_pi, _, _ = _run(N, T, seed=7)
    assert np.array_equal(a_pi.view(np.uint32), b_pi.view(np.uint32))
    h0 = _run(N // 2, T, seed=7, nenv_total=N, rank_offset=0)[0]
    h1 = _run(N // 2, T, seed=7, nenv_total=N, rank_offset=N // 2)[0]
    assert np.array_equal(np.concatenate([h0, h1], 1).view(np.uint32), a_pi.view(np.uint32))
    # ids: unique within an environment, a fresh id is above every id handed out before, max_id never decreases
    assert np.array_equal(a_pi[..., 1].astype(np.int64), a_id)
    for t in range(T + 1):
        s = np.sort(a_id[t], 1)
        assert (s[:, 1:] != s[:, :-1]).all()
        assert (a_id[t].max(1) < a_max[t]).all()
        if t:
            fresh = a_id[t] != a_id[t - 1]
            assert (a_id[t][fresh] >= np.repeat(a_max[t - 1][:, None], 20, 1)[fresh]).all()
            assert (a_max[t] >= a_max[t - 1]).all()
    assert (a_max[-1] > 20).any()


def test_recorder_equals_host_filter():
    from crowdnav_prediction_attngraph_b200.collect import Recorder
    N, T, C = 4096, 24, 10
    env = _env(num_envs=N, human_num=20, randomize_attributes=1, random_goal_changing=1, robot_policy=1, seed=11)
    rec = Recorder(N, 20, C, "cuda:0")
    zero = torch.zeros(N, 2, device="cuda:0")
    pi = env.reset_device()
    host = [[] for _ in range(N)]
    for t in range(T):
        o = pi.cpu().numpy()
        for e in range(N):
            host[e].append(o[e][~np.isinf(o[e, :, -1])])
        rec.append(pi)
        if rec.pending() == C or t == T - 1:
            rows, counts = rec.flush()
            host_chunk = [np.concatenate(h).reshape(-1, 4) for h in host]
            assert np.array_equal(counts, [len(h) for h in host_chunk])
            assert np.array_equal(rows.view(np.uint32), np.concatenate(host_chunk).view(np.uint32))
            host = [[] for _ in range(N)]
        pi = env.step_device(zero)[0]
    rec.close()
    env.close()


def test_make_vec_envs_collect_numpy_and_torch():
    from crowdnav_prediction_attngraph_b200.collect import reference_default_config
    from crowdnav_prediction_attngraph_b200.vec_env import make_vec_envs
    cfg = reference_default_config()
    envs = make_vec_envs("CrowdSimVarNumCollect-v0", 2 ** 31 + 9, 4, 0.99, None, "cuda:0", True, config=cfg,
                         wrap_pytorch=False)
    ob = envs.reset()
    assert isinstance(ob["pred_info"], np.ndarray) and ob["pred_info"].shape == (4, 20, 4)
    assert ob["pred_info"].dtype == np.float32
    ob, rew, done, infos = envs.step(np.zeros((4, 2)))
    assert isinstance(ob["pred_info"], np.ndarray) and np.all(ob["pred_info"][:, :, 0] == 1.0)
    assert isinstance(rew, np.ndarray) and not rew.any() and done.dtype == bool and len(infos) == 4
    envs.close()
    envs = make_vec_envs("CrowdSimVarNumCollect-v0", 425, 4, 0.99, None, "cuda:0", True, config=cfg, wrap_pytorch=True)
    ob = envs.reset()
    assert torch.is_tensor(ob["pred_info"]) and ob["pred_info"].is_cuda
    ob, rew, done, infos = envs.step(torch.zeros(4, 2, device="cuda:0"))
    assert torch.is_tensor(ob["pred_info"]) and rew.shape == (4, 1)
    envs.close()
