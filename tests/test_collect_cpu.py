"""The data-collection environment CrowdSimVarNumCollect-v0 on the CPU: the host build of the collect step kernel's
logic against golden vectors recorded from the unmodified reference (tools/make_golden_collect.py), the recorder's text
writer against the files the unmodified collect_data.py wrote, and the configurations the engine refuses."""
import os

import numpy as np
import pytest

from tests.collect_util import COLLECT_CASES, CollectHarnessEnv, load_collect_case, replay_collect
from tests.golden_util import GOLD


@pytest.mark.parametrize("name", COLLECT_CASES)
def test_collect_kernel_logic_host_build_matches_reference_golden(name):
    g, case, over = load_collect_case(name)
    env = CollectHarnessEnv(**over)
    bad = replay_collect(g, env.reset, env.step, env.get)
    assert not bad, bad[:5]


def test_collect_goldens_cover_both_goal_branches_and_collisions():
    med = uni = col = 0
    big_seed = False
    for name in COLLECT_CASES:
        g, case, _ = load_collect_case(name)
        big_seed |= case["seed"] >= 2 ** 31
        col += int((g["info"] == 2).sum())
        for t, k in zip(*np.nonzero(g["info"] == 3)):
            m = np.median(np.stack([g["hpx"][t - 1, k], g["hpy"][t - 1, k]], -1), axis=0)
            if np.array_equal(g["robot"][t, k, 4:6], m):
                med += 1
            else:
                uni += 1
    assert med > 0 and uni > 0 and col > 0 and big_seed


def _golden_rows(texts_npz):
    """The rows collect_data.py wrote, parsed back to float32 (the text is the repr of float32 values)."""
    out = []
    for text in texts_npz["texts"]:
        rows = [[float(x) for x in line.split("\t")] for line in str(text).splitlines()]
        out.append(np.asarray(rows, dtype=np.float32).reshape(-1, 4))
    return out


def test_text_writer_reproduces_collect_data_files(tmp_path):
    from crowdnav_prediction_attngraph_b200.collect import write_rows_txt
    f = np.load(os.path.join(GOLD, "collect_files.npz"))
    rows = _golden_rows(f)
    for rel in f["names"]:
        assert str(rel).startswith("train/")
    packed = np.concatenate(rows).astype(np.float32)
    counts = np.array([len(r) for r in rows], np.int64)
    write_rows_txt(str(tmp_path), packed, counts, env_base=0)
    for rel, text in zip(f["names"], f["texts"]):
        got = (tmp_path / os.path.basename(str(rel))).read_text()
        assert got == str(text), rel


def test_text_writer_formats_like_python_repr():
    from crowdnav_prediction_attngraph_b200.collect import format_rows
    rng = np.random.RandomState(0)
    vals = np.concatenate([rng.uniform(-20, 20, 4000), rng.uniform(-1e-4, 1e-4, 400), 2.0 ** rng.randint(-30, 60, 400),
                           np.array([0.0, -0.0, 1e-5, 1e-4, 1e16, 1e15, 123456789.0, 3.0517578125e-05, 40000.0])])
    rows = vals.astype(np.float32)[: (len(vals) // 4) * 4].reshape(-1, 4)
    want = "".join("\t".join(str(x) for x in r) + "\n" for r in rows.tolist())
    assert format_rows(rows) == want


def _config(**kw):
    from tests.test_robot_policy import _reference_like_config
    cfg = _reference_like_config("orca")
    for k, v in kw.items():
        sec, attr = k.split("__")
        setattr(getattr(cfg, sec), attr, v)
    return cfg


def test_collect_refusals():
    from crowdnav_prediction_attngraph_b200.vec_env import config_dict_from_reference
    name = "CrowdSimVarNumCollect-v0"
    d = config_dict_from_reference(_config(), 4, 2 ** 32 - 2005, name)
    assert d["seed"] == (2 ** 32 - 2005) - 2 ** 32 and d["const_vel"] == 0 and d["robot_policy"] == 1
    with pytest.raises(NotImplementedError, match="human_num_range"):
        config_dict_from_reference(_config(sim__human_num_range=2), 4, 425, name)
    with pytest.raises(NotImplementedError, match="human_visibility"):
        config_dict_from_reference(_config(), 1, 425, name)              # one environment: phase 'test'
    with pytest.raises(NotImplementedError, match="human_visibility"):
        config_dict_from_reference(_config(humans__policy="social_force"), 1, 425, name)
    # np.random.seed(2000 + case_counter + seed + rank) must stay below 2**32, as in the reference
    with pytest.raises(ValueError, match="2\\*\\*32"):
        config_dict_from_reference(_config(), 4, 2 ** 32 - 2003, name)
    with pytest.raises(ValueError, match="seed"):
        config_dict_from_reference(_config(), 4, 2 ** 32, name)
    # a network-policy robot takes the caller's action
    assert config_dict_from_reference(_config(robot__policy="srnn"), 4, 425, name)["robot_policy"] == 0
    with pytest.raises(NotImplementedError, match="[Rr]endering"):
        from crowdnav_prediction_attngraph_b200.collect import collect_dataset
        cfg = _config(data__render=True)
        collect_dataset(cfg, 4, 10, "/nonexistent", 425, True)
