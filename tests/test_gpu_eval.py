"""GPU: test-phase evaluation (SURVEY.md 8f row 1).  The batched evaluation (test_size parallel environments) must
report exactly what the reference's sequential protocol reports when both run on the CUDA engine, and the
protocol's seeding quirks (two resets per episode, case counter wrap) must hold."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _policy(N, dev):
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    from crowdnav_prediction_attngraph_b200.policy import Policy, make_reference_like_state_dict

    class Args(object):
        num_processes, seq_length, num_mini_batch = N, 30, 2
    spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((20, 12)),
              'detected_human_num': Box((1,))}
    pol = Policy(spaces, Box((2,)), base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    sd = make_reference_like_state_dict(12, seed=5)
    # a goal-seeking bias so that episodes end in all three ways within the time limit
    pol.load_state_dict(sd, strict=False)
    return pol


def test_batched_evaluation_equals_sequential_protocol():
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate, evaluate_batched
    dev = torch.device("cuda:0")
    test_size = 7                       # odd on purpose: the case counter wraps at test_size (0,2,4,6,1,3,5)
    d = _capi.default_config_dict(num_envs=1, nenv_total=1, seed=19, human_num=20, phase=2, test_size=test_size,
                                  time_limit=20.0)
    pol = _policy(1, dev)
    env = CudaCrowdVecEnv(device=dev, cfg=d)
    seq = evaluate(pol, env, 1, dev, test_size, None, None, None)
    env.close()
    bat = evaluate_batched(pol, None, "CrowdSimPred-v0", 19, test_size, dev, cfg_dict=d)
    assert seq["episode_steps"] == bat["episode_steps"]
    for k in ("success_rate", "collision_rate", "timeout_rate", "collision_cases", "timeout_cases"):
        assert seq[k] == bat[k], k
    for k in ("avg_nav_time", "path_length", "intrusion_ratio", "mean_episode_reward"):
        assert seq[k] == pytest.approx(bat[k], rel=1e-12, abs=1e-12), k
    if not np.isnan(seq["min_intrusion_dist"]):
        assert seq["min_intrusion_dist"] == pytest.approx(bat["min_intrusion_dist"], rel=1e-9)
    assert abs(seq["success_rate"] + seq["collision_rate"] + seq["timeout_rate"] - 1.0) < 1e-12


def test_single_env_defaults_to_test_phase_and_val_is_rejected():
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.vec_env import CudaCrowdVecEnv
    with pytest.raises(RuntimeError):
        CudaCrowdVecEnv(device="cuda:0", cfg=_capi.default_config_dict(num_envs=2, phase=1))


SHIPPED_COLLISIONS = [0, 1, 12, 17, 31, 34, 35, 42, 48, 57, 60, 68, 71, 89, 98, 99, 113, 117, 119, 121, 131, 142, 153, 158,
                      161, 164, 170, 214, 239, 246, 248, 250, 251, 262, 267, 281, 284, 285, 292, 298, 307, 310, 318, 321,
                      339, 348, 349, 363, 367, 369, 371, 381, 392, 403, 408, 411, 414, 420, 464, 489, 496, 498]


def test_shipped_checkpoint_reproduces_shipped_test_log():
    """End-to-end results parity (config 3, phase 'test'): the reference's 500-case protocol with its shipped policy
    checkpoint and GST predictor on this engine vs trained_models/GST_predictor_rand/test/test_41665.pt.log
    (success 0.88, collision 0.12, timeout 0.00, nav time 14.14, path length 20.08, intrusion ratio 8.35 %, min
    distance 0.41).  Needs the 10 MB checkpoint at local_ckpt/41665.pt (a reference artefact, not committed)."""
    import os
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate_batched
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ckpt = os.path.join(repo, "local_ckpt", "41665.pt")
    if not os.path.exists(ckpt):
        pytest.skip("shipped checkpoint not present (copy trained_models/GST_predictor_rand/checkpoints/41665.pt to local_ckpt/)")
    dev = torch.device("cuda:0")

    class Args(object):
        num_processes, seq_length, num_mini_batch = 500, 30, 2
    spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((20, 12)),
              'detected_human_num': Box((1,)), 'visible_masks': Box((20,), np.bool_)}
    pol = Policy(spaces, Box((2,)), base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    pol.load_state_dict(torch.load(ckpt, map_location="cpu", weights_only=True))
    gst = dict(np.load(os.path.join(repo, "tests", "golden", "gst_params.npz")))
    d = _capi.default_config_dict(num_envs=500, nenv_total=1, seed=425, human_num=20, phase=2, test_size=500,
                                  randomize_attributes=1, random_goal_changing=1, goal_change_chance=0.5)
    out = evaluate_batched(pol, None, "CrowdSimPredRealGST-v0", 425, 500, dev, cfg_dict=d, gst_params=gst)
    assert round(out["success_rate"], 2) == 0.88 and round(out["collision_rate"], 2) == 0.12 and out["timeout_rate"] == 0.0
    assert abs(out["avg_nav_time"] - 14.14) < 0.2 and abs(out["path_length"] - 20.08) < 0.15
    assert abs(out["intrusion_ratio"] - 8.35) < 0.3 and abs(out["min_intrusion_dist"] - 0.41) < 0.02
    same = len(set(out["collision_cases"]) & set(SHIPPED_COLLISIONS))
    assert same >= 56, "only %d of the 62 collision episodes of the shipped log collide here" % same
    # the case counter wraps at test_size: episode k + 250 repeats episode k
    assert all(((c + 250) % 500) in out["collision_cases"] for c in out["collision_cases"])


def test_shipped_non_rand_checkpoint_reproduces_its_test_log_exactly():
    """trained_models/GST_predictor_non_rand (fixed human attributes, seed 125, predictor ..._seed_1000): every episode
    outcome listed in test/test_41200.pt.log is reproduced.  Needs local_ckpt/41200.pt and local_ckpt/gst_params_nonrand.npz
    (reference artefacts, not committed; tools/eval_shipped.py documents how they are made)."""
    import os
    from crowdnav_prediction_attngraph_b200 import _capi
    from crowdnav_prediction_attngraph_b200.vec_env import Box
    from crowdnav_prediction_attngraph_b200.policy import Policy
    from crowdnav_prediction_attngraph_b200.evaluation import evaluate_batched
    repo = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ckpt, gstp = os.path.join(repo, "local_ckpt", "41200.pt"), os.path.join(repo, "local_ckpt", "gst_params_nonrand.npz")
    if not (os.path.exists(ckpt) and os.path.exists(gstp)):
        pytest.skip("shipped non_rand checkpoint / predictor parameters not present under local_ckpt/")
    dev = torch.device("cuda:0")

    class Args(object):
        num_processes, seq_length, num_mini_batch = 500, 30, 2
    spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((20, 12)),
              'detected_human_num': Box((1,)), 'visible_masks': Box((20,), np.bool_)}
    pol = Policy(spaces, Box((2,)), base_kwargs=Args(), base='selfAttn_merge_srnn').to(dev)
    pol.load_state_dict(torch.load(ckpt, map_location="cpu", weights_only=True))
    d = _capi.default_config_dict(num_envs=500, nenv_total=1, seed=125, human_num=20, phase=2, test_size=500)
    out = evaluate_batched(pol, None, "CrowdSimPredRealGST-v0", 125, 500, dev, cfg_dict=d, gst_params=dict(np.load(gstp)))
    assert out["collision_cases"] == [5, 71, 74, 95, 98, 103, 111, 159, 166, 171, 182, 186, 191, 205, 209, 227, 233, 235, 255,
                                      321, 324, 345, 348, 353, 361, 409, 416, 421, 432, 436, 441, 455, 459, 477, 483, 485]
    assert out["timeout_cases"] == [49, 299]
    assert round(out["avg_nav_time"], 2) == 15.42 and round(out["path_length"], 2) == 20.96
    # every episode outcome above is exact; the intrusion ratio counts single frames, where the 1e-6 summation-order
    # difference of the predictor's compact rows (masked neighbours enter the soft-max as one term) moves one or two
    # frames (4.237 vs the log's 4.23)
    assert abs(out["intrusion_ratio"] - 4.23) < 0.015 and round(out["min_intrusion_dist"], 2) == 0.44
