#!/usr/bin/env python
"""Golden vectors for BASELINE config 3 (row a16): the GST trajectory predictor and the VecPretextNormalize
wrapper, recorded from the UNMODIFIED reference code (runs only in the build container).

  tests/golden/gst_params.npz   the 67 269 parameters of the shipped predictor checkpoint (config.pred.model_dir
                                = gst_updated/results/...seed_1000_rand/sj/checkpoint/epoch_100.pt), loaded with
                                weights_only=True + an allowlist of the numpy scalar types the file pickles
  tests/golden/gst_io.npz       CrowdNavPredInterfaceMultiEnv.forward on random (partially masked) 5-frame windows
  tests/golden/gst_rollout.npz  CrowdSimPredRealGST-v0 environments stepped like the vec-env workers, their raw
                                observations, and what VecPretextNormalize.process_obs_rew makes of them

Opt-in modes (named on the command line; the default list is params, io, rollout) record larger crowds:
  io_h13, io_h128               gst_io_h13.npz / gst_io_h128.npz: the predictor on 13 and 128 humans
  rollout_h10_range3            gst_rollout_h10_range3.npz: 10 humans, human_num_range 3 (13 rows, humans join / leave)
  rollout_h50                   gst_rollout_h50.npz: 50 humans
  rollout_h100_x2               gst_rollout_h100_x2.npz: 100 humans, circle and arena x2 (BASELINE config 5's crowd)

The reference objects are created without running their __init__ (which torch.load()s / unpickles files);
the model arguments are the literal content of checkpoint/args.pickle.
"""
import argparse
import os
import sys
from collections import deque

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, "oracle", "shims"))
from reference_root import reference_root  # noqa: E402
REF = reference_root()
sys.path.insert(0, REF)
sys.path.insert(0, REPO)

import numpy as np  # noqa: E402
import torch  # noqa: E402

CKPT = os.path.join(REF, "gst_updated/results/100-gumbel_social_transformer-faster_lstm-lr_0.001-init_temp_0.5-"
        "edge_head_0-ebd_64-snl_1-snh_8-seed_1000_rand/sj/checkpoint/epoch_100.pt")
GST_ARGS = dict(spatial='gumbel_social_transformer', temporal='faster_lstm', output_dim=5, embedding_size=64,
                spatial_num_heads=8, lstm_hidden_size=64, lstm_num_layers=1, decode_style='recursive',
                detach_sample=False, motion_dim=2, obs_seq_len=5, pred_seq_len=5, num_epochs=100,
                spatial_num_layers=1, only_observe_full_period=False, spatial_num_heads_edges=0, ghost=False,
                init_temp=0.5)
GOLD = os.path.join(REPO, "tests", "golden")


def load_state_dict():
    allow = [(np._core.multiarray.scalar, "numpy.core.multiarray.scalar"), np.dtype, np.dtypes.Float64DType,
             np.dtypes.Float32DType, np.dtypes.Int64DType]
    with torch.serialization.safe_globals(allow):
        ck = torch.load(CKPT, map_location="cpu", weights_only=True)
    return ck["model_state_dict"]


def build_interface(num_env):
    from gst_updated.src.gumbel_social_transformer.st_model import st_model
    from gst_updated.scripts.wrapper.crowd_nav_interface_parallel import CrowdNavPredInterfaceMultiEnv
    args = argparse.Namespace(**GST_ARGS)
    model = st_model(args, device="cpu")
    model.load_state_dict(load_state_dict())
    model.eval()
    itf = object.__new__(CrowdNavPredInterfaceMultiEnv)
    itf.args = itf.args_eval = args
    itf.device = torch.device("cpu")
    itf.nenv = num_env
    itf.model = model
    return itf


def make_params():
    sd = load_state_dict()
    np.savez_compressed(os.path.join(GOLD, "gst_params.npz"), **{k: v.numpy() for k, v in sd.items()})
    print("wrote gst_params.npz", sum(v.numel() for v in sd.values()), "parameters")


def make_io(name="gst_io.npz", N=6, H=20, seed=3):
    rng = np.random.RandomState(seed)
    itf = build_interface(N)
    # smooth random walks + random visibility patterns (full, partial, never visible, appearing, disappearing)
    start = rng.uniform(-6, 6, (N, H, 1, 2))
    vel = rng.uniform(-0.3, 0.3, (N, H, 1, 2))
    traj = start + vel * np.arange(5).reshape(1, 1, 5, 1) + rng.normal(0, 0.02, (N, H, 5, 2))
    mask = (rng.uniform(size=(N, H, 5, 1)) < 0.8)
    mask[:, 0] = True
    mask[:, 1] = False
    mask[:, 2, :3] = False
    mask[:, 2, 3:] = True
    mask[:, 3, 4] = False
    traj = np.where(mask, traj, -999.0)
    with torch.no_grad():
        out_traj, out_mask = itf.forward(torch.tensor(traj, dtype=torch.float32), torch.tensor(mask, dtype=torch.float32))
    np.savez_compressed(os.path.join(GOLD, name), in_traj=traj.astype(np.float32), in_mask=mask,
                        out_traj=out_traj.numpy(), out_mask=out_mask.numpy())
    print("wrote", name, out_traj.shape, float(out_mask.mean()))


def make_rollout(name="gst_rollout.npz", N=3, T=90, H=20, human_num_range=0, seed=425, scale=1):
    """scale: factor on sim.circle_radius and sim.arena_size (2 for the 100-human crowd, which the reference's spawner
    cannot place on the default circle)"""
    sys.argv = ["x", "--no-cuda", "--env-name", "CrowdSimPredRealGST-v0"]
    import gym
    import crowd_sim  # noqa: F401
    import rvo2
    rvo2.ONLY_AGENT0 = False
    from crowd_nav.configs.config import Config
    from rl.vec_env.vec_pretext_normalize import VecPretextNormalize
    cfg = Config()
    cfg.sim.human_num = H
    # Config's sections are shared class objects: set every field a mode changes, so that modes run in one process
    # do not see each other's settings (the values at scale 1 are the reference's defaults)
    cfg.sim.human_num_range = human_num_range
    cfg.sim.circle_radius = 6 * np.sqrt(2) * scale
    cfg.sim.arena_size = 6 * scale
    HM = H + human_num_range                      # VecPretextNormalize.max_human_num: rows of every observation
    cfg.sim.predict_method = "inferred"
    cfg.env.use_wrapper = True
    cfg.orca.neighbor_dist = 10
    cfg.training.device = "cpu"
    envs = []
    for k in range(N):
        env = gym.make("CrowdSimPredRealGST-v0")
        env.configure(cfg)
        env.thisSeed = seed + k
        env.nenv = N
        env.phase = "train"
        envs.append(env)
    w = object.__new__(VecPretextNormalize)
    w.config = cfg
    w.device = torch.device("cpu")
    w.num_envs = N
    w.max_human_num = HM
    w.predictor = build_interface(N)
    w.pred_interval = int(cfg.data.pred_timestep // cfg.env.time_step)
    w.buffer_len = (GST_ARGS["obs_seq_len"] - 1) * w.pred_interval + 1
    # VecPretextNormalize.reset() without the venv call
    w.traj_buffer = deque(list(-torch.ones((w.buffer_len, N, HM, 2)) * 999), maxlen=w.buffer_len)
    w.mask_buffer = deque(list(torch.zeros((w.buffer_len, N, HM, 1), dtype=torch.bool)), maxlen=w.buffer_len)
    w.step_counter = 0
    w.last_pos = torch.zeros(N, HM, 2)

    def stack(obs_list):
        out = {}
        for key in ("robot_node", "temporal_edges", "spatial_edges", "detected_human_num", "visible_masks"):
            arr = np.stack([np.asarray(o[key]) for o in obs_list])
            out[key] = torch.tensor(arr, dtype=torch.bool if key == "visible_masks" else torch.float32)
        out["robot_node"] = out["robot_node"].reshape(N, 1, 7)
        out["temporal_edges"] = out["temporal_edges"].reshape(N, 1, 2)
        out["detected_human_num"] = out["detected_human_num"].reshape(N, 1)
        return out

    rec = dict(actions=np.zeros((T, N, 2), np.float32), reward_env=np.zeros((T, N)), reward=np.zeros((T, N)),
               done=np.zeros((T, N), bool))
    raw, fin = [], []
    rng = np.random.RandomState(5)
    obs_list = [e.reset() for e in envs]
    O = stack(obs_list)
    raw.append({k: v.numpy().copy() for k, v in O.items()})
    obs, _ = w.process_obs_rew(O, np.zeros(N))
    fin.append({k: v.numpy().copy() for k, v in obs.items()})
    for t in range(T):
        acts = []
        for k in range(N):
            rn = np.asarray(obs_list[k]["robot_node"], dtype=np.float64).reshape(-1)
            g = np.array([rn[3] - rn[0], rn[4] - rn[1]])
            a = (g / (np.linalg.norm(g) + 1e-9) * 0.9 + rng.normal(0, 0.3, 2)).astype(np.float32)
            acts.append(a)
        rec["actions"][t] = np.stack(acts)
        rews = np.zeros((N, 1))
        for k in range(N):
            ob, rew, done, info = envs[k].step(acts[k].copy())
            rec["reward_env"][t, k] = rew
            rec["done"][t, k] = done
            rews[k, 0] = rew
            if done:
                ob = envs[k].reset()
            obs_list[k] = ob
        O = stack(obs_list)
        raw.append({k: v.numpy().copy() for k, v in O.items()})
        obs, rews = w.process_obs_rew(O, rec["done"][t], rews=rews)
        rec["reward"][t] = np.asarray(rews).reshape(N)
        fin.append({k: v.numpy().copy() for k, v in obs.items()})
    out = dict(rec)
    for key in raw[0]:
        out["raw_" + key] = np.stack([r[key] for r in raw])
        out["fin_" + key] = np.stack([r[key] for r in fin])
    meta = dict(nenv=N, steps=T, human_num=H, seed=seed)
    if name != "gst_rollout.npz":                    # the default file's meta stays as it was recorded
        meta.update(human_num_range=human_num_range, circle_radius=float(cfg.sim.circle_radius),
                    arena_size=float(cfg.sim.arena_size))
    out["meta"] = np.array([repr(meta)])
    np.savez_compressed(os.path.join(GOLD, name), **out)
    print("wrote %s; episodes:" % name, rec["done"].sum(0), "penalised steps:",
          int((np.abs(rec["reward"] - rec["reward_env"]) > 0).sum()))


# opt-in crowds beyond the shipped 20 humans: mode -> (function, keyword arguments)
EXTRA = {
    "io_h13": (make_io, dict(name="gst_io_h13.npz", N=6, H=13, seed=13)),
    "io_h128": (make_io, dict(name="gst_io_h128.npz", N=3, H=128, seed=128)),
    "rollout_h10_range3": (make_rollout, dict(name="gst_rollout_h10_range3.npz", N=3, T=90, H=10, human_num_range=3)),
    "rollout_h50": (make_rollout, dict(name="gst_rollout_h50.npz", N=2, T=60, H=50)),
    "rollout_h100_x2": (make_rollout, dict(name="gst_rollout_h100_x2.npz", N=2, T=40, H=100, scale=2)),
}

if __name__ == "__main__":
    which = sys.argv[1:] or ["params", "io", "rollout"]
    unknown = [m for m in which if m not in ("params", "io", "rollout") and m not in EXTRA]
    if unknown:
        sys.exit("unknown mode(s) %s; modes: params io rollout %s" % (unknown, " ".join(EXTRA)))
    if "params" in which:
        make_params()
    if "io" in which:
        make_io()
    if "rollout" in which:
        make_rollout()
    for m in which:
        if m in EXTRA:
            EXTRA[m][0](**EXTRA[m][1])
