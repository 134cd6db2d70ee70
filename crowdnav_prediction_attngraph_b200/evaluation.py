"""Test-phase evaluation with the reference's protocol and metrics (rl/evaluation.py:7-160, test.py:136-158).

`evaluate(...)` keeps the reference's signature and runs its sequential protocol against the CUDA vec env
(one environment in phase 'test': ground-truth ORCA look-ahead before the reward, 'future' danger zone, test
seeds).  `evaluate_batched(...)` runs the SAME test cases as N = test_size parallel environments and returns
identical numbers (tests/test_gpu_eval.py): episode k of the sequential protocol is seeded with
1000 + (2k mod test_size) + seed (every episode consumes two resets: the explicit `eval_envs.reset()` of the
loop and the vec env's auto-reset at `done`, rl/evaluation.py:52 + shmem_vec_env.py:140), so environment k of the
batch gets case_counter 2k mod test_size, nenv = 1 and a zero per-env seed offset.

Quirks of the reference that are reproduced on purpose (they shape the numbers in its shipped test logs):
  * path length includes the jump from the final robot position to the start of the auto-reset episode,
    because the observation returned with `done` already belongs to the next episode (evaluation.py:96-97);
  * navigation time is the simulation time at the BEGINNING of the last step (evaluation.py:76-77);
  * with test_size = env.test_size = 500 the case counter wraps: episodes 250..499 repeat episodes 0..249.
"""
import numpy as np
import torch

from .vec_env import (CudaCrowdVecEnv, CudaPretextVecEnv, Danger, ReachGoal, Collision, Timeout,
                      config_dict_from_reference)

INFO_TIMEOUT, INFO_COLLISION, INFO_REACHGOAL, INFO_DANGER = 1, 2, 3, 4


def _summary(test_size, time_limit, end_codes, end_times, path_len, too_close_ratio, min_dist, ep_rewards, logging=None):
    end_codes = np.asarray(end_codes)
    success = end_codes == INFO_REACHGOAL
    collision = end_codes == INFO_COLLISION
    timeout = end_codes == INFO_TIMEOUT
    assert int(success.sum() + collision.sum() + timeout.sum()) == test_size, "invalid end signal from environment"
    success_times = [t for t, s in zip(end_times, success) if s]
    out = dict(
        success_rate=float(success.sum()) / test_size, collision_rate=float(collision.sum()) / test_size,
        timeout_rate=float(timeout.sum()) / test_size,
        avg_nav_time=float(sum(success_times) / len(success_times)) if success_times else float(time_limit),
        path_length=float(np.mean(path_len)), intrusion_ratio=float(np.mean(too_close_ratio)),
        min_intrusion_dist=float(np.mean(min_dist)) if len(min_dist) else float("nan"),
        collision_cases=[int(k) for k in np.nonzero(collision)[0]], timeout_cases=[int(k) for k in np.nonzero(timeout)[0]],
        mean_episode_reward=float(np.mean(ep_rewards)) if len(ep_rewards) else float("nan"),
        episode_steps=None)
    if logging is not None:
        logging.info(
            'Testing success rate: {:.2f}, collision rate: {:.2f}, timeout rate: {:.2f}, '
            'nav time: {:.2f}, path length: {:.2f}, average intrusion ratio: {:.2f}%, '
            'average minimal distance during intrusions: {:.2f}'.format(
                out["success_rate"], out["collision_rate"], out["timeout_rate"], out["avg_nav_time"],
                out["path_length"], out["intrusion_ratio"], out["min_intrusion_dist"]))
        logging.info('Collision cases: ' + ' '.join(str(x) for x in out["collision_cases"]))
        logging.info('Timeout cases: ' + ' '.join(str(x) for x in out["timeout_cases"]))
    return out


def _initial_hxs(actor_critic, n, dev):
    """Zero recurrent state of n environments (rl/evaluation.py:16-21); the DS-RNN policy (base='srnn') also carries
    its edge state [n, H+1, 256] from step to step, starting from an expanded zero (never materialised: the engine
    takes it as the zero state)."""
    hxs = {'human_node_rnn': torch.zeros(n, 1, 128, device=dev)}
    if getattr(actor_critic, 'dsrnn', False):
        b = actor_critic.base
        hxs['human_human_edge_rnn'] = torch.zeros(1, 1, 1, device=dev).expand(n, b.human_num + 1,
                                                                              b.human_human_edge_rnn_size)
    return hxs


def _act(actor_critic, obs, hxs, masks, n, dev):
    """(action, hxs): the policy's deterministic action and new recurrent state, or zeros for actor_critic=None (the
    ORCA / social-force robot baselines drive the robot inside env.step; the loop passes zeros, rl/evaluation.py:64-73)."""
    if actor_critic is None:
        return torch.zeros(n, 2, device=dev), hxs
    with torch.no_grad():
        _, action, _, hxs = actor_critic.act(obs, hxs, masks, deterministic=True)
    return action, hxs


def evaluate(actor_critic, eval_envs, num_processes, device, test_size, logging, config, args, visualize=False):
    """rl/evaluation.py:7-160 against a CudaCrowdVecEnv with ONE environment (phase 'test').  Returns the
    metrics as a dict (the reference only logs them)."""
    assert num_processes == 1 and eval_envs.num_envs == 1, "the reference's evaluate() drives a single environment"
    dev = torch.device(device)
    time_limit = float(eval_envs.cfgd["time_limit"])
    dt = float(eval_envs.cfgd["time_step"])
    hxs = _initial_hxs(actor_critic, 1, dev)
    masks = torch.zeros(1, 1, device=dev)
    end_codes, end_times, all_path_len, too_close_ratios, min_dist, ep_rewards, steps = [], [], [], [], [], [], []
    for k in range(test_size):
        done = False
        step_counter, too_close, path_len = 0, 0.0, 0.0
        obs = eval_envs.reset()
        last_pos = obs['robot_node'][0, 0, :2].cpu().numpy()
        global_time = 0.0
        infos = None
        while not done:
            step_counter += 1
            action, hxs = _act(actor_critic, obs, hxs, masks, 1, dev)
            global_time = (step_counter - 1) * dt            # baseEnv.global_time read before the step
            obs, rew, done_arr, infos = eval_envs.step(action)
            done = bool(done_arr[0])
            pos = obs['robot_node'][0, 0, :2].cpu().numpy()
            # float32 norm accumulated in float64 (NumPy 1.x promotion of `python float + np.float32`, the
            # reference's environment; NumPy 2 would keep float32)
            path_len = path_len + float(np.linalg.norm(pos - last_pos))
            last_pos = pos
            info0 = infos[0]
            if isinstance(info0['info'], Danger):
                too_close += 1
                min_dist.append(info0['info'].min_dist)
            masks = torch.tensor([[0.0] if d else [1.0] for d in done_arr], dtype=torch.float32, device=dev)
            if 'episode' in info0:
                ep_rewards.append(info0['episode']['r'])
        all_path_len.append(path_len)
        too_close_ratios.append(too_close / step_counter * 100)
        steps.append(step_counter)
        last = infos[0]['info']
        if isinstance(last, ReachGoal):
            end_codes.append(INFO_REACHGOAL); end_times.append(global_time)
        elif isinstance(last, Collision):
            end_codes.append(INFO_COLLISION); end_times.append(global_time)
        elif isinstance(last, Timeout):
            end_codes.append(INFO_TIMEOUT); end_times.append(time_limit)
        else:
            raise ValueError('Invalid end signal from environment')
    out = _summary(test_size, time_limit, end_codes, end_times, all_path_len, too_close_ratios, min_dist, ep_rewards, logging)
    out["episode_steps"] = steps
    out.update(case_code=[int(c) for c in end_codes], case_nav_time=list(end_times), case_path_len=list(all_path_len))
    return out


def _freeze_robot_sim(base, d, dev):
    """Create the robot's rvo2 simulator the way the sequential protocol does (first step of case 0 on a single
    environment) and install it in every environment of `base`."""
    one = dict(d)
    one.update(num_envs=1)
    env1 = CudaCrowdVecEnv(device=dev, cfg=one)
    try:
        env1.set_state("seed_off", np.zeros(1, np.int32))
        env1.set_state("case_counter", np.zeros(1, np.uint32))
        env1.reset()
        env1.step(torch.zeros(1, 2, device=dev))
        N, H = base.num_envs, base.human_num
        base.set_state("rsim_exists", np.ones(N, np.uint8))
        base.set_state("rsim_nd", np.repeat(env1.get_state("rsim_nd"), N))
        base.set_state("rsim_rother", np.tile(env1.get_state("rsim_rother"), N))
    finally:
        env1.close()


def evaluate_batched(actor_critic, config, env_name, seed, test_size, device, logging=None, cfg_dict=None, gst_params=None):
    """The same test cases as `evaluate`, as test_size parallel environments on one GPU.
    config: reference Config object (or pass cfg_dict = a flat cn_config dict).  gst_params: predictor parameters
    for CrowdSimPredRealGST-v0 + VecPretextNormalize (config 3); the wrapper's buffers start empty for every test
    case exactly like the sequential protocol's explicit reset().

    actor_critic=None runs the ORCA / social-force robot baselines (robot.policy 'orca' / 'social_force').  The
    reference creates the robot's rvo2 simulator once per process, at the first step of case 0, and reuses it for
    every later case; its neighborDist and radii are frozen then.  To give every parallel case those same frozen
    parameters, one step of case 0 runs first on a one-environment handle and its robot simulator (rsim_*) is
    uploaded to all N environments before the batch starts.  Without randomised attributes the frozen values are the
    configured constants and the hand-off changes nothing."""
    dev = torch.device(device)
    N = test_size
    if cfg_dict is None:
        cfg_dict = config_dict_from_reference(config, N, seed, env_name, nenv_total=1, rank_offset=0,
                                              device_index=dev.index or 0, phase="test")
    d = dict(cfg_dict)
    d.update(num_envs=N, nenv_total=1, rank_offset=0, seed=seed, phase=2)
    env = CudaPretextVecEnv(gst_params, device=dev, cfg=d) if gst_params is not None else CudaCrowdVecEnv(device=dev, cfg=d)
    base = env.env if gst_params is not None else env
    size = int(d["test_size"])
    base.set_state("seed_off", np.zeros(N, np.int32))
    base.set_state("case_counter", ((2 * np.arange(N)) % size).astype(np.uint32))
    if int(d.get("robot_policy", 0)) == 1:
        _freeze_robot_sim(base, d, dev)
    time_limit, dt = float(d["time_limit"]), float(d["time_step"])
    hxs = _initial_hxs(actor_critic, N, dev)
    masks = torch.zeros(N, 1, device=dev)
    obs = env.reset()
    last_pos = obs['robot_node'][:, 0, :2].cpu().numpy()
    alive = np.ones(N, bool)
    steps = np.zeros(N, np.int64)
    too_close = np.zeros(N)
    path_len = np.zeros(N)
    end_codes = np.zeros(N, np.int64)
    end_times = np.zeros(N)
    ep_rewards = np.zeros(N)
    min_dist = [[] for _ in range(N)]
    max_steps = int(round(time_limit / dt)) + 2
    for _ in range(max_steps):
        if not alive.any():
            break
        action, hxs = _act(actor_critic, obs, hxs, masks, N, dev)
        obs, rew, done, infos = env.step(action)
        codes, aux = infos._codes, infos._aux
        pos = obs['robot_node'][:, 0, :2].cpu().numpy()
        seg = np.linalg.norm(pos - last_pos, axis=1)           # float32, like the per-episode loop
        last_pos = pos
        steps[alive] += 1
        path_len[alive] = path_len[alive] + seg[alive]
        danger = alive & (codes == INFO_DANGER)
        too_close[danger] += 1
        for k in np.nonzero(danger)[0]:
            min_dist[k].append(float(aux[k]))
        finished = alive & done
        for k in np.nonzero(finished)[0]:
            end_codes[k] = codes[k]
            end_times[k] = time_limit if codes[k] == INFO_TIMEOUT else (steps[k] - 1) * dt
            ep_rewards[k] = infos[k]['episode']['r']
        alive &= ~done
        masks = torch.from_numpy(1.0 - done.astype(np.float32)).reshape(N, 1).to(dev)
    assert not alive.any(), "some test episodes did not terminate within the time limit"
    flat_min = [x for k in range(N) for x in min_dist[k]]
    out = _summary(N, time_limit, end_codes, list(end_times), list(path_len), list(too_close / steps * 100), flat_min,
                   list(ep_rewards), logging)
    out["episode_steps"] = [int(x) for x in steps]
    # per-case records (the reference logs only the aggregates): outcome, nav time, path length, too-close frames and
    # the min distances of those frames
    out.update(case_code=[int(c) for c in end_codes], case_nav_time=[float(x) for x in end_times],
               case_path_len=[float(x) for x in path_len], case_too_close=[int(x) for x in too_close],
               case_min_dist=min_dist)
    env.close()
    return out
