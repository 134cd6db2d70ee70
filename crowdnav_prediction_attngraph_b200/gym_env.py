"""Single-environment Gym surface of the reference (`gym.make('CrowdSimPred-v0')`, SURVEY.md §8b row 1) over the
CUDA engine: one environment resident on the GPU, host numpy in / out.

Mirrors crowd_sim/envs/crowd_sim_pred.py:20-58,100-213, crowd_sim_var_num.py:37-58,303-363 and
crowd_sim_pred_real_gst.py:27-62 at the call surface make_env uses (rl/networks/envs.py:36-94):
`configure(config)`, attribute writes `thisSeed / nenv / phase / render_axis / test_case`, `seed()`,
`observation_space`, `action_space`, `reset()`, `step(action)`, `talk2Env()`, `close()`, and the attributes
rl/evaluation.py reads (`time_limit`, `global_time`, `episode_k`).

Episode boundaries: the engine resets an environment inside the step that ends its episode (that is what the
reference's vec-env worker does, shmem_vec_env.py:138-142) and returns the FIRST observation of the next episode
with `done`.  A `reset()` that directly follows such a step returns that observation without starting yet another
episode, so the case counter advances once per episode exactly as in the reference; a `reset()` at any other
time starts a new episode."""
import numpy as np
import torch

from . import _capi
from .vec_env import CudaCrowdVecEnv, Box, _DictSpace, config_dict_from_reference

_ENV_IDS = {"CrowdSimPred": "CrowdSimPred-v0", "CrowdSimVarNum": "CrowdSimVarNum-v0",
            "CrowdSimPredRealGST": "CrowdSimVarNum-v0"}


class _GymCrowdEnv(object):
    metadata = {'render.modes': ['human']}
    _engine_id = None            # engine mode of the subclass
    _unsorted = False            # CrowdSimPredRealGST: raw, unsorted observation (the wrapper sorts)

    def __init__(self):
        self.config = None
        self.thisSeed = None
        self.nenv = None
        self.phase = None
        self.test_case = None
        self.render_axis = None
        self.episode_k = 0
        self.time_limit = None
        self.time_step = None
        self.human_num = None
        self.observation_space = None
        self.action_space = None
        self._venv = None
        self._pending_reset_obs = None
        self._device = None

    # ------------------------------------------------------------------ configuration
    def configure(self, config):
        self.config = config
        self.time_limit = config.env.time_limit
        self.time_step = config.env.time_step
        self.human_num = config.sim.human_num
        H = config.sim.human_num + config.sim.human_num_range
        W = 2 * (config.sim.predict_steps + 1) if self._engine_id == "CrowdSimPred-v0" else 2
        spaces = {'robot_node': Box((1, 7)), 'temporal_edges': Box((1, 2)), 'spatial_edges': Box((H, W)),
                  'detected_human_num': Box((1,))}
        if self._engine_id != "CrowdSimPred-v0":
            spaces['visible_masks'] = Box((H,), np.bool_)
        self.observation_space = _DictSpace(spaces)
        self.action_space = Box((2,))
        dev = getattr(getattr(config, "training", None), "device", "cuda:0")
        self._device = torch.device(dev if str(dev).startswith("cuda") else "cuda:0")

    def seed(self, seed=None):
        return [seed]

    def _build(self):
        if self.config is None:
            raise AttributeError('robot has to be set!')      # the reference's error for an unconfigured env
        if self.thisSeed is None or self.nenv is None:
            raise AttributeError("env.thisSeed and env.nenv must be set before reset() (rl/networks/envs.py:51-58)")
        phase = self.phase if self.phase is not None else 'train'
        d = config_dict_from_reference(self.config, 1, int(self.thisSeed), self._engine_id, nenv_total=int(self.nenv),
                                       rank_offset=0, device_index=self._device.index or 0, phase=phase,
                                       allow_unsorted=self._unsorted)
        if self._unsorted:
            d.update(sort_humans=0)
        self._venv = CudaCrowdVecEnv(device=self._device, cfg=d)
        if self.test_case is not None and self.test_case >= 0:
            self._venv.set_state("case_counter", np.array([self.test_case], np.uint32))

    def _to_host(self, obs):
        out = {}
        for k, v in obs.items():
            a = v[0].cpu().numpy()
            out[k] = a
        return out

    # ------------------------------------------------------------------ Gym API
    def reset(self, phase='train', test_case=None):
        if self._venv is None:
            self._build()
        if self._pending_reset_obs is not None:
            ob, self._pending_reset_obs = self._pending_reset_obs, None
            return ob
        if test_case is not None:
            self._venv.set_state("case_counter", np.array([test_case], np.uint32))
        return self._to_host(self._venv.reset())

    def step(self, action, update=True):
        if self._venv is None:
            raise RuntimeError("step() before reset()")
        a = np.asarray(action, dtype=np.float32).reshape(2)
        # SRNN.clip_action mutates the caller's array in place (crowd_nav/policy/srnn.py:17-33)
        v_pref = np.float32(self.config.robot.v_pref)
        norm = np.linalg.norm(a)
        if norm > v_pref and isinstance(action, np.ndarray) and action.dtype == np.float32:
            action[0] = a[0] / norm * v_pref
            action[1] = a[1] / norm * v_pref
        self._pending_reset_obs = None
        obs, reward, done, infos = self._venv.step(torch.from_numpy(a.copy()).unsqueeze(0).to(self._device))
        ob = self._to_host(obs)
        info = infos[0]
        d = bool(done[0])
        if d:
            self._pending_reset_obs = ob
        return ob, float(reward[0, 0]), d, {'info': info['info']}

    @property
    def global_time(self):
        if self._venv is None:
            return 0.0
        return float(self._venv.get_state("step_count")[0]) * float(self.time_step)

    def talk2Env(self, data):
        return True

    def render(self, mode='human'):
        return None

    def close(self):
        if self._venv is not None:
            self._venv.close()
            self._venv = None

    @property
    def unwrapped(self):
        return self


class CrowdSimPred(_GymCrowdEnv):
    """crowd_sim/envs/crowd_sim_pred.py, with sim.predict_method 'const_vel' (constant-velocity predictions) or 'truth'
    (every observation runs the ground-truth look-ahead; robot.visible = True is covered there)."""
    _engine_id = "CrowdSimPred-v0"


class CrowdSimVarNum(_GymCrowdEnv):
    """crowd_sim/envs/crowd_sim_var_num.py."""
    _engine_id = "CrowdSimVarNum-v0"


class CrowdSimPredRealGST(_GymCrowdEnv):
    """crowd_sim/envs/crowd_sim_pred_real_gst.py: the raw (unsorted, 2-wide) observation the GST wrapper consumes."""
    _engine_id = "CrowdSimVarNum-v0"
    _unsorted = True


class CrowdSimVarNumCollect(_GymCrowdEnv):
    """crowd_sim/envs/crowd_sim_var_num_collect.py: the data-collection environment of collect_data.py, observation
    {'pred_info': [H, 4]} (frame, prediction id, px, py; inf where the robot does not see the human)."""
    _engine_id = "CrowdSimVarNumCollect-v0"

    def configure(self, config):
        super().configure(config)
        H = config.sim.human_num + config.sim.human_num_range
        self.observation_space = _DictSpace({'pred_info': Box((H, 4))})

    def _build(self):
        from .collect import CudaCollectVecEnv
        if self.config is None:
            raise AttributeError('robot has to be set!')
        if self.thisSeed is None or self.nenv is None:
            raise AttributeError("env.thisSeed and env.nenv must be set before reset() (rl/networks/envs.py:51-58)")
        phase = self.phase if self.phase is not None else 'train'
        d = config_dict_from_reference(self.config, 1, int(self.thisSeed), self._engine_id, nenv_total=int(self.nenv),
                                       rank_offset=0, device_index=self._device.index or 0, phase=phase)
        self._venv = CudaCollectVecEnv(device=self._device, cfg=d)

    def reset(self, phase='train', test_case=None):
        if self._venv is None:
            self._build()
        return {'pred_info': self._venv.reset_device()[0].cpu().numpy()}

    def step(self, action, update=True):
        if self._venv is None:
            raise RuntimeError("step() before reset()")
        a = torch.from_numpy(np.asarray(action, dtype=np.float32).reshape(1, 2).copy()).to(self._device)
        obs, _, done, infos = self._venv.step(a)
        return {'pred_info': obs['pred_info'][0]}, 0, bool(done[0]), {'info': infos[0]['info']}
