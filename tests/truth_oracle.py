"""ORACLE (test infrastructure): one reference CrowdSimPred-v0 environment with sim.predict_method = 'truth'.  A scalar
restatement on top of oracle/crowd_env.py: CrowdSimPred.generate_ob (crowd_sim_pred.py:62-97) calls
calc_human_future_traj('truth') on every observation, reset included, and observes its kept rows; the look-ahead's
solves go through (and create) the humans' rvo2 simulators.  Everything else is CrowdSimPred-v0 as the base class runs it
for 'const_vel': the next step's reward penalises the stored trajectory, humans join / leave by CrowdSimPred's rule.
Pinned against the reference by the 'truth' goldens of tools/make_golden.py (tests/test_env_harness_truth_pred.py)."""
import numpy as np

from oracle.crowd_env import CrowdEnvOracle


class TruthPredOracle(CrowdEnvOracle):
    """CrowdEnvOracle of CrowdSimPred-v0 whose observation and stored trajectory come from the ground-truth look-ahead.
    `cfg.predict_method` is 'const_vel' (the base class's CrowdSimPred-v0 mode, whose reward and join / leave rules
    'truth' shares)."""

    def __init__(self, cfg, this_seed, nenv, phase="train"):
        if cfg.predict_method != "const_vel":
            raise ValueError("TruthPredOracle runs CrowdSimPred-v0: pass cfg.predict_method = 'const_vel'")
        super().__init__(cfg, this_seed, nenv, phase)

    def _generate_ob(self, reset):
        # visibility, belief update and the rest of the observation as for 'const_vel'; then the rows of the humans the
        # robot sees (this observation's visibility) come from the look-ahead, which also replaces the stored trajectory
        ob = super()._generate_ob(reset)
        H, P = self.H, self.P
        traj = self._truth_future_traj()
        vis = np.array(self.human_visibility, dtype=bool)
        spatial = np.ones((self.Hmax, 2 * (P + 1))) * np.inf
        pred_pos = np.transpose(traj[:, :, :2], (1, 0, 2)) - np.array([self.rpx, self.rpy])
        spatial[:H][vis] = pred_pos.reshape((H, -1))[vis]
        if self.cfg.sort_humans:
            spatial = np.array(sorted(spatial, key=lambda x: np.linalg.norm(x[:2])))
        spatial[np.isinf(spatial)] = 15
        ob["spatial_edges"] = np.asarray(spatial, dtype=np.float32)
        return ob
