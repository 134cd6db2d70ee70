"""ORACLE (test infrastructure): one reference environment whose robot runs its own policy, robot.policy 'orca' or
'social_force' (crowd_sim_var_num.py:371-377: env.step ignores the incoming action and calls
robot.act(last_human_states)).  A scalar restatement on top of oracle/crowd_env.py, with ORCA through oracle/rvo2_ref.cpp;
pinned against the reference by the robot goldens of tools/make_golden.py (tests/test_robot_policy.py)."""
import numpy as np

from oracle.crowd_env import CrowdEnvOracle, _norm2, rvo2


class RobotPolicyOracle(CrowdEnvOracle):
    """CrowdEnvOracle with robot.policy = `robot_policy` ('orca' | 'social_force')."""

    def __init__(self, cfg, this_seed, nenv, phase="train", robot_policy="orca"):
        if robot_policy not in ("orca", "social_force"):
            raise ValueError("robot_policy must be 'orca' or 'social_force'")
        if cfg.human_num_range or cfg.predict_method != "none":
            raise ValueError("the robot policies are restated for CrowdSimVarNum-v0 with human_num_range 0")
        super().__init__(cfg, this_seed, nenv, phase)
        self.robot_policy = robot_policy
        # the robot's rvo2 simulator: robot.policy is created once per env process (crowd_sim.py:184) and its simulator
        # is never rebuilt (the agent count stays H + 1), so it outlives every reset
        self.robot_sim = None

    def _robot_act(self):
        """robot.act(last_human_states) (crowd_sim_var_num.py:371-377): ORCA.predict (orca.py:64-117) with the robot as
        agent 0 of its own persistent simulator, or SOCIAL_FORCE.predict (social_force.py:11-49).  The neighbours are the
        belief rows as they are, (15, 15, 0, 0, 0.3) rows and dead-reckoned unseen humans included."""
        c = self.cfg
        hs = self.last_human_states.tolist()
        if self.robot_policy == "social_force":
            dx, dy = self.rgx - self.rpx, self.rgy - self.rpy
            dist = np.sqrt(dx ** 2 + dy ** 2)
            dvx = c.sf_KI * ((dx / dist) * c.robot_v_pref - self.rvx)
            dvy = c.sf_KI * ((dy / dist) * c.robot_v_pref - self.rvy)
            ivx = ivy = 0
            for ox, oy, _, _, orad in hs:
                ex, ey = self.rpx - ox, self.rpy - oy
                d = np.sqrt(ex ** 2 + ey ** 2)
                ivx += c.sf_A * np.exp((c.robot_radius + orad - d) / c.sf_B) * (ex / d)
                ivy += c.sf_A * np.exp((c.robot_radius + orad - d) / c.sf_B) * (ey / d)
            nvx = self.rvx + (dvx + ivx) * c.time_step
            nvy = self.rvy + (dvy + ivy) * c.time_step
            nrm = np.linalg.norm([nvx, nvy])
            if nrm > c.robot_v_pref:
                return nvx / nrm * c.robot_v_pref, nvy / nrm * c.robot_v_pref
            return nvx, nvy
        sim = self.robot_sim
        if sim is None:
            params = (self.nd_global, len(hs), c.orca_time_horizon, c.orca_time_horizon)
            sim = self.robot_sim = rvo2.PyRVOSimulator(c.time_step, *params, c.robot_radius, 1)
            sim.addAgent((self.rpx, self.rpy), *params, c.robot_radius + 0.01 + c.orca_safety_space, c.robot_v_pref,
                         (self.rvx, self.rvy))
            for px, py, vx, vy, r in hs:
                sim.addAgent((px, py), *params, r + 0.01 + c.orca_safety_space, 1, (vx, vy))
        else:
            sim.setAgentPosition(0, (self.rpx, self.rpy))
            sim.setAgentVelocity(0, (self.rvx, self.rvy))
            for k, (px, py, vx, vy, _) in enumerate(hs):
                sim.setAgentPosition(k + 1, (px, py))
                sim.setAgentVelocity(k + 1, (vx, vy))
        velocity = np.array((self.rgx - self.rpx, self.rgy - self.rpy))
        speed = np.linalg.norm(velocity)
        pref_vel = velocity / speed if speed > 1 else velocity
        sim.setAgentPrefVelocity(0, tuple(pref_vel))
        for k in range(len(hs)):
            sim.setAgentPrefVelocity(k + 1, (0, 0))
        sim.doStep()
        return sim.getAgentVelocity(0)

    def step(self, action):
        """CrowdEnvOracle.step with the robot's own velocity instead of the clipped `action` (which is ignored).
        The velocity is applied as computed: an ORCA result is not clipped, a social-force one stays fp64."""
        c, H = self.cfg, self.H
        avx, avy = self._robot_act()
        self.last_robot_action = (avx, avy)
        human_actions = self._human_actions()
        self.last_sim_actions = human_actions
        if self.phase == "test":
            self._truth_future_traj()
        reward, done, info, min_danger = self._calc_reward()
        self.rpx = self.rpx + avx * c.time_step
        self.rpy = self.rpy + avy * c.time_step
        self.rvx, self.rvy = avx, avy
        for i, (vx, vy) in enumerate(human_actions):
            self.hpx[i] = self.hpx[i] + vx * c.time_step
            self.hpy[i] = self.hpy[i] + vy * c.time_step
            self.hvx[i], self.hvy[i] = vx, vy
        self.global_time += c.time_step
        self.step_counter += 1
        ob = self._generate_ob(reset=False)
        if c.random_goal_changing and self.global_time % 5 == 0:
            self._update_goals_randomly()
        if c.end_goal_changing:
            for i in range(H):
                if _norm2(self.hgx[i] - self.hpx[i], self.hgy[i] - self.hpy[i]) < self.hrad[i]:
                    px, py, v_pref, radius = self._circle_crossing_human()
                    self.hpx[i], self.hpy[i], self.hgx[i], self.hgy[i] = px, py, -px, -py
                    self.hvx[i], self.hvy[i] = 0, 0
                    self.hvpref[i], self.hrad[i] = v_pref, radius
                    self.sims[i] = None
        self.last_human_actions = human_actions
        return ob, reward, done, {"info": info, "min_danger": min_danger}
