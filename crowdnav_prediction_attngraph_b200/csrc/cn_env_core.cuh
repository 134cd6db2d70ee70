// Per-environment step / reset / observation logic of the crowd simulator, written as
// "phase" functions for the (environment, human) thread mapping of the step kernel.
//
// Follows the reference's order of operations exactly (see DESIGN.md §path):
//   crowd_sim/envs/crowd_sim_pred.py:100-213       CrowdSimPred.step
//   crowd_sim/envs/crowd_sim_var_num.py:303-363    reset / generate_robot_humans
//   crowd_sim/envs/crowd_sim_var_num.py:465-561    calc_reward (train phase) + crowd_sim_pred.py:216-233
//   crowd_sim/envs/crowd_sim_pred.py:62-97         generate_ob  (VarNum: crowd_sim_var_num.py:233-279)
//   crowd_sim/envs/crowd_sim.py:243-273,513-572    belief update / visibility
//   crowd_sim/envs/crowd_sim.py:415-450            update_human_goals_randomly
//   crowd_sim/envs/crowd_sim_var_num.py:116-146    generate_circle_crossing_human
//   crowd_nav/policy/orca.py:64-117                per-human cached rvo2 simulator
//   crowd_nav/policy/srnn.py:17-33                 clip_action (fp32)
//
// Numeric conventions (what makes done/collision masks bit-exact against the oracle):
//   * positions, goals, radii, potential, reward: fp64, same expression trees as the Python;
//   * numpy's 1-D `norm((a, b))` is sqrt(dot) with dot = fma(b, b, a*a)  -> cn_norm_dot();
//     numpy's axis-norm and fp32 dot are plain a*a + b*b               -> cn_norm_plain();
//   * ORCA in fp32 without contraction (cn_orca.cuh); this TU is built with --fmad=false.
//
// Between phases the caller synchronises the threads of one environment (block barrier
// on the GPU; a plain loop over humans in the CPU test harness).
#pragma once
#include "cn_common.cuh"
#include "cn_rng.cuh"
#include "cn_orca.cuh"

#define CN_PI 3.141592653589793
#define CN_MAX_SPAWN_TRIES 20000
// heavy (CTA-scope) rejection sampling: threads per try, and the warp-scope budget of tries before an event is deferred
#define CN_HEAVY_SUB 4
#define CN_HEAVY_THREADS 512
#define CN_DEFER_TRIES 136

// robot.visible code paths (cn_orca_build, cn_sf_action) exist only in the step kernel's VIS instantiations, so the
// network policy's kernels without a visible robot carry none of them.  The host build of this header (the test
// harness) keeps them all and lets CnParams::robot_visible decide at run time.
#if defined(__CUDA_ARCH__)
#define CN_VIS(VIS) (VIS)
#else
#define CN_VIS(VIS) true
#endif

CN_HD double cn_fma(double a, double b, double c) {
#if defined(__CUDA_ARCH__)
  return __fma_rn(a, b, c);
#else
  return fma(a, b, c);
#endif
}
CN_HD double cn_norm_dot(double x, double y) { return sqrt(cn_fma(y, y, x * x)); }
CN_HD double cn_norm_plain(double x, double y) { return sqrt(x * x + y * y); }
CN_HD double cn_dot2(double a0, double a1, double b0, double b1) { return cn_fma(a1, b1, a0 * b0); }

// phase-dependent constants (crowd_sim.py:103-105, crowd_sim_var_num.py:329-334).  phase: 0 'train', 2 'test'.
// Call after P / time_step / pred_dt are set.
inline void cn_fill_phase(CnParams& p, int phase, int val_size, int test_size) {
  (void)val_size;
  p.test_phase = (phase == 2) ? 1 : 0;
  p.phase_offset = p.test_phase ? 1000u : 2000u;
  p.case_size = p.test_phase ? (uint32_t)(test_size > 0 ? test_size : 1) : (4294967295u - 2000u);
  int interval = (int)floor(p.pred_dt / p.time_step + 0.5);
  if (interval < 1) interval = 1;
  p.pred_interval = interval;
  p.lookahead_steps = p.P * interval;
}

// Working set of ONE environment while a step is in flight (shared memory on the GPU).
struct CnEnvSh {
  // human arrays, length H
  double *px, *py, *gx, *gy, *rad, *vpref;
  float *vx, *vy;        // current velocities (fp32-valued)
  double *wx, *wy, *nwx, *nwy;   // social-force humans only: current / new velocity in fp64 (null otherwise)
  float *fx, *fy;        // positions narrowed to fp32 (what the Cython boundary hands to rvo2)
  float *nvx, *nvy;      // ORCA output
  double *t0;            // scratch: closest distance / sort key
  double *t1;            // scratch: per-human future penalty
  uint8_t *visr;         // visible to the robot
  // robot + scalars
  double rpx, rpy, rgx, rgy;
  float rvx, rvy;
  double rwx, rwy;       // social-force robot: fp64 velocity (state) and the one computed for this step
  double nrwx, nrwy;
  float ax, ay;          // clipped action (or the robot policy's velocity)
  double reward;
  int done, info, reset_flag;
  int nvis;
  int hn;                // live humans of this environment (slots [hn, H) are empty; == H unless sim.human_num_range > 0)
  int goal_flag;         // some human is within its radius of its goal (respawn pending)
  int lp3_cost;          // humans of this environment whose solve fell through to linearProgram3 (balancing)
  int lean;              // step kernel: gx / gy / rad / vpref point straight into HBM (read-only there)
};

CN_HD size_t cn_idx(const CnParams& p, int e, int h) { return (size_t)e * p.H + h; }

// ------------------------------------------------------------------------------------------
// visibility helpers (crowd_sim.py:513-552)
CN_HD bool cn_in_fov(double x1, double y1, double vx1, double vy1, double x2, double y2, double fov) {
  if (fov >= 2.0 * CN_PI) {
    // offset = arccos(.) in [0, pi] <= fov/2 unless NaN (coincident centres -> 0/0)
    return !(x1 == x2 && y1 == y2);
  }
  const double th = atan2(vy1, vx1);
  double f0 = cos(th), f1 = sin(th);
  double d0 = x2 - x1, d1 = y2 - y1;
  const double nf = cn_norm_dot(f0, f1), nd = cn_norm_dot(d0, d1);
  f0 = f0 / nf; f1 = f1 / nf; d0 = d0 / nd; d1 = d1 / nd;
  double c = cn_dot2(f0, f1, d0, d1);
  if (c != c) return false;
  c = c < -1.0 ? -1.0 : (c > 1.0 ? 1.0 : c);
  return fabs(acos(c)) <= fov / 2;
}

// ------------------------------------------------------------------------------------------
// Robot policy inside the step (robot_policy != 0; crowd_sim_var_num.py:371-377: the env ignores the incoming action and
// calls robot.act(last_human_states)).  Leader thread, serial, at the end of cn_phase_load of a step, on the state the
// previous step left behind: the robot's position / velocity just loaded into s and its belief rows bpx..brad in HBM,
// which the step rewrites only in cn_phase_obs_a, after the reward.  Sets s.ax / s.ay (fp32 velocity) and, for social
// force, s.nrwx / s.nrwy (fp64), which cn_phase_reward integrates.
//
// 'orca' (crowd_nav/policy/orca.py:64-117, the robot as agent 0 of its own rvo2 simulator): neighbours are ALL H belief
// rows narrowed to float, including the (15, 15, 0, 0, 0.3) rows and the dead-reckoned rows of unseen humans (no FOV
// test, no (7, 7) dummy); maxNeighbors = H; own radius robot.radius + 0.01 + safety_space, maxSpeed robot.v_pref; the
// other radii and neighborDist are frozen when the simulator is created (rsim_*); the result is applied unclipped.
// 'social_force' (crowd_nav/policy/social_force.py): pull towards the goal with v_pref, push from every belief row, fp64
// in the reference's expression order, speed clipped to v_pref.
template <int MAXH>
CN_HD_NOINLINE void cn_robot_act(const CnParams& p, const CnState& g, CnEnvSh& s, int e) {
  const int H = p.H;
  const size_t row = (size_t)e * H;
  if (p.robot_policy == 2) {
    const double px = s.rpx, py = s.rpy, vx = s.rwx, vy = s.rwy, vp = p.robot_vpref;
    const double dx = s.rgx - px, dy = s.rgy - py;
    const double dist = sqrt(dx * dx + dy * dy);
    const double dvx = p.sf_KI * ((dx / dist) * vp - vx);
    const double dvy = p.sf_KI * ((dy / dist) * vp - vy);
    double ivx = 0.0, ivy = 0.0;
    for (int j = 0; j < H; ++j) {
      const double ex = px - g.bpx[row + j], ey = py - g.bpy[row + j];
      const double d = sqrt(ex * ex + ey * ey);
      const double w = p.sf_A * exp((p.robot_radius + g.brad[row + j] - d) / p.sf_B);
      ivx += w * (ex / d);
      ivy += w * (ey / d);
    }
    double nvx = vx + (dvx + ivx) * p.time_step;
    double nvy = vy + (dvy + ivy) * p.time_step;
    const double nrm = cn_norm_dot(nvx, nvy);                  // np.linalg.norm([new_vx, new_vy])
    if (nrm > vp) { nvx = nvx / nrm * vp; nvy = nvy / nrm * vp; }
    s.nrwx = nvx; s.nrwy = nvy;
    s.ax = (float)nvx; s.ay = (float)nvy;
    return;
  }
  const double pad = 0.01;
  if (!g.rsim_exists[e]) {                                     // first solve of this environment: create the simulator
    g.rsim_nd[e] = (float)g.nd_global[e];
    for (int j = 0; j < H; ++j) g.rsim_rother[row + j] = (float)(g.brad[row + j] + pad + p.orca_safety_space);
    g.rsim_exists[e] = 1;
  }
  const float nd = g.rsim_nd[e];
  const float rself = (float)(p.robot_radius + pad + p.orca_safety_space);
  const float vmax = (float)p.robot_vpref;
  const double dvx = s.rgx - s.rpx, dvy = s.rgy - s.rpy;
  const double speed = cn_norm_dot(dvx, dvy);
  const CnF2 pref = speed > 1 ? f2((float)(dvx / speed), (float)(dvy / speed)) : f2((float)dvx, (float)dvy);
  const CnF2 pos = f2((float)s.rpx, (float)s.rpy);
  const CnF2 vel = f2(s.rvx, s.rvy);
  const float rangeSq = nd * nd;
  const float invTimeHorizon = 1.0f / p.orca_time_horizon;
  const float timeStep = (float)p.time_step;
  // neighbours inside neighborDist, ascending distance, ties in index order; counting rank as in cn_orca_build
  float vd[MAXH];
  uint8_t vj[MAXH];
  int nl = 0;
  for (int j = 0; j < H; ++j) {
    const float d = f2abssq(f2sub(pos, f2((float)g.bpx[row + j], (float)g.bpy[row + j])));
    if (d < rangeSq) { vd[nl] = d; vj[nl] = (uint8_t)j; ++nl; }
  }
  CnLocalLines<MAXH> lines;
  for (int a = 0; a < nl; ++a) {
    const float da = vd[a];
    int rank = 0;
    for (int b = 0; b < nl; ++b) rank += (vd[b] < da || (vd[b] == da && b < a)) ? 1 : 0;
    const size_t i = row + vj[a];
    lines.set(rank, cn_orca_line(pos, vel, rself, f2((float)g.bpx[i], (float)g.bpy[i]), f2((float)g.bvx[i], (float)g.bvy[i]),
                                 g.rsim_rother[i], invTimeHorizon, timeStep));
  }
  CnF2 result;
  const int fail = cn_lp2(lines, nl, vmax, pref, false, result);
  if (fail < nl) cn_lp3<MAXH>(lines, nl, fail, vmax, result);
  s.ax = result.x; s.ay = result.y;
}

// ------------------------------------------------------------------------------------------
// Phase LOAD: every (env, human) thread loads its human; the leader (h == 0) loads the robot
// and clips the action (srnn.py:17-33, fp32), or with robot_policy != 0 runs the robot's own policy instead.
// ROBOT = false (the step kernel of a network policy) compiles the robot policy out; MAXH bounds its neighbour arrays.
template <int MAXH = 128, bool ROBOT = true>
CN_HD void cn_phase_load(const CnParams& p, const CnState& g, CnEnvSh& s, int e, int h,
                         const float* action /* [N,2] or null (reset) */) {
  const size_t i = cn_idx(p, e, h);
  s.px[h] = g.hpx[i]; s.py[h] = g.hpy[i];
  if (!s.lean) { s.gx[h] = g.hgx[i]; s.gy[h] = g.hgy[i]; s.rad[h] = g.hrad[i]; s.vpref[h] = g.hvpref[i]; }
  s.vx[h] = g.hvx[i]; s.vy[h] = g.hvy[i];
  if (p.social_force) { s.wx[h] = g.hwx[i]; s.wy[h] = g.hwy[i]; }
  s.fx[h] = (float)s.px[h]; s.fy[h] = (float)s.py[h];
  if (h == 0) {
    s.rpx = g.rpx[e]; s.rpy = g.rpy[e]; s.rgx = g.rgx[e]; s.rgy = g.rgy[e];
    s.rvx = g.rvx[e]; s.rvy = g.rvy[e];
    if (p.robot_policy == 2) { s.rwx = g.rwx[e]; s.rwy = g.rwy[e]; }
    s.done = 0; s.info = 0; s.reward = 0.0; s.reset_flag = 0; s.nvis = 0; s.goal_flag = 0; s.lp3_cost = 0;
    s.hn = g.hn[e];
    if (ROBOT && action && p.robot_policy) {
      cn_robot_act<MAXH>(p, g, s, e);
    } else if (action) {
      float ax = action[2 * e], ay = action[2 * e + 1];
      const float nrm = sqrtf(ax * ax + ay * ay);          // np.linalg.norm(float32[2])
      const float vp = (float)p.robot_vpref;
      if (nrm > vp) { ax = ax / nrm * vp; ay = ay / nrm * vp; }
      s.ax = ax; s.ay = ay;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Phase ORCA, part 1 (per thread = one human's rvo2 simulator, crowd_sim.py:680-703, orca.py:64-117):
// neighbour selection and ORCA half-plane construction into `lines` (sorted by distance).
// `mark`: value written to sim_exists for a simulator this call creates: 1, or 2 = PROVISIONAL when the solve runs ahead of
// the step it belongs to (pre-solve on the side stream, cn_env_kernels.cu): the finishing pass of that step promotes 2 / 3 -> 1;
// a full solve treats anything but 1 as missing, so an abandoned pre-solve (state uploaded in between) leaves no trace.
// VIS (robot.visible, crowd_sim.py:695-699): get_human_actions (use_fov) appends the robot -- or, outside the human's FOV,
// the dummy robot at (7, 7) with velocity 0 -- as the simulator's last agent, index hn; its radius is robot.radius either
// way.  The ground-truth look-ahead (use_fov = false) shows the humans only, so in phase 'test' the agent count alternates
// between hn + 1 and hn and every count change re-creates the simulator (orca.py:80-89).
template <int MAXH, bool VIS = false>
CN_HD void cn_orca_build(const CnParams& p, const CnState& g, CnEnvSh& s, int e, int h, CnLineStore lines, int& nl_out,
                         float& vmax_out, CnF2& pref_out, bool use_fov = true, uint8_t mark = 1) {
  const int H = p.H;            // slots (row pitch of the [N][H] arrays)
  const int hn = s.hn;          // live humans: the simulator of human h holds the other hn - 1 (orca.py:80-95)
  const size_t i = cn_idx(p, e, h);
  const double fov = p.human_fov;
  float nd, rself, vmax;
  const double pad = 0.01;
  const bool with_robot = CN_VIS(VIS) && p.robot_visible && use_fov;
  // --- cached simulator parameters (frozen at creation; orca.py:80-95 only updates pos/vel)
  if (p.randomize) {
    // (re)created when missing or when the agent count changed since its creation (orca.py:80-82): humans joined /
    // left, or (robot visible) the robot joined / left between get_human_actions and the look-ahead
    const uint8_t ex = g.sim_exists[i];
    const uint8_t count = (uint8_t)(hn + (with_robot ? 1 : 0));
    if (ex != 1 || ((p.hrange > 0 || CN_VIS(VIS)) && g.sim_n[i] != count)) {
      g.sim_n[i] = count;
      g.sim_nd[i] = (float)g.nd_global[e];
      g.sim_rself[i] = (float)(s.rad[h] + pad + p.orca_safety_space);
      g.sim_vmax[i] = (float)s.vpref[h];
      for (int j = 0; j < hn; ++j) {
        if (j == h) continue;
        // a simulator the look-ahead creates takes every human as is (no FOV dummies)
        const bool v = (CN_VIS(VIS) && !use_fov) || cn_in_fov(s.px[h], s.py[h], s.vx[h], s.vy[h], s.px[j], s.py[j], fov);
        g.sim_rother[i * H + j] = (float)((v ? s.rad[j] : 0.3) + pad + p.orca_safety_space);
      }
      // a pre-solve that RE-creates an official simulator (human count changed) marks it 3: still "exists" to a reader
      g.sim_exists[i] = mark == 2 ? ((ex == 1 || ex == 3) ? (uint8_t)3 : (uint8_t)2) : (uint8_t)1;
    }
    nd = g.sim_nd[i]; rself = g.sim_rself[i]; vmax = g.sim_vmax[i];
  } else {
    // non-randomised attributes never change, so the frozen-at-creation values equal these
    nd = (float)p.orca_neighbor_dist;
    rself = (float)(s.rad[h] + pad + p.orca_safety_space);
    vmax = (float)s.vpref[h];
    if (g.sim_exists[i] != 1) g.sim_exists[i] = mark;
  }
  // --- preferred velocity (orca.py:98-100), fp64 then narrowed
  const double dvx = s.gx[h] - s.px[h], dvy = s.gy[h] - s.py[h];
  const double speed = cn_norm_dot(dvx, dvy);
  const CnF2 pref = speed > 1 ? f2((float)(dvx / speed), (float)(dvy / speed)) : f2((float)dvx, (float)dvy);

  const CnF2 pos = f2(s.fx[h], s.fy[h]);
  const CnF2 vel = f2(s.vx[h], s.vy[h]);
  const float rangeSq = nd * nd;
  const float invTimeHorizon = 1.0f / p.orca_time_horizon;
  const float timeStep = (float)p.time_step;

  // --- neighbour selection: dist^2 < neighborDist^2, ascending, ties in insertion (index) order
  // (Agent::insertAgentNeighbor).  Pass 1 compresses the in-range neighbours; pass 2 ranks them by
  // counting (independent loads, no serial insertion chain through local memory) and builds each
  // ORCA line directly at its sorted position.
  float vd[MAXH];
  uint8_t vj[MAXH];          // bit 7 = dummy (invisible) neighbour, bits 0..6 = human index
  int nl = 0;
  for (int j = 0; j < hn; ++j) {
    if (j == h) continue;
    // use_fov = false: act_joint_state of the ground-truth look-ahead passes every other human as is
    const bool v = !use_fov || cn_in_fov(s.px[h], s.py[h], s.vx[h], s.vy[h], s.px[j], s.py[j], fov);
    const CnF2 op = v ? f2(s.fx[j], s.fy[j]) : f2(7.0f, 7.0f);     // dummy_human (crowd_sim.py:130-133)
    const float d = f2abssq(f2sub(pos, op));
    if (d < rangeSq) { vd[nl] = d; vj[nl] = (uint8_t)(j | (v ? 0 : 0x80)); ++nl; }
  }
  // the robot (VIS) is kept out of vd / vj: it is the last agent, so it ranks behind every human at an equal distance
  float rd = 0.0f;
  bool rin = false;
  if (with_robot) {
    const bool v = cn_in_fov(s.px[h], s.py[h], s.vx[h], s.vy[h], s.rpx, s.rpy, fov);
    const CnF2 op = v ? f2((float)s.rpx, (float)s.rpy) : f2(7.0f, 7.0f);        // dummy_robot (crowd_sim.py:135-139)
    const CnF2 ov = v ? f2(s.rvx, s.rvy) : f2(0.0f, 0.0f);
    rd = f2abssq(f2sub(pos, op));
    rin = rd < rangeSq;
    if (rin) {
      int rank = 0;
      for (int b = 0; b < nl; ++b) rank += (vd[b] <= rd) ? 1 : 0;
      lines.set(rank, cn_orca_line(pos, vel, rself, op, ov, (float)(p.robot_radius + pad + p.orca_safety_space),
                                   invTimeHorizon, timeStep));
    }
  }
  for (int a = 0; a < nl; ++a) {
    const float da = vd[a];
    int rank = (rin && rd < da) ? 1 : 0;
    for (int b = 0; b < nl; ++b) rank += (vd[b] < da || (vd[b] == da && b < a)) ? 1 : 0;
    const int j = vj[a] & 0x7f;
    const bool dummy = (vj[a] & 0x80) != 0;
    const CnF2 op = dummy ? f2(7.0f, 7.0f) : f2(s.fx[j], s.fy[j]);
    const CnF2 ov = dummy ? f2(0.0f, 0.0f) : f2(s.vx[j], s.vy[j]);
    const float orad = p.randomize ? g.sim_rother[i * H + j]
                                   : (float)((dummy ? 0.3 : s.rad[j]) + pad + p.orca_safety_space);
    lines.set(rank, cn_orca_line(pos, vel, rself, op, ov, orad, invTimeHorizon, timeStep));
  }
  nl_out = nl + (rin ? 1 : 0); vmax_out = vmax; pref_out = pref;
}

// Social-force humans (humans.policy = 'social_force', crowd_nav/policy/social_force.py:11-49): pull towards the goal
// with relaxation K_I, exponential push A exp((r_i + r_j - d) / B) from every other human (the ones outside the FOV are
// replaced by the dummy at (7, 7), crowd_sim.py:680-703), explicit Euler step, speed clipped to v_pref.  fp64 like the
// reference's Python floats, same expression order.  Writes s.nwx / s.nwy and the robot-collision distance.
// VIS (robot.visible): the robot, or outside the FOV the dummy robot at (7, 7), pushes too, radius robot.radius; it is
// the last term of the sum.
template <bool VIS = false>
CN_HD void cn_sf_action(const CnParams& p, const CnState& g, CnEnvSh& s, int e, int h, bool use_fov = true) {
  const int hn = s.hn;
  const double px = s.px[h], py = s.py[h], vx = s.wx[h], vy = s.wy[h];
  const double dx = s.gx[h] - px, dy = s.gy[h] - py;
  const double dist = sqrt(dx * dx + dy * dy);
  const double dvx = p.sf_KI * ((dx / dist) * s.vpref[h] - vx);
  const double dvy = p.sf_KI * ((dy / dist) * s.vpref[h] - vy);
  double ivx = 0.0, ivy = 0.0;
  for (int j = 0; j < hn; ++j) {
    if (j == h) continue;
    const bool v = !use_fov || cn_in_fov(px, py, vx, vy, s.px[j], s.py[j], p.human_fov);
    const double ox = v ? s.px[j] : 7.0, oy = v ? s.py[j] : 7.0, orad = v ? s.rad[j] : 0.3;
    const double ex = px - ox, ey = py - oy;
    const double d = sqrt(ex * ex + ey * ey);
    const double w = p.sf_A * exp((s.rad[h] + orad - d) / p.sf_B);
    ivx += w * (ex / d);
    ivy += w * (ey / d);
  }
  if (CN_VIS(VIS) && p.robot_visible && use_fov) {
    const bool v = cn_in_fov(px, py, vx, vy, s.rpx, s.rpy, p.human_fov);
    const double ex = px - (v ? s.rpx : 7.0), ey = py - (v ? s.rpy : 7.0);
    const double d = sqrt(ex * ex + ey * ey);
    const double w = p.sf_A * exp((s.rad[h] + p.robot_radius - d) / p.sf_B);
    ivx += w * (ex / d);
    ivy += w * (ey / d);
  }
  double nvx = vx + (dvx + ivx) * p.time_step;
  double nvy = vy + (dvy + ivy) * p.time_step;
  const double nrm = cn_norm_dot(nvx, nvy);                  // np.linalg.norm([new_vx, new_vy])
  if (nrm > s.vpref[h]) { nvx = nvx / nrm * s.vpref[h]; nvy = nvy / nrm * s.vpref[h]; }
  s.nwx[h] = nvx; s.nwy[h] = nvy;
  s.nvx[h] = (float)nvx; s.nvy[h] = (float)nvy;
  const size_t i = cn_idx(p, e, h);
  g.last_hvx[i] = (float)nvx; g.last_hvy[i] = (float)nvy; g.orca_nlines[i] = 0; g.orca_fail[i] = -1;
  const double rx = px - s.rpx, ry = py - s.rpy;
  s.t0[h] = sqrt(rx * rx + ry * ry) - s.rad[h] - p.robot_radius;
}

// Diagnostics of the LAST ORCA solve of a human's simulator (what reading the reference's rvo2 sims after a
// step shows; in the test phase that is the final look-ahead solve).
CN_HD void cn_orca_diag(const CnParams& p, const CnState& g, int e, int h, CnF2 result, int nl, int fail) {
  const size_t i = cn_idx(p, e, h);
  g.last_hvx[i] = result.x; g.last_hvy[i] = result.y;
  g.orca_nlines[i] = nl; g.orca_fail[i] = fail;
}

// Ground-truth look-ahead bookkeeping (calc_human_future_traj('truth') + the 'future' danger zone,
// crowd_sim_var_num.py:180-228,495-511, crowd_sim_pred.py:216-233): one human's kept future position k
// (1-based) against the robot's CURRENT position.  Humans the robot does not see sit at (15, 15).
struct CnLookahead {
  double min_rd;     // min distance among intruding future positions (+inf: none)
  double pen;        // min over k of [intrusion] * collision_penalty / 2^(k+1)  (<= 0)
};
CN_HD void cn_lookahead_accumulate(const CnParams& p, const CnEnvSh& s, bool visible, double x, double y, int k,
                                   CnLookahead& la) {
  const double rx = (visible ? x : 15.0) - s.rpx, ry = (visible ? y : 15.0) - s.rpy;
  const double rd = cn_norm_plain(rx, ry);                    // np.linalg.norm(axis=-1): no fma
  if (rd < p.robot_radius + p.human_radius) {
    la.min_rd = rd < la.min_rd ? rd : la.min_rd;
    double coef = 2.0;
    for (int q = 0; q < k; ++q) coef = coef * 2.0;            // 2^(k+1)
    const double c = p.collision_penalty / coef;
    la.pen = c < la.pen ? c : la.pen;
  }
}

// Phase ORCA, part 3 (per thread): publish the solved velocity + the robot-collision distance.
CN_HD void cn_orca_finish(const CnParams& p, const CnState& g, CnEnvSh& s, int e, int h, CnF2 result, int nl, int fail) {
  const size_t i = cn_idx(p, e, h);
  s.nvx[h] = result.x; s.nvy[h] = result.y;
  cn_orca_diag(p, g, e, h, result, nl, fail);
  // collision distance to the robot for calc_reward (state BEFORE the action is applied)
  const double dx = s.px[h] - s.rpx, dy = s.py[h] - s.rpy;
  s.t0[h] = sqrt(dx * dx + dy * dy) - s.rad[h] - p.robot_radius;
}

// ------------------------------------------------------------------------------------------
// Phase REWARD (leader): calc_reward + robot integration + time.
CN_HD void cn_phase_reward(const CnParams& p, const CnState& g, CnEnvSh& s, int e, const CnStepOut& out) {
  const int H = s.hn;           // live humans
  double dmin = INFINITY;
  bool collision = false;
  for (int i = 0; i < H; ++i) {
    double c;
    if (p.test_phase) {        // t0 carries the look-ahead's min distance there: closest distance recomputed
      const double dx = s.px[i] - s.rpx, dy = s.py[i] - s.rpy;
      c = sqrt(dx * dx + dy * dy) - s.rad[i] - p.robot_radius;
    } else {
      c = s.t0[i];
    }
    if (c < 0) { collision = true; break; }
    else if (c < dmin) dmin = c;
  }
  const bool reaching_goal = cn_norm_dot(s.rpx - s.rgx, s.rpy - s.rgy) < p.robot_radius;
  bool danger;
  double min_danger = 0.0, fut_pen;
  if (p.test_phase) {
    // 'future' danger zone on the ground-truth look-ahead (crowd_sim_var_num.py:495-511)
    double mr = INFINITY, pen = 0.0;
    for (int i = 0; i < H; ++i) { mr = s.t0[i] < mr ? s.t0[i] : mr; pen = s.t1[i] < pen ? s.t1[i] : pen; }
    danger = mr < INFINITY;
    if (danger) min_danger = mr;
    fut_pen = pen;
  } else {
    danger = dmin < p.discomfort_dist;                        // phase == 'train' (crowd_sim_var_num.py:495-497)
    fut_pen = g.fut_pen[e];
  }
  const int step = g.step_count[e];
  const double global_time = step * p.time_step;
  double reward; int done, info;
  if (global_time >= p.time_limit - 1) { reward = 0; done = 1; info = CN_INFO_TIMEOUT; }
  else if (collision) { reward = p.collision_penalty; done = 1; info = CN_INFO_COLLISION; }
  else if (reaching_goal) { reward = p.success_reward; done = 1; info = CN_INFO_REACHGOAL; }
  else if (danger) {
    reward = (dmin - p.discomfort_dist) * p.discomfort_penalty_factor * p.time_step;
    done = 0; info = CN_INFO_DANGER;
  } else {
    const double pot = cn_norm_dot(s.rpx - s.rgx, s.rpy - s.rgy);
    reward = 2 * (-fabs(pot) - g.potential[e]);
    g.potential[e] = -fabs(pot);
    done = 0; info = CN_INFO_NOTHING;
  }
  if (p.const_vel) reward = reward + fut_pen;                 // crowd_sim_pred.py:216-233
  s.reward = reward; s.done = done; s.info = info;
  // Monitor bookkeeping + outputs
  const double ret = g.ep_ret[e] + reward;
  const int len = g.ep_len[e] + 1;
  g.ep_ret[e] = ret; g.ep_len[e] = len;
  out.reward[e] = (float)reward;
  out.done[e] = (uint8_t)done;
  out.info[e] = info;
  out.info_aux[e] = (info == CN_INFO_DANGER) ? (float)min_danger : 0.0f;     // Danger(min_dist)
  if (out.not_done) out.not_done[e] = done ? 0.0f : 1.0f;
  if (done) { out.ep_ret[e] = ret; out.ep_len[e] = len; }
  // robot.step(action) (agent.py:170-183); time
  if (p.robot_policy == 2) {
    s.rpx = s.rpx + s.nrwx * p.time_step;
    s.rpy = s.rpy + s.nrwy * p.time_step;
    s.rwx = s.nrwx; s.rwy = s.nrwy;
  } else {
    s.rpx = s.rpx + (double)s.ax * p.time_step;
    s.rpy = s.rpy + (double)s.ay * p.time_step;
  }
  s.rvx = s.ax; s.rvy = s.ay;
  g.step_count[e] = step + 1;
}

// Phase INTEGRATE (per human): humans[i].step(human_action).
CN_HD void cn_phase_integrate(const CnParams& p, CnEnvSh& s, int h) {
  if (p.social_force) {
    s.px[h] = s.px[h] + s.nwx[h] * p.time_step;
    s.py[h] = s.py[h] + s.nwy[h] * p.time_step;
    s.wx[h] = s.nwx[h]; s.wy[h] = s.nwy[h];
    s.vx[h] = (float)s.nwx[h]; s.vy[h] = (float)s.nwy[h];
  } else {
    s.px[h] = s.px[h] + (double)s.nvx[h] * p.time_step;
    s.py[h] = s.py[h] + (double)s.nvy[h] * p.time_step;
    s.vx[h] = s.nvx[h]; s.vy[h] = s.nvy[h];
  }
  // end-goal respawn is due when a human is within its radius of its goal (crowd_sim_pred.py:207-211);
  // the RNG-consuming work itself runs in the event kernel.  (benign race: all writers store 1)
  if (p.end_goal_changing && cn_norm_dot(s.gx[h] - s.px[h], s.gy[h] - s.py[h]) < s.rad[h]) s.goal_flag = 1;
}

// Event flag of one environment after the step (leader): 2 = finished, 1 = goal dynamics pending.
CN_HD int cn_event_flag(const CnParams& p, const CnState& g, const CnEnvSh& s, int e) {
  if (s.done) return 2;
  if (s.goal_flag) return 1;
  if (p.goal_changing && fmod(g.step_count[e] * p.time_step, 5.0) == 0.0) return 1;
  return 0;
}

// ------------------------------------------------------------------------------------------
// RNG-consuming pieces (leader thread only, serial — they share one MT19937 stream).
struct CnSpawn { double px, py, vpref, rad; };

CN_HD void cn_new_human_attrs(const CnParams& p, CnRng& rng, const CnCoop& co, double& nd_global, double& vpref,
                              double& rad) {
  vpref = p.human_vpref; rad = p.human_radius;
  if (p.randomize) {                      // agent.py:20-23 then agent.py:44-50
    nd_global = cn_rng_uniform(rng, co, 5, 10);
    vpref = cn_rng_uniform(rng, co, 0.5, 1.5);
    rad = cn_rng_uniform(rng, co, 0.3, 0.5);
  }
}

// Rejection sampling of a point near the circle that keeps `rad_i + r_k + discomfort_dist` clear of the
// position AND the goal of the robot and of humans [0, n) except `skip`
// (crowd_sim_var_num.py:116-146 spawn: noise = U[0,1)*2; crowd_sim.py:415-450 goal change: noise =
// (U[0,1) - 0.5) * v_pref).  Every try consumes exactly three random_sample() = six MT19937 words, so a
// warp evaluates up to 32 CONSECUTIVE tries at once (lane j peeks at words [pos + 6j, pos + 6j + 6),
// checks its candidate against every agent) and accepts the first free one: same result and same
// stream position as the sequential loop.  Near the 624-word twist boundary (and in the single-thread
// host build) it falls back to one try at a time with a lane-strided scan.
// The reference loops forever when no free spot exists (it cannot place more than ~76 humans); a
// kernel must not hang, so try number CN_MAX_SPAWN_TRIES is accepted as is and the environment flagged.
struct CnCand { double x, y; };
CN_HD bool cn_cand_collides(const CnParams& p, const CnEnvSh& s, double x, double y, double rad_i, int k) {
  double ax, ay, agx, agy, ar;
  if (k < 0) { ax = s.rpx; ay = s.rpy; agx = s.rgx; agy = s.rgy; ar = p.robot_radius; }
  else { ax = s.px[k]; ay = s.py[k]; agx = s.gx[k]; agy = s.gy[k]; ar = s.rad[k]; }
  const double min_dist = rad_i + ar + p.discomfort_dist;
  // exact predicate: np.linalg.norm(d) < min_dist for the position AND the goal of agent k.
  // (1) fp32 screen: coordinates are below ~25 m, so an fp32 squared distance is within 1e-4 (abs, near the threshold)
  //     resp. 3e-7 (rel, far away) of the exact one; anything farther than 1e-3 (1 + d2) from the threshold is decided
  //     here -- that is > 99.9 % of the tests, and these searches are latency-bound chains of fp64 instructions.
  {
    const float m2f = (float)(min_dist * min_dist);
    const float fx = (float)x, fy = (float)y;
    const float dxf = fx - (float)ax, dyf = fy - (float)ay, exf = fx - (float)agx, eyf = fy - (float)agy;
    const float d2f = dxf * dxf + dyf * dyf, e2f = exf * exf + eyf * eyf;
    const float md = 1e-3f * (1.0f + d2f), me = 1e-3f * (1.0f + e2f);
    if (d2f < m2f - md || e2f < m2f - me) return true;
    if (d2f > m2f + md && e2f > m2f + me) return false;
  }
  // (2) fp64 squared distances decide every case that is not within 1e-14 (relative) of the boundary without the
  //     square root; (3) the boundary band takes the reference's exact expression.
  const double m2 = min_dist * min_dist, lo = m2 * (1.0 - 1e-14), hi = m2 * (1.0 + 1e-14);
  const double dx = x - ax, dy = y - ay, ex = x - agx, ey = y - agy;
  const double d2 = dx * dx + dy * dy, e2 = ex * ex + ey * ey;
  if (d2 < lo || e2 < lo) return true;
  if (d2 > hi && e2 > hi) return false;
  return cn_norm_dot(dx, dy) < min_dist || cn_norm_dot(ex, ey) < min_dist;
}
CN_HD CnCand cn_cand_point(const CnParams& p, double u0, double u1, double u2, int goal_kind, double vp) {
  const double angle = u0 * CN_PI * 2;
  const double nx = goal_kind ? (u1 - 0.5) * vp : u1 * 2;
  const double ny = goal_kind ? (u2 - 0.5) * vp : u2 * 2;
  CnCand c;
#if defined(__CUDA_ARCH__)
  double sn, cs;
  sincos(angle, &sn, &cs);            // one argument reduction for both (same values as sin() / cos())
#else
  const double sn = sin(angle), cs = cos(angle);
#endif
  c.x = p.circle_radius * cs + nx;
  c.y = p.circle_radius * sn + ny;
  return c;
}
CN_HD CnCand cn_rejection_sample(const CnParams& p, const CnEnvSh& s, CnRng& rng, const CnCoop& co, int goal_kind, int n,
                                 int skip, double rad_i, double vp, uint8_t* overflow) {
  CnCand c; c.x = 0; c.y = 0;
  bool tab_ready = false;       // CTA scope: fp32 agent table of this search built
  for (int tries = 0;;) {
    // warp scope: a search that has used up its budget is handed to cn_env_event_heavy_kernel (warp-uniform exit)
    if (rng.budget > 0 && tries >= rng.budget) { rng.deferred = 1; return c; }
    int nb = (624 - rng.pos) / 6;                              // whole tries left before the next twist
    if (co.nlanes <= 32 && nb > co.nlanes) nb = co.nlanes;
    if (nb > CN_MAX_SPAWN_TRIES - tries + 1) nb = CN_MAX_SPAWN_TRIES - tries + 1;
#if defined(__CUDA_ARCH__)
    if (co.nlanes > 32 && nb >= 1) {
      // CTA scope (heavy path): all <= 104 tries up to the next twist at once, CN_HEAVY_SUB consecutive threads share
      // one try and split the agent list; the FIRST free try wins, exactly like the sequential loop.
      // These searches are mostly doomed (the crowd has filled the goal ring; the reference would spin forever, the
      // engine gives up after CN_MAX_SPAWN_TRIES), so what matters is the latency of one batch.  Measured with
      // clock64: 5 400 cycles per batch when every thread ran the fp64 path (fp64 sincos + dependent shared-memory
      // loads through the CnEnvSh pointers + early-exit loop).  Now an fp32 SCREEN runs first: candidate from sincosf,
      // agents from a flat fp32 table in shared memory (built once per search), no early exit (independent loads),
      // "surely collides" only when the fp32 squared distance is below the threshold by 1e-3 (1 + d2) -- 50x the
      // fp32 error.  Only candidates the screen cannot reject take the exact path.
      const int t = co.lane / CN_HEAVY_SUB, sub = co.lane - t * CN_HEAVY_SUB;
      if (nb > co.nlanes / CN_HEAVY_SUB) nb = co.nlanes / CN_HEAVY_SUB;
      float* tab = co.ftab;
      if (!tab_ready) {                                         // (first batch of this search) agent table: index k + 1
        tab_ready = true;
        for (int k = -1 + co.lane; k < n; k += co.nlanes) {
          double ax, ay, agx, agy, ar;
          if (k < 0) { ax = s.rpx; ay = s.rpy; agx = s.rgx; agy = s.rgy; ar = p.robot_radius; }
          else { ax = s.px[k]; ay = s.py[k]; agx = s.gx[k]; agy = s.gy[k]; ar = s.rad[k]; }
          const double md = rad_i + ar + p.discomfort_dist;
          tab[k + 1] = (float)ax; tab[CN_FTAB + k + 1] = (float)ay; tab[2 * CN_FTAB + k + 1] = (float)agx;
          tab[3 * CN_FTAB + k + 1] = (float)agy;
          tab[4 * CN_FTAB + k + 1] = (k == skip) ? -1.0f : (float)(md * md);     // skipped agent: can never collide
        }
      }
      if (co.lane == 0) { co.scratch[0] = 0x7fffffff; co.scratch[1] += 1; }      // scratch[1]: batches of this CTA (diagnostic)
      const long long tq0 = clock64();
      __syncthreads();
      bool sure = false;
      if (t < nb) {
        const int off = 6 * t;
        const double u0 = cn_rng_peek_double(rng, off), u1 = cn_rng_peek_double(rng, off + 2), u2 = cn_rng_peek_double(rng, off + 4);
        float sn, cs;
        sincosf((float)(u0 * CN_PI * 2), &sn, &cs);
        const float fx = (float)p.circle_radius * cs + (goal_kind ? ((float)u1 - 0.5f) * (float)vp : (float)u1 * 2.0f);
        const float fy = (float)p.circle_radius * sn + (goal_kind ? ((float)u2 - 0.5f) * (float)vp : (float)u2 * 2.0f);
        for (int k = sub; k < n + 1; k += CN_HEAVY_SUB) {
          const float dx = fx - tab[k], dy = fy - tab[CN_FTAB + k], ex = fx - tab[2 * CN_FTAB + k], ey = fy - tab[3 * CN_FTAB + k];
          const float m2 = tab[4 * CN_FTAB + k];
          const float d2 = dx * dx + dy * dy, e2 = ex * ex + ey * ey;
          sure = sure || (d2 < m2 - 1e-3f * (1.0f + d2)) || (e2 < m2 - 1e-3f * (1.0f + e2));
        }
      }
      const uint32_t gmask = ((1u << CN_HEAVY_SUB) - 1u) << ((threadIdx.x & 31) / CN_HEAVY_SUB * CN_HEAVY_SUB);
      const bool try_sure = (__ballot_sync(0xffffffffu, sure) & gmask) != 0;
      bool collide = false;
      if (t < nb && !try_sure) {                                // exact path for the few candidates the screen let through
        const int off = 6 * t;
        const CnCand cc = cn_cand_point(p, cn_rng_peek_double(rng, off), cn_rng_peek_double(rng, off + 2),
                                        cn_rng_peek_double(rng, off + 4), goal_kind, vp);
        for (int k = -1 + sub; k < n && !collide; k += CN_HEAVY_SUB)
          if (k != skip) collide = cn_cand_collides(p, s, cc.x, cc.y, rad_i, k);
      }
      const uint32_t m = __ballot_sync(0xffffffffu, collide);
      if (t < nb && sub == 0 && !try_sure && !(m & gmask)) atomicMin(co.scratch, t);
      __syncthreads();
      const int first = co.scratch[0];
      __syncthreads();
      if (co.lane == 0) co.scratch[2] += (int)((clock64() - tq0) >> 4);          // diagnostic: cycles / 16 in candidate batches
      const bool last = (tries + nb - 1 >= CN_MAX_SPAWN_TRIES);
      if (first != 0x7fffffff || last) {
        const int j = (first != 0x7fffffff) ? first : nb - 1;
        c = cn_cand_point(p, cn_rng_peek_double(rng, 6 * j), cn_rng_peek_double(rng, 6 * j + 2),
                          cn_rng_peek_double(rng, 6 * j + 4), goal_kind, vp);
        rng.pos += 6 * (j + 1);
        if (first == 0x7fffffff && co.lane == 0) *overflow = 1;
        return c;
      }
      rng.pos += 6 * nb; tries += nb;
      continue;
    }
#endif
    if (co.nlanes > 1 && co.nlanes <= 32 && nb >= 1) {
      // Warp scope.  Most searches succeed within the first few candidates (acceptance 0.3 - 0.5 in a 50-human crowd),
      // so evaluating 32 candidates at once wastes 10x the distance tests on the warp's critical path.  The first
      // batches therefore take 4 candidates x 8 lanes (each lane tests an eighth of the agents: a 4x shorter
      // dependent chain); a search that is still running after 8 candidates widens to 32 x 1.
      const int sub = (tries < 8) ? 8 : 1;                     // lanes per candidate
      const int nbt = (nb < co.nlanes / sub) ? nb : co.nlanes / sub;
      const int t = co.lane / sub, j = co.lane - t * sub;
      const uint32_t gmask = (sub == 32 ? 0xffffffffu : ((1u << sub) - 1u)) << (t * sub);
      bool try_sure = false;
#if defined(__CUDA_ARCH__)
      if (co.ftab) {
        // fp32 screen first (see the CTA-scope branch): flat agent table in shared memory, candidate from sincosf,
        // no early exit; only candidates it cannot reject run the exact fp64 path below
        float* tab = co.ftab;
        if (!tab_ready) {
          tab_ready = true;
          for (int k = -1 + co.lane; k < n; k += co.nlanes) {
            double ax, ay, agx, agy, ar;
            if (k < 0) { ax = s.rpx; ay = s.rpy; agx = s.rgx; agy = s.rgy; ar = p.robot_radius; }
            else { ax = s.px[k]; ay = s.py[k]; agx = s.gx[k]; agy = s.gy[k]; ar = s.rad[k]; }
            const double md = rad_i + ar + p.discomfort_dist;
            tab[k + 1] = (float)ax; tab[CN_FTAB + k + 1] = (float)ay; tab[2 * CN_FTAB + k + 1] = (float)agx;
            tab[3 * CN_FTAB + k + 1] = (float)agy;
            tab[4 * CN_FTAB + k + 1] = (k == skip) ? -1.0f : (float)(md * md);
          }
          __syncwarp();
        }
        bool sure = false;
        if (t < nbt) {
          const int off = 6 * t;
          const double u0 = cn_rng_peek_double(rng, off), u1 = cn_rng_peek_double(rng, off + 2), u2 = cn_rng_peek_double(rng, off + 4);
          float sn, cs;
          sincosf((float)(u0 * CN_PI * 2), &sn, &cs);
          const float fx = (float)p.circle_radius * cs + (goal_kind ? ((float)u1 - 0.5f) * (float)vp : (float)u1 * 2.0f);
          const float fy = (float)p.circle_radius * sn + (goal_kind ? ((float)u2 - 0.5f) * (float)vp : (float)u2 * 2.0f);
          for (int k = j; k < n + 1; k += sub) {
            const float dx = fx - tab[k], dy = fy - tab[CN_FTAB + k], ex = fx - tab[2 * CN_FTAB + k], ey = fy - tab[3 * CN_FTAB + k];
            const float m2 = tab[4 * CN_FTAB + k];
            const float d2 = dx * dx + dy * dy, e2 = ex * ex + ey * ey;
            sure = sure || (d2 < m2 - 1e-3f * (1.0f + d2)) || (e2 < m2 - 1e-3f * (1.0f + e2));
          }
        }
        try_sure = (__ballot_sync(0xffffffffu, sure) & gmask) != 0;
      }
#endif
      bool collide = try_sure;
      if (t < nbt && !try_sure) {
        const int off = 6 * t;
        c = cn_cand_point(p, cn_rng_peek_double(rng, off), cn_rng_peek_double(rng, off + 2),
                          cn_rng_peek_double(rng, off + 4), goal_kind, vp);
        for (int k = -1 + j; k < n && !collide; k += sub)
          if (k != skip) collide = cn_cand_collides(p, s, c.x, c.y, rad_i, k);
      }
      const uint32_t cm = cn_ballot(co, collide);
      const uint32_t free_mask = cn_ballot(co, t < nbt && j == 0 && !(cm & gmask));      // bit = first lane of a free try
      const bool last = (tries + nbt - 1 >= CN_MAX_SPAWN_TRIES);
      if (free_mask || last) {
        const int lane_j = free_mask ? cn_ffs(free_mask) : (nbt - 1) * sub;
        const int tj = lane_j / sub;
        // every lane recomputes the accepted candidate (a candidate accepted at the try limit may have been rejected
        // by the fp32 screen, in which case no lane holds its fp64 coordinates)
        c = cn_cand_point(p, cn_rng_peek_double(rng, 6 * tj), cn_rng_peek_double(rng, 6 * tj + 2),
                          cn_rng_peek_double(rng, 6 * tj + 4), goal_kind, vp);
        rng.pos += 6 * (tj + 1);
        if (!free_mask && co.lane == 0) *overflow = 1;
        return c;
      }
      rng.pos += 6 * nbt; tries += nbt;
    } else {
      const double u0 = cn_rng_double(rng, co), u1 = cn_rng_double(rng, co), u2 = cn_rng_double(rng, co);
      c = cn_cand_point(p, u0, u1, u2, goal_kind, vp);
      bool collide = false;
      for (int k = -1 + co.lane; k < n; k += co.nlanes) {
        if (k == skip) continue;
        if (cn_cand_collides(p, s, c.x, c.y, rad_i, k)) { collide = true; break; }
      }
      if (!cn_any(co, collide)) return c;
      if (tries >= CN_MAX_SPAWN_TRIES) { if (co.lane == 0) *overflow = 1; return c; }
      ++tries;
    }
  }
}

// generate_circle_crossing_human (crowd_sim_var_num.py:116-146) against robot + humans[0..n_present).
CN_HD CnSpawn cn_circle_crossing_human(const CnParams& p, const CnEnvSh& s, CnRng& rng, const CnCoop& co, int n_present,
                                       double& nd_global, uint8_t* overflow) {
  CnSpawn sp;
  cn_new_human_attrs(p, rng, co, nd_global, sp.vpref, sp.rad);
  const CnCand c = cn_rejection_sample(p, s, rng, co, 0, n_present, -2, sp.rad, 0.0, overflow);
  sp.px = c.x; sp.py = c.y;
  return sp;
}

// PREPARE the next episode of environment e (crowd_sim_var_num.py:303-363 up to generate_ob): seed the
// legacy MT19937 with the CURRENT case_counter, sample robot + humans into the scratch working set `s`
// and publish the result in g.prep_*.  Pure function of (seed, case_counter): it runs off the critical
// path.  `key` = 624-word scratch; every lane of `co` runs this function (replicated), lane 0 writes.
// Returns true when a rejection-sampling search exhausted `budget` tries (warp scope only): nothing was published and
// the caller hands the environment to the CTA-scope kernel, which redoes the preparation with budget 0.
CN_HD bool cn_prepare_env(const CnParams& p, const CnState& g, CnEnvSh& s, int e, uint32_t* key, const CnCoop& co,
                          int budget = 0) {
  const int H = p.H;
  CnRng rng; rng.key = key; rng.pos = 624; rng.budget = budget; rng.deferred = 0;
  const uint32_t cc = g.case_counter[e];
  const uint32_t this_seed = p.seed_base + (uint32_t)g.seed_off[e];
  cn_rng_seed(rng, p.phase_offset + cc + this_seed, co);
  for (;;) {
    const double px = cn_rng_uniform(rng, co, -p.arena_size, p.arena_size);
    const double py = cn_rng_uniform(rng, co, -p.arena_size, p.arena_size);
    const double gx = cn_rng_uniform(rng, co, -p.arena_size, p.arena_size);
    const double gy = cn_rng_uniform(rng, co, -p.arena_size, p.arena_size);
    if (cn_norm_dot(px - gx, py - gy) >= 8) {
      if (co.lane == 0) { s.rpx = px; s.rpy = py; s.rgx = gx; s.rgy = gy; }
      break;
    }
  }
  cn_coop_sync(co);
  double nd = g.nd_global[e];
  // human_num = randint(human_num - range, human_num + range + 1) (crowd_sim_var_num.py:103-104; no draw when range == 0)
  const int hn = p.hrange > 0 ? cn_rng_randint(rng, co, p.hbase - p.hrange, p.hbase + p.hrange + 1) : H;
  for (int i = 0; i < hn; ++i) {
    const CnSpawn sp = cn_circle_crossing_human(p, s, rng, co, i, nd, g.spawn_overflow + e);
    if (rng.deferred) return true;
    if (co.lane == 0) {
      s.px[i] = sp.px; s.py[i] = sp.py; s.gx[i] = -sp.px; s.gy[i] = -sp.py; s.rad[i] = sp.rad; s.vpref[i] = sp.vpref;
    }
    cn_coop_sync(co);
  }
  for (int i = co.lane; i < H; i += co.nlanes) {
    const size_t gi = cn_idx(p, e, i);
    const bool live = i < hn;       // empty slots: zeros
    g.prep_hpx[gi] = live ? s.px[i] : 0.0; g.prep_hpy[gi] = live ? s.py[i] : 0.0;
    g.prep_hrad[gi] = live ? s.rad[i] : 0.0; g.prep_hvpref[gi] = live ? s.vpref[i] : 0.0;
  }
  if (co.lane == 0) {
    double* r = g.prep_robot + (size_t)e * 4;
    r[0] = s.rpx; r[1] = s.rpy; r[2] = s.rgx; r[3] = s.rgy;
    g.prep_nd[e] = nd;
    g.prep_hn[e] = hn;
    g.prep_mt_pos[e] = rng.pos;
  }
  cn_coop_sync(co);
  return false;
}

// INSTALL the prepared episode (per human thread; the leader also installs the per-env scalars).
// Called for finished episodes right after the reward, and for every environment on a full reset.
CN_HD void cn_install_env(const CnParams& p, const CnState& g, CnEnvSh& s, int e, int h) {
  const int H = p.H;
  const size_t i = cn_idx(p, e, h);
  const double px = g.prep_hpx[i], py = g.prep_hpy[i];
  s.px[h] = px; s.py[h] = py; s.gx[h] = -px; s.gy[h] = -py;        // lean: gx / gy / rad / vpref alias HBM
  s.rad[h] = g.prep_hrad[i]; s.vpref[h] = g.prep_hvpref[i];
  s.vx[h] = 0.0f; s.vy[h] = 0.0f; s.fx[h] = (float)px; s.fy[h] = (float)py;
  if (p.social_force) { s.wx[h] = 0.0; s.wy[h] = 0.0; }
  g.sim_exists[i] = 0;
  g.bpx[i] = 0; g.bpy[i] = 0; g.bvx[i] = 0; g.bvy[i] = 0; g.brad[i] = 0;   // last_human_states = zeros
  for (int w = h; w < 624; w += H) g.mt[(size_t)e * 624 + w] = g.prep_mt[(size_t)e * 624 + w];
  if (h == 0) {
    const double* r = g.prep_robot + (size_t)e * 4;
    s.rpx = r[0]; s.rpy = r[1]; s.rgx = r[2]; s.rgy = r[3]; s.rvx = 0.0f; s.rvy = 0.0f; s.rwx = 0.0; s.rwy = 0.0;
    // the robot's rvo2 simulator (rsim_*) is NOT reset: robot.policy outlives the episode
    // case_counter = (case_counter + nenv) % case_size[phase]  (train: UINT32_MAX - 2000, test: env.test_size)
    g.case_counter[e] = (uint32_t)(((uint64_t)g.case_counter[e] + (uint64_t)p.nenv_total) % (uint64_t)p.case_size);
    g.potential[e] = -fabs(cn_norm_dot(s.rgx - s.rpx, s.rgy - s.rpy));
    g.step_count[e] = 0;
    g.ep_ret[e] = 0.0; g.ep_len[e] = 0;
    g.mt_pos[e] = g.prep_mt_pos[e];
    if (p.randomize) g.nd_global[e] = g.prep_nd[e];
    s.reset_flag = 1; s.nvis = 0; s.goal_flag = 0;
    s.hn = g.prep_hn[e]; g.hn[e] = s.hn;
  }
}

// Humans join / leave every 5 s of simulation (sim.human_num_range > 0): CrowdSimPred.step (crowd_sim_pred.py:165-194)
// and CrowdSimVarNum.step (crowd_sim_var_num.py:404-437), AFTER the agents moved and BEFORE the observation.
// Single thread (the environment's leader), generator state used in place (`key` = g.mt row of the environment):
// it runs once per 20 steps and environment, so it is not worth a cooperative version.  The LAST humans leave
// (never one the robot currently observes: CrowdSimVarNum only -- CrowdSimPred never refreshes observed_human_ids),
// joining humans spawn on the circle like at reset and are unknown to the robot (belief (15, 15, 0, 0, 0.3)).
CN_HD void cn_phase_add_remove(const CnParams& p, const CnState& g, CnEnvSh& s, int e) {
  const CnCoop co = {0, 1, nullptr, nullptr};
  CnRng rng; rng.key = g.mt + (size_t)e * 624; rng.pos = g.mt_pos[e]; rng.budget = 0; rng.deferred = 0;
  const int hn = s.hn, hmin = p.hbase - p.hrange;
  int hnew = hn;
  if (cn_rng_double(rng, co) < 0.5) {
    int max_seen = -1;
    if (!p.const_vel)
      for (int k = 0; k < hn; ++k) if (g.vis[cn_idx(p, e, k)]) max_seen = k;
    int remove_num;
    if (p.const_vel) {
      const int max_remove = max_seen < 0 ? hn - 1 : (hn - 1) - max_seen;
      remove_num = cn_rng_randint(rng, co, 0, (p.hrange < max_remove ? p.hrange : max_remove) + 1);
    } else {
      int max_remove = hn - hmin;
      if (max_seen >= 0 && (hn - 1) - max_seen < max_remove) max_remove = (hn - 1) - max_seen;
      remove_num = cn_rng_randint(rng, co, 0, max_remove + 1);
    }
    hnew = hn - remove_num;
  } else {
    const int add_num = cn_rng_randint(rng, co, 0, p.hrange + 1);
    double nd = g.nd_global[e];
    for (int i = hn; i < hn + add_num && i < p.H; ++i) {
      s.hn = i;                                   // the spawn checks the robot and humans [0, i)
      const CnSpawn sp = cn_circle_crossing_human(p, s, rng, co, i, nd, g.spawn_overflow + e);
      s.px[i] = sp.px; s.py[i] = sp.py; s.gx[i] = -sp.px; s.gy[i] = -sp.py; s.rad[i] = sp.rad; s.vpref[i] = sp.vpref;
      s.vx[i] = 0.0f; s.vy[i] = 0.0f; s.fx[i] = (float)sp.px; s.fy[i] = (float)sp.py;
      if (p.social_force) { s.wx[i] = 0.0; s.wy[i] = 0.0; }
      const size_t gi = cn_idx(p, e, i);
      g.bpx[gi] = 15.; g.bpy[gi] = 15.; g.bvx[gi] = 0.; g.bvy[gi] = 0.; g.brad[gi] = 0.3;
      g.vis[gi] = 0; g.sim_exists[gi] = 0;
      hnew = i + 1;
    }
    if (p.randomize) g.nd_global[e] = nd;
  }
  // departed humans take their simulators with them; the survivors' simulators are rebuilt lazily at their next solve
  // (agent-count mismatch, cn_orca_build), exactly when the reference does it
  for (int k = hnew; k < hn; ++k) g.sim_exists[cn_idx(p, e, k)] = 0;
  s.hn = hnew; g.hn[e] = hnew;
  g.mt_pos[e] = rng.pos;
}
CN_HD bool cn_add_remove_due(const CnParams& p, const CnState& g, const CnEnvSh& s, int e) {
  return p.hrange > 0 && !s.done && fmod(g.step_count[e] * p.time_step, 5.0) == 0.0;
}

// ------------------------------------------------------------------------------------------
// Phase OBS-A (per human): robot visibility, belief update, prediction, sort key, future penalty.
// Writes the fp32 observation row into `row` (W floats, caller-provided per-thread scratch).
template <int MAXW>
CN_HD void cn_phase_obs_a(const CnParams& p, const CnState& g, CnEnvSh& s, int e, int h, float* row) {
  const size_t i = cn_idx(p, e, h);
  if (h >= s.hn) {           // empty slot: an all-inf row of the reference's max_human_num storage (sorts last, reads 15)
    s.visr[h] = 0; g.vis[i] = 0; s.t0[h] = INFINITY; s.t1[h] = 0.0;
    return;
  }
  const double dist = cn_norm_dot(s.rpx - s.px[h], s.rpy - s.py[h]) - p.robot_radius - s.rad[h];
  const double rvx = p.robot_policy == 2 ? s.rwx : (double)s.rvx, rvy = p.robot_policy == 2 ? s.rwy : (double)s.rvy;
  const bool in_fov = cn_in_fov(s.rpx, s.rpy, rvx, rvy, s.px[h], s.py[h], p.robot_fov);
  const bool vis = in_fov && (dist <= p.sensor_range);
  s.visr[h] = vis ? 1 : 0;
  g.vis[i] = vis ? 1 : 0;
  // prev_human_pos[:, 2:4] = belief velocity BEFORE this update (crowd_sim_pred.py:71)
  const double pvx = g.bvx[i], pvy = g.bvy[i];
  double bx, by;
  if (vis) {
    g.bpx[i] = s.px[h]; g.bpy[i] = s.py[h]; g.bvx[i] = p.social_force ? s.wx[h] : (double)s.vx[h];
    g.bvy[i] = p.social_force ? s.wy[h] : (double)s.vy[h];
    g.brad[i] = s.rad[h];
    bx = s.px[h]; by = s.py[h];
  } else if (s.reset_flag) {
    g.bpx[i] = 15.; g.bpy[i] = 15.; g.bvx[i] = 0.; g.bvy[i] = 0.; g.brad[i] = 0.3;
    bx = 15.; by = 15.;
  } else {
    bx = g.bpx[i] + pvx * p.time_step; by = g.bpy[i] + pvy * p.time_step;
    g.bpx[i] = bx; g.bpy[i] = by;
  }
  if (p.const_vel) {
    // calc_human_future_traj('const_vel') (crowd_sim_var_num.py:152-228)
    double pen = 0.0;   // min over k of [dist < r_robot + humans.radius] * penalty / 2^(k+1)
    const double thresh = p.robot_radius + p.human_radius;
    double coef = 2.0;
    for (int k = 0; k <= p.P; ++k) {
      double tx, ty;
      if (vis) { const double t = (double)k * p.pred_dt; tx = s.px[h] + t * pvx; ty = s.py[h] + t * pvy; }
      else { tx = 15.; ty = 15.; }
      const double rx = tx - s.rpx, ry = ty - s.rpy;
      row[2 * k] = (float)rx; row[2 * k + 1] = (float)ry;
      if (k == 0) s.t0[h] = vis ? cn_norm_dot(rx, ry) : INFINITY;
      else {
        coef = coef * 2.0;                                   // 2^(k+1)
        const double c = (cn_norm_plain(rx, ry) < thresh) ? (p.collision_penalty / coef) : 0.0;
        pen = c < pen ? c : pen;
      }
    }
    s.t1[h] = pen;
  } else {
    const double rx = bx - s.rpx, ry = by - s.rpy;
    row[0] = (float)rx; row[1] = (float)ry;
    s.t0[h] = vis ? cn_norm_dot(rx, ry) : INFINITY;
    s.t1[h] = 0.0;
  }
}

// Phase OBS-B (per human): stable rank by key, write the row; leader writes the per-env parts.
CN_HD void cn_phase_obs_b(const CnParams& p, const CnState& g, CnEnvSh& s, int e, int h, const float* row,
                          const CnObs& ob) {
  const int H = p.H, W = p.W;
  int rank = h;
  if (p.sort_humans) {
    rank = 0;
    const double kh = s.t0[h];
    for (int k = 0; k < H; ++k) {
      const double kk = s.t0[k];
      rank += (kk < kh || (kk == kh && k < h)) ? 1 : 0;
    }
  }
  float* dst = ob.spatial_edges + ((size_t)e * H + rank) * W;
  const bool vis = s.visr[h] != 0;
  for (int c = 0; c < W; ++c) dst[c] = vis ? row[c] : 15.0f;
  if (h == 0) {
    int nvis = 0; double pen = 0.0;
    for (int k = 0; k < H; ++k) { nvis += s.visr[k]; pen = s.t1[k] < pen ? s.t1[k] : pen; }
    s.nvis = nvis;
    g.fut_pen[e] = pen;
    float* rn = ob.robot_node + (size_t)e * 7;
    rn[0] = (float)s.rpx; rn[1] = (float)s.rpy; rn[2] = (float)p.robot_radius; rn[3] = (float)s.rgx;
    rn[4] = (float)s.rgy; rn[5] = (float)p.robot_vpref; rn[6] = (float)(CN_PI / 2);
    ob.temporal_edges[2 * e] = s.rvx; ob.temporal_edges[2 * e + 1] = s.rvy;
    ob.detected_human_num[e] = (float)(nvis > 0 ? nvis : 1);
  }
  if (ob.visible_masks) {
    // sorted: first num_visibles entries True (crowd_sim_var_num.py:262-266); unsorted: by id
    // (written in cn_phase_obs_c once nvis is known when sorted)
    if (!p.sort_humans) ob.visible_masks[(size_t)e * H + h] = vis ? 1 : 0;
  }
}
CN_HD void cn_phase_obs_c(const CnParams& p, CnEnvSh& s, int e, int h, const CnObs& ob) {
  if (ob.visible_masks && p.sort_humans) ob.visible_masks[(size_t)e * p.H + h] = (h < s.nvis) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------
// Phase GOALS (only when the episode continues): random goal changes every 5 s and end-goal respawns
// (crowd_sim_pred.py:202-211).  Replicated execution over the lanes of `co` (see CnCoop): every lane
// draws the same random numbers from `key`; collision scans are lane-strided; lane 0 owns the writes.
// Returns true when a search exhausted `budget` tries (see cn_prepare_env): the caller must NOT store the working set.
CN_HD bool cn_phase_goals(const CnParams& p, const CnState& g, CnEnvSh& s, int e, uint32_t* key, const CnCoop& co,
                          int budget = 0) {
  const int H = s.hn;           // live humans
  CnRng rng; rng.key = key; rng.pos = g.mt_pos[e]; rng.budget = budget; rng.deferred = 0;
  double nd = g.nd_global[e];
  const int step = g.step_count[e];
  // global_time % 5 == 0 with global_time = step * 0.25 accumulated exactly
  const double gt = step * p.time_step;
  if (p.goal_changing && fmod(gt, 5.0) == 0.0) {
    for (int i = 0; i < H; ++i) {
      if (s.vpref[i] == 0) continue;
      if (cn_rng_double(rng, co) <= p.goal_change_chance) {
        const double vp = (s.vpref[i] == 0) ? 1.0 : s.vpref[i];
        const CnCand c = cn_rejection_sample(p, s, rng, co, 1, H, i, s.rad[i], vp, g.spawn_overflow + e);
        if (rng.deferred) return true;
        const double gx = c.x, gy = c.y;
        cn_coop_sync(co);
        if (co.lane == 0) { s.gx[i] = gx; s.gy[i] = gy; }
        cn_coop_sync(co);
      }
    }
  }
  if (p.end_goal_changing) {
    for (int i = 0; i < H; ++i) {
      if (cn_norm_dot(s.gx[i] - s.px[i], s.gy[i] - s.py[i]) < s.rad[i]) {
        const CnSpawn sp = cn_circle_crossing_human(p, s, rng, co, H, nd, g.spawn_overflow + e);
        if (rng.deferred) return true;
        cn_coop_sync(co);
        if (co.lane == 0) {
          s.px[i] = sp.px; s.py[i] = sp.py; s.gx[i] = -sp.px; s.gy[i] = -sp.py;
          s.vx[i] = 0.0f; s.vy[i] = 0.0f; s.rad[i] = sp.rad; s.vpref[i] = sp.vpref;
          if (p.social_force) { s.wx[i] = 0.0; s.wy[i] = 0.0; }
          g.sim_exists[cn_idx(p, e, i)] = 0;       // new Human => new ORCA policy => new rvo2 sim
        }
        cn_coop_sync(co);
      }
    }
  }
  if (co.lane == 0) { g.mt_pos[e] = rng.pos; if (p.randomize) g.nd_global[e] = nd; }
  return false;
}

// Phase STORE: write the working set back to HBM.
CN_HD void cn_phase_store(const CnParams& p, const CnState& g, const CnEnvSh& s, int e, int h) {
  const size_t i = cn_idx(p, e, h);
  g.hpx[i] = s.px[h]; g.hpy[i] = s.py[h];
  if (!s.lean) { g.hgx[i] = s.gx[h]; g.hgy[i] = s.gy[h]; g.hrad[i] = s.rad[h]; g.hvpref[i] = s.vpref[h]; }
  g.hvx[i] = s.vx[h]; g.hvy[i] = s.vy[h];
  if (p.social_force) { g.hwx[i] = s.wx[h]; g.hwy[i] = s.wy[h]; }
  if (h == 0) {
    g.rpx[e] = s.rpx; g.rpy[e] = s.rpy; g.rgx[e] = s.rgx; g.rgy[e] = s.rgy;
    g.rvx[e] = s.rvx; g.rvy[e] = s.rvy;
    if (p.robot_policy == 2) { g.rwx[e] = s.rwx; g.rwy[e] = s.rwy; }
  }
}
