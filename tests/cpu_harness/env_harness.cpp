// TEST INFRASTRUCTURE: host (g++) build of the environment step, cn_env_step_kernel in cn_env_kernels.cu over the
// per-phase logic of crowdnav_prediction_attngraph_b200/csrc/cn_env_core.cuh, so the environment arithmetic can be
// checked against the oracle / golden vectors without a GPU.  step_env runs the kernel's phases in its order and takes
// each branch from CnParams as pick_kernel takes the kernel's instantiation: robot policy, robot.visible, social-force
// humans, phase 'test', 'truth' observations (const_vel 2) and the collect environment.  Thread barriers become plain
// loops over humans.  This is NOT a CPU fallback of the product: nothing under crowdnav_prediction_attngraph_b200/
// loads it.
#include <stdlib.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

struct float4 { float x, y, z, w; };
#include "../../crowdnav_prediction_attngraph_b200/csrc/cn_env_core.cuh"
#include "../../include/crowdnav_b200.h"

struct Harness {
  CnParams p;
  CnState g;
  std::map<std::string, std::pair<void*, size_t>> fields;
  std::vector<void*> allocs;
};

template <class T>
static void halloc(Harness* hn, const char* name, T** ptr, size_t count) {
  *ptr = static_cast<T*>(calloc(count ? count : 1, sizeof(T)));
  hn->allocs.push_back(*ptr);
  hn->fields[name] = {(void*)*ptr, count * sizeof(T)};
}

// Working set of one environment (the kernel's shared memory), reused by every environment of a call, plus the
// look-ahead's saved rows.  A human's ORCA lines hold up to H agents: the other humans and the visible robot.
struct Scratch {
  std::vector<double> d, sx, sy, swx, swy, lx, ly, pen;
  std::vector<float> f, rows, svx, svy, lvx, lvy;
  std::vector<uint8_t> u, seen;
  std::vector<float4> lines;
  std::vector<CnF2> res;
  std::vector<CnD2> v;
  std::vector<int> nls, fails;
  std::vector<CnLookahead> la;
  explicit Scratch(int H)
      : d(12 * H), sx(H), sy(H), swx(H), swy(H), lx(H), ly(H), pen(H), f(6 * H), rows((size_t)H * 16), svx(H), svy(H),
        lvx(H), lvy(H), u(H), seen(H), lines((size_t)H * (H + 1)), res(H), v(H), nls(H), fails(H), la(H) {}
};

static const CnCoop kCo = {0, 1, nullptr, nullptr};

// One ORCA solve of human h on the joint state in s: a single-lane "warp", so the cooperative solver degenerates to
// the sequential RVO2 order.  W.cap = 3 keeps both tiers of the line store (shared memory, overflow rows) exercised.
template <int MAXH>
static void solve(const CnParams& p, const CnState& g, Scratch& w, CnEnvSh& s, int e, int h, bool use_fov, CnF2& result,
                  int& nl, int& fail) {
  const int H = p.H;
  float4 projbuf[MAXH + 1];
  CnWarpLines W; W.smem0 = w.lines.data() + (size_t)h * (H + 1); W.stride = 1; W.cap = 3;
  W.ovf0 = W.smem0 + 3; W.ovf_stride = 0;
  CnLineStore proj; proj.base = projbuf; proj.stride = 1; proj.cap = MAXH + 1; proj.ovf = nullptr;
  float vmax = 0; CnF2 pref = f2(0, 0);
  nl = 0; fail = -1; result = f2(0, 0);
  cn_orca_build<MAXH>(p, g, s, e, h, W.of(0), nl, vmax, pref, use_fov);
  cn_orca_lp2_warp(kCo, W, nl, vmax, pref, result, fail);
  cn_orca_lp3_warp(kCo, W, nl, vmax, proj, result, fail);
}

// Ground-truth look-ahead (calc_human_future_traj('truth')): lookahead_steps nested steps of the n live humans from the
// joint state in s -- ORCA solves without FOV, or social-force velocities -- after which s is restored.  Every row of
// step t is complete before any solve of step t + 1 reads it, as across the kernel's barriers.  kept(h, k, x, y) sees
// the k-th kept row (every pred_interval-th step).  An ORCA simulator's last solve is its diagnostics (cn_orca_diag).
template <int MAXH, class Kept>
static void lookahead(const CnParams& p, const CnState& g, Scratch& w, CnEnvSh& s, int e, int n, Kept kept) {
  for (int h = 0; h < n; ++h) {
    w.sx[h] = s.px[h]; w.sy[h] = s.py[h]; w.svx[h] = s.vx[h]; w.svy[h] = s.vy[h];
    if (p.social_force) { w.swx[h] = s.wx[h]; w.swy[h] = s.wy[h]; }
    w.lx[h] = w.sx[h]; w.ly[h] = w.sy[h]; w.lvx[h] = w.svx[h]; w.lvy[h] = w.svy[h];
  }
  for (int t = 1; t <= p.lookahead_steps; ++t) {
    if (p.social_force) {
      for (int h = 0; h < n; ++h) w.v[h] = cn_sf_velocity(p, s, h, false);
      for (int h = 0; h < n; ++h) {
        w.lx[h] = s.px[h] + w.v[h].x * p.time_step; w.ly[h] = s.py[h] + w.v[h].y * p.time_step;
        s.px[h] = w.lx[h]; s.py[h] = w.ly[h]; s.wx[h] = w.v[h].x; s.wy[h] = w.v[h].y;
      }
    } else {
      for (int h = 0; h < n; ++h) {
        s.px[h] = w.lx[h]; s.py[h] = w.ly[h]; s.fx[h] = (float)w.lx[h]; s.fy[h] = (float)w.ly[h];
        s.vx[h] = w.lvx[h]; s.vy[h] = w.lvy[h];
      }
      for (int h = 0; h < n; ++h) solve<MAXH>(p, g, w, s, e, h, false, w.res[h], w.nls[h], w.fails[h]);
      for (int h = 0; h < n; ++h) {
        w.lx[h] = w.lx[h] + (double)w.res[h].x * p.time_step; w.ly[h] = w.ly[h] + (double)w.res[h].y * p.time_step;
        w.lvx[h] = w.res[h].x; w.lvy[h] = w.res[h].y;
      }
    }
    if (t % p.pred_interval == 0)
      for (int h = 0; h < n; ++h) kept(h, t / p.pred_interval, w.lx[h], w.ly[h]);
  }
  for (int h = 0; h < n; ++h) {
    s.px[h] = w.sx[h]; s.py[h] = w.sy[h]; s.fx[h] = (float)w.sx[h]; s.fy[h] = (float)w.sy[h];
    s.vx[h] = w.svx[h]; s.vy[h] = w.svy[h];
    if (p.social_force) { s.wx[h] = w.swx[h]; s.wy[h] = w.swy[h]; }
    else if (p.lookahead_steps > 0) cn_orca_diag(p, g, e, h, w.res[h], w.nls[h], w.fails[h]);
  }
}

// mode 1: reset (no step, every environment installs); 0: step.
template <int MAXH>
static void step_env(const CnParams& p, const CnState& g, Scratch& w, int e, const float* action, const CnObs& ob,
                     const CnStepOut& out, int mode) {
  const int H = p.H;
  CnEnvSh s;
  s.px = w.d.data(); s.py = s.px + H; s.gx = s.py + H; s.gy = s.gx + H; s.rad = s.gy + H; s.vpref = s.rad + H;
  s.t0 = s.vpref + H; s.t1 = s.t0 + H;
  s.wx = s.t1 + H; s.wy = s.wx + H; s.nwx = s.wy + H; s.nwy = s.nwx + H;      // social-force humans only
  s.vx = w.f.data(); s.vy = s.vx + H; s.fx = s.vy + H; s.fy = s.fx + H; s.nvx = s.fy + H; s.nvy = s.nvx + H;
  s.visr = w.u.data();
  s.lean = 0;
  uint32_t* prep_key = g.prep_mt + (size_t)e * 624;
  if (mode == 1) {
    // full reset = prepare (event kernel, forced) -> install + first observation (step kernel, mode 1)
    cn_prepare_env(p, g, s, e, prep_key, kCo);
    s.done = 1; s.info = 0; s.reward = 0.0; s.reset_flag = 0; s.nvis = 0; s.goal_flag = 0; s.hn = 0;
    for (int h = H - 1; h >= 0; --h) cn_install_env(p, g, s, e, h);
    if (p.collect) g.rgoal_due[e] = 0;
  } else {
    for (int h = H - 1; h >= 0; --h) cn_phase_load(p, g, s, e, h, action);   // + the robot's policy
    const int hn = s.hn;                       // live humans (slots [hn, H) are empty)
    if (p.social_force) {
      for (int h = 0; h < hn; ++h) cn_sf_action(p, g, s, e, h);
    } else {
      // The kernel finishes after its phase-'test' look-ahead, whose linearProgram3 queue borrows nvx / t0; here
      // nothing the look-ahead reads is written by cn_orca_finish, and the look-ahead's diagnostics still come last.
      for (int h = 0; h < hn; ++h) {
        CnF2 result; int nl, fail;
        solve<MAXH>(p, g, w, s, e, h, true, result, nl, fail);
        cn_orca_finish(p, g, s, e, h, result, nl, fail);
      }
    }
    if (p.test_phase && !p.collect) {
      // phase 'test': the 'future' danger zone inputs t0 / t1 of the reward, from the rows of the humans the previous
      // observation saw
      for (int h = 0; h < hn; ++h) { w.la[h].min_rd = INFINITY; w.la[h].pen = 0.0; }
      lookahead<MAXH>(p, g, w, s, e, hn, [&](int h, int k, double x, double y) {
        cn_lookahead_accumulate(p, s, g.vis[cn_idx(p, e, h)] != 0, x, y, k, w.la[h]);
      });
      for (int h = 0; h < hn; ++h) { s.t0[h] = w.la[h].min_rd; s.t1[h] = w.la[h].pen; }
    }
    if (p.collect) cn_collect_reward(p, g, s, e, out);
    else cn_phase_reward(p, g, s, e, out);
    if (s.done) { for (int h = H - 1; h >= 0; --h) cn_install_env(p, g, s, e, h); }   // prepared next episode
    else { for (int h = 0; h < hn; ++h) cn_phase_integrate(p, s, h); }
    if (cn_add_remove_due(p, g, s, e)) cn_phase_add_remove(p, g, s, e);
  }
  if (p.collect) for (int h = 0; h < H; ++h) w.seen[h] = h < s.hn && g.vis[cn_idx(p, e, h)] != 0;
  for (int h = 0; h < H; ++h) cn_phase_obs_a<16>(p, g, s, e, h, w.rows.data() + (size_t)h * 16);
  if (p.const_vel == 2) {
    // 'truth': the rows of the humans alive now, from their state after this step, become the observation columns
    // 2.. and the future-collision penalty of the humans the robot sees
    const int hn = s.hn;
    for (int h = 0; h < hn; ++h) w.pen[h] = 0.0;
    lookahead<MAXH>(p, g, w, s, e, hn, [&](int h, int k, double x, double y) {
      if (s.visr[h]) cn_truth_row(p, s, x, y, k, w.rows.data() + (size_t)h * 16, w.pen[h]);
    });
    for (int h = 0; h < hn; ++h) if (s.visr[h]) s.t1[h] = w.pen[h];
  }
  int evt;
  if (p.collect) {
    // prediction ids of the humans that left the robot's view, numbered in ascending human index
    uint32_t leaving[4] = {0, 0, 0, 0};
    for (int h = 0; h < H; ++h)
      if (w.seen[h] && !s.reset_flag && !s.visr[h]) leaving[h >> 5] |= 1u << (h & 31);
    for (int h = 0; h < H; ++h) cn_collect_ids(p, g, s, e, h, leaving, 0, ob);
    cn_collect_ids_done(p, g, s, e, leaving, 0);
    evt = cn_event_flag(p, g, s, e);
    if (evt == 0 && g.rgoal_due[e]) evt = 1;                        // the robot's goal draw
  } else {
    for (int h = 0; h < H; ++h) cn_phase_obs_b(p, g, s, e, h, w.rows.data() + (size_t)h * 16, ob);
    for (int h = 0; h < H; ++h) cn_phase_obs_c(p, s, e, h, ob);
    evt = cn_event_flag(p, g, s, e);
  }
  // event kernel: goal dynamics (evt 1) or preparation of the next episode (evt 2)
  uint32_t* key = g.mt + (size_t)e * 624;
  if (evt == 1 && p.collect) cn_phase_goals<true>(p, g, s, e, key, kCo);
  else if (evt == 1) cn_phase_goals<false>(p, g, s, e, key, kCo);
  for (int h = 0; h < H; ++h) cn_phase_store(p, g, s, e, h);
  if (evt == 2) cn_prepare_env(p, g, s, e, prep_key, kCo);
}

static void dispatch(Harness* hn, const float* action, const cn_obs_ptrs* o, const cn_step_ptrs* r, float* pred_info,
                     int mode) {
  CnObs ob{};
  if (o) ob = CnObs{o->robot_node, o->temporal_edges, o->spatial_edges, o->detected_human_num, o->visible_masks};
  ob.pred_info = pred_info;
  CnStepOut out;
  memset(&out, 0, sizeof(out));
  if (r) out = CnStepOut{r->reward, r->done, r->info, r->info_aux, r->ep_ret, r->ep_len, r->not_done};
  const int H = hn->p.H;
  auto step = H <= 32 ? step_env<32> : H <= 64 ? step_env<64> : step_env<128>;
  Scratch w(H);
  for (int e = 0; e < hn->p.N; ++e) step(hn->p, hn->g, w, e, action, ob, out, mode);
}

extern "C" {

// collect != 0: the collect environment (cn_env_create_collect), whose observation is pred_info
void* harness_create(const cn_config* cfg, int collect) {
  Harness* hn = new Harness();
  CnParams& p = hn->p;
  memset(&p, 0, sizeof(p));
  p.hbase = cfg->human_num; p.hrange = cfg->human_num_range;
  p.N = cfg->num_envs; p.H = cfg->human_num + cfg->human_num_range; p.P = cfg->predict_steps;
  p.const_vel = cfg->const_vel;
  p.W = p.const_vel ? 2 * (p.P + 1) : 2;
  p.randomize = cfg->randomize_attributes; p.goal_changing = cfg->random_goal_changing;
  p.end_goal_changing = cfg->end_goal_changing; p.sort_humans = cfg->sort_humans;
  p.nenv_total = cfg->nenv_total; p.seed_base = (uint32_t)(cfg->seed + cfg->rank_offset);
  p.time_step = cfg->time_step; p.time_limit = cfg->time_limit;
  p.pred_dt = cfg->time_step * (double)(int)floor(cfg->pred_timestep / cfg->time_step);
  cn_fill_phase(p, cfg->phase, cfg->val_size, cfg->test_size);
  p.circle_radius = cfg->circle_radius; p.arena_size = cfg->arena_size;
  p.discomfort_dist = cfg->discomfort_dist; p.discomfort_penalty_factor = cfg->discomfort_penalty_factor;
  p.success_reward = cfg->success_reward; p.collision_penalty = cfg->collision_penalty;
  p.human_radius = cfg->human_radius; p.human_vpref = cfg->human_v_pref;
  p.robot_radius = cfg->robot_radius; p.robot_vpref = cfg->robot_v_pref; p.sensor_range = cfg->sensor_range;
  p.human_fov = CN_PI * cfg->human_fov; p.robot_fov = CN_PI * cfg->robot_fov;
  p.goal_change_chance = cfg->goal_change_chance;
  p.orca_safety_space = cfg->orca_safety_space; p.orca_neighbor_dist = cfg->orca_neighbor_dist;
  p.orca_time_horizon = (float)cfg->orca_time_horizon;
  p.social_force = cfg->human_policy == 1 ? 1 : 0; p.sf_A = cfg->sf_A; p.sf_B = cfg->sf_B; p.sf_KI = cfg->sf_KI;
  p.robot_policy = cfg->robot_policy; p.robot_visible = cfg->robot_visible;
  if (collect) { p.collect = 1; p.frame_dt = cfg->pred_timestep; }
  // every field any configuration uses: cn_env_core.cuh never tests a state pointer, so unused ones cost only memory
  const size_t N = p.N, NH = N * p.H;
  CnState& g = hn->g;
#define A(field, count) halloc(hn, #field, &g.field, (count))
  A(rpx, N); A(rpy, N); A(rgx, N); A(rgy, N); A(rvx, N); A(rvy, N); A(potential, N); A(fut_pen, N);
  A(nd_global, N); A(ep_ret, N); A(ep_len, N); A(step_count, N); A(case_counter, N); A(seed_off, N);
  A(hpx, NH); A(hpy, NH); A(hgx, NH); A(hgy, NH); A(hrad, NH); A(hvpref, NH); A(hvx, NH); A(hvy, NH);
  A(bpx, NH); A(bpy, NH); A(bvx, NH); A(bvy, NH); A(brad, NH); A(vis, NH);
  A(sim_exists, NH); A(sim_nd, NH); A(sim_rself, NH); A(sim_vmax, NH); A(sim_rother, NH * p.H);
  A(mt, N * 624); A(mt_pos, N);
  A(prep_robot, N * 4); A(prep_hpx, NH); A(prep_hpy, NH); A(prep_hrad, NH); A(prep_hvpref, NH); A(prep_nd, N);
  A(prep_mt, N * 624); A(prep_mt_pos, N);
  A(last_hvx, NH); A(last_hvy, NH); A(orca_nlines, NH); A(orca_fail, NH); A(evt, N); A(spawn_overflow, N); A(lp_cost, N); A(hn, N); A(prep_hn, N); A(sim_n, NH); A(hwx, NH); A(hwy, NH);
  A(rwx, N); A(rwy, N); A(rsim_exists, N); A(rsim_nd, N); A(rsim_rother, NH);
  if (collect) { A(pred_id, NH); A(max_id, N); A(rgoal_due, N); A(rgoal_med, 2 * N); }
#undef A
  for (size_t e = 0; e < N; ++e) { g.nd_global[e] = cfg->orca_neighbor_dist; g.seed_off[e] = (int32_t)e; }
  return hn;
}

void harness_destroy(void* h) {
  Harness* hn = static_cast<Harness*>(h);
  for (void* q : hn->allocs) free(q);
  delete hn;
}

// o: the training observation (null for the collect environment); pred_info: the collect observation (null otherwise)
void harness_reset(void* h, const cn_obs_ptrs* o, float* pred_info) {
  dispatch(static_cast<Harness*>(h), nullptr, o, nullptr, pred_info, 1);
}
void harness_step(void* h, const float* action, const cn_obs_ptrs* o, const cn_step_ptrs* r, float* pred_info) {
  dispatch(static_cast<Harness*>(h), action, o, r, pred_info, 0);
}
size_t harness_state_bytes(void* h, const char* name) {
  Harness* hn = static_cast<Harness*>(h);
  auto it = hn->fields.find(name);
  return it == hn->fields.end() ? 0 : it->second.second;
}
int harness_state_copy(void* h, const char* name, void* buf, size_t bytes, int dir) {
  Harness* hn = static_cast<Harness*>(h);
  auto it = hn->fields.find(name);
  if (it == hn->fields.end() || it->second.second != bytes) return 1;
  if (dir) memcpy(it->second.first, buf, bytes); else memcpy(buf, it->second.first, bytes);
  return 0;
}

// MT19937 unit-test hooks
void harness_rng_doubles(uint32_t seed, int n, double* out) {
  uint32_t key[624];
  CnRng r; r.key = key; r.pos = 624;
  cn_rng_seed(r, seed, kCo);
  for (int i = 0; i < n; ++i) out[i] = cn_rng_double(r, kCo);
}

}  // extern "C"
