// TEST INFRASTRUCTURE: the host (g++) build of the step kernel's logic for CrowdSimPred-v0 with sim.predict_method =
// 'truth' (cn_config.const_vel 2, the TRUTH instantiations of cn_env_step_kernel in cn_env_kernels.cu): every
// observation, the first one of an episode included, runs the ground-truth look-ahead after cn_phase_obs_a -- ORCA
// humans through their cached simulators (cn_orca_build with use_fov = false), social-force humans with cn_sf_velocity
// -- and the kept rows of the humans the robot sees become observation columns 2.. and the future-collision penalty
// (cn_truth_row).  The rest of the step is env_harness.cpp's loop (ORCA humans, phase 'test' look-ahead) and
// sf_test_harness.cpp's (social-force humans), in the kernel's phase order, thread barriers as plain loops over humans.
// It builds on sf_test_harness.cpp, so that robot.visible (vis_harness_create) runs here too.
#include "sf_test_harness.cpp"

template <int MAXH>
static void run_truth(Harness* hn, const float* action, const cn_obs_ptrs* o, const cn_step_ptrs* r, int mode) {
  const CnParams& p = hn->p;
  CnState& g = hn->g;
  const int H = p.H;
  CnObs ob{o->robot_node, o->temporal_edges, o->spatial_edges, o->detected_human_num, o->visible_masks};
  CnStepOut out;
  memset(&out, 0, sizeof(out));
  if (r) out = CnStepOut{r->reward, r->done, r->info, r->info_aux, r->ep_ret, r->ep_len, r->not_done};
  std::vector<double> d(12 * H);
  std::vector<float> f(6 * H);
  std::vector<uint8_t> u(H);
  std::vector<float4> lines((size_t)H * (H + 1));
  std::vector<float> rows((size_t)H * 16);
  std::vector<float4> projbuf(MAXH + 1);
  std::vector<double> sx(H), sy(H), sw(H), sv(H), lx(H), ly(H), pen(H);
  std::vector<float> svx(H), svy(H), lvx(H), lvy(H);
  std::vector<CnF2> res(H);
  std::vector<CnD2> v(H);
  std::vector<int> nls(H), fails(H);
  std::vector<CnLookahead> la(H);
  const CnCoop co = {0, 1, nullptr, nullptr};
  // one ORCA solve of human h on the joint state in s (single-lane "warp": the sequential RVO2 order)
  auto solve = [&](CnEnvSh& s, int e, int h, bool use_fov, CnF2& result, int& nl, int& fail) {
    CnWarpLines W; W.smem0 = lines.data() + (size_t)h * (H + 1); W.stride = 1; W.cap = 3;    // exercise both tiers
    W.ovf0 = lines.data() + (size_t)h * (H + 1) + 3; W.ovf_stride = 0;
    CnLineStore proj; proj.base = projbuf.data(); proj.stride = 1; proj.cap = MAXH + 1; proj.ovf = nullptr;
    float vmax = 0; CnF2 pref = f2(0, 0);
    nl = 0; fail = -1; result = f2(0, 0);
    cn_orca_build<MAXH>(p, g, s, e, h, W.of(0), nl, vmax, pref, use_fov);
    cn_orca_lp2_warp(co, W, nl, vmax, pref, result, fail);
    cn_orca_lp3_warp(co, W, nl, vmax, proj, result, fail);
  };
  for (int e = 0; e < p.N; ++e) {
    CnEnvSh s;
    s.px = d.data(); s.py = s.px + H; s.gx = s.py + H; s.gy = s.gx + H; s.rad = s.gy + H; s.vpref = s.rad + H;
    s.t0 = s.vpref + H; s.t1 = s.t0 + H;
    s.wx = s.t1 + H; s.wy = s.wx + H; s.nwx = s.wy + H; s.nwy = s.nwx + H;
    s.vx = f.data(); s.vy = s.vx + H; s.fx = s.vy + H; s.fy = s.fx + H; s.nvx = s.fy + H; s.nvy = s.nvx + H;
    s.visr = u.data();
    s.lean = 0;
    uint32_t* prep_key = g.prep_mt + (size_t)e * 624;
    if (mode == 1) {
      // full reset = prepare (event kernel, forced) -> install + first observation (step kernel, mode 1)
      cn_prepare_env(p, g, s, e, prep_key, co);
      s.done = 1; s.info = 0; s.reward = 0.0; s.reset_flag = 0; s.nvis = 0; s.goal_flag = 0; s.hn = 0;
      for (int h = H - 1; h >= 0; --h) cn_install_env(p, g, s, e, h);
    } else {
      for (int h = H - 1; h >= 0; --h) cn_phase_load(p, g, s, e, h, action);
      const int hn0 = s.hn;
      if (p.social_force) {
        for (int h = 0; h < hn0; ++h) cn_sf_action(p, g, s, e, h);
        if (p.test_phase) {                    // cn_sf_lookahead
          for (int h = 0; h < hn0; ++h) { s.t0[h] = INFINITY; s.t1[h] = 0.0; }
          for (int t = 1; t <= p.lookahead_steps; ++t) {
            for (int h = 0; h < hn0; ++h) v[h] = cn_sf_velocity(p, s, h, false);
            for (int h = 0; h < hn0; ++h) {
              const double x = s.px[h] + v[h].x * p.time_step, y = s.py[h] + v[h].y * p.time_step;
              s.px[h] = x; s.py[h] = y; s.wx[h] = v[h].x; s.wy[h] = v[h].y;
              if (t % p.pred_interval == 0) {
                CnLookahead l; l.min_rd = s.t0[h]; l.pen = s.t1[h];
                cn_lookahead_accumulate(p, s, g.vis[cn_idx(p, e, h)] != 0, x, y, t / p.pred_interval, l);
                s.t0[h] = l.min_rd; s.t1[h] = l.pen;
              }
            }
          }
          for (int h = 0; h < hn0; ++h) {
            const size_t i = cn_idx(p, e, h);
            s.px[h] = g.hpx[i]; s.py[h] = g.hpy[i]; s.wx[h] = g.hwx[i]; s.wy[h] = g.hwy[i];
          }
        }
      } else {
        for (int h = 0; h < hn0; ++h) {
          CnF2 result; int nl, fail;
          solve(s, e, h, true, result, nl, fail);
          cn_orca_finish(p, g, s, e, h, result, nl, fail);
        }
        if (p.test_phase) {                    // the ORCA look-ahead before the reward
          for (int h = 0; h < hn0; ++h) {
            sx[h] = s.px[h]; sy[h] = s.py[h]; svx[h] = s.vx[h]; svy[h] = s.vy[h];
            lx[h] = sx[h]; ly[h] = sy[h]; lvx[h] = svx[h]; lvy[h] = svy[h];
            la[h].min_rd = INFINITY; la[h].pen = 0.0;
          }
          for (int t = 1; t <= p.lookahead_steps; ++t) {
            for (int h = 0; h < hn0; ++h) {
              s.px[h] = lx[h]; s.py[h] = ly[h]; s.fx[h] = (float)lx[h]; s.fy[h] = (float)ly[h];
              s.vx[h] = lvx[h]; s.vy[h] = lvy[h];
            }
            for (int h = 0; h < hn0; ++h) solve(s, e, h, false, res[h], nls[h], fails[h]);
            for (int h = 0; h < hn0; ++h) {
              lx[h] = lx[h] + (double)res[h].x * p.time_step; ly[h] = ly[h] + (double)res[h].y * p.time_step;
              lvx[h] = res[h].x; lvy[h] = res[h].y;
              if (t % p.pred_interval == 0)
                cn_lookahead_accumulate(p, s, g.vis[cn_idx(p, e, h)] != 0, lx[h], ly[h], t / p.pred_interval, la[h]);
              if (t == p.lookahead_steps) cn_orca_diag(p, g, e, h, res[h], nls[h], fails[h]);
            }
          }
          for (int h = 0; h < hn0; ++h) {
            s.px[h] = sx[h]; s.py[h] = sy[h]; s.fx[h] = (float)sx[h]; s.fy[h] = (float)sy[h];
            s.vx[h] = svx[h]; s.vy[h] = svy[h];
            s.t0[h] = la[h].min_rd; s.t1[h] = la[h].pen;
          }
        }
      }
      cn_phase_reward(p, g, s, e, out);
      if (s.done) { for (int h = H - 1; h >= 0; --h) cn_install_env(p, g, s, e, h); }   // prepared next episode
      else { for (int h = 0; h < hn0; ++h) cn_phase_integrate(p, s, h); }
      if (cn_add_remove_due(p, g, s, e)) cn_phase_add_remove(p, g, s, e);
    }
    for (int h = 0; h < H; ++h) cn_phase_obs_a<16>(p, g, s, e, h, rows.data() + (size_t)h * 16);
    // the observation look-ahead over the humans alive now, from their state after this step
    const int hn = s.hn;
    for (int h = 0; h < hn; ++h) {
      sx[h] = s.px[h]; sy[h] = s.py[h]; svx[h] = s.vx[h]; svy[h] = s.vy[h]; pen[h] = 0.0;
      if (p.social_force) { sw[h] = s.wx[h]; sv[h] = s.wy[h]; }
      lx[h] = sx[h]; ly[h] = sy[h]; lvx[h] = svx[h]; lvy[h] = svy[h];
    }
    for (int t = 1; t <= p.lookahead_steps; ++t) {
      if (p.social_force) {
        for (int h = 0; h < hn; ++h) v[h] = cn_sf_velocity(p, s, h, false);
        for (int h = 0; h < hn; ++h) {
          lx[h] = s.px[h] + v[h].x * p.time_step; ly[h] = s.py[h] + v[h].y * p.time_step;
          s.px[h] = lx[h]; s.py[h] = ly[h]; s.wx[h] = v[h].x; s.wy[h] = v[h].y;
        }
      } else {
        for (int h = 0; h < hn; ++h) {
          s.px[h] = lx[h]; s.py[h] = ly[h]; s.fx[h] = (float)lx[h]; s.fy[h] = (float)ly[h];
          s.vx[h] = lvx[h]; s.vy[h] = lvy[h];
        }
        for (int h = 0; h < hn; ++h) solve(s, e, h, false, res[h], nls[h], fails[h]);
        for (int h = 0; h < hn; ++h) {
          lx[h] = lx[h] + (double)res[h].x * p.time_step; ly[h] = ly[h] + (double)res[h].y * p.time_step;
          lvx[h] = res[h].x; lvy[h] = res[h].y;
          if (t == p.lookahead_steps) cn_orca_diag(p, g, e, h, res[h], nls[h], fails[h]);
        }
      }
      for (int h = 0; h < hn; ++h)
        if (s.visr[h] && t % p.pred_interval == 0)
          cn_truth_row(p, s, lx[h], ly[h], t / p.pred_interval, rows.data() + (size_t)h * 16, pen[h]);
    }
    for (int h = 0; h < hn; ++h) {
      s.px[h] = sx[h]; s.py[h] = sy[h]; s.fx[h] = (float)sx[h]; s.fy[h] = (float)sy[h];
      s.vx[h] = svx[h]; s.vy[h] = svy[h];
      if (p.social_force) { s.wx[h] = sw[h]; s.wy[h] = sv[h]; }
      if (s.visr[h]) s.t1[h] = pen[h];
    }
    for (int h = 0; h < H; ++h) cn_phase_obs_b(p, g, s, e, h, rows.data() + (size_t)h * 16, ob);
    for (int h = 0; h < H; ++h) cn_phase_obs_c(p, s, e, h, ob);
    const int evt = cn_event_flag(p, g, s, e);
    if (evt == 1) cn_phase_goals(p, g, s, e, g.mt + (size_t)e * 624, co);
    for (int h = 0; h < H; ++h) cn_phase_store(p, g, s, e, h);
    if (evt == 2) cn_prepare_env(p, g, s, e, prep_key, co);
  }
}

static int truth_dispatch(void* h, const float* a, const cn_obs_ptrs* o, const cn_step_ptrs* r, int mode) {
  Harness* hn = static_cast<Harness*>(h);
  if (hn->p.const_vel != 2 || hn->p.robot_policy != 0) return 1;
  if (hn->p.H <= 32) run_truth<32>(hn, a, o, r, mode);
  else if (hn->p.H <= 64) run_truth<64>(hn, a, o, r, mode);
  else run_truth<128>(hn, a, o, r, mode);
  return 0;
}

extern "C" {

// vis_harness_create with the 'truth' observation (cn_config.const_vel 2)
void* truth_harness_create(const cn_config* cfg) {
  Harness* hn = static_cast<Harness*>(vis_harness_create(cfg));
  hn->p.const_vel = cfg->const_vel;
  return hn;
}
int truth_harness_reset(void* h, const cn_obs_ptrs* o) { return truth_dispatch(h, nullptr, o, nullptr, 1); }
int truth_harness_step(void* h, const float* action, const cn_obs_ptrs* o, const cn_step_ptrs* r) {
  return truth_dispatch(h, action, o, r, 0);
}

}  // extern "C"
