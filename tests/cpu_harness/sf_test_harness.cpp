// TEST INFRASTRUCTURE: the host (g++) build of the step kernel's logic for social-force humans in phase 'test'
// (cn_config.human_policy 1, phase 2): cn_sf_action, then the ground-truth look-ahead of cn_sf_lookahead in
// cn_env_kernels.cu -- lookahead_steps fp64 SOCIAL_FORCE.predict steps of the live humans (cn_sf_velocity, no FOV, never
// the robot) on scratch rows, every pred_interval-th row folded into the 'future' danger zone inputs t0 / t1.
// env_harness.cpp's step loop runs the ORCA look-ahead in phase 'test'; sf_harness_step is that loop with the
// social-force look-ahead in its place (same phase order, thread barriers as plain loops over humans).  It builds on
// vis_harness.cpp, so that robot.visible and the ORCA / social-force robot (vis_harness_create) run here too.
#include "vis_harness.cpp"

static void run_sf(Harness* hn, const float* action, const cn_obs_ptrs* o, const cn_step_ptrs* r) {
  const CnParams& p = hn->p;
  CnState& g = hn->g;
  const int H = p.H;
  CnObs ob{o->robot_node, o->temporal_edges, o->spatial_edges, o->detected_human_num, o->visible_masks};
  CnStepOut out{r->reward, r->done, r->info, r->info_aux, r->ep_ret, r->ep_len, r->not_done};
  std::vector<double> d(12 * H);
  std::vector<float> f(6 * H);
  std::vector<uint8_t> u(H);
  std::vector<float> rows((size_t)H * 16);
  std::vector<CnD2> v(H);
  for (int e = 0; e < p.N; ++e) {
    CnEnvSh s;
    s.px = d.data(); s.py = s.px + H; s.gx = s.py + H; s.gy = s.gx + H; s.rad = s.gy + H; s.vpref = s.rad + H;
    s.t0 = s.vpref + H; s.t1 = s.t0 + H;
    s.wx = s.t1 + H; s.wy = s.wx + H; s.nwx = s.wy + H; s.nwy = s.nwx + H;
    s.vx = f.data(); s.vy = s.vx + H; s.fx = s.vy + H; s.fy = s.fx + H; s.nvx = s.fy + H; s.nvy = s.nvx + H;
    s.visr = u.data();
    s.lean = 0;
    const CnCoop co = {0, 1, nullptr, nullptr};
    uint32_t* prep_key = g.prep_mt + (size_t)e * 624;
    for (int h = H - 1; h >= 0; --h) cn_phase_load(p, g, s, e, h, action);
    const int hn = s.hn;                       // live humans (slots [hn, H) are empty)
    for (int h = 0; h < hn; ++h) cn_sf_action(p, g, s, e, h);
    // ground-truth look-ahead: the rows of step t - 1 are complete before any velocity of step t is computed, and every
    // velocity is computed before any row is overwritten (the kernel's two barriers)
    for (int h = 0; h < hn; ++h) { s.t0[h] = INFINITY; s.t1[h] = 0.0; }
    for (int t = 1; t <= p.lookahead_steps; ++t) {
      for (int h = 0; h < hn; ++h) v[h] = cn_sf_velocity(p, s, h, false);
      for (int h = 0; h < hn; ++h) {
        const double x = s.px[h] + v[h].x * p.time_step, y = s.py[h] + v[h].y * p.time_step;
        s.px[h] = x; s.py[h] = y; s.wx[h] = v[h].x; s.wy[h] = v[h].y;
        if (t % p.pred_interval == 0) {
          CnLookahead la; la.min_rd = s.t0[h]; la.pen = s.t1[h];
          cn_lookahead_accumulate(p, s, g.vis[cn_idx(p, e, h)] != 0, x, y, t / p.pred_interval, la);
          s.t0[h] = la.min_rd; s.t1[h] = la.pen;
        }
      }
    }
    for (int h = 0; h < hn; ++h) {             // the rows come back from the persistent state, as in the kernel
      const size_t i = cn_idx(p, e, h);
      s.px[h] = g.hpx[i]; s.py[h] = g.hpy[i]; s.wx[h] = g.hwx[i]; s.wy[h] = g.hwy[i];
    }
    cn_phase_reward(p, g, s, e, out);
    if (s.done) { for (int h = H - 1; h >= 0; --h) cn_install_env(p, g, s, e, h); }   // prepared next episode
    else { for (int h = 0; h < hn; ++h) cn_phase_integrate(p, s, h); }
    if (cn_add_remove_due(p, g, s, e)) cn_phase_add_remove(p, g, s, e);
    for (int h = 0; h < H; ++h) cn_phase_obs_a<16>(p, g, s, e, h, rows.data() + (size_t)h * 16);
    for (int h = 0; h < H; ++h) cn_phase_obs_b(p, g, s, e, h, rows.data() + (size_t)h * 16, ob);
    for (int h = 0; h < H; ++h) cn_phase_obs_c(p, s, e, h, ob);
    const int evt = cn_event_flag(p, g, s, e);
    if (evt == 1) cn_phase_goals(p, g, s, e, g.mt + (size_t)e * 624, co);
    for (int h = 0; h < H; ++h) cn_phase_store(p, g, s, e, h);
    if (evt == 2) cn_prepare_env(p, g, s, e, prep_key, co);
  }
}

// harness_step for social-force humans in phase 'test' (the reset is harness_reset's)
extern "C" int sf_harness_step(void* h, const float* action, const cn_obs_ptrs* o, const cn_step_ptrs* r) {
  Harness* hn = static_cast<Harness*>(h);
  if (!hn->p.social_force || !hn->p.test_phase) return 1;
  run_sf(hn, action, o, r);
  return 0;
}
