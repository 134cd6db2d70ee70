// TEST INFRASTRUCTURE: the host (g++) build of the collect environment's step (CrowdSimVarNumCollect-v0,
// cn_env_create_collect).  Same phases as the COLLECT instantiation of cn_env_step_kernel in cn_env_kernels.cu, with
// thread barriers turned into loops over humans: the humans' actions, cn_collect_reward, integration, visibility and
// belief (cn_phase_obs_a), the prediction ids from the bit string of humans that left the robot's view
// (cn_collect_ids), then the event kernel's part (cn_phase_goals<true>: the robot's goal draw first).
#include "robot_harness.cpp"

extern "C" void* collect_harness_create(const cn_config* cfg) {
  Harness* hn = static_cast<Harness*>(robot_harness_create(cfg));
  hn->p.robot_visible = cfg->robot_visible;
  hn->p.collect = 1;
  hn->p.frame_dt = cfg->pred_timestep;
  const size_t N = hn->p.N, NH = N * hn->p.H;
  CnState& g = hn->g;
  halloc(hn, "pred_id", &g.pred_id, NH); halloc(hn, "max_id", &g.max_id, N);
  halloc(hn, "rgoal_due", &g.rgoal_due, N); halloc(hn, "rgoal_med", &g.rgoal_med, 2 * N);
  return hn;
}

template <int MAXH>
static void collect_run(Harness* hn, const float* action, float* pred_info, const cn_step_ptrs* r, int mode) {
  const CnParams& p = hn->p;
  CnState& g = hn->g;
  const int H = p.H;
  CnObs ob{};
  ob.pred_info = pred_info;
  CnStepOut out;
  memset(&out, 0, sizeof(out));
  if (r) out = CnStepOut{r->reward, r->done, r->info, r->info_aux, r->ep_ret, r->ep_len, r->not_done};
  std::vector<double> d(12 * H);
  std::vector<float> f(6 * H);
  std::vector<uint8_t> u(H), seen(H);
  std::vector<float4> lines((size_t)H * H);
  std::vector<float> rows((size_t)H * 16);
  std::vector<float4> projbuf(MAXH);
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
    if (mode == 1) {
      cn_prepare_env(p, g, s, e, prep_key, co);
      s.done = 1; s.info = 0; s.reward = 0.0; s.reset_flag = 0; s.nvis = 0; s.goal_flag = 0; s.hn = 0;
      for (int h = H - 1; h >= 0; --h) cn_install_env(p, g, s, e, h);
      g.rgoal_due[e] = 0;
    } else {
      for (int h = H - 1; h >= 0; --h) cn_phase_load(p, g, s, e, h, action);
      const int hn = s.hn;
      if (p.social_force) for (int h = 0; h < hn; ++h) cn_sf_action(p, g, s, e, h);
      for (int h = 0; h < hn && !p.social_force; ++h) {
        CnWarpLines W; W.smem0 = lines.data() + (size_t)h * H; W.stride = 1; W.cap = 3;
        W.ovf0 = lines.data() + (size_t)h * H + 3; W.ovf_stride = 0;
        CnLineStore proj; proj.base = projbuf.data(); proj.stride = 1; proj.cap = MAXH; proj.ovf = nullptr;
        int nl = 0, fail = -1; float vmax = 0; CnF2 pref = f2(0, 0), result = f2(0, 0);
        cn_orca_build<MAXH>(p, g, s, e, h, W.of(0), nl, vmax, pref);
        cn_orca_lp2_warp(co, W, nl, vmax, pref, result, fail);
        cn_orca_lp3_warp(co, W, nl, vmax, proj, result, fail);
        cn_orca_finish(p, g, s, e, h, result, nl, fail);
      }
      cn_collect_reward(p, g, s, e, out);
      if (s.done) { for (int h = H - 1; h >= 0; --h) cn_install_env(p, g, s, e, h); }
      else { for (int h = 0; h < hn; ++h) cn_phase_integrate(p, s, h); }
    }
    for (int h = 0; h < H; ++h) seen[h] = h < s.hn && g.vis[cn_idx(p, e, h)] != 0;
    for (int h = 0; h < H; ++h) cn_phase_obs_a<16>(p, g, s, e, h, rows.data() + (size_t)h * 16);
    uint32_t leaving[4] = {0, 0, 0, 0};
    for (int h = 0; h < H; ++h)
      if (seen[h] && !s.reset_flag && !s.visr[h]) leaving[h >> 5] |= 1u << (h & 31);
    for (int h = 0; h < H; ++h) cn_collect_ids(p, g, s, e, h, leaving, 0, ob);
    cn_collect_ids_done(p, g, s, e, leaving, 0);
    int evt = cn_event_flag(p, g, s, e);
    if (evt == 0 && g.rgoal_due[e]) evt = 1;
    if (evt == 1) cn_phase_goals<true>(p, g, s, e, g.mt + (size_t)e * 624, co);
    for (int h = 0; h < H; ++h) cn_phase_store(p, g, s, e, h);
    if (evt == 2) cn_prepare_env(p, g, s, e, prep_key, co);
  }
}

static void collect_dispatch(Harness* hn, const float* a, float* pi, const cn_step_ptrs* r, int mode) {
  if (hn->p.H <= 32) collect_run<32>(hn, a, pi, r, mode);
  else if (hn->p.H <= 64) collect_run<64>(hn, a, pi, r, mode);
  else collect_run<128>(hn, a, pi, r, mode);
}

extern "C" void collect_harness_reset(void* h, float* pred_info) {
  collect_dispatch(static_cast<Harness*>(h), nullptr, pred_info, nullptr, 1);
}
extern "C" void collect_harness_step(void* h, const float* action, float* pred_info, const cn_step_ptrs* r) {
  collect_dispatch(static_cast<Harness*>(h), action, pred_info, r, 0);
}
