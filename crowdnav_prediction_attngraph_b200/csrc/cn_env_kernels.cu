// crowd_sim step()/reset() for thousands of environments: one fused sm_90a kernel per
// rollout step over the SoA state in HBM.  Thread mapping: one thread per (environment,
// human); a CTA owns EPB whole environments; neighbour tiles (positions, velocities, radii)
// and the ORCA half-plane lines live in shared memory.  See cn_env_core.cuh for the per-phase
// arithmetic and the reference lines each phase follows.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false  (no FMA contraction: the
// fp32 ORCA sequence and the fp64 reward/visibility tests must round exactly like the oracle).
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include <map>

#include "../../include/crowdnav_b200.h"
#include "cn_env_core.cuh"
#include "cn_host_util.h"

namespace {

// shared-memory carve-up of one environment's working set
struct EnvSmemLayout {
  size_t per_env;      // bytes per environment (without lines)
  size_t off_dbl;      // 8 double arrays
  size_t off_flt;      // 6 float arrays
  size_t off_u8;
};

__host__ __device__ inline size_t align16(size_t x) { return (x + 15) & ~(size_t)15; }

// lean = step kernel: goals / radii / preferred speeds are read-only there and stay in HBM, only what
// other threads read or what changes lives in shared memory (px, py, t0, t1 + 6 float arrays)
__host__ __device__ inline EnvSmemLayout env_layout(int H, bool lean, bool sf = false) {
  EnvSmemLayout L;
  size_t o = align16(sizeof(CnEnvSh));
  L.off_dbl = o; o += (size_t)((lean ? 4 : 8) + (sf ? 4 : 0)) * H * sizeof(double);   // sf: + wx, wy, nwx, nwy
  L.off_flt = o; o += (size_t)6 * H * sizeof(float);
  L.off_u8 = o; o += (size_t)H;
  L.per_env = align16(o);
  return L;
}

__device__ inline CnEnvSh* env_view(unsigned char* base, const EnvSmemLayout& L, int H, bool lean, const CnState& g,
                                    int e, bool sf = false) {
  CnEnvSh* s = reinterpret_cast<CnEnvSh*>(base);
  double* d = reinterpret_cast<double*>(base + L.off_dbl);
  float* f = reinterpret_cast<float*>(base + L.off_flt);
  s->px = d; s->py = d + H; s->t0 = d + 2 * H; s->t1 = d + 3 * H;
  if (lean) {
    const size_t o = (size_t)e * H;
    s->gx = g.hgx + o; s->gy = g.hgy + o; s->rad = g.hrad + o; s->vpref = g.hvpref + o;
  } else {
    s->gx = d + 4 * H; s->gy = d + 5 * H; s->rad = d + 6 * H; s->vpref = d + 7 * H;
  }
  s->lean = lean ? 1 : 0;
  {
    double* w = d + (lean ? 4 : 8) * H;
    s->wx = sf ? w : nullptr; s->wy = sf ? w + H : nullptr; s->nwx = sf ? w + 2 * H : nullptr; s->nwy = sf ? w + 3 * H : nullptr;
  }
  s->vx = f; s->vy = f + H; s->fx = f + 2 * H; s->fy = f + 3 * H; s->nvx = f + 4 * H; s->nvy = f + 5 * H;
  s->visr = base + L.off_u8;
  return s;
}

// Ground-truth look-ahead of social-force humans in phase 'test' (crowd_sim_var_num.py:180-206): lookahead_steps fp64
// SOCIAL_FORCE.predict steps of the humans only (no FOV dummies, never the robot).  The scratch rows are the humans'
// own px / py / wx / wy in shared memory, and the 'future' danger zone inputs accumulate in t0 / t1 (free in phase
// 'test': the reward recomputes the collision distance): across a barrier a thread holds nothing but its new velocity.
// The rows are restored from HBM, which holds them unchanged until cn_phase_store.  The real action (nwx / nwy / nvx /
// nvy) is not touched.  CTA-uniform call (barriers); `live` = the thread owns a human.
__device__ __forceinline__ void cn_sf_lookahead(const CnParams& p, const CnState& g, CnEnvSh* s, int e, int h, bool live) {
  const bool vis_prev = live && g.vis[cn_idx(p, e, h)] != 0;
  if (live) { s->t0[h] = INFINITY; s->t1[h] = 0.0; }
  for (int t = 1; t <= p.lookahead_steps; ++t) {
    __syncthreads();                                                  // row t - 1 complete
    CnD2 v = {0.0, 0.0};
    if (live) v = cn_sf_velocity(p, *s, h, false);
    __syncthreads();                                                  // every read of row t - 1 done
    if (live) {
      const double x = s->px[h] + v.x * p.time_step, y = s->py[h] + v.y * p.time_step;   // agent.py:185-192
      s->px[h] = x; s->py[h] = y; s->wx[h] = v.x; s->wy[h] = v.y;
      if (t % p.pred_interval == 0) {
        CnLookahead la; la.min_rd = s->t0[h]; la.pen = s->t1[h];
        cn_lookahead_accumulate(p, *s, vis_prev, x, y, t / p.pred_interval, la);
        s->t0[h] = la.min_rd; s->t1[h] = la.pen;                      // reward inputs (test phase)
      }
    }
  }
  __syncthreads();
  if (live) {
    const size_t i = cn_idx(p, e, h);
    s->px[h] = g.hpx[i]; s->py[h] = g.hpy[i]; s->wx[h] = g.hwx[i]; s->wy[h] = g.hwy[i];
  }
}

// Observation look-ahead of social-force humans with sim.predict_method = 'truth' (generate_ob ->
// calc_human_future_traj('truth')): the steps of cn_sf_lookahead from the state after this step (integrated, humans
// joined / left, episodes installed), whose rows are not in HBM yet, so each thread keeps its own human's row in
// registers and puts it back.  Every pred_interval-th row of a human the robot sees goes into its observation row and
// the future-collision penalty t1 (cn_truth_row); t0 (cn_phase_obs_a's sort key) is untouched.  CTA-uniform call.
__device__ __forceinline__ void cn_sf_obs_lookahead(const CnParams& p, CnEnvSh* s, int h, bool live, float* row) {
  const bool seen = live && s->visr[h] != 0;
  double spx = 0.0, spy = 0.0, swx = 0.0, swy = 0.0, pen = 0.0;
  if (live) { spx = s->px[h]; spy = s->py[h]; swx = s->wx[h]; swy = s->wy[h]; }
  for (int t = 1; t <= p.lookahead_steps; ++t) {
    __syncthreads();                                                  // row t - 1 complete
    CnD2 v = {0.0, 0.0};
    if (live) v = cn_sf_velocity(p, *s, h, false);
    __syncthreads();                                                  // every read of row t - 1 done
    if (live) {
      const double x = s->px[h] + v.x * p.time_step, y = s->py[h] + v.y * p.time_step;
      s->px[h] = x; s->py[h] = y; s->wx[h] = v.x; s->wy[h] = v.y;
      if (seen && t % p.pred_interval == 0) cn_truth_row(p, *s, x, y, t / p.pred_interval, row, pen);
    }
  }
  __syncthreads();
  if (live) {
    s->px[h] = spx; s->py[h] = spy; s->wx[h] = swx; s->wy[h] = swy;
    if (seen) s->t1[h] = pen;
  }
}

// One rollout step of every environment.  Episodes that finish INSTALL their prepared successor
// (g.prep_*, computed off the critical path by cn_env_event_kernel) and emit its first observation in
// the same launch.  mode 1 = reset of the whole vector env: no step, every environment installs.
// ROBOT: robot_policy != 0 (the robot's ORCA / social-force solve, cn_robot_act); a separate instantiation so the network
// policy's kernel carries none of its code.  VIS: robot_visible != 0 (the humans' solves see the robot), likewise.
// COLLECT: CrowdSimVarNumCollect-v0 (p.collect): collect reward, prediction ids and the pred_info rows instead of the
// training observation.  Phase 'train' only (cn_env_create_collect), so it carries no ground-truth look-ahead.
// SFLA: social-force humans in phase 'test' (cn_sf_lookahead); its own instantiations, so the kernels of ORCA humans and
// of phase 'train' carry none of the look-ahead's code.
// TRUTH: CrowdSimPred-v0 with sim.predict_method = 'truth' (p.const_vel 2): every observation runs the ground-truth
// look-ahead and observes its rows, ORCA humans (SFLA false) or social-force humans (SFLA true, whose phase-'test'
// look-ahead then runs in phase 'test' only).  Robot policy 0; robot visibility is a run-time parameter (VIS true), which
// also makes a simulator the look-ahead creates freeze every human's true radius (cn_orca_build).
template <int MAXH, int MAXW, bool ROBOT, bool VIS, bool COLLECT = false, bool SFLA = false, bool TRUTH = false>
__global__ void __launch_bounds__(288, 2) cn_env_step_kernel(CnParams p, CnState g, const float* __restrict__ action,
                                                          CnObs ob, CnStepOut out, int epb, int line_cap, int mode) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int H = p.H;
  const int le = threadIdx.x / H;
  const int h = threadIdx.x - le * H;
  // slot -> environment through the balancing permutation (cn_env_balance_kernel): CTAs get environments of
  // similar total linear-programming cost; results do not depend on the assignment
  const int e = (le < epb) ? g.perm[blockIdx.x * epb + le] : p.N;
  const bool active = (le < epb) && (e < p.N);
  const EnvSmemLayout L = env_layout(H, true, p.social_force != 0);
  CnEnvSh* s = nullptr;
  if (le < epb) {
    s = reinterpret_cast<CnEnvSh*>(smem + (size_t)le * L.per_env);
    if (h == 0 && e < p.N) env_view(smem + (size_t)le * L.per_env, L, H, true, g, e, p.social_force != 0);
  }
  __syncthreads();
  // ORCA line storage of this warp: first `line_cap` lines of every thread in shared memory
  // ([line][thread]), the rest in a global scratch row per thread; projected lines of the
  // cooperative linearProgram3 in a per-warp shared scratch.
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float4* lines_smem = reinterpret_cast<float4*>(smem + align16((size_t)epb * L.per_env));
  // line slots only for the epb * H threads that own a human (the <= 31 padding threads of the last warp own none)
  const int lstride = epb * H;
  CnWarpLines W;
  W.smem0 = lines_smem + warp * 32;
  W.stride = lstride;
  W.cap = line_cap;
  W.ovf_stride = g.ovf_stride;
  W.ovf0 = reinterpret_cast<float4*>(g.line_ovf) + ((size_t)blockIdx.x * blockDim.x + warp * 32) * g.ovf_stride;
  // The two HALVES of a warp run the cooperative linear programs of different humans at the same time (a scan over the
  // <= H - 1 previous lines rarely has work for more than 16 lanes): half-warp contexts and one projection scratch
  // (<= H - 2 projected lines of linearProgram3) per half.
  const int half = lane >> 4;
  const CnCoop hco = {lane & 15, 16, nullptr, nullptr, half ? 0xffff0000u : 0x0000ffffu, half << 4};
  CnLineStore proj;
  proj.base = lines_smem + (size_t)line_cap * lstride + (size_t)(2 * warp + half) * H;
  proj.stride = 1; proj.cap = H; proj.ovf = nullptr;
  // CTA-wide linearProgram3 task queue: {count, head, tasks[blockDim]} after the projection scratch
  unsigned char* lp3_q = reinterpret_cast<unsigned char*>(lines_smem + (size_t)line_cap * lstride +
                                                          (size_t)(blockDim.x >> 4) * H);
  if (threadIdx.x == 0) { reinterpret_cast<int*>(lp3_q)[0] = 0; reinterpret_cast<int*>(lp3_q)[1] = 0; }
  const CnCoop co = {lane, 32, nullptr, nullptr};

  if (mode == 1) {
    if (active && h == 0) { s->done = 1; s->info = 0; s->reward = 0.0; s->reset_flag = 0; s->nvis = 0; s->goal_flag = 0; s->lp3_cost = 0; s->hn = 0; }
  } else if (active) {
    cn_phase_load<MAXH, ROBOT>(p, g, *s, e, h, mode == 3 ? nullptr : action);   // ROBOT: + the robot's own policy
  }
  __syncthreads();
  // live = this thread's slot holds a human (slots [hn, H) are empty when sim.human_num_range > 0)
  const bool live = active && h < s->hn;
  // One ORCA solve of every human of the CTA on the joint state currently in shared memory (CTA-uniform call: contains
  // barriers; `lv` = this thread's slot holds a human).  linearProgram3 (needed by ~30 % of the humans in steady state)
  // is balanced across the whole CTA: failed humans are queued in shared memory and every warp pops tasks until the
  // queue is dry.
  int* lp3_count = reinterpret_cast<int*>(lp3_q);
  int* lp3_head = lp3_count + 1;
  unsigned short* lp3_tasks = reinterpret_cast<unsigned short*>(lp3_count + 2);
  auto orca_solve = [&](bool lv, bool use_fov, CnF2& result, int& nl, int& fail) {
    nl = 0; fail = -1;
    float vmax = 0.0f;
    CnF2 pref = f2(0.0f, 0.0f);
    result = f2(0.0f, 0.0f);
    if (lv) cn_orca_build<MAXH, VIS>(p, g, *s, e, h, W.of(lane), nl, vmax, pref, use_fov, mode == 3 ? (uint8_t)2 : (uint8_t)1);
    __syncwarp();
    cn_orca_lp2_warp(hco, W, nl, vmax, pref, result, fail);           // per half-warp; idle lanes with nl = 0
    if (fail >= 0) {
      s->nvx[h] = result.x; s->nvy[h] = result.y;                     // LP2 result at the failure point
      reinterpret_cast<int*>(&s->t0[h])[0] = nl | (fail << 8);        // t0 is free until the solve is published
      reinterpret_cast<float*>(&s->t0[h])[1] = vmax;
      lp3_tasks[atomicAdd(lp3_count, 1)] = (unsigned short)threadIdx.x;
    }
    __syncthreads();
    const int ntask = *lp3_count;
    for (;;) {                                                        // every HALF-warp pops its own tasks
      int t = 0;
      if (hco.lane == 0) t = atomicAdd(lp3_head, 1);
      t = __shfl_sync(hco.mask, t, hco.base);
      if (t >= ntask) break;
      const int owner = lp3_tasks[t];
      const int ole = owner / H, oh = owner - ole * H;
      CnEnvSh* os = reinterpret_cast<CnEnvSh*>(smem + (size_t)ole * L.per_env);
      const int packed = reinterpret_cast<const int*>(&os->t0[oh])[0];
      const float ovmax = reinterpret_cast<const float*>(&os->t0[oh])[1];
      CnF2 ores = f2(os->nvx[oh], os->nvy[oh]);
      CnLineStore ol;
      ol.base = lines_smem + owner; ol.stride = lstride; ol.cap = line_cap;
      ol.ovf = reinterpret_cast<float4*>(g.line_ovf) + ((size_t)blockIdx.x * blockDim.x + owner) * g.ovf_stride;
      cn_lp3_coop(hco, ol, packed & 0xff, packed >> 8, ovmax, ores, proj);
      if (hco.lane == 0) { os->nvx[oh] = ores.x; os->nvy[oh] = ores.y; }
    }
    __syncthreads();
    if (fail >= 0) result = f2(s->nvx[h], s->nvy[h]);
    if (threadIdx.x == 0) { *lp3_count = 0; *lp3_head = 0; }          // ready for the next solve (a barrier follows)
  };
  if (mode != 1 && p.social_force) {
    if (live) cn_sf_action<VIS>(p, g, *s, e, h);                           // social-force humans: no linear programs
    if (SFLA && (!TRUTH || p.test_phase)) cn_sf_lookahead(p, g, s, e, h, live);   // phase 'test' (CTA-uniform: barriers)
  } else if (mode == 2) {
    // finishing pass of a step whose ORCA solve already ran on the side stream (mode 3, same state: the humans' solve
    // reads the robot's position and velocity as the previous step left them, never this step's action)
    if (live) {
      const size_t i = cn_idx(p, e, h);
      const int nlf = g.pre_nlf[i];
      cn_orca_finish(p, g, *s, e, h, f2(g.pre_vx[i], g.pre_vy[i]), nlf & 0xff, (nlf >> 8) - 1);
      if (g.sim_exists[i] >= 2) g.sim_exists[i] = 1;                  // simulators the pre-solve created become official
    }
  } else if (mode != 1) {
    CnF2 result; int nl, fail;
    orca_solve(live, true, result, nl, fail);                         // get_human_actions (crowd_sim.py:680-703)
    if (live && fail >= 0) atomicAdd(&s->lp3_cost, 1);              // cost estimate for the next step's balancing
    if (mode == 3) {                                                  // pre-solve: publish the result and stop
      if (live) {
        const size_t i = cn_idx(p, e, h);
        g.pre_vx[i] = result.x; g.pre_vy[i] = result.y; g.pre_nlf[i] = nl | ((fail + 1) << 8);
      }
      __syncthreads();
      if (active && h == 0) g.lp_cost[e] = s->lp3_cost;
      return;
    }
    if (p.test_phase && !COLLECT) {
      // phase 'test': ground-truth look-ahead (crowd_sim_pred.py:136-138 -> crowd_sim_var_num.py:180-206):
      // lookahead_steps nested solves on a scratch copy of the joint state kept in the same shared arrays
      // (every thread saves / restores its own human), then the 'future' danger zone inputs for the reward.
      double spx = 0, spy = 0, lx = 0, ly = 0;
      float svx = 0, svy = 0, lvx = 0, lvy = 0;
      bool vis_prev = false;
      if (live) {
        spx = s->px[h]; spy = s->py[h]; svx = s->vx[h]; svy = s->vy[h];
        lx = spx; ly = spy; lvx = svx; lvy = svy;
        vis_prev = g.vis[cn_idx(p, e, h)] != 0;
      }
      CnLookahead la; la.min_rd = INFINITY; la.pen = 0.0;
      CnF2 lres = f2(0.0f, 0.0f); int lnl = 0, lfail = -1;
      for (int t = 1; t <= p.lookahead_steps; ++t) {
        __syncthreads();
        if (live) {
          s->px[h] = lx; s->py[h] = ly; s->fx[h] = (float)lx; s->fy[h] = (float)ly; s->vx[h] = lvx; s->vy[h] = lvy;
        }
        __syncthreads();
        orca_solve(live, false, lres, lnl, lfail);
        lx = lx + (double)lres.x * p.time_step; ly = ly + (double)lres.y * p.time_step;
        lvx = lres.x; lvy = lres.y;
        if (live && t % p.pred_interval == 0) cn_lookahead_accumulate(p, *s, vis_prev, lx, ly, t / p.pred_interval, la);
      }
      __syncthreads();
      if (live) {
        s->px[h] = spx; s->py[h] = spy; s->fx[h] = (float)spx; s->fy[h] = (float)spy; s->vx[h] = svx; s->vy[h] = svy;
      }
      __syncthreads();
      if (live) {
        cn_orca_finish(p, g, *s, e, h, result, nl, fail);
        cn_orca_diag(p, g, e, h, lres, lnl, lfail);                   // the simulators' LAST solve
        s->t0[h] = la.min_rd; s->t1[h] = la.pen;                      // reward inputs (test phase)
      }
    } else if (live) {
      cn_orca_finish(p, g, *s, e, h, result, nl, fail);
    }
  }
  __syncthreads();
  if (mode != 1 && active && h == 0) {
    if (COLLECT) cn_collect_reward(p, g, *s, e, out);
    else cn_phase_reward(p, g, *s, e, out);
  }
  if (COLLECT && mode == 1 && active && h == 0) g.rgoal_due[e] = 0;
  __syncthreads();
  if (active) {
    if (s->done) cn_install_env(p, g, *s, e, h);      // finished: the prepared next episode takes over
    else if (live) cn_phase_integrate(p, *s, h);
  }
  __syncthreads();
  if (p.hrange > 0) {                                 // humans join / leave every 5 s, before the observation (leader)
    if (mode != 1 && active && h == 0 && cn_add_remove_due(p, g, *s, e)) cn_phase_add_remove(p, g, *s, e);
    __syncthreads();
  }
  float row[MAXW];
  if (COLLECT) {
    // generate_ob of the collect environment: visibility and belief as usual (cn_phase_obs_a), then the prediction ids
    // of the humans that left the robot's view, numbered in ascending human index across the environment's threads
    // (which may span two warps): one ballot per warp, prefix popcounts over the CTA's bit string
    __shared__ uint32_t leaving[(288 + 31) / 32];
    const bool seen_before = active && h < s->hn && g.vis[cn_idx(p, e, h)] != 0;
    if (active) cn_phase_obs_a<MAXW>(p, g, *s, e, h, row);
    __syncthreads();
    const uint32_t b = __ballot_sync(0xffffffffu, seen_before && !s->reset_flag && !s->visr[h]);
    if (lane == 0) leaving[warp] = b;
    __syncthreads();
    if (active) cn_collect_ids(p, g, *s, e, h, leaving, le * H, ob);
    __syncthreads();
    if (active) cn_phase_store(p, g, *s, e, h);
    if (active && h == 0) {
      cn_collect_ids_done(p, g, *s, e, leaving, le * H);
      int evt = cn_event_flag(p, g, *s, e);
      if (evt == 0 && g.rgoal_due[e]) evt = 1;                        // the robot's goal draw (cn_phase_goals<true>)
      g.evt[e] = (uint8_t)evt;
      if (mode != 2) g.lp_cost[e] = s->lp3_cost;
    }
    return;
  }
  if (active) cn_phase_obs_a<MAXW>(p, g, *s, e, h, row);
  __syncthreads();
  if (TRUTH) {
    // generate_ob with sim.predict_method = 'truth' (crowd_sim_pred.py:62-97): after the visibility and belief update
    // (cn_phase_obs_a, whose row holds the k = 0 columns and the sort key) calc_human_future_traj('truth') runs
    // lookahead_steps nested solves of the live humans from their true state after this step: humans joined / left
    // and installed episodes included, so liveness is taken from the current count.  The rows of the humans the
    // robot sees (visibility of this observation) replace the 'const_vel' columns 2.. and the penalty t1; the others
    // keep cn_phase_obs_a's (15, 15) penalty and are written as 15 by cn_phase_obs_b.
    const bool olive = active && h < s->hn;
    if (SFLA) {
      cn_sf_obs_lookahead(p, s, h, olive, row);
    } else {
      // ORCA humans: the solves go through each human's cached simulator (orca_solve, use_fov = false: every other human
      // as is, never the robot), creating it when missing or when the agent count changed; every thread keeps its own
      // human's row and the sort key (the LP3 queue borrows t0) in registers.  The last solve is the simulator's
      // diagnostics (cn_orca_diag).  The loop is the test phase's above, written out again: one loop shared by both
      // changes the instruction schedule of the instantiations without TRUTH.
      const bool seen = olive && s->visr[h] != 0;
      double spx = 0, spy = 0, lx = 0, ly = 0, key = 0, pen = 0.0;
      float svx = 0, svy = 0, lvx = 0, lvy = 0;
      if (olive) {
        spx = s->px[h]; spy = s->py[h]; svx = s->vx[h]; svy = s->vy[h]; key = s->t0[h];
        lx = spx; ly = spy; lvx = svx; lvy = svy;
      }
      CnF2 lres = f2(0.0f, 0.0f); int lnl = 0, lfail = -1;
      for (int t = 1; t <= p.lookahead_steps; ++t) {
        __syncthreads();
        if (olive) {
          s->px[h] = lx; s->py[h] = ly; s->fx[h] = (float)lx; s->fy[h] = (float)ly; s->vx[h] = lvx; s->vy[h] = lvy;
        }
        __syncthreads();
        orca_solve(olive, false, lres, lnl, lfail);
        lx = lx + (double)lres.x * p.time_step; ly = ly + (double)lres.y * p.time_step;
        lvx = lres.x; lvy = lres.y;
        if (seen && t % p.pred_interval == 0) cn_truth_row(p, *s, lx, ly, t / p.pred_interval, row, pen);
      }
      __syncthreads();
      if (olive) {
        s->px[h] = spx; s->py[h] = spy; s->fx[h] = (float)spx; s->fy[h] = (float)spy; s->vx[h] = svx; s->vy[h] = svy;
        s->t0[h] = key;
        if (seen) s->t1[h] = pen;
        if (p.lookahead_steps > 0) cn_orca_diag(p, g, e, h, lres, lnl, lfail);
      }
    }
    __syncthreads();
  }
  if (active) cn_phase_obs_b(p, g, *s, e, h, row, ob);
  __syncthreads();
  if (active) {
    cn_phase_obs_c(p, *s, e, h, ob);
    cn_phase_store(p, g, *s, e, h);
  }
  if (active && h == 0) {
    g.evt[e] = (uint8_t)cn_event_flag(p, g, *s, e);
    if (mode != 2) g.lp_cost[e] = s->lp3_cost;                        // mode 2: the pre-solve already stored it
  }
}

// Event kernel: ONE WARP per environment, for everything that consumes the legacy numpy MT19937
// stream (624-word state per environment): PREPARATION of the next episode (CrowdSimVarNum.reset up
// to generate_ob, evt 2), end-goal respawns and random goal changes (evt 1).  The generator state is
// staged in shared memory (lane-parallel twist) and the rejection-sampling collision scans are
// lane-strided.  Nothing here touches observation buffers, so the kernel runs on the engine's side
// stream, overlapped with the policy; the next step kernel waits for it.  Warps whose environment has
// no event (g.evt == 0) exit immediately.
// COLLECT: the collect environment's instantiation, whose goal dynamics start with the robot's goal draw.
#define CN_EVENT_WARPS 4
template <bool COLLECT = false>
__global__ void __launch_bounds__(CN_EVENT_WARPS * 32) cn_env_event_kernel(CnParams p, CnState g, int force,
                                                                           size_t per_warp_bytes) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.x * CN_EVENT_WARPS + warp;
  if (e >= p.N) return;
  const int evt = force ? 2 : g.evt[e];
  if (evt == 0) return;
  const int H = p.H;
  const EnvSmemLayout L = env_layout(H, false, p.social_force != 0);
  unsigned char* base = smem + (size_t)warp * per_warp_bytes;
  CnEnvSh* s = reinterpret_cast<CnEnvSh*>(base);
  if (lane == 0) env_view(base, L, H, false, g, e, p.social_force != 0);
  __syncwarp();
  uint32_t* key = reinterpret_cast<uint32_t*>(base + L.per_env);
  // per-warp fp32 agent table of the rejection sampler, behind the MT19937 state
  const CnCoop co = {lane, 32, nullptr, reinterpret_cast<float*>(key + 624)};
  bool deferred;
  if (evt == 2) {
    deferred = cn_prepare_env(p, g, *s, e, key, co, p.defer_tries);
    if (!deferred)
      for (int i = lane; i < 624; i += 32) g.prep_mt[(size_t)e * 624 + i] = key[i];
  } else {
    // goal dynamics on the state the step kernel just stored
    for (int h = lane; h < H; h += 32) cn_phase_load(p, g, *s, e, h, nullptr);
    for (int i = lane; i < 624; i += 32) key[i] = g.mt[(size_t)e * 624 + i];
    __syncwarp();
    deferred = cn_phase_goals<COLLECT>(p, g, *s, e, key, co, p.defer_tries);
    __syncwarp();
    if (!deferred) {
      for (int h = lane; h < H; h += 32) cn_phase_store(p, g, *s, e, h);
      for (int i = lane; i < 624; i += 32) g.mt[(size_t)e * 624 + i] = key[i];
    }
  }
  // a rejection-sampling search that ran out of its warp-scope budget: nothing was published; the whole event of
  // this environment is redone by a 512-thread CTA (cn_env_event_heavy_kernel, launched right behind this kernel)
  if (deferred && lane == 0) {
    g.defer_list[atomicAdd(g.defer_ctl, 1)] = e | (evt << 24);
    atomicAdd(g.defer_ctl + 2, 1);
  }
}

// Heavy path of the event kernel.  In crowded configurations (BASELINE config 4: 50 randomised humans with random
// goal changes) a few environments per step reach a state where a free goal / spawn position is found only after
// thousands of candidates -- or never: the reference would spin there; the engine accepts candidate number
// CN_MAX_SPAWN_TRIES (cn_env_core.cuh).  One warp needs milliseconds for such a search (every candidate is tested
// against the position and the goal of every agent in fp64), and the next step kernel waits for it.  Here a CTA of
// CN_HEAVY_THREADS threads redoes the event of ONE deferred environment from scratch with the same code in CTA
// scope: the MT19937 twist runs 224 words at a time and the <= 104 candidates up to the next twist are evaluated at
// once, CN_HEAVY_SUB threads per candidate splitting the agent list.  Results are identical to the sequential loop
// (first free candidate, same stream position).
template <bool COLLECT = false>
__global__ void __launch_bounds__(CN_HEAVY_THREADS) cn_env_event_heavy_kernel(CnParams p, CnState g) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int H = p.H;
  const EnvSmemLayout L = env_layout(H, false, p.social_force != 0);
  CnEnvSh* s = reinterpret_cast<CnEnvSh*>(smem);
  uint32_t* key = reinterpret_cast<uint32_t*>(smem + L.per_env);
  int* scratch = reinterpret_cast<int*>(key + 624);                    // 16 ints
  float* ftab = reinterpret_cast<float*>(scratch + 16);               // 5 x CN_FTAB floats
  const int count = g.defer_ctl[0];
  if (threadIdx.x == 0) { scratch[1] = 0; scratch[2] = 0; }
  const long long tk0 = clock64();
  const CnCoop co = {(int)threadIdx.x, (int)blockDim.x, scratch, ftab};
  for (int idx = blockIdx.x; idx < count; idx += gridDim.x) {
    const int entry = g.defer_list[idx];
    const int e = entry & 0xffffff, evt = entry >> 24;
    if (threadIdx.x == 0) env_view(smem, L, H, false, g, e, p.social_force != 0);
    __syncthreads();
    if (evt == 2) {
      cn_prepare_env(p, g, *s, e, key, co, 0);
      for (int i = threadIdx.x; i < 624; i += blockDim.x) g.prep_mt[(size_t)e * 624 + i] = key[i];
    } else {
      for (int h = threadIdx.x; h < H; h += blockDim.x) cn_phase_load(p, g, *s, e, h, nullptr);
      for (int i = threadIdx.x; i < 624; i += blockDim.x) key[i] = g.mt[(size_t)e * 624 + i];
      __syncthreads();
      cn_phase_goals<COLLECT>(p, g, *s, e, key, co, 0);
      __syncthreads();
      for (int h = threadIdx.x; h < H; h += blockDim.x) cn_phase_store(p, g, *s, e, h);
      for (int i = threadIdx.x; i < 624; i += blockDim.x) g.mt[(size_t)e * 624 + i] = key[i];
    }
    __syncthreads();
  }
  // the last CTA to finish clears the list for the next event kernel
  if (threadIdx.x == 0) {
    if (scratch[1]) {
      atomicAdd(g.defer_ctl + 3, scratch[1]); atomicMax(g.defer_ctl + 4, scratch[1]);
      atomicAdd(g.defer_ctl + 5, scratch[2] >> 6);                               // kilo-cycles in candidate batches
      atomicAdd(g.defer_ctl + 6, (int)((clock64() - tk0) >> 10));               // kilo-cycles of working CTAs in total
    }   // diagnostics: total / max batches per CTA
    __threadfence();
    if (atomicAdd(g.defer_ctl + 1, 1) == (int)gridDim.x - 1) { g.defer_ctl[0] = 0; g.defer_ctl[1] = 0; }
  }
}

// Load balancing for the step kernel (side stream, off the critical path).  The kernel's duration is set by its
// slowest SM (ncu: SMs busy 78 % on average); the work of an environment is dominated by its linearProgram3
// fall-throughs, which change slowly from step to step.  Cost estimate = number of humans whose last solve needed
// linearProgram3 (counted by the step kernel); environments are bucketed by cost (counting sort, one CTA) and dealt to the CTAs in
// serpentine order, heaviest first, so every CTA gets a similar sum.
__global__ void __launch_bounds__(1024) cn_env_balance_kernel(CnParams p, CnState g, int grid, int epb) {
  __shared__ int bucket[130];                 // cost 0..H (H <= 128) -> count, then start offset
  __shared__ int cursor[130];
  const int H = p.H, N = p.N, slots = grid * epb;
  for (int i = threadIdx.x; i <= H; i += blockDim.x) bucket[i] = 0;
  __syncthreads();
  for (int e = threadIdx.x; e < N; e += blockDim.x) atomicAdd(&bucket[min(g.lp_cost[e], H)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {                       // descending cost: offsets of the buckets H, H-1, ..., 0
    int off = 0;
    for (int c = H; c >= 0; --c) { cursor[c] = off; off += bucket[c]; }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < slots; i += blockDim.x) g.perm[i] = N;          // empty
  __syncthreads();
  for (int e = threadIdx.x; e < N; e += blockDim.x) {
    const int k = atomicAdd(&cursor[min(g.lp_cost[e], H)], 1);     // rank in the descending order (ties arbitrary)
    const int round = k / grid, pos = k - round * grid;
    const int cta = (round & 1) ? grid - 1 - pos : pos;                         // serpentine deal
    g.perm[cta * epb + round] = e;
  }
}

// Several small device-to-device copies in one launch (RolloutStorage.insert): blockIdx.y = segment.
struct CopySegs {
  cn_copy_seg s[CN_MAX_COPY_SEGS];
};
__global__ void __launch_bounds__(256) cn_copy_segments_kernel(CopySegs p) {
  const cn_copy_seg sg = p.s[blockIdx.y];
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
  if ((((uintptr_t)sg.dst | (uintptr_t)sg.src | sg.bytes) & 15) == 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(sg.src);
    uint4* d4 = reinterpret_cast<uint4*>(sg.dst);
    for (size_t i = tid; i < sg.bytes / 16; i += nth) d4[i] = s4[i];
  } else {
    const unsigned char* s1 = reinterpret_cast<const unsigned char*>(sg.src);
    unsigned char* d1 = reinterpret_cast<unsigned char*>(sg.dst);
    for (size_t i = tid; i < sg.bytes; i += nth) d1[i] = s1[i];
  }
}

struct Field {
  void* ptr;
  size_t bytes;
};

}  // namespace

struct cn_env {
  cn_config cfg;
  CnParams p;
  CnState g;
  int device;
  int epb;
  int threads;
  size_t smem_bytes;
  int line_cap;
  size_t reset_warp_bytes;
  int heavy_grid;          // CTAs of cn_env_event_heavy_kernel (each loops over the deferred list)
  size_t heavy_smem;
  int maxh;
  int64_t launches;
  std::map<std::string, Field> fields;
  std::vector<void*> allocs;
  // side stream of the event kernel (overlaps the caller's policy work between two steps)
  cudaStream_t side;
  cudaEvent_t ev_step, ev_side;
  // optional timing of the env launches (cn_env_profile): [0..1] step / finishing kernel on the caller's stream,
  // [2..3] event kernel(s) + balancing, [3..4] pre-solve kernel on the side stream
  bool profile = false;
  cudaEvent_t pev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  bool side_pending;      // an event kernel is in flight: the next launch on the caller's stream waits for it
  bool use_side;
  bool presolve;          // run the humans' ORCA solve of the next step on the side stream behind the event kernel
  bool presolved;         // ... and one is in flight / done for the current state
  bool balance;           // re-deal environments to CTAs by their linearProgram3 load after every step (side stream)
  bool prep_dirty;        // a state upload may have invalidated the prepared episodes
  // staging for the host-buffer entry point
  float* d_action;
  cn_obs_ptrs d_obs;
  cn_step_ptrs d_out;
};

namespace {

template <class T>
int dev_alloc(cn_env* env, const char* name, T** ptr, size_t count) {
  void* q = nullptr;
  const size_t bytes = count * sizeof(T);
  cudaError_t err = cudaMalloc(&q, bytes ? bytes : 16);
  if (err != cudaSuccess) return cn_set_error("cudaMalloc(%s, %zu bytes): %s", name, bytes, cudaGetErrorString(err));
  err = cudaMemset(q, 0, bytes ? bytes : 16);
  if (err != cudaSuccess) return cn_set_error("cudaMemset(%s): %s", name, cudaGetErrorString(err));
  *ptr = static_cast<T*>(q);
  env->allocs.push_back(q);
  if (name) env->fields[name] = Field{q, bytes};
  return 0;
}

typedef void (*KernelFn)(CnParams, CnState, const float*, CnObs, CnStepOut, int, int, int);

template <bool VIS>
KernelFn pick_kernel_vis(int maxh, bool robot) {
  if (robot) {
    if (maxh <= 32) return cn_env_step_kernel<32, 16, true, VIS>;
    if (maxh <= 64) return cn_env_step_kernel<64, 16, true, VIS>;
    return cn_env_step_kernel<128, 16, true, VIS>;
  }
  if (maxh <= 32) return cn_env_step_kernel<32, 16, false, VIS>;
  if (maxh <= 64) return cn_env_step_kernel<64, 16, false, VIS>;
  return cn_env_step_kernel<128, 16, false, VIS>;
}

// the collect environment: robot policy and visibility stay run-time parameters there (it runs no network policy)
KernelFn pick_kernel_collect(int maxh) {
  if (maxh <= 32) return cn_env_step_kernel<32, 16, true, true, true>;
  if (maxh <= 64) return cn_env_step_kernel<64, 16, true, true, true>;
  return cn_env_step_kernel<128, 16, true, true, true>;
}

// social-force humans in phase 'test' (the SF look-ahead): robot policy and visibility stay run-time parameters too
KernelFn pick_kernel_sfla(int maxh) {
  if (maxh <= 32) return cn_env_step_kernel<32, 16, true, true, false, true>;
  if (maxh <= 64) return cn_env_step_kernel<64, 16, true, true, false, true>;
  return cn_env_step_kernel<128, 16, true, true, false, true>;
}

// CrowdSimPred-v0 with sim.predict_method = 'truth' (the observation look-ahead): ORCA or social-force humans, robot
// visibility a run-time parameter, robot policy 0
template <bool SF>
KernelFn pick_kernel_truth(int maxh) {
  if (maxh <= 32) return cn_env_step_kernel<32, 16, false, true, false, SF, true>;
  if (maxh <= 64) return cn_env_step_kernel<64, 16, false, true, false, SF, true>;
  return cn_env_step_kernel<128, 16, false, true, false, SF, true>;
}

KernelFn pick_kernel(const CnParams& p, int maxh) {
  if (p.collect) return pick_kernel_collect(maxh);
  if (p.const_vel == 2) return p.social_force ? pick_kernel_truth<true>(maxh) : pick_kernel_truth<false>(maxh);
  if (p.social_force && p.test_phase) return pick_kernel_sfla(maxh);
  const bool robot = p.robot_policy != 0, vis = p.robot_visible != 0;
  return vis ? pick_kernel_vis<true>(maxh, robot) : pick_kernel_vis<false>(maxh, robot);
}

CnObs to_obs(const cn_obs_ptrs* o) {
  CnObs ob;
  ob.robot_node = o->robot_node; ob.temporal_edges = o->temporal_edges; ob.spatial_edges = o->spatial_edges;
  ob.detected_human_num = o->detected_human_num; ob.visible_masks = o->visible_masks;
  ob.pred_info = nullptr;
  return ob;
}

int event_kernel(cn_env* env, int force, cudaStream_t stream) {
  const int grid = (env->p.N + CN_EVENT_WARPS - 1) / CN_EVENT_WARPS;
  if (env->p.collect)
    cn_env_event_kernel<true><<<grid, CN_EVENT_WARPS * 32, CN_EVENT_WARPS * env->reset_warp_bytes, stream>>>(
        env->p, env->g, force, env->reset_warp_bytes);
  else
    cn_env_event_kernel<<<grid, CN_EVENT_WARPS * 32, CN_EVENT_WARPS * env->reset_warp_bytes, stream>>>(
        env->p, env->g, force, env->reset_warp_bytes);
  env->launches += 1;
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("cn_env_event_kernel launch: %s", cudaGetErrorString(err));
  // deferred (pathological) searches, one CTA each; an empty list costs one ~2 us launch on the side stream
  if (env->p.collect)
    cn_env_event_heavy_kernel<true><<<env->heavy_grid, CN_HEAVY_THREADS, env->heavy_smem, stream>>>(env->p, env->g);
  else
    cn_env_event_heavy_kernel<<<env->heavy_grid, CN_HEAVY_THREADS, env->heavy_smem, stream>>>(env->p, env->g);
  env->launches += 1;
  err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("cn_env_event_heavy_kernel launch: %s", cudaGetErrorString(err));
  return 0;
}

// make `stream` wait for the event kernel in flight on the side stream (if any)
int join_side(cn_env* env, cudaStream_t stream) {
  if (!env->side_pending) return 0;
  cudaError_t err = cudaStreamWaitEvent(stream, env->ev_side, 0);
  if (err != cudaSuccess) return cn_set_error("cudaStreamWaitEvent(side): %s", cudaGetErrorString(err));
  env->side_pending = false;
  return 0;
}

// step (or mode 1: install-everything) kernel on the caller's stream, then the event kernel behind it
// on the side stream
int launch_step(cn_env* env, const float* d_action, const cn_obs_ptrs* o, const cn_step_ptrs* r, int mode,
                cudaStream_t stream, float* d_pred_info = nullptr) {
  CnStepOut out;
  memset(&out, 0, sizeof(out));
  if (r) {
    out.reward = r->reward; out.done = r->done; out.info = r->info; out.info_aux = r->info_aux;
    out.ep_ret = r->ep_ret; out.ep_len = r->ep_len; out.not_done = r->not_done;
  }
  int rc = join_side(env, stream);
  if (rc) return rc;
  if (mode == 1 || env->prep_dirty) {
    // (re)compute every prepared episode first: a pure function of (seed, case_counter)
    rc = event_kernel(env, 1, stream);
    if (rc) return rc;
    env->prep_dirty = false;
  }
  const int grid = (env->p.N + env->epb - 1) / env->epb;
  KernelFn fn = pick_kernel(env->p, env->maxh);
  CnObs ob = to_obs(o);
  ob.pred_info = d_pred_info;
  // mode 0 with a pre-solve of this state done on the side stream (joined above) -> finishing pass only (mode 2)
  const int kmode = (mode == 0 && env->presolved) ? 2 : mode;
  env->presolved = false;
  if (env->profile) cudaEventRecord(env->pev[0], stream);
  fn<<<grid, env->threads, env->smem_bytes, stream>>>(env->p, env->g, d_action, ob, out, env->epb, env->line_cap, kmode);
  if (env->profile) cudaEventRecord(env->pev[1], stream);
  env->launches += 1;
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("cn_env_step_kernel launch: %s", cudaGetErrorString(err));
  if (!env->use_side) return event_kernel(env, 0, stream);      // CN_NO_SIDE_STREAM=1: everything in stream order
  err = cudaEventRecord(env->ev_step, stream);
  if (err == cudaSuccess) err = cudaStreamWaitEvent(env->side, env->ev_step, 0);
  if (err != cudaSuccess) return cn_set_error("fork to side stream: %s", cudaGetErrorString(err));
  if (env->profile) cudaEventRecord(env->pev[2], env->side);
  rc = event_kernel(env, 0, env->side);
  if (rc) return rc;
  if (env->balance && mode == 0) {
    cn_env_balance_kernel<<<1, 1024, 0, env->side>>>(env->p, env->g, grid, env->epb);
    env->launches += 1;
  }
  if (env->profile) cudaEventRecord(env->pev[3], env->side);
  if (env->presolve) {
    // PRE-SOLVE: the humans' ORCA solve of the NEXT step depends on the state this step leaves behind (after the event
    // kernel's goal changes and the installed episodes) and on nothing the policy is about to compute.  With the robot
    // visible it also reads the robot's position and velocity, and both are final once this step has integrated (the
    // next action moves the robot only after the humans' solve).  It runs here, on the side stream, while the caller's
    // stream runs the policy; the next step only finishes (robot move, reward, integration, observation).
    fn<<<grid, env->threads, env->smem_bytes, env->side>>>(env->p, env->g, nullptr, ob, out, env->epb, env->line_cap, 3);
    env->launches += 1;
    err = cudaGetLastError();
    if (err != cudaSuccess) return cn_set_error("cn_env_step_kernel (pre-solve) launch: %s", cudaGetErrorString(err));
    env->presolved = true;
  }
  if (env->profile) cudaEventRecord(env->pev[4], env->side);
  err = cudaEventRecord(env->ev_side, env->side);
  if (err != cudaSuccess) return cn_set_error("cudaEventRecord(side): %s", cudaGetErrorString(err));
  env->side_pending = true;
  return 0;
}

}  // namespace

extern "C" {

int cn_abi_version(void) { return CN_ABI_VERSION; }

}  // extern "C"

namespace {

int env_create(const cn_config* cfg, cn_env** out, bool collect) {
  if (!cfg || !out) return cn_set_error("cn_env_create: null argument");
  *out = nullptr;
  if (cfg->num_envs <= 0 || cfg->human_num <= 0 || cfg->human_num_range < 0 || cfg->human_num_range >= cfg->human_num ||
      cfg->human_num + cfg->human_num_range > 128)
    return cn_set_error("cn_env_create: need num_envs > 0, 0 <= human_num_range < human_num and human_num + range <= 128 "
                        "(got %d, %d, %d)", cfg->num_envs, cfg->human_num, cfg->human_num_range);
  if (cfg->const_vel < 0 || cfg->const_vel > 2)
    return cn_set_error("cn_env_create: const_vel %d unsupported (0 = CrowdSimVarNum-v0, 1 = CrowdSimPred-v0 'const_vel', "
                        "2 = CrowdSimPred-v0 'truth')", cfg->const_vel);
  if (cfg->const_vel && (cfg->predict_steps < 0 || 2 * (cfg->predict_steps + 1) > 16))
    return cn_set_error("cn_env_create: predict_steps %d unsupported (row width > 16)", cfg->predict_steps);
  {
    // global_time is kept as step_count * time_step; the reference ACCUMULATES `global_time += time_step`
    // (crowd_sim_pred.py:160).  The two agree bit for bit iff every partial sum is exact, i.e. time_step is a
    // dyadic rational with a short mantissa (0.25, the reference's value; 0.5; 0.125 ...).  Anything else (0.1)
    // could shift the time-out / 5-second events by one step, so it is refused rather than approximated.
    const double ts = cfg->time_step * 1024.0;
    if (!(cfg->time_step > 0) || ts != floor(ts))
      return cn_set_error("cn_env_create: time_step %.17g is not a multiple of 1/1024 (the engine keeps global_time as "
                          "step * time_step, exact only for such steps)", cfg->time_step);
  }
  int ndev = 0;
  cudaError_t err = cudaGetDeviceCount(&ndev);
  if (err != cudaSuccess || ndev == 0)
    return cn_set_error("cn_env_create: no CUDA device (%s); this engine has no CPU fallback",
                        err == cudaSuccess ? "device count 0" : cudaGetErrorString(err));
  if (cfg->device < 0 || cfg->device >= ndev) return cn_set_error("cn_env_create: bad device %d", cfg->device);
  err = cudaSetDevice(cfg->device);
  if (err != cudaSuccess) return cn_set_error("cudaSetDevice: %s", cudaGetErrorString(err));

  cn_env* env = new cn_env();
  env->cfg = *cfg;
  env->device = cfg->device;
  env->launches = 0;
  env->side = nullptr; env->ev_step = nullptr; env->ev_side = nullptr;
  env->side_pending = false; env->prep_dirty = true;
  {
    const char* ns = getenv("CN_NO_SIDE_STREAM");       // debugging / profiling aid
    env->use_side = !(ns && ns[0] == '1');
    // pre-solve of the next step's ORCA on the side stream (launch_step).  Not with social-force humans (no linear
    // programs to move) nor in the test phase (its look-ahead solves stay with the step) nor with 'truth' predictions (the
    // observation look-ahead creates simulators, which the pre-solve's provisional marks do not cover).  Default: on for crowds of up
    // to 32 human slots (measured: 20 humans 0.455 -> 0.442 ms/step, e2e 0.534 -> 0.501), off above (50 humans 2.15 ->
    // 2.19, 100 humans 4.9 -> 5.1 ms/step: the many short CTAs of the large-H solve take SMs from the policy's GEMMs
    // instead of filling gaps); CN_PRESOLVE=1 / 0 forces it.
    const char* ps = getenv("CN_PRESOLVE");
    const bool want = ps ? ps[0] != '0' : (cfg->human_num + cfg->human_num_range <= 32);
    env->presolve = env->use_side && want && cfg->human_policy == 0 && cfg->phase != 2 && cfg->const_vel != 2;
    env->presolved = false;
  }
  err = cudaStreamCreateWithFlags(&env->side, cudaStreamNonBlocking);
  if (err == cudaSuccess) err = cudaEventCreateWithFlags(&env->ev_step, cudaEventDisableTiming);
  if (err == cudaSuccess) err = cudaEventCreateWithFlags(&env->ev_side, cudaEventDisableTiming);
  if (err != cudaSuccess) { cn_env_destroy(env); return cn_set_error("side stream: %s", cudaGetErrorString(err)); }
  CnParams& p = env->p;
  memset(&p, 0, sizeof(p));
  p.hbase = cfg->human_num; p.hrange = cfg->human_num_range;
  p.N = cfg->num_envs; p.H = cfg->human_num + cfg->human_num_range; p.P = cfg->predict_steps;
  p.const_vel = cfg->const_vel;                 // 0, 1 or 2 ('truth': the TRUTH instantiations, pick_kernel)
  p.W = p.const_vel ? 2 * (p.P + 1) : 2;
  p.randomize = cfg->randomize_attributes; p.goal_changing = cfg->random_goal_changing;
  p.end_goal_changing = cfg->end_goal_changing; p.sort_humans = cfg->sort_humans;
  p.nenv_total = cfg->nenv_total; p.seed_base = (uint32_t)(cfg->seed + cfg->rank_offset);
  p.time_step = cfg->time_step; p.time_limit = cfg->time_limit;
  {
    // pred_interval = int(pred_timestep // time_step) (crowd_sim.py:187)
    const double q = floor(cfg->pred_timestep / cfg->time_step);
    p.pred_dt = cfg->time_step * (double)(int)q;
  }
  if (cfg->human_policy != 0 && cfg->human_policy != 1) {
    cn_env_destroy(env);
    return cn_set_error("cn_env_create: human_policy %d unsupported (0 = 'orca', 1 = 'social_force')", cfg->human_policy);
  }
  if (cfg->robot_policy < 0 || cfg->robot_policy > 2) {
    cn_env_destroy(env);
    return cn_set_error("cn_env_create: robot_policy %d unsupported (0 = the caller's action, 1 = 'orca', 2 = 'social_force')",
                        cfg->robot_policy);
  }
  if (cfg->robot_policy != 0 && (cfg->const_vel || cfg->human_num_range > 0)) {
    cn_env_destroy(env);
    return cn_set_error("cn_env_create: the ORCA / social-force robot is covered for CrowdSimVarNum-v0 (const_vel 0) with "
                        "human_num_range 0");
  }
  if (cfg->robot_visible != 0 && cfg->robot_visible != 1) {
    cn_env_destroy(env);
    return cn_set_error("cn_env_create: robot_visible %d unsupported (0 or 1)", cfg->robot_visible);
  }
  if (cfg->robot_visible && cfg->const_vel == 1) {
    cn_env_destroy(env);
    return cn_set_error("cn_env_create: robot_visible is covered for CrowdSimVarNum-v0 (const_vel 0) and 'truth' (const_vel "
                        "2) only: the reference's CrowdSimPred-v0 with 'const_vel' cannot run it "
                        "(calc_human_future_traj('const_vel') assigns the humans' (H, 2) velocities into an (H + 1, 2) "
                        "slice and raises on the first reset)");
  }
  if (cfg->phase != 0 && cfg->phase != 2) {
    cn_env_destroy(env);
    return cn_set_error("cn_env_create: phase %d unsupported (0 = 'train', 2 = 'test')", cfg->phase);
  }
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
  p.social_force = cfg->human_policy == 1 ? 1 : 0;
  p.sf_A = cfg->sf_A; p.sf_B = cfg->sf_B; p.sf_KI = cfg->sf_KI;
  p.robot_policy = cfg->robot_policy;
  p.robot_visible = cfg->robot_visible;
  p.collect = collect ? 1 : 0;
  p.frame_dt = cfg->pred_timestep;
  {
    // warp-scope budget of rejection-sampling tries before an event goes to the CTA-scope kernel
    // (CN_DEFER_TRIES=1 sends every search that needs a second candidate there: parity tests of the heavy path)
    const char* dt = getenv("CN_DEFER_TRIES");
    p.defer_tries = dt ? atoi(dt) : CN_DEFER_TRIES;
    if (p.defer_tries < 1) p.defer_tries = 1;
  }

  const size_t N = (size_t)p.N, NH = N * p.H;
  CnState& g = env->g;
  memset(&g, 0, sizeof(g));
  int rc = 0;
#define A(field, count) if (!rc) rc = dev_alloc(env, #field, &g.field, (count))
  A(rpx, N); A(rpy, N); A(rgx, N); A(rgy, N); A(rvx, N); A(rvy, N); A(potential, N); A(fut_pen, N);
  A(nd_global, N); A(ep_ret, N); A(ep_len, N); A(step_count, N); A(case_counter, N); A(seed_off, N);
  A(hpx, NH); A(hpy, NH); A(hgx, NH); A(hgy, NH); A(hrad, NH); A(hvpref, NH); A(hvx, NH); A(hvy, NH);
  A(bpx, NH); A(bpy, NH); A(bvx, NH); A(bvy, NH); A(brad, NH); A(vis, NH);
  A(sim_exists, NH); A(sim_nd, NH); A(sim_rself, NH); A(sim_vmax, NH);
  A(sim_rother, p.randomize ? NH * p.H : (size_t)4);
  A(mt, N * 624); A(mt_pos, N);
  A(prep_robot, N * 4); A(prep_hpx, NH); A(prep_hpy, NH); A(prep_hrad, NH); A(prep_hvpref, NH); A(prep_nd, N);
  A(prep_mt, N * 624); A(prep_mt_pos, N);
  A(last_hvx, NH); A(last_hvy, NH); A(orca_nlines, NH); A(orca_fail, NH); A(evt, N); A(spawn_overflow, N);
  A(lp_cost, N); A(defer_list, N); A(defer_ctl, 8); A(hn, N); A(prep_hn, N); A(sim_n, NH);
  A(pre_vx, NH); A(pre_vy, NH); A(pre_nlf, NH);
  A(hwx, cfg->human_policy ? NH : (size_t)4); A(hwy, cfg->human_policy ? NH : (size_t)4);
  A(rwx, cfg->robot_policy == 2 ? N : (size_t)4); A(rwy, cfg->robot_policy == 2 ? N : (size_t)4);
  A(rsim_exists, N); A(rsim_nd, N); A(rsim_rother, cfg->robot_policy == 1 ? NH : (size_t)4);
  if (collect) { A(pred_id, NH); A(max_id, N); A(rgoal_due, N); A(rgoal_med, 2 * N); }
#undef A
  if (!rc) {
    // nd_global starts at the configured value (config.orca.neighbor_dist)
    std::vector<double> nd(N, cfg->orca_neighbor_dist);
    err = cudaMemcpy(g.nd_global, nd.data(), N * sizeof(double), cudaMemcpyHostToDevice);
    if (err != cudaSuccess) rc = cn_set_error("init nd_global: %s", cudaGetErrorString(err));
  }
  if (!rc) {
    std::vector<int32_t> so(N);
    for (size_t i = 0; i < N; ++i) so[i] = (int32_t)i;
    err = cudaMemcpy(g.seed_off, so.data(), N * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (err != cudaSuccess) rc = cn_set_error("init seed_off: %s", cudaGetErrorString(err));
  }
  // staging buffers for cn_env_step_host
  memset(&env->d_obs, 0, sizeof(env->d_obs)); memset(&env->d_out, 0, sizeof(env->d_out));
  env->d_action = nullptr;
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_action, N * 2);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_obs.robot_node, N * 7);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_obs.temporal_edges, N * 2);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_obs.spatial_edges, NH * p.W);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_obs.detected_human_num, N);
  if (!rc && !p.const_vel) rc = dev_alloc(env, nullptr, &env->d_obs.visible_masks, NH);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_out.reward, N);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_out.done, N);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_out.info, N);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_out.info_aux, N);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_out.ep_ret, N);
  if (!rc) rc = dev_alloc(env, nullptr, &env->d_out.ep_len, N);
  env->d_out.not_done = nullptr;
  if (rc) { cn_env_destroy(env); return rc; }

  // launch geometry: EPB whole environments per CTA (<= 288 threads); the first `line_cap` ORCA lines
  // of every thread live in shared memory.  Search (epb, cap) for the largest cap whose launch is
  // resident in ONE wave on this device (shared memory is the occupancy limiter; a partial second wave costs a whole
  // wave of the slowest CTAs).
  env->maxh = p.H <= 32 ? 32 : (p.H <= 64 ? 64 : 128);
  const EnvSmemLayout L = env_layout(p.H, true, p.social_force != 0);
  int nsm = 0;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, cfg->device);
  KernelFn fn = pick_kernel(p, env->maxh);
  // dynamic shared memory: 227 KiB less the kernel's static part (the collect instantiation's ballot words)
  size_t smem_cap = 227 * 1024;
  {
    cudaFuncAttributes fa;
    err = cudaFuncGetAttributes(&fa, fn);
    if (err != cudaSuccess) { cn_env_destroy(env); return cn_set_error("cudaFuncGetAttributes: %s", cudaGetErrorString(err)); }
    smem_cap -= fa.sharedSizeBytes;
  }
  err = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_cap);
  if (err != cudaSuccess) { cn_env_destroy(env); return cn_set_error("cudaFuncSetAttribute: %s", cudaGetErrorString(err)); }
  // ORCA lines per human: one per other human, plus one for the robot when it is visible
  const int max_lines = p.H - 1 + p.robot_visible;
  const int cap_max = max_lines > 1 ? max_lines : 1;
  int best_epb = 0, best_cap = 0, best_threads = 0;
  size_t best_need = 0;
  bool best_single = false;
  for (int epb = 288 / p.H > 0 ? 288 / p.H : 1; epb >= 1; --epb) {
    const int threads = ((epb * p.H + 31) / 32) * 32;
    if (threads > 288) continue;
    const int grid_try = (p.N + epb - 1) / epb;
    for (int cap = cap_max; cap >= 1; --cap) {
      const size_t need = align16((size_t)epb * L.per_env) + (size_t)cap * epb * p.H * sizeof(float4) +
                          (size_t)(threads / 16) * p.H * sizeof(float4) +         // + per-half-warp LP3 scratch
                          align16(8 + 2 * (size_t)threads);                       // + CTA LP3 task queue
      if (need > smem_cap) continue;
      int per_sm = 0;
      err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, threads, need);
      if (err != cudaSuccess) { cn_env_destroy(env); return cn_set_error("occupancy query: %s", cudaGetErrorString(err)); }
      const bool single = (long long)per_sm * nsm >= grid_try;
      // preference: single wave first, then larger cap, then larger epb (fewer CTAs)
      const bool better = !best_epb || (single && !best_single) ||
                          (single == best_single && (cap > best_cap || (cap == best_cap && epb > best_epb)));
      if (better && (single || !best_single)) {
        best_epb = epb; best_cap = cap; best_threads = threads; best_need = need; best_single = single;
      }
      if (single) break;          // smaller caps of this epb cannot be better
    }
  }
  if (!best_epb) { cn_env_destroy(env); return cn_set_error("cn_env_create: human_num %d does not fit shared memory", p.H); }
  env->epb = best_epb; env->threads = best_threads; env->line_cap = best_cap; env->smem_bytes = best_need;
  const int grid = (p.N + env->epb - 1) / env->epb;
  {
    // global scratch for the overflow lines (k >= line_cap) of every step-kernel thread
    float4* ovf = nullptr;
    env->g.ovf_stride = (max_lines - env->line_cap) > 0 ? (max_lines - env->line_cap) : 1;
    int rc2 = dev_alloc(env, nullptr, &ovf, (size_t)grid * env->threads * env->g.ovf_stride);
    if (rc2) { cn_env_destroy(env); return rc2; }
    env->g.line_ovf = ovf;
  }
  {
    // slot -> environment permutation of the step kernel, identity to start with
    int* perm = nullptr;
    int rc3 = dev_alloc(env, nullptr, &perm, (size_t)grid * env->epb);
    if (rc3) { cn_env_destroy(env); return rc3; }
    std::vector<int> id((size_t)grid * env->epb);
    for (size_t i = 0; i < id.size(); ++i) id[i] = (int)i;      // entries >= N are empty slots
    err = cudaMemcpy(perm, id.data(), id.size() * sizeof(int), cudaMemcpyHostToDevice);
    if (err != cudaSuccess) { cn_env_destroy(env); return cn_set_error("init perm: %s", cudaGetErrorString(err)); }
    env->g.perm = perm;
    const char* nb = getenv("CN_NO_BALANCE");
    env->balance = !(nb && nb[0] == '1') && env->use_side;
  }
  // event kernel: per-warp working set + MT19937 state
  env->reset_warp_bytes = align16(env_layout(p.H, false, p.social_force != 0).per_env + 624 * sizeof(uint32_t) + 5 * CN_FTAB * sizeof(float));
  err = collect ? cudaFuncSetAttribute(cn_env_event_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(CN_EVENT_WARPS * env->reset_warp_bytes))
                : cudaFuncSetAttribute(cn_env_event_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(CN_EVENT_WARPS * env->reset_warp_bytes));
  if (err != cudaSuccess) { cn_env_destroy(env); return cn_set_error("cudaFuncSetAttribute(reset): %s", cudaGetErrorString(err)); }
  // heavy path: working set + MT19937 state + a few ints of scratch per CTA; half an SM-wave of CTAs (the list
  // is short, and these CTAs share the GPU with the caller's policy kernels)
  env->heavy_smem = align16(env_layout(p.H, false, p.social_force != 0).per_env + 624 * sizeof(uint32_t) + 64 + 5 * CN_FTAB * sizeof(float));
  {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, cfg->device);
    env->heavy_grid = sms / 2 > 0 ? sms / 2 : 1;
    if (env->heavy_grid > p.N) env->heavy_grid = p.N;
  }
  err = collect ? cudaFuncSetAttribute(cn_env_event_heavy_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)env->heavy_smem)
                : cudaFuncSetAttribute(cn_env_event_heavy_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)env->heavy_smem);
  if (err != cudaSuccess) { cn_env_destroy(env); return cn_set_error("cudaFuncSetAttribute(heavy): %s", cudaGetErrorString(err)); }
  *out = env;
  return 0;
}

}  // namespace

extern "C" {

int cn_env_create(const cn_config* cfg, cn_env** out) { return env_create(cfg, out, false); }

int cn_env_create_collect(const cn_config* cfg, cn_env** out) {
  if (!cfg || !out) return cn_set_error("cn_env_create_collect: null argument");
  *out = nullptr;
  if (cfg->const_vel)
    return cn_set_error("cn_env_create_collect: CrowdSimVarNumCollect-v0 subclasses CrowdSimVarNum-v0 (const_vel 0)");
  if (cfg->human_num_range > 0)
    return cn_set_error("cn_env_create_collect: human_num_range > 0 is not covered: the reference raises there "
                        "(crowd_sim_var_num_collect.py:121-123 joins human_num frame rows with human_num + range position rows)");
  if (cfg->phase != 0)
    return cn_set_error("cn_env_create_collect: phase 'test' is not covered: the reference raises on the first step (the "
                        "ground-truth look-ahead reads self.human_visibility, crowd_sim_var_num.py:225, which the collect "
                        "environment's generate_ob never sets)");
  return env_create(cfg, out, true);
}

int cn_env_reset_collect(cn_env* env, float* d_pred_info, void* stream) {
  if (!env || !d_pred_info) return cn_set_error("cn_env_reset_collect: null argument");
  if (!env->p.collect) return cn_set_error("cn_env_reset_collect: the handle was not made by cn_env_create_collect");
  CnDeviceGuard guard(env->device);
  return launch_step(env, nullptr, &env->d_obs, nullptr, 1, (cudaStream_t)stream, d_pred_info);
}

int cn_env_step_collect(cn_env* env, const float* d_action, float* d_pred_info, const cn_step_ptrs* d_out, void* stream) {
  if (!env || !d_action || !d_pred_info || !d_out) return cn_set_error("cn_env_step_collect: null argument");
  if (!env->p.collect) return cn_set_error("cn_env_step_collect: the handle was not made by cn_env_create_collect");
  if (!d_out->reward || !d_out->done || !d_out->info || !d_out->info_aux || !d_out->ep_ret || !d_out->ep_len)
    return cn_set_error("cn_env_step_collect: every cn_step_ptrs field must be set");
  CnDeviceGuard guard(env->device);
  return launch_step(env, d_action, &env->d_obs, d_out, 0, (cudaStream_t)stream, d_pred_info);
}

int cn_env_destroy(cn_env* env) {
  if (!env) return 0;
  cudaSetDevice(env->device);
  cudaDeviceSynchronize();
  if (env->side) cudaStreamDestroy(env->side);
  if (env->ev_step) cudaEventDestroy(env->ev_step);
  if (env->ev_side) cudaEventDestroy(env->ev_side);
  for (int i = 0; i < 5; ++i) if (env->pev[i]) cudaEventDestroy(env->pev[i]);
  for (void* q : env->allocs) cudaFree(q);
  delete env;
  return 0;
}

int cn_env_reset(cn_env* env, const cn_obs_ptrs* d_obs, void* stream) {
  if (!env || !d_obs) return cn_set_error("cn_env_reset: null argument");
  if (env->p.collect) return cn_set_error("cn_env_reset: a collect environment resets with cn_env_reset_collect");
  CnDeviceGuard guard(env->device);
  // a reset of the whole vec env restarts Monitor bookkeeping but NOT case_counter (it keeps advancing)
  return launch_step(env, nullptr, d_obs, nullptr, 1, (cudaStream_t)stream);
}

int cn_env_step(cn_env* env, const float* d_action, const cn_obs_ptrs* d_obs, const cn_step_ptrs* d_out,
                void* stream) {
  if (!env || !d_action || !d_obs || !d_out) return cn_set_error("cn_env_step: null argument");
  if (env->p.collect) return cn_set_error("cn_env_step: a collect environment steps with cn_env_step_collect");
  if (!d_out->reward || !d_out->done || !d_out->info || !d_out->info_aux || !d_out->ep_ret || !d_out->ep_len)
    return cn_set_error("cn_env_step: every cn_step_ptrs field must be set");
  CnDeviceGuard guard(env->device);
  return launch_step(env, d_action, d_obs, d_out, 0, (cudaStream_t)stream);
}

int cn_env_step_host(cn_env* env, const float* h_action, const cn_obs_ptrs* h_obs, const cn_step_ptrs* h_out) {
  if (!env || !h_action || !h_obs || !h_out) return cn_set_error("cn_env_step_host: null argument");
  if (env->p.collect) return cn_set_error("cn_env_step_host: a collect environment steps with cn_env_step_collect");
  cudaSetDevice(env->device);
  const size_t N = (size_t)env->p.N, NH = N * env->p.H;
  cudaStream_t st = 0;
  cudaError_t err = cudaMemcpyAsync(env->d_action, h_action, N * 2 * sizeof(float), cudaMemcpyHostToDevice, st);
  if (err != cudaSuccess) return cn_set_error("H2D action: %s", cudaGetErrorString(err));
  int rc = launch_step(env, env->d_action, &env->d_obs, &env->d_out, 0, st);
  if (rc) return rc;
#define D2H(dst, src, bytes) if (dst) { err = cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st); \
    if (err != cudaSuccess) return cn_set_error("D2H " #dst ": %s", cudaGetErrorString(err)); }
  D2H(h_obs->robot_node, env->d_obs.robot_node, N * 7 * sizeof(float));
  D2H(h_obs->temporal_edges, env->d_obs.temporal_edges, N * 2 * sizeof(float));
  D2H(h_obs->spatial_edges, env->d_obs.spatial_edges, NH * env->p.W * sizeof(float));
  D2H(h_obs->detected_human_num, env->d_obs.detected_human_num, N * sizeof(float));
  if (env->d_obs.visible_masks) D2H(h_obs->visible_masks, env->d_obs.visible_masks, NH);
  D2H(h_out->reward, env->d_out.reward, N * sizeof(float));
  D2H(h_out->done, env->d_out.done, N);
  D2H(h_out->info, env->d_out.info, N * sizeof(int32_t));
  D2H(h_out->info_aux, env->d_out.info_aux, N * sizeof(float));
  D2H(h_out->ep_ret, env->d_out.ep_ret, N * sizeof(double));
  D2H(h_out->ep_len, env->d_out.ep_len, N * sizeof(int32_t));
#undef D2H
  err = cudaStreamSynchronize(st);
  if (err != cudaSuccess) return cn_set_error("cn_env_step_host: %s", cudaGetErrorString(err));
  return 0;
}

size_t cn_env_state_bytes(cn_env* env, const char* name) {
  if (!env || !name) return 0;
  auto it = env->fields.find(name);
  return it == env->fields.end() ? 0 : it->second.bytes;
}

int cn_env_state_copy(cn_env* env, const char* name, void* h_buf, size_t bytes, int dir) {
  if (!env || !name || !h_buf) return cn_set_error("cn_env_state_copy: null argument");
  auto it = env->fields.find(name);
  if (it == env->fields.end()) return cn_set_error("cn_env_state_copy: unknown field '%s'", name);
  if (bytes != it->second.bytes)
    return cn_set_error("cn_env_state_copy: field '%s' is %zu bytes, got %zu", name, it->second.bytes, bytes);
  cudaSetDevice(env->device);
  cudaError_t err = cudaDeviceSynchronize();
  if (err == cudaSuccess)
    err = dir ? cudaMemcpy(it->second.ptr, h_buf, bytes, cudaMemcpyHostToDevice)
              : cudaMemcpy(h_buf, it->second.ptr, bytes, cudaMemcpyDeviceToHost);
  if (err != cudaSuccess) return cn_set_error("cn_env_state_copy(%s): %s", name, cudaGetErrorString(err));
  if (dir) { env->prep_dirty = true; env->presolved = false; }     // an uploaded state invalidates the pre-solve in flight
  if (!dir && strcmp(name, "sim_exists") == 0) {
    // 2 = created, 3 = re-created by a pre-solve that belongs to the NEXT step: report the state as of the last step
    unsigned char* b = static_cast<unsigned char*>(h_buf);
    for (size_t i = 0; i < bytes; ++i) if (b[i] >= 2) b[i] = (unsigned char)(b[i] == 3);
  }
  return 0;
}

int cn_copy_segments(const cn_copy_seg* segs, int n, int device, void* stream) {
  if (!segs || n < 0 || n > CN_MAX_COPY_SEGS) return cn_set_error("cn_copy_segments: need 0 <= n <= %d segments", CN_MAX_COPY_SEGS);
  if (n == 0) return 0;
  CopySegs p;
  size_t maxb = 0;
  for (int i = 0; i < n; ++i) {
    if (!segs[i].dst || !segs[i].src) return cn_set_error("cn_copy_segments: null pointer in segment %d", i);
    p.s[i] = segs[i];
    if (segs[i].bytes > maxb) maxb = segs[i].bytes;
  }
  CnDeviceGuard guard(device);
  size_t blocks = (maxb / 16 + 255) / 256;
  if (blocks < 1) blocks = 1;
  if (blocks > 1184) blocks = 1184;
  cn_copy_segments_kernel<<<dim3((unsigned)blocks, (unsigned)n), 256, 0, (cudaStream_t)stream>>>(p);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("cn_copy_segments launch: %s", cudaGetErrorString(err));
  return 0;
}

int cn_fetch_sync(void* h_dst, const void* d_src, size_t bytes, int device, void* stream) {
  if (!h_dst || !d_src) return cn_set_error("cn_fetch_sync: null argument");
  CnDeviceGuard guard(device);
  cudaError_t err = cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)stream);
  if (err == cudaSuccess) err = cudaStreamSynchronize((cudaStream_t)stream);
  if (err != cudaSuccess) return cn_set_error("cn_fetch_sync: %s", cudaGetErrorString(err));
  return 0;
}

int cn_env_profile(cn_env* env, int enable) {
  if (!env) return cn_set_error("cn_env_profile: null argument");
  CnDeviceGuard guard(env->device);
  if (enable && !env->pev[0]) {
    for (int i = 0; i < 5; ++i)
      if (cudaEventCreate(&env->pev[i]) != cudaSuccess) return cn_set_error("cn_env_profile: cudaEventCreate failed");
  }
  env->profile = enable != 0;
  return 0;
}

int cn_env_stage_ms(cn_env* env, float* out3) {
  if (!env || !out3) return cn_set_error("cn_env_stage_ms: null argument");
  if (!env->pev[0]) return cn_set_error("cn_env_stage_ms: call cn_env_profile(env, 1) before the step");
  CnDeviceGuard guard(env->device);
  cudaError_t err = cudaDeviceSynchronize();
  out3[0] = out3[1] = out3[2] = 0.0f;
  if (err == cudaSuccess) err = cudaEventElapsedTime(&out3[0], env->pev[0], env->pev[1]);
  if (err == cudaSuccess && env->use_side) {
    err = cudaEventElapsedTime(&out3[1], env->pev[2], env->pev[3]);
    if (err == cudaSuccess) err = cudaEventElapsedTime(&out3[2], env->pev[3], env->pev[4]);
  }
  if (err != cudaSuccess) return cn_set_error("cn_env_stage_ms: %s", cudaGetErrorString(err));
  return 0;
}

int64_t cn_env_launch_count(cn_env* env) { return env ? env->launches : 0; }

}  // extern "C"
