// Shared definitions for the crowd-navigation rollout engine (sm_90a).
//
// Everything that is pure per-environment arithmetic is written as CN_HD (host+device)
// functions so the SAME source can be compiled by g++ into a unit-test harness
// (tests/cpu_harness) and checked against the oracle without a GPU.  The harness is
// test infrastructure only: the product entry points (cn_api.cu) launch CUDA kernels and
// fail loudly if no device is present.
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define CN_HD __host__ __device__ __forceinline__
#define CN_HD_NOINLINE __host__ __device__ __noinline__
#else
#define CN_HD inline
#define CN_HD_NOINLINE inline
#endif

// info codes (crowd_sim/envs/utils/info.py): Nothing, Timeout, Collision, ReachGoal, Danger
enum { CN_INFO_NOTHING = 0, CN_INFO_TIMEOUT = 1, CN_INFO_COLLISION = 2, CN_INFO_REACHGOAL = 3, CN_INFO_DANGER = 4 };

// Device-side mirror of cn_config (include/crowdnav_b200.h) with derived constants.
struct CnParams {
  int N;            // environments in this shard
  int H;            // human SLOTS per environment = sim.human_num + sim.human_num_range (max_human_num); the live
                    // count of an environment is CnState::hn[e] (== H when hrange == 0)
  int hrange;       // sim.human_num_range: humans join / leave every 5 s (crowd_sim_pred.py:165-194)
  int hbase;        // sim.human_num
  int P;            // sim.predict_steps
  int W;            // spatial_edges row width: 2*(P+1) (CrowdSimPred) or 2 (CrowdSimVarNum)
  int const_vel;    // 1: CrowdSimPred-v0 'const_vel'; 0: CrowdSimVarNum-v0 'none'
  int randomize;    // env.randomize_attributes
  int goal_changing;      // humans.random_goal_changing
  int end_goal_changing;  // humans.end_goal_changing
  int sort_humans;        // args.sort_humans
  int nenv_total;         // env.nenv (global, across shards)
  uint32_t seed_base;     // thisSeed of env 0 of this shard = seed + rank_offset
  uint32_t phase_offset;  // 2000 'train', 0 'val', 1000 'test' (crowd_sim_var_num.py:329-334)
  uint32_t case_size;     // case_counter wraps at case_size[phase] (crowd_sim.py:104-105)
  int test_phase;         // 1: phase == 'test' (ground-truth look-ahead + 'future' danger zone)
  int lookahead_steps;    // buffer_len = predict_steps * pred_interval
  int pred_interval;
  double time_step, time_limit, pred_dt;   // pred_dt = time_step * pred_interval
  double circle_radius, arena_size;
  double discomfort_dist, discomfort_penalty_factor, success_reward, collision_penalty;
  double human_radius, human_vpref, robot_radius, robot_vpref, sensor_range;
  double human_fov, robot_fov;             // radians (config value * pi)
  double goal_change_chance;
  double orca_safety_space, orca_neighbor_dist;   // neighbor_dist: initial value of the global
  float orca_time_horizon;
  int social_force;       // humans.policy == 'social_force' (crowd_nav/policy/social_force.py) instead of ORCA
  double sf_A, sf_B, sf_KI;   // config.sf
  int defer_tries;        // warp-scope rejection-sampling budget (cn_env_event_kernel -> cn_env_event_heavy_kernel)
  int robot_policy;       // robot.policy: 0 caller's action, 1 'orca', 2 'social_force' (cn_robot_act)
  int robot_visible;      // robot.visible: the humans' solves take the robot as one more agent (cn_orca_build, cn_sf_action)
};

// Struct-of-arrays environment state in HBM.  Per-human arrays are [N][H] (human index
// fastest) so that the (env, human) thread mapping of the step kernel is coalesced.
struct CnState {
  // robot
  double *rpx, *rpy, *rgx, *rgy;     // fp64 like the reference's Python floats
  float *rvx, *rvy;                  // fp32-valued (clipped action)
  double *rwx, *rwy;                 // fp64 velocity of a social-force robot (the reference keeps Python floats; rvx / rvy
                                     // hold it narrowed, as the observation's temporal_edges read it)
  // the robot's own rvo2 simulator (robot_policy 1): created at the environment's FIRST robot solve and never rebuilt
  // (crowd_sim.py:184 creates robot.policy once per env process), so these survive episode installs
  uint8_t *rsim_exists;              // [N]
  float *rsim_nd;                    // [N] neighborDist frozen at creation (config.orca.neighbor_dist then)
  float *rsim_rother;                // [N][H] radii of the belief rows frozen at creation (+ 0.01 + safety_space)
  double *potential;                 // -|goal - pos| bookkeeping (crowd_sim_var_num.py:351-352)
  double *fut_pen;                   // future-intrusion penalty of the STORED prediction (crowd_sim_pred.py:222-231)
  double *nd_global;                 // process-global config.orca.neighbor_dist (agent.py:21-22)
  double *ep_ret;                    // bench.Monitor episode return
  int *ep_len;
  int *step_count;                   // global_time = step_count * time_step
  int *hn;                           // [N] live humans (slots [hn, H) are empty), constant H unless hrange > 0
  int *prep_hn;                      // [N] live humans of the prepared next episode
  uint32_t *case_counter;            // case_counter[phase]
  int32_t *seed_off;                 // thisSeed - seed_base of every environment (default: its index; a batched
                                     // evaluation replays the single-env test protocol with all zeros)
  // humans [N][H]
  double *hpx, *hpy, *hgx, *hgy, *hrad, *hvpref;
  float *hvx, *hvy;
  double *hwx, *hwy;                 // fp64 velocities of social-force humans (the reference keeps Python floats;
                                     // ORCA velocities are fp32-valued and live in hvx / hvy)
  // robot belief (last_human_states) [N][H]
  double *bpx, *bpy, *bvx, *bvy, *brad;
  uint8_t *vis;                      // human_visibility (to the robot)
  // per-human cached rvo2 simulator parameters (crowd_nav/policy/orca.py:79-95): frozen at creation
  uint8_t *sim_exists;               // [N][H]
  uint8_t *sim_n;                    // [N][H] agent count when the simulator was created (human_num_range > 0 or robot visible)
  float *sim_nd, *sim_rself, *sim_vmax;   // [N][H]
  float *sim_rother;                 // [N][H][H] (only when randomize)
  // legacy numpy MT19937 per environment
  uint32_t *mt;                      // [N][624]
  int *mt_pos;                       // [N]
  // PREPARED next episode (an episode's initial state is a pure function of (seed, case_counter), so
  // it is computed off the critical path and merely installed when the current episode ends)
  double *prep_robot;                // [N][4] px, py, gx, gy
  double *prep_hpx, *prep_hpy, *prep_hrad, *prep_hvpref;   // [N][H]
  double *prep_nd;                   // [N] config.orca.neighbor_dist after the spawn draws
  uint32_t *prep_mt;                 // [N][624] generator state after the reset draws
  int *prep_mt_pos;                  // [N]
  // diagnostics of the last step (parity tests)
  float *last_hvx, *last_hvy;        // ORCA output velocities [N][H]
  int *orca_nlines, *orca_fail;      // [N][H]
  // pre-solve (cn_env_kernels.cu, mode 3 -> mode 2): the humans' ORCA solve of the NEXT step, computed on the side stream
  // while the policy runs, handed to that step's finishing pass
  float *pre_vx, *pre_vy;            // [N][H]
  int *pre_nlf;                      // [N][H] nl | (fail + 1) << 8
  // per-step event flags written by the step kernel, consumed by the event kernel:
  // 0 = nothing, 1 = goal dynamics (respawn / goal change) pending, 2 = episode finished (reset)
  uint8_t *evt;                      // [N]
  // load balancing of the step kernel: slot -> environment permutation (identity until the first balance pass)
  int *perm;                         // [grid * epb] (entries >= N: empty slot)
  int *lp_cost;                      // [N] humans whose last solve needed linearProgram3 (cost estimate)
  uint8_t *spawn_overflow;           // [N] set when a rejection-sampling loop hit CN_MAX_SPAWN_TRIES
  // events whose rejection sampling exceeded the warp-scope budget, redone by cn_env_event_heavy_kernel:
  int *defer_list;                   // [N] env | event kind << 24
  int *defer_ctl;                    // [8] {count, finished-CTA ticket, total deferrals, total CTA batches, max batches of one CTA launch, ..}
  // overflow ORCA lines (k >= line_cap) of every step-kernel thread: [grid * block][ovf_stride] float4
  void *line_ovf;
  int ovf_stride;
};

// Caller-owned observation/result buffers (PyTorch tensors in the host mirror).
struct CnObs {
  float *robot_node;          // [N,1,7]
  float *temporal_edges;      // [N,1,2]
  float *spatial_edges;       // [N,H,W]
  float *detected_human_num;  // [N,1]
  uint8_t *visible_masks;     // [N,H] or nullptr
};

struct CnStepOut {
  float *reward;       // [N]
  uint8_t *done;       // [N]
  int32_t *info;       // [N] CN_INFO_*
  float *info_aux;     // [N] Danger.min_dist (0 in train phase)
  double *ep_ret;      // [N] episode return at done (bench.Monitor 'r')
  int32_t *ep_len;     // [N] episode length at done
  float *not_done;     // [N] optional: 1 - done (rollout-storage mask row)
};
