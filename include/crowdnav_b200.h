/*
 * crowdnav_b200 — C ABI of the CUDA-native (H100 / sm_90a) crowd-navigation rollout engine.
 *
 * Drop-in boundary for the reference's PPO-rollout hot path (SURVEY.md §8b).  The reference
 * has no FFI today (it is duck-typed Python); each entry point below names the reference
 * interface it replaces.  The Python host mirror (crowdnav_prediction_attngraph_b200/) binds these
 * with ctypes and re-exposes the reference's own VecEnv / Policy surface; INTEGRATION.md
 * shows the stub a maintainer of the reference would add.
 *
 * Conventions
 *   - every pointer named d_* is CALLER-OWNED DEVICE memory (e.g. a PyTorch CUDA tensor);
 *     h_* is caller-owned host memory.  Step calls never allocate.
 *   - calls enqueue work on `stream` (a cudaStream_t passed as void*) and do not synchronise,
 *     except the *_host variants, which copy through host buffers and return when done.
 *   - return value: 0 = ok, non-zero = error; cn_last_error() gives the message of the last
 *     failure on the calling thread.  A missing CUDA device is an error, never a CPU fallback.
 *   - one host thread per handle; handles on different GPUs are independent.
 *   - current device: the per-step entry points (cn_env_reset / cn_env_step, cn_policy_act, cn_gst_step,
 *     cn_copy_segments, cn_fetch_sync, cn_env_profile / cn_env_stage_ms) run on the handle's device and RESTORE the
 *     caller's current device before returning; the set-up calls (create / destroy / set_param / finalize,
 *     cn_env_state_copy, cn_env_step_host, cn_gst_reset) leave the handle's device current, like cudaSetDevice.
 */
#ifndef CROWDNAV_B200_H
#define CROWDNAV_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CN_ABI_VERSION 3

/* info codes — crowd_sim/envs/utils/info.py (Nothing, Timeout, Collision, ReachGoal, Danger) */
#define CN_INFO_NOTHING_C 0
#define CN_INFO_TIMEOUT_C 1
#define CN_INFO_COLLISION_C 2
#define CN_INFO_REACHGOAL_C 3
#define CN_INFO_DANGER_C 4

/* Flat snapshot of the reference Config the hot path reads
 * (crowd_nav/configs/config.py:16-120, arguments.py:47,206; make_env: rl/networks/envs.py:51-58). */
typedef struct cn_config {
  int32_t num_envs;          /* environments owned by this handle (this GPU's shard)            */
  int32_t nenv_total;        /* env.nenv: total environments of the job (case_counter stride)   */
  int32_t rank_offset;       /* global index of this shard's env 0 (thisSeed = seed + rank)     */
  int32_t seed;              /* --seed (arguments.py:47)                                        */
  int32_t human_num;         /* sim.human_num                                                    */
  int32_t predict_steps;     /* sim.predict_steps                                               */
  int32_t const_vel;         /* 1: CrowdSimPred-v0 / 'const_vel'; 0: CrowdSimVarNum-v0 / 'none' */
  int32_t randomize_attributes;   /* env.randomize_attributes                                   */
  int32_t random_goal_changing;   /* humans.random_goal_changing                                */
  int32_t end_goal_changing;      /* humans.end_goal_changing                                   */
  int32_t sort_humans;            /* args.sort_humans                                           */
  int32_t device;                 /* CUDA device ordinal                                        */
  int32_t phase;                  /* env.phase: 0 'train', 2 'test' (ground-truth look-ahead, 'future'
                                   * danger zone, test seeds; crowd_sim_pred.py:136-138)          */
  int32_t val_size, test_size;    /* env.val_size / env.test_size: case_counter wrap of the phase */
  int32_t human_num_range;        /* sim.human_num_range: humans join / leave every 5 s; observations are padded to
                                   * human_num + human_num_range rows (crowd_sim_pred.py:165-194)             */
  int32_t human_policy;           /* humans.policy: 0 'orca', 1 'social_force' (crowd_nav/policy/social_force.py) */
  int16_t robot_policy;           /* robot.policy: 0 the caller's action (a network policy), 1 'orca', 2 'social_force':
                                   * the step computes the robot's velocity itself and ignores d_action
                                   * (crowd_sim_var_num.py:371-377); CrowdSimVarNum-v0 with human_num_range 0 only */
  int16_t robot_visible;          /* robot.visible: 1 = every human's ORCA / social-force solve sees the robot (or, outside
                                   * the human's FOV, the dummy robot at (7, 7)) as one more agent (crowd_sim.py:695-699);
                                   * CrowdSimVarNum-v0 only.  robot_policy and robot_visible share the 4 bytes robot_policy
                                   * had as an int32, so the struct keeps its size and every offset (little-endian: a caller
                                   * that stores robot_policy as an int32 below 32768 leaves robot_visible 0)          */
  double time_step, time_limit, pred_timestep;
  double circle_radius, arena_size;
  double discomfort_dist, discomfort_penalty_factor, success_reward, collision_penalty;
  double human_radius, human_v_pref, human_fov;     /* FOV as multiples of pi, like the Config  */
  double robot_radius, robot_v_pref, robot_fov, sensor_range;
  double goal_change_chance;
  double orca_neighbor_dist, orca_safety_space, orca_time_horizon;
  double sf_A, sf_B, sf_KI;       /* config.sf (social-force humans)                                          */
} cn_config;

/* Observation buffers: the dict rl/networks/shmem_vec_env.py:109-116 returns, float32.       */
typedef struct cn_obs_ptrs {
  float *robot_node;          /* [N,1,7]                                                       */
  float *temporal_edges;      /* [N,1,2]                                                       */
  float *spatial_edges;       /* [N,H,W]  W = 2*(predict_steps+1) or 2                         */
  float *detected_human_num;  /* [N,1]                                                         */
  uint8_t *visible_masks;     /* [N,H] or NULL (CrowdSimVarNum-v0 only)                        */
} cn_obs_ptrs;

/* Per-step results: (rews, dones, infos) of ShmemVecEnv.step_wait + bench.Monitor's episode. */
typedef struct cn_step_ptrs {
  float *reward;       /* [N]                                                                  */
  uint8_t *done;       /* [N]                                                                  */
  int32_t *info;       /* [N] CN_INFO_*                                                        */
  float *info_aux;     /* [N] Danger.min_dist                                                  */
  double *ep_ret;      /* [N] info['episode']['r'] (valid where done)                          */
  int32_t *ep_len;     /* [N] info['episode']['l'] (valid where done)                          */
  float *not_done;     /* [N] optional (may be NULL): 1 - done, the `masks` row train.py:185 builds */
} cn_step_ptrs;

/* replaces: the per-tensor copies of RolloutStorage.insert (rl/networks/storage.py:70-86) -- up to
 * CN_MAX_COPY_SEGS device-to-device copies in ONE kernel launch on `stream`.                    */
#define CN_MAX_COPY_SEGS 16
typedef struct cn_copy_seg {
  void *dst;
  const void *src;
  size_t bytes;
} cn_copy_seg;
int cn_copy_segments(const cn_copy_seg *segs, int n, int device, void *stream);
/* cn_copy_segments sources may also be PINNED host memory (the reward / mask tensors train.py builds on the host,
 * rl/networks/storage.py:70-86 `insert`): the kernel reads them over the bus, no separate cudaMemcpyAsync per tensor.
 *
 * replaces: the result read-back of ShmemVecEnv.step_wait (rl/networks/shmem_vec_env.py:75-80: pipe recv + shared-memory
 * read of every worker) -- ONE device->pinned-host copy of the packed step outputs on `stream`, then a wait for the stream. */
int cn_fetch_sync(void *h_dst, const void *d_src, size_t bytes, int device, void *stream);

/* BASELINE config 3: GST trajectory predictor + VecPretextNormalize processing (one chain of launches per step).
 * replaces: VecPretextNormalize.reset / process_obs_rew (rl/vec_env/vec_pretext_normalize.py:85-191) and
 * CrowdNavPredInterfaceMultiEnv.forward (gst_updated/scripts/wrapper/crowd_nav_interface_parallel.py:45-114).     */
typedef struct cn_gst cn_gst;
int cn_gst_create(int num_envs, int human_num, int predict_steps, double robot_radius, double human_radius,
                  double collision_penalty, int device, cn_gst **out);
int cn_gst_destroy(cn_gst *g);
/* name = key of the predictor checkpoint's model_state_dict (st_model), data = float32 host array              */
int cn_gst_set_param(cn_gst *g, const char *name, const float *data, size_t count);
int cn_gst_finalize(cn_gst *g);
int cn_gst_reset(cn_gst *g, void *stream);
/* d_robot_node [N,7], d_spatial2 [N,H,2], d_visible [N,H]: raw CrowdSimPredRealGST-v0 observation (unsorted);
 * d_reward [N] in/out or NULL (+= future-collision penalty), d_penalty [N] out or NULL,
 * d_spatial_out [N,H,2*(predict_steps+1)]: predicted, distance-sorted spatial_edges.                           */
int cn_gst_step(cn_gst *g, const float *d_robot_node, const float *d_spatial2, const uint8_t *d_visible,
                float *d_reward, float *d_penalty, float *d_spatial_out, void *stream);
int64_t cn_gst_launch_count(cn_gst *g);

typedef struct cn_env cn_env;

const char *cn_last_error(void);
int cn_abi_version(void);

/* replaces: make_vec_envs / ShmemVecEnv.__init__ + env.configure (rl/networks/envs.py:97-140,
 * rl/networks/shmem_vec_env.py:26-58): N environments resident in HBM on cfg->device.          */
int cn_env_create(const cn_config *cfg, cn_env **out);
int cn_env_destroy(cn_env *env);

/* replaces: ShmemVecEnv.reset (shmem_vec_env.py:62-68) -> CrowdSimVarNum.reset for every env.  */
int cn_env_reset(cn_env *env, const cn_obs_ptrs *d_obs, void *stream);

/* replaces: ShmemVecEnv.step_async/step_wait + _subproc_worker 'step' (shmem_vec_env.py:70-80,
 * 138-142): CrowdSimPred.step for every env, auto-reset where done.  d_action: float32 [N,2].   */
int cn_env_step(cn_env *env, const float *d_action, const cn_obs_ptrs *d_obs,
                const cn_step_ptrs *d_out, void *stream);

/* Same as cn_env_step with HOST buffers (the numpy arrays of the reference's VecEnv contract):
 * H2D of the actions, the step, D2H of observations and results; synchronous.                  */
int cn_env_step_host(cn_env *env, const float *h_action, const cn_obs_ptrs *h_obs,
                     const cn_step_ptrs *h_out);

/* Parity-test access to the persistent state (SURVEY.md §8a'): copies the named field
 * ("hpx", "rpx", "bvx", "mt", ...) device->host (dir 0) or host->device (dir 1).
 * cn_env_state_bytes returns the field size in bytes (0 if unknown).                            */
size_t cn_env_state_bytes(cn_env *env, const char *name);
int cn_env_state_copy(cn_env *env, const char *name, void *h_buf, size_t bytes, int dir);

/* Number of kernels this library launched since the handle was created (bench gpu_launches).  */
int64_t cn_env_launch_count(cn_env *env);
/* measurement hooks (no reference equivalent): with profiling enabled every step records CUDA events around its launches;
 * cn_env_stage_ms synchronises and returns, for the LAST step, out3[0] = step kernel on the caller's stream (the whole
 * step, or only its finishing pass when the ORCA solve ran ahead on the side stream), out3[1] = event kernel(s) +
 * balancing pass and out3[2] = pre-solve of the next step, both on the engine's side stream (ms).                      */
int cn_env_profile(cn_env *env, int enable);
int cn_env_stage_ms(cn_env *env, float *out3);

/* ------------------------------------------------------------------------------------------ */
/* Attention-graph policy (rl/networks/model.py:56-80, selfAttn_srnn_temp_node.py:360-449).    */

typedef struct cn_policy cn_policy;

typedef struct cn_policy_config {
  int32_t num_envs;     /* N                                                                   */
  int32_t human_num;    /* H                                                                   */
  int32_t input_size;   /* spatial_edges row width (12 for Pred envs, 2 for VarNum)            */
  int32_t device;
  int32_t gemm_mode;    /* 0: fp32 CUDA-core GEMM; 1: wgmma 3xFP16 error-compensated GEMM      */
} cn_policy_config;

int cn_policy_create(const cn_policy_config *cfg, cn_policy **out);
int cn_policy_destroy(cn_policy *pol);

/* Upload one state_dict tensor by its reference key (SURVEY.md §2.3), float32 host data.       */
int cn_policy_set_param(cn_policy *pol, const char *key, const float *h_data, size_t count);
/* Fold/convert the uploaded parameters into the kernels' layouts; call after all set_param.    */
int cn_policy_finalize(cn_policy *pol, void *stream);

typedef struct cn_act_ptrs {
  /* inputs */
  const float *robot_node, *temporal_edges, *spatial_edges, *detected_human_num;
  const float *h_in;    /* rnn_hxs['human_node_rnn'] [N,1,128]                                  */
  const float *masks;   /* [N,1]                                                                */
  const float *noise;   /* [N,2] standard normal draws, or NULL for deterministic (mode)        */
  /* outputs */
  float *value;         /* [N,1]                                                                */
  float *action;        /* [N,2]                                                                */
  float *log_prob;      /* [N,1]                                                                */
  float *h_out;         /* [N,1,128]                                                            */
  float *action_mean;   /* [N,2] (dist.fc_mean output; parity tests)                            */
} cn_act_ptrs;

/* replaces: Policy.act (rl/networks/model.py:56-74) with infer=True.                           */
int cn_policy_act(cn_policy *pol, const cn_act_ptrs *d, void *stream);
int64_t cn_policy_launch_count(cn_policy *pol);
/* Rows (valid humans, sum over envs of detected_human_num) the last cn_policy_act processed;
 * synchronises the device.  The per-human pipeline runs on these compacted rows only.          */
int64_t cn_policy_last_rows(cn_policy *pol);

/* Per-stage device timing of cn_policy_act (CUDA events on the launching stream), for bench.py's
 * roofline line.  enable != 0 records events around every stage of subsequent calls;
 * cn_policy_stage_ms synchronises and writes the last call's stage durations (ms) into out[0..n).
 * Stage names: cn_policy_stage_name(i), i < cn_policy_stage_count().                            */
int cn_policy_profile(cn_policy *pol, int enable);
int cn_policy_stage_count(void);
const char *cn_policy_stage_name(int i);
int cn_policy_stage_ms(cn_policy *pol, float *out, int n);

/* ------------------------------------------------------------------------------------------ */
/* PPO update path (rl/ppo/ppo.py:36-101 -> Policy.evaluate_actions, selfAttn_srnn_temp_node.py:63-91): the
 * per-human linear layers forward / backward on the wgmma 3xFP16 GEMM in fp32-equivalent accuracy.
 * Stateless: every buffer (outputs, `d_saved` = what the backward needs from the forward, workspace) is caller-owned
 * device memory; sizes from the *_bytes functions.  Dimensions: N and K multiples of 64, M arbitrary.
 * act: 0 none, 1 ReLU.  replaces: torch F.linear(+ReLU) and its autograd backward for these layers.            */
size_t cn_update_linear_saved_bytes(int M, int K);
size_t cn_update_linear_ws_bytes(int M, int N, int K);
/* Y[M,N] = act(X[M,K] W[N,K]^T + b[N])                                                                         */
int cn_update_linear_fwd(const float *d_x, const float *d_w, const float *d_b, float *d_y, void *d_saved, void *d_ws,
                         size_t ws_bytes, int M, int N, int K, int act, int device, void *stream);
/* dZ = dY o [Y > 0] (ReLU); dX[M,K] = dZ W (d_dx may be NULL); dW[N,K] = dZ^T X; db[N] = colsum(dZ) (may be NULL) */
int cn_update_linear_bwd(const float *d_dy, const float *d_y, const void *d_saved, const float *d_w, float *d_dx,
                         float *d_dw, float *d_db, void *d_ws, size_t ws_bytes, int M, int N, int K, int act, int device,
                         void *stream);

/* Human-human multi-head attention core (softmax(q k^T / 8) v, 8 heads x 64) over COMPACTED rows: only the valid
 * humans of every sample have rows.  d_qkv [Mc,1536] = (q | k | v); d_row_start [B+1] prefix sums of the per-sample
 * human counts; d_row_env [Mc] sample index of a row; d_stats [Mc,16] soft-max max / sum per head (forward -> backward);
 * d_delta [Mc,8] scratch.  replaces: nn.MultiheadAttention's attention product with key_padding_mask
 * (rl/networks/selfAttn_srnn_temp_node.py:83-87) and its autograd backward.                                      */
int cn_update_attn_fwd(const float *d_qkv, const int *d_row_start, const int *d_row_env, int Mc, float *d_out,
                       float *d_stats, int device, void *stream);
int cn_update_attn_bwd(const float *d_qkv, const float *d_out, const float *d_dout, const float *d_stats,
                       const int *d_row_start, const int *d_row_env, int Mc, float *d_dqkv, float *d_delta, int device,
                       void *stream);

/* EndRNN's GRU over the T steps of a [T, N] minibatch with done-mask resets, one launch forward, one backward.
 * d_gi [T,N,384] = W_ih x + b_ih (precomputed), d_h0 [N,128], d_masks [T,N], d_whh [384,128], d_bhh [384];
 * d_out [T,N,128] hidden state after every step; d_saved [T,N,512] gates for the backward.  Backward: d_dout [T,N,128]
 * (+ optional d_dhT [N,128]) -> d_dgi [T,N,384], d_dghn [T,N,128] (n-gate part of the recurrent pre-activation; its r / z
 * parts equal d_dgi's), d_dh0 [N,128].  replaces: RNNBase._forward_gru (rl/networks/srnn_model.py:35-103).        */
int cn_update_gru_fwd(const float *d_gi, const float *d_h0, const float *d_masks, const float *d_whh, const float *d_bhh,
                      int T, int N, float *d_out, float *d_saved, int device, void *stream);
int cn_update_gru_bwd(const float *d_dout, const float *d_dhT, const float *d_out, const float *d_h0, const float *d_masks,
                      const float *d_saved, const float *d_whh, int T, int N, float *d_dgi, float *d_dghn, float *d_dh0,
                      int device, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* CROWDNAV_B200_H */
