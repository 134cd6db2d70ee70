// Host side of the attention-graph policy forward: parameter upload / folding and the
// per-rollout-step launch sequence behind cn_policy_act (replaces Policy.act,
// rl/networks/model.py:56-74, for base = selfAttn_merge_SRNN with sort_humans = True).
//
// Algebraic folds done once per parameter upload (fp64 accumulate, exact same function):
//   q/k/v_linear  o  MultiheadAttention.in_proj   ->  one 512 -> 1536 projection
//   MultiheadAttention.out_proj  o  spatial_linear -> one 512 -> 256 projection (ReLU after)
//   spatial_edge_layer folded into the robot side of the dot-product attention (u = W_s^T te)
//
// no_self_attn = 1 (the reference's use_self_attn = False, selfAttn_srnn_temp_node.py:340-345, :402-416): no
// human-human attention; spatial_linear = Linear(W, 128), ReLU, Linear(128, 256), ReLU runs straight on the compacted
// spatial_edges rows (layer 1 in the embed1 slot, layer 2 into sout) and feeds the unchanged robot-human attention.
//
// visible_masks = 1 (the reference's sort_humans = False, selfAttn_srnn_temp_node.py:375-383, :398-416): the attention
// masks are the caller's visible_masks instead of the detected_human_num prefix.  cn_mask_slots_kernel turns them into
// per-environment counts and slot lists; the same scan then gives row_start / mc, and the two gathers (pack_inputs,
// embed1) read slot row_slot[r] instead of r - row_start[e].  Every later kernel reads row_start / row_env only.
//
// gemm_mode 0: every layer on the fp32 CUDA-core GEMM (cn_gemm_f32_kernel).
// gemm_mode 1: every layer with K >= 64 on the wgmma 3xFP16 GEMM (cn_gemm_tc_kernel): activations
//              travel between layers as (hi, lo) fp16 pairs written by the producing kernel's epilogue.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

#include "../../include/crowdnav_b200.h"
#include "cn_host_util.h"
#include "cn_gemm_tc.h"
#include "cn_launch.cuh"
#include "cn_policy_kernels.cuh"
#include "cn_qkv_attn.cuh"

struct cn_policy {
  cn_policy_config cfg;
  int N, H, Win, M;
  bool nsa;           // cfg.no_self_attn: spatial_linear(spatial_edges), no human-human attention
  bool vm;            // cfg.visible_masks: rows = the visible slots of cn_act_ptrs.visible_masks
  const char* const* stage_names;   // this network's stages (kStageNames, kStageNamesNsa or their Vm variants)
  int num_stages;
  CnLaunchCtx lc;     // launch counter, PDL, first launch error, device allocations
  bool fuse_qkv;      // QKV projection + human-human attention in ONE kernel (cn_qkv_attn.cuh; opt-in, CN_FUSE_QKV=1)
  TcMat tWqkvH;       // folded QKV weight, rows head-major: [8][Q 64 | K 64 | V 64][512]
  CUtensorMap qa_ah, qa_al, qa_bh, qa_bl;   // 32-wide (SWIZZLE_64B) boxes of tE2 and tWqkvH for the fused kernel
  float* bqkvH = nullptr;
  int* tile_tab = nullptr;   // row tiles of the fused kernel (cn_qkv_tiles_kernel)
  cudaEvent_t ev_tiles;
  // human-human attention instance: R queries of an environment per warp (CN_ATTN_R = 1 (default), 2 or 4; R = 1 is
  // the fastest at H = 20, R = 2 at H = 50 and 100, DESIGN.md 3.4c)
  void (*attn_kernel)(const float*, const int*, const int*, const int*, const int*, float*, __half*, __half*);
  int attn_warps;
  int qkv_chunks;     // 1 (default): single pass; 2 (CN_QKV_CHUNKS=2): QKV + attention in two row chunks with overlap
  bool finalized;
  std::map<std::string, std::vector<float>> host;
  size_t ws_allocs;   // lc.allocs[0..ws_allocs) = workspace (kept); the rest = parameters of the last finalize
  // device parameters (fp32 kernel layouts)
  // no_self_attn: W1 / b1 = spatial_linear.0 and W2 / b2 = spatial_linear.2; Wqkv ... bos are not allocated
  float *W1, *b1, *W2, *b2, *Wqkv, *bqkv, *Wos, *bos;
  float *Wr, *br, *Wet, *bet, *WsT, *bs, *Wa, *ba, *Wih, *bih, *Whh, *bhh, *Wo, *bo;
  float *Woac, *boac;      // (actor.0 | critic.0) o output_linear folded: 128 -> 512
  float *Wac1, *bac1, *Wa2, *ba2, *Wc2, *bc2, *wv_, *bv, *Wm, *bm, *logstd;
  // tensor-core path: split weights (B operands; tile rows = 256 for per-human layers, 64 for per-env layers)
  TcMat tW2, tWqkv, tWos, tWet, tWsT, tWa, tWih, tWhh, tWo, tWac1, tWoac, tWa2, tWc2;
  // tensor-core path: split activations (A operands)
  TcMat tE1, tE2, tAo;                                  // per human rows
  TcMat tRs, tT1, tTe, tWv, tH0, tH1, tOut, tAc1, tA1, tC1;   // per environment rows (tTe / tA1 / tC1 = column views)
  // second stream: the robot branch / gh / critic.2 are independent of the per-human chain and run
  // concurrently with it (fork / join with events; capturable in a CUDA graph)
  cudaStream_t st2, st3;
  cudaEvent_t ev_fork, ev_join, ev_fork2, ev_join2, ev_fork3, ev_join3;
  // optional per-stage profiling
  bool profile;
  std::vector<cudaEvent_t> ev;
  // workspace
  int *row_start, *row_env, *mc;
  int *slot_tab, *row_slot;   // visible_masks only: [N * H] visible slots per environment, [M] slot of each row
  float* vis_count;           // visible_masks only: [N] rows per environment (the scan's input)
  float *x16, *e1, *e2, *qkv, *ao, *sout, *xr, *rs, *t1, *u, *wv, *h0, *gi, *gh, *outb, *ac1, *a2, *c2;
  TcStoreMap qkv_st, sout_st;   // store maps of the fp32 outputs of the BN = 256 GEMMs (gemm_mode 1)
};

// The robot-human attention in its dense layout, for the DS-RNN forward (cn_dsrnn.cu): the kernel template is
// defined, instantiated and launched in this translation unit only.
void cn_hr_attention_dense(CnLaunchCtx* c, cudaStream_t st, const float* s_out, const float* u, const float* te, int ldte,
                           int te_off, const float* b_s, int env_pitch, int env_off, int N, int H, float* wv,
                           __half* wv_hi, __half* wv_lo, int ldwh) {
  launch_k(c, cn_hr_attention_kernel<true>, dim3((N + 3) / 4), dim3(128), 0, st, s_out, u, te, ldte, te_off, b_s,
           (const int*)nullptr, env_pitch, env_off, N, H, wv, wv_hi, wv_lo, ldwh);
}

namespace {

int upload(cn_policy* p, float** dst, const std::vector<float>& src) {
  int rc = palloc(&p->lc, dst, src.size());
  if (rc) return rc;
  cudaError_t err = cudaMemcpy(*dst, src.data(), src.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) return cn_set_error("H2D param: %s", cudaGetErrorString(err));
  return 0;
}

const std::vector<float>* get(cn_policy* p, const char* key, size_t count) {
  auto it = p->host.find(key);
  if (it == p->host.end()) { cn_set_error("cn_policy_finalize: parameter '%s' was not set", key); return nullptr; }
  if (it->second.size() != count) {
    cn_set_error("cn_policy_finalize: parameter '%s' has %zu elements, expected %zu", key, it->second.size(), count);
    return nullptr;
  }
  return &it->second;
}

void gemm(cn_policy* p, cudaStream_t st, const float* A, int lda, const float* W, int ldw, const float* bias,
          float* C, int ldc, int M, int N, int K, int act, int act_lo = 0, int act_hi = 1 << 30,
          const int* m_ptr = nullptr, __half* oh = nullptr, __half* ol = nullptr) {
  dim3 grid((N + CN_GEMM_BN - 1) / CN_GEMM_BN, (M + CN_GEMM_BM - 1) / CN_GEMM_BM);
  launch_k(&p->lc, cn_gemm_f32_kernel, grid, dim3(256), 0, st, A, lda, W, ldw, bias, C, ldc, M, N, K, act, act_lo, act_hi, m_ptr, oh, ol);
}

const char* kStageNames[] = {"pack_inputs", "embed1_gemm", "embed2_gemm", "qkv_gemm", "hh_attention",
                             "outproj_spatial_gemm", "robot_branch_join", "hr_attention", "gru", "actor_critic_heads"};
const int kNumStages = sizeof(kStageNames) / sizeof(kStageNames[0]);
// no_self_attn: the two spatial_linear layers, then the same tail as stages 6-9 above
const char* kStageNamesNsa[] = {"pack_inputs", "spatial_linear0", "spatial_linear2", "robot_branch_join",
                                "hr_attention", "gru", "actor_critic_heads"};
const int kNumStagesNsa = sizeof(kStageNamesNsa) / sizeof(kStageNamesNsa[0]);
// visible_masks: the mask compaction first, then the stages above
const char* kStageNamesVm[] = {"mask_rows", "pack_inputs", "embed1_gemm", "embed2_gemm", "qkv_gemm", "hh_attention",
                               "outproj_spatial_gemm", "robot_branch_join", "hr_attention", "gru", "actor_critic_heads"};
const char* kStageNamesNsaVm[] = {"mask_rows", "pack_inputs", "spatial_linear0", "spatial_linear2",
                                  "robot_branch_join", "hr_attention", "gru", "actor_critic_heads"};

inline void mark(cn_policy* p, cudaStream_t st, int i) {
  p->lc.cur_stage = i < p->num_stages ? p->stage_names[i] : "end";
  if (p->profile) cudaEventRecord(p->ev[i], st);
}

}  // namespace

extern "C" {

int cn_policy_profile(cn_policy* p, int enable) {
  if (!p) return cn_set_error("cn_policy_profile: null argument");
  cudaSetDevice(p->cfg.device);
  if (enable && p->ev.empty()) {
    p->ev.resize(p->num_stages + 1);
    for (auto& e : p->ev) cudaEventCreate(&e);
  }
  p->profile = enable != 0;
  return 0;
}
int cn_policy_stage_count(void) { return kNumStages; }
const char* cn_policy_stage_name(int i) { return (i >= 0 && i < kNumStages) ? kStageNames[i] : ""; }
const char* cn_policy_handle_stage_name(cn_policy* p, int i) {
  return (p && i >= 0 && i < p->num_stages) ? p->stage_names[i] : "";
}
int cn_policy_handle_stage_count(cn_policy* p) { return p ? p->num_stages : 0; }
int cn_policy_stage_ms(cn_policy* p, float* out, int n) {
  if (!p || !out) return cn_set_error("cn_policy_stage_ms: null argument");
  if (p->ev.empty()) return cn_set_error("cn_policy_stage_ms: profiling was never enabled");
  cudaSetDevice(p->cfg.device);
  cudaError_t err = cudaEventSynchronize(p->ev[p->num_stages]);
  if (err != cudaSuccess) return cn_set_error("cn_policy_stage_ms: %s", cudaGetErrorString(err));
  for (int i = 0; i < n && i < p->num_stages; ++i) cudaEventElapsedTime(&out[i], p->ev[i], p->ev[i + 1]);
  return 0;
}

int cn_policy_create(const cn_policy_config* cfg, cn_policy** out) {
  if (!cfg || !out) return cn_set_error("cn_policy_create: null argument");
  *out = nullptr;
  if (cfg->num_envs <= 0 || cfg->human_num <= 0 || cfg->human_num > 128 || cfg->input_size <= 0 || cfg->input_size > 16)
    return cn_set_error("cn_policy_create: unsupported dims N=%d H=%d input=%d", cfg->num_envs, cfg->human_num,
                        cfg->input_size);
  int ndev = 0;
  cudaError_t err = cudaGetDeviceCount(&ndev);
  if (err != cudaSuccess || ndev == 0)
    return cn_set_error("cn_policy_create: no CUDA device (%s); this engine has no CPU fallback",
                        err == cudaSuccess ? "device count 0" : cudaGetErrorString(err));
  if (cfg->device < 0 || cfg->device >= ndev) return cn_set_error("cn_policy_create: bad device %d", cfg->device);
  cudaSetDevice(cfg->device);
  cn_policy* p = new cn_policy();
  p->cfg = *cfg;
  p->N = cfg->num_envs; p->H = cfg->human_num; p->Win = cfg->input_size; p->M = p->N * p->H;
  p->nsa = cfg->no_self_attn != 0;
  p->vm = cfg->visible_masks != 0;
  p->stage_names = p->nsa ? (p->vm ? kStageNamesNsaVm : kStageNamesNsa) : (p->vm ? kStageNamesVm : kStageNames);
  p->num_stages = (p->nsa ? kNumStagesNsa : kNumStages) + (p->vm ? 1 : 0);
  p->finalized = false; p->profile = false;
  cn_launch_init(&p->lc, cfg->device);
  {
    const char* qc = getenv("CN_QKV_CHUNKS");
    p->qkv_chunks = (qc && qc[0] == '2') ? 2 : 1;
    const char* ar = getenv("CN_ATTN_R");
    const int attn_r = ar ? atoi(ar) : 1;
    p->attn_kernel = attn_r == 1 ? cn_hh_attention_kernel<1, 4, 4> : (attn_r == 4 ? cn_hh_attention_kernel<4, 2, 2> : cn_hh_attention_kernel<2, 4, 4>);
    p->attn_warps = attn_r == 4 ? 2 : 4;
    const char* fq = getenv("CN_FUSE_QKV");
    // opt-in (CN_FUSE_QKV=1): parity green, but its attention is bound by the SM's shared-memory bandwidth, which it
    // shares with the operand fetch of the MMAs, and it does not overlap the next tile's MMAs (DESIGN.md 3.4b)
    p->fuse_qkv = !p->nsa && cfg->gemm_mode == 1 && p->qkv_chunks == 1 && (fq && fq[0] == '1') && p->N <= QA_MAX_ENVS && p->H <= 128;
  }
  cudaEventCreateWithFlags(&p->ev_tiles, cudaEventDisableTiming);
  cudaStreamCreateWithFlags(&p->st2, cudaStreamNonBlocking);
  cudaStreamCreateWithFlags(&p->st3, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&p->ev_fork3, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_join3, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_fork2, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_join2, cudaEventDisableTiming);
  const size_t M = (size_t)p->M, N = (size_t)p->N;
  const int Mi = p->M, Ni = p->N;
  int rc = 0;
#define WS(name, count) if (!rc) rc = palloc(&p->lc, &p->name, (count))
  {
    float* q = nullptr;
    if (!rc) rc = palloc(&p->lc, &q, N + 2);
    p->row_start = reinterpret_cast<int*>(q);
    if (!rc) rc = palloc(&p->lc, &q, 4);
    p->mc = reinterpret_cast<int*>(q);
    if (!rc) rc = palloc(&p->lc, &q, M + 1);
    p->row_env = reinterpret_cast<int*>(q);
    if (!rc) rc = palloc(&p->lc, &q, 2 * N + 4);
    p->tile_tab = reinterpret_cast<int*>(q);
    if (p->vm) {
      if (!rc) rc = palloc(&p->lc, &q, M);
      p->slot_tab = reinterpret_cast<int*>(q);
      if (!rc) rc = palloc(&p->lc, &q, M + 1);
      p->row_slot = reinterpret_cast<int*>(q);
      if (!rc) rc = palloc(&p->lc, &p->vis_count, N);
    }
  }
  WS(x16, M * 16); WS(e1, M * 128); WS(sout, M * 256);
  if (!p->nsa) { WS(e2, M * 512); WS(qkv, M * 1536); WS(ao, M * 512); }   // human-human attention only
  WS(xr, N * 16); WS(rs, N * 256); WS(t1, N * 128); WS(u, N * 256); WS(wv, N * 256); WS(h0, N * 128);
  WS(gi, N * 384); WS(gh, N * 384); WS(outb, N * 256); WS(ac1, N * 512); WS(a2, N * 256); WS(c2, N * 256);
#undef WS
  if (!rc && cfg->gemm_mode == 1) {
    // A operands: box rows = 128 (TC_BM)
    // per-human rows feed the BN = 256 instance, per-environment rows the BN = 64 one
    rc = tc_alloc(&p->lc, p->tE1, Mi, 128, TC_BM, tc_box_k(256));
    if (!rc && !p->nsa) rc = tc_alloc(&p->lc, p->tE2, Mi, 512, TC_BM, tc_box_k(256));
    if (!rc && !p->nsa) rc = tc_alloc(&p->lc, p->tAo, Mi, 512, TC_BM, tc_box_k(256));
    if (!rc) rc = tc_alloc(&p->lc, p->tRs, Ni, 256, TC_BM, tc_box_k(64));
    if (!rc) rc = tc_alloc(&p->lc, p->tT1, Ni, 128, TC_BM, tc_box_k(64));   // [enc | te] then [enc | emb]
    if (!rc) rc = tc_view(p->tTe, p->tT1, 64, Ni, 64, TC_BM);           // te = columns 64..127
    if (!rc) rc = tc_alloc(&p->lc, p->tWv, Ni, 256, TC_BM, tc_box_k(64));
    if (!rc) rc = tc_alloc(&p->lc, p->tH0, Ni, 128, TC_BM, tc_box_k(64));
    if (!rc) rc = tc_alloc(&p->lc, p->tH1, Ni, 128, TC_BM, tc_box_k(64));
    if (!rc) rc = tc_alloc(&p->lc, p->tOut, Ni, 256, TC_BM, tc_box_k(64));
    if (!rc) rc = tc_alloc(&p->lc, p->tAc1, Ni, 512, TC_BM, tc_box_k(64));
    if (!rc) rc = tc_view(p->tA1, p->tAc1, 0, Ni, 256, TC_BM);          // actor.0 half
    if (!rc) rc = tc_view(p->tC1, p->tAc1, 256, Ni, 256, TC_BM);        // critic.0 half
    // fp32 outputs of the BN = 256 GEMMs (qkv, outproj_spatial)
    if (!rc && !p->nsa) rc = make_store_map(&p->qkv_st, p->qkv, 4, Mi, 1536, 1536);
    if (!rc) rc = make_store_map(&p->sout_st, p->sout, 4, Mi, 256, 256);
    if (!rc) rc = tc_set_attrs();
    if (!rc && !p->nsa) {
      err = cudaFuncSetAttribute(cn_qkv_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, QA_SMEM_BYTES);
      if (err != cudaSuccess) rc = cn_set_error("cudaFuncSetAttribute(qkv_attn): %s", cudaGetErrorString(err));
    }
  }
  if (rc) { cn_policy_destroy(p); return rc; }
  p->ws_allocs = p->lc.allocs.size();
  *out = p;
  return 0;
}

int cn_policy_destroy(cn_policy* p) {
  if (!p) return 0;
  cudaSetDevice(p->cfg.device);
  cn_launch_free(&p->lc);
  for (auto& e : p->ev) cudaEventDestroy(e);
  if (p->st2) {
    cudaStreamDestroy(p->st2);
    cudaStreamDestroy(p->st3); cudaEventDestroy(p->ev_fork3); cudaEventDestroy(p->ev_join3); cudaEventDestroy(p->ev_tiles);
    cudaEventDestroy(p->ev_fork); cudaEventDestroy(p->ev_join); cudaEventDestroy(p->ev_fork2); cudaEventDestroy(p->ev_join2);
  }
  delete p;
  return 0;
}

int cn_policy_set_param(cn_policy* p, const char* key, const float* h_data, size_t count) {
  if (!p || !key || !h_data) return cn_set_error("cn_policy_set_param: null argument");
  p->host[key] = std::vector<float>(h_data, h_data + count);
  p->finalized = false;
  return 0;
}

int cn_policy_finalize(cn_policy* p, void* stream) {
  if (!p) return cn_set_error("cn_policy_finalize: null argument");
  cudaSetDevice(p->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  const int Win = p->Win;
  // the per-human chain: embedding_layer -> q/k/v_linear -> multihead_attn -> spatial_linear (512 -> 256), or with
  // no_self_attn spatial_linear alone (W -> 128 -> 256) and no spatial_attn.* key at all
  const std::vector<float> *w1, *b1, *w2, *b2, *wq = nullptr, *bq = nullptr, *wk = nullptr, *bk = nullptr;
  const std::vector<float> *wvv = nullptr, *bvv = nullptr, *win = nullptr, *bin = nullptr, *wout = nullptr;
  const std::vector<float> *bout = nullptr, *wsl = nullptr, *bsl = nullptr;
#define GETP(var, key, count) if (!(var = get(p, key, (count)))) return 1
  if (p->nsa) {
    GETP(w1, "base.spatial_linear.0.weight", (size_t)128 * Win);
    GETP(b1, "base.spatial_linear.0.bias", 128);
    GETP(w2, "base.spatial_linear.2.weight", (size_t)256 * 128);
    GETP(b2, "base.spatial_linear.2.bias", 256);
  } else {
    GETP(w1, "base.spatial_attn.embedding_layer.0.weight", (size_t)128 * Win);
    GETP(b1, "base.spatial_attn.embedding_layer.0.bias", 128);
    GETP(w2, "base.spatial_attn.embedding_layer.2.weight", (size_t)512 * 128);
    GETP(b2, "base.spatial_attn.embedding_layer.2.bias", 512);
    GETP(wq, "base.spatial_attn.q_linear.weight", (size_t)512 * 512);
    GETP(bq, "base.spatial_attn.q_linear.bias", 512);
    GETP(wk, "base.spatial_attn.k_linear.weight", (size_t)512 * 512);
    GETP(bk, "base.spatial_attn.k_linear.bias", 512);
    GETP(wvv, "base.spatial_attn.v_linear.weight", (size_t)512 * 512);
    GETP(bvv, "base.spatial_attn.v_linear.bias", 512);
    GETP(win, "base.spatial_attn.multihead_attn.in_proj_weight", (size_t)1536 * 512);
    GETP(bin, "base.spatial_attn.multihead_attn.in_proj_bias", 1536);
    GETP(wout, "base.spatial_attn.multihead_attn.out_proj.weight", (size_t)512 * 512);
    GETP(bout, "base.spatial_attn.multihead_attn.out_proj.bias", 512);
    GETP(wsl, "base.spatial_linear.0.weight", (size_t)256 * 512);
    GETP(bsl, "base.spatial_linear.0.bias", 256);
  }
#undef GETP
#define GET(var, key, count) const std::vector<float>* var = get(p, key, (count)); if (!var) return 1
  GET(wr, "base.robot_linear.0.weight", (size_t)256 * 9);
  GET(br, "base.robot_linear.0.bias", 256);
  GET(wt, "base.attn.temporal_edge_layer.0.weight", (size_t)64 * 256);
  GET(bt, "base.attn.temporal_edge_layer.0.bias", 64);
  GET(ws, "base.attn.spatial_edge_layer.0.weight", (size_t)64 * 256);
  GET(bs, "base.attn.spatial_edge_layer.0.bias", 64);
  GET(we, "base.humanNodeRNN.encoder_linear.weight", (size_t)64 * 256);
  GET(be, "base.humanNodeRNN.encoder_linear.bias", 64);
  GET(wa, "base.humanNodeRNN.edge_attention_embed.weight", (size_t)64 * 256);
  GET(ba, "base.humanNodeRNN.edge_attention_embed.bias", 64);
  GET(wih, "base.humanNodeRNN.gru.weight_ih_l0", (size_t)384 * 128);
  GET(whh, "base.humanNodeRNN.gru.weight_hh_l0", (size_t)384 * 128);
  GET(bih, "base.humanNodeRNN.gru.bias_ih_l0", 384);
  GET(bhh, "base.humanNodeRNN.gru.bias_hh_l0", 384);
  GET(wo, "base.humanNodeRNN.output_linear.weight", (size_t)256 * 128);
  GET(bo, "base.humanNodeRNN.output_linear.bias", 256);
  GET(wa0, "base.actor.0.weight", (size_t)256 * 256);
  GET(ba0, "base.actor.0.bias", 256);
  GET(wa2, "base.actor.2.weight", (size_t)256 * 256);
  GET(ba2, "base.actor.2.bias", 256);
  GET(wc0, "base.critic.0.weight", (size_t)256 * 256);
  GET(bc0, "base.critic.0.bias", 256);
  GET(wc2, "base.critic.2.weight", (size_t)256 * 256);
  GET(bc2, "base.critic.2.bias", 256);
  GET(wcl, "base.critic_linear.weight", 256);
  GET(bcl, "base.critic_linear.bias", 1);
  GET(wm, "dist.fc_mean.weight", (size_t)2 * 256);
  GET(bm, "dist.fc_mean.bias", 2);
  GET(ls, "dist.logstd._bias", 2);
#undef GET
  // release device parameters of a previous finalize (workspace allocations come first and stay)
  cudaStreamSynchronize(st);
  for (size_t i = p->ws_allocs; i < p->lc.allocs.size(); ++i) cudaFree(p->lc.allocs[i]);
  p->lc.allocs.resize(p->ws_allocs);
  int rc = 0;
  auto pad_k = [](const std::vector<float>& w, int rows, int k, int kp) {
    std::vector<float> o((size_t)rows * kp, 0.0f);
    for (int r = 0; r < rows; ++r) for (int c = 0; c < k; ++c) o[(size_t)r * kp + c] = w[(size_t)r * k + c];
    return o;
  };
  auto cat = [](const std::vector<float>& a, const std::vector<float>& b) {
    std::vector<float> o(a); o.insert(o.end(), b.begin(), b.end()); return o;
  };
#define UP(dst, vec) if (!rc) rc = upload(p, &p->dst, (vec))
  UP(W1, pad_k(*w1, 128, Win, 16)); UP(b1, *b1); UP(W2, *w2); UP(b2, *b2);
  UP(Wr, pad_k(*wr, 256, 9, 16)); UP(br, *br);
  UP(Wet, cat(*we, *wt)); UP(bet, cat(*be, *bt));           // rows 0..63 encoder_linear, 64..127 temporal_edge_layer
  {
    std::vector<float> wst((size_t)256 * 64);                // W_s^T: [256][64]
    for (int r = 0; r < 64; ++r) for (int c = 0; c < 256; ++c) wst[(size_t)c * 64 + r] = (*ws)[(size_t)r * 256 + c];
    UP(WsT, wst);
  }
  UP(bs, *bs); UP(Wa, *wa); UP(ba, *ba); UP(Wih, *wih); UP(bih, *bih); UP(Whh, *whh); UP(bhh, *bhh);
  UP(Wo, *wo); UP(bo, *bo);
  UP(Wac1, cat(*wa0, *wc0)); UP(bac1, cat(*ba0, *bc0));      // rows 0..255 actor.0, 256..511 critic.0
  UP(Wa2, *wa2); UP(ba2, *ba2); UP(Wc2, *wc2); UP(bc2, *bc2);
  UP(wv_, *wcl); UP(bv, *bcl); UP(Wm, *wm); UP(bm, *bm); UP(logstd, *ls);
#undef UP
  if (!rc) rc = palloc(&p->lc, &p->Woac, (size_t)512 * 128);
  if (!rc) rc = palloc(&p->lc, &p->boac, 512);
  if (rc) return rc;
  // Woac = [actor.0 ; critic.0] (512x256) @ output_linear (256x128);  boac = [actor.0 ; critic.0] @ bo + bac1
  // (output_linear has no activation and feeds only the two MLPs, selfAttn_srnn_temp_node.py:438-447)
  cn_fold_mm_kernel<<<dim3(1, 512), 128, 0, st>>>(p->Wac1, p->Wo, p->Woac, 512, 128, 256);
  cn_fold_mv_kernel<<<4, 128, 0, st>>>(p->Wac1, p->bo, p->bac1, p->boac, 512, 256);
  if (!p->nsa) {
    // folded projections of the human-human attention
    float *d_win = nullptr, *d_bin = nullptr, *d_wl[3] = {nullptr, nullptr, nullptr}, *d_bl[3] = {nullptr, nullptr, nullptr};
    float *d_wout = nullptr, *d_bout = nullptr, *d_wsl = nullptr, *d_bsl = nullptr;
    if (!rc) rc = upload(p, &d_win, *win);
    if (!rc) rc = upload(p, &d_bin, *bin);
    const std::vector<float>* wl[3] = {wq, wk, wvv};
    const std::vector<float>* bl[3] = {bq, bk, bvv};
    for (int i = 0; i < 3 && !rc; ++i) { rc = upload(p, &d_wl[i], *wl[i]); if (!rc) rc = upload(p, &d_bl[i], *bl[i]); }
    if (!rc) rc = upload(p, &d_wout, *wout);
    if (!rc) rc = upload(p, &d_bout, *bout);
    if (!rc) rc = upload(p, &d_wsl, *wsl);
    if (!rc) rc = upload(p, &d_bsl, *bsl);
    if (!rc) rc = palloc(&p->lc, &p->Wqkv, (size_t)1536 * 512);
    if (!rc) rc = palloc(&p->lc, &p->bqkv, 1536);
    if (!rc) rc = palloc(&p->lc, &p->Wos, (size_t)256 * 512);
    if (!rc) rc = palloc(&p->lc, &p->bos, 256);
    if (rc) return rc;
    for (int i = 0; i < 3; ++i) {
      // Wf_i = Win_i (512x512) @ Wl_i (512x512);  bf_i = Win_i @ bl_i + bin_i
      cn_fold_mm_kernel<<<dim3(4, 512), 128, 0, st>>>(d_win + (size_t)i * 512 * 512, d_wl[i],
                                                       p->Wqkv + (size_t)i * 512 * 512, 512, 512, 512);
      cn_fold_mv_kernel<<<4, 128, 0, st>>>(d_win + (size_t)i * 512 * 512, d_bl[i], d_bin + i * 512, p->bqkv + i * 512, 512, 512);
    }
    // Wos = Wsl (256x512) @ Wout (512x512);  bos = Wsl @ bout + bsl
    cn_fold_mm_kernel<<<dim3(4, 256), 128, 0, st>>>(d_wsl, d_wout, p->Wos, 256, 512, 512);
    cn_fold_mv_kernel<<<2, 128, 0, st>>>(d_wsl, d_bout, d_bsl, p->bos, 256, 512);
  }
  if (p->cfg.gemm_mode == 1) {
    // fp16 (hi, lo) split of the tensor-core weights, pre-scaled by 2^6 (exact) so lo stays normal.
    // B-tile rows: 256 for the per-human layers (large M), 64 for the per-environment layers.
    // no_self_attn: W2 is spatial_linear.2 [256, 128]; there is no Wqkv / Wos (rows = 0: skipped)
    const int nh = p->nsa ? 0 : 1;
    struct { float* src; TcMat* t; int rows, k, bn; } tw[13] = {
        {p->Woac, &p->tWoac, 512, 128, 64},
        {p->W2, &p->tW2, p->nsa ? 256 : 512, 128, 256}, {p->Wqkv, &p->tWqkv, 1536 * nh, 512, 256},
        {p->Wos, &p->tWos, 256 * nh, 512, 256},
        {p->Wet, &p->tWet, 128, 256, 64},   {p->WsT, &p->tWsT, 256, 64, 64},      {p->Wa, &p->tWa, 64, 256, 64},
        {p->Wih, &p->tWih, 384, 128, 64},   {p->Whh, &p->tWhh, 384, 128, 64},     {p->Wo, &p->tWo, 256, 128, 64},
        {p->Wac1, &p->tWac1, 512, 256, 64}, {p->Wa2, &p->tWa2, 256, 256, 64},     {p->Wc2, &p->tWc2, 256, 256, 64}};
    for (auto& t : tw) {
      if (!t.rows) continue;
      rc = tc_alloc(&p->lc, *t.t, t.rows, t.k, t.bn, tc_box_k(t.bn));
      if (rc) return rc;
      split16(&p->lc, st, t.src, 64.0f, t.t->hi, t.t->lo, (size_t)t.rows * t.k);
    }
    if (p->fuse_qkv) {
      // head-major copy of the folded QKV projection for the fused kernel: row h * 192 + s * 64 + d <- row s * 512 + h * 64 + d
      float* wh = nullptr;
      rc = palloc(&p->lc, &wh, (size_t)1536 * 512);
      if (!rc) rc = palloc(&p->lc, &p->bqkvH, 1536);
      if (!rc) rc = tc_alloc(&p->lc, p->tWqkvH, 1536, 512, QA_BN, QA_BK);
      if (!rc) rc = make_map(&p->qa_bh, p->tWqkvH.hi, 1536, 512, QA_BN, 512, QA_BK);
      if (!rc) rc = make_map(&p->qa_bl, p->tWqkvH.lo, 1536, 512, QA_BN, 512, QA_BK);
      if (!rc) rc = make_map(&p->qa_ah, p->tE2.hi, p->M, 512, TC_BM, 512, QA_BK);
      if (!rc) rc = make_map(&p->qa_al, p->tE2.lo, p->M, 512, TC_BM, 512, QA_BK);
      if (rc) return rc;
      cn_head_major_kernel<<<1536, 128, 0, st>>>(p->Wqkv, p->bqkv, wh, p->bqkvH);
      split16(&p->lc, st, wh, 64.0f, p->tWqkvH.hi, p->tWqkvH.lo, (size_t)1536 * 512);
    }
  }
  cudaError_t err = cudaStreamSynchronize(st);
  if (err != cudaSuccess) return cn_set_error("cn_policy_finalize: %s", cudaGetErrorString(err));
  p->finalized = true;
  return 0;
}

int cn_policy_act(cn_policy* p, const cn_act_ptrs* d, void* stream) {
  if (!p || !d) return cn_set_error("cn_policy_act: null argument");
  if (!p->finalized) return cn_set_error("cn_policy_act: call cn_policy_finalize after setting parameters");
  if (!d->robot_node || !d->temporal_edges || !d->spatial_edges || !d->detected_human_num || !d->h_in || !d->masks ||
      !d->value || !d->action || !d->log_prob || !d->h_out)
    return cn_set_error("cn_policy_act: missing input/output pointer");
  if (p->vm && !d->visible_masks)
    return cn_set_error("cn_policy_act: visible_masks is NULL, and this handle was created with visible_masks = 1 "
                        "(sort_humans = False)");
  CnDeviceGuard guard(p->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  const int N = p->N, H = p->H, M = p->M;
  const bool tcm = p->cfg.gemm_mode == 1;
  const int* mc = p->mc;
  const int ALL = 1 << 30;
  // o: stage index offset (visible_masks: stage 0 is the mask compaction)
  const int o = p->vm ? 1 : 0;
  if (p->vm) {
    mark(p, st, 0);
    launch_k(&p->lc, cn_mask_slots_kernel, dim3((N + 7) / 8), dim3(256), 0, st, d->visible_masks, N, H, p->vis_count,
             p->slot_tab);
  }
  mark(p, st, o);
  // 0. compaction offsets, pack / pad inputs, h0 = h * mask
  {
    launch_k(&p->lc, cn_row_offsets_kernel, dim3(1), dim3(1024), 0, st, p->vm ? p->vis_count : d->detected_human_num, N, H,
             p->row_start, p->mc);
    const int total = (!tcm && M * 16 > N * 128) ? M * 16 : N * 128;
    launch_k(&p->lc, p->vm ? cn_pack_inputs_kernel<true> : cn_pack_inputs_kernel<false>, dim3((total + 255) / 256), dim3(256), 0, st,
                                                               d->spatial_edges, p->Win, H, N, p->row_start, p->row_env,
                                                               p->slot_tab, p->row_slot, tcm ? nullptr : p->x16,
                                                               d->temporal_edges, d->robot_node, d->h_in, d->masks, p->xr,
                                                               p->h0, tcm ? p->tH0.hi : nullptr, tcm ? p->tH0.lo : nullptr);
  }
  // fork: the robot branch (rs, [enc|te], u) and gh only depend on the packed inputs
  cudaStream_t s2 = p->st2;
  cudaEventRecord(p->ev_fork, st);
  cudaStreamWaitEvent(s2, p->ev_fork, 0);
  if (p->fuse_qkv) {
    cn_qkv_tiles_kernel<<<1, 1024, 0, s2>>>(p->row_start, N, p->tile_tab);
    p->lc.launches += 1;
    cudaEventRecord(p->ev_tiles, s2);
  }
  if (tcm) {
    gemm(p, s2, p->xr, 16, p->Wr, 16, p->br, nullptr, 256, N, 256, 16, CN_ACT_RELU, 0, ALL, nullptr, p->tRs.hi, p->tRs.lo);
    gemm_tc(&p->lc, s2, p->tRs, p->tWet, N, 128, 256, 64, p->bet, CN_ACT_RELU, out_both(p->t1, 128, p->tT1), nullptr, 0, 64);
    gemm_tc(&p->lc, s2, p->tTe, p->tWsT, N, 256, 64, 64, nullptr, CN_ACT_NONE, out32(p->u, 256));
    gemm_tc(&p->lc, s2, p->tH0, p->tWhh, N, 384, 128, 64, p->bhh, CN_ACT_NONE, out32(p->gh, 384));
  } else {
    gemm(p, s2, p->xr, 16, p->Wr, 16, p->br, p->rs, 256, N, 256, 16, CN_ACT_RELU);
    gemm(p, s2, p->rs, 256, p->Wet, 256, p->bet, p->t1, 128, N, 128, 256, CN_ACT_RELU, 0, 64);   // [enc | te]
    gemm(p, s2, p->t1 + 64, 128, p->WsT, 64, nullptr, p->u, 256, N, 256, 64, CN_ACT_NONE);        // u = W_s^T te
    gemm(p, s2, p->h0, 128, p->Whh, 128, p->bhh, p->gh, 384, N, 384, 128, CN_ACT_NONE);
  }
  cudaEventRecord(p->ev_join, s2);
  // 1. human-human branch over the Mc = sum_e n_e valid rows (device-side count p->mc)
  mark(p, st, o + 1);
  if (tcm) {
    launch_k(&p->lc, p->vm ? cn_embed1_kernel<true> : cn_embed1_kernel<false>, dim3(p->lc.num_sms * 6), dim3(256), 0, st,
             d->spatial_edges, p->Win, H, p->row_start, p->row_env, p->row_slot, p->mc, p->W1, p->b1, p->tE1.hi, p->tE1.lo);
  } else gemm(p, st, p->x16, 16, p->W1, 16, p->b1, p->e1, 128, M, 128, 16, CN_ACT_RELU, 0, ALL, mc);
  mark(p, st, o + 2);
  if (p->nsa) {
    // no_self_attn: spatial_linear.2 + ReLU is the last per-human layer, straight into sout
    if (tcm) gemm_tc(&p->lc, st, p->tE1, p->tW2, M, 256, 128, 256, p->b2, CN_ACT_RELU, out32(p->sout, 256, &p->sout_st), mc);
    else gemm(p, st, p->e1, 128, p->W2, 128, p->b2, p->sout, 256, M, 256, 128, CN_ACT_RELU, 0, ALL, mc);
  } else {
    if (tcm) gemm_tc(&p->lc, st, p->tE1, p->tW2, M, 512, 128, 256, p->b2, CN_ACT_RELU, out16(p->tE2), mc);
    else gemm(p, st, p->e1, 128, p->W2, 128, p->b2, p->e2, 512, M, 512, 128, CN_ACT_RELU, 0, ALL, mc);
    mark(p, st, o + 3);
    if (tcm) {
      // Optional experiment (CN_QKV_CHUNKS=2): QKV projection + attention in two row chunks split at an environment
      // boundary so that chunk 0's attention (side stream) overlaps chunk 1's GEMM.  Off by default: at H = 20 the
      // attention is load-latency bound, not L2-capacity bound, and the overlap does not pay; at H = 50 and 100 it
      // saves 0.4-3 % of the forward (DESIGN.md 3.4c).
      const int* mid = p->row_start + N / 2;
      __half* ah = p->tAo.hi;
      __half* al = p->tAo.lo;
      if (p->fuse_qkv) {
        // one kernel: projection tile (128 rows of whole environments x one head's Q | K | V) -> attention -> tAo
        cudaStreamWaitEvent(st, p->ev_tiles, 0);                 // tile table from the side stream
        launch_k(&p->lc, cn_qkv_attn_kernel, dim3(p->lc.num_sms), dim3(QA_THREADS), QA_SMEM_BYTES, st, p->qa_ah, p->qa_al, p->qa_bh,
                 p->qa_bl, p->bqkvH, 1.0f / 64.0f, p->tile_tab, p->row_start, p->row_env, ah, al,
                 getenv("CN_QA_DBG") ? atoi(getenv("CN_QA_DBG")) : 0);
        mark(p, st, o + 4);
      } else if (p->qkv_chunks == 1) {
        gemm_tc(&p->lc, st, p->tE2, p->tWqkv, M, 1536, 512, 256, p->bqkv, CN_ACT_NONE, out32(p->qkv, 1536, &p->qkv_st), mc);
        mark(p, st, o + 4);
        launch_k(&p->lc, p->attn_kernel, dim3(p->lc.num_sms * 64 / p->attn_warps), dim3(p->attn_warps * 32), 0, st, p->qkv, p->row_start, p->row_env, mc, nullptr,
                                                                               nullptr, ah, al);
      } else {
      gemm_tc(&p->lc, st, p->tE2, p->tWqkv, M, 1536, 512, 256, p->bqkv, CN_ACT_NONE, out32(p->qkv, 1536, &p->qkv_st), mid);
      cudaEventRecord(p->ev_fork3, st);
      cudaStreamWaitEvent(p->st3, p->ev_fork3, 0);
      launch_k(&p->lc, p->attn_kernel, dim3(p->lc.num_sms * 32 / p->attn_warps), dim3(p->attn_warps * 32), 0, p->st3, p->qkv, p->row_start, p->row_env, mid, nullptr,
                                                                                nullptr, ah, al);
      cudaEventRecord(p->ev_join3, p->st3);
      gemm_tc(&p->lc, st, p->tE2, p->tWqkv, M, 1536, 512, 256, p->bqkv, CN_ACT_NONE, out32(p->qkv, 1536, &p->qkv_st), mc, 0, 1 << 30, mid);
      mark(p, st, o + 4);
      launch_k(&p->lc, p->attn_kernel, dim3(p->lc.num_sms * 64 / p->attn_warps), dim3(p->attn_warps * 32), 0, st, p->qkv, p->row_start, p->row_env, mc, mid, nullptr,
                                                                             ah, al);
      cudaStreamWaitEvent(st, p->ev_join3, 0);
      }
    } else {
      gemm(p, st, p->e2, 512, p->Wqkv, 512, p->bqkv, p->qkv, 1536, M, 1536, 512, CN_ACT_NONE, 0, ALL, mc);
      mark(p, st, o + 4);
      launch_k(&p->lc, p->attn_kernel, dim3(p->lc.num_sms * 64 / p->attn_warps), dim3(p->attn_warps * 32), 0, st, p->qkv, p->row_start, p->row_env, p->mc, nullptr,
                                                                             p->ao, nullptr, nullptr);
    }
    mark(p, st, o + 5);
    if (tcm) gemm_tc(&p->lc, st, p->tAo, p->tWos, M, 256, 512, 256, p->bos, CN_ACT_RELU, out32(p->sout, 256, &p->sout_st), mc);
    else gemm(p, st, p->ao, 512, p->Wos, 512, p->bos, p->sout, 256, M, 256, 512, CN_ACT_RELU, 0, ALL, mc);
  }
  // 2. join the robot branch (stage indices from here on: the last four of the handle's stages)
  const int tail = p->num_stages - 4;
  mark(p, st, tail);
  cudaStreamWaitEvent(st, p->ev_join, 0);
  mark(p, st, tail + 1);
  launch_k(&p->lc, cn_hr_attention_kernel<false>, dim3((N + 3) / 4), dim3(128), 0, st, p->sout, p->u, p->t1, 128, 64, p->bs, p->row_start, 0, 0,
                                                      N, H, p->wv, tcm ? p->tWv.hi : nullptr, tcm ? p->tWv.lo : nullptr, 256);
  // 3. GRU: emb overwrites the te half of t1 -> t1 = [enc | emb] = GRU input (gh came from the side stream)
  mark(p, st, tail + 2);
  if (tcm) {
    TcOut o; o.oh = p->tT1.hi + 64; o.ol = p->tT1.lo + 64; o.ldh = 128;
    gemm_tc(&p->lc, st, p->tWv, p->tWa, N, 64, 256, 64, p->ba, CN_ACT_RELU, o);
    gemm_tc(&p->lc, st, p->tT1, p->tWih, N, 384, 128, 64, p->bih, CN_ACT_NONE, out32(p->gi, 384));
  } else {
    gemm(p, st, p->wv, 256, p->Wa, 256, p->ba, p->t1 + 64, 128, N, 64, 256, CN_ACT_RELU);
    gemm(p, st, p->t1, 128, p->Wih, 128, p->bih, p->gi, 384, N, 384, 128, CN_ACT_NONE);
  }
  launch_k(&p->lc, cn_gru_gate_kernel, dim3((N * 128 + 255) / 256), dim3(256), 0, st, p->gi, p->gh, p->h0, N, d->h_out, tcm ? p->tH1.hi : nullptr,
                                                            tcm ? p->tH1.lo : nullptr);
  // 4. output_linear, actor / critic MLPs (critic.2 on the side stream), heads
  mark(p, st, tail + 3);
  if (tcm) {
    gemm_tc(&p->lc, st, p->tH1, p->tWoac, N, 512, 128, 64, p->boac, CN_ACT_TANH, out16(p->tAc1));     // [actor.0 | critic.0]
    cudaEventRecord(p->ev_fork2, st);
    cudaStreamWaitEvent(s2, p->ev_fork2, 0);
    gemm_tc(&p->lc, s2, p->tC1, p->tWc2, N, 256, 256, 64, p->bc2, CN_ACT_TANH, out32(p->c2, 256));
    cudaEventRecord(p->ev_join2, s2);
    gemm_tc(&p->lc, st, p->tA1, p->tWa2, N, 256, 256, 64, p->ba2, CN_ACT_TANH, out32(p->a2, 256));
  } else {
    gemm(p, st, d->h_out, 128, p->Woac, 128, p->boac, p->ac1, 512, N, 512, 128, CN_ACT_TANH);
    cudaEventRecord(p->ev_fork2, st);
    cudaStreamWaitEvent(s2, p->ev_fork2, 0);
    gemm(p, s2, p->ac1 + 256, 512, p->Wc2, 256, p->bc2, p->c2, 256, N, 256, 256, CN_ACT_TANH);
    cudaEventRecord(p->ev_join2, s2);
    gemm(p, st, p->ac1, 512, p->Wa2, 256, p->ba2, p->a2, 256, N, 256, 256, CN_ACT_TANH);
  }
  cudaStreamWaitEvent(st, p->ev_join2, 0);
  launch_k(&p->lc, cn_heads_kernel, dim3((N + 3) / 4), dim3(128), 0, st, p->a2, 256, p->c2, 256, p->wv_, p->bv, p->Wm, p->bm, p->logstd, d->noise, N,
                                               d->value, d->action, d->log_prob, d->action_mean);
  mark(p, st, p->num_stages);
  cudaError_t err = cudaGetLastError();
  if (p->lc.launch_error) { p->lc.launch_error = false; return 1; }      // cn_last_error names the stage
  if (err != cudaSuccess) return cn_set_error("cn_policy_act launch: %s", cudaGetErrorString(err));
  return 0;
}

int64_t cn_policy_launch_count(cn_policy* p) { return p ? p->lc.launches : 0; }

int64_t cn_policy_last_rows(cn_policy* p) {
  if (!p) return -1;
  cudaSetDevice(p->cfg.device);
  int v = 0;
  if (cudaDeviceSynchronize() != cudaSuccess || cudaMemcpy(&v, p->mc, sizeof(int), cudaMemcpyDeviceToHost) != cudaSuccess)
    return -1;
  return v;
}

// Internal test hook (not part of the public header): where one named workspace buffer of the policy forward lives,
// so a test can read every stage's input and output back after cn_policy_act.  *kind = 0: fp32 at *ptr; 1: fp16
// (hi, lo) pair at *ptr / *ptr_lo (value = hi + lo); 2: int32.  Row r of the buffer starts at element r * *ld.
//   row_start [N + 1], row_env [Mc], mc [1]: compacted row layout (rows of environment e: row_start[e] .. [e + 1])
//   row_slot [Mc] (visible_masks only): the slot of spatial_edges each compacted row holds
//   e1 [Mc,128], e2 [Mc,512], qkv [Mc,1536] (not in the fused kernel's mode), ao [Mc,512], sout [Mc,256]
//   rs [N,256], t1 [N,128], u [N,256], wv [N,256], h0 [N,128], gi / gh [N,384], h1 [N,128], ac1 [N,512],
//   a2 / c2 [N,256];  folded weights Wqkv [1536,512], bqkv, Wos [256,512], bos, Woac [512,128], boac.
// In gemm_mode 1 a name gives what the tensor-core consumer reads (the split pair where there is one);
// "t1.f32", "wv.f32" and "h0.f32" give the fp32 copies that are also written there.  Overwritten buffers:
//   t1: the GRU input [enc | emb].  The edge embedding (stage gru) overwrites the te half of [enc | te]; in
//       gemm_mode 1 only the split pair is overwritten and "t1.f32" keeps [enc | te].
//   h1: gemm_mode 1 only (gemm_mode 0 reads the caller's h_out).
// no_self_attn: "e1" is the output of spatial_linear.0 + ReLU and "sout" that of spatial_linear.2 + ReLU; e2, qkv, ao
// and the folded Wqkv / bqkv / Wos / bos do not exist.
int cn_internal_policy_buffer(cn_policy* p, const char* name, void** ptr, void** ptr_lo, int* rows, int* cols, int* ld,
                              int* kind) {
  if (!p || !name || !ptr || !ptr_lo || !rows || !cols || !ld || !kind)
    return cn_set_error("cn_internal_policy_buffer: null argument");
  const bool tcm = p->cfg.gemm_mode == 1;
  const int N = p->N, M = p->M;
  const std::string s(name);
  *ptr_lo = nullptr;
  auto f32 = [&](const float* q, int r, int c, int l) { *ptr = (void*)q; *rows = r; *cols = c; *ld = l; *kind = 0; return 0; };
  auto i32 = [&](const int* q, int r) { *ptr = (void*)q; *rows = r; *cols = 1; *ld = 1; *kind = 2; return 0; };
  auto f16 = [&](const TcMat& t, int r, int c) {
    *ptr = t.hi; *ptr_lo = t.lo; *rows = r; *cols = c; *ld = t.pitch; *kind = 1; return 0;
  };
  if (s == "row_start") return i32(p->row_start, N + 1);
  if (s == "row_env") return i32(p->row_env, M);
  if (s == "mc") return i32(p->mc, 1);
  if (s == "row_slot") {
    if (!p->vm) return cn_set_error("cn_internal_policy_buffer: 'row_slot' exists with visible_masks = 1 only");
    return i32(p->row_slot, M);
  }
  if (p->nsa && (s == "e2" || s == "qkv" || s == "ao" || s == "Wqkv" || s == "bqkv" || s == "Wos" || s == "bos"))
    return cn_set_error("cn_internal_policy_buffer: '%s' does not exist without human-human attention (no_self_attn)", name);
  if (s == "e1") return tcm ? f16(p->tE1, M, 128) : f32(p->e1, M, 128, 128);
  if (s == "e2") return tcm ? f16(p->tE2, M, 512) : f32(p->e2, M, 512, 512);
  if (s == "qkv") {
    if (p->fuse_qkv) return cn_set_error("cn_internal_policy_buffer: 'qkv' is never written by the fused QKV-attention kernel");
    return f32(p->qkv, M, 1536, 1536);
  }
  if (s == "ao") return tcm ? f16(p->tAo, M, 512) : f32(p->ao, M, 512, 512);
  if (s == "sout") return f32(p->sout, M, 256, 256);
  if (s == "rs") return tcm ? f16(p->tRs, N, 256) : f32(p->rs, N, 256, 256);
  if (s == "t1") return tcm ? f16(p->tT1, N, 128) : f32(p->t1, N, 128, 128);
  if (s == "u") return f32(p->u, N, 256, 256);
  if (s == "wv") return tcm ? f16(p->tWv, N, 256) : f32(p->wv, N, 256, 256);
  if (s == "h0") return tcm ? f16(p->tH0, N, 128) : f32(p->h0, N, 128, 128);
  if (s == "gi") return f32(p->gi, N, 384, 384);
  if (s == "gh") return f32(p->gh, N, 384, 384);
  if (s == "h1") {
    if (!tcm) return cn_set_error("cn_internal_policy_buffer: 'h1' exists in gemm_mode 1 only (gemm_mode 0 reads h_out)");
    return f16(p->tH1, N, 128);
  }
  if (s == "ac1") return tcm ? f16(p->tAc1, N, 512) : f32(p->ac1, N, 512, 512);
  if (s == "a2") return f32(p->a2, N, 256, 256);
  if (s == "c2") return f32(p->c2, N, 256, 256);
  if (tcm && s == "t1.f32") return f32(p->t1, N, 128, 128);
  if (tcm && s == "wv.f32") return f32(p->wv, N, 256, 256);
  if (tcm && s == "h0.f32") return f32(p->h0, N, 128, 128);
  if (!p->finalized && (s == "Wqkv" || s == "bqkv" || s == "Wos" || s == "bos" || s == "Woac" || s == "boac"))
    return cn_set_error("cn_internal_policy_buffer: '%s' needs cn_policy_finalize first", name);
  if (s == "Wqkv") return f32(p->Wqkv, 1536, 512, 512);
  if (s == "bqkv") return f32(p->bqkv, 1536, 1, 1);
  if (s == "Wos") return f32(p->Wos, 256, 512, 512);
  if (s == "bos") return f32(p->bos, 256, 1, 1);
  if (s == "Woac") return f32(p->Woac, 512, 128, 128);
  if (s == "boac") return f32(p->boac, 512, 1, 1);
  return cn_set_error("cn_internal_policy_buffer: unknown buffer '%s' (gemm_mode %d)", name, p->cfg.gemm_mode);
}

}  // extern "C"
