// DS-RNN policy forward (the reference's base = 'srnn', rl/networks/srnn_model.py:326-468) for one rollout step
// (infer = True): parameter upload / folding and the launch sequence behind cn_dsrnn_act.
//
// Folds done once per parameter upload (fp64 accumulate):
//   humanNodeRNN.encoder_linear o robot_linear          -> one 7 -> 64 layer (no activation between the two)
//   [actor.0 ; critic.0] o humanNodeRNN.output_linear    -> one 128 -> 512 layer (as cn_policy's Woac)
//   attn.spatial_edge_layer into the temporal side of the attention: u = W_s^T te, cst = <b_s, te>
//
// The two edge GRUs (temporal: one row per environment; spatial: one row per (environment, human slot), all H slots)
// are each ONE wgmma 3xFP16 GEMM with the GRU cell in the epilogue (gemm_tc_gru, cn_gemm_tc.cuh tc_epilogue_gru).  Their
// A operand [x_emb (64) | m h (256)] is written by cn_dsrnn_edge_pack_kernel, which also runs the K = W <= 12 edge
// encoder on the CUDA cores; the new edge state goes straight into the caller's edge_h_out.  The per-environment tail
// (robot-human attention, node GRU, actor / critic heads) launches the attention-graph policy's kernels, defined once
// in cn_policy.cu.  Tensor-core path only.
#include <cuda_runtime.h>
#include <stdio.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

#include "../../include/crowdnav_b200.h"
#include "cn_gemm_tc.h"
#include "cn_host_util.h"
#include "cn_launch.cuh"

// Shared with the attention-graph policy; defined in cn_policy.cu (cn_policy_kernels.cuh).  The robot-human attention
// (cn_hr_attention_kernel<true>, dense rows, no mask) is launched through cn_policy.cu.
void cn_hr_attention_dense(CnLaunchCtx* c, cudaStream_t st, const float* s_out, const float* u, const float* te, int ldte,
                           int te_off, const float* b_s, int env_pitch, int env_off, int N, int H, float* wv,
                           __half* wv_hi, __half* wv_lo, int ldwh);
__global__ void cn_gru_gate_kernel(const float* __restrict__ gi, const float* __restrict__ gh,
                                   const float* __restrict__ h0, int N, float* __restrict__ h1,
                                   __half* __restrict__ h1_hi, __half* __restrict__ h1_lo);
__global__ void cn_heads_kernel(const float* __restrict__ ha, int ldha, const float* __restrict__ hc, int ldhc,
                                const float* __restrict__ w_v, const float* __restrict__ b_v,
                                const float* __restrict__ w_m, const float* __restrict__ b_m,
                                const float* __restrict__ logstd, const float* __restrict__ noise, int N,
                                float* __restrict__ value, float* __restrict__ action, float* __restrict__ logp,
                                float* __restrict__ mean_out);

namespace {
constexpr int kEdge = 256;      // human_human_edge_rnn_size
constexpr int kEmb = 64;        // human_human_edge_embedding_size
constexpr int kK = kEmb + kEdge;  // K of the edge-GRU GEMM
constexpr int kNode = 128;      // human_node_rnn_size
}  // namespace

// A operand of one edge GRU: row r (environment r / group, slot r % group) =
//   [ReLU(W_enc x_r + b_enc) (64) | mask[env] * h_in[env * pitch + off + slot] (256)] as a split fp16 pair [rows, 320].
// One thread per column pair.  h_in null: zero state.
__global__ void __launch_bounds__(256) cn_dsrnn_edge_pack_kernel(const float* __restrict__ x, int W, int rows, int group,
                                                                 int pitch, int off, const float* __restrict__ h_in,
                                                                 const float* __restrict__ masks,
                                                                 const float* __restrict__ w_enc /* [64, W] */,
                                                                 const float* __restrict__ b_enc,
                                                                 __half* __restrict__ a_hi, __half* __restrict__ a_lo) {
  cn_pdl_prologue();
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)rows * (kK / 2)) return;
  const int r = (int)(idx / (kK / 2)), c = 2 * (int)(idx % (kK / 2));
  const int env = r / group;
  float v0, v1;
  if (c < kEmb) {
    const float* xr = x + (size_t)r * W;
    float s0 = __ldg(b_enc + c), s1 = __ldg(b_enc + c + 1);
    for (int k = 0; k < W; ++k) {
      const float xk = __ldg(xr + k);
      s0 = fmaf(__ldg(w_enc + c * W + k), xk, s0);
      s1 = fmaf(__ldg(w_enc + (c + 1) * W + k), xk, s1);
    }
    v0 = fmaxf(s0, 0.0f); v1 = fmaxf(s1, 0.0f);
  } else if (h_in) {
    const size_t hrow = (size_t)env * pitch + off + (r - env * group);
    const float2 h = __ldg(reinterpret_cast<const float2*>(h_in + hrow * kEdge + (c - kEmb)));
    const float m = __ldg(masks + env);
    v0 = h.x * m; v1 = h.y * m;
  } else {
    v0 = 0.0f; v1 = 0.0f;
  }
  uint32_t lo;
  const uint32_t hi = tc::split_pair_hi(v0, v1, &lo);
  const size_t o = (size_t)r * kK + c;
  *reinterpret_cast<uint32_t*>(a_hi + o) = hi;
  *reinterpret_cast<uint32_t*>(a_lo + o) = lo;
}

// Node side inputs, one thread per (environment, unit < 128): enc = ReLU(W_rob robot_node + b_rob) into columns 0..63 of
// the node GRU's input t1 (split fp16, pitch 128); h0 = h_in * mask (fp32 and split fp16).
__global__ void __launch_bounds__(256) cn_dsrnn_node_in_kernel(const float* __restrict__ robot, const float* __restrict__ h_in,
                                                               const float* __restrict__ masks,
                                                               const float* __restrict__ w_rob /* [64, 7] */,
                                                               const float* __restrict__ b_rob, int N,
                                                               __half* __restrict__ t1_hi, __half* __restrict__ t1_lo,
                                                               float* __restrict__ h0, __half* __restrict__ h0_hi,
                                                               __half* __restrict__ h0_lo) {
  cn_pdl_prologue();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * kNode) return;
  const int e = idx / kNode, c = idx % kNode;
  const float hv = h_in[idx] * masks[e];
  h0[idx] = hv;
  const float hc = fminf(fmaxf(hv, -65504.0f), 65504.0f);
  const __half hh = __float2half_rn(hc);
  h0_hi[idx] = hh;
  h0_lo[idx] = __float2half_rn(hc - __half2float(hh));
  if (c < 64) {
    float s = b_rob[c];
#pragma unroll
    for (int k = 0; k < 7; ++k) s = fmaf(w_rob[c * 7 + k], robot[(size_t)e * 7 + k], s);
    s = fminf(fmaxf(s, 0.0f), 65504.0f);
    const __half eh = __float2half_rn(s);
    t1_hi[(size_t)e * 128 + c] = eh;
    t1_lo[(size_t)e * 128 + c] = __float2half_rn(s - __half2float(eh));
  }
}

struct cn_dsrnn {
  cn_dsrnn_config cfg;
  int N, H, W;
  CnLaunchCtx lc;
  bool finalized = false;
  std::map<std::string, std::vector<float>> host;
  size_t ws_allocs = 0;
  // parameters (device): encoders, interleaved GRU biases, per-environment layers
  float *We_s, *be_s, *We_t, *be_t, *bg_s, *bg_t, *Wrob, *brob;
  float *bt, *bs, *ba, *bih, *bhh, *boac, *ba2, *bc2, *wv_, *bv, *Wm, *bm, *logstd;
  TcMat tBs, tBt;                                   // interleaved edge-GRU weights [1024, 320]
  TcMat tWt, tWsT, tWa, tWih, tWhh, tWoac, tWa2, tWc2;
  // workspace
  TcMat tAs, tAt;                                   // edge-GRU A operands: [N H, 320], [N, 320]
  TcMat tHW, tHt;                                   // [h_t' | wv] [N, 512]; tHt = its columns 0..255
  TcMat tTe, tT1, tH0, tH1, tAc1, tA1, tC1;
  float *te, *u, *wv, *h0, *gi, *gh, *a2, *c2;
  cudaStream_t st2 = nullptr;
  cudaEvent_t ev_fork, ev_join, ev_fork2, ev_join2;
  bool profile = false;
  std::vector<cudaEvent_t> ev;
};

namespace {

const char* kStageNames[] = {"spatial_edge_pack", "spatial_edge_gru", "temporal_robot_join", "edge_attention",
                             "node_gru", "actor_critic_heads"};
const int kNumStages = sizeof(kStageNames) / sizeof(kStageNames[0]);

inline void mark(cn_dsrnn* p, cudaStream_t st, int i) {
  p->lc.cur_stage = i < kNumStages ? kStageNames[i] : "end";
  if (p->profile) cudaEventRecord(p->ev[i], st);
}

int upload(cn_dsrnn* p, float** dst, const std::vector<float>& src) {
  int rc = palloc(&p->lc, dst, src.size());
  if (rc) return rc;
  cudaError_t err = cudaMemcpy(*dst, src.data(), src.size() * sizeof(float), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) return cn_set_error("H2D param: %s", cudaGetErrorString(err));
  return 0;
}

const std::vector<float>* get(cn_dsrnn* p, const char* key, size_t count) {
  auto it = p->host.find(key);
  if (it == p->host.end()) { cn_set_error("cn_dsrnn_finalize: parameter '%s' was not set", key); return nullptr; }
  if (it->second.size() != count) {
    cn_set_error("cn_dsrnn_finalize: parameter '%s' has %zu elements, expected %zu", key, it->second.size(), count);
    return nullptr;
  }
  return &it->second;
}

// C[m, n] = sum_k A[m, k] B[k, n] (+ d[m] for the bias form), fp64 accumulate
std::vector<float> fold_mm(const std::vector<float>& A, const std::vector<float>& B, int M, int K, int N) {
  std::vector<float> C((size_t)M * N);
  for (int m = 0; m < M; ++m)
    for (int n = 0; n < N; ++n) {
      double s = 0.0;
      for (int k = 0; k < K; ++k) s += (double)A[(size_t)m * K + k] * (double)B[(size_t)k * N + n];
      C[(size_t)m * N + n] = (float)s;
    }
  return C;
}
std::vector<float> fold_mv(const std::vector<float>& A, const std::vector<float>& b, const std::vector<float>& d, int M, int K) {
  std::vector<float> c(M);
  for (int m = 0; m < M; ++m) {
    double s = d[m];
    for (int k = 0; k < K; ++k) s += (double)A[(size_t)m * K + k] * (double)b[k];
    c[m] = (float)s;
  }
  return c;
}

// B operand and bias of the edge-GRU GEMM: column tile t (256 columns) holds, for hidden units 64 t .. 64 t + 63,
//   r: [W_ir | W_hr], b_ir + b_hr;  z: [W_iz | W_hz], b_iz + b_hz;  gi_n: [W_in | 0], b_in;  gh_n: [0 | W_hn], b_hn.
void interleave_gru(const std::vector<float>& wih /* [768, 64] */, const std::vector<float>& whh /* [768, 256] */,
                    const std::vector<float>& bih, const std::vector<float>& bhh, std::vector<float>& B,
                    std::vector<float>& bias) {
  B.assign((size_t)1024 * kK, 0.0f);
  bias.assign(1024, 0.0f);
  for (int col = 0; col < 1024; ++col) {
    const int t = col / 256, q = (col % 256) / 64, u = 64 * t + col % 64;
    float* row = &B[(size_t)col * kK];
    const int g = q < 2 ? q : 2;                    // PyTorch gate block: r 0, z 1, n 2
    const size_t src = (size_t)(g * kEdge + u);
    if (q != 3) for (int k = 0; k < kEmb; ++k) row[k] = wih[src * kEmb + k];
    if (q != 2) for (int k = 0; k < kEdge; ++k) row[kEmb + k] = whh[src * kEdge + k];
    bias[col] = (q == 3 ? 0.0f : bih[src]) + (q == 2 ? 0.0f : bhh[src]);
  }
}

}  // namespace

extern "C" {

int cn_dsrnn_create(const cn_dsrnn_config* cfg, cn_dsrnn** out) {
  if (!cfg || !out) return cn_set_error("cn_dsrnn_create: null argument");
  *out = nullptr;
  if (cfg->num_envs <= 0 || cfg->human_num <= 0 || cfg->human_num > 128 || cfg->input_size <= 0 || cfg->input_size > 16)
    return cn_set_error("cn_dsrnn_create: unsupported dims N=%d H=%d input=%d", cfg->num_envs, cfg->human_num,
                        cfg->input_size);
  int ndev = 0;
  cudaError_t err = cudaGetDeviceCount(&ndev);
  if (err != cudaSuccess || ndev == 0)
    return cn_set_error("cn_dsrnn_create: no CUDA device (%s); this engine has no CPU fallback",
                        err == cudaSuccess ? "device count 0" : cudaGetErrorString(err));
  if (cfg->device < 0 || cfg->device >= ndev) return cn_set_error("cn_dsrnn_create: bad device %d", cfg->device);
  cudaSetDevice(cfg->device);
  cn_dsrnn* p = new cn_dsrnn();
  p->cfg = *cfg;
  p->N = cfg->num_envs; p->H = cfg->human_num; p->W = cfg->input_size;
  cn_launch_init(&p->lc, cfg->device);
  cudaStreamCreateWithFlags(&p->st2, cudaStreamNonBlocking);
  cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_join, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_fork2, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&p->ev_join2, cudaEventDisableTiming);
  const int N = p->N, MS = p->N * p->H;
  const size_t Nz = (size_t)N;
  int rc = 0;
  if (!rc) rc = palloc(&p->lc, &p->te, Nz * 64);
  if (!rc) rc = palloc(&p->lc, &p->u, Nz * 256);
  if (!rc) rc = palloc(&p->lc, &p->wv, Nz * 256);
  if (!rc) rc = palloc(&p->lc, &p->h0, Nz * 128);
  if (!rc) rc = palloc(&p->lc, &p->gi, Nz * 384);
  if (!rc) rc = palloc(&p->lc, &p->gh, Nz * 384);
  if (!rc) rc = palloc(&p->lc, &p->a2, Nz * 256);
  if (!rc) rc = palloc(&p->lc, &p->c2, Nz * 256);
  const int k256 = tc_box_k(256), k64 = tc_box_k(64);
  if (!rc) rc = tc_alloc(&p->lc, p->tAs, MS, kK, TC_BM, k256);
  if (!rc) rc = tc_alloc(&p->lc, p->tAt, N, kK, TC_BM, k256);
  if (!rc) rc = tc_alloc(&p->lc, p->tHW, N, 512, TC_BM, k64);
  if (!rc) rc = tc_view(p->tHt, p->tHW, 0, N, 256, TC_BM);
  if (!rc) rc = tc_alloc(&p->lc, p->tTe, N, 64, TC_BM, k64);
  if (!rc) rc = tc_alloc(&p->lc, p->tT1, N, 128, TC_BM, k64);
  if (!rc) rc = tc_alloc(&p->lc, p->tH0, N, 128, TC_BM, k64);
  if (!rc) rc = tc_alloc(&p->lc, p->tH1, N, 128, TC_BM, k64);
  if (!rc) rc = tc_alloc(&p->lc, p->tAc1, N, 512, TC_BM, k64);
  if (!rc) rc = tc_view(p->tA1, p->tAc1, 0, N, 256, TC_BM);
  if (!rc) rc = tc_view(p->tC1, p->tAc1, 256, N, 256, TC_BM);
  if (!rc) rc = tc_set_attrs();
  if (rc) { cn_dsrnn_destroy(p); return rc; }
  p->ws_allocs = p->lc.allocs.size();
  *out = p;
  return 0;
}

int cn_dsrnn_destroy(cn_dsrnn* p) {
  if (!p) return 0;
  cudaSetDevice(p->cfg.device);
  cn_launch_free(&p->lc);
  for (auto& e : p->ev) cudaEventDestroy(e);
  if (p->st2) {
    cudaStreamDestroy(p->st2);
    cudaEventDestroy(p->ev_fork); cudaEventDestroy(p->ev_join); cudaEventDestroy(p->ev_fork2); cudaEventDestroy(p->ev_join2);
  }
  delete p;
  return 0;
}

int cn_dsrnn_set_param(cn_dsrnn* p, const char* key, const float* h_data, size_t count) {
  if (!p || !key || !h_data) return cn_set_error("cn_dsrnn_set_param: null argument");
  p->host[key] = std::vector<float>(h_data, h_data + count);
  p->finalized = false;
  return 0;
}

int cn_dsrnn_finalize(cn_dsrnn* p, void* stream) {
  if (!p) return cn_set_error("cn_dsrnn_finalize: null argument");
  cudaSetDevice(p->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  const int W = p->W;
#define GET(var, key, count) const std::vector<float>* var = get(p, key, (count)); if (!var) return 1
  GET(s_wih, "base.humanhumanEdgeRNN_spatial.gru.weight_ih_l0", (size_t)768 * 64);
  GET(s_whh, "base.humanhumanEdgeRNN_spatial.gru.weight_hh_l0", (size_t)768 * 256);
  GET(s_bih, "base.humanhumanEdgeRNN_spatial.gru.bias_ih_l0", 768);
  GET(s_bhh, "base.humanhumanEdgeRNN_spatial.gru.bias_hh_l0", 768);
  GET(s_we, "base.humanhumanEdgeRNN_spatial.encoder_linear.weight", (size_t)64 * W);
  GET(s_be, "base.humanhumanEdgeRNN_spatial.encoder_linear.bias", 64);
  GET(t_wih, "base.humanhumanEdgeRNN_temporal.gru.weight_ih_l0", (size_t)768 * 64);
  GET(t_whh, "base.humanhumanEdgeRNN_temporal.gru.weight_hh_l0", (size_t)768 * 256);
  GET(t_bih, "base.humanhumanEdgeRNN_temporal.gru.bias_ih_l0", 768);
  GET(t_bhh, "base.humanhumanEdgeRNN_temporal.gru.bias_hh_l0", 768);
  GET(t_we, "base.humanhumanEdgeRNN_temporal.encoder_linear.weight", (size_t)64 * 2);
  GET(t_be, "base.humanhumanEdgeRNN_temporal.encoder_linear.bias", 64);
  GET(wt, "base.attn.temporal_edge_layer.0.weight", (size_t)64 * 256);
  GET(bt, "base.attn.temporal_edge_layer.0.bias", 64);
  GET(ws, "base.attn.spatial_edge_layer.0.weight", (size_t)64 * 256);
  GET(bs, "base.attn.spatial_edge_layer.0.bias", 64);
  GET(wr, "base.robot_linear.weight", (size_t)3 * 7);
  GET(br, "base.robot_linear.bias", 3);
  GET(we, "base.humanNodeRNN.encoder_linear.weight", (size_t)64 * 3);
  GET(be, "base.humanNodeRNN.encoder_linear.bias", 64);
  GET(wa, "base.humanNodeRNN.edge_attention_embed.weight", (size_t)64 * 512);
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
  cudaStreamSynchronize(st);
  for (size_t i = p->ws_allocs; i < p->lc.allocs.size(); ++i) cudaFree(p->lc.allocs[i]);
  p->lc.allocs.resize(p->ws_allocs);
  auto cat = [](const std::vector<float>& a, const std::vector<float>& b) {
    std::vector<float> o(a); o.insert(o.end(), b.begin(), b.end()); return o;
  };
  // folds (fp64): encoder_linear o robot_linear; [actor.0 ; critic.0] o output_linear
  const std::vector<float> wrob = fold_mm(*we, *wr, 64, 3, 7), brob = fold_mv(*we, *br, *be, 64, 3);
  const std::vector<float> wac0 = cat(*wa0, *wc0), bac0 = cat(*ba0, *bc0);
  const std::vector<float> woac = fold_mm(wac0, *wo, 512, 256, 128), boac = fold_mv(wac0, *bo, bac0, 512, 256);
  std::vector<float> wst((size_t)256 * 64);                  // W_s^T: [256][64]
  for (int r = 0; r < 64; ++r) for (int c = 0; c < 256; ++c) wst[(size_t)c * 64 + r] = (*ws)[(size_t)r * 256 + c];
  std::vector<float> Bs, bgs, Bt, bgt;
  interleave_gru(*s_wih, *s_whh, *s_bih, *s_bhh, Bs, bgs);
  interleave_gru(*t_wih, *t_whh, *t_bih, *t_bhh, Bt, bgt);
  int rc = 0;
#define UP(dst, vec) if (!rc) rc = upload(p, &p->dst, (vec))
  UP(We_s, *s_we); UP(be_s, *s_be); UP(We_t, *t_we); UP(be_t, *t_be); UP(bg_s, bgs); UP(bg_t, bgt);
  UP(Wrob, wrob); UP(brob, brob);
  UP(bt, *bt); UP(bs, *bs); UP(ba, *ba); UP(bih, *bih); UP(bhh, *bhh); UP(boac, boac); UP(ba2, *ba2); UP(bc2, *bc2);
  UP(wv_, *wcl); UP(bv, *bcl); UP(Wm, *wm); UP(bm, *bm); UP(logstd, *ls);
#undef UP
  if (rc) return rc;
  // fp16 (hi, lo) split of the tensor-core weights, pre-scaled by 2^6 (exact) so lo stays normal
  struct { const std::vector<float>* src; TcMat* t; int rows, k, bn; } tw[10] = {
      {&Bs, &p->tBs, 1024, kK, 256},  {&Bt, &p->tBt, 1024, kK, 256}, {wt, &p->tWt, 64, 256, 64},
      {&wst, &p->tWsT, 256, 64, 64},  {wa, &p->tWa, 64, 512, 64},    {wih, &p->tWih, 384, 128, 64},
      {whh, &p->tWhh, 384, 128, 64},  {&woac, &p->tWoac, 512, 128, 64}, {wa2, &p->tWa2, 256, 256, 64},
      {wc2, &p->tWc2, 256, 256, 64}};
  for (auto& t : tw) {
    float* d = nullptr;
    rc = upload(p, &d, *t.src);
    if (!rc) rc = tc_alloc(&p->lc, *t.t, t.rows, t.k, t.bn, tc_box_k(t.bn));
    if (rc) return rc;
    split16(&p->lc, st, d, 64.0f, t.t->hi, t.t->lo, (size_t)t.rows * t.k);
  }
  cudaError_t err = cudaStreamSynchronize(st);
  if (err != cudaSuccess) return cn_set_error("cn_dsrnn_finalize: %s", cudaGetErrorString(err));
  p->finalized = true;
  return 0;
}

int cn_dsrnn_act(cn_dsrnn* p, const cn_dsrnn_act_ptrs* d, void* stream) {
  if (!p || !d) return cn_set_error("cn_dsrnn_act: null argument");
  if (!p->finalized) return cn_set_error("cn_dsrnn_act: call cn_dsrnn_finalize after setting parameters");
  if (!d->robot_node || !d->temporal_edges || !d->spatial_edges || !d->h_in || !d->masks || !d->value || !d->action ||
      !d->log_prob || !d->h_out || !d->edge_h_out)
    return cn_set_error("cn_dsrnn_act: missing input/output pointer");
  CnDeviceGuard guard(p->cfg.device);
  cudaStream_t st = (cudaStream_t)stream;
  const int N = p->N, H = p->H, MS = N * H;
  float* eh = d->edge_h_out;
  const float* eh_in = d->edge_h_in;
  // fork: temporal edge GRU, te / u, the robot side and gh only depend on the inputs
  mark(p, st, 0);
  cudaStream_t s2 = p->st2;
  cudaEventRecord(p->ev_fork, st);
  cudaStreamWaitEvent(s2, p->ev_fork, 0);
  launch_k(&p->lc, cn_dsrnn_edge_pack_kernel, dim3((N * (kK / 2) + 255) / 256), dim3(256), 0, s2, d->temporal_edges, 2, N,
           1, H + 1, 0, eh_in, d->masks, p->We_t, p->be_t, p->tAt.hi, p->tAt.lo);
  gemm_tc_gru(&p->lc, s2, p->tAt, p->tBt, N, p->bg_t, eh_in, d->masks, eh, 1, H + 1, 0, p->tHW.hi, p->tHW.lo, 512);
  gemm_tc(&p->lc, s2, p->tHt, p->tWt, N, 64, 256, 64, p->bt, CN_ACT_NONE, out_both(p->te, 64, p->tTe));
  gemm_tc(&p->lc, s2, p->tTe, p->tWsT, N, 256, 64, 64, nullptr, CN_ACT_NONE, out32(p->u, 256));
  launch_k(&p->lc, cn_dsrnn_node_in_kernel, dim3((N * kNode + 255) / 256), dim3(256), 0, s2, d->robot_node, d->h_in,
           d->masks, p->Wrob, p->brob, N, p->tT1.hi, p->tT1.lo, p->h0, p->tH0.hi, p->tH0.lo);
  gemm_tc(&p->lc, s2, p->tH0, p->tWhh, N, 384, 128, 64, p->bhh, CN_ACT_NONE, out32(p->gh, 384));
  cudaEventRecord(p->ev_join, s2);
  // spatial edge GRU over all N H slots, straight into rows 1..H of every environment's edge state
  launch_k(&p->lc, cn_dsrnn_edge_pack_kernel, dim3((unsigned)(((size_t)MS * (kK / 2) + 255) / 256)), dim3(256), 0, st,
           d->spatial_edges, p->W, MS, H, H + 1, 1, eh_in, d->masks, p->We_s, p->be_s, p->tAs.hi, p->tAs.lo);
  mark(p, st, 1);
  gemm_tc_gru(&p->lc, st, p->tAs, p->tBs, MS, p->bg_s, eh_in, d->masks, eh, H, H + 1, 1, nullptr, nullptr, 0);
  mark(p, st, 2);
  cudaStreamWaitEvent(st, p->ev_join, 0);
  // edge attention over the H spatial states (no mask); wv goes to columns 256..511 of [h_t' | wv]
  mark(p, st, 3);
  cn_hr_attention_dense(&p->lc, st, eh, p->u, p->te, 64, 0, p->bs, H + 1, 1, N, H, p->wv, p->tHW.hi + 256, p->tHW.lo + 256,
                        512);
  // node GRU: emb = ReLU(edge_attention_embed([h_t' | wv])) into columns 64..127 of t1 = [enc | emb]
  mark(p, st, 4);
  {
    TcOut o; o.oh = p->tT1.hi + 64; o.ol = p->tT1.lo + 64; o.ldh = 128;
    gemm_tc(&p->lc, st, p->tHW, p->tWa, N, 64, 512, 64, p->ba, CN_ACT_RELU, o);
  }
  gemm_tc(&p->lc, st, p->tT1, p->tWih, N, 384, 128, 64, p->bih, CN_ACT_NONE, out32(p->gi, 384));
  launch_k(&p->lc, cn_gru_gate_kernel, dim3((N * 128 + 255) / 256), dim3(256), 0, st, (const float*)p->gi,
           (const float*)p->gh, (const float*)p->h0, N, d->h_out, p->tH1.hi, p->tH1.lo);
  // output_linear folded into [actor.0 | critic.0], actor / critic MLPs (critic.2 on the side stream), heads
  mark(p, st, 5);
  gemm_tc(&p->lc, st, p->tH1, p->tWoac, N, 512, 128, 64, p->boac, CN_ACT_TANH, out16(p->tAc1));
  cudaEventRecord(p->ev_fork2, st);
  cudaStreamWaitEvent(s2, p->ev_fork2, 0);
  gemm_tc(&p->lc, s2, p->tC1, p->tWc2, N, 256, 256, 64, p->bc2, CN_ACT_TANH, out32(p->c2, 256));
  cudaEventRecord(p->ev_join2, s2);
  gemm_tc(&p->lc, st, p->tA1, p->tWa2, N, 256, 256, 64, p->ba2, CN_ACT_TANH, out32(p->a2, 256));
  cudaStreamWaitEvent(st, p->ev_join2, 0);
  launch_k(&p->lc, cn_heads_kernel, dim3((N + 3) / 4), dim3(128), 0, st, (const float*)p->a2, 256, (const float*)p->c2,
           256, (const float*)p->wv_, (const float*)p->bv, (const float*)p->Wm, (const float*)p->bm,
           (const float*)p->logstd, d->noise, N, d->value, d->action, d->log_prob, d->action_mean);
  mark(p, st, kNumStages);
  cudaError_t err = cudaGetLastError();
  if (p->lc.launch_error) { p->lc.launch_error = false; return 1; }
  if (err != cudaSuccess) return cn_set_error("cn_dsrnn_act launch: %s", cudaGetErrorString(err));
  return 0;
}

int cn_dsrnn_profile(cn_dsrnn* p, int enable) {
  if (!p) return cn_set_error("cn_dsrnn_profile: null argument");
  cudaSetDevice(p->cfg.device);
  if (enable && p->ev.empty()) {
    p->ev.resize(kNumStages + 1);
    for (auto& e : p->ev) cudaEventCreate(&e);
  }
  p->profile = enable != 0;
  return 0;
}
int cn_dsrnn_stage_count(void) { return kNumStages; }
const char* cn_dsrnn_stage_name(int i) { return (i >= 0 && i < kNumStages) ? kStageNames[i] : ""; }
int cn_dsrnn_stage_ms(cn_dsrnn* p, float* out, int n) {
  if (!p || !out) return cn_set_error("cn_dsrnn_stage_ms: null argument");
  if (p->ev.empty()) return cn_set_error("cn_dsrnn_stage_ms: profiling was never enabled");
  cudaSetDevice(p->cfg.device);
  cudaError_t err = cudaEventSynchronize(p->ev[kNumStages]);
  if (err != cudaSuccess) return cn_set_error("cn_dsrnn_stage_ms: %s", cudaGetErrorString(err));
  for (int i = 0; i < n && i < kNumStages; ++i) cudaEventElapsedTime(&out[i], p->ev[i], p->ev[i + 1]);
  return 0;
}

int64_t cn_dsrnn_launch_count(cn_dsrnn* p) { return p ? p->lc.launches : 0; }

// Internal test hook (not part of the public header): where a workspace buffer of the forward lives, so a test can read
// every stage's input and output back after cn_dsrnn_act.  *kind = 0: fp32 at *ptr; 1: fp16 (hi, lo) pair at *ptr /
// *ptr_lo (value = hi + lo); 2: int32 (none here).  Row r of the buffer starts at element r * *ld.
//   As [N H, 320], At [N, 320]  split A operands of the spatial / temporal edge GRUs: [x_emb | m h]
//   HW [N, 512]                 split [h_t' | wv] (h_t' from the temporal GRU's epilogue, wv from the attention)
//   te [N, 64], Te [N, 64]      temporal_edge_layer(h_t'), fp32 and split
//   u, wv [N, 256]              W_s^T te and the attention's fp32 output
//   T1 [N, 128]                 split node-GRU input [enc | emb]
//   h0 [N, 128], H0 [N, 128]    h_in * mask, fp32 and split
//   gi, gh [N, 384]             node-GRU pre-activations
//   H1 [N, 128]                 split h_out
//   Ac1 [N, 512], a2, c2 [N, 256]  tanh([actor.0 | critic.0] o output_linear), actor.2, critic.2
int cn_internal_dsrnn_buffer(cn_dsrnn* p, const char* name, void** ptr, void** ptr_lo, int* rows, int* cols, int* ld,
                             int* kind) {
  if (!p || !name || !ptr || !ptr_lo || !rows || !cols || !ld || !kind)
    return cn_set_error("cn_internal_dsrnn_buffer: null argument");
  const int N = p->N;
  const std::string s(name);
  *ptr_lo = nullptr;
  auto f32 = [&](const float* q, int r, int c) { *ptr = (void*)q; *rows = r; *cols = c; *ld = c; *kind = 0; return 0; };
  auto f16 = [&](const TcMat& t, int r, int c) {
    *ptr = t.hi; *ptr_lo = t.lo; *rows = r; *cols = c; *ld = t.pitch; *kind = 1; return 0;
  };
  if (s == "As") return f16(p->tAs, N * p->H, kK);
  if (s == "At") return f16(p->tAt, N, kK);
  if (s == "HW") return f16(p->tHW, N, 512);
  if (s == "te") return f32(p->te, N, 64);
  if (s == "Te") return f16(p->tTe, N, 64);
  if (s == "u") return f32(p->u, N, 256);
  if (s == "wv") return f32(p->wv, N, 256);
  if (s == "T1") return f16(p->tT1, N, 128);
  if (s == "h0") return f32(p->h0, N, 128);
  if (s == "H0") return f16(p->tH0, N, 128);
  if (s == "gi") return f32(p->gi, N, 384);
  if (s == "gh") return f32(p->gh, N, 384);
  if (s == "H1") return f16(p->tH1, N, 128);
  if (s == "Ac1") return f16(p->tAc1, N, 512);
  if (s == "a2") return f32(p->a2, N, 256);
  if (s == "c2") return f32(p->c2, N, 256);
  return cn_set_error("cn_internal_dsrnn_buffer: unknown buffer '%s'", name);
}

}  // extern "C"
