// BASELINE config 3 (SURVEY.md row a16): the GST trajectory predictor and the VecPretextNormalize processing,
// fused into ONE kernel launch per rollout step.
//
//   reference: rl/vec_env/vec_pretext_normalize.py:85-191 (traj / mask deques, process_obs_rew),
//              gst_updated/scripts/wrapper/crowd_nav_interface_parallel.py:45-114 (input masks, cumsum of mu),
//              gst_updated/src/gumbel_social_transformer/st_model.py:271-455 + node_encoder_layer_no_ghost.py +
//              mha.py:236-242 for the shipped predictor configuration (full connectivity, one 8-head layer,
//              'faster_lstm', recursive decoding, sampling=False).
//
// One CTA per environment: the five observed frames are stacked as 5*H rows so every weight matrix of the encoder
// layer is read once for them, the LSTM runs its five steps on the H nodes, four more encoder + LSTM steps decode
// the future, and the CTA finishes the wrapper's work: future-collision penalty added to the reward, predicted
// relative positions written into the 2(P+1)-wide spatial_edges rows, rows sorted by distance to the robot.
// All activations live in shared memory; weights are stored transposed ([K][N]) so the register-tiled dense
// layers read them coalesced (they stay L2 resident: 269 KB).  fp32 CUDA cores: this first version favours
// parity (<= 2e-5 on the predicted positions).  The default path since is cn_gst_tc.cu (batched wgmma GEMMs over
// all environments + row-wise kernels); this fused kernel stays as CN_GST_MODE=fused (one launch, no workspace).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

#include "../../include/crowdnav_b200.h"
#include "cn_host_util.h"

namespace {

#define GST_D 64
#define GST_T 5          // observed frames = predicted steps
#define GST_THREADS 1024
#define GST_INVALID (-999.0f)

struct GstW {
  const float *We_t, *be, *ln0_g, *ln0_b, *Win_t, *bin, *Wout_t, *bout, *ln1_g, *ln1_b;
  const float *W1_t, *b1, *W2_t, *b2, *Wih_t, *bih, *Whh_t, *bhh, *Wp, *bp;
};

// out[r][c] = act(res[r][c] + bias[c] + sum_k in[r][k] * Wt[k][c]); RT x 4 register tiles, column tiles fastest
// across the threads (coalesced float4 weight loads, broadcast activation loads).  R % RT == 0, Nout % 4 == 0.
template <int RT>
__device__ void gst_dense_t(const float* __restrict__ in, int ldi, const float* __restrict__ Wt, const float* __restrict__ bias,
                            const float* res, int ldr, float* out, int ldo, int R, int K, int Nout, bool relu) {
  const int ct = Nout >> 2, rt = R / RT;
  for (int tile = threadIdx.x; tile < ct * rt; tile += blockDim.x) {
    const int c0 = (tile % ct) << 2, r0 = (tile / ct) * RT;
    float acc[RT][4];
    const float4 b = *reinterpret_cast<const float4*>(bias + c0);
#pragma unroll
    for (int i = 0; i < RT; ++i) { acc[i][0] = b.x; acc[i][1] = b.y; acc[i][2] = b.z; acc[i][3] = b.w; }
    const float* ip = in + (size_t)r0 * ldi;
    for (int k = 0; k < K; k += 4) {                       // K % 4 == 0; activations fetched as LDS.128 over k
      float4 wv[4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wv[kk] = __ldg(reinterpret_cast<const float4*>(Wt + (size_t)(k + kk) * Nout + c0));
#pragma unroll
      for (int i = 0; i < RT; ++i) {
        const float4 a4 = *reinterpret_cast<const float4*>(ip + i * ldi + k);
        const float a[4] = {a4.x, a4.y, a4.z, a4.w};
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          acc[i][0] = fmaf(a[kk], wv[kk].x, acc[i][0]); acc[i][1] = fmaf(a[kk], wv[kk].y, acc[i][1]);
          acc[i][2] = fmaf(a[kk], wv[kk].z, acc[i][2]); acc[i][3] = fmaf(a[kk], wv[kk].w, acc[i][3]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < RT; ++i) {
      float4 v = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
      if (res) {
        const float4 r = *reinterpret_cast<const float4*>(res + (size_t)(r0 + i) * ldr + c0);
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      if (relu) { v.x = fmaxf(v.x, 0.0f); v.y = fmaxf(v.y, 0.0f); v.z = fmaxf(v.z, 0.0f); v.w = fmaxf(v.w, 0.0f); }
      *reinterpret_cast<float4*>(out + (size_t)(r0 + i) * ldo + c0) = v;
    }
  }
}
// tile height chosen so that (almost) every thread of the CTA gets a tile
__device__ void gst_dense(const float* __restrict__ in, int ldi, const float* __restrict__ Wt, const float* __restrict__ bias,
                          const float* res, int ldr, float* out, int ldo, int R, int K, int Nout, bool relu) {
  const int ct = Nout >> 2;
  if ((R >> 2) * ct >= (int)blockDim.x) gst_dense_t<4>(in, ldi, Wt, bias, res, ldr, out, ldo, R, K, Nout, relu);
  else if ((R >> 1) * ct >= (int)blockDim.x) gst_dense_t<2>(in, ldi, Wt, bias, res, ldr, out, ldo, R, K, Nout, relu);
  else gst_dense_t<1>(in, ldi, Wt, bias, res, ldr, out, ldo, R, K, Nout, relu);
}

// LayerNorm over the 64 features of every row (one warp per row, two features per lane), optional row mask.
__device__ void gst_layernorm(const float* in, float* out, int R, const float* __restrict__ g, const float* __restrict__ b,
                              const float* rowmask) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  for (int r = warp; r < R; r += nw) {
    const float a0 = in[r * GST_D + lane], a1 = in[r * GST_D + lane + 32];
    float s = a0 + a1;
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s * (1.0f / GST_D);
    const float d0 = a0 - mean, d1 = a1 - mean;
    float v = d0 * d0 + d1 * d1;
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const float inv = rsqrtf(v * (1.0f / GST_D) + 1e-5f);
    const float m = rowmask ? rowmask[r] : 1.0f;
    out[r * GST_D + lane] = (d0 * inv * g[lane] + b[lane]) * m;
    out[r * GST_D + lane + 32] = (d1 * inv * g[lane + 32] + b[lane + 32]) * m;
  }
}

// One node-encoder layer on R = G * H rows (G groups of H nodes attend within their group).
//   xin  [R][2]   displacements            rowm [R]  node validity (attn_mask[i][j] = rowm[i] * rowm[j])
//   X    [R][64]  work / result            Y    [R][64] work        BIG [R][192 | 128] work
__device__ void gst_encoder(const GstW& w, const float* xin, const float* rowm, float* X, float* Y, float* BIG, int R, int H) {
  // node embedding (K = 2) fused with norm_node and the pedestrian mask
  for (int i = threadIdx.x; i < R * GST_D; i += blockDim.x) {
    const int r = i >> 6, c = i & 63;
    Y[i] = fmaf(xin[2 * r + 1], w.We_t[GST_D + c], fmaf(xin[2 * r], w.We_t[c], w.be[c]));
  }
  __syncthreads();
  gst_layernorm(Y, X, R, w.ln0_g, w.ln0_b, rowm);
  __syncthreads();
  gst_dense(X, GST_D, w.Win_t, w.bin, nullptr, 0, BIG, 192, R, GST_D, 192, false);
  __syncthreads();
  // attention: one thread per (row, head); soft-max over ALL H neighbours, then mask and renormalise (mha.py:236-242)
  for (int i = threadIdx.x; i < R * 8; i += blockDim.x) {
    const int r = i >> 3, hd = i & 7;
    const int g0 = (r / H) * H;
    const float scaling = 0.35355339059327373f;       // 8 ** -0.5
    float q[8];
#pragma unroll
    for (int d = 0; d < 8; ++d) q[d] = BIG[r * 192 + hd * 8 + d] * scaling;
    float mx = -INFINITY;
    for (int j = 0; j < H; ++j) {
      const float* kj = BIG + (g0 + j) * 192 + 64 + hd * 8;
      float s = 0.0f;
#pragma unroll
      for (int d = 0; d < 8; ++d) s = fmaf(q[d], kj[d], s);
      mx = fmaxf(mx, s);
    }
    float den = 0.0f, dm = 0.0f, o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    const float mi = rowm[r];
    for (int j = 0; j < H; ++j) {
      const float* kj = BIG + (g0 + j) * 192 + 64 + hd * 8;
      const float* vj = BIG + (g0 + j) * 192 + 128 + hd * 8;
      float s = 0.0f;
#pragma unroll
      for (int d = 0; d < 8; ++d) s = fmaf(q[d], kj[d], s);
      const float e = expf(s - mx);
      den += e;
      const float em = e * (mi * rowm[g0 + j]);
      dm += em;
#pragma unroll
      for (int d = 0; d < 8; ++d) o[d] = fmaf(em, vj[d], o[d]);
    }
    // w = softmax * mask; w /= (sum(w) + 1e-10)  ==  (e*m/den) / (dm/den + 1e-10)
    const float scale = (1.0f / den) / (dm / den + 1e-10f);
#pragma unroll
    for (int d = 0; d < 8; ++d) Y[r * GST_D + hd * 8 + d] = o[d] * scale;
  }
  __syncthreads();
  gst_dense(Y, GST_D, w.Wout_t, w.bout, X, GST_D, X, GST_D, R, GST_D, GST_D, false);      // x = x + out_proj(attn)
  __syncthreads();
  gst_layernorm(X, Y, R, w.ln1_g, w.ln1_b, nullptr);
  __syncthreads();
  gst_dense(Y, GST_D, w.W1_t, w.b1, nullptr, 0, BIG, 128, R, GST_D, 128, true);
  __syncthreads();
  gst_dense(BIG, 128, w.W2_t, w.b2, X, GST_D, X, GST_D, R, 128, GST_D, false);             // x = x + ffn(norm1(x))
  __syncthreads();
}

__device__ __forceinline__ float gst_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

struct GstShared {
  float* X; float* Y; float* BIG; float* GH;      // [R][64], [R][64], [R][256], [H][256]
  float* h; float* c;                             // [H][64]
  float* xin;                                     // [R][2]
  float* rowm;                                    // [R]
  float* pos_last; float* mu_cum; float* fp;      // [H][2], [H][2], [H]
  float* pred;                                    // [H][GST_T][2] predicted world positions
};

// smem floats needed for H nodes
__host__ __device__ inline size_t gst_smem_floats(int H) {
  const size_t R = (size_t)GST_T * H;
  return R * 64 * 2 + R * 256 + (size_t)H * 256 + (size_t)H * 64 * 2 + R * 2 + R + (size_t)H * (2 + 2 + 1) + (size_t)H * GST_T * 2 + 64;
}

__global__ void __launch_bounds__(GST_THREADS) cn_pretext_kernel(GstW w, int N, int H, int P, float thr, float collision_penalty,
                                                                 float* __restrict__ ring_pos /* [5][N][H][2] */,
                                                                 uint8_t* __restrict__ ring_mask /* [5][N][H] */, int newest,
                                                                 const float* __restrict__ robot_node /* [N][7] */,
                                                                 const float* __restrict__ sp2 /* [N][H][2] */,
                                                                 const uint8_t* __restrict__ vis /* [N][H] */,
                                                                 float* __restrict__ reward /* [N] or null */,
                                                                 float* __restrict__ penalty_out /* [N] or null */,
                                                                 float* __restrict__ out_sp /* [N][H][2(P+1)] */) {
  extern __shared__ __align__(16) float sm[];
  const int e = blockIdx.x;
  if (e >= N) return;
  const int R = GST_T * H;
  GstShared s;
  float* q = sm;
  s.X = q; q += R * 64; s.Y = q; q += R * 64; s.BIG = q; q += R * 256; s.GH = q; q += H * 256;
  s.h = q; q += H * 64; s.c = q; q += H * 64; s.xin = q; q += R * 2; s.rowm = q; q += R;
  s.pos_last = q; q += H * 2; s.mu_cum = q; q += H * 2; s.fp = q; q += H; s.pred = q;
  const float rx = robot_node[e * 7], ry = robot_node[e * 7 + 1];
  // ---- traj_buffer.append(robot + spatial_edges[:, :2]); mask_buffer.append(visible_masks)
  for (int i = threadIdx.x; i < H; i += blockDim.x) {
    const size_t o = ((size_t)newest * N + e) * H + i;
    ring_pos[2 * o] = rx + sp2[((size_t)e * H + i) * 2];
    ring_pos[2 * o + 1] = ry + sp2[((size_t)e * H + i) * 2 + 1];
    ring_mask[o] = vis[(size_t)e * H + i] ? 1 : 0;
  }
  __syncthreads();
  // ---- interface.forward input processing: frames oldest -> newest
  for (int i = threadIdx.x; i < R; i += blockDim.x) {
    const int t = i / H, n = i - t * H;
    const int slot = (newest + 1 + t) % GST_T, slot_prev = (newest + t) % GST_T, slot_last = newest;
    const size_t o = ((size_t)slot * N + e) * H + n, op = ((size_t)slot_prev * N + e) * H + n,
                 ol = ((size_t)slot_last * N + e) * H + n;
    // loss_mask_rel_obs: frame 0 = mask[0]; frame t >= 1 = mask[t-1] * mask[LAST] (sic, interface.forward:77-78)
    const float m = t == 0 ? (float)ring_mask[o] : (float)ring_mask[op] * (float)ring_mask[ol];
    float dx = 0.0f, dy = 0.0f;
    if (t > 0) { dx = ring_pos[2 * o] - ring_pos[2 * op]; dy = ring_pos[2 * o + 1] - ring_pos[2 * op + 1]; }
    s.xin[2 * i] = GST_INVALID * (1.0f - m) + dx * m;
    s.xin[2 * i + 1] = GST_INVALID * (1.0f - m) + dy * m;
    s.rowm[i] = m;
    if (t == GST_T - 1) { s.fp[n] = m; s.pos_last[2 * n] = ring_pos[2 * o]; s.pos_last[2 * n + 1] = ring_pos[2 * o + 1]; }
  }
  for (int i = threadIdx.x; i < H * 64; i += blockDim.x) { s.h[i] = 0.0f; s.c[i] = 0.0f; }
  for (int i = threadIdx.x; i < H * 2; i += blockDim.x) s.mu_cum[i] = 0.0f;
  __syncthreads();
  // ---- observation period: encoder on the 5 stacked frames, mask, LSTM
  gst_encoder(w, s.xin, s.rowm, s.X, s.Y, s.BIG, R, H);
  for (int i = threadIdx.x; i < R * 64; i += blockDim.x) s.X[i] *= s.rowm[i >> 6];
  __syncthreads();
  gst_dense(s.X, GST_D, w.Wih_t, w.bih, nullptr, 0, s.BIG, 256, R, GST_D, 256, false);      // W_ih x_t + b_ih, all frames
  __syncthreads();
  for (int t = 0; t < GST_T; ++t) {
    gst_dense(s.h, GST_D, w.Whh_t, w.bhh, nullptr, 0, s.GH, 256, H, GST_D, 256, false);
    __syncthreads();
    for (int i = threadIdx.x; i < H * 64; i += blockDim.x) {
      const int n = i >> 6, j = i & 63;
      const float* gx = s.BIG + (size_t)(t * H + n) * 256;
      const float* gh = s.GH + (size_t)n * 256;
      const float ig = gst_sigmoid(gx[j] + gh[j]), fg = gst_sigmoid(gx[64 + j] + gh[64 + j]);
      const float gg = tanhf(gx[128 + j] + gh[128 + j]), og = gst_sigmoid(gx[192 + j] + gh[192 + j]);
      const float c2 = fg * s.c[i] + ig * gg;
      s.c[i] = c2; s.h[i] = og * tanhf(c2);
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < H * 64; i += blockDim.x) { const float m = s.fp[i >> 6]; s.h[i] *= m; s.c[i] *= m; }
  __syncthreads();
  // ---- prediction period (recursive decoding, the mean is fed back)
  for (int tt = 0; tt < GST_T; ++tt) {
    if (tt > 0) {
      gst_encoder(w, s.xin, s.fp, s.X, s.Y, s.BIG, H, H);            // xin = masked mean of the previous step
      for (int i = threadIdx.x; i < H * 64; i += blockDim.x) s.X[i] *= s.fp[i >> 6];
      __syncthreads();
      gst_dense(s.X, GST_D, w.Wih_t, w.bih, nullptr, 0, s.BIG, 256, H, GST_D, 256, false);
      gst_dense(s.h, GST_D, w.Whh_t, w.bhh, nullptr, 0, s.GH, 256, H, GST_D, 256, false);
      __syncthreads();
      for (int i = threadIdx.x; i < H * 64; i += blockDim.x) {
        const int n = i >> 6, j = i & 63;
        const float* gx = s.BIG + (size_t)n * 256;
        const float* gh = s.GH + (size_t)n * 256;
        const float ig = gst_sigmoid(gx[j] + gh[j]), fg = gst_sigmoid(gx[64 + j] + gh[64 + j]);
        const float gg = tanhf(gx[128 + j] + gh[128 + j]), og = gst_sigmoid(gx[192 + j] + gh[192 + j]);
        const float c2 = fg * s.c[i] + ig * gg, h2 = og * tanhf(c2);
        const float m = s.fp[n];
        s.c[i] = c2 * m + s.c[i] * (1.0f - m);
        s.h[i] = h2 * m + s.h[i] * (1.0f - m);
      }
      __syncthreads();
    }
    // hidden2pos: only the mean is consumed downstream (sigma / corr are dropped by process_obs_rew)
    for (int i = threadIdx.x; i < H * 2; i += blockDim.x) {
      const int n = i >> 1, d = i & 1;
      float a = w.bp[d];
      for (int k = 0; k < 64; ++k) a = fmaf(s.h[n * 64 + k], w.Wp[d * 64 + k], a);
      const float m = s.fp[n];
      s.xin[i] = a * m;                                               // x_sample (masked) = next encoder input
      const float cum = s.mu_cum[i] + a;
      s.mu_cum[i] = cum;
      s.pred[(n * GST_T + tt) * 2 + d] = (cum + s.pos_last[i]) * m + GST_INVALID * (1.0f - m);
    }
    __syncthreads();
  }
  // ---- process_obs_rew: future-collision penalty, predicted relative positions, sort by distance
  if (threadIdx.x < 32) {
    float pen = 0.0f;
    for (int i = threadIdx.x; i < H * GST_T; i += 32) {
      const int n = i / GST_T, k = i - n * GST_T;
      if (k < P && s.fp[n] != 0.0f) {
        const float dx = s.pred[i * 2] - rx, dy = s.pred[i * 2 + 1] - ry;
        if (sqrtf(dx * dx + dy * dy) < thr) pen = fminf(pen, collision_penalty / (float)(4 << k));
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) pen = fminf(pen, __shfl_xor_sync(0xffffffffu, pen, o));
    if (threadIdx.x == 0) {
      if (reward) reward[e] += pen;
      if (penalty_out) penalty_out[e] = pen;
    }
  }
  const int W = 2 * (P + 1);
  for (int n = threadIdx.x; n < H; n += blockDim.x) {
    const float cx = sp2[((size_t)e * H + n) * 2], cy = sp2[((size_t)e * H + n) * 2 + 1];
    const float key = sqrtf(cx * cx + cy * cy);
    int rank = 0;
    for (int j = 0; j < H; ++j) {
      const float ox = sp2[((size_t)e * H + j) * 2], oy = sp2[((size_t)e * H + j) * 2 + 1];
      const float kj = sqrtf(ox * ox + oy * oy);
      rank += (kj < key || (kj == key && j < n)) ? 1 : 0;
    }
    float* dst = out_sp + ((size_t)e * H + rank) * W;
    dst[0] = cx; dst[1] = cy;
    const bool ok = s.fp[n] != 0.0f;
    for (int k = 0; k < P; ++k) {
      // unpredicted humans keep the tiled current relative position (crowd_sim_pred_real_gst.py generate_ob)
      dst[2 + 2 * k] = ok ? s.pred[(n * GST_T + k) * 2] - rx : cx;
      dst[3 + 2 * k] = ok ? s.pred[(n * GST_T + k) * 2 + 1] - ry : cy;
    }
  }
}

const char* kParamNames[] = {
    "gumbel_social_transformer.node_embedding.weight", "gumbel_social_transformer.node_embedding.bias",
    "gumbel_social_transformer.node_encoder_layers.0.norm_node.weight", "gumbel_social_transformer.node_encoder_layers.0.norm_node.bias",
    "gumbel_social_transformer.node_encoder_layers.0.self_attn.in_proj_weight",
    "gumbel_social_transformer.node_encoder_layers.0.self_attn.in_proj_bias",
    "gumbel_social_transformer.node_encoder_layers.0.self_attn.out_proj.weight",
    "gumbel_social_transformer.node_encoder_layers.0.self_attn.out_proj.bias",
    "gumbel_social_transformer.node_encoder_layers.0.norm1_node.weight", "gumbel_social_transformer.node_encoder_layers.0.norm1_node.bias",
    "gumbel_social_transformer.node_encoder_layers.0.linear1.weight", "gumbel_social_transformer.node_encoder_layers.0.linear1.bias",
    "gumbel_social_transformer.node_encoder_layers.0.linear2.weight", "gumbel_social_transformer.node_encoder_layers.0.linear2.bias",
    "lstm.weight_ih_l0", "lstm.bias_ih_l0", "lstm.weight_hh_l0", "lstm.bias_hh_l0", "hidden2pos.weight", "hidden2pos.bias"};
const int kParamRows[] = {64, 64, 64, 64, 192, 192, 64, 64, 64, 64, 128, 128, 64, 64, 256, 256, 256, 256, 5, 5};
const int kParamCols[] = {2, 1, 1, 1, 64, 1, 64, 1, 1, 1, 64, 1, 128, 1, 64, 1, 64, 1, 64, 1};
const bool kTranspose[] = {true, false, false, false, true, false, true, false, false, false,
                           true, false, true, false, true, false, true, false, false, false};
const int kNumParams = 20;

}  // namespace

// tensor-core implementation (cn_gst_tc.cu)
void* cn_gst_tc_create(int N, int H, int P, float thr, float pen, int device, const float* const* host, const int* rows,
                       const int* cols);
void cn_gst_tc_destroy(void* handle);
int64_t cn_gst_tc_launches(void* handle);
int cn_gst_tc_step(void* handle, float* ring_pos, uint8_t* ring_mask, int newest, const float* robot, const float* sp2,
                   const uint8_t* vis, float* reward, float* penalty, float* out_sp, cudaStream_t st);
int cn_gst_tcc_step(void* handle, float* ring_pos, uint8_t* ring_mask, int newest, const float* robot, const float* sp2,
                    const uint8_t* vis, float* reward, float* penalty, float* out_sp, cudaStream_t st);

struct cn_gst {
  void* tc;           // non-null: dense layers on the tensor-core GEMM (CN_GST_MODE=tcc (default) or tc)
  bool compact;       // tcc: only the rows whose mask is 1 are computed (cn_gst_tcc_step)
  int N, H, P, device;
  float thr, collision_penalty;
  std::map<std::string, std::vector<float>> host;
  std::vector<void*> allocs;
  const float* dev[kNumParams];
  float* ring_pos;
  uint8_t* ring_mask;
  int newest;         // ring slot of the most recent frame
  bool finalized;
  int64_t launches;
  size_t smem;
};

extern "C" {

int cn_gst_create(int num_envs, int human_num, int predict_steps, double robot_radius, double human_radius,
                  double collision_penalty, int device, cn_gst** out) {
  if (!out) return cn_set_error("cn_gst_create: null argument");
  *out = nullptr;
  if (num_envs <= 0 || human_num <= 0 || human_num % 4 || predict_steps < 1 || predict_steps > GST_T)
    return cn_set_error("cn_gst_create: need num_envs > 0, human_num %% 4 == 0 and 1 <= predict_steps <= %d (got %d, %d, %d)",
                        GST_T, num_envs, human_num, predict_steps);
  int ndev = 0;
  cudaError_t err = cudaGetDeviceCount(&ndev);
  if (err != cudaSuccess || ndev == 0)
    return cn_set_error("cn_gst_create: no CUDA device (%s); this engine has no CPU fallback",
                        err == cudaSuccess ? "device count 0" : cudaGetErrorString(err));
  if (device < 0 || device >= ndev) return cn_set_error("cn_gst_create: bad device %d", device);
  if (human_num > 32) return cn_set_error("cn_gst_create: human_num %d > 32 is not supported by the predictor kernels", human_num);
  const size_t smem = gst_smem_floats(human_num) * sizeof(float);
  if (smem > 227 * 1024)
    return cn_set_error("cn_gst_create: human_num %d needs %zu bytes of shared memory (max 232448)", human_num, smem);
  cudaSetDevice(device);
  cn_gst* g = new cn_gst();
  g->N = num_envs; g->H = human_num; g->P = predict_steps; g->device = device;
  g->thr = (float)(robot_radius + human_radius); g->collision_penalty = (float)collision_penalty;
  g->newest = GST_T - 1; g->finalized = false; g->launches = 0; g->smem = smem; g->tc = nullptr; g->compact = true;
  g->ring_pos = nullptr; g->ring_mask = nullptr;
  void* q = nullptr;
  err = cudaMalloc(&q, (size_t)GST_T * num_envs * human_num * 2 * sizeof(float));
  if (err == cudaSuccess) { g->ring_pos = (float*)q; g->allocs.push_back(q); err = cudaMalloc(&q, (size_t)GST_T * num_envs * human_num); }
  if (err == cudaSuccess) { g->ring_mask = (uint8_t*)q; g->allocs.push_back(q); }
  if (err == cudaSuccess) err = cudaFuncSetAttribute(cn_pretext_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) {
    for (void* a : g->allocs) cudaFree(a);
    delete g;
    return cn_set_error("cn_gst_create: %s", cudaGetErrorString(err));
  }
  *out = g;
  return 0;
}

int cn_gst_destroy(cn_gst* g) {
  if (!g) return 0;
  cudaSetDevice(g->device);
  cudaDeviceSynchronize();
  if (g->tc) cn_gst_tc_destroy(g->tc);
  for (void* a : g->allocs) cudaFree(a);
  delete g;
  return 0;
}

// name = key of the reference checkpoint's model_state_dict (st_model), data = float32 host array
int cn_gst_set_param(cn_gst* g, const char* name, const float* data, size_t count) {
  if (!g || !name || !data) return cn_set_error("cn_gst_set_param: null argument");
  for (int i = 0; i < kNumParams; ++i) {
    if (strcmp(name, kParamNames[i]) == 0) {
      if (count != (size_t)kParamRows[i] * kParamCols[i])
        return cn_set_error("cn_gst_set_param: '%s' has %zu elements, expected %d", name, count, kParamRows[i] * kParamCols[i]);
      g->host[name].assign(data, data + count);
      g->finalized = false;
      return 0;
    }
  }
  return cn_set_error("cn_gst_set_param: unknown parameter '%s'", name);
}

int cn_gst_finalize(cn_gst* g) {
  if (!g) return cn_set_error("cn_gst_finalize: null argument");
  cudaSetDevice(g->device);
  for (int i = 0; i < kNumParams; ++i) {
    auto it = g->host.find(kParamNames[i]);
    if (it == g->host.end()) return cn_set_error("cn_gst_finalize: parameter '%s' was not set", kParamNames[i]);
    std::vector<float> v = it->second;
    const int rows = kParamRows[i], cols = kParamCols[i];
    if (kTranspose[i]) {                       // [out][in] -> [in][out]
      std::vector<float> t(v.size());
      for (int r = 0; r < rows; ++r) for (int c = 0; c < cols; ++c) t[(size_t)c * rows + r] = v[(size_t)r * cols + c];
      v.swap(t);
    }
    void* q = nullptr;
    cudaError_t err = cudaMalloc(&q, v.size() * sizeof(float));
    if (err == cudaSuccess) err = cudaMemcpy(q, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice);
    if (err != cudaSuccess) return cn_set_error("cn_gst_finalize: %s", cudaGetErrorString(err));
    g->allocs.push_back(q);
    g->dev[i] = (const float*)q;
  }
  // default: dense layers as batched tensor-core GEMMs over all environments (cn_gst_tc.cu, 2.5x faster at N = 4096);
  // CN_GST_MODE=fused selects the single fused CUDA-core kernel of this file (no workspace, one launch)
  const char* mode = getenv("CN_GST_MODE");
  g->compact = !(mode && strcmp(mode, "tc") == 0);          // default "tcc": compact rows; "tc": every row
  if (!(mode && strcmp(mode, "fused") == 0)) {
    if (g->tc) { cn_gst_tc_destroy(g->tc); g->tc = nullptr; }
    const float* hp[kNumParams];
    for (int i = 0; i < kNumParams; ++i) hp[i] = g->host[kParamNames[i]].data();
    g->tc = cn_gst_tc_create(g->N, g->H, g->P, g->thr, g->collision_penalty, g->device, hp, kParamRows, kParamCols);
    if (!g->tc) return 1;                       // cn_last_error holds the reason
  }
  g->finalized = true;
  return 0;
}

// VecPretextNormalize.reset(): traj_buffer <- -999, mask_buffer <- False (rl/vec_env/vec_pretext_normalize.py:85-101)
int cn_gst_reset(cn_gst* g, void* stream) {
  if (!g) return cn_set_error("cn_gst_reset: null argument");
  cudaSetDevice(g->device);
  const size_t n = (size_t)GST_T * g->N * g->H;
  std::vector<float> inv(n * 2, GST_INVALID);
  cudaError_t err = cudaMemcpyAsync(g->ring_pos, inv.data(), n * 2 * sizeof(float), cudaMemcpyHostToDevice, (cudaStream_t)stream);
  if (err == cudaSuccess) err = cudaStreamSynchronize((cudaStream_t)stream);
  if (err == cudaSuccess) err = cudaMemsetAsync(g->ring_mask, 0, n, (cudaStream_t)stream);
  if (err != cudaSuccess) return cn_set_error("cn_gst_reset: %s", cudaGetErrorString(err));
  g->newest = GST_T - 1;
  return 0;
}

// VecPretextNormalize.process_obs_rew for the N environments of this shard (device pointers, caller's stream):
//   d_robot_node [N,7], d_spatial2 [N,H,2] + d_visible [N,H] = raw CrowdSimPredRealGST-v0 observation (the engine's
//   CrowdSimVarNum-v0 mode with sort_humans = 0 produces exactly these), d_reward [N] (in/out, may be NULL),
//   d_penalty [N] (out, may be NULL), d_spatial_out [N,H,2(P+1)] = predicted, distance-sorted spatial_edges.
int cn_gst_step(cn_gst* g, const float* d_robot_node, const float* d_spatial2, const uint8_t* d_visible, float* d_reward,
                float* d_penalty, float* d_spatial_out, void* stream) {
  if (!g || !d_robot_node || !d_spatial2 || !d_visible || !d_spatial_out) return cn_set_error("cn_gst_step: null argument");
  if (!g->finalized) return cn_set_error("cn_gst_step: call cn_gst_finalize after setting the parameters");
  CnDeviceGuard guard(g->device);
  g->newest = (g->newest + 1) % GST_T;
  if (g->tc) {
    g->launches += 1;
    if (g->compact)
      return cn_gst_tcc_step(g->tc, g->ring_pos, g->ring_mask, g->newest, d_robot_node, d_spatial2, d_visible, d_reward, d_penalty,
                             d_spatial_out, (cudaStream_t)stream);
    return cn_gst_tc_step(g->tc, g->ring_pos, g->ring_mask, g->newest, d_robot_node, d_spatial2, d_visible, d_reward, d_penalty,
                          d_spatial_out, (cudaStream_t)stream);
  }
  GstW w;
  w.We_t = g->dev[0]; w.be = g->dev[1]; w.ln0_g = g->dev[2]; w.ln0_b = g->dev[3]; w.Win_t = g->dev[4]; w.bin = g->dev[5];
  w.Wout_t = g->dev[6]; w.bout = g->dev[7]; w.ln1_g = g->dev[8]; w.ln1_b = g->dev[9]; w.W1_t = g->dev[10]; w.b1 = g->dev[11];
  w.W2_t = g->dev[12]; w.b2 = g->dev[13]; w.Wih_t = g->dev[14]; w.bih = g->dev[15]; w.Whh_t = g->dev[16]; w.bhh = g->dev[17];
  w.Wp = g->dev[18]; w.bp = g->dev[19];
  cn_pretext_kernel<<<g->N, GST_THREADS, g->smem, (cudaStream_t)stream>>>(w, g->N, g->H, g->P, g->thr, g->collision_penalty,
                                                                           g->ring_pos, g->ring_mask, g->newest, d_robot_node,
                                                                           d_spatial2, d_visible, d_reward, d_penalty, d_spatial_out);
  g->launches += 1;
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("cn_pretext_kernel launch: %s", cudaGetErrorString(err));
  return 0;
}

int64_t cn_gst_launch_count(cn_gst* g) { return !g ? 0 : (g->tc ? cn_gst_tc_launches(g->tc) : g->launches); }

}  // extern "C"
