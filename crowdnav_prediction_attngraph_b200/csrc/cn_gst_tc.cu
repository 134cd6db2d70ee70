// Config 3's GST predictor with its dense layers on the wgmma 3xFP16 GEMM (cn_gemm_tc.h).  Same arithmetic as the
// fused CUDA-core kernel of cn_gst.cu (reference lines are cited there); here every layer is a batched [rows, K] GEMM over ALL environments:
//   observation period: rows = N * 5 * H (frames of one environment contiguous: row = (e * 5 + t) * H + n)
//   decoding steps:     rows = N * H
// and small row-wise kernels do embedding + LayerNorm, the H x H attention, residuals, the LSTM cell and the wrapper's
// tail.  Default path of cn_gst_step (CN_GST_MODE=fused selects the single-kernel version); validated by the same
// tests as the fused kernel.
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

#include "cn_gemm_tc.h"
#include "cn_host_util.h"
#include "cn_launch.cuh"

namespace {

#define GT_T 5
#define GT_INVALID (-999.0f)

struct GstTcW {   // fp32 device parameters used by the row-wise kernels
  const float *We_t, *be, *ln0_g, *ln0_b, *ln1_g, *ln1_b, *Wp, *bp;
  const float *bin, *bout, *b1, *b2, *bih, *bhh;
};

__device__ __forceinline__ void gt_split_store(__half* hi, __half* lo, size_t idx, float x) {
  const float c = fminf(fmaxf(x, -65504.0f), 65504.0f);
  const __half h = __float2half_rn(c);
  hi[idx] = h;
  lo[idx] = __float2half_rn(c - __half2float(h));
}

// LayerNorm of one 64-wide row held as two values per lane
__device__ __forceinline__ void gt_ln(float a0, float a1, const float* g, const float* b, int lane, float& o0, float& o1) {
  float s = a0 + a1;
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s * (1.0f / 64.0f);
  const float d0 = a0 - mean, d1 = a1 - mean;
  float v = d0 * d0 + d1 * d1;
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const float inv = rsqrtf(v * (1.0f / 64.0f) + 1e-5f);
  o0 = d0 * inv * g[lane] + b[lane];
  o1 = d1 * inv * g[lane + 32] + b[lane + 32];
}

// ring append + input processing of the 5 observed frames + node embedding + norm_node + mask.  One warp per row.
__global__ void __launch_bounds__(256) gt_prep_kernel(GstTcW w, int N, int H, float* __restrict__ ring_pos,
                                                      uint8_t* __restrict__ ring_mask, int newest,
                                                      const float* __restrict__ robot, const float* __restrict__ sp2,
                                                      const uint8_t* __restrict__ vis, float* __restrict__ X0,
                                                      __half* __restrict__ xh, __half* __restrict__ xl, float* __restrict__ rowm,
                                                      float* __restrict__ fp, float* __restrict__ pos_last,
                                                      float* __restrict__ h32, __half* __restrict__ hh, __half* __restrict__ hl,
                                                      float* __restrict__ c32, float* __restrict__ mu_cum) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int R = N * GT_T * H;
  if (r >= R) return;
  const int n = r % H, t = (r / H) % GT_T, e = r / (H * GT_T);
  // positions / masks of frame t, t-1 and the newest frame; the newest comes straight from this step's observation
  auto frame_pos = [&](int tt, float& x, float& y, float& m) {
    if (tt == GT_T - 1) {
      x = robot[e * 7] + sp2[((size_t)e * H + n) * 2];
      y = robot[e * 7 + 1] + sp2[((size_t)e * H + n) * 2 + 1];
      m = vis[(size_t)e * H + n] ? 1.0f : 0.0f;
    } else {
      const int slot = (newest + 1 + tt) % GT_T;
      const size_t o = ((size_t)slot * N + e) * H + n;
      x = ring_pos[2 * o]; y = ring_pos[2 * o + 1]; m = (float)ring_mask[o];
    }
  };
  float x, y, m, xp = 0, yp = 0, mp = 0, xl_, yl_, ml_;
  frame_pos(t, x, y, m);
  frame_pos(GT_T - 1, xl_, yl_, ml_);
  if (t > 0) frame_pos(t - 1, xp, yp, mp);
  const float mrel = t == 0 ? m : mp * ml_;                  // interface.forward:77-78 (sic)
  const float dx = t == 0 ? 0.0f : x - xp, dy = t == 0 ? 0.0f : y - yp;
  const float ix = GT_INVALID * (1.0f - mrel) + dx * mrel, iy = GT_INVALID * (1.0f - mrel) + dy * mrel;
  float e0 = fmaf(iy, w.We_t[64 + lane], fmaf(ix, w.We_t[lane], w.be[lane]));
  float e1 = fmaf(iy, w.We_t[96 + lane], fmaf(ix, w.We_t[32 + lane], w.be[32 + lane]));
  float o0, o1;
  gt_ln(e0, e1, w.ln0_g, w.ln0_b, lane, o0, o1);
  o0 *= mrel; o1 *= mrel;
  const size_t b = (size_t)r * 64;
  X0[b + lane] = o0; X0[b + lane + 32] = o1;
  gt_split_store(xh, xl, b + lane, o0); gt_split_store(xh, xl, b + lane + 32, o1);
  if (lane == 0) rowm[r] = mrel;
  if (t == GT_T - 1) {
    const size_t rd = (size_t)e * H + n;
    if (lane == 0) {
      fp[rd] = mrel; pos_last[2 * rd] = x; pos_last[2 * rd + 1] = y; mu_cum[2 * rd] = 0.0f; mu_cum[2 * rd + 1] = 0.0f;
      // traj_buffer.append / mask_buffer.append (readers of this slot in this launch use the observation directly)
      const size_t o = ((size_t)newest * N + e) * H + n;
      ring_pos[2 * o] = x; ring_pos[2 * o + 1] = y; ring_mask[o] = m != 0.0f ? 1 : 0;
    }
    h32[rd * 64 + lane] = 0.0f; h32[rd * 64 + lane + 32] = 0.0f;
    c32[rd * 64 + lane] = 0.0f; c32[rd * 64 + lane + 32] = 0.0f;
    hh[rd * 64 + lane] = __float2half_rn(0.0f); hh[rd * 64 + lane + 32] = __float2half_rn(0.0f);
    hl[rd * 64 + lane] = __float2half_rn(0.0f); hl[rd * 64 + lane + 32] = __float2half_rn(0.0f);
  }
}

// decoding step: node embedding of x_sample + norm_node + mask.  One warp per row of [N*H].
__global__ void __launch_bounds__(256) gt_embed_kernel(GstTcW w, int Rd, const float* __restrict__ xin, const float* __restrict__ fp,
                                                       float* __restrict__ X0, __half* __restrict__ xh, __half* __restrict__ xl) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= Rd) return;
  const float ix = xin[2 * r], iy = xin[2 * r + 1];
  float e0 = fmaf(iy, w.We_t[64 + lane], fmaf(ix, w.We_t[lane], w.be[lane]));
  float e1 = fmaf(iy, w.We_t[96 + lane], fmaf(ix, w.We_t[32 + lane], w.be[32 + lane]));
  float o0, o1;
  gt_ln(e0, e1, w.ln0_g, w.ln0_b, lane, o0, o1);
  const float m = fp[r];
  o0 *= m; o1 *= m;
  const size_t b = (size_t)r * 64;
  X0[b + lane] = o0; X0[b + lane + 32] = o1;
  gt_split_store(xh, xl, b + lane, o0); gt_split_store(xh, xl, b + lane + 32, o1);
}

// attention within groups of H consecutive rows: one CTA per group (8 H threads = one per (row, head)), the group's
// q | k | v rows staged once in shared memory (every key / value row is read by all 8 H threads of the group: served
// from L1 this kernel was 1/3 of the predictor's time).  rowm: per-row validity.
#define GT_MAXH 32
__global__ void __launch_bounds__(8 * GT_MAXH) gt_attn_kernel(int R, int H, const float* __restrict__ qkv,
                                                              const float* __restrict__ rowm, __half* __restrict__ ah,
                                                              __half* __restrict__ al) {
  cn_pdl_prologue();
  __shared__ __align__(16) float sq[GT_MAXH * 192];
  __shared__ float sm_[GT_MAXH];
  const int g0 = blockIdx.x * H;
  if (g0 >= R) return;
  for (int i = threadIdx.x; i < H * 48; i += blockDim.x)
    reinterpret_cast<float4*>(sq)[i] = __ldg(reinterpret_cast<const float4*>(qkv + (size_t)g0 * 192) + i);
  for (int i = threadIdx.x; i < H; i += blockDim.x) sm_[i] = rowm[g0 + i];
  __syncthreads();
  const int lr = threadIdx.x >> 3, hd = threadIdx.x & 7;
  if (lr >= H) return;
  const float scaling = 0.35355339059327373f;
  float q[8];
#pragma unroll
  for (int d = 0; d < 8; ++d) q[d] = sq[lr * 192 + hd * 8 + d] * scaling;
  float mx = -INFINITY;
  for (int j = 0; j < H; ++j) {
    const float* kj = sq + j * 192 + 64 + hd * 8;
    float s = 0.0f;
#pragma unroll
    for (int d = 0; d < 8; ++d) s = fmaf(q[d], kj[d], s);
    mx = fmaxf(mx, s);
  }
  float den = 0.0f, dm = 0.0f, o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  const float mi = sm_[lr];
  for (int j = 0; j < H; ++j) {
    const float* kj = sq + j * 192 + 64 + hd * 8;
    const float* vj = sq + j * 192 + 128 + hd * 8;
    float s = 0.0f;
#pragma unroll
    for (int d = 0; d < 8; ++d) s = fmaf(q[d], kj[d], s);
    const float ex = expf(s - mx);
    den += ex;
    const float em = ex * (mi * sm_[j]);
    dm += em;
#pragma unroll
    for (int d = 0; d < 8; ++d) o[d] = fmaf(em, vj[d], o[d]);
  }
  const float scale = (1.0f / den) / (dm / den + 1e-10f);
  const size_t ob = (size_t)(g0 + lr) * 64 + hd * 8;
#pragma unroll
  for (int d = 0; d < 8; ++d) gt_split_store(ah, al, ob + d, o[d] * scale);
}

// X1 = X0 + O (fp32), Y = norm1(X1) as fp16 hi/lo.  One warp per row.
__global__ void __launch_bounds__(256) gt_res_ln_kernel(GstTcW w, int R, const float* __restrict__ X0, const float* __restrict__ O,
                                                        float* __restrict__ X1, __half* __restrict__ yh, __half* __restrict__ yl) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= R) return;
  const size_t b = (size_t)r * 64;
  const float a0 = X0[b + lane] + O[b + lane], a1 = X0[b + lane + 32] + O[b + lane + 32];
  X1[b + lane] = a0; X1[b + lane + 32] = a1;
  float o0, o1;
  gt_ln(a0, a1, w.ln1_g, w.ln1_b, lane, o0, o1);
  gt_split_store(yh, yl, b + lane, o0); gt_split_store(yh, yl, b + lane + 32, o1);
}

// XS = (X1 + O2) * rowmask as fp16 hi/lo (input of W_ih)
__global__ void __launch_bounds__(256) gt_res_mask_kernel(size_t count, const float* __restrict__ X1, const float* __restrict__ O2,
                                                          const float* __restrict__ rowm, __half* __restrict__ sh, __half* __restrict__ sl) {
  cn_pdl_prologue();
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  gt_split_store(sh, sl, i, (X1[i] + O2[i]) * rowm[i >> 6]);
}

__device__ __forceinline__ float gt_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// LSTM cell.  gx row of (e, n) = gx_row0 + (e * gx_env_stride + n); masked update when fp != null (decoding).
__global__ void __launch_bounds__(256) gt_cell_kernel(int N, int H, const float* __restrict__ GX, int gx_env_stride, int gx_row0,
                                                      const float* __restrict__ GH, const float* __restrict__ fp,
                                                      float* __restrict__ h32, float* __restrict__ c32, __half* __restrict__ hh,
                                                      __half* __restrict__ hl) {
  cn_pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * H * 64) return;
  const int j = i & 63, rd = i >> 6, e = rd / H, n = rd - e * H;
  const float* gx = GX + ((size_t)gx_row0 + (size_t)e * gx_env_stride + n) * 256;
  const float* gh = GH + (size_t)rd * 256;
  const float ig = gt_sigmoid(gx[j] + gh[j]), fg = gt_sigmoid(gx[64 + j] + gh[64 + j]);
  const float gg = tanhf(gx[128 + j] + gh[128 + j]), og = gt_sigmoid(gx[192 + j] + gh[192 + j]);
  float c2 = fg * c32[i] + ig * gg, h2 = og * tanhf(c2);
  if (fp) {
    const float m = fp[rd];
    c2 = c2 * m + c32[i] * (1.0f - m);
    h2 = h2 * m + h32[i] * (1.0f - m);
  }
  c32[i] = c2; h32[i] = h2;
  gt_split_store(hh, hl, i, h2);
}

// after the observation period: h, c *= fp
__global__ void __launch_bounds__(256) gt_mask_state_kernel(int count, const float* __restrict__ fp, float* __restrict__ h32,
                                                            float* __restrict__ c32, __half* __restrict__ hh, __half* __restrict__ hl) {
  cn_pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float m = fp[i >> 6];
  const float h = h32[i] * m;
  h32[i] = h; c32[i] *= m;
  gt_split_store(hh, hl, i, h);
}

// hidden2pos (mean only) -> x_sample, cumulative mean, predicted world position of step tt
__global__ void __launch_bounds__(256) gt_h2p_kernel(GstTcW w, int Rd, int tt, const float* __restrict__ h32, const float* __restrict__ fp,
                                                     const float* __restrict__ pos_last, float* __restrict__ xin,
                                                     float* __restrict__ mu_cum, float* __restrict__ pred) {
  cn_pdl_prologue();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Rd * 2) return;
  const int n = i >> 1, d = i & 1;
  float a = w.bp[d];
  for (int k = 0; k < 64; ++k) a = fmaf(h32[(size_t)n * 64 + k], w.Wp[d * 64 + k], a);
  const float m = fp[n];
  xin[i] = a * m;
  const float cum = mu_cum[i] + a;
  mu_cum[i] = cum;
  pred[((size_t)n * GT_T + tt) * 2 + d] = (cum + pos_last[i]) * m + GT_INVALID * (1.0f - m);
}

// process_obs_rew tail: one CTA (32 threads) per environment
__global__ void __launch_bounds__(32) gt_final_kernel(int N, int H, int P, float thr, float collision_penalty,
                                                      const float* __restrict__ robot, const float* __restrict__ sp2,
                                                      const float* __restrict__ fp, const float* __restrict__ pred,
                                                      float* __restrict__ reward, float* __restrict__ penalty_out,
                                                      float* __restrict__ out_sp) {
  cn_pdl_prologue();
  const int e = blockIdx.x;
  const float rx = robot[e * 7], ry = robot[e * 7 + 1];
  float pen = 0.0f;
  for (int i = threadIdx.x; i < H * GT_T; i += 32) {
    const int n = i / GT_T, k = i - n * GT_T;
    if (k < P && fp[(size_t)e * H + n] != 0.0f) {
      const float dx = pred[((size_t)e * H * GT_T + i) * 2] - rx, dy = pred[((size_t)e * H * GT_T + i) * 2 + 1] - ry;
      if (sqrtf(dx * dx + dy * dy) < thr) pen = fminf(pen, collision_penalty / (float)(4 << k));
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) pen = fminf(pen, __shfl_xor_sync(0xffffffffu, pen, o));
  if (threadIdx.x == 0) {
    if (reward) reward[e] += pen;
    if (penalty_out) penalty_out[e] = pen;
  }
  const int W = 2 * (P + 1);
  for (int n = threadIdx.x; n < H; n += 32) {
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
    const bool ok = fp[(size_t)e * H + n] != 0.0f;
    for (int k = 0; k < P; ++k) {
      dst[2 + 2 * k] = ok ? pred[(((size_t)e * H + n) * GT_T + k) * 2] - rx : cx;
      dst[3 + 2 * k] = ok ? pred[(((size_t)e * H + n) * GT_T + k) * 2 + 1] - ry : cy;
    }
  }
}

// ==========================================================================================================
// COMPACT path (default).  Every row-wise quantity of the predictor is multiplied by a 0/1 mask: the node embedding by
// the row's input mask, attention weights by the query's and the key's mask (a masked query's output is exactly 0, a
// masked key has weight exactly 0), the encoder output by the row mask again before W_ih, the LSTM state by the
// "visible in the newest frame" flag fp after the observation period and in every decoding step, the prediction by fp.
// So a masked row carries constants (its Q|K|V row is the bias, its W_ih input is 0 -> its gate pre-activation is
// b_ih) and a human with fp = 0 carries nothing at all.  With the robot seeing ~4.4 of 20 humans, 78 % of the
// N*5*H observation rows and of the N*H decoding rows are such constants.  Here only the valid rows exist:
//   observation period: rows with mask 1, compacted in (env, frame) group order  (count counts[0], group g = e*5+t owns
//                       compact rows [gstart[g], gstart[g+1]))
//   LSTM + decoding:    humans with fp = 1, compacted in env order             (count counts[1], env e owns [estart[e], ..))
// The only place masked rows enter a valid row's arithmetic is the soft-max denominator (soft-max over ALL H neighbours,
// then mask and renormalise, mha.py:236-242): all masked keys share the key vector b_k, so their H - n terms are
// (H - n) * exp(q . b_k - max).  Results equal the dense path up to the order of that sum (~1e-9 relative).
#define GTC_WARPS 8

// one warp per (env, frame) group, lane = human: masks, masked input displacement, group counts, newest-frame bookkeeping
__global__ void __launch_bounds__(GTC_WARPS * 32) gtc_prep_kernel(int N, int H, float* __restrict__ ring_pos, uint8_t* __restrict__ ring_mask,
                                                                   int newest, const float* __restrict__ robot, const float* __restrict__ sp2,
                                                                   const uint8_t* __restrict__ vis, float* __restrict__ rowm,
                                                                   float* __restrict__ inp, int* __restrict__ gcount,
                                                                   int* __restrict__ ecount, float* __restrict__ fp,
                                                                   float* __restrict__ pos_last) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * GTC_WARPS + (threadIdx.x >> 5);
  if (g >= N * GT_T) return;
  const int e = g / GT_T, t = g - e * GT_T, n = lane;
  bool valid = false, vnow = false;
  if (n < H) {
    auto frame_pos = [&](int tt, float& x, float& y, float& m) {
      if (tt == GT_T - 1) {
        x = robot[e * 7] + sp2[((size_t)e * H + n) * 2];
        y = robot[e * 7 + 1] + sp2[((size_t)e * H + n) * 2 + 1];
        m = vis[(size_t)e * H + n] ? 1.0f : 0.0f;
      } else {
        const int slot = (newest + 1 + tt) % GT_T;
        const size_t o = ((size_t)slot * N + e) * H + n;
        x = ring_pos[2 * o]; y = ring_pos[2 * o + 1]; m = (float)ring_mask[o];
      }
    };
    float x, y, m, xp = 0, yp = 0, mp = 0, xl_, yl_, ml_;
    frame_pos(t, x, y, m);
    frame_pos(GT_T - 1, xl_, yl_, ml_);
    if (t > 0) frame_pos(t - 1, xp, yp, mp);
    const float mrel = t == 0 ? m : mp * ml_;                  // interface.forward:77-78 (sic)
    const float dx = t == 0 ? 0.0f : x - xp, dy = t == 0 ? 0.0f : y - yp;
    const size_t r = (size_t)g * H + n;
    rowm[r] = mrel;
    inp[2 * r] = GT_INVALID * (1.0f - mrel) + dx * mrel;
    inp[2 * r + 1] = GT_INVALID * (1.0f - mrel) + dy * mrel;
    valid = mrel != 0.0f;
    if (t == GT_T - 1) {
      const size_t rd = (size_t)e * H + n;
      fp[rd] = mrel; pos_last[2 * rd] = x; pos_last[2 * rd + 1] = y;
      vnow = valid;
    }
  }
  const uint32_t b = __ballot_sync(0xffffffffu, valid);
  if (lane == 0) gcount[g] = __popc(b);
  if (t == GT_T - 1) {
    const uint32_t bn = __ballot_sync(0xffffffffu, vnow);
    if (lane == 0) ecount[e] = __popc(bn);
    // traj_buffer.append / mask_buffer.append.  Other groups of this launch read the newest frame from the observation,
    // never from this slot (frame_pos), so the write cannot race with them.
    if (n < H) {
      const size_t o = ((size_t)newest * N + e) * H + n;
      ring_pos[2 * o] = robot[e * 7] + sp2[((size_t)e * H + n) * 2];
      ring_pos[2 * o + 1] = robot[e * 7 + 1] + sp2[((size_t)e * H + n) * 2 + 1];
      ring_mask[o] = vis[(size_t)e * H + n] ? 1 : 0;
    }
  }
}

// exclusive prefix sums of the group counts (G) and of the per-env visible counts (N); totals -> counts[0], counts[1]
__global__ void __launch_bounds__(1024) gtc_scan_kernel(const int* __restrict__ gcount, int G, int* __restrict__ gstart,
                                                        const int* __restrict__ ecount, int N, int* __restrict__ estart,
                                                        int* __restrict__ counts) {
  cn_pdl_prologue();
  __shared__ int part[1024];
  for (int pass = 0; pass < 2; ++pass) {
    const int* in = pass ? ecount : gcount;
    int* out = pass ? estart : gstart;
    const int L = pass ? N : G;
    const int per = (L + 1023) / 1024, b0 = threadIdx.x * per;
    int s = 0;
    for (int i = b0; i < b0 + per && i < L; ++i) s += in[i];
    part[threadIdx.x] = s;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {                      // Hillis-Steele inclusive scan of the 1024 partials
      const int v = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
      __syncthreads();
      part[threadIdx.x] += v;
      __syncthreads();
    }
    int run = part[threadIdx.x] - s;                          // exclusive
    for (int i = b0; i < b0 + per && i < L; ++i) { out[i] = run; run += in[i]; }
    if (threadIdx.x == 1023) { out[L] = part[1023]; counts[pass] = part[1023]; }
    __syncthreads();
  }
}

// compaction maps: cidx[r] (compact row or -1), crow[c] (source row), drow[d] (env * H + human of decode row d)
__global__ void __launch_bounds__(GTC_WARPS * 32) gtc_index_kernel(int N, int H, const float* __restrict__ rowm, const float* __restrict__ fp,
                                                                    const int* __restrict__ gstart, const int* __restrict__ estart,
                                                                    int* __restrict__ cidx, int* __restrict__ crow, int* __restrict__ drow) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * GTC_WARPS + (threadIdx.x >> 5);
  if (g >= N * GT_T) return;
  const int e = g / GT_T, t = g - e * GT_T;
  const size_t r = (size_t)g * H + lane;
  const bool valid = lane < H && rowm[r] != 0.0f;
  const uint32_t b = __ballot_sync(0xffffffffu, valid);
  const int c = gstart[g] + __popc(b & ((1u << lane) - 1u));
  if (lane < H) cidx[r] = valid ? c : -1;
  if (valid) crow[c] = (int)r;
  if (t == GT_T - 1) {
    const size_t rd = (size_t)e * H + lane;
    const bool vnow = lane < H && fp[rd] != 0.0f;
    const uint32_t bn = __ballot_sync(0xffffffffu, vnow);
    if (vnow) drow[estart[e] + __popc(bn & ((1u << lane) - 1u))] = (int)rd;
  }
}

// node embedding + norm_node of the compact rows (mask == 1).  src: crow (observation period, input from inp[row]) or
// null (decoding: input = xin[c]).  One warp per row, grid-stride.
__global__ void __launch_bounds__(256) gtc_embed_kernel(GstTcW w, const int* __restrict__ count, const int* __restrict__ src,
                                                        const float* __restrict__ in2, float* __restrict__ X0, __half* __restrict__ xh,
                                                        __half* __restrict__ xl) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31, C = cn_ld_after_wait(count);
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < C; c += (gridDim.x * blockDim.x) >> 5) {
    const int r = src ? src[c] : c;
    const float ix = in2[2 * (size_t)r], iy = in2[2 * (size_t)r + 1];
    const float e0 = fmaf(iy, w.We_t[64 + lane], fmaf(ix, w.We_t[lane], w.be[lane]));
    const float e1 = fmaf(iy, w.We_t[96 + lane], fmaf(ix, w.We_t[32 + lane], w.be[32 + lane]));
    float o0, o1;
    gt_ln(e0, e1, w.ln0_g, w.ln0_b, lane, o0, o1);
    const size_t b = (size_t)c * 64;
    X0[b + lane] = o0; X0[b + lane + 32] = o1;
    gt_split_store(xh, xl, b + lane, o0); gt_split_store(xh, xl, b + lane + 32, o1);
  }
}

// attention within a group's compact rows [start[g], start[g+1]); the H - n masked neighbours enter the soft-max
// denominator through their common key b_k (see the header of this section).  One CTA per group.
__global__ void __launch_bounds__(8 * GT_MAXH) gtc_attn_kernel(int H, const int* __restrict__ start, const float* __restrict__ qkv,
                                                               const float* __restrict__ bk /* b_in + 64 */, __half* __restrict__ ah,
                                                               __half* __restrict__ al) {
  cn_pdl_prologue();
  __shared__ __align__(16) float sq[GT_MAXH * 192];
  const int c0 = cn_ld_after_wait(start + blockIdx.x), ng = cn_ld_after_wait(start + blockIdx.x + 1) - c0;
  if (ng <= 0) return;
  for (int i = threadIdx.x; i < ng * 48; i += blockDim.x)
    reinterpret_cast<float4*>(sq)[i] = __ldg(reinterpret_cast<const float4*>(qkv + (size_t)c0 * 192) + i);
  __syncthreads();
  const int lr = threadIdx.x >> 3, hd = threadIdx.x & 7;
  if (lr >= ng) return;
  const float scaling = 0.35355339059327373f;
  float q[8];
#pragma unroll
  for (int d = 0; d < 8; ++d) q[d] = sq[lr * 192 + hd * 8 + d] * scaling;
  const int nmask = H - ng;
  float sm = 0.0f;
#pragma unroll
  for (int d = 0; d < 8; ++d) sm = fmaf(q[d], __ldg(bk + hd * 8 + d), sm);
  float mx = nmask > 0 ? sm : -INFINITY;
  for (int j = 0; j < ng; ++j) {
    const float* kj = sq + j * 192 + 64 + hd * 8;
    float s = 0.0f;
#pragma unroll
    for (int d = 0; d < 8; ++d) s = fmaf(q[d], kj[d], s);
    mx = fmaxf(mx, s);
  }
  float den = 0.0f, dm = 0.0f, o[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < ng; ++j) {
    const float* kj = sq + j * 192 + 64 + hd * 8;
    const float* vj = sq + j * 192 + 128 + hd * 8;
    float s = 0.0f;
#pragma unroll
    for (int d = 0; d < 8; ++d) s = fmaf(q[d], kj[d], s);
    const float ex = expf(s - mx);
    den += ex;
    dm += ex;
#pragma unroll
    for (int d = 0; d < 8; ++d) o[d] = fmaf(ex, vj[d], o[d]);
  }
  if (nmask > 0) den += (float)nmask * expf(sm - mx);
  const float scale = (1.0f / den) / (dm / den + 1e-10f);
  const size_t ob = (size_t)(c0 + lr) * 64 + hd * 8;
#pragma unroll
  for (int d = 0; d < 8; ++d) gt_split_store(ah, al, ob + d, o[d] * scale);
}

// X1 = X0 + O, Y = norm1(X1) (compact rows, grid-stride)
__global__ void __launch_bounds__(256) gtc_res_ln_kernel(GstTcW w, const int* __restrict__ count, const float* __restrict__ X0,
                                                         const float* __restrict__ O, float* __restrict__ X1, __half* __restrict__ yh,
                                                         __half* __restrict__ yl) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31, C = cn_ld_after_wait(count);
  for (int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < C; c += (gridDim.x * blockDim.x) >> 5) {
    const size_t b = (size_t)c * 64;
    const float a0 = X0[b + lane] + O[b + lane], a1 = X0[b + lane + 32] + O[b + lane + 32];
    X1[b + lane] = a0; X1[b + lane + 32] = a1;
    float o0, o1;
    gt_ln(a0, a1, w.ln1_g, w.ln1_b, lane, o0, o1);
    gt_split_store(yh, yl, b + lane, o0); gt_split_store(yh, yl, b + lane + 32, o1);
  }
}

// XS = X1 + O2 (row mask == 1) as fp16 hi / lo
__global__ void __launch_bounds__(256) gtc_res_kernel(const int* __restrict__ count, const float* __restrict__ X1,
                                                      const float* __restrict__ O2, __half* __restrict__ sh, __half* __restrict__ sl) {
  cn_pdl_prologue();
  const size_t total = (size_t)cn_ld_after_wait(count) * 64;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x)
    gt_split_store(sh, sl, i, X1[i] + O2[i]);
}

// LSTM cell over the compact decode rows.  t >= 0: observation frame t, the row's gate input is GX[cidx] or, when that
// frame of the human is masked, the constant b_ih;  t < 0: decoding, gate input GX[d].  Also initialises (t == 0).
__global__ void __launch_bounds__(256) gtc_cell_kernel(int H, int t, const int* __restrict__ count, const int* __restrict__ drow,
                                                       const int* __restrict__ cidx, const float* __restrict__ GX,
                                                       const float* __restrict__ bih, const float* __restrict__ bhh,
                                                       const float* __restrict__ GH, float* __restrict__ h32,
                                                       float* __restrict__ c32, __half* __restrict__ hh, __half* __restrict__ hl) {
  cn_pdl_prologue();
  const size_t total = (size_t)cn_ld_after_wait(count) * 64;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int j = (int)(i & 63);
    const size_t d = i >> 6;
    const float* gx;
    if (t >= 0) {
      const int rd = drow[d], e = rd / H, n = rd - e * H;
      const int c = cidx[((size_t)e * GT_T + t) * H + n];
      gx = c >= 0 ? GX + (size_t)c * 256 : bih;
    } else {
      gx = GX + d * 256;
    }
    const float* gh = t == 0 ? bhh : GH + d * 256;            // h0 = 0: W_hh h + b_hh = b_hh
    const float cprev = t == 0 ? 0.0f : c32[i];
    const float ig = gt_sigmoid(gx[j] + gh[j]), fg = gt_sigmoid(gx[64 + j] + gh[64 + j]);
    const float gg = tanhf(gx[128 + j] + gh[128 + j]), og = gt_sigmoid(gx[192 + j] + gh[192 + j]);
    const float c2 = fg * cprev + ig * gg, h2 = og * tanhf(c2);
    c32[i] = c2; h32[i] = h2;
    gt_split_store(hh, hl, i, h2);
  }
}

// hidden2pos (mean only) of the compact decode rows -> next input, cumulative mean, predicted world position
__global__ void __launch_bounds__(256) gtc_h2p_kernel(GstTcW w, int tt, const int* __restrict__ count, const int* __restrict__ drow,
                                                      const float* __restrict__ h32, const float* __restrict__ pos_last,
                                                      float* __restrict__ xin, float* __restrict__ mu_cum, float* __restrict__ pred) {
  cn_pdl_prologue();
  const int total = cn_ld_after_wait(count) * 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int d = i >> 1, dim = i & 1, rd = drow[d];
    float a = w.bp[dim];
    for (int k = 0; k < 64; ++k) a = fmaf(h32[(size_t)d * 64 + k], w.Wp[dim * 64 + k], a);
    xin[i] = a;
    const float cum = (tt == 0 ? 0.0f : mu_cum[i]) + a;
    mu_cum[i] = cum;
    pred[((size_t)rd * GT_T + tt) * 2 + dim] = cum + pos_last[2 * (size_t)rd + dim];
  }
}

struct GstTc {
  CnLaunchCtx ctx;
  int N, H, P;
  float thr, pen;
  GstTcW w;
  TcMat tWin, tWout, tW1, tW2, tWih, tWhh;                   // weights (x 2^6, fp16 hi/lo)
  TcMat tX, tA, tY, tF, tXS, tHd;                            // activations (fp16 hi/lo A operands)
  float *X0, *QKV, *O, *X1, *GX, *GH, *rowm, *fp, *pos_last, *h32, *c32, *mu_cum, *xin, *pred;
  TcStoreMap GX_R, GX_Rd, GH_Rd;                             // store maps of the BN = 256 gate GEMMs' outputs, per row extent
  // compact path (cn_gst_tcc_step): only rows whose mask is 1 are computed
  float* inp;                                                // [R, 2] masked input displacement of every (env, frame, human) row
  int *cidx, *crow, *gcount, *gstart, *ecount, *estart, *drow, *counts;   // compaction maps (see gtc_* kernels)
};

int gt_upload(CnLaunchCtx* ctx, const float** dst, const float* src, size_t count) {
  float* q = nullptr;
  int rc = palloc(ctx, &q, count);
  if (rc) return rc;
  if (cudaMemcpy(q, src, count * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return cn_set_error("gst tc: H2D failed");
  *dst = q;
  return 0;
}

}  // namespace

// C++ entry points used by cn_gst.cu (not part of the public C ABI)
void* cn_gst_tc_create(int N, int H, int P, float thr, float pen, int device, const float* const* host /* 20 params, cn_gst.cu order, */,
                       const int* rows, const int* cols) {
  cudaSetDevice(device);
  GstTc* g = new GstTc();
  CnLaunchCtx* ctx = &g->ctx;
  cn_launch_init(ctx, device);
  g->N = N; g->H = H; g->P = P; g->thr = thr; g->pen = pen;
  int rc = tc_set_attrs();
  // indices in cn_gst.cu's kParamNames: 0 We 1 be 2 ln0g 3 ln0b 4 Win 5 bin 6 Wout 7 bout 8 ln1g 9 ln1b 10 W1 11 b1 12 W2 13 b2
  //                                     14 Wih 15 bih 16 Whh 17 bhh 18 Wp 19 bp
  std::vector<float> wet(128);
  for (int c = 0; c < 64; ++c) { wet[c] = host[0][c * 2]; wet[64 + c] = host[0][c * 2 + 1]; }     // [64][2] -> [2][64]
  if (!rc) rc = gt_upload(ctx, &g->w.We_t, wet.data(), 128);
  const float** fdst[] = {&g->w.be, &g->w.ln0_g, &g->w.ln0_b, &g->w.bin, &g->w.bout, &g->w.ln1_g, &g->w.ln1_b, &g->w.b1, &g->w.b2,
                          &g->w.bih, &g->w.bhh, &g->w.Wp, &g->w.bp};
  const int fidx[] = {1, 2, 3, 5, 7, 8, 9, 11, 13, 15, 17, 18, 19};
  for (int i = 0; i < 13 && !rc; ++i) rc = gt_upload(ctx, fdst[i], host[fidx[i]], (size_t)rows[fidx[i]] * cols[fidx[i]]);
  struct { int idx; TcMat* t; } tw[6] = {{4, &g->tWin}, {6, &g->tWout}, {10, &g->tW1}, {12, &g->tW2}, {14, &g->tWih}, {16, &g->tWhh}};
  for (int i = 0; i < 6 && !rc; ++i) {
    const int r = rows[tw[i].idx], k = cols[tw[i].idx];
    const float* d = nullptr;
    rc = gt_upload(ctx, &d, host[tw[i].idx], (size_t)r * k);
    const int bn = r == 256 ? 256 : 64;                                       // the 256-wide gate GEMMs use BN = 256 tiles
    if (!rc) rc = tc_alloc(ctx, *tw[i].t, r, k, bn, tc_box_k(bn));
    if (!rc) split16(ctx, 0, d, 64.0f, tw[i].t->hi, tw[i].t->lo, (size_t)r * k);
  }
  const size_t R = (size_t)N * GT_T * H, Rd = (size_t)N * H;
  if (!rc) rc = tc_alloc(ctx, g->tX, (int)R, 64, TC_BM, tc_box_k(64));
  if (!rc) rc = tc_alloc(ctx, g->tA, (int)R, 64, TC_BM, tc_box_k(64));
  if (!rc) rc = tc_alloc(ctx, g->tY, (int)R, 64, TC_BM, tc_box_k(64));
  if (!rc) rc = tc_alloc(ctx, g->tF, (int)R, 128, TC_BM, tc_box_k(64));
  if (!rc) rc = tc_alloc(ctx, g->tXS, (int)R, 64, TC_BM, tc_box_k(256));     // A of the BN = 256 gate GEMMs
  if (!rc) rc = tc_alloc(ctx, g->tHd, (int)Rd, 64, TC_BM, tc_box_k(256));
#define GA(name, count) if (!rc) rc = palloc(ctx, &g->name, (count))
  GA(X0, R * 64); GA(QKV, R * 192); GA(O, R * 64); GA(X1, R * 64); GA(GX, R * 256); GA(GH, Rd * 256); GA(rowm, R); GA(fp, Rd);
  GA(pos_last, Rd * 2); GA(h32, Rd * 64); GA(c32, Rd * 64); GA(mu_cum, Rd * 2); GA(xin, Rd * 2); GA(pred, Rd * GT_T * 2);
  GA(inp, R * 2);
#undef GA
  // the encoder runs over all R observation rows and over the Rd rows of the newest frame: one GX map per row extent
  if (!rc) rc = make_store_map(&g->GX_R, g->GX, 4, (int)R, 256, 256);
  if (!rc) rc = make_store_map(&g->GX_Rd, g->GX, 4, (int)Rd, 256, 256);
  if (!rc) rc = make_store_map(&g->GH_Rd, g->GH, 4, (int)Rd, 256, 256);
#define GI(name, count) if (!rc) { float* q_ = nullptr; rc = palloc(ctx, &q_, (count)); g->name = reinterpret_cast<int*>(q_); }
  GI(cidx, R); GI(crow, R); GI(gcount, (size_t)N * GT_T); GI(gstart, (size_t)N * GT_T + 1); GI(ecount, N); GI(estart, N + 1);
  GI(drow, Rd); GI(counts, 4);
#undef GI
  if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = cn_set_error("gst tc: setup failed");
  if (rc) { return nullptr; }
  return g;
}

void cn_gst_tc_destroy(void* handle) {
  GstTc* g = static_cast<GstTc*>(handle);
  if (!g) return;
  cn_launch_free(&g->ctx);
  delete g;
}

int64_t cn_gst_tc_launches(void* handle) { return handle ? static_cast<GstTc*>(handle)->ctx.launches : 0; }

int cn_gst_tc_step(void* handle, float* ring_pos, uint8_t* ring_mask, int newest, const float* robot, const float* sp2,
                   const uint8_t* vis, float* reward, float* penalty, float* out_sp, cudaStream_t st) {
  GstTc* g = static_cast<GstTc*>(handle);
  CnLaunchCtx* p = &g->ctx;
  const int N = g->N, H = g->H;
  const int R = N * GT_T * H, Rd = N * H;
  auto warps = [](int rows) { return dim3((unsigned)((rows + 7) / 8)); };          // 8 warps (rows) per 256-thread CTA
  auto encoder = [&](int rows, const float* rowm) {
    gemm_tc(p, st, g->tX, g->tWin, rows, 192, 64, 64, g->w.bin, CN_ACT_NONE, out32(g->QKV, 192));
    launch_k(p, gt_attn_kernel, dim3((unsigned)(rows / H)), dim3((unsigned)(8 * H)), 0, st, rows, H, g->QKV, rowm, g->tA.hi, g->tA.lo);
    gemm_tc(p, st, g->tA, g->tWout, rows, 64, 64, 64, g->w.bout, CN_ACT_NONE, out32(g->O, 64));
    launch_k(p, gt_res_ln_kernel, warps(rows), dim3(256), 0, st, g->w, rows, g->X0, g->O, g->X1, g->tY.hi, g->tY.lo);
    gemm_tc(p, st, g->tY, g->tW1, rows, 128, 64, 64, g->w.b1, CN_ACT_RELU, out16(g->tF));
    gemm_tc(p, st, g->tF, g->tW2, rows, 64, 128, 64, g->w.b2, CN_ACT_NONE, out32(g->O, 64));
    launch_k(p, gt_res_mask_kernel, dim3((unsigned)(((size_t)rows * 64 + 255) / 256)), dim3(256), 0, st, (size_t)rows * 64, g->X1, g->O,
             rowm, g->tXS.hi, g->tXS.lo);
    gemm_tc(p, st, g->tXS, g->tWih, rows, 256, 64, 256, g->w.bih, CN_ACT_NONE, out32(g->GX, 256, rows == R ? &g->GX_R : &g->GX_Rd));
  };
  launch_k(p, gt_prep_kernel, warps(R), dim3(256), 0, st, g->w, N, H, ring_pos, ring_mask, newest, robot, sp2, vis, g->X0, g->tX.hi,
           g->tX.lo, g->rowm, g->fp, g->pos_last, g->h32, g->tHd.hi, g->tHd.lo, g->c32, g->mu_cum);
  encoder(R, g->rowm);
  const unsigned cell_grid = (unsigned)((Rd * 64 + 255) / 256);
  for (int t = 0; t < GT_T; ++t) {
    gemm_tc(p, st, g->tHd, g->tWhh, Rd, 256, 64, 256, g->w.bhh, CN_ACT_NONE, out32(g->GH, 256, &g->GH_Rd));
    launch_k(p, gt_cell_kernel, dim3(cell_grid), dim3(256), 0, st, N, H, g->GX, GT_T * H, t * H, g->GH, (const float*)nullptr, g->h32,
             g->c32, g->tHd.hi, g->tHd.lo);
  }
  launch_k(p, gt_mask_state_kernel, dim3(cell_grid), dim3(256), 0, st, Rd * 64, g->fp, g->h32, g->c32, g->tHd.hi, g->tHd.lo);
  for (int tt = 0; tt < GT_T; ++tt) {
    if (tt > 0) {
      launch_k(p, gt_embed_kernel, warps(Rd), dim3(256), 0, st, g->w, Rd, g->xin, g->fp, g->X0, g->tX.hi, g->tX.lo);
      encoder(Rd, g->fp);
      gemm_tc(p, st, g->tHd, g->tWhh, Rd, 256, 64, 256, g->w.bhh, CN_ACT_NONE, out32(g->GH, 256, &g->GH_Rd));
      launch_k(p, gt_cell_kernel, dim3(cell_grid), dim3(256), 0, st, N, H, g->GX, H, 0, g->GH, g->fp, g->h32, g->c32, g->tHd.hi,
               g->tHd.lo);
    }
    launch_k(p, gt_h2p_kernel, dim3((unsigned)((Rd * 2 + 255) / 256)), dim3(256), 0, st, g->w, Rd, tt, g->h32, g->fp, g->pos_last, g->xin,
             g->mu_cum, g->pred);
  }
  launch_k(p, gt_final_kernel, dim3((unsigned)N), dim3(32), 0, st, N, H, g->P, g->thr, g->pen, robot, sp2, g->fp, g->pred, reward, penalty,
           out_sp);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("gst tc step: %s", cudaGetErrorString(err));
  if (p->launch_error) { p->launch_error = false; return 1; }
  return 0;
}

// Compact variant of cn_gst_tc_step (default): same outputs, only the valid rows are computed.
int cn_gst_tcc_step(void* handle, float* ring_pos, uint8_t* ring_mask, int newest, const float* robot, const float* sp2,
                    const uint8_t* vis, float* reward, float* penalty, float* out_sp, cudaStream_t st) {
  GstTc* g = static_cast<GstTc*>(handle);
  CnLaunchCtx* p = &g->ctx;
  const int N = g->N, H = g->H;
  const int R = N * GT_T * H, Rd = N * H, G = N * GT_T;
  p->dbg_launch_idx = 0;
  const int* cntR = g->counts;          // valid observation rows
  const int* cntD = g->counts + 1;      // humans visible in the newest frame
  const dim3 rows_grid((unsigned)(p->num_sms * 4)), grp_grid((unsigned)((G + GTC_WARPS - 1) / GTC_WARPS));
  auto encoder = [&](int maxrows, const int* cnt, int groups, const int* start) {
    gemm_tc(p, st, g->tX, g->tWin, maxrows, 192, 64, 64, g->w.bin, CN_ACT_NONE, out32(g->QKV, 192), cnt);
    launch_k(p, gtc_attn_kernel, dim3((unsigned)groups), dim3((unsigned)(8 * H)), 0, st, H, start, g->QKV, g->w.bin + 64, g->tA.hi, g->tA.lo);
    gemm_tc(p, st, g->tA, g->tWout, maxrows, 64, 64, 64, g->w.bout, CN_ACT_NONE, out32(g->O, 64), cnt);
    launch_k(p, gtc_res_ln_kernel, rows_grid, dim3(256), 0, st, g->w, cnt, g->X0, g->O, g->X1, g->tY.hi, g->tY.lo);
    gemm_tc(p, st, g->tY, g->tW1, maxrows, 128, 64, 64, g->w.b1, CN_ACT_RELU, out16(g->tF), cnt);
    gemm_tc(p, st, g->tF, g->tW2, maxrows, 64, 128, 64, g->w.b2, CN_ACT_NONE, out32(g->O, 64), cnt);
    launch_k(p, gtc_res_kernel, rows_grid, dim3(256), 0, st, cnt, g->X1, g->O, g->tXS.hi, g->tXS.lo);
    gemm_tc(p, st, g->tXS, g->tWih, maxrows, 256, 64, 256, g->w.bih, CN_ACT_NONE,
            out32(g->GX, 256, maxrows == R ? &g->GX_R : &g->GX_Rd), cnt);
  };
  launch_k(p, gtc_prep_kernel, grp_grid, dim3(GTC_WARPS * 32), 0, st, N, H, ring_pos, ring_mask, newest, robot, sp2, vis, g->rowm, g->inp,
           g->gcount, g->ecount, g->fp, g->pos_last);
  launch_k(p, gtc_scan_kernel, dim3(1), dim3(1024), 0, st, g->gcount, G, g->gstart, g->ecount, N, g->estart, g->counts);
  launch_k(p, gtc_index_kernel, grp_grid, dim3(GTC_WARPS * 32), 0, st, N, H, g->rowm, g->fp, g->gstart, g->estart, g->cidx, g->crow,
           g->drow);
  launch_k(p, gtc_embed_kernel, rows_grid, dim3(256), 0, st, g->w, cntR, g->crow, g->inp, g->X0, g->tX.hi, g->tX.lo);
  encoder(R, cntR, G, g->gstart);
  // LSTM over the 5 observed frames, humans visible now only (h0 = c0 = 0: frame 0 has no recurrent GEMM, its
  // hidden-state gate term is b_hh)
  for (int t = 0; t < GT_T; ++t) {
    if (t > 0) gemm_tc(p, st, g->tHd, g->tWhh, Rd, 256, 64, 256, g->w.bhh, CN_ACT_NONE, out32(g->GH, 256, &g->GH_Rd), cntD);
    launch_k(p, gtc_cell_kernel, rows_grid, dim3(256), 0, st, H, t, cntD, g->drow, g->cidx, g->GX, g->w.bih, g->w.bhh, g->GH, g->h32,
             g->c32, g->tHd.hi, g->tHd.lo);
  }
  for (int tt = 0; tt < GT_T; ++tt) {
    if (tt > 0) {
      launch_k(p, gtc_embed_kernel, rows_grid, dim3(256), 0, st, g->w, cntD, (const int*)nullptr, g->xin, g->X0, g->tX.hi, g->tX.lo);
      encoder(Rd, cntD, N, g->estart);
      gemm_tc(p, st, g->tHd, g->tWhh, Rd, 256, 64, 256, g->w.bhh, CN_ACT_NONE, out32(g->GH, 256, &g->GH_Rd), cntD);
      launch_k(p, gtc_cell_kernel, rows_grid, dim3(256), 0, st, H, -1, cntD, g->drow, g->cidx, g->GX, g->w.bih, g->w.bhh, g->GH, g->h32,
               g->c32, g->tHd.hi, g->tHd.lo);
    }
    launch_k(p, gtc_h2p_kernel, rows_grid, dim3(256), 0, st, g->w, tt, cntD, g->drow, g->h32, g->pos_last, g->xin, g->mu_cum, g->pred);
  }
  launch_k(p, gt_final_kernel, dim3((unsigned)N), dim3(32), 0, st, N, H, g->P, g->thr, g->pen, robot, sp2, g->fp, g->pred, reward, penalty,
           out_sp);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("gst tcc step: %s", cudaGetErrorString(err));
  if (p->launch_error) { p->launch_error = false; return 1; }
  return 0;
}
