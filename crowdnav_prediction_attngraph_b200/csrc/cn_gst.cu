// BASELINE config 3 (SURVEY.md row a16): the GST trajectory predictor and the VecPretextNormalize processing.
//
//   reference: rl/vec_env/vec_pretext_normalize.py:85-191 (traj / mask deques, process_obs_rew),
//              gst_updated/scripts/wrapper/crowd_nav_interface_parallel.py:45-114 (input masks, cumsum of mu),
//              gst_updated/src/gumbel_social_transformer/st_model.py:271-455 + node_encoder_layer_no_ghost.py +
//              mha.py:236-242 for the shipped predictor configuration (full connectivity, one 8-head layer,
//              'faster_lstm', recursive decoding, sampling=False).
//
// Every dense layer is a batched [rows, K] GEMM over ALL environments on the wgmma 3xFP16 GEMM (cn_gemm_tc.h), over
// the rows whose mask is 1 only (see the compact-row comment below), and small row-wise kernels do embedding +
// LayerNorm, the H x H attention, residuals, the LSTM cell and the wrapper's tail: future-collision penalty added to the
// reward, predicted relative positions written into the 2(P+1)-wide spatial_edges rows, rows sorted by distance to the
// robot.  The launches of one step form a chain with programmatic dependent launch (cn_launch.cuh).
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <map>
#include <string>
#include <vector>

#include "../../include/crowdnav_b200.h"
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

__device__ __forceinline__ float gt_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

#define GT_MAXH 128   // humans per environment (max_human_num), as in the environment and the policy

// process_obs_rew tail: one CTA per environment, one thread per human (32 * ceil(H / 32) threads).  The distance keys
// are computed once into shared memory; a row's rank counts the closer rows and the equally close rows of lower index.
__global__ void __launch_bounds__(GT_MAXH) gt_final_kernel(int N, int H, int P, float thr, float collision_penalty,
                                                           const float* __restrict__ robot, const float* __restrict__ sp2,
                                                           const float* __restrict__ fp, const float* __restrict__ pred,
                                                           float* __restrict__ reward, float* __restrict__ penalty_out,
                                                           float* __restrict__ out_sp) {
  cn_pdl_prologue();
  __shared__ float skey[GT_MAXH], spen[GT_MAXH / 32];
  const int e = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const float rx = robot[e * 7], ry = robot[e * 7 + 1];
  float pen = 0.0f;
  for (int i = threadIdx.x; i < H * GT_T; i += blockDim.x) {
    const int n = i / GT_T, k = i - n * GT_T;
    if (k < P && fp[(size_t)e * H + n] != 0.0f) {
      const float dx = pred[((size_t)e * H * GT_T + i) * 2] - rx, dy = pred[((size_t)e * H * GT_T + i) * 2 + 1] - ry;
      if (sqrtf(dx * dx + dy * dy) < thr) pen = fminf(pen, collision_penalty / (float)(4 << k));
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) pen = fminf(pen, __shfl_xor_sync(0xffffffffu, pen, o));
  if (lane == 0) spen[warp] = pen;
  for (int n = threadIdx.x; n < H; n += blockDim.x) {
    const float cx = sp2[((size_t)e * H + n) * 2], cy = sp2[((size_t)e * H + n) * 2 + 1];
    skey[n] = sqrtf(cx * cx + cy * cy);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < nw; ++w) pen = fminf(pen, spen[w]);
    if (reward) reward[e] += pen;
    if (penalty_out) penalty_out[e] = pen;
  }
  const int W = 2 * (P + 1);
  for (int n = threadIdx.x; n < H; n += blockDim.x) {
    const float cx = sp2[((size_t)e * H + n) * 2], cy = sp2[((size_t)e * H + n) * 2 + 1];
    const float key = skey[n];
    int rank = 0;
    for (int j = 0; j < H; ++j) {
      const float kj = skey[j];
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
// Compact rows.  Every row-wise quantity of the predictor is multiplied by a 0/1 mask: the node embedding by
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
// (H - n) * exp(q . b_k - max).  Results equal a computation over every row up to the order of that sum (~1e-9
// relative).  gtc_attn_kernel stages the Q|K|V rows of one group in dynamic shared memory: H * 768 bytes, 96 KB at
// GT_MAXH = 128 humans.
#define GTC_WARPS 8

// one warp per (env, frame) group, humans in chunks of 32 (lane = human - n0): masks, masked input displacement, group
// counts, newest-frame bookkeeping
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
  const int e = g / GT_T, t = g - e * GT_T;
  int gc = 0, ec = 0;
  for (int n0 = 0; n0 < H; n0 += 32) {
    const int n = n0 + lane;
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
    gc += __popc(__ballot_sync(0xffffffffu, valid));
    if (t == GT_T - 1) {
      ec += __popc(__ballot_sync(0xffffffffu, vnow));
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
  if (lane == 0) {
    gcount[g] = gc;
    if (t == GT_T - 1) ecount[e] = ec;
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

// compaction maps: cidx[r] (compact row or -1), crow[c] (source row), drow[d] (env * H + human of decode row d).  One
// warp per (env, frame) group, humans in chunks of 32 with a running offset: compact rows stay in ascending row order.
__global__ void __launch_bounds__(GTC_WARPS * 32) gtc_index_kernel(int N, int H, const float* __restrict__ rowm, const float* __restrict__ fp,
                                                                    const int* __restrict__ gstart, const int* __restrict__ estart,
                                                                    int* __restrict__ cidx, int* __restrict__ crow, int* __restrict__ drow) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * GTC_WARPS + (threadIdx.x >> 5);
  if (g >= N * GT_T) return;
  const int e = g / GT_T, t = g - e * GT_T;
  const uint32_t below = (1u << lane) - 1u;
  int c0 = cn_ld_after_wait(gstart + g), d0 = t == GT_T - 1 ? cn_ld_after_wait(estart + e) : 0;
  for (int n0 = 0; n0 < H; n0 += 32) {
    const int n = n0 + lane;
    const size_t r = (size_t)g * H + n;
    const bool valid = n < H && rowm[r] != 0.0f;
    const uint32_t b = __ballot_sync(0xffffffffu, valid);
    const int c = c0 + __popc(b & below);
    if (n < H) cidx[r] = valid ? c : -1;
    if (valid) crow[c] = (int)r;
    c0 += __popc(b);
    if (t == GT_T - 1) {
      const size_t rd = (size_t)e * H + n;
      const bool vnow = n < H && fp[rd] != 0.0f;
      const uint32_t bn = __ballot_sync(0xffffffffu, vnow);
      if (vnow) drow[d0 + __popc(bn & below)] = (int)rd;
      d0 += __popc(bn);
    }
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
// denominator through their common key b_k (see the header of this section).  One CTA of 8 * H threads per group, one
// thread per (row, head); H * 192 floats of dynamic shared memory.
__global__ void __launch_bounds__(8 * GT_MAXH) gtc_attn_kernel(int H, const int* __restrict__ start, const float* __restrict__ qkv,
                                                               const float* __restrict__ bk /* b_in + 64 */, __half* __restrict__ ah,
                                                               __half* __restrict__ al) {
  cn_pdl_prologue();
  extern __shared__ __align__(16) float sq[];
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
const int kNumParams = 20;

int gt_upload(CnLaunchCtx* ctx, const float** dst, const float* src, size_t count) {
  float* q = nullptr;
  int rc = palloc(ctx, &q, count);
  if (rc) return rc;
  if (cudaMemcpy(q, src, count * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return cn_set_error("cn_gst_finalize: H2D failed");
  *dst = q;
  return 0;
}

}  // namespace

struct cn_gst {
  CnLaunchCtx ctx;
  size_t ws_allocs;   // ctx.allocs[0..ws_allocs) = ring buffers + workspace (kept); the rest = parameters of the last finalize
  int N, H, P, device;
  float thr, collision_penalty;
  std::map<std::string, std::vector<float>> host;
  bool finalized;
  float* ring_pos;    // [5][N][H][2] traj_buffer
  uint8_t* ring_mask; // [5][N][H] mask_buffer
  int newest;         // ring slot of the most recent frame
  GstTcW w;
  TcMat tWin, tWout, tW1, tW2, tWih, tWhh;                   // weights (x 2^6, fp16 hi/lo)
  TcMat tX, tA, tY, tF, tXS, tHd;                            // activations (fp16 hi/lo A operands)
  float *X0, *QKV, *O, *X1, *GX, *GH, *rowm, *fp, *pos_last, *h32, *c32, *mu_cum, *xin, *pred;
  TcStoreMap GX_R, GX_Rd, GH_Rd;                             // store maps of the BN = 256 gate GEMMs' outputs, per row extent
  float* inp;                                                // [R, 2] masked input displacement of every (env, frame, human) row
  int *cidx, *crow, *gcount, *gstart, *ecount, *estart, *drow, *counts;   // compaction maps (see gtc_* kernels)
  std::string stop_after;   // cn_internal_gst_stop_after: the next cn_gst_step returns after this stage (empty: never)
};

namespace {

// Stages of one cn_gst_step in launch order, as cn_internal_gst_stop_after names them.  An encoder pass ("obs." over the
// observation rows, "decK." in decoding step K = 1..4) is embed, qkv, attn, out, res_ln, ffn1, ffn2, res, gx; "lstmT"
// is the LSTM cell of observed frame T (after its recurrent GEMM for T > 0); a decoding step K >= 1 continues with gh,
// cell, h2p; "final" is the penalty / sort / write-out.
std::vector<std::string> gst_stage_names() {
  static const char* enc[] = {"embed", "qkv", "attn", "out", "res_ln", "ffn1", "ffn2", "res", "gx"};
  std::vector<std::string> s = {"prep", "scan", "index"};
  for (const char* e : enc) s.push_back(std::string("obs.") + e);
  for (int t = 0; t < GT_T; ++t) s.push_back("lstm" + std::to_string(t));
  s.push_back("dec0.h2p");
  for (int k = 1; k < GT_T; ++k) {
    const std::string p = "dec" + std::to_string(k) + ".";
    for (const char* e : enc) s.push_back(p + e);
    for (const char* e : {"gh", "cell", "h2p"}) s.push_back(p + e);
  }
  s.push_back("final");
  return s;
}

}  // namespace

extern "C" {

int cn_gst_destroy(cn_gst* g) {
  if (!g) return 0;
  cudaSetDevice(g->device);
  cudaDeviceSynchronize();
  cn_launch_free(&g->ctx);
  delete g;
  return 0;
}

int cn_gst_create(int num_envs, int human_num, int predict_steps, double robot_radius, double human_radius,
                  double collision_penalty, int device, cn_gst** out) {
  if (!out) return cn_set_error("cn_gst_create: null argument");
  *out = nullptr;
  if (num_envs <= 0 || human_num <= 0 || human_num > GT_MAXH || predict_steps < 1 || predict_steps > GT_T)
    return cn_set_error("cn_gst_create: need num_envs > 0, 1 <= human_num <= %d and 1 <= predict_steps <= %d (got %d, %d, %d)",
                        GT_MAXH, GT_T, num_envs, human_num, predict_steps);
  int ndev = 0;
  cudaError_t err = cudaGetDeviceCount(&ndev);
  if (err != cudaSuccess || ndev == 0)
    return cn_set_error("cn_gst_create: no CUDA device (%s); this engine has no CPU fallback",
                        err == cudaSuccess ? "device count 0" : cudaGetErrorString(err));
  if (device < 0 || device >= ndev) return cn_set_error("cn_gst_create: bad device %d", device);
  cudaSetDevice(device);
  cn_gst* g = new cn_gst();
  g->N = num_envs; g->H = human_num; g->P = predict_steps; g->device = device;
  g->thr = (float)(robot_radius + human_radius); g->collision_penalty = (float)collision_penalty;
  g->newest = GT_T - 1; g->finalized = false;
  CnLaunchCtx* ctx = &g->ctx;
  cn_launch_init(ctx, device);
  int rc = tc_set_attrs();
  if (!rc && cudaFuncSetAttribute(gtc_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GT_MAXH * 192 * (int)sizeof(float)) !=
                 cudaSuccess)
    rc = cn_set_error("cn_gst_create: shared memory attribute of the attention kernel failed");
  // workspace, sized for every row although only the live ones are used: 4125 bytes per observation row (R = N * 5 * H:
  // fp32 X0 | QKV | O | X1 | GX, the split fp16 A operands, ring, masks, inputs, maps) + ~1.9 KB per decode row (N * H),
  // 9.2 GB at N = 4096, H = 100
  const size_t R = (size_t)num_envs * GT_T * human_num, Rd = (size_t)num_envs * human_num;
  float* q = nullptr;
  if (!rc) rc = palloc(ctx, &g->ring_pos, R * 2);
  if (!rc) rc = palloc(ctx, &q, (R + 3) / 4);
  g->ring_mask = reinterpret_cast<uint8_t*>(q);
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
  GI(cidx, R); GI(crow, R); GI(gcount, (size_t)num_envs * GT_T); GI(gstart, (size_t)num_envs * GT_T + 1); GI(ecount, num_envs);
  GI(estart, num_envs + 1); GI(drow, Rd); GI(counts, 4);
#undef GI
  if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = cn_set_error("cn_gst_create: setup failed");
  if (rc) { cn_gst_destroy(g); return rc; }
  g->ws_allocs = ctx->allocs.size();
  *out = g;
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
  const float* host[kNumParams];
  for (int i = 0; i < kNumParams; ++i) {
    auto it = g->host.find(kParamNames[i]);
    if (it == g->host.end()) return cn_set_error("cn_gst_finalize: parameter '%s' was not set", kParamNames[i]);
    host[i] = it->second.data();
  }
  cudaSetDevice(g->device);
  g->finalized = false;
  // release the device parameters of a previous finalize (ring buffers and workspace come first and stay)
  CnLaunchCtx* ctx = &g->ctx;
  cudaDeviceSynchronize();
  for (size_t i = g->ws_allocs; i < ctx->allocs.size(); ++i) cudaFree(ctx->allocs[i]);
  ctx->allocs.resize(g->ws_allocs);
  // indices in kParamNames: 0 We 1 be 2 ln0g 3 ln0b 4 Win 5 bin 6 Wout 7 bout 8 ln1g 9 ln1b 10 W1 11 b1 12 W2 13 b2
  //                         14 Wih 15 bih 16 Whh 17 bhh 18 Wp 19 bp
  std::vector<float> wet(128);
  for (int c = 0; c < 64; ++c) { wet[c] = host[0][c * 2]; wet[64 + c] = host[0][c * 2 + 1]; }     // [64][2] -> [2][64]
  int rc = gt_upload(ctx, &g->w.We_t, wet.data(), 128);
  const float** fdst[] = {&g->w.be, &g->w.ln0_g, &g->w.ln0_b, &g->w.bin, &g->w.bout, &g->w.ln1_g, &g->w.ln1_b, &g->w.b1, &g->w.b2,
                          &g->w.bih, &g->w.bhh, &g->w.Wp, &g->w.bp};
  const int fidx[] = {1, 2, 3, 5, 7, 8, 9, 11, 13, 15, 17, 18, 19};
  for (int i = 0; i < 13 && !rc; ++i) rc = gt_upload(ctx, fdst[i], host[fidx[i]], (size_t)kParamRows[fidx[i]] * kParamCols[fidx[i]]);
  struct { int idx; TcMat* t; } tw[6] = {{4, &g->tWin}, {6, &g->tWout}, {10, &g->tW1}, {12, &g->tW2}, {14, &g->tWih}, {16, &g->tWhh}};
  for (int i = 0; i < 6 && !rc; ++i) {
    const int r = kParamRows[tw[i].idx], k = kParamCols[tw[i].idx];
    const float* d = nullptr;
    rc = gt_upload(ctx, &d, host[tw[i].idx], (size_t)r * k);
    const int bn = r == 256 ? 256 : 64;                                       // the 256-wide gate GEMMs use BN = 256 tiles
    if (!rc) rc = tc_alloc(ctx, *tw[i].t, r, k, bn, tc_box_k(bn));
    if (!rc) split16(ctx, 0, d, 64.0f, tw[i].t->hi, tw[i].t->lo, (size_t)r * k);
  }
  if (!rc && cudaDeviceSynchronize() != cudaSuccess) rc = cn_set_error("cn_gst_finalize: weight upload failed");
  if (rc) return rc;
  g->finalized = true;
  return 0;
}

// VecPretextNormalize.reset(): traj_buffer <- -999, mask_buffer <- False (rl/vec_env/vec_pretext_normalize.py:85-101)
int cn_gst_reset(cn_gst* g, void* stream) {
  if (!g) return cn_set_error("cn_gst_reset: null argument");
  cudaSetDevice(g->device);
  const size_t n = (size_t)GT_T * g->N * g->H;
  std::vector<float> inv(n * 2, GT_INVALID);
  cudaError_t err = cudaMemcpyAsync(g->ring_pos, inv.data(), n * 2 * sizeof(float), cudaMemcpyHostToDevice, (cudaStream_t)stream);
  if (err == cudaSuccess) err = cudaStreamSynchronize((cudaStream_t)stream);
  if (err == cudaSuccess) err = cudaMemsetAsync(g->ring_mask, 0, n, (cudaStream_t)stream);
  if (err != cudaSuccess) return cn_set_error("cn_gst_reset: %s", cudaGetErrorString(err));
  g->newest = GT_T - 1;
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
  g->newest = (g->newest + 1) % GT_T;
  CnLaunchCtx* p = &g->ctx;
  cudaStream_t st = (cudaStream_t)stream;
  const int N = g->N, H = g->H;
  const int R = N * GT_T * H, Rd = N * H, G = N * GT_T;
  const int* cntR = g->counts;          // valid observation rows
  const int* cntD = g->counts + 1;      // humans visible in the newest frame
  const dim3 rows_grid((unsigned)(p->num_sms * 4)), grp_grid((unsigned)((G + GTC_WARPS - 1) / GTC_WARPS));
  // test hook (cn_internal_gst_stop_after): one string compare per stage while a stop is set, one empty() otherwise
  const std::string stop = g->stop_after;
  g->stop_after.clear();
  auto at = [&](const std::string& pfx, const char* s) { return !stop.empty() && stop == pfx + s; };
  auto finish = [&]() -> int {
    cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) return cn_set_error("cn_gst_step: %s", cudaGetErrorString(err));
    if (p->launch_error) { p->launch_error = false; return 1; }
    return 0;
  };
  // one encoder pass; true when the step stops inside it
  auto encoder = [&](const std::string& pfx, int maxrows, const int* cnt, int groups, const int* start) {
    gemm_tc(p, st, g->tX, g->tWin, maxrows, 192, 64, 64, g->w.bin, CN_ACT_NONE, out32(g->QKV, 192), cnt);
    if (at(pfx, "qkv")) return true;
    launch_k(p, gtc_attn_kernel, dim3((unsigned)groups), dim3((unsigned)(8 * H)), (size_t)H * 192 * sizeof(float), st, H, start,
             g->QKV, g->w.bin + 64, g->tA.hi, g->tA.lo);
    if (at(pfx, "attn")) return true;
    gemm_tc(p, st, g->tA, g->tWout, maxrows, 64, 64, 64, g->w.bout, CN_ACT_NONE, out32(g->O, 64), cnt);
    if (at(pfx, "out")) return true;
    launch_k(p, gtc_res_ln_kernel, rows_grid, dim3(256), 0, st, g->w, cnt, g->X0, g->O, g->X1, g->tY.hi, g->tY.lo);
    if (at(pfx, "res_ln")) return true;
    gemm_tc(p, st, g->tY, g->tW1, maxrows, 128, 64, 64, g->w.b1, CN_ACT_RELU, out16(g->tF), cnt);
    if (at(pfx, "ffn1")) return true;
    gemm_tc(p, st, g->tF, g->tW2, maxrows, 64, 128, 64, g->w.b2, CN_ACT_NONE, out32(g->O, 64), cnt);
    if (at(pfx, "ffn2")) return true;
    launch_k(p, gtc_res_kernel, rows_grid, dim3(256), 0, st, cnt, g->X1, g->O, g->tXS.hi, g->tXS.lo);
    if (at(pfx, "res")) return true;
    gemm_tc(p, st, g->tXS, g->tWih, maxrows, 256, 64, 256, g->w.bih, CN_ACT_NONE,
            out32(g->GX, 256, maxrows == R ? &g->GX_R : &g->GX_Rd), cnt);
    return at(pfx, "gx");
  };
  launch_k(p, gtc_prep_kernel, grp_grid, dim3(GTC_WARPS * 32), 0, st, N, H, g->ring_pos, g->ring_mask, g->newest, d_robot_node, d_spatial2,
           d_visible, g->rowm, g->inp, g->gcount, g->ecount, g->fp, g->pos_last);
  if (at("", "prep")) return finish();
  launch_k(p, gtc_scan_kernel, dim3(1), dim3(1024), 0, st, g->gcount, G, g->gstart, g->ecount, N, g->estart, g->counts);
  if (at("", "scan")) return finish();
  launch_k(p, gtc_index_kernel, grp_grid, dim3(GTC_WARPS * 32), 0, st, N, H, g->rowm, g->fp, g->gstart, g->estart, g->cidx, g->crow,
           g->drow);
  if (at("", "index")) return finish();
  launch_k(p, gtc_embed_kernel, rows_grid, dim3(256), 0, st, g->w, cntR, g->crow, g->inp, g->X0, g->tX.hi, g->tX.lo);
  if (at("obs.", "embed") || encoder("obs.", R, cntR, G, g->gstart)) return finish();
  // LSTM over the 5 observed frames, humans visible now only (h0 = c0 = 0: frame 0 has no recurrent GEMM, its
  // hidden-state gate term is b_hh)
  for (int t = 0; t < GT_T; ++t) {
    if (t > 0) gemm_tc(p, st, g->tHd, g->tWhh, Rd, 256, 64, 256, g->w.bhh, CN_ACT_NONE, out32(g->GH, 256, &g->GH_Rd), cntD);
    launch_k(p, gtc_cell_kernel, rows_grid, dim3(256), 0, st, H, t, cntD, g->drow, g->cidx, g->GX, g->w.bih, g->w.bhh, g->GH, g->h32,
             g->c32, g->tHd.hi, g->tHd.lo);
    if (!stop.empty() && stop == "lstm" + std::to_string(t)) return finish();
  }
  for (int tt = 0; tt < GT_T; ++tt) {
    const std::string pfx = stop.empty() ? std::string() : "dec" + std::to_string(tt) + ".";
    if (tt > 0) {
      launch_k(p, gtc_embed_kernel, rows_grid, dim3(256), 0, st, g->w, cntD, (const int*)nullptr, g->xin, g->X0, g->tX.hi, g->tX.lo);
      if (at(pfx, "embed") || encoder(pfx, Rd, cntD, N, g->estart)) return finish();
      gemm_tc(p, st, g->tHd, g->tWhh, Rd, 256, 64, 256, g->w.bhh, CN_ACT_NONE, out32(g->GH, 256, &g->GH_Rd), cntD);
      if (at(pfx, "gh")) return finish();
      launch_k(p, gtc_cell_kernel, rows_grid, dim3(256), 0, st, H, -1, cntD, g->drow, g->cidx, g->GX, g->w.bih, g->w.bhh, g->GH, g->h32,
               g->c32, g->tHd.hi, g->tHd.lo);
      if (at(pfx, "cell")) return finish();
    }
    launch_k(p, gtc_h2p_kernel, rows_grid, dim3(256), 0, st, g->w, tt, cntD, g->drow, g->h32, g->pos_last, g->xin, g->mu_cum, g->pred);
    if (at(pfx, "h2p")) return finish();
  }
  launch_k(p, gt_final_kernel, dim3((unsigned)N), dim3((unsigned)((H + 31) / 32 * 32)), 0, st, N, H, g->P, g->thr,
           g->collision_penalty, d_robot_node, d_spatial2, g->fp, g->pred, d_reward, d_penalty, d_spatial_out);
  return finish();
}

int64_t cn_gst_launch_count(cn_gst* g) { return g ? g->ctx.launches : 0; }

// ---- test-only hooks (not in crowdnav_b200.h): tests/test_gpu_gst_stages.py reads the workspace stage by stage ----
// Workspace buffer `name`: device pointer, rows, columns, row pitch (elements) and kind -- 0: fp32, 1: split fp16
// (hi, lo) pair at *ptr / *ptr_lo (value = hi + lo), 2: int32, 3: uint8.  Row r starts at element r * *ld.  R = N*5*H
// observation rows (compact: the first counts[0] are live), Rd = N*H decode rows (compact: the first counts[1]).
//   ring_pos [5*N*H, 2], ring_mask [5*N*H] (slot-major [5][N][H]);  rowm [R], inp [R, 2], gcount [N*5], gstart [N*5+1],
//   ecount [N], estart [N+1], counts [4], cidx / crow [R], drow [Rd], fp [Rd], pos_last [Rd, 2];
//   X0 [R, 64], tX / tA / tY / tXS pairs [R, 64], QKV [R, 192], O / X1 [R, 64], tF pair [R, 128], GX [R, 256];
//   GH [Rd, 256], h32 / c32 [Rd, 64], tHd pair [Rd, 64], xin / mu_cum [Rd, 2], pred [Rd, 10] (5 frames x (x, y)).
// The decoding encoder reuses the observation encoder's buffers; see cn_internal_gst_stop_after.
int cn_internal_gst_buffer(cn_gst* g, const char* name, void** ptr, void** ptr_lo, int* rows, int* cols, int* ld, int* kind) {
  if (!g || !name || !ptr || !ptr_lo || !rows || !cols || !ld || !kind) return cn_set_error("cn_internal_gst_buffer: null argument");
  const int R = g->N * GT_T * g->H, Rd = g->N * g->H, G = g->N * GT_T;
  const std::string s(name);
  *ptr_lo = nullptr;
  auto set = [&](const void* q, int r, int c, int l, int k) { *ptr = (void*)q; *rows = r; *cols = c; *ld = l; *kind = k; return 0; };
  auto f32 = [&](const float* q, int r, int c) { return set(q, r, c, c, 0); };
  auto i32 = [&](const int* q, int r) { return set(q, r, 1, 1, 2); };
  auto f16 = [&](const TcMat& t, int r, int c) { *ptr_lo = t.lo; return set(t.hi, r, c, t.pitch, 1); };
  if (s == "ring_pos") return f32(g->ring_pos, R, 2);
  if (s == "ring_mask") return set(g->ring_mask, R, 1, 1, 3);
  if (s == "rowm") return f32(g->rowm, R, 1);
  if (s == "inp") return f32(g->inp, R, 2);
  if (s == "gcount") return i32(g->gcount, G);
  if (s == "gstart") return i32(g->gstart, G + 1);
  if (s == "ecount") return i32(g->ecount, g->N);
  if (s == "estart") return i32(g->estart, g->N + 1);
  if (s == "counts") return i32(g->counts, 4);
  if (s == "cidx") return i32(g->cidx, R);
  if (s == "crow") return i32(g->crow, R);
  if (s == "drow") return i32(g->drow, Rd);
  if (s == "fp") return f32(g->fp, Rd, 1);
  if (s == "pos_last") return f32(g->pos_last, Rd, 2);
  if (s == "X0") return f32(g->X0, R, 64);
  if (s == "tX") return f16(g->tX, R, 64);
  if (s == "QKV") return f32(g->QKV, R, 192);
  if (s == "tA") return f16(g->tA, R, 64);
  if (s == "O") return f32(g->O, R, 64);
  if (s == "X1") return f32(g->X1, R, 64);
  if (s == "tY") return f16(g->tY, R, 64);
  if (s == "tF") return f16(g->tF, R, 128);
  if (s == "tXS") return f16(g->tXS, R, 64);
  if (s == "GX") return f32(g->GX, R, 256);
  if (s == "GH") return f32(g->GH, Rd, 256);
  if (s == "h32") return f32(g->h32, Rd, 64);
  if (s == "c32") return f32(g->c32, Rd, 64);
  if (s == "tHd") return f16(g->tHd, Rd, 64);
  if (s == "xin") return f32(g->xin, Rd, 2);
  if (s == "mu_cum") return f32(g->mu_cum, Rd, 2);
  if (s == "pred") return f32(g->pred, Rd, GT_T * 2);
  return cn_set_error("cn_internal_gst_buffer: unknown buffer '%s'", name);
}

// The next cn_gst_step returns right after stage `stage` (names: gst_stage_names), leaving the workspace as that stage
// wrote it; null or "" clears.  The stopped step has still advanced the ring.  Off by default.
int cn_internal_gst_stop_after(cn_gst* g, const char* stage) {
  if (!g) return cn_set_error("cn_internal_gst_stop_after: null argument");
  const std::string s(stage ? stage : "");
  if (!s.empty()) {
    bool known = false;
    for (const std::string& n : gst_stage_names()) known = known || n == s;
    if (!known) return cn_set_error("cn_internal_gst_stop_after: unknown stage '%s'", stage);
  }
  g->stop_after = s;
  return 0;
}

}  // extern "C"
