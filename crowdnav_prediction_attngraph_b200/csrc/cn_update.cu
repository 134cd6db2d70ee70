// PPO update path (SURVEY.md §8f row 3; rl/ppo/ppo.py:36-101 -> Policy.evaluate_actions): the per-human linear
// layers of the attention encoder -- 98 % of the update's FLOPs -- forward, data gradient and weight gradient on
// the wgmma 3xFP16 GEMM (cn_gemm_tc.cuh), in fp32-equivalent accuracy:
//
//   forward   Y[M,N]  = act(X[M,K] W[N,K]^T + b)
//   dgrad     dX[M,K] = dZ[M,N] W[N,K]            dZ = dY o act'(Y)
//   wgrad     dW[N,K] = dZ[M,N]^T X[M,K]          K-dimension of this GEMM = M rows (hundreds of thousands):
//                                                 split-K over the CTAs, partial tiles added atomically
//   db[N]     = column sums of dZ
//
// Every operand travels as a (hi, lo) fp16 pair.  Unlike the rollout (whose activations have known ranges and whose
// weights carry a fixed 2^6 scale) gradients span many orders of magnitude, so each tensor gets a DYNAMIC
// power-of-two scale from its amax (|x| max * scale in [2^13, 2^14)): exact to undo, keeps hi and lo in fp16's
// normal range for everything within ~2^-24 of the tensor's largest entry.  The scales stay on the device
// (no host synchronisation); the GEMM epilogue multiplies by 1 / (scale_a * scale_b).
//
// The C ABI below is stateless: the caller (crowdnav_prediction_attngraph_b200/update_ops.py, a torch.autograd
// Function) owns every buffer, including the workspace.
#include <cuda_runtime.h>
#include <stdint.h>

#include "cn_gemm_tc.h"
#include "cn_host_util.h"

namespace {

inline size_t up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---------------------------------------------------------------------------------------------- small kernels
// amax of |x| (optionally of x o [y > 0]): non-negative floats order like their bit patterns.  16-byte loads.
__global__ void __launch_bounds__(256) cn_upd_amax_kernel(const float* __restrict__ x, const float* __restrict__ relu_y,
                                                          size_t count, unsigned int* __restrict__ out) {
  float m = 0.0f;
  const size_t n4 = count / 4;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  const float4* y4 = reinterpret_cast<const float4*>(relu_y);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 v = __ldg(x4 + i);
    if (relu_y) {
      const float4 y = __ldg(y4 + i);
      if (!(y.x > 0.0f)) v.x = 0.0f;
      if (!(y.y > 0.0f)) v.y = 0.0f;
      if (!(y.z > 0.0f)) v.z = 0.0f;
      if (!(y.w > 0.0f)) v.w = 0.0f;
    }
    const float a = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));   // fmaxf drops NaNs
    if (a < 3.0e38f) m = fmaxf(m, a);                     // inf does not poison the scale (it poisons the result)
  }
  if (blockIdx.x == 0 && threadIdx.x < (count & 3)) {      // tail
    const size_t i = n4 * 4 + threadIdx.x;
    float v = fabsf(x[i]);
    if (relu_y && !(relu_y[i] > 0.0f)) v = 0.0f;
    if (v == v && v < 3.0e38f) m = fmaxf(m, v);
  }
  for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  __shared__ float sm[8];
  if ((threadIdx.x & 31) == 0) sm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, sm[w]);
    atomicMax(out, __float_as_uint(m));
  }
}

// scale[0] = 2^k with amax * 2^k in [2^13, 2^14), scale[1] = 2^-k  (amax == 0: 1, 1)
__global__ void cn_upd_scale_kernel(const unsigned int* __restrict__ amax_bits, float* __restrict__ scale) {
  const float a = __uint_as_float(*amax_bits);
  float s = 1.0f;
  if (a > 0.0f) {
    int e;
    frexpf(a, &e);                                    // a = f * 2^e, f in [0.5, 1)
    int k = 14 - e;
    k = k > 100 ? 100 : (k < -100 ? -100 : k);
    s = ldexpf(1.0f, k);
  }
  scale[0] = s;
  scale[1] = 1.0f / s;
}

// (hi, lo) split of a row-major fp32 matrix src[M, C] (C and ld multiples of 4; optionally masked by relu_y > 0),
// scaled by *scale:
//   hi/lo    [M, Cp]   row-major (pitch Cp >= C, multiple of 64; padding columns zero) -- or null
//   hiT/loT  [C, Mp]   transposed (pitch Mp >= M, multiple of 64; padding zero)       -- or null
//   colsum   [C]       += column sums of the masked, UNscaled values (db), fp64 accumulators (the partial sums of
//                         ~M/64 CTAs arrive in arbitrary order: in fp32 that costs ~1e-5 relative)  -- or null
// One 64 x 64 tile per CTA iteration (grid-stride): 16-byte loads, 8-byte row-major stores, and the transposed copy
// leaves through shared memory as 4-byte (two rows) stores, 128 contiguous bytes per warp.
__global__ void __launch_bounds__(256) cn_upd_split_kernel(const float* __restrict__ src, int ld, const float* __restrict__ relu_y,
                                                           int ldy, int M, int C, const float* __restrict__ scale,
                                                           __half* __restrict__ hi, __half* __restrict__ lo, int Cp,
                                                           __half* __restrict__ hiT, __half* __restrict__ loT, int Mp,
                                                           double* __restrict__ colsum) {
  __shared__ float tile[64][65];
  __shared__ float colpart[64];
  const float sc = __ldg(scale);
  const int tid = threadIdx.x;
  const int lx = tid & 15, ly = tid >> 4;                       // load layout: 16 float4 per row, 16 rows per pass
  const int tiles_c = ((Cp > C ? Cp : C) + 63) / 64, tiles_m = ((Mp > M ? Mp : M) + 63) / 64;
  const long long total = (long long)tiles_m * tiles_c;
  for (long long t = blockIdx.x; t < total; t += gridDim.x) {
    const int tm = (int)(t / tiles_c), tcn = (int)(t - (long long)tm * tiles_c);
    const int r0 = tm * 64, c0 = tcn * 64;
    if (colsum && tid < 64) colpart[tid] = 0.0f;
    if (colsum) __syncthreads();
    float cs[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = r0 + ly + 16 * j, c = c0 + 4 * lx;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < M && c < C) {
        v = *reinterpret_cast<const float4*>(src + (size_t)r * ld + c);
        if (relu_y) {
          const float4 y = *reinterpret_cast<const float4*>(relu_y + (size_t)r * ldy + c);
          if (!(y.x > 0.0f)) v.x = 0.0f;
          if (!(y.y > 0.0f)) v.y = 0.0f;
          if (!(y.z > 0.0f)) v.z = 0.0f;
          if (!(y.w > 0.0f)) v.w = 0.0f;
        }
      }
      cs[0] += v.x; cs[1] += v.y; cs[2] += v.z; cs[3] += v.w;
      float x[4] = {v.x * sc, v.y * sc, v.z * sc, v.w * sc};
      uint32_t ph[2], pl[2];
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float x0 = fminf(fmaxf(x[2 * q], -65504.0f), 65504.0f), x1 = fminf(fmaxf(x[2 * q + 1], -65504.0f), 65504.0f);
        x[2 * q] = x0; x[2 * q + 1] = x1;
        const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
        const __half l0 = __float2half_rn(x0 - __half2float(h0)), l1 = __float2half_rn(x1 - __half2float(h1));
        ph[q] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
        pl[q] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
      }
      float* trow = &tile[ly + 16 * j][4 * lx];
      trow[0] = x[0]; trow[1] = x[1]; trow[2] = x[2]; trow[3] = x[3];
      if (hi && r < M && c < Cp) {
        *reinterpret_cast<uint2*>(hi + (size_t)r * Cp + c) = make_uint2(ph[0], ph[1]);
        *reinterpret_cast<uint2*>(lo + (size_t)r * Cp + c) = make_uint2(pl[0], pl[1]);
      }
    }
    if (colsum) {
#pragma unroll
      for (int q = 0; q < 4; ++q) if (cs[q] != 0.0f) atomicAdd(&colpart[4 * lx + q], cs[q]);
    }
    __syncthreads();
    if (colsum && tid < 64 && c0 + tid < C && colpart[tid] != 0.0f) atomicAdd(colsum + c0 + tid, (double)colpart[tid]);
    if (hiT) {
      const int warp = tid >> 5, lane = tid & 31;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int cl = warp + 8 * j;                               // column of the tile handled by this warp
        const int c = c0 + cl, r = r0 + 2 * lane;                  // this lane writes rows r, r + 1
        if (c < C && r < Mp) {
          const float x0 = tile[2 * lane][cl], x1 = tile[2 * lane + 1][cl];
          const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
          const __half l0 = __float2half_rn(x0 - __half2float(h0)), l1 = __float2half_rn(x1 - __half2float(h1));
          *reinterpret_cast<uint32_t*>(hiT + (size_t)c * Mp + r) = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
          *reinterpret_cast<uint32_t*>(loT + (size_t)c * Mp + r) = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
        }
      }
    }
    __syncthreads();
  }
}

__global__ void cn_upd_d2f_kernel(const double* __restrict__ src, float* __restrict__ dst, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = (float)src[i];
}

// ---------------------------------------------------------------------------------------------- attention (update)
// Human-human multi-head self attention over COMPACTED rows, forward with soft-max statistics and backward
// (selfAttn_srnn_temp_node.py:63-91 -> nn.MultiheadAttention core: softmax(q k^T / 8) v over the n valid humans of a
// sample).  qkv [Mc, 1536] = (q | k | v) per row, 8 heads x 64.  One warp per row, all heads at once; lane l owns the
// float4 #(l + 32 c), c = 0..3, of every 512-wide row = 4 elements of head 2 c + (l >= 16), so a head's dot product is
// a butterfly over the 16 lanes of a half-warp.  The padded torch formulation this replaces materialised
// [B, H, 1536] tensors (7.5 GB per minibatch at the bench shape); here only real rows move.
#define CN_UPD_ATTN_WARPS 4
#define CN_UPD_MAXKEYS 128

__device__ __forceinline__ void upd_load_row(const float* __restrict__ p, int lane, float4 (&r)[4]) {
  const float4* v = reinterpret_cast<const float4*>(p) + lane;
#pragma unroll
  for (int c = 0; c < 4; ++c) r[c] = __ldg(v + 32 * c);
}
// per-head dot products of two 512-wide rows: s[c] = <a, b> restricted to head 2 c + (lane >= 16), on every lane of the half
__device__ __forceinline__ void upd_dot_heads(const float4 (&a)[4], const float4 (&b)[4], float (&s)[4]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    float x = a[c].x * b[c].x;
    x = fmaf(a[c].y, b[c].y, x); x = fmaf(a[c].z, b[c].z, x); x = fmaf(a[c].w, b[c].w, x);
#pragma unroll
    for (int o = 8; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    s[c] = x;
  }
}
__device__ __forceinline__ void upd_axpy(float4 (&acc)[4], const float (&w)[4], const float4 (&x)[4]) {
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    acc[c].x = fmaf(w[c], x[c].x, acc[c].x); acc[c].y = fmaf(w[c], x[c].y, acc[c].y);
    acc[c].z = fmaf(w[c], x[c].z, acc[c].z); acc[c].w = fmaf(w[c], x[c].w, acc[c].w);
  }
}

// forward: out[r] = softmax_j(q_r . k_j / 8) v_j ; stats[r] = {max[8], sum[8]} (head h at index h and 8 + h)
__global__ void __launch_bounds__(CN_UPD_ATTN_WARPS * 32) cn_upd_attn_fwd_kernel(const float* __restrict__ qkv,
                                                                                const int* __restrict__ row_start,
                                                                                const int* __restrict__ row_env, int Mc,
                                                                                float* __restrict__ out, float* __restrict__ stats) {
  __shared__ float sc[CN_UPD_ATTN_WARPS][CN_UPD_MAXKEYS][8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, half = lane >> 4;
  float (*my)[8] = sc[warp];
  for (int r = blockIdx.x * CN_UPD_ATTN_WARPS + warp; r < Mc; r += gridDim.x * CN_UPD_ATTN_WARPS) {
    const int e = row_env[r], row0 = row_start[e], n = row_start[e + 1] - row0;
    float4 q[4];
    upd_load_row(qkv + (size_t)r * 1536, lane, q);
#pragma unroll
    for (int c = 0; c < 4; ++c) { q[c].x *= 0.125f; q[c].y *= 0.125f; q[c].z *= 0.125f; q[c].w *= 0.125f; }
    float m[4] = {-INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int j = 0; j < n; ++j) {
      float4 k[4];
      upd_load_row(qkv + (size_t)(row0 + j) * 1536 + 512, lane, k);
      float s[4];
      upd_dot_heads(q, k, s);
#pragma unroll
      for (int c = 0; c < 4; ++c) m[c] = fmaxf(m[c], s[c]);
      if ((lane & 15) == 0) {
#pragma unroll
        for (int c = 0; c < 4; ++c) my[j][half * 4 + c] = s[c];
      }
    }
    __syncwarp();
    float4 acc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    float l[4] = {0.f, 0.f, 0.f, 0.f};
    for (int j = 0; j < n; ++j) {
      float4 v[4];
      upd_load_row(qkv + (size_t)(row0 + j) * 1536 + 1024, lane, v);
      float p[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) { p[c] = expf(my[j][half * 4 + c] - m[c]); l[c] += p[c]; }
      upd_axpy(acc, p, v);
    }
    float4* o = reinterpret_cast<float4*>(out + (size_t)r * 512) + lane;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float inv = 1.0f / l[c];
      o[32 * c] = make_float4(acc[c].x * inv, acc[c].y * inv, acc[c].z * inv, acc[c].w * inv);
    }
    if ((lane & 15) == 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {                    // head = 2 c + half
        stats[(size_t)r * 16 + 2 * c + half] = m[c];
        stats[(size_t)r * 16 + 8 + 2 * c + half] = l[c];
      }
    }
    __syncwarp();
  }
}

// backward, pass A (per query row i): delta_i = <dO_i, O_i> per head, dQ_i = (1/8) sum_j dS_ij K_j with
// dS_ij = P_ij (dO_i . V_j - delta_i).  Writes dqkv[:, 0:512] and delta [Mc, 8].
__global__ void __launch_bounds__(CN_UPD_ATTN_WARPS * 32) cn_upd_attn_bwd_q_kernel(
    const float* __restrict__ qkv, const float* __restrict__ out, const float* __restrict__ dout, const float* __restrict__ stats,
    const int* __restrict__ row_start, const int* __restrict__ row_env, int Mc, float* __restrict__ dqkv,
    float* __restrict__ delta) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, half = lane >> 4;
  for (int r = blockIdx.x * CN_UPD_ATTN_WARPS + warp; r < Mc; r += gridDim.x * CN_UPD_ATTN_WARPS) {
    const int e = row_env[r], row0 = row_start[e], n = row_start[e + 1] - row0;
    float4 q[4], dO[4], O[4];
    upd_load_row(qkv + (size_t)r * 1536, lane, q);
    upd_load_row(dout + (size_t)r * 512, lane, dO);
    upd_load_row(out + (size_t)r * 512, lane, O);
    float dl[4], m[4], linv[4];
    upd_dot_heads(dO, O, dl);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      q[c].x *= 0.125f; q[c].y *= 0.125f; q[c].z *= 0.125f; q[c].w *= 0.125f;
      m[c] = stats[(size_t)r * 16 + 2 * c + half];
      linv[c] = 1.0f / stats[(size_t)r * 16 + 8 + 2 * c + half];
    }
    if ((lane & 15) == 0) {
#pragma unroll
      for (int c = 0; c < 4; ++c) delta[(size_t)r * 8 + 2 * c + half] = dl[c];
    }
    float4 acc[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[c] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < n; ++j) {
      float4 k[4], v[4];
      upd_load_row(qkv + (size_t)(row0 + j) * 1536 + 512, lane, k);
      upd_load_row(qkv + (size_t)(row0 + j) * 1536 + 1024, lane, v);
      float s[4], dp[4], ds[4];
      upd_dot_heads(q, k, s);
      upd_dot_heads(dO, v, dp);
#pragma unroll
      for (int c = 0; c < 4; ++c) ds[c] = expf(s[c] - m[c]) * linv[c] * (dp[c] - dl[c]) * 0.125f;
      upd_axpy(acc, ds, k);
    }
    float4* o = reinterpret_cast<float4*>(dqkv + (size_t)r * 1536) + lane;
#pragma unroll
    for (int c = 0; c < 4; ++c) o[32 * c] = acc[c];
  }
}

// backward, pass B (per key row j): dV_j = sum_i P_ij dO_i, dK_j = (1/8) sum_i dS_ij Q_i.  Writes dqkv[:, 512:1536].
__global__ void __launch_bounds__(CN_UPD_ATTN_WARPS * 32) cn_upd_attn_bwd_kv_kernel(
    const float* __restrict__ qkv, const float* __restrict__ dout, const float* __restrict__ stats, const float* __restrict__ delta,
    const int* __restrict__ row_start, const int* __restrict__ row_env, int Mc, float* __restrict__ dqkv) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, half = lane >> 4;
  for (int r = blockIdx.x * CN_UPD_ATTN_WARPS + warp; r < Mc; r += gridDim.x * CN_UPD_ATTN_WARPS) {
    const int e = row_env[r], row0 = row_start[e], n = row_start[e + 1] - row0;
    float4 k[4], v[4];
    upd_load_row(qkv + (size_t)r * 1536 + 512, lane, k);
    upd_load_row(qkv + (size_t)r * 1536 + 1024, lane, v);
    float4 dk[4], dv[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) { dk[c] = make_float4(0.f, 0.f, 0.f, 0.f); dv[c] = make_float4(0.f, 0.f, 0.f, 0.f); }
    for (int i = 0; i < n; ++i) {
      const size_t ri = (size_t)(row0 + i);
      float4 q[4], dO[4];
      upd_load_row(qkv + ri * 1536, lane, q);
      upd_load_row(dout + ri * 512, lane, dO);
      float s[4], dp[4], p[4], ds[4];
      upd_dot_heads(q, k, s);
      upd_dot_heads(dO, v, dp);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float mi = stats[ri * 16 + 2 * c + half], li = stats[ri * 16 + 8 + 2 * c + half];
        p[c] = expf(s[c] * 0.125f - mi) / li;
        ds[c] = p[c] * (dp[c] - delta[ri * 8 + 2 * c + half]) * 0.125f;
      }
      upd_axpy(dv, p, dO);
      upd_axpy(dk, ds, q);
    }
    float4* ok = reinterpret_cast<float4*>(dqkv + (size_t)r * 1536 + 512) + lane;
    float4* ov = reinterpret_cast<float4*>(dqkv + (size_t)r * 1536 + 1024) + lane;
#pragma unroll
    for (int c = 0; c < 4; ++c) { ok[32 * c] = dk[c]; ov[32 * c] = dv[c]; }
  }
}

// ---------------------------------------------------------------------------------------------- GRU over a rollout (update)
// EndRNN's GRU cell over the T steps of a minibatch with done-mask resets (rl/networks/srnn_model.py:35-103,
// selfAttn_srnn_temp_node.py:262-285), forward and backward in ONE launch each.  The eager formulation costs ~40
// tiny kernels and autograd nodes per step and made the update launch-bound on the host.  gi = W_ih x + b_ih comes in
// precomputed for all steps (one GEMM); here, per step:  h <- h * mask_t;  gh = W_hh h + b_hh;  r = s(gi_r + gh_r),
// z = s(gi_z + gh_z), n = tanh(gi_n + r gh_n), h <- (1 - z) n + z h   (PyTorch gate order r, z, n).
// A CTA owns 16 environments for the whole sequence; W_hh (384 x 128 fp32 = 192 KB) stays in shared memory.
#define CN_GRU_ROWS 16
#define CN_GRU_THREADS 256
#define CN_GRU_SMEM (384 * 128 * 4 + CN_GRU_ROWS * 384 * 4 + 384 * 4)

__device__ __forceinline__ float upd_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

// saved [T, N, 4, 128] = (r, z, n, gh_n) per step; out [T, N, 128] = h after each step
__global__ void __launch_bounds__(CN_GRU_THREADS, 1) cn_upd_gru_fwd_kernel(
    const float* __restrict__ gi, const float* __restrict__ h0, const float* __restrict__ masks, const float* __restrict__ whh,
    const float* __restrict__ bhh, int T, int N, float* __restrict__ out, float* __restrict__ saved) {
  extern __shared__ __align__(16) float gsm[];
  float* wt = gsm;                              // [128][384]: W_hh transposed (k-major) -> conflict-free over the gate columns
  float* hs = wt + 128 * 384;                   // [16][128] current (masked) hidden state  (tile is 16 x 384 floats: reused below)
  float* bs = hs + CN_GRU_ROWS * 384;           // [384]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < 384 * 128; i += CN_GRU_THREADS) { const int j = i / 128, k = i - j * 128; wt[k * 384 + j] = whh[i]; }
  for (int i = tid; i < 384; i += CN_GRU_THREADS) bs[i] = bhh[i];
  const int row0 = blockIdx.x * CN_GRU_ROWS;
  const int r0 = 2 * warp, r1 = 2 * warp + 1;                    // this warp's two rows; lane owns columns lane + 32 j
  const int e0 = row0 + r0, e1 = row0 + r1;
  float h[2][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    h[0][j] = e0 < N ? h0[(size_t)e0 * 128 + lane + 32 * j] : 0.0f;
    h[1][j] = e1 < N ? h0[(size_t)e1 * 128 + lane + 32 * j] : 0.0f;
  }
  __syncthreads();
  for (int t = 0; t < T; ++t) {
    const float m0 = e0 < N ? masks[(size_t)t * N + e0] : 0.0f, m1 = e1 < N ? masks[(size_t)t * N + e1] : 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      h[0][j] *= m0; h[1][j] *= m1;
      hs[r0 * 128 + lane + 32 * j] = h[0][j]; hs[r1 * 128 + lane + 32 * j] = h[1][j];
    }
    __syncwarp();                                                 // rows r0, r1 are private to this warp
    float acc[2][12];
#pragma unroll
    for (int q = 0; q < 12; ++q) { acc[0][q] = 0.0f; acc[1][q] = 0.0f; }
#pragma unroll 4
    for (int k = 0; k < 128; ++k) {
      const float a0 = hs[r0 * 128 + k], a1 = hs[r1 * 128 + k];
      const float* w = wt + k * 384 + lane;
#pragma unroll
      for (int q = 0; q < 12; ++q) {                              // q = gate * 4 + j -> column gate * 128 + lane + 32 j
        const float wv = w[32 * q];
        acc[0][q] = fmaf(a0, wv, acc[0][q]); acc[1][q] = fmaf(a1, wv, acc[1][q]);
      }
    }
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int e = rr ? e1 : e0;
      if (e < N) {
        const float* g = gi + ((size_t)t * N + e) * 384;
        float* sv = saved + ((size_t)t * N + e) * 512;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = lane + 32 * j;
          const float ghr = acc[rr][j] + bs[c], ghz = acc[rr][4 + j] + bs[128 + c], ghn = acc[rr][8 + j] + bs[256 + c];
          const float r = upd_sigmoid(g[c] + ghr), z = upd_sigmoid(g[128 + c] + ghz);
          const float n = tanhf(g[256 + c] + r * ghn);
          const float hn = (1.0f - z) * n + z * h[rr][j];
          h[rr][j] = hn;
          out[((size_t)t * N + e) * 128 + c] = hn;
          sv[c] = r; sv[128 + c] = z; sv[256 + c] = n; sv[384 + c] = ghn;
        }
      }
    }
    __syncwarp();
  }
}

// backward: d_out [T, N, 128] (gradient w.r.t. every step's output), optional d_hT [N, 128] (gradient w.r.t. the final state).
// Writes d_gi [T, N, 384] (= gradient w.r.t. gi, and the r / z parts of gh), d_ghn [T, N, 128] (n part of gh) and d_h0 [N, 128];
// dW_hh = [d_gi_r | d_gi_z | d_ghn]^T hm and db_hh follow from these by one GEMM / column sum in the caller.
__global__ void __launch_bounds__(CN_GRU_THREADS, 1) cn_upd_gru_bwd_kernel(
    const float* __restrict__ d_out, const float* __restrict__ d_hT, const float* __restrict__ out, const float* __restrict__ h0,
    const float* __restrict__ masks, const float* __restrict__ saved, const float* __restrict__ whh, int T, int N,
    float* __restrict__ d_gi, float* __restrict__ d_ghn, float* __restrict__ d_h0) {
  extern __shared__ __align__(16) float gsm[];
  float* ws = gsm;                              // [384][128] W_hh as stored: row j contiguous over the hidden columns
  float* ds = ws + 384 * 128;                   // [16][384] gradient w.r.t. gh of the current step
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < 384 * 128; i += CN_GRU_THREADS) ws[i] = whh[i];
  const int row0 = blockIdx.x * CN_GRU_ROWS;
  const int r0 = 2 * warp, r1 = 2 * warp + 1;
  const int e0 = row0 + r0, e1 = row0 + r1;
  float dh[2][4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    dh[0][j] = (d_hT && e0 < N) ? d_hT[(size_t)e0 * 128 + lane + 32 * j] : 0.0f;
    dh[1][j] = (d_hT && e1 < N) ? d_hT[(size_t)e1 * 128 + lane + 32 * j] : 0.0f;
  }
  __syncthreads();
  for (int t = T - 1; t >= 0; --t) {
    float dhm[2][4];
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const int e = rr ? e1 : e0, rl = rr ? r1 : r0;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = lane + 32 * j;
        float gr = 0.0f, gz = 0.0f, gn = 0.0f, ghn_g = 0.0f, carry = 0.0f;
        if (e < N) {
          const float m = masks[(size_t)t * N + e];
          const float hprev = (t > 0 ? out[((size_t)(t - 1) * N + e) * 128 + c] : h0[(size_t)e * 128 + c]) * m;
          const float* sv = saved + ((size_t)t * N + e) * 512;
          const float r = sv[c], z = sv[128 + c], n = sv[256 + c], ghn = sv[384 + c];
          const float d = dh[rr][j] + d_out[((size_t)t * N + e) * 128 + c];
          const float dn = d * (1.0f - z), dz = d * (hprev - n);
          carry = d * z;
          const float dpn = dn * (1.0f - n * n);
          gn = dpn; ghn_g = dpn * r;
          gr = dpn * ghn * r * (1.0f - r);
          gz = dz * z * (1.0f - z);
          float* gg = d_gi + ((size_t)t * N + e) * 384;
          gg[c] = gr; gg[128 + c] = gz; gg[256 + c] = gn;
          d_ghn[((size_t)t * N + e) * 128 + c] = ghn_g;
        }
        ds[rl * 384 + c] = gr; ds[rl * 384 + 128 + c] = gz; ds[rl * 384 + 256 + c] = ghn_g;
        dhm[rr][j] = carry;
      }
    }
    __syncwarp();
    // dhm += d_gh W_hh  ([2 rows, 384] x [384, 128]) for this warp's rows
    float acc[2][4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { acc[0][j] = 0.0f; acc[1][j] = 0.0f; }
#pragma unroll 4
    for (int q = 0; q < 384; ++q) {
      const float a0 = ds[r0 * 384 + q], a1 = ds[r1 * 384 + q];
      const float* w = ws + q * 128 + lane;
#pragma unroll
      for (int j = 0; j < 4; ++j) { const float wv = w[32 * j]; acc[0][j] = fmaf(a0, wv, acc[0][j]); acc[1][j] = fmaf(a1, wv, acc[1][j]); }
    }
    const float m0 = e0 < N ? masks[(size_t)t * N + e0] : 0.0f, m1 = e1 < N ? masks[(size_t)t * N + e1] : 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) { dh[0][j] = (dhm[0][j] + acc[0][j]) * m0; dh[1][j] = (dhm[1][j] + acc[1][j]) * m1; }
    __syncwarp();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (e0 < N) d_h0[(size_t)e0 * 128 + lane + 32 * j] = dh[0][j];
    if (e1 < N) d_h0[(size_t)e1 * 128 + lane + 32 * j] = dh[1][j];
  }
}

struct Dev {
  int sms;
  bool attrs;
};
Dev g_dev[64];

int setup_device(int device) {
  if (device < 0 || device >= 64) return cn_set_error("cn_update: bad device %d", device);
  cudaError_t e = cudaSetDevice(device);
  if (e != cudaSuccess) return cn_set_error("cudaSetDevice(%d): %s", device, cudaGetErrorString(e));
  if (!g_dev[device].attrs) {
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (tc_set_attrs()) return 1;
    g_dev[device].sms = sms;
    g_dev[device].attrs = true;
  }
  return 0;
}

int run_amax_scale(cudaStream_t st, const float* x, const float* relu_y, size_t count, unsigned int* amax_bits, float* scale) {
  cudaMemsetAsync(amax_bits, 0, sizeof(unsigned int), st);
  const size_t want = (count / 4 + 255) / 256;
  const int grid = want < 132 * 16 ? (int)want : 132 * 16;
  cn_upd_amax_kernel<<<grid > 0 ? grid : 1, 256, 0, st>>>(x, relu_y, count, amax_bits);
  cn_upd_scale_kernel<<<1, 1, 0, st>>>(amax_bits, scale);
  return 0;
}

void run_split(cudaStream_t st, const float* src, int ld, const float* relu_y, int ldy, int M, int C, const float* scale,
               __half* hi, __half* lo, int Cp, __half* hiT, __half* loT, int Mp, double* colsum) {
  const long long tiles = (long long)((Mp > M ? Mp : M) + 63) / 64 * (((Cp > C ? Cp : C) + 63) / 64);
  const int grid = tiles < 132 * 8 ? (int)tiles : 132 * 8;
  cn_upd_split_kernel<<<grid > 0 ? grid : 1, 256, 0, st>>>(src, ld, relu_y, ldy, M, C, scale, hi, lo, Cp, hiT, loT, Mp, colsum);
}

struct Carve {
  unsigned char* p;
  size_t off, cap;
  void* take(size_t bytes) {
    off = up(off, 1024);
    void* q = p + off;
    off += bytes;
    return q;
  }
};

}  // namespace

extern "C" {

// rows of padding the transposed activation copies use
static inline int mpad(int M) { return (int)up((size_t)M, 64); }

size_t cn_update_linear_saved_bytes(int M, int K) {
  // X^T as (hi, lo) fp16 [K, Mp] + its scale {s, 1/s} (+ slack for alignment)
  return up((size_t)2 * K * mpad(M) * sizeof(__half), 1024) + 1024;
}

size_t cn_update_linear_ws_bytes(int M, int N, int K) {
  const size_t Mp = mpad(M), Np = up(N, 64), Kp = up(K, 64);
  size_t fwd = 2 * (size_t)M * Kp * 2 + 2 * (size_t)N * Kp * 2;                                 // X split, W split
  size_t bwd = 2 * (size_t)M * Np * 2 + 2 * (size_t)N * Mp * 2 + 2 * (size_t)K * Np * 2;        // dZ, dZ^T, W^T splits
  return (fwd > bwd ? fwd : bwd) + 16 * 1024 + (size_t)N * 8;
}

// replaces (inside Policy.evaluate_actions of the PPO update): F.linear + ReLU of one per-human layer.
// d_saved receives X^T split for the weight gradient of the backward pass.
int cn_update_linear_fwd(const float* d_x, const float* d_w, const float* d_b, float* d_y, void* d_saved, void* d_ws,
                         size_t ws_bytes, int M, int N, int K, int act, int device, void* stream) {
  if (!d_x || !d_w || !d_y || !d_saved || !d_ws) return cn_set_error("cn_update_linear_fwd: null argument");
  if (M <= 0 || N % 64 || K % 64) return cn_set_error("cn_update_linear_fwd: need M > 0, N %% 64 == 0, K %% 64 == 0 (M=%d N=%d K=%d)", M, N, K);
  if (ws_bytes < cn_update_linear_ws_bytes(M, N, K)) return cn_set_error("cn_update_linear_fwd: workspace too small");
  int rc = setup_device(device);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int Mp = mpad(M);
  Carve c{(unsigned char*)d_ws, 0, ws_bytes};
  unsigned int* amax = (unsigned int*)c.take(64);
  float* sw = (float*)c.take(64);
  __half* xh = (__half*)c.take((size_t)M * K * 2);
  __half* xl = (__half*)c.take((size_t)M * K * 2);
  __half* wh = (__half*)c.take((size_t)N * K * 2);
  __half* wl = (__half*)c.take((size_t)N * K * 2);
  unsigned char* sv = (unsigned char*)d_saved;
  __half* xTh = (__half*)sv;
  __half* xTl = xTh + (size_t)K * Mp;
  float* sx = (float*)(sv + up((size_t)2 * K * Mp * 2, 1024));
  run_amax_scale(st, d_x, nullptr, (size_t)M * K, amax, sx);
  run_split(st, d_x, K, nullptr, 0, M, K, sx, xh, xl, K, xTh, xTl, Mp, nullptr);
  run_amax_scale(st, d_w, nullptr, (size_t)N * K, amax + 1, sw);
  run_split(st, d_w, K, nullptr, 0, N, K, sw, wh, wl, K, nullptr, nullptr, 0, nullptr);
  rc = gemm_tc_promote(g_dev[device].sms, st, xh, xl, M, K, wh, wl, N, K, K, d_y, N, d_b, act, sx + 1, sw + 1, 1);
  if (rc) return rc;
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cn_set_error("cn_update_linear_fwd: %s", cudaGetErrorString(e));
  return 0;
}

// Backward of the same layer: dZ = dY o [Y > 0] (act == ReLU), dX = dZ W, dW = dZ^T X, db = colsum(dZ).
// d_dx may be null (first layer of a chain).  d_dw [N, K] and d_db [N] are OVERWRITTEN.
int cn_update_linear_bwd(const float* d_dy, const float* d_y, const void* d_saved, const float* d_w, float* d_dx, float* d_dw,
                         float* d_db, void* d_ws, size_t ws_bytes, int M, int N, int K, int act, int device, void* stream) {
  if (!d_dy || !d_saved || !d_w || !d_dw || !d_ws) return cn_set_error("cn_update_linear_bwd: null argument");
  if (act == 1 && !d_y) return cn_set_error("cn_update_linear_bwd: ReLU layer needs its forward output");
  if (act != 0 && act != 1) return cn_set_error("cn_update_linear_bwd: activation %d unsupported (0 none, 1 ReLU)", act);
  if (M <= 0 || N % 64 || K % 64) return cn_set_error("cn_update_linear_bwd: need M > 0, N %% 64 == 0, K %% 64 == 0");
  if (ws_bytes < cn_update_linear_ws_bytes(M, N, K)) return cn_set_error("cn_update_linear_bwd: workspace too small");
  int rc = setup_device(device);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int Mp = mpad(M);
  Carve c{(unsigned char*)d_ws, 0, ws_bytes};
  unsigned int* amax = (unsigned int*)c.take(64);
  float* sdz = (float*)c.take(64);
  float* sw = (float*)c.take(64);
  __half* zh = (__half*)c.take((size_t)M * N * 2);
  __half* zl = (__half*)c.take((size_t)M * N * 2);
  __half* zTh = (__half*)c.take((size_t)N * Mp * 2);
  __half* zTl = (__half*)c.take((size_t)N * Mp * 2);
  __half* wTh = (__half*)c.take((size_t)K * N * 2);
  __half* wTl = (__half*)c.take((size_t)K * N * 2);
  const unsigned char* sv = (const unsigned char*)d_saved;
  const __half* xTh = (const __half*)sv;
  const __half* xTl = xTh + (size_t)K * Mp;
  const float* sx = (const float*)(sv + up((size_t)2 * K * Mp * 2, 1024));
  const float* mask = act == 1 ? d_y : nullptr;
  run_amax_scale(st, d_dy, mask, (size_t)M * N, amax, sdz);
  double* db64 = (double*)c.take((size_t)N * sizeof(double));
  if (d_db) cudaMemsetAsync(db64, 0, (size_t)N * sizeof(double), st);
  run_split(st, d_dy, N, mask, N, M, N, sdz, d_dx ? zh : nullptr, d_dx ? zl : nullptr, N, zTh, zTl, Mp, d_db ? db64 : nullptr);
  if (d_db) cn_upd_d2f_kernel<<<(N + 255) / 256, 256, 0, st>>>(db64, d_db, N);
  if (d_dx) {
    run_amax_scale(st, d_w, nullptr, (size_t)N * K, amax + 1, sw);
    run_split(st, d_w, K, nullptr, 0, N, K, sw, nullptr, nullptr, 0, wTh, wTl, N, nullptr);     // W^T [K, N]
    rc = gemm_tc_promote(g_dev[device].sms, st, zh, zl, M, N, wTh, wTl, K, N, N, d_dx, K, nullptr, 0, sdz + 1, sw + 1, 1);
    if (rc) return rc;
  }
  // wgrad: dW[N, K] = dZ^T[N, Mp] . X^T[K, Mp]^T, reduction over the rows, split across CTAs
  cudaMemsetAsync(d_dw, 0, (size_t)N * K * sizeof(float), st);
  {
    const int mn = ((N + TC_BM - 1) / TC_BM) * (K / 64);          // output tiles of gemm_tc_promote (64 columns)
    const int kblocks = Mp / TC_BK;
    int ksplit = (g_dev[device].sms + mn - 1) / mn;
    if (ksplit > kblocks) ksplit = kblocks;
    if (ksplit < 1) ksplit = 1;
    // every slice must own at least one k-block (an empty slice would add an uninitialised accumulator):
    // ksplit = ceil(kblocks / ceil(kblocks / ksplit)) has that property; C is zeroed above for the reduce path
    const int kb_per = (kblocks + ksplit - 1) / ksplit;
    ksplit = (kblocks + kb_per - 1) / kb_per;
    rc = gemm_tc_promote(g_dev[device].sms, st, zTh, zTl, N, Mp, xTh, xTl, K, Mp, M, d_dw, K, nullptr, 0, sdz + 1, sx + 1, ksplit);
    if (rc) return rc;
  }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cn_set_error("cn_update_linear_bwd: %s", cudaGetErrorString(e));
  return 0;
}

// replaces (update path): the nn.MultiheadAttention core over the valid humans of every sample.
// d_qkv [Mc,1536]; d_row_start [B+1] (prefix sums of the per-sample human counts), d_row_env [Mc] (sample of a row);
// outputs d_out [Mc,512], d_stats [Mc,16] (soft-max max / sum per head, consumed by the backward).
int cn_update_attn_fwd(const float* d_qkv, const int* d_row_start, const int* d_row_env, int Mc, float* d_out, float* d_stats,
                       int device, void* stream) {
  if (!d_qkv || !d_row_start || !d_row_env || !d_out || !d_stats) return cn_set_error("cn_update_attn_fwd: null argument");
  if (Mc <= 0) return 0;
  int rc = setup_device(device);
  if (rc) return rc;
  int grid = (Mc + CN_UPD_ATTN_WARPS - 1) / CN_UPD_ATTN_WARPS;
  if (grid > g_dev[device].sms * 16) grid = g_dev[device].sms * 16;
  cn_upd_attn_fwd_kernel<<<grid, CN_UPD_ATTN_WARPS * 32, 0, (cudaStream_t)stream>>>(d_qkv, d_row_start, d_row_env, Mc, d_out, d_stats);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cn_set_error("cn_update_attn_fwd: %s", cudaGetErrorString(e));
  return 0;
}

// d_dqkv [Mc,1536] = gradient w.r.t. (q | k | v) given d_dout [Mc,512]; d_delta [Mc,8] is scratch.
int cn_update_attn_bwd(const float* d_qkv, const float* d_out, const float* d_dout, const float* d_stats, const int* d_row_start,
                       const int* d_row_env, int Mc, float* d_dqkv, float* d_delta, int device, void* stream) {
  if (!d_qkv || !d_out || !d_dout || !d_stats || !d_row_start || !d_row_env || !d_dqkv || !d_delta)
    return cn_set_error("cn_update_attn_bwd: null argument");
  if (Mc <= 0) return 0;
  int rc = setup_device(device);
  if (rc) return rc;
  int grid = (Mc + CN_UPD_ATTN_WARPS - 1) / CN_UPD_ATTN_WARPS;
  if (grid > g_dev[device].sms * 16) grid = g_dev[device].sms * 16;
  cudaStream_t st = (cudaStream_t)stream;
  cn_upd_attn_bwd_q_kernel<<<grid, CN_UPD_ATTN_WARPS * 32, 0, st>>>(d_qkv, d_out, d_dout, d_stats, d_row_start, d_row_env, Mc, d_dqkv, d_delta);
  cn_upd_attn_bwd_kv_kernel<<<grid, CN_UPD_ATTN_WARPS * 32, 0, st>>>(d_qkv, d_dout, d_stats, d_delta, d_row_start, d_row_env, Mc, d_dqkv);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cn_set_error("cn_update_attn_bwd: %s", cudaGetErrorString(e));
  return 0;
}

// replaces (update path): the per-step GRU loop of EndRNN / RNNBase._forward_gru with done-mask resets
// (rl/networks/srnn_model.py:49-103) over a [T, N] minibatch.  gi [T,N,384] = W_ih x + b_ih, h0 [N,128], masks [T,N],
// whh [384,128], bhh [384]; out [T,N,128], saved [T,N,512] (r, z, n, gh_n for the backward).
int cn_update_gru_fwd(const float* d_gi, const float* d_h0, const float* d_masks, const float* d_whh, const float* d_bhh, int T, int N,
                      float* d_out, float* d_saved, int device, void* stream) {
  if (!d_gi || !d_h0 || !d_masks || !d_whh || !d_bhh || !d_out || !d_saved) return cn_set_error("cn_update_gru_fwd: null argument");
  if (T <= 0 || N <= 0) return 0;
  int rc = setup_device(device);
  if (rc) return rc;
  static bool attr[64];
  if (!attr[device]) {
    cudaError_t e = cudaFuncSetAttribute(cn_upd_gru_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CN_GRU_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(cn_upd_gru_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CN_GRU_SMEM);
    if (e != cudaSuccess) return cn_set_error("cudaFuncSetAttribute(gru): %s", cudaGetErrorString(e));
    attr[device] = true;
  }
  const int grid = (N + CN_GRU_ROWS - 1) / CN_GRU_ROWS;
  cn_upd_gru_fwd_kernel<<<grid, CN_GRU_THREADS, CN_GRU_SMEM, (cudaStream_t)stream>>>(d_gi, d_h0, d_masks, d_whh, d_bhh, T, N, d_out, d_saved);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cn_set_error("cn_update_gru_fwd: %s", cudaGetErrorString(e));
  return 0;
}

// d_out [T,N,128] (+ optional d_hT [N,128]) -> d_gi [T,N,384], d_ghn [T,N,128], d_h0 [N,128]  (see the kernel comment)
int cn_update_gru_bwd(const float* d_dout, const float* d_dhT, const float* d_out, const float* d_h0, const float* d_masks,
                      const float* d_saved, const float* d_whh, int T, int N, float* d_dgi, float* d_dghn, float* d_dh0, int device,
                      void* stream) {
  if (!d_dout || !d_out || !d_h0 || !d_masks || !d_saved || !d_whh || !d_dgi || !d_dghn || !d_dh0)
    return cn_set_error("cn_update_gru_bwd: null argument");
  if (T <= 0 || N <= 0) return 0;
  int rc = setup_device(device);
  if (rc) return rc;
  const int grid = (N + CN_GRU_ROWS - 1) / CN_GRU_ROWS;
  cn_upd_gru_bwd_kernel<<<grid, CN_GRU_THREADS, CN_GRU_SMEM, (cudaStream_t)stream>>>(d_dout, d_dhT, d_out, d_h0, d_masks, d_saved, d_whh,
                                                                                     T, N, d_dgi, d_dghn, d_dh0);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cn_set_error("cn_update_gru_bwd: %s", cudaGetErrorString(e));
  return 0;
}

}  // extern "C"
