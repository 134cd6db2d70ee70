// Device kernels of the attention-graph policy forward (rollout / infer=True path):
//   rl/networks/selfAttn_srnn_temp_node.py:360-449 (selfAttn_merge_SRNN.forward)
//   rl/networks/selfAttn_srnn_temp_node.py:63-91   (SpatialEdgeSelfAttn, nn.MultiheadAttention 8 heads)
//   rl/networks/selfAttn_srnn_temp_node.py:145-223 (EdgeAttention_M)
//   rl/networks/selfAttn_srnn_temp_node.py:262-285 + srnn_model.py:35-47 (EndRNN / GRU step)
//   rl/networks/distributions.py:76-95,36-44       (DiagGaussian / FixedNormal)
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "cn_launch.cuh"

// ------------------------------------------------------------------------------------------
// fp32 CUDA-core GEMM:  C[M,N] = act(A[M,K] * W[N,K]^T + bias[N]),  act on columns [act_lo, act_hi).
// 128x128x16 tiles, 256 threads, 8x8 register tile per thread, register-prefetched double
// buffering through shared memory.  K % 16 == 0 (buffers are zero padded), M and N ragged.
#define CN_GEMM_BM 128
#define CN_GEMM_BN 128
#define CN_GEMM_BK 16
#define CN_GEMM_PAD 4

__device__ __forceinline__ float cn_apply_act(float v, int act) {
  if (act == CN_ACT_RELU) return v > 0.0f ? v : 0.0f;
  if (act == CN_ACT_TANH) return tanhf(v);
  return v;
}

__global__ void __launch_bounds__(256) cn_gemm_f32_kernel(const float* __restrict__ A, int lda,
                                                          const float* __restrict__ W, int ldw,
                                                          const float* __restrict__ bias, float* __restrict__ Cout,
                                                          int ldc, int M, int N, int K, int act, int act_lo,
                                                          int act_hi, const int* __restrict__ m_ptr,
                                                          __half* __restrict__ out_hi, __half* __restrict__ out_lo) {
  cn_pdl_prologue();
  // m_ptr: optional device-side row count (compacted human rows); tiles past it exit immediately
  if (m_ptr) { const int mc = *m_ptr; M = mc < M ? mc : M; }
  if ((int)(blockIdx.y * CN_GEMM_BM) >= M) return;
  __shared__ __align__(16) float As[2][CN_GEMM_BK][CN_GEMM_BM + CN_GEMM_PAD];
  __shared__ __align__(16) float Bs[2][CN_GEMM_BK][CN_GEMM_BN + CN_GEMM_PAD];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * CN_GEMM_BM, n0 = blockIdx.x * CN_GEMM_BN;
  const int tx = tid & 15, ty = tid >> 4;
  // global -> register staging: each thread moves two float4 of A and two of W per k-tile
  const int lrow = tid >> 2;          // 0..63
  const int lk = (tid & 3) * 4;       // 0,4,8,12
  float4 ra[2], rb[2];
  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int m = m0 + lrow + i * 64;
      ra[i] = (m < M) ? *reinterpret_cast<const float4*>(A + (size_t)m * lda + k0 + lk) : make_float4(0, 0, 0, 0);
      const int n = n0 + lrow + i * 64;
      rb[i] = (n < N) ? *reinterpret_cast<const float4*>(W + (size_t)n * ldw + k0 + lk) : make_float4(0, 0, 0, 0);
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int r = lrow + i * 64;
      As[buf][lk + 0][r] = ra[i].x; As[buf][lk + 1][r] = ra[i].y; As[buf][lk + 2][r] = ra[i].z; As[buf][lk + 3][r] = ra[i].w;
      Bs[buf][lk + 0][r] = rb[i].x; Bs[buf][lk + 1][r] = rb[i].y; Bs[buf][lk + 2][r] = rb[i].z; Bs[buf][lk + 3][r] = rb[i].w;
    }
  };
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;

  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  const int nk = K / CN_GEMM_BK;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * CN_GEMM_BK);
#pragma unroll
    for (int k = 0; k < CN_GEMM_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      store_tiles(buf ^ 1);
      __syncthreads();
    }
  }
  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int nb = n0 + (jj == 0 ? tx * 4 : 64 + tx * 4);
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = nb + j;
        float x = acc[i][jj * 4 + j];
        if (n < N) {
          if (bias) x += bias[n];
          if (n >= act_lo && n < act_hi) x = cn_apply_act(x, act);
        }
        v[j] = x;
      }
      if (out_hi) {    // (hi, lo) fp16 split for the tensor-core consumer; same leading dimension
        if (nb + 3 < N && ((ldc & 3) == 0)) {
          uint32_t ph[2], pl[2];
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const float c0 = fminf(fmaxf(v[2 * t], -65504.0f), 65504.0f), c1 = fminf(fmaxf(v[2 * t + 1], -65504.0f), 65504.0f);
            const __half h0 = __float2half_rn(c0), h1 = __float2half_rn(c1);
            const __half l0 = __float2half_rn(c0 - __half2float(h0)), l1 = __float2half_rn(c1 - __half2float(h1));
            ph[t] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
            pl[t] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
          }
          *reinterpret_cast<uint2*>(out_hi + (size_t)m * ldc + nb) = make_uint2(ph[0], ph[1]);
          *reinterpret_cast<uint2*>(out_lo + (size_t)m * ldc + nb) = make_uint2(pl[0], pl[1]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (nb + j < N) {
              const float c = fminf(fmaxf(v[j], -65504.0f), 65504.0f);
              const __half hh = __float2half_rn(c);
              out_hi[(size_t)m * ldc + nb + j] = hh;
              out_lo[(size_t)m * ldc + nb + j] = __float2half_rn(c - __half2float(hh));
            }
        }
        if (!Cout) continue;
      }
      float* dst = Cout + (size_t)m * ldc + nb;
      if (nb + 3 < N && ((ldc & 3) == 0)) {
        *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (nb + j < N) dst[j] = v[j];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Weight folding at parameter-load time (fp64 accumulate):  C[m,n] = sum_k A[m,k] * B[k,n]
// and  c[m] = sum_k A[m,k] * b[k] + d[m].   Not on the rollout path.
__global__ void cn_fold_mm_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ Cm,
                                  int M, int N, int K) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
  if (n >= N || m >= M) return;
  double acc = 0.0;
  for (int k = 0; k < K; ++k) acc += (double)A[(size_t)m * K + k] * (double)B[(size_t)k * N + n];
  Cm[(size_t)m * N + n] = (float)acc;
}
__global__ void cn_fold_mv_kernel(const float* __restrict__ A, const float* __restrict__ b, const float* __restrict__ d,
                                  float* __restrict__ c, int M, int K) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= M) return;
  double acc = d ? (double)d[m] : 0.0;
  for (int k = 0; k < K; ++k) acc += (double)A[(size_t)m * K + k] * (double)b[k];
  c[m] = (float)acc;
}

// ------------------------------------------------------------------------------------------
// Row compaction.  Humans are sorted by distance and rows j >= n_e = detected_human_num[e] are
// padding: as attention KEYS they are masked (key_padding_mask), and as attention QUERIES their
// outputs only reach the robot-human softmax, where masked_fill(-1e9) gives them weight exactly 0
// (selfAttn_srnn_temp_node.py:49-60,165-170).  They cannot influence any output, so the per-human
// pipeline runs on the compacted valid rows only:  row_start[e] = sum_{e' < e} n_e',  *mc = total.
// Single CTA, 1024 threads, chunked inclusive scan (N <= a few 10^4).
__global__ void __launch_bounds__(1024) cn_row_offsets_kernel(const float* __restrict__ detected, int N, int H,
                                                              int* __restrict__ row_start, int* __restrict__ mc) {
  cn_pdl_prologue();
  __shared__ int warp_sums[32];
  __shared__ int carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < N; base += 1024) {
    const int e = base + tid;
    int n = 0;
    if (e < N) { n = (int)detected[e]; n = n < 1 ? 1 : (n > H ? H : n); }
    int x = n;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = warp_sums[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += y; }
      warp_sums[lane] = w;
    }
    __syncthreads();
    const int incl = x + (warp > 0 ? warp_sums[warp - 1] : 0) + carry;
    if (e < N) row_start[e] = incl - n;
    __syncthreads();
    if (tid == 1023) carry = incl;
    __syncthreads();
  }
  if (tid == 0) { *mc = carry; row_start[N] = carry; }
}

// Row compaction by the visible mask (sort_humans = False, selfAttn_srnn_temp_node.py:375-383): the attention masks
// are visible_masks, in slot (human id) order and not a prefix.  The argument above holds for any mask, so only the
// choice of rows changes.  One warp per environment: slot_tab[e * H + k] = the k-th visible slot in ascending order
// (ballot + popc of the lower lanes per 32 slots) and count[e] = the number of visible slots, as a float so that
// cn_row_offsets_kernel scans it as it scans detected_human_num.  An environment with no visible human keeps slot 0
// only (the reference's dummy_human_mask, :351-358, :382-383).
__global__ void __launch_bounds__(256) cn_mask_slots_kernel(const uint8_t* vis /* [N, H], nonzero = visible */, int N,
                                                            int H, float* __restrict__ count, int* __restrict__ slot_tab) {
  cn_pdl_prologue();
  const int lane = threadIdx.x & 31;
  const int e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (e >= N) return;
  const uint8_t* m = vis + (size_t)e * H;
  int* tab = slot_tab + (size_t)e * H;
  int n = 0;
  for (int s0 = 0; s0 < H; s0 += 32) {
    const int s = s0 + lane;
    const bool v = s < H && m[s] != 0;
    const unsigned b = __ballot_sync(0xffffffffu, v);
    if (v) tab[n + __popc(b & ((1u << lane) - 1u))] = s;
    n += __popc(b);
  }
  if (lane == 0) {
    if (n == 0) { tab[0] = 0; n = 1; }
    count[e] = (float)n;
  }
}

// Input packing: x16[row_start[e] + j, 16] = spatial_edges[e, s] zero-padded to K=16 for j < n_e, with s = j
// (kSlot false: the first n_e rows, sorted humans) or s = slot_tab[e * H + j] (kSlot true: the visible slots, and
// row_slot[row_start[e] + j] = s); xr[N,16] = cat(temporal_edges(2), robot_node(7)) zero padded; h0 = h_in * mask.
template <bool kSlot>
__global__ void cn_pack_inputs_kernel(const float* __restrict__ spatial, int Win, int H, int N,
                                      const int* __restrict__ row_start, int* __restrict__ row_env,
                                      const int* __restrict__ slot_tab, int* __restrict__ row_slot,
                                      float* __restrict__ x16,
                                      const float* __restrict__ temporal, const float* __restrict__ robot,
                                      const float* __restrict__ h_in, const float* __restrict__ masks,
                                      float* __restrict__ xr, float* __restrict__ h0, __half* __restrict__ h0_hi,
                                      __half* __restrict__ h0_lo) {
  cn_pdl_prologue();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (x16 && idx < N * H * 16) {
    const int r = idx >> 4, c = idx & 15;
    const int e = r / H, j = r - e * H;
    const int rs = row_start[e], n = row_start[e + 1] - rs;
    if (j < n) {
      const int s = kSlot ? slot_tab[r] : j;
      x16[(size_t)(rs + j) * 16 + c] = c < Win ? spatial[((size_t)e * H + s) * Win + c] : 0.0f;
      if (c == 0) {
        row_env[rs + j] = e;
        if (kSlot) row_slot[rs + j] = s;
      }
    }
  }
  if (!x16 && idx < N) {                  // tensor-core mode: row -> environment (and slot) map of the compacted rows
    const int rs = row_start[idx], n = row_start[idx + 1] - rs;
    for (int j = 0; j < n; ++j) {
      row_env[rs + j] = idx;
      if (kSlot) row_slot[rs + j] = slot_tab[(size_t)idx * H + j];
    }
  }
  if (idx < N * 16) {
    const int e = idx >> 4, c = idx & 15;
    float v = 0.0f;
    if (c < 2) v = temporal[2 * e + c];
    else if (c < 9) v = robot[7 * e + (c - 2)];
    xr[idx] = v;
  }
  if (idx < N * 128) {
    const float hv = h_in[idx] * masks[idx >> 7];
    h0[idx] = hv;
    if (h0_hi) {
      const float c = fminf(fmaxf(hv, -65504.0f), 65504.0f);
      const __half hh = __float2half_rn(c);
      h0_hi[idx] = hh;
      h0_lo[idx] = __float2half_rn(c - __half2float(hh));
    }
  }
}

// ------------------------------------------------------------------------------------------
// First embedding layer of the human-human branch fused with the row compaction gather (tensor-core
// mode): e1[row_start[e] + j] = relu(W1 spatial_edges[e, j] + b1) for j < n_e, written directly as the
// fp16 (hi, lo) A operand of the next tensor-core GEMM.  K = input width (12 or 2) is far too small for a
// tensor-core tile: one warp per compacted human row, lane l owns outputs 4l..4l+3, the 128 x 16 weights sit
// transposed in shared memory (conflict-free LDS.128), the input row is broadcast by shuffles, and each lane
// issues one 8-byte store per half (256 B coalesced per warp).  Latency bound: sized for many resident warps.
// kSlot: row r gathers slot row_slot[r] (visible-mask compaction) instead of slot r - row_start[e].
template <bool kSlot>
__global__ void __launch_bounds__(256) cn_embed1_kernel(const float* __restrict__ spatial, int Win, int H,
                                                        const int* __restrict__ row_start, const int* __restrict__ row_env,
                                                        const int* __restrict__ row_slot,
                                                        const int* __restrict__ mc_ptr,
                                                        const float* __restrict__ W1 /* [128][16], zero padded */,
                                                        const float* __restrict__ b1, __half* __restrict__ e_hi,
                                                        __half* __restrict__ e_lo /* [Mc,128] */) {
  cn_pdl_prologue();
  __shared__ __align__(16) float ws[16][128];        // transposed weights: ws[c][out]
  for (int i = threadIdx.x; i < 128 * 16; i += blockDim.x) ws[i & 15][i >> 4] = W1[i];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  const float4 b = __ldg(reinterpret_cast<const float4*>(b1) + lane);
  const int mc = *mc_ptr;
  for (int r = gw; r < mc; r += nw) {
    const int e = row_env[r];
    const int j = kSlot ? row_slot[r] : r - row_start[e];
    const float x = lane < Win ? __ldg(spatial + ((size_t)e * H + j) * Win + lane) : 0.0f;
    float acc[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const float xc = __shfl_sync(0xffffffffu, x, c);
      const float4 w = *reinterpret_cast<const float4*>(&ws[c][4 * lane]);
      acc[0] = fmaf(xc, w.x, acc[0]); acc[1] = fmaf(xc, w.y, acc[1]);
      acc[2] = fmaf(xc, w.z, acc[2]); acc[3] = fmaf(xc, w.w, acc[3]);
    }
    const float bb[4] = {b.x, b.y, b.z, b.w};
    uint32_t ph[2], pl[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      float c0 = acc[2 * t] + bb[2 * t], c1 = acc[2 * t + 1] + bb[2 * t + 1];
      c0 = fminf(fmaxf(c0, 0.0f), 65504.0f); c1 = fminf(fmaxf(c1, 0.0f), 65504.0f);       // ReLU + fp16 range
      const __half h0 = __float2half_rn(c0), h1 = __float2half_rn(c1);
      const __half l0 = __float2half_rn(c0 - __half2float(h0)), l1 = __float2half_rn(c1 - __half2float(h1));
      ph[t] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
      pl[t] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
    }
    const size_t o = (size_t)r * 128 + 4 * lane;
    *reinterpret_cast<uint2*>(e_hi + o) = make_uint2(ph[0], ph[1]);
    *reinterpret_cast<uint2*>(e_lo + o) = make_uint2(pl[0], pl[1]);
  }
}

// ------------------------------------------------------------------------------------------
// Human-human multi-head self attention over the compacted rows.
// qkv: [Mc, 1536] rows = (q | k | v), head hd uses columns hd*64..hd*64+63 of each third.
// Only valid humans have rows (keys j >= n_e of the reference's key_padding_mask do not exist here).
//
// One WARP per query row, all 8 heads at once.  Every 512-float q / k / v / o row is touched with four
// fully coalesced LDG.128 per warp: lane l owns float4 #(l + 32 c), c = 0..3, i.e. elements
// 128 c + 4 l .. + 3, which belong to head 2 c + (l >= 16).  The kernel was instruction-issue bound
// (ncu: 3 200 warp instructions per query, 59 % issue active) on redundant work: every lane reduced and
// exponentiated all four of its heads.  Now
//  * the four per-lane partial dot products are reduced over the 16 lanes of a half with a PACKED
//    butterfly (2 + 1 + 2 shuffles instead of 16): afterwards lane l holds the complete score of ONE
//    head chunk own = 2 (l & 1) + ((l >> 1) & 1), so each lane exponentiates one head, not four;
//  * soft-max is two-pass (pass 1: scores -> shared memory + running max; pass 2: p = exp(s - max),
//    P V): one exp per (key, head) and no rescaling of the accumulators;
//  * the p of the other three chunks come from the neighbouring lanes of the aligned 4-lane group.
//  * template parameter R: R query rows of the SAME environment share every K / V row a warp loads (each loaded
//    element then feeds R FMAs).  At 4096 envs and H = 20 (about 4 keys per query) R = 1 is the fastest of the
//    three -- the L1 delivery rate (one FMA per 4 bytes) is not what limits the kernel, the extra registers cost
//    occupancy.  At H = 50 and 100 R = 2 is faster (0.219 against 0.232-0.235 ms, 0.663 against 0.772-0.776 ms;
//    DESIGN.md §3.4c).  R = 1 is the default; CN_ATTN_R selects the others.
#define CN_ATTN_WARPS 4
#define CN_ATTN_MAXKEYS 128
template <int R, int KB /* keys whose rows are in flight together */, int W /* warps per CTA */>
__global__ void __launch_bounds__(W * 32) cn_hh_attention_kernel(const float* __restrict__ qkv,
                                                                             const int* __restrict__ row_start,
                                                                             const int* __restrict__ row_env,
                                                                             const int* __restrict__ mc_ptr,
                                                                             const int* __restrict__ r0_ptr /* first row or null */,
                                                                             float* __restrict__ out /* [Mc,512] or null */,
                                                                             __half* __restrict__ out_hi,
                                                                             __half* __restrict__ out_lo) {
  cn_pdl_prologue();
  __shared__ float sc[W][R][CN_ATTN_MAXKEYS][8];                // scores [query][key][half * 4 + chunk]
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int mc = cn_ld_after_wait(mc_ptr);
  const int nwarps = gridDim.x * W;
  const float scale = 0.125f;   // 1/sqrt(head_dim = 64); torch scales q before q k^T
  const bool b0 = (lane & 1) != 0, b1 = (lane & 2) != 0;
  const int own = (b0 ? 2 : 0) + (b1 ? 1 : 0);                  // head chunk this lane finishes
  const int col = ((lane >> 4) << 2) + own;                     // its column in sc[][][][8]
  const int grp = lane & ~3;
  // grid-stride over the compacted rows: the launch is sized to the machine, not to the worst case.  The warp that
  // meets the first row of a group of R consecutive queries of an environment does the whole group.
  const int r_first = r0_ptr ? cn_ld_after_wait(r0_ptr) : 0;   // row chunk [r_first, mc) of this launch
  for (int r = r_first + blockIdx.x * W + warp; r < mc; r += nwarps) {
    const int e = row_env[r];
    const int row0 = row_start[e];
    const int n = row_start[e + 1] - row0;
    if ((r - row0) % R != 0) continue;
    const int nq = (row0 + n - r) < R ? (row0 + n - r) : R;     // queries r .. r + nq - 1 (warp-uniform)
    float4 q[R][4];
#pragma unroll
    for (int u = 0; u < R; ++u) {
      const int ru = u < nq ? r + u : r;                        // a missing query repeats the first (results dropped)
      const float4* qv = reinterpret_cast<const float4*>(qkv + (size_t)ru * 1536) + lane;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const float4 a = __ldg(qv + 32 * c);
        q[u][c] = make_float4(a.x * scale, a.y * scale, a.z * scale, a.w * scale);
      }
    }
    // ---- pass 1: scores.  Keys are processed in blocks of KB with all of a block's K rows requested before the
    // first is used (memory-level parallelism).
    float m[R];
#pragma unroll
    for (int u = 0; u < R; ++u) m[u] = -INFINITY;
    for (int jb = 0; jb < n; jb += KB) {
      float4 kr[KB][4];
#pragma unroll
      for (int t = 0; t < KB; ++t) {
        const int j = (jb + t < n) ? jb + t : n - 1;             // clamped: the duplicate load hits L1
        const float4* kv = reinterpret_cast<const float4*>(qkv + (size_t)(row0 + j) * 1536 + 512) + lane;
#pragma unroll
        for (int c = 0; c < 4; ++c) kr[t][c] = __ldg(kv + 32 * c);
      }
#pragma unroll
      for (int t = 0; t < KB; ++t) {
        if (jb + t < n) {                                        // warp-uniform
#pragma unroll
          for (int u = 0; u < R; ++u) {
            float s[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              float x = q[u][c].x * kr[t][c].x;
              x = fmaf(q[u][c].y, kr[t][c].y, x); x = fmaf(q[u][c].z, kr[t][c].z, x); x = fmaf(q[u][c].w, kr[t][c].w, x);
              s[c] = x;
            }
            // packed butterfly over the 16 lanes of the half: 4 values -> 1 per lane
            const float x0 = b0 ? s[0] : s[2], x1 = b0 ? s[1] : s[3];               // what the xor-1 partner keeps
            const float r0 = __shfl_xor_sync(0xffffffffu, x0, 1), r1 = __shfl_xor_sync(0xffffffffu, x1, 1);
            const float u0 = (b0 ? s[2] : s[0]) + r0, u1 = (b0 ? s[3] : s[1]) + r1; // chunks (2 b0, 2 b0 + 1) over 2 lanes
            const float y = b1 ? u0 : u1;
            float v = (b1 ? u1 : u0) + __shfl_xor_sync(0xffffffffu, y, 2);          // chunk `own` over 4 lanes
            v += __shfl_xor_sync(0xffffffffu, v, 4);
            v += __shfl_xor_sync(0xffffffffu, v, 8);                                // ... over the 16 lanes of the half
            m[u] = fmaxf(m[u], v);
            if ((lane & 12) == 0) sc[warp][u][jb + t][col] = v;                     // lanes 0-3 and 16-19
          }
        }
      }
    }
    __syncwarp();
    // ---- pass 2: p = exp(s - max), accumulate P V
    float4 acc[R][4];
    float l[R];
#pragma unroll
    for (int u = 0; u < R; ++u) {
      l[u] = 0.0f;
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[u][c] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    }
    for (int jb = 0; jb < n; jb += KB) {
      float4 vr[KB][4];
#pragma unroll
      for (int t = 0; t < KB; ++t) {
        const int j = (jb + t < n) ? jb + t : n - 1;
        const float4* vv = reinterpret_cast<const float4*>(qkv + (size_t)(row0 + j) * 1536 + 1024) + lane;
#pragma unroll
        for (int c = 0; c < 4; ++c) vr[t][c] = __ldg(vv + 32 * c);
      }
#pragma unroll
      for (int t = 0; t < KB; ++t) {
        if (jb + t < n) {
#pragma unroll
          for (int u = 0; u < R; ++u) {
            const float p = expf(sc[warp][u][jb + t][col] - m[u]);
            l[u] += p;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              // chunk c was finished by the lane of this 4-lane group with (b0, b1) = (c >> 1, c & 1)
              const float pc = __shfl_sync(0xffffffffu, p, grp | (c >> 1) | ((c & 1) << 1));
              acc[u][c].x = fmaf(pc, vr[t][c].x, acc[u][c].x); acc[u][c].y = fmaf(pc, vr[t][c].y, acc[u][c].y);
              acc[u][c].z = fmaf(pc, vr[t][c].z, acc[u][c].z); acc[u][c].w = fmaf(pc, vr[t][c].w, acc[u][c].w);
            }
          }
        }
      }
    }
    __syncwarp();                                      // sc is reused by this warp's next group
#pragma unroll
    for (int u = 0; u < R; ++u) {
      if (u < nq) {                                    // warp-uniform
        const float linv = 1.0f / l[u];
        float4 a[4];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const float inv = __shfl_sync(0xffffffffu, linv, grp | (c >> 1) | ((c & 1) << 1));
          a[c] = make_float4(acc[u][c].x * inv, acc[u][c].y * inv, acc[u][c].z * inv, acc[u][c].w * inv);
        }
        if (out) {
          float4* dst = reinterpret_cast<float4*>(out + (size_t)(r + u) * 512) + lane;
#pragma unroll
          for (int c = 0; c < 4; ++c) dst[32 * c] = a[c];
        }
        if (out_hi) {     // (hi, lo) fp16 split = A operand of the tensor-core out-projection
          uint2* dh = reinterpret_cast<uint2*>(out_hi + (size_t)(r + u) * 512) + lane;
          uint2* dl = reinterpret_cast<uint2*>(out_lo + (size_t)(r + u) * 512) + lane;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const float cv[4] = {fminf(fmaxf(a[c].x, -65504.0f), 65504.0f), fminf(fmaxf(a[c].y, -65504.0f), 65504.0f),
                                 fminf(fmaxf(a[c].z, -65504.0f), 65504.0f), fminf(fmaxf(a[c].w, -65504.0f), 65504.0f)};
            uint32_t ph[2], pl[2];
#pragma unroll
            for (int w = 0; w < 2; ++w) {
              const __half h0 = __float2half_rn(cv[2 * w]), h1 = __float2half_rn(cv[2 * w + 1]);
              const __half l0 = __float2half_rn(cv[2 * w] - __half2float(h0)), l1 = __float2half_rn(cv[2 * w + 1] - __half2float(h1));
              ph[w] = (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
              pl[w] = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
            }
            dh[32 * c] = make_uint2(ph[0], ph[1]);
            dl[32 * c] = make_uint2(pl[0], pl[1]);
          }
        }
      }
    }
  }   // row loop
}

// ------------------------------------------------------------------------------------------
// Robot-human attention (EdgeAttention_M.att_func) for one environment per warp:
//   score_j = <W_t robot + b_t, W_s s_j + b_s> * (H / sqrt(64))  ==  (u . s_j + cst) * H/8
// with u = W_s^T te (precomputed by a GEMM), cst = <b_s, te>;  masked_fill(-1e9) for j >= n_e;
// softmax over all H; weighted sum of the 256-d human features.
// Row layouts of s_out (kDense): compacted (false: rows row_start[e] .. row_start[e + 1] - 1 of environment e, the
// rest masked; env_pitch, env_off and ldwh unused, wv_hi / wv_lo have row pitch 256), or dense without a mask (true:
// the H rows e * env_pitch + env_off + j, j < H, DS-RNN's spatial edge states inside its [N, H + 1, 256] edge state,
// srnn_model.py:256-323; row_start unused, wv_hi / wv_lo have row pitch ldwh).  A template, so that the compacted
// instance compiles to the same code as before the dense layout existed (a run-time switch cost 16 us per rollout
// step at N = 4096, H = 20 on an H100).  cn_policy.cu launches the dense instance for cn_dsrnn.cu.
template <bool kDense>
__global__ void __launch_bounds__(128) cn_hr_attention_kernel(const float* __restrict__ s_out /* [*,256] */,
                                                              const float* __restrict__ u /* [N,256] */,
                                                              const float* __restrict__ te /* [N, ldte] cols te_off.. */,
                                                              int ldte, int te_off, const float* __restrict__ b_s,
                                                              const int* __restrict__ row_start, int env_pitch,
                                                              int env_off, int N, int H,
                                                              float* __restrict__ wv /* [N,256] */,
                                                              __half* __restrict__ wv_hi, __half* __restrict__ wv_lo,
                                                              int ldwh) {
  cn_pdl_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.x * 4 + warp;
  if (e >= N) return;
  const size_t row0 = kDense ? (size_t)e * env_pitch + env_off : (size_t)row_start[e];
  const int n = kDense ? H : row_start[e + 1] - row_start[e];
  float ur[8];
#pragma unroll
  for (int t = 0; t < 8; ++t) ur[t] = u[(size_t)e * 256 + lane + 32 * t];
  float cst = b_s[lane] * te[(size_t)e * ldte + te_off + lane] + b_s[lane + 32] * te[(size_t)e * ldte + te_off + lane + 32];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cst += __shfl_xor_sync(0xffffffffu, cst, o);
  const float temperature = (float)H / 8.0f;
  // scores for valid humans; lanes cooperate on each 256-d dot product
  float sc[4] = {-1e9f, -1e9f, -1e9f, -1e9f};   // lane holds score of human lane + 32 t
  for (int j = 0; j < n; ++j) {
    const float* sr = s_out + (row0 + j) * 256;
    float d = 0.0f;
#pragma unroll
    for (int t = 0; t < 8; ++t) d = fmaf(ur[t], sr[lane + 32 * t], d);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    const float s = (d + cst) * temperature;
    if ((j & 31) == lane) sc[j >> 5] = s;
  }
  float mx = -INFINITY;
#pragma unroll
  for (int t = 0; t < 4; ++t) if (lane + 32 * t < H) mx = fmaxf(mx, sc[t]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.0f;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    sc[t] = (lane + 32 * t < H) ? expf(sc[t] - mx) : 0.0f;   // masked entries: exp(-1e9 - mx) == 0
    sum += sc[t];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float inv = 1.0f / sum;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < n; ++j) {
    const float pj = __shfl_sync(0xffffffffu, sc[j >> 5], j & 31) * inv;
    const float* sr = s_out + (row0 + j) * 256;
#pragma unroll
    for (int t = 0; t < 8; ++t) acc[t] = fmaf(pj, sr[lane + 32 * t], acc[t]);
  }
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const size_t o = (size_t)e * 256 + lane + 32 * t;
    wv[o] = acc[t];
    if (wv_hi) {
      const float c = fminf(fmaxf(acc[t], -65504.0f), 65504.0f);
      const __half hh = __float2half_rn(c);
      const size_t oh = (size_t)e * (kDense ? ldwh : 256) + lane + 32 * t;
      wv_hi[oh] = hh;
      wv_lo[oh] = __float2half_rn(c - __half2float(hh));
    }
  }
}

// ------------------------------------------------------------------------------------------
// GRU cell gates (PyTorch order r, z, n; h' = (1 - z) * n + z * h), one thread per (env, unit).
__device__ __forceinline__ float cn_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

__global__ void cn_gru_gate_kernel(const float* __restrict__ gi, const float* __restrict__ gh,
                                   const float* __restrict__ h0, int N, float* __restrict__ h1,
                                   __half* __restrict__ h1_hi, __half* __restrict__ h1_lo) {
  cn_pdl_prologue();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= N * 128) return;
  const int e = idx >> 7, c = idx & 127;
  const float* a = gi + (size_t)e * 384;
  const float* b = gh + (size_t)e * 384;
  const float r = cn_sigmoid(a[c] + b[c]);
  const float z = cn_sigmoid(a[128 + c] + b[128 + c]);
  const float n = tanhf(a[256 + c] + r * b[256 + c]);
  const float hv = (1.0f - z) * n + z * h0[idx];
  h1[idx] = hv;
  if (h1_hi) {       // (hi, lo) fp16 split for the tensor-core output_linear
    const __half hh = __float2half_rn(hv);
    h1_hi[idx] = hh;
    h1_lo[idx] = __float2half_rn(hv - __half2float(hh));
  }
}

// ------------------------------------------------------------------------------------------
// Output heads, one warp per environment: value = critic_linear(hc); mean = fc_mean(ha);
// action = mean + exp(logstd) * noise (torch.normal = randn * std + mean); log-prob summed.
__global__ void __launch_bounds__(128) cn_heads_kernel(const float* __restrict__ ha, int ldha,
                                                       const float* __restrict__ hc, int ldhc,
                                                       const float* __restrict__ w_v, const float* __restrict__ b_v,
                                                       const float* __restrict__ w_m, const float* __restrict__ b_m,
                                                       const float* __restrict__ logstd,
                                                       const float* __restrict__ noise, int N,
                                                       float* __restrict__ value, float* __restrict__ action,
                                                       float* __restrict__ logp, float* __restrict__ mean_out) {
  cn_pdl_prologue();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = blockIdx.x * 4 + warp;
  if (e >= N) return;
  float v = 0.0f, m0 = 0.0f, m1 = 0.0f;
#pragma unroll
  for (int t = 0; t < 8; ++t) {
    const int c = lane + 32 * t;
    const float a = ha[(size_t)e * ldha + c], cc = hc[(size_t)e * ldhc + c];
    v = fmaf(cc, w_v[c], v);
    m0 = fmaf(a, w_m[c], m0);
    m1 = fmaf(a, w_m[256 + c], m1);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    v += __shfl_xor_sync(0xffffffffu, v, o);
    m0 += __shfl_xor_sync(0xffffffffu, m0, o);
    m1 += __shfl_xor_sync(0xffffffffu, m1, o);
  }
  if (lane == 0) {
    v += b_v[0]; m0 += b_m[0]; m1 += b_m[1];
    value[e] = v;
    if (mean_out) { mean_out[2 * e] = m0; mean_out[2 * e + 1] = m1; }
    const float ls0 = logstd[0], ls1 = logstd[1];
    const float s0 = expf(ls0), s1 = expf(ls1);
    float a0 = m0, a1 = m1;
    if (noise) {
      a0 = __fadd_rn(__fmul_rn(noise[2 * e], s0), m0);
      a1 = __fadd_rn(__fmul_rn(noise[2 * e + 1], s1), m1);
    }
    action[2 * e] = a0; action[2 * e + 1] = a1;
    // Normal.log_prob: -((x - mu)^2) / (2 var) - log(std) - log(sqrt(2 pi))
    const float c = 0.91893853320467274178f;
    const float d0 = a0 - m0, d1 = a1 - m1;
    const float l0 = -(d0 * d0) / (2.0f * (s0 * s0)) - logf(s0) - c;   // log_scale = scale.log()
    const float l1 = -(d1 * d1) / (2.0f * (s1 * s1)) - logf(s1) - c;
    logp[e] = l0 + l1;
  }
}
