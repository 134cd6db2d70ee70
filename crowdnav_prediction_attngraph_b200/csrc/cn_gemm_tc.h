// Host API of the wgmma 3xFP16 GEMM (cn_gemm_tc.cuh); cn_gemm_tc.cu is the only translation unit that instantiates
// cn_gemm_tc_kernel.  The rollout (policy, GST predictor) keeps its operands as split fp16 matrices with prebuilt TMA
// maps (TcMat) and launches through gemm_tc; the PPO update launches the PROMOTE instance through gemm_tc_promote.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "cn_gemm_tc.cuh"
#include "cn_launch.cuh"

// TMA store map of an output of the BN = 256 GEMM instances: [rows, cols], boxes of 64 rows x 128 bytes, 128-byte
// swizzle (cn_gemm_tc.cuh, tc_epilogue_tma).  rows = 0: no map (TMA needs a 16-byte-aligned base and a row pitch that
// is a multiple of 16 bytes).
struct TcStoreMap {
  CUtensorMap map;
  int rows = 0, cols = 0;
};

// A split-fp16 matrix [rows, K] (row pitch `pitch` elements) and its TMA descriptors.
struct TcMat {
  __half *hi = nullptr, *lo = nullptr;
  CUtensorMap mh, ml;
  int pitch = 0;
  int box_k = 0;   // k width of the TMA box of mh / ml: the k-block of the GEMM instance that reads it
  TcStoreMap sh, sl;   // store maps of hi / lo, for a BN = 256 GEMM that writes this matrix
};

// Outputs of one gemm_tc launch.  The BN = 256 instances store through TMA: each output they write needs its store map
// (sc for c32, sh / sl for oh / ol), built where the buffer is allocated, of [M rows, N columns].
struct TcOut {
  float* c32 = nullptr; int ldc = 0;
  __half *oh = nullptr, *ol = nullptr; int ldh = 0;
  const TcStoreMap *sc = nullptr, *sh = nullptr, *sl = nullptr;
};
inline TcOut out32(float* c, int ldc, const TcStoreMap* sc = nullptr) { TcOut o; o.c32 = c; o.ldc = ldc; o.sc = sc; return o; }
inline TcOut out16(const TcMat& t) { TcOut o; o.oh = t.hi; o.ol = t.lo; o.ldh = t.pitch; o.sh = &t.sh; o.sl = &t.sl; return o; }
inline TcOut out_both(float* c, int ldc, const TcMat& t) { TcOut o = out16(t); o.c32 = c; o.ldc = ldc; return o; }

// k width of the TMA boxes of the GEMM instance with B-tile rows bn (32 for BN = 256, 64 for BN = 64)
inline int tc_box_k(int bn) { return bn == 256 ? TcCfg<256>::kBK : TcCfg<64>::kBK; }

// TMA can store a box into a matrix with this base and row pitch (bytes)
inline bool tma_store_ok(const void* ptr, size_t pitch_bytes) { return ((uintptr_t)ptr % 16) == 0 && pitch_bytes % 16 == 0; }

// 2-D fp16 row-major [rows, K] tensor with row pitch `pitch`, box = 64 (K) x box_rows, 128-byte swizzle
// (box_k = 32: 64-byte rows with SWIZZLE_64B, the half-width K blocks of cn_qkv_attn.cuh); elements past the extent
// load as zeros
int make_map(CUtensorMap* map, const __half* ptr, int rows, int K, int box_rows, int pitch, int box_k = TC_BK);
// store map of a BN = 256 output: fp32 (esize 4) or fp16 (esize 2) [rows, cols], row pitch `pitch` elements
int make_store_map(TcStoreMap* s, const void* ptr, int esize, int rows, int cols, int pitch);
// allocate a split matrix [rows, K] in the context and build its maps (box_rows = 128 for A operands, BN for B operands;
// box_k = tc_box_k(BN) of the instance that reads it)
int tc_alloc(CnLaunchCtx* c, TcMat& t, int rows, int K, int box_rows, int box_k);
// view of columns [col0, col0 + K) of an existing split matrix (same box width as the source)
int tc_view(TcMat& v, const TcMat& src, int col0, int rows, int K, int box_rows);
// (hi, lo) = fp16 split of src * scale (scale an exact power of two)
void split16(CnLaunchCtx* c, cudaStream_t st, const float* src, float scale, __half* hi, __half* lo, size_t count);
// maximum dynamic shared memory of every instance (once per device before the first launch)
int tc_set_attrs();

// C = act((Ahi+Alo)(Bhi+Blo)^T / 64 + bias) on columns [act_lo, act_hi); bn = B tile rows (256 or 64).  m_ptr / m0_ptr:
// optional device-side row count / first row.  A failure is recorded in the context (launch_error, cn_last_error).
void gemm_tc(CnLaunchCtx* c, cudaStream_t st, const TcMat& A, const TcMat& B, int M, int N, int K, int bn, const float* bias,
             int act, const TcOut& o, const int* m_ptr = nullptr, int act_lo = 0, int act_hi = 1 << 30,
             const int* m0_ptr = nullptr);

// One GRU cell step (hidden size 256, input size 64) over M rows as ONE GEMM with the gate math in the epilogue
// (TC_OUT_GRU): A = [x (64) | m h (256)] split fp16 [M, 320]; B = the interleaved gate weights [1024, 320] (cn_dsrnn.cu),
// bias [1024] in the same order.  h' of GEMM row r goes to the fp32 state row (r / group) * pitch + off + r % group of
// h_out [*, 256]; h_in (same rows; null = zero state) times mask[r / group] is the previous state.  oh / ol (or null):
// split fp16 copy of h' in GEMM row order, row pitch ldh.
void gemm_tc_gru(CnLaunchCtx* c, cudaStream_t st, const TcMat& A, const TcMat& B, int M, const float* bias,
                 const float* h_in, const float* mask, float* h_out, int group, int pitch, int off, __half* oh, __half* ol,
                 int ldh);

// The PPO update's GEMM (PROMOTE instance, BN = 64, plain launch on `st` with a grid of at most num_sms CTAs):
// C[Mr, Nc] (+)= act((A_hi + A_lo)[Mr, Kd] (B_hi + B_lo)[Nc, Kd]^T * *inv_a * *inv_b + bias); Kd multiple of 64 in
// storage (pitches), logical extents may be smaller (TMA zero-fills).  ksplit > 1: atomic adds into a zeroed C.
int gemm_tc_promote(int num_sms, cudaStream_t st, const __half* ahi, const __half* alo, int a_rows, int a_pitch,
                    const __half* bhi, const __half* blo, int b_rows, int b_pitch, int Kd, float* C, int ldc,
                    const float* bias, int act, const float* inv_a, const float* inv_b, int ksplit);
