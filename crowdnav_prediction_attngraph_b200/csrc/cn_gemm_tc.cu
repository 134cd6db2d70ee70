// Host side of the wgmma 3xFP16 GEMM (cn_gemm_tc.cuh): TMA maps, split fp16 operands, the instance table and the
// launches of the rollout (gemm_tc) and of the PPO update (gemm_tc_promote), and the GEMM test hooks.  The only
// translation unit that instantiates cn_gemm_tc_kernel.
#include "cn_gemm_tc.h"

// fp32 -> (hi, lo) fp16 split with an exact power-of-two pre-scale (weights at finalize time,
// and the generic "split this activation" helper).
__global__ void cn_split_f16_kernel(const float* __restrict__ src, float scale, __half* __restrict__ hi,
                                    __half* __restrict__ lo, size_t count) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float x = fminf(fmaxf(src[i] * scale, -65504.0f), 65504.0f);
  const __half h = __float2half_rn(x);
  hi[i] = h;
  lo[i] = __float2half_rn(x - __half2float(h));
}

namespace {

typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                             const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeFn get_encode() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void* sym = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeFn>(sym);
  }
  return fn;
}

int halloc16(CnLaunchCtx* c, __half** ptr, size_t count) {
  float* q = nullptr;
  int rc = palloc(c, &q, (count + 1) / 2);
  *ptr = reinterpret_cast<__half*>(q);
  return rc;
}

// store maps of the hi / lo halves of a split matrix (left empty where TMA cannot store: an unaligned column view)
int tc_store_maps(TcMat& t, int rows, int K) {
  if (!tma_store_ok(t.hi, (size_t)t.pitch * 2) || !tma_store_ok(t.lo, (size_t)t.pitch * 2)) return 0;
  int rc = make_store_map(&t.sh, t.hi, 2, rows, K, t.pitch);
  if (!rc) rc = make_store_map(&t.sl, t.lo, 2, rows, K, t.pitch);
  return rc;
}

// the non-PROMOTE instance of cn_gemm_tc_kernel with B-tile rows BN, activation act (CN_ACT_*) and output kind out (TC_OUT_*)
typedef void (*TcKernel)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, int, int, int, TcEpilogue, CUtensorMap,
                         CUtensorMap, CUtensorMap);
template <int BN>
TcKernel tc_kernel(int act, int out) {
  static const TcKernel k[3][3] = {
      {cn_gemm_tc_kernel<BN, false, CN_ACT_NONE, TC_OUT_F32>, cn_gemm_tc_kernel<BN, false, CN_ACT_NONE, TC_OUT_F16>,
       cn_gemm_tc_kernel<BN, false, CN_ACT_NONE, TC_OUT_BOTH>},
      {cn_gemm_tc_kernel<BN, false, CN_ACT_RELU, TC_OUT_F32>, cn_gemm_tc_kernel<BN, false, CN_ACT_RELU, TC_OUT_F16>,
       cn_gemm_tc_kernel<BN, false, CN_ACT_RELU, TC_OUT_BOTH>},
      {cn_gemm_tc_kernel<BN, false, CN_ACT_TANH, TC_OUT_F32>, cn_gemm_tc_kernel<BN, false, CN_ACT_TANH, TC_OUT_F16>,
       cn_gemm_tc_kernel<BN, false, CN_ACT_TANH, TC_OUT_BOTH>}};
  return k[act][out - 1];
}

#ifdef CN_GEMM_TRACE
unsigned long long* g_tc_trace = nullptr;   // per-tile trace buffer of every following gemm_tc launch (or null)
int g_tc_trace_cap = 0;
#endif

}  // namespace

int make_map(CUtensorMap* map, const __half* ptr, int rows, int K, int box_rows, int pitch, int box_k) {
  EncodeFn enc = get_encode();
  if (!enc) return cn_set_error("cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)pitch * sizeof(__half)};
  cuuint32_t box[2] = {(cuuint32_t)box_k, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(ptr), gdim, gstride, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, box_k == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cn_set_error("cuTensorMapEncodeTiled failed (%d) rows=%d K=%d pitch=%d", (int)r, rows, K, pitch);
  return 0;
}

int make_store_map(TcStoreMap* s, const void* ptr, int esize, int rows, int cols, int pitch) {
  s->rows = s->cols = 0;
  if (!tma_store_ok(ptr, (size_t)pitch * esize))
    return cn_set_error("TMA store map: base %p / row pitch %d B not 16-byte aligned", ptr, pitch * esize);
  EncodeFn enc = get_encode();
  if (!enc) return cn_set_error("cuTensorMapEncodeTiled entry point not available");
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)pitch * esize};
  cuuint32_t box[2] = {(cuuint32_t)(128 / esize), 64};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(&s->map, esize == 4 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                   const_cast<void*>(ptr), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return cn_set_error("cuTensorMapEncodeTiled(store) failed (%d) rows=%d cols=%d", (int)r, rows, cols);
  s->rows = rows; s->cols = cols;
  return 0;
}

int tc_alloc(CnLaunchCtx* c, TcMat& t, int rows, int K, int box_rows, int box_k) {
  int rc = halloc16(c, &t.hi, (size_t)rows * K);
  if (!rc) rc = halloc16(c, &t.lo, (size_t)rows * K);
  t.pitch = K; t.box_k = box_k;
  if (!rc) rc = make_map(&t.mh, t.hi, rows, K, box_rows, K, box_k);
  if (!rc) rc = make_map(&t.ml, t.lo, rows, K, box_rows, K, box_k);
  if (!rc) rc = tc_store_maps(t, rows, K);
  return rc;
}

int tc_view(TcMat& v, const TcMat& src, int col0, int rows, int K, int box_rows) {
  v.hi = src.hi + col0; v.lo = src.lo + col0; v.pitch = src.pitch; v.box_k = src.box_k;
  int rc = make_map(&v.mh, v.hi, rows, K, box_rows, src.pitch, src.box_k);
  if (!rc) rc = make_map(&v.ml, v.lo, rows, K, box_rows, src.pitch, src.box_k);
  if (!rc) rc = tc_store_maps(v, rows, K);
  return rc;
}

void split16(CnLaunchCtx* c, cudaStream_t st, const float* src, float scale, __half* hi, __half* lo, size_t count) {
  cn_split_f16_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(src, scale, hi, lo, count);
  c->launches += 1;
}

int tc_set_attrs() {
  cudaError_t e = cudaSuccess;
  for (int act = CN_ACT_NONE; act <= CN_ACT_TANH; ++act)
    for (int out = TC_OUT_F32; out <= TC_OUT_BOTH; ++out) {
      if (e == cudaSuccess)
        e = cudaFuncSetAttribute(tc_kernel<256>(act, out), cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<256>::kSmemBytes);
      if (e == cudaSuccess)
        e = cudaFuncSetAttribute(tc_kernel<64>(act, out), cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<64>::kSmemBytes);
    }
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(cn_gemm_tc_kernel<64, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<64>::kSmemBytes);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(cn_gemm_tc_kernel<256, false, CN_ACT_NONE, TC_OUT_GRU>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, TcCfg<256>::kSmemBytes);
  if (e != cudaSuccess) return cn_set_error("cudaFuncSetAttribute(tc): %s", cudaGetErrorString(e));
  return 0;
}

void gemm_tc(CnLaunchCtx* c, cudaStream_t st, const TcMat& A, const TcMat& B, int M, int N, int K, int bn, const float* bias,
             int act, const TcOut& o, const int* m_ptr, int act_lo, int act_hi, const int* m0_ptr) {
  TcEpilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.bias = bias; ep.inv_scale = 1.0f / 64.0f; ep.act = act; ep.act_lo = act_lo; ep.act_hi = act_hi;
  ep.c32 = o.c32; ep.ldc = o.ldc; ep.out_hi = o.oh; ep.out_lo = o.ol; ep.ldh = o.ldh; ep.m_ptr = m_ptr; ep.m0_ptr = m0_ptr;
  {
    static const int nostore = (getenv("CN_DBG_NOSTORE") && getenv("CN_DBG_NOSTORE")[0] == '1') ? 1 : 0;
    ep.dbg_nostore = nostore;
  }
  // the operand maps must have the box width this instance loads, or its barriers would wait for bytes that never come
  if (A.box_k != tc_box_k(bn) || B.box_k != tc_box_k(bn)) {
    if (!c->launch_error) {
      c->launch_error = true;
      cn_set_error("gemm_tc in stage '%s': operand boxes %d / %d wide, the BN = %d instance loads %d",
                   c->cur_stage ? c->cur_stage : "?", A.box_k, B.box_k, bn, tc_box_k(bn));
    }
    return;
  }
  const int out_kind = (o.c32 ? TC_OUT_F32 : 0) | (o.oh ? TC_OUT_F16 : 0);
  if (act < CN_ACT_NONE || act > CN_ACT_TANH || !out_kind) {
    if (!c->launch_error) {
      c->launch_error = true;
      cn_set_error("gemm_tc in stage '%s': activation %d / no output", c->cur_stage ? c->cur_stage : "?", act);
    }
    return;
  }
#ifdef CN_GEMM_TRACE
  ep.trace = g_tc_trace; ep.trace_cap = g_tc_trace_cap;
#endif
  static const CUtensorMap no_map = {};                 // placeholder for the store maps an instance does not read
  const CUtensorMap *mc = &no_map, *mh = &no_map, *ml = &no_map;
  if (bn == 256) {
    // TMA stores: every output needs a map of exactly [M, N] (the row extent clips the last tile's rows)
    auto fits = [&](const TcStoreMap* s) { return s && s->rows == M && s->cols == N; };
    const bool ok = (!o.c32 || fits(o.sc)) && (!o.oh || (fits(o.sh) && fits(o.sl)));
    if (!ok) {
      if (!c->launch_error) {
        c->launch_error = true;
        cn_set_error("gemm_tc in stage '%s': a BN = 256 output needs a TMA store map of [%d x %d] (16-byte-aligned "
                     "base, row pitch a multiple of 16 bytes)", c->cur_stage ? c->cur_stage : "?", M, N);
      }
      return;
    }
    if (o.c32) mc = &o.sc->map;
    if (o.oh) { mh = &o.sh->map; ml = &o.sl->map; }
  }
  // persistent: one CTA per SM at most; tiles beyond the device-side row count are never touched
  const int tiles = (N / bn) * ((M + TC_BM - 1) / TC_BM);
  dim3 grid(tiles < c->num_sms ? tiles : c->num_sms);
  if (bn == 256)
    launch_k(c, tc_kernel<256>(act, out_kind), grid, dim3(TC_THREADS), TcCfg<256>::kSmemBytes, st, A.mh, A.ml, B.mh, B.ml, M, N, K, ep,
             *mc, *mh, *ml);
  else
    launch_k(c, tc_kernel<64>(act, out_kind), grid, dim3(TC_THREADS), TcCfg<64>::kSmemBytes, st, A.mh, A.ml, B.mh, B.ml, M, N, K, ep,
             *mc, *mh, *ml);
}

void gemm_tc_gru(CnLaunchCtx* c, cudaStream_t st, const TcMat& A, const TcMat& B, int M, const float* bias,
                 const float* h_in, const float* mask, float* h_out, int group, int pitch, int off, __half* oh, __half* ol,
                 int ldh) {
  const int N = 4 * 256, K = 64 + 256;
  if (A.box_k != tc_box_k(256) || B.box_k != tc_box_k(256) || !bias || !h_out || !mask || group <= 0) {
    if (!c->launch_error) {
      c->launch_error = true;
      cn_set_error("gemm_tc_gru in stage '%s': operand boxes %d / %d wide (need %d), or a missing bias / mask / output",
                   c->cur_stage ? c->cur_stage : "?", A.box_k, B.box_k, tc_box_k(256));
    }
    return;
  }
  TcEpilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.bias = bias; ep.inv_scale = 1.0f / 64.0f; ep.act_hi = 1 << 30;
  ep.c32 = h_out; ep.ldc = 256; ep.out_hi = oh; ep.out_lo = ol; ep.ldh = ldh;
  ep.gru_h = h_in; ep.gru_mask = mask; ep.gru_group = group; ep.gru_pitch = pitch; ep.gru_off = off;
  static const CUtensorMap no_map = {};
  const int tiles = (N / 256) * ((M + TC_BM - 1) / TC_BM);
  dim3 grid(tiles < c->num_sms ? tiles : c->num_sms);
  launch_k(c, cn_gemm_tc_kernel<256, false, CN_ACT_NONE, TC_OUT_GRU>, grid, dim3(TC_THREADS), TcCfg<256>::kSmemBytes, st,
           A.mh, A.ml, B.mh, B.ml, M, N, K, ep, no_map, no_map, no_map);
}

int gemm_tc_promote(int num_sms, cudaStream_t st, const __half* ahi, const __half* alo, int a_rows, int a_pitch,
                    const __half* bhi, const __half* blo, int b_rows, int b_pitch, int Kd, float* C, int ldc,
                    const float* bias, int act, const float* inv_a, const float* inv_b, int ksplit) {
  // 64-column tiles: the per-k-block promoted accumulation (cn_gemm_tc.cuh) needs a second accumulator in registers
  const int bn = 64;
  if (b_rows % bn) return cn_set_error("cn_update gemm: output columns %d not a multiple of 64", b_rows);
  const int Kp = (Kd + TC_BK - 1) / TC_BK * TC_BK;
  CUtensorMap mah, mal, mbh, mbl;
  int rc = make_map(&mah, ahi, a_rows, Kd, TC_BM, a_pitch);
  if (!rc) rc = make_map(&mal, alo, a_rows, Kd, TC_BM, a_pitch);
  if (!rc) rc = make_map(&mbh, bhi, b_rows, Kd, bn, b_pitch);
  if (!rc) rc = make_map(&mbl, blo, b_rows, Kd, bn, b_pitch);
  if (rc) return rc;
  TcEpilogue ep;
  memset(&ep, 0, sizeof(ep));
  ep.bias = bias; ep.inv_scale = 1.0f; ep.act = act; ep.act_lo = 0; ep.act_hi = 1 << 30;
  ep.c32 = C; ep.ldc = ldc; ep.inv_scale_a = inv_a; ep.inv_scale_b = inv_b; ep.ksplit = ksplit;
  const int tiles = (b_rows / bn) * ((a_rows + TC_BM - 1) / TC_BM) * (ksplit > 1 ? ksplit : 1);
  const int grid = tiles < num_sms ? tiles : num_sms;
  static const CUtensorMap no_map = {};        // the PROMOTE instance stores directly; its store maps are not read
  cn_gemm_tc_kernel<64, true><<<grid, TC_THREADS, TcCfg<64>::kSmemBytes, st>>>(mah, mal, mbh, mbl, a_rows, b_rows, Kp, ep,
                                                                                no_map, no_map, no_map);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return cn_set_error("cn_update gemm launch (M=%d N=%d K=%d ksplit=%d): %s", a_rows, b_rows, Kd, ksplit, cudaGetErrorString(e));
  return 0;
}

extern "C" {

// Internal test hooks (not part of the public header): C = act(A[M,K] W[N,K]^T + bias) through the
// wgmma 3xFP16 kernel with B-tile rows `bn` (256 or 64), fp32 device pointers in/out.  cn_internal_gemm_tc_ex adds
// the epilogue and operand variants the rollout uses (zero / null = off):
//   m_ptr, m0_ptr   device-side row count and first row (rows [*m0_ptr, *m_ptr) of the M-row extent);
//   a_col0, a_pitch A is the column view [a_col0, a_col0 + K) of an fp32 matrix [M, a_pitch] (pitch 0 = K);
//   out_hi, out_lo  fp16 (hi, lo) split output with leading dimension ldh (pointers already at the column offset);
//                   dC may then be null;
//   act_lo, act_hi  the activation applies to columns [act_lo, act_hi) only (act_hi 0 = all columns).
int cn_internal_gemm_tc_ex(const float* dA, const float* dW, const float* dbias, float* dC, int M, int N, int K, int act,
                           int bn, const int* m_ptr, const int* m0_ptr, int a_col0, int a_pitch, __half* out_hi,
                           __half* out_lo, int ldh, int act_lo, int act_hi) {
  if (a_pitch == 0) a_pitch = K;
  if ((bn != 256 && bn != 64) || M <= 0 || N <= 0 || K <= 0 || N % bn || K % TC_BK || a_col0 < 0 ||
      a_col0 + K > a_pitch || a_col0 % 8 || a_pitch % 8 || (!dC && !out_hi) || (!out_hi != !out_lo) ||
      (out_hi && ldh < N))
    return cn_set_error("cn_internal_gemm_tc_ex: need bn in {64,256}, M, N, K > 0, N %% bn == 0, K %% 64 == 0, "
                        "a_col0 + K <= a_pitch (both multiples of 8), an output and ldh >= N");
  // the BN = 256 instances store with TMA (gemm_tc); check here, before anything is launched
  if (bn == 256 && ((dC && !tma_store_ok(dC, (size_t)N * 4)) ||
                    (out_hi && (!tma_store_ok(out_hi, (size_t)ldh * 2) || !tma_store_ok(out_lo, (size_t)ldh * 2)))))
    return cn_set_error("cn_internal_gemm_tc_ex: a BN = 256 output needs a 16-byte-aligned base and a row pitch that is "
                        "a multiple of 16 bytes");
  CnLaunchCtx ctx;                                 // no PDL
  cudaDeviceGetAttribute(&ctx.num_sms, cudaDevAttrMultiProcessorCount, 0);
  TcMat Af, A, B;
  int rc = tc_alloc(&ctx, Af, M, a_pitch, TC_BM, tc_box_k(bn));
  if (!rc) rc = tc_view(A, Af, a_col0, M, K, TC_BM);
  if (!rc) rc = tc_alloc(&ctx, B, N, K, bn, tc_box_k(bn));
  if (!rc) rc = tc_set_attrs();
  TcOut o = out32(dC, N);
  o.oh = out_hi; o.ol = out_lo; o.ldh = ldh;
  TcStoreMap sc, sh, sl;                           // store maps of this call's outputs (BN = 256)
  if (bn == 256) {
    if (!rc && dC) rc = make_store_map(&sc, dC, 4, M, N, N);
    if (!rc && out_hi) rc = make_store_map(&sh, out_hi, 2, M, N, ldh);
    if (!rc && out_hi) rc = make_store_map(&sl, out_lo, 2, M, N, ldh);
    o.sc = &sc; o.sh = &sh; o.sl = &sl;
  }
  if (!rc) {
    split16(&ctx, 0, dA, 1.0f, Af.hi, Af.lo, (size_t)M * a_pitch);
    split16(&ctx, 0, dW, 64.0f, B.hi, B.lo, (size_t)N * K);
    gemm_tc(&ctx, 0, A, B, M, N, K, bn, dbias, act, o, m_ptr, act_lo, act_hi > 0 ? act_hi : 1 << 30, m0_ptr);
    cudaError_t err = cudaDeviceSynchronize();
    if (err != cudaSuccess) rc = cn_set_error("cn_internal_gemm_tc_ex: %s", cudaGetErrorString(err));
    else if (ctx.launch_error) rc = 1;
  }
  cn_launch_free(&ctx);
  return rc;
}
// the plain form: whole rows, A with pitch K, fp32 output [M, N], activation on every column
int cn_internal_gemm_tc(const float* dA, const float* dW, const float* dbias, float* dC, int M, int N, int K, int act,
                        int bn) {
  return cn_internal_gemm_tc_ex(dA, dW, dbias, dC, M, N, K, act, bn, nullptr, nullptr, 0, 0, nullptr, nullptr, 0, 0, 0);
}
// The edge-GRU instance (TC_OUT_GRU, gemm_tc_gru) on its own: A fp32 [M, 320] = [x | m h] split at scale 1, dB fp32
// [1024, 320] and dbias [1024] already interleaved (cn_dsrnn.cu, interleave_gru) and split at scale 64, as in the
// rollout.  h_in (null: zero state), mask and h_out are indexed as gemm_tc_gru documents (h_out needs
// ceil(M / group) * pitch rows of 256); out_hi / out_lo (both or neither): split copy of h' [M, ldh].
int cn_internal_gemm_tc_gru(const float* dA, const float* dB, const float* dbias, const float* h_in, const float* mask,
                            float* h_out, int M, int group, int pitch, int off, __half* out_hi, __half* out_lo, int ldh) {
  const int N = 4 * 256, K = 64 + 256;
  if (M <= 0 || group <= 0 || off < 0 || off + group > pitch || !dA || !dB || !dbias || !mask || !h_out ||
      (!out_hi != !out_lo) || (out_hi && (ldh < 256 || ldh % 2)))
    return cn_set_error("cn_internal_gemm_tc_gru: need M, group > 0, 0 <= off, off + group <= pitch, A, B, bias, mask "
                        "and h_out, and out_hi / out_lo both or neither with an even ldh >= 256");
  CnLaunchCtx ctx;                                 // no PDL
  cudaDeviceGetAttribute(&ctx.num_sms, cudaDevAttrMultiProcessorCount, 0);
  TcMat A, B;
  int rc = tc_alloc(&ctx, A, M, K, TC_BM, tc_box_k(256));
  if (!rc) rc = tc_alloc(&ctx, B, N, K, 256, tc_box_k(256));
  if (!rc) rc = tc_set_attrs();
  if (!rc) {
    split16(&ctx, 0, dA, 1.0f, A.hi, A.lo, (size_t)M * K);
    split16(&ctx, 0, dB, 64.0f, B.hi, B.lo, (size_t)N * K);
    gemm_tc_gru(&ctx, 0, A, B, M, dbias, h_in, mask, h_out, group, pitch, off, out_hi, out_lo, ldh);
    cudaError_t err = cudaDeviceSynchronize();
    if (err != cudaSuccess) rc = cn_set_error("cn_internal_gemm_tc_gru: %s", cudaGetErrorString(err));
    else if (ctx.launch_error) rc = 1;
  }
  cn_launch_free(&ctx);
  return rc;
}

#ifdef CN_GEMM_TRACE
// Traced builds only (tools/gemm_tile_trace.py): every following gemm_tc launch writes per-tile records
// [gridDim.x][cap][TC_TRACE_REC] (cn_gemm_tc.cuh) to dtrace.
int cn_internal_gemm_trace(unsigned long long* dtrace, int cap) {
  g_tc_trace = dtrace; g_tc_trace_cap = dtrace ? cap : 0;
  return 0;
}
#endif

}  // extern "C"
