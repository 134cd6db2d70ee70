// wgmma / TMA GEMM for the policy's 512-wide projections (sm_90a only).
//
//   C[M,N] = act( (A_hi + A_lo)[M,K] . (B_hi + B_lo)[N,K]^T * (1/scale_b) + bias[N] )
//
// "3xFP16" error-compensated product: every fp32 operand is split into two fp16 pieces
// (hi = rn(x), lo = rn(x - hi): 22 significand bits) and the three significant partial
// products  A_hi.B_hi + A_hi.B_lo + A_lo.B_hi  are accumulated by the Hopper tensor cores
// (wgmma) in an fp32 register accumulator.  Measured against the fp32 reference policy this keeps
// the action mean / value within 2e-5 (same as a plain fp32 CUDA-core GEMM), where single-pass
// TF32/BF16 would break the 1e-4 tolerance (see DESIGN.md).  Weights are pre-scaled by 2^6 so
// their lo pieces stay in fp16's normal range; the epilogue undoes the power-of-two scale exactly.
//
// Tiling: one 128 x BN output tile per CTA (BN = 256 for the large per-human GEMMs, BN = 64 for the
// per-environment layers where M is only a few thousand rows and more CTAs matter more than tile
// efficiency), TMA->smem ring of 4 stages of 48 KB.  BN = 64: k-blocks of 64 fp16 (one 128-byte swizzle
// atom).  BN = 256: k-blocks of 32 fp16 (64-byte swizzle), so a slot is refilled after a quarter of the ring's
// MMA time instead of half of it; each output element still sees the same wgmma instructions in the same order.
// Warp groups: 0 = TMA producer (one thread), 1 and 2 = consumers: each issues wgmma.m64nBNk16 for 64 rows of the
// tile, keeps that 64 x BN fp32 accumulator in registers and runs the epilogue (bias, activation, stores) from them:
// BN = 64 stores straight to global memory, BN = 256 stages boxes in shared memory and stores them with TMA while the
// warp group goes on (tc_epilogue_tma).  The activation and the output kind are template parameters of the non-PROMOTE instances: an epilogue
// that chose them at run time inlined every path into each of the 64 unrolled column groups of BN = 256 (20 680
// instructions, ~330 KB of code walked on every tile), and that epilogue, not the MMAs, set the time of a tile (QKV:
// 31 of 46 us; now 9 of 24 us, DESIGN.md 3.2).  The QKV instance is now 1 048 instructions.
//
// PROMOTE (the PPO update's GEMMs, which must be fp32-equivalent): the tensor core sums each 64-wide k-block on its own
// and the CUDA cores add the block sums into a second register accumulator with IEEE round-to-nearest.  wgmma's fp32
// accumulation truncates inside every instruction, so over K = 512..1536 one long chain drifts to ~5e-6 relative
// error, several times torch's fp32 GEMM; per-block sums keep the truncated chain 12 instructions long.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "cn_launch.cuh"

#define TC_BM 128
#define TC_BK 64                                      // k-block of the BN = 64 instances (and the PPO update's maps)
#define TC_CONSUMER_WARPS 8                           // two consumer warp groups
#define TC_THREADS (128 + 32 * TC_CONSUMER_WARPS)

template <int BN>
struct TcCfg {
  static constexpr int kBK = (BN >= 256) ? 32 : TC_BK;        // k-block width (fp16) = TMA box width
  static constexpr int kSwizzle = 2 * kBK;                    // bytes per smem row: 64- or 128-byte swizzle
  static constexpr int kStages = 4;
  static constexpr int kATile = TC_BM * kBK * 2;
  static constexpr int kBTile = BN * kBK * 2;
  static constexpr int kStageBytes = 2 * kATile + 2 * kBTile;
  // BN = 256: the epilogue stages its output in shared memory, in boxes of 64 rows x 128 bytes (32 fp32 or 64 fp16
  // columns, 128-byte swizzle) that TMA stores; kStoreBoxes boxes per consumer warp group (tc_epilogue_tma).  Two boxes
  // fit beside the 4-stage ring (230 656 B of the 232 448 B opt-in limit).  A 3-stage ring with four boxes measured the
  // same for embed2 and qkv and 6 % slower for outproj_spatial, whose main loop then waits for operands (DESIGN.md 3.2).
  static constexpr int kStoreBoxes = (BN >= 256) ? 2 : 0;
  static constexpr int kBoxBytes = 64 * 128;
  static constexpr int kStagingBytes = 2 * kStoreBoxes * kBoxBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + kStagingBytes + 256 /*barriers*/ + 1024 /*align slack*/;
};

struct TcEpilogue {
  const float* bias;     // [N] or null
  float inv_scale;       // 1 / scale_b
  int act;               // CN_ACT_* applied to columns [act_lo, act_hi)
  int act_lo, act_hi;
  float* c32;            // fp32 output [M, ldc] or null
  int ldc;
  __half* out_hi;        // split fp16 output [M, ldh] or null (A operand of the next GEMM)
  __half* out_lo;
  int ldh;
  const int* m_ptr;      // optional device-side row count (compacted rows); tiles past it exit
  int dbg_nostore;       // diagnostic: run the epilogue arithmetic but skip the global stores
  const int* m0_ptr;     // optional device-side first row: the launch covers rows [*m0_ptr, *m_ptr) (row chunks)
  // --- PPO update path (cn_update.cu); all zero / null in the rollout ---
  const float* inv_scale_a;   // optional device scalars: the result is also multiplied by *inv_scale_a * *inv_scale_b
  const float* inv_scale_b;   // (dynamic power-of-two operand scales chosen from the tensors' amax)
  int ksplit;                 // > 1 (PROMOTE only): the K range is cut into `ksplit` slices, every slice is its own tile and ADDS its
                              // partial product into a zero-initialised fp32 C with atomic adds (bias from slice 0
                              // only, no activation): wgrad has K = #rows (hundreds of thousands) and a tiny output
  // --- GRU cell epilogue (TC_OUT_GRU, the DS-RNN edge GRUs); all zero / null otherwise ---
  // GEMM row r is the state row  out_r = (r / gru_group) * gru_pitch + gru_off + r % gru_group  of the [*, 256] fp32
  // state: h = gru_h[out_r] * gru_mask[r / gru_group] (gru_h null: h = 0); h' goes to c32[out_r] (ldc = 256) and, with
  // out_hi, as a split fp16 pair to out_hi / out_lo [r, ldh].
  const float* gru_h;
  const float* gru_mask;
  int gru_group, gru_pitch, gru_off;
#ifdef CN_GEMM_TRACE
  unsigned long long* trace;  // [gridDim.x][trace_cap][TC_TRACE_REC] per-tile records (tools/gemm_tile_trace.py)
  int trace_cap;
#endif
};

#ifdef CN_GEMM_TRACE
// per-tile trace record: tile start, first full-barrier pass, main-loop end, epilogue end (%globaltimer, ns; for
// BN = 256 the moment the recording thread handed the tile's last box to TMA), failed polls of the full barriers;
// BN = 256 only: staging-buffer waits that blocked, and the clock cycles spent in all staging-buffer waits
#define TC_TRACE_REC 7
#define TC_TRACE_WAIT_CLK 100     // a wait on a buffer that is already free returns well within this many cycles
#endif

// Output kinds of the non-PROMOTE instances (template parameter OUT): fp32 C, split fp16 (hi, lo), or both; or
// (BN = 256 only) the GRU cell epilogue tc_epilogue_gru
enum { TC_OUT_F32 = 1, TC_OUT_F16 = 2, TC_OUT_BOTH = 3, TC_OUT_GRU = 4 };

#ifdef CN_GEMM_TRACE
#define TC_TRACE(...) __VA_ARGS__
#else
#define TC_TRACE(...)
#endif

namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
  } while (!ok);
}
#ifdef CN_GEMM_TRACE
// mbar_wait that returns the number of failed polls
__device__ __forceinline__ uint32_t mbar_wait_polls(uint32_t bar, uint32_t parity) {
  uint32_t ok, n = 0;
  while (true) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n" : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    if (ok) return n;
    ++n;
  }
}
__device__ __forceinline__ uint64_t globaltimer() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#endif
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void st_shared_v2(uint32_t addr, float a, float b) {
  asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(addr), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// TMA store of one box from shared memory (bulk-group completion) and the bulk-group bookkeeping of the issuing thread
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(map), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy writes to shared memory -> visible to the async proxy (TMA) after the next barrier
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// K-major shared-memory matrix descriptor of wgmma (cute::GMMA::DescriptorSW128 / SW64) for a tile written by TMA
// with SWIZZLE_128B (SW = 128: 128-byte rows) or SWIZZLE_64B (SW = 64: 64-byte rows):
//   [0,14) start address >> 4 | [16,30) LBO >> 4 (=1, unused for swizzled K-major) |
//   [32,46) SBO >> 4 (8 rows * SW bytes) | [62,64) layout (1 = 128B swizzle, 2 = 64B swizzle)
template <int SW>
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | (1ull << 16) | ((uint64_t)((8 * SW) >> 4) << 32) |
         ((SW == 128 ? 1ull : 2ull) << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int NREG>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(NREG)); }
template <int NREG>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(NREG)); }

// D[64 x N] (+)= A[64 x 16] . B[N x 16]^T, fp16 operands from shared memory, fp32 accumulator in registers.
// accum = 0 overwrites D.  Register i of the calling thread (warp w of the group, lane l) holds
//   row 16 w + l / 4 + 8 ((i / 2) & 1),  column 8 (i / 4) + 2 (l & 3) + (i & 1).
template <int N>
__device__ __forceinline__ void wgmma_f16(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accum);
template <>
__device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, %32, %33, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accum));
}
template <>
__device__ __forceinline__ void wgmma_f16<192>(float (&d)[96], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %98, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
      "}, %96, %97, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(da), "l"(db), "r"(accum));
}
template <>
__device__ __forceinline__ void wgmma_f16<256>(float (&d)[128], uint64_t da, uint64_t db, uint32_t accum) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, %130, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, "
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, "
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, p, 1, 1, 0, 0;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accum));
}

// tanh(x) = 1 - 2 / (exp(2x) + 1) with the accurate expf and an IEEE division: ~2e-7 absolute error
// (cheaper than tanhf in the 256-column epilogue, and far inside the 1e-4 policy tolerance)
__device__ __forceinline__ float fast_tanh(float x) {
  const float e = expf(2.0f * x);
  return 1.0f - 2.0f / (e + 1.0f);
}
__device__ __forceinline__ uint32_t split_pair_hi(float x0, float x1, uint32_t* lo) {
  x0 = fminf(fmaxf(x0, -65504.0f), 65504.0f);
  x1 = fminf(fmaxf(x1, -65504.0f), 65504.0f);
  const __half h0 = __float2half_rn(x0), h1 = __float2half_rn(x1);
  const __half l0 = __float2half_rn(x0 - __half2float(h0)), l1 = __float2half_rn(x1 - __half2float(h1));
  *lo = (uint32_t)__half_as_ushort(l0) | ((uint32_t)__half_as_ushort(l1) << 16);
  return (uint32_t)__half_as_ushort(h0) | ((uint32_t)__half_as_ushort(h1) << 16);
}

}  // namespace tc

// Epilogue of the non-PROMOTE instances: scale, bias, activation and stores straight from the 64 x BN accumulator of
// one consumer warp group (this thread: rows r0, r0 + 8; columns 8 g + cq, + 1).  The activation (CN_ACT_*) and the
// output kind (TC_OUT_*) are compile-time, so each instance holds only the code it runs; the [act_lo, act_hi) window
// is a per-column select.  Rows at or past m_ext (the output's extent) are not stored.
template <int BN, int ACT, int OUT>
__device__ __forceinline__ void tc_epilogue_store(const float (&acc)[BN / 2], const TcEpilogue& ep, float inv_scale,
                                                  int n0, int r0, int cq, int m_ext) {
  static_assert(ACT >= 0 && ACT <= 2 && OUT >= TC_OUT_F32 && OUT <= TC_OUT_BOTH, "epilogue kind");
  const int row_end = ep.dbg_nostore ? 0 : m_ext;       // CN_DBG_NOSTORE: all the arithmetic, no stores
#pragma unroll
  for (int g = 0; g < BN / 8; ++g) {
    const int col = n0 + 8 * g + cq;
    const float b0 = ep.bias ? __ldg(ep.bias + col) : 0.0f, b1 = ep.bias ? __ldg(ep.bias + col + 1) : 0.0f;
    const bool w0 = col >= ep.act_lo && col < ep.act_hi, w1 = col + 1 >= ep.act_lo && col + 1 < ep.act_hi;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      float v0 = fmaf(acc[4 * g + 2 * h], inv_scale, b0), v1 = fmaf(acc[4 * g + 2 * h + 1], inv_scale, b1);
      if constexpr (ACT == 1) {
        v0 = w0 ? fmaxf(v0, 0.0f) : v0; v1 = w1 ? fmaxf(v1, 0.0f) : v1;
      } else if constexpr (ACT == 2) {
        if (w0) v0 = tc::fast_tanh(v0);
        if (w1) v1 = tc::fast_tanh(v1);
      }
      if (row >= row_end) continue;
      if constexpr ((OUT & TC_OUT_F32) != 0) {
        *reinterpret_cast<float2*>(ep.c32 + (size_t)row * ep.ldc + col) = make_float2(v0, v1);
      }
      if constexpr ((OUT & TC_OUT_F16) != 0) {
        uint32_t lo;
        const uint32_t hi = tc::split_pair_hi(v0, v1, &lo);
        const size_t o = (size_t)row * ep.ldh + col;
        *reinterpret_cast<uint32_t*>(ep.out_hi + o) = hi;
        *reinterpret_cast<uint32_t*>(ep.out_lo + o) = lo;
      }
    }
  }
}

// Staging buffers of tc_epilogue_tma.  Acquire: the issuing thread waits until at most PENDING of its box stores may
// still be reading shared memory (so the buffers about to be written are free), then the warp group (named barrier
// bar_id, 128 threads) goes on.  Release: every thread's writes are made visible to the async proxy before the
// barrier after which the issuing thread hands the boxes to TMA.
struct TcStaging {
  uint32_t base;     // this warp group's kStoreBoxes boxes (1024-byte aligned)
  uint32_t box;      // running box counter: box b is staged in buffer b % kStoreBoxes
  bool leader;       // the warp group's thread that issues (and drains) the TMA stores
  int bar_id;
#ifdef CN_GEMM_TRACE
  uint32_t waits;    // acquires that blocked (TC_TRACE_WAIT_CLK), and the cycles spent in all of them
  uint64_t wait_clk;
#endif
  template <int PENDING>
  __device__ __forceinline__ void acquire() {
    if (leader) {
#ifdef CN_GEMM_TRACE
      const long long c0 = clock64();
      tc::bulk_wait_read<PENDING>();
      const long long d = clock64() - c0;
      waits += d > TC_TRACE_WAIT_CLK ? 1u : 0u;
      wait_clk += (uint64_t)d;
#else
      tc::bulk_wait_read<PENDING>();
#endif
    }
    tc::named_bar_sync(bar_id, 128);
  }
  __device__ __forceinline__ void release() {
    tc::fence_proxy_async_smem();
    tc::named_bar_sync(bar_id, 128);
  }
  __device__ __forceinline__ uint32_t buf(uint32_t b) const { return base + (b % TcCfg<256>::kStoreBoxes) * TcCfg<256>::kBoxBytes; }
};

// Epilogue of the BN = 256 non-PROMOTE instances: the arithmetic of tc_epilogue_store (same operations, same order),
// but the warp group's 64 x 256 result goes through shared memory.  Each box of 64 rows x 128 bytes (fp32: 32 columns;
// split fp16: 64 columns of hi and, in a second box, of lo) is written in the 128-byte swizzle of the output maps: a
// 16-byte chunk c of row r sits at chunk c ^ (r & 7), so the eight rows of a warp's store land in different banks.
// One thread then stores the box with TMA and the warp group moves on without waiting for the global writes; the map's
// row extent (the output's extent M) clips rows as `row < m_ext` does in tc_epilogue_store.  CN_DBG_NOSTORE: stage,
// issue nothing.  This thread: rows wr, wr + 8 of the half starting at row m_half; columns 8 g + cq, + 1.
template <int ACT, int OUT>
__device__ __forceinline__ void tc_epilogue_tma(const float (&acc)[128], const TcEpilogue& ep, float inv_scale, int n0,
                                                int m_half, int wr, int lane, TcStaging& sg, const CUtensorMap* map_c,
                                                const CUtensorMap* map_oh, const CUtensorMap* map_ol) {
  static_assert(ACT >= 0 && ACT <= 2 && OUT >= TC_OUT_F32 && OUT <= TC_OUT_BOTH, "epilogue kind");
  constexpr int NB = TcCfg<256>::kStoreBoxes;
  static_assert(NB >= 2 && (NB & (NB - 1)) == 0, "the split fp16 output stages hi and lo boxes together");
  const int cq = 2 * (lane & 3);
  const bool issue = sg.leader && !ep.dbg_nostore;
  const uint32_t rsw = (uint32_t)(wr & 7);                        // swizzle phase of rows wr and wr + 8
  const uint32_t row_off = (uint32_t)wr * 128u;
  if constexpr ((OUT & TC_OUT_F32) != 0) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {                                 // box j: columns [32 j, 32 j + 32) of the tile
      sg.acquire<NB - 1>();
      const uint32_t b = sg.buf(sg.box) + row_off + 8u * (uint32_t)(lane & 1);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int g = 4 * j + q, col = n0 + 8 * g + cq;
        const float b0 = ep.bias ? __ldg(ep.bias + col) : 0.0f, b1 = ep.bias ? __ldg(ep.bias + col + 1) : 0.0f;
        const bool w0 = col >= ep.act_lo && col < ep.act_hi, w1 = col + 1 >= ep.act_lo && col + 1 < ep.act_hi;
        const uint32_t chunk = (uint32_t)(2 * q + ((lane & 3) >> 1));
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v0 = fmaf(acc[4 * g + 2 * h], inv_scale, b0), v1 = fmaf(acc[4 * g + 2 * h + 1], inv_scale, b1);
          if constexpr (ACT == 1) {
            v0 = w0 ? fmaxf(v0, 0.0f) : v0; v1 = w1 ? fmaxf(v1, 0.0f) : v1;
          } else if constexpr (ACT == 2) {
            if (w0) v0 = tc::fast_tanh(v0);
            if (w1) v1 = tc::fast_tanh(v1);
          }
          tc::st_shared_v2(b + 1024u * h + ((chunk ^ rsw) << 4), v0, v1);
        }
      }
      sg.release();
      if (issue) {
        tc::tma_store_2d(map_c, sg.buf(sg.box), n0 + 32 * j, m_half);
        tc::bulk_commit();
      }
      ++sg.box;
    }
  }
  if constexpr ((OUT & TC_OUT_F16) != 0) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {                                 // boxes of hi and lo: columns [64 j, 64 j + 64)
      sg.acquire<NB - 2>();
      const uint32_t bh = sg.buf(sg.box) + row_off + 4u * (uint32_t)(lane & 3);
      const uint32_t bl = sg.buf(sg.box + 1) + row_off + 4u * (uint32_t)(lane & 3);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const int g = 8 * j + q, col = n0 + 8 * g + cq;
        const float b0 = ep.bias ? __ldg(ep.bias + col) : 0.0f, b1 = ep.bias ? __ldg(ep.bias + col + 1) : 0.0f;
        const bool w0 = col >= ep.act_lo && col < ep.act_hi, w1 = col + 1 >= ep.act_lo && col + 1 < ep.act_hi;
        const uint32_t sw_off = ((uint32_t)q ^ rsw) << 4;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float v0 = fmaf(acc[4 * g + 2 * h], inv_scale, b0), v1 = fmaf(acc[4 * g + 2 * h + 1], inv_scale, b1);
          if constexpr (ACT == 1) {
            v0 = w0 ? fmaxf(v0, 0.0f) : v0; v1 = w1 ? fmaxf(v1, 0.0f) : v1;
          } else if constexpr (ACT == 2) {
            if (w0) v0 = tc::fast_tanh(v0);
            if (w1) v1 = tc::fast_tanh(v1);
          }
          uint32_t lo;
          const uint32_t hi = tc::split_pair_hi(v0, v1, &lo);
          tc::st_shared_b32(bh + 1024u * h + sw_off, hi);
          tc::st_shared_b32(bl + 1024u * h + sw_off, lo);
        }
      }
      sg.release();
      if (issue) {
        tc::tma_store_2d(map_oh, sg.buf(sg.box), n0 + 64 * j, m_half);
        tc::bulk_commit();
        tc::tma_store_2d(map_ol, sg.buf(sg.box + 1), n0 + 64 * j, m_half);
        tc::bulk_commit();
      }
      sg.box += 2;
    }
  }
}

// GRU cell epilogue (TC_OUT_GRU, BN = 256): the B operand is interleaved so that columns [0, 64), [64, 128),
// [128, 192), [192, 256) of the tile at n0 hold the pre-activations r, z, gi_n = W_in x + b_in and gh_n = W_hn h + b_hn
// of hidden units n0 / 4 .. n0 / 4 + 63.  Accumulator column group g (< 8) of this thread and the groups g + 8, + 16,
// + 24 are then the four gates of the same two units, and the cell finishes in registers (PyTorch's GRU,
// h' = (1 - z) n + z h with n = tanh(gi_n + r gh_n)).  No gate leaves the SM: h' is stored in fp32 straight into the
// state row of the GEMM row (TcEpilogue::gru_*), and optionally as a split fp16 pair in GEMM row order.
__device__ __forceinline__ float tc_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ void tc_epilogue_gru(const float (&acc)[128], const TcEpilogue& ep, float inv_scale, int n0,
                                                int r0, int cq, int m_ext) {
  const int u0 = n0 / 4;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = r0 + 8 * h;
    if (row >= m_ext) continue;
    const int env = row / ep.gru_group;
    const size_t orow = (size_t)env * ep.gru_pitch + ep.gru_off + (row - env * ep.gru_group);
    const float m = ep.gru_h ? __ldg(ep.gru_mask + env) : 0.0f;
#pragma unroll
    for (int g = 0; g < 8; ++g) {
      const int c = 8 * g + cq, u = u0 + c;
      float hv[2] = {0.0f, 0.0f};
      if (ep.gru_h) {
        const float2 t = __ldg(reinterpret_cast<const float2*>(ep.gru_h + orow * 256 + u));
        hv[0] = t.x * m; hv[1] = t.y * m;
      }
      float o[2];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const int a = 4 * g + 2 * h + k;
        const float r = tc_sigmoid(fmaf(acc[a], inv_scale, __ldg(ep.bias + n0 + c + k)));
        const float z = tc_sigmoid(fmaf(acc[a + 32], inv_scale, __ldg(ep.bias + n0 + 64 + c + k)));
        const float gin = fmaf(acc[a + 64], inv_scale, __ldg(ep.bias + n0 + 128 + c + k));
        const float ghn = fmaf(acc[a + 96], inv_scale, __ldg(ep.bias + n0 + 192 + c + k));
        const float n = tanhf(gin + r * ghn);
        o[k] = (1.0f - z) * n + z * hv[k];
      }
      if (ep.dbg_nostore) continue;
      *reinterpret_cast<float2*>(ep.c32 + orow * 256 + u) = make_float2(o[0], o[1]);
      if (ep.out_hi) {
        uint32_t lo;
        const uint32_t hi = tc::split_pair_hi(o[0], o[1], &lo);
        const size_t q = (size_t)row * ep.ldh + u;
        *reinterpret_cast<uint32_t*>(ep.out_hi + q) = hi;
        *reinterpret_cast<uint32_t*>(ep.out_lo + q) = lo;
      }
    }
  }
}

// Persistent kernel: grid = min(#tiles, #SMs); every CTA walks tiles t = blockIdx.x, blockIdx.x + grid, ...
// (n fastest, so CTAs running at the same time share A rows in L2).  The row count may live on the
// device (ep.m_ptr, compacted human rows): no CTA is ever launched for an empty tile.  Rows are stored
// up to M (the output's extent), columns up to N (a multiple of BN).
// ACT (CN_ACT_*) and OUT (TC_OUT_*) select the epilogue of the non-PROMOTE instances (tc_epilogue_tma for BN = 256,
// tc_epilogue_store for BN = 64); the PROMOTE instance keeps the run-time epilogue below (activation from ep.act, atomic
// adds with split-K) and ignores them.  map_c / map_oh / map_ol: TMA store maps of the fp32 and split fp16 outputs,
// [M rows, N columns] with boxes of 64 rows x 128 bytes and the 128-byte swizzle; read by the BN = 256 non-PROMOTE
// instances only (the others get unused placeholders).
template <int BN, bool PROMOTE = false, int ACT = 0, int OUT = TC_OUT_F32>
__global__ void __launch_bounds__(TC_THREADS, 1)
cn_gemm_tc_kernel(const __grid_constant__ CUtensorMap map_ahi, const __grid_constant__ CUtensorMap map_alo,
                  const __grid_constant__ CUtensorMap map_bhi, const __grid_constant__ CUtensorMap map_blo,
                  int M, int N, int K, TcEpilogue ep, const __grid_constant__ CUtensorMap map_c,
                  const __grid_constant__ CUtensorMap map_oh, const __grid_constant__ CUtensorMap map_ol) {
  cn_pdl_trigger();                                 // PDL: the successor may be scheduled while this grid runs
  constexpr int TC_STAGES = TcCfg<BN>::kStages;
  constexpr int BK = TcCfg<BN>::kBK;
  constexpr int SW = TcCfg<BN>::kSwizzle;
  constexpr int TC_A_TILE_BYTES = TcCfg<BN>::kATile;
  constexpr int TC_B_TILE_BYTES = TcCfg<BN>::kBTile;
  constexpr int TC_STAGE_BYTES = TcCfg<BN>::kStageBytes;
  constexpr bool kTmaStore = !PROMOTE && BN == 256 && OUT != TC_OUT_GRU;
  static_assert(OUT != TC_OUT_GRU || (BN == 256 && !PROMOTE), "the GRU epilogue reads four 64-column gate blocks");
  static_assert(!PROMOTE || BK == 64, "PROMOTE sums 64-wide k-blocks");
  static_assert(!kTmaStore || TcCfg<BN>::kStoreBoxes > 0, "BN = 256 stages its output");
  extern __shared__ uint8_t tc_smem_raw[];
  const uint32_t raw = tc::smem_u32(tc_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                 // swizzled tiles need 1024-byte alignment
  const uint32_t staging = base + TC_STAGES * TC_STAGE_BYTES;   // BN = 256: output staging after the operand ring
  const uint32_t bar_base = staging + TcCfg<BN>::kStagingBytes; // barriers after them
  const uint32_t bar_full = bar_base, bar_empty = bar_base + 64;   // full[s] = +8 s ; empty[s] = +64 + 8 s

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
  const int num_kb = K / BK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < TC_STAGES; ++s) {
      tc::mbar_init(bar_full + 8 * s, 1);                     // producer's arrive.expect_tx
      tc::mbar_init(bar_empty + 8 * s, TC_CONSUMER_WARPS);    // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_ahi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_alo) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_bhi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_blo) : "memory");
    if constexpr (kTmaStore) {
      if constexpr ((OUT & TC_OUT_F32) != 0) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_c) : "memory");
      if constexpr ((OUT & TC_OUT_F16) != 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_oh) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&map_ol) : "memory");
      }
    }
  }
  __syncthreads();
  // PDL: everything above (barrier init, descriptor prefetch) overlaps the predecessor's tail;
  // global memory written by it (row counts, operands, bias) is only touched after this wait
  cn_pdl_wait();
  const int m_ext = M;
  if (ep.m_ptr) { const int mc = *ep.m_ptr; M = mc < M ? mc : M; }
  int m_lo = ep.m0_ptr ? *ep.m0_ptr : 0;
  if (m_lo > M) m_lo = M;
  const int n_ntiles = N / BN;
  const int n_mn = ((M - m_lo + TC_BM - 1) / TC_BM) * n_ntiles;
  // split-K only with PROMOTE: its block sums start from zero, so an empty slice adds zeros.  Without PROMOTE every
  // tile covers the whole K range (K >= 64), so the accumulator is always written and the slot ring stays in step.
  const int ksplit = (PROMOTE && ep.ksplit > 1) ? ep.ksplit : 1;
  const int kb_per = (num_kb + ksplit - 1) / ksplit;                 // k-blocks per slice (the last may be shorter)
  const int n_tiles = n_mn * ksplit;                                 // CTAs beyond it run zero tiles and exit

  if (wg == 0) {
    // ===================== TMA producer =====================
    tc::setmaxnreg_dec<40>();
    if (threadIdx.x == 0) {
      uint32_t it = 0;                                            // running k-block counter across tiles
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int mn = tile % n_mn, ks = tile / n_mn;
        const int m0 = m_lo + (mn / n_ntiles) * TC_BM, n0 = (mn % n_ntiles) * BN;
        const int kb0 = ks * kb_per, kb1 = (kb0 + kb_per < num_kb) ? kb0 + kb_per : num_kb;
        for (int kb = kb0; kb < kb1; ++kb, ++it) {
          const uint32_t s = it % TC_STAGES, ph = (it / TC_STAGES) & 1u;
          tc::mbar_wait(bar_empty + 8 * s, ph ^ 1u);              // slot free (first pass returns immediately)
          const uint32_t full = bar_full + 8 * s;
          tc::mbar_expect_tx(full, TC_STAGE_BYTES);
          const uint32_t st = base + s * TC_STAGE_BYTES;
          tc::tma_load_2d(st, &map_ahi, full, kb * BK, m0);
          tc::tma_load_2d(st + TC_A_TILE_BYTES, &map_alo, full, kb * BK, m0);
          tc::tma_load_2d(st + 2 * TC_A_TILE_BYTES, &map_bhi, full, kb * BK, n0);
          tc::tma_load_2d(st + 2 * TC_A_TILE_BYTES + TC_B_TILE_BYTES, &map_blo, full, kb * BK, n0);
        }
      }
    }
    return;
  }
  // ===================== consumers (warp groups 1, 2): MMA + epilogue =====================
  tc::setmaxnreg_inc<232>();
  float inv_scale = ep.inv_scale;
  if (ep.inv_scale_a) inv_scale *= __ldg(ep.inv_scale_a);
  if (ep.inv_scale_b) inv_scale *= __ldg(ep.inv_scale_b);
  const int half = wg - 1;                                        // rows [64 half, 64 half + 64) of the tile
  const int wr = 16 * (warp & 3) + (lane >> 2);                   // first accumulator row of this thread in its half
  const int cq = 2 * (lane & 3);                                  // first accumulator column inside each 8-column group
  uint32_t it = 0;
  TcStaging sg;                                                   // BN = 256: this warp group's output staging
  sg.base = staging + half * TcCfg<BN>::kStoreBoxes * TcCfg<BN>::kBoxBytes;
  sg.box = 0; sg.leader = (threadIdx.x & 127) == 0; sg.bar_id = wg;   // named barriers 1, 2 (0 = __syncthreads)
  TC_TRACE(sg.waits = 0; sg.wait_clk = 0;)
  // trace (CN_GEMM_TRACE builds only): consumer warp 0 (the issuing thread of warp group 1) records one
  // TC_TRACE_REC record per tile
  TC_TRACE(const bool tr = ep.trace && warp == 4 && lane == 0; int tr_n = 0;)
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const int mn = tile % n_mn, ks = tile / n_mn;
    const int m0 = m_lo + (mn / n_ntiles) * TC_BM, n0 = (mn % n_ntiles) * BN;
    const int kb0 = ks * kb_per, kb1 = (kb0 + kb_per < num_kb) ? kb0 + kb_per : num_kb;
    TC_TRACE(const uint64_t t_tile = tc::globaltimer(); uint64_t t_first = 0; uint32_t polls = 0;)
    float acc[BN / 2];
    float sum[PROMOTE ? BN / 2 : 1];
    if constexpr (PROMOTE) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) sum[i] = 0.0f;
    }
    uint32_t prev = 0;
    for (int kb = kb0; kb < kb1; ++kb, ++it) {
      const uint32_t s = it % TC_STAGES, ph = (it / TC_STAGES) & 1u;
#ifdef CN_GEMM_TRACE
      polls += tc::mbar_wait_polls(bar_full + 8 * s, ph);
      if (kb == kb0) t_first = tc::globaltimer();
#else
      tc::mbar_wait(bar_full + 8 * s, ph);                        // TMA bytes landed
#endif
      const uint32_t st = base + s * TC_STAGE_BYTES;
      const uint32_t a_hi = st + half * (TC_A_TILE_BYTES / 2), a_lo = a_hi + TC_A_TILE_BYTES,
                     b_hi = st + 2 * TC_A_TILE_BYTES, b_lo = b_hi + TC_B_TILE_BYTES;
      tc::fence_regs(acc);
      tc::wgmma_fence();
#pragma unroll
      for (int k = 0; k < BK / 16; ++k) {
        const uint32_t koff = k * 32;                             // 16 fp16 = 32 bytes inside the swizzle atom
        const uint64_t dah = tc::make_desc<SW>(a_hi + koff), dal = tc::make_desc<SW>(a_lo + koff);
        const uint64_t dbh = tc::make_desc<SW>(b_hi + koff), dbl = tc::make_desc<SW>(b_lo + koff);
        const bool first = k == 0 && (PROMOTE || kb == kb0);      // the MMA that starts a new sum overwrites acc
        tc::wgmma_f16<BN>(acc, dah, dbh, first ? 0u : 1u);
        tc::wgmma_f16<BN>(acc, dah, dbl, 1u);
        tc::wgmma_f16<BN>(acc, dal, dbh, 1u);
      }
      tc::wgmma_commit();
      tc::fence_regs(acc);
      if constexpr (PROMOTE) {
        tc::wgmma_wait<0>();                                      // this block's sum is needed now
        tc::fence_regs(acc);
        __syncwarp();
        if (lane == 0) tc::mbar_arrive(bar_empty + 8 * s);
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) sum[i] += acc[i];
      } else {
        // one k-block of MMAs stays in flight: the previous block's are done reading their slot
        tc::wgmma_wait<1>();
        if (kb != kb0) {
          __syncwarp();
          if (lane == 0) tc::mbar_arrive(bar_empty + 8 * prev);
        }
        prev = s;
      }
    }
    if constexpr (PROMOTE) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = sum[i];
    } else {
      tc::wgmma_wait<0>();
      tc::fence_regs(acc);
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(bar_empty + 8 * prev);
    }

    TC_TRACE(const uint64_t t_loop = tc::globaltimer();)
    if constexpr (!PROMOTE) {
      TC_TRACE(const uint32_t waits0 = sg.waits; const uint64_t clk0 = sg.wait_clk;)
      if constexpr (OUT == TC_OUT_GRU) {
        tc_epilogue_gru(acc, ep, inv_scale, n0, m0 + 64 * half + wr, cq, m_ext);
      } else if constexpr (kTmaStore) {
        tc_epilogue_tma<ACT, OUT>(acc, ep, inv_scale, n0, m0 + 64 * half, wr, lane, sg, &map_c, &map_oh, &map_ol);
      } else {
        tc_epilogue_store<BN, ACT, OUT>(acc, ep, inv_scale, n0, m0 + 64 * half + wr, cq, m_ext);
      }
      TC_TRACE(
        if (tr && tr_n < ep.trace_cap) {
          unsigned long long* rec = ep.trace + ((size_t)blockIdx.x * ep.trace_cap + tr_n) * TC_TRACE_REC;
          rec[0] = t_tile; rec[1] = t_first; rec[2] = t_loop; rec[3] = tc::globaltimer(); rec[4] = polls;
          rec[5] = sg.waits - waits0; rec[6] = sg.wait_clk - clk0;
        }
        ++tr_n;)
      continue;
    }
    // ---- PROMOTE epilogue: scale, bias, activation, stores (atomic adds with split-K) from the accumulator ----
    // activation is uniform over the tile unless the [act_lo, act_hi) window cuts through it
    const bool act_full = ep.act_lo <= n0 && ep.act_hi >= n0 + BN;
    const bool act_none = ep.act == 0 || ep.act_hi <= n0 || ep.act_lo >= n0 + BN;
    const int act_mode = act_none ? 0 : (act_full ? ep.act : 3);
    const bool with_bias = ep.bias && ks == 0;
    const int r0 = m0 + 64 * half + wr;
#pragma unroll
    for (int g = 0; g < BN / 8; ++g) {
      const int col = n0 + 8 * g + cq;
      const float b0 = with_bias ? __ldg(ep.bias + col) : 0.0f, b1 = with_bias ? __ldg(ep.bias + col + 1) : 0.0f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        float v0 = fmaf(acc[4 * g + 2 * h], inv_scale, b0), v1 = fmaf(acc[4 * g + 2 * h + 1], inv_scale, b1);
        if (act_mode == 1) {
          v0 = fmaxf(v0, 0.0f); v1 = fmaxf(v1, 0.0f);
        } else if (act_mode == 2) {
          v0 = tc::fast_tanh(v0); v1 = tc::fast_tanh(v1);
        } else if (act_mode == 3) {
          if (col >= ep.act_lo && col < ep.act_hi) v0 = (ep.act == 1) ? fmaxf(v0, 0.0f) : tc::fast_tanh(v0);
          if (col + 1 >= ep.act_lo && col + 1 < ep.act_hi) v1 = (ep.act == 1) ? fmaxf(v1, 0.0f) : tc::fast_tanh(v1);
        }
        if (row >= m_ext || ep.dbg_nostore) continue;
        if (ep.c32) {
          float* c = ep.c32 + (size_t)row * ep.ldc + col;
          if (ksplit > 1) {
            atomicAdd(c, v0);
            atomicAdd(c + 1, v1);
          } else {
            *reinterpret_cast<float2*>(c) = make_float2(v0, v1);
          }
        }
        if (ep.out_hi) {
          uint32_t lo;
          const uint32_t hi = tc::split_pair_hi(v0, v1, &lo);
          const size_t o = (size_t)row * ep.ldh + col;
          *reinterpret_cast<uint32_t*>(ep.out_hi + o) = hi;
          *reinterpret_cast<uint32_t*>(ep.out_lo + o) = lo;
        }
      }
    }
  }
  // BN = 256: the box stores must have completed before the CTA exits.  Its shared memory is released then, and a
  // dependent launch (griddepcontrol.wait after this grid) reads the output, visible only once the writes are done.
  if constexpr (kTmaStore) {
    if (sg.leader) tc::bulk_wait_all();
  }
}
