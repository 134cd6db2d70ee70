// Bulk recorder of the collect environment's pred_info observations (collect_data.py:54-62 at thousands of
// environments).  collect_data.py keeps, every pred_interval steps, each environment's rows whose py is finite, in frame
// order then human index, and writes one text file per environment.  Here the rows stay on the device for a whole chunk
// of frames: every append copies one observation into the chunk and counts each environment's visible rows (one warp per
// environment, ballot + popcount); a flush turns the per-(environment, frame) counts into offsets with a device prefix
// sum, scatters the visible rows packed in environment-major order (environment, frame, human) and copies only those
// rows, plus the per-environment row counts, to the host: one synchronisation per chunk, none per step.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "../../include/crowdnav_b200.h"
#include "cn_host_util.h"

namespace {

#define CN_REC_SCAN_THREADS 1024

// chunk slot `c` <- the observation; cnt[e * C + c] = visible rows of environment e
__global__ void __launch_bounds__(256) cn_rec_append_kernel(const float4* __restrict__ obs, float4* __restrict__ chunk,
                                                           int* __restrict__ cnt, int N, int H, int C, int c) {
  const int e = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (e >= N) return;
  const float4* src = obs + (size_t)e * H;
  float4* dst = chunk + ((size_t)c * N + e) * H;
  int n = 0;
  for (int h0 = 0; h0 < H; h0 += 32) {
    const int h = h0 + lane;
    bool vis = false;
    if (h < H) {
      const float4 r = src[h];
      dst[h] = r;
      vis = !isinf(r.w);                       // np.isinf(pred_info[i, :, -1])
    }
    n += __popc(__ballot_sync(0xffffffffu, vis));
  }
  if (lane == 0) cnt[(size_t)e * C + c] = n;
}

// exclusive prefix sum of cnt[0..M) -> off[0..M], off[M] = total; env_rows[e] = rows of environment e (C slots each)
__global__ void __launch_bounds__(CN_REC_SCAN_THREADS) cn_rec_scan_kernel(const int* __restrict__ cnt, int64_t* __restrict__ off,
                                                                          int64_t* __restrict__ env_rows, int M, int C) {
  __shared__ int64_t part[CN_REC_SCAN_THREADS];
  const int t = threadIdx.x;
  const int per = (M + CN_REC_SCAN_THREADS - 1) / CN_REC_SCAN_THREADS;
  const int lo = t * per, hi = min(M, lo + per);
  int64_t sum = 0;
  for (int i = lo; i < hi; ++i) sum += cnt[i];
  part[t] = sum;
  __syncthreads();
  for (int d = 1; d < CN_REC_SCAN_THREADS; d <<= 1) {   // Hillis-Steele inclusive scan of the segment sums
    const int64_t v = t >= d ? part[t - d] : 0;
    __syncthreads();
    part[t] += v;
    __syncthreads();
  }
  int64_t run = part[t] - sum;
  for (int i = lo; i < hi; ++i) { off[i] = run; run += cnt[i]; }
  if (t == CN_REC_SCAN_THREADS - 1) off[M] = part[t];
  __syncthreads();
  for (int e = t; e < M / C; e += CN_REC_SCAN_THREADS) env_rows[e] = off[(size_t)(e + 1) * C] - off[(size_t)e * C];
}

// one warp per (environment, frame slot): the visible rows in human order at their packed offset
__global__ void __launch_bounds__(256) cn_rec_scatter_kernel(const float4* __restrict__ chunk, const int64_t* __restrict__ off,
                                                            float4* __restrict__ packed, int N, int H, int C, int frames) {
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= N * frames) return;
  const int e = w / frames, c = w - e * frames;
  const float4* src = chunk + ((size_t)c * N + e) * H;
  int64_t o = off[(size_t)e * C + c];
  for (int h0 = 0; h0 < H; h0 += 32) {
    const int h = h0 + lane;
    float4 r = make_float4(0.f, 0.f, 0.f, INFINITY);
    if (h < H) r = src[h];
    const bool vis = h < H && !isinf(r.w);
    const uint32_t m = __ballot_sync(0xffffffffu, vis);
    if (vis) packed[o + __popc(m & ((1u << lane) - 1u))] = r;
    o += __popc(m);
  }
}

}  // namespace

struct cn_recorder {
  int N, H, C, device;
  int frames;            // frames appended since the last flush
  float4* chunk;         // [C][N][H]
  float4* packed;        // [C * N * H] (worst case: every row visible)
  int* cnt;              // [N][C]
  int64_t* off;          // [N * C + 1]
  int64_t* env_rows;     // [N]
  int64_t rows_total;    // rows flushed so far (all chunks)
};

extern "C" {

int cn_recorder_create(int num_envs, int human_num, int chunk_frames, int device, cn_recorder** out) {
  if (!out) return cn_set_error("cn_recorder_create: null argument");
  *out = nullptr;
  if (num_envs <= 0 || human_num <= 0 || human_num > 128 || chunk_frames <= 0)
    return cn_set_error("cn_recorder_create: need num_envs > 0, 0 < human_num <= 128, chunk_frames > 0 (got %d, %d, %d)",
                        num_envs, human_num, chunk_frames);
  CnDeviceGuard guard(device);
  cn_recorder* r = new cn_recorder();
  r->N = num_envs; r->H = human_num; r->C = chunk_frames; r->device = device; r->frames = 0; r->rows_total = 0;
  const size_t rows = (size_t)chunk_frames * num_envs * human_num, M = (size_t)num_envs * chunk_frames;
  cudaError_t err = cudaMalloc(&r->chunk, rows * sizeof(float4));
  if (err == cudaSuccess) err = cudaMalloc(&r->packed, rows * sizeof(float4));
  if (err == cudaSuccess) err = cudaMalloc(&r->cnt, M * sizeof(int));
  if (err == cudaSuccess) err = cudaMalloc(&r->off, (M + 1) * sizeof(int64_t));
  if (err == cudaSuccess) err = cudaMalloc(&r->env_rows, num_envs * sizeof(int64_t));
  if (err == cudaSuccess) err = cudaMemset(r->cnt, 0, M * sizeof(int));
  if (err != cudaSuccess) {
    cn_recorder_destroy(r);
    return cn_set_error("cn_recorder_create: %s", cudaGetErrorString(err));
  }
  *out = r;
  return 0;
}

int cn_recorder_destroy(cn_recorder* r) {
  if (!r) return 0;
  CnDeviceGuard guard(r->device);
  cudaDeviceSynchronize();
  cudaFree(r->chunk); cudaFree(r->packed); cudaFree(r->cnt); cudaFree(r->off); cudaFree(r->env_rows);
  delete r;
  return 0;
}

int cn_recorder_append(cn_recorder* r, const float* d_pred_info, void* stream) {
  if (!r || !d_pred_info) return cn_set_error("cn_recorder_append: null argument");
  if (r->frames >= r->C) return cn_set_error("cn_recorder_append: chunk full (%d frames): flush first", r->C);
  CnDeviceGuard guard(r->device);
  cn_rec_append_kernel<<<(r->N + 7) / 8, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float4*>(d_pred_info), r->chunk, r->cnt, r->N, r->H, r->C, r->frames);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("cn_recorder_append launch: %s", cudaGetErrorString(err));
  r->frames += 1;
  return 0;
}

int cn_recorder_pending(cn_recorder* r) { return r ? r->frames : 0; }

int cn_recorder_flush(cn_recorder* r, float* h_rows, int64_t* h_env_rows, int64_t* n_rows, void* stream) {
  if (!r || !h_rows || !h_env_rows || !n_rows) return cn_set_error("cn_recorder_flush: null argument");
  CnDeviceGuard guard(r->device);
  cudaStream_t st = (cudaStream_t)stream;
  *n_rows = 0;
  if (r->frames == 0) {
    memset(h_env_rows, 0, r->N * sizeof(int64_t));
    return 0;
  }
  // slots the chunk did not fill count nothing
  if (r->frames < r->C)
    cudaMemset2DAsync(r->cnt + r->frames, r->C * sizeof(int), 0, (r->C - r->frames) * sizeof(int), r->N, st);
  const int M = r->N * r->C;
  cn_rec_scan_kernel<<<1, CN_REC_SCAN_THREADS, 0, st>>>(r->cnt, r->off, r->env_rows, M, r->C);
  const int warps = r->N * r->frames;
  cn_rec_scatter_kernel<<<(warps + 7) / 8, 256, 0, st>>>(r->chunk, r->off, r->packed, r->N, r->H, r->C, r->frames);
  cudaError_t err = cudaGetLastError();
  if (err != cudaSuccess) return cn_set_error("cn_recorder_flush launch: %s", cudaGetErrorString(err));
  int64_t total = 0;
  err = cudaMemcpyAsync(&total, r->off + M, sizeof(int64_t), cudaMemcpyDeviceToHost, st);
  if (err == cudaSuccess) err = cudaMemcpyAsync(h_env_rows, r->env_rows, r->N * sizeof(int64_t), cudaMemcpyDeviceToHost, st);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);
  if (err == cudaSuccess && total > 0)
    err = cudaMemcpyAsync(h_rows, r->packed, (size_t)total * sizeof(float4), cudaMemcpyDeviceToHost, st);
  if (err == cudaSuccess) err = cudaStreamSynchronize(st);
  if (err != cudaSuccess) return cn_set_error("cn_recorder_flush: %s", cudaGetErrorString(err));
  *n_rows = total;
  r->rows_total += total;
  r->frames = 0;
  return 0;
}

}  // extern "C"
