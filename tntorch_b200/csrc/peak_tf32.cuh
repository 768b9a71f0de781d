// Measured dense TF32 peaks of the tensor-core instructions the kernels use (SURVEY.md §8d: "the builder must measure a
// TF32 peak ... before quoting tensor-pipe fractions").  Every warp of two 256-thread CTAs per SM issues
// mma.sync.m16n8k8 .tf32 back to back on register operands into eight independent accumulators (no shared or global
// traffic: the tensor pipe is the only thing exercised); `reps` x `per_commit` MMAs per accumulator.
// FLOP = 2*16*8*8 per MMA.
// The Gram / A^T B kernel issues wgmma instead: peak_tf32_wgmma_kernel measures wgmma.mma_async m64n256k8 .tf32 with A
// from registers and B from a fixed K-major SWIZZLE_128B shared-memory buffer, two warpgroups per CTA, one CTA per SM,
// each warpgroup into its own 128 accumulators (the shape and operand sources of the Gram's 128 x 256 tile).
// `reps` commit groups of 4 x `per_commit` wgmma per warpgroup; FLOP = 2*64*256*8 per wgmma.
// The TT inner product (tt_dot.cuh) issues mma.sync m16n8k16 .f64 (DMMA): peak_f64_kernel measures it the way
// peak_tf32_kernel measures the TF32 MMA, two 256-thread CTAs per SM; FLOP = 2*16*8*16 per MMA.
#pragma once
#include "common.cuh"
#include "gram_tc.cuh"
#include "tt_dot.cuh"

namespace tnb {

constexpr int PK_THREADS = 256;
constexpr int PK_ACC = 8;

__global__ void __launch_bounds__(PK_THREADS) peak_tf32_kernel(int reps, int per_commit, float* sink) {
  const uint32_t x = __float_as_uint(1.0f + (float)(threadIdx.x & 7) * 0.125f);
  const uint32_t y = __float_as_uint(0.5f + (float)(threadIdx.x >> 5) * 0.0625f);
  float acc[PK_ACC][4] = {};
  for (int r = 0; r < reps; ++r)
    for (int m = 0; m < per_commit; ++m)
#pragma unroll
      for (int a = 0; a < PK_ACC; ++a) mma_tf32(acc[a], x, y, x, y, x, y);
  float s = 0.f;
#pragma unroll
  for (int a = 0; a < PK_ACC; ++a) s += acc[a][0] + acc[a][1] + acc[a][2] + acc[a][3];
  if (sink && s == 12345.f) sink[0] = s;  // keeps the products live; never true for these operands
}

__global__ void __launch_bounds__(PK_THREADS) peak_f64_kernel(int reps, int per_commit, double* sink) {
  const double x = 1.0 + (double)(threadIdx.x & 7) * 0.125, y = 0.5 + (double)(threadIdx.x >> 5) * 0.0625;
  const double a[8] = {x, y, x, y, x, y, x, y}, b[4] = {y, x, y, x};
  double acc[PK_ACC][4] = {};
  for (int r = 0; r < reps; ++r)
    for (int m = 0; m < per_commit; ++m)
#pragma unroll
      for (int k = 0; k < PK_ACC; ++k) dmma_16816(acc[k], a, b);
  double s = 0.0;
#pragma unroll
  for (int k = 0; k < PK_ACC; ++k) s += acc[k][0] + acc[k][1] + acc[k][2] + acc[k][3];
  if (sink && s == 12345.0) sink[0] = s;  // keeps the products live; never true for these operands
}

constexpr int PKW_THREADS = 256;

__global__ void __launch_bounds__(PKW_THREADS, 1) peak_tf32_wgmma_kernel(int reps, int per_commit, float* sink) {
  __shared__ __align__(1024) float b_sm[256 * 32];  // 256 rows of B^T x 32 k: four k8 slices
  for (int i = threadIdx.x; i < 256 * 32; i += PKW_THREADS) b_sm[i] = 0.25f + (float)(i & 7) * 0.03125f;
  fence_proxy_async_smem();
  __syncthreads();
  const uint32_t x = __float_as_uint(1.0f + (float)(threadIdx.x & 7) * 0.125f);
  const uint32_t y = __float_as_uint(0.5f + (float)(threadIdx.x >> 5) * 0.0625f);
  const uint32_t a[4] = {x, y, x, y};
  const uint64_t desc0 = wgmma_desc_kmajor_sw128(b_sm);
  const uint64_t desc[4] = {desc0, desc0 + 2, desc0 + 4, desc0 + 6};
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  wgmma_fence_operand(acc);
  for (int r = 0; r < reps; ++r) {
    wgmma_fence();
    for (int m = 0; m < per_commit; ++m)
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma_tf32<8>(acc, a, desc[kk]);
    wgmma_commit();
    wgmma_wait<0>();
  }
  wgmma_fence_operand(acc);
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 128; ++i) s += acc[i];
  if (sink && s == 12345.f) sink[0] = s;  // keeps the products live; never true for these operands
}

// Returns TFLOP/s of the best of `trials` timed launches (CUDA events on `st`); wgmma selects peak_tf32_wgmma_kernel,
// f64 peak_f64_kernel.
inline int measure_tf32_peak(int reps, int per_commit, int trials, double* tflops_out, double* ms_out, cudaStream_t st,
                             bool wgmma = false, bool f64 = false) {
  if (!tc_path_available()) return fail(TNB_ERR_UNSUPPORTED, "tensor-core path not available on this device");
  const int blocks = (wgmma ? 1 : 2) * device_info().sm_count;
  void* sink = nullptr;
  TNB_CUDA(cudaMalloc(&sink, 256));
  cudaEvent_t e0, e1;
  TNB_CUDA(cudaEventCreate(&e0));
  TNB_CUDA(cudaEventCreate(&e1));
  double best = 1e30;
  for (int t = 0; t < trials + 2; ++t) {
    TNB_CUDA(cudaEventRecord(e0, st));
    if (f64)
      peak_f64_kernel<<<blocks, PK_THREADS, 0, st>>>(reps, per_commit, static_cast<double*>(sink));
    else if (wgmma)
      peak_tf32_wgmma_kernel<<<blocks, PKW_THREADS, 0, st>>>(reps, per_commit, static_cast<float*>(sink));
    else
      peak_tf32_kernel<<<blocks, PK_THREADS, 0, st>>>(reps, per_commit, static_cast<float*>(sink));
    TNB_CUDA(cudaEventRecord(e1, st));
    TNB_CUDA(cudaEventSynchronize(e1));
    TNB_COUNT_LAUNCH();
    cudaError_t le = cudaGetLastError();
    if (le != cudaSuccess) return fail(TNB_ERR_CUDA, "peak kernel: %s", cudaGetErrorString(le));
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    if (t >= 2 && ms < best) best = ms;
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(sink);
  const double flop = f64 ? 2.0 * 16 * 8 * 16 * PK_ACC * (double)reps * per_commit * (PK_THREADS / 32) * blocks
                    : wgmma ? 2.0 * 64 * 256 * 8 * 4 * (double)reps * per_commit * (PKW_THREADS / 128) * blocks
                            : 2.0 * 16 * 8 * 8 * PK_ACC * (double)reps * per_commit * (PK_THREADS / 32) * blocks;
  *tflops_out = flop / (best * 1e-3) / 1e12;
  if (ms_out) *ms_out = best;
  return TNB_OK;
}

}  // namespace tnb
