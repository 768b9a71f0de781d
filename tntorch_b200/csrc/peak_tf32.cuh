// Measured dense TF32 peak of the tensor-core instruction the kernels use (SURVEY.md §8d: "the builder must measure a
// TF32 peak ... before quoting tensor-pipe fractions").  Every warp of two 256-thread CTAs per SM issues
// mma.sync.m16n8k8 .tf32 back to back on register operands into eight independent accumulators (no shared or global
// traffic: the tensor pipe is the only thing exercised); `reps` x `per_commit` MMAs per accumulator.
// FLOP = 2*16*8*8 per MMA.
#pragma once
#include "common.cuh"
#include "gram_tc.cuh"

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

// Returns TFLOP/s of the best of `trials` timed launches (CUDA events on `st`).
inline int measure_tf32_peak(int reps, int per_commit, int trials, double* tflops_out, double* ms_out, cudaStream_t st) {
  if (!tc_path_available()) return fail(TNB_ERR_UNSUPPORTED, "tensor-core path not available on this device");
  const int blocks = 2 * device_info().sm_count;
  float* sink = nullptr;
  TNB_CUDA(cudaMalloc(&sink, 256));
  cudaEvent_t e0, e1;
  TNB_CUDA(cudaEventCreate(&e0));
  TNB_CUDA(cudaEventCreate(&e1));
  double best = 1e30;
  for (int t = 0; t < trials + 2; ++t) {
    TNB_CUDA(cudaEventRecord(e0, st));
    peak_tf32_kernel<<<blocks, PK_THREADS, 0, st>>>(reps, per_commit, sink);
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
  const double flop = 2.0 * 16 * 8 * 8 * PK_ACC * (double)reps * per_commit * (PK_THREADS / 32) * blocks;
  *tflops_out = flop / (best * 1e-3) / 1e12;
  if (ms_out) *ms_out = best;
  return TNB_OK;
}

}  // namespace tnb
