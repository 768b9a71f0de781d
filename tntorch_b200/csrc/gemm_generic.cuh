// Generic CUDA-core GEMM used for every shape/dtype the tensor-core kernels do not cover:
// fp64 everywhere, fp32 with fp32 or fp64 accumulation, bf16 or fp16 operands (dense TT-SVD input), ragged sizes, both
// storage orders.
//
//   C[M,N] = alpha * sum_k A(m,k) * B(k,n)  (+ beta * D + gamma * E)
//
// A(m,k) is stored either [M][K] (A_KMAJ: k contiguous) or [K][M] (m contiguous);
// B(k,n) is stored either [N][K] (B_KMAJ: k contiguous) or [K][N] (n contiguous).
// 64x64x16 tiles, 256 threads, 4x4 register micro-tile; optional split-K over gridDim.z with
// a deterministic second pass (no atomics, bit-reproducible).
#pragma once
#include "common.cuh"

namespace tnb {

constexpr int GEMM_BM = 64, GEMM_BN = 64, GEMM_BK = 16, GEMM_THREADS = 256;

// Operand load: the one place an element becomes the accumulation type (bf16 and fp16 through fp32, exactly).
template <typename TAcc, typename T>
__device__ __forceinline__ TAcc gemm_ld(const T& v) {
  return (TAcc)v;
}
template <typename TAcc>
__device__ __forceinline__ TAcc gemm_ld(const __nv_bfloat16& v) {
  return (TAcc)__bfloat162float(v);
}
template <typename TAcc>
__device__ __forceinline__ TAcc gemm_ld(const __half& v) {
  return (TAcc)__half2float(v);
}

template <typename TA, typename TB, typename TAcc, typename TC>
struct GemmArgs {
  int64_t M, N, K;
  const TA* A;
  int64_t lda;
  const TB* B;
  int64_t ldb;
  // split-K
  int64_t k_per_split;
  TAcc* partial;  // [splits][M][N] when !DIRECT
  // direct epilogue
  TC* C;
  int64_t ldc;
  TAcc alpha;
  const TC* D;
  int64_t ldd;
  TAcc beta;
  const TC* E;
  int64_t lde;
  TAcc gamma;
  int symmetric;  // only tiles with tn >= tm (A and B describe the same matrix)
  // batched accumulation: C = sum_b A_b * B_b with A_b = A + b*batch_stride_a (same K each); split z then owns
  // batches [z*batches_per_split, ...) instead of a K range.  nbatch == 0: plain GEMM.
  int64_t nbatch, batches_per_split, batch_stride_a, batch_stride_b;
  // speculative enqueue (common.cuh::tnb_skip): nullptr = always run
  const int* skip_words;
  int skip_stage;
};

template <typename TA, typename TB, typename TAcc, typename TC, bool A_KMAJ, bool B_KMAJ, bool DIRECT>
__global__ void __launch_bounds__(GEMM_THREADS) gemm_tile_kernel(const GemmArgs<TA, TB, TAcc, TC> p) {
  __shared__ __align__(16) TAcc As[GEMM_BK][GEMM_BM + 4];
  __shared__ __align__(16) TAcc Bs[GEMM_BK][GEMM_BN + 4];
  const int tm = blockIdx.x, tn = blockIdx.y, z = blockIdx.z;
  if (p.symmetric && tn < tm) return;
  if (tnb_skip(p.skip_words, p.skip_stage)) return;
  const int64_t m0 = (int64_t)tm * GEMM_BM, n0 = (int64_t)tn * GEMM_BN;
  int64_t kbeg = (int64_t)z * p.k_per_split;
  int64_t kend = (kbeg + p.k_per_split < p.K) ? kbeg + p.k_per_split : p.K;
  int64_t b0 = 0, b1 = 1;
  if (p.nbatch > 0) {
    kbeg = 0;
    kend = p.K;
    b0 = (int64_t)z * p.batches_per_split;
    b1 = b0 + p.batches_per_split < p.nbatch ? b0 + p.batches_per_split : p.nbatch;
  }
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  TAcc acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = TAcc(0);

  for (int64_t bb = b0; bb < b1; ++bb) {
  const TA* Ab = p.A + bb * p.batch_stride_a;
  const TB* Bb = p.B + bb * p.batch_stride_b;
  for (int64_t k0 = kbeg; k0 < kend; k0 += GEMM_BK) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + i * GEMM_THREADS;
      int kk, mm;
      if (A_KMAJ) {
        mm = idx >> 4;
        kk = idx & 15;
      } else {
        kk = idx >> 6;
        mm = idx & 63;
      }
      const int64_t gm = m0 + mm, gk = k0 + kk;
      TAcc v = TAcc(0);
      if (gm < p.M && gk < kend) v = gemm_ld<TAcc>(A_KMAJ ? Ab[gm * p.lda + gk] : Ab[gk * p.lda + gm]);
      As[kk][mm] = v;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int idx = tid + i * GEMM_THREADS;
      int kk, nn;
      if (B_KMAJ) {
        nn = idx >> 4;
        kk = idx & 15;
      } else {
        kk = idx >> 6;
        nn = idx & 63;
      }
      const int64_t gn = n0 + nn, gk = k0 + kk;
      TAcc v = TAcc(0);
      if (gn < p.N && gk < kend) v = gemm_ld<TAcc>(B_KMAJ ? Bb[gn * p.ldb + gk] : Bb[gk * p.ldb + gn]);
      Bs[kk][nn] = v;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < GEMM_BK; ++kk) {
      TAcc a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t gm = m0 + ty * 4 + i;
    if (gm >= p.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t gn = n0 + tx * 4 + j;
      if (gn >= p.N) continue;
      if (DIRECT) {
        TAcc v = p.alpha * acc[i][j];
        if (p.D) v += p.beta * (TAcc)p.D[gm * p.ldd + gn];
        if (p.E) v += p.gamma * (TAcc)p.E[gm * p.lde + gn];
        p.C[gm * p.ldc + gn] = (TC)v;
      } else {
        p.partial[((int64_t)z * p.M + gm) * p.N + gn] = acc[i][j];
      }
    }
  }
}

// Second pass of split-K: sum the partials in a fixed order, apply the epilogue, mirror the
// upper tiles of a symmetric product into the lower triangle, convert to the output type.
// Optionally writes a second copy C2 (type TC2) — used to emit G in fp64 and fp32 at once.
template <typename TAcc, typename TC, typename TC2>
__global__ void gemm_finalize_kernel(const TAcc* __restrict__ partial, int splits, int64_t M, int64_t N, TC* C,
                                     int64_t ldc, TAcc alpha, const TC* D, int64_t ldd, TAcc beta, const TC* E,
                                     int64_t lde, TAcc gamma, int symmetric, TC2* C2, int64_t ldc2,
                                     const int* skip_words = nullptr, int skip_stage = 0) {
  if (tnb_skip(skip_words, skip_stage)) return;
  const int64_t total = M * N;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = idx / N, n = idx % N;
    int64_t sm = m, sn = n;
    if (symmetric && (m / GEMM_BM) > (n / GEMM_BN)) {
      sm = n;
      sn = m;
    }
    TAcc s = TAcc(0);
    for (int z = 0; z < splits; ++z) s += partial[((int64_t)z * M + sm) * N + sn];
    TAcc v = alpha * s;
    if (D) v += beta * (TAcc)D[m * ldd + n];
    if (E) v += gamma * (TAcc)E[m * lde + n];
    C[m * ldc + n] = (TC)v;
    if (C2) C2[m * ldc2 + n] = (TC2)v;
  }
}

struct GemmPlan {
  int splits = 1;
  int64_t k_per_split = 0;
  size_t partial_elems = 0;
};

// Pick a split-K factor that fills the machine (~2 waves of CTAs) without making slices tiny.
inline GemmPlan plan_gemm(int64_t M, int64_t N, int64_t K, bool symmetric, int force_splits = 0) {
  GemmPlan pl;
  const int64_t tm = ceil_div<int64_t>(M, GEMM_BM), tn = ceil_div<int64_t>(N, GEMM_BN);
  int64_t tiles = symmetric ? tm * (tn + 1) / 2 : tm * tn;
  if (tiles < 1) tiles = 1;
  int sms = device_info().valid ? device_info().sm_count : 132;
  int64_t want = ceil_div<int64_t>(2 * (int64_t)sms * 2, tiles);  // 2 CTAs/SM resident, 2 waves
  int64_t max_by_k = K / 64 > 0 ? K / 64 : 1;
  int64_t s = want < max_by_k ? want : max_by_k;
  if (s < 1) s = 1;
  if (s > 64) s = 64;
  if (force_splits > 0) s = force_splits;
  int64_t kps = ceil_div<int64_t>(K, s);
  kps = ceil_div<int64_t>(kps, GEMM_BK) * GEMM_BK;
  if (kps < GEMM_BK) kps = GEMM_BK;
  s = ceil_div<int64_t>(K, kps);
  if (s < 1) s = 1;
  pl.splits = (int)s;
  pl.k_per_split = kps;
  pl.partial_elems = (size_t)s * (size_t)M * (size_t)N;
  return pl;
}

template <typename TA, typename TB, typename TAcc, typename TC, bool DIRECT>
inline int launch_gemm_tiles(const GemmArgs<TA, TB, TAcc, TC>& a, bool a_kmaj, bool b_kmaj, int splits,
                             cudaStream_t st) {
  if (a.M <= 0 || a.N <= 0) return TNB_OK;
  const int64_t tm = ceil_div<int64_t>(a.M, GEMM_BM), tn = ceil_div<int64_t>(a.N, GEMM_BN);
  if (tn > 65535 || splits > 65535) return fail(TNB_ERR_UNSUPPORTED, "gemm: N tile count %lld too large", (long long)tn);
  dim3 grid((unsigned)tm, (unsigned)tn, (unsigned)splits);
  if (a_kmaj && b_kmaj)
    gemm_tile_kernel<TA, TB, TAcc, TC, true, true, DIRECT><<<grid, GEMM_THREADS, 0, st>>>(a);
  else if (a_kmaj && !b_kmaj)
    gemm_tile_kernel<TA, TB, TAcc, TC, true, false, DIRECT><<<grid, GEMM_THREADS, 0, st>>>(a);
  else if (!a_kmaj && b_kmaj)
    gemm_tile_kernel<TA, TB, TAcc, TC, false, true, DIRECT><<<grid, GEMM_THREADS, 0, st>>>(a);
  else
    gemm_tile_kernel<TA, TB, TAcc, TC, false, false, DIRECT><<<grid, GEMM_THREADS, 0, st>>>(a);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// One-pass GEMM with fused epilogue (no split-K): C = alpha*A*B + beta*D + gamma*E.
template <typename TA, typename TB, typename TAcc, typename TC>
inline int gemm_direct(int64_t M, int64_t N, int64_t K, const TA* A, int64_t lda, bool a_kmaj, const TB* B,
                       int64_t ldb, bool b_kmaj, TC* C, int64_t ldc, TAcc alpha, const TC* D, int64_t ldd, TAcc beta,
                       const TC* E, int64_t lde, TAcc gamma, cudaStream_t st) {
  GemmArgs<TA, TB, TAcc, TC> a{};
  a.M = M; a.N = N; a.K = K; a.A = A; a.lda = lda; a.B = B; a.ldb = ldb;
  a.k_per_split = K > 0 ? K : 1; a.partial = nullptr;
  a.C = C; a.ldc = ldc; a.alpha = alpha; a.D = D; a.ldd = ldd; a.beta = beta; a.E = E; a.lde = lde; a.gamma = gamma;
  a.symmetric = 0;
  return launch_gemm_tiles<TA, TB, TAcc, TC, true>(a, a_kmaj, b_kmaj, 1, st);
}

// Split-K GEMM: partial sums into `partial` (plan.partial_elems of TAcc), then finalize.
template <typename TA, typename TB, typename TAcc, typename TC, typename TC2 = TC>
inline int gemm_splitk(const GemmPlan& pl, int64_t M, int64_t N, int64_t K, const TA* A, int64_t lda, bool a_kmaj,
                       const TB* B, int64_t ldb, bool b_kmaj, TAcc* partial, TC* C, int64_t ldc, TAcc alpha,
                       const TC* D, int64_t ldd, TAcc beta, const TC* E, int64_t lde, TAcc gamma, bool symmetric,
                       TC2* C2, int64_t ldc2, cudaStream_t st, const int* skip_words = nullptr, int skip_stage = 0) {
  if (M <= 0 || N <= 0) return TNB_OK;
  GemmArgs<TA, TB, TAcc, TC> a{};
  a.M = M; a.N = N; a.K = K; a.A = A; a.lda = lda; a.B = B; a.ldb = ldb;
  a.k_per_split = pl.k_per_split; a.partial = partial;
  a.C = nullptr; a.symmetric = symmetric ? 1 : 0;
  a.skip_words = skip_words; a.skip_stage = skip_stage;
  TNB_TRY((launch_gemm_tiles<TA, TB, TAcc, TC, false>(a, a_kmaj, b_kmaj, pl.splits, st)));
  const int64_t total = M * N;
  int blocks = (int)(ceil_div<int64_t>(total, 256) < 4096 ? ceil_div<int64_t>(total, 256) : 4096);
  gemm_finalize_kernel<TAcc, TC, TC2><<<blocks, 256, 0, st>>>(partial, pl.splits, M, N, C, ldc, alpha, D, ldd, beta, E,
                                                              lde, gamma, symmetric ? 1 : 0, C2, ldc2, skip_words, skip_stage);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// C = sum_{b < nbatch} A_b B_b (same shapes, A_b = A + b*stride): split over batches, deterministic reduce.
// partial must hold plan_batched(...).partial_elems TAcc's.
inline GemmPlan plan_batched(int64_t M, int64_t N, int64_t nbatch, bool symmetric) {
  GemmPlan pl;
  const int64_t tm = ceil_div<int64_t>(M, GEMM_BM), tn = ceil_div<int64_t>(N, GEMM_BN);
  int64_t tiles = symmetric ? tm * (tn + 1) / 2 : tm * tn;
  int sms = device_info().valid ? device_info().sm_count : 132;
  int64_t s = ceil_div<int64_t>(4 * (int64_t)sms, tiles);
  if (s > nbatch) s = nbatch;
  if (s > 256) s = 256;
  if (s < 1) s = 1;
  const int64_t bps = ceil_div<int64_t>(nbatch, s);
  s = ceil_div<int64_t>(nbatch, bps);
  pl.splits = (int)s;
  pl.k_per_split = bps;  // re-used as batches per split
  pl.partial_elems = (size_t)s * (size_t)M * (size_t)N;
  return pl;
}

template <typename TA, typename TB, typename TAcc, typename TC>
inline int gemm_batched_sum(const GemmPlan& pl, int64_t M, int64_t N, int64_t K, int64_t nbatch, const TA* A, int64_t lda,
                            bool a_kmaj, int64_t bsa, const TB* B, int64_t ldb, bool b_kmaj, int64_t bsb, TAcc* partial,
                            TC* C, int64_t ldc, bool symmetric, cudaStream_t st) {
  if (M <= 0 || N <= 0) return TNB_OK;
  GemmArgs<TA, TB, TAcc, TC> a{};
  a.M = M; a.N = N; a.K = K; a.A = A; a.lda = lda; a.B = B; a.ldb = ldb;
  a.k_per_split = K; a.partial = partial; a.C = nullptr; a.symmetric = symmetric ? 1 : 0;
  a.nbatch = nbatch; a.batches_per_split = pl.k_per_split; a.batch_stride_a = bsa; a.batch_stride_b = bsb;
  TNB_TRY((launch_gemm_tiles<TA, TB, TAcc, TC, false>(a, a_kmaj, b_kmaj, pl.splits, st)));
  const int64_t total = M * N;
  int blocks = (int)(ceil_div<int64_t>(total, 256) < 4096 ? ceil_div<int64_t>(total, 256) : 4096);
  gemm_finalize_kernel<TAcc, TC, TC><<<blocks, 256, 0, st>>>(partial, pl.splits, M, N, C, ldc, (TAcc)1, nullptr, 0, (TAcc)0,
                                                            nullptr, 0, (TAcc)0, symmetric ? 1 : 0, (TC*)nullptr, 0);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

}  // namespace tnb
