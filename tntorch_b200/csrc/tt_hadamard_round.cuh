// Rounding of the elementwise (Hadamard) product of two tensor trains (tnb_tt_hadamard_round): round_tt(a * b) without
// forming the Kronecker cores C_k[:, i, :] = A_k[:, i, :] (x) B_k[:, i, :] of bond rank R_k = ra_k rb_k.
//
// It is a Gram form of the sweep tt_round_impl runs on C:
//   left Grams   GL_0 = [1],  GL_{k+1} = sum_i C_i^T GL_k C_i   (R_{k+1} x R_{k+1}),  kept for k = 1 .. N-1;
//   truncation   W_N = [1];  at bond mu = N-1 .. 1:  Y = C_mu W_{mu+1}  (R_mu x I_mu r'),  H = Y^T GL_mu Y  (the Gram of
//                the carry tt_round_impl truncates at this bond),  eigenpairs of H -> the rank rule of truncate_step,
//                core mu = V_r^T (orthonormal rows),  W_mu = Y V_r;  core 0 = C_0 W_1.
// No square root or inverse of GL is taken, so a singular GL (more Kronecker rank than the left unfolding has) is harmless.
// The nested projections' errors are mutually orthogonal: the discarded eigenvalues of every bond add up to
// ||C - round(C)||^2, returned with ||C||^2 = trace(H) at the first bond.
//
// GL_k is read as a 4-index tensor [a, b, c, d] (row (a, b), column (c, d)); one mode of the recurrence is four
// contractions of the leading index, each one GEMM  out(m, n) = sum_k X(k, m) Y(k, n)  per mode value i:
//   T1[b c d, a'] = sum_a  GL[a, b c d]   A[a, i, a']
//   T2[c d a', b'] = sum_b  T1[b, c d a']  B[b, i, b']
//   T3[d a' b', c'] = sum_c  T2[c, d a' b'] A[c, i, c']
//   GL'[a' b' c', d'] += sum_d T3[d, a' b' c'] B[d, i, d']      (8 I r^5 flops a mode at equal ranks)
// A launch takes a chunk of tthr_chunk mode values (blockIdx.z); the last contraction sums its chunk in registers, in i
// order, and adds the chunk to GL' chunk after chunk: no atomics, so a call is bitwise reproducible, and the chunk depends
// on the shapes only.  Y, GL Y, H and W use the same GEMM.
//
// All arithmetic is fp64: fp32 cores are widened exactly as they are loaded; the output cores take the input dtype.
// Inside the envelope (tthr_mode_path: every rank of the mode in [16, 256]) a mode runs tthr_gemm_tc_kernel, fp64
// mma.sync m16n8k16 (DMMA, the fragments of ttd_mode_tc_kernel); outside it, and always under TNB_FLAG_NO_TENSORCORE,
// tthr_gemm_generic_kernel, fp64 FMAs on the CUDA cores.  The bond GEMMs take the tensor cores when their n and k are at
// least 16 (tthr_bond_path).
#pragma once
#include <algorithm>

#include "common.cuh"
#include "round_impl.cuh"
#include "small_kernels.cuh"
#include "sweep.cuh"
#include "tt_dot.cuh"

namespace tnb {

constexpr int TTHR_TC_MIN_R = 16;
constexpr int TTHR_TC_MAX_R = 256;
constexpr int TTHR_MAX_RANK = 4096;             // of either operand
constexpr int64_t TTHR_MAX_R = 65536;           // of the product: GL_k is R_k^2 doubles
constexpr int TTHR_MAX_KEEP = 256;              // no eigen stage keeps more (Jacobi: L <= 256; ChFSI: <= 240)
constexpr int64_t TTHR_CHUNK_DOUBLES = (int64_t)1 << 26;  // per chunk: the T1 / T3 and T2 buffers together (512 MB)

enum TthrPath {
  TTHR_PATH_TC = 0,
  TTHR_PATH_RANK_MIN = 1,  // a rank below TTHR_TC_MIN_R (always the first and last modes)
  TTHR_PATH_RANK_MAX = 2,  // a rank above TTHR_TC_MAX_R
  TTHR_PATH_FORCED = 3,    // TNB_FLAG_NO_TENSORCORE
};

// The path of the left-Gram recurrence at a mode of ranks (ra, rb) -> (ra', rb').  The one place the envelope is defined.
inline int tthr_mode_path(int64_t ra, int64_t rb, int64_t rao, int64_t rbo, bool allow_tc) {
  if (!allow_tc) return TTHR_PATH_FORCED;
  const int64_t lo = std::min(std::min(ra, rb), std::min(rao, rbo)), hi = std::max(std::max(ra, rb), std::max(rao, rbo));
  if (hi > TTHR_TC_MAX_R) return TTHR_PATH_RANK_MAX;
  if (lo < TTHR_TC_MIN_R) return TTHR_PATH_RANK_MIN;
  return TTHR_PATH_TC;
}

// The path of a bond GEMM (Y, GL Y, H, W) of n columns and inner dimension k.
inline int tthr_bond_path(int64_t n, int64_t k, bool allow_tc) {
  if (!allow_tc) return TTHR_PATH_FORCED;
  return std::min(n, k) < TTHR_TC_MIN_R ? TTHR_PATH_RANK_MIN : TTHR_PATH_TC;
}

// The per-i intermediates of one mode (doubles): T1 / T3 share a buffer, T2 has its own.
inline int64_t tthr_t13(int64_t ra, int64_t rb, int64_t rao, int64_t rbo) {
  return std::max(rb * ra * rb * rao, rb * rao * rbo * rao);
}
inline int64_t tthr_t2(int64_t ra, int64_t rb, int64_t rao, int64_t rbo) { return ra * rb * rao * rbo; }

// Mode values per launch: as many as keep both buffers within TTHR_CHUNK_DOUBLES, at least 1, at most n and 65535.
inline int64_t tthr_chunk(int64_t n, int64_t ra, int64_t rb, int64_t rao, int64_t rbo) {
  const int64_t per = tthr_t13(ra, rb, rao, rbo) + tthr_t2(ra, rb, rao, rbo);
  int64_t c = TTHR_CHUNK_DOUBLES / std::max<int64_t>(per, 1);
  c = std::max<int64_t>(1, std::min<int64_t>(c, std::min<int64_t>(n, 65535)));
  return c;
}

// ---------------------------------------------------------------------------------------------
// The GEMM: out(m, n) = beta * out(m, n) + sum_{z} sum_k X(k, m) Y(k, n), with every operand addressed through strides
// (m splits into (m / M2, m % M2) with one stride each, so a permuted output needs no copy).  zsum: the Z batches are
// summed into one output, in z order; else batch z writes its own output (blockIdx.z).
// ---------------------------------------------------------------------------------------------
struct TthrGemm {
  const void* X;
  int64_t xk, xm1, xm2, xz;
  const void* Y;
  int64_t yk, yn, yz;
  void* O;
  int64_t om1, om2, on, oz;
  int64_t M, M2;
  int N, K, Z;
  int zsum, beta;
};

template <typename TX>
__device__ __forceinline__ double tthr_x(const TthrGemm& g, int64_t k, int64_t m, int64_t z) {
  const int64_t m1 = g.M2 == g.M ? 0 : m / g.M2, m2 = m - m1 * g.M2;
  return (double)static_cast<const TX*>(g.X)[k * g.xk + m1 * g.xm1 + m2 * g.xm2 + z * g.xz];
}
template <typename TY>
__device__ __forceinline__ double tthr_y(const TthrGemm& g, int64_t k, int64_t n, int64_t z) {
  return (double)static_cast<const TY*>(g.Y)[k * g.yk + n * g.yn + z * g.yz];
}
template <typename TO>
__device__ __forceinline__ void tthr_store(const TthrGemm& g, int64_t m, int64_t n, int64_t z, double v) {
  const int64_t m1 = g.M2 == g.M ? 0 : m / g.M2, m2 = m - m1 * g.M2;
  TO* p = static_cast<TO*>(g.O) + m1 * g.om1 + m2 * g.om2 + n * g.on + z * g.oz;
  if (g.beta) v += (double)*p;
  *p = (TO)v;
}

constexpr int TTHR_BM = 64, TTHR_BN = 64, TTHR_KC = 32;
constexpr int TTHR_S = TTHR_BM + 4;  // 4 mod 16 doubles: the 16 lanes of a half-warp fragment load hit distinct banks
constexpr int TTHR_TC_THREADS = 128;
constexpr int TTHR_GEN_THREADS = 256;

// Tensor cores: 4 warps as 2 x 2, each a 32 x 32 tile (2 m16 by 4 n8); KC = 32 rows of X and Y staged per barrier.
template <typename TX, typename TY, typename TO>
__global__ void __launch_bounds__(TTHR_TC_THREADS) tthr_gemm_tc_kernel(const TthrGemm g) {
  __shared__ double Xs[TTHR_KC * TTHR_S];
  __shared__ double Ys[TTHR_KC * TTHR_S];
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, gq = lane >> 2, t = lane & 3;
  const int wm = w & 1, wn = w >> 1;
  const int64_t m0 = (int64_t)blockIdx.x * TTHR_BM;
  const int n0 = blockIdx.y * TTHR_BN;
  double acc[2][4][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[h][j][e] = 0.0;
  const int z0 = g.zsum ? 0 : blockIdx.z, z1 = g.zsum ? g.Z : blockIdx.z + 1;
  for (int z = z0; z < z1; ++z) {
    for (int k0 = 0; k0 < g.K; k0 += TTHR_KC) {
      const int kc = min(TTHR_KC, (g.K - k0 + 15) / 16 * 16);
      for (int e = tid; e < kc * TTHR_BM; e += TTHR_TC_THREADS) {
        const int kk = e / TTHR_BM, mm = e % TTHR_BM;
        const int64_t k = k0 + kk, m = m0 + mm;
        Xs[kk * TTHR_S + mm] = (k < g.K && m < g.M) ? tthr_x<TX>(g, k, m, z) : 0.0;
      }
      for (int e = tid; e < kc * TTHR_BN; e += TTHR_TC_THREADS) {
        const int kk = e / TTHR_BN, nn = e % TTHR_BN;
        const int k = k0 + kk, n = n0 + nn;
        Ys[kk * TTHR_S + nn] = (k < g.K && n < g.N) ? tthr_y<TY>(g, k, n, z) : 0.0;
      }
      __syncthreads();
      for (int ks = 0; ks < kc; ks += 16) {
        double a[2][8];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int i = 0; i < 8; ++i)
            a[h][i] = Xs[(ks + t + 4 * (i >> 1)) * TTHR_S + 32 * wm + 16 * h + gq + 8 * (i & 1)];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          double b[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) b[i] = Ys[(ks + t + 4 * i) * TTHR_S + 32 * wn + 8 * j + gq];
#pragma unroll
          for (int h = 0; h < 2; ++h) dmma_16816(acc[h][j], a[h], b);
        }
      }
      __syncthreads();
    }
    if (!g.zsum) break;
  }
  const int zo = g.zsum ? 0 : blockIdx.z;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int64_t m = m0 + 32 * wm + 16 * h + gq + 8 * (e >> 1);
        const int n = n0 + 32 * wn + 8 * j + 2 * t + (e & 1);
        if (m < g.M && n < g.N) tthr_store<TO>(g, m, n, zo, acc[h][j][e]);
      }
}

// CUDA cores: 256 threads, a 64 x 64 tile, 4 x 4 outputs a thread (rows ty + 16 i, columns tx + 16 j).
template <typename TX, typename TY, typename TO>
__global__ void __launch_bounds__(TTHR_GEN_THREADS) tthr_gemm_generic_kernel(const TthrGemm g) {
  __shared__ double Xs[TTHR_KC][TTHR_BM + 1];
  __shared__ double Ys[TTHR_KC][TTHR_BN + 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.x * TTHR_BM;
  const int n0 = blockIdx.y * TTHR_BN;
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
  const int z0 = g.zsum ? 0 : blockIdx.z, z1 = g.zsum ? g.Z : blockIdx.z + 1;
  for (int z = z0; z < z1; ++z) {
    for (int k0 = 0; k0 < g.K; k0 += TTHR_KC) {
      const int kc = min(TTHR_KC, g.K - k0);
      for (int e = tid; e < kc * TTHR_BM; e += TTHR_GEN_THREADS) {
        const int kk = e / TTHR_BM, mm = e % TTHR_BM;
        const int64_t m = m0 + mm;
        Xs[kk][mm] = m < g.M ? tthr_x<TX>(g, k0 + kk, m, z) : 0.0;
      }
      for (int e = tid; e < kc * TTHR_BN; e += TTHR_GEN_THREADS) {
        const int kk = e / TTHR_BN, nn = e % TTHR_BN;
        const int n = n0 + nn;
        Ys[kk][nn] = n < g.N ? tthr_y<TY>(g, k0 + kk, n, z) : 0.0;
      }
      __syncthreads();
      for (int kk = 0; kk < kc; ++kk) {
        double a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = Xs[kk][ty + 16 * i], b[i] = Ys[kk][tx + 16 * i];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  const int zo = g.zsum ? 0 : blockIdx.z;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t m = m0 + ty + 16 * i;
      const int n = n0 + tx + 16 * j;
      if (m < g.M && n < g.N) tthr_store<TO>(g, m, n, zo, acc[i][j]);
    }
}

template <typename TX, typename TY, typename TO>
inline int tthr_gemm(bool tc, const TthrGemm& g, cudaStream_t st) {
  if (g.M < 1 || g.N < 1 || g.K < 1 || g.Z < 1) return TNB_OK;
  const dim3 grid((unsigned)ceil_div<int64_t>(g.M, TTHR_BM), (unsigned)ceil_div<int64_t>(g.N, TTHR_BN),
                  g.zsum ? 1u : (unsigned)g.Z);
  if (tc)
    tthr_gemm_tc_kernel<TX, TY, TO><<<grid, TTHR_TC_THREADS, 0, st>>>(g);
  else
    tthr_gemm_generic_kernel<TX, TY, TO><<<grid, TTHR_GEN_THREADS, 0, st>>>(g);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// A contiguous operand of one stride for m (M2 = M).
inline TthrGemm tthr_op(int64_t M, int N, int K) {
  TthrGemm g;
  std::memset(&g, 0, sizeof(g));
  g.M = M, g.M2 = M, g.N = N, g.K = K, g.Z = 1;
  return g;
}

// H <- (H + H^T) / 2: GL_k and H are symmetric in exact arithmetic, not bit for bit.
__global__ void tthr_symmetrize_kernel(double* H, int64_t n) {
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n * n; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = idx / n, j = idx % n;
    if (j <= i) continue;
    const double v = 0.5 * (H[i * n + j] + H[j * n + i]);
    H[i * n + j] = v;
    H[j * n + i] = v;
  }
}

// Discarded energy of a bond: trace - sum of the kept eigenvalues (the whole trace for a zero carry), added in bond order.
__global__ void tthr_energy_kernel(const double* __restrict__ w, int rank, int zero, const SweepScalars* sc, double* acc) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double head = 0.0;
  if (!zero)
    for (int j = 0; j < rank; ++j) head += w[j] > 0.0 ? w[j] : 0.0;
  const double d = sc->trace - head;
  acc[0] += d > 0.0 ? d : 0.0;
}

// ||C||^2 of a one-mode product (its only core) into sc->norm2.
template <typename T>
__global__ void tthr_sumsq_kernel(const T* __restrict__ c, int64_t n, SweepScalars* sc) {
  __shared__ double red[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += (double)c[i] * (double)c[i];
  s = block_reduce_sum(s, red);
  if (threadIdx.x == 0) sc->norm2 = s;
}

// ---------------------------------------------------------------------------------------------
// Dimensions and the output layout
// ---------------------------------------------------------------------------------------------
struct HrDims {
  int N = 0;
  std::vector<int64_t> shape, ra, rb, R;  // R = ra rb
  std::vector<int64_t> rorth;             // rank bound of the orthogonalised left unfoldings (make_round_dims' ra)
  std::vector<int64_t> rcap;              // rank caps after truncation (also at most TTHR_MAX_KEEP)
  std::vector<int64_t> slot;              // element offset of output core k, [rcap_k, I_k, rcap_{k+1}]
  std::vector<int64_t> chunk;             // mode values per launch of the left-Gram recurrence, per mode
  int64_t capacity = 0;
};

inline int make_hr_dims(int ndim, const int64_t* shape, const int32_t* ranks_a, const int32_t* ranks_b, const int32_t* rmax,
                        HrDims& d) {
  if (ndim < 1 || ndim > 62) return fail(TNB_ERR_INVALID, "tt_hadamard_round: ndim=%d out of range", ndim);
  if (!shape || !ranks_a || !ranks_b) return fail(TNB_ERR_INVALID, "tt_hadamard_round: null argument");
  const int N = ndim;
  d.N = N;
  d.shape.assign(shape, shape + N);
  d.ra.resize(N + 1), d.rb.resize(N + 1), d.R.resize(N + 1);
  for (int k = 0; k < N; ++k)
    if (shape[k] < 1) return fail(TNB_ERR_INVALID, "tt_hadamard_round: mode sizes must be >= 1");
  for (int k = 0; k <= N; ++k) {
    d.ra[k] = ranks_a[k], d.rb[k] = ranks_b[k];
    if (d.ra[k] < 1 || d.rb[k] < 1) return fail(TNB_ERR_INVALID, "tt_hadamard_round: rank[%d] < 1", k);
  }
  if (d.ra[0] != 1 || d.ra[N] != 1 || d.rb[0] != 1 || d.rb[N] != 1)
    return fail(TNB_ERR_INVALID, "tt_hadamard_round: boundary TT ranks must be 1");
  for (int k = 0; k <= N; ++k) {
    if (d.ra[k] > TTHR_MAX_RANK || d.rb[k] > TTHR_MAX_RANK)
      return fail(TNB_ERR_UNSUPPORTED, "tt_hadamard_round: rank %lld above %d", (long long)std::max(d.ra[k], d.rb[k]),
                  TTHR_MAX_RANK);
    d.R[k] = d.ra[k] * d.rb[k];
    if (d.R[k] > TTHR_MAX_R)
      return fail(TNB_ERR_UNSUPPORTED, "tt_hadamard_round: product rank %lld at bond %d above %lld", (long long)d.R[k], k,
                  (long long)TTHR_MAX_R);
  }
  d.rorth.assign(N + 1, 1);
  for (int k = 0; k < N - 1; ++k) d.rorth[k + 1] = std::min<int64_t>(d.rorth[k] * shape[k], d.R[k + 1]);
  d.rcap.assign(N + 1, 1);
  for (int mu = N - 1; mu >= 1; --mu) {
    int64_t c = std::min<int64_t>(d.rorth[mu], shape[mu] * d.rcap[mu + 1]);
    if (rmax && rmax[mu - 1] > 0 && rmax[mu - 1] < c) c = rmax[mu - 1];
    d.rcap[mu] = std::min<int64_t>(c, TTHR_MAX_KEEP);
  }
  d.slot.assign(N, 0);
  int64_t off = 0;
  for (int k = 0; k < N; ++k) {
    d.slot[k] = off;
    off += d.rcap[k] * shape[k] * d.rcap[k + 1];
    off = (off + 63) / 64 * 64;
  }
  d.capacity = off;
  d.chunk.assign(N, 1);
  for (int k = 0; k < N; ++k) d.chunk[k] = tthr_chunk(shape[k], d.ra[k], d.rb[k], d.ra[k + 1], d.rb[k + 1]);
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// The driver.  Workspace: the step scalars and the energy accumulator, GL_0 .. GL_{N-1}; then, overlapping, the
// recurrence's two chunk buffers, or the truncation's carries W (two), Z, Y, GL Y, H, the eigen stage and V_r.
// ---------------------------------------------------------------------------------------------
template <typename T, class ArenaT>
inline int tt_hadamard_round_impl(ArenaT& ar, bool dry, const T* const* ca, const T* const* cb, const HrDims& d,
                                  const int32_t* rmax, double eps, uint32_t flags, T* cores_out, int32_t* ranks_host,
                                  double* energies_host, cudaStream_t st) {
  const int N = d.N;
  const bool allow_tc = tc_allowed(flags, dry);
  StepCtx cx = make_step_ctx(ar, dry, N, eps, flags | TNB_FLAG_NO_TENSORCORE, nullptr, st, false);
  double* acc = ar.template take<double>(1);
  std::vector<double*> GL(N, nullptr);
  for (int k = 0; k < N; ++k) GL[k] = ar.template take<double>((size_t)d.R[k] * d.R[k]);
  const size_t base = ar.off;
  size_t peak = ar.off;

  // ---- sizing of the recurrence's chunk buffers
  int64_t t13 = 1, t2 = 1;
  for (int k = 0; k + 1 < N; ++k) {
    t13 = std::max(t13, d.chunk[k] * tthr_t13(d.ra[k], d.rb[k], d.ra[k + 1], d.rb[k + 1]));
    t2 = std::max(t2, d.chunk[k] * tthr_t2(d.ra[k], d.rb[k], d.ra[k + 1], d.rb[k + 1]));
  }
  double* T13 = N > 1 ? ar.template take<double>((size_t)t13) : nullptr;
  double* T2b = N > 1 ? ar.template take<double>((size_t)t2) : nullptr;
  peak = std::max(peak, ar.off);
  if (!dry) {
    if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_hadamard_round: workspace too small (need > %zu bytes)", ar.off);
    cx.h_sc = static_cast<int*>(pinned_scratch(sizeof(SweepScalars) + 2 * sizeof(double)));
    if (!cx.h_sc) return fail(TNB_ERR_CUDA, "pinned scratch allocation failed");
    ranks_host[0] = 1;
    ranks_host[N] = 1;
    TNB_CUDA(cudaMemsetAsync(acc, 0, sizeof(double), st));
    TNB_CUDA(cudaMemsetAsync(cx.sc, 0, sizeof(SweepScalars), st));
    fill_kernel<double><<<1, 32, 0, st>>>(GL[0], 1, 1.0);
    TNB_LAUNCH_CHECK();
    // ---------------- left Grams: GL_{k+1} = sum_i C_i^T GL_k C_i ----------------
    for (int k = 0; k + 1 < N; ++k) {
      const int64_t ra = d.ra[k], rb = d.rb[k], rao = d.ra[k + 1], rbo = d.rb[k + 1], I = d.shape[k], R = d.R[k];
      const bool tc = tthr_mode_path(ra, rb, rao, rbo, allow_tc) == TTHR_PATH_TC;
      const T* A = ca[k];
      const T* B = cb[k];
      const int64_t s1 = rb * R * rao, s2 = ra * rb * rao * rbo, s3 = rb * rao * rbo * rao;
      for (int64_t i0 = 0; i0 < I; i0 += d.chunk[k]) {
        const int Z = (int)std::min<int64_t>(d.chunk[k], I - i0);
        // T1[z][b c d][a'] = sum_a GL[a][b c d] A[a, i, a']
        TthrGemm g = tthr_op(rb * R, (int)rao, (int)ra);
        g.X = GL[k], g.xk = rb * R, g.xm2 = 1, g.xz = 0;
        g.Y = A + i0 * rao, g.yk = I * rao, g.yn = 1, g.yz = rao;
        g.O = T13, g.om2 = rao, g.on = 1, g.oz = s1, g.Z = Z;
        TNB_TRY((tthr_gemm<double, T, double>(tc, g, st)));
        // T2[z][c d a'][b'] = sum_b T1[z][b][c d a'] B[b, i, b']
        g = tthr_op(ra * rb * rao, (int)rbo, (int)rb);
        g.X = T13, g.xk = ra * rb * rao, g.xm2 = 1, g.xz = s1;
        g.Y = B + i0 * rbo, g.yk = I * rbo, g.yn = 1, g.yz = rbo;
        g.O = T2b, g.om2 = rbo, g.on = 1, g.oz = s2, g.Z = Z;
        TNB_TRY((tthr_gemm<double, T, double>(tc, g, st)));
        // T3[z][d a' b'][c'] = sum_c T2[z][c][d a' b'] A[c, i, c']
        g = tthr_op(rb * rao * rbo, (int)rao, (int)ra);
        g.X = T2b, g.xk = rb * rao * rbo, g.xm2 = 1, g.xz = s2;
        g.Y = A + i0 * rao, g.yk = I * rao, g.yn = 1, g.yz = rao;
        g.O = T13, g.om2 = rao, g.on = 1, g.oz = s3, g.Z = Z;
        TNB_TRY((tthr_gemm<double, T, double>(tc, g, st)));
        // GL'[a' b' c'][d'] (+)= sum_z sum_d T3[z][d][a' b' c'] B[d, i, d']
        g = tthr_op(rao * rbo * rao, (int)rbo, (int)rb);
        g.X = T13, g.xk = rao * rbo * rao, g.xm2 = 1, g.xz = s3;
        g.Y = B + i0 * rbo, g.yk = I * rbo, g.yn = 1, g.yz = rbo;
        g.O = GL[k + 1], g.om2 = rbo, g.on = 1, g.Z = Z, g.zsum = 1, g.beta = i0 > 0;
        TNB_TRY((tthr_gemm<double, T, double>(tc, g, st)));
      }
    }
  }
  ar.off = base;

  // ---------------- truncation from the right ----------------
  int64_t wmax = 1;
  for (int mu = 1; mu <= N; ++mu) wmax = std::max(wmax, d.R[mu] * d.rcap[mu]);
  double* W[2] = {ar.template take<double>((size_t)wmax), ar.template take<double>((size_t)wmax)};
  if (!dry) {
    if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_hadamard_round: workspace too small (need > %zu bytes)", ar.off);
    fill_kernel<double><<<1, 32, 0, st>>>(W[0], 1, 1.0);  // W_N = [1]
    TNB_LAUNCH_CHECK();
  }
  const SweepScalars* hs = reinterpret_cast<const SweepScalars*>(cx.h_sc);
  int64_t r_next = 1;
  int cur = 0;
  for (int mu = N - 1; mu >= 0; --mu) {
    const size_t mark = ar.off;
    const int64_t I = d.shape[mu], ra = d.ra[mu], rb = d.rb[mu], rao = d.ra[mu + 1], rbo = d.rb[mu + 1], R = d.R[mu];
    const int64_t rn = dry ? d.rcap[mu + 1] : r_next;
    const int64_t n = I * rn;
    const int64_t kcap = std::min<int64_t>(d.rcap[mu], n);
    const bool have_rmax = mu >= 1 && rmax && rmax[mu - 1] > 0;
    double* Zb = ar.template take<double>((size_t)(I * rao * rn * rb + (N == 1 ? I : 0)));
    double* Yb = mu >= 1 ? ar.template take<double>((size_t)(R * n)) : nullptr;
    double* G1 = mu >= 1 ? ar.template take<double>((size_t)(R * n)) : nullptr;
    double* H = mu >= 1 ? ar.template take<double>((size_t)(n * n)) : nullptr;
    EigWork<double> ew;
    double* fac = nullptr;
    if (mu >= 1) {
      TNB_TRY(eig_carve<double>(ar, n, kcap, have_rmax, ew));
      fac = ar.template take<double>((size_t)(n * kcap));
    }
    peak = std::max(peak, ar.off);
    if (dry) {
      ar.off = mark;
      continue;
    }
    if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_hadamard_round: workspace too small (need > %zu bytes)", ar.off);
    // Z[i][a'][j][b] = sum_b' W[a'][b'][j] B[b, i, b']
    const bool tz = tthr_bond_path(rb, rbo, allow_tc) == TTHR_PATH_TC;
    TthrGemm g = tthr_op(rao * rn, (int)rb, (int)rbo);
    g.M2 = rn;
    g.X = W[cur], g.xk = rn, g.xm1 = rbo * rn, g.xm2 = 1, g.xz = 0;
    g.Y = cb[mu], g.yk = 1, g.yn = I * rbo, g.yz = rbo;
    g.O = Zb, g.om1 = rn * rb, g.om2 = rb, g.on = 1, g.oz = rao * rn * rb, g.Z = (int)I;
    TNB_TRY((tthr_gemm<double, T, double>(tz, g, st)));
    // Y[a b][i j] = sum_a' A[a, i, a'] Z[i][a'][j][b]   (core 0 itself when mu = 0)
    const bool ty = tthr_bond_path(ra, rao, allow_tc) == TTHR_PATH_TC;
    g = tthr_op(rn * rb, (int)ra, (int)rao);
    g.M2 = rb;
    g.X = Zb, g.xk = rn * rb, g.xm1 = rb, g.xm2 = 1, g.xz = rao * rn * rb;
    g.Y = ca[mu], g.yk = 1, g.yn = I * rao, g.yz = rao;
    g.om1 = 1, g.om2 = I * rn, g.on = rb * I * rn, g.oz = rn, g.Z = (int)I;
    if (mu == 0) {
      if (N == 1) {  // ||C||^2 of the fp64 product, before the core takes the input dtype
        g.O = Zb + I * rao * rn * rb;
        TNB_TRY((tthr_gemm<double, T, double>(ty, g, st)));
        tthr_sumsq_kernel<double><<<1, 256, 0, st>>>(Zb + I * rao * rn * rb, I, cx.sc);
        TNB_LAUNCH_CHECK();
        convert_kernel<double, T><<<grid_for(I), 256, 0, st>>>(Zb + I * rao * rn * rb, cores_out + d.slot[0], I);
        TNB_LAUNCH_CHECK();
        break;
      }
      g.O = cores_out + d.slot[0];
      TNB_TRY((tthr_gemm<double, T, T>(ty, g, st)));
      break;
    }
    g.O = Yb;
    TNB_TRY((tthr_gemm<double, T, double>(ty, g, st)));
    // G1 = GL_mu Y  (R x n);  H = Y^T G1  (n x n)
    const bool tg = tthr_bond_path(n, R, allow_tc) == TTHR_PATH_TC;
    g = tthr_op(R, (int)n, (int)R);
    g.X = GL[mu], g.xk = R, g.xm2 = 1;
    g.Y = Yb, g.yk = n, g.yn = 1;
    g.O = G1, g.om2 = n, g.on = 1;
    TNB_TRY((tthr_gemm<double, double, double>(tg, g, st)));
    g = tthr_op(n, (int)n, (int)R);
    g.X = Yb, g.xk = n, g.xm2 = 1;
    g.Y = G1, g.yk = n, g.yn = 1;
    g.O = H, g.om2 = n, g.on = 1;
    TNB_TRY((tthr_gemm<double, double, double>(tg, g, st)));
    tthr_symmetrize_kernel<<<grid_for(n * n), 256, 0, st>>>(H, n);
    TNB_LAUNCH_CHECK();
    trace_kernel<<<1, 256, 0, st>>>(H, (int)n, (int)n, cx.sc, mu == N - 1 ? 1 : 0, cx.eps_scaled2);
    TNB_LAUNCH_CHECK();
    // the eigen stage and rank rule of truncate_step (one synchronisation; an eps-only ChFSI solve may take more)
    TNB_TRY(eig_solve_and_rank<double>(H, nullptr, n, ew, cx.sc, cx.h_sc, have_rmax ? rmax[mu - 1] : 0, 0, nullptr,
                                       nullptr, st, false, false));
    const bool zero = hs->zero_flag != 0;
    const int64_t rank = zero ? 1 : std::min<int64_t>(hs->rank, kcap);
    ranks_host[mu] = (int32_t)rank;
    tthr_energy_kernel<<<1, 32, 0, st>>>(ew.w, (int)rank, zero ? 1 : 0, cx.sc, acc);
    TNB_LAUNCH_CHECK();
    T* core = cores_out + d.slot[mu];
    double* Wn = W[cur ^ 1];
    if (zero) {
      fill_kernel<T><<<grid_for(n), 256, 0, st>>>(core, n, (T)0);
      TNB_LAUNCH_CHECK();
      fill_kernel<double><<<grid_for(R), 256, 0, st>>>(Wn, R, 0.0);
      TNB_LAUNCH_CHECK();
    } else {
      // core mu = V_r^T (rank x n);  W_mu = Y V_r  (R x rank)
      scale_extract_kernel<T><<<grid_for(n * rank), 256, 0, st>>>(ew.V, ew.ldv, (int)n, (int)rank, ew.w, core, 0, 1);
      TNB_LAUNCH_CHECK();
      scale_extract_kernel<double><<<grid_for(n * rank), 256, 0, st>>>(ew.V, ew.ldv, (int)n, (int)rank, ew.w, fac, 0, 0);
      TNB_LAUNCH_CHECK();
      g = tthr_op(R, (int)rank, (int)n);
      g.X = Yb, g.xk = 1, g.xm2 = n;
      g.Y = fac, g.yk = rank, g.yn = 1;
      g.O = Wn, g.om2 = rank, g.on = 1;
      TNB_TRY((tthr_gemm<double, double, double>(tthr_bond_path(rank, n, allow_tc) == TTHR_PATH_TC, g, st)));
    }
    cur ^= 1;
    r_next = rank;
    ar.off = mark;
  }
  if (dry) {
    ar.off = peak;
    return TNB_OK;
  }
  double* he = reinterpret_cast<double*>(reinterpret_cast<char*>(cx.h_sc) + sizeof(SweepScalars));
  TNB_CUDA(cudaMemcpyAsync(cx.h_sc, cx.sc, sizeof(SweepScalars), cudaMemcpyDeviceToHost, st));
  TNB_CUDA(cudaMemcpyAsync(he, acc, sizeof(double), cudaMemcpyDeviceToHost, st));
  TNB_CUDA(cudaStreamSynchronize(st));
  if (energies_host) {
    energies_host[0] = hs->norm2;
    energies_host[1] = he[0];
  }
  return TNB_OK;
}

}  // namespace tnb
