// CP-ALS on the device: tn.Tensor(X, ranks_cp=R, max_iter, tol)  (tensor.py:210-400).
//
//   init (tensor.py:217-277): per mode n, G_n = X_(n) X_(n)^T, top-R eigenvectors -> factor A_n (I_n x R)
//   sweep (tensor.py:323-361): for n = 0..N-1:  M_n = MTTKRP_n(X; A_m, m != n),  P = hadamard_{m != n}(A_m^T A_m),
//                              A_n = M_n P^+,  gram_n = A_n^T A_n
//   error (tensor.py:373-381): ||X - [[A]]|| / ||X||, here from ||X||^2 - 2<X,[[A]]> + ||[[A]]||^2 with
//                              <X,[[A]]> = sum(M_{N-1} .* A_{N-1}) and ||[[A]]||^2 = sum(hadamard_n gram_n),
//                              i.e. without the reference's extra full reconstruction pass.
//
// MTTKRP never materialises the Khatri-Rao product nor a permuted copy of X (the reference does both,
// tensor.py:351-357, tools.py:226-228): the last (or, for n = N-1, the first) mode is contracted by one GEMM
// over X with R output columns, the remaining modes by cheap "Khatri-Rao reductions" on the (rest x R) result.
#pragma once
#include "sweep.cuh"

namespace tnb {

// out[l, q, r] = sum_i Y[l, i, q, r] * A[i, r]     (Y: L x I x Q x R row-major, A: I x R)
template <typename T>
__global__ void khatri_reduce_kernel(const T* __restrict__ Y, const T* __restrict__ A, T* __restrict__ out, int64_t L,
                                     int I, int64_t Q, int R) {
  const int64_t total = L * Q * R;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(idx % R);
    const int64_t q = (idx / R) % Q, l = idx / (R * Q);
    const T* y = Y + ((l * I) * Q + q) * R + r;
    const T* a = A + r;
    const int64_t stride = Q * R;
    double acc = 0.0;
    int i = 0;
    if (sizeof(T) == 4) {
      // fp32 data: eight products per fp32 partial (eight independent loads in flight), partials summed in fp64 — one
      // fp64 addition per eight products instead of one fp64 FMA per product
      for (; i + 8 <= I; i += 8) {
        float part = 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) part = fmaf((float)y[(int64_t)(i + u) * stride], (float)a[(size_t)(i + u) * R], part);
        acc += (double)part;
      }
    }
    for (; i < I; ++i) acc += (double)y[(int64_t)i * stride] * (double)a[(size_t)i * R];
    out[idx] = (T)acc;
  }
}

// The same reduction for fp32 data with an even R: two adjacent r per thread (8-byte loads), eight rows in flight.  The
// scalar kernel keeps only 1280 threads x 8 x 4 B = 40 KB in flight per SM, too little to cover HBM latency.
__global__ void __launch_bounds__(256) khatri_reduce2_kernel(const float* __restrict__ Y, const float* __restrict__ A,
                                                             float* __restrict__ out, int64_t L, int I, int64_t Q, int R) {
  const int R2 = R >> 1;
  const int64_t total = L * Q * R2;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int rv = (int)(idx % R2);
    const int64_t q = (idx / R2) % Q, l = idx / ((int64_t)R2 * Q);
    const float2* y = reinterpret_cast<const float2*>(Y + ((l * I) * Q + q) * R) + rv;
    const float2* a = reinterpret_cast<const float2*>(A) + rv;
    const int64_t stride = Q * R2;  // in float2
    double acc0 = 0.0, acc1 = 0.0;
    int i = 0;
    for (; i + 8 <= I; i += 8) {
      float2 yv[8], av[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) yv[u] = __ldcs(y + (int64_t)(i + u) * stride);  // streamed once
#pragma unroll
      for (int u = 0; u < 8; ++u) av[u] = __ldg(a + (size_t)(i + u) * R2);
      float p0 = 0.f, p1 = 0.f;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        p0 = fmaf(yv[u].x, av[u].x, p0);
        p1 = fmaf(yv[u].y, av[u].y, p1);
      }
      acc0 += (double)p0;
      acc1 += (double)p1;
    }
    for (; i < I; ++i) {
      const float2 yv = y[(int64_t)i * stride], av = a[(size_t)i * R2];
      acc0 += (double)yv.x * (double)av.x;
      acc1 += (double)yv.y * (double)av.y;
    }
    reinterpret_cast<float2*>(out)[idx] = make_float2((float)acc0, (float)acc1);
  }
}

// Few outputs (the inner steps of a chain: L*Q*R/2 of a few thousand): eight lanes share one output pair, each summing
// every eighth row, so that the I rows are not walked by one thread alone (80 us -> latency of I/8 rows).
__global__ void __launch_bounds__(256) khatri_reduce2_split_kernel(const float* __restrict__ Y, const float* __restrict__ A,
                                                                   float* __restrict__ out, int64_t L, int I, int64_t Q,
                                                                   int R) {
  const int R2 = R >> 1;
  const int64_t total = L * Q * R2;
  const int g = threadIdx.x & 7;
  const int64_t idx = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 3;
  double acc0 = 0.0, acc1 = 0.0;
  if (idx < total) {
    const int rv = (int)(idx % R2);
    const int64_t q = (idx / R2) % Q, l = idx / ((int64_t)R2 * Q);
    const float2* y = reinterpret_cast<const float2*>(Y + ((l * I) * Q + q) * R) + rv;
    const float2* a = reinterpret_cast<const float2*>(A) + rv;
    const int64_t stride = Q * R2;
#pragma unroll 4
    for (int i = g; i < I; i += 8) {
      const float2 yv = y[(int64_t)i * stride], av = __ldg(a + (size_t)i * R2);
      acc0 += (double)yv.x * (double)av.x;
      acc1 += (double)yv.y * (double)av.y;
    }
  }
  for (int o = 4; o > 0; o >>= 1) {  // the eight lanes of a group are adjacent lanes of one warp
    acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
    acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
  }
  if (g == 0 && idx < total) reinterpret_cast<float2*>(out)[idx] = make_float2((float)acc0, (float)acc1);
}

struct GramPtrs {
  const double* g[16];
};
// P[r][s] = prod_{m != skip} gram_m[r][s]  (skip < 0: all modes)
__global__ void hadamard_grams_kernel(GramPtrs gp, int nmodes, int skip, int R, double* __restrict__ P) {
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < R * R; idx += gridDim.x * blockDim.x) {
    double v = 1.0;
    for (int m = 0; m < nmodes; ++m)
      if (m != skip) v *= gp.g[m][idx];
    P[idx] = v;
  }
}
// Pinv = Q diag(1/lam_i if lam_i > rcond*lam_0 else 0) Q^T   (lam descending; minimum-norm solve like lstsq)
__global__ void pinv_from_eig_kernel(const double* __restrict__ Q, const double* __restrict__ lam, int R, double rcond,
                                     double* __restrict__ Pinv) {
  const double thr = rcond * (lam[0] > 0.0 ? lam[0] : 0.0);
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < R * R; idx += gridDim.x * blockDim.x) {
    const int i = idx / R, j = idx % R;
    double s = 0.0;
    for (int k = 0; k < R; ++k) {
      const double l = lam[k];
      if (l > thr && l > 0.0) s += Q[(size_t)i * R + k] * Q[(size_t)j * R + k] / l;
    }
    Pinv[idx] = s;
  }
}
// acc[0] += sum(M .* A) ; acc[1] += sum(P)   (fp64)
template <typename T>
__global__ void cp_error_terms_kernel(const T* __restrict__ M, const T* __restrict__ A, int64_t n, const double* __restrict__ P,
                                      int rr, double* __restrict__ acc) {
  __shared__ double red[32];
  double s = 0.0, t = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    s += (double)M[i] * (double)A[i];
  if (blockIdx.x == 0)
    for (int i = threadIdx.x; i < rr; i += blockDim.x) t += P[i];
  s = block_reduce_sum(s, red);
  t = block_reduce_sum(t, red);
  if (threadIdx.x == 0) {
    atomicAdd(&acc[0], s);
    if (blockIdx.x == 0) atomicAdd(&acc[1], t);
  }
}
// A (I x R) <- first R columns of V (I x ldv, fp64); columns beyond `have` filled pseudo-randomly (tensor.py:258-272)
template <typename T>
__global__ void cp_init_factor_kernel(const double* __restrict__ V, int ldv, int I, int R, int have, T* __restrict__ A,
                                      uint32_t seed) {
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < I * R; idx += gridDim.x * blockDim.x) {
    const int i = idx / R, r = idx % R;
    double v;
    if (r < have) v = V[(size_t)i * ldv + r];
    else {
      const uint32_t h = hash_u32((uint32_t)idx * 2654435761U + seed);
      v = ((double)(h >> 8) + 0.5) * (2.0 / 16777216.0) - 1.0;
    }
    A[idx] = (T)v;
  }
}

struct CpDims {
  int N;
  std::vector<int64_t> shape, left, right;  // left[n] = prod_{m<n} I_m, right[n] = prod_{m>n} I_m
  int64_t numel;
  std::vector<int64_t> foff;  // factor offsets
  int64_t ftotal;
};
inline int make_cp_dims(int ndim, const int64_t* shape, int R, CpDims& d) {
  if (ndim < 2 || ndim > 16) return fail(TNB_ERR_INVALID, "cp_als: ndim=%d must be in [2,16]", ndim);
  if (R < 1 || R > JACOBI_MAX_N) return fail(TNB_ERR_UNSUPPORTED, "cp_als: rank %d outside [1,%d]", R, JACOBI_MAX_N);
  d.N = ndim;
  d.shape.assign(shape, shape + ndim);
  d.left.assign(ndim, 1);
  d.right.assign(ndim, 1);
  d.numel = 1;
  for (int n = 0; n < ndim; ++n) {
    if (shape[n] < 1 || shape[n] > 2147483647LL / (R + 1)) return fail(TNB_ERR_INVALID, "cp_als: bad shape[%d]", n);
    d.left[n] = d.numel;
    d.numel *= shape[n];
  }
  int64_t r = 1;
  for (int n = ndim - 1; n >= 0; --n) {
    d.right[n] = r;
    r *= shape[n];
  }
  d.foff.assign(ndim, 0);
  int64_t off = 0;
  for (int n = 0; n < ndim; ++n) {
    d.foff[n] = off;
    off += (shape[n] * R + 63) / 64 * 64;
  }
  d.ftotal = off;
  return TNB_OK;
}

// MTTKRP for mode n into Mout (I_n x R).  Y0/Y1: ping-pong buffers of numel/min(I_0,I_{N-1}) * R elements.
template <typename T>
inline int cp_mttkrp(const T* X, const CpDims& d, int n, int R, T* const* A, T* Y0, T* Y1, T* Mout, cudaStream_t st,
                     void* tc_ws = nullptr, size_t tc_ws_bytes = 0) {
  const int N = d.N;
  T* cur = Y0;
  T* nxt = Y1;
  int lo, hi;  // modes still alive in `cur`: [lo, hi]
  if (n != N - 1) {
    // contract the last mode:  cur[(i_0..i_{N-2}), r] = sum_i X[.., i] A_{N-1}[i, r]
    const int64_t rows = d.numel / d.shape[N - 1];
    TNB_TRY(project_any<T>(X, rows, d.shape[N - 1], A[N - 1], R, cur, st, tc_ws, tc_ws_bytes));  // 3xTF32 on the tensor cores when it fits
    lo = 0;
    hi = N - 2;
  } else {
    // contract the first mode:  cur[(i_1..i_{N-1}), r] = sum_i X[i, ..] A_0[i, r]
    const int64_t rest = d.numel / d.shape[0];
    TNB_TRY((gemm_direct<T, T, T, T>(rest, R, d.shape[0], X, rest, false, A[0], R, false, cur, R, (T)1, nullptr, 0, (T)0,
                                     nullptr, 0, (T)0, st)));
    lo = 1;
    hi = N - 1;
  }
  // reduce right modes hi..n+1 (fast index side), then left modes lo..n-1
  while (hi > n) {
    int64_t L = 1;
    for (int m = lo; m < hi; ++m) L *= d.shape[m];
    T* dst = (hi - 1 == n && lo == n) ? Mout : nxt;
    khatri_reduce_kernel<T><<<grid_for(L * R, 256, 8192), 256, 0, st>>>(cur, A[hi], dst, L, (int)d.shape[hi], 1, R);
    TNB_LAUNCH_CHECK();
    if (dst != Mout) { T* t = cur; cur = nxt; nxt = t; } else cur = Mout;
    --hi;
  }
  while (lo < n) {
    int64_t Q = 1;
    for (int m = lo + 1; m <= hi; ++m) Q *= d.shape[m];
    T* dst = (lo + 1 == n && hi == n) ? Mout : nxt;
    khatri_reduce_kernel<T><<<grid_for(Q * R, 256, 8192), 256, 0, st>>>(cur, A[lo], dst, 1, (int)d.shape[lo], Q, R);
    TNB_LAUNCH_CHECK();
    if (dst != Mout) { T* t = cur; cur = nxt; nxt = t; } else cur = Mout;
    ++lo;
  }
  if (cur != Mout)  // N == 2: the single GEMM already produced the I_n x R result
    TNB_CUDA(cudaMemcpyAsync(Mout, cur, sizeof(T) * (size_t)d.shape[n] * R, cudaMemcpyDeviceToDevice, st));
  return TNB_OK;
}

// out[c, r] = in[r, c]   (in: rows x cols row-major).  32 x 32 tiles through shared memory, both sides coalesced.
template <typename T>
__global__ void cp_transpose_kernel(const T* __restrict__ in, T* __restrict__ out, int64_t rows, int64_t cols) {
  __shared__ T tile[32][33];
  const int64_t r0 = (int64_t)blockIdx.x * 32;
  for (int64_t c0 = (int64_t)blockIdx.y * 32; c0 < cols; c0 += (int64_t)gridDim.y * 32) {
    for (int j = threadIdx.y; j < 32; j += 8) {
      const int64_t r = r0 + j, c = c0 + threadIdx.x;
      if (r < rows && c < cols) tile[j][threadIdx.x] = in[r * cols + c];
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += 8) {
      const int64_t c = c0 + j, r = r0 + threadIdx.x;
      if (r < rows && c < cols) out[c * rows + r] = tile[threadIdx.x][j];
    }
    __syncthreads();
  }
}

// One ALS sweep's MTTKRPs as a dimension tree (N >= 3).  Within a sweep the factors of modes > n are still the old ones
// when mode n is updated, so
//   * Y = X x_{N-1} A_{N-1} (ONE pass over X) serves modes 0..N-2, and the right-to-left chain
//     R_k = R_{k+1} x_{k+1} A_{k+1} (R_{N-2} = Y, alive modes [0, k]) is built once; M_n = R_n reduced over modes < n
//     with the freshly updated factors;
//   * mode N-1 contracts the last mode of XT (X with mode N-1 moved to the front, transposed once per call) with
//     A_{N-2} through the same projection kernel and reduces modes N-3..0 — instead of a first-mode (strided) GEMM.
// Per sweep X is read twice (not N times); the reference recomputes the full Khatri-Rao product and a permuted copy of
// X for every mode (tensor.py:351-357).
template <typename T>
struct CpTree {
  T* Yk = nullptr;      // max(numel / I_{N-1}, numel / I_{N-2}) * R
  T* T0 = nullptr;      // reduction ping-pong
  T* T1 = nullptr;
  T* XT = nullptr;      // numel
  std::vector<T*> chain;  // chain[k], k = 0..N-3: prod_{m<=k} I_m * R
};

template <typename T>
inline void cp_khatri(const T* Y, const T* A, T* out, int64_t L, int64_t I, int64_t Q, int R, cudaStream_t st) {
  const bool al8 = ((reinterpret_cast<uintptr_t>(Y) | reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(out)) & 7u) == 0;
  if (std::is_same<T, float>::value && (R & 1) == 0 && al8 && L * Q * (R / 2) < (int64_t)usable_sms() * 256) {
    const int64_t threads = L * Q * (R / 2) * 8;
    khatri_reduce2_split_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(
        reinterpret_cast<const float*>(Y), reinterpret_cast<const float*>(A), reinterpret_cast<float*>(out), L, (int)I, Q, R);
    return;
  }
  if (std::is_same<T, float>::value && (R & 1) == 0 && al8) {
    khatri_reduce2_kernel<<<grid_for(L * Q * (R / 2), 256, 16384), 256, 0, st>>>(
        reinterpret_cast<const float*>(Y), reinterpret_cast<const float*>(A), reinterpret_cast<float*>(out), L, (int)I, Q, R);
    return;
  }
  khatri_reduce_kernel<T><<<grid_for(L * Q * R, 256, 8192), 256, 0, st>>>(Y, A, out, L, (int)I, Q, R);
}

template <typename T>
inline int cp_tree_mttkrp(const T* X, const CpDims& d, int n, int R, T* const* A, CpTree<T>& tr, T* Mout, cudaStream_t st,
                          void* tc_ws, size_t tc_ws_bytes) {
  const int N = d.N;
  if (n == 0) {
    TNB_TRY(project_any<T>(X, d.numel / d.shape[N - 1], d.shape[N - 1], A[N - 1], R, tr.Yk, st, tc_ws, tc_ws_bytes));
    const T* src = tr.Yk;
    for (int k = N - 3; k >= 0; --k) {  // R_k = R_{k+1} x_{k+1} A_{k+1}
      cp_khatri<T>(src, A[k + 1], tr.chain[k], d.left[k + 1], d.shape[k + 1], 1, R, st);
      TNB_LAUNCH_CHECK();
      src = tr.chain[k];
    }
    TNB_CUDA(cudaMemcpyAsync(Mout, tr.chain[0], sizeof(T) * (size_t)d.shape[0] * R, cudaMemcpyDeviceToDevice, st));
    return TNB_OK;
  }
  const T* cur;
  T* bufs[2] = {tr.T0, tr.T1};
  int flip = 0;
  if (n <= N - 2) {
    cur = (n == N - 2) ? tr.Yk : tr.chain[n];  // alive modes [0, n]
    for (int lo = 0; lo < n; ++lo) {
      int64_t Q = 1;
      for (int m = lo + 1; m <= n; ++m) Q *= d.shape[m];
      T* dst = (lo + 1 == n) ? Mout : bufs[flip];
      cp_khatri<T>(cur, A[lo], dst, 1, d.shape[lo], Q, R, st);
      TNB_LAUNCH_CHECK();
      cur = dst;
      flip ^= 1;
    }
    return TNB_OK;
  }
  // n == N-1: XT is [I_{N-1}, I_0, ..., I_{N-2}]
  TNB_TRY(project_any<T>(tr.XT, d.numel / d.shape[N - 2], d.shape[N - 2], A[N - 2], R, tr.Yk, st, tc_ws, tc_ws_bytes));
  cur = tr.Yk;
  for (int m = N - 3; m >= 0; --m) {
    T* dst = (m == 0) ? Mout : bufs[flip];
    cp_khatri<T>(cur, A[m], dst, d.shape[N - 1] * d.left[m], d.shape[m], 1, R, st);
    TNB_LAUNCH_CHECK();
    cur = dst;
    flip ^= 1;
  }
  return TNB_OK;
}

// acc[0] += sum x^2 (fp64)
template <typename T>
__global__ void cp_sumsq_kernel(const T* __restrict__ X, int64_t n, double* __restrict__ acc) {
  __shared__ double red[32];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double x = (double)X[i];
    s = fma(x, x, s);
  }
  s = block_reduce_sum(s, red);
  if (threadIdx.x == 0) atomicAdd(acc, s);
}

// init_given: `factors` already holds the starting factors (the reference's random start of CP on a Tucker core,
// tensor.py:278-302) and the HOSVD initialisation is skipped.
template <typename T, class ArenaT>
inline int cp_als_impl(ArenaT& ar, bool dry, const T* X, const CpDims& d, int R, int max_iter, double tol, T* factors,
                       double* errors_host, int32_t* iters_host, cudaStream_t st, bool init_given = false) {
  const int N = d.N;
  int64_t imax = 0;
  for (int n = 0; n < N; ++n) imax = std::max<int64_t>(imax, d.shape[n]);
  const int64_t ymax = d.numel / std::min<int64_t>(d.shape[0], d.shape[N - 1]) * R;
  T* Y0 = ar.template take<T>(N == 2 ? ymax : 64);  // the plain two-GEMM path of N == 2
  T* Y1 = ar.template take<T>(N == 2 ? ymax + 64 : 64);
  T* Mbuf = ar.template take<T>(imax * R);
  T* Anew = ar.template take<T>(imax * R);
  double* grams = ar.template take<double>((size_t)N * R * R);
  double* P = ar.template take<double>((size_t)R * R);
  double* Pinv = ar.template take<double>((size_t)R * R);
  T* PinvT = ar.template take<T>((size_t)R * R);
  double* lam = ar.template take<double>(R);
  double* Q = ar.template take<double>((size_t)R * R);
  double* js = ar.template take<double>(jacobi_scratch_doubles(R));
  int* jinfo = ar.template take<int>(4);
  double* acc = ar.template take<double>(4);
  GemmPlan plg = plan_gemm(R, R, imax, false);
  double* gpart = ar.template take<double>(plg.partial_elems + 64);
  void* ptc_ws = nullptr;
  size_t ptc_bytes = 0;
  const bool tree = N >= 3;  // dimension-tree sweeps (cp_tree_mttkrp); N == 2 keeps the two plain GEMMs
  for (int m = tree ? N - 2 : N - 1; m < N; ++m)
    if (std::is_same<T, float>::value && R <= PT_MAX_N && d.shape[m] % 4 == 0 && d.shape[m] >= 32)
      ptc_bytes = std::max(ptc_bytes, project_tc_workspace_bytes(d.shape[m], R));
  if (ptc_bytes) ptc_ws = ar.template take<char>(ptc_bytes);
  CpTree<T> tr;
  if (tree) {
    int64_t imin = d.shape[0];
    for (int n = 1; n < N; ++n) imin = std::min<int64_t>(imin, d.shape[n]);
    const int64_t yk = d.numel / std::min<int64_t>(d.shape[N - 1], d.shape[N - 2]) * R;
    tr.Yk = ar.template take<T>(yk);
    tr.T0 = ar.template take<T>(yk / imin + 64);
    tr.T1 = ar.template take<T>(yk / imin + 64);
    tr.XT = ar.template take<T>(d.numel);
    tr.chain.resize(N - 2);
    for (int k = 0; k <= N - 3; ++k) tr.chain[k] = ar.template take<T>(d.left[k + 1] * R + 64);
  }
  // HOSVD init scratch: mode Gram (I x I) + eigen workspace, sized for the largest mode
  size_t peak = ar.off;
  for (int n = 0; n < N; ++n) {
    const size_t mark = ar.off;
    const int64_t I = d.shape[n];
    GemmPlan pb = plan_batched(I, I, std::max<int64_t>(d.left[n], 1), true);
    GemmPlan pk = plan_gemm(I, I, d.numel / I, true);
    ar.template take<double>(std::max(pb.partial_elems, pk.partial_elems));
    ar.template take<double>((size_t)I * I);
    EigWork<T> ew;
    TNB_TRY(eig_carve<T>(ar, I, std::min<int64_t>(R, I), true, ew));
    if (ar.off > peak) peak = ar.off;
    ar.off = mark;
  }
  if (dry) {
    ar.off = peak;
    return TNB_OK;
  }
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "cp_als: workspace too small (need %zu bytes)", peak);
  std::vector<T*> A(N);
  for (int n = 0; n < N; ++n) A[n] = factors + d.foff[n];
  double* h = static_cast<double*>(pinned_scratch(4 * sizeof(double)));
  if (!h) return fail(TNB_ERR_CUDA, "pinned scratch allocation failed");

  // ---------------- HOSVD initialisation (tensor.py:217-277) ----------------
  double normX2 = 0.0;
  if (init_given) {
    TNB_CUDA(cudaMemsetAsync(acc, 0, 4 * sizeof(double), st));
    cp_sumsq_kernel<T><<<grid_for(d.numel, 256, 1184), 256, 0, st>>>(X, d.numel, acc);
    TNB_LAUNCH_CHECK();
    TNB_CUDA(cudaMemcpyAsync(h, acc, sizeof(double), cudaMemcpyDeviceToHost, st));
    TNB_CUDA(cudaStreamSynchronize(st));
    normX2 = h[0];
  }
  for (int n = 0; n < N && !init_given; ++n) {
    const size_t mark = ar.off;
    const int64_t I = d.shape[n];
    GemmPlan pb = plan_batched(I, I, std::max<int64_t>(d.left[n], 1), true);
    GemmPlan pk = plan_gemm(I, I, d.numel / I, true);
    double* part = ar.template take<double>(std::max(pb.partial_elems, pk.partial_elems));
    double* G = ar.template take<double>((size_t)I * I);
    EigWork<T> ew;
    TNB_TRY(eig_carve<T>(ar, I, std::min<int64_t>(R, I), true, ew));
    if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "cp_als: workspace too small");
    float* Gf = (ew.chfsi && std::is_same<T, float>::value) ? reinterpret_cast<float*>(ew.Gb) : nullptr;
    if (n == N - 1) {  // X viewed (rest x I): G = C^T C
      TNB_TRY((gemm_splitk<T, T, double, double, float>(pk, I, I, d.numel / I, X, I, false, X, I, false, part, G, I, 1.0,
                                                        nullptr, 0, 0.0, nullptr, 0, 0.0, true, Gf, I, st)));
    } else if (d.left[n] == 1) {  // X viewed (I x rest): G = C C^T, split over the long contraction
      TNB_TRY((gemm_splitk<T, T, double, double, float>(pk, I, I, d.numel / I, X, d.numel / I, true, X, d.numel / I, true,
                                                        part, G, I, 1.0, nullptr, 0, 0.0, nullptr, 0, 0.0, true, Gf, I, st)));
    } else {  // sum over the left index l of A_l A_l^T with A_l = X[l] (I x right), k contiguous
      const int64_t Rt = d.right[n];
      TNB_TRY((gemm_batched_sum<T, T, double, double>(pb, I, I, Rt, d.left[n], X, Rt, true, I * Rt, X, Rt, true, I * Rt,
                                                      part, G, I, true, st)));
      if (Gf) {
        convert_kernel<double, float><<<grid_for(I * I), 256, 0, st>>>(G, Gf, I * I);
        TNB_LAUNCH_CHECK();
      }
    }
    SweepScalars* sc = reinterpret_cast<SweepScalars*>(acc);  // only .trace is used by the subspace solver
    (void)sc;
    double* d_trace = nullptr;
    ChfsiStats cs;
    TNB_TRY(eig_run<T>(G, reinterpret_cast<const T*>(Gf), I, ew, d_trace, &cs, st, false));
    const int have = (int)std::min<int64_t>(R, I);
    cp_init_factor_kernel<T><<<grid_for(I * R), 256, 0, st>>>(ew.V, ew.ldv, (int)I, R, have, A[n], 0x5151u + n);
    TNB_LAUNCH_CHECK();
    if (n == 0) {  // ||X||^2 = trace of any mode Gram
      TNB_CUDA(cudaMemsetAsync(acc, 0, 4 * sizeof(double), st));
      trace_kernel<<<1, 256, 0, st>>>(G, (int)I, (int)I, reinterpret_cast<SweepScalars*>(js), 0, 0.0);
      TNB_LAUNCH_CHECK();
      TNB_CUDA(cudaMemcpyAsync(h, &reinterpret_cast<SweepScalars*>(js)->trace, sizeof(double), cudaMemcpyDeviceToHost, st));
      TNB_CUDA(cudaStreamSynchronize(st));
      normX2 = h[0];
    }
    ar.off = mark;
  }
  // grams[n] = A_n^T A_n for n >= 1 (tensor.py:307-310; gram_0 is produced by the first update)
  GramPtrs gp;
  for (int n = 0; n < 16; ++n) gp.g[n] = grams + (size_t)std::min(n, N - 1) * R * R;
  for (int n = 1; n < N; ++n) {
    GemmPlan pl = plan_gemm(R, R, d.shape[n], false);
    TNB_TRY((gemm_splitk<T, T, double, double, double>(pl, R, R, d.shape[n], A[n], R, false, A[n], R, false, gpart,
                                                       grams + (size_t)n * R * R, R, 1.0, nullptr, 0, 0.0, nullptr, 0, 0.0,
                                                       false, (double*)nullptr, 0, st)));
  }

  // ---------------- ALS sweeps (tensor.py:323-400) ----------------
  if (tree) {  // XT[i_{N-1}, rest] = X[rest, i_{N-1}], once per call
    const int64_t rows = d.numel / d.shape[N - 1], cols = d.shape[N - 1];
    dim3 grid((unsigned)((rows + 31) / 32), (unsigned)std::min<int64_t>((cols + 31) / 32, 65535));
    cp_transpose_kernel<T><<<grid, dim3(32, 8), 0, st>>>(X, tr.XT, rows, cols);
    TNB_LAUNCH_CHECK();
  }
  int it = 0;
  double prev_err = 0.0;
  for (; it < max_iter; ++it) {
    for (int n = 0; n < N; ++n) {
      if (tree)
        TNB_TRY(cp_tree_mttkrp<T>(X, d, n, R, A.data(), tr, Mbuf, st, ptc_ws, ptc_bytes));
      else
        TNB_TRY(cp_mttkrp<T>(X, d, n, R, A.data(), Y0, Y1, Mbuf, st, ptc_ws, ptc_bytes));
      hadamard_grams_kernel<<<grid_for(R * R), 256, 0, st>>>(gp, N, n, R, P);
      TNB_LAUNCH_CHECK();
      if (n == N - 1) {  // <X, [[A]]> needs M_{N-1} and the NEW A_{N-1}; ||[[A]]||^2 needs all new grams
        TNB_CUDA(cudaMemsetAsync(acc, 0, 2 * sizeof(double), st));
      }
      // A_n = M P^+  (lstsq, tensor.py:358-360)
      TNB_TRY(jacobi2_eigh(P, R, R, lam, Q, js, jinfo, st));
      pinv_from_eig_kernel<<<grid_for(R * R), 256, 0, st>>>(Q, lam, R, 2.220446049250313e-16 * std::max<int64_t>(R, 1), Pinv);
      TNB_LAUNCH_CHECK();
      convert_kernel<double, T><<<grid_for(R * R), 256, 0, st>>>(Pinv, PinvT, (int64_t)R * R);
      TNB_LAUNCH_CHECK();
      TNB_TRY((gemm_direct<T, T, T, T>(d.shape[n], R, R, Mbuf, R, true, PinvT, R, false, A[n], R, (T)1, nullptr, 0, (T)0,
                                       nullptr, 0, (T)0, st)));
      GemmPlan pl = plan_gemm(R, R, d.shape[n], false);
      TNB_TRY((gemm_splitk<T, T, double, double, double>(pl, R, R, d.shape[n], A[n], R, false, A[n], R, false, gpart,
                                                         grams + (size_t)n * R * R, R, 1.0, nullptr, 0, 0.0, nullptr, 0,
                                                         0.0, false, (double*)nullptr, 0, st)));
    }
    // relative error of this sweep
    hadamard_grams_kernel<<<grid_for(R * R), 256, 0, st>>>(gp, N, -1, R, P);
    TNB_LAUNCH_CHECK();
    cp_error_terms_kernel<T><<<64, 256, 0, st>>>(Mbuf, A[N - 1], d.shape[N - 1] * R, P, R * R, acc);
    TNB_LAUNCH_CHECK();
    TNB_CUDA(cudaMemcpyAsync(h, acc, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
    TNB_CUDA(cudaStreamSynchronize(st));
    double e2 = normX2 - 2.0 * h[0] + h[1];
    if (e2 < 0.0) e2 = 0.0;
    const double err = normX2 > 0.0 ? std::sqrt(e2 / normX2) : 0.0;
    if (errors_host) errors_host[it] = err;
    if (it >= 1 && prev_err - err < tol) {  // tensor.py:380-381
      ++it;
      break;
    }
    prev_err = err;
  }
  if (iters_host) *iters_host = it;
  return TNB_OK;
}

}  // namespace tnb
