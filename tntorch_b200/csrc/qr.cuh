// Tall-skinny Householder QR on the device, one CTA per matrix (batched), fp64.
// A (rows x n, rows >= 1) = Q R with Q (rows x k) explicit, k = min(rows, n): the geqr2 / org2r recurrences
// (the ones LAPACK's geqrf/orgqr block), so Q matches torch.linalg.qr(V)[0] up to rounding, including its
// sign convention (beta = -sign(alpha) ||x||) and its completion of rank-deficient columns — which is what
// tn.cross needs before maxvol (cross.py:398, 430): an orthonormal basis with ALL n columns even when the
// sampled fibres are numerically rank deficient.
//
// Column operations are warp-per-column: the inner products v^T a_c are lane-strided sums finished with
// shuffles, the reflector norm is a block reduction, one barrier per reflector.
//
// The reflector is formed like LAPACK dlarfg: the norm of x = col[j+1:] is taken as m * sqrt(sum (x_i/m)^2) with
// m = max |x_i| (one more block reduction per column), and beta = -sign(alpha) hypot(alpha, ||x||).  An unscaled
// sum of squares underflows to 0 below |x| ~ 1e-160 (every tau 0, Q = I) and overflows above ~ 1e154, so Q would
// depend on the scale of the input; with the scaled norm Q(c A) = Q(A) and R(c A) = c R(A) to rounding for any
// normal c.  dlarfg's extra rescaling of |beta| < 2e-292 (subnormal-range results) is not reproduced.  The max keeps
// NaN, so a NaN input still reaches Q and R.
#pragma once
#include <cfloat>

#include "common.cuh"
#include "jacobi.cuh"

namespace tnb {

// max that keeps NaN (fmax would drop it): a NaN anywhere below the diagonal makes m, and so Q and R, NaN
struct NanMaxOp {
  __device__ __forceinline__ double operator()(double a, double b) const { return (b != b || b > a) ? b : a; }
};

// work: [nbatch][n][rows] (column-major copy of A, holds the reflectors), Qout: [nbatch][rows][k] row-major,
// Rout (optional): [nbatch][k][n] row-major upper-trapezoidal factor.
__global__ void __launch_bounds__(512) householder_qr_kernel(const double* __restrict__ A_all, int rows, int n,
                                                             double* __restrict__ work_all, double* __restrict__ Q_all,
                                                             double* __restrict__ R_all) {
  extern __shared__ double qr_tau[];  // k taus
  __shared__ double red[32];
  __shared__ double s_scal[2];
  const int k = rows < n ? rows : n;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  const double* A = A_all + (size_t)blockIdx.x * rows * n;
  double* W = work_all + (size_t)blockIdx.x * rows * n;  // W[c*rows + i] = A[i][c]
  double* Q = Q_all + (size_t)blockIdx.x * rows * k;
  for (int idx = tid; idx < rows * n; idx += nt) {
    const int i = idx / n, c = idx % n;
    W[(size_t)c * rows + i] = A[idx];
  }
  __syncthreads();
  for (int j = 0; j < k; ++j) {
    double* col = W + (size_t)j * rows;
    double m = 0.0;
    for (int i = j + 1 + tid; i < rows; i += nt) m = NanMaxOp{}(m, fabs(col[i]));
    m = block_reduce(m, red, NanMaxOp{}, 0.0);
    double s = 0.0;
    if (m != 0.0) {
      if (m >= DBL_MIN) {  // 1/m is finite for a normal m: one reciprocal, then multiplies
        const double inv_m = 1.0 / m;
        for (int i = j + 1 + tid; i < rows; i += nt) {
          const double x = col[i] * inv_m;
          s = fma(x, x, s);
        }
      } else {  // subnormal (1/m would overflow) or NaN
        for (int i = j + 1 + tid; i < rows; i += nt) {
          const double x = col[i] / m;
          s = fma(x, x, s);
        }
      }
      s = block_reduce_sum(s, red);
    }
    if (tid == 0) {
      const double alpha = col[j];
      double tau = 0.0, scale = 0.0, beta = alpha;
      if (m != 0.0) {
        beta = -copysign(hypot(alpha, m * sqrt(s)), alpha);
        tau = (beta - alpha) / beta;
        scale = 1.0 / (alpha - beta);
      }
      qr_tau[j] = tau;
      s_scal[0] = scale;
      col[j] = beta;
    }
    __syncthreads();
    const double scale = s_scal[0], tau = qr_tau[j];
    for (int i = j + 1 + tid; i < rows; i += nt) col[i] *= scale;  // v (v_j = 1 implicit)
    __syncthreads();
    if (tau != 0.0) {
      for (int c = j + 1 + warp; c < n; c += nwarps) {
        double* a = W + (size_t)c * rows;
        double w = (lane == 0) ? a[j] : 0.0;
        for (int i = j + 1 + lane; i < rows; i += 32) w = fma(col[i], a[i], w);
        for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
        const double tw = tau * w;
        if (lane == 0) a[j] -= tw;
        for (int i = j + 1 + lane; i < rows; i += 32) a[i] = fma(-tw, col[i], a[i]);
      }
    }
    __syncthreads();
  }
  if (R_all) {
    double* R = R_all + (size_t)blockIdx.x * k * n;
    for (int idx = tid; idx < k * n; idx += nt) {
      const int i = idx / n, c = idx % n;
      R[idx] = (c >= i) ? W[(size_t)c * rows + i] : 0.0;
    }
  }
  // Q = H_0 ... H_{k-1} [I_k; 0]  (org2r): built column-major in the tail of the work area is not possible (W holds v),
  // so Q is accumulated directly in its row-major output with warp-per-column updates.
  for (int idx = tid; idx < rows * k; idx += nt) Q[idx] = (idx / k == idx % k) ? 1.0 : 0.0;
  __syncthreads();
  for (int j = k - 1; j >= 0; --j) {
    const double tau = qr_tau[j];
    const double* v = W + (size_t)j * rows;
    if (tau != 0.0) {
      for (int c = j + warp; c < k; c += nwarps) {
        double w = (lane == 0) ? Q[(size_t)j * k + c] : 0.0;
        for (int i = j + 1 + lane; i < rows; i += 32) w = fma(v[i], Q[(size_t)i * k + c], w);
        for (int o = 16; o > 0; o >>= 1) w += __shfl_xor_sync(0xffffffffu, w, o);
        const double tw = tau * w;
        if (lane == 0) Q[(size_t)j * k + c] -= tw;
        for (int i = j + 1 + lane; i < rows; i += 32) Q[(size_t)i * k + c] = fma(-tw, v[i], Q[(size_t)i * k + c]);
      }
    }
    __syncthreads();
  }
}

inline size_t householder_qr_workspace_bytes(int nbatch, int rows, int n) {
  return align_up((size_t)nbatch * rows * n * sizeof(double));
}
inline int householder_qr_run(const double* A, int nbatch, int rows, int n, void* ws, size_t ws_bytes, double* Q, double* R,
                              cudaStream_t st) {
  if (nbatch < 1 || rows < 1 || n < 1) return fail(TNB_ERR_INVALID, "qr: bad shape");
  if (ws_bytes < householder_qr_workspace_bytes(nbatch, rows, n)) return fail(TNB_ERR_WORKSPACE, "qr: workspace too small");
  const int k = rows < n ? rows : n;
  if ((size_t)k * sizeof(double) > 40 * 1024) return fail(TNB_ERR_UNSUPPORTED, "qr: more than 5120 columns");
  householder_qr_kernel<<<nbatch, 512, (size_t)k * sizeof(double), st>>>(A, rows, n, static_cast<double*>(ws), Q, R);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

}  // namespace tnb
