// Small dense symmetric eigenproblems on one CTA: parallel-order one-sided (Hestenes) Jacobi with
// warp-shuffle reductions, fp64 throughout.  Replaces torch.linalg.eigh (round.py:114) and the
// U,S part of torch.linalg.svd (round.py:96) for Gram matrices up to JACOBI_MAX_N.
#pragma once
#include "common.cuh"

namespace tnb {

constexpr int JACOBI_MAX_N = 256;      // one-CTA solver limit (matrix in L1/L2-backed global memory above ~100)
constexpr int JACOBI_SMEM_MAX_N = 104; // A and V both in shared memory up to this size
constexpr int JACOBI_THREADS = 1024;

// Block-wide reduction of one double per thread with the associative `op` (identity: the value the unused slots of
// the second stage hold); every thread returns the result.
template <class Op>
__device__ __forceinline__ double block_reduce(double v, double* red /*>=32 doubles smem*/, Op op, double identity) {
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  double t = (threadIdx.x < nw) ? red[threadIdx.x] : identity;
  if (w == 0) {
    for (int o = 16; o > 0; o >>= 1) t = op(t, __shfl_xor_sync(0xffffffffu, t, o));
    if (lane == 0) red[0] = t;
  }
  __syncthreads();
  const double out = red[0];
  __syncthreads();
  return out;
}

struct SumOp {
  __device__ __forceinline__ double operator()(double a, double b) const { return a + b; }
};

__device__ __forceinline__ double block_reduce_sum(double v, double* red /*>=32 doubles smem*/) {
  return block_reduce(v, red, SumOp{}, 0.0);
}

// Rotation (c, s) that orthogonalises two columns with squared norms dpp, dqq and inner product dpq:
//   t = sign(tau)/(|tau| + sqrt(1+tau^2)), tau = (dqq-dpp)/(2 dpq);  c = 1/sqrt(1+t^2);  s = t c.
// ANY t gives an exactly orthogonal rotation as long as c and s are consistent, so t is evaluated in
// fp32 on exponent-normalised inputs (MUFU sqrt / division: a handful of instructions instead of three
// software fp64 divisions/square roots), and only c = rsqrt(1+t^2) is refined to full precision with two
// Newton steps.  A pair is then annihilated to ~1e-7 relative per rotation instead of 1e-16, which the
// next sweep finishes (convergence stays superlinear); V stays orthogonal to working precision.
__device__ __forceinline__ void jacobi_rotation(double dpp, double dqq, double dpq, double& c, double& s) {
  const double h = dqq - dpp, b2 = 2.0 * dpq;
  const double big = fmax(fabs(h), fabs(b2));
  // 2^-e with e = exponent of big, built from the exponent bits (big is a normal number: dpq passed the threshold)
  const int ebits = (__double2hiint(big) >> 20) & 0x7ff;
  int sbits = 2046 - ebits;               // biased exponent of 2^-(e)
  sbits = sbits < 1 ? 1 : (sbits > 2046 ? 2046 : sbits);
  const double scale = __hiloint2double(sbits << 20, 0);
  const float hf = (float)(h * scale), bf = (float)(b2 * scale);
  const float radf = sqrtf(fmaf(hf, hf, bf * bf));
  float tf = __fdividef(bf, fabsf(hf) + radf);
  if (hf < 0.f) tf = -tf;
  const double t = (double)tf;
  const double x = fma(t, t, 1.0);  // in [1, 2]
  double y = (double)rsqrtf((float)x);
  y = y * fma(-0.5 * x, y * y, 1.5);
  y = y * fma(-0.5 * x, y * y, 1.5);
  c = y;
  s = t * y;
}
__device__ __forceinline__ void jacobi_rotation(float dpp, float dqq, float dpq, float& c, float& s) {
  const float h = dqq - dpp, b2 = 2.f * dpq;
  const float radf = sqrtf(fmaf(h, h, b2 * b2));
  float t = __fdividef(b2, fabsf(h) + radf);
  if (h < 0.f) t = -t;
  c = rsqrtf(fmaf(t, t, 1.f));
  s = t * c;
}

template <typename R> struct JacTraits;
template <> struct JacTraits<double> { static constexpr double floor_rel = 1e-30; };
template <> struct JacTraits<float> { static constexpr float floor_rel = 1e-13f; };

// Eigen-decomposition of the symmetric PSD n x n matrix Gin (leading dimension ldg) by ONE-SIDED
// (Hestenes) Jacobi in precision R (double for the truncation step, float for the b x b problems of the
// fp32 subspace iteration).  W = G V is kept column by column; a group of LANES lanes owns one column
// pair per round (32/LANES pairs per warp, so the per-pair scalar work is issued once per warp), takes
// the three inner products with shuffle reductions, rotates its two columns of W and V; the only
// block-wide synchronisation is one barrier per round (np-1 rounds per sweep, circle ordering).
// At convergence W = V diag(lambda), lambda_c = v_c . w_c.
//   w_out[0..n)   eigenvalues, descending (fp64)
//   V_out[n x n]  row-major fp64, column j = eigenvector of w_out[j]
//   scratch       2*np*np R's when !SMEM (np = n rounded up to even)
//   info[0]       number of sweeps used (negative if max_sweeps hit without convergence)
template <typename R, bool SMEM, int LANES, int EPL>
__global__ void __launch_bounds__(JACOBI_THREADS) jacobi_eigh_kernel(const double* __restrict__ Gin, int n, int ldg,
                                                                     double* __restrict__ w_out,
                                                                     double* __restrict__ V_out,
                                                                     R* __restrict__ scratch, int max_sweeps,
                                                                     R tol, int* __restrict__ info, int v_in_smem) {
  extern __shared__ __align__(16) unsigned char jac_smem_raw[];
  const int np = n + (n & 1);
  const int m = np >> 1;
  const int ld = np + 8;  // padded column stride: the lane groups of a warp hit different banks
  R* Wt;  // column-major: Wt[c*ld + r] = W[r][c]
  R* Vt;
  // SMEM: W (the matrix every round reads three inner products from) lives in shared memory; V joins it when
  // both fit (v_in_smem), otherwise V stays in the L1/L2-backed global scratch (it is only touched by rotations)
  if (SMEM) {
    Wt = reinterpret_cast<R*>(jac_smem_raw);
    Vt = v_in_smem ? Wt + (size_t)np * ld : scratch;
  } else {
    Wt = scratch;
    Vt = scratch + (size_t)np * ld;
  }
  __shared__ double s_w[JACOBI_MAX_N + 2];
  __shared__ int s_rank[JACOBI_MAX_N + 2];
  __shared__ double s_gmax;
  __shared__ int s_nrot;
  const int tid = threadIdx.x, nt = blockDim.x;
  const int lane = tid & 31, warp = tid >> 5, nwarps = nt >> 5;
  constexpr int PPW = 32 / LANES;           // pairs per warp per pass
  const int sub = lane / LANES, sl = lane % LANES;

  // scale by the largest diagonal entry (keeps fp32 in range; eigenvalues are scaled back at the end)
  double dmax_local = 0.0;
  for (int i = tid; i < n; i += nt) dmax_local = fmax(dmax_local, fabs(Gin[(size_t)i * ldg + i]));
  for (int o = 16; o > 0; o >>= 1) dmax_local = fmax(dmax_local, __shfl_xor_sync(0xffffffffu, dmax_local, o));
  if (tid == 0) s_gmax = 0.0;
  __syncthreads();
  if (lane == 0)  // non-negative doubles order like their bit patterns
    atomicMax(reinterpret_cast<unsigned long long*>(&s_gmax), (unsigned long long)__double_as_longlong(dmax_local));
  __syncthreads();
  const double gscale = s_gmax > 0.0 ? s_gmax : 1.0;
  const double ginv = 1.0 / gscale;
  __syncthreads();

  for (int idx = tid; idx < np * np; idx += nt) {
    const int c = idx / np, r = idx % np;
    double v = 0.0;
    if (r < n && c < n) v = 0.5 * (Gin[(size_t)r * ldg + c] + Gin[(size_t)c * ldg + r]) * ginv;  // symmetrise, scale
    Wt[(size_t)c * ld + r] = (R)v;
    Vt[(size_t)c * ld + r] = (r == c) ? (R)1 : (R)0;
  }
  __syncthreads();
  // reference scale: largest squared column norm (~ lambda_max^2 in scaled units)
  for (int c = warp; c < np; c += nwarps) {
    R sacc = 0;
    for (int r = lane; r < np; r += 32) { const R a = Wt[(size_t)c * ld + r]; sacc += a * a; }
    for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
    if (lane == 0) s_w[c] = (double)sacc;
  }
  __syncthreads();
  if (tid == 0) {
    double g = 0.0;
    for (int c = 0; c < np; ++c) g = s_w[c] > g ? s_w[c] : g;
    s_gmax = g;
  }
  __syncthreads();
  const R floor2 = (R)(JacTraits<R>::floor_rel * s_gmax);  // pairs of columns both at the noise level are left alone
  const R tol2 = tol * tol;

  int sweeps_done = 0;
  bool converged = false;
  for (int sweep = 0; sweep < max_sweeps; ++sweep) {
    if (tid == 0) s_nrot = 0;
    __syncthreads();
    int rot = 0;
    for (int step = 0; step < np - 1; ++step) {
      for (int base = warp * PPW; base < m; base += nwarps * PPW) {  // warp-uniform trip count
        const int pi = base + sub;
        const bool active = pi < m;
        int p = 0, q = 1;
        if (active) {
          if (pi == 0) {
            p = np - 1;
            q = step;  // step < np - 1
          } else {      // circle method: (step + pi) and (step - pi) modulo np - 1
            p = step + pi;
            if (p >= np - 1) p -= np - 1;
            q = step - pi;
            if (q < 0) q += np - 1;
          }
          if (p > q) { const int t = p; p = q; q = t; }
        }
        R* wp = Wt + (size_t)p * ld;
        R* wq = Wt + (size_t)q * ld;
        // this lane's slice of both columns lives in registers for the whole pair update
        R a[EPL], bq[EPL];
        R dpp = 0, dqq = 0, dpq = 0;
#pragma unroll
        for (int i = 0; i < EPL; ++i) {
          const int r = sl + i * LANES;
          const bool ok = active && r < np;
          a[i] = ok ? wp[r] : (R)0;
          bq[i] = ok ? wq[r] : (R)0;
        }
#pragma unroll
        for (int i = 0; i < EPL; ++i) {
          dpp = fma(a[i], a[i], dpp);
          dqq = fma(bq[i], bq[i], dqq);
          dpq = fma(a[i], bq[i], dpq);
        }
#pragma unroll
        for (int o = LANES / 2; o > 0; o >>= 1) {
          dpp += __shfl_xor_sync(0xffffffffu, dpp, o);
          dqq += __shfl_xor_sync(0xffffffffu, dqq, o);
          dpq += __shfl_xor_sync(0xffffffffu, dpq, o);
        }
        const R prod = dpp * dqq;
        if (active && dpq * dpq > tol2 * prod && prod > floor2 * floor2) {  // uniform within the lane group
          rot = 1;
          R c, s;
          jacobi_rotation(dpp, dqq, dpq, c, s);
          R* vp = Vt + (size_t)p * ld;
          R* vq = Vt + (size_t)q * ld;
#pragma unroll
          for (int i = 0; i < EPL; ++i) {
            const int r = sl + i * LANES;
            if (r < np) {
              const R x = vp[r], y = vq[r];
              wp[r] = c * a[i] - s * bq[i];
              wq[r] = s * a[i] + c * bq[i];
              vp[r] = c * x - s * y;
              vq[r] = s * x + c * y;
            }
          }
        }
      }
      __syncthreads();
    }
    if (rot) atomicAdd(&s_nrot, 1);
    __syncthreads();
    sweeps_done = sweep + 1;
    const int nrot = s_nrot;
    __syncthreads();
    if (nrot == 0) {  // a full sweep without a single rotation: converged
      converged = true;
      break;
    }
  }

  // eigenvalues as Rayleigh quotients lambda_c = v_c . (G v_c) = v_c . w_c (fp64 accumulate); sort; write out
  for (int c = warp; c < n; c += nwarps) {
    double sacc = 0.0;
    for (int r = lane; r < np; r += 32) sacc = fma((double)Vt[(size_t)c * ld + r], (double)Wt[(size_t)c * ld + r], sacc);
    for (int o = 16; o > 0; o >>= 1) sacc += __shfl_xor_sync(0xffffffffu, sacc, o);
    if (lane == 0) s_w[c] = sacc * gscale;
  }
  __syncthreads();
  for (int i = tid; i < n; i += nt) {
    const double wi = s_w[i];
    int r = 0;
    for (int j = 0; j < n; ++j) {
      const double wj = s_w[j];
      r += (wj > wi) || (wj == wi && j < i);
    }
    s_rank[i] = r;
    w_out[r] = wi;
  }
  __syncthreads();
  for (int idx = tid; idx < n * n; idx += nt) {
    const int k = idx / n, i = idx % n;
    V_out[(size_t)k * n + s_rank[i]] = (double)Vt[(size_t)i * ld + k];
  }
  if (tid == 0 && info) info[0] = converged ? sweeps_done : -sweeps_done;
}

inline size_t jacobi_scratch_doubles(int n) {
  const int np = n + (n & 1);
  return (size_t)2 * np * (np + 8);
}

template <typename R, bool SMEM>
inline void jacobi_launch(int n, size_t smem, const double* G, int ldg, double* w, double* V, R* scratch, int max_sweeps,
                          R tol, int* info, cudaStream_t st, int v_in_smem = 1) {
  // lanes per column pair (LANES) x elements per lane (EPL) >= n; small problems use 8 lanes (4 pairs per warp)
  // the block is sized to the warps that own a pair (idle warps would only lengthen every barrier)
  if (n <= 64)
    jacobi_eigh_kernel<R, SMEM, 8, 8><<<1, 256, smem, st>>>(G, n, ldg, w, V, scratch, max_sweeps, tol, info, v_in_smem);
  else if (n <= 128)
    jacobi_eigh_kernel<R, SMEM, 8, 16><<<1, 512, smem, st>>>(G, n, ldg, w, V, scratch, max_sweeps, tol, info, v_in_smem);
  else
    jacobi_eigh_kernel<R, SMEM, 16, 16><<<1, JACOBI_THREADS, smem, st>>>(G, n, ldg, w, V, scratch, max_sweeps, tol, info, v_in_smem);
}

// G: n x n fp64 (ld = ldg). w: n, V: n x n. scratch: jacobi_scratch_doubles(n) doubles.
// single_precision: run the rotations in fp32 (for the b x b problems of the fp32 subspace iteration).
// loose_tol > 0 overrides the convergence threshold (Rayleigh-Ritz inside the subspace iteration only needs the
// Ritz basis to ~1e-5: the rotations stay exactly orthogonal and the captured energy is second order in it).
inline int jacobi_eigh(const double* G, int n, int ldg, double* w, double* V, double* scratch, int* info,
                       cudaStream_t st, bool single_precision = false, double loose_tol = 0.0) {
  if (n < 1 || n > JACOBI_MAX_N) return fail(TNB_ERR_UNSUPPORTED, "jacobi_eigh: n=%d outside [1,%d]", n, JACOBI_MAX_N);
  const int np = n + (n & 1);
  const int max_sweeps = 30;
  const int maxb = 2 * (JACOBI_SMEM_MAX_N) * (JACOBI_SMEM_MAX_N + 8) * (int)sizeof(double);
  static PerDeviceFlag attr_done[6];
  TNB_CUDA(ensure_dyn_smem(attr_done[0], jacobi_eigh_kernel<double, true, 8, 8>, maxb));
  TNB_CUDA(ensure_dyn_smem(attr_done[1], jacobi_eigh_kernel<float, true, 8, 8>, maxb));
  TNB_CUDA(ensure_dyn_smem(attr_done[2], jacobi_eigh_kernel<double, true, 8, 16>, maxb));
  TNB_CUDA(ensure_dyn_smem(attr_done[3], jacobi_eigh_kernel<float, true, 8, 16>, maxb));
  TNB_CUDA(ensure_dyn_smem(attr_done[4], jacobi_eigh_kernel<double, true, 16, 16>, maxb));
  TNB_CUDA(ensure_dyn_smem(attr_done[5], jacobi_eigh_kernel<float, true, 16, 16>, maxb));
  if (single_precision) {
    const float tol = loose_tol > 0.0 ? (float)loose_tol : 2e-6f;  // default ~ eps_fp32 * sqrt(n)
    const size_t one = (size_t)np * (np + 8) * sizeof(float);
    if (2 * one <= (size_t)maxb)
      jacobi_launch<float, true>(n, 2 * one, G, ldg, w, V, reinterpret_cast<float*>(scratch), max_sweeps, tol, info, st, 1);
    else if (one <= (size_t)maxb)
      jacobi_launch<float, true>(n, one, G, ldg, w, V, reinterpret_cast<float*>(scratch), max_sweeps, tol, info, st, 0);
    else
      jacobi_launch<float, false>(n, 0, G, ldg, w, V, reinterpret_cast<float*>(scratch), max_sweeps, tol, info, st);
  } else {
    const double tol = loose_tol > 0.0 ? loose_tol : 1e-14;  // relative threshold |w_p.w_q| <= tol*|w_p||w_q|
    const size_t one = (size_t)np * (np + 8) * sizeof(double);
    if (2 * one <= (size_t)maxb)
      jacobi_launch<double, true>(n, 2 * one, G, ldg, w, V, scratch, max_sweeps, tol, info, st, 1);
    else if (one <= (size_t)maxb)
      jacobi_launch<double, true>(n, one, G, ldg, w, V, scratch, max_sweeps, tol, info, st, 0);
    else
      jacobi_launch<double, false>(n, 0, G, ldg, w, V, scratch, max_sweeps, tol, info, st);
  }
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

}  // namespace tnb
