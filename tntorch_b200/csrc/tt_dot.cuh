// Inner products of tensor-train pairs (tnb_tt_dot): for each pair p, trains a and b of one shape (n_0 .. n_{N-1}),
// boundary ranks 1, each pair with its own rank profile,
//   F_0 = [1],   F_{k+1} = sum_i A_k[:, i, :]^T F_k B_k[:, i, :]   (ra_{k+1} x rb_{k+1}),   <a, b> = F_N[0, 0].
// Neither tensor is formed.  All arithmetic is fp64: fp64 cores are read as they are, fp32 cores are widened as they are
// loaded (exact), so every product is exact and every sum is an fp64 sum.
//
// Per mode and pair, ttd_order picks the cheaper association: "A first" contracts F with A (G_i = A_i^T F, then
// G_i B_i), "B first" contracts F with B (G_i = B_i^T F^T, then G_i A_i, the transpose of the result).  Both are one
// computation, P = sum_i X_i^T F' Y_i, with (X, Y) = (A, B) and F' = F, or (X, Y) = (B, A) and F' = F^T; the kernels
// read F through strides and the reduction writes F_{k+1} back in (ra x rb) orientation.
//
// Work items are (pair, chunk of i, 32-row tile of X's columns); a CTA keeps its G_i rows in shared memory and
// accumulates its partial P in registers over the chunk, then writes it to the workspace.  ttd_reduce_kernel sums the
// chunks of each pair in a fixed order into F_{k+1} (or, after the last mode, into out[p]): no atomics, so a call is
// bitwise reproducible.  The number of chunks per pair (ttd_chunks) depends on the shapes and the pair count only, so
// the result does not depend on the device either.
//
// Inside the envelope (ttd_mode_path) a mode runs ttd_mode_tc_kernel on mma.sync m16n8k16 .f64 (DMMA): each barrier
// stages up to 64 rows of X_i / F / Y_i in shared memory (four k16 steps), zero padded to multiples of 16.  Everything else (tiny, ragged or
// large ranks, and always the boundary modes, whose rank is 1) runs ttd_mode_generic_kernel, fp64 FMAs on the CUDA
// cores, under the same driver.
#pragma once
#include <algorithm>

#include "common.cuh"
#include "small_kernels.cuh"

namespace tnb {

// ---------------------------------------------------------------------------------------------
// The envelope, the association order and the split over i
// ---------------------------------------------------------------------------------------------
constexpr int TTD_TC_MAX_R = 256;   // the rank envelope of the library's other tensor-core kernels
constexpr int TTD_TC_MIN_R = 16;    // below one k16 step of padding most of every DMMA would multiply zeros
constexpr int TTD_BM = 32;          // rows of X's columns (rx') per work item
constexpr int TTD_GN = 64;          // columns of Y (ry') per generic work item
constexpr int TTD_TARGET_ITEMS = 512;  // work items per mode over all pairs (about four per SM)
constexpr int TTD_GROUP = 32;       // pairs per launch (the per-pair table travels in the kernel parameters)

enum TtdPath {
  TTD_PATH_TC = 0,
  TTD_PATH_RANK_MIN = 1,  // a rank below TTD_TC_MIN_R (always the boundary modes)
  TTD_PATH_RANK_MAX = 2,  // a rank above TTD_TC_MAX_R
};

// The path of one mode of one pair, in the roles the order gave: X is [rx, n, rxo], Y is [ry, n, ryo].  The one place
// the envelope is defined.
inline int ttd_mode_path(int64_t rx, int64_t ry, int64_t rxo, int64_t ryo) {
  const int64_t lo = std::min(std::min(rx, ry), std::min(rxo, ryo)), hi = std::max(std::max(rx, ry), std::max(rxo, ryo));
  if (hi > TTD_TC_MAX_R) return TTD_PATH_RANK_MAX;
  if (lo < TTD_TC_MIN_R) return TTD_PATH_RANK_MIN;
  return TTD_PATH_TC;
}

// true: B first (X = B, Y = A).  Multiply-adds per i: A first ra' rb (ra + rb'), B first rb' ra (rb + ra'); ties go A
// first.
inline bool ttd_order(int64_t ra, int64_t rb, int64_t rao, int64_t rbo) {
  return rbo * ra * (rb + rao) < rao * rb * (ra + rbo);
}

// Work items of one chunk: 32-row tiles of rxo, and on the generic path 64-column tiles of ryo.
inline int64_t ttd_tiles(int path, int64_t rxo, int64_t ryo) {
  return ceil_div<int64_t>(rxo, TTD_BM) * (path == TTD_PATH_TC ? 1 : ceil_div<int64_t>(ryo, TTD_GN));
}

// Chunks of i for one pair in a call of npairs pairs: enough that all pairs together make about TTD_TARGET_ITEMS work
// items, at most n, and no chunk empty.
inline int64_t ttd_chunks(int64_t npairs, int64_t n, int64_t tiles) {
  int64_t c = ceil_div<int64_t>(TTD_TARGET_ITEMS, npairs * tiles);
  c = c < 1 ? 1 : c > n ? n : c;
  return ceil_div<int64_t>(n, ceil_div<int64_t>(n, c));
}

// ---------------------------------------------------------------------------------------------
// Per-launch tables
// ---------------------------------------------------------------------------------------------
template <typename T>
struct TtdPair {
  const T* X;            // [rx][n][rxo]
  const T* Y;            // [ry][n][ryo]
  int rx, ry, rxo, ryo;
  int swap;              // 1: B first (F is read transposed, P is written back transposed)
  int nch, tn;           // chunks of i; generic: 64-column tiles of ryo
  int64_t len;           // length of a chunk
  int64_t item0;         // first work item of this pair in the launch
  int64_t f_off;         // F_k of this pair in the workspace (doubles); ignored at the first mode
  int64_t p_off;         // its partials: nch blocks of rxo x ryo doubles
};

template <typename T>
struct TtdTable {
  int np;
  int64_t n;             // mode size
  const double* F;       // the F region; nullptr at the first mode (F_0 = [1])
  double* part;
  TtdPair<T> p[TTD_GROUP];
};

// F'(x, y) of one pair: F_k (ra x rb, row-major) or its transpose; F_0 = [1] when F is null
__device__ __forceinline__ double ttd_f(const double* F, int swap, int rx, int ry, int x, int y) {
  if (!F) return 1.0;
  return swap ? F[(int64_t)y * rx + x] : F[(int64_t)x * ry + y];
}

template <typename T>
__device__ __forceinline__ int ttd_find(const TtdTable<T>& t, int64_t item) {
  int q = 0;
  while (q + 1 < t.np && item >= t.p[q + 1].item0) ++q;
  return q;
}

// ---------------------------------------------------------------------------------------------
// Tensor-core mode: 8 warps; G (32 x ry) and P (32 x ryo) are 2 m16 tiles by up to 32 n8 tiles, warp w taking n8 tiles
// w, w + 8, w + 16, w + 24.  Row strides are 4 mod 16 doubles, so the 16 lanes of a half-warp fragment load hit distinct bank
// pairs.
// ---------------------------------------------------------------------------------------------
constexpr int TTD_THREADS = 256;
constexpr int TTD_KC = 64;                       // rows of X_i / F / Y_i staged per barrier: four k16 steps
constexpr int TTD_SX = TTD_BM + 4;               // Xs[KC][SX]: X_i rows a, columns m of the tile
constexpr int TTD_SW = TTD_TC_MAX_R + 4;         // Fs / Ys [KC][SW] and Gs[32][SW]
constexpr int TTD_SMEM_BYTES = (TTD_KC * TTD_SX + TTD_KC * TTD_SW + TTD_BM * TTD_SW) * 8;
static_assert(TTD_SMEM_BYTES <= 227 * 1024, "ttd_mode_tc: shared memory");

__device__ __forceinline__ void dmma_16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5, %6, %7, %8, %9, %10, %11}, "
      "{%12, %13, %14, %15}, {%0, %1, %2, %3};"
      : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
      : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]),
        "d"(b[2]), "d"(b[3]));
}

// acc[h][jj] += A (32 x 16, A(m, k) = a_at(m, k)) times B (16 x N, B(k, n) = Bs[k * SW + n]) for the warp's n8 tiles.
// Fragments (PTX m16n8k16 .f64): a_i at row g + 8 (i & 1), column t + 4 (i >> 1); b_i at row t + 4 i, column g;
// c at rows g, g + 8 and columns 2t, 2t + 1.
template <class AAt>
__device__ __forceinline__ void ttd_mma_k16(double (&acc)[2][4][4], AAt a_at, const double* Bs, int nt, int w, int g,
                                            int t) {
  double a[2][8];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int i = 0; i < 8; ++i) a[h][i] = a_at(16 * h + g + 8 * (i & 1), t + 4 * (i >> 1));
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    const int j = w + 8 * jj;
    if (j < nt) {
      double b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) b[i] = Bs[(t + 4 * i) * TTD_SW + 8 * j + g];
#pragma unroll
      for (int h = 0; h < 2; ++h) dmma_16816(acc[h][jj], a[h], b);
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(TTD_THREADS, 1) ttd_mode_tc_kernel(const TtdTable<T> tab) {
  extern __shared__ double ttd_smem[];
  double* Xs = ttd_smem;               // [KC][SX]
  double* Ws = Xs + TTD_KC * TTD_SX;   // Fs or Ys [KC][SW]
  double* Gs = Ws + TTD_KC * TTD_SW;   // [32][SW]
  const int q = ttd_find(tab, blockIdx.x);
  const TtdPair<T>& P = tab.p[q];
  const int64_t local = blockIdx.x - P.item0;
  const int mtiles = (P.rxo + TTD_BM - 1) / TTD_BM;
  const int mt = (int)(local % mtiles), ch = (int)(local / mtiles);
  const int m0 = mt * TTD_BM;
  const int64_t n = tab.n, i0 = (int64_t)ch * P.len, i1 = min(n, i0 + P.len);
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int rx = P.rx, ry = P.ry, rxo = P.rxo, ryo = P.ryo;
  const double* F = tab.F ? tab.F + P.f_off : nullptr;
  const int ntg = (ry + 15) / 16 * 2, ntp = (ryo + 7) / 8;  // n8 tiles of G (padded to k16) and of P
  double pacc[2][4][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int jj = 0; jj < 4; ++jj)
#pragma unroll
      for (int e = 0; e < 4; ++e) pacc[h][jj][e] = 0.0;

  for (int64_t i = i0; i < i1; ++i) {
    // ---- G = X_i[:, m0 : m0 + 32]^T F' (32 x ry), K = rx in k16 steps
    double gacc[2][4][4];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int e = 0; e < 4; ++e) gacc[h][jj][e] = 0.0;
    for (int k0 = 0; k0 < rx; k0 += TTD_KC) {
      const int kc = min(TTD_KC, (rx - k0 + 15) / 16 * 16);  // rows staged: the k16 steps that reach into rx
      for (int e = tid; e < kc * TTD_BM; e += TTD_THREADS) {
        const int kk = e / TTD_BM, m = e % TTD_BM;
        const int a = k0 + kk, col = m0 + m;
        Xs[kk * TTD_SX + m] = (a < rx && col < rxo) ? (double)P.X[((int64_t)a * n + i) * rxo + col] : 0.0;
      }
      for (int e = tid; e < kc * ntg * 8; e += TTD_THREADS) {
        const int kk = e / (ntg * 8), y = e % (ntg * 8);
        const int a = k0 + kk;
        Ws[kk * TTD_SW + y] = (a < rx && y < ry) ? ttd_f(F, P.swap, rx, ry, a, y) : 0.0;
      }
      __syncthreads();
      for (int ks = 0; ks < kc; ks += 16)
        ttd_mma_k16(gacc, [&](int m, int k) { return Xs[(ks + k) * TTD_SX + m]; }, Ws + ks * TTD_SW, ntg, w, g, t);
      __syncthreads();
    }
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int j = w + 8 * jj;
        if (j < ntg) {
          double* r0 = Gs + (16 * h + g) * TTD_SW + 8 * j + 2 * t;
          r0[0] = gacc[h][jj][0], r0[1] = gacc[h][jj][1];
          r0[8 * TTD_SW] = gacc[h][jj][2], r0[8 * TTD_SW + 1] = gacc[h][jj][3];
        }
      }
    // ---- P += G Y_i (32 x ryo), K = ry in k16 steps (G's columns past ry are zero)
    for (int k0 = 0; k0 < ry; k0 += TTD_KC) {
      const int kc = min(TTD_KC, (ry - k0 + 15) / 16 * 16);
      for (int e = tid; e < kc * ntp * 8; e += TTD_THREADS) {
        const int kk = e / (ntp * 8), c = e % (ntp * 8);
        const int b = k0 + kk;
        Ws[kk * TTD_SW + c] = (b < ry && c < ryo) ? (double)P.Y[((int64_t)b * n + i) * ryo + c] : 0.0;
      }
      __syncthreads();
      for (int ks = 0; ks < kc; ks += 16)
        ttd_mma_k16(pacc, [&](int m, int k) { return Gs[m * TTD_SW + k0 + ks + k]; }, Ws + ks * TTD_SW, ntp, w, g, t);
      __syncthreads();
    }
  }
  double* out = tab.part + P.p_off + (int64_t)ch * rxo * ryo;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int j = w + 8 * jj;
      if (j >= ntp) continue;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = m0 + 16 * h + g + 8 * (e >> 1), c = 8 * j + 2 * t + (e & 1);
        if (m < rxo && c < ryo) out[(int64_t)m * ryo + c] = pacc[h][jj][e];
      }
    }
}

// ---------------------------------------------------------------------------------------------
// Generic mode: any ranks.  Work item (pair, chunk, 32-row tile of rxo, 64-column tile of ryo); per i and per 32-wide
// slice of ry, G (32 x 32) is formed in shared memory from X_i and F', then P (32 x 64, eight per thread) takes G Y_i.
// ---------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(TTD_THREADS) ttd_mode_generic_kernel(const TtdTable<T> tab) {
  __shared__ double Gs[TTD_BM][33];
  const int q = ttd_find(tab, blockIdx.x);
  const TtdPair<T>& P = tab.p[q];
  const int64_t local = blockIdx.x - P.item0;
  const int64_t mtiles = (P.rxo + TTD_BM - 1) / TTD_BM;
  const int tn = (int)(local % P.tn), mt = (int)(local / P.tn % mtiles), ch = (int)(local / P.tn / mtiles);
  const int m0 = mt * TTD_BM, c0 = tn * TTD_GN;
  const int64_t n = tab.n, i0 = (int64_t)ch * P.len, i1 = min(n, i0 + P.len);
  const int tid = threadIdx.x;
  const int rx = P.rx, ry = P.ry, rxo = P.rxo, ryo = P.ryo;
  const double* F = tab.F ? tab.F + P.f_off : nullptr;
  const int pm = tid >> 3, pc = tid & 7;  // this thread's P entries: row pm, columns pc + 8 j
  double acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.0;
  for (int64_t i = i0; i < i1; ++i) {
    for (int b0 = 0; b0 < ry; b0 += 32) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int e = tid + TTD_THREADS * u, m = e >> 5, bb = e & 31;
        const int col = m0 + m, b = b0 + bb;
        double s = 0.0;
        if (col < rxo && b < ry)
          for (int a = 0; a < rx; ++a)
            s = fma((double)P.X[((int64_t)a * n + i) * rxo + col], ttd_f(F, P.swap, rx, ry, a, b), s);
        Gs[m][bb] = s;
      }
      __syncthreads();
      const int bl = min(32, ry - b0);
      for (int bb = 0; bb < bl; ++bb) {
        const double gv = Gs[pm][bb];
        const T* yr = P.Y + ((int64_t)(b0 + bb) * n + i) * ryo;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = c0 + pc + 8 * j;
          if (c < ryo) acc[j] = fma(gv, (double)yr[c], acc[j]);
        }
      }
      __syncthreads();
    }
  }
  const int m = m0 + pm;
  if (m >= rxo) return;
  double* out = tab.part + P.p_off + ((int64_t)ch * rxo + m) * ryo;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c0 + pc + 8 * j;
    if (c < ryo) out[c] = acc[j];
  }
}

// ---------------------------------------------------------------------------------------------
// Reduction: F_{k+1}[a'][b'] = sum over chunks, in chunk order, of P[x'][y'] ((x', y') = (a', b'), or (b', a') when
// swapped); after the last mode F_N is 1 x 1 and goes to out[pair].
// ---------------------------------------------------------------------------------------------
struct TtdReduceTable {
  int np;
  const double* part;
  double* F;               // F_{k+1} region, or nullptr after the last mode
  double* out;             // out + first pair of the group, after the last mode
  int64_t end[TTD_GROUP];  // running sum of the pairs' output entries
  int64_t p_off[TTD_GROUP], f_off[TTD_GROUP];
  int rao[TTD_GROUP], rbo[TTD_GROUP], nch[TTD_GROUP], swap[TTD_GROUP];
};

__global__ void ttd_reduce_kernel(const TtdReduceTable tab) {
  const int64_t total = tab.end[tab.np - 1];
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int q = 0;
    while (idx >= tab.end[q]) ++q;
    const int64_t e = idx - (q ? tab.end[q - 1] : 0);
    const int ra = tab.rao[q], rb = tab.rbo[q];
    const int a = (int)(e / rb), b = (int)(e % rb);
    const int64_t src = tab.swap[q] ? (int64_t)b * ra + a : e;
    const double* p = tab.part + tab.p_off[q];
    double s = 0.0;
    for (int c = 0; c < tab.nch[q]; ++c) s += p[(int64_t)c * ra * rb + src];
    if (tab.F)
      tab.F[tab.f_off[q] + e] = s;
    else
      tab.out[q] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// The driver
// ---------------------------------------------------------------------------------------------
constexpr int TTD_MAX_D = 1024;
constexpr int64_t TTD_MAX_ELEMS = (int64_t)1 << 46;  // of every core

// ndim >= 1, npairs >= 1, every mode size and rank >= 1, unit boundary ranks (TNB_ERR_INVALID); ndim <= TTD_MAX_D, each
// core within TTD_MAX_ELEMS and each rank below 2^31 / 64 (TNB_ERR_UNSUPPORTED).
inline int ttd_check_dims(int npairs, int ndim, const int64_t* shape, const int32_t* ra, const int32_t* rb) {
  if (npairs < 1) return fail(TNB_ERR_INVALID, "tt_dot: npairs=%d must be >= 1", npairs);
  if (ndim < 1) return fail(TNB_ERR_INVALID, "tt_dot: ndim=%d must be >= 1", ndim);
  if (ndim > TTD_MAX_D) return fail(TNB_ERR_UNSUPPORTED, "tt_dot: ndim=%d above %d", ndim, TTD_MAX_D);
  for (int k = 0; k < ndim; ++k)
    if (shape[k] < 1) return fail(TNB_ERR_INVALID, "tt_dot: mode sizes must be >= 1");
  for (int p = 0; p < npairs; ++p) {
    const int32_t* r[2] = {ra + (int64_t)p * (ndim + 1), rb + (int64_t)p * (ndim + 1)};
    for (int s = 0; s < 2; ++s) {
      if (r[s][0] != 1 || r[s][ndim] != 1) return fail(TNB_ERR_INVALID, "tt_dot: pair %d: boundary ranks must be 1", p);
      for (int k = 1; k < ndim; ++k) {
        if (r[s][k] < 1) return fail(TNB_ERR_INVALID, "tt_dot: pair %d: ranks must be >= 1", p);
        if (r[s][k] >= (1 << 25)) return fail(TNB_ERR_UNSUPPORTED, "tt_dot: pair %d: rank %d too large", p, (int)r[s][k]);
      }
      for (int k = 0; k < ndim; ++k)
        if ((unsigned __int128)r[s][k] * shape[k] * r[s][k + 1] > (unsigned __int128)TTD_MAX_ELEMS)
          return fail(TNB_ERR_UNSUPPORTED, "tt_dot: pair %d: core %d too large", p, k);
    }
  }
  return TNB_OK;
}

// One mode of one pair, as the driver plans it.
struct TtdPlan {
  int swap, path;
  int64_t rx, ry, rxo, ryo, tn, tiles, nch, len;
};

inline TtdPlan ttd_plan(int npairs, int64_t n, int64_t ra, int64_t rb, int64_t rao, int64_t rbo) {
  TtdPlan pl;
  pl.swap = ttd_order(ra, rb, rao, rbo) ? 1 : 0;
  pl.rx = pl.swap ? rb : ra, pl.ry = pl.swap ? ra : rb, pl.rxo = pl.swap ? rbo : rao, pl.ryo = pl.swap ? rao : rbo;
  pl.path = ttd_mode_path(pl.rx, pl.ry, pl.rxo, pl.ryo);
  pl.tn = pl.path == TTD_PATH_TC ? 1 : ceil_div<int64_t>(pl.ryo, TTD_GN);
  pl.tiles = ttd_tiles(pl.path, pl.rxo, pl.ryo);
  pl.nch = ttd_chunks(npairs, n, pl.tiles);
  pl.len = ceil_div<int64_t>(n, pl.nch);
  return pl;
}

template <typename T>
inline int ttd_launch_mode(bool tc, TtdTable<T>& tab, int64_t items, cudaStream_t st) {
  if (items == 0) return TNB_OK;
  if (tc) {
    static PerDeviceFlag attr_done;
    TNB_CUDA(ensure_dyn_smem(attr_done, ttd_mode_tc_kernel<T>, TTD_SMEM_BYTES));
    ttd_mode_tc_kernel<T><<<(unsigned)items, TTD_THREADS, TTD_SMEM_BYTES, st>>>(tab);
  } else {
    ttd_mode_generic_kernel<T><<<(unsigned)items, TTD_THREADS, 0, st>>>(tab);
  }
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// T: float or double.  Workspace: one F region (each pair's largest interior F_k) and one partials region (the largest
// mode's chunks over all pairs); mode k reads F_k and writes partials, its reduction then overwrites F_k with F_{k+1}.
template <typename T, class ArenaT>
inline int tt_dot_impl(ArenaT& ar, bool dry, const T* const* ca, const T* const* cb, int npairs, int ndim,
                       const int64_t* shape, const int32_t* ranks_a, const int32_t* ranks_b, double* out,
                       cudaStream_t st) {
  const int64_t R = ndim + 1;
  int64_t f_total = 0, p_max = 0;
  for (int p = 0; p < npairs; ++p) {
    int64_t fm = 0;
    for (int k = 1; k < ndim; ++k) fm = std::max(fm, (int64_t)ranks_a[p * R + k] * ranks_b[p * R + k]);
    f_total += fm;
  }
  for (int k = 0; k < ndim; ++k) {
    int64_t s = 0;
    for (int p = 0; p < npairs; ++p) {
      const int32_t *a = ranks_a + p * R, *b = ranks_b + p * R;
      const TtdPlan pl = ttd_plan(npairs, shape[k], a[k], b[k], a[k + 1], b[k + 1]);
      s += pl.nch * pl.rxo * pl.ryo;
    }
    p_max = std::max(p_max, s);
  }
  double* F = f_total > 0 ? ar.template take<double>((size_t)f_total) : nullptr;
  double* part = ar.template take<double>((size_t)p_max);
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_dot: workspace too small (need %zu bytes)", ar.off);

  for (int k = 0; k < ndim; ++k) {
    const bool last = k + 1 == ndim;
    int64_t p_off = 0, f_off = 0;  // this pair's partials and F_k
    for (int g0 = 0; g0 < npairs; g0 += TTD_GROUP) {
      const int gn = std::min(TTD_GROUP, npairs - g0);
      TtdTable<T> tab[2];  // [generic, tensor cores]
      int64_t items[2] = {0, 0};
      TtdReduceTable red;
      red.np = gn, red.part = part, red.F = last ? nullptr : F, red.out = out + g0;
      for (int s = 0; s < 2; ++s) tab[s].np = 0, tab[s].n = shape[k], tab[s].F = k == 0 ? nullptr : F, tab[s].part = part;
      for (int q = 0; q < gn; ++q) {
        const int p = g0 + q;
        const int32_t *a = ranks_a + p * R, *b = ranks_b + p * R;
        const TtdPlan pl = ttd_plan(npairs, shape[k], a[k], b[k], a[k + 1], b[k + 1]);
        const int s = pl.path == TTD_PATH_TC ? 1 : 0;
        TtdPair<T>& e = tab[s].p[tab[s].np++];
        e.X = pl.swap ? cb[(int64_t)p * ndim + k] : ca[(int64_t)p * ndim + k];
        e.Y = pl.swap ? ca[(int64_t)p * ndim + k] : cb[(int64_t)p * ndim + k];
        e.rx = (int)pl.rx, e.ry = (int)pl.ry, e.rxo = (int)pl.rxo, e.ryo = (int)pl.ryo;
        e.swap = pl.swap, e.nch = (int)pl.nch, e.len = pl.len, e.tn = (int)pl.tn;
        e.item0 = items[s];
        e.f_off = f_off;
        e.p_off = p_off;
        items[s] += pl.nch * pl.tiles;
        red.end[q] = (q ? red.end[q - 1] : 0) + (int64_t)a[k + 1] * b[k + 1];
        red.p_off[q] = p_off, red.f_off[q] = f_off;
        red.rao[q] = a[k + 1], red.rbo[q] = b[k + 1], red.nch[q] = (int)pl.nch, red.swap[q] = pl.swap;
        p_off += pl.nch * pl.rxo * pl.ryo;
        int64_t fm = 0;
        for (int j = 1; j < ndim; ++j) fm = std::max(fm, (int64_t)a[j] * b[j]);
        f_off += fm;
      }
      TNB_TRY(ttd_launch_mode<T>(true, tab[1], items[1], st));
      TNB_TRY(ttd_launch_mode<T>(false, tab[0], items[0], st));
      ttd_reduce_kernel<<<grid_for(red.end[gn - 1]), 256, 0, st>>>(red);
      TNB_LAUNCH_CHECK();
    }
  }
  return TNB_OK;
}

}  // namespace tnb
