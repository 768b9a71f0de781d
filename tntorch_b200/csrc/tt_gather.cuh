// Entries of tensor trains at many multi-indices (tnb_tt_gather): for each train t and point p, over the mode range
// [first, last),
//   out[t][a][p][b] = (G_first[:, i_p0, :] G_{first+1}[:, i_p1, :] ... G_{last-1}[:, i_p(M-1), :])[a, b],   M = last - first.
// Nothing is formed but the running state of each point: rows (p, a), a < r_first, of r_k columns.
//
// Two paths, chosen by the shapes and P only (ttg_path):
//   F (fused)   one launch per train: one CTA per point keeps its r_first x r_k state in shared memory and walks every
//               mode, reading each core slice through L1 / L2.  For latency-sized calls (a single entry, cross
//               validation sets).
//   G (grouped) mode by mode.  The first mode only gathers G_first[a, i_p, :] into the state.  Before every later mode a
//               counting sort (histogram, one-CTA exclusive scan, scatter) groups the state rows by that mode's index
//               and writes a tile list of (index value, first row, row count), tiles of at most TTG_T rows that never
//               cross an index value.  The step kernel then stages the slice G_k[:, i, :] once per tile and multiplies
//               the tile's gathered rows by it, writing the new rows at their own row ids in the other state buffer.
//               Inside the envelope of ttg_mode_path a step runs on the tensor cores: fp64 on mma.sync m16n8k16 .f64
//               (dmma_16816 of tt_dot.cuh), fp32 on 3xTF32 mma.sync m16n8k8 with operands split hi / lo as they are
//               staged, as tt_multiply.cuh does.  Everything else runs the same tiles on the CUDA cores.
//
// A row's value depends only on its indices, the cores and each mode's path: every output row is its own chain of
// products and sums in a fixed order, whatever other rows share its tile.  So a call is bitwise reproducible, and a
// shuffled index set gives the shuffled outputs, although the scatter orders rows inside a bucket by atomics.
// An index outside [0, I_k) is never used to address a core: it gives that point NaN.
#pragma once
#include <algorithm>

#include "common.cuh"
#include "gram_tc.cuh"
#include "expand_tc.cuh"
#include "small_kernels.cuh"
#include "tt_dot.cuh"

namespace tnb {

// ---------------------------------------------------------------------------------------------
// The choosers
// ---------------------------------------------------------------------------------------------
constexpr int TTG_TC_MIN_R = 16;             // below one k16 step most of every DMMA would multiply padding zeros
constexpr int TTG_TC_MAX_R = 256;            // the rank envelope of the library's other tensor-core kernels
constexpr int64_t TTG_FUSED_MAX_ROWS = 4096;  // above this P r_first one CTA per point re-reads each slice P / I_k
                                              // times from L2, where the grouped path reads it once per tile
constexpr int64_t TTG_FUSED_MAX_STATE = 2048;  // r_first x max r: two fp64 state buffers in 32 KB of the 48 KB default
constexpr int TTG_FUSED_MAX_MODES = 64;      // the fused kernel's parameter table holds 64 modes
constexpr int TTG_T = 64;                    // state rows per tile
constexpr int TTG_BN = 64;                   // output columns per step CTA
constexpr int TTG_BK = 32;                   // state columns staged per barrier

enum TtgPath { TTG_PATH_FUSED = 0, TTG_PATH_GROUPED = 1 };
enum TtgModePath {
  TTG_MODE_TC = 0,
  TTG_MODE_RANK_MIN = 1,  // r_k or r_{k+1} below TTG_TC_MIN_R (always the boundary modes of a full range)
  TTG_MODE_RANK_MAX = 2,  // r_k or r_{k+1} above TTG_TC_MAX_R
};

// The largest state width of train `r` (its ranks[first .. last]): columns r_{k+1} of every mode but the last, which
// writes the output.
inline int64_t ttg_state_cols(const int32_t* r, int first, int last) {
  int64_t m = 0;
  for (int k = first + 1; k < last; ++k) m = std::max<int64_t>(m, r[k]);
  return m;
}

// F or G for a call: the fused path when every train's rows fit TTG_FUSED_MAX_ROWS, its state fits shared memory and
// the range fits the parameter table.
inline int ttg_path(int ntrains, int ndim, const int32_t* ranks, int first, int last, int64_t npoints) {
  if (last - first > TTG_FUSED_MAX_MODES) return TTG_PATH_GROUPED;
  for (int t = 0; t < ntrains; ++t) {
    const int32_t* r = ranks + (int64_t)t * (ndim + 1);
    int64_t w = r[last];
    for (int k = first + 1; k < last; ++k) w = std::max<int64_t>(w, r[k]);
    if (npoints * r[first] > TTG_FUSED_MAX_ROWS || (int64_t)r[first] * w > TTG_FUSED_MAX_STATE) return TTG_PATH_GROUPED;
  }
  return TTG_PATH_FUSED;
}

// The path of one grouped step (a mode after the first): the state's r_k columns times the slice's r_{k+1}.
inline int ttg_mode_path(int64_t rk, int64_t rk1) {
  if (std::max(rk, rk1) > TTG_TC_MAX_R) return TTG_MODE_RANK_MAX;
  if (std::min(rk, rk1) < TTG_TC_MIN_R) return TTG_MODE_RANK_MIN;
  return TTG_MODE_TC;
}

// Tiles of one grouped step: each nonempty bucket (the I_k index values and one for out-of-range indices) ends at most
// one partial tile.
inline int64_t ttg_tile_bound(int64_t rows, int64_t n) { return ceil_div<int64_t>(rows, TTG_T) + n + 1; }

// ---------------------------------------------------------------------------------------------
// Fused path: one CTA per point, the state of its r_first rows in shared memory
// ---------------------------------------------------------------------------------------------
template <typename T>
struct TtgFusedTable {
  const T* core[TTG_FUSED_MAX_MODES];
  int64_t n[TTG_FUSED_MAX_MODES];
  int r[TTG_FUSED_MAX_MODES + 1];
  int m;            // modes in the range
};

constexpr int TTG_FUSED_THREADS = 128;

template <typename T>
__global__ void __launch_bounds__(TTG_FUSED_THREADS) ttg_fused_kernel(const TtgFusedTable<T> tab, const int64_t* idx,
                                                                      int64_t P, int wmax, T* out) {
  extern __shared__ __align__(16) unsigned char ttg_fsmem[];
  T* s0 = reinterpret_cast<T*>(ttg_fsmem);
  T* s1 = s0 + (int64_t)tab.r[0] * wmax;
  const int64_t p = blockIdx.x;
  const int M = tab.m, ra = tab.r[0];
  const int64_t* ip = idx + p * M;
  bool bad = false;
  for (int k = 0; k < M; ++k) bad |= ip[k] < 0 || ip[k] >= tab.n[k];
  if (bad) {
    const int rl = tab.r[M];
    for (int e = threadIdx.x; e < ra * rl; e += blockDim.x)
      out[((int64_t)(e / rl) * P + p) * rl + e % rl] = (T)NAN;
    return;
  }
  for (int k = 0; k < M; ++k) {
    const int r0 = tab.r[k], r1 = tab.r[k + 1];
    const int64_t i = ip[k], n = tab.n[k];
    const T* G = tab.core[k];
    const bool lastk = k + 1 == M;
    for (int e = threadIdx.x; e < ra * r1; e += blockDim.x) {
      const int a = e / r1, c = e % r1;
      T s;
      if (k == 0) {
        s = G[((int64_t)a * n + i) * r1 + c];
      } else {
        s = 0;
        for (int b = 0; b < r0; ++b) s = fma(s0[a * wmax + b], G[((int64_t)b * n + i) * r1 + c], s);
      }
      if (lastk)
        out[((int64_t)a * P + p) * r1 + c] = s;
      else
        s1[a * wmax + c] = s;
    }
    __syncthreads();
    T* tmp = s0;
    s0 = s1, s1 = tmp;
  }
}

// ---------------------------------------------------------------------------------------------
// Grouped path: indices, counting sort, tile list
// ---------------------------------------------------------------------------------------------
// idx [P][M] int64 -> idx32 [M][P] (a value outside int32 becomes -1, out of every mode's range); zeroes the counts.
__global__ void ttg_narrow_kernel(const int64_t* __restrict__ idx, int64_t P, int M, int* __restrict__ idx32,
                                  int* __restrict__ counts, int64_t ncounts) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < P * M; e += stride) {
    const int64_t p = e / M, m = e % M;
    const int64_t v = idx[e];
    idx32[m * P + p] = (v >= 0 && v <= INT32_MAX) ? (int)v : -1;
  }
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < ncounts; e += stride) counts[e] = 0;
}

// The bucket of an index of a mode of size n: the value, or n when it is out of range.
__device__ __forceinline__ int ttg_bucket(int v, int n) { return (v < 0 || v >= n) ? n : v; }

// counts[b] += r_first for each point in bucket b
__global__ void ttg_hist_kernel(const int* __restrict__ ix, int64_t P, int n, int ra, int* __restrict__ counts) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(counts + ttg_bucket(ix[p], n), ra);
}

// One CTA: over the n + 1 buckets, cursor[b] = first row of bucket b (exclusive scan of counts), the tile list
// (value, first row, row count) in bucket order, *ntiles; counts are zeroed for the next step.
constexpr int TTG_SCAN_THREADS = 1024;
__global__ void __launch_bounds__(TTG_SCAN_THREADS) ttg_scan_kernel(int* __restrict__ counts, int n,
                                                                    int* __restrict__ cursor, int* __restrict__ tiles,
                                                                    int* __restrict__ ntiles) {
  __shared__ int s_rows[TTG_SCAN_THREADS], s_tiles[TTG_SCAN_THREADS], s_cnt[TTG_SCAN_THREADS];
  __shared__ int s_carry[2];
  if (threadIdx.x == 0) s_carry[0] = 0, s_carry[1] = 0;
  __syncthreads();
  const int nb = n + 1;
  for (int b0 = 0; b0 < nb; b0 += TTG_SCAN_THREADS) {
    const int b = b0 + threadIdx.x;
    const int c = b < nb ? counts[b] : 0;
    if (b < nb) counts[b] = 0;
    s_cnt[threadIdx.x] = c;
    s_rows[threadIdx.x] = c;
    s_tiles[threadIdx.x] = (c + TTG_T - 1) / TTG_T;
    __syncthreads();
    for (int off = 1; off < TTG_SCAN_THREADS; off <<= 1) {  // inclusive Hillis-Steele scans
      const int x = threadIdx.x >= off ? s_rows[threadIdx.x - off] : 0;
      const int y = threadIdx.x >= off ? s_tiles[threadIdx.x - off] : 0;
      __syncthreads();
      s_rows[threadIdx.x] += x, s_tiles[threadIdx.x] += y;
      __syncthreads();
    }
    const int row0 = s_carry[0], tile0 = s_carry[1];
    if (b < nb) cursor[b] = row0 + s_rows[threadIdx.x] - c;
    const int chunk_tiles = s_tiles[TTG_SCAN_THREADS - 1];
    // tile j of the chunk: its bucket is the first whose inclusive tile count exceeds j (binary search)
    for (int j = threadIdx.x; j < chunk_tiles; j += TTG_SCAN_THREADS) {
      int lo = 0, hi = TTG_SCAN_THREADS - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_tiles[mid] > j) hi = mid; else lo = mid + 1;
      }
      const int tb = lo, first_tile = s_tiles[tb] - (s_cnt[tb] + TTG_T - 1) / TTG_T;
      const int q = j - first_tile;
      const int start = row0 + s_rows[tb] - s_cnt[tb] + q * TTG_T;
      int* e = tiles + 3 * (int64_t)(tile0 + j);
      e[0] = b0 + tb, e[1] = start, e[2] = min(TTG_T, s_cnt[tb] - q * TTG_T);
    }
    __syncthreads();
    if (threadIdx.x == 0) s_carry[0] = row0 + s_rows[TTG_SCAN_THREADS - 1], s_carry[1] = tile0 + chunk_tiles;
    __syncthreads();
  }
  if (threadIdx.x == 0) *ntiles = s_carry[1];
}

// perm[cursor[b] ...] = the rows p r_first + a of the points of bucket b
__global__ void ttg_scatter_kernel(const int* __restrict__ ix, int64_t P, int n, int ra, int* __restrict__ cursor,
                                   int* __restrict__ perm) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x) {
    const int pos = atomicAdd(cursor + ttg_bucket(ix[p], n), ra);
    for (int a = 0; a < ra; ++a) perm[pos + a] = (int)(p * ra + a);
  }
}

// The first mode: state[p r_first + a][c] = G[a, i_p, c] (or straight into out when the range has one mode).
template <typename T>
__global__ void ttg_init_kernel(const T* __restrict__ G, int64_t n, int ra, int r1, const int* __restrict__ ix,
                                int64_t P, T* __restrict__ state, T* __restrict__ out) {
  const int64_t total = P * ra * r1;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / r1, c = e % r1, p = row / ra, a = row % ra;
    const int v = ix[p];
    const T s = (v < 0 || v >= n) ? (T)NAN : G[((int64_t)a * n + v) * r1 + c];
    if (out)
      out[(a * P + p) * r1 + c] = s;
    else
      state[e] = s;
  }
}

// ---------------------------------------------------------------------------------------------
// Grouped step: tile (value i, rows) x column block; new[row][c] = sum_b S[row][b] G[b, i, c]
// ---------------------------------------------------------------------------------------------
constexpr int TTG_THREADS = 256;
constexpr int TTG_SS = TTG_BK + 4;  // fp64 row stride of the staged state: 4 mod 16 doubles (see tt_dot.cuh)
constexpr int TTG_SG = TTG_BN + 4;

struct TtgStep {
  int64_t n;         // mode size
  int64_t P;
  int rk, rk1, ra;   // state columns, new columns, r_first
  const int* tiles;
  const int* ntiles;
  const int* perm;
};

// where row `rid` column c of the step's result goes: the next state, or out[a][p][c] after the last mode
template <typename T>
__device__ __forceinline__ T* ttg_dst(const TtgStep& s, T* nxt, T* out, int rid, int c) {
  if (out) {
    const int64_t p = rid / s.ra, a = rid % s.ra;
    return out + (a * s.P + p) * s.rk1 + c;
  }
  return nxt + (int64_t)rid * s.rk1 + c;
}

// Row `j` of a step's bucket order: perm holds row ids, or with PPERM point ids (the backward's stable order), row j
// being row j % r_first of the point at j / r_first.
template <bool PPERM>
__device__ __forceinline__ int ttg_rid(const TtgStep& s, int j) {
  if constexpr (PPERM) return s.perm[j / s.ra] * s.ra + j % s.ra;
  return s.perm[j];
}

// Slice entry (k, c) of the step's right operand: G[k, i, c], or with TRANS (the backward's reverse step, whose rk
// columns are r_{k+1} and rk1 columns r_k) G[c, i, k], the slice transposed.
template <bool TRANS, typename T>
__device__ __forceinline__ T ttg_slice(const TtgStep& s, const T* G, int i, int k, int c) {
  if constexpr (TRANS) return G[((int64_t)c * s.n + i) * s.rk + k];
  return G[((int64_t)k * s.n + i) * s.rk1 + c];
}

// The step on CUDA cores: each thread 4 rows x 4 columns (rows ty + 16 u, columns tx + 16 v).
template <typename T, bool PPERM = false, bool TRANS = false>
__global__ void __launch_bounds__(TTG_THREADS) ttg_step_generic_kernel(const TtgStep s, const T* __restrict__ G,
                                                                       const T* __restrict__ cur, T* nxt, T* out) {
  __shared__ T Ss[TTG_T][TTG_BK + 1];
  __shared__ T Gs[TTG_BK][TTG_BN + 1];
  __shared__ int rids[TTG_T];
  const int tile = blockIdx.x;
  if (tile >= *s.ntiles) return;
  const int* te = s.tiles + 3 * (int64_t)tile;
  const int i = te[0], row0 = te[1], cnt = te[2];
  const int c0 = blockIdx.y * TTG_BN, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  if (tid < TTG_T) rids[tid] = tid < cnt ? ttg_rid<PPERM>(s, row0 + tid) : 0;
  __syncthreads();
  if (i >= s.n) {  // out-of-range index: NaN
    for (int e = tid; e < cnt * TTG_BN; e += TTG_THREADS) {
      const int r = e / TTG_BN, c = c0 + e % TTG_BN;
      if (c < s.rk1) *ttg_dst(s, nxt, out, rids[r], c) = (T)NAN;
    }
    return;
  }
  T acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) acc[u][v] = 0;
  for (int k0 = 0; k0 < s.rk; k0 += TTG_BK) {
    for (int e = tid; e < TTG_T * TTG_BK; e += TTG_THREADS) {
      const int r = e / TTG_BK, kk = e % TTG_BK, k = k0 + kk;
      Ss[r][kk] = (r < cnt && k < s.rk) ? cur[(int64_t)rids[r] * s.rk + k] : (T)0;
    }
    for (int e = tid; e < TTG_BK * TTG_BN; e += TTG_THREADS) {
      // transposed, consecutive threads walk k, the slice's contiguous index
      const int kk = TRANS ? e % TTG_BK : e / TTG_BN, cc = TRANS ? e / TTG_BK : e % TTG_BN, k = k0 + kk, c = c0 + cc;
      Gs[kk][cc] = (k < s.rk && c < s.rk1) ? ttg_slice<TRANS>(s, G, i, k, c) : (T)0;
    }
    __syncthreads();
    const int kl = min(TTG_BK, s.rk - k0);
    for (int kk = 0; kk < kl; ++kk) {
      T gv[4];
#pragma unroll
      for (int v = 0; v < 4; ++v) gv[v] = Gs[kk][tx + 16 * v];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const T sv = Ss[ty + 16 * u][kk];
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fma(sv, gv[v], acc[u][v]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int r = ty + 16 * u;
    if (r >= cnt) continue;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int c = c0 + tx + 16 * v;
      if (c < s.rk1) *ttg_dst(s, nxt, out, rids[r], c) = acc[u][v];
    }
  }
}

// One staged 64 x 32 by 32 x 64 block product on the tensor cores, accumulated into a warp's 16 x 32 share of the
// 64 x 64 block: rows mrow .. + 16, n8 tiles at ncol .. + 32 (fp64 k16 DMMA steps; fp32 k8 3xTF32 steps on hi / lo).
template <typename T, typename Acc>
__device__ __forceinline__ void ttg_mma_block(Acc (&acc)[4][4], const T (*Ss)[TTG_T][TTG_SS], const T (*Gs)[TTG_BK][TTG_SG],
                                              int mrow, int ncol, int g, int t) {
  constexpr bool F64 = sizeof(T) == 8;
  if constexpr (F64) {
#pragma unroll
    for (int ks = 0; ks < TTG_BK; ks += 16) {
      double a[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) a[q] = Ss[0][mrow + g + 8 * (q & 1)][ks + t + 4 * (q >> 1)];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        double b[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) b[q] = Gs[0][ks + t + 4 * q][ncol + 8 * j + g];
        dmma_16816(acc[j], a, b);
      }
    }
  } else {
#pragma unroll
    for (int ks = 0; ks < TTG_BK; ks += 8) {
      uint32_t ah[4], al[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int r = mrow + g + 8 * (q & 1), k = ks + t + 4 * (q >> 1);
        ah[q] = __float_as_uint(Ss[0][r][k]), al[q] = __float_as_uint(Ss[1][r][k]);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int c = ncol + 8 * j + g;
        const uint32_t bh0 = __float_as_uint(Gs[0][ks + t][c]), bh1 = __float_as_uint(Gs[0][ks + t + 4][c]);
        const uint32_t bl0 = __float_as_uint(Gs[1][ks + t][c]), bl1 = __float_as_uint(Gs[1][ks + t + 4][c]);
        mma_tf32(acc[j], ah[0], ah[1], ah[2], ah[3], bl0, bl1);  // S_hi G_lo
        mma_tf32(acc[j], al[0], al[1], al[2], al[3], bh0, bh1);  // S_lo G_hi
        mma_tf32(acc[j], ah[0], ah[1], ah[2], ah[3], bh0, bh1);  // S_hi G_hi
      }
    }
  }
}

// The step on the tensor cores.  Eight warps over the 64 x 64 output block: warp w takes rows 16 (w & 3) .. + 16 and
// n8 tiles 4 (w >> 2) .. + 4.  fp64: k16 DMMA steps on the staged operands.  fp32: k8 3xTF32 steps, each operand
// stored hi / lo (rounded to nearest) as it is staged.
template <typename T, bool PPERM = false, bool TRANS = false>
__global__ void __launch_bounds__(TTG_THREADS) ttg_step_tc_kernel(const TtgStep s, const T* __restrict__ G,
                                                                  const T* __restrict__ cur, T* nxt, T* out) {
  constexpr bool F64 = sizeof(T) == 8;
  constexpr int PLANES = F64 ? 1 : 2;  // hi / lo for 3xTF32
  __shared__ T Ss[PLANES][TTG_T][TTG_SS];
  __shared__ T Gs[PLANES][TTG_BK][TTG_SG];
  __shared__ int rids[TTG_T];
  const int tile = blockIdx.x;
  if (tile >= *s.ntiles) return;
  const int* te = s.tiles + 3 * (int64_t)tile;
  const int i = te[0], row0 = te[1], cnt = te[2];
  const int c0 = blockIdx.y * TTG_BN, tid = threadIdx.x;
  const int w = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int mrow = 16 * (w & 3), ncol = 32 * (w >> 2);
  if (tid < TTG_T) rids[tid] = tid < cnt ? ttg_rid<PPERM>(s, row0 + tid) : 0;
  __syncthreads();
  if (i >= s.n) {
    for (int e = tid; e < cnt * TTG_BN; e += TTG_THREADS) {
      const int r = e / TTG_BN, c = c0 + e % TTG_BN;
      if (c < s.rk1) *ttg_dst(s, nxt, out, rids[r], c) = (T)NAN;
    }
    return;
  }
  using Acc = typename std::conditional<F64, double, float>::type;
  Acc acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0;
  for (int k0 = 0; k0 < s.rk; k0 += TTG_BK) {
    for (int e = tid; e < TTG_T * TTG_BK; e += TTG_THREADS) {
      const int r = e / TTG_BK, kk = e % TTG_BK, k = k0 + kk;
      const T v = (r < cnt && k < s.rk) ? cur[(int64_t)rids[r] * s.rk + k] : (T)0;
      if constexpr (F64) {
        Ss[0][r][kk] = v;
      } else {
        const float hi = ex_tf32_rn(v);
        Ss[0][r][kk] = hi, Ss[1][r][kk] = ex_tf32_rn(v - hi);
      }
    }
    for (int e = tid; e < TTG_BK * TTG_BN; e += TTG_THREADS) {
      const int kk = TRANS ? e % TTG_BK : e / TTG_BN, cc = TRANS ? e / TTG_BK : e % TTG_BN, k = k0 + kk, c = c0 + cc;
      const T v = (k < s.rk && c < s.rk1) ? ttg_slice<TRANS>(s, G, i, k, c) : (T)0;
      if constexpr (F64) {
        Gs[0][kk][cc] = v;
      } else {
        const float hi = ex_tf32_rn(v);
        Gs[0][kk][cc] = hi, Gs[1][kk][cc] = ex_tf32_rn(v - hi);
      }
    }
    __syncthreads();
    ttg_mma_block<T>(acc, Ss, Gs, mrow, ncol, g, t);
    __syncthreads();
  }
  // c fragment: e at row g + 8 (e >> 1), column 2 t + (e & 1) of each n8 tile
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int r = mrow + g + 8 * (e >> 1), c = c0 + ncol + 8 * j + 2 * t + (e & 1);
      if (r < cnt && c < s.rk1) *ttg_dst(s, nxt, out, rids[r], c) = (T)acc[j][e];
    }
}

// ---------------------------------------------------------------------------------------------
// The driver
// ---------------------------------------------------------------------------------------------
constexpr int TTG_MAX_D = 1024;
constexpr int64_t TTG_MAX_ELEMS = (int64_t)1 << 46;  // of every core, state and output

// ntrains >= 1, ndim >= 1, 0 <= first < last <= ndim, npoints >= 1, mode sizes and ranks >= 1 (TNB_ERR_INVALID);
// ndim <= TTG_MAX_D, mode sizes below 2^31 - 1, ranks below 2^21 (the step grid's 65535 column blocks of 64), P r_first
// below 2^31 rows, every core, state and output within TTG_MAX_ELEMS (TNB_ERR_UNSUPPORTED).
inline int ttg_check_dims(int ntrains, int ndim, const int64_t* shape, const int32_t* ranks, int first, int last,
                          int64_t npoints) {
  if (ntrains < 1) return fail(TNB_ERR_INVALID, "tt_gather: ntrains=%d must be >= 1", ntrains);
  if (ndim < 1) return fail(TNB_ERR_INVALID, "tt_gather: ndim=%d must be >= 1", ndim);
  if (first < 0 || last > ndim || first >= last)
    return fail(TNB_ERR_INVALID, "tt_gather: mode range [%d, %d) is not inside [0, %d)", first, last, ndim);
  if (npoints < 1) return fail(TNB_ERR_INVALID, "tt_gather: npoints=%lld must be >= 1", (long long)npoints);
  if (ndim > TTG_MAX_D) return fail(TNB_ERR_UNSUPPORTED, "tt_gather: ndim=%d above %d", ndim, TTG_MAX_D);
  for (int k = 0; k < ndim; ++k) {
    if (shape[k] < 1) return fail(TNB_ERR_INVALID, "tt_gather: mode sizes must be >= 1");
    if (shape[k] >= INT32_MAX) return fail(TNB_ERR_UNSUPPORTED, "tt_gather: mode size %lld too large", (long long)shape[k]);
  }
  const unsigned __int128 lim = (unsigned __int128)TTG_MAX_ELEMS;
  for (int t = 0; t < ntrains; ++t) {
    const int32_t* r = ranks + (int64_t)t * (ndim + 1);
    for (int k = 0; k <= ndim; ++k) {
      if (r[k] < 1) return fail(TNB_ERR_INVALID, "tt_gather: train %d: ranks must be >= 1", t);
      if (r[k] >= (1 << 21)) return fail(TNB_ERR_UNSUPPORTED, "tt_gather: train %d: rank %d too large", t, (int)r[k]);
    }
    for (int k = 0; k < ndim; ++k)
      if ((unsigned __int128)r[k] * shape[k] * r[k + 1] > lim)
        return fail(TNB_ERR_UNSUPPORTED, "tt_gather: train %d: core %d too large", t, k);
    const unsigned __int128 rows = (unsigned __int128)npoints * r[first];
    if (rows >= (unsigned __int128)INT32_MAX)
      return fail(TNB_ERR_UNSUPPORTED, "tt_gather: train %d: %lld points x rank %d above 2^31 rows", t,
                  (long long)npoints, (int)r[first]);
    if (rows * ttg_state_cols(r, first, last) > lim || rows * r[last] > lim)
      return fail(TNB_ERR_UNSUPPORTED, "tt_gather: train %d: state or output too large", t);
  }
  return TNB_OK;
}

// T: float or double.  Workspace (grouped path only): the narrowed indices [M][P], the counts, cursors and tile list of
// one step, one permutation, and two state buffers of P r_first max r_k, all sized by the largest train and reused by
// every train and mode.  The fused path takes none.
template <typename T, class ArenaT>
inline int tt_gather_impl(ArenaT& ar, bool dry, const T* const* cores, int ntrains, int ndim, const int64_t* shape,
                          const int32_t* ranks, int first, int last, const int64_t* idx, int64_t P, T* out,
                          cudaStream_t st) {
  const int M = last - first;
  const int64_t R = ndim + 1;
  const int path = ttg_path(ntrains, ndim, ranks, first, last, P);
  if (path == TTG_PATH_FUSED) {
    if (dry) return TNB_OK;
    int64_t off = 0;
    for (int t = 0; t < ntrains; ++t) {
      const int32_t* r = ranks + t * R;
      TtgFusedTable<T> tab;
      tab.m = M;
      int wmax = r[last];
      for (int k = 0; k < M; ++k) {
        tab.core[k] = cores[t * ndim + first + k];
        tab.n[k] = shape[first + k];
        tab.r[k] = r[first + k];
        if (k > 0) wmax = std::max(wmax, (int)r[first + k]);
      }
      tab.r[M] = r[last];
      const int smem = (int)(2 * (int64_t)r[first] * wmax * sizeof(T));
      ttg_fused_kernel<T><<<(unsigned)P, TTG_FUSED_THREADS, smem, st>>>(tab, idx, P, wmax, out + off);
      TNB_LAUNCH_CHECK();
      off += P * r[first] * r[last];
    }
    return TNB_OK;
  }

  int64_t nmax = 0, rows_max = 0, state_max = 0, tiles_max = 0;
  for (int k = first; k < last; ++k) nmax = std::max(nmax, shape[k]);
  for (int t = 0; t < ntrains; ++t) {
    const int32_t* r = ranks + t * R;
    const int64_t rows = P * r[first];
    rows_max = std::max(rows_max, rows);
    state_max = std::max(state_max, rows * ttg_state_cols(r, first, last));
    for (int k = first + 1; k < last; ++k) tiles_max = std::max(tiles_max, ttg_tile_bound(rows, shape[k]));
  }
  int* idx32 = ar.template take<int>((size_t)(P * M));
  int* counts = ar.template take<int>((size_t)(nmax + 1));
  int* cursor = M > 1 ? ar.template take<int>((size_t)(nmax + 1)) : nullptr;
  int* tiles = M > 1 ? ar.template take<int>((size_t)(3 * tiles_max + 1)) : nullptr;
  int* perm = M > 1 ? ar.template take<int>((size_t)rows_max) : nullptr;
  T* sbuf[2] = {nullptr, nullptr};
  if (state_max > 0) sbuf[0] = ar.template take<T>((size_t)state_max), sbuf[1] = ar.template take<T>((size_t)state_max);
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_gather: workspace too small (need %zu bytes)", ar.off);
  int* ntiles = tiles ? tiles + 3 * tiles_max : nullptr;

  ttg_narrow_kernel<<<grid_for(std::max(P * M, nmax + 1)), 256, 0, st>>>(idx, P, M, idx32, counts, nmax + 1);
  TNB_LAUNCH_CHECK();
  int64_t off = 0;
  for (int t = 0; t < ntrains; ++t) {
    const int32_t* r = ranks + t * R;
    const int ra = r[first];
    const int64_t rows = P * ra;
    T* o = out + off;
    ttg_init_kernel<T><<<grid_for(rows * r[first + 1]), 256, 0, st>>>(cores[t * ndim + first], shape[first], ra,
                                                                      r[first + 1], idx32, P, sbuf[0],
                                                                      M == 1 ? o : nullptr);
    TNB_LAUNCH_CHECK();
    int cur = 0;
    for (int k = first + 1; k < last; ++k) {
      const int* ix = idx32 + (int64_t)(k - first) * P;
      const int n = (int)shape[k];
      ttg_hist_kernel<<<grid_for(P), 256, 0, st>>>(ix, P, n, ra, counts);
      TNB_LAUNCH_CHECK();
      ttg_scan_kernel<<<1, TTG_SCAN_THREADS, 0, st>>>(counts, n, cursor, tiles, ntiles);
      TNB_LAUNCH_CHECK();
      ttg_scatter_kernel<<<grid_for(P), 256, 0, st>>>(ix, P, n, ra, cursor, perm);
      TNB_LAUNCH_CHECK();
      TtgStep s;
      s.n = n, s.P = P, s.rk = r[k], s.rk1 = r[k + 1], s.ra = ra, s.tiles = tiles, s.ntiles = ntiles, s.perm = perm;
      const bool lastk = k + 1 == last;
      const dim3 grid((unsigned)ttg_tile_bound(rows, n), (unsigned)ceil_div<int64_t>(r[k + 1], TTG_BN));
      if (ttg_mode_path(r[k], r[k + 1]) == TTG_MODE_TC)
        ttg_step_tc_kernel<T><<<grid, TTG_THREADS, 0, st>>>(s, cores[t * ndim + k], sbuf[cur], sbuf[cur ^ 1],
                                                            lastk ? o : nullptr);
      else
        ttg_step_generic_kernel<T><<<grid, TTG_THREADS, 0, st>>>(s, cores[t * ndim + k], sbuf[cur], sbuf[cur ^ 1],
                                                                 lastk ? o : nullptr);
      TNB_LAUNCH_CHECK();
      cur ^= 1;
    }
    off += rows * r[last];
  }
  return TNB_OK;
}

}  // namespace tnb
