// The gradient of tnb_tt_gather (tnb_tt_gather_grad): for each train t, from grad_out[t][a][p][b] = d loss / d out[t][a][p][b],
//   dG_k[:, i, :] = sum over the points p with i_pk = i of L_k[p]^T W_k[p],   k in [first, last),
// with L_k[p] = G_first[:, i_p0, :] ... G_{k-1}[:, i_p(k-1-first), :] (r_first x r_k; the identity for k = first) and
// W_k[p] = grad_out[p] G_{last-1}[:, i_p(M-1), :]^T ... G_{k+1}[:, i_p(k+1-first), :]^T (r_first x r_{k+1}).
// Rows are (p, a), a < r_first, as in the forward's grouped path.
//
// Once per call, for every mode of the range: a stable counting sort of the points by that mode's index (an LSD pass
// over each 8-bit digit of the bucket: per-block digit histograms, one digit-major exclusive scan, a scatter with
// block-local stable ranks), so the order of a bucket's points depends on idx alone, never on how atomics resolve.
// Per train:
//   plans   per mode, the tile list of the steps (TTG_T rows, as the forward's) and the chunk list of the reduction
//           (ttgg_chunk_rows rows, from the shapes and P only), both over the stable order;
//   forward ttg_init_kernel and the forward step kernels (stable order) recompute and keep every L_k;
//   reverse W_{last-1} is grad_out; then for k = last-1 down to first: the reduction dG_k = sum L_k^T W_k, a
//           segmented GEMM over the rows of each bucket (an identity L_first makes the first mode a segmented sum of
//           W rows), and, above first, W_{k-1} = W_k G_k[:, i, :]^T, the forward step with the slice staged transposed.
// Both run on the tensor cores inside the envelope of ttg_mode_path (fp64 mma.sync m16n8k16, fp32 3xTF32), on CUDA-core
// tiles outside it.  A bucket of one chunk writes its slice directly; a longer one writes per-chunk partials that
// ttgg_combine_kernel sums in chunk order (in fp64 for fp32 cores) and rounds once.  Slices no point reaches stay zero.
// No atomics touch a value, so a call is bitwise reproducible.  A point with any index outside its mode is sent to the
// out-of-range bucket of every mode: it takes no part in any gradient and never addresses a core.
#pragma once
#include <algorithm>
#include <vector>

#include "tt_gather.cuh"

namespace tnb {

constexpr int TTGG_SORT_THREADS = 256;
constexpr int TTGG_SORT_ITEMS = 16;
constexpr int TTGG_SORT_CHUNK = TTGG_SORT_THREADS * TTGG_SORT_ITEMS;  // points per sort block
constexpr int TTGG_DIGITS = 256;
constexpr int64_t TTGG_CHUNK_MIN = 256;      // rows per reduction chunk, at least
constexpr int64_t TTGG_CHUNK_MAX = 1 << 16;  // and at most
constexpr int64_t TTGG_CHUNK_CTAS = 1024;    // reduction CTAs a mode aims for

// 8-bit digit passes that sort the buckets 0 .. n
inline int ttgg_sort_passes(int64_t n) {
  int p = 1;
  while (p < 4 && (n >> (8 * p)) > 0) ++p;
  return p;
}
inline int64_t ttgg_sort_blocks(int64_t P) { return ceil_div<int64_t>(P, TTGG_SORT_CHUNK); }

// Rows per chunk of one mode's reduction: about TTGG_CHUNK_CTAS CTAs over the rows and the r_k x r_{k+1} output tiles.
inline int64_t ttgg_chunk_rows(int64_t rows, int64_t rk, int64_t rk1) {
  const int64_t otiles = ceil_div<int64_t>(rk, TTG_T) * ceil_div<int64_t>(rk1, TTG_BN);
  const int64_t ch = ceil_div<int64_t>(ceil_div<int64_t>(rows * otiles, TTGG_CHUNK_CTAS), TTG_BK) * TTG_BK;
  return std::min(std::max(ch, TTGG_CHUNK_MIN), TTGG_CHUNK_MAX);
}
// Chunks of one mode: each nonempty bucket ends at most one partial chunk.
inline int64_t ttgg_chunk_bound(int64_t rows, int64_t n, int64_t ch) { return ceil_div<int64_t>(rows, ch) + n + 1; }
// Partial slices of one mode: only buckets of more than one chunk take them, ceil(c / ch) < 2 c / ch each.
inline int64_t ttgg_slot_bound(int64_t rows, int64_t ch) { return rows > ch ? 2 * rows / ch : 0; }

// ---------------------------------------------------------------------------------------------
// Indices and the stable order
// ---------------------------------------------------------------------------------------------
struct TtggModes {
  int m;
  int n[TTG_MAX_D];
};

// idx [P][M] int64 -> idx32 [M][P]; every index of a point with any index outside its mode becomes -1 (the
// out-of-range bucket of every mode).  Zeroes the bucket counts.
__global__ void ttgg_narrow_kernel(const TtggModes md, const int64_t* __restrict__ idx, int64_t P,
                                   int* __restrict__ idx32, int* __restrict__ counts, int64_t ncounts) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int M = md.m;
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += stride) {
    bool bad = false;
    for (int m = 0; m < M; ++m) {
      const int64_t v = idx[p * M + m];
      bad |= v < 0 || v >= md.n[m];
    }
    for (int m = 0; m < M; ++m) idx32[m * P + p] = bad ? -1 : (int)idx[p * M + m];
  }
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < ncounts; e += stride) counts[e] = 0;
}

// points per bucket
__global__ void ttgg_count_kernel(const int* __restrict__ ix, int64_t P, int n, int* __restrict__ counts) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < P; p += (int64_t)gridDim.x * blockDim.x)
    atomicAdd(counts + ttg_bucket(ix[p], n), 1);
}

__device__ __forceinline__ int ttgg_digit(const int* ix, int p, int n, int shift) {
  return (ttg_bucket(ix[p], n) >> shift) & (TTGG_DIGITS - 1);
}

// hist[d * nblocks + block] = points of the block (TTGG_SORT_CHUNK of src, the identity when src is null) with digit d
__global__ void __launch_bounds__(TTGG_SORT_THREADS) ttgg_digit_hist_kernel(const int* __restrict__ ix,
                                                                            const int* __restrict__ src, int64_t P,
                                                                            int n, int shift, int* __restrict__ hist) {
  __shared__ int h[TTGG_DIGITS];
  h[threadIdx.x] = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * TTGG_SORT_CHUNK;
  for (int j = threadIdx.x; j < TTGG_SORT_CHUNK; j += TTGG_SORT_THREADS) {
    const int64_t q = base + j;
    if (q < P) atomicAdd(&h[ttgg_digit(ix, src ? src[q] : (int)q, n, shift)], 1);
  }
  __syncthreads();
  hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// One CTA: exclusive scan of hist[len] in place (each thread a contiguous segment, then a scan of the segment sums).
constexpr int TTGG_SCAN_THREADS = 1024;
__global__ void __launch_bounds__(TTGG_SCAN_THREADS) ttgg_digit_scan_kernel(int* __restrict__ hist, int64_t len) {
  __shared__ int s[TTGG_SCAN_THREADS];
  const int64_t seg = (len + TTGG_SCAN_THREADS - 1) / TTGG_SCAN_THREADS;
  const int64_t lo = min(len, (int64_t)threadIdx.x * seg), hi = min(len, lo + seg);
  int sum = 0;
  for (int64_t e = lo; e < hi; ++e) sum += hist[e];
  s[threadIdx.x] = sum;
  __syncthreads();
  for (int off = 1; off < TTGG_SCAN_THREADS; off <<= 1) {
    const int x = threadIdx.x >= off ? s[threadIdx.x - off] : 0;
    __syncthreads();
    s[threadIdx.x] += x;
    __syncthreads();
  }
  int run = s[threadIdx.x] - sum;
  for (int64_t e = lo; e < hi; ++e) {
    const int v = hist[e];
    hist[e] = run;
    run += v;
  }
}

// dst[hist[d][block] + stable rank] = the points of the block, in src order within each digit: a point's rank is the
// number of earlier points of the block with its digit (warp match, then the warps before it, then earlier rounds).
__global__ void __launch_bounds__(TTGG_SORT_THREADS) ttgg_digit_scatter_kernel(const int* __restrict__ ix,
                                                                               const int* __restrict__ src, int64_t P,
                                                                               int n, int shift,
                                                                               const int* __restrict__ hist,
                                                                               int* __restrict__ dst) {
  constexpr int WARPS = TTGG_SORT_THREADS / 32;
  __shared__ int run[TTGG_DIGITS];
  __shared__ int wc[WARPS][TTGG_DIGITS];
  const int tid = threadIdx.x, w = tid >> 5, lane = tid & 31;
  run[tid] = hist[(int64_t)tid * gridDim.x + blockIdx.x];
  const int64_t base = (int64_t)blockIdx.x * TTGG_SORT_CHUNK;
  for (int it = 0; it < TTGG_SORT_ITEMS; ++it) {
    const int64_t q = base + (int64_t)it * TTGG_SORT_THREADS + tid;
    const bool valid = q < P;
    const int p = valid ? (src ? src[q] : (int)q) : 0;
    const int d = valid ? ttgg_digit(ix, p, n, shift) : TTGG_DIGITS;
    for (int e = tid; e < WARPS * TTGG_DIGITS; e += TTGG_SORT_THREADS) wc[e / TTGG_DIGITS][e % TTGG_DIGITS] = 0;
    __syncthreads();
    const unsigned mask = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(mask & ((1u << lane) - 1u));
    if (valid && rank == 0) wc[w][d] = __popc(mask);
    __syncthreads();
    if (valid) {
      int pos = run[d] + rank;
      for (int v = 0; v < w; ++v) pos += wc[v][d];
      dst[pos] = p;
    }
    __syncthreads();
    int add = 0;
    for (int v = 0; v < WARPS; ++v) add += wc[v][tid];
    run[tid] += add;
    __syncthreads();
  }
}

// One CTA: from the points per bucket, the list of one mode's tiles of at most `tile` rows (r_first per point) that never
// cross a bucket, in bucket order: (value, first row, row count) and, with width 4, the first partial slot of a
// bucket of more than one tile plus the tile's place in it (-1 for a bucket of one tile); *nlist.
constexpr int TTGG_PLAN_THREADS = 1024;
__global__ void __launch_bounds__(TTGG_PLAN_THREADS) ttgg_plan_kernel(const int* __restrict__ counts, int n, int ra,
                                                                      int tile, int width, int* __restrict__ list,
                                                                      int* __restrict__ nlist) {
  __shared__ int s_rows[TTGG_PLAN_THREADS], s_tiles[TTGG_PLAN_THREADS], s_slots[TTGG_PLAN_THREADS];
  __shared__ int s_cnt[TTGG_PLAN_THREADS];
  __shared__ int s_carry[3];
  if (threadIdx.x == 0) s_carry[0] = 0, s_carry[1] = 0, s_carry[2] = 0;
  __syncthreads();
  const int nb = n + 1;
  for (int b0 = 0; b0 < nb; b0 += TTGG_PLAN_THREADS) {
    const int b = b0 + threadIdx.x;
    const int c = b < nb ? counts[b] * ra : 0;
    const int nt = (c + tile - 1) / tile;
    s_cnt[threadIdx.x] = c, s_rows[threadIdx.x] = c, s_tiles[threadIdx.x] = nt, s_slots[threadIdx.x] = nt > 1 ? nt : 0;
    __syncthreads();
    for (int off = 1; off < TTGG_PLAN_THREADS; off <<= 1) {  // inclusive Hillis-Steele scans
      const int x = threadIdx.x >= off ? s_rows[threadIdx.x - off] : 0;
      const int y = threadIdx.x >= off ? s_tiles[threadIdx.x - off] : 0;
      const int z = threadIdx.x >= off ? s_slots[threadIdx.x - off] : 0;
      __syncthreads();
      s_rows[threadIdx.x] += x, s_tiles[threadIdx.x] += y, s_slots[threadIdx.x] += z;
      __syncthreads();
    }
    const int row0 = s_carry[0], tile0 = s_carry[1], slot0 = s_carry[2];
    const int chunk_tiles = s_tiles[TTGG_PLAN_THREADS - 1];
    for (int j = threadIdx.x; j < chunk_tiles; j += TTGG_PLAN_THREADS) {
      int lo = 0, hi = TTGG_PLAN_THREADS - 1;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (s_tiles[mid] > j) hi = mid; else lo = mid + 1;
      }
      const int tb = lo, ntb = (s_cnt[tb] + tile - 1) / tile, q = j - (s_tiles[tb] - ntb);
      int* e = list + (int64_t)width * (tile0 + j);
      e[0] = b0 + tb, e[1] = row0 + s_rows[tb] - s_cnt[tb] + q * tile, e[2] = min(tile, s_cnt[tb] - q * tile);
      if (width == 4) e[3] = ntb > 1 ? slot0 + s_slots[tb] - ntb + q : -1;
    }
    __syncthreads();
    if (threadIdx.x == 0)
      s_carry[0] = row0 + s_rows[TTGG_PLAN_THREADS - 1], s_carry[1] = tile0 + chunk_tiles,
      s_carry[2] = slot0 + s_slots[TTGG_PLAN_THREADS - 1];
    __syncthreads();
  }
  if (threadIdx.x == 0) *nlist = s_carry[1];
}

// W_{last-1}[p r_first + a][c] = grad_out[a][p][c]
template <typename T>
__global__ void ttgg_load_kernel(const T* __restrict__ gout, int64_t P, int ra, int rl, T* __restrict__ W) {
  const int64_t total = P * ra * rl;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = e / rl, c = e % rl, p = row / ra, a = row % ra;
    W[e] = gout[(a * P + p) * rl + c];
  }
}

// ---------------------------------------------------------------------------------------------
// The reduction: chunk (value i, rows) x output block (b, c); sum over the chunk's rows of L[row][b] W[row][c]
// ---------------------------------------------------------------------------------------------
template <typename T>
struct TtggReduce {
  int64_t n;       // mode size
  int rk, rk1, ra;
  const int* chunks;
  const int* nchunks;
  const int* perm;  // the stable order of the mode's points
  const T* L;       // [rows][rk], or null for the first mode: row (p, a) is e_a
  const T* W;       // [rows][rk1]
  T* dG;            // [rk][n][rk1]
  T* part;          // [slot][rk][rk1]
};

__device__ __forceinline__ int ttgg_rid(const int* perm, int ra, int j) { return perm[j / ra] * ra + j % ra; }

template <typename T>
__device__ __forceinline__ T ttgg_left(const TtggReduce<T>& s, int rid, int b) {
  if (!s.L) return rid % s.ra == b ? (T)1 : (T)0;
  return s.L[(int64_t)rid * s.rk + b];
}

template <typename T>
__device__ __forceinline__ T* ttgg_dst(const TtggReduce<T>& s, int i, int slot, int b, int c) {
  return slot < 0 ? s.dG + ((int64_t)b * s.n + i) * s.rk1 + c : s.part + ((int64_t)slot * s.rk + b) * s.rk1 + c;
}

// On CUDA cores: each thread 4 x 4 of the 64 x 64 block, rows of the chunk in order.
template <typename T>
__global__ void __launch_bounds__(TTG_THREADS) ttgg_reduce_generic_kernel(const TtggReduce<T> s) {
  __shared__ T Ls[TTG_T][TTG_BK + 1];
  __shared__ T Ws[TTG_BK][TTG_BN + 1];
  __shared__ int rids[TTG_BK];
  const int ch = blockIdx.x;
  if (ch >= *s.nchunks) return;
  const int* ce = s.chunks + 4 * (int64_t)ch;
  const int i = ce[0], row0 = ce[1], cnt = ce[2], slot = ce[3];
  if (i >= s.n) return;  // points with an index out of range take no part
  const int b0 = blockIdx.y * TTG_T, c0 = blockIdx.z * TTG_BN, tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  T acc[4][4];
#pragma unroll
  for (int u = 0; u < 4; ++u)
#pragma unroll
    for (int v = 0; v < 4; ++v) acc[u][v] = 0;
  for (int k0 = 0; k0 < cnt; k0 += TTG_BK) {
    if (tid < TTG_BK) rids[tid] = k0 + tid < cnt ? ttgg_rid(s.perm, s.ra, row0 + k0 + tid) : 0;
    __syncthreads();
    for (int e = tid; e < TTG_T * TTG_BK; e += TTG_THREADS) {
      const int kk = e / TTG_T, b = e % TTG_T;
      Ls[b][kk] = (k0 + kk < cnt && b0 + b < s.rk) ? ttgg_left(s, rids[kk], b0 + b) : (T)0;
    }
    for (int e = tid; e < TTG_BK * TTG_BN; e += TTG_THREADS) {
      const int kk = e / TTG_BN, cc = e % TTG_BN;
      Ws[kk][cc] = (k0 + kk < cnt && c0 + cc < s.rk1) ? s.W[(int64_t)rids[kk] * s.rk1 + c0 + cc] : (T)0;
    }
    __syncthreads();
    const int kl = min(TTG_BK, cnt - k0);
    for (int kk = 0; kk < kl; ++kk) {
      T wv[4];
#pragma unroll
      for (int v = 0; v < 4; ++v) wv[v] = Ws[kk][tx + 16 * v];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const T lv = Ls[ty + 16 * u][kk];
#pragma unroll
        for (int v = 0; v < 4; ++v) acc[u][v] = fma(lv, wv[v], acc[u][v]);
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const int b = b0 + ty + 16 * u;
    if (b >= s.rk) continue;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
      const int c = c0 + tx + 16 * v;
      if (c < s.rk1) *ttgg_dst(s, i, slot, b, c) = acc[u][v];
    }
  }
}

// On the tensor cores: L^T staged as the 64 x 32 left operand, W as the 32 x 64 right one, ttg_mma_block per 32 rows.
template <typename T>
__global__ void __launch_bounds__(TTG_THREADS) ttgg_reduce_tc_kernel(const TtggReduce<T> s) {
  constexpr bool F64 = sizeof(T) == 8;
  constexpr int PLANES = F64 ? 1 : 2;
  __shared__ T Ls[PLANES][TTG_T][TTG_SS];
  __shared__ T Ws[PLANES][TTG_BK][TTG_SG];
  __shared__ int rids[TTG_BK];
  const int ch = blockIdx.x;
  if (ch >= *s.nchunks) return;
  const int* ce = s.chunks + 4 * (int64_t)ch;
  const int i = ce[0], row0 = ce[1], cnt = ce[2], slot = ce[3];
  if (i >= s.n) return;
  const int b0 = blockIdx.y * TTG_T, c0 = blockIdx.z * TTG_BN, tid = threadIdx.x;
  const int w = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int mrow = 16 * (w & 3), ncol = 32 * (w >> 2);
  using Acc = typename std::conditional<F64, double, float>::type;
  Acc acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[j][e] = 0;
  for (int k0 = 0; k0 < cnt; k0 += TTG_BK) {
    if (tid < TTG_BK) rids[tid] = k0 + tid < cnt ? ttgg_rid(s.perm, s.ra, row0 + k0 + tid) : 0;
    __syncthreads();
    for (int e = tid; e < TTG_T * TTG_BK; e += TTG_THREADS) {
      const int kk = e / TTG_T, b = e % TTG_T;
      const T v = (k0 + kk < cnt && b0 + b < s.rk) ? ttgg_left(s, rids[kk], b0 + b) : (T)0;
      if constexpr (F64) {
        Ls[0][b][kk] = v;
      } else {
        const float hi = ex_tf32_rn(v);
        Ls[0][b][kk] = hi, Ls[1][b][kk] = ex_tf32_rn(v - hi);
      }
    }
    for (int e = tid; e < TTG_BK * TTG_BN; e += TTG_THREADS) {
      const int kk = e / TTG_BN, cc = e % TTG_BN;
      const T v = (k0 + kk < cnt && c0 + cc < s.rk1) ? s.W[(int64_t)rids[kk] * s.rk1 + c0 + cc] : (T)0;
      if constexpr (F64) {
        Ws[0][kk][cc] = v;
      } else {
        const float hi = ex_tf32_rn(v);
        Ws[0][kk][cc] = hi, Ws[1][kk][cc] = ex_tf32_rn(v - hi);
      }
    }
    __syncthreads();
    ttg_mma_block<T>(acc, Ls, Ws, mrow, ncol, g, t);
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int b = b0 + mrow + g + 8 * (e >> 1), c = c0 + ncol + 8 * j + 2 * t + (e & 1);
      if (b < s.rk && c < s.rk1) *ttgg_dst(s, i, slot, b, c) = (T)acc[j][e];
    }
}

// The slices of buckets of more than one chunk: the first chunk of such a bucket sums its bucket's partials in chunk
// order, in fp64, and rounds once.
template <typename T>
__global__ void ttgg_combine_kernel(const TtggReduce<T> s) {
  const int ch = blockIdx.x;
  if (ch >= *s.nchunks) return;
  const int* ce = s.chunks + 4 * (int64_t)ch;
  const int i = ce[0], slot = ce[3];
  if (i >= s.n || slot < 0 || (ch > 0 && ce[-4] == i)) return;
  int nq = 1;
  while (ch + nq < *s.nchunks && ce[4 * nq] == i) ++nq;
  const int64_t area = (int64_t)s.rk * s.rk1;
  for (int64_t e = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; e < area; e += (int64_t)gridDim.y * blockDim.x) {
    double sum = 0;
    for (int q = 0; q < nq; ++q) sum += (double)s.part[(slot + q) * area + e];
    const int64_t b = e / s.rk1, c = e % s.rk1;
    s.dG[(b * s.n + i) * s.rk1 + c] = (T)sum;
  }
}

// ---------------------------------------------------------------------------------------------
// The driver
// ---------------------------------------------------------------------------------------------
// T: float or double.  Workspace: the narrowed indices [M][P]; per mode the bucket counts and the stable order [P]
// (plus one [P] buffer and the digit histograms of a sort pass); per mode of one train its tile and chunk lists; the
// kept L_k (P r_first sum r_k over the modes after the first); two W buffers of P r_first max r_{k+1}; one mode's chunk
// partials.  The lists, states and partials are sized by the largest train and reused by every train.  Never a core.
template <typename T, class ArenaT>
inline int tt_gather_grad_impl(ArenaT& ar, bool dry, const T* const* cores, int ntrains, int ndim,
                               const int64_t* shape, const int32_t* ranks, int first, int last, const int64_t* idx,
                               int64_t P, const T* gout, T* const* gcores, cudaStream_t st) {
  const int M = last - first;
  const int64_t R = ndim + 1;
  int64_t ncounts = 0;
  int passes_max = 1;
  for (int k = first; k < last; ++k) ncounts += shape[k] + 1, passes_max = std::max(passes_max, ttgg_sort_passes(shape[k]));
  const int64_t nblocks = ttgg_sort_blocks(P);
  int64_t lsum_max = 0, w_max = 0, tiles_max = 0, chunks_max = 0, part_max = 0;
  for (int t = 0; t < ntrains; ++t) {
    const int32_t* r = ranks + t * R;
    const int64_t rows = P * r[first];
    int64_t lsum = 0, wcols = 0, tl = 0, cl = 0;
    for (int k = first; k < last; ++k) {
      if (k > first) lsum += rows * r[k], tl += 3 * ttg_tile_bound(rows, shape[k]) + 1;
      wcols = std::max<int64_t>(wcols, r[k + 1]);
      const int64_t ch = ttgg_chunk_rows(rows, r[k], r[k + 1]);
      cl += 4 * ttgg_chunk_bound(rows, shape[k], ch) + 1;
      part_max = std::max(part_max, ttgg_slot_bound(rows, ch) * r[k] * r[k + 1]);
    }
    lsum_max = std::max(lsum_max, lsum), w_max = std::max(w_max, rows * wcols);
    tiles_max = std::max(tiles_max, tl), chunks_max = std::max(chunks_max, cl);
  }
  int* idx32 = ar.template take<int>((size_t)(P * M));
  int* counts = ar.template take<int>((size_t)ncounts);
  int* order = ar.template take<int>((size_t)(P * M));
  int* otmp = passes_max > 1 ? ar.template take<int>((size_t)P) : nullptr;
  int* dhist = ar.template take<int>((size_t)(TTGG_DIGITS * nblocks));
  int* tiles = tiles_max > 0 ? ar.template take<int>((size_t)tiles_max) : nullptr;
  int* chunks = ar.template take<int>((size_t)chunks_max);
  T* lbuf = lsum_max > 0 ? ar.template take<T>((size_t)lsum_max) : nullptr;
  T* wbuf[2] = {ar.template take<T>((size_t)w_max), ar.template take<T>((size_t)w_max)};
  T* part = part_max > 0 ? ar.template take<T>((size_t)part_max) : nullptr;
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_gather_grad: workspace too small (need %zu bytes)", ar.off);

  // the stable order of every mode, shared by all trains
  TtggModes md;
  md.m = M;
  for (int m = 0; m < M; ++m) md.n[m] = (int)shape[first + m];
  ttgg_narrow_kernel<<<grid_for(std::max(P, ncounts)), 256, 0, st>>>(md, idx, P, idx32, counts, ncounts);
  TNB_LAUNCH_CHECK();
  std::vector<int*> cnt_of(M), ord_of(M);
  int64_t coff = 0;
  for (int m = 0; m < M; ++m) {
    const int n = (int)shape[first + m];
    const int* ix = idx32 + (int64_t)m * P;
    cnt_of[m] = counts + coff, ord_of[m] = order + (int64_t)m * P;
    coff += n + 1;
    ttgg_count_kernel<<<grid_for(P), 256, 0, st>>>(ix, P, n, cnt_of[m]);
    TNB_LAUNCH_CHECK();
    const int passes = ttgg_sort_passes(n);
    const int* src = nullptr;
    for (int q = 0; q < passes; ++q) {
      int* dst = ((passes - 1 - q) % 2 == 0) ? ord_of[m] : otmp;  // the last pass writes the mode's order
      ttgg_digit_hist_kernel<<<(unsigned)nblocks, TTGG_SORT_THREADS, 0, st>>>(ix, src, P, n, 8 * q, dhist);
      TNB_LAUNCH_CHECK();
      ttgg_digit_scan_kernel<<<1, TTGG_SCAN_THREADS, 0, st>>>(dhist, TTGG_DIGITS * nblocks);
      TNB_LAUNCH_CHECK();
      ttgg_digit_scatter_kernel<<<(unsigned)nblocks, TTGG_SORT_THREADS, 0, st>>>(ix, src, P, n, 8 * q, dhist, dst);
      TNB_LAUNCH_CHECK();
      src = dst;
    }
  }

  for (int t = 0; t < ntrains; ++t) {
    const int32_t* r = ranks + t * R;
    const int ra = r[first];
    const int64_t rows = P * ra;
    // plans of every mode
    std::vector<int*> tl_of(M, nullptr), cl_of(M);
    std::vector<int64_t> ch_of(M);
    int64_t toff = 0, choff = 0;
    for (int m = 0; m < M; ++m) {
      const int k = first + m, n = (int)shape[k];
      if (m > 0) {
        tl_of[m] = tiles + toff;
        const int64_t tb = ttg_tile_bound(rows, n);
        toff += 3 * tb + 1;
        ttgg_plan_kernel<<<1, TTGG_PLAN_THREADS, 0, st>>>(cnt_of[m], n, ra, TTG_T, 3, tl_of[m], tl_of[m] + 3 * tb);
        TNB_LAUNCH_CHECK();
      }
      ch_of[m] = ttgg_chunk_rows(rows, r[k], r[k + 1]);
      cl_of[m] = chunks + choff;
      const int64_t cb = ttgg_chunk_bound(rows, n, ch_of[m]);
      choff += 4 * cb + 1;
      ttgg_plan_kernel<<<1, TTGG_PLAN_THREADS, 0, st>>>(cnt_of[m], n, ra, (int)ch_of[m], 4, cl_of[m], cl_of[m] + 4 * cb);
      TNB_LAUNCH_CHECK();
    }
    // forward: L_{first+1} .. L_{last-1}
    std::vector<T*> L_of(M, nullptr);
    int64_t loff = 0;
    for (int m = 1; m < M; ++m) L_of[m] = lbuf + loff, loff += rows * r[first + m];
    if (M > 1) {
      ttg_init_kernel<T><<<grid_for(rows * r[first + 1]), 256, 0, st>>>(cores[t * ndim + first], shape[first], ra,
                                                                        r[first + 1], idx32, P, L_of[1], nullptr);
      TNB_LAUNCH_CHECK();
    }
    for (int m = 1; m + 1 < M; ++m) {
      const int k = first + m, n = (int)shape[k];
      TtgStep s;
      s.n = n, s.P = P, s.rk = r[k], s.rk1 = r[k + 1], s.ra = ra, s.tiles = tl_of[m];
      s.ntiles = tl_of[m] + 3 * ttg_tile_bound(rows, n), s.perm = ord_of[m];
      const dim3 grid((unsigned)ttg_tile_bound(rows, n), (unsigned)ceil_div<int64_t>(r[k + 1], TTG_BN));
      if (ttg_mode_path(r[k], r[k + 1]) == TTG_MODE_TC)
        ttg_step_tc_kernel<T, true, false><<<grid, TTG_THREADS, 0, st>>>(s, cores[t * ndim + k], L_of[m], L_of[m + 1],
                                                                         nullptr);
      else
        ttg_step_generic_kernel<T, true, false><<<grid, TTG_THREADS, 0, st>>>(s, cores[t * ndim + k], L_of[m],
                                                                              L_of[m + 1], nullptr);
      TNB_LAUNCH_CHECK();
    }
    // reverse
    for (int k = first; k < last; ++k)
      TNB_CUDA(cudaMemsetAsync(gcores[t * ndim + k], 0, sizeof(T) * (size_t)r[k] * shape[k] * r[k + 1], st));
    ttgg_load_kernel<T><<<grid_for(rows * r[last]), 256, 0, st>>>(gout + (int64_t)t * rows * r[last], P, ra, r[last],
                                                                  wbuf[0]);
    TNB_LAUNCH_CHECK();
    int cur = 0;
    for (int m = M - 1; m >= 0; --m) {
      const int k = first + m, n = (int)shape[k];
      const int64_t cb = ttgg_chunk_bound(rows, n, ch_of[m]);
      TtggReduce<T> red;
      red.n = n, red.rk = r[k], red.rk1 = r[k + 1], red.ra = ra, red.chunks = cl_of[m], red.nchunks = cl_of[m] + 4 * cb;
      red.perm = ord_of[m], red.L = L_of[m], red.W = wbuf[cur], red.dG = gcores[t * ndim + k], red.part = part;
      const dim3 rgrid((unsigned)cb, (unsigned)ceil_div<int64_t>(r[k], TTG_T), (unsigned)ceil_div<int64_t>(r[k + 1], TTG_BN));
      if (ttg_mode_path(r[k], r[k + 1]) == TTG_MODE_TC)
        ttgg_reduce_tc_kernel<T><<<rgrid, TTG_THREADS, 0, st>>>(red);
      else
        ttgg_reduce_generic_kernel<T><<<rgrid, TTG_THREADS, 0, st>>>(red);
      TNB_LAUNCH_CHECK();
      const int64_t area = (int64_t)r[k] * r[k + 1];
      const dim3 cgrid((unsigned)cb, (unsigned)std::min<int64_t>(ceil_div<int64_t>(area, 256), 65535));
      ttgg_combine_kernel<T><<<cgrid, 256, 0, st>>>(red);
      TNB_LAUNCH_CHECK();
      if (m == 0) break;
      TtgStep s;  // W_{k-1} = W_k G_k[:, i, :]^T: r_{k+1} columns in, r_k out
      s.n = n, s.P = P, s.rk = r[k + 1], s.rk1 = r[k], s.ra = ra, s.tiles = tl_of[m];
      s.ntiles = tl_of[m] + 3 * ttg_tile_bound(rows, n), s.perm = ord_of[m];
      const dim3 grid((unsigned)ttg_tile_bound(rows, n), (unsigned)ceil_div<int64_t>(r[k], TTG_BN));
      if (ttg_mode_path(r[k], r[k + 1]) == TTG_MODE_TC)
        ttg_step_tc_kernel<T, true, true><<<grid, TTG_THREADS, 0, st>>>(s, cores[t * ndim + k], wbuf[cur],
                                                                        wbuf[cur ^ 1], nullptr);
      else
        ttg_step_generic_kernel<T, true, true><<<grid, TTG_THREADS, 0, st>>>(s, cores[t * ndim + k], wbuf[cur],
                                                                             wbuf[cur ^ 1], nullptr);
      TNB_LAUNCH_CHECK();
      cur ^= 1;
    }
  }
  return TNB_OK;
}

}  // namespace tnb
