// TT-matrix times a batch (tnb_tt_multiply): Y (b x O) = X (b x I) M, where M (I x O, I = prod i_k, O = prod o_k) is
// given by d cores [r_k, i_k, o_k, r_{k+1}] (r_0 = r_d = 1) and is never formed.
//
// Step k contracts (i_k, r_k) of the running intermediate with core k and appends (o_k, r_{k+1}).  The intermediates keep
// the batch index outermost:
//   T_k [b][i_k .. i_{d-1}][o_0 .. o_{k-1}][r_k],   T_0 = X (r_0 = 1),   T_d = Y (r_d = 1),
// so with R_k = (i_{k+1} .. i_{d-1}) (o_0 .. o_{k-1}) rows per batch element, step k is
//   T_{k+1}[b R_k + j][o_k r_{k+1}] = sum_{i, r} T_k[b][i][j][r] core_k[r][i][o_k r_{k+1}],
// a GEMM with M = b R_k rows, K = i_k r_k and N = o_k r_{k+1}.  Its A operand is T_k as the previous step wrote it (for a
// fixed (b, i) an R_k x r_k row-major block) and its output is row-major in exactly the layout step k + 1 reads: no step
// copies, transposes or permutes an operand, step 0 reads X and step d - 1 writes Y.
//
// ttm_step_tc_kernel runs a step on the tensor cores at fp32 accuracy ("3xTF32" as in project_tc.cuh / expand_tc.cuh):
//   * A chunks of 128 rows j x 32 columns r of one (b, i) are staged by TMA (a 4-D map over (r_k, R_k, i_k, b),
//     SWIZZLE_128B, zero fill past R_k and r_k) and split in registers (A_lo = A - trunc_tf32(A)) as in project_tc;
//   * the cores' hi / lo images (ttm_image_kernel, one launch for all tensor-core steps of the call) are stored per
//     (column tile, i, 32-wide r chunk) as kcr rows of EX_RS floats, the expand_tc R-image layout, so each chunk is one
//     contiguous run brought in by a TMA bulk copy behind the same mbarrier as its A chunk;
//   * persistent CTAs over 128 x 128 output tiles, column tile fastest so the CTAs that share an A block run together
//     and it is read from HBM once; the expand_tc warp layout (eight MMA warps of 32 x 64, mma.sync m16n8k8 .tf32), n8
//     tiles past N skipped; each warp stores its piece from registers with 8-byte stores (whole 32-byte sectors).
//
// Everything outside the kernel's envelope (ttm_step_path) runs ttm_step_generic_kernel, the 64 x 64 x 16 CUDA-core
// tiles of gemm_generic.cuh with the step's addressing, under the same driver.  That includes every step with r_k = 1
// (always step 0): its A blocks are single columns, M-major, which the K-major TMA tiles do not read.
#pragma once
#include "expand_tc.cuh"
#include "project_tc.cuh"

namespace tnb {

// ---------------------------------------------------------------------------------------------
// The envelope of the tensor-core step
// ---------------------------------------------------------------------------------------------
constexpr int TTM_TC_MAX_R = 256;      // the rank envelope of the library's other tensor-core kernels
constexpr int TTM_TC_MIN_ROWS = 64;    // rows per batch element: below half a tile most of every A block is padding
// Below this many output elements a step cannot fill the GPU with 128 x 128 tiles (64 of them) and the generic tiles
// are used.
constexpr int64_t TTM_TC_MIN_ELEMS = (int64_t)1 << 20;

enum TtmPath {
  TTM_PATH_TC = 0,
  TTM_PATH_F64 = 1,         // fp64 operands
  TTM_PATH_RANK_ALIGN = 2,  // r_k % 4 != 0: the A rows are not 16-byte multiples that TMA can address
  TTM_PATH_RANK_MAX = 3,    // r_k > TTM_TC_MAX_R
  TTM_PATH_N_ODD = 4,       // o_k r_{k+1} odd: the 8-byte stores need even row lengths
  TTM_PATH_EXTENT = 5,      // R_k below TTM_TC_MIN_ROWS, or R_k, i_k or N at or past 2^31 (32-bit TMA coordinates)
  TTM_PATH_SMALL = 6,       // fewer than TTM_TC_MIN_ELEMS output elements
  TTM_PATH_OUT_ALIGN = 7,   // output not 8-byte aligned (only Y can be: the intermediates are the workspace's)
};

// The path of one step: rows = R_k, nb = batch, I = i_k, r = r_k, N = o_k r_{k+1}.  The one place the envelope is
// defined.
inline int ttm_step_path(bool f32, int64_t rows, int64_t nb, int64_t I, int64_t r, int64_t N, bool out_aligned) {
  if (!f32) return TTM_PATH_F64;
  if (r % 4 != 0) return TTM_PATH_RANK_ALIGN;
  if (r > TTM_TC_MAX_R) return TTM_PATH_RANK_MAX;
  if (N % 2 != 0) return TTM_PATH_N_ODD;
  constexpr int64_t lim = (int64_t)1 << 31;
  if (rows < TTM_TC_MIN_ROWS || rows >= lim || I >= lim || N >= lim) return TTM_PATH_EXTENT;
  if (nb * rows * N < TTM_TC_MIN_ELEMS) return TTM_PATH_SMALL;
  if (!out_aligned) return TTM_PATH_OUT_ALIGN;
  return TTM_PATH_TC;
}

// ---------------------------------------------------------------------------------------------
// Tensor-core step
// ---------------------------------------------------------------------------------------------
constexpr int TTM_STAGES = 4;
constexpr int TTM_B_MAX_BYTES = 2 * EX_KC * EX_RS * 4;          // hi + lo of one 32-row image chunk
constexpr int TTM_STAGE_BYTES = PT_A_BYTES + TTM_B_MAX_BYTES;   // 50 KB, a multiple of 1024 (swizzle alignment)
constexpr int TTM_SMEM_BYTES = TTM_STAGES * TTM_STAGE_BYTES + 1024 /*align*/ + 64 /*barriers*/;
static_assert(TTM_STAGE_BYTES % 1024 == 0, "each A tile starts 1024-byte aligned");
static_assert(TTM_SMEM_BYTES <= 227 * 1024, "ttm_step_tc: shared memory");

struct TtmStepParams {
  int64_t R;        // rows per batch element
  int I, r, N;      // i_k, r_k, o_k r_{k+1}
  int nrc;          // 32-wide chunks of r_k
  int kcr;          // image rows per chunk: r_k rounded up to 8 when r_k <= 32, else 32
  int64_t num_tj, num_tn, num_tiles;
  const float* img;  // [tn][i][rc][hi | lo][kcr][EX_RS]
  float* out;        // [nb R][N]
};

__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
      : "memory");
}

// tile -> (batch element, row tile, column tile), column tile fastest
__device__ __forceinline__ void ttm_tile(const TtmStepParams& p, int64_t tile, int64_t& b, int64_t& tj, int64_t& tn) {
  tn = tile % p.num_tn;
  tile /= p.num_tn;
  tj = tile % p.num_tj;
  b = tile / p.num_tj;
}

__global__ void __launch_bounds__(EX_THREADS, 1)
ttm_step_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const TtmStepParams p) {
  extern __shared__ unsigned char ttm_smem_raw[];
  unsigned char* base = ttm_smem_raw + ((1024u - (smem_u32(ttm_smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(base + TTM_STAGES * TTM_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + TTM_STAGES;
  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < TTM_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EX_MMA_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int64_t my_tiles = (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;  // may be 0
  const int chunk_floats = 2 * p.kcr * EX_RS;

  if (warp_idx == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      const uint32_t b_bytes = (uint32_t)chunk_floats * 4u;
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t it = 0; it < my_tiles; ++it) {
        int64_t b, tj, tn;
        ttm_tile(p, blockIdx.x + it * gridDim.x, b, tj, tn);
        for (int i = 0; i < p.I; ++i)
          for (int rc = 0; rc < p.nrc; ++rc) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            unsigned char* sb = base + stage * TTM_STAGE_BYTES;
            mbar_expect_tx(&full_bar[stage], (uint32_t)PT_A_BYTES + b_bytes);
            tma_load_4d(sb, &tmap_a, &full_bar[stage], rc * EX_KC, (int)(tj * EX_BM), i, (int)b);
            bulk_load(sb + PT_A_BYTES, p.img + ((tn * p.I + i) * p.nrc + rc) * (int64_t)chunk_floats, b_bytes,
                      &full_bar[stage]);
            if (++stage == TTM_STAGES) { stage = 0; phase ^= 1u; }
          }
      }
    }
    return;
  }

  // ================= MMA warps =================
  const int w = warp_idx - 1, g = lane >> 2, t = lane & 3;
  const int wm = (w >> 1) * EX_WM, wn = (w & 1) * EX_WN;
  const int nk = p.I * p.nrc;
  int stage = 0;
  uint32_t phase = 0;
  for (int64_t it = 0; it < my_tiles; ++it) {
    int64_t b, tj, tn;
    ttm_tile(p, blockIdx.x + it * gridDim.x, b, tj, tn);
    const int64_t col0 = tn * EX_BN + wn;
    const int64_t left = (p.N - col0 + 7) / 8;  // n8 tiles of this warp inside N
    const int nj = left < 0 ? 0 : left > 8 ? 8 : (int)left;
    float out[2][8][4];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) out[a][j][e] = 0.f;
    int rc = 0;
    for (int kc = 0; kc < nk; ++kc) {
      mbar_wait(&full_bar[stage], phase);
      const unsigned char* sa = base + stage * TTM_STAGE_BYTES;
      const uint32_t* Bh = reinterpret_cast<const uint32_t*>(sa + PT_A_BYTES);
      const uint32_t* Bl = Bh + p.kcr * EX_RS;
      float acc[2][8][4];
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[a][j][e] = 0.f;
      const int steps = min(p.kcr, p.r - rc * EX_KC + 7) / 8;  // the k-steps past r_k hold zeros
#pragma unroll 1
      for (int ks = 0; ks < steps; ++ks) {
        const int k0 = 8 * ks;
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int a = 0; a < 2; ++a) {
          const int m = wm + 16 * a + g;
          ah[a][0] = km_ld(sa, m, k0 + t);
          ah[a][1] = km_ld(sa, m + 8, k0 + t);
          ah[a][2] = km_ld(sa, m, k0 + t + 4);
          ah[a][3] = km_ld(sa, m + 8, k0 + t + 4);
#pragma unroll
          for (int q = 0; q < 4; ++q)
            al[a][q] = __float_as_uint(__uint_as_float(ah[a][q]) - __uint_as_float(ah[a][q] & 0xFFFFE000u));
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (j < nj) {
            const int o = (k0 + t) * EX_RS + wn + 8 * j + g;
            const uint32_t bh0 = Bh[o], bh1 = Bh[o + 4 * EX_RS], bl0 = Bl[o], bl1 = Bl[o + 4 * EX_RS];
#pragma unroll
            for (int a = 0; a < 2; ++a) {
              mma_tf32(acc[a][j], ah[a][0], ah[a][1], ah[a][2], ah[a][3], bl0, bl1);  // A_hi B_lo
              mma_tf32(acc[a][j], al[a][0], al[a][1], al[a][2], al[a][3], bh0, bh1);  // A_lo B_hi
              mma_tf32(acc[a][j], ah[a][0], ah[a][1], ah[a][2], ah[a][3], bh0, bh1);  // A_hi B_hi
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == TTM_STAGES) { stage = 0; phase ^= 1u; }
      if (++rc == p.nrc) rc = 0;
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) out[a][j][e] += acc[a][j][e];
    }
    // fragment (a, j): rows 16a + g (c0, c1) and 16a + g + 8 (c2, c3), columns 8j + 2t, 8j + 2t + 1 of the warp's piece
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t j = tj * EX_BM + wm + 16 * a + g + 8 * h;
        if (j >= p.R) continue;
        float* row = p.out + (b * p.R + j) * p.N;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          const int64_t c = col0 + 8 * jj + 2 * t;
          if (c < p.N) *reinterpret_cast<float2*>(row + c) = make_float2(out[a][jj][2 * h], out[a][jj][2 * h + 1]);
        }
      }
  }
}

// The hi / lo images of the cores of up to TTM_IMG_BATCH tensor-core steps, one launch.
constexpr int TTM_IMG_BATCH = 16;
struct TtmImageTable {
  int n;
  const float* core[TTM_IMG_BATCH];
  float* img[TTM_IMG_BATCH];
  int I[TTM_IMG_BATCH], r[TTM_IMG_BATCH], N[TTM_IMG_BATCH], nrc[TTM_IMG_BATCH], kcr[TTM_IMG_BATCH];
  int64_t end[TTM_IMG_BATCH];  // running sum of the images' hi-term elements
};

inline int64_t ttm_num_tn(int64_t N) { return ceil_div<int64_t>(N, EX_BN); }
inline int ttm_kcr(int64_t r) { return r <= EX_KC ? (int)ceil_div<int64_t>(r, 8) * 8 : EX_KC; }
inline int ttm_nrc(int64_t r) { return (int)ceil_div<int64_t>(r, EX_KC); }
// floats of one core's image (hi and lo)
inline size_t ttm_image_elems(int64_t I, int64_t r, int64_t N) {
  return (size_t)ttm_num_tn(N) * I * ttm_nrc(r) * 2 * ttm_kcr(r) * EX_RS;
}

// core (r x I x N, row-major) -> image [tn][i][rc][hi | lo][kcr][EX_RS], element (kk, c) = core[rc 32 + kk][i][tn 128 + c],
// zero past r and N; hi / lo rounded to nearest (ex_split_store)
__global__ void ttm_image_kernel(const TtmImageTable tab) {
  const int64_t total = tab.end[tab.n - 1];
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    int q = 0;
    while (idx >= tab.end[q]) ++q;
    const int64_t e = idx - (q ? tab.end[q - 1] : 0);
    const int kcr = tab.kcr[q], nrc = tab.nrc[q], I = tab.I[q], r = tab.r[q], N = tab.N[q];
    const int c = (int)(e % EX_RS), kk = (int)(e / EX_RS % kcr);
    const int64_t blk = e / ((int64_t)kcr * EX_RS);
    const int rr = (int)(blk % nrc) * EX_KC + kk, i = (int)(blk / nrc % I);
    const int64_t n = blk / ((int64_t)nrc * I) * EX_BN + c;
    const float v = (c < EX_BN && rr < r && n < N) ? tab.core[q][((int64_t)rr * I + i) * N + n] : 0.f;
    ex_split_store(v, tab.img[q] + blk * (2 * kcr * EX_RS) + kk * EX_RS + c, kcr * EX_RS);
  }
}

inline int ttm_step_tc(const float* A, int64_t nb, int64_t R, int64_t I, int64_t r, int64_t N, const float* img, float* out,
                       cudaStream_t st) {
  TtmStepParams p;
  p.R = R; p.I = (int)I; p.r = (int)r; p.N = (int)N;
  p.nrc = ttm_nrc(r);
  p.kcr = ttm_kcr(r);
  p.num_tj = ceil_div<int64_t>(R, EX_BM);
  p.num_tn = ttm_num_tn(N);
  p.num_tiles = nb * p.num_tj * p.num_tn;
  p.img = img; p.out = out;
  CUtensorMap ta;  // (r, R, I, b), box (32, 128, 1, 1): one 128 x 32 swizzled tile of one (b, i)
  cuuint64_t gdim[4] = {(cuuint64_t)r, (cuuint64_t)R, (cuuint64_t)I, (cuuint64_t)nb};
  cuuint64_t gstride[3] = {(cuuint64_t)r * 4, (cuuint64_t)(R * r) * 4, (cuuint64_t)(I * R * r) * 4};
  cuuint32_t box[4] = {(cuuint32_t)EX_KC, (cuuint32_t)EX_BM, 1, 1}, estr[4] = {1, 1, 1, 1};
  CUresult cr = get_encode_tiled()(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(A), gdim, gstride, box, estr,
                                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return fail(TNB_ERR_CUDA, "tt_multiply: cuTensorMapEncodeTiled failed (%d)", (int)cr);
  static PerDeviceFlag attr_done;
  TNB_CUDA(ensure_dyn_smem(attr_done, ttm_step_tc_kernel, TTM_SMEM_BYTES));
  const int sms = usable_sms();
  const int64_t grid = p.num_tiles < sms ? p.num_tiles : sms;
  ttm_step_tc_kernel<<<(unsigned)grid, EX_THREADS, TTM_SMEM_BYTES, st>>>(ta, p);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// Generic step: the 64 x 64 x 16 tiles and 4 x 4 micro-tiles of gemm_tile_kernel, A(m, kk) at
// (m / R) I R r + (kk / r) R r + (m % R) r + kk % r and B(kk, n) = core[kk % r][kk / r][n].  Persistent over the tiles
// (a grid-stride loop), so M and N have no launch-grid limit.  KMAJ (r_k >= 16): a thread loads four rows at one k,
// reading runs of r_k; otherwise one row at four k, reading runs along j (r_k = 1: the rows of X).
// ---------------------------------------------------------------------------------------------
template <typename T, bool KMAJ>
__global__ void __launch_bounds__(GEMM_THREADS) ttm_step_generic_kernel(const T* __restrict__ A, const T* __restrict__ core,
                                                                        T* __restrict__ out, int64_t M, int64_t R, int64_t I,
                                                                        int r, int64_t N, int64_t num_tn,
                                                                        int64_t num_tiles) {
  __shared__ __align__(16) T As[GEMM_BK][GEMM_BM + 4];
  __shared__ __align__(16) T Bs[GEMM_BK][GEMM_BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t K = I * r, Rr = R * r;
  for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const int64_t m0 = tile / num_tn * GEMM_BM, n0 = tile % num_tn * GEMM_BN;
    // this thread's A rows: KMAJ rows (tid >> 4) + 16 q at column tid & 15, else row tid & 63 at columns (tid >> 6) + 4 q
    int64_t arow[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int64_t m = m0 + (KMAJ ? (tid >> 4) + 16 * q : (tid & 63));
      arow[q] = m < M ? (m / R) * I * Rr + (m % R) * r : -1;
    }
    T acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = T(0);
    for (int64_t k0 = 0; k0 < K; k0 += GEMM_BK) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int kk = KMAJ ? (tid & 15) : (tid >> 6) + 4 * q, mm = KMAJ ? (tid >> 4) + 16 * q : (tid & 63);
        const int64_t gk = k0 + kk;
        T v = T(0);
        if (arow[q] >= 0 && gk < K) v = A[arow[q] + (gk / r) * Rr + gk % r];
        As[kk][mm] = v;
      }
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int idx = tid + q * GEMM_THREADS, kk = idx >> 6, nn = idx & 63;
        const int64_t gk = k0 + kk, gn = n0 + nn;
        T v = T(0);
        if (gn < N && gk < K) v = core[((gk % r) * I + gk / r) * N + gn];
        Bs[kk][nn] = v;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < GEMM_BK; ++kk) {
        T a[4], bv[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) bv[j] = Bs[kk][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t gm = m0 + ty * 4 + i;
      if (gm >= M) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int64_t gn = n0 + tx * 4 + j;
        if (gn < N) out[gm * N + gn] = acc[i][j];
      }
    }
  }
}

template <typename T>
inline int ttm_step_generic(const T* A, int64_t nb, int64_t R, int64_t I, int64_t r, int64_t N, const T* core, T* out,
                            cudaStream_t st) {
  const int64_t M = nb * R;
  const int64_t num_tn = ceil_div<int64_t>(N, GEMM_BN), tiles = ceil_div<int64_t>(M, GEMM_BM) * num_tn;
  const int64_t cap = (int64_t)8 * device_sms();
  const unsigned grid = (unsigned)(tiles < cap ? tiles : cap);
  if (r >= 16)
    ttm_step_generic_kernel<T, true><<<grid, GEMM_THREADS, 0, st>>>(A, core, out, M, R, I, (int)r, N, num_tn, tiles);
  else
    ttm_step_generic_kernel<T, false><<<grid, GEMM_THREADS, 0, st>>>(A, core, out, M, R, I, (int)r, N, num_tn, tiles);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// The driver
// ---------------------------------------------------------------------------------------------
constexpr int TTM_MAX_D = 64;
constexpr int64_t TTM_MAX_ELEMS = (int64_t)1 << 46;  // of X, Y, every intermediate and every core

// d in [1, TTM_MAX_D], every extent and rank >= 1, unit boundary ranks (TNB_ERR_INVALID); batch < 2^31 (a TMA
// coordinate), and X, Y, each core and each step's input and output within TTM_MAX_ELEMS (TNB_ERR_UNSUPPORTED).
inline int ttm_check_dims(int d, const int64_t* idims, const int64_t* odims, const int32_t* ranks, int64_t batch) {
  if (d < 1 || d > TTM_MAX_D) return fail(TNB_ERR_INVALID, "tt_multiply: d=%d outside [1, %d]", d, TTM_MAX_D);
  if (ranks[0] != 1 || ranks[d] != 1) return fail(TNB_ERR_INVALID, "tt_multiply: boundary ranks must be 1");
  if (batch < 1) return fail(TNB_ERR_INVALID, "tt_multiply: batch must be >= 1");
  for (int k = 0; k < d; ++k)
    if (idims[k] < 1 || odims[k] < 1 || ranks[k + 1] < 1)
      return fail(TNB_ERR_INVALID, "tt_multiply: dims and ranks must be >= 1");
  if (batch >= ((int64_t)1 << 31)) return fail(TNB_ERR_UNSUPPORTED, "tt_multiply: batch must be below 2^31");
  const unsigned __int128 cap = (unsigned __int128)TTM_MAX_ELEMS;
  // step k reads (b, i_k .. i_{d-1}, o_0 .. o_{k-1}, r_k) and writes (b, i_{k+1} .. , o_0 .. o_k, r_{k+1}); k = 0 reads
  // X and k = d - 1 writes Y.  Every factor is >= 1 and each is checked as it joins, so nothing wraps.
  unsigned __int128 rows = (unsigned __int128)batch;
  for (int k = 0; k < d; ++k) {
    rows *= (unsigned __int128)idims[k];
    if (rows > cap) return fail(TNB_ERR_UNSUPPORTED, "tt_multiply: sizes too large");
  }
  for (int k = 0; k < d; ++k) {  // rows = b (i_k .. i_{d-1}) (o_0 .. o_{k-1})
    const unsigned __int128 core = (unsigned __int128)ranks[k] * idims[k] * odims[k] * ranks[k + 1];
    const unsigned __int128 in = rows * (unsigned __int128)ranks[k];
    const unsigned __int128 out = rows / (unsigned __int128)idims[k] * odims[k] * ranks[k + 1];
    if (core > cap || in > cap || out > cap) return fail(TNB_ERR_UNSUPPORTED, "tt_multiply: sizes too large");
    rows = rows / (unsigned __int128)idims[k] * odims[k];
  }
  return TNB_OK;
}

// T: float or double.  Y may be misaligned (the last step then takes the generic tiles); the workspace size does not
// depend on it.
template <typename T, class ArenaT>
inline int tt_multiply_impl(ArenaT& ar, bool dry, const T* const* cores, int d, const int64_t* idims, const int64_t* odims,
                            const int32_t* ranks, const T* X, int64_t nb, T* Y, cudaStream_t st) {
  constexpr bool F32 = std::is_same<T, float>::value;
  int64_t R[TTM_MAX_D], N[TTM_MAX_D];
  {
    int64_t rows = 1;  // R_k = (i_{k+1} .. i_{d-1}) (o_0 .. o_{k-1})
    for (int k = 1; k < d; ++k) rows *= idims[k];
    for (int k = 0; k < d; ++k) {
      R[k] = rows;
      N[k] = odims[k] * ranks[k + 1];
      if (k + 1 < d) rows = rows / idims[k + 1] * odims[k];
    }
  }
  int64_t inter = 0;  // the largest intermediate T_1 .. T_{d-1}
  for (int k = 0; k + 1 < d; ++k) inter = nb * R[k] * N[k] > inter ? nb * R[k] * N[k] : inter;
  T* buf[2] = {nullptr, nullptr};
  if (d > 1) buf[0] = ar.template take<T>((size_t)inter), buf[1] = d > 2 ? ar.template take<T>((size_t)inter) : nullptr;
  float* img[TTM_MAX_D];
  int path[TTM_MAX_D];
  for (int k = 0; k < d; ++k) {
    const bool out_aligned = dry || k + 1 < d || (reinterpret_cast<uintptr_t>(Y) & 7u) == 0;
    path[k] = ttm_step_path(F32, R[k], nb, idims[k], ranks[k], N[k], out_aligned);
    img[k] = nullptr;
    if (ttm_step_path(F32, R[k], nb, idims[k], ranks[k], N[k], true) == TTM_PATH_TC)
      img[k] = ar.template take<float>(ttm_image_elems(idims[k], ranks[k], N[k]));
  }
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_multiply: workspace too small (need %zu bytes)", ar.off);

  if constexpr (F32) {
    TtmImageTable tab;
    tab.n = 0;
    for (int k = 0; k < d; ++k) {
      if (path[k] != TTM_PATH_TC) continue;
      const int q = tab.n++;
      tab.core[q] = cores[k];
      tab.img[q] = img[k];
      tab.I[q] = (int)idims[k], tab.r[q] = ranks[k], tab.N[q] = (int)N[k];
      tab.nrc[q] = ttm_nrc(ranks[k]), tab.kcr[q] = ttm_kcr(ranks[k]);
      tab.end[q] = (q ? tab.end[q - 1] : 0) + (int64_t)(ttm_image_elems(idims[k], ranks[k], N[k]) / 2);
      if (tab.n == TTM_IMG_BATCH) {
        ttm_image_kernel<<<grid_for(tab.end[q]), 256, 0, st>>>(tab);
        TNB_LAUNCH_CHECK();
        tab.n = 0;
      }
    }
    if (tab.n > 0) {
      ttm_image_kernel<<<grid_for(tab.end[tab.n - 1]), 256, 0, st>>>(tab);
      TNB_LAUNCH_CHECK();
    }
  }
  for (int k = 0; k < d; ++k) {
    const T* in = k == 0 ? X : buf[(k - 1) & 1];
    T* out = k + 1 == d ? Y : buf[k & 1];
    if constexpr (F32)
      if (path[k] == TTM_PATH_TC) {
        TNB_TRY(ttm_step_tc(in, nb, R[k], idims[k], ranks[k], N[k], img[k], out, st));
        continue;
      }
    TNB_TRY(ttm_step_generic<T>(in, nb, R[k], idims[k], ranks[k], N[k], cores[k], out, st));
  }
  return TNB_OK;
}

template <class ArenaT>
inline int tt_multiply_dispatch(ArenaT& ar, bool dry, int dtype, const void* const* cores, int d, const int64_t* idims,
                                const int64_t* odims, const int32_t* ranks, const void* X, int64_t batch, void* Y,
                                cudaStream_t st) {
  if (dtype == TNB_F64)
    return tt_multiply_impl<double>(ar, dry, reinterpret_cast<const double* const*>(cores), d, idims, odims, ranks,
                                    static_cast<const double*>(X), batch, static_cast<double*>(Y), st);
  return tt_multiply_impl<float>(ar, dry, reinterpret_cast<const float* const*>(cores), d, idims, odims, ranks,
                                 static_cast<const float*>(X), batch, static_cast<float*>(Y), st);
}

}  // namespace tnb
