// TT -> dense: the cores of one tensor train expanded into a caller-owned row-major buffer (tnb_tt_decompress).
//
// Meet in the middle.  For a split bond k the left chain F_j = F_{j-1} core_j gives L ((I_0 .. I_{k-1}) x r_k), the
// right chain H_j = core_j H_{j+1} gives R (r_k x (I_k .. I_{N-1})), and the tensor is L R.  decompress_split picks the k
// with the smallest numel(L) + numel(R), so every chain step is a small product (gemm_direct) and the one large
// product has K = r_k: it reads almost nothing and is bound by writing the result once.  The left-to-right chain of
// Tensor.torch() instead writes and re-reads F_{N-2}, half the size of an fp32 result per 64-wide last mode.
//
// expand_tc_kernel, C (M x Nc) = L (M x K) R (K x Nc) at fp32 accuracy on the tensor cores, C fp32, bf16 or fp16:
//   * "3xTF32" as in project_tc.cuh (C = L_hi R_lo + L_lo R_hi + L_hi R_hi, low-order products first, each 32-wide K
//     chunk folded into an fp32 running sum).  Both operands are small, so expand_split_{l,r}_kernel split them once
//     into hi / lo images in the workspace and the hot loop has no per-element splitting;
//   * the images are stored tile by tile in the order the MMA warps read them: per (row tile, K chunk) 128 rows of
//     EX_LS = 36 floats for L, per (column tile, K chunk) 32 rows of EX_RS = 136 floats for R, hi then lo, zero past
//     M, Nc and K.  The paddings make every mma.sync fragment load hit 32 distinct banks, and an operand chunk is one
//     contiguous run, so the producer thread brings a stage in with two TMA bulk copies (cp.async.bulk) behind an
//     mbarrier.  Two stages: the next tile's operands arrive while the current tile is computed and stored;
//   * persistent CTAs over 128 x 128 tiles, eight MMA warps of 32 x 64 each (mma.sync m16n8k8 .tf32);
//   * epilogue: each warp stages its 32 x 64 piece in its own shared-memory patch (no CTA-wide barrier: the warps
//     drift apart and one warp's stores overlap another's MMAs) and writes whole rows of it with 16-byte streaming
//     stores, 256 B (fp32) or 128 B (16-bit) contiguous per row, converting once, round-to-nearest-even, at the store.
//     Rows past M and columns past Nc are predicated off; Nc % 8 == 0 keeps every 16-byte store whole and aligned.
// Tiles are walked column-fastest when R's image is the smaller one (it stays in L2 while each L chunk is reused by
// the tiles of one tile row) and row-fastest otherwise.
//
// Outside the kernel's envelope (expand_tc_shape_ok: fp32 cores, 8 <= K <= 256, Nc % 8 == 0, M Nc >= EXPAND_TC_MIN_ELEMS,
// out 16-byte aligned) the last product is gemm_direct with the output type as its store type: the same driver, the
// same single rounding, CUDA cores.
#pragma once
#include <type_traits>

#include "gemm_generic.cuh"
#include "gram_tc.cuh"
#include "small_kernels.cuh"

namespace tnb {

constexpr int EX_BM = 128, EX_BN = 128, EX_KC = 32;
constexpr int EX_LS = EX_KC + 4;                  // L image row stride (floats): 4 mod 8, A fragments conflict-free
constexpr int EX_RS = EX_BN + 8;                  // R image row stride (floats): 8 mod 32, B fragments conflict-free
constexpr int EX_L_TERM = EX_BM * EX_LS, EX_R_TERM = EX_KC * EX_RS;  // floats per hi or lo term of a chunk
constexpr int EX_L_BYTES = 2 * EX_L_TERM * 4, EX_R_BYTES = 2 * EX_R_TERM * 4;
constexpr int EX_STAGE_BYTES = EX_L_BYTES + EX_R_BYTES;
constexpr int EX_STAGES = 2;
constexpr int EX_MMA_WARPS = 8, EX_THREADS = 32 * (1 + EX_MMA_WARPS);
constexpr int EX_WM = 32, EX_WN = 64;             // warp tile: 4 x 2 warps per CTA tile
constexpr int EX_CS = EX_WN + 8;                  // staging row stride (floats): float2 fragment stores conflict-free
constexpr int EX_STG_BYTES = EX_MMA_WARPS * EX_WM * EX_CS * 4;
constexpr int EX_SMEM_BYTES = EX_STAGES * EX_STAGE_BYTES + EX_STG_BYTES + 128 /*align*/ + 64 /*barriers*/;
static_assert(EX_SMEM_BYTES <= 227 * 1024, "expand_tc: shared memory");
static_assert(EX_L_BYTES % 16 == 0 && EX_R_BYTES % 16 == 0, "bulk copies move multiples of 16 bytes");
constexpr int EX_MAX_K = 256;
// Below this many output elements the tile kernel cannot fill the GPU (64 tiles of 128 x 128) and the generic product
// is used.
constexpr int64_t EXPAND_TC_MIN_ELEMS = (int64_t)1 << 20;

struct ExpandTcParams {
  int64_t M, Nc;
  int k8;        // 8-wide k-steps that hold K
  int nkc;       // 32-wide K chunks
  int64_t num_tm, num_tn, num_tiles;
  int tm_fastest;
  const float* Limg;
  const float* Rimg;
  void* out;
};

__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :
               : "r"(smem_u32(smem_dst)), "l"(__cvta_generic_to_global(gsrc)), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ void ex_tile(const ExpandTcParams& p, int64_t tile, int64_t& tm, int64_t& tn) {
  if (p.tm_fastest) {
    tn = tile / p.num_tm;
    tm = tile % p.num_tm;
  } else {
    tm = tile / p.num_tn;
    tn = tile % p.num_tn;
  }
}

// two fp32 values as one 32-bit word of 16-bit elements (the first in the low half), round-to-nearest-even
template <typename TOut>
__device__ __forceinline__ uint32_t ex_pack2(float a, float b) {
  if constexpr (std::is_same<TOut, __half>::value) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  } else {
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
  }
}

template <typename TOut>
__global__ void __launch_bounds__(EX_THREADS, 1) expand_tc_kernel(const ExpandTcParams p) {
  extern __shared__ unsigned char ex_smem_raw[];
  unsigned char* base = ex_smem_raw + ((128u - (smem_u32(ex_smem_raw) & 127u)) & 127u);
  unsigned char* stg_base = base + EX_STAGES * EX_STAGE_BYTES;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stg_base + EX_STG_BYTES);
  uint64_t* empty_bar = full_bar + EX_STAGES;
  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < EX_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], EX_MMA_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int64_t my_tiles = (p.num_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;  // may be 0

  if (warp_idx == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t i = 0; i < my_tiles; ++i) {
        int64_t tm, tn;
        ex_tile(p, blockIdx.x + i * gridDim.x, tm, tn);
        for (int kc = 0; kc < p.nkc; ++kc) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          unsigned char* sb = base + stage * EX_STAGE_BYTES;
          mbar_expect_tx(&full_bar[stage], EX_STAGE_BYTES);
          bulk_load(sb, p.Limg + (tm * p.nkc + kc) * (2 * EX_L_TERM), EX_L_BYTES, &full_bar[stage]);
          bulk_load(sb + EX_L_BYTES, p.Rimg + (tn * p.nkc + kc) * (2 * EX_R_TERM), EX_R_BYTES, &full_bar[stage]);
          if (++stage == EX_STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ================= MMA warps =================
  const int w = warp_idx - 1, g = lane >> 2, t = lane & 3;
  const int wm = (w >> 1) * EX_WM, wn = (w & 1) * EX_WN;
  float* stg = reinterpret_cast<float*>(stg_base) + w * (EX_WM * EX_CS);
  int stage = 0;
  uint32_t phase = 0;
  for (int64_t i = 0; i < my_tiles; ++i) {
    int64_t tm, tn;
    ex_tile(p, blockIdx.x + i * gridDim.x, tm, tn);
    float out[2][8][4];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) out[a][j][e] = 0.f;
    for (int kc = 0; kc < p.nkc; ++kc) {
      mbar_wait(&full_bar[stage], phase);
      const uint32_t* Lh = reinterpret_cast<const uint32_t*>(base + stage * EX_STAGE_BYTES);
      const uint32_t* Ll = Lh + EX_L_TERM;
      const uint32_t* Rh = Lh + 2 * EX_L_TERM;
      const uint32_t* Rl = Rh + EX_R_TERM;
      float acc[2][8][4];
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) acc[a][j][e] = 0.f;
      const int steps = min(EX_KC / 8, p.k8 - kc * (EX_KC / 8));  // the k-steps past K hold zeros
#pragma unroll 1
      for (int ks = 0; ks < steps; ++ks) {
        const int k0 = 8 * ks;
        uint32_t ah[2][4], al[2][4];
#pragma unroll
        for (int a = 0; a < 2; ++a) {
          const int o = (wm + 16 * a + g) * EX_LS + k0 + t;
          ah[a][0] = Lh[o], ah[a][1] = Lh[o + 8 * EX_LS], ah[a][2] = Lh[o + 4], ah[a][3] = Lh[o + 8 * EX_LS + 4];
          al[a][0] = Ll[o], al[a][1] = Ll[o + 8 * EX_LS], al[a][2] = Ll[o + 4], al[a][3] = Ll[o + 8 * EX_LS + 4];
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int o = (k0 + t) * EX_RS + wn + 8 * j + g;
          const uint32_t bh0 = Rh[o], bh1 = Rh[o + 4 * EX_RS], bl0 = Rl[o], bl1 = Rl[o + 4 * EX_RS];
#pragma unroll
          for (int a = 0; a < 2; ++a) {
            mma_tf32(acc[a][j], ah[a][0], ah[a][1], ah[a][2], ah[a][3], bl0, bl1);  // L_hi R_lo
            mma_tf32(acc[a][j], al[a][0], al[a][1], al[a][2], al[a][3], bh0, bh1);  // L_lo R_hi
            mma_tf32(acc[a][j], ah[a][0], ah[a][1], ah[a][2], ah[a][3], bh0, bh1);  // L_hi R_hi
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);
      if (++stage == EX_STAGES) { stage = 0; phase ^= 1u; }
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e) out[a][j][e] += acc[a][j][e];
    }
    // fragment (a, j): rows 16a + g (c0, c1) and 16a + g + 8 (c2, c3), columns 8j + 2t, 8j + 2t + 1 of the warp's piece
    __syncwarp();  // the last tile's copy-out has read the patch
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<float2*>(stg + (16 * a + g + 8 * h) * EX_CS + 8 * j + 2 * t) =
              make_float2(out[a][j][2 * h], out[a][j][2 * h + 1]);
    __syncwarp();
    const int64_t row0 = tm * EX_BM + wm, col0 = tn * EX_BN + wn;
    if constexpr (sizeof(TOut) == 4) {  // 16 lanes x 16 B per row, two rows per pass
      float* C = static_cast<float*>(p.out);
      const int c = (lane & 15) * 4;
#pragma unroll 4
      for (int r = lane >> 4; r < EX_WM; r += 2)
        if (row0 + r < p.M && col0 + c < p.Nc)
          __stcs(reinterpret_cast<float4*>(C + (row0 + r) * p.Nc + col0 + c),
                 *reinterpret_cast<const float4*>(stg + r * EX_CS + c));
    } else {  // 8 lanes x 16 B (eight 16-bit elements) per row, four rows per pass
      TOut* C = static_cast<TOut*>(p.out);
      const int c = (lane & 7) * 8;
#pragma unroll 4
      for (int r = lane >> 3; r < EX_WM; r += 4)
        if (row0 + r < p.M && col0 + c < p.Nc) {
          const float4 x = *reinterpret_cast<const float4*>(stg + r * EX_CS + c);
          const float4 y = *reinterpret_cast<const float4*>(stg + r * EX_CS + c + 4);
          __stcs(reinterpret_cast<uint4*>(C + (row0 + r) * p.Nc + col0 + c),
                 make_uint4(ex_pack2<TOut>(x.x, x.y), ex_pack2<TOut>(x.z, x.w), ex_pack2<TOut>(y.x, y.y),
                            ex_pack2<TOut>(y.z, y.w)));
        }
    }
  }
}

__device__ __forceinline__ float ex_tf32_rn(float v) {
  uint32_t u;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(u) : "f"(v));
  return __uint_as_float(u);
}
// hi = v rounded to TF32, lo = the exact remainder v - hi rounded to TF32: both to nearest, so that what the pair drops
// (below 2^-22 |v|) has no sign bias, where the tensor core's own truncation of raw fp32 bits would always shrink.
__device__ __forceinline__ void ex_split_store(float v, float* hi_at, int term) {
  const float hi = ex_tf32_rn(v);
  hi_at[0] = hi;
  hi_at[term] = ex_tf32_rn(v - hi);
}
// L (M x K, row-major) -> image [row tile][K chunk][hi | lo][128][EX_LS]
__global__ void expand_split_l_kernel(const float* __restrict__ L, int64_t M, int K, int nkc, int64_t num_tm,
                                      float* __restrict__ img) {
  const int64_t total = num_tm * nkc * EX_L_TERM;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % EX_LS), r = (int)(idx / EX_LS % EX_BM);
    const int64_t blk = idx / EX_L_TERM;
    const int64_t row = blk / nkc * EX_BM + r;
    const int k = (int)(blk % nkc) * EX_KC + c;
    const float v = (c < EX_KC && row < M && k < K) ? L[row * K + k] : 0.f;
    ex_split_store(v, img + blk * (2 * EX_L_TERM) + r * EX_LS + c, EX_L_TERM);
  }
}
// R (K x Nc, row-major) -> image [column tile][K chunk][hi | lo][32][EX_RS]
__global__ void expand_split_r_kernel(const float* __restrict__ R, int K, int64_t Nc, int nkc, int64_t num_tn,
                                      float* __restrict__ img) {
  const int64_t total = num_tn * nkc * EX_R_TERM;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(idx % EX_RS), kk = (int)(idx / EX_RS % EX_KC);
    const int64_t blk = idx / EX_R_TERM;
    const int64_t col = blk / nkc * EX_BN + c;
    const int k = (int)(blk % nkc) * EX_KC + kk;
    const float v = (c < EX_BN && col < Nc && k < K) ? R[(int64_t)k * Nc + col] : 0.f;
    ex_split_store(v, img + blk * (2 * EX_R_TERM) + kk * EX_RS + c, EX_R_TERM);
  }
}

inline bool expand_tc_shape_ok(int64_t M, int64_t K, int64_t Nc) {
  return K >= 8 && K <= EX_MAX_K && Nc % 8 == 0 && M * Nc >= EXPAND_TC_MIN_ELEMS;
}
inline size_t expand_tc_limg_elems(int64_t M, int64_t K) {
  return (size_t)ceil_div<int64_t>(M, EX_BM) * ceil_div<int64_t>(K, EX_KC) * (2 * EX_L_TERM);
}
inline size_t expand_tc_rimg_elems(int64_t K, int64_t Nc) {
  return (size_t)ceil_div<int64_t>(Nc, EX_BN) * ceil_div<int64_t>(K, EX_KC) * (2 * EX_R_TERM);
}

// C (M x Nc, row-major, 16-byte aligned) = L (M x K) R (K x Nc); Limg / Rimg: expand_tc_{l,r}img_elems floats.
template <typename TOut>
inline int expand_tc(const float* L, const float* R, int64_t M, int64_t K, int64_t Nc, TOut* C, float* Limg, float* Rimg,
                     cudaStream_t st) {
  ExpandTcParams p;
  p.M = M; p.Nc = Nc;
  p.k8 = (int)ceil_div<int64_t>(K, 8);
  p.nkc = (int)ceil_div<int64_t>(K, EX_KC);
  p.num_tm = ceil_div<int64_t>(M, EX_BM);
  p.num_tn = ceil_div<int64_t>(Nc, EX_BN);
  p.num_tiles = p.num_tm * p.num_tn;
  p.tm_fastest = expand_tc_limg_elems(M, K) < expand_tc_rimg_elems(K, Nc) ? 1 : 0;
  p.Limg = Limg; p.Rimg = Rimg; p.out = C;
  expand_split_l_kernel<<<grid_for(p.num_tm * p.nkc * EX_L_TERM), 256, 0, st>>>(L, M, (int)K, p.nkc, p.num_tm, Limg);
  TNB_LAUNCH_CHECK();
  expand_split_r_kernel<<<grid_for(p.num_tn * p.nkc * EX_R_TERM), 256, 0, st>>>(R, (int)K, Nc, p.nkc, p.num_tn, Rimg);
  TNB_LAUNCH_CHECK();
  static PerDeviceFlag attr_done;
  TNB_CUDA(ensure_dyn_smem(attr_done, expand_tc_kernel<TOut>, EX_SMEM_BYTES));
  const int sms = usable_sms();
  const int64_t grid = p.num_tiles < sms ? p.num_tiles : sms;
  expand_tc_kernel<TOut><<<(unsigned)grid, EX_THREADS, EX_SMEM_BYTES, st>>>(p);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// Row-major C = A B on the generic tiles, C stored as TC; wide C in column blocks the launch grid can hold.
template <typename T, typename TC>
inline int gemm_rowmajor(int64_t M, int64_t N, int64_t K, const T* A, const T* B, TC* C, cudaStream_t st) {
  constexpr int64_t NB = (int64_t)65535 * GEMM_BN;
  for (int64_t n0 = 0; n0 < N; n0 += NB)
    TNB_TRY((gemm_direct<T, T, T, TC>(M, N - n0 < NB ? N - n0 : NB, K, A, K, true, B + n0, N, false, C + n0, N, (T)1,
                                      nullptr, 0, (T)0, nullptr, 0, (T)0, st)));
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// The driver
// ---------------------------------------------------------------------------------------------
constexpr int64_t DECOMPRESS_MAX_ELEMS = (int64_t)1 << 46;  // of the result and of every chain buffer

// Shapes and ranks the driver can size without overflow: extents and ranks >= 1, unit boundary ranks, the result and
// every partial product of either chain (taken at any split) within DECOMPRESS_MAX_ELEMS.
inline int decompress_check_dims(int N, const int64_t* shape, const int32_t* ranks) {
  if (N < 1 || N > 62) return fail(TNB_ERR_INVALID, "tt_decompress: ndim=%d outside [1, 62]", N);
  if (ranks[0] != 1 || ranks[N] != 1) return fail(TNB_ERR_INVALID, "tt_decompress: boundary ranks must be 1");
  unsigned __int128 left = 1;
  for (int j = 0; j < N; ++j) {
    if (shape[j] < 1 || ranks[j] < 1) return fail(TNB_ERR_INVALID, "tt_decompress: extents and ranks must be >= 1");
    left *= (unsigned __int128)shape[j];
    if (left > (unsigned __int128)DECOMPRESS_MAX_ELEMS) return fail(TNB_ERR_UNSUPPORTED, "tt_decompress: tensor too large");
  }
  return TNB_OK;
}

// The split bond k (1 <= k <= N - 1, N >= 2) with the smallest numel(L) + numel(R) = r_k (I_0 .. I_{k-1} + I_k .. I_{N-1});
// of equal ones the last, whose R is the smaller operand.
inline int decompress_split(int N, const int64_t* shape, const int32_t* ranks) {
  unsigned __int128 total = 1, left = 1, best = 0;
  for (int j = 0; j < N; ++j) total *= (unsigned __int128)shape[j];
  int best_k = 1;
  for (int k = 1; k < N; ++k) {
    left *= (unsigned __int128)shape[k - 1];
    const unsigned __int128 cost = (unsigned __int128)ranks[k] * (left + total / left);
    if (k == 1 || cost <= best) best = cost, best_k = k;
  }
  return best_k;
}

// T: the cores' type (float, double); TOut: T, or bf16 / fp16 with float cores.
template <typename T, typename TOut, class ArenaT>
inline int tt_decompress_impl(ArenaT& ar, bool dry, const T* const* cores, int N, const int64_t* shape,
                              const int32_t* ranks, TOut* out, cudaStream_t st) {
  if (N == 1) {
    if (dry) return TNB_OK;
    convert_kernel<T, TOut><<<grid_for(shape[0]), 256, 0, st>>>(cores[0], out, shape[0]);
    TNB_LAUNCH_CHECK();
    return TNB_OK;
  }
  const int k = decompress_split(N, shape, ranks);
  // F_j ((I_0 .. I_j) x r_{j+1}), j = 1 .. k-1, and H_j (r_j x (I_j .. I_{N-1})), j = N-2 .. k, ping-pong by parity of j
  unsigned __int128 fl[2] = {0, 0}, fr[2] = {0, 0}, rows128 = (unsigned __int128)shape[0], cols128 = (unsigned __int128)shape[N - 1];
  for (int j = 1; j < k; ++j) {
    rows128 *= (unsigned __int128)shape[j];
    const unsigned __int128 e = rows128 * (unsigned __int128)ranks[j + 1];
    if (e > fl[j & 1]) fl[j & 1] = e;
  }
  for (int j = N - 2; j >= k; --j) {
    cols128 *= (unsigned __int128)shape[j];
    const unsigned __int128 e = cols128 * (unsigned __int128)ranks[j];
    if (e > fr[j & 1]) fr[j & 1] = e;
  }
  const int64_t M = (int64_t)rows128, Nc = (int64_t)cols128, K = ranks[k];
  const unsigned __int128 cap = (unsigned __int128)DECOMPRESS_MAX_ELEMS;
  if (fl[0] > cap || fl[1] > cap || fr[0] > cap || fr[1] > cap || (unsigned __int128)K * (rows128 + cols128) > cap)
    return fail(TNB_ERR_UNSUPPORTED, "tt_decompress: ranks too large for this shape");
  T* FL[2] = {ar.template take<T>((size_t)fl[0]), ar.template take<T>((size_t)fl[1])};
  T* FR[2] = {ar.template take<T>((size_t)fr[0]), ar.template take<T>((size_t)fr[1])};
  bool fast = false;
  float *Limg = nullptr, *Rimg = nullptr;
  if constexpr (std::is_same<T, float>::value) {
    fast = expand_tc_shape_ok(M, K, Nc);
    if (fast) {
      Limg = ar.template take<float>(expand_tc_limg_elems(M, K));
      Rimg = ar.template take<float>(expand_tc_rimg_elems(K, Nc));
    }
  }
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "tt_decompress: workspace too small (need %zu bytes)", ar.off);

  const T* L = cores[0];  // F_0 = core_0 as (I_0 x r_1)
  int64_t rows = shape[0];
  for (int j = 1; j < k; ++j) {  // F_j (rows I_j x r_{j+1}) = F_{j-1} (rows x r_j) core_j (r_j x I_j r_{j+1})
    TNB_TRY((gemm_rowmajor<T, T>(rows, shape[j] * ranks[j + 1], ranks[j], L, cores[j], FL[j & 1], st)));
    L = FL[j & 1];
    rows *= shape[j];
  }
  const T* R = cores[N - 1];  // H_{N-1} = core_{N-1} as (r_{N-1} x I_{N-1})
  int64_t cols = shape[N - 1];
  for (int j = N - 2; j >= k; --j) {  // H_j (r_j I_j x cols) = core_j (r_j I_j x r_{j+1}) H_{j+1} (r_{j+1} x cols)
    TNB_TRY((gemm_rowmajor<T, T>(ranks[j] * shape[j], cols, ranks[j + 1], cores[j], R, FR[j & 1], st)));
    R = FR[j & 1];
    cols *= shape[j];
  }
  if constexpr (std::is_same<T, float>::value)
    if (fast && (reinterpret_cast<uintptr_t>(out) & 15u) == 0) return expand_tc<TOut>(L, R, M, K, Nc, out, Limg, Rimg, st);
  return gemm_rowmajor<T, TOut>(M, Nc, K, L, R, out, st);
}

// fp32 cores to fp32, bf16 or fp16; fp64 cores to fp64
inline bool decompress_pair_ok(int core_dtype, int out_dtype) {
  return core_dtype == TNB_F32 ? (out_dtype == TNB_F32 || out_dtype == TNB_BF16 || out_dtype == TNB_F16)
                               : (core_dtype == TNB_F64 && out_dtype == TNB_F64);
}
template <class ArenaT>
inline int tt_decompress_dispatch(ArenaT& ar, bool dry, int core_dtype, int out_dtype, const void* const* cores, int ndim,
                                  const int64_t* shape, const int32_t* ranks, void* out, cudaStream_t st) {
  if (core_dtype == TNB_F64)
    return tt_decompress_impl<double, double>(ar, dry, reinterpret_cast<const double* const*>(cores), ndim, shape, ranks,
                                              static_cast<double*>(out), st);
  const float* const* c32 = reinterpret_cast<const float* const*>(cores);
  if (out_dtype == TNB_BF16)
    return tt_decompress_impl<float, __nv_bfloat16>(ar, dry, c32, ndim, shape, ranks, static_cast<__nv_bfloat16*>(out), st);
  if (out_dtype == TNB_F16)
    return tt_decompress_impl<float, __half>(ar, dry, c32, ndim, shape, ranks, static_cast<__half*>(out), st);
  return tt_decompress_impl<float, float>(ar, dry, c32, ndim, shape, ranks, static_cast<float*>(out), st);
}

}  // namespace tnb
