// Gram matrix G = C^T C of a tall row-major fp32 matrix C (rows x n) on the Hopper tensor cores.
//
//   * row slabs of C are staged HBM -> shared memory by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle,
//     out-of-bounds rows/columns zero-filled by the TMA unit), 4-stage mbarrier ring;
//   * the contraction runs over the ROW index of C, so both operands are "MN-major" views of the very same
//     slab.  tf32 wgmma only takes K-major shared-memory operands, so the products run on the warp-level
//     tensor-core MMA (mma.sync m16n8k8 .tf32, fp32 accumulation in registers) with the fragments read
//     straight out of the swizzled slab (mma_frag_* below: conflict-free, no transpose pass);
//   * G is symmetric: only tiles that touch the upper triangle are computed, and on diagonal tiles the
//     A operand is a sub-block of the B slab (loaded once);
//   * split-K over row ranges across CTAs; partial tiles go registers -> global and are summed in fp64 by a
//     deterministic second kernel (no atomics).
//
// 256 threads = eight MMA warps, a 2 x 4 grid of 64 x tn/4 warp tiles over the 128 x tn output tile; thread 0 also
// issues the TMA loads, TC_STAGES - 1 stages ahead.  (A separate producer warp would make it 288 threads, which the
// register allocator rounds up to 384: 168 registers per thread, too few for the 128 accumulators of a 64 x 64 tile.)
//
// Replaces, for large fp32 unfoldings, the QR of tensor.py:1816 / the Gram of round.py:104-110.
#pragma once
#include <cuda.h>

#include <cstdlib>

#include "common.cuh"

namespace tnb {

constexpr int TC_KC = 32;                       // rows of C per pipeline stage
constexpr int TC_BOX_BYTES = TC_KC * 128;       // one TMA box: 32 fp32 columns x KC rows
constexpr int TC_STAGES = 4;
constexpr int TC_MAX_BOXES = 12;                // 4 (A) + 8 (B)
constexpr int TC_STAGE_BYTES = TC_MAX_BOXES * TC_BOX_BYTES;
constexpr int TC_MMA_WARPS = 8;
constexpr int TC_THREADS = 32 * TC_MMA_WARPS;
constexpr int TC_SMEM_BYTES = TC_STAGES * TC_STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
// Longest run of rows one CTA accumulates in fp32 registers (512 stages = 16384 rows).  The diagonal of a Gram grows with
// the row count while the rounding error of an fp32 sum grows faster; 16384-row partial sums keep that error well below
// the TF32 operand noise the accept rule of the sweep budgets for.
constexpr int64_t TC_MAX_SPLIT_ITERS = 512;

struct GramTcParams {
  int64_t rows;    // contraction length K (rows of both operands)
  int n;           // columns of B (= of A in the symmetric Gram case)
  int m;           // columns of A
  int symmetric;   // 1: A == B, only tiles touching the upper triangle; 0: general A^T B
  int tn;          // B tile width (multiple of 32, <= 256)
  int num_bm;      // ceil(m / 128)
  int num_bn;      // ceil(n / tn)
  int num_tiles;   // kept tiles
  int ksplit;
  int64_t iters_total;      // ceil(rows / KC)
  int64_t iters_per_split;
  float* partial;  // [ksplit][num_tiles][128][tn]
  int fold;              // > 1: the matrix was viewed as (rows/fold) x (fold*n_orig); G = sum of the diagonal blocks
  int n_orig;
  // direct epilogue (general A^T B with ksplit == 1): C = alpha * acc + beta * D + gamma * E written by the
  // MMA warps, no partial tiles and no finalize kernel.  One CTA per output tile: the narrow form used
  // when several decompositions share the GPU (few SMs busy per product instead of all of them).
  int direct;
  float* C;
  const float* D;
  const float* E;
  int ldc, ldd, lde;
  float alpha, beta, gamma;
};

// ---------------------------------------------------------------------------------------------
// PTX wrappers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a wrong box or byte count must surface as an error, never as a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;  // fast path: no clock read when the phase has already completed
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) {  // ~2 s
      printf("tnb200: mbarrier wait timed out (block %d,%d thread %d)\n", blockIdx.x, blockIdx.y, threadIdx.x);
      __trap();
    }
  }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// D += A * B, m16n8k8, tf32 operands as raw fp32 bits (the tensor core ignores the low 13 mantissa bits: truncation).
__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Fragments from an MN-major region written by TMA with CU_TENSOR_MAP_SWIZZLE_128B: boxes of 32 fp32 columns x
// TC_KC rows, box j (columns 32j..32j+31) at base + j*TC_BOX_BYTES; element (row k, column c) of a box sits at
// k*128 + (((c/4) ^ (k%8)) * 16) + (c%4)*4.  The k index of an 8-row step is permuted (fragment k = t -> row 2t,
// k = t+4 -> row 2t+1) identically for both operands, which leaves the product unchanged and makes every fragment
// load hit 32 distinct banks.
__device__ __forceinline__ uint32_t mn_ld(const unsigned char* base, int k, int c) {
  return *reinterpret_cast<const uint32_t*>(base + (c >> 5) * TC_BOX_BYTES + k * 128 + ((((c & 31) >> 2) ^ (k & 7)) << 4) +
                                            ((c & 3) << 2));
}
// A fragment of the 16 x 8 block (columns c0..c0+15 as rows of A^T, rows k0..k0+7); g = lane/4, t = lane%4.
__device__ __forceinline__ void mma_frag_a_mn(const unsigned char* base, int k0, int c0, int g, int t, uint32_t (&a)[4]) {
  a[0] = mn_ld(base, k0 + 2 * t, c0 + g);
  a[1] = mn_ld(base, k0 + 2 * t, c0 + g + 8);
  a[2] = mn_ld(base, k0 + 2 * t + 1, c0 + g);
  a[3] = mn_ld(base, k0 + 2 * t + 1, c0 + g + 8);
}
__device__ __forceinline__ void mma_frag_b_mn(const unsigned char* base, int k0, int c0, int g, int t, uint32_t (&b)[2]) {
  b[0] = mn_ld(base, k0 + 2 * t, c0 + g);
  b[1] = mn_ld(base, k0 + 2 * t + 1, c0 + g);
}

// ---------------------------------------------------------------------------------------------
// The kernel
// ---------------------------------------------------------------------------------------------
// NT = tn / 32: n8 tiles per warp (each warp covers tn / 4 columns)
// Loads of pipeline iteration `it` (rows it_begin + it) into its ring slot, once the MMA warps have released it.
__device__ __forceinline__ void gram_tc_produce(const CUtensorMap* tmap, const CUtensorMap* tmap_b, unsigned char* stage_base,
                                                uint64_t* full_bar, uint64_t* empty_bar, int64_t it, int64_t it_begin,
                                                int nbox_a, int nbox_b, int a_col0, int b_col0) {
  const int stage = (int)(it % TC_STAGES);
  const uint32_t phase = (uint32_t)(it / TC_STAGES) & 1u;
  mbar_wait(&empty_bar[stage], phase ^ 1u);
  unsigned char* sb = stage_base + stage * TC_STAGE_BYTES;
  mbar_expect_tx(&full_bar[stage], (uint32_t)(nbox_a + nbox_b) * TC_BOX_BYTES);
  const int row0 = (int)((it_begin + it) * TC_KC);
  // B boxes first (slots 0..nbox_b), then A boxes (slots 8..11)
  for (int j = 0; j < nbox_b; ++j) tma_load_2d(sb + j * TC_BOX_BYTES, tmap_b, &full_bar[stage], b_col0 + 32 * j, row0);
  for (int j = 0; j < nbox_a; ++j) tma_load_2d(sb + (8 + j) * TC_BOX_BYTES, tmap, &full_bar[stage], a_col0 + 32 * j, row0);
}

template <int NT>
__device__ __forceinline__ void gram_tc_consume(const CUtensorMap* tmap, const CUtensorMap* tmap_b, const GramTcParams& p,
                                                unsigned char* stage_base, uint64_t* full_bar, uint64_t* empty_bar,
                                                int64_t it_begin, int64_t iters, int nbox_a, int a_box, int tile_id,
                                                int split, int a_col0, int b_col0) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int wm = w >> 2, wn = w & 3;      // 64-row half of the tile, quarter of its columns
  const int cm = wm * 64, cn = wn * NT * 8;
  float acc[4][NT][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;

  if (threadIdx.x == 0)
    for (int64_t it = 0; it < TC_STAGES - 1 && it < iters; ++it)
      gram_tc_produce(tmap, tmap_b, stage_base, full_bar, empty_bar, it, it_begin, nbox_a, NT, a_col0, b_col0);
  int stage = 0;
  uint32_t phase = 0;
  for (int64_t it = 0; it < iters; ++it) {
    if (threadIdx.x == 0 && it + TC_STAGES - 1 < iters)  // refill the slot iteration it - 1 used
      gram_tc_produce(tmap, tmap_b, stage_base, full_bar, empty_bar, it + TC_STAGES - 1, it_begin, nbox_a, NT, a_col0,
                      b_col0);
    __syncwarp();
    mbar_wait(&full_bar[stage], phase);
    const unsigned char* sb = stage_base + stage * TC_STAGE_BYTES;
    const unsigned char* sa = sb + a_box * TC_BOX_BYTES;
#pragma unroll
    for (int ks = 0; ks < TC_KC; ks += 8) {
      uint32_t bf[NT][2];
#pragma unroll
      for (int j = 0; j < NT; ++j) mma_frag_b_mn(sb, ks, cn + 8 * j, g, t, bf[j]);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        uint32_t af[4];
        mma_frag_a_mn(sa, ks, cm + 16 * i, g, t, af);
#pragma unroll
        for (int j = 0; j < NT; ++j) mma_tf32(acc[i][j], af[0], af[1], af[2], af[3], bf[j][0], bf[j][1]);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);  // this warp is done reading the slot
    if (++stage == TC_STAGES) { stage = 0; phase ^= 1u; }
  }

  // epilogue: accumulator element (row r, column c) of the 128 x tn tile; c0/c1 and c2/c3 are column pairs
  if (p.direct) {
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int gi = a_col0 + cm + 16 * i + g + 8 * h;
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int gj = b_col0 + cn + 8 * j + 2 * t + e;
            if (gi < p.m && gj < p.n) {
              float x = p.alpha * acc[i][j][2 * h + e];
              if (p.D) x += p.beta * p.D[(size_t)gi * p.ldd + gj];
              if (p.E) x += p.gamma * p.E[(size_t)gi * p.lde + gj];
              p.C[(size_t)gi * p.ldc + gj] = x;
            }
          }
      }
    return;
  }
  float* out = p.partial + ((size_t)split * p.num_tiles + tile_id) * 128 * (size_t)p.tn;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float* orow = out + (size_t)(cm + 16 * i + g + 8 * h) * p.tn + cn + 2 * t;
#pragma unroll
      for (int j = 0; j < NT; ++j)
        *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
    }
}

__global__ void __launch_bounds__(TC_THREADS, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_b,
               const GramTcParams p) {
  extern __shared__ unsigned char tc_smem_raw[];
  // 1024-byte aligned stage buffers (SWIZZLE_128B atoms are 1024 B)
  const uint32_t raw_addr = smem_u32(tc_smem_raw);
  const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
  unsigned char* stage_base = tc_smem_raw + pad;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stage_base + TC_STAGES * TC_STAGE_BYTES);
  uint64_t* empty_bar = full_bar + TC_STAGES;
  int* tile_smem = reinterpret_cast<int*>(empty_bar + TC_STAGES);  // bm, bn

  const int tile_id = blockIdx.x, split = blockIdx.y;

  if (threadIdx.x == 0) {
    // flat tile id -> (bm, bn) among the tiles that touch the upper triangle
    int cnt = 0, fbm = 0, fbn = 0;
    if (p.symmetric) {
      for (int bm = 0; bm < p.num_bm; ++bm)
        for (int bn = 0; bn < p.num_bn; ++bn)
          if ((bn + 1) * p.tn > bm * 128) {
            if (cnt == tile_id) { fbm = bm; fbn = bn; }
            ++cnt;
          }
    } else {
      fbm = tile_id / p.num_bn;
      fbn = tile_id % p.num_bn;
    }
    tile_smem[0] = fbm;
    tile_smem[1] = fbn;
    for (int s = 0; s < TC_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], TC_MMA_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int bm = tile_smem[0], bn = tile_smem[1];
  const int a_col0 = bm * 128, b_col0 = bn * p.tn;
  const int nbox_b = p.tn / 32;
  const bool a_in_b = p.symmetric && (a_col0 >= b_col0) && (a_col0 + 128 <= b_col0 + p.tn);
  const int nbox_a = a_in_b ? 0 : 4;
  const int a_box = a_in_b ? (a_col0 - b_col0) / 32 : 8;  // first box of the A operand in a stage
  const int64_t it_begin = (int64_t)split * p.iters_per_split;
  int64_t it_end = it_begin + p.iters_per_split;
  if (it_end > p.iters_total) it_end = p.iters_total;
  const int64_t iters = it_end > it_begin ? it_end - it_begin : 0;

#define TNB_GRAM_CONSUME(NT)                                                                                    \
  gram_tc_consume<NT>(&tmap, &tmap_b, p, stage_base, full_bar, empty_bar, it_begin, iters, nbox_a, a_box, tile_id, split, \
                      a_col0, b_col0)
  switch (nbox_b) {
    case 1: TNB_GRAM_CONSUME(1); break;
    case 2: TNB_GRAM_CONSUME(2); break;
    case 3: TNB_GRAM_CONSUME(3); break;
    case 4: TNB_GRAM_CONSUME(4); break;
    case 5: TNB_GRAM_CONSUME(5); break;
    case 6: TNB_GRAM_CONSUME(6); break;
    case 7: TNB_GRAM_CONSUME(7); break;
    default: TNB_GRAM_CONSUME(8); break;
  }
#undef TNB_GRAM_CONSUME
}

// Sum the split-K partial tiles in fp64 (fixed order), mirror to the lower triangle.
__global__ void gram_tc_finalize_kernel(const GramTcParams p, double* __restrict__ G, float* __restrict__ Gf) {
  if (p.fold > 1) {  // single 128 x 128 tile; fold the diagonal n_orig x n_orig blocks
    // one WARP per output element: the ksplit * fold terms (hundreds, strided) are dealt to the lanes and combined by a
    // shuffle tree in a fixed order — deterministic like the serial sum, without its 300-deep dependent chain per thread
    const int no = p.n_orig;
    const size_t split_stride = (size_t)p.num_tiles * 128 * p.tn;
    const int lane = threadIdx.x & 31;
    const int warps = (gridDim.x * blockDim.x) >> 5;
    const int nterms = p.ksplit * p.fold;
    for (int idx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; idx < no * no; idx += warps) {
      const int i = idx / no, j = idx % no;
      double s = 0.0;
      for (int t = lane; t < nterms; t += 32) {
        const int z = t / p.fold, a = t - z * p.fold;
        s += (double)p.partial[(size_t)z * split_stride + (size_t)(a * no + i) * p.tn + (a * no + j)];
      }
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) {
        G[idx] = s;
        if (Gf) Gf[idx] = (float)s;
      }
    }
    return;
  }
  const int64_t total = (int64_t)p.n * p.n;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / p.n), j = (int)(idx % p.n);
    const int ii = i <= j ? i : j, jj = i <= j ? j : i;
    const int bm = ii / 128, bn = jj / p.tn;
    // flat index of (bm, bn) among kept tiles: row a keeps the column tiles b >= first(a) = floor(a*128 / tn)
    int tile = 0;
    for (int a = 0; a < bm; ++a) tile += p.num_bn - (a * 128) / p.tn;
    tile += bn - (bm * 128) / p.tn;
    const size_t off = ((size_t)tile * 128 + (ii - bm * 128)) * (size_t)p.tn + (jj - bn * p.tn);
    const size_t split_stride = (size_t)p.num_tiles * 128 * p.tn;
    double s = 0.0;
    for (int z = 0; z < p.ksplit; ++z) s += (double)p.partial[(size_t)z * split_stride + off];
    G[idx] = s;
    if (Gf) Gf[idx] = (float)s;
  }
}

// ---------------------------------------------------------------------------------------------
// Host side
// ---------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled load_encode_tiled() {
  void* f = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &q) == cudaSuccess &&
      q == cudaDriverEntryPointSuccess)
    return reinterpret_cast<PFN_encodeTiled>(f);
  cudaGetLastError();
  return nullptr;
}
inline PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = load_encode_tiled();  // thread-safe one-time initialisation
  return fn;
}

inline bool tc_path_available() {
  const DeviceInfo& di = device_info();
  return di.valid && di.cc_major == 9 && get_encode_tiled() != nullptr;
}

inline bool gram_tc_shape_ok(int64_t rows, int64_t n) {
  return n >= 16 && n % 4 == 0 && n <= 16384 && rows >= 1 && rows < ((int64_t)1 << 31) - 64;
}

inline void gram_tc_plan(int64_t rows, int64_t n, GramTcParams& p, int64_t m_cols = -1) {
  p.rows = rows;
  p.n = (int)n;
  p.symmetric = m_cols < 0 ? 1 : 0;
  p.m = p.symmetric ? (int)n : (int)m_cols;
  int tn = n >= 256 ? 256 : (int)((n + 31) / 32 * 32);
  p.tn = tn;
  p.num_bm = (int)((p.m + 127) / 128);
  p.num_bn = (int)((n + tn - 1) / tn);
  int cnt = 0;
  if (p.symmetric) {
    for (int bm = 0; bm < p.num_bm; ++bm)
      for (int bn = 0; bn < p.num_bn; ++bn)
        if ((bn + 1) * tn > bm * 128) ++cnt;
  } else {
    cnt = p.num_bm * p.num_bn;
  }
  p.num_tiles = cnt;
  p.iters_total = (rows + TC_KC - 1) / TC_KC;
  // split-K factor: at least sms / cnt and enough splits that no fp32 accumulation chain is longer than
  // TC_MAX_SPLIT_ITERS stages (the splits are summed in fp64), then up to 8x that if it fills the last wave of CTAs better
  // while every split keeps >= 64 stages (72 tiles of 262144 rows on 128 SMs: 16 splits, 9 full waves)
  const int sms = usable_sms();
  const int64_t base = std::max<int64_t>(cnt < sms ? sms / cnt : 1, (p.iters_total + TC_MAX_SPLIT_ITERS - 1) / TC_MAX_SPLIT_ITERS);
  int64_t ks = base;
  double best = 0.0;
  for (int64_t k = base; k <= 8 * base && k <= p.iters_total && (k == base || 64 * k <= p.iters_total); ++k) {
    const int64_t ctas = k * cnt, waves = (ctas + sms - 1) / sms;
    const double eff = (double)ctas / (double)(waves * sms);
    if (eff > best + 0.02) { best = eff; ks = k; }
  }
  if (ks > p.iters_total) ks = p.iters_total;
  p.iters_per_split = (p.iters_total + ks - 1) / ks;
  ks = (p.iters_total + p.iters_per_split - 1) / p.iters_per_split;
  p.ksplit = (int)ks;
  p.partial = nullptr;
  p.fold = 1;
  p.n_orig = (int)n;
  p.direct = 0;
  p.C = nullptr;
  p.D = p.E = nullptr;
  p.ldc = p.ldd = p.lde = 0;
  p.alpha = 1.f;
  p.beta = p.gamma = 0.f;
}

// Narrow matrices (n = 32 or 64) are viewed as (rows/f) x 128, f = 128/n: one full-width 128 x 128 tile with
// every TMA box useful (16 KB per stage in flight instead of 8 KB padded with zero boxes); the Gram matrix is
// the sum of the f diagonal n x n blocks.
inline int gram_tc_fold(int64_t rows, int64_t n) {
  if (n >= 128 || n < 32 || 128 % n != 0) return 1;
  const int f = (int)(128 / n);
  return (rows % f == 0) ? f : 1;
}

inline size_t gram_tc_workspace_bytes(int64_t rows, int64_t n) {
  GramTcParams p;
  const int f = gram_tc_fold(rows, n);
  gram_tc_plan(rows / f, n * f, p);
  return align_up((size_t)p.ksplit * p.num_tiles * 128 * p.tn * sizeof(float));
}

inline int encode_rowmajor_f32(CUtensorMap* tmap, const float* ptr, int64_t rows, int64_t cols, int box_rows = TC_KC) {
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * sizeof(float)};
  cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult cr = get_encode_tiled()(tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), gdim, gstride, box,
                                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return fail(TNB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)cr);
  return TNB_OK;
}

// G (n x n fp64) and optionally Gf (fp32 copy) = A^T A, A: rows x n fp32 row-major (device).
inline int gram_tc_f32(const float* A, int64_t rows, int64_t n, double* G, float* Gf, void* ws, size_t ws_bytes,
                       cudaStream_t st) {
  if (!tc_path_available()) return fail(TNB_ERR_UNSUPPORTED, "gram_tc: TMA tensor-core path needs an sm_90 device");
  if (!gram_tc_shape_ok(rows, n)) return fail(TNB_ERR_UNSUPPORTED, "gram_tc: unsupported shape rows=%lld n=%lld", (long long)rows, (long long)n);
  if ((reinterpret_cast<uintptr_t>(A) & 15u) != 0) return fail(TNB_ERR_INVALID, "gram_tc: input must be 16-byte aligned");
  GramTcParams p;
  const int fold = gram_tc_fold(rows, n);
  const int64_t n_in = n;
  rows /= fold;
  n *= fold;
  gram_tc_plan(rows, n, p);
  p.fold = fold;
  p.n_orig = (int)n_in;
  const size_t need = (size_t)p.ksplit * p.num_tiles * 128 * p.tn * sizeof(float);
  if (ws_bytes < need) return fail(TNB_ERR_WORKSPACE, "gram_tc: workspace %zu < %zu", ws_bytes, need);
  p.partial = static_cast<float*>(ws);

  CUtensorMap tmap;
  TNB_TRY(encode_rowmajor_f32(&tmap, A, rows, n));

  static PerDeviceFlag attr_done;
  TNB_CUDA(ensure_dyn_smem(attr_done, gram_tc_kernel, TC_SMEM_BYTES));
  dim3 grid((unsigned)p.num_tiles, (unsigned)p.ksplit);
  gram_tc_kernel<<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(tmap, tmap, p);
  TNB_LAUNCH_CHECK();
  const int64_t total = n_in * n_in * (p.fold > 1 ? 32 : 1);  // folded form: one warp per element
  gram_tc_finalize_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, 4096), 256, 0, st>>>(p, G, Gf);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// General C (m x n) = alpha * A^T B + beta * D + gamma * E on the same kernel: A is K x m, B is K x n,
// both row-major fp32 (TF32 operands, fp32 accumulation).  Used for the filter products G*Y of the
// subspace iteration (G symmetric, so A = G).  Finalize fuses the three-term epilogue.
// ---------------------------------------------------------------------------------------------
__global__ void atb_tc_finalize_kernel(const GramTcParams p, float* __restrict__ C, int ldc, float alpha,
                                       const float* __restrict__ D, int ldd, float beta, const float* __restrict__ E,
                                       int lde, float gamma) {
  const int64_t total = (int64_t)p.m * p.n;
  const size_t split_stride = (size_t)p.num_tiles * 128 * p.tn;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / p.n), j = (int)(idx % p.n);
    const int bm = i / 128, bn = j / p.tn;
    const int tile = bm * p.num_bn + bn;
    const size_t off = ((size_t)tile * 128 + (i - bm * 128)) * (size_t)p.tn + (j - bn * p.tn);
    float s = 0.f;
    for (int z = 0; z < p.ksplit; ++z) s += p.partial[(size_t)z * split_stride + off];
    float v = alpha * s;
    if (D) v += beta * D[(size_t)i * ldd + j];
    if (E) v += gamma * E[(size_t)i * lde + j];
    C[(size_t)i * ldc + j] = v;
  }
}

inline bool atb_tc_shape_ok(int64_t K, int64_t m, int64_t n) {
  return m >= 32 && n >= 32 && m % 4 == 0 && n % 4 == 0 && m <= 65536 && n <= 65536 && K >= 1 && K < ((int64_t)1 << 31) - 64;
}
inline size_t atb_tc_workspace_bytes(int64_t K, int64_t m, int64_t n) {
  GramTcParams p;
  gram_tc_plan(K, n, p, m);
  return align_up((size_t)p.ksplit * p.num_tiles * 128 * p.tn * sizeof(float));
}

inline int atb_tc_f32(const float* A, int64_t K, int64_t m, const float* B, int64_t n, float* C, int ldc, float alpha,
                      const float* D, int ldd, float beta, const float* E, int lde, float gamma, void* ws,
                      size_t ws_bytes, cudaStream_t st, bool narrow = false) {
  if (!tc_path_available()) return fail(TNB_ERR_UNSUPPORTED, "atb_tc: TMA tensor-core path needs an sm_90 device");
  if (!atb_tc_shape_ok(K, m, n)) return fail(TNB_ERR_UNSUPPORTED, "atb_tc: unsupported shape K=%lld m=%lld n=%lld", (long long)K, (long long)m, (long long)n);
  if (((reinterpret_cast<uintptr_t>(A) | reinterpret_cast<uintptr_t>(B)) & 15u) != 0)
    return fail(TNB_ERR_INVALID, "atb_tc: operands must be 16-byte aligned");
  GramTcParams p;
  gram_tc_plan(K, n, p, m);
  if (narrow) {  // one CTA per output tile, epilogue writes C directly
    p.ksplit = 1;
    p.iters_per_split = p.iters_total;
    p.direct = 1;
    p.C = C; p.ldc = ldc; p.alpha = alpha;
    p.D = beta != 0.f ? D : nullptr; p.ldd = ldd; p.beta = beta;
    p.E = gamma != 0.f ? E : nullptr; p.lde = lde; p.gamma = gamma;
  }
  const size_t need = narrow ? 0 : (size_t)p.ksplit * p.num_tiles * 128 * p.tn * sizeof(float);
  if (ws_bytes < need) return fail(TNB_ERR_WORKSPACE, "atb_tc: workspace %zu < %zu", ws_bytes, need);
  p.partial = static_cast<float*>(ws);
  CUtensorMap ta, tb;
  TNB_TRY(encode_rowmajor_f32(&ta, A, K, m));
  TNB_TRY(encode_rowmajor_f32(&tb, B, K, n));
  static PerDeviceFlag attr_done;
  TNB_CUDA(ensure_dyn_smem(attr_done, gram_tc_kernel, TC_SMEM_BYTES));
  dim3 grid((unsigned)p.num_tiles, (unsigned)p.ksplit);
  gram_tc_kernel<<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(ta, tb, p);
  TNB_LAUNCH_CHECK();
  if (narrow) return TNB_OK;
  const int64_t total = m * n;
  atb_tc_finalize_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, 4096), 256, 0, st>>>(p, C, ldc, alpha, D, ldd,
                                                                                                 beta, E, lde, gamma);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

}  // namespace tnb
