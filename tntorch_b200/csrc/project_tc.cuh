// Tall-skinny projection C (rows x r) = A (rows x K) * V (K x r) on the Hopper tensor cores at fp32 accuracy
// ("3xTF32": A = A_hi + A_lo, V = V_hi + V_lo, C = A_hi V_hi + A_hi V_lo + A_lo V_hi, error ~2^-21 relative,
// i.e. the accuracy class of an fp32 FFMA product — a plain TF32 projection would put a 2^-11 relative error
// straight into the reconstruction).  This is the "C <- C V_r" step of the sweep (round.py:181, tensor.py:2081-2083).
//
//   * A row blocks (128 rows x 32 k) are staged by TMA (K-major, SWIZZLE_128B) into a deep mbarrier ring (11 x 16 KB
//     when V fits in shared memory, else 8 x 24 KB with the V chunk riding in the stage); V_hi^T / V_lo^T are
//     prepared once (split_v_kernel) and staged as K-major tiles of npad rows each;
//   * eight MMA warps, 16 rows of the block each, read their A fragments from the swizzled tile (conflict-free),
//     split them in registers (A_lo = A - trunc_tf32(A); the tensor core truncates the raw bits of A_hi itself) and
//     issue the three products per 8-wide k-step with mma.sync m16n8k8 .tf32; every 32-wide chunk is folded into an
//     fp32 running sum so that the accumulation error does not grow with K;
//   * persistent CTAs, static round-robin over row blocks; each warp stores its 16 x r piece of C from registers.
//
// Two more layouts serve the K-blocked carry of the sweep (the next step's matrix M, rows' x n', stored as wgmma's K-major
// core matrices [rows'/8][n'/8][2][8][4] so that its Gram loads K-major operands, gram_tc.cuh):
//   * PT_OUT_KBLOCKED writes C in that layout.  C's row a * inner + i is row a of M, columns i * r .. i * r + r - 1.  A
//     row block is 8 a's x 16 i's (warp w: a0 + w) loaded by a 3-D map as the same 128 x 32 swizzled tile, so the
//     products are unchanged; its output is one contiguous 16 x r x 8 run of the carry, staged through shared memory past
//     the ring (the ring keeps its depth) and stored with 16-byte writes.
//   * PT_IN_KBLOCKED reads A in that layout (a 1 KB run per 8 rows and 32 columns, no swizzle) and writes C row-major.
//
// bf16 A (the dense TT-SVD's input, step 0 only), V and C fp32: V is split once into three bf16 terms v1 = bf16(v),
// v2 = bf16(v - v1), v3 = bf16(v - v1 - v2), which together hold fp32's 24 significand bits, and every 16-wide k-step
// issues mma.sync m16n8k16 .bf16 for C v3, C v2, C v1 in that order.  The products of two bf16 values are exact and
// accumulate in fp32, so C comes out at fp32 accuracy without an fp32 image of A.  A chunk is 64 bf16 columns: the
// same 128-byte swizzled rows as 32 fp32 columns, so the tiles, the ring, the schedule and both output layouts are
// shared, and the 32-bit fragment words sit where the tf32 fragments sit.
//
// fp16 A takes the same path with mma.sync m16n8k16 .f16 and two terms of V, scaled per column: fp16's smallest normal
// is 2^-14, and the second term of an orthonormal V's entries (|v| ~ 0.02-0.1, remainder ~|v| 2^-11) would fall below
// it.  split_v_f16_kernel picks for column j a power of two s_j that puts max_i |V_ij| s_j in [2^14, 2^15) and stores
// v1 = fp16(v s_j), v2 = fp16(v s_j - v1) (22 significant bits, what V_hi + V_lo carry on the fp32 path) and 1 / s_j;
// the epilogue multiplies column j by 1 / s_j, which is exact.  The products stay exact in fp32
// (|A| |v s| <= 65504 * 2^15 < 2^31).  The scale is chosen on the device: the speculative sweep enqueues the projection
// without a host read.
//
// fp8 A (e4m3 or e5m2) uses those two scaled fp16 terms of V as they are.  A chunk is 128 fp8 columns (TMA boxes of
// UINT8, the same 128-byte swizzled rows, so A's tiles and ring are the fp32 path's), and each V term of a chunk is two
// 64-column fp16 boxes.  A fragment word (km_ld, the tf32 access pattern) holds four consecutive k; it is widened to two
// f16x2 words in registers (exact) and feeds two mma.sync m16n8k16 .f16 whose k order is permuted the same way for A and
// V: word w of the row pairs with the 8-byte V load of k 4w .. 4w + 3.  An fp8 value times an fp16 term has at most
// 4 + 11 significant bits, so the products stay exact in fp32 (|A| |v s| <= 57344 * 2^15).  K need only be a multiple of
// 16 and >= 64: the A box reads zeros past K, the V boxes past K are not loaded, and the 32-wide k-steps past K are
// skipped (K = 64, the 64^5 step-0 shape, fills half an A box and one V box per term).
#pragma once
#include <type_traits>

#include "gram_tc.cuh"

namespace tnb {

constexpr int PT_BM = 128, PT_KC = 32, PT_MAX_STAGES = 12, PT_MMA_WARPS = 8, PT_THREADS = 32 * (1 + PT_MMA_WARPS);
constexpr int PT_A_BYTES = PT_BM * PT_KC * 4;      // 16 KB
constexpr int PT_MAX_N = 64;                        // r padded to a multiple of 16, <= 64
constexpr int PT_RING_BYTES = 192 * 1024;           // stage ring (+ resident V when it fits)
constexpr int PT_STG_MAX_BYTES = 29 * 1024;         // PT_OUT_KBLOCKED output staging (r <= 48), past the ring
constexpr int PT_SMEM_BYTES = PT_RING_BYTES + PT_STG_MAX_BYTES + 1024 + 256;
constexpr int PT_VRES_MAX_BYTES = 32 * 1024;        // V_hi|V_lo kept in shared memory for the whole kernel up to this size
constexpr int PT_ROWMAJOR = 0, PT_OUT_KBLOCKED = 1, PT_IN_KBLOCKED = 2;

struct ProjTcParams {
  int64_t rows;
  int K;
  int r;       // real output columns
  int npad;    // r rounded up to a multiple of 16
  int64_t num_row_blocks;
  int nk;      // K chunks
  int vres;         // 1: all V chunks resident in shared memory (small K), stages hold A only
  int stage_bytes;  // 16 KB (+ 2*npad*128 B of V chunk when streaming V)
  int nstages;      // ring depth that fits PT_RING_BYTES: the HBM latency needs >= ~140 KB in flight per SM
  float* C;
  int inner16;      // PT_OUT_KBLOCKED: inner / 16 row blocks per 8 rows of M
  int64_t out_ld;   // PT_OUT_KBLOCKED: n' = inner * r
  const float* vscale;  // fp16 A: 1 / s_j of the npad columns of V (split_v_f16_kernel), else nullptr
};

// element (row m, column k) of a 128 x 32 tile of a K-blocked matrix: 16 runs of 32 columns x 8 rows, each four 8 x 8
// blocks of two 4-row core matrices (column-minor)
__device__ __forceinline__ uint32_t kb_ld(const unsigned char* base, int m, int k) {
  return *reinterpret_cast<const uint32_t*>(
      base + (((m >> 3) << 8) + (((((k >> 3) << 1) + ((m & 7) >> 2)) << 5) + ((k & 7) << 2) + (m & 3)) << 2));
}
// Staging of a PT_OUT_KBLOCKED tile: warp w's 16 x R piece at w * SW + row * RS + column.  RS = R + 8 makes the float2
// stores of each half-warp conflict-free, SW = 16 RS + 4 (4 SW = 16 mod 32 banks) the gathers of the copy-out.
template <int R>
struct PtStage {
  static constexpr int RS = R + 8, SW = 16 * RS + 4;
  static_assert(8 * SW * 4 <= PT_STG_MAX_BYTES, "staging must fit past the ring");
};


// D += A * B, m16n8k16, 16-bit operands of type T16 (bf16 or fp16, two per 32-bit word, the lower k in the low half),
// fp32 accumulation.
template <typename T16>
__device__ __forceinline__ void mma_k16(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                        uint32_t b1) {
  static_assert(std::is_same<T16, __half>::value || std::is_same<T16, __nv_bfloat16>::value, "bf16 or fp16 operands");
  if constexpr (std::is_same<T16, __half>::value)
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
  else
    asm volatile(
        "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
        "{%0, %1, %2, %3};"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// Per A element type: columns per 128-byte chunk row and the number of V terms (fp32: V_hi, V_lo; bf16: v1, v2, v3;
// fp16 and fp8: the scaled fp16 v1, v2), their element type TV and the 128-byte V boxes per term and chunk.
template <typename TA>
struct PtType {
  static constexpr int KC = 128 / (int)sizeof(TA);
  static constexpr int VTERMS = std::is_same<TA, __nv_bfloat16>::value ? 3 : 2;
  static constexpr bool SCALED = sizeof(TA) <= 2 && !std::is_same<TA, __nv_bfloat16>::value;  // per-column 2^e scale of V
  using TV = std::conditional_t<sizeof(TA) == 1, __half, TA>;
  static constexpr int VSUB = sizeof(TA) == 1 ? 2 : 1;
};

// fp8 A: V boxes of chunk kc that start inside K (the second 64 columns of the last chunk may lie past it)
__device__ __forceinline__ int pt_f8_vsub(const ProjTcParams& p, int kc) { return kc * 128 + 64 < p.K ? 2 : 1; }

// element (row m, column k) of a K-major tile of 32 fp32 columns written by TMA with SWIZZLE_128B
__device__ __forceinline__ uint32_t km_ld(const unsigned char* base, int m, int k) {
  return *reinterpret_cast<const uint32_t*>(base + m * 128 + ((((k >> 2) ^ (m & 7))) << 4) + ((k & 3) << 2));
}

// fp8 A: the fp16 values of one V term at column `col`, k 4w .. 4w + 3 of the chunk (two f16x2 words), from the term's
// two boxes of 64 columns (box w / 16: npad rows of 128 bytes, 128-byte swizzle)
__device__ __forceinline__ uint2 pt_f8_vld(const unsigned char* v, int npad, int col, int w) {
  return *reinterpret_cast<const uint2*>(v + (w >> 4) * npad * 128 + col * 128 + ((((w & 15) >> 1) ^ (col & 7)) << 4) +
                                         ((w & 1) << 3));
}

// fp8 A: TMA loads of V chunk kc, both terms and the boxes pt_f8_vsub keeps, into dst as [term][box][npad rows][128 B]
__device__ __forceinline__ void pt_f8_load_v(unsigned char* dst, const CUtensorMap* th, const CUtensorMap* tl,
                                             uint64_t* bar, const ProjTcParams& p, int kc) {
  for (int h = 0; h < pt_f8_vsub(p, kc); ++h) {
    tma_load_2d(dst + h * p.npad * 128, th, bar, kc * 128 + 64 * h, 0);
    tma_load_2d(dst + (2 + h) * p.npad * 128, tl, bar, kc * 128 + 64 * h, 0);
  }
}

// NT = npad / 8 n8 tiles
template <int NT, int MODE, typename TA>
__device__ __forceinline__ void project_tc_consume(const ProjTcParams& p, const unsigned char* stage_base,
                                                   const unsigned char* v_res, float* stg, uint64_t* full_bar,
                                                   uint64_t* empty_bar, uint64_t* v_bar, int64_t total_items) {
  const int w = (threadIdx.x >> 5) - 1, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int m0 = 16 * w;
  const int vchunk_bytes = PtType<TA>::VTERMS * PtType<TA>::VSUB * p.npad * 128;
  const int vlo_off = PtType<TA>::VSUB * p.npad * 128;  // between V terms
  if (p.vres && total_items > 0) mbar_wait(v_bar, 0);
  float vsc[NT][2];  // fp16 A: 1 / s_j of this thread's output columns 8j + 2t, 8j + 2t + 1
  if constexpr (PtType<TA>::SCALED)
#pragma unroll
    for (int j = 0; j < NT; ++j) vsc[j][0] = p.vscale[8 * j + 2 * t], vsc[j][1] = p.vscale[8 * j + 2 * t + 1];
  float out[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j)
#pragma unroll
    for (int e = 0; e < 4; ++e) out[j][e] = 0.f;
  int stage = 0, kc = 0;
  uint32_t phase = 0;
  int64_t rb = blockIdx.x;
  for (int64_t item = 0; item < total_items; ++item) {
    mbar_wait(&full_bar[stage], phase);
    const unsigned char* sa = stage_base + (size_t)stage * p.stage_bytes;
    const unsigned char* vh = p.vres ? v_res + (size_t)kc * vchunk_bytes : sa + PT_A_BYTES;
    const unsigned char* vl = vh + vlo_off;
    float acc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[j][e] = 0.f;
#pragma unroll
    for (int ks = 0; ks < PT_KC; ks += 8) {  // 8 fragment words: 8 fp32, 16 bf16 / fp16 or 32 fp8 columns
      if constexpr (sizeof(TA) == 1)
        if (kc * 128 + 4 * ks >= p.K) break;  // past K: A and V are zero there
      uint32_t a[4], lo[4];
      if constexpr (MODE == PT_IN_KBLOCKED) {
        a[0] = kb_ld(sa, m0 + g, ks + t);
        a[1] = kb_ld(sa, m0 + g + 8, ks + t);
        a[2] = kb_ld(sa, m0 + g, ks + t + 4);
        a[3] = kb_ld(sa, m0 + g + 8, ks + t + 4);
      } else {
        a[0] = km_ld(sa, m0 + g, ks + t);
        a[1] = km_ld(sa, m0 + g + 8, ks + t);
        a[2] = km_ld(sa, m0 + g, ks + t + 4);
        a[3] = km_ld(sa, m0 + g + 8, ks + t + 4);
      }
      if constexpr (sizeof(TA) == 1) {  // fp8: C v2, C v1 (scaled fp16 terms), k 4w, 4w + 1 in x, 4w + 2, 4w + 3 in y
        uint32_t x[4], y[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) f8x4_to_f16x2<TA>(a[i], x[i], y[i]);
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const int col = 8 * j + g;
          const uint2 l0 = pt_f8_vld(vl, p.npad, col, ks + t), l1 = pt_f8_vld(vl, p.npad, col, ks + t + 4);
          const uint2 h0 = pt_f8_vld(vh, p.npad, col, ks + t), h1 = pt_f8_vld(vh, p.npad, col, ks + t + 4);
          mma_k16<__half>(acc[j], x[0], x[1], x[2], x[3], l0.x, l1.x);
          mma_k16<__half>(acc[j], y[0], y[1], y[2], y[3], l0.y, l1.y);
          mma_k16<__half>(acc[j], x[0], x[1], x[2], x[3], h0.x, h1.x);
          mma_k16<__half>(acc[j], y[0], y[1], y[2], y[3], h0.y, h1.y);
        }
      } else if constexpr (sizeof(TA) == 2) {  // bf16: C v3, C v2, C v1; fp16: C v2, C v1 (scaled terms)
        const unsigned char* v3 = vl + vlo_off;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          if constexpr (PtType<TA>::VTERMS == 3)
            mma_k16<TA>(acc[j], a[0], a[1], a[2], a[3], km_ld(v3, 8 * j + g, ks + t), km_ld(v3, 8 * j + g, ks + t + 4));
          mma_k16<TA>(acc[j], a[0], a[1], a[2], a[3], km_ld(vl, 8 * j + g, ks + t), km_ld(vl, 8 * j + g, ks + t + 4));
          mma_k16<TA>(acc[j], a[0], a[1], a[2], a[3], km_ld(vh, 8 * j + g, ks + t), km_ld(vh, 8 * j + g, ks + t + 4));
        }
      } else {
#pragma unroll
        for (int i = 0; i < 4; ++i)
          lo[i] = __float_as_uint(__uint_as_float(a[i]) - __uint_as_float(a[i] & 0xFFFFE000u));
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const uint32_t bh0 = km_ld(vh, 8 * j + g, ks + t), bh1 = km_ld(vh, 8 * j + g, ks + t + 4);
          const uint32_t bl0 = km_ld(vl, 8 * j + g, ks + t), bl1 = km_ld(vl, 8 * j + g, ks + t + 4);
          mma_tf32(acc[j], a[0], a[1], a[2], a[3], bl0, bl1);      // A_hi V_lo
          mma_tf32(acc[j], lo[0], lo[1], lo[2], lo[3], bh0, bh1);  // A_lo V_hi
          mma_tf32(acc[j], a[0], a[1], a[2], a[3], bh0, bh1);      // A_hi V_hi
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[stage]);
    if (++stage == p.nstages) { stage = 0; phase ^= 1u; }
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) out[j][e] += acc[j][e];
    if (++kc < p.nk) continue;
    // row block complete: rows m0+g (c0, c1) and m0+g+8 (c2, c3), columns 8j+2t, 8j+2t+1
    kc = 0;
    if constexpr (PtType<TA>::SCALED)  // undo the column scale of V: a power of two, exact
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) out[j][e] *= vsc[j][e & 1];
    if constexpr (MODE == PT_OUT_KBLOCKED) {  // r == npad
      constexpr int R = 8 * NT, RS = PtStage<R>::RS, SW = PtStage<R>::SW;
      asm volatile("bar.sync 1, %0;" ::"n"(PT_MMA_WARPS * 32) : "memory");  // the last copy-out has read the staging
      float* sw = stg + w * SW;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < NT; ++j)
          *reinterpret_cast<float2*>(sw + (g + 8 * h) * RS + 8 * j + 2 * t) = make_float2(out[j][2 * h], out[j][2 * h + 1]);
      asm volatile("bar.sync 1, %0;" ::"n"(PT_MMA_WARPS * 32) : "memory");
      // element (row ii of warp w, column col) is row a0 + w of M, column (i0 + ii) * R + col = (i0 * R) + pi: word
      // ((pi / 8) * 2 + w / 4) * 32 + (pi % 8) * 4 + w % 4 of the run that starts at M row group a0 / 8, column i0 * R
      float* dst = p.C + ((rb / p.inner16) * p.out_ld + (rb % p.inner16) * 16 * R) * 8;
      for (int q = threadIdx.x - 32; q < 32 * R; q += PT_MMA_WARPS * 32) {
        const int pi = ((q >> 4) << 3) + (q & 7);
        const float* src = stg + ((q >> 3) & 1) * 4 * SW + (pi / R) * RS + pi % R;
        *reinterpret_cast<float4*>(dst + 4 * (int64_t)q) = make_float4(src[0], src[SW], src[2 * SW], src[3 * SW]);
      }
    } else {
    const int64_t row0 = rb * PT_BM;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t grow = row0 + m0 + g + 8 * h;
      if (grow < p.rows) {
        float* crow = p.C + grow * p.r;
#pragma unroll
        for (int j = 0; j < NT; ++j) {
          const int c = 8 * j + 2 * t;
          if ((p.r & 1) == 0) {
            if (c < p.r) *reinterpret_cast<float2*>(crow + c) = make_float2(out[j][2 * h], out[j][2 * h + 1]);
          } else {
            if (c < p.r) crow[c] = out[j][2 * h];
            if (c + 1 < p.r) crow[c + 1] = out[j][2 * h + 1];
          }
        }
      }
    }
    }
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) out[j][e] = 0.f;
    rb += gridDim.x;
  }
}

// tmap_v3: the third V term (bf16 A only).
template <int MODE, typename TA>
__global__ void __launch_bounds__(PT_THREADS, 1)
project_tc_kernel(const __grid_constant__ CUtensorMap tmap_a, const __grid_constant__ CUtensorMap tmap_vhi,
                  const __grid_constant__ CUtensorMap tmap_vlo, const __grid_constant__ CUtensorMap tmap_v3,
                  const ProjTcParams p) {
  constexpr int VT = PtType<TA>::VTERMS;
  extern __shared__ unsigned char pt_smem_raw[];
  const uint32_t raw_addr = smem_u32(pt_smem_raw);
  const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
  unsigned char* stage_base = pt_smem_raw + pad;
  unsigned char* v_res = stage_base + (size_t)p.nstages * p.stage_bytes;   // resident V (vres): nk x [V_hi; V_lo] chunks
  float* stg = reinterpret_cast<float*>(stage_base + PT_RING_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stage_base + PT_RING_BYTES + PT_STG_MAX_BYTES);
  uint64_t* empty_bar = full_bar + PT_MAX_STAGES;
  uint64_t* v_bar = empty_bar + PT_MAX_STAGES;
  constexpr bool F8 = sizeof(TA) == 1;
  const int vchunk_bytes = VT * PtType<TA>::VSUB * p.npad * 128;

  const int warp_idx = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < PT_MAX_STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], PT_MMA_WARPS);
    }
    mbar_init(v_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int64_t my_blocks = (p.num_row_blocks - blockIdx.x + gridDim.x - 1) / gridDim.x;  // may be 0
  const int64_t total_items = my_blocks * p.nk;

  if (warp_idx == 0) {
    // ================= TMA producer =================
    if (lane == 0) {
      if constexpr (F8) {
        if (p.vres && total_items > 0) {
          uint32_t bytes = 0;
          for (int kc = 0; kc < p.nk; ++kc) bytes += (uint32_t)(VT * pt_f8_vsub(p, kc) * p.npad * 128);
          mbar_expect_tx(v_bar, bytes);
          for (int kc = 0; kc < p.nk; ++kc) pt_f8_load_v(v_res + (size_t)kc * vchunk_bytes, &tmap_vhi, &tmap_vlo, v_bar, p, kc);
        }
      } else if (p.vres && total_items > 0) {
        mbar_expect_tx(v_bar, (uint32_t)(p.nk * vchunk_bytes));
        for (int kc = 0; kc < p.nk; ++kc) {
          tma_load_2d(v_res + (size_t)kc * vchunk_bytes, &tmap_vhi, v_bar, kc * PtType<TA>::KC, 0);
          tma_load_2d(v_res + (size_t)kc * vchunk_bytes + p.npad * 128, &tmap_vlo, v_bar, kc * PtType<TA>::KC, 0);
          if (VT == 3) tma_load_2d(v_res + (size_t)kc * vchunk_bytes + 2 * p.npad * 128, &tmap_v3, v_bar, kc * PtType<TA>::KC, 0);
        }
      }
      const uint32_t tx_bytes = (uint32_t)PT_A_BYTES + (p.vres ? 0u : (uint32_t)vchunk_bytes);
      int stage = 0;
      uint32_t phase = 0;
      int kc = 0;
      int rb = (int)blockIdx.x;           // rows < 2^31 (checked on the host)
      for (int64_t item = 0; item < total_items; ++item) {
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        unsigned char* sb = stage_base + (size_t)stage * p.stage_bytes;
        if constexpr (F8)
          mbar_expect_tx(&full_bar[stage],
                         (uint32_t)PT_A_BYTES + (p.vres ? 0u : (uint32_t)(VT * pt_f8_vsub(p, kc) * p.npad * 128)));
        else
          mbar_expect_tx(&full_bar[stage], tx_bytes);
        constexpr int KC = PtType<TA>::KC;
        if (MODE == PT_OUT_KBLOCKED)
          tma_load_3d(sb, &tmap_a, &full_bar[stage], kc * KC, (rb % p.inner16) * 16, (rb / p.inner16) * 8);
        else if (MODE == PT_IN_KBLOCKED)
          tma_load_2d(sb, &tmap_a, &full_bar[stage], kc * KC * 8, rb * (PT_BM / 8));
        else
          tma_load_2d(sb, &tmap_a, &full_bar[stage], kc * KC, rb * PT_BM);
        if constexpr (F8) {
          if (!p.vres) pt_f8_load_v(sb + PT_A_BYTES, &tmap_vhi, &tmap_vlo, &full_bar[stage], p, kc);
        } else if (!p.vres) {
          tma_load_2d(sb + PT_A_BYTES, &tmap_vhi, &full_bar[stage], kc * KC, 0);
          tma_load_2d(sb + PT_A_BYTES + p.npad * 128, &tmap_vlo, &full_bar[stage], kc * KC, 0);  // rows npad..2npad-1
          if (VT == 3) tma_load_2d(sb + PT_A_BYTES + 2 * p.npad * 128, &tmap_v3, &full_bar[stage], kc * KC, 0);
        }
        if (++kc == p.nk) { kc = 0; rb += (int)gridDim.x; }
        if (++stage == p.nstages) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }
  switch (p.npad) {
    case 16: project_tc_consume<2, MODE, TA>(p, stage_base, v_res, stg, full_bar, empty_bar, v_bar, total_items); break;
    case 32: project_tc_consume<4, MODE, TA>(p, stage_base, v_res, stg, full_bar, empty_bar, v_bar, total_items); break;
    case 48: project_tc_consume<6, MODE, TA>(p, stage_base, v_res, stg, full_bar, empty_bar, v_bar, total_items); break;
    default:  // r <= 48 with a K-blocked output (project_tc)
      if constexpr (MODE != PT_OUT_KBLOCKED)
        project_tc_consume<8, MODE, TA>(p, stage_base, v_res, stg, full_bar, empty_bar, v_bar, total_items);
      break;
  }
}

// Vt_hi / Vt_lo (npad x K, row-major, K contiguous) from V (K x r): hi = tf32-truncated V, lo = V - hi.
__global__ void split_v_kernel(const float* __restrict__ V, int K, int r, int npad, float* __restrict__ Vhi,
                               float* __restrict__ Vlo) {
  const int total = npad * K;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int j = idx / K, k = idx % K;
    float v = 0.f;
    if (j < r) v = V[(size_t)k * r + j];
    const float hi = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    Vhi[idx] = hi;
    Vlo[idx] = v - hi;
  }
}

// v1, v2, v3 (npad x K bf16 each, K contiguous) from V (K x r): three round-to-nearest bf16 terms of v.
__global__ void split_v_bf16_kernel(const float* __restrict__ V, int K, int r, int npad, __nv_bfloat16* __restrict__ V1,
                                    __nv_bfloat16* __restrict__ V2, __nv_bfloat16* __restrict__ V3) {
  const int total = npad * K;
  for (int idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int j = idx / K, k = idx % K;
    float v = 0.f;
    if (j < r) v = V[(size_t)k * r + j];
    const __nv_bfloat16 b1 = __float2bfloat16_rn(v);
    const float r1 = v - __bfloat162float(b1);
    const __nv_bfloat16 b2 = __float2bfloat16_rn(r1);
    V1[idx] = b1;
    V2[idx] = b2;
    V3[idx] = __float2bfloat16_rn(r1 - __bfloat162float(b2));
  }
}

// v1, v2 (npad x K fp16 each, K contiguous) and inv_scale[j] = 1 / s_j from V (K x r), one block per column j:
// s_j = 2^(15 - e) with max_i |V_ij| = f 2^e, f in [0.5, 1), so that max_i |V_ij| s_j lies in [2^14, 2^15) and the
// second term stays clear of fp16's subnormals.  The exponent is clamped so that s_j and 1 / s_j are normal fp32 values.
__global__ void __launch_bounds__(256) split_v_f16_kernel(const float* __restrict__ V, int K, int r, __half* __restrict__ V1,
                                                          __half* __restrict__ V2, float* __restrict__ inv_scale) {
  __shared__ float red[8];
  const int j = blockIdx.x;
  float m = 0.f;
  if (j < r)
    for (int k = threadIdx.x; k < K; k += blockDim.x) m = fmaxf(m, fabsf(V[(size_t)k * r + j]));
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int w = 1; w < 8; ++w) m = fmaxf(m, red[w]);
  int e = 0;
  frexpf(m, &e);
  const int sh = m > 0.f ? min(max(15 - e, -126), 126) : 0;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float v = j < r ? ldexpf(V[(size_t)k * r + j], sh) : 0.f;  // exact: a power-of-two scale
    const __half h1 = __float2half_rn(v);
    V1[(size_t)j * K + k] = h1;
    V2[(size_t)j * K + k] = __float2half_rn(v - __half2float(h1));
  }
  if (threadIdx.x == 0) inv_scale[j] = ldexpf(1.f, -sh);
}

// fp32 A: K % 4 == 0 and K >= 32; bf16 / fp16 A: K % 8 == 0 and K >= 64 (16-byte rows, one full 128-byte chunk); fp8 A:
// K % 16 == 0 and K >= 64 (16-byte rows, one full V box).
template <typename TA = float>
inline bool project_tc_shape_ok(int64_t rows, int64_t K, int64_t r, const void* A, const void* C) {
  constexpr int KMIN = sizeof(TA) == 1 ? 64 : PtType<TA>::KC;
  return r >= 1 && r <= PT_MAX_N && K % (16 / (int)sizeof(TA)) == 0 && K >= KMIN && K <= (1 << 24) && rows >= 128 &&
         rows < ((int64_t)1 << 31) - 256 && (reinterpret_cast<uintptr_t>(A) & 15u) == 0 &&
         (reinterpret_cast<uintptr_t>(C) & 15u) == 0;
}
// the V terms, then (fp16 / fp8 A) the npad inverse column scales
template <typename TA = float>
inline size_t project_tc_workspace_bytes(int64_t K, int64_t r) {
  const int64_t npad = (r + 15) / 16 * 16;
  return PtType<TA>::VTERMS * align_up((size_t)npad * K * sizeof(typename PtType<TA>::TV)) +
         (PtType<TA>::SCALED ? align_up((size_t)npad * sizeof(float)) : 0);
}

// boxes of 128 bytes (32 fp32, 64 bf16 / fp16 or 128 fp8 columns) x box_rows rows
template <typename T = float>
inline int encode_kmajor_f32(CUtensorMap* tmap, const T* ptr, int64_t rows, int64_t cols, int box_rows) {
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * sizeof(T)};
  cuuint32_t box[2] = {(cuuint32_t)PtType<T>::KC, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult cr = get_encode_tiled()(tmap, tma_dtype<T>(), 2, const_cast<T*>(ptr), gdim, gstride, box,
                                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return fail(TNB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)cr);
  return TNB_OK;
}

// C (rows x r) = A (rows x K) V (K x r); ws: project_tc_workspace_bytes<TA>(K, r).  TA: float, __nv_bfloat16, __half,
// __nv_fp8_e4m3 or __nv_fp8_e5m2.
//   layout PT_ROWMAJOR:     A and C row-major;
//   layout PT_OUT_KBLOCKED: A row-major, C stored as the K-blocked (gram_tc.cuh) (rows / inner) x (inner * r) matrix;
//                           needs inner % 16 == 0, rows % (8 * inner) == 0, r % 16 == 0, r <= 48;
//   layout PT_IN_KBLOCKED:  A stored K-blocked (rows % 8 == 0, K % 8 == 0), C row-major (fp32 A only).
template <typename TA>
inline int project_tc(const TA* A, int64_t rows, int64_t K, const float* V, int r, float* C, void* ws, size_t ws_bytes,
                      cudaStream_t st, int layout = PT_ROWMAJOR, int64_t inner = 0) {
  constexpr bool BF16 = std::is_same<TA, __nv_bfloat16>::value, F16 = std::is_same<TA, __half>::value;
  constexpr bool F8 = sizeof(TA) == 1;
  constexpr int KC = PtType<TA>::KC, VT = PtType<TA>::VTERMS;
  using TV = typename PtType<TA>::TV;
  if (!tc_path_available()) return fail(TNB_ERR_UNSUPPORTED, "project_tc: needs an sm_90 device");
  if (!project_tc_shape_ok<TA>(rows, K, r, A, C)) return fail(TNB_ERR_UNSUPPORTED, "project_tc: unsupported shape");
  if (layout == PT_OUT_KBLOCKED && !(inner >= 16 && inner % 16 == 0 && rows % (8 * inner) == 0 && r % 16 == 0 && r <= 48))
    return fail(TNB_ERR_UNSUPPORTED,
                "project_tc: K-blocked output needs inner %% 16 == 0, rows %% (8 inner) == 0, r %% 16 == 0, r <= 48");
  if (layout == PT_IN_KBLOCKED && (sizeof(TA) != 4 || rows % 8 != 0 || K % 8 != 0))
    return fail(TNB_ERR_UNSUPPORTED, "project_tc: K-blocked input needs fp32, rows %% 8 == 0 and K %% 8 == 0");
  if (ws_bytes < project_tc_workspace_bytes<TA>(K, r)) return fail(TNB_ERR_WORKSPACE, "project_tc: workspace too small");
  ProjTcParams p;
  p.rows = rows; p.K = (int)K; p.r = r; p.npad = (r + 15) / 16 * 16;
  p.num_row_blocks = (rows + PT_BM - 1) / PT_BM;
  p.nk = (int)((K + KC - 1) / KC);
  p.C = C;
  p.inner16 = layout == PT_OUT_KBLOCKED ? (int)(inner / 16) : 1;
  p.out_ld = layout == PT_OUT_KBLOCKED ? inner * r : 0;
  const int vchunk = VT * PtType<TA>::VSUB * p.npad * 128;
  p.vres = ((int64_t)p.nk * vchunk <= PT_VRES_MAX_BYTES) ? 1 : 0;
  p.stage_bytes = PT_A_BYTES + (p.vres ? 0 : vchunk);
  p.nstages = (PT_RING_BYTES - (p.vres ? p.nk * vchunk : 0)) / p.stage_bytes;
  if (p.nstages > PT_MAX_STAGES) p.nstages = PT_MAX_STAGES;
  const size_t term_bytes = align_up((size_t)p.npad * K * sizeof(TV));
  TV* Vt[3];
  for (int q = 0; q < 3; ++q) Vt[q] = reinterpret_cast<TV*>(static_cast<char*>(ws) + (q < VT ? q : 0) * term_bytes);
  p.vscale = nullptr;
  if constexpr (BF16) {
    split_v_bf16_kernel<<<grid_for((int64_t)p.npad * K), 256, 0, st>>>(V, (int)K, r, p.npad, Vt[0], Vt[1], Vt[2]);
  } else if constexpr (F16 || F8) {
    float* inv_scale = reinterpret_cast<float*>(static_cast<char*>(ws) + VT * term_bytes);
    split_v_f16_kernel<<<p.npad, 256, 0, st>>>(V, (int)K, r, Vt[0], Vt[1], inv_scale);
    p.vscale = inv_scale;
  } else
    split_v_kernel<<<grid_for((int64_t)p.npad * K), 256, 0, st>>>(V, (int)K, r, p.npad, Vt[0], Vt[1]);
  TNB_LAUNCH_CHECK();
  CUtensorMap ta, th, tl, t3;
  CUresult cr = CUDA_SUCCESS;
  if (layout == PT_OUT_KBLOCKED) {  // (K, inner, rows / inner), box (KC, 16, 8): the 128 x KC tile of 8 rows of M
    cuuint64_t gdim[3] = {(cuuint64_t)K, (cuuint64_t)inner, (cuuint64_t)(rows / inner)};
    cuuint64_t gstride[2] = {(cuuint64_t)K * sizeof(TA), (cuuint64_t)(inner * K) * sizeof(TA)};
    cuuint32_t box[3] = {(cuuint32_t)KC, 16, 8}, estr[3] = {1, 1, 1};
    cr = get_encode_tiled()(&ta, tma_dtype<TA>(), 3, const_cast<TA*>(A), gdim, gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else if (layout == PT_IN_KBLOCKED) {  // (8 K, rows / 8), box (8 x 32 columns, 16 row groups), no swizzle
    cuuint64_t gdim[2] = {(cuuint64_t)(8 * K), (cuuint64_t)(rows / 8)};
    cuuint64_t gstride[1] = {(cuuint64_t)(8 * K) * sizeof(float)};
    cuuint32_t box[2] = {8 * PT_KC, PT_BM / 8}, estr[2] = {1, 1};
    cr = get_encode_tiled()(&ta, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<TA*>(A), gdim, gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    TNB_TRY(encode_kmajor_f32<TA>(&ta, A, rows, K, PT_BM));
  }
  if (cr != CUDA_SUCCESS) return fail(TNB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)cr);
  TNB_TRY(encode_kmajor_f32<TV>(&th, Vt[0], p.npad, K, p.npad));
  TNB_TRY(encode_kmajor_f32<TV>(&tl, Vt[1], p.npad, K, p.npad));
  t3 = th;
  if (VT == 3) TNB_TRY(encode_kmajor_f32<TV>(&t3, Vt[2], p.npad, K, p.npad));
  const int sms = usable_sms();
  const int64_t grid = p.num_row_blocks < sms ? p.num_row_blocks : sms;
  if (layout == PT_OUT_KBLOCKED) {
    static PerDeviceFlag attr_done;
    TNB_CUDA(ensure_dyn_smem(attr_done, project_tc_kernel<PT_OUT_KBLOCKED, TA>, PT_SMEM_BYTES));
    project_tc_kernel<PT_OUT_KBLOCKED, TA><<<(unsigned)grid, PT_THREADS, PT_SMEM_BYTES, st>>>(ta, th, tl, t3, p);
  } else if (layout == PT_IN_KBLOCKED) {
    if constexpr (sizeof(TA) == 4) {
      static PerDeviceFlag attr_done;
      TNB_CUDA(ensure_dyn_smem(attr_done, project_tc_kernel<PT_IN_KBLOCKED, TA>, PT_SMEM_BYTES));
      project_tc_kernel<PT_IN_KBLOCKED, TA><<<(unsigned)grid, PT_THREADS, PT_SMEM_BYTES, st>>>(ta, th, tl, t3, p);
    }
  } else {
    static PerDeviceFlag attr_done;
    TNB_CUDA(ensure_dyn_smem(attr_done, project_tc_kernel<PT_ROWMAJOR, TA>, PT_SMEM_BYTES));
    project_tc_kernel<PT_ROWMAJOR, TA><<<(unsigned)grid, PT_THREADS, PT_SMEM_BYTES, st>>>(ta, th, tl, t3, p);
  }
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

}  // namespace tnb
