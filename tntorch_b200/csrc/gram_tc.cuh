// Gram matrix G = C^T C of a tall row-major fp32 matrix C (rows x n) on the Hopper tensor cores.
//
//   * row slabs of C are staged HBM -> shared memory by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle,
//     out-of-bounds rows/columns zero-filled by the TMA unit), 4-stage mbarrier ring;
//   * the contraction runs over the ROW index of C, so both operands are "MN-major" views of the very same
//     slab.  tf32 wgmma takes its shared-memory B operand K-major only, but takes A from registers: the A
//     fragments are read straight out of the swizzled slab (mma_frag_a_mn: conflict-free), and only the B
//     columns of each stage are transposed into a K-major, 128-byte-swizzled buffer that a wgmma descriptor reads;
//   * G is symmetric: only tiles that touch the upper triangle are computed, and on diagonal tiles the
//     A operand is a sub-block of the B slab (loaded once);
//   * split-K over row ranges across CTAs; partial tiles go registers -> global and are summed in fp64 by a
//     deterministic second kernel (no atomics).
//
// 384 threads = three warpgroups, warp-specialized.  Warpgroup 0 is the producer: its warp 0 issues the TMA loads of a
// TC_STAGES-deep slab ring, its warps 1-3 transpose the B boxes of each stage into one of TC_TB_STAGES K-major buffers.
// Warpgroups 1 and 2 are the consumers: each owns 64 rows of the 128 x tn output tile and runs
// wgmma.mma_async m64n{tn}k8 .f32.tf32.tf32 with A from registers, accumulating in registers.  setmaxnreg moves the
// register file to the consumers (TC_CONSUMER_REGS: 128 accumulators plus two stages of A fragments).
//
// K-blocked mode (gram_tc(..., kblocked)): C is stored as wgmma's K-major core matrices, [rows/8][n/8][2][8][4]:
// element (k, c) at (((k/8 * n/8 + c/8) * 2 + k%8/4) * 8 + c%8) * 4 + k%4, the layout the sweep's projection writes for
// the next step.  Each 8 x 4 core matrix is 128 contiguous bytes and the 8 rows of a k8 step over 256 columns are one
// contiguous 8 KB run, so TMA loads both operands (256-byte lines, no swizzle) straight into the layout tf32 wgmma reads
// from shared memory: no transposers, A and B through descriptors, and the freed shared memory holds a
// TC_BLK_STAGES-deep slab ring.  The 8 rows each k8 step sums are the same 8 rows as in the row-major mode.
//
// bf16 mode (gram_tc_bf16): C is a row-major bf16 matrix (the dense TT-SVD's input).  wgmma takes 16-bit operands from
// shared memory MN-major, so TMA loads boxes of 64 bf16 columns x TC_KC rows (128-byte rows, 128-byte swizzle) and both
// operands go through descriptors of those boxes as they are: no transposers, a TC_BF16_STAGES-deep ring of 24 KB
// stages, wgmma.mma_async m64n128k16 .f32.bf16.bf16 on 128 x 128 tiles.  A product of two bf16 values is exact in
// fp32, so G rounds only in the accumulation.  The tensor core's fp32 accumulation is biased toward zero: over a whole
// 16384-row split it shrank G by ~5e-5 and left a non-uniform part of 8.5e-6 ||G|| on a rank-6 signal.  So each
// consumer accumulates TC_BF16_FLUSH stages into a scratch accumulator (the first wgmma of a group overwrites it) and
// adds that into its running sum with round-to-nearest fp32 adds, which needs the register room of 128-column tiles.
// Plan (with tn capped at 128), split-K, tile set, fold, partial layout and finalize are those of the fp32 modes.
// The mode takes its 16-bit element type as a parameter: fp16 input (gram_tc_f16) runs the same kernel with
// wgmma m64n128k16 .f32.f16.f16 (same MN-major descriptors) on a TMA map of FLOAT16 elements; an fp16 product is exact
// in fp32 as well (11-bit significands), and nothing else differs.
//
// Replaces, for large fp32 unfoldings, the QR of tensor.py:1816 / the Gram of round.py:104-110.
#pragma once
#include <cuda.h>

#include <cstdlib>
#include <type_traits>

#include "common.cuh"

namespace tnb {

constexpr int TC_KC = 32;                       // rows of C per pipeline stage
constexpr int TC_BOX_BYTES = TC_KC * 128;       // one TMA box: 32 fp32 columns x KC rows
constexpr int TC_STAGES = 3;                    // slab ring depth
constexpr int TC_MAX_BOXES = 12;                // 4 (A) + 8 (B)
constexpr int TC_STAGE_BYTES = TC_MAX_BOXES * TC_BOX_BYTES;
constexpr int TC_TB_STAGES = 2;                 // transposed-B ring depth (the consumer loop is unrolled by it)
constexpr int TC_TB_BYTES = 256 * TC_KC * 4;    // up to 256 columns x KC rows, K-major
constexpr int TC_TRANSPOSE_THREADS = 96;        // producer warps 1-3
constexpr int TC_THREADS = 384;
constexpr int TC_PRODUCER_REGS = 40;
constexpr int TC_CONSUMER_REGS = 232;
constexpr int TC_RING_BYTES = TC_STAGES * TC_STAGE_BYTES + TC_TB_STAGES * TC_TB_BYTES;
constexpr int TC_SMEM_BYTES = TC_RING_BYTES + 1024 /*align*/ + 256 /*barriers*/;
constexpr int TC_BLK_STAGES = 4;                // slab ring depth of the K-blocked mode (no transposed-B buffers)
static_assert(TC_BLK_STAGES * TC_STAGE_BYTES <= TC_RING_BYTES, "K-blocked ring must fit the row-major mode's buffers");
constexpr int TC_BF16_STAGE_BYTES = 6 * TC_BOX_BYTES;  // bf16 mode: 4 B boxes (256 columns) + 2 A boxes, TC_KC rows each
constexpr int TC_BF16_STAGES = 8;
constexpr int TC_BF16_FLUSH = 16;               // stages (512 rows) per scratch accumulation of the bf16 mode
static_assert(TC_BF16_STAGES * TC_BF16_STAGE_BYTES <= TC_RING_BYTES, "bf16 ring must fit the row-major mode's buffers");
constexpr int TC_MAX_RING = 8;                  // mbarriers per ring
constexpr int TC_ROWMAJOR = 0, TC_KBLOCKED = 1, TC_BF16 = 2;  // gram_tc_kernel modes
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
// The same bound without the printf, for kernels that issue wgmma: a function call anywhere in such a kernel makes ptxas
// serialize the wgmma pipeline.
__device__ __forceinline__ void mbar_wait_quiet(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > 4000000000LL) __trap();
}
// Unbounded wait, for warps that raised their register budget with setmaxnreg: a trap in that region makes ptxas fall
// back to the launch budget (spills, serialized wgmma).  Only use it on barriers whose producer waits with a bound, so
// that a stuck pipeline still ends in that producer's trap.
__device__ __forceinline__ void mbar_wait_spin(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* tmap, uint64_t* bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      :
      : "r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
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
// wgmma: tf32, A from registers, B from a K-major SWIZZLE_128B shared-memory buffer
// ---------------------------------------------------------------------------------------------
// Shared-memory descriptor of a K-major SWIZZLE_128B operand: rows of 128 bytes (32 tf32 along K), 8-row atoms of
// 1024 bytes stacked along N (stride byte offset 1024; the leading byte offset is unused by this layout).  The buffer is
// 1024-byte aligned, so the base offset is 0.  Adding 2 (32 bytes) to the descriptor selects the next k8 slice.
__device__ __forceinline__ uint64_t wgmma_desc_kmajor_sw128(const void* p) {
  return (uint64_t)((smem_u32(p) & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}
// K-major operand without swizzle: 8 x 16-byte core matrices of 128 contiguous bytes, the two of a k8 step 128 bytes
// apart (leading byte offset), 8-row groups 256 bytes apart along M/N (stride byte offset).
__device__ __forceinline__ uint64_t wgmma_desc_kmajor_core(const void* p) {
  return (uint64_t)((smem_u32(p) & 0x3FFFFu) >> 4) | ((uint64_t)(128 >> 4) << 16) | ((uint64_t)(256 >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from moving accesses of an accumulator across the asynchronous wgmma window.
template <int R>
__device__ __forceinline__ void wgmma_fence_operand(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Orders this thread's generic-proxy shared-memory writes before later async-proxy (wgmma, TMA) accesses.
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}

// D (64 x 32*NT fp32) += A (64 x 8) * B (8 x 32*NT), wgmma.mma_async m64n{32*NT}k8 .f32.tf32.tf32.  A is the m16n8k8 row
// fragment of each warp's 16 rows (a0: row g, k t; a1: row g+8, k t; a2: row g, k t+4; a3: row g+8, k t+4); d[4j+2h+e]
// is row 16*warp + g + 8h, column 8j + 2t + e.  B is read through `desc`.  The tensor core truncates the operands to tf32.
template <int NT>
__device__ void wgmma_tf32(float (&d)[NT * 16], const uint32_t (&a)[4], uint64_t desc);
template <>
__device__ __forceinline__ void wgmma_tf32<1>(float (&d)[16], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
      "}, {%16, %17, %18, %19}, %20, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<2>(float (&d)[32], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
      "}, {%32, %33, %34, %35}, %36, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<3>(float (&d)[48], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
      "}, {%48, %49, %50, %51}, %52, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<4>(float (&d)[64], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
      "}, {%64, %65, %66, %67}, %68, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<5>(float (&d)[80], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n160k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
      "}, {%80, %81, %82, %83}, %84, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<6>(float (&d)[96], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n192k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95"
      "}, {%96, %97, %98, %99}, %100, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<7>(float (&d)[112], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n224k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111"
      "}, {%112, %113, %114, %115}, %116, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
template <>
__device__ __forceinline__ void wgmma_tf32<8>(float (&d)[128], const uint32_t (&a)[4], uint64_t desc) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, {%128, %129, %130, %131}, %132, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc));
}
// MN-major operand of a 16-bit type with 128-byte swizzle, as TMA writes a box of 64 columns x TC_KC rows: each k is one
// 128-byte row, 8 rows form a 1024-byte swizzle atom (stride byte offset 1024 between the 8-k groups), and the 64-column
// blocks along M/N are `lbo` bytes apart (leading byte offset).  Adding 128 (2048 bytes) selects the next k16 slice.
__device__ __forceinline__ uint64_t wgmma_desc_mn_sw128(const void* p, uint32_t lbo) {
  return (uint64_t)((smem_u32(p) & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(1024 >> 4) << 32) |
         ((uint64_t)1 << 62);
}

// D (64 x 128 fp32) = A (64 x 16) * B (16 x 128) + (accumulate ? D : 0), both operands MN-major through descriptors, of
// the 16-bit type T16 (bf16 or fp16).
#define TNB_WGMMA_M64N128K16_SS(TY)                                                                              \
  asm volatile(                                                                                                  \
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"                                                         \
      "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " {"                                              \
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"                                    \
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"                          \
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"                          \
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"                            \
      "}, %64, %65, p, 1, 1, 1, 1;\n\t}"                                                                        \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),          \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),    \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),  \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),  \
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),  \
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),  \
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),  \
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])   \
      : "l"(desc_a), "l"(desc_b), "r"(accumulate))
template <typename T16>
__device__ __forceinline__ void wgmma_16_ss(float (&d)[64], uint64_t desc_a, uint64_t desc_b, int accumulate) {
  static_assert(std::is_same<T16, __half>::value || std::is_same<T16, __nv_bfloat16>::value, "bf16 or fp16 operands");
  if constexpr (std::is_same<T16, __half>::value)
    TNB_WGMMA_M64N128K16_SS("f16");
  else
    TNB_WGMMA_M64N128K16_SS("bf16");
}
#undef TNB_WGMMA_M64N128K16_SS

// The same m64n256k8 with A read from shared memory through `desc_a` as well (K-blocked mode).
__device__ __forceinline__ void wgmma_tf32_ss(float (&d)[128], uint64_t desc_a, uint64_t desc_b) {
  asm volatile(
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15,"
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47,"
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
      "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79,"
      "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
      "%96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111,"
      "%112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127"
      "}, %128, %129, 1, 1, 1;"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]),
        "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]),
        "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]),
        "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]),
        "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]),
        "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]),
        "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]),
        "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]),
        "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(desc_a), "l"(desc_b));
}

// ---------------------------------------------------------------------------------------------
// The kernel
// ---------------------------------------------------------------------------------------------
// Ring geometry of each mode.
template <int MODE>
struct TcRing {
  static constexpr int STAGES = MODE == TC_KBLOCKED ? TC_BLK_STAGES : MODE == TC_BF16 ? TC_BF16_STAGES : TC_STAGES;
  static constexpr int STAGE_BYTES = MODE == TC_BF16 ? TC_BF16_STAGE_BYTES : TC_STAGE_BYTES;
  static constexpr int A_SLOT = MODE == TC_BF16 ? 4 : 8;  // first box of a separately loaded A operand
  static constexpr int BOX_COLS = MODE == TC_BF16 ? 64 : 32;
};
static_assert(TcRing<TC_BF16>::STAGES <= TC_MAX_RING && TcRing<TC_KBLOCKED>::STAGES <= TC_MAX_RING, "mbarrier arrays");

// Loads of pipeline iteration `it` (rows it_begin + it) into its ring slot, once the transposers and the consumers have
// released it.  B first (slots 0..nbox_b), then A (slots A_SLOT..).  Row-major: boxes of 32 columns.  bf16: boxes of 64
// columns.  K-blocked: one box of (64, tn / 8 column groups, 4 row groups) for B and one of (64, 16, 4) for A, i.e.
// four k8 slices of tn (128) columns x 32 bytes.
template <int MODE>
__device__ __forceinline__ void gram_tc_produce(const CUtensorMap* tmap, const CUtensorMap* tmap_b, unsigned char* stage_base,
                                                uint64_t* full_bar, uint64_t* empty_bar, int64_t it, int64_t it_begin,
                                                int nbox_a, int nbox_b, int a_col0, int b_col0) {
  using R = TcRing<MODE>;
  const int stage = (int)(it % R::STAGES);
  const uint32_t phase = (uint32_t)(it / R::STAGES) & 1u;
  mbar_wait_quiet(&empty_bar[stage], phase ^ 1u);
  unsigned char* sb = stage_base + stage * R::STAGE_BYTES;
  mbar_expect_tx(&full_bar[stage], (uint32_t)(nbox_a + nbox_b) * TC_BOX_BYTES);
  const int row0 = (int)((it_begin + it) * TC_KC);
  if constexpr (MODE == TC_KBLOCKED) {
    tma_load_3d(sb, tmap_b, &full_bar[stage], 0, b_col0 / 8, row0 / 8);
    if (nbox_a) tma_load_3d(sb + 8 * TC_BOX_BYTES, tmap, &full_bar[stage], 0, a_col0 / 8, row0 / 8);
  } else {
    for (int j = 0; j < nbox_b; ++j)
      tma_load_2d(sb + j * TC_BOX_BYTES, tmap_b, &full_bar[stage], b_col0 + R::BOX_COLS * j, row0);
    for (int j = 0; j < nbox_a; ++j)
      tma_load_2d(sb + (R::A_SLOT + j) * TC_BOX_BYTES, tmap, &full_bar[stage], a_col0 + R::BOX_COLS * j, row0);
  }
}

// Transposes the nbox B boxes of a slab stage into the K-major buffer tb: element (row k, column c) of box j, at
// j*TC_BOX_BYTES + k*128 + ((((c%32)/4) ^ (k%8)) * 16) + (c%4)*4, goes to (column c, fragment index kl) at
// c*128 + (((kl/4) ^ (c%8)) * 16) + (kl%4)*4.  kl is the k index of mma_frag_a_mn: inside each 8-row step kl = t is row
// 2t and kl = t+4 is row 2t+1, so B carries the permutation of the A fragments and the product is unchanged.
// A work unit is a 4 x 4 block, 4 columns (16-byte chunk cq of a box row) by 4 fragment indices (16-byte chunk q of a
// tb row): four 16-byte loads, a register transpose, four 16-byte stores.  The 8 lanes of a quarter-warp take cq = l
// and q = (l/2) ^ s for one s in 0..7; then both the loads (chunk cq ^ (k%8)) and the stores (chunk q ^ (c%8)) reach 8
// distinct 16-byte bank groups: no bank conflicts on either side.
__device__ __forceinline__ void gram_tc_transpose_b(const unsigned char* sb, unsigned char* tb, int nbox, int tid) {
  for (int u = tid; u < nbox * 64; u += TC_TRANSPOSE_THREADS) {
    const int l = u & 7, s = (u >> 3) & 7, j = u >> 6;
    const int q = (l >> 1) ^ s;
    const int k0 = 8 * (q >> 1) + (q & 1);  // rows k0, k0+2, k0+4, k0+6 hold kl = 4q .. 4q+3
    float4 v[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int k = k0 + 2 * r;
      v[r] = *reinterpret_cast<const float4*>(sb + j * TC_BOX_BYTES + k * 128 + ((l ^ (k & 7)) << 4));
    }
    const int c0 = 32 * j + 4 * l;
    *reinterpret_cast<float4*>(tb + (c0 + 0) * 128 + ((q ^ ((c0 + 0) & 7)) << 4)) = make_float4(v[0].x, v[1].x, v[2].x, v[3].x);
    *reinterpret_cast<float4*>(tb + (c0 + 1) * 128 + ((q ^ ((c0 + 1) & 7)) << 4)) = make_float4(v[0].y, v[1].y, v[2].y, v[3].y);
    *reinterpret_cast<float4*>(tb + (c0 + 2) * 128 + ((q ^ ((c0 + 2) & 7)) << 4)) = make_float4(v[0].z, v[1].z, v[2].z, v[3].z);
    *reinterpret_cast<float4*>(tb + (c0 + 3) * 128 + ((q ^ ((c0 + 3) & 7)) << 4)) = make_float4(v[0].w, v[1].w, v[2].w, v[3].w);
  }
}

// Producer warps 1-3: for every stage, transpose its B boxes into the transposed-B ring and release the slab slot.
__device__ __forceinline__ void gram_tc_transposer(unsigned char* stage_base, unsigned char* tb_base, uint64_t* full_bar,
                                                   uint64_t* empty_bar, uint64_t* tb_full, uint64_t* tb_empty,
                                                   int64_t iters, int nbox_b) {
  const int tid = threadIdx.x - 32;
  for (int64_t it = 0; it < iters; ++it) {
    const int s = (int)(it % TC_STAGES), b = (int)(it % TC_TB_STAGES);
    mbar_wait_quiet(&full_bar[s], (uint32_t)(it / TC_STAGES) & 1u);
    mbar_wait_quiet(&tb_empty[b], ((uint32_t)(it / TC_TB_STAGES) & 1u) ^ 1u);
    gram_tc_transpose_b(stage_base + s * TC_STAGE_BYTES, tb_base + b * TC_TB_BYTES, nbox_b, tid);
    fence_proxy_async_smem();  // the stores are read by wgmma (async proxy)
    mbar_arrive(&tb_full[b]);
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(&empty_bar[s]);
  }
}

template <int NT>
__device__ __forceinline__ void gram_tc_epilogue(const GramTcParams& p, const float (&acc)[NT * 16], int cm, int lane,
                                                 int tile_id, int split, int a_col0, int b_col0);

// One pipeline stage of a consumer warp: A fragments of stage `it` into `af`, four k8 wgmma into `acc`, then release
// the slab slot and, once the previous stage's group has completed, its transposed-B buffer.
template <int NT>
__device__ __forceinline__ void gram_tc_consume_stage(float (&acc)[NT * 16], uint32_t (&af)[4][4], int64_t it,
                                                      const unsigned char* stage_base, uint64_t* full_bar, uint64_t* empty_bar, uint64_t* tb_full,
                                                      uint64_t* tb_empty, uint64_t desc, int a_box, int cm, int lane) {
  const int g = lane >> 2, t = lane & 3;
  const int s = (int)(it % TC_STAGES), b = (int)(it % TC_TB_STAGES);
  mbar_wait_spin(&full_bar[s], (uint32_t)(it / TC_STAGES) & 1u);
  const unsigned char* sa = stage_base + s * TC_STAGE_BYTES + a_box * TC_BOX_BYTES;
#pragma unroll
  for (int kk = 0; kk < TC_KC / 8; ++kk) mma_frag_a_mn(sa, 8 * kk, cm, g, t, af[kk]);
  mbar_wait_spin(&tb_full[b], (uint32_t)(it / TC_TB_STAGES) & 1u);
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < TC_KC / 8; ++kk) wgmma_tf32<NT>(acc, af[kk], desc + 2 * kk);
  wgmma_commit();
  __syncwarp();
  if (lane == 0) mbar_arrive(&empty_bar[s]);  // A of this stage is in registers: the slab slot may be refilled
  wgmma_wait<1>();                            // the previous stage's wgmma group has finished reading its buffer
  if (it > 0 && lane == 0) mbar_arrive(&tb_empty[(it - 1) % TC_TB_STAGES]);
}

// Consumer warpgroup cw (0 or 1): rows 64*cw .. 64*cw+63 of the 128 x tn tile, tn = 32*NT, as one m64n{tn} wgmma
// accumulator.  A fragments of a stage are read from the slab into registers (two register sets: the loads of a stage
// overlap the wgmma of the previous one), B through the descriptor of the stage's transposed buffer.
template <int NT>
__device__ __forceinline__ void gram_tc_consumer(const GramTcParams& p, const unsigned char* stage_base,
                                                 const unsigned char* tb_base, uint64_t* full_bar, uint64_t* empty_bar,
                                                 uint64_t* tb_full, uint64_t* tb_empty, int64_t iters, int a_box,
                                                 int tile_id, int split, int a_col0, int b_col0) {
  const int ct = threadIdx.x - 128;
  const int lane = ct & 31, w = (ct >> 5) & 3;
  const int cm = 64 * (ct >> 7) + 16 * w;  // first of this warp's 16 rows of the tile
  float acc[NT * 16];
#pragma unroll
  for (int i = 0; i < NT * 16; ++i) acc[i] = 0.f;
  wgmma_fence_operand(acc);

  // TC_TB_STAGES == 2: even stages read transposed buffer 0 (A fragments af0), odd stages buffer 1 (af1)
  const uint64_t desc0 = wgmma_desc_kmajor_sw128(tb_base), desc1 = wgmma_desc_kmajor_sw128(tb_base + TC_TB_BYTES);
  uint32_t af0[4][4], af1[4][4];
  // The loop leaves right after an odd number of stages: on the back edge only the af1 group can be in flight, so
  // ptxas can prove that loading af0 does not overwrite registers a pending wgmma reads (else it serializes them).
  for (int64_t it = 0; it < iters; it += 2) {
    gram_tc_consume_stage<NT>(acc, af0, it, stage_base, full_bar, empty_bar, tb_full, tb_empty, desc0, a_box, cm, lane);
    if (it + 1 == iters) break;
    gram_tc_consume_stage<NT>(acc, af1, it + 1, stage_base, full_bar, empty_bar, tb_full, tb_empty, desc1, a_box, cm,
                              lane);
  }
  wgmma_wait<0>();
  wgmma_fence_operand(acc);
  gram_tc_epilogue<NT>(p, acc, cm, lane, tile_id, split, a_col0, b_col0);
}

// Consumer warpgroup cw of the K-blocked mode (tn = 256): both operands through descriptors of the stage's k8 slices.  B slice kk is at kk * 8 KB; A (this warpgroup's 64 rows) at a_off + kk * a_slice + 64 * cw rows.  A slot is
// released once the wgmma group that read it has completed, i.e. one stage later.
__device__ __forceinline__ void gram_tc_consumer_blocked(const GramTcParams& p, const unsigned char* stage_base,
                                                         uint64_t* full_bar, uint64_t* empty_bar, int64_t iters,
                                                         int a_off, int a_slice, int tile_id, int split, int a_col0,
                                                         int b_col0) {
  const int ct = threadIdx.x - 128;
  const int lane = ct & 31, w = (ct >> 5) & 3, cw = ct >> 7;
  const int cm = 64 * cw + 16 * w;
  float acc[128];
#pragma unroll
  for (int i = 0; i < 128; ++i) acc[i] = 0.f;
  wgmma_fence_operand(acc);
  for (int64_t it = 0; it < iters; ++it) {
    const int s = (int)(it % TC_BLK_STAGES);
    mbar_wait_spin(&full_bar[s], (uint32_t)(it / TC_BLK_STAGES) & 1u);
    const unsigned char* sb = stage_base + s * TC_STAGE_BYTES;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < TC_KC / 8; ++kk)
      wgmma_tf32_ss(acc, wgmma_desc_kmajor_core(sb + a_off + kk * a_slice + 64 * cw * 32),
                    wgmma_desc_kmajor_core(sb + kk * 256 * 32));
    wgmma_commit();
    wgmma_wait<1>();
    __syncwarp();
    if (it > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % TC_BLK_STAGES]);
  }
  wgmma_wait<0>();
  wgmma_fence_operand(acc);
  gram_tc_epilogue<8>(p, acc, cm, lane, tile_id, split, a_col0, b_col0);
}

// Consumer warpgroup cw of the bf16 mode (tn = 128): A (this warpgroup's 64 columns of C, box a_box + cw) and B (the
// stage's two boxes, TC_BOX_BYTES apart) through MN-major descriptors, two k16 slices per stage, into the scratch
// accumulator `part`; every TC_BF16_FLUSH stages (and at the end) `part` is added into `acc` with fp32 adds.  A slot is
// released once the wgmma group that read it has completed, i.e. one stage later.  T16: bf16 or fp16 operands.
template <typename T16>
__device__ __forceinline__ void gram_tc_consumer_bf16(const GramTcParams& p, const unsigned char* stage_base,
                                                      uint64_t* full_bar, uint64_t* empty_bar, int64_t iters, int a_box,
                                                      int tile_id, int split, int a_col0, int b_col0) {
  using R = TcRing<TC_BF16>;
  const int ct = threadIdx.x - 128;
  const int lane = ct & 31, w = (ct >> 5) & 3, cw = ct >> 7;
  const int cm = 64 * cw + 16 * w;
  float acc[64], part[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f, part[i] = 0.f;
  wgmma_fence_operand(part);
  for (int64_t it = 0; it < iters; ++it) {
    const int s = (int)(it % R::STAGES);
    mbar_wait_spin(&full_bar[s], (uint32_t)(it / R::STAGES) & 1u);
    const unsigned char* sb = stage_base + s * R::STAGE_BYTES;
    const int first = it % TC_BF16_FLUSH == 0;
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < TC_KC / 16; ++kk)
      wgmma_16_ss<T16>(part, wgmma_desc_mn_sw128(sb + (a_box + cw) * TC_BOX_BYTES + kk * 2048, TC_BOX_BYTES),
                    wgmma_desc_mn_sw128(sb + kk * 2048, TC_BOX_BYTES), (first && kk == 0) ? 0 : 1);
    wgmma_commit();
    if ((it + 1) % TC_BF16_FLUSH == 0 || it + 1 == iters) {
      wgmma_wait<0>();
      wgmma_fence_operand(part);
#pragma unroll
      for (int i = 0; i < 64; ++i) acc[i] += part[i];
      wgmma_fence_operand(part);
    } else {
      wgmma_wait<1>();
    }
    __syncwarp();
    if (it > 0 && lane == 0) mbar_arrive(&empty_bar[(it - 1) % R::STAGES]);
  }
  gram_tc_epilogue<4>(p, acc, cm, lane, tile_id, split, a_col0, b_col0);
}

// Output of one consumer warp: acc[4j + 2h + e] is (row cm + g + 8h, column 8j + 2t + e) of the 128 x tn tile.
template <int NT>
__device__ __forceinline__ void gram_tc_epilogue(const GramTcParams& p, const float (&acc)[NT * 16], int cm, int lane,
                                                 int tile_id, int split, int a_col0, int b_col0) {
  const int g = lane >> 2, t = lane & 3;
  if (p.direct) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int gi = a_col0 + cm + g + 8 * h;
#pragma unroll
      for (int j = 0; j < 4 * NT; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int gj = b_col0 + 8 * j + 2 * t + e;
          if (gi < p.m && gj < p.n) {
            float x = p.alpha * acc[4 * j + 2 * h + e];
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
  for (int h = 0; h < 2; ++h) {
    float* orow = out + (size_t)(cm + g + 8 * h) * p.tn + 2 * t;
#pragma unroll
    for (int j = 0; j < 4 * NT; ++j)
      *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
  }
}

// TC_KBLOCKED: the operands are K-blocked (see the top of the file); tmap / tmap_b are 3-D maps with boxes (64, 16, 4)
// and (64, 32, 4).  TC_ROWMAJOR: row-major fp32, 2-D maps with boxes of 32 columns x TC_KC rows.  TC_BF16: row-major
// T16 (bf16 or fp16; the other modes ignore it), 2-D maps with boxes of 64 columns x TC_KC rows.
template <int MODE, typename T16 = __nv_bfloat16>
__global__ void __launch_bounds__(TC_THREADS, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ CUtensorMap tmap_b,
               const GramTcParams p) {
  extern __shared__ unsigned char tc_smem_raw[];
  // 1024-byte aligned stage buffers (SWIZZLE_128B atoms are 1024 B)
  const uint32_t raw_addr = smem_u32(tc_smem_raw);
  const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
  unsigned char* stage_base = tc_smem_raw + pad;
  unsigned char* tb_base = stage_base + TC_STAGES * TC_STAGE_BYTES;  // row-major mode only
  constexpr bool BLOCKED = MODE == TC_KBLOCKED, BF16 = MODE == TC_BF16;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(stage_base + TC_RING_BYTES);
  uint64_t* empty_bar = full_bar + TC_MAX_RING;
  uint64_t* tb_full = empty_bar + TC_MAX_RING;
  uint64_t* tb_empty = tb_full + TC_TB_STAGES;
  int* tile_smem = reinterpret_cast<int*>(tb_empty + TC_TB_STAGES);  // bm, bn

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
    for (int s = 0; s < TcRing<MODE>::STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      // per warp: transposers and consumers (K-blocked, bf16: consumers only)
      mbar_init(&empty_bar[s], (MODE == TC_ROWMAJOR ? TC_TRANSPOSE_THREADS / 32 : 0) + 8);
    }
    for (int b = 0; b < TC_TB_STAGES; ++b) {
      mbar_init(&tb_full[b], TC_TRANSPOSE_THREADS);  // per thread: each orders its own stores for the async proxy
      mbar_init(&tb_empty[b], 8);                    // per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int bm = tile_smem[0], bn = tile_smem[1];
  const int a_col0 = bm * 128, b_col0 = bn * p.tn;
  constexpr int BOX_COLS = TcRing<MODE>::BOX_COLS;
  const int nbox_b = p.tn / BOX_COLS;
  const bool a_in_b = p.symmetric && (a_col0 >= b_col0) && (a_col0 + 128 <= b_col0 + p.tn);
  const int nbox_a = a_in_b ? 0 : 128 / BOX_COLS;
  const int a_box = a_in_b ? (a_col0 - b_col0) / BOX_COLS : TcRing<MODE>::A_SLOT;  // first box of the A operand in a stage
  const int64_t it_begin = (int64_t)split * p.iters_per_split;
  int64_t it_end = it_begin + p.iters_per_split;
  if (it_end > p.iters_total) it_end = p.iters_total;
  const int64_t iters = it_end > it_begin ? it_end - it_begin : 0;

  if (threadIdx.x < 128) {  // producer warpgroup
    setmaxnreg_dec<TC_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      for (int64_t it = 0; it < iters; ++it)
        gram_tc_produce<MODE>(&tmap, &tmap_b, stage_base, full_bar, empty_bar, it, it_begin, nbox_a, nbox_b, a_col0,
                              b_col0);
    } else if (MODE == TC_ROWMAJOR && threadIdx.x >= 32) {
      gram_tc_transposer(stage_base, tb_base, full_bar, empty_bar, tb_full, tb_empty, iters, nbox_b);
    }
    return;
  }
  setmaxnreg_inc<TC_CONSUMER_REGS>();
  if constexpr (BF16) {  // tn = 128
    gram_tc_consumer_bf16<T16>(p, stage_base, full_bar, empty_bar, iters, a_box, tile_id, split, a_col0, b_col0);
    return;
  } else if constexpr (BLOCKED) {  // tn == 256; A inside B: its k8 slices are rows of B's (8 KB apart), else 128-row slices in slot 8
    gram_tc_consumer_blocked(p, stage_base, full_bar, empty_bar, iters,
                             a_in_b ? (a_col0 - b_col0) * 32 : 8 * TC_BOX_BYTES, a_in_b ? 256 * 32 : 128 * 32, tile_id,
                             split, a_col0, b_col0);
    return;
  } else {
#define TNB_GRAM_CONSUME(NT)                                                                                          \
  gram_tc_consumer<NT>(p, stage_base, tb_base, full_bar, empty_bar, tb_full, tb_empty, iters, a_box, tile_id, split, \
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

// max_tn: widest column tile (256; 128 for the bf16 mode)
inline void gram_tc_plan(int64_t rows, int64_t n, GramTcParams& p, int64_t m_cols = -1, int max_tn = 256) {
  p.rows = rows;
  p.n = (int)n;
  p.symmetric = m_cols < 0 ? 1 : 0;
  p.m = p.symmetric ? (int)n : (int)m_cols;
  int tn = n >= max_tn ? max_tn : (int)((n + 31) / 32 * 32);
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

inline size_t gram_tc_workspace_bytes(int64_t rows, int64_t n, int max_tn = 256) {
  GramTcParams p;
  const int f = gram_tc_fold(rows, n);
  gram_tc_plan(rows / f, n * f, p, -1, max_tn);
  return align_up((size_t)p.ksplit * p.num_tiles * 128 * p.tn * sizeof(float));
}

// TMA element type of the kernels' inputs: fp32, bf16 or fp16
template <typename T>
inline CUtensorMapDataType tma_dtype() {
  static_assert(std::is_same<T, float>::value || std::is_same<T, __nv_bfloat16>::value || std::is_same<T, __half>::value,
                "fp32, bf16 or fp16 elements");
  return std::is_same<T, float>::value           ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32
         : std::is_same<T, __nv_bfloat16>::value ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
                                                 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}

// boxes of 128 bytes per row: 32 fp32 or 64 bf16 / fp16 columns
template <typename T = float>
inline int encode_rowmajor_f32(CUtensorMap* tmap, const T* ptr, int64_t rows, int64_t cols, int box_rows = TC_KC) {
  cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t gstride[1] = {(cuuint64_t)cols * sizeof(T)};
  cuuint32_t box[2] = {128 / (cuuint32_t)sizeof(T), (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult cr = get_encode_tiled()(tmap, tma_dtype<T>(), 2, const_cast<T*>(ptr), gdim, gstride, box,
                                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return fail(TNB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)cr);
  return TNB_OK;
}

// 3-D map over a K-blocked matrix (64 floats per 8 rows x 8 columns, cols / 8 column groups, rows / 8 row groups):
// box (64, box_cols / 8, TC_KC / 8) lands in shared memory as TC_KC / 8 k8 slices of box_cols columns x 32 bytes.
inline int encode_kblocked_f32(CUtensorMap* tmap, const float* ptr, int64_t rows, int64_t cols, int box_cols) {
  cuuint64_t gdim[3] = {64, (cuuint64_t)(cols / 8), (cuuint64_t)(rows / 8)};
  cuuint64_t gstride[2] = {64 * sizeof(float), (cuuint64_t)cols * 8 * sizeof(float)};
  cuuint32_t box[3] = {64, (cuuint32_t)box_cols / 8, TC_KC / 8};
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult cr = get_encode_tiled()(tmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(ptr), gdim, gstride, box,
                                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) return fail(TNB_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)cr);
  return TNB_OK;
}

inline bool gram_tc_kblocked_shape_ok(int64_t rows, int64_t n) {
  return gram_tc_shape_ok(rows, n) && n >= 256 && n % 8 == 0 && rows % 8 == 0;
}

// bf16 / fp16 input: 16-byte rows (n % 8 == 0) and 128-column tiles: a folded n = 32 / 64, n = 128, or n >= 256 (where
// the upper-triangle tile set of 128 x 128 tiles covers no more than that of the fp32 modes' 128 x 256 tiles).
inline bool gram_tc_bf16_shape_ok(int64_t rows, int64_t n) {
  return gram_tc_shape_ok(rows, n) && n % 8 == 0 && (gram_tc_fold(rows, n) > 1 || n == 128 || n >= 256);
}
template <typename T>
inline size_t gram_tc_input_workspace_bytes(int64_t rows, int64_t n) {
  return gram_tc_workspace_bytes(rows, n, sizeof(T) == 2 ? 128 : 256);
}
template <typename T>
inline bool gram_tc_input_ok(int64_t rows, int64_t n) {
  if (std::is_same<T, float>::value) return gram_tc_shape_ok(rows, n);
  if (std::is_same<T, __nv_bfloat16>::value || std::is_same<T, __half>::value) return gram_tc_bf16_shape_ok(rows, n);
  return false;
}

// G (n x n fp64) and optionally Gf (fp32 copy) = A^T A, A: rows x n fp32, bf16 or fp16 (device), row-major or, with
// kblocked (fp32 only), stored K-blocked (then n >= 256, n % 8 == 0 and rows % 8 == 0).
template <typename T>
inline int gram_tc(const T* A, int64_t rows, int64_t n, double* G, float* Gf, void* ws, size_t ws_bytes,
                   cudaStream_t st, bool kblocked = false) {
  constexpr bool BF16 = sizeof(T) == 2;  // the 16-bit mode, bf16 or fp16
  if (!tc_path_available()) return fail(TNB_ERR_UNSUPPORTED, "gram_tc: TMA tensor-core path needs an sm_90 device");
  if (!(kblocked ? !BF16 && gram_tc_kblocked_shape_ok(rows, n) : gram_tc_input_ok<T>(rows, n)))
    return fail(TNB_ERR_UNSUPPORTED, "gram_tc: unsupported shape rows=%lld n=%lld", (long long)rows, (long long)n);
  if ((reinterpret_cast<uintptr_t>(A) & 15u) != 0) return fail(TNB_ERR_INVALID, "gram_tc: input must be 16-byte aligned");
  GramTcParams p;
  const int fold = gram_tc_fold(rows, n);  // 1 for n >= 128
  const int64_t n_in = n;
  rows /= fold;
  n *= fold;
  gram_tc_plan(rows, n, p, -1, BF16 ? 128 : 256);
  p.fold = fold;
  p.n_orig = (int)n_in;
  const size_t need = (size_t)p.ksplit * p.num_tiles * 128 * p.tn * sizeof(float);
  if (ws_bytes < need) return fail(TNB_ERR_WORKSPACE, "gram_tc: workspace %zu < %zu", ws_bytes, need);
  p.partial = static_cast<float*>(ws);

  dim3 grid((unsigned)p.num_tiles, (unsigned)p.ksplit);
  if constexpr (BF16) {
    CUtensorMap tmap;
    TNB_TRY(encode_rowmajor_f32<T>(&tmap, A, rows, n));
    static PerDeviceFlag attr_done;
    TNB_CUDA(ensure_dyn_smem(attr_done, gram_tc_kernel<TC_BF16, T>, TC_SMEM_BYTES));
    gram_tc_kernel<TC_BF16, T><<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(tmap, tmap, p);
  } else if (kblocked) {
    CUtensorMap ta, tb;
    TNB_TRY(encode_kblocked_f32(&ta, A, rows, n, 128));
    TNB_TRY(encode_kblocked_f32(&tb, A, rows, n, 256));
    static PerDeviceFlag attr_done;
    TNB_CUDA(ensure_dyn_smem(attr_done, gram_tc_kernel<TC_KBLOCKED>, TC_SMEM_BYTES));
    gram_tc_kernel<TC_KBLOCKED><<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(ta, tb, p);
  } else {
    CUtensorMap tmap;
    TNB_TRY(encode_rowmajor_f32(&tmap, A, rows, n));
    static PerDeviceFlag attr_done;
    TNB_CUDA(ensure_dyn_smem(attr_done, gram_tc_kernel<TC_ROWMAJOR>, TC_SMEM_BYTES));
    gram_tc_kernel<TC_ROWMAJOR><<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(tmap, tmap, p);
  }
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
  TNB_CUDA(ensure_dyn_smem(attr_done, gram_tc_kernel<TC_ROWMAJOR>, TC_SMEM_BYTES));
  dim3 grid((unsigned)p.num_tiles, (unsigned)p.ksplit);
  gram_tc_kernel<TC_ROWMAJOR><<<grid, TC_THREADS, TC_SMEM_BYTES, st>>>(ta, tb, p);
  TNB_LAUNCH_CHECK();
  if (narrow) return TNB_OK;
  const int64_t total = m * n;
  atb_tc_finalize_kernel<<<(unsigned)std::min<int64_t>((total + 255) / 256, 4096), 256, 0, st>>>(p, C, ldc, alpha, D, ldd,
                                                                                                 beta, E, lde, gamma);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

}  // namespace tnb
