// Chebyshev filter of the subspace iteration (eig.cuh) as ONE resident kernel.
//
// The filter is m products Y_s = a_s * G*Y_{s-1} + b_s * Y_{s-1} + g_s * Y_{s-2} with the same symmetric G
// (n x n fp32, <= 16 MB).  Launched one product at a time it is latency-bound (15 us tensor-core kernel +
// 5 us split-K finalize per product, 60 products per eigensolve).  Here G is partitioned ONCE over the
// shared memories of the grid and stays there for all m products:
//
//   * a cluster of 8 CTAs owns a 128-row slab of the output; CTA q of the cluster holds the G block
//     (K-slice q: rows [q*n/8, (q+1)*n/8)) x (128 slab columns) — G is symmetric, so this block is the
//     MN-major A operand of the slab's product — loaded by TMA (128B swizzle) before step 1;
//   * each step: TMA-load the matching K-slice of Y_{s-1} (n/8 x b, L2 resident), 128 x b x n/8 tf32 product
//     on the tensor cores (mma.sync, four warps of 32 rows, accumulators in registers) into shared memory,
//     cluster barrier, every CTA sums 16 of the slab's rows over the 8 partial tiles through distributed
//     shared memory, applies the three-term recurrence and writes its 16 rows of Y_s;
//   * a grid-wide barrier (all CTAs are co-resident: cooperative launch) separates the steps.
//
// When the GPU cannot hold n/128 clusters of 8 CTAs with this shared-memory footprint at once
// (cudaOccupancyMaxActiveClusters, asked once per device), the 8 partial tiles of a slab go through L2 instead
// (row-major partial tiles, coalesced both ways) with a second grid barrier per step.
//
// Only the FILTER runs here (TF32 operands: operator accuracy affects the convergence rate only); the
// Rayleigh-Ritz product stays on the fp32 FFMA path (eig.cuh).
#pragma once
#include <mutex>

#include "common.cuh"
#include "gram_tc.cuh"

namespace tnb {

constexpr int CF_KS = 8;          // cluster size = K-slices per slab
constexpr int CF_THREADS = 128;
constexpr int CF_MAX_STEPS = 48;
constexpr int CF_RED_LD = 129;    // odd column stride of the partial-tile buffer: conflict-free both ways

// Device-resident control block of the sync-free subspace eigensolver (chfsi_dev.cuh).  The first three ints are the
// skip words of common.cuh::tnb_skip.  The Rayleigh-Ritz kernel of stage s writes the degree, the coefficients and the
// ring position of the NEXT filter here; the filter kernel reads them (nothing about the filter passes through the host).
struct ChfsiCtrl {
  int done;        // 1 once the captured energy has converged
  int error;       // 0 ok, 1 Cholesky breakdown (numerically dependent block), 2 not converged, 3 non-finite values
  int conv_stage;  // stage at which `done` was raised
  int outer;       // Rayleigh-Ritz steps completed
  int products;    // filter products executed
  int steps;       // degree of the next filter
  int xin;         // ring buffer holding the input block of the next filter; its result lands in ring[0]
  int jac_sweeps;  // Jacobi sweeps summed over the Rayleigh-Ritz solves (diagnostic)
  double prev_cap, prev_delta, trace, cap;
  float a[48], bc[48], g[48];  // CF_MAX_STEPS
};

struct ChebFilterParams {
  int n, b;        // G is n x n, blocks are n x b (ld = b)
  int nbox;        // ceil(b / 32)
  int ksl;         // n / 8 rows of Y per CTA
  int steps;
  float a[CF_MAX_STEPS], bc[CF_MAX_STEPS], g[CF_MAX_STEPS];
  float* buf[3];   // rotating n x b blocks: step s reads buf[(s-1)%3] (and buf[(s-2)%3]), writes buf[s%3]
  unsigned* counter;  // zeroed grid-barrier counter
  int dsmem;          // 1: launched as clusters of 8, partial tiles reduced through distributed shared memory
  float* partial;     // dsmem == 0: [slab][q][128][nbox*32] partial tiles in global memory (L2 resident)
  const ChfsiCtrl* ctrl;  // non-null: steps / coefficients / ring rotation come from the device control block
  int stage;
};

inline size_t cheb_filter_smem_bytes(int n, int b) {
  const int nbox = (b + 31) / 32, ksl = n / CF_KS;
  return (size_t)ksl * 128 * 4 + (size_t)ksl * nbox * 128 + (size_t)nbox * 32 * CF_RED_LD * 4 + 1024 + 64;
}
inline bool cheb_filter_shape_ok(int n, int b) {
  if (n % 256 != 0 || n < 256 || b < 8 || b % 4 != 0 || b > 128) return false;
  if ((n / 128) * CF_KS > device_info().sm_count) return false;
  return cheb_filter_smem_bytes(n, b) <= (size_t)227 * 1024;
}

__device__ __forceinline__ void cf_grid_barrier(unsigned* ctr, unsigned target) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(ctr) : "memory");
  unsigned v;
  const long long t0 = clock64();
  for (;;) {
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(ctr) : "memory");
    if (v >= target) break;
    if (clock64() - t0 > 4000000000LL) {
      printf("tnb200: filter grid barrier timed out (block %d, %u < %u)\n", blockIdx.x, v, target);
      __trap();
    }
  }
}

// NB = nbox: the warp's 32 x (32 NB) share of the 128 x bn partial tile of this CTA's K-slice
template <int NB>
__device__ __forceinline__ void cf_product(const unsigned char* g_sm, const unsigned char* y_sm, int nchunk, int nbox,
                                           float (&acc)[2][4 * NB][4]) {
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4 * NB; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
  for (int c = 0; c < nchunk; ++c) {
    const unsigned char* ga = g_sm + (size_t)c * 4 * TC_BOX_BYTES;
    const unsigned char* yb = y_sm + (size_t)c * nbox * TC_BOX_BYTES;
#pragma unroll
    for (int ks = 0; ks < 32; ks += 8) {
      uint32_t af[2][4];
      mma_frag_a_mn(ga, ks, 32 * w, g, t, af[0]);
      mma_frag_a_mn(ga, ks, 32 * w + 16, g, t, af[1]);
#pragma unroll
      for (int j = 0; j < 4 * NB; ++j) {
        uint32_t bf[2];
        mma_frag_b_mn(yb, ks, 8 * j, g, t, bf);
        mma_tf32(acc[0][j], af[0][0], af[0][1], af[0][2], af[0][3], bf[0], bf[1]);
        mma_tf32(acc[1][j], af[1][0], af[1][1], af[1][2], af[1][3], bf[0], bf[1]);
      }
    }
  }
}

template <int NB>
__global__ void __launch_bounds__(CF_THREADS, 1)
cheb_filter_kernel(const __grid_constant__ CUtensorMap tmap_g, const __grid_constant__ CUtensorMap tmap_y0,
                   const __grid_constant__ CUtensorMap tmap_y1, const __grid_constant__ CUtensorMap tmap_y2,
                   const ChebFilterParams p) {
  extern __shared__ unsigned char cf_smem_raw[];
  int nsteps = p.steps, rot = 0;
  if (p.ctrl) {  // speculative enqueue: the whole grid leaves at once when the solve has converged or failed
    if (tnb_skip(&p.ctrl->done, p.stage)) return;
    nsteps = __ldcg(&p.ctrl->steps);
    rot = __ldcg(&p.ctrl->xin);
    if (nsteps < 1 || nsteps > CF_MAX_STEPS) return;
  }
  const uint32_t raw_addr = smem_u32(cf_smem_raw);
  const uint32_t pad = (1024u - (raw_addr & 1023u)) & 1023u;
  unsigned char* g_sm = cf_smem_raw + pad;                                  // ksl/32 chunks x 4 boxes
  unsigned char* y_sm = g_sm + (size_t)p.ksl * 512;                         // ksl/32 chunks x nbox boxes
  float* red = reinterpret_cast<float*>(y_sm + (size_t)p.ksl * p.nbox * 128);  // [nbox*32][CF_RED_LD]
  uint64_t* bars = reinterpret_cast<uint64_t*>(red + (size_t)p.nbox * 32 * CF_RED_LD);
  uint64_t* g_bar = bars;
  uint64_t* y_bar = bars + 1;

  const int tid = threadIdx.x, warp_idx = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t = lane & 3;
  const uint32_t q = blockIdx.x % CF_KS;         // K-slice of this CTA (= its rank in the cluster, if any)
  const int slab = blockIdx.x / CF_KS;           // 128-row slab of the output
  const int m0 = slab * 128, k0 = (int)q * p.ksl;
  const int nchunk = p.ksl / 32;
  const int bn = p.nbox * 32;

  if (tid == 0) {
    mbar_init(g_bar, 1);
    mbar_init(y_bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (tid == 0) {
    // resident block of G: rows k0..k0+ksl, columns m0..m0+128
    mbar_expect_tx(g_bar, (uint32_t)p.ksl * 512u);
    for (int c = 0; c < nchunk; ++c)
      for (int j = 0; j < 4; ++j)
        tma_load_2d(g_sm + ((size_t)c * 4 + j) * TC_BOX_BYTES, &tmap_g, g_bar, m0 + 32 * j, k0 + 32 * c);
  }
  if (p.dsmem) cluster_sync_all();  // every CTA of the cluster is running before any DSMEM access

  const uint32_t red_addr = smem_u32(red);
  const int row_base = m0 + 16 * (int)q;  // the 16 output rows this CTA reduces and writes

  for (int s = 1; s <= nsteps; ++s) {
    const uint32_t par = (uint32_t)(s - 1) & 1u;
    const int icur = (s - 1 + rot) % 3, iprev = (s + 1 + rot) % 3, iout = (s + rot) % 3;
    const float* ycur = p.buf[icur];   // written by other CTAs in earlier steps: read through L2 (__ldcg)
    const float* yprev = p.buf[iprev];
    float* yout = p.buf[iout];
    const float ca = p.ctrl ? __ldcg(&p.ctrl->a[s - 1]) : p.a[s - 1];
    const float cb = p.ctrl ? __ldcg(&p.ctrl->bc[s - 1]) : p.bc[s - 1];
    const float cg = p.ctrl ? __ldcg(&p.ctrl->g[s - 1]) : p.g[s - 1];
    if (tid == 0) {
      asm volatile("fence.proxy.async;" ::: "memory");  // Y_{s-1} was written with generic stores by other CTAs
      const CUtensorMap* tm = icur == 0 ? &tmap_y0 : (icur == 1 ? &tmap_y1 : &tmap_y2);
      mbar_expect_tx(y_bar, (uint32_t)p.ksl * (uint32_t)p.nbox * 128u);
      for (int c = 0; c < nchunk; ++c)
        for (int j = 0; j < p.nbox; ++j)
          tma_load_2d(y_sm + ((size_t)c * p.nbox + j) * TC_BOX_BYTES, tm, y_bar, 32 * j, k0 + 32 * c);
    }
    // operands of the recurrence for this thread's share of the 16 x b output rows (independent of the product)
    float vc[16], vp[16];
#pragma unroll
    for (int cnt = 0; cnt < 16; ++cnt) {
      const int idx = tid + cnt * CF_THREADS;
      const int r = idx / bn, j = idx - r * bn;
      vc[cnt] = 0.f;
      vp[cnt] = 0.f;
      if (idx < 16 * bn && j < p.b) {
        const size_t off = (size_t)(row_base + r) * p.b + j;
        if (cb != 0.f) vc[cnt] = __ldcg(ycur + off);
        if (cg != 0.f) vp[cnt] = __ldcg(yprev + off);
      }
    }
    if (s == 1) mbar_wait(g_bar, 0);
    mbar_wait(y_bar, par);
    float acc[2][4 * NB][4];
    cf_product<NB>(g_sm, y_sm, nchunk, NB, acc);
    // accumulator (row 32w + 16i + g + 8h, column 8j + 2t + e) of the 128 x bn partial tile
    if (p.dsmem) {
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4 * NB; ++j)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            red[(size_t)(8 * j + 2 * t + (e & 1)) * CF_RED_LD + 32 * warp_idx + 16 * i + g + 8 * (e >> 1)] = acc[i][j][e];
      cluster_sync_all();  // all 8 partial tiles of the slab are in shared memory
#pragma unroll
      for (int cnt = 0; cnt < 16; ++cnt) {
        const int idx = tid + cnt * CF_THREADS;
        if (idx >= 16 * bn) break;
        const int r = idx / bn, j = idx - r * bn;
        const uint32_t laddr = red_addr + (uint32_t)((j * CF_RED_LD + 16 * (int)q + r) * 4);
        float sum = 0.f;
#pragma unroll
        for (uint32_t peer = 0; peer < CF_KS; ++peer) {
          uint32_t raddr;
          float x;
          asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(raddr) : "r"(laddr), "r"(peer));
          asm volatile("ld.shared::cluster.f32 %0, [%1];" : "=f"(x) : "r"(raddr) : "memory");
          sum += x;
        }
        if (j < p.b) yout[(size_t)(row_base + r) * p.b + j] = ca * sum + cb * vc[cnt] + cg * vp[cnt];
      }
    } else {
      float* out = p.partial + ((size_t)slab * CF_KS + q) * 128 * (size_t)bn;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float* orow = out + (size_t)(32 * warp_idx + 16 * i + g + 8 * h) * bn + 2 * t;
#pragma unroll
          for (int j = 0; j < 4 * NB; ++j)
            *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(acc[i][j][2 * h], acc[i][j][2 * h + 1]);
        }
      __threadfence();
      __syncthreads();
      if (tid == 0) cf_grid_barrier(p.counter, (unsigned)gridDim.x * (unsigned)(2 * s - 1));
      __syncthreads();
#pragma unroll
      for (int cnt = 0; cnt < 16; ++cnt) {
        const int idx = tid + cnt * CF_THREADS;
        if (idx >= 16 * bn) break;
        const int r = idx / bn, j = idx - r * bn;
        const float* src = p.partial + (((size_t)slab * CF_KS) * 128 + 16 * q + r) * (size_t)bn + j;
        float sum = 0.f;
#pragma unroll
        for (int peer = 0; peer < CF_KS; ++peer) sum += __ldcg(src + (size_t)peer * 128 * bn);
        if (j < p.b) yout[(size_t)(row_base + r) * p.b + j] = ca * sum + cb * vc[cnt] + cg * vp[cnt];
      }
    }
    __threadfence();
    asm volatile("fence.proxy.async;" ::: "memory");
    __syncthreads();
    if (tid == 0) cf_grid_barrier(p.counter, (unsigned)gridDim.x * (unsigned)(p.dsmem ? s : 2 * s));
    __syncthreads();
  }

  if (p.dsmem) cluster_sync_all();  // the peers may still be reading this CTA's partial tile
}

inline size_t cheb_filter_workspace_bytes(int n, int b) {
  return align_up((size_t)n * CF_KS * (size_t)((b + 31) / 32 * 32) * sizeof(float)) + 256;
}

// Runs `steps` filter products.  bufs[0] holds the input block; the result is left in bufs[steps % 3].
// ws: cheb_filter_workspace_bytes(n, b) of device scratch (grid-barrier counter + partial tiles).
// Returns TNB_ERR_UNSUPPORTED (without touching the blocks, reason in the last-error string) outside the
// envelope or when the driver refuses the cooperative launch, so that the caller can run the products one by one.
inline int cheb_filter_f32(const float* G, int n, int b, float* const bufs[3], int steps, const float* a,
                           const float* bc, const float* g, void* ws, size_t ws_bytes, cudaStream_t st,
                           const ChfsiCtrl* ctrl = nullptr, int stage = 0) {
  if (ctrl) steps = 1;  // the degree comes from the control block
  if (!tc_path_available() || !cheb_filter_shape_ok(n, b) || steps < 1 || steps > CF_MAX_STEPS ||
      ws_bytes < cheb_filter_workspace_bytes(n, b)) {
    last_error_ref() = "resident filter: shape outside the envelope or workspace too small";
    return TNB_ERR_UNSUPPORTED;
  }
  // everything remembered about the launch is per device: refused sizes, the chaining event, the cluster occupancy
  struct DevState {
    std::mutex mu;
    cudaEvent_t last = nullptr;
    int max_clusters = -1;  // co-resident clusters of 8 CTAs at the largest footprint
    unsigned refused = 0;   // sizes whose cooperative launch the driver refused once
  };
  static DevState states[TNB_MAX_DEVICES];
  DevState& ds = states[current_device_index()];
  if (ds.refused & (1u << (n / 256))) return TNB_ERR_UNSUPPORTED;
  ChebFilterParams p;
  p.n = n;
  p.b = b;
  p.nbox = (b + 31) / 32;
  p.ksl = n / CF_KS;
  p.steps = steps;
  p.ctrl = ctrl;
  p.stage = stage;
  for (int i = 0; i < steps && !ctrl; ++i) { p.a[i] = a[i]; p.bc[i] = bc[i]; p.g[i] = g[i]; }
  for (int i = 0; i < 3; ++i) p.buf[i] = bufs[i];
  p.counter = static_cast<unsigned*>(ws);
  p.partial = reinterpret_cast<float*>(static_cast<char*>(ws) + 256);
  CUtensorMap tg, ty[3];
  TNB_TRY(encode_rowmajor_f32(&tg, G, n, n));
  for (int i = 0; i < 3; ++i) TNB_TRY(encode_rowmajor_f32(&ty[i], bufs[i], n, b));
  const size_t smem = cheb_filter_smem_bytes(n, b);
  std::lock_guard<std::mutex> lk(ds.mu);
  cudaEvent_t& last = ds.last;
  int& max_clusters = ds.max_clusters;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)((n / 128) * CF_KS));
  cfg.blockDim = dim3(CF_THREADS);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  // Speculatively enqueued stages (ctrl != nullptr) are NOT cooperative launches: a cooperative launch — even of a stage
  // that will return at once because the solve has converged — waits until all of its CTAs fit on the GPU at the same
  // time, i.e. for a gap between the whole-GPU kernels of the other in-flight tensors.  A plain launch lets the CTAs of a
  // skipped stage drain through whatever SMs are free.  Co-residency of a stage that does run is still guaranteed:
  // grid <= SM count with one CTA per SM (checked in cheb_filter_shape_ok), the filter kernels of all streams are
  // chained by the event below so two of them never hold SMs at the same time, and no other kernel of this library waits
  // on a filter while holding SMs; the grid barrier additionally times out instead of spinning for ever.
  cudaLaunchAttribute attrs[2];
  attrs[0].id = cudaLaunchAttributeCooperative;
  attrs[0].val.cooperative = ctrl ? 0 : 1;
  attrs[1].id = cudaLaunchAttributeClusterDimension;
  attrs[1].val.clusterDim.x = CF_KS;
  attrs[1].val.clusterDim.y = 1;
  attrs[1].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  void (*const kernels[4])(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, ChebFilterParams) = {
      cheb_filter_kernel<1>, cheb_filter_kernel<2>, cheb_filter_kernel<3>, cheb_filter_kernel<4>};
  const auto kernel = kernels[p.nbox - 1];
  if (max_clusters < 0) {
    for (auto k : kernels) TNB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    TNB_CUDA(cudaEventCreateWithFlags(&last, cudaEventDisableTiming));
    cudaLaunchConfig_t probe = cfg;
    probe.dynamicSmemBytes = 227 * 1024 - 2048;
    probe.numAttrs = 2;
    int nc = 0;
    if (cudaOccupancyMaxActiveClusters(&nc, kernels[3], &probe) != cudaSuccess) nc = 0;
    cudaGetLastError();
    max_clusters = nc;
  }
  p.dsmem = (n / 128 <= max_clusters && !getenv("TNB_FILTER_NO_DSMEM")) ? 1 : 0;
  cfg.numAttrs = p.dsmem ? 2 : 1;
  TNB_CUDA(cudaMemsetAsync(p.counter, 0, sizeof(unsigned), st));
  // two resident filter kernels that each hold part of the SMs would wait on each other for ever:
  // chain them across streams
  TNB_CUDA(cudaStreamWaitEvent(st, last, 0));
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, tg, ty[0], ty[1], ty[2], p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    fail(TNB_ERR_UNSUPPORTED, "resident filter launch refused: %s (n=%d b=%d smem=%zu dsmem=%d, max active clusters %d)",
         cudaGetErrorString(e), n, b, smem, p.dsmem, max_clusters);
    if (getenv("TNB_DEBUG")) fprintf(stderr, "tnb200: %s\n", last_error_ref().c_str());
    ds.refused |= 1u << (n / 256);
    return TNB_ERR_UNSUPPORTED;
  }
  TNB_CUDA(cudaEventRecord(last, st));
  return TNB_OK;
}

}  // namespace tnb
