// Host orchestration of the right-to-left Gram sweep (dense TT-SVD), the TT rounding sweeps and
// the two-factor split.  Each routine is written once over an arena type so that the very same
// sequence of `take` calls sizes the workspace (ArenaSizer) and carves it (Arena).
//
// Dense TT-SVD (tn.Tensor(data, ranks_tt=r): tensor.py:401-408 -> round_tt tensor.py:2008-2083):
//   C <- T viewed (rows x I_{N-1});  for mu = N-1 .. 1:
//     G = C^T C (or C C^T when rows < cols)      Gram, fp64 accumulation   [replaces QR tensor.py:1816 + SVD round.py:96]
//     (lambda, V) = leading eigenpairs of G       Jacobi / Chebyshev subspace iteration
//     rank by the tail-energy rule                round.py:147-158
//     core_mu = V_r^T, C <- C V_r                 round.py:166-172 + tensor.py:2078-2083
//   core_0 = C.
// This is algebraically the reference's result (same subspaces, same gauge: cores 1..N-1 have
// orthonormal right unfoldings, core 0 carries the norm) without the identity-flanked full-rank TT.
#pragma once
#include "common.cuh"
#include "eig.cuh"
#include "gemm_generic.cuh"
#include "jacobi.cuh"
#include "jacobi2.cuh"
#include "small_kernels.cuh"
#include "gram_tc.cuh"
#include "project.cuh"
#include "project_tc.cuh"
#include "chfsi_dev.cuh"

namespace tnb {

// The input of the dense TT-SVD may be bf16 or fp16 (TIn); only step 0 reads it, every carry and core is T (fp32 for
// 16-bit input).
template <typename TIn>
constexpr bool tc_input() {
  return std::is_same<TIn, float>::value || std::is_same<TIn, __nv_bfloat16>::value || std::is_same<TIn, __half>::value;
}

// C (rows x r) = A (rows x n) * V (n x r) in the data precision (fp32 for 16-bit A): tensor-core kernel, streaming FFMA
// kernel for fp32 when the shape allows, generic tiled GEMM otherwise.
constexpr int64_t PROJ_TC_MIN_ROWS = 16384;
template <typename TIn = float>
inline bool project_use_tc(int64_t rows, int64_t n, int64_t r, const void* A, const void* C) {
  return tc_input<TIn>() && rows >= PROJ_TC_MIN_ROWS && project_tc_shape_ok<TIn>(rows, n, r, A, C);
}
template <typename T, typename TIn = T>
inline int project_any(const TIn* A, int64_t rows, int64_t n, const T* V, int64_t r, T* C, cudaStream_t st,
                       void* tc_ws = nullptr, size_t tc_ws_bytes = 0) {
  if constexpr (tc_input<TIn>())
    if (tc_ws && tc_path_available() && project_use_tc<TIn>(rows, n, r, A, C))
      return project_tc<TIn>(A, rows, n, reinterpret_cast<const float*>(V), (int)r, reinterpret_cast<float*>(C), tc_ws,
                             tc_ws_bytes, st);
  if (std::is_same<TIn, float>::value && project_f32_fast_ok(rows, n, r, A, C))
    return project_f32_fast(reinterpret_cast<const float*>(A), rows, n, reinterpret_cast<const float*>(V), (int)r,
                            reinterpret_cast<float*>(C), st);
  return gemm_direct<TIn, T, T, T>(rows, r, n, A, n, true, V, r, false, C, r, (T)1, nullptr, 0, (T)0, nullptr, 0, (T)0, st);
}
// Workspace of the tensor-core projection of a step (0: the step projects elsewhere).
template <typename TIn>
inline size_t project_tc_carve_bytes(bool allow_tc, int64_t rows, int64_t n, int64_t kcap) {
  if (!allow_tc || !tc_input<TIn>() || rows < n || !project_use_tc<TIn>(rows, n, kcap, nullptr, nullptr)) return 0;
  return project_tc_workspace_bytes<TIn>(n, kcap);
}

constexpr int64_t TC_MIN_ROWS = 2048;  // below this the generic fp64-accumulating Gram is used

struct SweepDims {
  int N = 0;
  std::vector<int64_t> shape;
  std::vector<int64_t> rows;   // rows[mu] = prod_{j<mu} shape[j]
  std::vector<int64_t> rcap;   // rcap[k], k=0..N : max possible rank at bond k
  std::vector<int64_t> slot;   // element offset of core k in the cores buffer
  int64_t capacity = 0;
};

inline int make_dims(int ndim, const int64_t* shape, const int32_t* rmax, SweepDims& d) {
  if (ndim < 1 || ndim > 62) return fail(TNB_ERR_INVALID, "ndim=%d out of range", ndim);
  d.N = ndim;
  d.shape.assign(shape, shape + ndim);
  for (int k = 0; k < ndim; ++k)
    if (shape[k] < 1) return fail(TNB_ERR_INVALID, "shape[%d]=%lld must be >= 1", k, (long long)shape[k]);
  d.rows.assign(ndim + 1, 1);
  for (int k = 0; k < ndim; ++k) {
    if (d.rows[k] > (int64_t)1 << 56) return fail(TNB_ERR_INVALID, "tensor too large");
    d.rows[k + 1] = d.rows[k] * shape[k];
  }
  d.rcap.assign(ndim + 1, 1);
  for (int mu = ndim - 1; mu >= 1; --mu) {
    int64_t c = shape[mu] * d.rcap[mu + 1];
    if (d.rows[mu] < c) c = d.rows[mu];
    if (rmax && rmax[mu - 1] > 0 && rmax[mu - 1] < c) c = rmax[mu - 1];
    d.rcap[mu] = c;
  }
  d.slot.assign(ndim, 0);
  int64_t off = 0;
  for (int k = 0; k < ndim; ++k) {
    d.slot[k] = off;
    off += d.rcap[k] * shape[k] * d.rcap[k + 1];
    off = (off + 63) / 64 * 64;  // keep every core 256-byte aligned for fp32
  }
  d.capacity = off;
  return TNB_OK;
}

// The carry that step mu + 1 writes and step mu reads, M (rows' x n' = d.rows[mu] x shape[mu] * rcap[mu+1]), is stored
// K-blocked, as wgmma's K-major core matrices (gram_tc.cuh), when the speculative sweep runs both ends on kernels that have that form:
// step mu takes the tensor-core Gram unfolded (n' >= 256) and the tensor-core projection, and step mu + 1 projects on the
// tensor cores with an epilogue that can write it (rcap[mu+1] % 16 == 0 and <= 48, shape[mu] % 16 == 0).  Its Gram then loads
// K-major operands directly instead of transposing every slab in shared memory.  The writer's own input must be
// row-major (fp32, or the bf16 / fp16 input when the writer is step 0), and the last carry (step mu = 0's core) stays
// row-major.
template <typename T, typename TIn = T>
inline bool carry_kblocked(const SweepDims& d, int mu, bool allow_tc) {
  if (!std::is_same<T, float>::value || !allow_tc || mu < 1 || mu + 1 > d.N - 1) return false;
  const int64_t rows = d.rows[mu], n = d.shape[mu] * d.rcap[mu + 1], k = std::min<int64_t>(d.rcap[mu], n);
  const bool reader = rows >= n && rows >= std::max(TC_MIN_ROWS, PROJ_TC_MIN_ROWS) && gram_tc_kblocked_shape_ok(rows, n) &&
                      k <= PT_MAX_N && project_tc_shape_ok(rows, n, k, nullptr, nullptr);
  const int64_t wrows = d.rows[mu + 1], wn = d.shape[mu + 1] * d.rcap[mu + 2], r = d.rcap[mu + 1];
  const bool wtc = mu + 1 == d.N - 1 ? project_use_tc<TIn>(wrows, wn, r, nullptr, nullptr)
                                     : project_use_tc<T>(wrows, wn, r, nullptr, nullptr);
  const bool writer = wrows >= wn && wn >= 32 && wtc && r % 16 == 0 && r <= 48 && d.shape[mu] % 16 == 0;
  return reader && writer && !carry_kblocked<T, TIn>(d, mu + 1, allow_tc);
}

// ---------------------------------------------------------------------------------------------
// Gram of a (rows x n) row-major matrix on whichever side is smaller, into fp64 G (L x L).
// ---------------------------------------------------------------------------------------------
struct GramWork {  // untyped buffers: the same for every input type
  double* partial = nullptr;
  size_t partial_elems = 0;
  void* tc_ws = nullptr;
  size_t tc_bytes = 0;
};

template <typename T, class ArenaT>
inline void gram_carve(ArenaT& ar, int64_t rows, int64_t n, bool allow_tc, GramWork& w) {  // T: the input type
  const bool tall = rows >= n;
  const int64_t L = tall ? n : rows;
  const int64_t K = tall ? rows : n;
  GemmPlan pl = plan_gemm(L, L, K, true);
  w.partial_elems = pl.partial_elems;
  w.partial = ar.template take<double>(pl.partial_elems);
  w.tc_bytes = 0;
  w.tc_ws = nullptr;
  if (allow_tc && tall && rows >= TC_MIN_ROWS && gram_tc_input_ok<T>(rows, n)) {
    w.tc_bytes = gram_tc_input_workspace_bytes<T>(rows, n);
    w.tc_ws = ar.template take<char>(w.tc_bytes);
  }
}

// *used_tc: 0 exact-product Gram, 1 TF32 tensor-core Gram, 2 bf16 tensor-core Gram, 3 fp16 tensor-core Gram (gram_noise)
template <typename T>
inline int gram_small_side(const T* C, int64_t rows, int64_t n, double* G, float* Gf, GramWork& w, bool use_tc,
                           int* used_tc, cudaStream_t st) {
  const bool tall = rows >= n;
  if (used_tc) *used_tc = 0;
  if (tall) {
    if constexpr (tc_input<T>())
      if (use_tc && w.tc_ws) {
        if (used_tc) *used_tc = std::is_same<T, __nv_bfloat16>::value ? 2 : std::is_same<T, __half>::value ? 3 : 1;
        return gram_tc<T>(C, rows, n, G, Gf, w.tc_ws, w.tc_bytes, st);
      }
    GemmPlan pl = plan_gemm(n, n, rows, true);
    return gemm_splitk<T, T, double, double, float>(pl, n, n, rows, C, n, false, C, n, false, w.partial, G, n, 1.0,
                                                    nullptr, 0, 0.0, nullptr, 0, 0.0, true, Gf, n, st);
  }
  GemmPlan pl = plan_gemm(rows, rows, n, true);
  return gemm_splitk<T, T, double, double, float>(pl, rows, rows, n, C, n, true, C, n, true, w.partial, G, rows, 1.0,
                                                  nullptr, 0, 0.0, nullptr, 0, 0.0, true, Gf, rows, st);
}

// The accept rule's noise level for a Gram made as gram_small_side's *used_tc says (0: exact, nothing to guard), and,
// when its eigenpairs come from an fp32 solve, at least the TF32 level that covers the solve (spec_step_eig_begin).
inline double gram_noise(int used_tc, bool fp32_solve = false) {
  const double g = used_tc == 3 ? FP16_GRAM_NOISE : used_tc == 2 ? BF16_GRAM_NOISE : used_tc ? TF32_GRAM_NOISE : 0.0;
  return fp32_solve ? std::max(g, TF32_GRAM_NOISE) : g;
}

// ---------------------------------------------------------------------------------------------
// Eigen stage: all eigenpairs (Jacobi) when L <= JACOBI_MAX_N, else k leading pairs (ChFSI).
// Outputs: w (>= L or b doubles, descending), V (L x ldv doubles, columns = vectors).
// ---------------------------------------------------------------------------------------------
template <typename TBk>
struct EigWork {
  double* w = nullptr;
  double* V = nullptr;
  int ldv = 0;
  double* jscratch = nullptr;
  int* jinfo = nullptr;
  bool chfsi = false;
  bool adaptive = false;  // eps-only: k grows until the rank rule is decided
  int k = 0, b = 0;       // capacity (carved); k_run / b_run are what the last solve used
  int k_run = 0, b_run = 0;
  TBk* Gb = nullptr;  // G in block precision (ChFSI only)
  ChfsiWork<TBk> cw;
};

template <typename TBk, class ArenaT>
inline int eig_carve(ArenaT& ar, int64_t L, int64_t rcap, bool have_rmax, EigWork<TBk>& e) {
  if (L <= JACOBI_MAX_N) {
    e.chfsi = false;
    e.w = ar.template take<double>(L);
    e.V = ar.template take<double>((size_t)L * L);
    e.ldv = (int)L;
    e.jscratch = ar.template take<double>(jacobi_scratch_doubles((int)L));
    e.jinfo = ar.template take<int>(4);
    return TNB_OK;
  }
  // eps-only truncation (no rank cap) of a large Gram matrix: the leading values are computed in growing blocks
  // (k = 32, 64, 128, 240) until the tail-energy rule is decided; ranks above 240 are out of reach of the subspace
  // eigensolver and raise.
  e.adaptive = !have_rmax;
  if (have_rmax && rcap + 16 > JACOBI_MAX_N)
    return fail(TNB_ERR_UNSUPPORTED, "target rank %lld too large for the subspace eigensolver (limit %d) at Gram size %lld",
                (long long)rcap, JACOBI_MAX_N - 16, (long long)L);
  if (!have_rmax || rcap + 16 > JACOBI_MAX_N) rcap = JACOBI_MAX_N - 16;
  if (L > 46000) return fail(TNB_ERR_UNSUPPORTED, "Gram size %lld too large", (long long)L);
  e.chfsi = true;
  e.k = (int)rcap;
  e.b = chfsi_default_block((int)L, e.k);
  e.w = ar.template take<double>(e.b);
  e.V = ar.template take<double>((size_t)L * e.b);
  e.ldv = e.b;
  if (!std::is_same<TBk, double>::value) e.Gb = ar.template take<TBk>((size_t)L * L);
  chfsi_carve<TBk>(ar, (int)L, e.b, e.cw);
  return TNB_OK;
}

template <typename TBk>
inline int eig_run(const double* G, const TBk* Gb_in, int64_t L, EigWork<TBk>& e, const double* d_trace,
                   ChfsiStats* stats, cudaStream_t st, bool allow_tc = false, bool shared_gpu = false, int k_try = 0,
                   double tol = 1e-6) {
  if (!e.chfsi) return jacobi2_eigh(G, (int)L, (int)L, e.w, e.V, e.jscratch, e.jinfo, st);
  e.cw.use_tc = allow_tc;
  e.cw.shared_gpu = shared_gpu;
  e.cw.narrow = shared_gpu && getenv("TNB_NARROW") != nullptr;
  e.k_run = (k_try > 0 && k_try < e.k) ? k_try : e.k;
  e.b_run = chfsi_default_block((int)L, e.k_run);
  if (e.b_run > e.b) e.b_run = e.b;
  e.ldv = e.b_run;
  const TBk* Gb = Gb_in;
  if (std::is_same<TBk, double>::value) Gb = reinterpret_cast<const TBk*>(G);
  return eig_topk_chfsi<TBk>(Gb, (int)L, e.k_run, e.b_run, d_trace, tol, e.cw, e.w, e.V, stats, st);
}

// Eigen stage + rank rule + host read-back of the step scalars (one sync, which the caller needs anyway for the rank).
// eps-only truncation of a large Gram matrix (EigWork::adaptive) repeats the subspace solve with k = 32, 64, 128, 240
// leading values until the tail-energy rule is decided, with a stopping rule fine enough to resolve delta^2.
template <typename TBk>
inline int eig_solve_and_rank(const double* G, const TBk* Gb, int64_t L, EigWork<TBk>& ew, SweepScalars* sc, int* h_sc,
                              int32_t rm, int batch_mode, ChfsiStats* total, int* solves, cudaStream_t st, bool allow_tc,
                              bool shared_gpu, int used_tc = 0) {
  const SweepScalars* hs = reinterpret_cast<const SweepScalars*>(h_sc);
  const bool adaptive = ew.chfsi && ew.adaptive;
  int k_try = adaptive ? 32 : 0;
  double tol = 1e-6;
  if (adaptive) {
    TNB_CUDA(cudaMemcpyAsync(h_sc, sc, sizeof(SweepScalars), cudaMemcpyDeviceToHost, st));
    TNB_CUDA(cudaStreamSynchronize(st));
    const double floor_tol = std::is_same<TBk, float>::value ? 1e-7 : 1e-12;  // what fp32 / fp64 Ritz sums can resolve
    if (hs->trace > 0.0) tol = std::min(1e-6, std::max(floor_tol, 0.05 * hs->delta2 / hs->trace));
  }
  for (;;) {
    ChfsiStats cs;
    TNB_TRY(eig_run<TBk>(G, Gb, L, ew, &sc->trace, &cs, st, allow_tc, shared_gpu, k_try, tol));
    if (total)
      total->products += cs.products, total->fused_filters += cs.fused_filters, total->outer += cs.outer,
          total->rr_sweeps += cs.rr_sweeps;
    if (solves) *solves += 1;
    rank_rule_kernel<<<1, 32, 0, st>>>(ew.w, (int)L, ew.chfsi ? ew.k_run : (int)L, rm, ew.chfsi ? 1 : 0, batch_mode, sc,
                                       gram_noise(used_tc), ew.chfsi ? ew.b_run : (int)L);
    TNB_LAUNCH_CHECK();
    TNB_CUDA(cudaMemcpyAsync(h_sc, sc, sizeof(SweepScalars), cudaMemcpyDeviceToHost, st));
    TNB_CUDA(cudaStreamSynchronize(st));
    if (!adaptive || !hs->undecided || hs->zero_flag) return TNB_OK;
    if (ew.k_run >= ew.k)
      return fail(TNB_ERR_UNSUPPORTED,
                  "eps-only truncation of a %lld x %lld Gram matrix needs a rank above %d; pass rmax / ranks_tt "
                  "(the direct eigensolver stops at %d)", (long long)L, (long long)L, ew.k, JACOBI_MAX_N);
    k_try = 2 * ew.k_run > 128 ? ew.k : 2 * ew.k_run;
  }
}

// ---------------------------------------------------------------------------------------------
// One truncation step, shared by the dense sweep and by phase B of TT rounding.
//   C (rows x n, row-major)  ->  core (rank x n, orthonormal rows)  and  Cn (rows x rank) with
//   C ~= Cn * core, exactly what tn.truncated_svd(M, left_ortho=False) returns (round.py:166-172,181)
//   for M = the right unfolding the reference holds at tensor.py:2054.
// ---------------------------------------------------------------------------------------------
struct SweepInfo {
  double norm = 0;
  int eig_solves = 0;
  int chfsi_products = 0;
  int fused_filters = 0;  // Chebyshev filters run as one resident kernel (cheb_filter.cuh)
  int rr_sweeps = 0, rr_solves = 0;  // Jacobi sweeps / solves of the Rayleigh-Ritz steps (diagnostic)
  int tc_grams = 0;
  int kblocked_steps = 0;  // steps whose Gram and projection read a K-blocked carry (carry_kblocked)
  int speculative = 0;  // 1: the sync-free sweep was accepted (one host synchronisation in total)
  int spec_flags = 0;   // why a speculative sweep was repeated on the host-driven path (spec_check_kernel bits)
  // TNB_FLAG_PROFILE: CUDA-event timings (ms) on the launching stream, per step (t = 0 is the first Gram)
  int nsteps = 0;
  double gram_ms[8] = {0}, eig_ms[8] = {0}, factor_ms[8] = {0};
};

// Event-based phase profiler (only active under TNB_FLAG_PROFILE; events are recorded on the stream the
// kernels are launched on, and read after the per-step synchronisation the sweep performs anyway).
struct Prof {
  bool on = false;
  std::vector<cudaEvent_t> ev;
  int used = 0;
  cudaEvent_t next() {
    if (used == (int)ev.size()) {
      cudaEvent_t e;
      cudaEventCreate(&e);
      ev.push_back(e);
    }
    return ev[used++];
  }
  void mark(cudaStream_t st) {
    if (on) cudaEventRecord(next(), st);
  }
  // after the stream has been synchronised; 4 events per step: start, after Gram, after eigen+rank, after
  // factor/projection
  void collect(SweepInfo* info) {
    if (on && info) {
      const int steps = used / 4;
      info->nsteps = steps;
      for (int t = 0; t < steps && t < 8; ++t) {
        float a = 0, b = 0, c = 0;
        cudaEventElapsedTime(&a, ev[4 * t], ev[4 * t + 1]);
        cudaEventElapsedTime(&b, ev[4 * t + 1], ev[4 * t + 2]);
        cudaEventElapsedTime(&c, ev[4 * t + 2], ev[4 * t + 3]);
        info->gram_ms[t] = a;
        info->eig_ms[t] = b;
        info->factor_ms[t] = c;
      }
    }
    on = false;
  }
  static Prof& get() {
    static thread_local Prof p;
    return p;
  }
};

struct StepCtx {
  SweepScalars* sc = nullptr;   // device
  int* h_sc = nullptr;          // pinned host mirror
  uint32_t flags = 0;
  bool allow_tc = false;
  double eps_scaled2 = 0;       // (eps / max(1, sqrt(N-1)))^2
  SweepInfo* info = nullptr;
  cudaStream_t st = 0;
  bool exact_gram = false;      // a TF32 Gram was rejected for this tensor: take the exact-product Gram throughout
  // speculative (sync-free) sweep
  int* d_flags = nullptr;       // device flags raised by spec_check_kernel / cd_finish_kernel
  int32_t* d_ranks = nullptr;   // device copy of the ranks the rule chose, [N + 1]
};

// The context of a sweep over N modes.  Carves the device scalars and, for a speculative sweep, then its flags and ranks.
template <class ArenaT>
inline StepCtx make_step_ctx(ArenaT& ar, int N, double eps, uint32_t flags, bool allow_tc, SweepInfo* info,
                             cudaStream_t st, bool speculative) {
  StepCtx cx;
  cx.flags = flags;
  cx.allow_tc = allow_tc;
  cx.info = info;
  cx.st = st;
  const double epsN = eps / std::max(1.0, std::sqrt((double)(N - 1)));
  cx.eps_scaled2 = epsN * epsN;
  cx.sc = ar.template take<SweepScalars>(1);
  if (speculative) {
    cx.d_flags = ar.template take<int>(4);
    cx.d_ranks = ar.template take<int32_t>(N + 1);
  }
  return cx;
}

// The end of a truncation step at rank `rank`, from the step's eigenpairs (w descending, V with leading dimension ldv):
//   tall (rows >= n): core = V_r^T (rank x n);  Cn = C V_r;
//   wide:             core = diag(1/s) U_r^T C (rank x n);  Cn = U_r diag(s).
// fac (L x rank) is scratch; ptc_ws the tensor-core projection's workspace (project_tc_carve_bytes).  `layout` is
// PT_ROWMAJOR unless the speculative sweep reads (PT_IN_KBLOCKED) or writes (PT_OUT_KBLOCKED, out_inner) a K-blocked carry.
template <typename T, typename TIn>
inline int step_factors(const StepCtx& cx, const TIn* C, int64_t rows, int64_t n, int64_t rank, const double* w,
                        const double* V, int ldv, T* fac, void* ptc_ws, size_t ptc_bytes, T* core, T* Cn,
                        int layout = PT_ROWMAJOR, int64_t out_inner = 0) {
  cudaStream_t st = cx.st;
  if (rows >= n) {
    scale_extract_kernel<T><<<grid_for(n * rank), 256, 0, st>>>(V, ldv, (int)n, (int)rank, w, core, 0, 1);
    TNB_LAUNCH_CHECK();
    scale_extract_kernel<T><<<grid_for(n * rank), 256, 0, st>>>(V, ldv, (int)n, (int)rank, w, fac, 0, 0);
    TNB_LAUNCH_CHECK();
    BigKernelGate gate(st, (cx.flags & TNB_FLAG_CONCURRENT) && rows >= PROJ_TC_MIN_ROWS);
    if constexpr (tc_input<TIn>())
      if (layout != PT_ROWMAJOR)
        return project_tc<TIn>(C, rows, n, reinterpret_cast<const float*>(fac), (int)rank, reinterpret_cast<float*>(Cn),
                               ptc_ws, ptc_bytes, st, layout, out_inner);
    return project_any<T, TIn>(C, rows, n, fac, rank, Cn, st, ptc_ws, ptc_bytes);
  }
  scale_extract_kernel<T><<<grid_for(rows * rank), 256, 0, st>>>(V, ldv, (int)rows, (int)rank, w, fac, 1, 0);
  TNB_LAUNCH_CHECK();
  TNB_TRY((gemm_direct<T, TIn, T, T>(rank, n, rows, fac, rank, false, C, n, false, core, n, (T)1, nullptr, 0, (T)0,
                                     nullptr, 0, (T)0, st)));
  scale_extract_kernel<T><<<grid_for(rows * rank), 256, 0, st>>>(V, ldv, (int)rows, (int)rank, w, Cn, 2, 0);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// TIn: the element type of C (the dense input at step 0, else T).
template <typename T, typename TIn, class ArenaT>
inline int truncate_step(ArenaT& ar, bool dry, const StepCtx& cx, const TIn* C, int64_t rows, int64_t n, int64_t rank_cap,
                         bool have_rmax, int32_t rm, bool first_step, T* core, T* Cn, int64_t* rank_out) {
  typedef T TBk;  // block precision of the subspace eigensolver follows the data
  const bool tall = rows >= n;
  const int64_t L = tall ? n : rows;
  const int batch_mode = (cx.flags & TNB_FLAG_BATCH_MODE) ? 1 : 0;
  cudaStream_t st = cx.st;
  GramWork gw;
  EigWork<TBk> ew;
  // The TF32 Gram equals (1 - c) * G, c ~ 7e-4 (operand truncation shrinks every product alike: harmless, the rank
  // rule works on ratios) plus noise of ~1.6e-6 * ||G|| (measured, tests/test_model.py) — a floor under the tail
  // energies the rank rule can resolve.  An eps budget between "inactive" and 1e-4 of the trace needs finer
  // resolution than that: those sweeps take the exact-product fp64-accumulating Gram instead.
  const bool tc_gram = cx.allow_tc && !cx.exact_gram && (dry || cx.eps_scaled2 < 1e-20 || cx.eps_scaled2 >= 1e-4);
  gram_carve<TIn>(ar, rows, n, tc_gram, gw);
  double* G = ar.template take<double>((size_t)L * L);
  float* Gf = nullptr;
  const int64_t kcap = std::min<int64_t>(rank_cap, L);
  TNB_TRY(eig_carve<TBk>(ar, L, kcap, have_rmax, ew));
  if (ew.chfsi && std::is_same<TBk, float>::value) Gf = reinterpret_cast<float*>(ew.Gb);
  T* fac = ar.template take<T>((size_t)L * (size_t)kcap);  // V_r or U_r/s
  const size_t ptc_bytes = project_tc_carve_bytes<TIn>(cx.allow_tc, rows, n, kcap);
  void* ptc_ws = ptc_bytes ? ar.template take<char>(ptc_bytes) : nullptr;
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "workspace too small (need > %zu bytes)", ar.off);
  Prof& prof = Prof::get();
  prof.mark(st);
  int used_tc = 0;
  const bool concurrent = (cx.flags & TNB_FLAG_CONCURRENT) != 0;
  {
    BigKernelGate gate(st, concurrent && gw.tc_ws != nullptr);
    TNB_TRY(gram_small_side<TIn>(C, rows, n, G, Gf, gw, tc_gram, &used_tc, st));
  }
  if (cx.info) cx.info->tc_grams += used_tc ? 1 : 0;
  trace_kernel<<<1, 256, 0, st>>>(G, (int)L, (int)L, cx.sc, first_step ? 1 : 0, cx.eps_scaled2);
  TNB_LAUNCH_CHECK();
  prof.mark(st);
  ChfsiStats cs;
  int solves = 0;
  TNB_TRY(eig_solve_and_rank<TBk>(G, reinterpret_cast<const TBk*>(Gf), L, ew, cx.sc, cx.h_sc, rm, batch_mode, &cs, &solves, st,
                                  cx.allow_tc, concurrent, used_tc));
  if (used_tc && reinterpret_cast<const SweepScalars*>(cx.h_sc)->tf32_reject) {
    // the spectrum is too steep for the TF32 noise floor (small_kernels.cuh::tf32_gram_rejected): same step again on
    // the exact-product, fp64-accumulated Gram
    if (cx.info) cx.info->tc_grams -= 1;
    used_tc = 0;
    TNB_TRY(gram_small_side<TIn>(C, rows, n, G, Gf, gw, false, nullptr, st));
    trace_kernel<<<1, 256, 0, st>>>(G, (int)L, (int)L, cx.sc, first_step ? 1 : 0, cx.eps_scaled2);
    TNB_LAUNCH_CHECK();
    TNB_TRY(eig_solve_and_rank<TBk>(G, reinterpret_cast<const TBk*>(Gf), L, ew, cx.sc, cx.h_sc, rm, batch_mode, &cs, &solves,
                                    st, cx.allow_tc, concurrent, 0));
  }
  if (cx.info) cx.info->eig_solves += solves, cx.info->chfsi_products += cs.products, cx.info->fused_filters += cs.fused_filters,
        cx.info->rr_sweeps += cs.rr_sweeps, cx.info->rr_solves += cs.outer;
  prof.mark(st);
  const SweepScalars* hs = reinterpret_cast<const SweepScalars*>(cx.h_sc);
  if (first_step && cx.info) cx.info->norm = std::sqrt(hs->norm2 > 0 ? hs->norm2 : 0.0);
  int64_t rank = hs->rank;
  if (rank > kcap) rank = kcap;
  if (hs->zero_flag) {  // round.py:137-145: rank-1 zero factors
    rank = 1;
    fill_kernel<T><<<grid_for(n), 256, 0, st>>>(core, n, (T)0);
    TNB_LAUNCH_CHECK();
    fill_kernel<T><<<grid_for(rows), 256, 0, st>>>(Cn, rows, (T)0);
    TNB_LAUNCH_CHECK();
  } else {
    TNB_TRY((step_factors<T, TIn>(cx, C, rows, n, rank, ew.w, ew.V, ew.ldv, fac, ptc_ws, ptc_bytes, core, Cn)));
  }
  prof.mark(st);
  *rank_out = rank;
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// The same truncation step, SPECULATIVE: enqueued without any host round trip, assuming the rank rule will return the
// cap (rank_cap) — which it does whenever a rank cap decides (ranks_tt= with an inactive eps budget, the benchmark's
// and the common case).  The rule still runs on the device; spec_check_kernel records what it chose and raises a flag
// if it differs (rank-deficient data, zero unfolding), if the TF32 Gram is not accurate enough for this spectrum, or if
// the sync-free subspace solver failed; the caller looks at the flags ONCE, after the whole sweep, and repeats the
// decomposition on the host-driven path when any is set.  Eligibility is decided up front by spec_eligible().
// ---------------------------------------------------------------------------------------------
template <typename T>
inline bool spec_step_ok(int64_t rows, int64_t n, int64_t rank_cap, bool allow_tc) {
  const int64_t L = rows >= n ? n : rows;
  if (L <= JACOBI_MAX_N) return true;
  if (!std::is_same<T, float>::value || !allow_tc) return false;
  const int64_t k = std::min<int64_t>(rank_cap, L);
  if (k + 16 > JACOBI_MAX_N) return false;
  return chfsi_dev_ok((int)L, chfsi_dev_block((int)L, (int)k));
}

// The step is split in enqueue phases so that a batch of tensors can be interleaved phase by phase (spec_enqueue: all
// Gram kernels of a step first, then every tensor's eigen stages, then every tensor's projection): the whole-GPU kernels
// of the batch then run back to back while the latency-bound eigen chains of the other tensors run beside them on their
// own streams.
template <typename T>
struct SpecStep {
  GramWork gw;
  double *G = nullptr, *w = nullptr, *V = nullptr, *jscratch = nullptr;
  int* jinfo = nullptr;
  float* Gf = nullptr;
  CdWork<float> cw;
  T* fac = nullptr;
  void* ptc_ws = nullptr;
  size_t ptc_bytes = 0;
  int ldv = 0, b = 0, used_tc = 0;
  bool chfsi = false, tc_gram = false;
  bool fp32_solve = false;    // the small Gram's eigenpairs come from fp32 Jacobi rotations
  bool in_kblocked = false;   // C is K-blocked (carry_kblocked of this step)
  int64_t out_inner = 0;      // > 0: write Cn K-blocked for the next step, whose rows hold out_inner rows of Cn each
  int64_t L = 0, kcap = 0;
  CdRun cd;  // the subspace solve of this step, enqueued stage by stage
};

template <typename T, typename TIn, class ArenaT>
inline void spec_step_carve(ArenaT& ar, const StepCtx& cx, int64_t rows, int64_t n, int64_t rank_cap, SpecStep<T>& s) {
  const bool tall = rows >= n;
  s.L = tall ? n : rows;
  const int64_t L = s.L;
  s.tc_gram = cx.allow_tc && !cx.exact_gram;
  gram_carve<TIn>(ar, rows, n, s.tc_gram, s.gw);
  s.G = ar.template take<double>((size_t)L * L);
  s.kcap = std::min<int64_t>(rank_cap, L);
  s.chfsi = L > JACOBI_MAX_N;
  s.ldv = (int)L;
  s.b = 0;
  s.Gf = nullptr;
  if (!s.chfsi) {
    s.w = ar.template take<double>(L);
    s.V = ar.template take<double>((size_t)L * L);
    s.jscratch = ar.template take<double>(jacobi_scratch_doubles((int)L));
    s.jinfo = ar.template take<int>(4);
  } else {
    s.b = chfsi_dev_block((int)L, (int)s.kcap);
    s.w = ar.template take<double>(s.b);
    s.V = ar.template take<double>((size_t)L * s.b);
    s.ldv = s.b;
    s.Gf = ar.template take<float>((size_t)L * L);
    chfsi_dev_carve<float>(ar, (int)L, s.b, s.cw);
  }
  s.fac = ar.template take<T>((size_t)L * (size_t)s.kcap);
  s.ptc_bytes = project_tc_carve_bytes<TIn>(cx.allow_tc, rows, n, s.kcap);
  s.ptc_ws = s.ptc_bytes ? ar.template take<char>(s.ptc_bytes) : nullptr;
}

// phase 1: Gram + trace
template <typename T, typename TIn>
inline int spec_step_gram(const StepCtx& cx, const TIn* C, int64_t rows, int64_t n, bool first_step, SpecStep<T>& s, bool prof_on) {
  cudaStream_t st = cx.st;
  Prof& prof = Prof::get();
  if (prof_on) prof.mark(st);
  const bool concurrent = (cx.flags & TNB_FLAG_CONCURRENT) != 0;
  {
    BigKernelGate gate(st, concurrent && s.gw.tc_ws != nullptr);
    if (s.in_kblocked) {
      s.used_tc = 1;
      TNB_TRY(gram_tc(reinterpret_cast<const float*>(C), rows, n, s.G, s.Gf, s.gw.tc_ws, s.gw.tc_bytes, st, true));
    } else {
      TNB_TRY(gram_small_side<TIn>(C, rows, n, s.G, s.Gf, s.gw, s.tc_gram, &s.used_tc, st));
    }
  }
  if (cx.info) cx.info->tc_grams += s.used_tc ? 1 : 0, cx.info->kblocked_steps += s.in_kblocked ? 1 : 0;
  trace_kernel<<<1, 256, 0, st>>>(s.G, (int)s.L, (int)s.L, cx.sc, first_step ? 1 : 0, cx.eps_scaled2);
  TNB_LAUNCH_CHECK();
  if (prof_on) prof.mark(st);
  return TNB_OK;
}

// phase 2a: start the eigen stage — a small Gram matrix is solved right here (one Jacobi kernel), a large one begins its
// subspace solve, whose stages are enqueued one at a time by spec_step_eig_stage so that a batch can interleave them
template <typename T>
inline int spec_step_eig_begin(const StepCtx& cx, SpecStep<T>& s) {
  const int64_t L = s.L;
  cudaStream_t st = cx.st;
  if (!s.chfsi) {
    // a TF32 Gram is accurate to ~2e-6 ||G||: rotating it in fp32 (backward error ~1e-6 ||G||, covered by the accept rule's
    // noise allowance) is consistent with it and cheaper than fp64 rotations.  The stop is at 2e-7, near the fp32
    // resolution, not at the noise level: the eigenvectors at the rank cutoff decide what the next steps see (a 2e-6 stop
    // moved a flat-spectrum randn 64^4 decomposition by 3e-6 in relative error against the fp64 rotations);
    // eigenvalues still come out as fp64 Rayleigh quotients and the vectors are re-orthonormalised (jacobi2.cuh).
    // The same holds for fp32 DATA whatever Gram kernel produced G, as long as the accept rule — which then guards the
    // fp32 solve instead of the TF32 Gram, same noise allowance — finds the spectrum benign; a rejected step is repeated
    // on the host-driven path with fp64 rotations.
    // The rule then allows for the larger of the Gram kernel's noise and the fp32 solve's (gram_noise).
    const bool single = std::is_same<T, float>::value && (cx.allow_tc && !cx.exact_gram) && jacobi2_ok((int)L, true);
    s.fp32_solve = single;
    return jacobi2_eigh(s.G, (int)L, (int)L, s.w, s.V, s.jscratch, s.jinfo, st, single, single ? 2e-7 : 0.0);
  }
  if (cx.info) cx.info->eig_solves += 1;
  return cd_begin(s.cd, s.Gf, (int)L, (int)s.kcap, s.b, &cx.sc->trace, 1e-6, s.cw, s.w, s.V, cx.d_flags, st);
}
template <typename T>
inline int spec_step_eig_stage(SpecStep<T>& s, int stage) {
  return s.chfsi ? cd_stage(s.cd, stage) : TNB_OK;
}

// phase 2b: end of the eigen stage, rank rule + speculation check, factor extraction, projection
template <typename T, typename TIn>
inline int spec_step_rest(const StepCtx& cx, const TIn* C, int64_t rows, int64_t n, int32_t rm, T* core, T* Cn, int mu,
                          SpecStep<T>& s, bool prof_on) {
  const int64_t L = s.L;
  const int batch_mode = (cx.flags & TNB_FLAG_BATCH_MODE) ? 1 : 0;
  cudaStream_t st = cx.st;
  Prof& prof = Prof::get();
  if (!s.chfsi) {
    rank_rule_kernel<<<1, 32, 0, st>>>(s.w, (int)L, (int)L, rm, 0, batch_mode, cx.sc, gram_noise(s.used_tc, s.fp32_solve),
                                       (int)L);
  } else {
    TNB_TRY(cd_end(s.cd));
    rank_rule_kernel<<<1, 32, 0, st>>>(s.w, (int)L, (int)s.kcap, rm, 1, batch_mode, cx.sc, gram_noise(s.used_tc), s.b);
  }
  TNB_LAUNCH_CHECK();
  spec_check_kernel<<<1, 32, 0, st>>>(cx.sc, (int)s.kcap, cx.d_ranks + mu, cx.d_flags);
  TNB_LAUNCH_CHECK();
  if (prof_on) prof.mark(st);
  const int layout = s.in_kblocked ? PT_IN_KBLOCKED : s.out_inner > 0 ? PT_OUT_KBLOCKED : PT_ROWMAJOR;
  TNB_TRY((step_factors<T, TIn>(cx, C, rows, n, s.kcap, s.w, s.V, s.ldv, s.fac, s.ptc_ws, s.ptc_bytes, core, Cn, layout,
                                s.out_inner)));
  if (prof_on) prof.mark(st);
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// Dense TT-SVD
// ---------------------------------------------------------------------------------------------
// The two ping-pong carries, sized by the rank caps: step t writes carry[t & 1] (rows[mu] x rcap[mu]).
template <typename T, class ArenaT>
inline void carve_carries(ArenaT& ar, const SweepDims& d, T* carry[2]) {
  size_t elems[2] = {0, 0};
  for (int mu = d.N - 1, t = 0; mu >= 1; --mu, ++t) {
    const size_t e = (size_t)d.rows[mu] * (size_t)d.rcap[mu];
    if (e > elems[t & 1]) elems[t & 1] = e;
  }
  carry[0] = ar.template take<T>(elems[0]);
  carry[1] = ar.template take<T>(elems[1]);
}

// T: carries and cores; TIn: the dense input (T, or bf16 / fp16 with T = float), read by step 0 only.
template <typename T, typename TIn, class ArenaT>
inline int ttsvd_sync_impl(ArenaT& ar, bool dry, const TIn* data, const SweepDims& d, const int32_t* rmax, double eps,
                           uint32_t flags, T* cores, int32_t* ranks_host, SweepInfo* info, cudaStream_t st,
                           bool exact_gram = false) {
  const int N = d.N;
  StepCtx cx = make_step_ctx(ar, N, eps, flags, !(flags & TNB_FLAG_NO_TENSORCORE) && (dry || tc_path_available()), info,
                             st, false);
  cx.exact_gram = exact_gram;
  Prof& prof = Prof::get();
  prof.on = !dry && (flags & TNB_FLAG_PROFILE);
  prof.used = 0;
  if (!dry) {
    cx.h_sc = static_cast<int*>(pinned_scratch(sizeof(SweepScalars)));
    if (!cx.h_sc) return fail(TNB_ERR_CUDA, "pinned scratch allocation failed");
    ranks_host[0] = 1;
    ranks_host[N] = 1;
  }
  if (N == 1) {
    if (!dry) {
      if (std::is_same<T, TIn>::value) {
        TNB_CUDA(cudaMemcpyAsync(cores + d.slot[0], data, sizeof(T) * d.shape[0], cudaMemcpyDeviceToDevice, st));
      } else {  // the single core is the data, converted
        convert_kernel<T, TIn><<<grid_for(d.shape[0]), 256, 0, st>>>(data, d.shape[0], cores + d.slot[0]);
        TNB_LAUNCH_CHECK();
      }
      TNB_CUDA(cudaStreamSynchronize(st));
      if (info) info->norm = 0;
    }
    return TNB_OK;
  }
  T* carry[2];
  carve_carries(ar, d, carry);
  const T* C = nullptr;  // the carry step t > 0 reads; step 0 reads data
  int64_t r_next = 1;
  size_t peak = ar.off;
  for (int mu = N - 1, t = 0; mu >= 1; --mu, ++t) {
    const int64_t rows = d.rows[mu];
    const int64_t n = dry ? d.shape[mu] * d.rcap[mu + 1] : d.shape[mu] * r_next;
    const bool have_rmax = rmax && rmax[mu - 1] > 0;
    const size_t mark = ar.off;
    int64_t rank = d.rcap[mu];
    T* core = dry ? nullptr : cores + d.slot[mu];
    const int32_t rm = have_rmax ? rmax[mu - 1] : 0;
    if (t == 0)
      TNB_TRY((truncate_step<T, TIn>(ar, dry, cx, data, rows, n, d.rcap[mu], have_rmax, rm, true, core, carry[0], &rank)));
    else
      TNB_TRY((truncate_step<T, T>(ar, dry, cx, C, rows, n, d.rcap[mu], have_rmax, rm, false, core, carry[t & 1], &rank)));
    if (!dry) {
      ranks_host[mu] = (int32_t)rank;
      r_next = rank;
      C = carry[t & 1];
    }
    if (ar.off > peak) peak = ar.off;  // the sizing pass reports the largest step
    ar.off = mark;                     // release the step scratch
  }
  if (dry) ar.off = peak;
  if (!dry) {
    TNB_CUDA(cudaMemcpyAsync(cores + d.slot[0], C, sizeof(T) * (size_t)d.shape[0] * (size_t)r_next,
                             cudaMemcpyDeviceToDevice, st));
    TNB_CUDA(cudaStreamSynchronize(st));
    prof.collect(info);
  }
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// Speculative dense TT-SVD: the whole right-to-left sweep enqueued in one go, ONE synchronisation at the end.
// ---------------------------------------------------------------------------------------------
template <typename T>
inline bool spec_eligible(const SweepDims& d, const int32_t* rmax, double eps, uint32_t flags, bool allow_tc) {
  if ((flags & TNB_FLAG_NO_SPECULATE) || d.N < 2 || !rmax) return false;
  const double epsN = eps / std::max(1.0, std::sqrt((double)(d.N - 1)));
  if (!(epsN * epsN < 1e-20)) return false;  // an active eps budget decides ranks: host-driven path
  for (int mu = d.N - 1; mu >= 1; --mu) {
    if (rmax[mu - 1] <= 0) return false;
    if (!spec_step_ok<T>(d.rows[mu], d.shape[mu] * d.rcap[mu + 1], d.rcap[mu], allow_tc)) return false;
  }
  return true;
}

struct SpecHostBack {  // pinned read-back of one speculative sweep
  SweepScalars sc;
  int flags[4];
  int32_t ranks[64];
};

// One tensor of a speculative sweep (or of a batch of them): its arena, device scalars, carries and position.
template <typename T, typename TIn, class ArenaT>
struct SpecRun {
  ArenaT* ar = nullptr;
  StepCtx cx;
  SweepInfo info_local;
  const TIn* data = nullptr;  // read by step 0
  const T* C = nullptr;       // the carry later steps read
  T* carry[2] = {nullptr, nullptr};
  T* cores = nullptr;
  SpecStep<T> step;
  size_t mark = 0, peak = 0;
  SpecHostBack* hb = nullptr;
};

template <typename T, typename TIn, class ArenaT>
inline int spec_begin(SpecRun<T, TIn, ArenaT>& r, ArenaT& ar, bool dry, const TIn* data, const SweepDims& d, double eps,
                      uint32_t flags, T* cores, SweepInfo* info, cudaStream_t st, SpecHostBack* hb) {
  r.ar = &ar;
  r.cx = make_step_ctx(ar, d.N, eps, flags, !(flags & TNB_FLAG_NO_TENSORCORE) && (dry || tc_path_available()), info, st,
                       true);
  carve_carries(ar, d, r.carry);
  r.data = data;
  r.C = nullptr;
  r.cores = cores;
  r.peak = ar.off;
  r.hb = hb;
  if (!dry) TNB_CUDA(cudaMemsetAsync(r.cx.d_flags, 0, 4 * sizeof(int), st));
  return TNB_OK;
}

// the step scratch of step t+1 reuses that of step t: the kernels of one stream run in order, and every kernel of
// step t+1 that writes scratch is enqueued after every kernel of step t that reads it
template <typename T, typename TIn, class ArenaT>
inline int spec_phase1(SpecRun<T, TIn, ArenaT>& r, bool dry, const SweepDims& d, int mu, int t, bool prof_on) {
  ArenaT& ar = *r.ar;
  r.mark = ar.off;
  const int64_t rows = d.rows[mu], n = d.shape[mu] * d.rcap[mu + 1];
  if (t == 0)
    spec_step_carve<T, TIn>(ar, r.cx, rows, n, d.rcap[mu], r.step);
  else
    spec_step_carve<T, T>(ar, r.cx, rows, n, d.rcap[mu], r.step);
  r.step.in_kblocked = carry_kblocked<T, TIn>(d, mu, r.cx.allow_tc);
  r.step.out_inner = carry_kblocked<T, TIn>(d, mu - 1, r.cx.allow_tc) ? d.shape[mu - 1] : 0;
  if (ar.off > r.peak) r.peak = ar.off;
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "workspace too small (need > %zu bytes)", ar.off);
  if (t == 0) return spec_step_gram<T, TIn>(r.cx, r.data, rows, n, true, r.step, prof_on);
  return spec_step_gram<T, T>(r.cx, r.C, rows, n, false, r.step, prof_on);
}
template <typename T, typename TIn, class ArenaT>
inline int spec_phase2b(SpecRun<T, TIn, ArenaT>& r, bool dry, const SweepDims& d, const int32_t* rmax, int mu, int t,
                        bool prof_on) {
  ArenaT& ar = *r.ar;
  if (!dry) {
    const int64_t rows = d.rows[mu], n = d.shape[mu] * d.rcap[mu + 1];
    if (t == 0)
      TNB_TRY((spec_step_rest<T, TIn>(r.cx, r.data, rows, n, rmax[mu - 1], r.cores + d.slot[mu], r.carry[0], mu, r.step,
                                      prof_on)));
    else
      TNB_TRY((spec_step_rest<T, T>(r.cx, r.C, rows, n, rmax[mu - 1], r.cores + d.slot[mu], r.carry[t & 1], mu, r.step,
                                    prof_on)));
    r.C = r.carry[t & 1];
  }
  ar.off = r.mark;
  return TNB_OK;
}
// Enqueues the whole sweep of g >= 1 runs, each on its own stream, step by step: every run's Gram (phase 1), then every
// run's eigen start (phase 2a), then the subspace-solver stages interleaved run by run, then every run's rank rule and
// projection (phase 2b).  Interleaving the stages makes the resident filter kernels of the streams run one after the
// other (cheb_filter.cuh), so one run's Rayleigh-Ritz step is in flight while another run's filter runs.  With dry it
// only sizes the step scratch.
template <typename T, typename TIn, class ArenaT>
inline int spec_enqueue(SpecRun<T, TIn, ArenaT>* runs, int g, bool dry, const SweepDims& d, const int32_t* rmax,
                        bool prof_on) {
  for (int mu = d.N - 1, t = 0; mu >= 1; --mu, ++t) {
    for (int s = 0; s < g; ++s) TNB_TRY(spec_phase1(runs[s], dry, d, mu, t, prof_on));
    if (!dry) {
      for (int s = 0; s < g; ++s) TNB_TRY(spec_step_eig_begin<T>(runs[s].cx, runs[s].step));
      for (int stage = 0; stage <= CD_MAX_STAGES; ++stage)
        for (int s = 0; s < g; ++s) TNB_TRY(spec_step_eig_stage<T>(runs[s].step, stage));
    }
    for (int s = 0; s < g; ++s) TNB_TRY(spec_phase2b(runs[s], dry, d, rmax, mu, t, prof_on));
  }
  return TNB_OK;
}
template <typename T, typename TIn, class ArenaT>
inline int spec_end(SpecRun<T, TIn, ArenaT>& r, const SweepDims& d) {
  cudaStream_t st = r.cx.st;
  const int N = d.N;
  TNB_CUDA(cudaMemcpyAsync(r.cores + d.slot[0], r.C, sizeof(T) * (size_t)d.shape[0] * (size_t)d.rcap[1],
                           cudaMemcpyDeviceToDevice, st));
  TNB_CUDA(cudaMemcpyAsync(&r.hb->sc, r.cx.sc, sizeof(SweepScalars), cudaMemcpyDeviceToHost, st));
  TNB_CUDA(cudaMemcpyAsync(r.hb->flags, r.cx.d_flags, 4 * sizeof(int), cudaMemcpyDeviceToHost, st));
  TNB_CUDA(cudaMemcpyAsync(r.hb->ranks, r.cx.d_ranks, (size_t)(N + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  return TNB_OK;
}
// after the stream has been synchronised; returns the speculation flags (spec_check_kernel bits, 0: accepted)
inline int spec_collect(const SpecHostBack* hb, const SweepDims& d, int32_t* ranks_host, SweepInfo* info) {
  const int N = d.N;
  ranks_host[0] = 1;
  ranks_host[N] = 1;
  for (int mu = 1; mu < N; ++mu) ranks_host[mu] = (int32_t)d.rcap[mu];  // the flags say whether the rule agreed
  if (info) {
    info->norm = std::sqrt(hb->sc.norm2 > 0 ? hb->sc.norm2 : 0.0);
    info->chfsi_products += hb->flags[1];
    info->rr_solves += hb->flags[2];
    info->rr_sweeps += hb->flags[3];
    info->fused_filters += hb->flags[2] - info->eig_solves;  // every Rayleigh-Ritz step but the first of a solve follows a filter
  }
  return hb->flags[0];
}

// *spec_flags: what spec_collect returned (set when the sweep ran to its end)
template <typename T, typename TIn, class ArenaT>
inline int ttsvd_spec_impl(ArenaT& ar, bool dry, const TIn* data, const SweepDims& d, const int32_t* rmax, double eps,
                           uint32_t flags, T* cores, int32_t* ranks_host, SweepInfo* info, cudaStream_t st,
                           int* spec_flags) {
  Prof& prof = Prof::get();
  prof.on = !dry && (flags & TNB_FLAG_PROFILE);
  prof.used = 0;
  const bool prof_on = prof.on;
  SpecHostBack* hb = nullptr;
  if (!dry) {
    hb = static_cast<SpecHostBack*>(pinned_scratch(sizeof(SpecHostBack)));
    if (!hb) return fail(TNB_ERR_CUDA, "pinned scratch allocation failed");
  }
  SpecRun<T, TIn, ArenaT> r;
  TNB_TRY(spec_begin(r, ar, dry, data, d, eps, flags, cores, info, st, hb));
  const int rc = spec_enqueue(&r, 1, dry, d, rmax, prof_on);
  if (rc != TNB_OK) {
    if (!dry) cudaStreamSynchronize(st);  // part of the sweep is enqueued: drain it before the host-driven path
    prof.on = false;
    return rc;
  }
  if (dry) {
    ar.off = r.peak;
    return TNB_OK;
  }
  TNB_TRY(spec_end(r, d));
  TNB_CUDA(cudaStreamSynchronize(st));
  *spec_flags = spec_collect(hb, d, ranks_host, info);
  prof.collect(info);
  return TNB_OK;
}

// Dispatcher: speculative sweep when a rank cap decides every bond, host-driven sweep otherwise and as the fallback.
template <typename T, typename TIn, class ArenaT>
inline int ttsvd_impl(ArenaT& ar, bool dry, const TIn* data, const SweepDims& d, const int32_t* rmax, double eps,
                      uint32_t flags, T* cores, int32_t* ranks_host, SweepInfo* info, cudaStream_t st) {
  const bool allow_tc = !(flags & TNB_FLAG_NO_TENSORCORE) && (dry || tc_path_available());
  // the sizing pass cannot ask the device what it supports: size for both paths
  const bool spec = dry ? (d.N >= 2 && rmax != nullptr) : spec_eligible<T>(d, rmax, eps, flags, allow_tc);
  const size_t base = ar.off;
  size_t need_spec = 0;
  if (spec) {
    if (dry) {
      bool all_caps = true;
      for (int mu = 1; mu < d.N; ++mu) all_caps = all_caps && rmax[mu - 1] > 0;
      if (all_caps) {
        const int rc = ttsvd_spec_impl<T, TIn>(ar, true, data, d, rmax, eps, flags, cores, ranks_host, info, st, nullptr);
        if (rc == TNB_OK) need_spec = ar.off - base;
        ar.off = base;
      }
    } else {
      int sflags = 0;
      SweepInfo saved;
      if (info) saved = *info;
      const int rc = ttsvd_spec_impl<T, TIn>(ar, false, data, d, rmax, eps, flags, cores, ranks_host, info, st, &sflags);
      if (rc == TNB_OK && sflags == 0) {
        if (info) info->speculative = 1;
        return TNB_OK;
      }
      if (rc != TNB_OK && rc != TNB_ERR_UNSUPPORTED && rc != TNB_ERR_NOCONV) return rc;
      // the device disagreed with the speculation (or could not run the sync-free solver): host-driven sweep;
      // bit 0 = the TF32 Gram is too coarse for this spectrum, so the repeat takes exact-product Gram matrices
      if (info) { *info = saved; info->spec_flags = sflags; }
      ar.off = base;
      ar.ok = true;
      return ttsvd_sync_impl<T, TIn>(ar, false, data, d, rmax, eps, flags, cores, ranks_host, info, st, (sflags & 1) != 0);
    }
  }
  const int rc = ttsvd_sync_impl<T, TIn>(ar, dry, data, d, rmax, eps, flags, cores, ranks_host, info, st);
  if (dry && rc == TNB_OK && need_spec > ar.off - base) ar.off = base + need_spec;
  return rc;
}

// ---------------------------------------------------------------------------------------------
// A batch of independent dense tensors of one shape (the reference's `batch=True` constructor, tensor.py:401-408 with
// a leading batch dimension; north_star: "batched decompositions").  Up to `inflight` speculative sweeps are enqueued
// from ONE host thread, interleaved stage by stage on internal streams (spec_enqueue), and synchronised once; tensors
// whose speculation the device rejected are then repeated one by one on the host-driven path.
// ---------------------------------------------------------------------------------------------
constexpr int TNB_BATCH_MAX_INFLIGHT = 8;

struct StreamPool {
  cudaStream_t st[TNB_BATCH_MAX_INFLIGHT] = {};
  cudaEvent_t ev[TNB_BATCH_MAX_INFLIGHT + 1] = {};
  bool ready = false;
  std::mutex mu;
  int ensure() {
    if (ready) return TNB_OK;
    for (int i = 0; i < TNB_BATCH_MAX_INFLIGHT; ++i) TNB_CUDA(cudaStreamCreateWithFlags(&st[i], cudaStreamNonBlocking));
    for (int i = 0; i <= TNB_BATCH_MAX_INFLIGHT; ++i) TNB_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    ready = true;
    return TNB_OK;
  }
  // the first n internal streams start after whatever the caller enqueued on `caller`
  int fork(cudaStream_t caller, int n) {
    TNB_CUDA(cudaEventRecord(ev[TNB_BATCH_MAX_INFLIGHT], caller));
    for (int i = 0; i < n; ++i) TNB_CUDA(cudaStreamWaitEvent(st[i], ev[TNB_BATCH_MAX_INFLIGHT], 0));
    return TNB_OK;
  }
  // `caller` continues after the first n internal streams; unchecked, as it also runs after a failed enqueue
  void join(cudaStream_t caller, int n) {
    for (int i = 0; i < n; ++i) {
      cudaEventRecord(ev[i], st[i]);
      cudaStreamWaitEvent(caller, ev[i], 0);
    }
  }
  static StreamPool& get() {
    static StreamPool pools[TNB_MAX_DEVICES];
    return pools[current_device_index()];
  }
};

template <typename T, typename TIn>
inline int ttsvd_batch_impl(void* workspace, size_t per_tensor_bytes, int inflight, const TIn* const* data, int batch,
                            const SweepDims& d, const int32_t* rmax, double eps, uint32_t flags, T* const* cores,
                            int32_t* ranks_host, double* norms_host, int32_t* spec_host, cudaStream_t st) {
  const int N = d.N;
  const bool allow_tc = !(flags & TNB_FLAG_NO_TENSORCORE) && tc_path_available();
  const bool spec = batch > 0 && spec_eligible<T>(d, rmax, eps, flags, allow_tc);
  char* ws = static_cast<char*>(workspace);
  if (!spec || inflight < 2 || batch < 2) {  // one at a time through the dispatcher (speculative when eligible)
    for (int i = 0; i < batch; ++i) {
      Arena ar(ws, per_tensor_bytes);
      SweepInfo info;
      TNB_TRY((ttsvd_impl<T, TIn, Arena>(ar, false, data[i], d, rmax, eps, flags, cores[i], ranks_host + (size_t)i * (N + 1), &info,
                                         st)));
      if (norms_host) norms_host[i] = info.norm;
      if (spec_host) spec_host[i] = info.speculative;
    }
    return TNB_OK;
  }
  if (inflight > TNB_BATCH_MAX_INFLIGHT) inflight = TNB_BATCH_MAX_INFLIGHT;
  if (inflight > batch) inflight = batch;
  StreamPool& pool = StreamPool::get();
  std::lock_guard<std::mutex> lk(pool.mu);  // one batch at a time per device uses the internal streams
  TNB_TRY(pool.ensure());
  SpecHostBack* hbs = static_cast<SpecHostBack*>(pinned_scratch((size_t)batch * sizeof(SpecHostBack)));
  if (!hbs) return fail(TNB_ERR_CUDA, "pinned scratch allocation failed");
  TNB_TRY(pool.fork(st, inflight));
  const uint32_t bflags = (flags | TNB_FLAG_CONCURRENT) & ~TNB_FLAG_PROFILE;
  std::vector<SweepInfo> infos(batch);
  int rc = TNB_OK;
  for (int g0 = 0; g0 < batch && rc == TNB_OK; g0 += inflight) {
    const int g = std::min(inflight, batch - g0);
    std::vector<Arena> arenas;
    arenas.reserve(g);
    std::vector<SpecRun<T, TIn, Arena>> runs(g);
    for (int s = 0; s < g; ++s) arenas.emplace_back(ws + (size_t)s * per_tensor_bytes, per_tensor_bytes);
    for (int s = 0; s < g && rc == TNB_OK; ++s)
      rc = spec_begin(runs[s], arenas[s], false, data[g0 + s], d, eps, bflags, cores[g0 + s], &infos[g0 + s], pool.st[s],
                      hbs + g0 + s);
    if (rc == TNB_OK) rc = spec_enqueue(runs.data(), g, false, d, rmax, false);
    for (int s = 0; s < g && rc == TNB_OK; ++s) rc = spec_end(runs[s], d);
  }
  pool.join(st, inflight);  // then the one host synchronisation
  TNB_CUDA(cudaStreamSynchronize(st));
  if (rc != TNB_OK && rc != TNB_ERR_UNSUPPORTED && rc != TNB_ERR_NOCONV) return rc;
  // read every outcome out of the pinned block first: the host-driven repeats below reuse that scratch
  std::vector<int> sflags(batch, 0);
  for (int i = 0; i < batch; ++i)
    if (rc == TNB_OK) sflags[i] = spec_collect(hbs + i, d, ranks_host + (size_t)i * (N + 1), &infos[i]);
  for (int i = 0; i < batch; ++i) {
    int32_t* rk = ranks_host + (size_t)i * (N + 1);
    if (rc == TNB_OK && sflags[i] == 0) {
      if (norms_host) norms_host[i] = infos[i].norm;
      if (spec_host) spec_host[i] = 1;
      continue;
    }
    // repeat this tensor on the host-driven path (exact Gram when the TF32 one was rejected)
    Arena ar(ws, per_tensor_bytes);
    SweepInfo info;
    TNB_TRY((ttsvd_sync_impl<T, TIn, Arena>(ar, false, data[i], d, rmax, eps, flags & ~TNB_FLAG_PROFILE, cores[i], rk, &info, st,
                                       (sflags[i] & 1) != 0)));
    if (norms_host) norms_host[i] = info.norm;
    if (spec_host) spec_host[i] = 0;
  }
  return TNB_OK;
}

}  // namespace tnb
