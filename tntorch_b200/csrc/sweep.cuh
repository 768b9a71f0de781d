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

// The input of the dense TT-SVD may be bf16, fp16 or fp8 (TIn); only step 0 reads it, every carry and core is T (fp32
// for 16-bit and fp8 input).
template <typename TIn>
constexpr bool tc_input() {
  return std::is_same<TIn, float>::value || std::is_same<TIn, __nv_bfloat16>::value || std::is_same<TIn, __half>::value ||
         is_fp8<TIn>();
}
// The TMA tensor-core kernels need 16-byte aligned operands; the dense input is the caller's pointer and may not be.
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

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
// row-major (fp32, or the bf16 / fp16 / fp8 input when the writer is step 0), and the last carry (step mu = 0's core) stays
// row-major, and 16-byte aligned when it is the caller's input (`data`; nullptr when only sizing).
template <typename T, typename TIn = T>
inline bool carry_kblocked(const SweepDims& d, int mu, bool allow_tc, const void* data = nullptr) {
  if (!std::is_same<T, float>::value || !allow_tc || mu < 1 || mu + 1 > d.N - 1) return false;
  const int64_t rows = d.rows[mu], n = d.shape[mu] * d.rcap[mu + 1], k = std::min<int64_t>(d.rcap[mu], n);
  const bool reader = rows >= n && rows >= std::max(TC_MIN_ROWS, PROJ_TC_MIN_ROWS) && gram_tc_kblocked_shape_ok(rows, n) &&
                      k <= PT_MAX_N && project_tc_shape_ok(rows, n, k, nullptr, nullptr);
  const int64_t wrows = d.rows[mu + 1], wn = d.shape[mu + 1] * d.rcap[mu + 2], r = d.rcap[mu + 1];
  const bool wtc = mu + 1 == d.N - 1 ? project_use_tc<TIn>(wrows, wn, r, nullptr, nullptr)
                                     : project_use_tc<T>(wrows, wn, r, nullptr, nullptr);
  const bool writer = wrows >= wn && wn >= 32 && wtc && r % 16 == 0 && r <= 48 && d.shape[mu] % 16 == 0 &&
                      (mu + 1 != d.N - 1 || data == nullptr || aligned16(data));
  return reader && writer && !carry_kblocked<T, TIn>(d, mu + 1, allow_tc, data);
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

// Has a (rows x n) matrix of T a tensor-core Gram: tall, and enough rows for it to pay.
template <typename T>
inline bool gram_tc_tall_ok(int64_t rows, int64_t n) {
  return rows >= n && rows >= TC_MIN_ROWS && gram_tc_input_ok<T>(rows, n);
}

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
  if (allow_tc && gram_tc_tall_ok<T>(rows, n)) {
    w.tc_bytes = gram_tc_input_workspace_bytes<T>(rows, n);
    w.tc_ws = ar.template take<char>(w.tc_bytes);
  }
}

// *used_tc: 0 exact-product Gram, 1 TF32 tensor-core Gram, 2 bf16 tensor-core Gram, 3 fp16 tensor-core Gram, 4 / 5 e4m3 /
// e5m2 tensor-core Gram (gram_noise)
template <typename T>
inline int gram_small_side(const T* C, int64_t rows, int64_t n, double* G, float* Gf, GramWork& w, bool use_tc,
                           int* used_tc, cudaStream_t st) {
  const bool tall = rows >= n;
  if (used_tc) *used_tc = 0;
  if (tall) {
    if constexpr (tc_input<T>())
      if (use_tc && w.tc_ws && aligned16(C)) {  // a misaligned input takes the generic Gram, whose partials are always carved
        if (used_tc)
          *used_tc = std::is_same<T, __nv_bfloat16>::value   ? 2
                     : std::is_same<T, __half>::value        ? 3
                     : std::is_same<T, __nv_fp8_e4m3>::value ? 4
                     : std::is_same<T, __nv_fp8_e5m2>::value ? 5
                                                             : 1;
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
  const double g = used_tc >= 4   ? FP8_GRAM_NOISE
                   : used_tc == 3 ? FP16_GRAM_NOISE
                   : used_tc == 2 ? BF16_GRAM_NOISE
                   : used_tc      ? TF32_GRAM_NOISE
                                  : 0.0;
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
                   double tol = 1e-6, bool fp32_solve = false) {
  if (!e.chfsi) return jacobi2_eigh(G, (int)L, (int)L, e.w, e.V, e.jscratch, e.jinfo, st, fp32_solve, fp32_solve ? 2e-7 : 0.0);
  e.cw.use_tc = allow_tc;
  e.cw.shared_gpu = shared_gpu;
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
// fp32_solve: a small Gram's eigenpairs from fp32 rotations, as the speculative sweep takes them (spec_step_eig_begin).
template <typename TBk>
inline int eig_solve_and_rank(const double* G, const TBk* Gb, int64_t L, EigWork<TBk>& ew, SweepScalars* sc, int* h_sc,
                              int32_t rm, int batch_mode, ChfsiStats* total, int* solves, cudaStream_t st, bool allow_tc,
                              bool shared_gpu, int used_tc = 0, bool fp32_solve = false) {
  fp32_solve = fp32_solve && !ew.chfsi;
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
    // the eps-only solve must resolve the tail energy to 0.05 delta^2; TF32 filter products do not (on a 512 x 512 fp32
    // Gram with eps = 1e-2 they left ~3e-6 of the energy uncaptured and moved the relative error by 3 %): CUDA cores
    TNB_TRY(eig_run<TBk>(G, Gb, L, ew, &sc->trace, &cs, st, allow_tc && !adaptive, shared_gpu, k_try, tol, fp32_solve));
    if (total)
      total->products += cs.products, total->fused_filters += cs.fused_filters, total->outer += cs.outer,
          total->rr_sweeps += cs.rr_sweeps;
    if (solves) *solves += 1;
    rank_rule_kernel<<<1, 32, 0, st>>>(ew.w, (int)L, ew.chfsi ? ew.k_run : (int)L, rm, ew.chfsi ? 1 : 0, batch_mode, sc,
                                       gram_noise(used_tc, fp32_solve), ew.chfsi ? ew.b_run : (int)L);
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
  int stream_passes = 0, stream_chunks = 0;  // tnb_ttsvd_stream: passes over the host tensor, chunks per pass
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

  // May a host-driven step take a tensor-core Gram?  The TF32 Gram equals (1 - c) * G, c ~ 7e-4 (operand truncation
  // shrinks every product alike: harmless, the rank rule works on ratios) plus noise of ~1.6e-6 * ||G|| (measured,
  // tests/test_model.py) — a floor under the tail energies the rank rule can resolve.  An eps budget between "inactive"
  // and 1e-4 of the trace needs finer resolution than that: those sweeps take the exact-product fp64-accumulating Gram
  // instead.  The sizing pass sizes for the tensor-core Gram whatever the budget.
  bool tc_gram(bool dry) const { return allow_tc && !exact_gram && (dry || eps_scaled2 < 1e-20 || eps_scaled2 >= 1e-4); }
};

// The tensor-core kernels may run: the caller did not turn them off and the device has them (the sizing pass, which
// cannot ask the device, sizes for them).
inline bool tc_allowed(uint32_t flags, bool dry) {
  return !(flags & TNB_FLAG_NO_TENSORCORE) && (dry || tc_path_available());
}

// The context of a sweep over N modes.  Carves the device scalars and, for a speculative sweep, then its flags and ranks.
template <class ArenaT>
inline StepCtx make_step_ctx(ArenaT& ar, bool dry, int N, double eps, uint32_t flags, SweepInfo* info, cudaStream_t st,
                             bool speculative) {
  StepCtx cx;
  cx.flags = flags;
  cx.allow_tc = tc_allowed(flags, dry);
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

// A wide step's factor (step_factors) in fp64 scratch: F = U_r diag(1/d) (rows x kcap), the split-K partials of the
// kcap x kcap Gram of the core's rows (~4 sms kcap^2 / tiles doubles, at most n kcap^2 / 64), that Gram, the Cholesky-QR factors T and R,
// the factorisation's scratch, and a control block (tnb_skip words: word 1 set = the rows are already orthonormal).
// O(rows * kcap + kcap^2): nothing of the core's length n.
struct WideWork {
  double *F = nullptr, *partial = nullptr, *S = nullptr, *Tm = nullptr, *Rm = nullptr, *scratch = nullptr;
  int* ctrl = nullptr;
  int splits = 1;
};
template <class ArenaT>
inline void wide_carve(ArenaT& ar, int64_t rows, int64_t n, int64_t kcap, WideWork& ww) {
  // the Gram has a few output tiles and a long K: split it over ~4 CTAs per SM (plan_gemm stops at 64 splits, which left
  // a 64 x 64 Gram over 2^21 columns on half the SMs), at most n / 64 of them
  const int64_t tm = ceil_div<int64_t>(kcap, GEMM_BM), tiles = tm * (tm + 1) / 2;
  const int sms = device_info().valid ? device_info().sm_count : 132;
  const int64_t want = std::min<int64_t>(std::max<int64_t>(ceil_div<int64_t>(4 * (int64_t)sms, tiles), 1),
                                         std::max<int64_t>(n / 64, 1));
  const GemmPlan pl = plan_gemm(kcap, kcap, n, true, (int)std::min<int64_t>(want, 1024));
  ww.splits = pl.splits;
  ww.F = ar.template take<double>((size_t)rows * kcap);
  ww.partial = ar.template take<double>(pl.partial_elems);
  ww.S = ar.template take<double>((size_t)kcap * kcap);
  ww.Tm = ar.template take<double>((size_t)kcap * kcap);
  ww.Rm = ar.template take<double>((size_t)kcap * kcap);
  ww.scratch = ar.template take<double>((size_t)2 * kcap * (kcap | 1));
  ww.ctrl = ar.template take<int>(4);
}

// F[a][j] = U[a][j] / d_j and Cn[a][j] = U[a][j] d_j, d_j = max(s_j, 1e-8 s_0): F^T C has rows near unit length (at the
// Gram's noise floor, where s_j carries no information, shorter) and Cn (F^T C) = U_r U_r^T C exactly.
template <typename T>
__global__ void wide_prep_kernel(const double* __restrict__ V, int ldv, int64_t rows, int rank, const double* __restrict__ w,
                                 double* __restrict__ F, T* __restrict__ Cn) {
  const double s0 = sqrt(w[0] > 0.0 ? w[0] : 0.0);
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < rows * rank; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t a = idx / rank;
    const int j = (int)(idx % rank);
    const double d = fmax(sqrt(w[j] > 0.0 ? w[j] : 0.0), 1e-8 * s0);
    const double u = V[(size_t)a * ldv + j];
    F[idx] = d > 0.0 ? u / d : 0.0;
    Cn[idx] = (T)(u * d);
  }
}

// Are the core's rows orthonormal already (S = core core^T within tol of I)?  Then every later stage of the step is
// skipped (ctrl word 1, read by tnb_skip); otherwise they run.  One warp.
__global__ void wide_check_kernel(const double* __restrict__ S, int rank, double tol, int* ctrl) {
  double dev = 0.0;
  for (int idx = threadIdx.x; idx < rank * rank; idx += blockDim.x) {
    const int i = idx / rank, j = idx % rank;
    dev = fmax(dev, fabs(S[idx] - (i == j ? 1.0 : 0.0)));
  }
  for (int o = 16; o > 0; o >>= 1) dev = fmax(dev, __shfl_xor_sync(0xffffffffu, dev, o));
  if (threadIdx.x == 0) {
    ctrl[0] = 0;
    ctrl[1] = dev <= tol ? 1 : 0;
    ctrl[2] = 0;
  }
}

template <typename TB>
__global__ void __launch_bounds__(1024) wide_chol_kernel(const double* __restrict__ S, int b, double* scratch, TB* __restrict__ T,
                                                         int use_smem, TB* __restrict__ Rout, int* ctrl) {
  extern __shared__ __align__(16) unsigned char wide_chol_smem[];
  if (tnb_skip(ctrl, 0)) return;
  chol_orth_device<TB>(S, b, scratch, T, ctrl + 3, use_smem, Rout, wide_chol_smem);
}

// One Cholesky-QR step in place, from the factors of chol_orth_kernel for A = core^T (A T has orthonormal columns,
// A = (A T) R; T and R upper triangular with positive diagonals): core <- T^T core and Cn <- Cn R^T.  Each block takes
// 32 vectors (columns of core, or rows of Cn) into shared memory, then writes the products over them.  With `fill`, a
// core row that was exactly zero (S_jj <= 1e-30 max S: U_r's direction meets a null row space of C, or the tensor is
// zero) has no direction to keep: it becomes a fixed pseudo-random row and its Cn column zero, which leaves Cn core as it
// was; the next step orthonormalises it against the others.
// CORE picks the role (the orthonormalised factor, updated by T, or the other one, updated by R); KMAJOR the layout:
// X[k][g] (rank x nvec, a core's rows) or X[g][k] (nvec x rank, Cn's rows).  truncated_svd's tall form has them swapped.
template <typename T, bool CORE, bool KMAJOR = CORE>
__global__ void __launch_bounds__(256) wide_apply_kernel(const double* __restrict__ M, const double* __restrict__ S, int rank,
                                                         int64_t nvec, T* __restrict__ X, int fill, const int* ctrl) {
  extern __shared__ __align__(16) unsigned char wide_apply_smem[];
  if (tnb_skip(ctrl, 0)) return;
  double* x = reinterpret_cast<double*>(wide_apply_smem);  // [rank][32]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  double smax = 0.0;
  if (fill)
    for (int k = 0; k < rank; ++k) smax = fmax(smax, S[(size_t)k * rank + k]);
  for (int64_t v0 = (int64_t)blockIdx.x * 32; v0 < nvec; v0 += (int64_t)gridDim.x * 32) {
    __syncthreads();
    for (int idx = threadIdx.x; idx < rank * 32; idx += blockDim.x) {
      const int k = idx / 32, v = idx % 32;
      const int64_t g = v0 + v;
      x[idx] = g < nvec ? (double)(KMAJOR ? X[(size_t)k * nvec + g] : X[(size_t)g * rank + k]) : 0.0;
    }
    __syncthreads();
    const int64_t g = v0 + lane;
    if (g < nvec)
      for (int j = warp; j < rank; j += 8) {
        double acc = 0.0;
        if (CORE)
          for (int k = 0; k <= j; ++k) acc = fma(M[(size_t)k * rank + j], x[k * 32 + lane], acc);
        else
          for (int k = j; k < rank; ++k) acc = fma(M[(size_t)j * rank + k], x[k * 32 + lane], acc);
        if (fill && (S[(size_t)j * rank + j] <= 1e-30 * smax || !(smax > 0.0))) {
          if (CORE) {
            const uint64_t e = (uint64_t)j * nvec + g;
            const uint32_t h = hash_u32((uint32_t)e * 2654435761U + 0x5bd1e995U) ^ hash_u32((uint32_t)(e >> 32) + 0x9e3779b9U);
            acc = ((double)(h >> 8) + 0.5) * (2.0 / 16777216.0) - 1.0;
          } else {
            acc = 0.0;
          }
        }
        if (KMAJOR) X[(size_t)j * nvec + g] = (T)acc;
        else X[(size_t)g * rank + j] = (T)acc;
      }
  }
}

// Rows of a wide step's core that are orthonormal to this level skip the Cholesky-QR steps (fp64 accumulation of
// diag(1/d) U_r^T C leaves them within ~eps_64 lambda_0 / lambda_{r-1} of it, plus the storage rounding).
template <typename T>
constexpr double wide_orth_tol() { return std::is_same<T, double>::value ? 1e-13 : 1e-6; }

// The gauge repair of a split Q P (Q: `rank` vectors of length nq that should be orthonormal; P: the other factor, np
// vectors of length rank): the fp64 Gram of Q's vectors (split-K GEMM, ww.splits); when it is within wide_orth_tol of I
// the rest is skipped on the device; otherwise two Cholesky-QR steps (one-CTA Cholesky of the rank x rank Gram, in-place
// triangular updates of Q and P on the whole GPU, a second Gram).  Q_KMAJOR: Q is rank x nq row-major and P np x rank
// (a wide step's core and Cn), else Q is nq x rank and P rank x np (truncated_svd's tall form, left and right).
// Positive diagonals keep the basis; the product Q^T P^T (or Q P) is unchanged but for rounding.
template <typename T, bool Q_KMAJOR>
inline int chol_qr_repair(const WideWork& ww, int64_t rank, T* Q, int64_t nq, T* P, int64_t np, cudaStream_t st) {
  const GemmPlan pl = plan_gemm(rank, rank, nq, true, ww.splits);
  const size_t csm = (size_t)2 * rank * (rank | 1) * sizeof(double), asm_bytes = (size_t)rank * 32 * sizeof(double);
  const bool fits = csm <= 180 * 1024;
  static PerDeviceFlag attr_chol, attr_q, attr_p;
  TNB_CUDA(ensure_dyn_smem(attr_chol, wide_chol_kernel<double>, 180 * 1024));
  TNB_CUDA(ensure_dyn_smem(attr_q, wide_apply_kernel<T, true, Q_KMAJOR>, 64 * 1024));
  TNB_CUDA(ensure_dyn_smem(attr_p, wide_apply_kernel<T, false, !Q_KMAJOR>, 64 * 1024));
  const int grid_q = (int)std::min<int64_t>(ceil_div<int64_t>(nq, 32), 8 * usable_sms());
  const int grid_p = (int)std::min<int64_t>(ceil_div<int64_t>(np, 32), 8 * usable_sms());
  const int ldq = Q_KMAJOR ? (int)nq : (int)rank;
  // two Cholesky-QR steps, all of them skipped on the device when the first Gram finds the vectors orthonormal
  for (int pass = 0; pass < 2; ++pass) {
    TNB_TRY((gemm_splitk<T, T, double, double, float>(pl, rank, rank, nq, Q, ldq, Q_KMAJOR, Q, ldq, Q_KMAJOR, ww.partial, ww.S,
                                                      rank, 1.0, nullptr, 0, 0.0, nullptr, 0, 0.0, true, (float*)nullptr, 0, st,
                                                      pass ? ww.ctrl : nullptr, 0)));
    if (pass == 0) {
      wide_check_kernel<<<1, 32, 0, st>>>(ww.S, (int)rank, wide_orth_tol<T>(), ww.ctrl);
      TNB_LAUNCH_CHECK();
    }
    wide_chol_kernel<double><<<1, 1024, fits ? csm : 0, st>>>(ww.S, (int)rank, ww.scratch, ww.Tm, fits ? 1 : 0, ww.Rm, ww.ctrl);
    TNB_LAUNCH_CHECK();
    wide_apply_kernel<T, true, Q_KMAJOR><<<grid_q, 256, asm_bytes, st>>>(ww.Tm, ww.S, (int)rank, nq, Q, pass == 0, ww.ctrl);
    TNB_LAUNCH_CHECK();
    wide_apply_kernel<T, false, !Q_KMAJOR><<<grid_p, 256, asm_bytes, st>>>(ww.Rm, ww.S, (int)rank, np, P, pass == 0, ww.ctrl);
    TNB_LAUNCH_CHECK();
  }
  return TNB_OK;
}

// A tall step's factors from its eigenpairs (w descending, V with leading dimension ldv): core = V_r^T (rank x n) and
// fac = V_r (n x rank), the operand of the projection Cn = C V_r.
template <typename T>
inline int tall_factors(const double* w, const double* V, int ldv, int64_t n, int64_t rank, T* core, T* fac,
                        cudaStream_t st) {
  scale_extract_kernel<T><<<grid_for(n * rank), 256, 0, st>>>(V, ldv, (int)n, (int)rank, w, core, 0, 1);
  TNB_LAUNCH_CHECK();
  scale_extract_kernel<T><<<grid_for(n * rank), 256, 0, st>>>(V, ldv, (int)n, (int)rank, w, fac, 0, 0);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// The factors of a zero unfolding at the rank host_step_solve gives it (round.py:137-145).
template <typename T>
inline int zero_factors(int64_t rows, int64_t n, int64_t rank, T* core, T* Cn, cudaStream_t st) {
  fill_kernel<T><<<grid_for(n * rank), 256, 0, st>>>(core, n * rank, (T)0);
  TNB_LAUNCH_CHECK();
  fill_kernel<T><<<grid_for(rows * rank), 256, 0, st>>>(Cn, rows * rank, (T)0);
  TNB_LAUNCH_CHECK();
  return TNB_OK;
}

// The end of a truncation step at rank `rank`, from the step's eigenpairs (w descending, V with leading dimension ldv):
//   tall (rows >= n): core = V_r^T (rank x n);  Cn = C V_r;
//   wide:             core = diag(1/d) U_r^T C (accumulated in fp64), Cn = U_r diag(d), d_j = max(s_j, 1e-8 s_0), then
//                     the fp64 Gram of core's rows (split-K GEMM).  When it is within wide_orth_tol of I (a spectrum
//                     well above the Gram's noise floor) the step ends there, decided on the device; otherwise two
//                     Cholesky-QR steps follow (one-CTA Cholesky of the rank x rank Gram, in-place triangular updates of
//                     core and Cn on the whole GPU, a second Gram), which make the rows orthonormal when s_r nears the
//                     noise floor or the unfolding's rank is below the cap, where diag(1/s) U_r^T C alone is not.
//                     Positive diagonals keep the basis; Cn core = U_r U_r^T C throughout.
// fac (n x rank, tall steps) and ww (wide steps) are scratch; ptc_ws the tensor-core projection's workspace
// (project_tc_carve_bytes).  `layout` is PT_ROWMAJOR unless the speculative sweep reads (PT_IN_KBLOCKED) or writes
// (PT_OUT_KBLOCKED, out_inner) a K-blocked carry.
template <typename T, typename TIn>
inline int step_factors(const StepCtx& cx, const TIn* C, int64_t rows, int64_t n, int64_t rank, const double* w,
                        const double* V, int ldv, T* fac, const WideWork& ww, void* ptc_ws, size_t ptc_bytes, T* core,
                        T* Cn, int layout = PT_ROWMAJOR, int64_t out_inner = 0) {
  cudaStream_t st = cx.st;
  if (rows >= n) {
    TNB_TRY(tall_factors<T>(w, V, ldv, n, rank, core, fac, st));
    BigKernelGate gate(st, (cx.flags & TNB_FLAG_CONCURRENT) && rows >= PROJ_TC_MIN_ROWS);
    if constexpr (tc_input<TIn>())
      if (layout != PT_ROWMAJOR)
        return project_tc<TIn>(C, rows, n, reinterpret_cast<const float*>(fac), (int)rank, reinterpret_cast<float*>(Cn),
                               ptc_ws, ptc_bytes, st, layout, out_inner);
    return project_any<T, TIn>(C, rows, n, fac, rank, Cn, st, ptc_ws, ptc_bytes);
  }
  wide_prep_kernel<T><<<grid_for(rows * rank), 256, 0, st>>>(V, ldv, rows, (int)rank, w, ww.F, Cn);
  TNB_LAUNCH_CHECK();
  TNB_TRY((gemm_direct<double, TIn, double, T>(rank, n, rows, ww.F, rank, false, C, n, false, core, n, 1.0, nullptr, 0, 0.0,
                                               nullptr, 0, 0.0, st)));
  return chol_qr_repair<T, true>(ww, rank, core, n, Cn, rows, st);
}

// A host-driven truncation step of a (rows x n) matrix C of TIn, apart from its Gram scratch (GramWork): the fp64 Gram
// G (L x L), the eigen stage (its block precision follows the data), and the factors' scratch: fac = V_r (tall steps)
// or ww (wide steps), and ptc_ws the tensor-core projection's workspace (project_tc_carve_bytes).
template <typename T>
struct HostStep {
  int64_t L = 0, kcap = 0;
  double* G = nullptr;
  EigWork<T> ew;
  T* fac = nullptr;
  WideWork ww;
  void* ptc_ws = nullptr;
  size_t ptc_bytes = 0;
  float* Gf() const { return reinterpret_cast<float*>(ew.Gb); }  // G in fp32 for an fp32 subspace solve, else nullptr
};
template <typename T, typename TIn, class ArenaT>
inline int host_step_carve(ArenaT& ar, const StepCtx& cx, int64_t rows, int64_t n, int64_t rank_cap, bool have_rmax,
                           HostStep<T>& s) {
  s.L = std::min(rows, n);
  s.kcap = std::min<int64_t>(rank_cap, s.L);
  s.G = ar.template take<double>((size_t)s.L * s.L);
  TNB_TRY(eig_carve<T>(ar, s.L, s.kcap, have_rmax, s.ew));
  if (rows >= n) s.fac = ar.template take<T>((size_t)s.L * (size_t)s.kcap);
  else wide_carve(ar, rows, n, s.kcap, s.ww);
  s.ptc_bytes = project_tc_carve_bytes<TIn>(cx.allow_tc, rows, n, s.kcap);
  s.ptc_ws = s.ptc_bytes ? ar.template take<char>(s.ptc_bytes) : nullptr;
  return TNB_OK;
}

// The Gram, eigen stage and rank rule of a host-driven step.  gram(use_tc, &used_tc) makes s.G (and s.Gf()) and the
// step scalars' trace, and reports which Gram ran (gram_small_side's *used_tc).  Eigenpairs the accept rule rejects
// (tf32_reject: too steep a spectrum for a tensor-core Gram's or the fp32 solve's noise floor) are solved again with
// fp64 rotations, on a new exact Gram if the rejected one came from the tensor cores.  prof (nullptr: none) records
// the step's first three events, the caller the fourth.  Returns the step's rank, at most s.kcap, and whether the
// unfolding is zero: then the rank is 1 (round.py:137-145), but the batch rank rule (round.py:149-150) has no zero
// branch and keeps min(rmax, L), so a zero sample's factors are zero at that rank, like the other samples' of its batch.
template <typename T, class GramF>
inline int host_step_solve(const StepCtx& cx, HostStep<T>& s, GramF&& gram, bool use_tc, int32_t rm, bool first_step,
                           bool shared_gpu, bool fp32_solve, Prof* prof, int64_t* rank, bool* zero) {
  const int batch_mode = (cx.flags & TNB_FLAG_BATCH_MODE) ? 1 : 0;
  const SweepScalars* hs = reinterpret_cast<const SweepScalars*>(cx.h_sc);
  if (prof) prof->mark(cx.st);
  int used_tc = 0;
  TNB_TRY(gram(use_tc, &used_tc));
  if (prof) prof->mark(cx.st);
  ChfsiStats cs;
  int solves = 0;
  TNB_TRY(eig_solve_and_rank<T>(s.G, s.ew.Gb, s.L, s.ew, cx.sc, cx.h_sc, rm, batch_mode, &cs, &solves, cx.st,
                                cx.allow_tc, shared_gpu, used_tc, fp32_solve));
  if (hs->tf32_reject) {
    if (used_tc) TNB_TRY(gram(false, &used_tc));
    TNB_TRY(eig_solve_and_rank<T>(s.G, s.ew.Gb, s.L, s.ew, cx.sc, cx.h_sc, rm, batch_mode, &cs, &solves, cx.st,
                                  cx.allow_tc, shared_gpu, 0));
  }
  if (prof) prof->mark(cx.st);
  if (cx.info) {
    cx.info->tc_grams += used_tc ? 1 : 0;
    cx.info->eig_solves += solves, cx.info->chfsi_products += cs.products, cx.info->fused_filters += cs.fused_filters;
    cx.info->rr_sweeps += cs.rr_sweeps, cx.info->rr_solves += cs.outer;
    if (first_step) cx.info->norm = std::sqrt(hs->norm2 > 0 ? hs->norm2 : 0.0);
  }
  *zero = hs->zero_flag != 0;
  *rank = *zero && !batch_mode ? 1 : std::min<int64_t>(hs->rank, s.kcap);
  return TNB_OK;
}

// TIn: the element type of C (the dense input at step 0, else T).
template <typename T, typename TIn, class ArenaT>
inline int truncate_step(ArenaT& ar, bool dry, const StepCtx& cx, const TIn* C, int64_t rows, int64_t n, int64_t rank_cap,
                         bool have_rmax, int32_t rm, bool first_step, T* core, T* Cn, int64_t* rank_out) {
  cudaStream_t st = cx.st;
  const bool tc_gram = cx.tc_gram(dry);
  GramWork gw;
  gram_carve<TIn>(ar, rows, n, tc_gram, gw);
  HostStep<T> s;
  TNB_TRY((host_step_carve<T, TIn>(ar, cx, rows, n, rank_cap, have_rmax, s)));
  if (dry) return TNB_OK;
  if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "workspace too small (need > %zu bytes)", ar.off);
  const bool concurrent = (cx.flags & TNB_FLAG_CONCURRENT) != 0;
  auto gram = [&](bool use_tc, int* used_tc) -> int {
    {
      BigKernelGate gate(st, concurrent && use_tc && gw.tc_ws != nullptr);
      TNB_TRY(gram_small_side<TIn>(C, rows, n, s.G, s.Gf(), gw, use_tc, used_tc, st));
    }
    trace_kernel<<<1, 256, 0, st>>>(s.G, (int)s.L, (int)s.L, cx.sc, first_step ? 1 : 0, cx.eps_scaled2);
    TNB_LAUNCH_CHECK();
    return TNB_OK;
  };
  Prof& prof = Prof::get();
  int64_t rank = 0;
  bool zero = false;
  TNB_TRY(host_step_solve<T>(cx, s, gram, tc_gram, rm, first_step, concurrent, false, &prof, &rank, &zero));
  TNB_TRY((zero ? zero_factors<T>(rows, n, rank, core, Cn, st)
                : step_factors<T, TIn>(cx, C, rows, n, rank, s.ew.w, s.ew.V, s.ew.ldv, s.fac, s.ww, s.ptc_ws, s.ptc_bytes,
                                       core, Cn)));
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
  T* fac = nullptr;   // tall step: V_r
  WideWork ww;        // wide step
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
  s.fac = tall ? ar.template take<T>((size_t)L * (size_t)s.kcap) : nullptr;
  if (!tall) wide_carve(ar, rows, n, s.kcap, s.ww);
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
  TNB_TRY((step_factors<T, TIn>(cx, C, rows, n, s.kcap, s.w, s.V, s.ldv, s.fac, s.ww, s.ptc_ws, s.ptc_bytes, core, Cn,
                                layout, s.out_inner)));
  if (prof_on) prof.mark(st);
  return TNB_OK;
}

// ---------------------------------------------------------------------------------------------
// Dense TT-SVD
// ---------------------------------------------------------------------------------------------
// The carry step 0 wrote when it ran outside the sweep (the streamed step 0 of tnb_ttsvd_stream): C holds
// rows[N-1] x rank elements, K-blocked for step 1 (carry_kblocked(d, N - 2)) or row-major, in memory of its own (never one
// of the ping-pong pair, so that a host-driven repeat of the sweep can start from it again); sc: step 0's device scalars
// (norm2, delta2), copied into the sweep's own.
template <typename T>
struct Carry0 {
  T* C = nullptr;
  int64_t rank = 0;
  bool kblocked = false;
  const SweepScalars* sc = nullptr;
};

// The two ping-pong carries, sized by the rank caps: step t writes carry[t & 1] (rows[mu] x rcap[mu]); steps before t0
// write elsewhere.
template <typename T, class ArenaT>
inline void carve_carries(ArenaT& ar, const SweepDims& d, T* carry[2], int t0 = 0) {
  size_t elems[2] = {0, 0};
  for (int mu = d.N - 1 - t0, t = t0; mu >= 1; --mu, ++t) {
    const size_t e = (size_t)d.rows[mu] * (size_t)d.rcap[mu];
    if (e > elems[t & 1]) elems[t & 1] = e;
  }
  carry[0] = ar.template take<T>(elems[0]);
  carry[1] = ar.template take<T>(elems[1]);
}

// A K-blocked carry (rows' x n', gram_tc.cuh) rewritten row-major in place, one group of 8 rows (8 n' contiguous elements)
// per block through shared memory: what the host-driven sweep reads when it repeats a speculative one from a step-0 carry
// that was written K-blocked.
constexpr int UNBLOCK_MAX_SMEM = 192 * 1024;
__global__ void __launch_bounds__(256) unblock_carry_kernel(float* __restrict__ M, int64_t groups, int64_t n) {
  extern __shared__ __align__(16) float unblock_smem[];
  for (int64_t g = blockIdx.x; g < groups; g += gridDim.x) {
    float* p = M + (size_t)g * 8 * n;
    __syncthreads();
    for (int64_t i = threadIdx.x; i < 8 * n; i += blockDim.x) unblock_smem[i] = p[i];
    __syncthreads();
    for (int64_t i = threadIdx.x; i < 8 * n; i += blockDim.x) {
      const int64_t k = i / n, c = i % n;
      p[i] = unblock_smem[((c / 8 * 2 + k / 4) * 8 + c % 8) * 4 + k % 4];
    }
  }
}

// T: carries and cores; TIn: the dense input (T, or bf16 / fp16 / fp8 with T = float), read by step 0 only.  With c0 the
// sweep starts at step 1 from that step-0 carry (data unused).
template <typename T, typename TIn, class ArenaT>
inline int ttsvd_sync_impl(ArenaT& ar, bool dry, const TIn* data, const SweepDims& d, const int32_t* rmax, double eps,
                           uint32_t flags, T* cores, int32_t* ranks_host, SweepInfo* info, cudaStream_t st,
                           bool exact_gram = false, const Carry0<T>* c0 = nullptr) {
  const int N = d.N;
  StepCtx cx = make_step_ctx(ar, dry, N, eps, flags, info, st, false);
  cx.exact_gram = exact_gram;
  if (c0 && !dry) {
    TNB_CUDA(cudaMemcpyAsync(cx.sc, c0->sc, sizeof(SweepScalars), cudaMemcpyDeviceToDevice, st));
    if (c0->kblocked) {  // this path reads row-major carries
      if constexpr (std::is_same<T, float>::value) {
        const int64_t n = d.shape[N - 2] * c0->rank, groups = d.rows[N - 1] / d.shape[N - 2] / 8;
        static PerDeviceFlag attr;
        TNB_CUDA(ensure_dyn_smem(attr, unblock_carry_kernel, UNBLOCK_MAX_SMEM));
        unblock_carry_kernel<<<(unsigned)std::min<int64_t>(groups, 8 * usable_sms()), 256, 8 * n * sizeof(float), st>>>(
            c0->C, groups, n);
        TNB_LAUNCH_CHECK();
      }
    }
  }
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
  const int t0 = c0 ? 1 : 0;
  T* carry[2];
  carve_carries(ar, d, carry, t0);
  const T* C = c0 ? c0->C : nullptr;  // the carry step t > 0 reads; step 0 reads data
  int64_t r_next = c0 ? c0->rank : 1;
  size_t peak = ar.off;
  for (int mu = N - 1 - t0, t = t0; mu >= 1; --mu, ++t) {
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
inline bool spec_eligible(const SweepDims& d, const int32_t* rmax, double eps, uint32_t flags) {
  if ((flags & TNB_FLAG_NO_SPECULATE) || d.N < 2 || !rmax) return false;
  const bool allow_tc = tc_allowed(flags, false);
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
                      uint32_t flags, T* cores, SweepInfo* info, cudaStream_t st, SpecHostBack* hb,
                      const Carry0<T>* c0 = nullptr) {
  r.ar = &ar;
  r.cx = make_step_ctx(ar, dry, d.N, eps, flags, info, st, true);
  carve_carries(ar, d, r.carry, c0 ? 1 : 0);
  r.data = data;
  r.C = c0 ? c0->C : nullptr;
  r.cores = cores;
  r.peak = ar.off;
  r.hb = hb;
  if (!dry) TNB_CUDA(cudaMemsetAsync(r.cx.d_flags, 0, 4 * sizeof(int), st));
  if (!dry && c0) TNB_CUDA(cudaMemcpyAsync(r.cx.sc, c0->sc, sizeof(SweepScalars), cudaMemcpyDeviceToDevice, st));
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
  r.step.in_kblocked = carry_kblocked<T, TIn>(d, mu, r.cx.allow_tc, r.data);
  r.step.out_inner = carry_kblocked<T, TIn>(d, mu - 1, r.cx.allow_tc, r.data) ? d.shape[mu - 1] : 0;
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
// only sizes the step scratch.  t0 = 1: step 0 ran already (Carry0).
template <typename T, typename TIn, class ArenaT>
inline int spec_enqueue(SpecRun<T, TIn, ArenaT>* runs, int g, bool dry, const SweepDims& d, const int32_t* rmax,
                        bool prof_on, int t0 = 0) {
  for (int mu = d.N - 1 - t0, t = t0; mu >= 1; --mu, ++t) {
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
                           int* spec_flags, const Carry0<T>* c0 = nullptr) {
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
  TNB_TRY(spec_begin(r, ar, dry, data, d, eps, flags, cores, info, st, hb, c0));
  const int rc = spec_enqueue(&r, 1, dry, d, rmax, prof_on, c0 ? 1 : 0);
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
// With c0 the sweep starts at step 1 from that step-0 carry; it is speculative only if step 0 kept its rank cap.
template <typename T, typename TIn, class ArenaT>
inline int ttsvd_impl(ArenaT& ar, bool dry, const TIn* data, const SweepDims& d, const int32_t* rmax, double eps,
                      uint32_t flags, T* cores, int32_t* ranks_host, SweepInfo* info, cudaStream_t st,
                      const Carry0<T>* c0 = nullptr) {
  // the sizing pass cannot ask the device what it supports: size for both paths
  const bool spec = dry ? (d.N >= 2 && rmax != nullptr)
                        : spec_eligible<T>(d, rmax, eps, flags) && (!c0 || c0->rank == d.rcap[d.N - 1]);
  const size_t base = ar.off;
  size_t need_spec = 0;
  if (spec) {
    if (dry) {
      bool all_caps = true;
      for (int mu = 1; mu < d.N; ++mu) all_caps = all_caps && rmax[mu - 1] > 0;
      if (all_caps) {
        const int rc = ttsvd_spec_impl<T, TIn>(ar, true, data, d, rmax, eps, flags, cores, ranks_host, info, st, nullptr, c0);
        if (rc == TNB_OK) need_spec = ar.off - base;
        ar.off = base;
      }
    } else {
      int sflags = 0;
      SweepInfo saved;
      if (info) saved = *info;
      const int rc = ttsvd_spec_impl<T, TIn>(ar, false, data, d, rmax, eps, flags, cores, ranks_host, info, st, &sflags, c0);
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
      return ttsvd_sync_impl<T, TIn>(ar, false, data, d, rmax, eps, flags, cores, ranks_host, info, st, (sflags & 1) != 0,
                                     c0);
    }
  }
  const int rc = ttsvd_sync_impl<T, TIn>(ar, dry, data, d, rmax, eps, flags, cores, ranks_host, info, st, false, c0);
  if (dry && rc == TNB_OK && need_spec > ar.off - base) ar.off = base + need_spec;
  return rc;
}

// ---------------------------------------------------------------------------------------------
// Dense TT-SVD of a tensor in host memory (tnb_ttsvd_stream).  Only step 0 reads the input: C = T viewed
// (rows x I_{N-1}), and a row block of C is a contiguous byte range of the host tensor.  So step 0 streams C through the
// device in chunks of whole row blocks, twice: pass 1 sums the chunk Grams into one fp64 G (in chunk order), the eigen
// stage and rank rule run on G through host_step_solve as in truncate_step, and pass 2 projects each chunk into its row
// range of the step-0 carry.  A TF32 Gram that the accept rule rejects costs one more pass 1 with the exact Gram.
// Steps 1..N-1 then run through ttsvd_impl from that carry, which stays in memory of its own.  The device never holds
// more of the input than the chunk ring.
// ---------------------------------------------------------------------------------------------
constexpr size_t STREAM_DEFAULT_CHUNK = (size_t)256 << 20;
constexpr size_t STREAM_PIECE = (size_t)64 << 20;  // staging piece of a pageable source

// Chunks of whole row blocks: `unit` rows = lcm(16, the narrow Gram's fold (1, 2 or 4), 8 inner when the carry is written
// K-blocked: inner % 16 == 0), so every chunk keeps the full tensor's Gram kernel and the carry's 16-byte alignment; at
// least PROJ_TC_MIN_ROWS rows when the projection runs on the tensor cores, and never fewer rows than columns (a chunk's
// Gram is the n x n one).  A last piece shorter than that joins the chunk before it.
struct ChunkPlan {
  int64_t unit = 16, min_rows = 1, chunk_rows = 0, nchunks = 0, last_rows = 0;
  int64_t max_rows() const { return std::max(chunk_rows, last_rows); }
  int64_t rows_of(int64_t c) const { return c + 1 == nchunks ? last_rows : chunk_rows; }
};
inline ChunkPlan make_chunk_plan(int64_t rows, int64_t n, size_t row_bytes, size_t chunk_bytes, bool proj_tc,
                                 int64_t kb_inner) {
  ChunkPlan p;
  p.unit = kb_inner > 0 ? 8 * kb_inner : 16;
  p.min_rows = std::max<int64_t>(proj_tc ? PROJ_TC_MIN_ROWS : 1, n);
  if (chunk_bytes == 0) chunk_bytes = STREAM_DEFAULT_CHUNK;
  const int64_t want = (int64_t)(chunk_bytes / row_bytes) / p.unit * p.unit;
  p.chunk_rows = std::max(want, ceil_div<int64_t>(p.min_rows, p.unit) * p.unit);
  if (p.chunk_rows >= rows) {
    p.chunk_rows = p.last_rows = rows;
    p.nchunks = 1;
    return p;
  }
  p.nchunks = ceil_div<int64_t>(rows, p.chunk_rows);
  p.last_rows = rows - (p.nchunks - 1) * p.chunk_rows;
  if (p.last_rows < p.min_rows) {
    --p.nchunks;
    p.last_rows += p.chunk_rows;
  }
  return p;
}

// The copy side of the chunk ring, one per device: a copy stream, its events and (for a pageable source) two pinned
// staging pieces.  One streamed decomposition at a time per device uses it.
struct StreamRing {
  cudaStream_t copy = nullptr;
  cudaEvent_t start = nullptr, copied[2] = {}, freed[2] = {}, piece[2] = {};
  void* pinned[2] = {nullptr, nullptr};
  std::mutex mu;
  int ensure(bool staging) {
    if (!copy) {
      TNB_CUDA(cudaStreamCreateWithFlags(&copy, cudaStreamNonBlocking));
      cudaEvent_t* evs[7] = {&start, &copied[0], &copied[1], &freed[0], &freed[1], &piece[0], &piece[1]};
      for (cudaEvent_t* e : evs) TNB_CUDA(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    }
    for (int i = 0; i < 2 && staging; ++i)
      if (!pinned[i]) TNB_CUDA(cudaHostAlloc(&pinned[i], STREAM_PIECE, cudaHostAllocDefault));
    return TNB_OK;
  }
  static StreamRing& get() {
    static StreamRing rings[TNB_MAX_DEVICES];
    return rings[current_device_index()];
  }
};

// One pass over the host tensor: chunk c lands in buf[c & 1] on the copy stream while chunk c - 1 is computed on st
// (events order the two: a buffer is refilled after the kernels that read it).  A pinned source is one DMA per chunk; a
// pageable one is copied by this thread into the pinned pieces in turn, each piece's DMA overlapping the next memcpy.
// compute(c, X, first_row, rows) enqueues the chunk's kernels on st.
template <typename TIn, class F>
inline int stream_pass(StreamRing& ring, const char* host, bool pinned_src, size_t row_bytes, const ChunkPlan& p,
                       TIn* const buf[2], cudaStream_t st, F&& compute) {
  TNB_CUDA(cudaEventRecord(ring.start, st));
  TNB_CUDA(cudaStreamWaitEvent(ring.copy, ring.start, 0));
  int piece = 0;
  for (int64_t c = 0; c < p.nchunks; ++c) {
    const int b = (int)(c & 1);
    char* dst = reinterpret_cast<char*>(buf[b]);
    const size_t off = (size_t)(c * p.chunk_rows) * row_bytes, bytes = (size_t)p.rows_of(c) * row_bytes;
    if (c >= 2) TNB_CUDA(cudaStreamWaitEvent(ring.copy, ring.freed[b], 0));
    if (pinned_src) {
      TNB_CUDA(cudaMemcpyAsync(dst, host + off, bytes, cudaMemcpyHostToDevice, ring.copy));
    } else {
      for (size_t q = 0; q < bytes; q += STREAM_PIECE, ++piece) {
        const int s = piece & 1;
        const size_t nb = std::min(STREAM_PIECE, bytes - q);
        TNB_CUDA(cudaEventSynchronize(ring.piece[s]));  // the DMA out of this piece has finished
        std::memcpy(ring.pinned[s], host + off + q, nb);
        TNB_CUDA(cudaMemcpyAsync(dst + q, ring.pinned[s], nb, cudaMemcpyHostToDevice, ring.copy));
        TNB_CUDA(cudaEventRecord(ring.piece[s], ring.copy));
      }
    }
    TNB_CUDA(cudaEventRecord(ring.copied[b], ring.copy));
    TNB_CUDA(cudaStreamWaitEvent(st, ring.copied[b], 0));
    TNB_TRY(compute(c, reinterpret_cast<const TIn*>(dst), c * p.chunk_rows, p.rows_of(c)));
    TNB_CUDA(cudaEventRecord(ring.freed[b], st));
  }
  return TNB_OK;
}

__global__ void accumulate_kernel(double* __restrict__ G, const double* __restrict__ Gc, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) G[i] += Gc[i];
}

// ||T||_F^2 in fp64 over the chunks of pass 1, in a fixed order, when step 0 takes a tensor-core Gram: its trace is
// shrunk by operand truncation or fp32 accumulation (~7e-4 for TF32 on randn), which ||T||^2 - ||core_0||^2
// (ops.tt_relative_error_from_norm) cannot afford; an exact-product Gram's trace is the norm already.  part[b] = block
// b's sum over the chunk (64 blocks read a chunk far faster than it arrives); part[SUMSQ_BLOCKS] accumulates the chunks.
constexpr int SUMSQ_BLOCKS = 64;
template <typename TIn>
__global__ void __launch_bounds__(512) sumsq_kernel(const TIn* __restrict__ X, int64_t n, double* __restrict__ part) {
  __shared__ double red[32];
  double s = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const double v = gemm_ld<double>(X[i]);
    s = fma(v, v, s);
  }
  s = block_reduce_sum(s, red);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__global__ void sumsq_add_kernel(double* part, int first) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  double s = first ? 0.0 : part[SUMSQ_BLOCKS];
  for (int b = 0; b < SUMSQ_BLOCKS; ++b) s += part[b];
  part[SUMSQ_BLOCKS] = s;
}
// step 0's ||T||^2 (and the eps budget on it) from the exact sum instead of the Gram's trace
__global__ void set_norm2_kernel(SweepScalars* sc, const double* norm2, double eps_scaled) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  sc->norm2 = *norm2;
  sc->delta2 = eps_scaled * *norm2;
}

// true for page-locked host memory, false for pageable; device or managed memory is not a host tensor
inline int host_memory_kind(const void* p, bool* pinned) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    *pinned = false;
    return TNB_OK;
  }
  if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged)
    return fail(TNB_ERR_INVALID, "ttsvd_stream: data_host is device memory (decompose it with tnb_ttsvd)");
  *pinned = a.type == cudaMemoryTypeHost;
  return TNB_OK;
}

// *ring_bytes: the chunk ring's share of the workspace (sizing pass)
template <typename T, typename TIn, class ArenaT>
inline int ttsvd_stream_impl(ArenaT& ar, bool dry, const TIn* host, const SweepDims& d, const int32_t* rmax, double eps,
                             uint32_t flags, size_t chunk_bytes, T* cores, int32_t* ranks_host, SweepInfo* info,
                             cudaStream_t st, size_t* ring_bytes = nullptr) {
  const int N = d.N;
  if (N < 2) return fail(TNB_ERR_UNSUPPORTED, "ttsvd_stream: a tensor of %d mode(s) has no step to stream", N);
  const int mu = N - 1;
  const int64_t rows = d.rows[mu], n = d.shape[mu], kcap = d.rcap[mu];
  if (rows < n)
    return fail(TNB_ERR_UNSUPPORTED, "ttsvd_stream: step 0 is wide (%lld rows < %lld columns) and is not streamed",
                (long long)rows, (long long)n);
  if (kcap >= n)
    return fail(TNB_ERR_WORKSPACE,
                "ttsvd_stream: the step-0 carry (rank %lld of %lld columns) holds as many elements as the input, so it "
                "cannot fit where the input does not; decompose on the device or lower the last rank cap",
                (long long)kcap, (long long)n);
  flags &= ~TNB_FLAG_PROFILE;
  StepCtx cx = make_step_ctx(ar, dry, N, eps, flags, info, st, false);
  const bool have_rmax = rmax && rmax[mu - 1] > 0;
  T* carry0 = ar.template take<T>((size_t)rows * kcap);  // outside the ping-pong pair of the sweep that follows
  const size_t mark = ar.off;
  HostStep<T> s;
  TNB_TRY((host_step_carve<T, TIn>(ar, cx, rows, n, kcap, have_rmax, s)));
  // the chunks keep the full tensor's kernels: its Gram, its projection and its carry's layout
  const bool tc_gram = cx.tc_gram(dry) && gram_tc_tall_ok<TIn>(rows, n);
  const int64_t inner = d.shape[N - 2];
  const bool kb_ok = carry_kblocked<T, TIn>(d, N - 2, cx.allow_tc) && 8 * inner * kcap * sizeof(float) <= UNBLOCK_MAX_SMEM;
  const ChunkPlan plan = make_chunk_plan(rows, n, (size_t)n * sizeof(TIn), chunk_bytes, s.ptc_bytes > 0, kb_ok ? inner : 0);
  const size_t ring_start = ar.off;
  TIn* buf[2] = {ar.template take<TIn>((size_t)plan.max_rows() * n),
                 plan.nchunks > 1 ? ar.template take<TIn>((size_t)plan.max_rows() * n) : nullptr};
  if (ring_bytes) *ring_bytes = ar.off - ring_start;
  // a chunk's Gram scratch is carved for the larger need of the two chunk sizes: it is not monotone in the row count
  GramWork gw;
  for (int64_t r : {plan.chunk_rows, plan.last_rows}) {
    gw.partial_elems = std::max(gw.partial_elems, plan_gemm(n, n, r, true).partial_elems);
    if (tc_gram) gw.tc_bytes = std::max(gw.tc_bytes, gram_tc_input_workspace_bytes<TIn>(r, n));
  }
  gw.partial = ar.template take<double>(gw.partial_elems);
  gw.tc_ws = tc_gram ? ar.template take<char>(gw.tc_bytes) : nullptr;
  double* Gc = plan.nchunks > 1 ? ar.template take<double>((size_t)n * n) : nullptr;
  double* sq = tc_gram ? ar.template take<double>(SUMSQ_BLOCKS + 1) : nullptr;
  const size_t peak = ar.off;
  Carry0<T> c0{carry0, kcap, false, cx.sc};
  if (!dry) {
    if (!ar.ok) return fail(TNB_ERR_WORKSPACE, "workspace too small (need > %zu bytes)", ar.off);
    bool pinned_src = false;
    TNB_TRY(host_memory_kind(host, &pinned_src));
    cx.h_sc = static_cast<int*>(pinned_scratch(sizeof(SweepScalars)));
    if (!cx.h_sc) return fail(TNB_ERR_CUDA, "pinned scratch allocation failed");
    StreamRing& ring = StreamRing::get();
    std::lock_guard<std::mutex> lk(ring.mu);
    TNB_TRY(ring.ensure(!pinned_src));
    struct Drain {  // no DMA may still read the caller's memory or the staging pieces when this returns
      cudaStream_t s;
      ~Drain() { cudaStreamSynchronize(s); }
    } drain{ring.copy};
    const char* src = reinterpret_cast<const char*>(host);
    const size_t row_bytes = (size_t)n * sizeof(TIn);
    int passes = 0;
    auto gram_pass = [&](bool use_tc, int* used_tc) -> int {
      const bool first_pass = ++passes == 1;
      TNB_TRY(stream_pass<TIn>(ring, src, pinned_src, row_bytes, plan, buf, st,
                               [&](int64_t c, const TIn* X, int64_t, int64_t rc) -> int {
                                 if (first_pass && sq) {
                                   sumsq_kernel<TIn><<<SUMSQ_BLOCKS, 512, 0, st>>>(X, rc * n, sq);
                                   TNB_LAUNCH_CHECK();
                                   sumsq_add_kernel<<<1, 32, 0, st>>>(sq, c == 0 ? 1 : 0);
                                   TNB_LAUNCH_CHECK();
                                 }
                                 TNB_TRY(gram_small_side<TIn>(X, rc, n, c == 0 ? s.G : Gc, nullptr, gw, use_tc, used_tc, st));
                                 if (c > 0) {
                                   accumulate_kernel<<<grid_for(n * n), 256, 0, st>>>(s.G, Gc, n * n);
                                   TNB_LAUNCH_CHECK();
                                 }
                                 return TNB_OK;
                               }));
      if (s.Gf()) {
        convert_kernel<double, float><<<grid_for(n * n), 256, 0, st>>>(s.G, s.Gf(), n * n);
        TNB_LAUNCH_CHECK();
      }
      trace_kernel<<<1, 256, 0, st>>>(s.G, (int)n, (int)n, cx.sc, 1, cx.eps_scaled2);
      TNB_LAUNCH_CHECK();
      if (sq) {
        set_norm2_kernel<<<1, 32, 0, st>>>(cx.sc, sq + SUMSQ_BLOCKS, cx.eps_scaled2);
        TNB_LAUNCH_CHECK();
      }
      return TNB_OK;
    };
    const bool spec_tail = spec_eligible<T>(d, rmax, eps, flags);
    // the eigenpairs come from fp32 rotations where the speculative device sweep takes them so (spec_step_eig_begin).
    // Whatever TNB_FLAG_CONCURRENT says, step 0's Gram is not gated and its solve does not share the GPU.
    const bool fp32_solve = spec_tail && std::is_same<T, float>::value && jacobi2_ok((int)n, true);
    int64_t rank = 0;
    bool zero = false;
    TNB_TRY(host_step_solve<T>(cx, s, gram_pass, tc_gram, have_rmax ? rmax[mu - 1] : 0, true, false, fp32_solve, nullptr,
                               &rank, &zero));
    T* core = cores + d.slot[mu];
    if (zero) {
      TNB_TRY(zero_factors<T>(rows, n, rank, core, carry0, st));
    } else {
      c0.kblocked = kb_ok && spec_tail && rank == kcap;
      TNB_TRY(tall_factors<T>(s.ew.w, s.ew.V, s.ew.ldv, n, rank, core, s.fac, st));
      ++passes;
      TNB_TRY(stream_pass<TIn>(ring, src, pinned_src, row_bytes, plan, buf, st,
                               [&](int64_t, const TIn* X, int64_t r0, int64_t rc) -> int {
                                 T* out = carry0 + (size_t)r0 * rank;
                                 if constexpr (tc_input<TIn>())
                                   if (s.ptc_ws)
                                     return project_tc<TIn>(X, rc, n, reinterpret_cast<const float*>(s.fac), (int)rank,
                                                            reinterpret_cast<float*>(out), s.ptc_ws, s.ptc_bytes, st,
                                                            c0.kblocked ? PT_OUT_KBLOCKED : PT_ROWMAJOR,
                                                            c0.kblocked ? inner : 0);
                                 return project_any<T, TIn>(X, rc, n, s.fac, rank, out, st);
                               }));
    }
    if (info) {
      info->stream_passes = passes;
      info->stream_chunks = (int)plan.nchunks;
      if (spec_tail && rank != kcap) info->spec_flags = zero ? 32 : 16;  // spec_check_kernel's bits
    }
    ranks_host[mu] = (int32_t)rank;  // the rest of the sweep sets the others
    c0.rank = rank;
  }
  ar.off = mark;  // the rest of the sweep reuses the chunk ring and step 0's scratch
  TNB_TRY((ttsvd_impl<T, TIn, ArenaT>(ar, dry, nullptr, d, rmax, eps, flags, cores, ranks_host, info, st, &c0)));
  if (dry && peak > ar.off) ar.off = peak;
  return TNB_OK;
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
  const bool spec = batch > 0 && spec_eligible<T>(d, rmax, eps, flags);
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
