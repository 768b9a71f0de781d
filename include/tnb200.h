/*
 * tnb200 — H100-native (sm_90a) decomposition / rounding hot path for tntorch.
 *
 * C-ABI drop-in boundary.  The reference (rballester/tntorch) is 100 % Python and has no
 * FFI of its own (SURVEY.md §8b); these entry points are what a ctypes binding added to the
 * reference would call in place of its torch.linalg call sites.  Each declaration cites the
 * reference interface it replaces (paths relative to the reference repo root).
 *
 * Conventions
 *   - all matrix / tensor arguments are DEVICE pointers unless the name ends in `_host`;
 *     dense tensors are C-contiguous (row-major), exactly torch's default layout;
 *   - `stream` is a cudaStream_t passed as void*; work is enqueued on it, and a call returns
 *     after at most the host synchronisations needed to report data-dependent ranks
 *     (the reference itself syncs once per round_tt: tensor.py:2051 `.item()`);
 *   - the library owns no device memory: workspaces are sized by the *_workspace_bytes
 *     queries and allocated by the caller (torch's caching allocator in the Python shim);
 *   - return value 0 = ok; non-zero = error code below, text via tnb_last_error();
 *   - there is NO CPU fallback: without a CUDA device every compute entry point fails.
 */
#ifndef TNB200_H
#define TNB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TNB_OK 0
#define TNB_ERR_INVALID 1      /* bad argument (maps to ValueError / AssertionError in the shim) */
#define TNB_ERR_CUDA 2         /* CUDA runtime / driver error                                     */
#define TNB_ERR_WORKSPACE 3    /* workspace or output buffer too small                            */
#define TNB_ERR_UNSUPPORTED 4  /* shape/mode outside what the kernels cover (raised, never faked) */
#define TNB_ERR_NOCONV 5       /* iterative eigensolver did not converge                          */

#define TNB_F32 0
#define TNB_F64 1
/* bf16 and fp16 dense input, accepted by tnb_ttsvd, tnb_ttsvd_batch, tnb_ttsvd_host, their *_workspace_bytes queries
 * and tnb_tt_relative_error (16-bit data, fp32 cores).  The cores, their capacity and info_host are fp32 for 16-bit
 * input; every other entry point rejects both codes with TNB_ERR_INVALID. */
#define TNB_BF16 2
#define TNB_F16 3

/* flags for tnb_ttsvd / tnb_tt_round */
#define TNB_FLAG_NO_TENSORCORE 1u /* force the generic fp32/fp64 CUDA-core kernels (debug / parity A-B) */
#define TNB_FLAG_BATCH_MODE 2u    /* reference `batch=True` rank rule: rank = min(rmax, len(S)), no eps  */
#define TNB_FLAG_PROFILE 4u       /* record CUDA events around each phase; timings returned in info_host  */
#define TNB_FLAG_CONCURRENT 8u    /* the caller runs several decompositions at once on different streams: the
                                    whole-GPU kernels (tensor-core Gram, projection) of all of them are chained
                                    one at a time and sized to leave tnb_set_reserved_sms() SMs free for the
                                    one-CTA eigen kernels of the others                                       */
#define TNB_FLAG_NO_SPECULATE 16u /* always take the host-driven sweep (one synchronisation per step).  By default a
                                    decomposition whose ranks are decided by rank caps is enqueued in one go with a
                                    single synchronisation at the end, and repeated on the host-driven path only if
                                    the device-side rank rule disagrees (info_host[26], [27])                  */

int tnb_version(void);
const char* tnb_last_error(void);
/* number of kernel launches issued by this library since process start (bench.py `gpu_launches`) */
uint64_t tnb_launch_count(void);
/* Number of SMs the one-CTA-per-SM kernels (tensor-core Gram, projection) leave free, so that the latency-bound
 * one-CTA kernels of another in-flight decomposition (other stream) can run beside them.  Default 0. */
void tnb_set_reserved_sms(int32_t n);
/* 1 if the TMA tensor-core kernels are usable on the current device (sm_90), else 0 */
int tnb_has_tensorcore_path(void);

/* ------------------------------------------------------------------------------------------
 * Dense tensor -> TT cores (TT-SVD).
 * Replaces: tn.Tensor(data, ranks_tt=...)  tensor.py:401-408  (= _full_rank_tt tensor.py:10-104
 *           + Tensor.round_tt tensor.py:2008-2083 + tn.truncated_svd round.py:52-187).
 *   dtype      TNB_F32 / TNB_F64 (cores come back in the same dtype, like the reference)
 *   data       dense tensor, shape[0..ndim), C-contiguous
 *   rmax       ndim-1 entries, <=0 meaning "no cap" (reference: rmax=None)
 *   eps        relative error budget of round_tt (reference default 1e-14)
 *   cores      output buffer; core k is written at element offset core_offsets_host[k] with shape
 *              [ranks_host[k], shape[k], ranks_host[k+1]]; capacity from tnb_ttsvd_cores_capacity()
 *   ranks_host ndim+1 ints (host), ranks_host[0] = ranks_host[ndim] = 1
 *   info_host  optional (may be NULL) 32 doubles: [0]=||T||_F, [1]=#eig solves, [2]=#ChFSI matrix products,
 *              [3]=#tensor-core Gram launches; with TNB_FLAG_PROFILE also [4]=Gram ms, [5]=eigen ms,
 *              [6]=factor/projection ms (totals), [7]=#steps, [8+3t..10+3t]=the same three for step t < 6;
 *              [26]=1 when the speculative (single-synchronisation) sweep was accepted, [27]=the device flags that
 *              made a speculative sweep repeat on the host-driven path (bit 0 TF32 Gram too coarse, bits 1-3 subspace
 *              solver, bit 4 rank below the cap, bit 5 zero unfolding);
 *              [29]=Jacobi sweeps summed over the Rayleigh-Ritz solves, [30]=#outer subspace iterations,
 *              [31]=#Chebyshev filters that ran as one resident cluster kernel
 * ------------------------------------------------------------------------------------------ */
int64_t tnb_ttsvd_cores_capacity(int ndim, const int64_t* shape, const int32_t* rmax, int64_t* core_offsets_host);
size_t tnb_ttsvd_workspace_bytes(int dtype, int ndim, const int64_t* shape, const int32_t* rmax, uint32_t flags);
int tnb_ttsvd(int dtype, const void* data, int ndim, const int64_t* shape, const int32_t* rmax, double eps,
              uint32_t flags, void* workspace, size_t workspace_bytes, void* cores, int64_t cores_capacity,
              int32_t* ranks_host, double* info_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * A batch of dense tensors of ONE shape -> their TT cores.
 * Replaces: tn.Tensor(data[B, ...], ranks_tt=..., batch=True)  tensor.py:401-408 with the leading batch dimension
 *           (_full_rank_tt tensor.py:58-104 batch branch + round_tt), and any caller that decomposes many tensors
 *           (north_star: "batched decompositions shard the batch dimension"; dist.py shards the batch over GPUs and
 *           calls this per rank).
 *   data[i] / cores[i]  device pointers of tensor i and of its cores buffer (cores_capacity elements each, layout as
 *                       in tnb_ttsvd); ranks_host: batch * (ndim + 1) ints
 *   workspace           k * per_tensor_bytes with k >= 1: up to min(k, 8) decompositions are in flight at once on
 *                       internal streams, enqueued from the calling thread step by step (all Gram kernels of a step,
 *                       then the eigen stages of all tensors interleaved, then every projection) and synchronised ONCE; `stream` is forked from
 *                       and joined to.  tnb_ttsvd_batch_workspace_bytes() returns the recommended size (8 in flight)
 *                       and, through per_tensor_bytes, the unit.
 *   norms_host          optional, batch doubles: ||T_i||_F
 *   speculative_host    optional, batch ints: 1 if tensor i was accepted from the single-synchronisation sweep
 * Tensors need rank caps on every bond for the in-flight path (see TNB_FLAG_NO_SPECULATE); otherwise, and for tensors
 * whose speculation the device rejected, the decomposition runs one tensor at a time like tnb_ttsvd.
 * ------------------------------------------------------------------------------------------ */
size_t tnb_ttsvd_batch_workspace_bytes(int dtype, int batch, int ndim, const int64_t* shape, const int32_t* rmax,
                                       uint32_t flags, size_t* per_tensor_bytes);
int tnb_ttsvd_batch(int dtype, const void* const* data, int batch, int ndim, const int64_t* shape, const int32_t* rmax,
                    double eps, uint32_t flags, void* workspace, size_t workspace_bytes, void* const* cores,
                    int64_t cores_capacity, int32_t* ranks_host, double* norms_host, int32_t* speculative_host,
                    void* stream);

/* Same as tnb_ttsvd, but `data_host` / `cores_host` are HOST buffers (pinned for full speed): the tensor is copied to
 * `device_buffer` in 256 MiB chunks on `stream` (so that a pageable source still overlaps its staging with the DMA), the
 * decomposition runs on the same stream AFTER the copy (nothing of it overlaps the transfer: at 4 GiB per tensor the call
 * is bound by the PCIe link either way), and the cores are copied back before returning.
 * `device_buffer` must hold the dense tensor (prod(shape) elements) and is left filled. */
int tnb_ttsvd_host(int dtype, const void* data_host, int ndim, const int64_t* shape, const int32_t* rmax, double eps,
                   uint32_t flags, void* device_buffer, void* workspace, size_t workspace_bytes, void* cores_dev,
                   int64_t cores_capacity, void* cores_host, int32_t* ranks_host, double* info_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * TT rounding of an existing tensor train.
 * Replaces: Tensor.round_tt(eps, rmax)  tensor.py:2008-2083 (phase A: orthogonalize tensor.py:1881-1909
 *           -> left_orthogonalize tensor.py:1800-1833; phase B: truncated_svd round.py:52-187).
 *   cores_in   ndim device pointers (host array of pointers), core k has shape [ranks_in[k], shape[k], ranks_in[k+1]]
 *   cores_out / ranks_host / capacity: as for tnb_ttsvd, with capacity from tnb_tt_round_cores_capacity()
 * ------------------------------------------------------------------------------------------ */
int64_t tnb_tt_round_cores_capacity(int ndim, const int64_t* shape, const int32_t* ranks_in, const int32_t* rmax,
                                    int64_t* core_offsets_host);
size_t tnb_tt_round_workspace_bytes(int dtype, int ndim, const int64_t* shape, const int32_t* ranks_in,
                                    const int32_t* rmax);
int tnb_tt_round(int dtype, const void* const* cores_in, int ndim, const int64_t* shape, const int32_t* ranks_in,
                 const int32_t* rmax, double eps, uint32_t flags, void* workspace, size_t workspace_bytes,
                 void* cores_out, int64_t cores_capacity, int32_t* ranks_host, void* stream);

/* A batch of TT tensors with ONE shape and ONE input rank profile, rounded with up to 8 of them in flight on internal
 * streams and a single synchronisation (the batched-throughput form of BASELINE.json config 3; Tensor.round_tt on a
 * batch=True tensor, tensor.py:2008-2083 with the leading batch dimension).  cores_in: batch * ndim device pointers,
 * tensor-major; cores_out[i]: buffer of cores_capacity elements for tensor i (layout as tnb_tt_round); ranks_host:
 * batch * (ndim + 1); workspace: k * per_tensor_bytes, k >= 1 tensors in flight.  Needs rank caps on every bond and
 * full-rank left unfoldings for the in-flight path; anything else runs one tensor at a time like tnb_tt_round. */
size_t tnb_tt_round_batch_workspace_bytes(int dtype, int batch, int ndim, const int64_t* shape, const int32_t* ranks_in,
                                          const int32_t* rmax, size_t* per_tensor_bytes);
int tnb_tt_round_batch(int dtype, const void* const* cores_in, int batch, int ndim, const int64_t* shape,
                       const int32_t* ranks_in, const int32_t* rmax, double eps, uint32_t flags, void* workspace,
                       size_t workspace_bytes, void* const* cores_out, int64_t cores_capacity, int32_t* ranks_host,
                       int32_t* speculative_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * Linear combinations of TT tensors, optionally fused with the rounding that follows them.
 * Replaces: Tensor.__add__ / __sub__ / scalar * for TT operands (tensor.py:445-520: block cores — first core side by
 *           side, interior cores block diagonal, last core stacked) and the `tn.round(function(a, b))` step of
 *           tools.reduce (tools.py:460-512), metrics.hadamard_sum (metrics.py:384-446) and every caller that adds and
 *           re-rounds in a loop (SURVEY.md §8f-3).
 *   cores_in   noperands * ndim device pointers, operand-major (cores_in[k * ndim + n] = core n of operand k, shape
 *              [r_n, I_n, r_{n+1}]); ranks_in: noperands * (ndim + 1) ints; alpha: noperands doubles (NULL = all 1),
 *              applied to the first core like the reference's `t * scalar`; at most 16 operands per call
 *   tnb_tt_sum        writes the block cores (summed ranks through tnb_tt_sum_cores_capacity)
 *   tnb_tt_sum_round  assembles them in the workspace and runs the tnb_tt_round sweeps on them in the same call: no
 *                     intermediate tensor exists on the host side; output layout as tnb_tt_round
 * ------------------------------------------------------------------------------------------ */
int64_t tnb_tt_sum_cores_capacity(int noperands, int ndim, const int64_t* shape, const int32_t* ranks_in,
                                  int32_t* ranks_sum_host, int64_t* core_offsets_host);
int tnb_tt_sum(int dtype, const void* const* cores_in, int noperands, const double* alpha, int ndim, const int64_t* shape,
               const int32_t* ranks_in, void* cores_out, int64_t cores_capacity, void* stream);
int64_t tnb_tt_sum_round_cores_capacity(int noperands, int ndim, const int64_t* shape, const int32_t* ranks_in,
                                        const int32_t* rmax, int64_t* core_offsets_host);
size_t tnb_tt_sum_round_workspace_bytes(int dtype, int noperands, int ndim, const int64_t* shape, const int32_t* ranks_in,
                                        const int32_t* rmax);
int tnb_tt_sum_round(int dtype, const void* const* cores_in, int noperands, const double* alpha, int ndim, const int64_t* shape,
                     const int32_t* ranks_in, const int32_t* rmax, double eps, uint32_t flags, void* workspace,
                     size_t workspace_bytes, void* cores_out, int64_t cores_capacity, int32_t* ranks_host, void* stream);
/* Elementwise product of two TT tensors: core n of the result is the row-wise Kronecker product of the operands' cores,
 * out[(a1 a2), i, (b1 b2)] = A[a1, i, b1] * B[a2, i, b2], written to cores_out[n] (ra_n rb_n x I_n x ra_{n+1} rb_{n+1}).
 * Replaces: Tensor.__mul__ for TT operands (tensor.py:560-640) — with tnb_tt_round the multiply-and-round loops of
 * metrics.hadamard_sum (metrics.py:384-446). */
int tnb_tt_hadamard(int dtype, const void* const* cores_a, const void* const* cores_b, int ndim, const int64_t* shape,
                    const int32_t* ranks_a, const int32_t* ranks_b, void* const* cores_out, void* stream);

/* Measurement helper (SURVEY.md §8d): dense TF32 peak of this GPU for the MMA the kernels use — two CTAs per SM whose
 * warps issue mma.sync.m16n8k8 .tf32 back to back on register operands into eight accumulators (no memory traffic),
 * `reps` x `per_commit` MMAs per accumulator; best of `trials` launches timed with CUDA events.  The denominator of the
 * tensor-bound roofline fractions. */
int tnb_measure_tf32_peak(int32_t reps, int32_t per_commit, int32_t trials, double* tflops_host, double* ms_host, void* stream);
/* The same for wgmma.mma_async m64n256k8 .tf32, the instruction of the Gram / A^T B kernel: one CTA per SM, two
 * warpgroups each issuing it with A from registers and B from a fixed shared-memory buffer into their own 128
 * accumulators; `reps` commit groups of 4 x `per_commit` wgmma per warpgroup. */
int tnb_measure_wgmma_tf32_peak(int32_t reps, int32_t per_commit, int32_t trials, double* tflops_host, double* ms_host,
                                void* stream);

/* ------------------------------------------------------------------------------------------
 * Two-factor rank-revealing split  M (m x n)  ->  left (m x r), right (r x n).
 * Replaces: tn.truncated_svd(M, delta, eps, rmax, left_ortho)  round.py:52-187.
 *   delta < 0 means "not given"; eps < 0 means "not given"; both given -> TNB_ERR_INVALID
 *   (round.py:77-78 ValueError).  rmax <= 0 means no cap.  left/right need m*min(m,n) and
 *   min(m,n)*n elements of capacity; *rank_host receives r.
 *   left_ortho: bit 0 = which factor is orthonormal (round.py:164-183); bit 1 = the reference's batch rank rule
 *   for one sample of a batch (round.py:149-150: r = min(rmax, len(S)), eps/delta ignored).  In that mode a zero
 *   sample keeps that rank (zero factors) and *rank_host receives -r, so the caller can apply round.py:138-142
 *   (rank-1 zeros only when every sample is zero).
 * ------------------------------------------------------------------------------------------ */
size_t tnb_truncated_svd_workspace_bytes(int dtype, int64_t m, int64_t n);
int tnb_truncated_svd(int dtype, const void* M, int64_t m, int64_t n, double delta, double eps, int32_t rmax,
                      int left_ortho, void* workspace, size_t workspace_bytes, void* left, void* right,
                      int32_t* rank_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * CP decomposition by alternating least squares.
 * Replaces: tn.Tensor(data, ranks_cp=R, max_iter=, tol=)  tensor.py:210-400 (HOSVD init 217-277, ALS sweeps
 *           323-361 with the MTTKRP of 355-357 and the lstsq of 358-360, stopping rule 373-381).
 *   factors      output, factor n (shape[n] x R, row-major) at element offset factor_offsets_host[n];
 *                capacity from tnb_cp_als_factors_capacity()
 *   errors_host  max_iter doubles: relative error after each sweep;  *iters_host: sweeps performed
 *   tol          stop when errors[-2] - errors[-1] < tol (pass -INFINITY for a fixed sweep count)
 *   workspace    for ndim >= 3 it holds one permuted copy of the data (mode ndim-1 moved to the front, numel elements)
 *                plus one numel / min(shape[ndim-1], shape[ndim-2]) * R intermediate: every sweep reads the data twice
 *                (one projection shared by modes 0..ndim-2, one over the permuted copy for the last mode)
 * ------------------------------------------------------------------------------------------ */
int64_t tnb_cp_als_factors_capacity(int ndim, const int64_t* shape, int32_t R, int64_t* factor_offsets_host);
size_t tnb_cp_als_workspace_bytes(int dtype, int ndim, const int64_t* shape, int32_t R);
int tnb_cp_als(int dtype, const void* data, int ndim, const int64_t* shape, int32_t R, int32_t max_iter, double tol,
               void* workspace, size_t workspace_bytes, void* factors, int64_t factors_capacity, double* errors_host,
               int32_t* iters_host, void* stream);
/* Same sweeps started from the factors already in `factors` (layout as above) instead of the HOSVD initialisation:
 * the reference's CP on a Tucker core starts from random factors (tensor.py:278-302). */
int tnb_cp_als_from(int dtype, const void* data, int ndim, const int64_t* shape, int32_t R, int32_t max_iter, double tol,
                    void* workspace, size_t workspace_bytes, void* factors, int64_t factors_capacity, double* errors_host,
                    int32_t* iters_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * maxvol: dominant r x r submatrix of each of `nbatch` tall N x r fp64 matrices (row-major, contiguous batch).
 * Replaces: py_maxvol(A, tol=1.05, max_iters=100)  tntorch/maxvol.py:114-170, called per TT core from tn.cross
 *           (cross.py:399-402, 431-434) after a device->host copy; here everything stays on the device.
 *   index_dev  nbatch x r int32 (device): selected rows      C_dev  nbatch x N x r (device): A inv(A[index]),
 *              i.e. the interpolation core cross.py:403 recomputes with lstsq
 *   iters_host optional nbatch ints (host): swap iterations used (forces a stream sync when given)
 * ------------------------------------------------------------------------------------------ */
size_t tnb_maxvol_workspace_bytes(int32_t nbatch, int32_t N, int32_t r);
int tnb_maxvol(const double* A, int32_t nbatch, int32_t N, int32_t r, double tol, int32_t max_iters, void* workspace,
               size_t workspace_bytes, int32_t* index_dev, double* C_dev, int32_t* iters_host, void* stream);

/* ------------------------------------------------------------------------------------------
 * rect_maxvol: rectangular 2-volume maximisation of each of `nbatch` tall N x r fp64 matrices (N > r).
 * Replaces: py_rect_maxvol(A, tol, maxK, min_add_K, minK, start_maxvol_iters=10, identity_submatrix=True)
 *           tntorch/maxvol.py:30-111 (called by tn.cross(..., _minimize=True), cross.py:399-400): maxvol with
 *           start_maxvol_iters swaps, then rows are added while the largest squared row norm of the coefficient matrix
 *           exceeds tol^2 (up to maxK rows) or fewer than minK rows are chosen.
 *   index_dev nbatch x maxK int32 (device), the first K_dev[b] entries valid;  C_dev nbatch x N x maxK (device, leading
 *   dimension maxK), the first K_dev[b] columns valid;  K_dev nbatch int32 (device).  r <= minK <= maxK <= N.
 * ------------------------------------------------------------------------------------------ */
size_t tnb_rect_maxvol_workspace_bytes(int32_t nbatch, int32_t N, int32_t r, int32_t maxK);
int tnb_rect_maxvol(const double* A, int32_t nbatch, int32_t N, int32_t r, double tol, int32_t minK, int32_t maxK,
                    int32_t start_maxvol_iters, void* workspace, size_t workspace_bytes, int32_t* index_dev, double* C_dev,
                    int32_t* K_dev, void* stream);

/* ------------------------------------------------------------------------------------------
 * Batched TT-cross plumbing: B independent cross problems on one grid with one rank profile advance together
 * (tntorch_b200/cross_batch.py).  Replaces, for tensor-product grids, the per-core host work of tn.cross:
 *   tnb_cross_gather_coords  the sample coordinates of core j — cross.py:316-321 (interface products selecting grid
 *                            values): X[k][(b, a, i, c)] = grid[k][index_k] for the multi-index
 *                            (lsets[b][a][0..j), i, rsets[b][c][0..N-j-1)); X is N vectors of B*Rl*I*Rr doubles
 *   tnb_cross_update_lsets   nested left index sets after a maxvol step — cross.py:405-411; `local` = row chosen by maxvol
 *                            in the (Rl*I) x Rn sample matrix; lnext [B][Rn][j+1]
 *   tnb_cross_update_rsets   nested right index sets — cross.py:437-443; `local` = row in the (I*Rr) x Rp matrix;
 *                            rprev [B][Rp][N-j]
 *   tnb_cross_tt_eval        out[b][p] = TT_b(idx[p]) for B trains with cores [B][r][I][r'] fp64 — the validation error
 *                            of cross.py:457-459 (Tensor.__getitem__ on a list of index vectors)
 * All index tensors are int32 on the device; `active` (may be NULL) masks problems that already converged.
 * ------------------------------------------------------------------------------------------ */
int tnb_cross_gather_coords(const int32_t* lsets, const int32_t* rsets, const double* grid, int32_t Imax, int32_t B,
                            int32_t N, int32_t j, int32_t Rl, int32_t I, int32_t Rr, double* X, void* stream);
int tnb_cross_update_lsets(const int32_t* lsets, const int32_t* local, int32_t B, int32_t j, int32_t Rl, int32_t I,
                           int32_t Rn, const int32_t* active, int32_t* lnext, void* stream);
int tnb_cross_update_rsets(const int32_t* rsets, const int32_t* local, int32_t B, int32_t N, int32_t j, int32_t I,
                           int32_t Rr, int32_t Rp, const int32_t* active, int32_t* rprev, void* stream);
int tnb_cross_tt_eval(const double* const* cores, int32_t N, const int32_t* ranks, const int32_t* shape, const int32_t* idx,
                      int32_t B, int32_t P, int32_t per_problem, double* out, void* stream);

/* C (M x N) = A (M x K) B (K x N), all row-major, same dtype (fp32: fp32 accumulate; fp64: fp64), CUDA-core tiles.
 * Replaces: `R @ right_unfolding(next)` tensor.py:1826-1832 and `leftcoreL @ L` tensor.py:1868-1878. */
int tnb_matmul(int dtype, const void* A, const void* B, void* C, int64_t M, int64_t N, int64_t K, void* stream);

/* Tall-skinny Householder QR of `nbatch` fp64 matrices (rows x n, row-major): Q (rows x min(rows,n)) explicit,
 * optional R (min(rows,n) x n).  Warp-shuffle reflector kernels, one CTA per matrix.
 * Replaces: torch.linalg.qr(V) before maxvol in tn.cross (cross.py:398, 430) and the QR of
 * Tensor.left_orthogonalize (tensor.py:1816) for small cores. */
size_t tnb_qr_workspace_bytes(int32_t nbatch, int32_t rows, int32_t n);
int tnb_qr_householder(const double* A, int32_t nbatch, int32_t rows, int32_t n, void* workspace, size_t workspace_bytes,
                       double* Q, double* R, void* stream);

/* ------------------------------------------------------------------------------------------
 * Building blocks (exposed for tests, profiling and the Python shim).
 * ------------------------------------------------------------------------------------------ */
/* G (n x n, fp64) = A^T A for A (rows x n), dtype f32/f64; fp64 accumulation on CUDA cores.
 * Replaces: `M.permute(dims) @ M` round.py:104-110 and the QR of tensor.py:1816 (via the Gram sweep). */
size_t tnb_gram_workspace_bytes(int dtype, int64_t rows, int64_t n);
int tnb_gram(int dtype, const void* A, int64_t rows, int64_t n, double* G, void* workspace, size_t workspace_bytes,
             void* stream);
/* Same Gram on the tensor cores: TMA-staged slabs, tf32 mma.sync, fp32 accumulation in registers
 * (fp32 input only, n % 4 == 0).  Output fp64 G like tnb_gram. */
size_t tnb_gram_tc_workspace_bytes(int64_t rows, int64_t n);
int tnb_gram_tc_f32(const float* A, int64_t rows, int64_t n, double* G, void* workspace, size_t workspace_bytes,
                    void* stream);
/* The same Gram of A stored K-blocked: element (k, c) of the rows x n matrix at
 * (((k / 8 * n / 8 + c / 8) * 2 + k % 8 / 4) * 8 + c % 8) * 4 + k % 4, the layout the speculative sweep uses for a carry
 * whose Gram has n >= 256 (both wgmma operands then load K-major, no shared-memory transpose).  n >= 256, n % 8 == 0,
 * rows % 8 == 0; workspace from tnb_gram_tc_workspace_bytes. */
int tnb_gram_tc_kblocked_f32(const float* A, int64_t rows, int64_t n, double* G, void* workspace, size_t workspace_bytes,
                             void* stream);
/* The same Gram of a row-major bf16 A (rows x n, n % 8 == 0; n = 32 / 64 with rows divisible by 128 / n, n = 128 or
 * n >= 256): bf16 wgmma, exact products, fp32 accumulation; workspace: tnb_gram_tc_bf16_workspace_bytes. */
size_t tnb_gram_tc_bf16_workspace_bytes(int64_t rows, int64_t n);
/* The noise level ||E|| / ||G|| the TT-SVD's accept rule allows for a tensor-core Gram of TNB_F32 (TF32), TNB_BF16 or
 * TNB_F16 input, E = G_tc - (1 - c) G after the uniform shrink c; 0 for other codes. */
double tnb_gram_noise_level(int dtype);
int tnb_gram_tc_bf16(const void* A, int64_t rows, int64_t n, double* G, void* workspace, size_t workspace_bytes,
                     void* stream);
/* The same Gram of a row-major fp16 A (same shapes as tnb_gram_tc_bf16): the same kernel with fp16 wgmma, exact
 * products, fp32 accumulation; workspace: tnb_gram_tc_f16_workspace_bytes. */
size_t tnb_gram_tc_f16_workspace_bytes(int64_t rows, int64_t n);
int tnb_gram_tc_f16(const void* A, int64_t rows, int64_t n, double* G, void* workspace, size_t workspace_bytes,
                    void* stream);
/* C (m x n) = alpha * A^T B + beta * D on the same tensor-core kernel (A: K x m, B: K x n, row-major fp32, TF32
 * operands, fp32 accumulation; m, n multiples of 4, >= 32).  The Chebyshev-filter products G*Y of
 * tnb_eig_topk's subspace iteration run through this entry (G symmetric => A = G).  D may be NULL. */
size_t tnb_atb_tc_workspace_bytes(int64_t K, int64_t m, int64_t n);
int tnb_atb_tc_f32(const float* A, int64_t K, int64_t m, const float* B, int64_t n, float* C, float alpha,
                   const float* D, float beta, void* workspace, size_t workspace_bytes, void* stream);
/* Chebyshev filter of the subspace iteration as ONE resident cluster kernel: `steps` products
 * Y_s = a[s-1] * G*Y_{s-1} + bc[s-1] * Y_{s-1} + g[s-1] * Y_{s-2}  (G symmetric n x n fp32, TF32 operands,
 * blocks n x b fp32).  G stays partitioned over the shared memories of the grid for all steps; clusters of 8
 * CTAs reduce their partial tiles through distributed shared memory.  bufs = three n x b device blocks,
 * bufs[0] = Y_0 on entry; the result is left in bufs[steps % 3].  n % 256 == 0, n <= 2048, b % 4 == 0,
 * steps <= 48.  When 8-CTA clusters for all slabs cannot be co-resident the partial tiles go
 * through L2 with a second grid barrier per step.  TNB_ERR_UNSUPPORTED outside that envelope. */
size_t tnb_cheb_filter_workspace_bytes(int32_t n, int32_t b);
int tnb_cheb_filter_f32(const float* G, int32_t n, int32_t b, float* buf0, float* buf1, float* buf2, int32_t steps,
                        const float* a_host, const float* bc_host, const float* g_host, void* workspace,
                        size_t workspace_bytes, void* stream);
/* C (rows x r) = A (rows x n) * V (n x r), same dtype throughout (fp32: FFMA, fp32 accumulate).
 * Replaces: `M @ left` round.py:181 / einsum absorb tensor.py:2081-2083. */
int tnb_project(int dtype, const void* A, int64_t rows, int64_t n, const void* V, int32_t r, void* C, void* stream);
/* The same projection on the tensor cores at fp32 accuracy (3xTF32 split: A_hi V_hi + A_hi V_lo + A_lo V_hi),
 * fp32 only, r <= 64, n % 4 == 0, rows >= 128.  Used by the sweep for the large carries. */
size_t tnb_project_tc_workspace_bytes(int64_t n, int32_t r);
int tnb_project_tc_f32(const float* A, int64_t rows, int64_t n, const float* V, int32_t r, float* C, void* workspace,
                       size_t workspace_bytes, void* stream);
/* The same products with C written K-blocked as the (rows / inner) x (inner * r) matrix whose row a is rows
 * a * inner .. a * inner + inner - 1 of C (inner % 16 == 0, rows % (8 * inner) == 0, r % 16 == 0, r <= 48), and with A read
 * K-blocked (rows % 8 == 0, n % 8 == 0; C row-major).  The K-blocked layout is that of tnb_gram_tc_kblocked_f32.  Each element of C
 * is the same sum as tnb_project_tc_f32's. */
int tnb_project_tc_kblocked_out_f32(const float* A, int64_t rows, int64_t n, const float* V, int32_t r, int64_t inner,
                                    float* C, void* workspace, size_t workspace_bytes, void* stream);
int tnb_project_tc_kblocked_in_f32(const float* A, int64_t rows, int64_t n, const float* V, int32_t r, float* C,
                                   void* workspace, size_t workspace_bytes, void* stream);
/* C (rows x r, fp32) = A (rows x n, bf16) V (n x r, fp32) at fp32 accuracy (V split into three bf16 terms); n % 8 == 0,
 * n >= 64, rows >= 128.  inner > 0 writes C K-blocked like tnb_project_tc_kblocked_out_f32.  Workspace:
 * tnb_project_tc_workspace_bytes. */
int tnb_project_tc_bf16(const void* A, int64_t rows, int64_t n, const float* V, int32_t r, int64_t inner, float* C,
                        void* workspace, size_t workspace_bytes, void* stream);
/* The same with A fp16: V is split into two fp16 terms of V scaled per column by a power of two (chosen on the device),
 * and the scale is divided out of C exactly.  Same shapes, layouts and workspace query as tnb_project_tc_bf16. */
int tnb_project_tc_f16(const void* A, int64_t rows, int64_t n, const float* V, int32_t r, int64_t inner, float* C,
                       void* workspace, size_t workspace_bytes, void* stream);
/* Symmetric eigendecomposition of a PSD matrix G (n x n fp64): all eigenpairs by one-CTA parallel
 * Jacobi (n <= 256), eigenvalues descending in w, eigenvectors in the columns of V (row-major n x n).
 * Replaces: torch.linalg.eigh round.py:114 / the U,S of torch.linalg.svd round.py:96. */
size_t tnb_eigh_workspace_bytes(int32_t n);
int tnb_eigh_jacobi(const double* G, int32_t n, double* w, double* V, void* workspace, size_t workspace_bytes,
                    void* stream);
/* k leading eigenpairs of PSD G (n x n fp64) by Chebyshev-filtered subspace iteration with block b
 * (b = 0 -> default 2k): w (b, descending Ritz values), V (n x b row-major, fp64). info_host[0] = #products. */
size_t tnb_eig_topk_workspace_bytes(int32_t n, int32_t k, int32_t b);
int tnb_eig_topk(const double* G, int32_t n, int32_t k, int32_t b, double tol, double* w, double* V, void* workspace,
                 size_t workspace_bytes, double* info_host, void* stream);
/* Relative reconstruction error ||T - TT(cores)||_F / ||T||_F, accumulated in fp64 on the device
 * (reference: metrics.relative_error metrics.py:135-151 on Tensor.torch() tensor.py:1639-1687). */
size_t tnb_tt_relative_error_workspace_bytes(int dtype, int ndim, const int64_t* shape, const int32_t* ranks);
int tnb_tt_relative_error(int dtype, const void* data, const void* const* cores, int ndim, const int64_t* shape,
                          const int32_t* ranks, void* workspace, size_t workspace_bytes, double* result_host,
                          void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TNB200_H */
