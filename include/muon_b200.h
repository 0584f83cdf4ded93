/*
 * muon_b200.h -- C ABI of the H100-native sparse hot path of scverse/muon.
 *
 * muon itself is pure Python and has no FFI: the reference boundary for this path is the
 * Python signature of mu.atac.pp.tfidf / mu.atac.tl.lsi / mu.tl.mofa (SURVEY.md section 8b).
 * This header is the boundary *below* that Python shim: every entry point is what a
 * ctypes / cffi / pybind binding of the reference would bind for the arithmetic the
 * reference delegates to scipy / ARPACK / mofapy2.  Each declaration cites the reference
 * lines whose arithmetic it replaces (paths relative to the muon checkout).
 *
 * Conventions (all entry points):
 *   - extern "C", plain pointers and sizes; no torch / C++ types.
 *   - return 0 on success, <0 on error; mub_last_error() returns a thread-local message.
 *   - every pointer is a DEVICE pointer unless its name ends in _h (host).
 *   - the library never allocates or frees caller memory; scratch space is passed in and
 *     sized by the matching *_workspace_bytes() query.
 *   - work is enqueued on the caller's stream (cudaStream_t passed as void*); nothing
 *     synchronises unless documented.  Re-entrant, no global mutable state.
 *   - CSR layout: indptr int64[n_rows+1], indices int32[nnz], values float32[nnz]
 *     (nnz may exceed 2^31: 6e9 at BASELINE configs[1]).
 *   - dense operands are row-major with a leading dimension `ld` (floats) that must be one
 *     of the padded widths 32, 64 or 128; columns >= the logical width must be zero.
 */
#ifndef MUON_B200_H
#define MUON_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* mub_stream_t; /* cudaStream_t */

/* flags of mub_tfidf_* : keyword arguments of tfidf(), muon/_atac/preproc.py:18-21,101 */
#define MUB_TFIDF_LOG_TF 1u    /* log_tf=True      preproc.py:103-104 */
#define MUB_TFIDF_LOG_IDF 2u   /* log_idf=True     preproc.py:107-108 */
#define MUB_TFIDF_LOG_TFIDF 4u /* log_tfidf=True   preproc.py:116-117 */
#define MUB_TFIDF_NO_SCALE 8u  /* scale_factor in {None,0,1}: multiply skipped, preproc.py:101 */
#define MUB_TFIDF_BINARIZE 16u /* treat every stored non-zero as 1: binarize() (preproc.py:132-152) fused in */

int mub_version(void);
const char* mub_last_error(void);
/* sm count, compute capability and L2 size of the current device */
int mub_device_info(int* sm_count, int* cc_major, int* cc_minor, int64_t* l2_bytes);

/* ---- TF-IDF (muon/_atac/preproc.py:92-119) -------------------------------------------- */
/* pass 1: row_sum[i] = sum_j c_ij (preproc.py:93);  col_sum[j] += sum_i c_ij (preproc.py:106).
 * row_sum is overwritten, col_sum is ACCUMULATED (zero it first; allreduce it across
 * cell shards before pass 2).  status (optional int32 word, zeroed by the caller) receives
 * bit0 if some row's column indices are not strictly increasing (unsorted or duplicate entries)
 * and bit1 if an explicit zero is stored: such input must be canonicalised first to reproduce
 * the reference's output pattern (scipy's matmul merges duplicates and drops zeros). */
int mub_tfidf_reduce_f32(const int64_t* indptr, const int32_t* indices, const float* data,
                         int64_t n_rows, int32_t n_cols, float* row_sum, float* col_sum,
                         int32_t* status, uint32_t flags, mub_stream_t stream);
int mub_tfidf_reduce_f64(const int64_t* indptr, const int32_t* indices, const double* data,
                         int64_t n_rows, int32_t n_cols, double* row_sum, double* col_sum,
                         int32_t* status, uint32_t flags, mub_stream_t stream);
/* pass 1, tiled variant for fp32 matrices whose rows hold SORTED column indices: a CTA owns mub_tfidf_tile_rows()
 * rows and sweeps the columns tile by tile with the tile's column sums and entry counts in shared memory (two
 * shared-memory atomics per non-zero, one global flush per tile) instead of one global atomic per non-zero.
 * Same outputs and status bits as mub_tfidf_reduce_f32; status is mandatory (bit0 set = some row is not sorted:
 * the sums are then invalid, use mub_tfidf_reduce_f32).  row_sum / indptr point at the first row of the call,
 * row_base = its absolute row number (a multiple of the tile height).  Optional by-product: col_count
 * [n_chunks x n_cols] int32 (zeroed by the caller, accumulated) = stored entries per (row chunk, column), row
 * chunks given by chunk_bounds[n_chunks+1] (absolute rows, multiples of the tile height): the histogram
 * mub_csr_transpose_count would otherwise compute in a pass of its own.  Second optional by-product: rb_count
 * uint16[ceil(n_rows_total / tile height)][n_cols] = stored entries per (row block, column), written (not accumulated)
 * for the blocks of this call; mub_csr_transpose_fill_tiled turns it into write offsets. */
int mub_tfidf_reduce_tiled_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                               int32_t n_cols, float* row_sum, float* col_sum, int32_t* status, uint32_t flags,
                               int32_t* col_count, const int64_t* chunk_bounds, int32_t n_chunks, int64_t row_base,
                               uint16_t* rb_count, mub_stream_t stream);
int mub_tfidf_tile_rows(void);
/* idf[j] = n_obs_total / col_sum[j], log1p if MUB_TFIDF_LOG_IDF (preproc.py:106-108) */
int mub_tfidf_idf_f32(const float* col_sum, int32_t n_cols, double n_obs_total, uint32_t flags,
                      float* idf, mub_stream_t stream);
int mub_tfidf_idf_f64(const double* col_sum, int32_t n_cols, double n_obs_total, uint32_t flags,
                      double* idf, mub_stream_t stream);
/* pass 2: out_ij = log1p(((1/r_i) * c_ij) * sf) * idf_j   (preproc.py:94-96,101-104,110-112,
 * 116-117), association order as written.  data_out may alias data_in (in place). */
int mub_tfidf_apply_f32(const int64_t* indptr, const int32_t* indices, const float* data_in,
                        float* data_out, int64_t n_rows, int32_t n_cols, const float* row_sum,
                        const float* idf, float scale_factor, uint32_t flags, mub_stream_t stream);
int mub_tfidf_apply_f64(const int64_t* indptr, const int32_t* indices, const double* data_in,
                        double* data_out, int64_t n_rows, int32_t n_cols, const double* row_sum,
                        const double* idf, double scale_factor, uint32_t flags, mub_stream_t stream);

/* ---- CSR x dense SpMM: the operator applications inside svds ------------------------------
 * C[n_rows x ld] (=|+=) A * B[n_cols x ld].  Replaces scipy's csr_matvec / csc_matvec loop
 * driven by ARPACK (scipy _svds.py:428-460 called from muon/_atac/tools.py:53) and the dense
 * Y^T Z / Y W contractions of mofapy2 (called from muon/_core/tools.py:583-585).
 * ld in {32,64,128}.  accumulate: 0 -> C = A*B, 1 -> C += A*B.
 * row_counter: optional device int64 scratch word, zeroed by the caller, enabling dynamic row
 * scheduling (recommended for skewed row lengths, e.g. transposed ATAC matrices); may be NULL.
 * flags: MUB_SPMM_ROWS_SORTED states that every row's column indices are ascending (a caller
 * promise, not checked: unsorted rows then give wrong results).  mub_spmm_csr_f32 then runs the
 * tiled kernel, which stages B in shared memory in column tiles once per band of 128 rows instead
 * of gathering a row of B from L2 per non-zero (row_counter is then unused).  The other three
 * entry points accept the flag and keep the row-warp kernel.  Both kernels return the same bits. */
#define MUB_SPMM_ROWS_SORTED 1u
int mub_spmm_csr_f32(const int64_t* indptr, const int32_t* indices, const float* data,
                     int64_t n_rows, int64_t n_cols, const float* B, int32_t ld, float* C,
                     int32_t accumulate, unsigned long long* row_counter, uint32_t flags,
                     mub_stream_t stream);

/* ---- CSR transpose (one-time per matrix): builds the CSR of A^T so that A^T * Y is again a
 * row-gather SpMM (scipy does the same implicitly through csc_matvec, _svds.py:447).
 * Step 1 counts entries per column into t_count[n_cols+1] (int64, zeroed by caller, slot 0 unused
 * so that an inclusive scan of t_count is t_indptr); the caller scans (any device scan), then
 * step 2 scatters.  cursor: int64[n_cols] scratch, overwritten.  Entry order inside a
 * transposed row is not deterministic (atomic slot claim): sums over it differ run to run in
 * the last fp32 bits. */
int mub_csr_transpose_count(const int32_t* indices, int64_t nnz, int32_t n_cols, int64_t* t_count,
                            mub_stream_t stream);
int mub_csr_transpose_fill(const int64_t* indptr, const int32_t* indices, const float* data,
                           int64_t n_rows, int32_t n_cols, int64_t row_offset,
                           const int64_t* t_indptr, int64_t* cursor, int32_t* t_indices,
                           float* t_data, mub_stream_t stream);
/* the same fill for float64 values (differential accessibility ranks a float64 matrix on its own values) */
int mub_csr_transpose_fill_f64(const int64_t* indptr, const int32_t* indices, const double* data,
                               int64_t n_rows, int32_t n_cols, int64_t row_offset,
                               const int64_t* t_indptr, int64_t* cursor, int32_t* t_indices,
                               double* t_data, mub_stream_t stream);

/* "Pairs" layout for transposed panels: entry k of row j is the 8-byte pair {int32 index, float32 value bits},
 * so the scatter writes once per non-zero and the product reads one 8-byte word per entry.
 * fill_pairs: like mub_csr_transpose_fill, writing t_pairs[2*nnz] (int32 view of the int2 array).
 * spmm_csrp : C (+)= A B for a pairs-layout matrix (same kernel family and rules as mub_spmm_csr_f32).
 * csrp_row_stats: per-row sum and sum of squares (fp64).  On the transposed panels these are the per-feature
 *                 moments behind MOFA's centring / intercepts (muon/_core/tools.py:283-287, mofapy2 process_data). */
int mub_csr_transpose_fill_pairs(const int64_t* indptr, const int32_t* indices, const float* data,
                                 int64_t n_rows, int32_t n_cols, int64_t row_offset, const int64_t* t_indptr,
                                 int64_t* cursor, int32_t* t_pairs, mub_stream_t stream);
/* fill_pairs without global atomics and in a fixed order (every transposed row lists its source rows in ascending
 * order, so sums over it are the same on every run), for a row panel that starts on a row-block boundary: rb_count points at the
 * panel's first row block (see mub_tfidf_reduce_tiled_f32), indptr at its first row, t_indptr[n_cols+1] are the panel's
 * transposed row offsets, base is uint32 scratch [ceil(n_rows / tile height)][n_cols] (the scanned write offsets),
 * status (int32, zeroed by the caller) gets bit0 if counts and t_indptr disagree, or if the pattern no longer matches
 * the counts (then the result is invalid; no slot past the panel's non-zeros is written either way). */
int mub_csr_transpose_fill_tiled(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                                 int32_t n_cols, const uint16_t* rb_count, const int64_t* t_indptr, uint32_t* base,
                                 int32_t* t_pairs, int32_t* status, mub_stream_t stream);
int mub_spmm_csrp_f32(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, int64_t n_cols,
                      const float* B, int32_t ld, float* C, int32_t accumulate, unsigned long long* row_counter,
                      uint32_t flags, mub_stream_t stream);
int mub_csrp_row_stats_f32(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, double* sum,
                           double* sumsq, mub_stream_t stream);

/* ---- CSR row-and-column selection: out = A[rows][:, kept columns], the kept columns renumbered.  Cuts a
 * device-resident MOFA view into (view, group) blocks restricted to its use_var features, the work of the scipy
 * fancy indexing X[rows][:, mask] on the host path (muon/_core/tools.py:172-176, 243-255).
 * rows[n_rows_out]: int64 source row of every output row (repeats and any order allowed; NULL = every row, then
 * n_rows_out == n_rows_src); the caller checks that every id is in [0, n_rows_src).  col_map[n_cols_src]: int32 new
 * column of every source column, -1 = dropped (NULL = keep every column); a map that is increasing on the kept
 * columns keeps sorted rows sorted.  indptr values are absolute offsets (they need not start at 0 and may exceed 2^31).
 *   count : out_len[n_rows_out] (int64) = kept entries of every output row; an inclusive scan of it, behind a leading
 *           0, is out_indptr.
 *   fill  : writes out_indices / out_data at out_indptr (absolute offsets), entry order within a row preserved.  No
 *           entry is written outside its output row's range, and a row with no kept entry is not read. */
int mub_csr_select_count(const int64_t* indptr, const int32_t* indices, int64_t n_rows_src, int32_t n_cols_src,
                         const int64_t* rows, int64_t n_rows_out, const int32_t* col_map, int64_t* out_len,
                         mub_stream_t stream);
int mub_csr_select_fill_f32(const int64_t* indptr, const int32_t* indices, const float* data, int32_t n_cols_src,
                            const int64_t* rows, int64_t n_rows_out, const int32_t* col_map, const int64_t* out_indptr,
                            int32_t* out_indices, float* out_data, mub_stream_t stream);

/* ---- tall-skinny Gram (the k x k contraction that is allreduced across cell shards) ------
 * G[l x l] = Y^T Y for Y[n x ld] row-major, float64 result (partials are fp32 per CTA slab,
 * combined in fp64 in a fixed order: deterministic).  Replaces the dense Gram inside
 * scipy.linalg.svd(Av) (_svds.py:511-521) and mofapy2's Z^T Z / W^T diag(tau) W.
 * weights: optional per-row weight w_i (G = Y^T diag(w) Y), may be NULL. */
size_t mub_gram_workspace_bytes(int64_t n, int32_t ld);
int mub_gram_f32(const float* Y, const float* weights, int64_t n, int32_t ld, int32_t l, double* G,
                 void* workspace, mub_stream_t stream);

/* ---- MOFA+ variational updates (mofapy2 training loop reached from muon/_core/tools.py:583-585;
 * equations restated in oracle/mofa_ref.py).  One thread per row, Gauss-Seidel over the K factors,
 * fp64 arithmetic on fp32 storage.  Dense operands are row-major with leading dimension ld >= K.
 * Centring is implicit: Praw = Y^T E[Z] of the UN-centred sparse view, mu[D] the feature means
 * (NULL = no centring), zsum[K] = column sums of E[Z]; inv_scale = 1/std for scale_views.
 *   update_w : spike-and-slab weights of one view over G groups of cells (G=1: no grouping).  Arrays
 *              carry a leading group dimension: Praw[G][D x ld], mu[G][D], zsum[G][K], inv_scale[G],
 *              ZZ[G][K x K] (E[Z^T Z] of the group's cells observed in this view, E[z^2] on the
 *              diagonal), tau[G][D] = E[tau]; alpha/lnth/ln1mth[K] = E[alpha], E[ln theta], E[ln(1-theta)].
 *              W is read (current means) and overwritten; WW = E[(sw)^2], S = q(s=1),
 *              What2 = E[what^2] (both branches) are written.
 *   update_z : factors; Q = sum_m Y_m (tau*W_m) un-centred, and per cell class c (group x set of views
 *              the cell is observed in; cls[N] or NULL = one class): qshift[C][K] the centring correction,
 *              GW[C][K x K] = sum_m W^T diag(tau) W, zvar[C][K] = Var[z_k].  Z read and overwritten.
 *   tau      : b_out[D] = b0 + 1/2 E||y_d - Z w_d||^2 from ssq[D] (centred sum of squares), one
 *              (view, group) block per call. */
int mub_mofa_update_w_f32(const float* Praw, const float* mu, const double* zsum, const double* inv_scale,
                          const double* ZZ, const float* tau, const double* alpha, const double* lnth,
                          const double* ln1mth, float* W, float* WW, float* S, float* What2, int64_t D,
                          int32_t ld, int32_t K, int32_t G, int32_t spikeslab, mub_stream_t stream);
int mub_mofa_update_z_f32(const float* Q, const double* qshift, const double* GW, const double* zvar,
                          const int32_t* cls, float* Z, int64_t N, int32_t ld, int32_t K, int32_t C,
                          mub_stream_t stream);
int mub_mofa_tau_f32(const float* Praw, const float* mu, const double* zsum, double inv_scale, const double* ZZ,
                     const double* ssq, const float* W, const float* WW, double b0, double* b_out, int64_t D,
                     int32_t ld, int32_t K, mub_stream_t stream);

/* Non-gaussian likelihoods (mofapy2 guesses "poisson" for integer and "bernoulli" for binary views when muon
 * passes likelihoods=None, muon/_core/tools.py:272-280): Seeger pseudo-data of a DENSE row-major view around
 * zeta = E[Z] E[W]^T at fixed precision kappa[D] (restated in oracle/mofa_ref.py::mofa_ref_general).
 * kind: 1 = poisson  yhat = zeta - sigmoid(zeta) (1 - y / ln(1+e^zeta)) / kappa_d
 *       2 = bernoulli yhat = zeta - (sigmoid(zeta) - y) / kappa_d
 * mofa_pseudo overwrites zeta[n_rows x D] with yhat; mofa_loglik ACCUMULATES sum ln p(y | zeta) into *out (device
 * double; poisson: y ln rate - rate, bernoulli: y zeta - ln(1+e^zeta)). */
int mub_mofa_pseudo_f32(float* zeta, const float* obs, const float* kappa, int64_t n_rows, int32_t D, int32_t kind,
                        mub_stream_t stream);
int mub_mofa_loglik_f32(const float* zeta, const float* obs, int64_t n_rows, int32_t D, int32_t kind, double* out,
                        mub_stream_t stream);

/* The same quantities for a SPARSE view, without materialising anything N x D.  With g(zeta) = zeta - sigmoid(zeta)
 * / kappa_d the pseudo-data are yhat = g(zeta) everywhere plus, at the stored entries only, s = y sigmoid(zeta) /
 * (kappa_d r(zeta)) (poisson, r = max(ln(1+e^zeta), 1e-30)) or s = y / kappa_d (bernoulli); ln p is -r(zeta)
 * (poisson) / -ln(1+e^zeta) (bernoulli) everywhere plus y ln r(zeta) / y zeta at the stored entries.
 * zeta = Z W^T for Z[n x ld], W[D x ld] (padded columns zero), ld in {32, 64}.  fp32 arithmetic as mub_mofa_pseudo_f32;
 * sums of ln p and of squares in fp64.  A call with n = 0 or D = 0 writes nothing.
 *   lowrank_rows : B[D x ld] given: out[n x ld] = g(zeta) B (accumulate = 0) or += (1), each output row written once,
 *                  deterministic.  B = NULL: *loglik += the everywhere-part of sum ln p (kappa, out unused).
 *   lowrank_cols : P[D x ld] = g(zeta)^T C for C[n x ld] (C = Z gives Yhat^T Z), ssq[D] = sum_n g(zeta)^2; both
 *                  written, deterministic.
 *   nnz_rows     : CSR of the observations (n_rows = n cells); B given: out[n x ld] += S B; B = NULL: *loglik += the
 *                  stored-entry part of sum ln p.
 *   nnz_cols     : one transposed row panel of the observations in the pairs layout (mub_csr_transpose_fill_pairs):
 *                  D rows, entries indexed by the panel's cells, Z and C pointing at the panel's first cell;
 *                  P[D x ld] += S^T C and ssq[D] += sum (2 g s + s^2) over the entries (the cross terms of sum yhat^2). */
int mub_mofa_lowrank_rows_f32(const float* Z, int64_t n, const float* W, int64_t D, const float* kappa, const float* B,
                              int32_t ld, int32_t kind, float* out, int32_t accumulate, double* loglik,
                              mub_stream_t stream);
int mub_mofa_lowrank_cols_f32(const float* Z, int64_t n, const float* W, int64_t D, const float* kappa, const float* C,
                              int32_t ld, int32_t kind, float* P, double* ssq, mub_stream_t stream);
int mub_mofa_nnz_rows_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                          const float* Z, const float* W, const float* kappa, const float* B, int32_t ld, int32_t kind,
                          float* out, double* loglik, mub_stream_t stream);
int mub_mofa_nnz_cols_f32(const int64_t* t_indptr, const int32_t* t_pairs, int64_t D, const float* Z, const float* W,
                          const float* kappa, const float* C, int32_t ld, int32_t kind, float* P, double* ssq,
                          mub_stream_t stream);


/* ---- exact k-nearest neighbours (groundwork for the WNN row, muon/_core/preproc.py:520-528: the reference asks
 * umap's NN-descent for n_multineighbors+1 = 201 neighbours per cell and modality; this search is exact).
 * For every row of X[nq x ld] (d meaningful columns) the k nearest rows of Y[nc x ld] in Euclidean distance,
 * ascending, ties by lower index; out_idx[nq x k] (-1 if fewer than k candidates), out_dist[nq x k] (not squared).
 * X == Y is allowed (a point is then its own first neighbour at distance exactly 0).  k <= 320. */
int mub_knn_l2_f32(const float* X, int64_t nq, const float* Y, int64_t nc, int32_t d, int32_t ld, int32_t k,
                   int32_t* out_idx, float* out_dist, mub_stream_t stream);

/* Same result (bit-identical indices and distances), tensor-core version: wgmma TF32 inner products (3xTF32 for
 * d <= 64) select the candidates (threshold widened by the TF32 error bound so that no true neighbour is lost), an
 * fp32 pass with the arithmetic of mub_knn_l2_f32 ranks them.  d <= 128, k <= 512.  `workspace` of
 * mub_knn_l2_tc_workspace_bytes(nq, nc, d) bytes; *status (zeroed by the caller) gets bit1 if some query had more than
 * ~900 points inside its error band (result then incomplete: use mub_knn_l2_f32). */
size_t mub_knn_l2_tc_workspace_bytes(int64_t nq, int64_t nc, int32_t d);
int mub_knn_l2_tc_f32(const float* X, int64_t nq, const float* Y, int64_t nc, int32_t d, int32_t ld, int32_t k,
                      int32_t* out_idx, float* out_dist, void* workspace, size_t workspace_bytes, int32_t* status,
                      mub_stream_t stream);

/* ---- WNN building blocks (muon/_core/preproc.py:264-640; numba helpers :46-159) ------------------------------
 * bandwidth: for every cell i the n_bw cells minimising the reference's tie-breaking metric
 *   (N - jd*N) + (bbox - e)/bbox  (jd = Jaccard distance of the kNN sets, e = Euclidean distance; preproc.py:51-76)
 *   among cells sharing a neighbour with i, enumerated exactly through the transposed kNN graph
 *   (g_* = kNN graph CSR with sorted rows, t_* = CSR of its transpose); sigma[i] = mean Euclidean distance to
 *   them (preproc.py:462-470).  First pass: cell_list = NULL (tables in shared memory); cells sharing neighbours
 *   with more than 1536 cells get sigma = -1 and status bit0, and are redone by a second call with cell_list
 *   (status bit1 = even the fallback tables were too small).
 * affinity_topk: union of the per-modality candidate lists cands[m][n x n_cand] (-1 = none), affinity
 *   sum_m weight[i,m] * exp(-||x^m_i - x^m_j|| / sigmas[m][i]), distance sqrt(0.5 (1 - affinity)) and the n_out
 *   smallest per cell, ascending (preproc.py:569-604 and _sparse_csr_fast_knn_ :114-135).  reps / dims / lds /
 *   cands / sigmas are HOST arrays of n_mod device pointers / ints. */
int mub_wnn_bandwidth_f32(const int64_t* g_indptr, const int32_t* g_indices, const int64_t* t_indptr,
                          const int32_t* t_indices, const float* X, int64_t n, int32_t d, int32_t ld, int32_t n_bw,
                          double bbox_norm, double* sigma, int32_t* status, const int64_t* cell_list,
                          int64_t n_cells, void* workspace, int32_t table_slots, int32_t n_tables,
                          mub_stream_t stream);
/* fallback pass for hub cells: cell_list[n_cells] = cells with sigma == -1 after the first pass, hash tables of
 * table_slots (power of two) entries in `workspace` (mub_wnn_bandwidth_workspace_bytes(table_slots, n_tables)) */
size_t mub_wnn_bandwidth_workspace_bytes(int32_t table_slots, int32_t n_tables);
int mub_wnn_affinity_topk_f32(int32_t n_mod, const float* const* reps, const int32_t* dims, const int32_t* lds,
                              const int32_t* const* cands, const double* const* sigmas, const double* weight,
                              int64_t n, int32_t n_cand, int32_t n_out, int32_t* out_idx, double* out_dist,
                              int32_t* status, mub_stream_t stream);

/* ---- half-precision dense operand for the early block-Lanczos steps of the svds replacement --------------
 * (scipy _svds.py:428-460 as driven from muon/_atac/tools.py:53).  The operator application is bound by the
 * 4*ld bytes of the dense operand every non-zero pulls through L2 -> L1; with B stored as IEEE half that is
 * 2*ld.  Products and sums stay fp32.  f32_to_f16_scaled: dst[i] = half(src[i] * scale), n a multiple of 4
 * (scale: a power of two that lifts orthonormal columns, |x| <= 1, out of the subnormal range).
 * spmm_csr_h16 / spmm_csrp_h16: C (=|+=) out_scale * A * B_half, same rules as mub_spmm_csr_f32. */
int mub_f32_to_f16_scaled(const float* src, int64_t n, float scale, void* dst, mub_stream_t stream);
int mub_spmm_csr_h16(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                     int64_t n_cols, const void* B_half, int32_t ld, float* C, int32_t accumulate,
                     float out_scale, unsigned long long* row_counter, uint32_t flags, mub_stream_t stream);
int mub_spmm_csrp_h16(const int64_t* indptr, const int32_t* pairs, int64_t n_rows, int64_t n_cols,
                      const void* B_half, int32_t ld, float* C, int32_t accumulate, float out_scale,
                      unsigned long long* row_counter, uint32_t flags, mub_stream_t stream);

/* ---- host <-> device staging (ingest side: adata.X is a pageable scipy CSR, muon/_atac/preproc.py:86-129
 * reads it and rebinds a freshly allocated host matrix).  A stager owns a ring of pinned buffers and a pool
 * of host threads; transfers are chunked through the ring so that the host-side copy of chunk i+1 overlaps
 * the DMA of chunk i.  Fused into the host-side copy: int64 -> int32 narrowing of scipy's index arrays
 * (nnz >= 2^31) and a position-dependent 64-bit fingerprint  sum_i (e_i + C1) * (i*C2 + C3)  of the 32-bit
 * element stream, by which a later call can prove a host array still equals its device twin.
 * Pointers ending in _h are HOST pointers.  A stager is not thread-safe: one transfer at a time.
 *   create : n_bufs pinned buffers of buf_bytes each (n_bufs = 0: thread pool only, no CUDA context needed)
 *   h2d    : src_elem_bytes 1, 4 or 8; narrow = 1 (8-byte sources): int64 -> int32; narrow = 2 (4-byte sources):
 *            float32 -> uint8 for count data (widen on the device with mub_u8_to_f32); *overflow_h = 1 if a value
 *            does not survive the narrowing (the destination is then garbage: resend without narrowing); hash_h
 *            (optional; 4-byte sources or narrow = 1) receives the fingerprint.  Chunks are enqueued on `stream`;
 *            returns when the last chunk is enqueued.
 *   d2h    : synchronous; hash_h (optional, n_bytes % 4 == 0) receives the fingerprint of what was written.
 *   host_fingerprint   : fingerprint of a host array (elem_bytes 4, or 8 = int64 read as narrowed int32).
 *   device_fingerprint : the same function of a device array of n 32-bit elements, ACCUMULATED into *out
 *            (device uint64, zeroed by the caller). */
int mub_stager_create(size_t buf_bytes, int32_t n_bufs, int32_t n_threads, void** out);
int mub_stager_destroy(void* stager);
int mub_stager_h2d(void* stager, const void* src_h, void* dst, size_t n_elems, int32_t src_elem_bytes,
                   int32_t narrow, uint64_t* hash_h, int32_t* overflow_h, mub_stream_t stream);
int mub_stager_d2h(void* stager, const void* src, void* dst_h, size_t n_bytes, uint64_t* hash_h,
                   mub_stream_t stream);
int mub_u8_to_f32(const void* src, int64_t n, float* dst, mub_stream_t stream);
int mub_host_fingerprint(void* stager, const void* src_h, size_t n_elems, int32_t elem_bytes, uint64_t* hash_h);
int mub_device_fingerprint(const void* src, int64_t n, uint64_t* out, mub_stream_t stream);

/* ---- synthetic ATAC count generator (benchmark / test input; SURVEY App. E) ---------------
 * Deterministic counter-based planted-topic model; bit-identical to the numpy generator in
 * muon_b200/_synth.py.  Step 1 writes nnz per row; caller scans into indptr; step 2 fills.
 * beta[n_cols], topic[n_topics x n_cols], row_topic[n_rows], row_scale[n_rows] are host-made
 * tables (device copies); row0 is the global index of the first row (shards hash identically). */
int mub_synth_count(int64_t row0, int64_t n_rows, int32_t n_cols, const float* beta, const float* topic,
                    const int32_t* row_topic, const float* row_scale, uint64_t seed, int64_t* row_nnz,
                    mub_stream_t stream);
int mub_synth_fill(int64_t row0, int64_t n_rows, int32_t n_cols, const float* beta, const float* topic,
                   const int32_t* row_topic, const float* row_scale, uint64_t seed, const int64_t* indptr,
                   int32_t* indices, float* data, mub_stream_t stream);

/* ---- DSB normalisation of protein counts (muon/_prot/preproc.py:161-218) ------------------
 * _f32 / _f64: the dtype of log(X + pseudocount), which is also the output dtype.  Count matrices
 * are CSR (indptr != NULL; canonical: no duplicate entries) or dense row-major (indptr == NULL).
 *   moments : mean[P] and ddof=1 stdev[P] (fp64) of log(x + pseudocount) over the empty droplets
 *             (preproc.py:173-175); only stored entries are read.  Deterministic (fixed-order sums).
 *   fit     : per cell, out[i,:] = (log(x + pc) - mean) [/ stdev if MUB_DSB_STANDARDIZE], rounded
 *             to the output dtype (preproc.py:161-177); with MUB_DSB_FIT also the tied and full
 *             2-component mixtures of preproc.py:183-198 in fp64 on the rounded row: bgmean[i] (min
 *             mean of the model with the smaller BIC, full on a tie, rounded to the output dtype),
 *             model[i] (0 tied, 1 full), n_iter[2i + m], converged[2i + m].  draws holds the uniform
 *             P x 2 blocks of sklearn's init_params="random": the block of fit m of cell i starts at
 *             draws + i*draw_cell_stride + m*draw_model_stride (strides 0: one block for every fit).
 *             A row with a non-finite scaled value sets bit0 of *status (device int32, zeroed by the
 *             caller) and gets bgmean NaN.
 *   cross   : sums[q + q*q + P + q*P] = [sum z | sum z z^T | sum y_j | sum z y_j] over cells, with
 *             z = [y[:, controls] | bgmean], q = n_controls + 1 <= MUB_DSB_MAX_CONTROLS + 1.
 *   apply   : y[i,j] -= (z_i . w - b) * beta[j] (skipped when beta == NULL), then with MUB_DSB_CLIP
 *             y[i,j] = min(max(y[i,j], lo), hi); arithmetic in fp64, rounded to the output dtype. */
#define MUB_DSB_MAX_PROTEINS 1024
#define MUB_DSB_MAX_CONTROLS 14
#define MUB_DSB_STANDARDIZE 1u /* scale_factor="standardize" */
#define MUB_DSB_FIT 2u         /* denoise_counts=True: run the mixture fits */
#define MUB_DSB_CLIP 1u        /* quantile_clipping=True */
size_t mub_dsb_moments_workspace_bytes(int64_t n_rows, int32_t n_prot);
int mub_dsb_moments_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_rows,
                        int32_t n_prot, float pseudocount, void* workspace, double* mean, double* stdev,
                        mub_stream_t stream);
int mub_dsb_moments_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n_rows,
                        int32_t n_prot, double pseudocount, void* workspace, double* mean, double* stdev,
                        mub_stream_t stream);
int mub_dsb_fit_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_cells,
                    int32_t n_prot, float pseudocount, const double* mean, const double* stdev, uint32_t flags,
                    const double* draws, int64_t draw_cell_stride, int64_t draw_model_stride, float* out,
                    double* bgmean, int8_t* model, int32_t* n_iter, int8_t* converged, int32_t* status,
                    mub_stream_t stream);
int mub_dsb_fit_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n_cells,
                    int32_t n_prot, double pseudocount, const double* mean, const double* stdev, uint32_t flags,
                    const double* draws, int64_t draw_cell_stride, int64_t draw_model_stride, double* out,
                    double* bgmean, int8_t* model, int32_t* n_iter, int8_t* converged, int32_t* status,
                    mub_stream_t stream);
size_t mub_dsb_cross_workspace_bytes(int64_t n_cells, int32_t n_prot, int32_t n_controls);
int mub_dsb_cross_f32(const float* y, int64_t n_cells, int32_t n_prot, const double* bgmean,
                      const int32_t* controls, int32_t n_controls, void* workspace, double* sums,
                      mub_stream_t stream);
int mub_dsb_cross_f64(const double* y, int64_t n_cells, int32_t n_prot, const double* bgmean,
                      const int32_t* controls, int32_t n_controls, void* workspace, double* sums,
                      mub_stream_t stream);
int mub_dsb_apply_f32(float* y, int64_t n_cells, int32_t n_prot, const double* bgmean, const int32_t* controls,
                      int32_t n_controls, const double* w, double b, const double* beta, double lo, double hi,
                      uint32_t flags, mub_stream_t stream);
int mub_dsb_apply_f64(double* y, int64_t n_cells, int32_t n_prot, const double* bgmean, const int32_t* controls,
                      int32_t n_controls, const double* w, double b, const double* beta, double lo, double hi,
                      uint32_t flags, mub_stream_t stream);

/* ---- UMAP layout (umap-learn optimize_layout_euclidean, as scanpy's sc.tl.umap calls it) ------------------
 *   epoch  : one Jacobi epoch.  Reads Y_in [n x dim] and writes Y_out (must not alias).  The head entries are the
 *            CSR (indptr, indices) of the pruned graph, the tail entries its transpose (t_indptr, t_indices); eps /
 *            t_eps hold each entry's epochs per sample w_max / w >= 1.  Entry e is sampled at epoch n iff
 *            floor(n/eps) > floor((n-1)/eps); its m-th sample draws floor(n*rate/eps) - floor(n'*rate/eps)
 *            negatives (n' = ceil((m-1)*eps), the first sample counts from 1 instead), vertex
 *            philox4x32_10(ctr = {e_lo, e_hi ^ s2, n, draw}, key = {s0, s1}).x mod n.  Y_out[i] = Y_in[i] +
 *            alpha_n * (sum of the clipped attraction terms of the sampled head and tail entries of i and the
 *            repulsion terms of their negatives, skipping draws equal to i).  Deterministic: fixed-order sums.
 *   philox : out[4t..4t+3] = Philox4x32-10(ctr[4t..4t+3], {k0, k1}) for t < n (the generator of the epoch). */
#define MUB_UMAP_MAX_COMPONENTS 16
int mub_umap_epoch_f32(const int64_t* indptr, const int32_t* indices, const float* eps, const int64_t* t_indptr,
                       const int32_t* t_indices, const float* t_eps, int64_t n, int32_t dim, const float* Y_in,
                       float* Y_out, float a, float b, float gamma, float alpha_n, int32_t epoch,
                       int32_t negative_sample_rate, uint32_t s0, uint32_t s1, uint32_t s2, mub_stream_t stream);
int mub_philox4x32_10(const uint32_t* ctr, int64_t n, uint32_t k0, uint32_t k1, uint32_t* out,
                      mub_stream_t stream);

/* ---- Leiden / Louvain (leidenalg / louvain-igraph on the multiplex RB-configuration objective) --------------------
 * One graph per level: CSR (indptr, indices) with int64 fixed-point weights w (sum_l w_l A^l_uv * 2^Se) and degrees
 * k [n x n_layers] (k^l_v * 2^Sk); ce = 2^-Se, cl_h[l] = w_l gamma_l / m_l * 2^-2Sk.  All sums are exact integer sums.
 * Every pointer is device memory except cl_h, a host array of n_layers doubles read at launch.
 *   scan    : mode 0 (local moving): for every vertex the best move out of memb[v] (neighbour communities, or the
 *             empty community n + v), target[v] = -1 unless its gain exceeds 2^-40 of its magnitude.  mode 1
 *             (refinement): memb is the refined partition, parent the communities; singletons whose coin for `key`
 *             is set move to the best sub-community of their parent they touch (gain >= 0) that is not a moving
 *             singleton; flags bit 0 is set when some singleton still has a non-negative move.  K / size are the
 *             totals of memb.  Rows longer than mub_leiden_max_shared_degree() go through hubs[n_hubs] with a table
 *             of hub_slots[i] (a power of two >= 2 x degree) slots at hub_off[i] in hub_keys / hub_vals (int64), and
 *             hub_slots[i] / 2 list entries at hub_off[i] / 2 in hub_lists.
 *   apply   : mode 0: prio[v] = the unique hashed priority of v's proposal (0 without one, prio is [n] uint64) and the
 *             proposals with priority >= min_priority move; mode 1: every proposal moves (prio unused).  counts =
 *             {moves, moves to an empty community}.
 *   totals  : K[c] = sum of k over memb == c, size[c] = members (size may be NULL).
 *   segment_sum : out[seg[i]] += w[i].   internal : out = sum of w over the entries inside one community. */
#define MUB_LEIDEN_MAX_LAYERS 4
int mub_leiden_scan(int32_t mode, const int64_t* indptr, const int32_t* indices, const int64_t* w, const int64_t* k,
                    int64_t n, int32_t n_layers, double ce, const double* cl_h, const int32_t* memb,
                    const int32_t* parent, const int64_t* K, const int32_t* size, uint64_t key, int32_t* target,
                    double* gain, int32_t* flags, const int32_t* hubs, int64_t n_hubs, const int64_t* hub_off,
                    const int32_t* hub_slots, int32_t* hub_keys, void* hub_vals, int32_t* hub_lists,
                    int32_t* hub_counts, mub_stream_t stream);
int32_t mub_leiden_max_shared_degree(void);
int mub_leiden_apply(int32_t mode, int64_t n, int32_t* memb, const int32_t* target, uint64_t key,
                     uint64_t min_priority, void* prio, int32_t* counts, mub_stream_t stream);
int mub_leiden_totals(int64_t n, int32_t n_layers, const int32_t* memb, const int64_t* k, int64_t n_comm, int64_t* K,
                      int32_t* size, mub_stream_t stream);
int mub_leiden_segment_sum(int64_t n, const int64_t* seg, const int64_t* w, int64_t n_seg, int64_t* out,
                           mub_stream_t stream);
int mub_leiden_internal(int64_t n, const int64_t* indptr, const int32_t* indices, const int64_t* w,
                        const int32_t* memb, int64_t* out, mub_stream_t stream);

/* ---- differential accessibility (scanpy's rank_genes_groups, called by muon/_atac/tools.py:371) ------------------
 * Input: the CSR of A^T (t_indptr [d+1], t_cells [nnz], t_vals [nnz]) and cell_code [n cells]: 0..K-2 = the tested
 * groups, K-1 = the other ranked cells (rest: cells of no tested group; MUB_RANK_VS_GROUP: the reference group),
 * -1 = not ranked (MUB_RANK_VS_GROUP only).  group_n [K] = cells per code; n_ranked = cells with a code >= 0
 * (< 2642245, so that the tie terms are exact in 64 bits).  K - 1 <= MUB_RANK_MAX_GROUPS.
 *   stats : rows [n_rows] of A^T, written to columns cols [n_rows] of stats [5][K][n_out] (float64): stored non-zeros,
 *           sum, sum of squares (each value squared in the input precision), rank sum, tie term sum(t^3 - t).  Rank sum
 *           (codes < K-1, MUB_RANK_WILCOXON): the group's average ranks among all ranked cells (rest), or among the
 *           group and the reference (MUB_RANK_VS_GROUP); exact.  The tie term is that of the same ranking.  Stored
 *           zeros count as implicit zeros; negative values rank below them.  Moments are fixed-order sums: the output
 *           does not depend on the entry order of the transposition.  cap: a power of two >= every row's length; rows
 *           up to mub_rank_shared_capacity() are sorted in shared memory (cap = the size class), longer ones in a
 *           workspace of ws_bytes >= mub_rank_workspace_slice_bytes(cap) (one slice per concurrently sorted row).
 *   score : per (group g < K-1, column) from stats: scores / pvals (Welch's t and its two-sided p, or the Wilcoxon z
 *           and erfc(|z|/sqrt 2); NaN score -> 0, NaN p -> 1), lfc = log2((expm1(mean_g) + 1e-9) / (expm1(mean_r) +
 *           1e-9)) (expm1(x ln base) when log_base > 0), pts [K][n_out] = stored non-zeros / cells (row K-1 with
 *           MUB_RANK_VS_GROUP only), pts_rest [K-1][n_out] (rest only, may be NULL).  n_total = cells of the matrix. */
#define MUB_RANK_WILCOXON 1u
#define MUB_RANK_VS_GROUP 2u
#define MUB_RANK_TIE_CORRECT 4u
#define MUB_RANK_OVERESTIM_VAR 8u
#define MUB_RANK_MAX_GROUPS 1024
int32_t mub_rank_shared_capacity(int32_t value_bytes);
int64_t mub_rank_workspace_slice_bytes(int32_t value_bytes, int32_t cap);
int mub_rank_stats_f32(const int64_t* t_indptr, const int32_t* t_cells, const float* t_vals, const int32_t* cell_code,
                       const int32_t* rows, const int32_t* cols, int32_t n_rows, int32_t n_out, int32_t K,
                       const int64_t* group_n, int64_t n_ranked, uint32_t flags, int32_t cap, void* ws, int64_t ws_bytes,
                       double* stats, mub_stream_t stream);
int mub_rank_stats_f64(const int64_t* t_indptr, const int32_t* t_cells, const double* t_vals, const int32_t* cell_code,
                       const int32_t* rows, const int32_t* cols, int32_t n_rows, int32_t n_out, int32_t K,
                       const int64_t* group_n, int64_t n_ranked, uint32_t flags, int32_t cap, void* ws, int64_t ws_bytes,
                       double* stats, mub_stream_t stream);
int mub_rank_score(const double* stats, int32_t K, int32_t n_out, const int64_t* group_n, int64_t n_total,
                   uint32_t flags, double log_base, double* scores, double* pvals, double* lfc, double* pts,
                   double* pts_rest, mub_stream_t stream);

/* ---- fragments file (muon/_atac/tools.py:746-1201: count_fragments_features, tss_enrichment, nucleosome_signal) ------
 * text: an inflated chunk of the fragments file whose last byte is a newline.
 *   newline_count / newline_fill : tile_counts [ceil(n_bytes / mub_frag_tile_bytes())] newlines per tile; with their
 *           exclusive scan tile_offsets, nl_pos [lines] receives every newline position in byte order.
 *   barcode_table : open addressing over the barcodes bc[bc_off[j] : bc_off[j+1]] (distinct, j < n_bc): keys [capacity]
 *           (zeroed; a power of two > n_bc) hold 64-bit hashes, slot_entry [capacity] the barcode index j.
 *   parse : one thread per line: start, end (int32), score (int32) of the 5 tab-separated fields, cell = bc_val[j] of the
 *           barcode equal byte for byte to the name field, else -1 (keys may be NULL: no lookup).  flags: bit0 = the
 *           line starts a contig run (first line, or a chromosome unlike the previous line's), bit1 = a '#' line.
 *           status int64[5] (caller initialises {INT64_MAX x3, 0, 0}): atomic minimum line_base + line of a malformed
 *           line, of a coordinate or score beyond int32, of a start below the previous line's on the same chromosome;
 *           maximum fragment length; count of '#' lines.
 *   overlap : one warp per query q over records [q_rec_lo, q_rec_hi) (one contig, start-sorted): hits are records with
 *           start < q_hi, end > q_lo and cell >= 0, searched from the first start >= q_lo - lmax + 1.  out_off NULL:
 *           counts [n_q] = hits; else hits go to out_off[q].. in record order as (cell, feat_base + q, score or 1).
 *   tss_pileup : same hits; +score at max(start - q_lo, 0) and -score at min(end - q_lo, width) of the cell's row of
 *           diff [cells][width + 1] (int64, zeroed).
 *   tss_rows : per cell, diff row -> its running sum (the pileup, in place); sums [cells][2] = sum over the first and the
 *           last `flank` positions, sum over [center_lo, center_hi).
 *   tss_scale : out [cells][width] = pile / flank_mean[cell] (float64, IEEE division).
 *   nucleosome : counts [cells][2] += 1 at column 0 when end - start < free_ub, else at column 1 when < mono_ub. */
int64_t mub_frag_tile_bytes(void);
int mub_frag_newline_count(const uint8_t* text, int64_t n_bytes, int64_t* tile_counts, mub_stream_t stream);
int mub_frag_newline_fill(const uint8_t* text, int64_t n_bytes, const int64_t* tile_offsets, int64_t* nl_pos,
                          mub_stream_t stream);
int mub_frag_barcode_table(const uint8_t* bc, const int64_t* bc_off, int32_t n_bc, uint64_t* keys, int32_t* slot_entry,
                           int64_t capacity, mub_stream_t stream);
int mub_frag_parse(const uint8_t* text, const int64_t* nl_pos, int64_t n_lines, int64_t line_base, const uint8_t* bc,
                   const int64_t* bc_off, const int32_t* bc_val, const uint64_t* keys, const int32_t* slot_entry,
                   int64_t capacity, int32_t* start, int32_t* end, int32_t* score, int32_t* cell, uint8_t* flags,
                   int64_t* status, mub_stream_t stream);
int mub_frag_overlap(const int32_t* start, const int32_t* end, const int32_t* cell, const int32_t* score,
                     const int64_t* q_rec_lo, const int64_t* q_rec_hi, const int64_t* q_lo, const int64_t* q_hi,
                     int32_t n_q, int64_t lmax, int32_t use_score, int32_t feat_base, int64_t* counts,
                     const int64_t* out_off, int32_t* out_cell, int32_t* out_feat, int64_t* out_val,
                     mub_stream_t stream);
int mub_frag_tss_pileup(const int32_t* start, const int32_t* end, const int32_t* cell, const int32_t* score,
                        const int64_t* q_rec_lo, const int64_t* q_rec_hi, const int64_t* q_lo, const int64_t* q_hi,
                        int32_t n_q, int64_t lmax, int32_t width, int64_t* diff, mub_stream_t stream);
int mub_frag_tss_rows(int64_t* diff, int64_t n_cells, int32_t width, int32_t flank, int32_t center_lo,
                      int32_t center_hi, int64_t* sums, mub_stream_t stream);
int mub_frag_tss_scale(const int64_t* pile, int64_t n_cells, int32_t width, const double* flank_mean, double* out,
                       mub_stream_t stream);
int mub_frag_nucleosome(const int32_t* start, const int32_t* end, const int32_t* cell, int64_t n, double free_ub,
                        double mono_ub, int32_t* counts, mub_stream_t stream);

/* ---- similarity network fusion (muon.tl.snf), float64 -------------------------------------------------------------
 * Dense N x N row-major matrices on the device.  A fused state is a raw bit-symmetric X with r[i] = sum_j X[i,j] -
 * X[i,i] (0 -> 1); its normalised matrix nv(X)[i,j] = 0.5 on the diagonal, else (X/(2 r_i) + X/(2 r_j)) / 2.  A null
 * r anywhere below means "X is used as is".
 *   symmetrise : D = (D + D^T) / 2 with a zero diagonal, in place.
 *   densify    : out = the canonical CSR (indptr, indices, data) as a dense matrix, unstored entries +inf, diagonal 0.
 *   select     : per row the k entries first in (value, column) order, ascending for SMALLEST (values X), DIST
 *                (0.5 - nv(X), zeros skipped) and CONN (nv(X), zeros skipped), descending value for LARGEST (nv(X)).
 *                out_idx / out_val [n x k] in that order; rows with fewer candidates are padded with -1 / 0 and
 *                out_count[i] (may be null) says how many are real.  k <= MUB_SNF_MAX_NEIGHBORS + 1.
 *   affinity   : means[i] = mean of the finite values of sel[i, 1..k] (sel is [n x (k+1)], the k+1 smallest of D's
 *                row) + eps; then in place D[i,j] = exp(-(y^2)/2) / sqrt(2 pi) / s with s = sigma ((m_i + m_j)/3 +
 *                D[i,j]/3 + eps), y = D[i,j] / s, and 0 where D[i,j] is +inf.
 *   rowsum     : r as above, fixed-order reduction.
 *   average    : out = (nv(xs[0]) + ... + nv(xs[count-1])) / div, summed in that order; xs / rs are host arrays of
 *                device pointers (rs[q] may be null); out may alias xs[0] only when count == 1.
 *   dominate   : (ptr, col, val) is the transposed top-k structure (row i lists the c with i in c's top k, ascending,
 *                val = nv(W)[c, i]); cs[i] = the sum of row i, out[e] = val[e] / cs[col[e]].
 *   diffuse    : C = S . B with S the CSR (s_ptr, s_col, s_val) and B read through nv(., rB).  TRANSPOSED writes
 *                out = C^T; SYMMETRIC computes the upper triangle of C and mirrors it, so out is bit-symmetric.
 *                B and out must not alias.  No float atomics: every call returns the same bits. */
#define MUB_SNF_MAX_NEIGHBORS 255
#define MUB_SNF_MAX_MODALITIES 16
#define MUB_SNF_MAX_CELLS 1048576
#define MUB_SNF_SELECT_SMALLEST 0
#define MUB_SNF_SELECT_LARGEST 1
#define MUB_SNF_SELECT_DIST 2
#define MUB_SNF_SELECT_CONN 3
#define MUB_SNF_DIFFUSE_TRANSPOSED 0
#define MUB_SNF_DIFFUSE_SYMMETRIC 1
int mub_snf_symmetrise_f64(double* D, int64_t n, mub_stream_t stream);
int mub_snf_densify_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t n, double* out,
                        mub_stream_t stream);
int mub_snf_select_f64(const double* X, const double* r, int64_t n, int32_t k, int32_t mode, int32_t* out_idx,
                       double* out_val, int32_t* out_count, mub_stream_t stream);
int mub_snf_affinity_f64(double* D, int64_t n, const double* sel, int32_t k, double sigma, double eps, double* means,
                         mub_stream_t stream);
int mub_snf_rowsum_f64(const double* X, int64_t n, double* r, mub_stream_t stream);
int mub_snf_average_f64(const double* const* xs, const double* const* rs, int32_t count, double div, int64_t n,
                        double* out, mub_stream_t stream);
int mub_snf_dominate_f64(const int64_t* ptr, const int32_t* col, const double* val, int64_t n, double* cs,
                         double* out, mub_stream_t stream);
int mub_snf_diffuse_f64(const int64_t* s_ptr, const int32_t* s_col, const double* s_val, int64_t n, const double* B,
                        const double* rB, double* out, int32_t mode, mub_stream_t stream);

/* ---- motif scanning (muon.atac.tl.scan_sequences), float64 -------------------------------------------------------
 *   encode : in place, A/a C/c G/g T/t -> 0..3, every other byte -> 4.
 *   count  : sequences are codes[seq_off[s] .. seq_off[s+1]), cut into tiles of MUB_MOTIF_TILE window starts
 *            (tile_seq[g] = its sequence, seq_tile0[s] = the sequence's first tile).  Motif m has the columns
 *            col_off[m] .. col_off[m+1] (length <= MUB_MOTIF_MAX_LEN) of tab, MUB_MOTIF_CODES scores per column, the
 *            fifth -inf; motifs are scanned in groups group_m0[q] .. group_m0[q+1] of at most MUB_MOTIF_GROUP_COLS
 *            columns.  A window's score is the float64 sum over its columns in order from 0.0; it is a hit when
 *            score >= thr[m].  counts[seq_tile0[s] * n_motifs + m * n_tiles(s) + (g - seq_tile0[s])] = hits of motif
 *            m in tile g, i.e. laid out in (sequence, motif, tile) order.
 *   fill   : with offsets = the exclusive scan of counts, writes every hit (sequence, motif, window start, score) at
 *            its offset, in (sequence, motif, position) order.  No float atomics: every call returns the same bits. */
#define MUB_MOTIF_MAX_LEN 64
#define MUB_MOTIF_TILE 512
#define MUB_MOTIF_CODES 5
#define MUB_MOTIF_GROUP_COLS 512
int mub_motif_encode(uint8_t* bytes, int64_t n, mub_stream_t stream);
int mub_motif_count(const uint8_t* codes, const int64_t* seq_off, const int32_t* tile_seq, const int64_t* seq_tile0,
                    int64_t n_tiles, const double* tab, const int32_t* col_off, const double* thr,
                    const int32_t* group_m0, int32_t n_groups, int32_t n_motifs, int32_t* counts,
                    mub_stream_t stream);
int mub_motif_fill(const uint8_t* codes, const int64_t* seq_off, const int32_t* tile_seq, const int64_t* seq_tile0,
                   int64_t n_tiles, const double* tab, const int32_t* col_off, const double* thr,
                   const int32_t* group_m0, int32_t n_groups, int32_t n_motifs, const int32_t* counts,
                   const int64_t* offsets, int32_t* out_seq, int32_t* out_motif, int32_t* out_pos, double* out_score,
                   mub_stream_t stream);

/* ---- independent component analysis (muon.tl.ica, muon/_core/tools.py:1365-1386: sklearn FastICA) -----------------
 * X [n x p] row-major in the input dtype (_f32 / _f64), p <= MUB_ICA_MAX_DIM; X1 [n x k] float64 row-major.  Every
 * sum is float64 in a fixed order (per-CTA partials in `workspace`, of mub_ica_workspace_bytes(n, p, k) bytes, summed
 * in CTA order): every call returns the same bits.
 *   moments : mean[p] = column means, gram[p x p] = (X - mean)^T (X - mean); *status (int32, zeroed by the caller)
 *             gets bit0 if a value is not finite.
 *   project : X1[i, :] = Kt^T (x_i - mean) (Kt [p x k], the whitening matrix transposed with sqrt(n) folded in); Kt ==
 *             NULL: X1 = x widened (k == p, mean unused).  Sets bit0 of *status as moments does.
 *   step    : one fixed-point pass for the r rows of W [r x k]: with y = W x1_i, out[r k + r] = [sum_i g(y) x1_i^T |
 *             sum_i g'(y)] for fun LOGCOSH (g = tanh(alpha y)), EXP (y e^(-y^2/2)) or CUBE (y^3).
 *   sources : v = T(Mt^T x1_i) (Mt [k x k], T the output type), then v = T(v / d1) and v = T(v / d2) for the non-null
 *             divisors [k].  Exactly one of out and stats: out [n x k] = v, or stats[2k] = the column means and ddof-0
 *             standard deviations of v (nothing written to out). */
#define MUB_ICA_MAX_DIM 128
#define MUB_ICA_LOGCOSH 0
#define MUB_ICA_EXP 1
#define MUB_ICA_CUBE 2
size_t mub_ica_workspace_bytes(int64_t n, int32_t p, int32_t k);
int mub_ica_moments_f32(const float* X, int64_t n, int32_t p, void* workspace, double* mean, double* gram,
                        int32_t* status, mub_stream_t stream);
int mub_ica_moments_f64(const double* X, int64_t n, int32_t p, void* workspace, double* mean, double* gram,
                        int32_t* status, mub_stream_t stream);
int mub_ica_project_f32(const float* X, int64_t n, int32_t p, const double* mean, const double* Kt, int32_t k,
                        double* X1, int32_t* status, mub_stream_t stream);
int mub_ica_project_f64(const double* X, int64_t n, int32_t p, const double* mean, const double* Kt, int32_t k,
                        double* X1, int32_t* status, mub_stream_t stream);
int mub_ica_step_f64(const double* X1, int64_t n, int32_t k, const double* W, int32_t r, int32_t fun, double alpha,
                     void* workspace, double* out, mub_stream_t stream);
int mub_ica_sources_f32(const double* X1, int64_t n, int32_t k, const double* Mt, const double* d1, const double* d2,
                        float* out, void* workspace, double* stats, mub_stream_t stream);
int mub_ica_sources_f64(const double* X1, int64_t n, int32_t k, const double* Mt, const double* d1, const double* d2,
                        double* out, void* workspace, double* stats, mub_stream_t stream);

/* ---- scOpen imputation (muon.atac.pp.scopen, muon/_atac/preproc.py:155-236: bounded NMF of the scaled pattern) ---
 * The reference factorises X [peaks x cells], X[p, c] = s_c where count(c, p) > 0, by coordinate descent.  Every sum
 * is float64 in a fixed order (per-CTA partials in `workspace`, of mub_scopen_workspace_bytes(rows, k) bytes, summed
 * in CTA order): every call returns the same bits.  Factors are row-major [rows x k] float64, k <= 64.
 *   pattern_count : count[i] = entries > 0 of CSR row i (int64 indptr, int32 indices; NaN does not count).
 *   pattern_fill  : out_indices[out_indptr[i] ..] = the columns of those entries in stored order (out_indptr is the
 *                   scan of count); with row_scale, out_data[..] = row_scale[i] (fp32, the SVD operand).
 *   spmm          : C[i, :] = row_scale[i] sum_{j in pattern row i} col_scale[j] B[j, :]; either scale may be NULL
 *                   (1).  B [cols x k], C [rows x k].
 *   gram          : G [k x k] = Y^T Y for Y [rows x k].
 *   cd            : one sweep of sklearn's _update_cdnmf_fast over the rows of W in place, components 0 .. k-1 in
 *                   order, with HHt = G + l2 I and the update projected onto [0, upper] (upper = +inf: sklearn's);
 *                   *violation = sum over rows and components of |projected gradient|.
 *   impute        : out[(p - p0) n + c] = clip(W[p, :] . Ht[c, :], 0, 1) for p0 <= p < p1 (at most 1048560 rows),
 *                   c < n: a block of rows of clip(W H, 0, 1) [m x n] row-major. */
#define MUB_SCOPEN_MAX_COMPONENTS 64
size_t mub_scopen_workspace_bytes(int64_t rows, int32_t k);
int mub_scopen_pattern_count_f32(const int64_t* indptr, const float* data, int64_t rows, int64_t* count,
                                 mub_stream_t stream);
int mub_scopen_pattern_count_f64(const int64_t* indptr, const double* data, int64_t rows, int64_t* count,
                                 mub_stream_t stream);
int mub_scopen_pattern_fill_f32(const int64_t* indptr, const int32_t* indices, const float* data, int64_t rows,
                                const int64_t* out_indptr, const float* row_scale, int32_t* out_indices,
                                float* out_data, mub_stream_t stream);
int mub_scopen_pattern_fill_f64(const int64_t* indptr, const int32_t* indices, const double* data, int64_t rows,
                                const int64_t* out_indptr, const float* row_scale, int32_t* out_indices,
                                float* out_data, mub_stream_t stream);
int mub_scopen_spmm_f64(const int64_t* indptr, const int32_t* indices, int64_t rows, const double* row_scale,
                        const double* col_scale, const double* B, int32_t k, double* C, mub_stream_t stream);
int mub_scopen_gram_f64(const double* Y, int64_t rows, int32_t k, void* workspace, double* G, mub_stream_t stream);
int mub_scopen_cd_f64(double* W, int64_t rows, int32_t k, const double* G, double l2, const double* XHt, double upper,
                      void* workspace, double* violation, mub_stream_t stream);
int mub_scopen_impute_f64(const double* W, int64_t p0, int64_t p1, const double* Ht, int64_t n, int32_t k,
                          double* out, mub_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* MUON_B200_H */
