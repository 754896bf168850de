/* scanpy_b200.h — C ABI of libscanpy_b200.so: the H100-native (sm_90a) kernels behind
 * scanpy's  sc.pp.pca -> sc.pp.neighbors -> sc.tl.leiden  hot path.
 *
 * The reference (scverse/scanpy @ fabadb94) is pure Python and has no FFI of its own: its hot
 * path is three call sites into third-party native code.  Each entry point below replaces one of
 * those call sites and is what a reference-side binding (ctypes, see INTEGRATION.md) would bind:
 *
 *   sb2_pca_csr_f32            <- sklearn PCA(svd_solver='arpack').fit_transform(csr)
 *                                 src/scanpy/preprocessing/_pca/__init__.py:282-291,308
 *                                 (solver 1: the covariance_eigh route, _pca/_dask.py:143-213 +
 *                                  _pca/_kernels.py:14-58)
 *   sb2_knn_l2_f32             <- KNeighborsTransformer(algorithm='brute').fit_transform(x)
 *                                 src/scanpy/neighbors/__init__.py:754-768,638
 *   sb2_fuzzy_simplicial_set_f32 <- umap.umap_.fuzzy_simplicial_set(...).tocsr()
 *                                 src/scanpy/neighbors/_connectivity.py:124-138
 *   sb2_leiden_csr_f32         <- leidenalg.find_partition / Graph.community_leiden
 *                                 src/scanpy/tools/_leiden.py:184-187,195-196 (graph build
 *                                 src/scanpy/_utils/__init__.py:278-306 is eliminated: CSR in)
 *
 * Conventions
 *   - every function returns int32: 0 ok, <0 error (SB2_E_*); sb2_last_error() gives the text
 *     (thread-local, library-owned, valid until the next failing call on that thread).
 *   - pointers prefixed d_ are DEVICE pointers into memory the caller owns (the Python host
 *     allocates them as torch CUDA tensors); h_ are HOST pointers.  No torch types cross the ABI.
 *   - work is enqueued on the ctx's CUDA stream.  Functions that return host-visible scalars
 *     (nnz, counters, modularity) synchronise that stream before returning; the others are async.
 *   - a ctx is bound to one device and is not thread-safe.  No callbacks, no exceptions.
 *   - indptr is int64 (10M x 4k at 5 % has > 2^31 non-zeros), column / neighbour indices int32.
 */
#ifndef SCANPY_B200_H
#define SCANPY_B200_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB2_OK 0
#define SB2_E_BADARG (-1)
#define SB2_E_CUDA (-2)
#define SB2_E_NCCL (-3)
#define SB2_E_OOM (-4)
#define SB2_E_NOTCONV (-5)
#define SB2_E_UNSUPPORTED (-6)

typedef struct sb2_ctx sb2_ctx;

typedef struct sb2_device_info {
  int32_t device;
  int32_t sm_count;
  int32_t cc_major, cc_minor;
  int32_t clock_khz;        /* max SM clock */
  int32_t mem_clock_khz;
  int32_t l2_bytes;
  int32_t smem_per_block_optin;
  int64_t total_mem;
  char name[64];
} sb2_device_info;

/* per-call statistics (all optional: pass NULL) */
typedef struct sb2_pca_info {
  int32_t iterations;       /* operator applications */
  int32_t converged;        /* 1 if residual test met */
  double max_rel_residual;  /* max_j ||A v_j - theta_j v_j|| / theta_1 over the k kept pairs */
  double total_var;         /* sum of per-gene variances (ddof=1) */
} sb2_pca_info;

typedef struct sb2_knn_info {
  int64_t n_uncertified;    /* query rows that needed the exact fallback */
  float max_norm;
  float pass1_ms;           /* CUDA-event duration of all first-pass sweep launches on the ctx stream */
  double pass1_flops;       /* 2 * n_query * n_points * d: the algorithmic flops of that launch */
  double pass1_issued_flops; /* flops actually issued (tensor path: padded tiles x split-precision K axis) */
  int32_t pass1_tensor;     /* 2 = knn_sweep2_kernel (wgmma, default), 0 = knn_pass1_kernel (fp32 FFMA) */
  int64_t n_resweep;        /* rows the fp16 tier left uncertified, swept again in split precision (tensor path) */
} sb2_knn_info;

typedef struct sb2_leiden_info {
  int32_t passes;           /* whole Leiden iterations run */
  int32_t levels;           /* aggregation levels of the last pass */
  int64_t moves;            /* accepted local moves, all levels */
} sb2_leiden_info;

int32_t sb2_version(void);
const char* sb2_last_error(void);

/* stream: the cudaStream_t (as void*) to enqueue on; NULL means the legacy default stream unless
 * flags has SB2_CTX_PRIVATE_STREAM, in which case the ctx creates its own non-blocking stream. */
#define SB2_CTX_PRIVATE_STREAM 1u
int32_t sb2_ctx_create(int32_t device, void* stream, uint32_t flags, sb2_ctx** out);
int32_t sb2_ctx_destroy(sb2_ctx* ctx);
int32_t sb2_ctx_sync(sb2_ctx* ctx);
int32_t sb2_device_info_get(sb2_ctx* ctx, sb2_device_info* out);
/* number of kernel launches this ctx has enqueued so far (bench.py's gpu_launches) */
int64_t sb2_ctx_launch_count(sb2_ctx* ctx);

/* Multi-GPU (one process per GPU): rank 0 calls sb2_comm_unique_id, the 128 bytes travel to the
 * other ranks through the host's own rendezvous (torch.distributed broadcast), every rank calls
 * sb2_comm_init.  With a communicator attached, sb2_pca_csr_f32 treats its CSR as the rank's row
 * shard and all-reduces its small dense reductions. */
int32_t sb2_comm_unique_id(void* h_id128);
int32_t sb2_comm_init(sb2_ctx* ctx, int32_t n_ranks, int32_t rank, const void* h_id128);
int32_t sb2_comm_allgather(sb2_ctx* ctx, const void* d_send, void* d_recv, int64_t bytes_per_rank);
int32_t sb2_comm_allreduce_f64(sb2_ctx* ctx, double* d_buf, int64_t count);

/* ---- PCA: top-k principal components of the implicitly centred CSR matrix (A1 in SURVEY.md) ----
 * solver 0: block subspace iteration driven by CSR x dense SpMM passes (replaces ARPACK).
 * solver 1: exact Gram route  G = X^T X (one CSR pass) -> covariance -> dense block iteration.
 * n_total = number of rows over ALL ranks (== n when no communicator is attached).
 * Outputs: d_x_pca [n x k] float32 row-major, d_components [k x g] float32 (rows = PCs, sign fixed by
 * svd_flip(u_based_decision=False)), h_var[k], h_var_ratio[k], h_mean[g] (host, float64). */
int32_t sb2_pca_csr_f32(sb2_ctx* ctx, int64_t n, int64_t n_total, int32_t g, const int64_t* d_indptr,
                        const int32_t* d_indices, const float* d_data, int32_t k, int32_t solver,
                        int32_t max_iter, double tol, uint64_t seed, float* d_x_pca, float* d_components,
                        double* h_var, double* h_var_ratio, double* h_mean, sb2_pca_info* info);

/* building blocks of the above, exported for tests / profiling */
int32_t sb2_csr_col_stats(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                          const float* d_data, double* d_col_sum, double* d_col_sumsq);
/* Y[n x l] = X * B[g x l] - 1 * shift[l]  (shift may be NULL) */
int32_t sb2_spmm_csr(sb2_ctx* ctx, int64_t n, int32_t g, int32_t l, const int64_t* d_indptr,
                     const int32_t* d_indices, const float* d_data, const float* d_b, const float* d_shift,
                     float* d_y);
/* Z[g x l] (float64) = X^T * Y[n x l] */
int32_t sb2_spmm_csr_t(sb2_ctx* ctx, int64_t n, int32_t g, int32_t l, const int64_t* d_indptr,
                       const int32_t* d_indices, const float* d_data, const float* d_y, double* d_z);
/* G[g x g] (float64, full symmetric) = X^T X */
int32_t sb2_csr_gram(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                     const float* d_data, double* d_gram);

/* sc.pp.pca(zero_center=False): replaces sklearn.decomposition.TruncatedSVD (src/scanpy/preprocessing/_pca/__init__.py:309-336).
 * Top-k singular triplets of X itself: d_x_pca = X V (= U Sigma), d_components = V^T with svd_flip(u_based_decision=False)
 * signs, h_var = np.var(X V, axis=0) (ddof 0), h_var_ratio = h_var / sum of per-gene variances (ddof 0). */
int32_t sb2_tsvd_csr_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                         const float* d_data, int32_t k, int32_t solver, int32_t max_iter, double tol, uint64_t seed,
                         float* d_x_pca, float* d_components, double* h_var, double* h_var_ratio, sb2_pca_info* info);

/* ---- out-of-core / chunked PCA: sc.pp.pca(chunked=True) (src/scanpy/preprocessing/_pca/__init__.py:245-271) ----
 * The reference streams row chunks through sklearn.decomposition.IncrementalPCA and asserts the result equals the full PCA
 * (tests/test_pca.py:357-386).  Here the chunks stream through the exact Gram route: device memory = one chunk + 2 g^2
 * doubles, independent of n.
 *   pass 1: sb2_pca_stream_accumulate_f32 adds the chunk's column sums / sums of squares into d_stats fp64 [2g] and its
 *           X^T X into d_gram fp64 [g x g] (caller zero-fills both before the first chunk);
 *   solve : sb2_pca_stream_solve_f32 -> d_components [k x g], h_var, h_var_ratio, h_mean as sb2_pca_csr_f32, plus the
 *           projection operator d_proj fp32 [g x 128] (first g * *h_l entries used), d_shift fp64 [128], *h_l (32/64/128);
 *   pass 2: sb2_pca_stream_project_f32 -> d_x_pca [n_chunk x k] = X_chunk U - mu^T U. */
int32_t sb2_pca_stream_accumulate_f32(sb2_ctx* ctx, int64_t n_chunk, int32_t g, const int64_t* d_indptr,
                                      const int32_t* d_indices, const float* d_data, double* d_stats, double* d_gram);
int32_t sb2_pca_stream_solve_f32(sb2_ctx* ctx, int64_t n_total, int32_t g, const double* d_stats, const double* d_gram,
                                 int32_t k, int32_t max_iter, double tol, uint64_t seed, float* d_components, double* h_var,
                                 double* h_var_ratio, double* h_mean, float* d_proj, double* d_shift, int32_t* h_l,
                                 sb2_pca_info* info);
int32_t sb2_pca_stream_project_f32(sb2_ctx* ctx, int64_t n_chunk, int32_t g, const int64_t* d_indptr,
                                   const int32_t* d_indices, const float* d_data, int32_t k, int32_t l, const float* d_proj,
                                   const double* d_shift, float* d_x_pca);

/* ---- exact brute-force kNN (euclidean) -----------------------------------------------------
 * points: d_x [n_points x d] float32 row-major.  Queries are rows [q0, q0+n_query) of the same
 * array (q0 % 128 == 0 unless n_query == n_points).  k includes the query itself: column 0 of
 * the outputs is the query row with distance 0 (src/scanpy/neighbors/_common.py:74-98).
 * Outputs [n_query x k]: d_idx int32 (global row ids), d_dist float64, ascending by (distance, id).
 * d <= 150, k <= 56.  Exactness: a fast first pass (wgmma fp16 / split-fp16 sweeps; SB2_KNN_PASS1=ffma selects the
 * fp32 CUDA-core sweep, k <= 30) proposes 32 (k <= 24) or 64 candidates per query, an fp64 re-score certifies the top-k
 * against a rounding-error bound, uncertified rows are recomputed exactly. */
int32_t sb2_knn_l2_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int64_t q0, int64_t n_query,
                       int32_t k, int32_t* d_idx, double* d_dist, sb2_knn_info* info);

/* test / debug entry: raw proposals (scores in the sweep's scaled units + ids, 64 per point) of ONE cold-start tensor-core
 * sweep in the operand format `terms` (1: fp16, 3: split fp16) and the quantities its rounding-error certificate uses:
 * h_meta[6] = { inv_s2 (score_true = score * inv_s2), largest squared norm R^2, max_p |x_p - fp16(x_p)|, c_q, c_n, list_m };
 * the certificate bounds |score * inv_s2 - (q.c - |c|^2/2)| by  c_n R^2/2 + c_q |q| R  (+ for terms = 1:
 * dnorm[q] R + (|q| + dnorm[q]) max dnorm).  d_dnorm [n_points] may be NULL. */
int32_t sb2_knn_debug_proposals_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int32_t terms,
                                    float* d_score, int32_t* d_idx, float* d_dnorm, double* h_meta);

/* test / debug entry: the tile screen of a whole-data-set kNN call (k neighbours, d <= 150, fp16 tier), as the default
 * sweep would use it at any size.  d_perm [n_points]: the kd order (position -> point; query block b holds the points
 * at positions [128 b, 128 b + 128)); d_lists [blocks x tiles] / d_len [blocks]: per query block the ascending candidate
 * tiles (of the order) it visits; d_ub [n_points]: per position the bound u >= the row's k-th neighbour distance that
 * justified the skipped tiles (+inf: none). */
int32_t sb2_knn_debug_screen_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int32_t k, int32_t* d_perm,
                                 int32_t* d_lists, int32_t* d_len, float* d_ub);

/* ---- UMAP fuzzy simplicial set -> symmetric connectivities CSR -------------------------------
 * d_knn_idx/d_knn_dist [n x k] (column 0 = self), as produced by sb2_knn_l2_f32; 2 <= k <= 64.
 * Output CSR: d_indptr int64[n+1], d_indices int32[cap], d_data float32[cap]; cap >= 2*n*(k-1) is
 * always enough.  Rows sorted by column, no explicit zeros, zero diagonal. */
int32_t sb2_fuzzy_simplicial_set_f32(sb2_ctx* ctx, int64_t n, int32_t k, const int32_t* d_knn_idx,
                                     const double* d_knn_dist, float set_op_mix_ratio, float local_connectivity,
                                     int64_t* d_indptr, int32_t* d_indices, float* d_data, int64_t cap,
                                     int64_t* h_nnz, float* d_sigmas, float* d_rhos);

/* method='gauss' (method 1) / 'jaccard' (method 2) connectivities from the same k-lists (SURVEY.md 8f row f3;
 * src/scanpy/neighbors/_connectivity.py:17-100 sparse kNN branch, :141-186).  float64 values like the reference. */
int32_t sb2_knn_connectivities_f64(sb2_ctx* ctx, int64_t n, int32_t k, const int32_t* d_knn_idx, const double* d_knn_dist,
                                   int32_t method, int64_t* d_indptr, int32_t* d_indices, double* d_data, int64_t cap,
                                   int64_t* h_nnz);

/* ---- Leiden on a symmetric weighted CSR graph ------------------------------------------------
 * n_iterations < 0: iterate until a whole pass moves nothing.  Output membership int32[n]
 * renumbered by decreasing community size; *h_modularity at the given resolution.  Weights must be finite and
 * non-negative (SB2_E_BADARG otherwise); results do not change when every weight is multiplied by a power of two.
 * sb2_modularity_csr_f32: d_membership ids in [0, n). */
int32_t sb2_leiden_csr_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                           const float* d_weights, double resolution, int32_t n_iterations, uint64_t seed,
                           int32_t* d_membership, double* h_modularity, int32_t* h_n_comms, sb2_leiden_info* info);
int32_t sb2_modularity_csr_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                               const float* d_weights, double resolution, const int32_t* d_membership,
                               double* h_modularity);
/* Louvain (SURVEY.md 8f row f3): local moving + aggregation, no refinement, one pass to its fixed point - replaces
 * `louvain.find_partition(g, RBConfigurationVertexPartition, ...)` / `g.community_multilevel(weights)` at
 * src/scanpy/tools/_louvain.py:150-176.  Outputs as sb2_leiden_csr_f32. */
int32_t sb2_louvain_csr_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                            const float* d_weights, double resolution, uint64_t seed, int32_t* d_membership,
                            double* h_modularity, int32_t* h_n_comms, sb2_leiden_info* info);

/* ---- preprocessing passes in front of the path (SURVEY.md 8f, row f2): normalize_total, log1p, HVG statistics ----
 * sb2_csr_row_sums_f32      <- numba `_normalize_csr` (src/scanpy/preprocessing/_normalization.py:29-66): per-cell
 *                              totals; with d_skip_cols only columns whose flag is 0 are summed
 * sb2_csr_hiexpr_count_f32  <- same function, the `exclude_highly_expressed` branch: per-gene count of entries
 *                              exceeding max_fraction * cell total
 * sb2_csr_scale_rows_f32    <- axis_mul_or_truediv(x, counts_per_cell, op=truediv, allow_divide_by_zero=False)
 *                              (src/scanpy/_utils/__init__.py:623-660), in place
 * sb2_log1p_f32             <- np.log1p(x.data) [/ log(base)] (src/scanpy/preprocessing/_simple.py:359-380), in place
 * sb2_csr_col_sums_f32      <- stats.mean_var(expm1(x), axis=0) inside highly_variable_genes(flavor='seurat')
 *                              (src/scanpy/preprocessing/_highly_variable_genes.py:337-346): per-gene sum and sum of
 *                              squares (fp64) of expm1(x * log_scale) (apply_expm1 = 1; the product is formed in fp64
 *                              and rounded once to float32, as numpy's `x *= np.log(base)` on float32 data) or of x */
int32_t sb2_csr_row_sums_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                             const float* d_data, const int32_t* d_skip_cols, float* d_out);
int32_t sb2_csr_hiexpr_count_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                                 const float* d_data, const float* d_row_sums, double max_fraction,
                                 int32_t* d_counts_per_col);
int32_t sb2_csr_scale_rows_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, float* d_data, const float* d_scale);
int32_t sb2_log1p_f32(sb2_ctx* ctx, int64_t nnz, float* d_data, double base);
int32_t sb2_csr_col_sums_f32(sb2_ctx* ctx, int64_t nnz, int32_t g, const int32_t* d_indices, const float* d_data,
                             int32_t apply_expm1, double log_scale, double* d_sum, double* d_sumsq);

/* ---- quality control and filtering in front of normalize_total (csrc/qc.cu) ----
 * sb2_csr_qc_rows_f32    <- describe_obs + top_segment_proportions_sparse_csr (src/scanpy/preprocessing/_qc.py:41-129,
 *                           :430-457) and the per-cell numbers of filter_cells (src/scanpy/preprocessing/_simple.py:53-196).
 *                           Per row: d_count int64 = #(data != 0), or #(data > 0) with positive_only; d_total fp64 = sum
 *                           of the stored values; d_qc_total fp64 [n x n_qc] = the sum over the genes whose bit b is set
 *                           in d_qc_bits[col] (n_qc <= 32; NULL when n_qc == 0); d_top fp64 [n x n_ns] = the sum of the
 *                           h_ns[i] largest non-zero stored values, padded with zeros up to max(h_ns) as the reference's
 *                           sparse branch does.  h_ns is a HOST array, sorted ascending, every entry in [1, g].  The top
 *                           sums are exact selections with a fixed-order fp64 prefix sum: they depend only on the
 *                           multiset of non-zero values in the row.  max(h_ns) beyond the shared-memory candidate
 *                           capacity (32768 on sm_90) is an error when some row has more stored values than that.
 * sb2_csr_col_counts_f32 <- describe_var's axis_nnz (_qc.py:178-180) and filter_genes' `data > 0` count (_simple.py:
 *                           284-286): d_counts int64 [g] = #(data != 0) (or > 0) per column, overwritten.  The per-gene
 *                           totals are sb2_csr_col_sums_f32 with apply_expm1 = 0. */
int32_t sb2_csr_qc_rows_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                            const float* d_data, int32_t positive_only, const uint32_t* d_qc_bits, int32_t n_qc,
                            const int32_t* h_ns, int32_t n_ns, int64_t* d_count, double* d_total, double* d_qc_total,
                            double* d_top);
int32_t sb2_csr_col_counts_f32(sb2_ctx* ctx, int64_t nnz, int32_t g, const int32_t* d_indices, const float* d_data,
                               int32_t positive_only, int64_t* d_counts);

/* ---- sc.pp.regress_out (src/scanpy/preprocessing/_simple.py:468-681; csrc/regress.cu) ----
 * X is a block of `rows` rows given either dense (d_x, row-major [rows x g]) or as CSR arrays (d_indptr pointing at the
 * block's first row, entry offsets absolute; column indices sorted within each row, no duplicates; d_x NULL), with
 * float32 (is_f64 = 0) or float64 values.
 * sb2_regress_col_sums  <- `regressor.T @ data` of numpy_regress_out and the per-category means of
 *                          _create_regressor_categorical.  Weighted (d_w != NULL, fp64 [rows x p], p <= 32): d_acc[k*g+j]
 *                          += sum_i w[i,k] x[i,j].  Grouped (d_w == NULL): d_acc[c*g+j] += sum of x[i,j] over the rows
 *                          with d_group[i] == c < n_groups; d_order lists the block's rows sorted by (i / TILE, group, i).
 *                          Also folds the per-gene min / max into d_min / d_max and sets d_nan[j] if column j holds a NaN
 *                          (implicit CSR zeros count as 0).  fp64 sums in a fixed order over TILE-row subtiles: calling it
 *                          over consecutive blocks whose lengths, except the last, are multiples of TILE gives the same
 *                          bits as one call over all rows.
 * sb2_regress_residual  <- `data[i] -= regressor[i] @ coeff` / the GLM residuals: d_out[i*g+j] = x[i,j] - fit[i,j], in fp64
 *                          rounded once to float32 (out_f64 = 0, float32 X only) or float64, fit = sum_k w[i,k] coef[k*g+j]
 *                          (d_w != NULL) or d_b0[j] + d_b1[j] * d_means[c*g+j] with c = d_code[i] (d_b0[j] for c < 0); genes
 *                          with d_pass[j] != 0 (d_pass may be NULL) are copied unchanged. */
#define SB2_REGRESS_TILE_ROWS 1024
int32_t sb2_regress_col_sums(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                             const int64_t* d_indptr, const int32_t* d_indices, const void* d_data, const double* d_w,
                             int32_t p, const int32_t* d_group, const int32_t* d_order, int32_t n_groups, double* d_acc,
                             double* d_min, double* d_max, int32_t* d_nan);
int32_t sb2_regress_residual(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                             const int64_t* d_indptr, const int32_t* d_indices, const void* d_data, const double* d_w,
                             int32_t p, const double* d_coef, const int32_t* d_code, const double* d_means,
                             const double* d_b0, const double* d_b1, const uint8_t* d_pass, int32_t out_f64,
                             void* d_out);

/* ---- sc.experimental.pp analytic Pearson residuals (src/scanpy/experimental/pp/_highly_variable_genes.py:35-287,
 * _normalization.py:36-75; csrc/pearson.cu) ----
 * X is a block of `rows` rows as for regress_out: dense (d_x) or CSR arrays (d_indptr pointing at the block's first row,
 * entry offsets absolute; sorted column indices, no duplicates), float32 (is_f64 = 0) or float64 values.  The residual
 * of x[i,j] is clip((x - mu) / sqrt(mu + mu*mu/theta)) with mu = gene[j] * cell[i] / total, in fp64; clip keeps NaN;
 * theta may be +inf.
 * sb2_pearson_row_sums       <- `x.sum(axis=1)`: d_out[i] = fp64 total of row i, in a fixed order.
 * sb2_pearson_residual_var   <- _calculate_res_sparse / _calculate_res_dense for one batch.  Row k of the call is X row
 *                               d_order[k] (d_order NULL: row k of the block; with CSR, d_indptr then indexes d_order's
 *                               rows), d_cell[k] its cell total.  Merges into d_acc fp64 [4 x g] (zeroed before the first
 *                               call of a batch): row 0 the count, 1 the mean residual, 2 the sum of squared deviations
 *                               (the variance is M2 / count), 3 Σx².  Blocks of one batch must be consecutive, and all but
 *                               the last a multiple of SB2_PEARSON_TILE_ROWS rows: the result then has the same bits as
 *                               one call over the batch.
 * sb2_pearson_residuals      <- _pearson_residuals: d_out[i*g+j] = the residual, rounded once to float32 (out_f64 = 0,
 *                               float32 X only) or float64; d_cell[i] is row i's total. */
#define SB2_PEARSON_TILE_ROWS 1024
int32_t sb2_pearson_row_sums(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                             const int64_t* d_indptr, const void* d_data, double* d_out);
int32_t sb2_pearson_residual_var(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                                 const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                                 const int64_t* d_order, const double* d_gene, const double* d_cell, double total,
                                 double clip, double theta, double* d_acc);
int32_t sb2_pearson_residuals(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                              const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                              const double* d_gene, const double* d_cell, double total, double clip, double theta,
                              int32_t out_f64, void* d_out);

/* ---- sc.pp.combat (src/scanpy/preprocessing/_combat.py:71-289; csrc/combat.cu) ----
 * X is a block of `rows` rows as for regress_out: dense (d_x) or CSR arrays (d_indptr pointing at the block's first row,
 * entry offsets absolute; sorted column indices, no duplicates), float32 (is_f64 = 0) or float64 values.  DᵀX is
 * sb2_regress_col_sums (grouped for the batch columns, weighted for the covariate columns).  With stand_mean[i,j] =
 * d_grand[j] + sum_k cov[i,k] d_beta[k*g+j] (cov fp64 [rows x p], p <= 32; p = 0: d_cov, d_beta may be NULL) and
 * r = x - stand_mean, all in fp64:
 * sb2_combat_moments <- the per-batch statistics of _standardize_data / combat for one batch.  Row k of the call is X row
 *                       d_order[k] (d_order NULL: row k of the block; with CSR, d_indptr then indexes d_order's rows),
 *                       d_cov row k its covariates.  Merges into d_acc fp64 [3 x g] (zeroed before the first call of a
 *                       batch): row 0 the count, 1 the mean of r, 2 the sum of squared deviations of r.  Blocks of one
 *                       batch must be consecutive, and all but the last a multiple of SB2_COMBAT_TILE_ROWS rows: the
 *                       result then has the same bits as one call over the batch.
 * sb2_combat_adjust  <- the parametric adjustment: d_out[i*g+j] (float64) = ((s - gamma[b*g+j]) / dsq[b*g+j]) *
 *                       sqrt_vp[j] + stand_mean[i,j] with b = d_batch[i], s = r / sqrt_vp[j] (0 where sqrt_vp[j] == 0);
 *                       d_cov row i belongs to block row i. */
#define SB2_COMBAT_TILE_ROWS 1024
int32_t sb2_combat_moments(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                           const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                           const int64_t* d_order, const double* d_cov, int32_t p, const double* d_grand,
                           const double* d_beta, double* d_acc);
int32_t sb2_combat_adjust(sb2_ctx* ctx, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                          const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                          const int32_t* d_batch, const double* d_cov, int32_t p, const double* d_grand,
                          const double* d_beta, const double* d_sqrt_vp, const double* d_gamma, const double* d_dsq,
                          double* d_out);

/* ---- sc.metrics.morans_i / sc.metrics.gearys_c (src/scanpy/metrics/_morans_i.py, _gearys_c.py; csrc/autocorr.cu) ----
 * X holds all n cells as rows: dense (d_x, row-major [n x g]) or CSR arrays (d_xindptr over all n rows; sorted column
 * indices, no duplicates; d_x NULL), float32 (is_f64 = 0) or float64 values.  The graph is a block of `rows` rows, cells
 * row0 .. row0 + rows - 1, as CSR arrays with fp64 weights (d_gindptr pointing at the block's first row, entry offsets
 * absolute; column indices in [0, n) in any order; explicit zeros, self-loops, empty rows and negative weights allowed).
 * The per-gene mean comes from sb2_regress_col_sums; Σx and the constancy flag are not recomputed here.
 * sb2_autocorr_sums <- the arc loops of _morans_i_vec_w and _gearys_c_vec_w.  With z = x - d_mean[j] for gene j, merges
 *                      into d_acc fp64 [3 x g] (zeroed before the first call): row 0 A = Σ_i z_i Σ_j w_ij z_j (`inum`),
 *                      row 1 B = Σ_i Σ_j w_ij (x_i - x_j)² (`total`), row 2 Q = Σ_i z_i², summed over the block's rows i
 *                      and their stored arcs i -> j, in fp64 on the centred and differenced values.  Blocks must be
 *                      consecutive, and all but the last a multiple of SB2_AUTOCORR_TILE_ROWS rows: the result then has
 *                      the same bits as one call over all rows. */
#define SB2_AUTOCORR_TILE_ROWS 1024
int32_t sb2_autocorr_sums(sb2_ctx* ctx, int64_t row0, int64_t rows, int32_t g, int32_t is_f64, const void* d_x,
                          const int64_t* d_xindptr, const int32_t* d_xindices, const void* d_xdata,
                          const int64_t* d_gindptr, const int32_t* d_gindices, const double* d_gweights,
                          const double* d_mean, double* d_acc);


/* ---- sc.get.aggregate (src/scanpy/get/_aggregated.py:47-190, 663-698; csrc/aggregate.cu) ----
 * sb2_aggregate_group_order <- the stable order of the kept rows by group: d_codes int32 [n] in [0, n_groups) or -1 (no
 *                              group); d_offsets int64 [n_groups + 1] = each group's first position (d_offsets[n_groups]
 *                              = kept rows) and d_order int64 [>= kept rows] the row ids, each group's rows ascending.
 * X is dense (d_x, row-major [rows x g]) or CSR arrays (sorted column indices, no duplicates), float32 (is_f64 = 0) or
 * float64 values; row k of a call is X row d_order[k] (d_order NULL: row k).  The call's rows form n_seg segments,
 * segment s = call rows h_seg_row[s] .. h_seg_row[s + 1] - 1 (host arrays), consecutive rows of group h_seg_group[s];
 * a group appears in at most one segment per call.
 * sb2_aggregate_moments <- Aggregate.sum / mean_var / count_nonzero: merges each segment's rows into its group's row
 *                          of d_sum, d_mean, d_m2 (fp64 [n_groups x g]: Σx, the mean, the sum of squared deviations)
 *                          and d_nnz (int64: the count of x != 0; implicit and stored zeros are zeros).  h_seg_n0[s] =
 *                          the group's rows merged by earlier calls, a multiple of SB2_AGGREGATE_TILE_ROWS (0: the
 *                          group's outputs are overwritten).  The bits depend only on each group's rows and their order.
 * sb2_aggregate_median  <- Aggregate.median: d_out [n_groups x g] (float32 when is_f64 = 0, else float64) row
 *                          h_seg_group[s] = np.median over the segment's rows, which must be all of the group's rows:
 *                          the mean, in the value type, of the order statistics (n-1)/2 and n/2 with zeros included.
 *                          A CSR's NaN sorts above +inf (sklearn's csc_median_axis_0); a dense group with a NaN gives
 *                          NaN (np.median). */
#define SB2_AGGREGATE_TILE_ROWS 1024
int32_t sb2_aggregate_group_order(sb2_ctx* ctx, int64_t n, const int32_t* d_codes, int32_t n_groups,
                                  int64_t* d_order, int64_t* d_offsets);
int32_t sb2_aggregate_moments(sb2_ctx* ctx, int32_t n_seg, const int64_t* h_seg_row, const int32_t* h_seg_group,
                              const int64_t* h_seg_n0, int32_t g, int32_t is_f64, const void* d_x,
                              const int64_t* d_indptr, const int32_t* d_indices, const void* d_data,
                              const int64_t* d_order, double* d_sum, double* d_mean, double* d_m2, int64_t* d_nnz);
int32_t sb2_aggregate_median(sb2_ctx* ctx, int32_t n_seg, const int64_t* h_seg_row, const int32_t* h_seg_group,
                             int32_t g, int32_t is_f64, const void* d_x, const int64_t* d_indptr,
                             const int32_t* d_indices, const void* d_data, const int64_t* d_order, void* d_out);

/* ---- sc.pp.scrublet / sc.pp.scrublet_simulate_doublets (src/scanpy/preprocessing/_scrublet/core.py:188-238, 313-386;
 * csrc/scrublet.cu) ----
 * sb2_scrublet_pair_sums  <- scipy's canonical `x[p0] + x[p1]` for every row pair of d_pairs int64 [n_sim x 2] of the
 *                            observed CSR (int64 indptr, sorted unique int32 indices, float32 data): d_out_indptr int64
 *                            [n_sim + 1]; d_out_indices / d_out_data hold at least Σ_s (nnz(p0) + nnz(p1)) entries, of
 *                            which d_out_indptr[n_sim] are written.  Entries whose fp32 sum is 0 are dropped.
 * sb2_knn_label_count_f32 <- the k-neighbour label count of Scrublet's classifier over the points d_x [n x d] fp32
 *                            row-major (1 <= k <= n < 2^31, d <= 256, |x| <= 2^55 and finite).  Point i's neighbour set
 *                            is i plus its k - 1 nearest other points in (fp64 squared distance, id) order, the fp64
 *                            squared distance summed over the columns in order with every operation rounded.
 *                            d_count int32 [n] = members with id >= n_first; d_kth fp64 [n] = the fp64 distance of the
 *                            (k - 1)-th other member (0 when k = 1); d_ids int32 [n x k] (may be NULL) = the set, i first,
 *                            the rest unordered. */
int32_t sb2_scrublet_pair_sums(sb2_ctx* ctx, int64_t n_obs, const int64_t* d_indptr, const int32_t* d_indices,
                               const float* d_data, int64_t n_sim, const int64_t* d_pairs, int64_t* d_out_indptr,
                               int32_t* d_out_indices, float* d_out_data);
int32_t sb2_knn_label_count_f32(sb2_ctx* ctx, int64_t n_points, int32_t d, const float* d_x, int64_t n_first,
                                int32_t k, int32_t* d_count, double* d_kth, int32_t* d_ids);

/* ---- extreme eigenpairs of diag(s) A diag(s), A symmetric fp32 CSR (csrc/eigs.cu: thick-restart Lanczos, fp64) ----
 * Replaces `scipy.sparse.linalg.eigsh(matrix.astype(float64), k=n_comps, which='LM', v0=...)` in
 * Neighbors.compute_eigen (src/scanpy/neighbors/__init__.py:832-884; sc.tl.diffmap) and the eigsh of umap's spectral
 * initialisation (sc.tl.umap).  d_scale may be NULL (s = 1).  which: 0 largest algebraic, 1 largest magnitude, 2 smallest
 * algebraic.  ncv <= 0 / tol <= 0 / max_restarts <= 0 pick defaults (max(2 nev + 16, 40), 1e-10, 400).  h_evals ascending
 * like eigsh; d_evecs fp64 [nev x n], row e = unit eigenvector of h_evals[e] (sign arbitrary, as with ARPACK).
 * A converged set is locked and searched again from a fresh start vector for copies of its eigenvalues that the start
 * vector missed.  info: n_converged = returned pairs whose residual estimate |beta_m y_m| is <= tol * max|theta|;
 * max_residual = the largest such estimate over the returned pairs, taken in the cycle that locked each pair. */
typedef struct sb2_eigs_info {
  int32_t restarts, matvecs, n_converged, reserved;
  double max_residual;
} sb2_eigs_info;
int32_t sb2_eigsh_csr_scaled(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                             const float* d_weights, const double* d_scale, int32_t nev, int32_t which, int32_t ncv,
                             double tol, int32_t max_restarts, const double* d_v0, double* h_evals, double* d_evecs,
                             sb2_eigs_info* info);
/* d_scale fp64[n] with T_sym = diag(d_scale) W diag(d_scale): the symmetrised transition matrix of
 * Neighbors.compute_transitions (src/scanpy/neighbors/__init__.py:791-830; density_normalize as there). */
int32_t sb2_transition_scale_f64(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                 const float* d_weights, int32_t density_normalize, double* d_scale);

/* ---- sc.tl.umap layout (SURVEY.md 8f row f1; csrc/umap.cu) ----
 * Replaces `umap.umap_.simplicial_set_embedding` as called at src/scanpy/tools/_umap.py:196-215.
 * sb2_umap_spectral_init_f32: init='spectral' (eigenvectors 2..dim+1 of D^-1/2 A D^-1/2, expanded to max|x| = 10, N(0,1e-4)
 *   jitter) into d_init fp32 [n x dim].
 * sb2_umap_layout_f32: d_embedding fp32 [n x dim] holds the initialisation on entry (rescaled to [0,10]^dim first, like the
 *   reference) and the optimised layout on return; graph = symmetric connectivities CSR (not modified); a, b from
 *   find_ab_params(spread, min_dist); deterministic in (graph, init, seed). */
int32_t sb2_umap_spectral_init_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                                   const float* d_weights, int32_t dim, uint64_t seed, float* d_init);
int32_t sb2_umap_layout_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices, const float* d_weights,
                            int32_t dim, int32_t n_epochs, double a, double b, double gamma, double initial_alpha,
                            int32_t negative_sample_rate, uint64_t seed, float* d_embedding);

/* ---- sc.tl.paga aggregation (SURVEY.md 8f row f3): d_counts int64 [G x G], counts[gi*G + gj] = stored arcs i -> j with
 * d_group[i] = gi, d_group[j] = gj.  Replaces igraph's VertexClustering.cluster_graph / subgraph(i).ecount() at
 * src/scanpy/tools/_paga.py:177-208 (inner-cluster edge counts are the diagonal). */
int32_t sb2_group_arc_counts(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices,
                             const int32_t* d_group, int32_t n_groups, int64_t* d_counts);

/* ---- sc.pp.scale (SURVEY.md 8f row f2 tail; src/scanpy/preprocessing/_scale.py:150-296) ----
 * sb2_csr_col_stats_rows_f32 <- mean_var(x[mask_obs, :], axis=0, correction=1): per-gene sum / sum of squares (fp64) over
 *                               the rows with d_mask[row] != 0 (d_mask == NULL: every row)
 * sb2_csr_scale_cols_f32     <- numba `scale_and_clip_csr` (:267-283): data[j] = min(max_value, data[j] / std[col]) on the
 *                               masked rows, in place (zero_center=False keeps the matrix sparse)
 * sb2_csr_scale_dense_f64    <- `x -= mean; x /= std; clip` on a CSR (:203-222): the dense float64 [n x g] result; rows
 *                               outside d_mask keep their values
 * sb2_dense_col_stats / sb2_dense_scale <- the same two steps for a dense float32 (is_f64 = 0) / float64 [n x g] input,
 *                               in place; d_mean == NULL means zero_center=False (then only the upper clip applies) */
int32_t sb2_csr_col_stats_rows_f32(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                                   const float* d_data, const uint8_t* d_mask, double* d_sum, double* d_sumsq);
int32_t sb2_csr_scale_cols_f32(sb2_ctx* ctx, int64_t n, const int64_t* d_indptr, const int32_t* d_indices, float* d_data,
                               const double* d_std, const uint8_t* d_mask, int32_t has_max, double max_value);
int32_t sb2_csr_scale_dense_f64(sb2_ctx* ctx, int64_t n, int32_t g, const int64_t* d_indptr, const int32_t* d_indices,
                                const float* d_data, const double* d_mean, const double* d_std, const uint8_t* d_mask,
                                int32_t has_max, double max_value, double* d_out);
int32_t sb2_dense_col_stats(sb2_ctx* ctx, int64_t n, int32_t g, const void* d_x, int32_t is_f64, const uint8_t* d_mask,
                            double* d_sum, double* d_sumsq);
int32_t sb2_dense_scale(sb2_ctx* ctx, int64_t n, int32_t g, void* d_x, int32_t is_f64, const double* d_mean,
                        const double* d_std, const uint8_t* d_mask, int32_t has_max, double max_value);

/* ---- sc.pp.harmony_integrate (src/scanpy/preprocessing/_harmony/core.py; csrc/harmony.cu) ----
 * Z, R, X and the outputs are row-major [n x d] / [n x k], float32 (is_f64 = 0) or float64; d_y, d_pen, d_w and every
 * sum are fp64.  d_codes [n x keys] int32 holds each cell's marginal code per key, in [0, n_codes).  A cell list d_idx
 * (int64, NULL: the identity) names the rows a call works on.  Sums have no floating-point atomics: per-CTA partials
 * fold in CTA order, and the CTA split depends only on the shapes, so equal inputs give equal bits.
 * sb2_harmony_normalize <- _normalize_rows_l2: d_out[i] = d_x[i] / max(||d_x[i]||, 1e-12).
 * sb2_harmony_wsums     <- d_out[g][c][j] = Σ_{rows of group g} w(i, c) * [z_i | 1][j], fp64 [groups x k x (d+1)].  The
 *                          call's rows are d_idx[0 .. h_bounds[groups]) (row i = d_idx[p]), group g owning positions
 *                          h_bounds[g] .. h_bounds[g+1] (host array).  w: d_r[i][c] (mode 0), 1 where d_labels[i] == c
 *                          (mode 1, float64 Z only), or 1 with k = 1 (mode 2).
 * sb2_harmony_step      <- one block of the clustering: for each listed cell, log r = term (1 - z·y_c) + Σ_keys
 *                          d_pen[code][c] (d_pen NULL: no penalty), minus its max, exp, divided by max(Σ, 1e-12), stored
 *                          to d_r; d_ent[i] = Σ_c r̂ log(r̂ + 1e-12) with r̂ = r / max(Σ r, 1e-12).
 * sb2_harmony_code_sums <- d_out fp64 [(n_codes + 1) x k]: row b the sum of d_r over the listed cells with code b for
 *                          any key, row n_codes the sum over all listed cells.
 * sb2_harmony_oe_update <- o += sign * sums[b], e += sign * pr_b[b] * sums[n_codes], then d_pen[b][c] = theta[b] *
 *                          (log(e + 1) - log(o + e + 1)) (stabilized) or theta[b] * (log(e + 1) - log(o + 1)).
 * sb2_harmony_sum       <- *d_out = Σ d_v[0 .. n).
 * sb2_harmony_center / sb2_harmony_kpp_search / sb2_harmony_kpp_dists / sb2_harmony_labels <- sklearn's KMeans on
 *                          the rows of Z: d_xc = z - d_mean and d_xx = ||d_xc||²; for each uniform d_u[t], the first i
 *                          with cumsum(d_v)[i] >= d_u[t] (n - 1 if none); for each candidate row d_ids[t],
 *                          d_dist[t][i] = min(d_closest[i], max(-2 xc_i·xc_c + ||xc_c||² + xx_i, 0)) (d_closest NULL: no
 *                          min) and d_pot[t] = Σ_i d_dist[t][i]; d_labels[i] = argmin_c ||c||² - 2 xc_i·c (first),
 *                          *d_changed = 1 if any label differs from d_old.
 * sb2_harmony_apply     <- the correction: for each group g of rows (as in wsums) with code tuple d_gcodes[g] [keys],
 *                          z_i = x_i - Σ_c r_ic Σ_keys d_w[c][code + 1] (d_w fp64 [k x (n_codes + 1) x d]) to d_zhat,
 *                          and z_i / max(||z_i||, 1e-12) to d_znorm. */
#define SB2_HARMONY_MAX_K 128
#define SB2_HARMONY_MAX_D 128
#define SB2_HARMONY_MAX_CODES 128
#define SB2_HARMONY_MAX_TUPLES 65536
#define SB2_HARMONY_MAX_TRIALS 8
int32_t sb2_harmony_normalize(sb2_ctx* ctx, int64_t n, int32_t d, int32_t is_f64, const void* d_x, void* d_out);
int32_t sb2_harmony_wsums(sb2_ctx* ctx, int32_t groups, const int64_t* h_bounds, const int64_t* d_idx, int32_t d,
                          int32_t k, int32_t is_f64, const void* d_z, int32_t mode, const void* d_r,
                          const int32_t* d_labels, double* d_out);
int32_t sb2_harmony_step(sb2_ctx* ctx, int64_t rows, const int64_t* d_idx, int32_t d, int32_t k, int32_t is_f64,
                         const void* d_z, const double* d_y, int32_t keys, const int32_t* d_codes, const double* d_pen,
                         double term, void* d_r, double* d_ent);
int32_t sb2_harmony_code_sums(sb2_ctx* ctx, int64_t rows, const int64_t* d_idx, int32_t k, int32_t is_f64,
                              const void* d_r, int32_t keys, const int32_t* d_codes, int32_t n_codes, double* d_out);
int32_t sb2_harmony_oe_update(sb2_ctx* ctx, int32_t n_codes, int32_t k, double sign, const double* d_sums,
                              const double* d_pr_b, const double* d_theta, int32_t stabilized, double* d_o, double* d_e,
                              double* d_pen);
int32_t sb2_harmony_sum(sb2_ctx* ctx, int64_t n, const double* d_v, double* d_out);
int32_t sb2_harmony_center(sb2_ctx* ctx, int64_t n, int32_t d, int32_t is_f64, const void* d_z, const double* d_mean,
                           double* d_xc, double* d_xx);
int32_t sb2_harmony_kpp_search(sb2_ctx* ctx, int64_t n, const double* d_v, int32_t trials, const double* d_u,
                               int64_t* d_ids);
int32_t sb2_harmony_kpp_dists(sb2_ctx* ctx, int64_t n, int32_t d, const double* d_xc, const double* d_xx,
                              int32_t trials, const int64_t* d_ids, const double* d_closest, double* d_dist,
                              double* d_pot);
int32_t sb2_harmony_labels(sb2_ctx* ctx, int64_t n, int32_t d, int32_t k, const double* d_xc, const double* d_centers,
                           const int32_t* d_old, int32_t* d_labels, int32_t* d_changed);
int32_t sb2_harmony_apply(sb2_ctx* ctx, int32_t groups, const int64_t* h_bounds, const int64_t* d_idx, int32_t d,
                          int32_t k, int32_t is_f64, int32_t keys, const int32_t* d_gcodes, int32_t n_codes,
                          const double* d_w, const void* d_x, const void* d_r, void* d_zhat, void* d_znorm);

#ifdef __cplusplus
}
#endif
#endif /* SCANPY_B200_H */
