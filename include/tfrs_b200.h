/*
 * tfrs_b200.h -- C ABI of libtfrs_b200.so: the H100 (sm_90a) kernels behind the TensorFlow
 * Recommenders retrieval / ranking hot path.
 *
 * The reference (tensorflow/recommenders v0.7.7) has no native/FFI layer: its boundary with native
 * code is "call public tf.* ops" from Python.  Each entry point below therefore replaces one TF op
 * call site of the reference (cited per function, paths relative to tensorflow_recommenders/).
 * The Python mirror of the reference API (recommenders_b200/) is the only intended caller and binds
 * these symbols with ctypes (see INTEGRATION.md for the binding a maintainer would add).
 *
 * Conventions
 *  - Every function returns 0 on success or a negative TFRS_ERR_* code; tfrs_last_error() returns a
 *    thread-local message.  No C++ exception or abort crosses the boundary.
 *  - All data pointers are DEVICE pointers owned by the caller (e.g. torch storage .data_ptr());
 *    the library never frees or retains them past the call.  Pointer ARRAYS (tables / ids lists)
 *    are HOST arrays of device pointers.
 *  - No hidden allocation: scratch memory is caller-provided, its size comes from *_workspace_bytes().
 *  - Every call is asynchronous on `stream` (a cudaStream_t passed as void*; NULL = default stream).
 *    No implicit synchronisation; calls are CUDA-graph capturable.
 *  - Matrices are row-major fp32 unless stated otherwise.
 */
#ifndef TFRS_B200_H_
#define TFRS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFRS_B200_VERSION 102 /* 0.1.2 */

enum {
  TFRS_OK = 0,
  TFRS_ERR_INVALID_ARG = -1,
  TFRS_ERR_UNSUPPORTED = -2,
  TFRS_ERR_CUDA = -3,
  TFRS_ERR_WORKSPACE_TOO_SMALL = -4,
  TFRS_ERR_NCCL = -5
};

enum { TFRS_I32 = 0, TFRS_I64 = 1 };

int tfrs_version(void);
const char* tfrs_last_error(void);
/* Number of kernels this library has launched in the calling process (bench.py's gpu_launches). */
int64_t tfrs_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * K1  embedding gather.  Replaces tf.keras.layers.Embedding -> tf.gather in the user towers
 * (README.md:62-66,77-78; experimental/layers/embedding/partial_tpu_embedding.py:81-85,127).
 *   out[i, out_col_off[t] .. +dims[t]) = tables[t][ids[t][i], :]     for t < n_tables, i < n
 * Writes straight into a concatenated [n, out_ld] activation (the layout Cross consumes).
 * Out-of-range ids produce zero rows.  dims[t] % 4 == 0 and 16-byte aligned rows take the
 * vectorised path; anything else a scalar path.  n == 0 writes nothing (out and ids may be NULL).
 * ------------------------------------------------------------------------------------------- */
int tfrs_gather_f32(const float* const* tables, const int64_t* rows, const int32_t* dims, int n_tables,
                    const void* const* ids, int ids_dtype, int64_t n, float* out, int64_t out_ld,
                    const int32_t* out_col_off, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K2  brute-force top-K scan.  Replaces  scores = matmul(q, c^T); top_k(scores, k)
 * (layers/factorized_top_k.py:603-605 BruteForce.call; :424-438,:440-472 Streaming.call).
 * Scores are the canonical sequential fmaf chain over k = 0..d-1; order = (score desc, index asc).
 * `state_*` (nullable, state_k entries per query) is Streaming's carried state; it takes part in
 * the selection with its own indices.  New candidates get index = index_offset + row (shard /
 * chunk offset).  Output: min(k, state_k + N) entries per query, written with row stride k.
 * k <= 2048.
 *
 * tfrs_topk_scan_f32      exact fp32 CUDA-core path (any N, d; used for small corpora/chunks).
 * tfrs_index_*            builds the tensor-core screening image of a corpus (fp16 after an exact
 *                         power-of-two rescale, GMMA SWIZZLE_128B K-major tiles + row-norm bound);
 *                         done once at index() time (BruteForce.index, factorized_top_k.py:540-584).
 * tfrs_topk_tc_f32        wgmma screening GEMM (fp16 in / fp32 accumulate in registers) with a fused
 *                         threshold filter, then exact fp32 rescoring of the survivors -- same
 *                         bit-exact result as tfrs_topk_scan_f32.  Needs d <= 128, k <= 256 and a
 *                         corpus of at least ~256*k rows (tfrs_topk_tc_workspace_bytes returns 0
 *                         outside the supported range; callers then use tfrs_topk_scan_f32).
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_topk_scan_workspace_bytes(int64_t Q, int64_t N, int d, int k);
int tfrs_topk_scan_f32(const float* q, int64_t Q, const float* corpus, int64_t N, int d, int k,
                       int64_t index_offset, const float* state_scores, const int64_t* state_idx,
                       int state_k, float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes,
                       void* stream);

size_t tfrs_index_bytes(int64_t N, int d);
int tfrs_index_build(const float* corpus, int64_t N, int d, void* index_buf, size_t index_bytes,
                     void* stream);
size_t tfrs_topk_tc_workspace_bytes(int64_t Q, int64_t N, int d, int k);
int tfrs_topk_tc_f32(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N,
                     int d, int k, int64_t index_offset, float* out_scores, int64_t* out_idx, void* ws,
                     size_t ws_bytes, void* stream);

/* The same tensor-core scan with `query_with_exclusions` fused into the finalize step (layers/factorized_top_k.py
 * :242-288 + `_exclude` :83-115): the k + n_excl best candidates are selected as above, candidates whose identifier
 * (identifiers[global index], or the global index itself when identifiers == NULL) appears in exclusions[q, :] get
 * score - 1e5, the k best ADJUSTED scores win (ties -> better original position) and the ORIGINAL scores / global
 * indices are written -- bit-for-bit what the reference computes from its over-fetched list.  int64 ids.
 * Workspace: tfrs_topk_tc_workspace_bytes(Q, N, d, k + n_excl). */
int tfrs_topk_tc_exclude_f32(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N, int d,
                             int k, int64_t index_offset, const int64_t* identifiers, const int64_t* exclusions,
                             int n_excl, float* out_scores, int64_t* out_idx, void* ws, size_t ws_bytes, void* stream);

/* The score branch of FactorizedTopK.update_state (metrics/factorized_top_k.py:133-137,181-192) without a top-K
 * list: out_count[q] = min(k, #{candidates whose exact score is > positive_scores[q]}); the metric for any k' <= k is
 * then  count < k'  (tf.math.in_top_k: fewer than k' predictions strictly above the target).  Same screening +
 * exact-rescoring guarantees as tfrs_topk_tc_f32 (only candidates within the error band of the positive are
 * re-scored).  Workspace: tfrs_topk_tc_workspace_bytes(Q, N, d, k). */
int tfrs_topk_tc_count_f32(const float* q, int64_t Q, const float* corpus, const void* index_buf, int64_t N, int d,
                           int k, const float* positive_scores, int32_t* out_count, void* ws, size_t ws_bytes,
                           void* stream);

/* `_exclude` (layers/factorized_top_k.py:83-115) on an already fetched, sorted [Q, k_fetched] list (Streaming and
 * the exact CUDA-core path): same rule as tfrs_topk_tc_exclude_f32.  idx are global indices into `identifiers`. */
int tfrs_topk_exclude_rerank_f32(const float* scores, const int64_t* idx, int64_t Q, int k_fetched,
                                 const int64_t* identifiers, const int64_t* exclusions, int n_excl, int k_out,
                                 float* out_scores, int64_t* out_idx, void* stream);

/* out_count[q] = #{t < k : scores[q*ld + t] > positive_scores[q]} -- the in_top_k count on a retrieved list. */
int tfrs_count_above_f32(const float* scores, int64_t ld, int k, const float* positive_scores, int64_t Q,
                         int32_t* out_count, void* stream);

/* Device-resident running sums of FactorizedTopK's Mean metrics (metrics/factorized_top_k.py:186-192):
 *   acc[j] += sum_q w_q * [count_q < ks[j] && isfinite(positive_q)]  (j < n_ks);   acc[n_ks] += sum_q w_q
 * (w = 1 when sample_weight == NULL).  `ks` is a HOST array (n_ks <= 16), `acc` n_ks + 1 doubles on the device.
 * Fixed-order fp64 reduction: deterministic; the host reads acc once, in result(). */
int tfrs_topk_hits_accumulate(const int32_t* count, const float* positive_scores, const float* sample_weight, int64_t Q,
                              const int32_t* ks, int n_ks, double* acc, void* stream);

/* Test/debug introspection of tfrs_topk_tc_f32's workspace: out10 = {count offset, fallback-flag offset,
 * threshold offset, survivor-list offset, parts, cap_part, padded Q, cut offset, bins of the sampled pass,
 * row-exponent offset} (byte offsets from the 16-byte-aligned workspace base).  Lets the tests assert which rows
 * took the exact fallback and which selection / threshold branch a call ran. */
int tfrs_topk_tc_layout(int64_t Q, int64_t N, int d, int k, int64_t* out10);

/* The same workspace's two-threshold state: out4 = {guaranteed-threshold offset (float [padded Q], the k-th bin bound
 * thr_safe), retry-mark offset (uint32 [padded Q], 1 = the row missed at its raised filter threshold and was filtered
 * again at thr_safe), bin rank K' of the filter threshold of a top-K / exclusion call, sample stride}.  The threshold
 * at the tfrs_topk_tc_layout offset is the one whose records the workspace holds: thr_safe for a retried row. */
int tfrs_topk_tc_retry_layout(int64_t Q, int64_t N, int d, int k, int64_t* out4);

/* The sampled pass on a norm-sample index (tfrs_index_build takes the floor(N/8) rows of largest norm as the sample
 * when N >= 2^19 and the norm spread predicts a tighter bound): out8 = {bin-maxima offset (float [padded Q, bins_ld]),
 * bins_ld, bins, tiles per bin, bins per corpus part and column half, corpus parts, sample tiles, margin offset
 * (float [padded Q])}.  Bins = 0: the shape has no norm-sample layout. */
int tfrs_topk_tc_sample_layout(int64_t Q, int64_t N, int d, int k, int64_t* out8);

/* Optional per-stage device timing of tfrs_topk_tc_f32 (CUDA events on the launch stream; used by
 * bench.py for the roofline figure).  tfrs_profile_read synchronises the device and returns the summed
 * times in ms of stage 0 = query image, 1 = sampled pass + threshold, 2 = full filter pass (the
 * dominant kernel), 3 = exact re-scoring (+ fallback), over `calls` recorded calls. */
int tfrs_profile_enable(int on);
int tfrs_profile_read(float* stage_ms, int* calls);

/* K2m  merge n_lists per-shard/per-chunk [Q, k_in] lists into the best k_out = min(k_out, n_lists*k_in) per query
 * (Streaming reduce :440-472; shard merge after the all-gather).  Order = (score desc, index asc).  The lists sit
 * `list_stride_*` elements apart: Q*k_in for a list-major [n_lists, Q, k_in] array, more in the receive buffer of the
 * single all-gather, where every rank's block is [scores | indices]. */
int tfrs_topk_merge_strided(const float* scores, const int64_t* idx, int64_t list_stride_scores,
                            int64_t list_stride_idx, int n_lists, int64_t Q, int k_in, int k_out,
                            float* out_scores, int64_t* out_idx, void* stream);

/* The same merge when every input list is already sorted in the total order (score desc, index asc) -- which is
 * what tfrs_topk_scan_f32 / tfrs_topk_tc_f32 emit, i.e. the per-shard lists of the sharded BruteForce: merged rank
 * = own position + binary-search counts in the other lists; no sort.  n_lists * k_in <= 16384. */
int tfrs_topk_merge_sorted_strided(const float* scores, const int64_t* idx, int64_t list_stride_scores,
                                   int64_t list_stride_idx, int n_lists, int64_t Q, int k_in, int k_out,
                                   float* out_scores, int64_t* out_idx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K26  multi-interest (maxsim) retrieval: a query is H >= 1 vectors q_h and scores candidate c by
 * m(q, c) = max_h s_h(c), s_h = the canonical fmaf chain of q_h . c (tasks/retrieval.py:172-176).  Heads that tie on the
 * maximum (+0 and -0 tie) report the lowest head's bits.  Order = (m desc, index asc).
 *
 * tfrs_topk_maxsim_merge_f32  scores / idx = [Q, H, w]: per query the H per-head top-w lists, each sorted by (score desc,
 *                             index asc) with distinct indices -- what the scans emit for the Q*H head rows with k = w.
 *                             Keeps each candidate's best entry (highest score, then lowest head) and writes the first
 *                             k_out (1 <= k_out <= w) kept entries in order to out_* [Q, k_out].  With w = min(k, N) the
 *                             result is the exact maxsim top-min(k, N) (DESIGN.md, K26).  H * w <=
 *                             TFRS_MAXSIM_MAX_ENTRIES, TFRS_ERR_UNSUPPORTED above.  No workspace; deterministic.
 * tfrs_rowwise_maxsim_f32     out[r] = max_h dot(q[r, h, :], c[r, :]) for q [rows, H, d], c [rows, d]: FactorizedTopK's
 *                             positive score for multi-head queries, each head by tfrs_rowwise_dot_f32's chain.
 * ------------------------------------------------------------------------------------------- */
#define TFRS_MAXSIM_MAX_ENTRIES 8192
int tfrs_topk_maxsim_merge_f32(const float* scores, const int64_t* idx, int64_t Q, int H, int w, int k_out,
                               float* out_scores, int64_t* out_idx, void* stream);
int tfrs_rowwise_maxsim_f32(const float* q, const float* c, int64_t rows, int H, int d, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K14  exact top-K with overridden rows, and its hit count: the device side of examples.movielens.evaluate
 * (examples/movielens.py:71-88, `scores[train_movies] = -1e6; top_movies = argsort(-scores)[:k]`).  Query u lists the
 * rows rows[offsets[u] .. offsets[u+1]) (CSR, int64, sorted and unique per query, in [0, N)); those rows score exactly
 * -1e6f instead of their canonical dot.  Order = (score desc, row asc); k_out = min(k, N) entries per query.
 * `users` (nullable = 0 .. n-1) maps position j of a call to query users[j]: its row of q, its list and its output row
 * (out_* rows are out_ld apart).  Both routes give the same bits.
 *
 * tfrs_topk_override_merge_f32   scan route: list_* = [n, w] the top w of each query by canonical score (what
 *                                tfrs_topk_scan_f32 / tfrs_topk_tc_f32 emit) with w >= min(N, k + list length) and
 *                                k_out <= w <= 256.  Drops the listed rows, merges the first k survivors with the listed
 *                                rows at -1e6, writes k_out.  No workspace.
 * tfrs_topk_overriding_dense_f32 dense route, any list length, k <= 2048: chunks of queries are scored into the workspace
 *                                ([chunk, N] fp32 plus the chunk's query rows and selections), the listed entries are
 *                                overwritten and the rows selected.  The chunk is the largest the given workspace holds;
 *                                tfrs_topk_overriding_dense_workspace_bytes sizes one of at most 256 MB.
 * tfrs_count_listed              out_count[u] = #{t in [offsets[u], offsets[u+1]) : rows[t] is among top_rows[u, 0..kk)}
 *                                (entries counted with multiplicity; rows need not be sorted here).  kk <= 2048.
 * ------------------------------------------------------------------------------------------- */
int tfrs_topk_override_merge_f32(const float* list_scores, const int64_t* list_idx, int64_t n, int w, const int64_t* users,
                                 const int64_t* offsets, const int64_t* rows, int k, int k_out, float* out_scores,
                                 int64_t* out_idx, int out_ld, void* stream);
size_t tfrs_topk_overriding_dense_workspace_bytes(int64_t n, int64_t N, int d, int k);
int tfrs_topk_overriding_dense_f32(const float* q, const int64_t* users, int64_t n, const float* corpus, int64_t N, int d,
                                   int k, const int64_t* offsets, const int64_t* rows, float* out_scores, int64_t* out_idx,
                                   int out_ld, void* ws, size_t ws_bytes, void* stream);
int tfrs_count_listed(const int64_t* top_rows, int64_t Q, int kk, int64_t ld, const int64_t* offsets, const int64_t* rows,
                      int32_t* out_count, void* stream);

/* ---------------------------------------------------------------------------------------------
 * C1  the collective of the row-sharded scan (SURVEY 8b/8e; the reference has no sharded scan -- its corpus is one
 * variable, layers/factorized_top_k.py:571-580 -- and its only collective helper is tasks/retrieval.py:238-321).
 * One process per GPU; shard g owns a contiguous row block, so global index order == (shard, local index) order and
 * the lowest-index tie rule survives the merge.  NCCL is bound at run time (dlopen libnccl.so.2: the copy the host
 * framework already loaded, else the system one; TFRS_NCCL_LIB overrides), so binders need only this header.
 *
 *   tfrs_comm_unique_id   rank 0 creates the 128-byte NCCL id; the host framework broadcasts it by any means
 *   tfrs_comm_create      collective over the group (ncclCommInitRank on the CURRENT device); tfrs_comm_destroy frees it
 *   tfrs_topk_allgather   every rank's [Q,k] (scores, global indices) -> all_s/all_i [world, Q, k] in rank order
 *   tfrs_topk_sharded_f32 the whole sharded BruteForce.call in one entry point: local scan (tensor-core path when
 *                         `index_buf` is given and the shape allows it, exact scan otherwise; shards shorter than k
 *                         are padded with (-inf, INT64_MAX)) written straight into the send block -> ONE all-gather
 *                         of the packed blocks -> sorted-list merge on every rank.  Every rank returns the same
 *                         [Q,k] result.  All ranks must call it with the same Q, d, k.
 * Handles need external locking; calls are asynchronous on `stream`.
 * ------------------------------------------------------------------------------------------- */
typedef struct tfrs_comm* tfrs_comm_t;
int tfrs_comm_unique_id(void* out128);
int tfrs_comm_create(tfrs_comm_t* comm, int rank, int world, const void* unique_id128);
int tfrs_comm_destroy(tfrs_comm_t comm);
/* Optional: map every rank's exchange buffer into every peer (cudaIpc over NVLink / NVSwitch), sized for calls up to
 * (max_Q, max_k).  Collective; synchronises the device.  With it tfrs_topk_sharded_f32 replaces the NCCL all-gather +
 * replicated merge by its own kernels: every rank STORES the slice of its lists owned by rank o straight into o's buffer
 * (owner = contiguous block of ceil(Q / world) queries), owners merge only their block and store the result into every
 * rank's result area, epoch flags order the steps -- 1/world of the all-gather's NVLink traffic and of the merge work.
 * Returns TFRS_ERR_UNSUPPORTED on EVERY rank when any peer mapping fails (the NCCL path stays in use).
 * tfrs_comm_p2p_capacity: 1 when the mapped buffers hold a (Q, k) call. */
int tfrs_comm_enable_p2p(tfrs_comm_t comm, int64_t max_Q, int max_k);
int tfrs_comm_p2p_capacity(tfrs_comm_t comm, int64_t Q, int k);
/* option 0: exchange a GLOBAL lower bound of the k-th best score between the threshold kernel and the filter pass of the
 * peer-memory path (default 1): each shard then keeps ~1/world of the survivors, so the per-rank select / re-score work
 * shrinks with the shard.  Must be set identically on every rank. */
int tfrs_comm_set_option(tfrs_comm_t comm, int option, int value);
int tfrs_comm_rank(tfrs_comm_t comm);
int tfrs_comm_world(tfrs_comm_t comm);
int tfrs_topk_allgather(tfrs_comm_t comm, const float* s, const int64_t* i, int64_t Q, int k, float* all_s,
                        int64_t* all_i, void* stream);
size_t tfrs_topk_sharded_workspace_bytes(int world, int64_t Q, int64_t N_local, int d, int k);
/* test introspection: out4 = {index byte offset inside a block, block bytes, send-block offset, receive-buffer offset} */
int tfrs_topk_sharded_layout(int world, int64_t Q, int64_t N_local, int d, int k, int64_t* out4);
int tfrs_topk_sharded_f32(tfrs_comm_t comm, const float* q, int64_t Q, const float* corpus_local, const void* index_buf,
                          int64_t N_local, int d, int k, int64_t index_offset, float* out_scores, int64_t* out_idx,
                          void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Score helpers (exact fp32, canonical fmaf chain, one owner thread per output).
 * tfrs_sgemm_f32: C[M,N] (+)= opA(A) . opB(B); opA(m,k) = transA ? A[k*lda+m] : A[m*lda+k],
 *   opB(k,n) = transB ? B[n*ldb+k] : B[k*ldb+n].  transA=0, transB=1 is `_compute_score`
 *   = matmul(q, c^T) (layers/factorized_top_k.py:320-333; tasks/retrieval.py:178-180); the other
 *   modes serve its backward and the low-rank Cross (dcn.py:131-148,178-179).
 * tfrs_rowwise_dot_f32: out[i] = sum_k a[i,k]*b[i,k]  (positive scores,
 *   metrics/factorized_top_k.py:133-134).
 * ------------------------------------------------------------------------------------------- */
int tfrs_sgemm_f32(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda,
                   const float* B, int64_t ldb, float* C, int64_t ldc, int accumulate, void* stream);
int tfrs_rowwise_dot_f32(const float* a, const float* b, int64_t rows, int d, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K3  in-batch softmax loss of tfrs.tasks.Retrieval (tasks/retrieval.py:178-185,187-188,210):
 *   s = (q . c^T) * inv_temperature ; loss = sum_i w_i * (logsumexp_j s_ij - s_ii)
 * C >= B (extra negatives, positives are the first B rows).  `lse` [B] is saved for backward.
 * Backward (tape.gradient at models/base.py:77): G = (softmax(s) - I) * w * grad_loss * inv_temperature,
 *   dq = G . c   [B,d] ;  dc = G^T . q   [C,d].
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_inbatch_softmax_workspace_bytes(int64_t B, int64_t C, int d);
int tfrs_inbatch_softmax_fwd(const float* q, const float* c, int64_t B, int64_t C, int d,
                             float inv_temperature, const float* sample_weight, float* loss, float* lse,
                             void* ws, size_t ws_bytes, void* stream);
int tfrs_inbatch_softmax_bwd(const float* q, const float* c, int64_t B, int64_t C, int d,
                             float inv_temperature, const float* sample_weight, const float* lse,
                             const float* grad_loss, float* dq, float* dc, void* ws, size_t ws_bytes,
                             void* stream);

/* K3 on the tensor cores, forward (same contract and outputs as tfrs_inbatch_softmax_fwd; d <= 128) and backward (same as
 * tfrs_inbatch_softmax_bwd; d <= 64).
 *   forward:  hi/lo fp16 split of q and c (|err| <= 2^-21 |q||c| on a score), wgmma GEMM with fp32 register accumulation
 *             and an online log-sum-exp epilogue -- the [B,C] logits are never written.
 *   backward: two launches of one flash-attention-backward-shaped kernel -- S = X.Y^T (wgmma, split fp16 operands), G built
 *             on the register fragment of S, dX += G.Y with G as the register A operand of the next wgmma and the Y tile as
 *             an MN-major operand; X = q gives dq, X = c gives dc.  Deterministic (no atomics).
 * The tfrs.tasks.Retrieval loss options (SURVEY 8f-3), each nullable:
 *   candidate_bias (float [C])       added to every logit of its column after the temperature: with
 *                                    bias_j = -log(clip(p_j, 1e-6, 1)) it is the sampling-probability correction of
 *                                    tasks/retrieval.py:190-192 / layers/loss.py:150-158
 *   candidate_ids  (int64 [C])       remove_accidental_hits: every candidate j != i whose id equals the id of query i's
 *                                    positive (candidate i) gets logit MIN_FLOAT (tasks/retrieval.py:194-200,
 *                                    layers/loss.py:114-147; `logits + dup * MIN_FLOAT` rounds to MIN_FLOAT in fp32)
 *   score_mask     (uint8 [B, C])    where(mask, s, MIN_FLOAT) (retrieval.py:202-203); row-major, nonzero = keep
 * ids and mask are applied after the temperature and the bias, in the reference's order.  The ids / keep-bits are tested against the fp32 accumulators in
 * registers: no [B,C] logits, labels or masks are materialised (the byte mask is packed to bits once).  Masked entries get
 * zero gradient.  *_workspace_bytes sizes `ws` for the options given (has_ids = candidate_ids != NULL, has_mask =
 * score_mask != NULL); it returns 0, and the call TFRS_ERR_UNSUPPORTED, outside the shape range; the caller then uses
 * tfrs_inbatch_softmax_fwd / _bwd. */
size_t tfrs_inbatch_softmax_tc_workspace_bytes(int64_t B, int64_t C, int d, int has_ids, int has_mask);
int tfrs_inbatch_softmax_tc_fwd(const float* q, const float* c, int64_t B, int64_t C, int d, float inv_temperature,
                                const float* sample_weight, const float* candidate_bias, const int64_t* candidate_ids,
                                const uint8_t* score_mask, float* loss, float* lse, void* ws, size_t ws_bytes, void* stream);
size_t tfrs_inbatch_softmax_tc_bwd_workspace_bytes(int64_t B, int64_t C, int d, int has_ids, int has_mask);
int tfrs_inbatch_softmax_tc_bwd(const float* q, const float* c, int64_t B, int64_t C, int d, float inv_temperature,
                                const float* sample_weight, const float* candidate_bias, const int64_t* candidate_ids,
                                const uint8_t* score_mask, const float* lse, const float* grad_loss, float* dq, float* dc,
                                void* ws, size_t ws_bytes, void* stream);

/* Multi-head queries (tasks/retrieval.py:172-176): q is [B,H,d] and  scores_ij = max_h q_ih . c_j  ("maxsim") before the same
 * loss.  Exact fp32 path: row blocks of the [B*H, C] head scores stay L2-resident, the head maximum is folded while the
 * row statistics are taken; nothing of size [B,C] reaches the caller.  The gradient goes to the head(s) attaining the maximum
 * (split evenly among exact ties, as tf.reduce_max's).  dq is [B,H,d]. */
size_t tfrs_inbatch_softmax_maxsim_workspace_bytes(int64_t B, int H, int64_t C, int d);
int tfrs_inbatch_softmax_maxsim_fwd(const float* q, const float* c, int64_t B, int H, int64_t C, int d, float inv_temperature,
                                    const float* sample_weight, float* loss, float* lse, void* ws, size_t ws_bytes, void* stream);
int tfrs_inbatch_softmax_maxsim_bwd(const float* q, const float* c, int64_t B, int H, int64_t C, int d, float inv_temperature,
                                    const float* sample_weight, const float* lse, const float* grad_loss, float* dq, float* dc,
                                    void* ws, size_t ws_bytes, void* stream);

/* Hard-negative mining inside the loss (tasks/retrieval.py:205-210, layers/loss.py:61-111) without the [B,C] logits: the
 * n + 1 best candidates of every query come from the top-K scan above (k1 = min(n + 1, C) entries per query, exact fp32
 * scores, sorted); tfrs_hardneg_loss_fwd keeps the positive (candidate i of query i, score `positive_scores[i]`) plus the
 * n best other candidates and computes  loss = sum_i w_i (logsumexp(kept logits / T) - positive / T)  and the gradient
 * coefficients `coef` [B, k1 + 2] (entry t of the list, then the positive, then the row loss; w_i / T folded in).
 * tfrs_hardneg_loss_bwd:  dq_i = g sum_t coef_it c_{j_t}  (fixed order),  dc_j += g coef_it q_i  (float atomics: the only
 * non-bit-reproducible kernel of the library; dc is zeroed by the call). */
int tfrs_hardneg_loss_fwd(const float* top_scores, const int64_t* top_idx, int64_t B, int k1, const float* positive_scores,
                          float inv_temperature, const float* sample_weight, float* loss, float* coef, void* stream);
int tfrs_hardneg_loss_bwd(const float* q, const float* c, int64_t B, int64_t C, int d, const int64_t* top_idx, int k1,
                          const float* coef, const float* grad_loss, float* dq, float* dc, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K4  sparse Adagrad on the rows touched by a batch (optimizer.apply_gradients with IndexedSlices,
 * models/base.py:77-78; Adagrad chosen by the user, README.md:84).  Duplicate ids are summed in
 * order of occurrence, then  acc += g*g ; var -= lr*g / sqrt(acc+eps)   (eps_inside_sqrt != 0)
 *                       or   acc += g*g ; var -= lr*g / (sqrt(acc)+eps) (eps_inside_sqrt == 0).
 * Deterministic (sort + segmented reduction, no float atomics).  n < 2^24.
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_sparse_adagrad_workspace_bytes(int64_t n, int d);
int tfrs_sparse_adagrad_f32(float* table, float* accum, int64_t rows, int d, const void* ids, int ids_dtype,
                            int64_t n, const float* grad_rows, float lr, float eps, int eps_inside_sqrt,
                            void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K7  ClippyAdagrad (experimental/optimizers/clippy_adagrad.py:81-249): Adagrad with one clipping factor per variable.
 * Per touched element, with g the gradient (duplicate ids summed in order of occurrence, as K4), v the variable and
 * a the accumulator, every step one IEEE fp32 operation:
 *   a1 = standard ? a + g*g : a ;  p = 1 / sqrt(a1 + eps) ;  delta = (lr*g) * p
 *   m  = (abs_thr + |v|*var_rel) + p*acc_rel ;  s = delta == 0 ? 1 : m / |delta|
 *   scale = min(1, min over the variable's touched elements of s)     (NaN ratios are ignored, as fminf)
 *   v' = v - delta*scale ;  a' = standard ? a1 : a + u*u,  u = clip ? g*scale : g
 * flags: bit 0 clip_accumulator_update (clip), bit 1 use_standard_accumulator_update (standard); not both.  Thresholds
 * must be >= 0.  The factor (1 when nothing is touched) is written to the device scalar clipping_factor_out, or kept in
 * `ws` when it is NULL.  Deterministic (atomicMin on the factor's bit pattern, no float atomics on the state).
 * Sparse: one table per call, the contract of tfrs_sparse_adagrad_f32 (I32/I64 ids, out-of-range ids skipped,
 * n < 2^24, d <= 1024).
 * Dense: every variable of one optimizer in one call; vars / grads / accums / numels are HOST arrays of nvars device
 * pointers and element counts, clipping_factors_out a device array of nvars floats (or NULL: kept in `ws`).
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_sparse_clippy_adagrad_workspace_bytes(int64_t n, int d);
int tfrs_sparse_clippy_adagrad_f32(float* table, float* accum, int64_t rows, int d, const void* ids, int ids_dtype,
                                   int64_t n, const float* grad_rows, float lr, float eps, float var_rel, float acc_rel,
                                   float abs_thr, int flags, float* clipping_factor_out, void* ws, size_t ws_bytes,
                                   void* stream);
size_t tfrs_clippy_adagrad_dense_workspace_bytes(int nvars);
int tfrs_clippy_adagrad_dense_f32(float* const* vars, const float* const* grads, float* const* accums,
                                  const int64_t* numels, int nvars, float lr, float eps, float var_rel, float acc_rel,
                                  float abs_thr, int flags, float* clipping_factors_out, void* ws, size_t ws_bytes,
                                  void* stream);

/* ---------------------------------------------------------------------------------------------
 * K10  Adam with tf-keras's legacy rules (optimizer_v2/adam.py).  The caller computes, per step,
 *   alpha = lr * sqrt(1 - beta2^t) / (1 - beta1^t)   (t = the optimizer's iterations + 1)
 * and the kernels use omb1 = 1 - beta1 and omb2 = 1 - beta2 in fp32.  Every step one IEEE fp32 operation:
 *   dense (_resource_apply_dense):  m' = m + (g - m)*omb1 ;  v' = v + (g*g - v)*omb2 ;
 *                                   var' = var - (m'*alpha) / (sqrt(v') + eps)
 *   sparse (_resource_apply_sparse), g = the row's gradient with duplicate ids summed in order of occurrence (as K4):
 *     touched rows:  m' = m*beta1 + g*omb1 ;  v' = v*beta2 + (g*g)*omb2
 *     other rows:    m' = m*beta1 ;  v' = v*beta2          (lazy != 0: other rows keep var, m and v bit for bit)
 *     every updated row:  var' = var - (alpha*m') / (sqrt(v') + eps)
 * Sparse: one table per call, the contract of tfrs_sparse_adagrad_f32 (I32/I64 ids, out-of-range ids skipped,
 * n < 2^24, d <= 1024, rows < 2^40); n == 0 is allowed (with lazy == 0 every row still decays).  Deterministic.
 * Dense: every variable of one optimizer in one call; vars / grads / ms / vs / numels are HOST arrays of nvars device
 * pointers and element counts.
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_sparse_adam_workspace_bytes(int64_t n, int64_t rows);
int tfrs_sparse_adam_f32(float* table, float* m, float* v, int64_t rows, int d, const void* ids, int ids_dtype,
                         int64_t n, const float* grad_rows, float alpha, float beta1, float beta2, float eps,
                         int lazy, void* ws, size_t ws_bytes, void* stream);
int tfrs_adam_dense_f32(float* const* vars, const float* const* grads, float* const* ms, float* const* vs,
                        const int64_t* numels, int nvars, float alpha, float beta1, float beta2, float eps, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K12  FTRL-Proximal with tf-keras's legacy rules (optimizer_v2/ftrl.py; TF's ApplyFtrl / ApplyFtrlV2).  The caller
 * folds beta into l2 once per call:  l2a = l2 + beta / (2*lr)  (fp32).  Power term:
 *   P(x) = sqrt(x) when lr_power == -0.5, else the fp32 rounding of the fp64 pow(x, -lr_power).
 * Every other step one IEEE fp32 operation, per element with g the gradient:
 *   gs = l2_shrinkage > 0 ? g + (2*l2_shrinkage)*var : g ;  na = acc + g*g
 *   lin' = lin + (gs - ((P(na) - P(acc)) / lr)*var) ;  y = P(na)/lr + 2*l2a
 *   var' = |lin'| > l1 ? (copysign(l1, lin') - lin') / y : +0 ;  acc' = na
 * TFRS_ERR_INVALID_ARG on a non-finite scalar, lr <= 0, lr_power > 0, or a negative l1, l2a or l2_shrinkage.
 * Sparse (_resource_apply_sparse): one table per call, the contract of tfrs_sparse_adagrad_f32 (I32/I64 ids, duplicate
 * ids summed in order of occurrence, out-of-range ids skipped, n < 2^24, d <= 1024, rows < 2^40); n == 0 is a no-op.
 * Only the touched rows change: every other row keeps var, accum and linear bit for bit.  Deterministic.
 * Dense: every variable of one optimizer in one call; vars / grads / accums / linears / numels are HOST arrays of nvars
 * device pointers and element counts.
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_sparse_ftrl_workspace_bytes(int64_t n);
int tfrs_sparse_ftrl_f32(float* table, float* accum, float* linear, int64_t rows, int d, const void* ids, int ids_dtype,
                         int64_t n, const float* grad_rows, float lr, float lr_power, float l1, float l2a,
                         float l2_shrinkage, void* ws, size_t ws_bytes, void* stream);
int tfrs_ftrl_dense_f32(float* const* vars, const float* const* grads, float* const* accums, float* const* linears,
                        const int64_t* numels, int nvars, float lr, float lr_power, float l1, float l2a,
                        float l2_shrinkage, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K5  DCN-v2 cross layer (layers/feature_interaction/dcn.py:176-186, full-rank, no preactivation):
 *   out = x0 * (x . W + bias + diag_scale * x) + x ,  W [D,D] in Keras [in,out] layout.
 * x0, x, out have row stride ld (>= D).  `prod` (nullable) receives x.W + bias + diag_scale*x for
 * the backward pass.  Backward:
 *   dx0 = g*prod ; gp = g*x0 ; dx = gp . W^T + diag_scale*gp + g ; dW = x^T . gp ; dbias = colsum(gp).
 * dx0/dx/dW/dbias are nullable (skipped when NULL).  ws holds gp: B*D floats.
 * ------------------------------------------------------------------------------------------- */
int tfrs_cross_fwd_f32(const float* x0, const float* x, const float* W, const float* bias, int64_t B, int D,
                       int64_t ld, float diag_scale, float* out, float* prod, void* stream);
size_t tfrs_cross_bwd_workspace_bytes(int64_t B, int D);
int tfrs_cross_bwd_f32(const float* x0, const float* x, const float* W, const float* prod, const float* dout,
                       int64_t B, int D, int64_t ld, float diag_scale, float* dx0, float* dx, float* dW,
                       float* dbias, void* ws, size_t ws_bytes, void* stream);

/* K5 on the tensor cores (forward): the same cross formula as tfrs_cross_fwd_f32, computed as one wgmma GEMM on
 * exactly-rescaled fp16 hi/lo splits of x and W (3 MMAs per K step, fp32 accumulation in registers; ~2^-21 relative
 * error, inside the 1e-5 bar) with the formula fused in the epilogue.  W [D,D] ([in,out]) is taken as stored; `ws`
 * holds the per-call images of x and W, and for D > 1024 the chunk partials of the reduction (summed in fixed order,
 * then the formula is applied).
 * For a STACK of cross layers (the reference chains `x = cross(x0, x)`): `out_amax_bits` (nullable, one uint32 on the
 * device) receives max |out| as float bits, accumulated by the epilogue; passing it as `x_amax_bits` (nullable) of the
 * next layer replaces that layer's pass over x for the power-of-two rescale statistic (identical bits, identical result). */
size_t tfrs_cross_tc_workspace_bytes(int64_t B, int D);
int tfrs_cross_tc_fwd_f32(const float* x0, const float* x, const float* W, const float* bias, int64_t B, int D, int64_t ld,
                          float diag_scale, float* out, float* prod, const unsigned int* x_amax_bits, unsigned int* out_amax_bits,
                          void* ws, size_t ws_bytes, void* stream);

/* K5b with both GEMMs on the tensor cores (same contract and outputs as tfrs_cross_bwd_f32): dx = gp.W^T + diag*gp + g
 * and dW = x^T.gp as split-fp16 wgmma GEMMs (dW accumulates the batch in chunks of 1024 rows, partials summed in
 * fixed order); gp = g*x0, dx0 = g*prod and dbias = colsum(gp) as in the exact path.  Deterministic. */
size_t tfrs_cross_tc_bwd_workspace_bytes(int64_t B, int D);
int tfrs_cross_tc_bwd_f32(const float* x0, const float* x, const float* W, const float* prod, const float* dout,
                          int64_t B, int D, int64_t ld, float diag_scale, float* dx0, float* dx, float* dW,
                          float* dbias, void* ws, size_t ws_bytes, void* stream);

/* General fp32-parity GEMM on the tensor cores (the same exact-rescale + fp16 hi/lo split scheme, ~2^-21 relative error):
 *   C[M,N] = opA(A) . opB(B),  opA(m,k) = transA ? A[k*lda+m] : A[m*lda+k],  opB(k,n) = transB ? B[n*ldb+k] : B[k*ldb+n].
 * Reductions longer than 1024 are accumulated in chunks of 1024 with a fixed-order sum of the partials (deterministic).
 * Needs ldc >= N, lda >= (transA ? M : K) and ldb >= (transB ? K : N).  Serves the projections of the low-rank Cross below and large `_compute_score`-style products. */
size_t tfrs_gemm_tc_workspace_bytes(int64_t M, int64_t N, int64_t K);
int tfrs_gemm_tc_f32(int transA, int transB, int64_t M, int64_t N, int64_t K, const float* A, int64_t lda, const float* B,
                     int64_t ldb, float* C, int64_t ldc, void* ws, size_t ws_bytes, void* stream);

/* Low-rank DCN-v2 cross layer on the tensor cores (layers/feature_interaction/dcn.py:131-148,178-179 `projection_dim`;
 * the layer of MultiLayerDCN, multi_layer_dcn.py:146-148):
 *   t = x . U  [B,p] ;  out = x0 * (t . V + bias + diag_scale * x) + x       U [D,p], V [p,D] in Keras [in,out] layout
 * Two wgmma GEMMs; the cross formula is the epilogue of the second one (no [B,D] product round trip).  `t` (required)
 * and `prod` (nullable) are kept for the backward pass:
 *   gp = g*x0 ; dx0 = g*prod ; dt = gp.V^T ; dV = t^T.gp ; dU = x^T.dt ; dx = dt.U^T + diag_scale*gp + g ; dbias = colsum(gp)
 * -- four tensor-core GEMMs, deterministic.  D, p <= 1024.  dx0 / dx / dU / dV / dbias are nullable. */
size_t tfrs_cross_lowrank_tc_workspace_bytes(int64_t B, int D, int p);
int tfrs_cross_lowrank_tc_fwd_f32(const float* x0, const float* x, const float* U, const float* V, const float* bias, int64_t B,
                                  int D, int p, int64_t ld, float diag_scale, float* out, float* prod, float* t, void* ws,
                                  size_t ws_bytes, void* stream);
size_t tfrs_cross_lowrank_tc_bwd_workspace_bytes(int64_t B, int D, int p);
int tfrs_cross_lowrank_tc_bwd_f32(const float* x0, const float* x, const float* U, const float* V, const float* t,
                                  const float* prod, const float* dout, int64_t B, int D, int p, int64_t ld, float diag_scale,
                                  float* dx0, float* dx, float* dU, float* dV, float* dbias, void* ws, size_t ws_bytes,
                                  void* stream);

/* ---------------------------------------------------------------------------------------------
 * K6  Dense layer (tf.keras.layers.Dense inside layers/blocks.py:24-61 MLP and the ranking models,
 * experimental/models/ranking.py:27-257):   y = act(x . W + bias)
 *   x [B,K], W [K,N] ([in,out], Keras layout), bias [N] nullable, act = TFRS_ACT_*.
 * Tensor cores (B >= 1024, K >= 64, N >= 64; tfrs_dense_uses_tc): the split-fp16 wgmma GEMM of the Cross backward with
 * bias + activation in the epilogue (fp32 parity, ~2^-21 relative); K > 1024 is accumulated in chunks of 1024, summed in
 * fixed order, and the bias + activation applied in that reduction.  Otherwise exact CUDA-core kernels: every output is
 * the canonical sequential fmaf chain over k from +0.0f, then + bias, then the activation (a warp per row when N <= 16).
 * `logits` (nullable, [B,N]) receives z = x.W + bias when act is sigmoid: the binary cross-entropy of a sigmoid output
 * is computed from it (tf-keras `_keras_logits`).
 * Backward from the saved OUTPUT y:  dz = dy * act'(y) + dlogits  (relu' = [y > 0], sigmoid' = y (1 - y); dy and dlogits
 * are nullable, at least one is given);  db = colsum(dz);  dx = dz . W^T;  dW = x^T . dz (batch chunks, fixed-order sum).
 * dx / dW / db are nullable.  Deterministic, no float atomics.
 * ------------------------------------------------------------------------------------------- */
enum { TFRS_ACT_LINEAR = 0, TFRS_ACT_RELU = 1, TFRS_ACT_SIGMOID = 2 };
int tfrs_dense_uses_tc(int64_t B, int K, int N);
size_t tfrs_dense_fwd_workspace_bytes(int64_t B, int K, int N);
int tfrs_dense_fwd_f32(const float* x, const float* W, const float* bias, int64_t B, int K, int N, int activation, float* y,
                       float* logits, void* ws, size_t ws_bytes, void* stream);
size_t tfrs_dense_bwd_workspace_bytes(int64_t B, int K, int N);
int tfrs_dense_bwd_f32(const float* x, const float* W, const float* y, const float* dy, const float* dlogits, int64_t B, int K,
                       int N, int activation, float* dx, float* dW, float* dbias, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K27  1-D convolution (tf.keras.layers.Conv1D, channels_last, groups = 1):  x [B, T, C], W [k, C, F] (Keras layout),
 * bias [F] nullable, stride s, dilation d, left pad p >= 0, T_out output steps, act = TFRS_ACT_*:
 *   y [B, T_out, F]:  y[b, t, n] = act(bias[n] + sum_j sum_c x[b, t s + j d - p, c] W[j, c, n]),  x outside [0, T) reads 0.
 * The caller maps Keras's padding to (p, T_out): "valid" p = 0, T_out = floor((T - d (k - 1) - 1) / s) + 1; "same"
 * T_out = ceil(T / s), p = floor(max((T_out - 1) s + d (k - 1) + 1 - T, 0) / 2); "causal" T_out = ceil(T / s),
 * p = d (k - 1).  Windows may read past either end of the sequence (the right pad is implied).
 * This is the Dense layer (K6) on the im2col matrix col [B T_out, k C] with W viewed as [k C, F], on K6's route rule
 * (tfrs_dense_uses_tc(B T_out, k C, F)).  Tensor cores: K6's split-fp16 GEMM and bias + activation epilogue, the A image
 * gathered from x window by window (col is never formed; its power-of-two rescale is taken from max |x| over all of x).
 * Otherwise col is gathered into the workspace and K6's exact CUDA-core kernels run on it.
 * Backward from the saved OUTPUT y, as K6:  dz = dy * act'(y);  dbias = colsum(dz);  dW [k, C, F] = col^T . dz (the
 * reduction over B T_out chunked by 1024 and summed in fixed order);  dx = col2im(dz . W^T): dx[b, t, c] is the sum over j
 * ascending of the terms whose window reads (b, t, c).  dx / dW / dbias are nullable.  Deterministic, no float atomics.
 * ws: tfrs_conv1d_fwd_workspace_bytes / tfrs_conv1d_bwd_workspace_bytes, 16-byte aligned.  B = 0 is a no-op forward.
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_conv1d_fwd_workspace_bytes(int64_t B, int T_out, int C, int k, int F);
int tfrs_conv1d_fwd_f32(const float* x, const float* W, const float* bias, int64_t B, int T, int C, int k, int F, int stride,
                        int dilation, int pad, int T_out, int activation, float* y, void* ws, size_t ws_bytes, void* stream);
size_t tfrs_conv1d_bwd_workspace_bytes(int64_t B, int T_out, int C, int k, int F);
int tfrs_conv1d_bwd_f32(const float* x, const float* W, const float* y, const float* dy, int64_t B, int T, int C, int k, int F,
                        int stride, int dilation, int pad, int T_out, int activation, float* dx, float* dW, float* dbias, void* ws,
                        size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Ranking loss + metrics (tasks/ranking.py:26-119 with the tf.keras losses / metrics the tutorials pass).
 * One pass over the B predictions computes the per-example loss, the reduced loss (fixed-order reduction to a device
 * scalar) and, in the same launch, the batch statistics of the ranking metrics:
 *   loss_kind TFRS_LOSS_BCE         BinaryCrossentropy(from_logits=False): p = clip(pred, 1e-7, 1 - 1e-7),
 *                                   l = -(y log(p + 1e-7) + (1 - y) log(1 - p + 1e-7))
 *             TFRS_LOSS_BCE_LOGITS  BinaryCrossentropy on logits: l = max(z, 0) - z y + log1p(exp(-|z|))
 *             TFRS_LOSS_MSE         MeanSquaredError: l = (pred - y)^2
 *   reduction TFRS_REDUCTION_NONE (per_example only), _SUM (sum_i w_i l_i), _SUM_OVER_BATCH_SIZE (sum_i w_i l_i / B).
 * `loss_in` is what the loss reads (the logits for BCE_LOGITS), `pred` what the metrics read; weights nullable (= 1).
 * stats (nullable, float64 [TFRS_RANKING_STATS + 2 T]) is WRITTEN with this batch's totals:
 *   [0] sum w   [1] sum w [(pred > threshold) == y]   [2] sum w pred   [3] sum w y   [4] sum w (pred - y)^2
 *   [5 .. 5+T) sum w y per AUC bucket, [5+T .. 5+2T) sum w (1 - y) per bucket; bucket = max(ceil(pred (T-1)) - 1, 0)
 *   (tf-keras AUC's evenly-spaced-threshold update, num_thresholds = T).  Per-block partials, fixed-order sums.
 * Backward: dL/d loss_in = g * w * dl/dx (* 1/B for SUM_OVER_BATCH_SIZE); g is a device scalar, or [B] for NONE.
 * ------------------------------------------------------------------------------------------- */
enum { TFRS_LOSS_BCE = 0, TFRS_LOSS_BCE_LOGITS = 1, TFRS_LOSS_MSE = 2 };
enum { TFRS_REDUCTION_NONE = 0, TFRS_REDUCTION_SUM = 1, TFRS_REDUCTION_SUM_OVER_BATCH_SIZE = 2 };
#define TFRS_RANKING_STATS 5
size_t tfrs_ranking_workspace_bytes(int64_t B, int num_thresholds);
int tfrs_ranking_loss_fwd_f32(const float* loss_in, const float* pred, const float* labels, const float* weights, int64_t B,
                              int loss_kind, int reduction, float* per_example, float* loss, double* stats, float threshold,
                              int num_thresholds, void* ws, size_t ws_bytes, void* stream);
int tfrs_ranking_loss_bwd_f32(const float* loss_in, const float* labels, const float* weights, int64_t B, int loss_kind,
                              int reduction, const float* grad, float* dloss_in, void* stream);
/* The metric statistics alone (a loss the library does not own) -- same layout and numbers as above.  The caller's metric
 * objects add them into their device-resident sums; nothing synchronises. */
int tfrs_ranking_metrics_f32(const float* pred, const float* labels, const float* weights, int64_t B, double* stats,
                                    float threshold, int num_thresholds, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K13  Listwise ranking losses and NDCG (TF-Ranking's ListMLELoss, PairwiseHingeLoss, SoftmaxLoss and NDCGMetric, as the
 * reference's listwise_ranking tutorial uses them).  pred, labels [B, L] row-major, 1 <= L <= TFRS_LISTWISE_MAX_LIST;
 * weights (nullable) [B], one per list.  An item with !(label >= 0) (negative or NaN) is padding: it takes no part in any
 * loss, pair, rank or gain, and gets dl/ds = +0.  s = pred * inv_temperature (fp32); n = the valid items of a list,
 * m = max of their s.  Per list, in fp64 unless stated:
 *   LISTMLE         pi = valid items by label descending, ties by mix32(seed, call, b, i) ascending, then by i;
 *                   e_k = exp(s_pi(k) - m), S_k = sum_{j >= k} e_j;  l = sum_k log S_k - (s_pi(k) - m);
 *                   dl/ds_pi(k) = e_k * sum_{j <= k} 1/S_j - 1.
 *                   mix32(seed, call, b, i) = f(f(f(f(seed) ^ call) ^ b) ^ i), f = murmur3's 32-bit finalizer.
 *   PAIRWISE_HINGE  pairs (i, j) with y_i > y_j; fp32: r_i = sum_{j asc} max(0, 1 - (s_i - s_j)), l = (sum_{i asc} r_i) / #pairs
 *                   (0 without a pair); dl/ds_k = (#active (i, k) - #active (k, j)) / #pairs, active: 1 - (s_i - s_j) > 0.
 *   SOFTMAX         Y = sum y;  l = Y log sum_i exp(s_i - m) - sum_i y_i (s_i - m);  dl/ds_i = Y softmax_i - y_i (0 when Y = 0).
 * The fp32 list loss l_b is the rounded fp64 value (hinge: the fp32 chain); per_list[b] = w_b * l_b (fp32) and
 * dlds[b, i] = (float)(w_b * dl/ds_i).  loss = sum_b per_list[b] in fp64 (/ B for SUM_OVER_BATCH_SIZE), rounded once.
 * NDCG at topn (<= 0: L), when `discount` (device fp32 [>= L], discount[r - 1] = 1 / log2(r + 1)) is given: gain =
 * exp2f(y) - 1, ranks by pred descending (ties to the lower i), ideal ranks by label descending; DCG / IDCG are sequential
 * fp32 sums in rank order over r < min(topn, n); ndcg[b] = DCG / IDCG, 0 when IDCG = 0.  ndcg_stats (float64 [2]) is WRITTEN
 * with [sum_b w_b ndcg_b, sum_b w'_b], w'_b = w_b, or for a list with IDCG = 0 the mean w_b of the lists with IDCG > 0.
 * loss_mode TFRS_LIST_LOSS_NONE computes NDCG alone.  The CTA records are folded in a fixed order by the last CTA: one kernel
 * per call, no float atomics, bitwise reproducible.  Backward: dx = (c * dlds) * inv_temperature + 0, c = grad[b] (NONE),
 * grad[0] (SUM) or grad[0] / B (SUM_OVER_BATCH_SIZE) in fp32.
 * ------------------------------------------------------------------------------------------- */
enum { TFRS_LIST_LOSS_NONE = 0, TFRS_LIST_LOSS_LISTMLE = 1, TFRS_LIST_LOSS_PAIRWISE_HINGE = 2, TFRS_LIST_LOSS_SOFTMAX = 3 };
#define TFRS_LISTWISE_MAX_LIST 1024
size_t tfrs_listwise_workspace_bytes(int64_t B, int L);
int tfrs_listwise_fwd_f32(const float* pred, const float* labels, const float* weights, int64_t B, int L, int loss_mode,
                          int reduction, float inv_temperature, uint32_t seed, uint32_t call, float* per_list, float* loss,
                          float* dlds, const float* discount, int topn, float* ndcg, double* ndcg_stats, void* ws,
                          size_t ws_bytes, void* stream);
int tfrs_listwise_bwd_f32(const float* dlds, int64_t B, int L, int reduction, float inv_temperature, const float* grad,
                          float* dx, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K8  UnifiedEmbedding lookup (layers/feature_multiplexing/unified_embedding.py:186-215): every chunk of a feature is
 * tf-keras Hashing(num_bins = table rows, salt) followed by an embedding lookup in a table shared with other features.
 *   bin = SipHash-2-4(k0 = salt[0], k1 = salt[1], message) mod num_bins   (tf.strings.to_hash_bucket_strong)
 * message: the bytes of a TFRS_BYTES value; for TFRS_I32 / TFRS_I64 values the decimal text of tf.as_string (a leading
 * '-' for negatives, no '+', no padding).
 *
 * A feature is one input stream of n values; its n_chunks slots are the next n_chunks entries of `slots` (features in
 * order, so slots of feature k follow those of feature k-1).  Each slot names its table ([rows, dim], rows = num_bins),
 * its salt, and where its dim columns go: out[i * ld + col_off ..].
 *  - row_splits == NULL: out row i = table[bin(value i)] for i < n.
 *  - row_splits != NULL ([n_bags + 1], non-decreasing from 0 to n, as tf.RaggedTensor.from_row_splits): out row b =
 *    the bag values[row_splits[b] .. row_splits[b+1]) pooled: the rows summed in value order in fp32 from +0, then one
 *    IEEE division by the count (MEAN) or by sqrtf(count) (SQRTN); an empty bag gives zeros.
 * `ids` (int64 [n], nullable unless pooled) receives the bucket ids; pointing the slots of one table at consecutive
 * ranges of one buffer gives that table's ids contiguous, in the caller's slot order.
 * dim, col_off and ld are multiples of 4; table, out, grad and grad_rows 16-byte aligned.
 * Launches: forward 1 for up to 64 features and 256 slots (+1 when a feature is pooled); longer calls take one (or two)
 * per group of whole features.  Backward 1 per group.
 * Backward: grad_rows (fp32 [n, dim]) row i = grad[i * ld + col_off ..] (unpooled) or the bag gradient of value i
 * divided as in the forward (pooled; a value outside every bag gets zeros).  Only n, row_splits, n_bags, combiner and
 * n_chunks of the features and dim, ld, col_off, grad and grad_rows of the slots are read.  No float atomics.
 * Pooled features need n_bags >= 1 unless n == 0.  An empty call (n == 0 and no bags) may pass NULL outputs.
 * tfrs_hash_bins: bins[i] = bin(value i) for one stream and one salt (I32, I64, or BYTES with offsets [n+1]); it is
 * tfrs_hashing (K18, below) with that salt and no mask.
 * ------------------------------------------------------------------------------------------- */
enum { TFRS_BYTES = 2 };
enum { TFRS_COMBINER_SUM = 0, TFRS_COMBINER_MEAN = 1, TFRS_COMBINER_SQRTN = 2 };
typedef struct tfrs_ue_feature {
  const void* values;          /* TFRS_I32 / TFRS_I64 values, or the bytes of TFRS_BYTES strings */
  const int64_t* offsets;      /* TFRS_BYTES: [n + 1]; string i = bytes [offsets[i], offsets[i+1]) of values */
  int64_t n;
  const int64_t* row_splits;   /* nullable: pooled bags */
  int64_t n_bags;
  int32_t kind;
  int32_t combiner;            /* TFRS_COMBINER_*, pooled features */
  int32_t n_chunks;
  int32_t reserved;
} tfrs_ue_feature;
typedef struct tfrs_ue_slot {
  const float* table;
  int64_t rows;                /* = num_bins */
  uint64_t salt[2];            /* the SipHash key (k0, k1), by value */
  float* out;
  int64_t ld;
  int32_t col_off;
  int32_t dim;
  int64_t* ids;                /* nullable unless pooled */
  const float* grad;           /* backward: gradient of out */
  float* grad_rows;            /* backward: [n, dim] */
} tfrs_ue_slot;
/* `salt` is a HOST array of two uint64 (k0, k1); values, offsets and bins are device pointers. */
int tfrs_hash_bins(const void* values, const int64_t* offsets, int kind, int64_t n, const uint64_t* salt, int64_t num_bins,
                   int64_t* bins, void* stream);
int tfrs_unified_lookup_fwd_f32(const tfrs_ue_feature* features, int n_features, const tfrs_ue_slot* slots, int n_slots,
                                void* stream);
int tfrs_unified_lookup_bwd_f32(const tfrs_ue_feature* features, int n_features, const tfrs_ue_slot* slots, int n_slots,
                                void* stream);

/* ---------------------------------------------------------------------------------------------
 * K11  Weighted multi-hot bag pooling (layers/embedding/tpu_embedding_layer.py off TPU: safe_embedding_lookup_sparse per
 * feature).  Every feature of a call in one launch (up to 128 features; longer calls take one launch per group of whole
 * features).  A feature reads `table` [rows, dim] (row-major) with n ids `values` (kind TFRS_I32 / TFRS_I64) and optional
 * fp32 `weights` [n] (NULL = 1), and writes output row r at out[r * ld + col_off ..]:
 *  - row_splits != NULL, max_seq_len == 0 (pooled, n_bags rows): row b = (sum of w*e over the valid values of the bag
 *    values[row_splits[b] .. row_splits[b+1]), in value order from +0.0f, each step one fp32 multiply and one add) / D;
 *    D = 1 (SUM), sum w (MEAN), sqrtf(sum w*w) (SQRTN), summed sequentially in fp32; one IEEE division; an empty bag
 *    gives zeros.  `denom` (fp32 [n_bags], nullable) receives D for MEAN / SQRTN; the backward reads it.
 *  - row_splits != NULL, max_seq_len L > 0 (sequence, n_bags * L rows): row b*L + j = w_j * e_j for j < bag size, zeros
 *    for the positions past the bag; values past L are cut.
 *  - row_splits == NULL (dense, n rows): row i = e_i; weights must be NULL.
 * Ids outside [0, rows) are dropped with their weight (zeros at their position, nothing added to a bag or to D).
 * `ids` (int64 [n], nullable) receives the ids as int64: pointing the features of one table at consecutive ranges of one
 * buffer gives that table's (ids, grad_rows) pair.  row_splits are non-decreasing from 0 to n, n_bags >= 1 unless n == 0.
 * Backward: grad_rows (fp32 [n, dim]) row v = grad[r * ld + col_off ..] of the value's output row r (dense), times w
 * (sequence; zeros past L), or g_b * w / D_b (pooled; g_b * w for SUM); zeros for dropped ids.  One launch per group.
 * No alignment is required: dim, col_off, ld multiples of 4 with 16-byte aligned pointers take float4 pieces, anything
 * else a scalar path with the same bits.  No float atomics.
 * ------------------------------------------------------------------------------------------- */
typedef struct tfrs_bag_feature {
  const float* table;
  int64_t rows;
  int32_t dim;
  int32_t kind;                /* TFRS_I32 / TFRS_I64 */
  const void* values;
  int64_t n;
  const int64_t* row_splits;   /* nullable: dense */
  int64_t n_bags;
  const float* weights;        /* nullable */
  int32_t combiner;            /* TFRS_COMBINER_*, pooled features */
  int32_t max_seq_len;         /* > 0: sequence feature */
  float* out;                  /* forward */
  int64_t ld;
  int32_t col_off;
  int32_t reserved;
  int64_t* ids;                /* forward, nullable */
  float* denom;                /* forward: written (nullable); backward: read (MEAN / SQRTN) */
  const float* grad;           /* backward: gradient of out (same ld / col_off) */
  float* grad_rows;            /* backward: [n, dim] */
} tfrs_bag_feature;
int tfrs_embedding_bag_fwd_f32(const tfrs_bag_feature* features, int n_features, void* stream);
int tfrs_embedding_bag_bwd_f32(const tfrs_bag_feature* features, int n_features, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SGD with tf-keras's legacy rules (optimizer_v2/gradient_descent.py, momentum 0), every step one IEEE fp32 operation:
 *   dense:   var' = var - lr*g
 *   sparse:  var[id] = var[id] - lr*g_i once per occurrence i of id, in order of occurrence (no deduplication)
 * Sparse: one table per call; I32/I64 ids, out-of-range ids skipped, n < 2^24, rows < 2^40; ws holds
 * tfrs_sparse_sgd_workspace_bytes(n) bytes.  Dense: vars / grads / numels are HOST arrays of nvars device pointers and
 * element counts.  Deterministic, no atomics.
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_sparse_sgd_workspace_bytes(int64_t n);
int tfrs_sparse_sgd_f32(float* table, int64_t rows, int d, const void* ids, int ids_dtype, int64_t n,
                        const float* grad_rows, float lr, void* ws, size_t ws_bytes, void* stream);
int tfrs_sgd_dense_f32(float* const* vars, const float* const* grads, const int64_t* numels, int nvars, float lr,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * K9  tree-AH approximate retrieval: the algorithm of ScaNN (layers/factorized_top_k.py:613-796) under the rules of
 * DESIGN.md §2 -- a k-means tree of L leaves over the rows, 4-bit product codes of every row's residual (blocks of dpb
 * dims, 16 centers each), and a search that scores the rows of the probed leaves with int8 lookup tables.
 * d <= 256, 1 <= dpb <= 8, B = ceil(d / dpb) blocks, W = ceil(B / 8) code words per row, N < 2^24 rows.
 *
 * Index build (the host runs the Lloyd iterations):
 *   tfrs_tree_ah_assign_f32: leaf[i] = top-1 of the canonical dot [x_i, 1] . [c_l, -0.5f * |c_l|^2] (squared L2, ties to
 *     the lower l), through tfrs_topk_scan_f32 in chunks of 65536 rows.
 *   tfrs_tree_ah_group: order[] = positions 0..n-1 grouped by leaf in ascending leaf order, positions ascending inside a
 *     leaf; offsets[l] .. offsets[l+1] is leaf l's range (offsets has L + 1 entries).
 *   tfrs_tree_ah_update_centroids_f32: every non-empty leaf's centroid = the float64 sum of its members' rows x[order[..]]
 *     taken sequentially in that order, divided once by the count, rounded to fp32.  Empty leaves keep theirs.
 *   Codebooks are fp32 [B][16][dpb] (the last block's unused dims are 0); residual r = x - c_leaf(x) (one fp32 subtraction).
 *   tfrs_tree_ah_init_codebooks_f32: center j of every block = the residual of position pos[j] (pos: 16 int64).
 *   tfrs_tree_ah_encode: codes of positions p < n (row = rows ? rows[p] : p; leaf indexed by row): per block the top-1 of
 *     [r_b, 1] . [cb_j, -0.5f |cb_j|^2]; packed 8 per uint32 (block 8w+e in bits 4e..4e+3), W words per position.
 *   tfrs_tree_ah_update_codebooks_f32: codebook update from the codes of positions 0..n-1, the same ordered float64 mean.
 * Search: per query, probe the top P leaves by canonical dot(q, c_l) (ties to the lower leaf); LUT T[b][j] = canonical
 *   dot of block b of q with center j, s = max|T| / 127 (0 if max|T| = 0), T8 = (int8) rint(T / s); the approximate
 *   score of a row of probed leaf l is  dot(q, c_l) + s * (float) sum_b T8[b][code_b]  (two rounded fp32 ops).  The top
 *   k' rows by that score are kept; with `rows` (fp32 [N, d], original row order) they are rescored with the canonical
 *   dot and the top k of those returned, otherwise k' == k and the approximate scores are returned.  Order = (score desc,
 *   row asc).  Positions with no row (the probed leaves hold fewer) get (NaN, 0).  out_*: [Q, k]; out_idx = row ids.
 *   P <= min(L, 2048), k <= k' <= 2048.
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_tree_ah_assign_workspace_bytes(int64_t n, int d, int L);
int tfrs_tree_ah_assign_f32(const float* x, int64_t n, int d, const float* centers, int L, int64_t* leaf, void* ws,
                            size_t ws_bytes, void* stream);
size_t tfrs_tree_ah_group_workspace_bytes(int64_t n);
int tfrs_tree_ah_group(const int64_t* leaf, int64_t n, int L, int32_t* offsets, int32_t* order, void* ws, size_t ws_bytes,
                       void* stream);
int tfrs_tree_ah_update_centroids_f32(const float* x, int d, const int32_t* order, const int32_t* offsets, int L,
                                      float* centroids, void* stream);
int tfrs_tree_ah_init_codebooks_f32(const float* x, int d, const int64_t* pos, const int64_t* leaf, const float* centroids,
                                    int dpb, float* codebooks, void* stream);
int tfrs_tree_ah_encode(const float* x, int d, const int32_t* rows, int64_t n, const int64_t* leaf, const float* centroids,
                        const float* codebooks, int dpb, uint32_t* codes, void* stream);
int tfrs_tree_ah_update_codebooks_f32(const float* x, int d, int64_t n, const int64_t* leaf, const float* centroids,
                                      const uint32_t* codes, int dpb, float* codebooks, void* stream);
size_t tfrs_tree_ah_search_workspace_bytes(int64_t Q, int d, int L, int P, int dpb, int k, int kp, int reorder, int64_t N);
int tfrs_tree_ah_search_f32(const float* q, int64_t Q, int d, const float* centroids, int L, const int32_t* leaf_offsets,
                            const float* codebooks, int dpb, const uint32_t* codes, const int32_t* order, int64_t N,
                            const float* rows, int P, int k, int kp, float* out_scores, int64_t* out_idx, void* ws,
                            size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DLRM DotInteraction (layers/feature_interaction/dot_interaction.py:53-104; SURVEY 8f-4): feats [B,F,d] ->
 * pairwise dots e_i.e_j of every sample; output = lower triangle in (i,j) row-major order without
 * (self_interaction=0) or with the diagonal, [B, out_dim], or the full [B,F*F] matrix with the excluded part
 * zeroed (skip_gather=1).  Every dot is the canonical sequential fmaf chain.  F <= 64.
 * Backward: dfeats[b,i,:] = sum_j G'(i,j) feats[b,j,:] with G' the symmetrised upstream gradient.
 * B == 0 writes nothing (pointers may be NULL); gout may be NULL when the output width is 0.
 * ------------------------------------------------------------------------------------------- */
int tfrs_dot_interaction_out_dim(int F, int self_interaction, int skip_gather);
int tfrs_dot_interaction_fwd_f32(const float* feats, int64_t B, int F, int d, int self_interaction, int skip_gather,
                                 float* out, void* stream);
int tfrs_dot_interaction_bwd_f32(const float* feats, const float* gout, int64_t B, int F, int d, int self_interaction,
                                 int skip_gather, float* dfeats, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K15 vocabulary lookup: tf.keras.layers.StringLookup / IntegerLookup (tf-keras index_lookup.py) as the reference's
 * towers use them (`Sequential([StringLookup(vocabulary=ids, mask_token=None), Embedding(len(ids) + 1, d)])`).
 *
 * A table maps each of V distinct keys (V < 2^30) to its position 0..V-1: an int64 vocabulary (kind TFRS_I64, `keys`
 * int64 [V]) or a string one (TFRS_BYTES, `keys` = the bytes back to back, `offsets` int64 [V+1]).  The caller keeps the
 * keys alive as long as the table; `slots` is tfrs_lookup_table_bytes(V, kind) bytes of device memory, 256-byte aligned,
 * that tfrs_lookup_build fills (its contents may differ from build to build; results never do).  The mask token
 * (has_mask != 0) is `mask` for TFRS_I64 and the mask_len bytes at `mask_bytes` (device) for TFRS_BYTES.
 *   tfrs_lookup_slots: the table's slot count for V keys (a power of two >= 2V, at least 64), -1 when V is out of range.
 *   tfrs_lookup_build: fills `slots`; *dup = 1 when two keys are equal (compared as int64, or as byte strings), else 0.
 *     One launch for TFRS_I64, two for TFRS_BYTES, after two memsets.
 *   tfrs_lookup: out[i] (int64) = 0 if value i equals the mask token, base + p if it equals key p, otherwise `oov` --
 *     or, when `miss` is not NULL, -1 and *miss = 1 (the caller zeroes *miss).  `values`: TFRS_I32 / TFRS_I64 against an
 *     I64 table (compared as int64), TFRS_BYTES with `offsets` [n+1] against a BYTES table.  One launch; n == 0 writes
 *     nothing.
 *   tfrs_lookup_invert: out[i] = keys[x - base] (or x - base when keys is NULL) for x = idx[i] (TFRS_I32 / TFRS_I64) in
 *     [base, base + V); mask_out for x == 0 when has_mask; oov_out for every other x.  One launch.
 * ------------------------------------------------------------------------------------------- */
typedef struct tfrs_lookup_table {
  const void* keys;            /* TFRS_I64: int64 [V]; TFRS_BYTES: the keys' bytes */
  const int64_t* offsets;      /* TFRS_BYTES: [V + 1]; key p = bytes [offsets[p], offsets[p+1]) of keys */
  int64_t V;
  int32_t kind;                /* TFRS_I64 or TFRS_BYTES */
  int32_t has_mask;
  int64_t mask;                /* TFRS_I64: the mask token */
  const uint8_t* mask_bytes;   /* TFRS_BYTES: the mask token's bytes */
  int64_t mask_len;
  void* slots;                 /* tfrs_lookup_table_bytes(V, kind) bytes */
} tfrs_lookup_table;

int64_t tfrs_lookup_slots(int64_t V);
size_t tfrs_lookup_table_bytes(int64_t V, int kind);
int tfrs_lookup_build(const tfrs_lookup_table* table, int32_t* dup, void* stream);
int tfrs_lookup(const tfrs_lookup_table* table, const void* values, const int64_t* offsets, int kind, int64_t n,
                int64_t base, int64_t oov, int32_t* miss, int64_t* out, void* stream);
int tfrs_lookup_invert(const void* idx, int kind, int64_t n, const int64_t* keys, int64_t V, int64_t base, int has_mask,
                       int64_t mask_out, int64_t oov_out, int64_t* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K16 text vectorization: tf.keras.layers.TextVectorization(output_mode="int", split="whitespace") as the reference's
 * movie towers use it (`TextVectorization(max_tokens=10_000)` -> `Embedding(..., mask_zero=True)` -> pooling).
 *
 * n strings (TFRS_BYTES layout: `data` with int64 `offsets` [n+1], nbytes = offsets[n] < 2^32 bytes in all).
 *   tfrs_text_standardize: for each string, ASCII-lowercases the bytes (flags & TFRS_TEXT_LOWER) and deletes the 32 bytes
 *     of Python's string.punctuation (flags & TFRS_TEXT_STRIP), writing the result to `scratch` at the string's own
 *     offsets and filling the rest of its range with spaces.  counts[i] (int32) = the number of tokens of string i: the
 *     runs of bytes other than " \t\n\v\f\r".  When max_count is not NULL, *max_count = the largest count (0 for n == 0).
 *     One launch after a 4-byte memset.
 *   tfrs_text_lookup: out [n, T] int64: token j of string i (j < T) looked up in a BYTES lookup table, base + p for
 *     vocabulary entry p and `oov` for any other token; 0 after the string's last token.  Tokens past T are dropped.
 *     One launch; no atomics.
 *   tfrs_text_spans: the tokens themselves: token j of string i is spans[2k] = its first byte's offset in scratch and
 *     spans[2k+1] = its length, k = token_offsets[i] + j (token_offsets [n+1]: the exclusive sum of counts).  One launch.
 * ------------------------------------------------------------------------------------------- */
enum { TFRS_TEXT_LOWER = 1, TFRS_TEXT_STRIP = 2 };

int tfrs_text_standardize(const uint8_t* data, const int64_t* offsets, int64_t n, int64_t nbytes, int flags,
                          uint8_t* scratch, int32_t* counts, int32_t* max_count, void* stream);
int tfrs_text_lookup(const tfrs_lookup_table* table, const uint8_t* scratch, const int64_t* offsets, int64_t n, int64_t T,
                     int64_t base, int64_t oov, int64_t* out, void* stream);
int tfrs_text_spans(const uint8_t* scratch, const int64_t* offsets, int64_t n, const int64_t* token_offsets,
                    int64_t* spans, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K17 numeric columns and pooling: tf.keras.layers.Discretization, Normalization and GlobalAveragePooling1D as the
 * reference's context-feature towers use them.  Values are TFRS_I32, TFRS_I64, TFRS_F32 or TFRS_F64 (device, contiguous).
 *   tfrs_bucketize: out[i] (int64) = #{j : b[j] <= x_i} over the nb sorted float32 boundaries (std::upper_bound; NaN gives
 *     nb).  Integers are rounded to float32 first; float64 values are compared as doubles.  One launch.
 *   tfrs_normalize: out[i] = (f32(x_i) - mean[c]) / max(sqrt(var[c]), 1e-7f), or with invert mean[c] + f32(x_i) *
 *     max(sqrt(var[c]), 1e-7f), c = i % C; one IEEE float32 operation per step, no FMA.  One launch.
 *   tfrs_normalization_adapt: merges the batches of x ([N, R] rows, channel of element (r, e) = e % C; C divides R) into
 *     state [2, C] = (mean, variance) float32 and *count (int64), as Keras's Normalization.update_state does: batch k holds
 *     rows [k*batch_rows, (k+1)*batch_rows).  Batch moments: float32 of the float64 sums (in row-major order) of f32(x)
 *     and of f32((f32(x) - m)^2), over the batch's count; then, in float32, w = n_b / n_total, mean' = mean*(1-w) +
 *     m*w, var' = (var + (mean-mean')^2)*(1-w) + (v + (m-mean')^2)*w.  One launch when N <= batch_rows, else two (every
 *     batch's moments, then one fold per channel); ws is tfrs_normalization_adapt_workspace_bytes bytes.
 *   tfrs_mean_pool_fwd: out [B, d] = sum_t x[b,t,:]*m[b,t] / sum_t m[b,t] (products and the sum in float32, t ascending
 *     from +0.0f; an all-masked row is 0/0), or without a mask sum_t x[b,t,:] / T.  x is addressed by element strides;
 *     mask [B, T] (a Keras mask, see TFRS_BOOL).  One launch.
 *   tfrs_mean_pool_bwd: dx [B, T, d] contiguous = f32(g[b,:] / sum_t m[b,t]) * m[b,t], or g[b,:] / T.  One launch.
 * ------------------------------------------------------------------------------------------- */
/* A Keras mask crosses the ABI as (const void* mask, int mask_kind): a device array of kind TFRS_BOOL (one byte per
 * element), TFRS_I32 or TFRS_I64, contiguous and row-major over the shape the entry names; nonzero = kept.  NULL keeps
 * every element.  A non-NULL mask of another kind is TFRS_ERR_INVALID_ARG. */
enum { TFRS_F32 = 3, TFRS_F64 = 4, TFRS_BOOL = 5 };

int tfrs_bucketize(const void* x, int kind, int64_t n, const float* bounds, int64_t nb, int64_t* out, void* stream);
int tfrs_normalize(const void* x, int kind, int64_t n, int64_t C, const float* mean, const float* var, int invert,
                   float* out, void* stream);
size_t tfrs_normalization_adapt_workspace_bytes(int64_t N, int64_t C, int64_t batch_rows);
int tfrs_normalization_adapt(const void* x, int kind, int64_t N, int64_t R, int64_t C, int64_t batch_rows, float* state,
                             int64_t* count, void* ws, size_t ws_bytes, void* stream);
int tfrs_mean_pool_fwd(const float* x, int64_t B, int64_t T, int64_t d, int64_t sb, int64_t st, int64_t sd,
                       const void* mask, int mask_kind, float* out, void* stream);
int tfrs_mean_pool_bwd(const float* g, int64_t B, int64_t T, int64_t d, const void* mask, int mask_kind, float* dx,
                       void* stream);

/* ---------------------------------------------------------------------------------------------
 * K18 feature hashing: tf.keras.layers.Hashing(num_bins, mask_value, salt) as the reference's uet and featurization
 * tutorials use it (`Sequential([Hashing(num_bins=buckets), Embedding(buckets, d)])`).
 *   h = FarmHash Fingerprint64(message) when `salt` is NULL (tf.strings.to_hash_bucket_fast), else
 *       SipHash-2-4(k0 = salt[0], k1 = salt[1], message) (to_hash_bucket_strong).  `salt` is a HOST array of two uint64.
 *   message: the bytes of a TFRS_BYTES value (offsets [n+1]; strings may start at any byte); for TFRS_I32 / TFRS_I64
 *       values the decimal text of tf.as_string.
 *   bins[i] (int64) = h mod num_bins, unsigned.  With has_mask and num_bins > 1, bin 0 is reserved: 0 when value i
 *       equals the mask (`mask` as int64 for integer values; the mask_len device bytes at mask_bytes for strings), else
 *       1 + h mod (num_bins - 1).  With num_bins == 1 nothing is reserved.
 * One launch; n == 0 writes nothing.
 * ------------------------------------------------------------------------------------------- */
int tfrs_hashing(const void* values, const int64_t* offsets, int kind, int64_t n, const uint64_t* salt, int64_t num_bins,
                 int has_mask, int64_t mask, const uint8_t* mask_bytes, int64_t mask_len, int64_t* bins, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K19 GRU recurrence: tf.keras.layers.GRU(units, reset_after=True) as the reference's sequential retrieval tutorial
 * builds its query tower (`Sequential([StringLookup, Embedding, GRU(32)])`).  Weights as Keras stores them, columns
 * ordered (z, r, h): kernel W [D, 3u], recurrent_kernel U [u, 3u], bias [2, 3u] = (b_i, b_r).  The input projection
 * gx = x.W + b_i ([B*T, 3u], row b*T + t) is the caller's, on K6 (tfrs_dense_fwd_f32 / tfrs_dense_bwd_f32).
 *   gr = h_{t-1}.U + b_r (fmaf chain over k ascending from +0.0f, then + b_r);  z = sigmoid(gx_z + gr_z),
 *   r = sigmoid(gx_r + gr_r),  hh = tanh(gx_h + r gr_h),  h_t = z h_{t-1} + (1 - z) hh;  sigmoid = 1 / (1 + expf(-x)).
 * h_0 = h0 [B, u], or zeros when h0 is NULL.  mask [B, T] (a Keras mask, see TFRS_BOOL): at a masked step h_t = h_{t-1}
 * and nothing is computed.  1 <= units <= TFRS_GRU_MAX_UNITS, T >= 1, B < 2^31; B == 0 writes nothing.
 *   tfrs_gru_fwd_f32: h_last [B, u] = h_T; out_seq [B, T, u] = every h_t (nullable); gates [B, T, 4u] = (z, r, hh, gr_h)
 *     and h_prev [B, T, u] = h_{t-1} (both or neither, for the backward; gates are not written at masked steps).
 *     One launch.
 *   tfrs_gru_bwd_f32: from the upstream gradients g_seq [B, T, u] (of out_seq) and g_last [B, u] (of h_last), either
 *     nullable, in reverse t with dh carried:  dh += g_seq[t] (+ g_last at T-1);  dz = dh (h_{t-1} - hh) z (1 - z);
 *     dn = dh (1 - z)(1 - hh^2);  dr = dn gr_h r (1 - r);  dgx = [dz | dr | dn];  dgr = [dz | dr | dn r];
 *     dh <- dh z + dgr.U^T (fmaf chain over the 3u columns ascending).  A masked step passes dh through and writes zero
 *     dgx rows.  Writes dgx [B*T, 3u] (the gradient of gx) and dh0 [B, u] (nullable) in one launch, then dU = h_prev^T .
 *     dgr and db_r = colsum(dgr) (each nullable) with tfrs_dense_bwd_f32.  ws: tfrs_gru_bwd_workspace_bytes, 16-byte
 *     aligned.  No float atomics.
 * ------------------------------------------------------------------------------------------- */
#define TFRS_GRU_MAX_UNITS 2048

int tfrs_gru_fwd_f32(const float* gx, const float* U, const float* b_r, const float* h0, const void* mask, int mask_kind,
                     int64_t B, int64_t T, int units, float* out_seq, float* h_last, float* gates, float* h_prev,
                     void* stream);
size_t tfrs_gru_bwd_workspace_bytes(int64_t B, int64_t T, int units);
int tfrs_gru_bwd_f32(const float* U, const float* gates, const float* h_prev, const void* mask, int mask_kind,
                     const float* g_seq, const float* g_last, int64_t B, int64_t T, int units, float* dgx, float* dU,
                     float* db_r, float* dh0, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K20 LSTM recurrence: tf.keras.layers.LSTM(units) with the TF2 defaults (tanh / sigmoid, implementation=2), the cell
 * users put in the sequential retrieval tutorial's query tower instead of the GRU.  Weights as Keras stores them,
 * columns ordered (i, f, c, o): kernel W [D, 4u], recurrent_kernel U [u, 4u], bias b [4u].  The input projection
 * gx = x.W + b ([B*T, 4u], row b*T + t) is the caller's, on K6 (tfrs_dense_fwd_f32 / tfrs_dense_bwd_f32).
 *   z = gx + h_{t-1}.U (fmaf chain over k ascending from +0.0f, then added to gx);  i = sigmoid(z_i), f = sigmoid(z_f),
 *   g = tanh(z_c), o = sigmoid(z_o);  c_t = f c_{t-1} + i g,  h_t = o tanh(c_t);  sigmoid = 1 / (1 + expf(-x)).
 * h_0 = h0 [B, u] and c_0 = c0 [B, u], each zeros when NULL.  mask [B, T] (a Keras mask, see TFRS_BOOL): at a masked
 * step h_t = h_{t-1}, c_t = c_{t-1} and nothing is computed.  1 <= units <= TFRS_LSTM_MAX_UNITS, T >= 1, B < 2^31;
 * B == 0 writes nothing.
 *   tfrs_lstm_fwd_f32: h_last [B, u] = h_T and c_last [B, u] = c_T; out_seq [B, T, u] = every h_t (nullable); gates
 *     [B, T, 4u] = (i, f, g, o), c_seq [B, T, u] = every c_t and h_prev [B, T, u] = h_{t-1} (all three or none, for the
 *     backward; gates are not written at masked steps).  One launch.
 *   tfrs_lstm_bwd_f32: from the upstream gradients g_seq [B, T, u] (of out_seq), g_h [B, u] (of h_last) and g_c [B, u]
 *     (of c_last), each nullable, in reverse t with dh and dc carried:  dh += g_seq[t] (+ g_h at T-1), dc (+= g_c at
 *     T-1);  do = dh tanh(c_t) o (1 - o);  dc += dh o (1 - tanh(c_t)^2);  di = dc g i (1 - i);  df = dc c_{t-1} f (1 - f);
 *     dg = dc i (1 - g^2);  dz = [di | df | dg | do];  dh <- dz.U^T (fmaf chain over the 4u columns ascending);
 *     dc <- dc f.  c0 is the forward's (nullable).  A masked step passes dh and dc through and writes zero dz rows.
 *     Writes dz [B*T, 4u] (the gradient of gx), dh0 and dc0 [B, u] (each nullable) in one launch, then dU = h_prev^T .
 *     dz (nullable; needs h_prev) with tfrs_dense_bwd_f32.  ws: tfrs_lstm_bwd_workspace_bytes, 16-byte aligned (only
 *     read when dU is written).  No float atomics.
 * ------------------------------------------------------------------------------------------- */
#define TFRS_LSTM_MAX_UNITS 2048

int tfrs_lstm_fwd_f32(const float* gx, const float* U, const float* h0, const float* c0, const void* mask, int mask_kind,
                      int64_t B, int64_t T, int units, float* out_seq, float* h_last, float* c_last, float* gates,
                      float* c_seq, float* h_prev, void* stream);
size_t tfrs_lstm_bwd_workspace_bytes(int64_t B, int64_t T, int units);
int tfrs_lstm_bwd_f32(const float* U, const float* gates, const float* c_seq, const float* h_prev, const float* c0,
                      const void* mask, int mask_kind, const float* g_seq, const float* g_h, const float* g_c, int64_t B,
                      int64_t T, int units, float* dz, float* dU, float* dh0, float* dc0, void* ws, size_t ws_bytes,
                      void* stream);

/* ---------------------------------------------------------------------------------------------
 * K21 attention core: tf.keras.layers.MultiHeadAttention between its projections (attention over the sequence axis, no
 * dropout).  The caller projects with K6 (tfrs_dense_fwd_f32): Q [B, T, H*dk], K [B, S, H*dk], V [B, S, H*dv], head h
 * in columns h*d .. h*d + d - 1, contiguous; they are read in place.  1 <= dk, dv <= TFRS_MHA_MAX_HEAD_DIM, T, S >= 1.
 *   scores s = (Q_h * scale) . K_h^T with scale = (float)(1 / sqrt(dk)) applied to Q in fp32 (Keras's order); where the
 *   combined mask drops (b, t, s), s += -1e9f (tf-keras Softmax), so a fully masked row is uniform; P = softmax over s;
 *   O_h = P . V_h.  masks (nullable; each a Keras mask, see TFRS_BOOL): query [B, T], value [B, S], key [B, S],
 *   attention [B, T, S], causal (keeps s <= t), combined by AND.
 *   tfrs_mha_fwd_f32: O [B, T, H*dv]; stats [B, H, T, 2] = (row max m, row sum l of e^{s - m}) -- the log-sum-exp
 *     m + log l, kept as two numbers because a fully masked row's m = -1e9 leaves no fp32 room for log l (nullable; the
 *     backward needs it); P [B, H, T, S] = e^{s - m} / l (nullable).  One launch.
 *   tfrs_mha_bwd_f32: from dO [B, T, H*dv] and the forward's O and stats: dQ, dK, dV (the gradients of the projected Q,
 *     K, V).  Three launches: delta = rowsum(dO * O); dK, dV per key row (P recomputed from stats); dQ per query row.
 *     ws: tfrs_mha_bwd_workspace_bytes, 16-byte aligned.  Fixed summation order, no float atomics.
 * ------------------------------------------------------------------------------------------- */
#define TFRS_MHA_MAX_HEAD_DIM 128

typedef struct TfrsMhaMasks {
  const void* query; int query_kind;
  const void* value; int value_kind;
  const void* key; int key_kind;
  const void* attention; int attention_kind;
  int causal;
} TfrsMhaMasks;

int tfrs_mha_fwd_f32(const float* Q, const float* K, const float* V, const TfrsMhaMasks* masks, int64_t B, int64_t T,
                     int64_t S, int H, int dk, int dv, float* O, float* stats, float* P, void* stream);
size_t tfrs_mha_bwd_workspace_bytes(int64_t B, int64_t T, int H);
int tfrs_mha_bwd_f32(const float* Q, const float* K, const float* V, const TfrsMhaMasks* masks, const float* O,
                     const float* stats, const float* dO, int64_t B, int64_t T, int64_t S, int H, int dk, int dv,
                     float* dQ, float* dK, float* dV, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dense attention (K21 dot scores, K25 tanh scores): tf.keras.layers.Attention and AdditiveAttention on query Q [B, Tq,
 * dim], key K [B, Tv, dim] and value V [B, Tv, dv] (float32, contiguous; 1 <= dim, dv <= TFRS_MHA_MAX_HEAD_DIM, Tq, Tv
 * >= 1), run as one head over the B * Tq query rows.  Scores in fp32:
 *   TFRS_DENSE_DOT:      s = scale * (q . k)                        (scale [1], NULL = 1)
 *   TFRS_DENSE_CONCAT:   s = wc * sum_d tanhf(scale (q_d + k_d))    (scale [1], NULL = 1; concat_weight wc [1])
 *   TFRS_DENSE_ADDITIVE: s = sum_d scale_d tanhf(q_d + k_d)         (scale [dim], NULL = 1)
 *   The weights are device pointers, read by the kernels.  keep(b, i, j) = value_mask[b, j] & (j <= i if causal); a
 *   dropped score gets s -= 1e9 in fp32, then P = softmax over j (a fully masked row is uniform).  With rate > 0 (a
 *   training call) the weights are dropped as K23 drops a [B, Tq, Tv] tensor: element e = (b Tq + i) Tv + j takes word
 *   e % 4 of Philox4x32-10 at counter (e/4 lo, e/4 hi, call lo, call hi) and key (seed lo, seed hi); keep <=> (word >>
 *   8) >= ceil(rate * 2^24); W = keep ? P * (float)(1 / (1 - rate)) : +0; else W = P.  O[b, i] = query_mask[b, i] *
 *   sum_j W_ij v_j.  query_mask [B, Tq] and value_mask [B, Tv] (Keras masks, see TFRS_BOOL).
 *   tfrs_dense_attention_fwd_f32: O [B, Tq, dv]; stats [B, Tq, 2] = (row max, row sum of e^{s - max}) (nullable; the
 *     backward needs it); P [B, Tq, Tv] = W (nullable).  One launch.
 *   tfrs_dense_attention_bwd_f32: from dO and the forward's O and stats: dQ, dK [B, Tv, dim], dV; dscale ([1], or [dim]
 *     for ADDITIVE; nullable) and dconcat_weight ([1], CONCAT only; nullable).  Three launches (delta, dK / dV per key
 *     row, dQ and the per-row partials of the weights' gradients per query row) and one fixed-order fold per weight
 *     gradient asked for.  ws: tfrs_dense_attention_bwd_workspace_bytes, 16-byte aligned.  No float atomics: bitwise
 *     reproducible.
 * ------------------------------------------------------------------------------------------- */
#define TFRS_DENSE_DOT 0
#define TFRS_DENSE_CONCAT 1
#define TFRS_DENSE_ADDITIVE 2

typedef struct TfrsDenseAttention {
  int mode;
  const float* scale;
  const float* concat_weight;
  const void* query_mask; int query_mask_kind;
  const void* value_mask; int value_mask_kind;
  int causal;
  double rate; uint64_t seed; uint64_t call;
} TfrsDenseAttention;

int tfrs_dense_attention_fwd_f32(const float* Q, const float* K, const float* V, const TfrsDenseAttention* desc,
                                 int64_t B, int64_t Tq, int64_t Tv, int dim, int dv, float* O, float* stats, float* P,
                                 void* stream);
size_t tfrs_dense_attention_bwd_workspace_bytes(int mode, int64_t B, int64_t Tq, int dim);
int tfrs_dense_attention_bwd_f32(const float* Q, const float* K, const float* V, const TfrsDenseAttention* desc,
                                 const float* O, const float* stats, const float* dO, int64_t B, int64_t Tq, int64_t Tv,
                                 int dim, int dv, float* dQ, float* dK, float* dV, float* dscale, float* dconcat_weight,
                                 void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K22 layer normalization: tf.keras.layers.LayerNormalization(axis=-1) over the rows of x [N, d] (d >= 1).
 *   mean = hi + lo with hi = sum(x) / d and lo = sum(x - hi) / d; var = sum((x - hi)^2) / d - lo^2 (population
 *   variance, corrected two-pass); rstd = 1 / sqrtf(var + eps); y = ((x - hi) - lo) * rstd * gamma + beta, gamma / beta
 *   [d] nullable (scale / center off).  Keeping the mean as the pair (hi, lo) keeps x - mean exact where |mean| >> std.
 *   tfrs_layer_norm_fwd_f32: y [N, d]; mean [N, 2] = (hi, lo) and rstd [N] (nullable together; the backward needs
 *     them).  One launch.
 *   tfrs_layer_norm_bwd_f32: from dy: dx [N, d] = rstd (g - mean(g) - xhat mean(g xhat)) with g = dy * gamma and
 *     xhat = ((x - hi) - lo) rstd; dparams [2, d] = (sum_rows dy xhat, sum_rows dy) = (dgamma, dbeta) (nullable) from
 *     per-CTA partials folded in fixed order by a second launch.  ws: tfrs_layer_norm_bwd_workspace_bytes, 16-byte
 *     aligned.  No float atomics.
 * ------------------------------------------------------------------------------------------- */
int tfrs_layer_norm_fwd_f32(const float* x, const float* gamma, const float* beta, int64_t N, int64_t d, float eps,
                            float* y, float* mean, float* rstd, void* stream);
size_t tfrs_layer_norm_bwd_workspace_bytes(int64_t N, int64_t d);
int tfrs_layer_norm_bwd_f32(const float* x, const float* gamma, const float* mean, const float* rstd, const float* dy,
                            int64_t N, int64_t d, float* dx, float* dparams, void* ws, size_t ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K23 dropout: tf.keras.layers.Dropout's training-mode output over x (contiguous float32, `rank` axes of `shape`):
 *   y[i] = keep(m(i)) ? x[i] * scale : +0.0f.  The same call on dy is the backward (the mask is regenerated, never
 *   stored).  A dropped element is +0 whatever x[i] is, so a dropped NaN or inf does not propagate.
 *   noise_shape [rank] (nullable = shape): each entry is 1 (one mask value broadcast along that axis) or shape[a].  Mask
 *   element j counts row-major over the noise shape; m(i) is the mask element of output element i.
 *   Philox4x32-10 (M = 0xD2511F53, 0xCD9E8D57; W = 0x9E3779B9, 0xBB67AE85) at key (seed lo, seed hi) and counter
 *   (g lo, g hi, call lo, call hi) with g = j / 4; element j takes output word j % 4.
 *   keep <=> (word >> 8) >= thr, thr = ceil(rate * 2^24) in float64;  scale = (float)(1 / (1 - rate)) from float64.
 *   0 <= rate < 1; 1 <= rank <= TFRS_DROPOUT_MAX_RANK (TFRS_ERR_UNSUPPORTED otherwise).  `call` is the caller's per-layer
 *   counter, advanced once per training call.  An empty x writes nothing.  One launch.
 * ------------------------------------------------------------------------------------------- */
#define TFRS_DROPOUT_MAX_RANK 4

int tfrs_dropout_f32(const float* x, int rank, const int64_t* shape, const int64_t* noise_shape, double rate,
                     uint64_t seed, uint64_t call, float* y, void* stream);

/* ---------------------------------------------------------------------------------------------
 * K24 batch normalization: tf.keras.layers.BatchNormalization(axis=-1) over the rows of x [N, d] (N >= 1, d >= 1; the
 * statistics are per column).  gamma / beta [d] nullable (scale / center off).  mask [N] (a Keras mask, see TFRS_BOOL)
 * restricts the batch moments to the kept rows (weighted moments, n = sum w); n = 0 gives mean 0 and variance 0.  Every
 * sum runs in a fixed order over a row chunking that depends on (N, d) only: no float atomics, bitwise reproducible.
 *   training: the batch mean as the fp32 pair hi = f32(mean), lo = f32(mean - hi) (per-chunk shifted sums folded in
 *     fp64), the population variance var, rstd = 1 / sqrtf(var + eps), y = ((x - hi) - lo) rstd gamma + beta; the
 *     moving statistics updated in place with decay = f32(1 - momentum): mm = mm - (mm - f32(hi + lo)) decay, mv = mv
 *     - (mv - var) decay (plain fp32, no contraction).
 *   inference: y = (x - mm) rstd_mv gamma + beta with rstd_mv = 1 / sqrtf(mv + eps); nothing is updated.
 *   tfrs_batch_norm_fwd_f32: y [N, d]; saved [3 d + 1] = (hi [d], lo [d], rstd [d], n) for the backward (nullable; at
 *     inference hi = mm, lo = 0, rstd = rstd_mv).  Training: three launches (chunk sums, fold + moving update,
 *     normalize); ws: tfrs_batch_norm_fwd_workspace_bytes, 16-byte aligned.  Inference: one launch, no workspace.
 *   tfrs_batch_norm_bwd_f32: from dy and the forward's saved: dparams [2, d] = (dgamma, dbeta) = (sum_rows dy xhat,
 *     sum_rows dy) over all rows, xhat = ((x - hi) - lo) rstd; dx [N, d] (nullable) = gamma rstd (dy - w (S1 + xhat S2)
 *     / n) in training (S1 = dbeta, S2 = dgamma), dy gamma rstd_mv at inference.  Training: three launches (chunk
 *     partials, fold, dx); inference: two (chunk partials with dx, fold).  ws: tfrs_batch_norm_bwd_workspace_bytes,
 *     16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
size_t tfrs_batch_norm_fwd_workspace_bytes(int64_t N, int64_t d);
int tfrs_batch_norm_fwd_f32(const float* x, const void* mask, int mask_kind, const float* gamma, const float* beta,
                            int64_t N, int64_t d, int training, double momentum, float eps, float* moving_mean,
                            float* moving_var, float* y, float* saved, void* ws, size_t ws_bytes, void* stream);
size_t tfrs_batch_norm_bwd_workspace_bytes(int64_t N, int64_t d);
int tfrs_batch_norm_bwd_f32(const float* x, const void* mask, int mask_kind, const float* gamma, const float* saved,
                            const float* dy, int64_t N, int64_t d, int training, float* dx, float* dparams, void* ws,
                            size_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFRS_B200_H_ */
