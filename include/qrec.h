/*
 * qrec.h -- C ABI of libqrec.so, the H100 (sm_90a) engine behind QRec's
 * embedding-training hot path.
 *
 * The reference (Coder-Yu/QRec) is pure Python and defines no FFI; its plugin
 * interface is the Recommender class surface.  Every entry point below replaces
 * one reference function on the hot path (cited as file:line relative to the
 * reference checkout) and is what the Python layer (qrec_b200/engine.py, via
 * ctypes) binds.  INTEGRATION.md shows the stub a QRec maintainer would add.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no torch / Python types.
 *   - every function returns int: 0 = QREC_OK, <0 = error; the message is
 *     available from qrec_last_error() (thread-local).  Nothing throws.
 *   - "dev" pointers are CUDA device pointers owned by the caller (in the Python
 *     layer: torch CUDA tensors -> data_ptr()).  The library allocates device
 *     memory only inside an opaque qrec_ctx (pipelined host path workspaces).
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream);
 *     all device entry points are asynchronous on that stream.
 *   - ids are int32 (U + I < 2^31 in every configuration); offsets/counts int64.
 *   - tables are row-major [rows, d], rows contiguous, 16-byte aligned.
 */
#ifndef QREC_H_
#define QREC_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define QREC_OK 0
#define QREC_ERR_ARG (-1)    /* bad argument (null pointer, unsupported d, ...) */
#define QREC_ERR_CUDA (-2)   /* a CUDA runtime call failed; see qrec_last_error */
#define QREC_ERR_STATE (-3)  /* object used in the wrong state */
#define QREC_ERR_NOMEM (-4)

const char* qrec_last_error(void);
/* "qrec-b200 <semver> sm_90a" */
const char* qrec_version(void);
/* number of kernels this library has launched in this process (bench `gpu_launches`) */
int64_t qrec_launch_count(void);

/* =====================================================================================
 * K0 (compat) -- CPython `random` (MT19937) clone, host side, bit exact.
 * Replaces the `random.choice / shuffle / randint / random` calls on the path:
 *   model/ranking/BPR.py:28,35-38   base/deepRecommender.py:30,47-49,69-71
 *   base/iterativeRecommender.py:101   util/dataSplit.py:15
 * State is caller-owned: 624 words + index, the layout of random.getstate()[1].
 * ===================================================================================== */
typedef struct qrec_mt19937 {
  uint32_t mt[624];
  uint32_t index;
} qrec_mt19937;

/* random.seed(int) -- init_by_array over the 32-bit little-endian words of |seed| */
int qrec_mt_seed(qrec_mt19937* st, uint64_t seed);
/* random.setstate / getstate: state625 = 624 words followed by the index */
int qrec_mt_set_state(qrec_mt19937* st, const uint32_t* state625);
int qrec_mt_get_state(const qrec_mt19937* st, uint32_t* state625);
uint32_t qrec_mt_next_u32(qrec_mt19937* st);           /* genrand_uint32            */
double qrec_mt_random(qrec_mt19937* st);               /* random.random()           */
uint32_t qrec_mt_randbelow(qrec_mt19937* st, uint32_t n); /* Random._randbelow(n), n>=1 */
/* random.shuffle applied to perm[0..n) in place (perm holds any int32 payload) */
int qrec_mt_shuffle_i32(qrec_mt19937* st, int64_t n, int32_t* perm);
/* the same swap sequence applied to two parallel arrays (the (user,item) columns of
 * trainingData): base/deepRecommender.py:30, base/iterativeRecommender.py:101 */
int qrec_mt_shuffle_pairs_i32(qrec_mt19937* st, int64_t n, int32_t* a, int32_t* b);
/* util/dataSplit.py:9-26: keep[k] = 0 if random() < test_ratio (goes to test) else 1 */
int qrec_mt_data_split(qrec_mt19937* st, int64_t n, double test_ratio, uint8_t* keep);

/* A user's rated-item set for rejection: CSR over users, column ids SORTED ascending
 * inside each row (membership = binary search).  rowptr has n_users+1 entries. */

/* model/ranking/BPR.py:31-38 -- one epoch of the numpy path's sampler.
 * Iterates users 0..n_users-1 and, per user, its positives in `pos_cols` order (the
 * reference's insertion order, CSR rowptr `pos_rowptr`); draws j = randbelow(num_items)
 * until j is not in the user's sorted positive set.  Emits n = pos_rowptr[n_users]
 * triples.  Users with an empty positive row are skipped (BPR.py:22-25). */
int qrec_sample_bpr_epoch(qrec_mt19937* st, int32_t n_users, int32_t num_items,
                          const int64_t* pos_rowptr, const int32_t* pos_cols,
                          const int64_t* sorted_rowptr, const int32_t* sorted_cols,
                          int32_t* out_u, int32_t* out_i, int32_t* out_j);

/* base/deepRecommender.py:44-50 (and model/ranking/BPR.py:67-74): for each row k of a
 * batch, j[k] = randbelow(num_items) until j not rated by u[k]. */
int qrec_sample_pairwise(qrec_mt19937* st, int64_t n, int32_t num_items, const int32_t* u,
                         const int64_t* sorted_rowptr, const int32_t* sorted_cols,
                         int32_t* out_j);

/* TBPR epoch of preference chains, model/ranking/TBPR.py:131-160 (host): for every listed user and every positive item
 * (insertion order) the chain  i > joint > weak > strong > unobserved  of the levels that exist for the user -- one
 * choice(list) per non-empty level in that order, then choice(item_list) until it is not one of the user's positives --
 * written as the chain's consecutive (u, a, b) steps; the same draws from the same MT19937 stream.  Pools: CSR over
 * user ids, items in list order.  out_u/a/b: capacity 4 * positives of the listed users; out_per_user[k]: steps of
 * order[k]; *out_n: steps written. */
int qrec_sample_tbpr_epoch(qrec_mt19937* st, int32_t n_order, const int32_t* order, int32_t num_items,
                           const int64_t* pos_rowptr, const int32_t* pos_cols, const int64_t* possorted_rowptr,
                           const int32_t* possorted_cols, const int64_t* joint_rowptr, const int32_t* joint_items,
                           const int64_t* weak_rowptr, const int32_t* weak_items, const int64_t* strong_rowptr,
                           const int32_t* strong_items, int32_t* out_u, int32_t* out_a, int32_t* out_b,
                           int64_t* out_per_user, int64_t* out_n);

/* SBPR minibatch rows, model/ranking/SBPR.py:84-100 (host): per row the social item k = choice(list(FPSet[user].keys()))
 * with its friend count S_uk (no social feedback: choice(item_list), weight 0), then the negative j = choice(item_list)
 * until j is neither rated by the user nor in FPSet[user] -- the same draws from the same MT19937 stream.
 * fp_items / fp_counts: every user's FPSet in dict (insertion) order, CSR over user ids; fp_sorted: the same sets
 * ascending (membership test); rated_*: all rated items per user, ascending. */
int qrec_sample_sbpr_batch(qrec_mt19937* st, int64_t n, int32_t num_items, const int32_t* u,
                           const int64_t* rated_rowptr, const int32_t* rated_cols, const int64_t* fp_rowptr,
                           const int32_t* fp_items, const int32_t* fp_counts, const int32_t* fp_sorted,
                           int32_t* out_k, int32_t* out_j, int32_t* out_w);

/* base/deepRecommender.py:65-76: per interaction emit (u,i,1) then 4 x (u, randint(0,I-1)
 * until unrated, 0).  Outputs have 5*n entries. */
int qrec_sample_pointwise(qrec_mt19937* st, int64_t n, int32_t num_items, const int32_t* u,
                          const int32_t* i, const int64_t* sorted_rowptr,
                          const int32_t* sorted_cols, int32_t* out_u, int32_t* out_i,
                          int32_t* out_y);

/* =====================================================================================
 * K0 (fast) -- device sampler: Philox4x32-10 counter RNG + binary-search rejection.
 * Same role as base/deepRecommender.py:47-49 for throughput runs (the MT19937 stream is
 * serial by construction).  j[k] = (philox(seed; k, attempt, epoch).x * num_items) >> 32,
 * attempt = 0,1,... until j is not rated by u[k].  Deterministic in (seed, epoch, k).  A user whose row
 * already contains every item gets the first draw (no valid negative exists; the kernel must not spin).
 * ===================================================================================== */
int qrec_sample_neg_philox(int64_t n, int32_t num_items, const int32_t* dev_u,
                           const int64_t* dev_sorted_rowptr, const int32_t* dev_sorted_cols,
                           uint64_t seed, uint32_t epoch, int32_t* dev_out_j, void* stream);

/* =====================================================================================
 * K1 -- BPR.optimization(u,i,j), model/ranking/BPR.py:45-53 (statement order as there).
 * ===================================================================================== */

/* Native reader of rating files (host; next row f-3): FileIO.loadDataSet (util/io.py:31-76) with the
 * default delimiter set -- strip, split at every single ' ', ',' or tab, optional header, column
 * selection, optional binarisation -- plus the first-appearance id mapping of Rating.__generateSet
 * (data/rating.py:33-54).  col_r < 0: no rating column (every rating 1.0).  Returns NULL with a message
 * in qrec_last_error() for anything it is not sure about (short line, unusual number syntax) so that
 * the caller can fall back to the reference-style Python path. */
typedef struct qrec_text_table qrec_text_table;
qrec_text_table* qrec_text_load(const char* path, int32_t col_u, int32_t col_i, int32_t col_r, int32_t header,
                                int32_t binarize, double threshold);
int64_t qrec_text_rows(const qrec_text_table* t);
int32_t qrec_text_vocab_size(const qrec_text_table* t, int32_t which /* 0 users, 1 items */);
int qrec_text_copy(const qrec_text_table* t, int32_t* u, int32_t* i, double* r);
/* names in id order joined by '\n'; returns the byte count (copies into buf when buf != NULL) */
int64_t qrec_text_names(const qrec_text_table* t, int32_t which, char* buf, int64_t capacity);
void qrec_text_free(qrec_text_table* t);

/* Per-user item sets of an id-mapped interaction list (host; next row f-3): the reference keeps them as
 * a dict of dicts (data/rating.py:48-55), so a repeated (user, item) line keeps the position of its
 * first occurrence and the value of its last.  Outputs (caller-allocated, column arrays of length n):
 *   sorted_rowptr / sorted_cols   every rated item per user, ascending ids (the rejection sets)
 *   pos_rowptr / pos_cols         items with rating >= positive_threshold in insertion order
 *                                 (the iteration order of model/ranking/BPR.py:22-25,31-33)
 *   possorted_cols                the same positives in ascending ids (rows as in pos_rowptr)
 * rating may be null (every rating 1).  Stable counting sort by user + a small sort per user, threaded. */
int qrec_build_rated_csr(int64_t n, const int64_t* u, const int64_t* i, const double* rating,
                         int32_t num_users, int32_t num_items, double positive_threshold,
                         int64_t* sorted_rowptr, int32_t* sorted_cols, int64_t* pos_rowptr,
                         int32_t* pos_cols, int32_t* possorted_cols);

/* Host prepass for the dependency-ordered kernel: for triple k, wait_x[k] = number of
 * earlier triples (k' < k) that touch the same table row (P[u_k]; Q[i_k]; Q[j_k], where a
 * Q row counts touches both as i and as j). */
int qrec_bpr_order_prepare(int64_t n, const int32_t* u, const int32_t* i, const int32_t* j,
                           int32_t num_users, int32_t num_items, int32_t* wait_u,
                           int32_t* wait_i, int32_t* wait_j);

/* Depth of the dependency DAG of the sequential loop (number of levels; n / depth = how many triples
 * are independent on average).  Host, O(n).  Returns -1 on an out-of-range id. */
int64_t qrec_bpr_order_depth(int64_t n, const int32_t* u, const int32_t* i, const int32_t* j,
                             int32_t num_users, int32_t num_items);

/* Parity mode: results identical to running BPR.optimization over the triples in array
 * order (Gauss-Seidel SGD, BPR.py:31-39), executed as a dataflow over the per-row
 * dependency chains.  dev_ver_p / dev_ver_q: int32[num_users] / int32[num_items] row
 * version counters, dev_ticket: uint64[1]; all three must be ZERO on entry.
 * dev_loss: double[1], the kernel ADDS sum_k -ln(s_k) (BPR.py:53).  Any d >= 1 (<= 256).
 * n_warps: number of polling warps (0 = fill the GPU); measured at width 4.6: 73 warps 2.59 s,
 * 2368 warps 2.91 s, 32 warps 4.18 s per 5 M triples -- the per-level latency (~2.5 us) dominates. */
int qrec_bpr_sgd_ordered_f32(float* dev_P, float* dev_Q, int32_t d, int64_t n,
                             const int32_t* dev_u, const int32_t* dev_i, const int32_t* dev_j,
                             const int32_t* dev_wait_u, const int32_t* dev_wait_i,
                             const int32_t* dev_wait_j, int32_t* dev_ver_p, int32_t* dev_ver_q,
                             unsigned long long* dev_ticket, float lr, float reg_u, float reg_i,
                             double* dev_loss, int32_t n_warps, void* stream);
int qrec_bpr_sgd_ordered_f64(double* dev_P, double* dev_Q, int32_t d, int64_t n,
                             const int32_t* dev_u, const int32_t* dev_i, const int32_t* dev_j,
                             const int32_t* dev_wait_u, const int32_t* dev_wait_i,
                             const int32_t* dev_wait_j, int32_t* dev_ver_p, int32_t* dev_ver_q,
                             unsigned long long* dev_ticket, double lr, double reg_u,
                             double reg_i, double* dev_loss, int32_t n_warps, void* stream);

/* Throughput mode: one fused gather -> 2 dots -> sigmoid -> BPR step -> scatter-add kernel.
 * Every triple reads its three rows, applies BPR.py:45-52 to its private copy and adds the
 * row deltas back with 128-bit vector reductions (red.global.add.v4.f32).  Triples that
 * share no row with another in-flight triple get exactly the reference update; rows shared
 * inside a launch receive the SUM of their deltas (atomic, order-free).
 * d must be a multiple of 4, 4 <= d <= 256.  dev_loss: double[1], accumulated. */
int qrec_bpr_sgd_batch_f32(float* dev_P, float* dev_Q, int32_t d, int64_t n,
                           const int32_t* dev_u, const int32_t* dev_i, const int32_t* dev_j,
                           float lr, float reg_u, float reg_i, double* dev_loss, void* stream);

/* Same step and semantics as qrec_bpr_sgd_batch_f32 for d = 64, with the scatter-add done by the
 * bulk-copy (TMA) engine: row deltas are staged in shared memory and reduced into the tables with
 * cp.reduce.async.bulk...add.f32 (one 256-byte operation per row) instead of per-lane REDG. */
int qrec_bpr_sgd_batch_tma_f32(float* dev_P, float* dev_Q, int32_t d, int64_t n,
                               const int32_t* dev_u, const int32_t* dev_i, const int32_t* dev_j,
                               float lr, float reg_u, float reg_i, double* dev_loss, void* stream);

/* Throughput mode in the reference's own order (model/ranking/BPR.py:31-33: users in id order, each
 * user's positives in CSR order): a lane group keeps P[u] in registers across the user's triples, so
 * P[u] is updated sequentially inside a user -- as in the reference -- and read/written once per
 * user; the item rows are gathered and scatter-added per triple (atomic sum across users).
 * rowptr: int64[n_users+1]; i, j: int32[n], n = rowptr[n_users], in that order; num_items = rows of Q.
 * Every user is processed whole by one lane group; the stream is swept in waves, each reading the item
 * table as the earlier waves left it, so the result does not depend on timing (up to the summation order
 * of the scatter-adds).  d multiple of 4, <= 128. */
int qrec_bpr_sgd_usermajor_f32(float* dev_P, float* dev_Q, int32_t d, int32_t n_users, int64_t n, int32_t num_items,
                               const int64_t* dev_rowptr, const int32_t* dev_i, const int32_t* dev_j,
                               float lr, float reg_u, float reg_i, double* dev_loss, void* stream);

/* One whole epoch of the numpy path (model/ranking/BPR.py:29-39) in a single launch: the user-major
 * kernel above with the negative sampling fused in.  Lane l of a lane group draws the negative of its
 * triple k with Philox counter (k, attempt, epoch) -- exactly what qrec_sample_neg_philox produces
 * for (u[k], k) -- rejecting items in the user's sorted rated row; j never touches HBM unless
 * dev_j_out is given.  rated_rowptr/rated_cols: CSR of the rejection sets (may equal rowptr's). */
int qrec_bpr_epoch_usermajor_f32(float* dev_P, float* dev_Q, int32_t d, int32_t n_users, int64_t n,
                                 const int64_t* dev_rowptr, const int32_t* dev_i,
                                 const int64_t* dev_rated_rowptr, const int32_t* dev_rated_cols,
                                 int32_t num_items, uint64_t seed, uint32_t epoch, int32_t* dev_j_out,
                                 float lr, float reg_u, float reg_i, double* dev_loss, void* stream);

/* The fused epoch with a pre-test in the sampler: rated_sig holds 16 words per user, bit (c & 511) set
 * for every rated column c (qrec_rated_signature_build; static per data set).  A clear bit proves a
 * draw is not rated, so about 1 - deg/512 of the draws skip the binary search -- the dependent-load
 * chain of the sampler.  No false negatives:
 * the negatives, hence P and Q, are identical to qrec_bpr_epoch_usermajor_f32.  d in {16,32,64,128}. */
int qrec_rated_signature_build(int32_t n_users, const int64_t* dev_rated_rowptr, const int32_t* dev_rated_cols,
                               uint32_t* dev_sig, void* stream);
int qrec_bpr_epoch_usermajor_sig_f32(float* dev_P, float* dev_Q, int32_t d, int32_t n_users, int64_t n,
                                     const int64_t* dev_rowptr, const int32_t* dev_i,
                                     const int64_t* dev_rated_rowptr, const int32_t* dev_rated_cols,
                                     const uint32_t* dev_rated_sig, int32_t num_items, uint64_t seed,
                                     uint32_t epoch, int32_t* dev_j_out, float lr, float reg_u, float reg_i,
                                     double* dev_loss, void* stream);

/* K1 for a row-sharded item table (SURVEY 8e, K7): the Q rows of the batch were fetched from their
 * owner ranks into dev_R (row pos_i[k] / pos_j[k] holds Q[i_k] / Q[j_k]).  Applies BPR.py:45-52,
 * updates P in place and writes the item-row deltas to dev_D at the same positions, ready to be
 * returned to the owners and scatter-added (qrec_scatter_add_rows_f32).  d multiple of 4, <= 128. */
int qrec_bpr_sgd_staged_f32(float* dev_P, int32_t d, int64_t n, const int32_t* dev_u,
                            const int32_t* dev_pos_i, const int32_t* dev_pos_j, const float* dev_R,
                            float* dev_D, float lr, float reg_u, float reg_i, double* dev_loss,
                            void* stream);

/* regU*sum(P*P) + regI*sum(Q*Q) building block (BPR.py:40): dev_out[0] += sum(x[k]^2). */
int qrec_sumsq_f32(const float* dev_x, int64_t n, double* dev_out, void* stream);
int qrec_sumsq_f64(const double* dev_x, int64_t n, double* dev_out, void* stream);

/* dev_dst[0 .. n) = dev_src[0 .. n): the item-table snapshot the user-major epoch takes before each wave (both
 * tables kept in L2 at evict_last).  n a multiple of 4, both pointers 16-byte aligned, no overlap. */
int qrec_table_snapshot_f32(const float* dev_src, float* dev_dst, int64_t n, void* stream);

/* =====================================================================================
 * Replicated item table across GPUs (SURVEY 8e, BPR throughput mode: users range-partitioned, Q
 * replicated; the data-parallel form of the in-place item updates of BPR.py:50-52).  B is the table all
 * ranks agreed on at the last exchange.  delta: D = Q - B (and S = D when S != NULL), one read of Q per
 * element while K1 may keep RED-adding into it.  merge: Q += S - D with float atomics, B += S, where S is
 * the sum of all ranks' D -- so updates that landed in Q after delta read it stay in Q - B and travel with
 * the next exchange; K1 never waits.  The two *_p2p entry points are the exchange itself over peer
 * memory (NVLink P2P loads; peer_* are host arrays of `world` device pointers to the ranks' symmetric
 * buffers): reduce-scatter of D into this rank's slice of S, then all-gather fused with the merge.
 * The caller separates the phases with a cross-rank barrier.  n multiple of 4, pointers 16-byte aligned.
 * ===================================================================================== */
int qrec_table_delta_f32(const float* dev_Q, const float* dev_B, float* dev_D, float* dev_S, int64_t n, void* stream);
int qrec_table_merge_f32(float* dev_Q, float* dev_B, const float* dev_D, const float* dev_S, int64_t n, void* stream);
int qrec_table_reduce_scatter_p2p_f32(const float* const* peer_D, int32_t world, int32_t rank, float* dev_S, int64_t n,
                                      void* stream);
int qrec_table_gather_merge_p2p_f32(const float* const* peer_S, int32_t world, float* dev_Q, float* dev_B,
                                    const float* dev_D, int64_t n, void* stream);

/* K8 (SURVEY 8f-1): batched ranking evaluation, replaces the per-user loop of Recommender.evalRanking
 * (base/recommender.py:143-152) + find_k_largest (util/qmath.py:134-146).  For every row r of the block:
 * scores = V . U[user_ids[r]] (fp32), rated items of that user (sorted CSR) score `rated_value` (the reference
 * writes 0, it does not remove them), the N best (score descending, ties by ascending item id) go to
 * out_ids / out_scores [n_rows, N].  The score matrix is never materialised.  1 <= N <= 100. */
int qrec_score_topn_f32(const float* dev_U, const float* dev_V, int32_t d, int32_t n_items,
                        const int32_t* dev_user_ids, int32_t n_rows, const int64_t* dev_rated_rowptr,
                        const int32_t* dev_rated_cols, float rated_value, int32_t N, int32_t* dev_out_ids,
                        float* dev_out_scores, void* stream);
/* The same contract with the scores computed on the tensor cores: wgmma TF32, error-compensated
 * (3xTF32: hi.hi + lo.hi + hi.lo of operands split into two TF32 values), fp32 accumulators in registers parked in
 * shared memory for the selection code -- fp32-level scores (2^-22 relative per product).
 * d <= 64 and a multiple of 4; tables 16-byte aligned.  csrc/topn_tc.cu. */
int qrec_score_topn_tc_f32(const float* dev_U, const float* dev_V, int32_t d, int32_t n_items,
                           const int32_t* dev_user_ids, int32_t n_rows, const int64_t* dev_rated_rowptr,
                           const int32_t* dev_rated_cols, float rated_value, int32_t N, int32_t* dev_out_ids,
                           float* dev_out_scores, void* stream);

/* =====================================================================================
 * f-2 -- the normalised joint adjacency and its per-epoch edge-dropout rebuild on the device
 * (base/graphRecommender.py:10-29; model/ranking/SGL.py:113-155, aug_type 1).  The joint CSR of the full graph
 * (rowptr int64[n_rows+1], cols int32 sorted per row) is built once; `pair` int32[nnz] maps every stored entry to
 * its undirected edge so that (u,i) and (i,u) share a weight; pair_w fp32[n_pairs] is the edge multiplicity
 * (number of kept interaction lines, duplicates summed like scipy's constructor; 0 = dropped).
 * ===================================================================================== */
/* deg[r] = sum of row r's weights; vals[e] = (deg_r^-1/2 * w) * deg_c^-1/2 in fp32 (isolated nodes: 0).
 * pair / pair_w may both be NULL (all weights 1). */
int qrec_adj_normalize_f32(int32_t n_rows, const int64_t* dev_rowptr, const int32_t* dev_cols, const int32_t* dev_pair,
                           const float* dev_pair_w, float* dev_deg, float* dev_vals, void* stream);
/* keep[k] = Philox-uniform(k; tag, epoch, seed) >= drop_rate, one flag per interaction line. */
int qrec_edge_keep_philox(int64_t n_lines, float drop_rate, uint64_t seed, uint32_t tag, uint32_t epoch,
                          uint8_t* dev_keep, void* stream);
/* pair_w[p] = number of lines k with line_pair[k] == p and keep[k] != 0 (keep NULL: all lines). */
int qrec_adj_line_weights_f32(int64_t n_lines, const int32_t* dev_line_pair, const uint8_t* dev_keep, int64_t n_pairs,
                              float* dev_pair_w, void* stream);
/* Sub-graph of the edges with pair_w > 0: degrees into dev_deg, the new row pointer into dev_new_rowptr
 * (int64[n_rows+1], exclusive scan of the surviving entries per row).  scan_scratch: int64[ceil((n_rows+1)/1024)]. */
int qrec_adj_subgraph_count(int32_t n_rows, const int64_t* dev_rowptr, const int32_t* dev_pair, const float* dev_pair_w,
                            float* dev_deg, int64_t* dev_new_rowptr, int64_t* dev_scan_scratch, void* stream);
/* Ordered compaction of the surviving entries (the CSR stays sorted) with the sub-graph's own D^-1/2 scaling. */
int qrec_adj_subgraph_fill_f32(int32_t n_rows, const int64_t* dev_rowptr, const int32_t* dev_cols, const int32_t* dev_pair,
                               const float* dev_pair_w, const float* dev_deg, const int64_t* dev_new_rowptr,
                               int32_t* dev_new_cols, float* dev_new_vals, void* stream);

/* Measurement aid for the K1 roofline (bench.py "row_op_peak"; not on the product path): issues
 * n_ops 256-byte row operations against random rows of dev_table [rows, 64] fp32 with nothing else in
 * the loop -- mode 0: LDG.E.128 gathers, 1: REDG.E.ADD.F32x4 scatter-adds (value 1e-9 alternating in
 * sign), 2: one gather + one scatter-add per op (K1's mix on the item table, BPR.py:45-52). */
int qrec_ubench_row_ops_f32(float* dev_table, int64_t rows, int64_t n_ops, int32_t mode, uint32_t seed,
                            float* dev_sink, void* stream);

/* =====================================================================================
 * Pipelined host entry (what trainModel calls when the triples live in HOST memory):
 * chunks the index arrays, overlaps H2D copies (copy stream) with the K1 kernel (compute
 * stream) through a ring of device staging buffers owned by the ctx, returns the loss.
 * ===================================================================================== */
typedef struct qrec_ctx qrec_ctx;
int qrec_ctx_create(int device, int64_t chunk_triples, qrec_ctx** out);
int qrec_ctx_destroy(qrec_ctx* ctx);
/* Optional: the rated-set signatures of ALL users ([n_users, 16] words, qrec_rated_signature_build) for the fused
 * sampler's pre-test in qrec_bpr_epoch_usermajor_host (same negatives, fewer dependent loads); NULL switches it off.
 * The array must stay alive while the ctx uses it. */
int qrec_ctx_set_rated_signature(qrec_ctx* ctx, const uint32_t* dev_rated_sig);
/* host u/i/j: pinned memory gives true overlap; pageable memory works but serialises.
 * *host_loss receives sum_k -ln(s_k) of this call.  Synchronous on return. */
int qrec_bpr_epoch_host(qrec_ctx* ctx, float* dev_P, float* dev_Q, int32_t d, int64_t n,
                        const int32_t* host_u, const int32_t* host_i, const int32_t* host_j,
                        float lr, float reg_u, float reg_i, double* host_loss);

/* The same pipeline for a user-major epoch (the reference's loop order): the positives live in HOST
 * memory as CSR (host_rowptr int64[n_users+1], host_i int32[n]); chunks of whole users are copied while
 * the fused sampling+SGD kernel (qrec_bpr_epoch_usermajor_f32) runs the previous chunk.  Negatives are
 * drawn on the device against the resident rejection CSR.  No user may have more positives than the
 * ctx chunk size.  Synchronous on return. */
int qrec_bpr_epoch_usermajor_host(qrec_ctx* ctx, float* dev_P, float* dev_Q, int32_t d, int32_t n_users,
                                  const int64_t* host_rowptr, const int32_t* host_i,
                                  const int64_t* dev_rated_rowptr, const int32_t* dev_rated_cols,
                                  int32_t num_items, uint64_t seed, uint32_t epoch, float lr,
                                  float reg_u, float reg_i, double* host_loss);

/* =====================================================================================
 * K2 -- Y = A * X for the normalised joint adjacency, CSR, fp32 values, int32 columns.
 * Replaces tf.sparse_tensor_dense_matmul(norm_adj, E): model/ranking/LightGCN.py:17,
 * model/ranking/NGCF.py:28, model/ranking/SimGCL.py:25,33.  A is symmetric, so the same
 * call is the backward pass.  Optional fused layer accumulation (LightGCN.py:19):
 * if dev_acc != NULL, acc[r,:] += acc_scale * Y[r,:].  d multiple of 4, <= 256.
 * nnz = rowptr[n_rows] (passed by value so the launch needs no device read-back).
 * ===================================================================================== */
int qrec_spmm_csr_f32(int32_t n_rows, int64_t nnz, const int64_t* dev_rowptr, const int32_t* dev_cols,
                      const float* dev_vals, const float* dev_X, float* dev_Y, int32_t d,
                      float* dev_acc, float acc_scale, void* stream);
/* Same product with plain row partitioning (one lane group per row, no atomics, bit-reproducible
 * summation order).  qrec_spmm_csr_f32 balances by non-zeros instead and is the default.  d = 64 runs
 * its own specialisation (a half warp per row, 8 gathered rows in flight per lane, 4 CTAs per SM). */
int qrec_spmm_csr_rowsplit_f32(int32_t n_rows, int64_t nnz, const int64_t* dev_rowptr, const int32_t* dev_cols,
                               const float* dev_vals, const float* dev_X, float* dev_Y, int32_t d,
                               float* dev_acc, float acc_scale, void* stream);

/* Sparse-source product (the first backward layer of a minibatch step: the loss gradient touches at
 * most 3B rows).  (rowptr, cols, vals) is a CSR whose ROWS are source nodes and whose column ids index
 * rows of Y; Y (n_rows rows) is zero-filled here, then Y[c] += a_rc X[r] over the edges of the n_src
 * listed source rows r; optional acc[c] += acc_scale * a_rc X[r].  With the symmetric joint adjacency
 * this is Y = A X for an X that is non-zero only in the listed rows. */
int qrec_spmm_csr_scatter_rows_f32(int32_t n_rows, int32_t n_src, const int32_t* dev_src_rows,
                                   const int64_t* dev_rowptr, const int32_t* dev_cols,
                                   const float* dev_vals, const float* dev_X, float* dev_Y, int32_t d,
                                   float* dev_acc, float acc_scale, void* stream);

/* Pull-side product on a list of OUTPUT rows (the last forward layer of a minibatch step: the loss of
 * model/ranking/LightGCN.py:22-26 reads the propagated embeddings of the batch's rows only).  For k < n_list with
 * r = rows[k] >= 0:  s = sum_e a_e X[col_e] over CSR row r;  Y[compact ? k : r] = s (Y may be NULL);
 * acc[r] += acc_scale * s (acc may be NULL; the listed rows must then be distinct).  Entries r = -1 are padding:
 * skipped, their row of a compact Y is zero-filled.  d % 4 == 0, d <= 128. */
int qrec_spmm_csr_rows_f32(int32_t n_list, const int32_t* dev_rows, const int64_t* dev_rowptr,
                           const int32_t* dev_cols, const float* dev_vals, const float* dev_X, float* dev_Y,
                           int32_t compact, int32_t d, float* dev_acc, float acc_scale, void* stream);

/* =====================================================================================
 * K3 -- gather rows of the propagated tables, bpr_loss + batch L2 and its gradient,
 * scatter-added into dense gradient buffers.  util/loss.py:3-6, LightGCN.py:22-24,28-30.
 *   y = u.p - u.n ; s = sigmoid(y) ; loss += -ln(s + eps) + reg*0.5*(|u|^2+|p|^2+|n|^2)
 *   dL/dy = -s(1-s)/(s+eps)
 *   gU[u] += dL/dy*(p-n) + reg*u ; gV[i] += dL/dy*u + reg*p ; gV[j] += -dL/dy*u + reg*n
 * dev_gU/dev_gV must be zeroed by the caller.  dev_loss: double[1], accumulated.
 * ===================================================================================== */
int qrec_bpr_grad_scatter_f32(const float* dev_U, const float* dev_V, int32_t d, int64_t n,
                              const int32_t* dev_u, const int32_t* dev_i, const int32_t* dev_j,
                              float eps, float reg, float* dev_gU, float* dev_gV,
                              double* dev_loss, void* stream);

/* K3 with a per-sample score scale c_k: the term is -ln(sigmoid(c_k y_k) + eps), dL/dy = -c s(1-s)/(s+eps) with
 * s = sigmoid(c_k y_k).  Replaces the first term of SBPR's minibatch loss, model/ranking/SBPR.py:110-113
 * (y_ik / (weights + 1): c_k = 1 / (S_uk + 1), the number of friends who consumed the social item k); the second term
 * (y_kj) is qrec_bpr_grad_scatter_f32 on (u, k, j).  dev_y_scale: float[n]. */
int qrec_bpr_grad_scatter_scaled_f32(const float* dev_U, const float* dev_V, int32_t d, int64_t n,
                                     const int32_t* dev_u, const int32_t* dev_i, const int32_t* dev_j,
                                     const float* dev_y_scale, float eps, float reg, float* dev_gU, float* dev_gV,
                                     double* dev_loss, void* stream);

/* The same step for ranks that each hold a COLUMN block of the tables (feature-parallel LightGCN: the propagation
 * A X is independent per column, so d/world columns of every row live on each rank and the only exchange of a
 * minibatch step is the sum of these partial scores).  d = the LOCAL width.
 *   partial scores: y_part[k] = sum over the local columns of U[u_k].(V[i_k] - V[j_k]); the local part of the batch L2
 *                   term (reg/2 * squared norms) is added to *loss.
 *   gradients     : given y_full = the ranks' y_part summed, scatter-adds the gradient of the local columns into gU / gV
 *                   exactly like qrec_bpr_grad_scatter_f32 and adds log_weight * sum_k -ln(sigmoid(y_k) + eps) to *loss
 *                   (log_weight = 1 on one rank, 0 on the others: the term is a function of the full score). */
int qrec_bpr_partial_scores_f32(const float* dev_U, const float* dev_V, int32_t d, int64_t n, const int32_t* dev_u,
                                const int32_t* dev_i, const int32_t* dev_j, float reg, float* dev_y_part,
                                double* dev_loss, void* stream);
int qrec_bpr_grad_from_scores_f32(const float* dev_U, const float* dev_V, int32_t d, int64_t n, const int32_t* dev_u,
                                  const int32_t* dev_i, const int32_t* dev_j, const float* dev_y_full, float eps,
                                  float reg, float log_weight, float* dev_gU, float* dev_gV, double* dev_loss,
                                  void* stream);

/* =====================================================================================
 * K4 -- tf.train.AdamOptimizer (TF 1.14) dense update over a whole variable:
 * LightGCN.py:31-32, NGCF.py:54, SimGCL.py:99, BPR.py:84.
 *   lr_t = lr*sqrt(1-b2^t)/(1-b1^t); m += (g-m)(1-b1); v += (g*g-v)(1-b2);
 *   var -= (m*lr_t) / (sqrt(v) + eps)            (t = 1-based step count; fp32 throughout)
 * ===================================================================================== */
int qrec_adam_dense_tf1_f32(float* dev_var, float* dev_m, float* dev_v, const float* dev_g,
                            int64_t n, float lr, float beta1, float beta2, float eps,
                            int64_t t, void* stream);
/* The same update with the step-dependent factor lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t) read from device
 * memory at run time: a training step captured in a CUDA graph replays with a new t without re-capturing. */
int qrec_adam_dense_tf1_devstep_f32(float* dev_var, float* dev_m, float* dev_v, const float* dev_g, int64_t n,
                                    const float* dev_lr_t, float beta1, float beta2, float eps, void* stream);

/* Layer mean helper (LightGCN.py:19): dst[k] = scale * (a[k] + b[k]); dst may alias a. */
int qrec_axpby_f32(float* dev_dst, const float* dev_a, const float* dev_b, float alpha,
                   float beta, int64_t n, void* stream);

/* =====================================================================================
 * K6 -- SimGCL pieces (model/ranking/SimGCL.py:30-38,60-78) and the small dense helpers of
 * NGCF (model/ranking/NGCF.py:27-41).  All fp32, row-major, d multiple of 4 where noted.
 * ===================================================================================== */

/* SimGCL.py:33-35: E += sign(E) * l2_normalize(U[0,1)^d, axis=1) * eps, in place.  The uniform
 * noise of element (row r, column c) is word (c & 3) of Philox4x32-10(key = seed;
 * counter = (r, c >> 2, tag, step)), mapped to [0,1) as (w >> 8) * 2^-24 -- `tag` separates
 * encoders/layers, `step` minibatches (tf.random.uniform draws fresh noise per sess.run).
 * Optional fused layer mean: acc[r,:] += acc_scale * E_new[r,:].  d multiple of 4; columns
 * >= d_valid (zero padding of a table whose logical width is not a multiple of 4) get no noise. */
int qrec_simgcl_perturb_f32(float* dev_E, int64_t n_rows, int32_t d, int32_t d_valid, float eps, uint64_t seed,
                            uint32_t tag, uint32_t step, float* dev_acc, float acc_scale,
                            void* stream);
/* The same perturbation for a block of rows of a ROW-SHARDED table: the noise of local row r is that of global
 * row row_offset + r, so a sharded run draws exactly the single-GPU run's noise (SURVEY 8e, config 5). */
int qrec_simgcl_perturb_rows_f32(float* dev_E, int64_t n_rows, int64_t row_offset, int32_t d, int32_t d_valid,
                                 float eps, uint64_t seed, uint32_t tag, uint32_t step, float* dev_acc,
                                 float acc_scale, void* stream);
/* The same perturbation for a LIST of rows held compactly: row k of dev_Ec ([n_list, d], e.g. the compact output of
 * qrec_spmm_csr_rows_f32) stands for table row dev_rows[k] (global row row_offset + dev_rows[k]); entries -1 are
 * skipped.  Ec[k] is perturbed in place and acc[dev_rows[k]] += acc_scale * Ec[k] (the last encoder layer of a
 * minibatch step, of which the losses of model/ranking/SimGCL.py:60-78,92-96 read the batch's rows only). */
int qrec_simgcl_perturb_listed_f32(float* dev_Ec, const int32_t* dev_rows, int64_t n_list, int64_t row_offset,
                                   int32_t d, int32_t d_valid, float eps, uint64_t seed, uint32_t tag, uint32_t step,
                                   float* dev_acc, float acc_scale, void* stream);

/* Z[r,:] = l2_normalize(T[idx[r],:]) (tf.nn.l2_normalize, epsilon 1e-12 on the squared norm);
 * norms[r] = the divisor.  SimGCL.py:61-69. */
int qrec_gather_normalize_f32(const float* dev_T, const int32_t* dev_idx, int32_t n, int32_t d,
                              float* dev_Z, float* dev_norms, void* stream);

/* InfoNCE over an n x n matrix of raw dots S_ij = z1_i . z2_j (SimGCL.py:70-78):
 * loss[0] += sum_i (log sum_j exp(S_ij/tau) - S_ii/tau);  S_ij <- dLoss/dS_ij. */
int qrec_infonce_rows_f32(float* dev_S, int32_t n, float tau, double* dev_loss, void* stream);

/* Gradient through the row normalisation, added into the dense gradient buffer:
 * G[idx[r],:] += scale * (dZ_r - Z_r (Z_r . dZ_r)) / norms[r]. */
int qrec_normalize_bwd_scatter_f32(const float* dev_dZ, const float* dev_Z, const float* dev_norms,
                                   const int32_t* dev_idx, int32_t n, int32_t d, float scale,
                                   float* dev_G, void* stream);

/* C[M,N] = alpha * op(A) * op(B) + beta * C, row-major fp32 (op = transpose when the flag is
 * non-zero).  tf.matmul at NGCF.py:29,31 and SimGCL.py:70-71 -- bandwidth-sized products. */
int qrec_sgemm_f32(int32_t trans_a, int32_t trans_b, int32_t M, int32_t N, int32_t K, float alpha,
                   const float* dev_A, int32_t lda, const float* dev_B, int32_t ldb, float beta,
                   float* dev_C, int32_t ldc, void* stream);

/* NGCF.py:32-40 forward: H = dropout(leaky_relu(Z, 0.2), keep) (training only; Philox mask,
 * counter (r, c>>2, tag, step)), out = l2_normalize(H) written with row stride ld_out (a column
 * block of the concatenated [N, 3d] table, NGCF.py:42), norms = divisor. */
int qrec_ngcf_act_fwd_f32(const float* dev_Z, int64_t n_rows, int32_t d, float keep,
                          int32_t training, uint64_t seed, uint32_t tag, uint32_t step,
                          float* dev_H, float* dev_out, int32_t ld_out, float* dev_norms,
                          void* stream);
/* ... and its backward: dZ from dOut (w.r.t. the normalised output) and the optional dH_extra
 * (w.r.t. H through the next layer). */
int qrec_ngcf_act_bwd_f32(const float* dev_dOut, int32_t ld_dout, const float* dev_dH_extra, const float* dev_H,
                          const float* dev_Z, const float* dev_norms, int64_t n_rows, int32_t d,
                          float keep, int32_t training, uint64_t seed, uint32_t tag, uint32_t step,
                          float* dev_dZ, void* stream);
/* dst = a * b elementwise (the bi-interaction term ego (.) side, NGCF.py:30). */
int qrec_mul_f32(float* dev_dst, const float* dev_a, const float* dev_b, int64_t n, void* stream);

/* =====================================================================================
 * K5 building block -- tensor-core GEMM for NeuMF's MLP (model/ranking/NeuMF.py:39-50):
 *   C[M,N] = epilogue(A[M,K] * B), fp32 storage, TF32 wgmma with fp32 accumulation in registers.
 * b_is_nk = 0: B is [K,N] row-major (a weight matrix, forward pass);
 * b_is_nk = 1: B is [N,K] row-major (dX = dY * W^T uses W as stored).
 * epilogue: 0 none | 1 relu(x + bias[n]) | 2 x * (mask[m,n] > 0) (ReLU backward) | 3 x + bias[n].
 * A 16-byte aligned, K % 4 == 0, lda % 4 == 0.
 * ===================================================================================== */
int qrec_tc_gemm_tf32(int32_t b_is_nk, int32_t M, int32_t N, int32_t K, const float* dev_A,
                      int32_t lda, const float* dev_B, int32_t ldb, float* dev_C, int32_t ldc,
                      int32_t epilogue, const float* dev_bias, const float* dev_mask,
                      int32_t ldmask, void* stream);
/* The same product through a persistent, warp-specialised pipeline: one CTA per SM keeps a 64-column
 * block of B resident in shared memory, A arrives by TMA (cp.async.bulk.tensor.2d, SWIZZLE_128B tensor
 * map) through a 4-stage mbarrier ring, two consumer warpgroups take the row tiles in turn (wgmma,
 * accumulators in registers) and write their epilogues while the other multiplies.  Same arguments and epilogues; K <= 320, N <= 64 x #SMs.
 * A is consumed as raw fp32 bits (TF32 truncation, error <= 2^-10 per operand; v1 rounds to nearest). */
int qrec_tc_gemm_tf32_v2(int32_t b_is_nk, int32_t M, int32_t N, int32_t K, const float* dev_A,
                         int32_t lda, const float* dev_B, int32_t ldb, float* dev_C, int32_t ldc,
                         int32_t epilogue, const float* dev_bias, const float* dev_mask,
                         int32_t ldmask, void* stream);

/* =====================================================================================
 * K5 -- NeuMF (model/ranking/NeuMF.py:12-123): row gather / scatter-add around the tensor-core
 * MLP and the three prediction heads with their BCE losses.
 * ===================================================================================== */
/* out[b, 0:d] = T[idx[b], :], output rows ld_out apart (tf.nn.embedding_lookup + tf.concat,
 * NeuMF.py:27-30,41). */
int qrec_gather_rows_f32(const float* dev_T, const int32_t* dev_idx, int64_t n, int32_t d,
                         float* dev_out, int32_t ld_out, void* stream);
/* G[idx[b], :] += scale * src[b, 0:d] (IndexedSlices gradient, duplicates summed). */
int qrec_scatter_add_rows_f32(float* dev_G, const int32_t* dev_idx, int64_t n, int32_t d,
                              const float* dev_src, int32_t ld_src, float scale, void* stream);
/* K7 (SURVEY 8e, row-sharded item table): device-side bucketing of the 2n item requests of a minibatch by owner
 * rank (owner = id / rows_per_rank) into FIXED-capacity buckets, so that the id / row / delta exchanges are
 * equal-split all-to-alls with no host round trip.  send[world*cap] receives the owner-local row ids (-1 = empty
 * slot; qrec_gather_rows_f32 returns zeros for it, qrec_scatter_add_rows_f32 skips it), pos[k] the slot of request
 * k (= the row of the fetched block it will read and the delta block it will write).  *overflow is set when a
 * bucket needs more than `cap` slots (the step is then invalid). */
int qrec_bucket_requests(const int32_t* dev_ids, int64_t n, int32_t rows_per_rank, int32_t world, int32_t cap,
                         int32_t* dev_count, int32_t* dev_send, int32_t* dev_pos, int32_t* dev_overflow, void* stream);
/* out[c] = beta*out[c] + alpha * sum_b A[b, c] * v[b] (v NULL: column sums; beta 0 or 1): the bias gradients
 * (tf.reduce_sum over the batch) and head-vector gradients of NeuMF.py:39-57 without a tiled GEMM. */
int qrec_gemv_t_f32(const float* dev_A, int32_t lda, int64_t rows, int32_t cols, const float* dev_v, float alpha,
                    float beta, float* dev_out, void* stream);
/* mode 0 GMF | 1 MLP | 2 NeuMF head: y = sigmoid(wg*(UG*IG).h_mf + wm*H3.h_mlp); when training,
 * loss += BCE(r, y; +1e-9) [+ reg*l2_loss(UG)+reg*l2_loss(IG), modes 0/2], dz = dLoss/dz, and the
 * per-sample gradients GMF=UG*IG, dUG, dIG (incl. reg), dH3 (ReLU-masked).  The h-vector terms of
 * the regulariser and all weight gradients are assembled by the caller from dz/GMF/dH3. */
int qrec_neumf_head_f32(int32_t mode, int32_t training, const float* dev_UG, const float* dev_IG,
                        const float* dev_H3, const float* dev_h_mf, const float* dev_h_mlp,
                        const float* dev_r, int64_t n, int32_t d, float reg, double* dev_loss,
                        float* dev_y, float* dev_dz, float* dev_GMF, float* dev_dUG, float* dev_dIG,
                        float* dev_dH3, void* stream);

/* =====================================================================================
 * K8 (next row f-1) -- batched evaluation helpers: scores = P[users] * Q^T comes from
 * qrec_sgemm_f32 (fp32, so the ranking matches the reference's GEMV to rounding), then the rated
 * positions are overwritten with `value` (0 in the reference: base/recommender.py:147-149,
 * base/iterativeRecommender.py:126-128).  rowptr/cols: the users' rated-item CSR.
 * ===================================================================================== */
int qrec_mask_rated_f32(float* dev_scores, int32_t n_rows, int64_t ld, const int32_t* dev_users,
                        const int64_t* dev_rowptr, const int32_t* dev_cols, float value,
                        void* stream);

/* =====================================================================================
 * K9 (next row f-4) -- the rating-prediction MF family: one entry (u, i, r) per step.
 *   kind 0  BasicMF  model/rating/BasicMF.py:13-23   P[u] += (lr*e)*Q[i];  Q[i] += (lr*e)*P[u]
 *   kind 1  PMF      model/rating/PMF.py:13-22       P[u] += lr*(e*Q[i]-regU*P[u]);  Q[i] += lr*(e*P[u]-regI*Q[i])
 *   kind 2  SVD      model/rating/SVD.py:17-32,84-90 kind 1 with e taken against P.Q + mean + Bi[i] + Bu[u]
 *                                                    and Bu[u] += lr*(e-regB*Bu[u]), Bi[i] likewise
 * e = r - prediction; the item row is updated from the NEW user row (`p` is a view in the reference).
 * dev_loss: double[1], accumulates sum e^2.  Bias pointers may be null unless kind == 2.
 * ===================================================================================== */
/* wait_u[k] / wait_i[k] = number of earlier entries touching P[u[k]] / Q[i[k]] (host, O(n)). */
int qrec_mf_order_prepare(int64_t n, const int32_t* u, const int32_t* i, int32_t num_users,
                          int32_t num_items, int32_t* wait_u, int32_t* wait_i);
/* Length of the longest dependency chain of the stream (n / depth = average parallel width). */
int64_t qrec_mf_order_depth(int64_t n, const int32_t* u, const int32_t* i, int32_t num_users,
                            int32_t num_items);
/* Parity mode: sequential-equivalent epoch (dataflow over row versions, see qrec_bpr_sgd_ordered_*).
 * ver_p[num_users], ver_q[num_items], ticket[1] must be zero on entry. */
int qrec_mf_sgd_ordered_f64(int32_t kind, double* dev_P, double* dev_Q, int32_t d, int64_t n,
                            const int32_t* dev_u, const int32_t* dev_i, const double* dev_r,
                            const int32_t* dev_wait_u, const int32_t* dev_wait_i, int32_t* dev_ver_p,
                            int32_t* dev_ver_q, unsigned long long* dev_ticket, double lr, double reg_u,
                            double reg_i, double* dev_Bu, double* dev_Bi, double reg_b, double global_mean,
                            double* dev_loss, int32_t n_warps, void* stream);
int qrec_mf_sgd_ordered_f32(int32_t kind, float* dev_P, float* dev_Q, int32_t d, int64_t n,
                            const int32_t* dev_u, const int32_t* dev_i, const float* dev_r,
                            const int32_t* dev_wait_u, const int32_t* dev_wait_i, int32_t* dev_ver_p,
                            int32_t* dev_ver_q, unsigned long long* dev_ticket, float lr, float reg_u,
                            float reg_i, float* dev_Bu, float* dev_Bi, float reg_b, float global_mean,
                            double* dev_loss, int32_t n_warps, void* stream);
/* Throughput mode: every entry reads its two rows, applies the step to its private copy and adds the
 * row deltas back with red.global.add.v4.f32 (rows shared inside a launch get the sum of the deltas).
 * d: multiple of 4, 4..128 (pad with zero columns; they stay zero).
 * max_inflight: 0 = fill the GPU; > 0 = size the grid so that about this many entries sit between
 * their row reads and their reductions at any time.  A row hit c times inside that window moves as
 * with c*lr (every hit reads the same stale row) and the squared-error gradient is unbounded, so
 * small or skewed data needs a window of roughly (0.25/lr) / (share of the most frequent row). */
int qrec_mf_sgd_batch_f32(int32_t kind, float* dev_P, float* dev_Q, int32_t d, int64_t n,
                          const int32_t* dev_u, const int32_t* dev_i, const float* dev_r, float lr,
                          float reg_u, float reg_i, float* dev_Bu, float* dev_Bi, float reg_b,
                          float global_mean, double* dev_loss, int64_t max_inflight, void* stream);
/* out[k] = P[u[k]].Q[i[k]]  (+ global_mean + Bi[i[k]] + Bu[u[k]] when the bias vectors are given):
 * predictForRating for known (user, item) pairs (iterativeRecommender.py:66-73, SVD.py:84-90). */
int qrec_mf_predict_pairs_f32(const float* dev_P, const float* dev_Q, int32_t d, int64_t n,
                              const int32_t* dev_u, const int32_t* dev_i, const float* dev_Bu,
                              const float* dev_Bi, float global_mean, float* dev_out, void* stream);
int qrec_mf_predict_pairs_f64(const double* dev_P, const double* dev_Q, int32_t d, int64_t n,
                              const int32_t* dev_u, const int32_t* dev_i, const double* dev_Bu,
                              const double* dev_Bi, double global_mean, double* dev_out, void* stream);

/* =====================================================================================
 * K10 -- WRMF (implicit-feedback ALS, model/ranking/WRMF.py:19-61).  A half-epoch solves every row of one
 * table X against the other table Z, which it only reads:
 *   A = Z^T Z + lambda*I + alpha * sum_k v_k z_k z_k^T,   b = sum_k (1 + alpha*v_k) z_k,   X[r] = A^-1 b
 * over the entries (c_k, v_k) of row r.  A and b are float64 for both table types.  d: 1..128.
 * ===================================================================================== */
/* Bytes of device workspace qrec_als_gram_* needs for n rows of width d (0 for n = 0); < 0 on bad arguments. */
int64_t qrec_als_gram_workspace_bytes(int64_t n, int32_t d);
/* G[d][d] (float64, row-major, exactly symmetric) = Z^T Z of the table Z[n][d].  Partial Grams of fixed 2048-row
 * chunks go to the caller's workspace (workspace_bytes >= qrec_als_gram_workspace_bytes(n, d)) and are summed in
 * chunk order, so G is bitwise the same from run to run and on any H100.  n = 0 gives G = 0. */
int qrec_als_gram_f32(const float* dev_Z, int64_t n, int32_t d, double* dev_G, void* dev_workspace,
                      int64_t workspace_bytes, void* stream);
int qrec_als_gram_f64(const double* dev_Z, int64_t n, int32_t d, double* dev_G, void* dev_workspace,
                      int64_t workspace_bytes, void* stream);
/* Solves the rows row_order[0..n_rows) of X (a different table from Z) with G = Z^T Z from qrec_als_gram_*:
 * row r's entries are cols[rowptr[r]..rowptr[r+1]) (rows of Z) with values vals[...].  One CTA solves one row
 * (Cholesky in float64), so X is bitwise reproducible; row_order only balances the work (longest rows first).
 * A row without entries gets x = 0.  dev_loss (optional, double[1]) accumulates sum_k (1 - x_old.z_k)^2 with the
 * row's value before the solve.  A row whose A has a pivot that is not positive is left unchanged and counted in
 * dev_n_failed (optional, int32[1]).  d > 128 is QREC_ERR_ARG. */
int qrec_als_solve_rows_f32(float* dev_X, const float* dev_Z, const double* dev_G, int32_t d, int64_t n_rows,
                            const int32_t* dev_row_order, const int64_t* dev_rowptr, const int32_t* dev_cols,
                            const float* dev_vals, double lambda, double alpha, double* dev_loss,
                            int32_t* dev_n_failed, void* stream);
int qrec_als_solve_rows_f64(double* dev_X, const double* dev_Z, const double* dev_G, int32_t d, int64_t n_rows,
                            const int32_t* dev_row_order, const int64_t* dev_rowptr, const int32_t* dev_cols,
                            const double* dev_vals, double lambda, double alpha, double* dev_loss,
                            int32_t* dev_n_failed, void* stream);

/* =====================================================================================
 * K11 -- SVD++ (model/rating/SVDPlusPlus.py:26-88).  Tables P[num_users][d], Q, Y[num_items][d], Bu, Bi.  Per entry
 * (u, i, r), with N(u) the user's distinct items (one CSR row) and w = |N(u)|:
 *   pred = (sum_{N(u)} Y / w).Q[i] + P[u].Q[i] + mean + Bi[i] + Bu[u];   e = r - pred;   dev_loss += e^2
 *   Bu[u], Bi[i] += lr*(e - regB*b);
 *   w > 1:  Y[j] += lr*(e*Q[i]/(w-1) - regY*Y[j]) for j in N(u), j != i;   Q[i] += lr*e*sum_{j != i} Y[j] / (w-1)
 *   P[u] += lr*(e*Q[i] - regU*P[u]);  Q[i] += lr*(e*P[u] - regI*Q[i])   (Q[i] after the implicit step, the new P[u])
 * rowptr (int64 [num_users + 1]) / cols (int32): N(u) in the order of the user's row.
 * ===================================================================================== */
/* Parity mode: the entries (u[k], i[k], r[k]) one after another in array order, by ONE CTA (parallel inside an
 * entry only), with the reference's evaluation order; float64 tables follow the reference to the grouping of the
 * two dot products.  d: 1..256. */
int qrec_svdpp_sgd_ordered_f64(double* dev_P, double* dev_Q, double* dev_Y, double* dev_Bu, double* dev_Bi, int32_t d,
                               int64_t n, const int32_t* dev_u, const int32_t* dev_i, const double* dev_r,
                               const int64_t* dev_rowptr, const int32_t* dev_cols, double lr, double reg_u,
                               double reg_i, double reg_b, double reg_y, double global_mean, double* dev_loss,
                               void* stream);
int qrec_svdpp_sgd_ordered_f32(float* dev_P, float* dev_Q, float* dev_Y, float* dev_Bu, float* dev_Bi, int32_t d,
                               int64_t n, const int32_t* dev_u, const int32_t* dev_i, const float* dev_r,
                               const int64_t* dev_rowptr, const int32_t* dev_cols, float lr, float reg_u, float reg_i,
                               float reg_b, float reg_y, float global_mean, double* dev_loss, void* stream);
/* Throughput mode: one user-major epoch over the CSR's entries (cols, vals: each user's distinct items and their
 * ratings), users taken from row_order[0..n_rows).  One lane group runs a user's entries in row order through the
 * per-user closed form (csrc/svdpp_step.cuh), so a step moves Q[i] and Y[i] instead of all the user's Y rows; the
 * Q / Y / Bi deltas are added back atomically, P[u] and Bu[u] are written once.
 * d: multiple of 4, 4..128 (pad with zero columns; they stay zero).
 * max_users_in_flight: 0 = fill the GPU; k > 0 = at most k users at a time.  Users in flight read each other's
 * rows stale, like qrec_mf_sgd_batch_f32's entries: small or skewed data needs about (0.25/lr) / (share of the users
 * who rated the most-rated item).  k = 1 applies the users one after another.  n_rows = 0 launches nothing. */
int qrec_svdpp_epoch_usermajor_f32(float* dev_P, float* dev_Q, float* dev_Y, float* dev_Bu, float* dev_Bi, int32_t d,
                                   int32_t n_rows, const int32_t* dev_row_order, const int64_t* dev_rowptr,
                                   const int32_t* dev_cols, const float* dev_vals, float lr, float reg_u, float reg_i,
                                   float reg_b, float reg_y, float global_mean, double* dev_loss,
                                   int64_t max_users_in_flight, void* stream);

/* =====================================================================================
 * K12 -- CoFactor (model/ranking/CoFactor.py): WRMF plus a co-factorisation of the item-item SPPMI matrix.  The user
 * half-epoch is K10's qrec_als_solve_rows_*; the SPPMI's co-occurrence counts and the item half-epoch are here.
 * ===================================================================================== */
/* Co-occurrence counts of the eligible items (at least `filter` distinct users): for each listed row i and each
 * eligible j != i, the number of users of both, kept when > filter.  item_rowptr / item_users: every item's DISTINCT
 * users; user_rowptr / user_items: its transpose, each user's items in ascending order.  One CTA per row, rows taken
 * from row_order[0..n_rows) (eligible items only; longest first balances the grid).  Two passes:
 *   out_rowptr == NULL: row_nnz[i] = number of kept entries of each listed row (other rows untouched);
 *   out_rowptr != NULL: the kept columns of row i, ascending, go to out_cols[out_rowptr[i]..] with their counts.
 * Exact integer counts, the same on every run. */
int qrec_cooc_count(int32_t n_items, const int64_t* dev_item_rowptr, const int32_t* dev_item_users,
                    const int64_t* dev_user_rowptr, const int32_t* dev_user_items, int32_t n_rows,
                    const int32_t* dev_row_order, int32_t filter, const int64_t* dev_out_rowptr, int64_t* dev_row_nnz,
                    int32_t* dev_out_cols, int32_t* dev_out_counts, void* stream);
/* One item half-epoch in item-id order, in place (tables Y, G [n_items][d], w, c [n_items]; X [num_users][d] only
 * read; XtX = X^T X from qrec_als_gram_*).  Item i's users are item_users[item_rowptr[i]..] with ratings item_vals,
 * its SPPMI contexts sppmi_cols[sppmi_rowptr[i]..] with values sppmi_vals (the SPPMI must be symmetric):
 *   Y_i = (XtX + alpha*sum r x x^T + lambda*I + sum_c G_c G_c^T)^-1 (sum (1 + alpha*r) x + sum_c ((m - w_i) - c_c) G_c)
 *   and, for an item with contexts, G_i = (sum_c Y_c Y_c^T + gamma*I)^-1 sum_c ((m - w_c) - c_i) Y_c,
 *   w_i = mean_c ((m - Y_i.G_c) - c_c), c_i = mean_c ((m - Y_c.G_i) - w_c)  with item i's values from before it.
 * Contexts c < i are read after their update in this sweep, c > i before it, as in the sequential loop: CTAs take
 * items in id order from dev_ticket (uint64[1], zero on entry) and wait until every smaller context's stamp
 * (dev_stamps int32[n_items], all sweep - 1 on entry) equals `sweep`; each item then adds 1 to its stamp.  A and b
 * are float64; the result is bitwise reproducible.  A system that is not positive definite leaves its row unchanged
 * and is counted in dev_n_failed (optional, int32[1]).  d: 1..128. */
int qrec_cofactor_item_sweep_f32(float* dev_Y, float* dev_G, float* dev_w, float* dev_c, const float* dev_X,
                                 const double* dev_XtX, int32_t d, int32_t n_items, const int64_t* dev_item_rowptr,
                                 const int32_t* dev_item_users, const float* dev_item_vals,
                                 const int64_t* dev_sppmi_rowptr, const int32_t* dev_sppmi_cols,
                                 const float* dev_sppmi_vals, double lambda, double gamma, double alpha,
                                 int32_t* dev_stamps, int32_t sweep, unsigned long long* dev_ticket,
                                 int32_t* dev_n_failed, void* stream);
int qrec_cofactor_item_sweep_f64(double* dev_Y, double* dev_G, double* dev_w, double* dev_c, const double* dev_X,
                                 const double* dev_XtX, int32_t d, int32_t n_items, const int64_t* dev_item_rowptr,
                                 const int32_t* dev_item_users, const double* dev_item_vals,
                                 const int64_t* dev_sppmi_rowptr, const int32_t* dev_sppmi_cols,
                                 const double* dev_sppmi_vals, double lambda, double gamma, double alpha,
                                 int32_t* dev_stamps, int32_t sweep, unsigned long long* dev_ticket,
                                 int32_t* dev_n_failed, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* QREC_H_ */
