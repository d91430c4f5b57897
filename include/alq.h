/*
 * alq.h -- C ABI of libalq.so, the H100 (sm_90a) acquisition-scoring engine that replaces the
 * per-round query tail of zeyademam/active_learning (`strategy.query(budget)`,
 * src/main_al.py:156).  Citations below are relative to active_learning/src/query_strategies/.
 *
 * Conventions
 *   - Every pointer is a DEVICE pointer owned by the caller unless its name ends in `_host`.
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream); calls are
 *     asynchronous on it unless stated otherwise.
 *   - Return value: ALQ_OK (0) or an ALQ_ERR_* code; `alq_last_error(ctx)` describes the failure.
 *   - All arithmetic is IEEE fp32 (fp64 only for the inverse-CDF search and the Ward clustering, K7/K8; K3 and K9
 *     contract on the tensor cores as 3xTF32, fp32 to about 2^-21 per product); index math is int32 on the device
 *     (n < 2^31), except the int64 offsets into K7/K8's distances.  There is no CPU fallback anywhere in this library.
 *   - Matrices are row-major with an explicit leading dimension (`ld*`, in elements).  The fast
 *     paths need the base pointer 16-byte aligned and ld % 4 == 0.
 */
#ifndef ALQ_H_
#define ALQ_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct alq_ctx alq_ctx;

enum {
    ALQ_OK = 0,
    ALQ_ERR_INVALID = 1, /* bad argument (shape, alignment, null pointer) */
    ALQ_ERR_CUDA = 2,    /* a CUDA runtime call failed */
    ALQ_ERR_NOMEM = 3,   /* scratch allocation failed */
    ALQ_ERR_STATE = 4,   /* call sequence / communicator state */
    ALQ_ERR_NUMERIC = 5  /* non-finite probability mass etc. */
};

enum { ALQ_MODE_MARGIN = 0, ALQ_MODE_LEAST_CONFIDENCE = 1, ALQ_MODE_ENTROPY = 2 };

/* ABI version of this header (bumped on any signature change). */
int alq_version(void);

/* One context per process and GPU.  Owns a grow-only device scratch arena, a private stream
 * and (optionally) the peer-memory windows of a multi-GPU group. */
int alq_create(alq_ctx** out, int device);
void alq_destroy(alq_ctx* ctx);
const char* alq_last_error(const alq_ctx* ctx);
/* Implementation knobs (defaults pick the fastest valid kernel):
 *   "k3_impl"        0 auto | 1 exact-fp32 SIMT contraction | 2 wgmma 3xTF32 contraction
 *   "greedy_variant" selection loop (K4/K5) only: 0 auto | 1 direct-load step kernel | 2 bulk-copy (TMA) pipeline |
 *                    3 persistent cooperative loop
 *   "l2_resident_mb" persistent selection loop: MB of the rows a GPU streams that are fetched L2::evict_last (the head of every
 *                    CTA's segment) so that they stay in the 50 MB L2 across the B steps; the rest is fetched evict_first.
 *                    Default 24; 0 turns the hints off
 *   "d2_fast_path"   1 (default): the persistent loop's D^2 draw first tries the certified path (one fp64 mass per CTA, the
 *                    rounding of NumPy's float32 probabilities bounded by a margin); 0: always the exact NumPy-tree machinery
 *   "tail_buckets"   1 (default): alq_uncertainty_tail on one GPU routes the candidates to per-CTA score buckets, each CTA sorts
 *                    its own bucket; 0: the general route (every CTA ranks its candidates against the whole list), which is also
 *                    what a pool whose scores do not spread (tie groups) falls back to inside the launch
 *   "spin_timeout_ms" how long a kernel waits for a peer GPU's flag before giving up with ALQ_ERR_STATE (default 20000)
 *   "select_impl"    0 auto | 1 multi-kernel radix select   | 2 single cluster-resident launch
 *   "base_impl"      0 auto | 1 sequential class loop       | 2 per-class candidate lists + in-order resolve
 *   "balancing_loop" 0 auto (K11 whenever its limits hold, otherwise K12 whenever its limits hold, otherwise the caller's
 *                    per-step path) | 1 per-step path: alq_balancing_select and alq_balancing_table_select decline
 *                    (n_picks_host = -1) and the caller runs its own step loop | 2 K11, ALQ_ERR_INVALID naming the limit
 *                    when the shape is beyond it; K12 declines | 3 K12, the same; K11 declines */
int alq_set_option(alq_ctx* ctx, const char* key, int64_t value);
/* Number of kernels this context has launched since creation (bench.py's `gpu_launches`). */
int64_t alq_launch_count(const alq_ctx* ctx);

/* ---- multi-GPU group: one process per GPU, peer-memory windows over NVLink ---------------------
 * alq_comm_create allocates this rank's window and returns its 64-byte CUDA IPC handle; the caller
 * exchanges the handles (e.g. torch.distributed.all_gather) and passes all of them, in rank order, to
 * alq_comm_connect.  The global (non-partitioned) CoreSet / k-means++ loops and BalancingSampler's loops then exchange
 * their per-step winner through these windows from inside the kernels (alq_greedy_desc.shard_off_host,
 * alq_balancing_desc.shard_off_host).                                                             */
#define ALQ_IPC_HANDLE_BYTES 64
int alq_comm_create(alq_ctx* ctx, int32_t world, int32_t rank, size_t window_bytes, void* handle_out);
int alq_comm_connect(alq_ctx* ctx, const void* all_handles);
int alq_comm_destroy(alq_ctx* ctx);

/* ---- K1: softmax-uncertainty score -------------------------------------------------------
 * Replaces the per-batch Softmax -> topk -> subtract of margin_sampler.py:33-35 and
 * confidence_sampler.py:31-33 (entropy: SURVEY.md section 8 row A3, new).
 * scores[i] = p(1)-p(2) | p(1) | sum_c p_c log p_c  of softmax(logits[i, :c]).                */
int alq_score_softmax(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld,
                      int32_t mode, float* scores, void* stream);

/* ---- K1b: stable top-B smallest -------------------------------------------------------------
 * Replaces torch.sort(ascending).indices[:B] of margin_sampler.py:42 / confidence_sampler.py:42
 * under the fixed tie-break "equal scores: lowest position first".  out_pos[0..b) = positions
 * in ascending (score, position) order.                                                       */
int alq_select_smallest(alq_ctx* ctx, const float* scores, int64_t n, int64_t b,
                        int32_t* out_pos, void* stream);

/* K1 + K1b as ONE launch: scores[i] as alq_score_softmax AND out_pos[0..b) as alq_select_smallest of those scores --
 * the whole tail of MarginSampler.query / ConfidenceSampler.query (margin_sampler.py:33-42) behind one call.  When the
 * pipelined scoring kernel applies (c % 4 == 0, contiguous rows, 4096 <= n <= ~240 000 per GPU) the selection runs in
 * that kernel's epilogue (one CTA per SM, device-wide spin barriers: per-CTA key lists in shared memory, two global
 * 2048-bin histogram levels, the winners ordered through per-CTA score buckets -- option "tail_buckets"); otherwise the
 * two kernels run back to back.  Same results either way.  Launches of this kernel (and of the persistent selection loop)
 * from different streams of one process are serialised against each other by the library.                              */
int alq_uncertainty_tail(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld, int32_t mode,
                         int64_t b, float* scores, int32_t* out_pos, void* stream);

/* Diagnostics of the LAST fused launch of alq_uncertainty_tail[_sharded] on this context (the caller has synchronised its
 * stream): out_ms_host[0] = kernel start -> every CTA has finished streaming its rows, [1] = kernel start -> end, both from
 * %globaltimer stamps of CTA 0.  ALQ_ERR_STATE if that call ran the separate kernels instead.                         */
int alq_uncertainty_tail_timing(alq_ctx* ctx, float* out_ms_host);

/* The same tail with the rows sharded over the G >= 1 ranks of the peer-memory group (alq_comm_create/connect): rank r holds
 * `n` rows that are positions [row_lo, row_lo + n) of the pool and every rank receives the same out_gpos[0..b): the global
 * positions of the b smallest scores over ALL ranks, ascending (score, position) -- exactly what a single GPU returns for
 * the concatenated pool.  K1, K1b and the exchange are ONE launch per rank: both histogram levels are summed over
 * the ranks and the b + few candidate words gathered through the windows from inside the kernel (8-byte {tag, value} words
 * and plain stores over NVLink; no collective library, nothing on the host).  Collective: every rank calls it with the same
 * c, mode, b, rows_min / rows_max (the smallest / largest shard; they decide, identically on every rank, whether the fused
 * kernel applies -- otherwise K1, K1b and alq_topb_exchange run back to back, same result).  The separate launches serve
 * b <= 16384 only (alq_topb_exchange's limit): a larger b that does not fuse returns ALQ_ERR_INVALID on every rank before
 * anything runs, and the caller exchanges the local winners itself (alq_topb_pack + alq_topb_merge).  Asynchronous; a
 * peer that never shows up is reported through alq_comm_check like alq_topb_exchange.                              */
int alq_uncertainty_tail_sharded(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld, int32_t mode,
                                 int64_t b, int64_t row_lo, int64_t rows_min, int64_t rows_max, float* scores,
                                 int32_t* out_gpos, void* stream);

/* Multi-GPU top-B (rows sharded over G ranks): each rank packs its local winners as
 * out[i] = ord(scores[pos[i]]) << 32 | (row_lo + pos[i])  (i < k; padded with ~0 up to b_pad),
 * the G*b_pad words are all-gathered by the caller (NCCL), and alq_topb_merge returns the global
 * positions of the b smallest words in ascending order -- the same (score, position) order as K1b.
 * list_len > 0 declares that keys is n / list_len individually sorted lists (what alq_topb_pack of
 * K1b output produces): they are merged by rank counting, without a sorting pass.               */
int alq_topb_pack(alq_ctx* ctx, const float* scores, const int32_t* pos, int64_t k, int64_t row_lo,
                  int64_t b_pad, uint64_t* out, void* stream);
int alq_topb_merge(alq_ctx* ctx, const uint64_t* keys, int64_t n, int64_t list_len, int64_t b,
                   int32_t* out_gpos, void* stream);

/* The same exchange over the peer-memory windows of alq_comm_create/connect (G >= 1 ranks) instead of a collective
 * library: pack + store into every peer's window + flag, then wait + merge (b <= 16384).  Collective: every rank of the
 * group must call it, in the same order relative to its other group calls.                      */
int alq_topb_exchange(alq_ctx* ctx, const float* scores, const int32_t* pos, int64_t k, int64_t row_lo,
                      int64_t b, int32_t* out_gpos, void* stream);
/* alq_topb_exchange is asynchronous, so a peer that never raises its flag (a dead or badly delayed rank; the bounded
 * spin lasts "spin_timeout_ms") cannot be reported by its return value: the merge then writes -1 into every output
 * position and records ALQ_ERR_STATE in a host-visible status word.  alq_comm_check returns (and clears) that status;
 * call it once the stream has been synchronised (e.g. after the positions were copied to the host).  The next
 * alq_topb_exchange on the context also reports it before doing anything.                         */
int alq_comm_check(alq_ctx* ctx);

/* Same tail for HOST buffers (what a CPU-tensor caller of MarginSampler.query has): pinned or
 * pageable host logits -> chunked H2D overlapped with K1 -> K1b -> positions back on the host.
 * Synchronous.                                                                                */
int alq_uncertainty_query_host(alq_ctx* ctx, const float* logits_host, int64_t n, int32_t c,
                               int32_t mode, int64_t b, int32_t* out_pos_host);

/* ---- K2: BADGE gradient-embedding factors --------------------------------------------------
 * badge_sampler.py:33-40: the logits-gradient of CE(mean) against the arg-max pseudo label is
 * a_i = (softmax(z_i) - onehot(argmax z_i)) / bs_i, bs_i = size of the loader batch holding row
 * i (`batch_size`, or n % batch_size for the last short batch).  The 2048*1000-d embedding is
 * a_i (x) h_i and is never materialised.  Writes a[n, c] (columns c..lda-1 zero-filled up to the
 * next multiple of 4) and a_norm2[i] = |a_i|^2.
 * A shard of a larger pool passes its offset: the rows are positions [row0, row0 + n) of a loader pass over
 * n_total rows (n_total <= 0 means the call covers the whole pool).                               */
int alq_badge_factors(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld,
                      int32_t batch_size, int64_t row0, int64_t n_total, float* a, int64_t lda,
                      float* a_norm2, void* stream);

/* K2p: the adaptive-pooled embedding of badge_sampler.py:41-44 (pool_h = min(16, c),
 * pool_w = 512 / pool_h) written materialised: out[i, r*pool_w + s] = pool(a_i)[r] * pool(h_i)[s]. */
int alq_badge_pooled_embedding(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld,
                               int32_t batch_size, const float* emb, int32_t d, int64_t lde,
                               float* out, int64_t ldo, void* stream);

/* out[i] = sum_k x[i,k]^2  (the norm_square column of coreset_sampler.py:61).                */
int alq_row_norm2(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ld, float* out,
                  void* stream);

/* ---- K3: min (or max) squared distance to a row set -------------------------------------------
 * Replaces get_pairwise_l2_dist + `[:, labeled].min(dim=1)` (coreset_sampler.py:59-64,79)
 * without forming N x N:  out[i] = red_j  fl(fl(xn[i] + yn[j]) - 2*<x_i, y_j>),  red = min, or
 * max when reduce_max != 0 (the minimax cold start, coreset_sampler.py:100).
 * With accumulate != 0 the result is folded into the existing out[i].
 * Factored (BADGE) rows: pass xa/ya (second factor, `c` columns) and the per-factor norms; then
 * <g_i,g_j> = <xa_i,ya_j> * <x_i,y_j> and |g|^2 = an*xn.  Pass xa = ya = NULL for dense rows.  */
int alq_min_dist(alq_ctx* ctx,
                 const float* x, int64_t ldx, const float* xn, int64_t n,
                 const float* y, int64_t ldy, const float* yn, int64_t m, int32_t d,
                 const float* xa, int64_t ldxa, const float* xan,
                 const float* ya, int64_t ldya, const float* yan, int32_t c,
                 int32_t reduce_max, int32_t accumulate, float* out, void* stream);

/* out_row[0] = argmin_i v[i] (lowest index on ties) -- second half of coreset_sampler.py:100. */
int alq_argmin(alq_ctx* ctx, const float* v, int64_t n, int32_t* out_row, void* stream);

/* balancing_sampler.py:114-119: out_row[0] = argmin_i num[i] / den[i] over the rows with avail[i] != 0 (lowest index on
 * ties; -1 if no row is available).  num == NULL stands for the constant 1 (the rarest class has no labeled row,
 * :104-107).  num / den are K3 outputs: squared distance to the rarest class centre / largest squared distance to a
 * majority class centre (alq_min_dist with reduce_max).                                                        */
int alq_ratio_argmin(alq_ctx* ctx, const float* num, const float* den, const unsigned char* avail, int64_t n,
                     int32_t* out_row, void* stream);

/* ---- K4 / K5: greedy k-center and k-means++ D^2 seeding ----------------------------------------
 * Replaces the step loop of coreset_sampler.py:77-103.  Candidates are the UNLABELED rows only;
 * `mind` arrives holding their min squared distance to the labeled set (K3; +inf if none) and is
 * updated in place with a running min against every new centre (SURVEY.md finding 4).
 * Partitions (partitioned_coreset_sampler.py:63-80) are a batch dimension: rows
 * [part_off[p], part_off[p+1]) form partition p with its own centre, mass and budget.
 *
 *   uniforms_host == NULL : arg-max of mind, lowest row on ties      (coreset_sampler.py:94)
 *   uniforms_host != NULL : D^2 sampling with NumPy-identical arithmetic (coreset_sampler.py:84-92):
 *        p = clip(mind,0); p[labeled]=0; p /= np.sum(p) (fp32 pairwise tree over the partition's
 *        full labeled+unlabeled array); NaN -> mind += 1e-5 retry; np.random.choice ==
 *        first k with cumsum64(p)[k]/total > u.  One pre-drawn uniform per step.
 */
typedef struct alq_greedy_desc {
    size_t struct_size;          /* sizeof(alq_greedy_desc), for forward compatibility */
    /* candidate rows: dense part x[n, d]; optional second factor a[n, c] (NULL for CoreSet) */
    const float* x;  int64_t ldx; int32_t d;
    const float* a;  int64_t lda; int32_t c;
    const float* xn;             /* [n] |x_i|^2 */
    const float* an;             /* [n] |a_i|^2, NULL iff a == NULL */
    float* mind;                 /* [n] in/out */
    int64_t n;
    /* partitions (host arrays) */
    int32_t n_parts;
    const int32_t* part_off_host;   /* [n_parts + 1] */
    const int32_t* budget_host;     /* [n_parts] picks per partition */
    /* D^2-sampling extras */
    const double* uniforms_host;    /* [sum budget] partition-major, or NULL */
    const int32_t* vpos;            /* [n] position of row i inside its partition's full array */
    const int32_t* full_n_host;     /* [n_parts] length of that array (labeled + unlabeled) */
    const int32_t* first_pick_host; /* [n_parts] or NULL: row already chosen by the caller as the
                                       first centre of a partition with nothing labeled, else -1 */
    /* output: [sum budget] partition-major, in pick order; row ids in [0, n) */
    int32_t* picks;
    /* kernel variant: 0 = auto, 1 = direct-load step kernel, 2 = bulk-copy (TMA) pipeline step kernel (one launch
       per step), 3 = ONE persistent cooperative launch for the whole loop (TMA pipeline that keeps prefetching the
       next step's rows while the grid agrees on the new centre).  Auto picks 3 whenever it fits. */
    int32_t variant;
    /* multi-GPU (needs alq_comm_create/connect; n_parts must be 1; variant 3 only).  Every array above is indexed
       by GLOBAL candidate row and REPLICATED on every rank (x/a/xn/an/vpos: n rows each; a few hundred MB next to
       180 GB of HBM), so a new centre is announced as a row id and read locally -- no row payload crosses NVLink.
       Rank r streams rows [shard_off[r], shard_off[r+1]) only and owns that range of `mind` (the rest of `mind` is
       not touched).  picks are global row ids, identical on every rank.  NULL => single GPU.  Given on a context with
       a group, whatever its size, the call takes the group path: a group of one rank runs the group path too (the
       window, its ready handshake and tags, on this GPU's own memory).  Given without a group, shard_off = {0, n} is
       ignored and anything else is ALQ_ERR_STATE.  An explicit variant 1 or 2 (or the option) is ALQ_ERR_INVALID.
       D^2 sampling additionally needs the shards aligned to the leaves of NumPy's pairwise-sum tree over the
       partition's full array: rank r's rows are exactly the candidates with vpos in
       [shard_pos[r], shard_pos[r+1]), every shard_pos a leaf boundary (alq_pairwise_leaf_bounds), shard_pos[0] = 0,
       shard_pos[world] = full_n[0].  Per step the ranks exchange 8-byte {tag, value} words through the peer-memory
       windows (leaf sums, leaf masses, the pick): one-way NVLink stores, no fences, no collective library. */
    const int32_t* shard_off_host;
    const int32_t* shard_pos_host;
    /* optional timing out-parameter (forces a stream synchronisation at the end of the call), 8 floats in ms:
       [0] mean time of the streaming phase of a step (variants 1/2: CUDA events around the step kernel; variant 3:
       %globaltimer stamps taken by CTA 0), [1] mean time of the selection phase (barrier + exchange + draw) of a step
       (variant 3 only), [2] steps measured, [3] the variant that ran, [4..7] variant 3 diagnostics: [4] [5] reserved, [6] the t = 0
       selection in ms, [7] the whole kernel in ms as its CTA 0 saw it. */
    float* step_kernel_ms_host;
} alq_greedy_desc;

int alq_greedy_select(alq_ctx* ctx, const alq_greedy_desc* desc, void* stream);

/* Leaf boundaries of NumPy's float32 pairwise summation over an array of n entries (blocks of <= 128 entries, splits
 * at n/2 rounded down to a multiple of 8): out[0..k] ascending with out[0] = 0, out[k] = n.  Returns k (the number of
 * leaves), or -1 if cap < k + 1.  Host-only helper for building leaf-aligned shards (alq_greedy_desc.shard_pos_host). */
int64_t alq_pairwise_leaf_bounds(int64_t n, int32_t* out_host, int64_t cap);

/* ---- K6: MASE / BASE (SURVEY.md section 8f rank 2) ---------------------------------------------
 * mase_sampler.py:52-80 measures, for every pool row, the distance of its embedding h_i to the decision
 * boundary between the predicted class p = argmax z_i (lowest index on ties) and every other class c:
 *     radius[i, c] = | -(w_p - w_c) * lam / 2 |,  lam = 2 (h_i.(w_p - w_c) + b_p - b_c) / |w_p - w_c|^2
 *                  = |z_ip - z_ic| / |w_p - w_c|            (the logit gap over the head geometry),
 * NaN (c == p, coinciding class rows) -> +inf (:77), min_margin[i] = min_c radius[i, c] (:79).
 *
 * alq_class_gap_inv: ginv[a, c] = 1 / |w_a - w_c| for the head weight[c, m] (:60-71; +inf where rows coincide and on
 *   the diagonal; columns c..ldg-1 are filled with +inf) and, if gmin != NULL (c + 1 floats), gmin[a] = min_c ginv[a, c]
 *   for a < c plus gmin[c] = max_a (largest finite ginv[a, :]) / gmin[a], the spread of the class rows.
 *   Once per query: the head changes every round.
 * alq_mase_margins: one streaming pass over the logits slab.  pred[i] = p, the arg-max of torch.max: the first
 *   maximum, and in a row with a NaN logit the first NaN (every radius of that row is then +inf, as in the reference,
 *   where the NaN gap becomes +inf at :77).  radius may be NULL (MASE needs only
 *   the minimum); columns c..ldr-1 of radius are unspecified.  gmin (optional, from alq_class_gap_inv of the same
 *   table) lets the minimum-only pass skip every class that provably cannot attain it (the skip is verified per
 *   row, with a full evaluation if the check fails) -- same result, the table is touched for a handful of
 *   classes per row instead of all C.                                                                       */
int alq_class_gap_inv(alq_ctx* ctx, const float* weight, int32_t c, int32_t m, int64_t ldw, float* ginv,
                      int64_t ldg, float* gmin, void* stream);
int alq_mase_margins(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, int64_t ld, const float* ginv,
                     int64_t ldg, const float* gmin, float* min_margin, int32_t* pred, float* radius, int64_t ldr,
                     void* stream);

/* base_sampler.py:22-38: class by class (c = 0..C-1), take the budget / C (+1 for c < budget % C) rows with the
 * smallest key  (pred[i] == c ? min_margin[i] : radius[i, c]),  rows taken by earlier classes pushed to +inf;
 * every per-class sort is K1b (stable).  out_pos[0..budget) = pool positions in pick order.  Synchronous.
 * With many classes and <= 32 picks per class the per-class lists are extracted for all classes at once and
 * resolved in class order on the device (same result; a class whose list runs short takes the ordinary step).
 * ALQ_ERR_NUMERIC if a row would be selected twice -- the condition the reference asserts on (:40).          */
int alq_base_select(alq_ctx* ctx, const float* min_margin, const float* radius, int64_t ldr, const int32_t* pred,
                    int64_t n, int32_t c, int64_t budget, int32_t* out_pos, void* stream);

/* ---- K7 / K8: Ward agglomerative clustering (MarginClusteringSampler) -----------------------------------------------
 * margin_clustering_sampler.py:59 clusters the pool embeddings with sklearn's AgglomerativeClustering(n_clusters=20),
 * i.e. scipy.cluster.hierarchy.ward(X): pdist + nn_chain over the full tree + sklearn's _hc_cut.  The three calls
 * below reproduce that tree bit for bit, so the labels are sklearn's.
 *
 * alq_pdist_f64 (K7): dist[i, j] (row-major, leading dimension ldd >= n) = scipy's pdist(X, 'euclidean') of the fp32
 *   rows x[i], x[j] in fp64: s summed over k = 0, 1, ... as `d = x[i,k] - x[j,k]; s = s + d*d` (no FMA), dist = sqrt(s).
 *   Every pair is computed once and written to (i, j) and (j, i); the diagonal holds 0.0 (K8 never reads it).  Zero
 *   pad columns (the 16-byte row padding of the pool-forward slab) leave every sum unchanged, so d may include them.
 *   Any ldx >= d and any alignment.  n <= 65535 * 64.  The caller owns `dist` (8 * n * ldd bytes: 51.2 GB at
 *   n = 80 000), so the caller frees it when the query ends (Engine.ward_tree hands it back to the device) and it
 *   never sits in the grow-only arena.  Offsets into `dist` are
 *   int64 -- the one exception to the int32 index rule above (n^2 passes 2^31 at n = 46 341).
 * alq_pdist_f64_condensed (K7, condensed layout): the same distances, bit for bit, written only once each into
 *   scipy's condensed vector -- pdist's own output: (i, j), i < j, at dist[n*i - i*(i+1)/2 + (j - i - 1)], n (n - 1) / 2
 *   entries (4 n (n - 1) bytes, half the square matrix: 25.6 GB at n = 80 000, 53.7 GB at n = 115 846).  Nothing past
 *   them is written.  Same arguments, limits and caller-owned buffer as alq_pdist_f64, without ldd.  Offsets are
 *   int64 (the vector passes 2^31 entries at n = 65 537).
 * alq_pdist_f64_condensed_rows (K7, a band of rows): the entries (i, j), row_lo <= i < row_hi, j > i, of the condensed
 *   vector -- bit for bit those alq_pdist_f64_condensed writes (a pair's sum does not depend on the tile computing it)
 *   -- at dist[cidx(i, j) - cidx(row_lo, row_lo + 1)], cidx(i, j) = n*i - i*(i+1)/2 + (j - i - 1): the band is one
 *   contiguous slice of cidx(row_hi, row_hi + 1) - cidx(row_lo, row_lo + 1) entries, nothing past it is written.
 *   Bands that cover [0, n) concatenate to alq_pdist_f64_condensed's vector.  An empty band (row_lo == row_hi) is
 *   valid and writes nothing.  ALQ_ERR_INVALID for row_lo < 0, row_hi > n, row_lo > row_hi, null pointers, and as
 *   alq_pdist_f64_condensed.  This is how the ranks of a group split K7 (sharding.py: ShardGroup.ward_labels).
 * alq_pdist_f64_expand: a condensed band as alq_pdist_f64_condensed_rows writes it (`rows`, same n, row_lo, row_hi)
 *   into the square matrix: dist[i, j] = dist[j, i] = its entry for row_lo <= i < row_hi and every j > i, and
 *   dist[i, i] = 0.0 (row-major, ldd >= n).  Nothing else is written.  Expanding bands that cover [0, n) gives exactly
 *   what alq_pdist_f64 writes, diagonal included.  HBM-bound (64 x 64 tiles staged through shared memory, so the
 *   row-wise and the mirrored stores are both coalesced).  Same argument checks as the band call, plus ldd < n.
 * alq_ward_nn_chain (K8): scipy's nn_chain with the Ward update, in ONE launch of one thread-block cluster, consuming
 *   `dist` in place (its contents are unspecified afterwards).  merge_xy[k] = (x, y) with x < y and merge_dist[k], for
 *   k < n - 1, in the chain's discovery order (before scipy's sort).  n >= 2.  Synchronous; ALQ_ERR_NUMERIC if a scan
 *   found no finite distance (non-finite input).
 * alq_ward_nn_chain_condensed (K8, condensed layout): the same walk and the same merge list, bit for bit, over a
 *   condensed vector of n (n - 1) / 2 entries (as alq_pdist_f64_condensed writes it), consumed in place.  Same
 *   arguments and contract as alq_ward_nn_chain, without ldd.
 * alq_ward_nn_chain_banded (K8, banded layout): the same walk and the same merge list, bit for bit, over the condensed
 *   vector cut into 1 <= nbands <= 8 bands of rows, each at its own device pointer (which may be a peer GPU's memory
 *   mapped with alq_band_open): band b holds rows [row_cuts_host[b], row_cuts_host[b + 1]) as
 *   alq_pdist_f64_condensed_rows writes them, at bands_host[b].  The nbands + 1 cuts run from 0 to n and never
 *   decrease (empty bands are allowed); a band without pairs (row n - 1 alone, or empty) may have a null pointer.
 *   Consumed in place.  Every band must stay untouched by any other stream, process or GPU until this call returns.
 *   ALQ_ERR_INVALID for cuts that decrease or do not cover [0, n), a null pointer for a band with pairs, nbands
 *   outside [1, 8], and as alq_ward_nn_chain_condensed.  This is how a group runs K8 over the ranks' bands without
 *   gathering them (sharding.py: ShardGroup.ward_labels, the distributed placement).
 * alq_band_alloc / alq_band_open / alq_band_close / alq_band_free: device memory for one band that another process can
 *   map.  alloc: a cudaMalloc allocation of `bytes` (> 0) of its own -- an IPC handle names the base of an allocation,
 *   so a block of a caching allocator cannot be exported -- and its ALQ_IPC_HANDLE_BYTES handle (ALQ_ERR_NOMEM if the
 *   device cannot hold it).  open: maps a handle from another process (cudaIpcOpenMemHandle; ALQ_ERR_CUDA without
 *   peer access).  close: unmaps what open returned.  free: releases what alloc returned; the owner frees only after
 *   every process that opened the band has closed it.
 * alq_ward_labels: host-only, needs no GPU.  From K8's merge list: the stable sort by distance and scipy's union-find
 *   relabelling (hierarchy.ward's Z), then sklearn's _hc_cut(n_clusters): labels_host[0..n) in [0, n_clusters),
 *   numbered in the order of the cut's final heap.  ALQ_ERR_INVALID if n_clusters > n, or if the list is not a merge
 *   tree: an index out of range, x == y, a NaN distance, or a pair whose clusters were already joined (the n - 1
 *   pairs must form a spanning tree of the n rows), so that every label is written on success.                   */
int alq_pdist_f64(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, double* dist, int64_t ldd,
                  void* stream);
int alq_ward_nn_chain(alq_ctx* ctx, double* dist, int64_t n, int64_t ldd, int32_t* merge_xy, double* merge_dist,
                      void* stream);
int alq_pdist_f64_condensed(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, double* dist, void* stream);
int alq_ward_nn_chain_condensed(alq_ctx* ctx, double* dist, int64_t n, int32_t* merge_xy, double* merge_dist,
                                void* stream);
int alq_pdist_f64_condensed_rows(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, int64_t row_lo,
                                 int64_t row_hi, double* dist, void* stream);
int alq_pdist_f64_expand(alq_ctx* ctx, const double* rows, int64_t n, int64_t row_lo, int64_t row_hi, double* dist,
                         int64_t ldd, void* stream);
int alq_ward_labels(const int32_t* merge_xy_host, const double* merge_dist_host, int64_t n, int32_t n_clusters,
                    int32_t* labels_host);
int alq_ward_nn_chain_banded(alq_ctx* ctx, const int64_t* row_cuts_host, void* const* bands_host, int32_t nbands,
                             int64_t n, int32_t* merge_xy, double* merge_dist, void* stream);
int alq_band_alloc(alq_ctx* ctx, size_t bytes, void** ptr_out, void* handle_out);
int alq_band_open(alq_ctx* ctx, const void* handle, void** ptr_out);
int alq_band_close(alq_ctx* ctx, void* ptr);
int alq_band_free(alq_ctx* ctx, void* ptr);

/* ---- K9: the VAAL discriminator (VAALSampler) ---------------------------------------------------------------------
 * vaal_sampler.py:57-58 scores every pool row by the discriminator of vaal_discriminator.py on the VAE's mu:
 *     p[i] = sigmoid(w3 . relu(W2 relu(W1 mu_i + b1) + b2) + b3)
 * for fp32 rows mu[n, z] (leading dimension ldmu >= z), W1 [hidden, z] (ldw1 >= z), b1 [hidden], W2 [hidden, hidden]
 * (ldw2 >= hidden), b2 [hidden], w3 [hidden] (the single row of the last Linear) and b3 [1], all device pointers.
 * hidden must be 512, the reference's only width.  Both contractions run on the tensor cores as 3xTF32 (fp32 to about
 * 2^-21 per product); the last layer is a fixed-order sum per row, so equal rows give equal p.  logits (optional, may
 * be NULL) receives the pre-sigmoid value.  mu, w1, w2 16-byte aligned and every ld a multiple of 4, otherwise
 * ALQ_ERR_INVALID.  The pool runs in slices of at most 131 072 rows, so the scratch is bounded (about 0.6 GB at
 * z = 64) whatever n is.  Rank the rows with alq_select_smallest on p.                                              */
int alq_vaal_scores(alq_ctx* ctx, const float* mu, int64_t n, int32_t z, int64_t ldmu, const float* w1, int64_t ldw1,
                    const float* b1, const float* w2, int64_t ldw2, const float* b2, const float* w3, const float* b3,
                    int32_t hidden, float* p, float* logits, void* stream);

/* ---- K10: per-class counts and class-balanced picks (BalancedRandomSampler) --------------------------------------
 * balanced_random_sampler.py:29-95 counts the available rows of every class and then, class by class, takes the
 * rows `cur_available_idxs.nonzero()[torch.randperm(n_c)][:k_c]`.  Inputs: labels[n] (int32, device) and avail[n]
 * (uint8, device; non-zero = the row may be picked), n < 2^31, 1 <= C <= ALQ_CLASS_MAX.  Rows whose avail is 0 are
 * never inspected.  Both calls read the pool once: the pool is cut into tiles of ALQ_CLASS_TILE * ceil(C /
 * ALQ_CLASS_TILE) rows, each tile's histogram is built in shared memory (4 C bytes, hence the bound on C) and
 * scanned per class.  The table lives in the context's scratch arena: 4 C (ceil(n / tile) + 1) bytes, at most
 * 4 (n + 2 C), plus 4 (C + 1) bytes of budget offsets for alq_class_pick.  The two calls share no state.
 *
 * alq_class_counts: counts[c] (int32, device) = the number of rows with avail != 0 and labels == c.  An available
 *   row whose label is outside [0, C) makes the call return ALQ_ERR_INVALID; alq_last_error names the smallest such
 *   row and its label.  Because that can only be seen on the device, this call synchronises the stream once, after
 *   the pass (the counts themselves stay on the device).
 * alq_class_pick: k[C] (int32, device) are per-class budgets and perm[B] (int32, device) the concatenated
 *   permutation prefixes, classes ascending: out[off_c + j] (int32, device; off_c = k_0 + ... + k_{c-1}) = the
 *   perm[off_c + j]-th (from 0) available row of class c in ascending row order, for j < k_c.  An output whose rank
 *   is not in [0, n_c), or that lies past the sum of k, is -1; a negative k_c counts as 0; available rows with a label
 *   outside [0, C) belong to no class.  Asynchronous; four launches whatever C and B are.  Deterministic.       */
#define ALQ_CLASS_MAX 32768
#define ALQ_CLASS_TILE 1024
int alq_class_counts(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int64_t n, int32_t c, int32_t* counts,
                     void* stream);
int alq_class_pick(alq_ctx* ctx, const int32_t* labels, const uint8_t* avail, int64_t n, int32_t c, const int32_t* k,
                   const int32_t* perm, int64_t b, int32_t* out, void* stream);

/* ---- K11: the whole query of BalancingSampler as one persistent launch -------------------------------------------
 * balancing_sampler.py:58-134 picks one row per step: when the labeled class histogram is imbalanced relative to the
 * remaining budget (:66-84, evaluated in fp32 exactly as torch does on the CPU) it takes the available row with the
 * smallest d2(row, rarest centre) / max over the majority centres of d2(row, centre) (numerator 1 when the rarest class
 * has no labeled row; lowest row on ties, NaN ranked as alq_ratio_argmin ranks it), otherwise one legacy
 * `np.random.choice` over the available rows (MT19937, masked rejection draws).  After a pick the row is labeled, its
 * class count rises and that class's centre is recomputed.
 *
 * Inputs (device unless _host): x[n, d] fp32 rows (d % 4 == 0, ldx % 4 == 0, 16-byte aligned), xn[n] = alq_row_norm2(x),
 * labels[n] int32, avail[n] / labeled[n] uint8 masks (not modified), c classes, the budget, and NumPy's MT19937 state
 * (np.random.get_state(): 624 key words and the position).  Class sums are fp64 in a fixed order (labeled rows in row
 * order per chunk of 65 536 rows, the chunks in order, then the picks in pick order); a centre is
 * fl32(sum / fl32(count + 1e-5)); a row's dot product with a centre is a fixed function of the row (lane-strided fmaf
 * chains folded by a butterfly), whatever the grid, so the picks are bit-reproducible.
 * Outputs: picks[0 .. *n_picks_host) int32 in pick order, *n_picks_host = min(budget, available rows),
 * *n_balancing_host = the steps that balanced, and the MT19937 key / position after the last draw (in place).
 * An available or labeled row whose label is outside [0, c) makes the call return ALQ_ERR_INVALID naming the row and
 * its label, before any draw.
 * Limits (option "balancing_loop"): every centre (4 c d bytes) plus the per-CTA tables fit the shared memory of one
 * CTA, and 1 KB per class for the fp64 set-up pass; at most 65 535 rows per CTA segment (n < 65 536 * SMs); every class
 * count plus the budget below 2^24 (the fp32 imbalance test is exact there).  Beyond them the call declines
 * (*n_picks_host = -1, nothing drawn) under option 0, 1 or 3 and fails with ALQ_ERR_INVALID under option 2.
 * Launches: K10's table pass (2), one segment count, two fp64 set-up passes and the loop: six, whatever the budget.
 * Synchronous (it reads the label check, the counts and the final RNG state back).
 *
 * Rows sharded over a group (K11 and K12; shard_off_host non-NULL; needs alq_comm_create/connect).  Every array stays
 * GLOBAL and REPLICATED on every rank (x, xn, labels, avail, labeled: n rows each); rank r streams rows
 * [shard_off[r], shard_off[r + 1]) only, so a pick is announced as a row id and read from the local replica.  Every rank
 * runs the same number of CTAs (from the smallest shard), counts the available rows of every rank's CTA segments and
 * keeps the same counts, centres or class sums and MT19937 state; a balancing step exchanges one 8-byte key word per CTA
 * through the peer-memory windows, a random step the owner's pick word.  The words share the window region of the
 * persistent selection loop (alq_greedy_select) and its start-of-call ready handshake, and their tags carry the call's
 * epoch.  Picks, the balancing steps and the written-back MT19937 state are identical on every rank and bit-identical to
 * the single-GPU call on the same inputs; with one rank and shard_off = {0, n} the CTA segments are exactly the
 * single-GPU ones.  Collective: every rank makes the call with the same inputs (the caller checks that; Engine does),
 * in the same order relative to its other group calls, and the ranks take the same run-or-decline decision (the shape
 * limits, the window's room for one word per pick, and K12's memory check on group_free_bytes).  Every wait is bounded
 * by "spin_timeout_ms": a rank that fails after the decision ends the call with ALQ_ERR_STATE on its peers, never with a
 * hang.  A descriptor whose struct_size ends before shard_off_host is a single-GPU call.                          */
typedef struct alq_balancing_desc {
    size_t struct_size;          /* sizeof(alq_balancing_desc) */
    const float* x;  int64_t ldx; int32_t d;
    const float* xn;             /* [n] |x_i|^2 */
    const int32_t* labels;       /* [n] */
    const uint8_t* avail;        /* [n] non-zero: the row may be picked */
    const uint8_t* labeled;      /* [n] non-zero: the row is labeled (class histogram, centres) */
    int64_t n;
    int32_t c;
    int64_t budget;
    uint32_t* mt_key_host;       /* [624] in/out: np.random.get_state()[1] */
    int32_t* mt_pos_host;        /* in/out: np.random.get_state()[2] */
    int32_t* picks;              /* [budget] out */
    int64_t* n_picks_host;       /* out: picks written, or -1 when the call declined (option / limits) */
    int64_t* n_balancing_host;   /* out: balancing steps among them */
    const int32_t* shard_off_host;   /* [world + 1] rows per rank of a sharded call, or NULL: one GPU */
    int64_t group_free_bytes;    /* sharded K12: the least free device memory (bytes) over the group's ranks, gathered by
                                    the caller before the call; the table check tests every rank's share against it */
} alq_balancing_desc;

int alq_balancing_select(alq_ctx* ctx, const alq_balancing_desc* desc, void* stream);

/* ---- K12: the same query at large class counts, over an incremental row x class table ----------------------------
 * Same descriptor, same semantics and same outputs as alq_balancing_select (the branch test, numerator 1, NumPy's
 * draws and state, the lowest row on ties, NaN ranked as alq_ratio_argmin ranks it, the label check); only the
 * distance arithmetic differs, so that it does not need the C x d centres in shared memory.
 * At the first balancing step every available row i gets a table row T[i, c] = <x_i, S_c> (fp64; S_c the fp64 sum of
 * class c's labeled rows, in row order) and xn64_i = <x_i, x_i> (fp64).  A balancing step scores
 *     d2(i, c) = xn64_i - 2 T[i, c] / den_c + q_c / den_c^2,   den_c = fl32(n_c + 1e-5),  q_c = <S_c, S_c> (fp64),
 * which is |x_i - m_c|^2 for the unrounded centre m_c = S_c / den_c (K11 rounds the centre to fp32), and ranks
 * the rows by (fl32(near / far), row) with the ratio formed in fp64 and rounded once.  After a pick p of class y every
 * table row gets T[i, y] += <x_i, x_p> (fp64 sums of exact fp32 products in a fixed order), applied while the next
 * balancing step streams the rows; a query that never balances builds no table.  The picks are bit-reproducible and
 * do not depend on the grid; they differ from K11's or the per-step path's only where fp32 rounding decides the
 * arg-min (two best ratios within about 1e-6 relative).
 * Limits (option "balancing_loop"): the per-class tables (20 c bytes), the per-segment counts, the MT state and at
 * least one pending row (4 d bytes) fit one CTA's shared memory; at most 65 535 rows per CTA segment; the labeled count
 * plus the budget below 2^24; the table (8 n_avail c bytes) plus one copy of the fp64 class sums per CTA (8 c d grid
 * bytes) fit the device's free memory, checked before any of it is reserved (the context's grow-only scratch keeps it
 * after the call).  Beyond them the call declines (*n_picks_host = -1, nothing drawn) under option 0 and fails with
 * ALQ_ERR_INVALID naming the limit under option 3; options 1 and 2 always decline.
 * Launches: K10's table pass (2), one segment count, one grouping of the labeled rows by class, one class-sum pass and
 * the loop: six, whatever the budget.  Synchronous.                                                               */
int alq_balancing_table_select(alq_ctx* ctx, const alq_balancing_desc* desc, void* stream);

/* ---- K13 / K14: ProbCover (Yehuda et al., NeurIPS 2022) --------------------------------------------------------------
 * alq_probcover_graph (K13): the delta-ball graph of x[n, d] (fp32, d % 4 == 0, ldx >= d, any alignment) as CSR.  Every
 *   row is L2-normalised into xhat[n, d] (caller-owned, 16-byte aligned): lane l of a warp sums the fp64 squares of
 *   columns l, l + 32, .. in order, a butterfly (xor 16, 8, 4, 2, 1) adds the 32 partials, norm = sqrt, and
 *   xhat = fl32(x / norm) in fp64 (a zero row stays zero).  There is an edge (i, j) iff scipy's fp64 euclidean distance of
 *   xhat_i and xhat_j (K7's pair arithmetic: d = a - b, s = s + d * d, k ascending, no FMA, sqrt) is < *delta_host, so
 *   every (i, i) is an edge.  The pairs are screened on the tensor cores (3xTF32) with a rigorous error bound (DESIGN
 *   section 4); only pairs inside the bound's band are recomputed exactly.  Two calls, same x, d and delta:
 *     count (cols == NULL): writes xhat, tile_cnt (caller-owned int32 [n * ceil(n / 128)], scratch of the fill), row_ptr
 *       (int64 [n + 1]), *nnz_host = row_ptr[n] and *recheck_host = the pairs decided by the exact recomputation.
 *     fill (cols != NULL, int32 [nnz]): reads xhat, tile_cnt and row_ptr as the count left them (x is not read) and
 *       writes every row's columns, ascending; (i, j) and (j, i) are both stored.
 *   The caller checks that nnz fits in memory between the two calls.  n in [1, 2^31), delta finite and > 0, otherwise
 *   ALQ_ERR_INVALID.  Synchronous.
 * alq_probcover_select (K14): the greedy coverage picks over that CSR.  covered[y] starts true for every y in the ball
 *   of a row with labeled[row] != 0 and deg[x] = |{y in N(x) : y uncovered}|; each step stops if max deg = 0, else picks
 *   c = the lowest row of the maximum and covers every uncovered y in N(c).  picks[0 .. *n_steps_host) (int32, device) in
 *   pick order, *n_steps_host <= budget <= n.  Set-up: two launches; then ONE launch runs every step (one CTA per SM,
 *   agreement over 8-byte LL words, every wait bounded by "spin_timeout_ms"); at most 65 535 rows per CTA segment.
 *   Synchronous. */
int alq_probcover_graph(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, const double* delta_host,
                        float* xhat, int32_t* tile_cnt, int64_t* row_ptr, int32_t* cols, int64_t* nnz_host,
                        int64_t* recheck_host, void* stream);
int alq_probcover_select(alq_ctx* ctx, const int64_t* row_ptr, const int32_t* cols, int64_t n, const uint8_t* labeled,
                         int64_t budget, int32_t* picks, int64_t* n_steps_host, void* stream);

/* ---- K15 / K16 / K17: TypiClust (Hacohen, Dekel & Weinshall, ICML 2022) ----------------------------------------------
 * alq_kmeans_rows: normalise != 0: xhat = x's rows L2-normalised exactly as alq_probcover_graph does; normalise == 0: xhat
 *   is the input.  Then hi / lo = the TF32 split of xhat and nrm2 = |xhat|^2 in fp64, the operands of alq_kmeans_assign.
 *   x[n, d] (fp32, ldx >= d), xhat, hi, lo [n, d] (16-byte aligned), d % 4 == 0.  Asynchronous on `stream`.
 * alq_kmeans_assign (K15): labels[i] = the lowest c of the minimum over c < K of the exact fp64 d2(xhat_i, centres_c)
 *   (K7's pair arithmetic: d = a - b, s = s + d * d, k ascending, no FMA).  The pairs are screened on the tensor cores
 *   (3xTF32) with a rigorous band (DESIGN section 4); a row whose nearest centre the band cannot isolate is recomputed
 *   exactly against every centre.  labels is read (the previous labels; any value outside [0, K) counts as a change)
 *   and written.  counts_host[0] = rows whose label changed, counts_host[1] = rows rechecked.  K in [1, 32768].
 *   Synchronous (one 8-byte copy).
 * alq_kmeans_update (K16): for every c < K with m_c = |{i : labels[i] == c}| > 0, centres[c] = fl32(S_c / m_c), S_c the
 *   fp64 sum of the member rows of xhat in ascending row order (one sequential chain per column).  Clusters with no
 *   member, and rows whose label is outside [0, K), are left alone.  K in [1, 32768].  Asynchronous on `stream`.
 * alq_typicality (K17): rows[group_off_host[g] .. group_off_host[g + 1]) (int32 row ids of xhat[., d], device) form group
 *   g, every group non-empty.  For each listed row, k = min(k_max, m_g / 2) and mean = the ascending fp64 sum of the k
 *   smallest exact fp64 d2 (K7's arithmetic) to the other rows of its group (itself excluded by position) divided by k;
 *   typ = 1 / (mean + 1e-5) (fp64, device, one per listed row; 0 for a group of one row).  best[g] = the position in
 *   rows of the group's largest typ, the lowest on ties.  k_max in [1, 32].  Synchronous.
 * alq_kmeans_nearest (K21): nearest[c] (int32, device) = for every c < K the row i with labels[i] == c and the smallest
 *   exact fp64 d2(xhat_i, centres_c) (K7's pair arithmetic), the lowest row on ties; -1 when no row is labeled c.  Rows
 *   whose label is outside [0, K) are skipped.  xhat [n, d], centres [K, d]: fp32, 16-byte aligned, d % 4 == 0.
 *   Asynchronous on `stream`. */
int alq_kmeans_rows(alq_ctx* ctx, const float* x, int64_t n, int32_t d, int64_t ldx, int32_t normalise, float* xhat,
                    float* hi, float* lo, double* nrm2, void* stream);
int alq_kmeans_assign(alq_ctx* ctx, const float* xhat, const float* hi, const float* lo, const double* nrm2, int64_t n,
                      int32_t d, const float* centres, int32_t k, int32_t* labels, int64_t* counts_host, void* stream);
int alq_kmeans_update(alq_ctx* ctx, const float* xhat, int64_t n, int32_t d, const int32_t* labels, int32_t k,
                      float* centres, void* stream);
int alq_typicality(alq_ctx* ctx, const float* xhat, int32_t d, const int32_t* rows, const int64_t* group_off_host,
                   int32_t groups, int32_t k_max, double* typ, int32_t* best, void* stream);
int alq_kmeans_nearest(alq_ctx* ctx, const float* xhat, int64_t n, int32_t d, const int32_t* labels, const float* centres,
                       int32_t k, int32_t* nearest, void* stream);

/* ---- K18 / K19: CAL (Margatina, Vernikos, Barrault & Aletras, EMNLP 2021) ---------------------------------------------
 * alq_knn (K18): for every row i of x[n, d], idx[i][0..k) = the k rows j of y[m, d] with the smallest exact fp64
 *   d2(x_i, y_j) (K7's pair arithmetic on the raw rows: d = a - b, s = s + d * d, k ascending, no FMA), in ascending
 *   (d2, j) order, and d2[i][0..k) their values.  When m < k the last k - m entries of a row are idx -1, d2 +inf.  The
 *   pairs are screened on the tensor cores (3xTF32) with a rigorous band (DESIGN section 4); each row keeps 32 candidate
 *   columns and takes an exact scan of all m rows when they cannot certify its k nearest.  x, y: fp32, contiguous rows
 *   (pitch d), 16-byte aligned, d % 4 == 0; every squared row norm finite and at most 2^100 (ALQ_ERR_INVALID otherwise).
 *   idx int32 [n, k], d2 fp64 [n, k], device.  k in [1, 32].  *fallback_rows_host = the rows that took the exact scan.
 *   Synchronous (two 4-byte copies).
 * alq_cal_scores (K19): per row r of cand_logits[n, C] and ref_logits[m, C] (fp32, contiguous rows), in fp64:
 *   lse_r = mx_r + log(sum_c exp(z_rc - mx_r)) (c ascending, mx_r = max_c z_rc), lp_rc = z_rc - lse_r, p_rc = exp(lp_rc).
 *   For candidate i and each idx[i][j] in [0, m) (other entries are skipped): KL_j = sum_c p_nc (lp_nc - lp_ic),
 *   c ascending; score[i] = (sum of the KL_j in list order) / (their number), 0 when there is none.  key[i] =
 *   -fl32(score[i]), +0.0 when fl32(score[i]) is zero and +NaN when score[i] is NaN: alq_select_smallest on key takes the
 *   largest scores first, the lowest row on ties.  idx int32 [n, k], score fp64 [n], key fp32 [n], device.  k in
 *   [1, 32].  Asynchronous on `stream`. */
int alq_knn(alq_ctx* ctx, const float* x, int64_t n, const float* y, int64_t m, int32_t d, int32_t k, int32_t* idx,
            double* d2, int64_t* fallback_rows_host, void* stream);
int alq_cal_scores(alq_ctx* ctx, const float* cand_logits, int64_t n, const float* ref_logits, int64_t m, int32_t c,
                   const int32_t* idx, int32_t k, double* score, float* key, void* stream);

/* ---- K20: ALFA-Mix (Parvaneh et al., CVPR 2022) -----------------------------------------------------------------------
 * alq_alfamix_rho (K20): the closed-form feature-mixing test of every row u of logits[n, C] (fp32, contiguous) with its
 *   embedding emb[n, dp] against the head weight[C, D] and the anchors[C, dp] (fp32, contiguous; emb and anchors padded
 *   with zero columns from D to dp, dp % 4 == 0).  In fp64: G = weight weight^T (ascending-d chain per entry);
 *   lse_u as alq_cal_scores forms it, yhat = the lowest class of the largest logit, r_c = exp(l_c - lse_u) - [c == yhat];
 *   w_k = sum_c G_kc r_c (c ascending); s2 = sum_k r_k w_k (k ascending); t* = min over {k : w_k > w_yhat} of
 *   ((l_yhat - l_k) sqrt(s2)) / (w_k - w_yhat), +inf when s2 <= 0 or no k qualifies; R2 = max_c of the exact fp64
 *   d2(emb_u, anchors_c) (K7's pair arithmetic); rho = (sqrt(D) t*) / sqrt(R2), +inf when R2 = 0 or t* = +inf.
 *   rho, r2 and tstar are fp64 [n] on the device; r2 and tstar may be NULL.  C >= 2, 1 <= D <= dp; a non-finite logit,
 *   embedding, anchor or weight entry is ALQ_ERR_INVALID.  Synchronous. */
int alq_alfamix_rho(alq_ctx* ctx, const float* logits, int64_t n, int32_t c, const float* emb, int32_t dp,
                    const float* anchors, const float* weight, int32_t d, double* rho, double* r2, double* tstar,
                    void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ALQ_H_ */
