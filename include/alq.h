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
 *   - All arithmetic is IEEE fp32 (fp64 only for the inverse-CDF search); index math is int32 on
 *     the device (n < 2^31).  There is no CPU fallback anywhere in this library.
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
 *   "greedy_variant" 0 auto | 1 direct-load step kernel     | 2 bulk-copy (TMA) pipeline | 3 persistent cooperative loop
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
 *   "base_impl"      0 auto | 1 sequential class loop       | 2 per-class candidate lists + in-order resolve */
int alq_set_option(alq_ctx* ctx, const char* key, int64_t value);
/* Number of kernels this context has launched since creation (bench.py's `gpu_launches`). */
int64_t alq_launch_count(const alq_ctx* ctx);

/* ---- multi-GPU group: one process per GPU, peer-memory windows over NVLink ---------------------
 * alq_comm_create allocates this rank's window and returns its 64-byte CUDA IPC handle; the caller
 * exchanges the handles (e.g. torch.distributed.all_gather) and passes all of them, in rank order, to
 * alq_comm_connect.  The global (non-partitioned) CoreSet / k-means++ loops then exchange their
 * per-step winner through these windows from inside the kernels (alq_greedy_desc.shard_off_host).   */
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

/* The same tail with the rows sharded over the G ranks of the peer-memory group (alq_comm_create/connect): rank r holds
 * `n` rows that are positions [row_lo, row_lo + n) of the pool and every rank receives the same out_gpos[0..b): the global
 * positions of the b smallest scores over ALL ranks, ascending (score, position) -- exactly what a single GPU returns for
 * the concatenated pool.  K1, K1b and the exchange are ONE launch per rank: both histogram levels are summed over
 * the ranks and the b + few candidate words gathered through the windows from inside the kernel (8-byte {tag, value} words
 * and plain stores over NVLink; no collective library, nothing on the host).  Collective: every rank calls it with the same
 * c, mode, b, rows_min / rows_max (the smallest / largest shard; they decide, identically on every rank, whether the fused
 * kernel applies -- otherwise K1, K1b and alq_topb_exchange run back to back, same result).  Asynchronous; a peer that never
 * shows up is reported through alq_comm_check like alq_topb_exchange.                                              */
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

/* The same exchange over the peer-memory windows of alq_comm_create/connect instead of a collective library:
 * pack + store into every peer's window + flag, then wait + merge (b <= 16384).  Collective: every rank of the
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
       not touched).  picks are global row ids, identical on every rank.  NULL => single GPU.
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
 * alq_mase_margins: one streaming pass over the logits slab.  pred[i] = p;  radius may be NULL (MASE needs only
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

#ifdef __cplusplus
}
#endif
#endif /* ALQ_H_ */
