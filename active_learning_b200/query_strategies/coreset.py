"""CoreSet (greedy k-center) and BADGE (k-means++ D^2 seeding) queries on the device
(kernels K2, K3, K4, K5).

Host glue of active_learning/src/query_strategies/coreset_sampler.py:21-41,107-133,
partitioned_coreset_sampler.py:36-84, badge_sampler.py:50-78 and partitioned_badge_sampler.py:
index bookkeeping and the NumPy RNG stream are reproduced call for call; everything numeric
(embeddings, distances, the B-step selection loop) stays on the GPU.
"""
from __future__ import annotations

import numpy as np
import torch

from .strategy import EngineMixin


def _gather(t, pos, dev):
    if t is None:
        return None
    return t.index_select(0, torch.as_tensor(np.asarray(pos), dtype=torch.long, device=dev))


class CoresetQuery(EngineMixin):
    RANDOMIZE = False          # CoreSet: arg-max; BADGE: D^2 sampling (badge_sampler.py:72-73)
    GRADIENT_EMBEDDING = False

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.saved_pairwise_l2_dist = None       # kept for pickle/attribute compatibility
        self._saved_embeddings = None
        self.freeze_feature = kwargs["freeze_feature"]
        self.subset_labeled = kwargs["subset_labeled"]
        self.subset_unlabeled = kwargs["subset_unlabeled"]
        self.cache_embeddings = kwargs.get("cache_embeddings", True)
        self.channels_last = kwargs.get("channels_last", True)

    # ---- coreset_sampler.py:21-41 ------------------------------------------------------------------
    def get_idxs_for_coreset(self, return_sep_idxs=False):
        idxs_for_query = self.available_query_idxs(boolean=False, shuffle=True)
        idxs_labeled = np.atleast_1d(self.already_labeled_idxs(boolean=False, shuffle=True))
        if self.subset_labeled is not None:
            subset_labeled = min(self.subset_labeled, len(idxs_labeled))
            idxs_labeled = idxs_labeled[:subset_labeled]
        if self.subset_unlabeled is not None:
            if self.subset_labeled is not None:
                cap = self.subset_labeled + self.subset_unlabeled - subset_labeled
            else:
                cap = self.subset_unlabeled
            idxs_for_query = idxs_for_query[:min(cap, len(idxs_for_query))]
        union = sorted(idxs_for_query.tolist() + idxs_labeled.tolist())
        if return_sep_idxs:
            return union, idxs_labeled.tolist(), idxs_for_query.tolist()
        return union

    # ---- embeddings ----------------------------------------------------------------------------------
    def _features(self, idxs):
        """Row features for `idxs` in loader order, on the device.

        CoreSet : (emb[n, D], None)                     coreset_sampler.py:43-57
        BADGE   : (emb[n, D], a[n, C]) rank-1 factors   badge_sampler.py:22-40 (never materialised)
        """
        self.feature_net.eval()
        if not self.GRADIENT_EMBEDDING:
            _, emb = self._forward_pool(idxs, self.feature_net, want_features=True)
            return emb, None
        logits, emb = self._forward_pool(idxs, self.net, want_features=True)
        bs = int(self.train_args["loader_te_args"]["batch_size"])
        a, _ = self.get_engine().badge_factors(logits, bs)
        return emb, a

    # ---- randomness: the reference's draws, in the reference's order -------------------------------
    def _draw(self, full_ns, n_labeled, budgets):
        """What `coreset(..., randomize=True)` pulls from np.random for each partition in turn
        (coreset_sampler.py:92,98): with nothing labeled one np.random.choice(n) for the first
        centre, then one uniform per np.random.choice(n, p=...)."""
        first, unif = [], []
        for n, nl, b in zip(full_ns, n_labeled, budgets):
            cold = int(nl == 0 and b > 0)
            first.append(int(np.random.choice(int(n))) if (cold and self.RANDOMIZE) else -1)
            u = np.zeros(b, dtype=np.float64)
            if self.RANDOMIZE and b - cold > 0:
                u[cold:] = np.random.random_sample(b - cold)
            unif.append(u)
        return first, unif

    # ---- one batched selection over P independent partitions ----------------------------------------
    def _select(self, feats, factors, lab_pos_list, cand_pos_list, bases, budgets, first, unif):
        """Partition p's labeled rows are feats[lab_pos_list[p]], its candidates
        feats[cand_pos_list[p]]; row r of the partition's matrix in the reference is feats[bases[p] + r].
        Returns, per partition, indices into cand_pos_list[p] in pick order."""
        eng = self.get_engine()
        dev = feats.device
        P = len(budgets)
        cand_all = np.concatenate([np.asarray(c, dtype=np.int64) for c in cand_pos_list])
        X = _gather(feats, cand_all, dev)
        XA = _gather(factors, cand_all, dev)
        xn = eng.row_norm2(X)
        xan = eng.row_norm2(XA) if XA is not None else None
        part_off = np.zeros(P + 1, dtype=np.int64)
        part_off[1:] = np.cumsum([len(c) for c in cand_pos_list])
        mind = torch.full((X.shape[0],), float("inf"), dtype=torch.float32, device=dev)
        first_pick = np.full(P, -1, dtype=np.int32)
        vpos = np.zeros(X.shape[0], dtype=np.int32)
        full_n = np.zeros(P, dtype=np.int32)

        def sl(t, lo, hi):
            return t[lo:hi] if t is not None else None

        for p in range(P):
            lo, hi = int(part_off[p]), int(part_off[p + 1])
            lab_pos = np.asarray(lab_pos_list[p], dtype=np.int64)
            full_n[p] = len(lab_pos) + (hi - lo)
            vpos[lo:hi] = np.asarray(cand_pos_list[p], dtype=np.int64) - bases[p]
            if budgets[p] <= 0:
                continue
            if len(lab_pos):
                Y, YA = _gather(feats, lab_pos, dev), _gather(factors, lab_pos, dev)
                eng.min_dist(X[lo:hi], xn[lo:hi], Y, eng.row_norm2(Y), sl(XA, lo, hi), sl(xan, lo, hi),
                             YA, eng.row_norm2(YA) if YA is not None else None, out=mind[lo:hi])
            elif self.RANDOMIZE:
                # nothing labeled: the matrix rows ARE the candidates, so position == candidate row
                first_pick[p] = lo + first[p]
            else:
                far = eng.min_dist(X[lo:hi], xn[lo:hi], X[lo:hi], xn[lo:hi], sl(XA, lo, hi), sl(xan, lo, hi),
                                   sl(XA, lo, hi), sl(xan, lo, hi), reduce_max=True)
                first_pick[p] = lo + eng.argmin(far)            # minimax centre, coreset_sampler.py:100
        picks = eng.greedy_select(
            X, xn, mind, part_off.astype(np.int32), np.asarray(budgets, dtype=np.int32), a=XA, an=xan,
            uniforms=np.concatenate(unif) if self.RANDOMIZE else None,
            vpos=torch.as_tensor(vpos, device=dev) if self.RANDOMIZE else None,
            full_n=full_n if self.RANDOMIZE else None, first_pick=first_pick)
        out, at = [], 0
        for p in range(P):
            b = int(budgets[p])
            out.append(np.asarray(picks[at:at + b], dtype=np.int64) - int(part_off[p]))
            at += b
        return out

    # ---- coreset_sampler.py:107-133 / badge_sampler.py:50-78 ---------------------------------------
    def query(self, budget):
        union = np.asarray(self.get_idxs_for_coreset(), dtype=np.int64)      # RNG: two permutations (:22-23)
        group = getattr(self, "_shard_group", None)
        if group is not None and group.world_size > 1:
            return self._query_global_sharded(union, budget, group)
        cacheable = (self.freeze_feature and not self.GRADIENT_EMBEDDING
                     and self.subset_unlabeled is None and self.subset_labeled is None)
        saved = getattr(self, "_saved_embeddings", None)
        if cacheable and saved is not None and saved[0].shape[0] == len(union):
            feats, factors = saved       # the reference caches the N x N matrix here (:112-121)
        else:
            feats, factors = self._features(union.tolist())
            if cacheable:
                self._saved_embeddings = (feats, factors)
        is_lab = self.already_labeled_idxs(boolean=True)[union]
        budget = int(min(self.available_query_idxs(boolean=True)[union].sum(), budget))
        if budget <= 0:
            return [], 0
        lab_pos, cand_pos = np.flatnonzero(is_lab), np.flatnonzero(~is_lab)
        first, unif = self._draw([len(union)], [len(lab_pos)], [budget])
        picks = self._select(feats, factors, [lab_pos], [cand_pos], [0], [budget], first, unif)[0]
        labeled_idxs_cur_rd = union[cand_pos[picks]].tolist()
        return labeled_idxs_cur_rd, len(labeled_idxs_cur_rd)

    # ---- the same query with the work sharded over the ranks of a ShardGroup ------------------------------
    def _query_global_sharded(self, union, budget, group):
        """Every rank forwards rows [lo, hi) of the sorted union; the embeddings (and BADGE factors) are
        all-gathered once, so every rank holds a replica of every row (a few hundred MB next to 180 GB).  The
        distance pass (K3) and the selection loop (K4 / K5) are then sharded by candidate row: a new centre is
        announced as a row id through the engine's peer-memory windows and read from the local replica.  Host
        bookkeeping and the RNG stream are replicated, so every rank returns the single-GPU list."""
        from ..sharding import plan_shards
        eng = self.get_engine()
        is_lab = self.already_labeled_idxs(boolean=True)[union]
        budget = int(min(self.available_query_idxs(boolean=True)[union].sum(), budget))
        if budget <= 0:
            return [], 0
        n_u, G, r = len(union), group.world_size, group.rank
        bounds = [group.row_range(n_u, q) for q in range(G)]
        lo, hi = bounds[r]
        lab_pos, cand_pos = np.flatnonzero(is_lab), np.flatnonzero(~is_lab)
        first, unif = self._draw([n_u], [len(lab_pos)], [budget])

        self.feature_net.eval()
        if self.GRADIENT_EMBEDDING:
            logits, emb = self._forward_pool(union[lo:hi].tolist(), self.net, want_features=True)
            bs = int(self.train_args["loader_te_args"]["batch_size"])
            factors, _ = eng.badge_factors(logits, bs, row0=lo, n_total=n_u)      # 1/bs of the GLOBAL loader pass
        else:
            _, emb = self._forward_pool(union[lo:hi].tolist(), self.feature_net, want_features=True)
            factors = None
        dev = emb.device
        counts = [b - a for a, b in bounds]
        feats = group.all_gather_rows(emb, counts)                                 # [n_u, D] on every rank
        factors = group.all_gather_rows(factors, counts) if factors is not None else None
        X, XA = _gather(feats, cand_pos, dev), _gather(factors, cand_pos, dev)
        xn = eng.row_norm2(X)
        xan = eng.row_norm2(XA) if XA is not None else None
        shard_off, shard_pos = plan_shards(cand_pos, n_u, G, leaf_aligned=self.RANDOMIZE)
        s0, s1 = int(shard_off[r]), int(shard_off[r + 1])

        def sl(t):
            return t[s0:s1] if t is not None else None

        mind = torch.full((X.shape[0],), float("inf"), dtype=torch.float32, device=dev)
        first_pick = -1
        if len(lab_pos):
            Y, YA = _gather(feats, lab_pos, dev), _gather(factors, lab_pos, dev)
            if s1 > s0:
                eng.min_dist(X[s0:s1], xn[s0:s1], Y, eng.row_norm2(Y), sl(XA), sl(xan), YA,
                             eng.row_norm2(YA) if YA is not None else None, out=mind[s0:s1])
        elif self.RANDOMIZE:
            first_pick = int(first[0])            # nothing labeled: position == candidate row (coreset_sampler.py:98)
        else:
            far = torch.empty(0, dtype=torch.float32, device=dev)
            if s1 > s0:
                far = eng.min_dist(X[s0:s1], xn[s0:s1], X, xn, sl(XA), sl(xan), XA, xan, reduce_max=True)
            far_all = group.all_gather_rows(far, [int(shard_off[q + 1] - shard_off[q]) for q in range(G)])
            first_pick = eng.argmin(far_all)      # minimax centre, coreset_sampler.py:100
        picks = eng.greedy_select(
            X, xn, mind, [0, X.shape[0]], [budget], a=XA, an=xan,
            uniforms=unif[0] if self.RANDOMIZE else None,
            vpos=torch.as_tensor(cand_pos.astype(np.int32), device=dev) if self.RANDOMIZE else None,
            full_n=[n_u] if self.RANDOMIZE else None, first_pick=[first_pick],
            shard_off=shard_off, shard_pos=shard_pos)
        labeled_idxs_cur_rd = union[cand_pos[np.asarray(picks, dtype=np.int64)]].tolist()
        return labeled_idxs_cur_rd, len(labeled_idxs_cur_rd)


class PoolQuery(CoresetQuery):
    """The query body of the samplers that pick from CoreSet's pool by a rule of their own (ProbCover, TypiClust, CAL,
    ALFA-Mix, MaxHerding, BAIT).

    The pool is CoreSet's (`get_idxs_for_coreset`: the same two shuffles, subset_labeled / subset_unlabeled honoured) and
    the budget is clamped to its available rows; a budget <= 0 returns ([], 0) before anything else runs.  A subclass's
    `_positions` returns pool positions in pick order, possibly fewer than the budget.  One deliberate deviation from the
    papers: where a sampler's rule runs out of picks (the authors' loops would repeat a pick or index an empty cluster),
    the rest of the budget is `np.random.choice(available-and-unpicked positions ascending, rest, replace=False)`, drawn
    only when something is left.  In a ShardGroup every rank runs the whole query on its own GPU and returns the same
    picks."""

    def query(self, budget):
        union = np.asarray(self.get_idxs_for_coreset(), dtype=np.int64)      # RNG: two permutations
        is_lab = self.already_labeled_idxs(boolean=True)[union]
        avail = self.available_query_idxs(boolean=True)[union]
        budget = int(min(int(avail.sum()), budget))
        if budget <= 0:
            return [], 0
        picks = self._positions(union, is_lab, avail, budget)
        rest = budget - len(picks)
        if rest > 0:
            free = avail.copy()
            free[picks] = False
            picks = np.concatenate([picks, np.random.choice(np.flatnonzero(free), rest, replace=False)])
        labeled_idxs_cur_rd = union[picks].tolist()
        return labeled_idxs_cur_rd, len(labeled_idxs_cur_rd)

    def _positions(self, union, is_lab, avail, budget):
        """Positions in the pool in pick order, at most `budget` of them."""
        raise NotImplementedError

    def _kmeans(self, xhat, k, max_iter):
        """Engine.kmeans of the rows of xhat into k clusters, seeded by CoresetQuery's D^2 cold start: one
        np.random.choice(n) for the first centre, then k - 1 np.random.random_sample uniforms."""
        first = int(np.random.choice(xhat.shape[0]))
        unif = np.random.random_sample(k - 1)
        return self.get_engine().kmeans(xhat, first, unif, k, max_iter)


class PartitionedCoresetQuery(CoresetQuery):
    """partitioned_coreset_sampler.py: the selection runs independently inside `partitions` random
    groups.  Here the groups are one batch dimension of the same kernels (and, multi-GPU, the unit
    that is dealt to ranks: no collective inside the loop)."""
    POOLED = False

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.partitions = kwargs["partitions"]

    def generate_partition_idxs_list(self, input_idxs):
        """partitioned_coreset_sampler.py:36-47."""
        idxs = np.array(input_idxs)
        np.random.shuffle(idxs)
        out, cum = [], 0
        for i in range(self.partitions):
            m = int(len(input_idxs) / self.partitions) + int(i < len(input_idxs) % self.partitions)
            out.append(idxs[cum:cum + m])
            cum += m
        return out

    def query(self, budget):
        _, labeled_idxs, unlabeled_idxs = self.get_idxs_for_coreset(return_sep_idxs=True)
        lab_parts = self.generate_partition_idxs_list(labeled_idxs)
        unl_parts = self.generate_partition_idxs_list(unlabeled_idxs)
        budget = int(min(len(unlabeled_idxs), budget))
        P = self.partitions
        budgets = [int(budget / P) + int(i < budget % P) for i in range(P)]
        rows = [np.concatenate((lab_parts[i], unl_parts[i])).astype(np.int64) for i in range(P)]
        # every rank draws for ALL partitions (identical stream everywhere) and runs its own share
        first, unif = self._draw([len(r) for r in rows], [len(l) for l in lab_parts], budgets)
        group = getattr(self, "_shard_group", None)
        if group is None or group.world_size == 1:
            picked = self._run_partitions(list(range(P)), rows, lab_parts, budgets, first, unif)
        else:
            mine = group.my_partitions(P)
            picked = group.all_gather_dict(self._run_partitions(mine, rows, lab_parts, budgets, first, unif))
        out = []
        for i in range(P):
            out += list(rows[i][len(lab_parts[i]) + picked[i]])
        return sorted(int(v) for v in out), len(out)

    def _run_partitions(self, which, rows, lab_parts, budgets, first, unif):
        """Embeds and selects for the partitions in `which` as one batch."""
        if not which:
            return {}
        eng = self.get_engine()
        sizes = [len(rows[i]) for i in which]
        flat = np.concatenate([rows[i] for i in which]).tolist()
        if self.GRADIENT_EMBEDDING and self.POOLED:
            # one loader pass per partition in the reference: each partition's short last batch has its
            # own 1/bs (badge_sampler.py:36-37), so K2p runs per partition slice
            self.feature_net.eval()
            logits, emb = self._forward_pool(flat, self.net, want_features=True)
            bs = int(self.train_args["loader_te_args"]["batch_size"])
            chunks, at = [], 0
            for m in sizes:
                chunks.append(eng.badge_pooled_embedding(logits[at:at + m], emb[at:at + m], bs))
                at += m
            feats, factors = torch.cat(chunks, dim=0), None
        else:
            feats, factors = self._features(flat)
        lab_pos, cand_pos, bases, at = [], [], [], 0
        for i, m in zip(which, sizes):
            nl = len(lab_parts[i])
            lab_pos.append(np.arange(at, at + nl))
            cand_pos.append(np.arange(at + nl, at + m))
            bases.append(at)
            at += m
        picks = self._select(feats, factors, lab_pos, cand_pos, bases, [budgets[i] for i in which],
                             [first[i] for i in which], [unif[i] for i in which])
        return {i: picks[k] for k, i in enumerate(which)}


class BADGEQuery(CoresetQuery):
    """badge_sampler.py: k-means++ over gradient embeddings, kept as rank-1 factors."""
    RANDOMIZE = True
    GRADIENT_EMBEDDING = True


class PartitionedBADGEQuery(PartitionedCoresetQuery):
    """partitioned_badge_sampler.py: pooled 512-d gradient embeddings, D^2 sampling per partition."""
    RANDOMIZE = True
    GRADIENT_EMBEDDING = True
    POOLED = True
