"""Query-path half of the reference's ``Strategy`` base class, plus the plumbing the accelerated
samplers share.

Mirrors active_learning/src/query_strategies/strategy.py for everything ``query()`` touches:
constructor signature and attributes (:74-124), ``available_query_idxs`` (:126-145),
``already_labeled_idxs`` (:147-163), ``update`` (:459-485).  Training / evaluation
(:249-442) is out of scope (SURVEY.md section 2, row 14): to keep it, bind the samplers onto the
reference's own base class with ``active_learning_b200.integration.make_drop_in``.

The global NumPy RNG is consumed in exactly the reference's order (SURVEY.md section 7, hard
part 6), because selected indices are compared bit-for-bit against it.
"""
from __future__ import annotations

import logging
import os

import numpy as np
import torch
from torch.utils.data import DataLoader, Subset


class Strategy:
    logger = logging.getLogger("ActiveLearning")

    def __init__(self, train_set, al_set, net, train_args, eval_idxs, comet_experiment,
                 test_set=None, **kwargs):
        self.train_args = train_args
        self.comet_experiment = comet_experiment
        url = getattr(comet_experiment, "url", ".") or "."
        tag = os.path.basename(os.path.normpath(url))[:9]
        self.comet_experiment_hash = "debug" if tag == "." else tag

        self.train_set, self.al_set, self.test_set = train_set, al_set, test_set
        self.num_classes = self.al_set.num_classes

        self.round = 0
        self.cumulative_cost = 0

        self.n_pool = len(self.al_set)
        self.eval_idxs = eval_idxs
        self.idxs_lb = np.zeros(self.n_pool, dtype=bool)
        self.idxs_lb_recent = np.zeros(self.n_pool, dtype=bool)

        patience = kwargs.get("early_stop_patience", 0)
        self.es_params = {"use_es": patience != 0, "patience": patience, "count": 0,
                          "success": False, "best_perf": 0}
        self.n_epoch = kwargs.get("n_epoch")
        self.imbalanced_training = train_args.get("imbalanced_training", False)
        self.world_size = kwargs.get("world_size", 1)

        self.device = torch.device("cuda" if torch.cuda.is_available() else "cpu")
        self.net = net
        self.net_name = kwargs.get("model")
        self.query_net = None
        self.feature_net = None
        self.freeze_feature = kwargs.get("freeze_feature", False)

        self.base_ckpt_path = kwargs.get("ckpt_path", ".")
        self.exp_name = kwargs.get("exp_name", "active_learning")
        self.exp_hash = "no_comet" if tag == "." else tag

    # ---- pool bookkeeping -----------------------------------------------------------------------
    def available_query_idxs(self, boolean=False, shuffle=True):
        """strategy.py:126-145.  The reference filters the evaluation indices with a Python list
        comprehension (`x not in eval_idxs`, O(N*|eval|)); np.isin keeps order and values and is
        applied after the permutation exactly like the reference, so the RNG stream is unchanged."""
        if boolean:
            mask = ~self.idxs_lb
            mask[self.eval_idxs] = False
            return mask
        cand = np.where(self.idxs_lb == False)[0]  # noqa: E712
        if shuffle:
            cand = np.random.permutation(cand)
        if len(self.eval_idxs):
            cand = cand[~np.isin(cand, np.asarray(self.eval_idxs))]
        return cand

    def already_labeled_idxs(self, boolean=False, shuffle=False):
        """strategy.py:147-163."""
        if boolean:
            return np.copy(self.idxs_lb)
        lab = np.argwhere(self.idxs_lb).squeeze()
        if shuffle:
            lab = np.random.permutation(lab)
        return lab

    def update(self, labeled_idxs, cur_cost):
        """strategy.py:459-485 (same assertion, same artefact file).  The reference walks the B new indices in a Python
        loop (:468-471); the check and the mask update are vectorised here (SURVEY.md section 8f rank 4): an index that is
        already labeled, or that appears twice in the list, trips the same assertion."""
        if isinstance(labeled_idxs, list):
            labeled_idxs = np.array(labeled_idxs)
        self.idxs_lb_recent = labeled_idxs
        idx = np.asarray(labeled_idxs).reshape(-1).astype(np.int64)
        assert not self.idxs_lb[idx].any() and len(np.unique(idx)) == len(idx)   # never re-label (:470)
        self.idxs_lb[idx] = True
        self.cumulative_cost += cur_cost
        exp = self.comet_experiment
        if exp is not None:
            exp.log_metric("cumulative_budget", self.cumulative_cost, include_context=False,
                           step=self.round)
            exp.log_asset_data(",".join(str(e) for e in labeled_idxs),
                               name=f"labeled_idxs_on_rd_{self.round}")
        self.logger.info(f"Cumulative budget used on round {self.round} = {self.cumulative_cost}")
        out_dir = os.path.join(self.base_ckpt_path, self.exp_name)
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "labeled_idxs_per_round.txt"), "a") as fh:
            fh.writelines(f"Round {self.round}: {labeled_idxs}\n")

    def init_network_weights(self):
        """Query-path effect of strategy.py:175-198: the feature network is the task network."""
        self.feature_net = self.net

    def query(self, budget):
        raise NotImplementedError

    def train(self, *a, **k):
        raise NotImplementedError(
            "training is outside the accelerated path; bind the samplers onto the reference's "
            "Strategy with active_learning_b200.integration.make_drop_in to keep it")

    test = load_best_ckpt = train


class EngineMixin:
    """What every accelerated sampler needs: the CUDA engine (lazily created, never pickled)
    and the pool forward pass that leaves logits / embeddings in device slabs."""

    _engine = None
    _shard_group = None

    def get_engine(self):
        if self._engine is None:
            from ..engine import Engine  # raises without GPU + libalq.so: no CPU fallback
            self._engine = Engine()
        return self._engine

    def set_engine(self, engine):
        self._engine = engine

    def __getstate__(self):
        # save_experiment pickles the whole Strategy every round (utils/resume_training.py:49) and
        # train() pickles it into mp.spawn workers (strategy.py:297): keep handles and caches out.
        state = dict(self.__dict__)
        for k in ("_engine", "_shard_group", "_saved_embeddings", "_emb_cache", "_bal_cache", "_pc_cache"):
            state.pop(k, None)
        return state

    def _query_device(self):
        eng = self.get_engine()
        return getattr(eng, "device", self.device)

    def _loader(self, idxs, dataset=None):
        return DataLoader(Subset(self.al_set if dataset is None else dataset, indices=idxs), shuffle=False,
                          **self.train_args["loader_te_args"], drop_last=False)

    # ---- pool-forward data path (SURVEY.md section 8f, rank 3) -----------------------------------------
    def _device_batches(self, loader, dev, net=None):
        """The loader's batches with x already on the device: batch k+1 is staged through one of two pinned host buffers
        and copied on a side stream while batch k runs through the network, so the H2D copy and the host-side collation
        overlap the forward pass instead of sitting in front of it.  Image batches (4-D) are handed over channels-last and
        the network is switched to channels-last once (same arithmetic, the tensor-core-friendly cuDNN kernels; opt out
        with the sampler kwarg channels_last=False).  Precision is untouched: fp32 weights and activations, torch's
        defaults for TF32."""
        dev = torch.device(dev)
        if dev.type != "cuda" or os.environ.get("ALQ_PREFETCH", "1") == "0":
            for x, y, i in loader:
                yield x.to(dev, non_blocking=True), y, i
            return
        cl = bool(getattr(self, "channels_last", True)) and os.environ.get("ALQ_CHANNELS_LAST", "1") != "0"
        if cl and net is not None and not getattr(net, "_alq_channels_last", False):
            try:
                net.to(memory_format=torch.channels_last)
                net._alq_channels_last = True
            except Exception:
                cl = False
        side = torch.cuda.Stream(device=dev)
        pinned = [None, None]

        def stage(batch, slot):
            x, y, i = batch
            if not x.is_pinned():
                if pinned[slot] is None or pinned[slot].shape != x.shape or pinned[slot].dtype != x.dtype:
                    pinned[slot] = torch.empty(x.shape, dtype=x.dtype).pin_memory()
                pinned[slot].copy_(x)
                x = pinned[slot]
            with torch.cuda.stream(side):
                xd = x.to(dev, non_blocking=True)
                if cl and xd.dim() == 4:
                    xd = xd.contiguous(memory_format=torch.channels_last)
                ev = torch.cuda.Event()
                ev.record(side)
            return xd, y, i, ev

        it = iter(loader)
        try:
            nxt = stage(next(it), 0)
        except StopIteration:
            return
        k = 0
        while nxt is not None:
            xd, y, i, ev = nxt
            k += 1
            try:
                nxt = stage(next(it), k & 1)      # the next batch's copy is in flight while this one is consumed
            except StopIteration:
                nxt = None
            cur = torch.cuda.current_stream(dev)
            cur.wait_event(ev)
            xd.record_stream(cur)
            yield xd, y, i

    # ---- cross-round embedding cache (SURVEY.md section 8f, rank 1) ---------------------------------
    def _cacheable(self, net):
        """Under --freeze_feature the encoder never changes (resnet_simclr.py:36-37 detaches it) and the
        al_set transforms are deterministic, so pool embeddings are round-invariant; only the linear head
        moves.  Needs the reference's encoder/linear layout and is opt-out with cache_embeddings=False."""
        return (bool(getattr(self, "freeze_feature", False)) and getattr(self, "cache_embeddings", True)
                and hasattr(net, "encoder") and hasattr(net, "linear"))

    @staticmethod
    def _encoder_fingerprint(net):
        """Every parameter AND buffer of the encoder (BatchNorm running statistics included): a partially loaded
        checkpoint, changed BN statistics or a fine-tuned last block must invalidate the cached embeddings.  Two
        moments per tensor, reduced on the tensor's own device and fetched with ONE transfer (no per-tensor sync:
        a ResNet-50 has 320 state tensors); runs once per query."""
        with torch.no_grad():
            sd = net.encoder.state_dict()
            if not sd:
                return (0,)
            names, shapes, moments = [], [], []
            for name, t in sd.items():
                t = t.detach()
                tf = t if t.is_floating_point() else t.double()
                names.append(name)
                shapes.append(tuple(t.shape))
                moments.append(tf.sum(dtype=torch.float64))
                moments.append(torch.linalg.vector_norm(tf.flatten(), 2, dtype=torch.float64))
            vals = torch.stack(moments).cpu().tolist()
            return (len(sd), tuple(names), tuple(shapes), tuple(vals))

    def _forward_pool_cached(self, idxs, net, want_features):
        """Same outputs as `_forward_pool`, but the encoder runs only for pool rows it has not seen: the
        embeddings live in a device slab [n_pool, D] (1.28 M x 2048 fp32 = 10.5 GB on a 180 GB part) and each
        query recomputes logits = linear(emb) per loader batch, exactly the GEMM the reference's forward ends
        with (resnet_simclr.py:38).  8 AL rounds cost one backbone pass over the pool instead of 8."""
        dev = self._query_device()
        net.to(dev)
        idxs_t = torch.as_tensor(np.asarray(idxs, dtype=np.int64), device=dev)
        fp = self._encoder_fingerprint(net)
        cache = getattr(self, "_emb_cache", None)
        if cache is not None and (cache["fp"] != fp or cache["emb"].device != dev):
            cache = None
        bs = int(self.train_args["loader_te_args"]["batch_size"])
        with torch.no_grad():
            if cache is None or len(idxs) == 0:
                have = None
            else:
                have = cache["have"][idxs_t]
            missing = np.asarray(idxs, dtype=np.int64) if have is None else np.asarray(idxs, dtype=np.int64)[(~have).cpu().numpy()]
            if len(missing):
                off = 0
                for x, _y, _i in self._device_batches(self._loader(missing.tolist()), dev, net):
                    em = net.encoder(x)
                    if cache is None:
                        dpad = (em.shape[1] + 3) & ~3
                        cache = {"fp": fp, "dim": em.shape[1],
                                 "emb": torch.zeros((self.n_pool, dpad), dtype=torch.float32, device=dev),
                                 "have": torch.zeros(self.n_pool, dtype=torch.bool, device=dev)}
                    rows = torch.as_tensor(missing[off:off + em.shape[0]], device=dev)
                    cache["emb"][rows, :em.shape[1]] = em.float()
                    cache["have"][rows] = True
                    off += em.shape[0]
                self._emb_cache = cache
            if cache is None:
                return (torch.empty((0, self.num_classes), dtype=torch.float32, device=dev),
                        torch.empty((0, 4), dtype=torch.float32, device=dev))
            emb = cache["emb"].index_select(0, idxs_t)
            logits = torch.empty((len(idxs), self.num_classes), dtype=torch.float32, device=dev)
            for lo in range(0, len(idxs), bs):
                logits[lo:lo + bs] = net.linear(emb[lo:lo + bs, :cache["dim"]])
        return logits, (emb if want_features else None)

    def _forward_pool(self, idxs, net, want_features, dataset=None, labels_out=None):
        """Loader loop of margin_sampler.py:29-37 / coreset_sampler.py:50-56 with the `.cpu()`
        removed: outputs land in preallocated device slabs [len(idxs), C] / [len(idxs), D].
        `dataset` overrides al_set (mase_sampler.py:30-33 can read the augmented train_set); `labels_out`, a list,
        collects the loader's label batches (mase_sampler.py:84).  Either one bypasses the embedding cache."""
        if dataset is None and labels_out is None and self._cacheable(net):
            return self._forward_pool_cached(idxs, net, want_features)
        dev = self._query_device()
        n = len(idxs)
        net.to(dev)
        logits = emb = None
        off = 0
        with torch.no_grad():
            for x, _y, _i in self._device_batches(self._loader(idxs, dataset), dev, net):
                if labels_out is not None:
                    labels_out.append(torch.as_tensor(_y).clone())
                if want_features:
                    lg, em = net(x, return_features="finalembed")
                else:
                    lg, em = net(x), None
                if logits is None:
                    logits = torch.empty((n, lg.shape[1]), dtype=torch.float32, device=dev)
                    if em is not None:
                        dpad = (em.shape[1] + 3) & ~3   # kernels want 16-byte rows
                        emb = torch.zeros((n, dpad), dtype=torch.float32, device=dev)
                b = lg.shape[0]
                logits[off:off + b] = lg
                if em is not None:
                    emb[off:off + b, :em.shape[1]] = em
                off += b
        if logits is None:
            logits = torch.empty((0, self.num_classes), dtype=torch.float32, device=dev)
            emb = torch.empty((0, 4), dtype=torch.float32, device=dev)
        return logits, emb
