"""NumPy twin of K11 (alq_balancing_select): the semantics of BalancingSampler's query as the persistent loop runs it.

  * NumPy's legacy RNG: MT19937 advanced from np.random.get_state(), `np.random.choice(a)` over the available rows as
    the masked rejection draw of random_bounded_uint64_fill (rng = n_avail - 1, draw `next_uint32 & mask(rng)` until it
    is <= rng; rng == 0 draws nothing);
  * the imbalance test of balancing_sampler.py:66-84 in fp32, the way torch evaluates it on the CPU;
  * the tie rule: lowest row among equal ratios;
  * the bookkeeping: class sums in fp64 in K11's fixed order (labeled rows in row order within chunks of CHUNK rows, the
    chunks in order, then the picks in pick order), fp32 centres fl32(sum / fl32(count + 1e-5));
  * distances in fp64 from the fp32 rows and centres, with the relative gap between the two best ratios of every
    balancing step recorded: where it is far above fp32 rounding, the device's fp32 arg-min is the same row.
"""
import numpy as np

CHUNK = 65536
F = np.float32


class MT19937Twin:
    """NumPy's mt19937 (numpy/random/src/mt19937) on a copy of a get_state() tuple."""
    N, M = 624, 397

    def __init__(self, state=None):
        state = np.random.get_state() if state is None else state
        assert state[0] == "MT19937"
        self.key = [int(v) for v in state[1]]
        self.pos = int(state[2])
        self.rest = tuple(state[3:])
        self.outputs = 0

    def _twist(self):
        k, n, m = self.key, self.N, self.M
        for i in range(n):
            y = (k[i] & 0x80000000) | (k[(i + 1) % n] & 0x7FFFFFFF)
            k[i] = k[(i + m) % n] ^ (y >> 1) ^ (0x9908B0DF if y & 1 else 0)
        self.pos = 0

    def next32(self):
        if self.pos >= self.N:
            self._twist()
        y = self.key[self.pos]
        self.pos += 1
        self.outputs += 1
        y ^= y >> 11
        y ^= (y << 7) & 0x9D2C5680
        y ^= (y << 15) & 0xEFC60000
        y ^= y >> 18
        return y & 0xFFFFFFFF

    def bounded(self, rng):
        """legacy randint(0, rng + 1): masked rejection; rng == 0 consumes nothing."""
        if rng == 0:
            return 0
        mask = (1 << int(rng).bit_length()) - 1
        while True:
            v = self.next32() & mask
            if v <= rng:
                return v

    def state(self):
        return ("MT19937", np.array(self.key, dtype=np.uint32), self.pos) + self.rest


def needs_balancing(counts, remaining):
    """balancing_sampler.py:66-84 in fp32: the majority mask if the step balances, else None."""
    cnt = np.asarray(counts, dtype=np.int64)
    c = len(cnt)
    mean = F(F(cnt.sum()) / F(c))
    above = cnt.astype(F) > mean
    na, nr = int(above.sum()), int((~above).sum())
    with np.errstate(invalid="ignore", divide="ignore"):
        avg_a = F(F(cnt[above].sum()) / F(na))
        avg_r = F(F(cnt[~above].sum()) / F(nr))
        rhs = F(F(nr) * F(avg_a - avg_r))
    return above if F(remaining) <= rhs else None


def class_sums(x, ys, labeled, c):
    """fp64 [c, d] sums of the labeled rows in K11's fixed order."""
    n, d = x.shape
    s = np.zeros((c, d), dtype=np.float64)
    for lo in range(0, n, CHUNK):
        p = np.zeros((c, d), dtype=np.float64)
        for r in np.flatnonzero(labeled[lo:lo + CHUNK]) + lo:
            if 0 <= ys[r] < c:
                p[ys[r]] += x[r].astype(np.float64)
        s += p
    return s


def centre(sum64, count):
    return (sum64 / np.float64(F(F(count) + F(1e-5)))).astype(F)


def balancing_loop(emb, ys, avail, labeled, num_classes, budget, state=None):
    """-> dict(picks, balancing_steps, branch (per step: True = balancing), state (get_state() tuple after the last
    draw), outputs (MT words consumed), min_gap (smallest relative gap between the two best ratios of a balancing step),
    gaps)."""
    x = np.ascontiguousarray(np.asarray(emb, dtype=F))
    ys = np.asarray(ys, dtype=np.int64).reshape(-1)
    avail = np.array(avail, dtype=bool).reshape(-1)
    labeled = np.array(labeled, dtype=bool).reshape(-1)
    lab0 = labeled.copy()
    c = int(num_classes)
    for name, m in (("labeled", labeled), ("available", avail)):
        bad = np.flatnonzero(m & ((ys < 0) | (ys >= c)))
        if len(bad):
            raise ValueError(f"{name} row {bad[0]} has label {ys[bad[0]]}, outside [0, {c})")
    rng = MT19937Twin(state)
    budget = int(min(int(avail.sum()), budget))
    out = dict(picks=[], balancing_steps=0, branch=[], min_gap=float("inf"), gaps=[])
    if budget > 0:
        counts = np.bincount(ys[labeled], minlength=c)[:c].astype(np.int64)
        sums = cents = cn = xn = None
        for t in range(budget):
            maj = needs_balancing(counts, budget - t)
            out["branch"].append(maj is not None)
            if maj is not None:
                if sums is None:                     # built on the first balancing step: no state depends on it
                    sums = class_sums(x, ys, lab0, c)
                    for r in out["picks"]:
                        sums[ys[r]] += x[r].astype(np.float64)
                    cents = np.stack([centre(sums[k], counts[k]) for k in range(c)]).astype(np.float64)
                    cn = (cents * cents).sum(axis=1)
                    xn = (x.astype(np.float64) ** 2).sum(axis=1)
                rows = np.flatnonzero(avail)
                xr = x[rows].astype(np.float64)
                rare = int(np.argmin(counts))
                mi = np.flatnonzero(maj)
                far = (xn[rows][:, None] + cn[mi][None, :] - 2.0 * (xr @ cents[mi].T)).max(axis=1)
                near = np.ones(len(rows)) if counts[rare] == 0 else xn[rows] + cn[rare] - 2.0 * (xr @ cents[rare])
                with np.errstate(invalid="ignore", divide="ignore"):
                    ratio = near / far
                i = int(np.argmin(ratio))
                pick = int(rows[i])
                if len(ratio) > 1:
                    two = np.partition(ratio, 1)[:2]
                    gap = float((two[1] - two[0]) / max(abs(two[1]), 1e-30))
                    out["gaps"].append(gap)
                    out["min_gap"] = min(out["min_gap"], gap)
                out["balancing_steps"] += 1
            else:
                k = rng.bounded(int(avail.sum()) - 1)
                pick = int(np.flatnonzero(avail)[k])
            avail[pick] = False
            labeled[pick] = True
            out["picks"].append(pick)
            y = ys[pick]
            counts[y] += 1
            if sums is not None:
                sums[y] += x[pick].astype(np.float64)
                cents[y] = centre(sums[y], counts[y]).astype(np.float64)
                cn[y] = (cents[y] * cents[y]).sum()
    out["state"] = rng.state()
    out["outputs"] = rng.outputs
    return out
