"""NumPy twin of K12 (alq_balancing_table_select): BalancingSampler's query over an incremental fp64 row x class table.

  * the branch test, NumPy's draws and the label checks are K11's (tests/balancing_loop_oracle.py);
  * class sums S_c in fp64 over the labeled rows in row order, then the picks in pick order; q_c = <S_c, S_c>;
  * at the first balancing step the table T[i, c] = <x_i, S_c> (fp64) and xn64_i = <x_i, x_i> of every available row;
    after that every pick p of class y is pending until the next balancing step, which applies T[i, y] += <x_i, x_p>
    in pick order;
  * d2(i, c) = xn64_i - 2 T[i, c] / den_c + q_c / den_c^2 with den_c = fl32(n_c + 1e-5), the ratio near / far in fp64
    rounded once to fp32, and the arg-min of (ord(fl32 ratio + 0), row): the lowest row on ties, NaN last;
  * the relative gap between the two best fp64 ratios of every balancing step is recorded: where it is far above the
    table's rounding (about 1e-13) the device makes the same pick.
"""
import numpy as np

from balancing_loop_oracle import MT19937Twin, needs_balancing

F = np.float32


def ord32(v):
    """alq_ord on float32: a monotone map to uint32 (NaN with the sign bit clear above +inf)."""
    u = np.asarray(v, dtype=F).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, (~u) & 0xFFFFFFFF, u | 0x80000000)


def class_sums(x, ys, labeled, c):
    """fp64 [c, d] sums of the labeled rows, each class in row order."""
    s = np.zeros((c, x.shape[1]), dtype=np.float64)
    rows = np.flatnonzero(labeled)
    np.add.at(s, ys[rows], x[rows].astype(np.float64))
    return s


def dist(xn, t, den, q):
    return xn - 2.0 * t / den + q / (den * den)


def balancing_table(emb, ys, avail, labeled, num_classes, budget, state=None):
    """-> dict(picks, balancing_steps, branch (per step: True = balancing), state (get_state() tuple after the last
    draw), outputs (MT words consumed), min_gap, gaps, and the final table: slots (its rows), table (pending picks
    applied), sums)."""
    x = np.ascontiguousarray(np.asarray(emb, dtype=F))
    ys = np.asarray(ys, dtype=np.int64).reshape(-1)
    avail = np.array(avail, dtype=bool).reshape(-1)
    labeled = np.array(labeled, dtype=bool).reshape(-1)
    c = int(num_classes)
    for name, m in (("labeled", labeled), ("available", avail)):
        bad = np.flatnonzero(m & ((ys < 0) | (ys >= c)))
        if len(bad):
            raise ValueError(f"{name} row {bad[0]} has label {ys[bad[0]]}, outside [0, {c})")
    rng = MT19937Twin(state)
    budget = int(min(int(avail.sum()), budget))
    out = dict(picks=[], balancing_steps=0, branch=[], min_gap=float("inf"), gaps=[], slots=None, table=None, sums=None)
    if budget <= 0:
        out["state"], out["outputs"] = rng.state(), rng.outputs
        return out
    counts = np.bincount(ys[labeled], minlength=c)[:c].astype(np.int64)
    sums = class_sums(x, ys, labeled, c)
    slots = table = xs = xn = None
    pend = []

    def apply_pending():
        for p in pend:
            table[:, ys[p]] += xs @ x[p].astype(np.float64)
        pend.clear()

    for t in range(budget):
        maj = needs_balancing(counts, budget - t)
        out["branch"].append(maj is not None)
        if maj is not None:
            if table is None:                        # built at the first balancing step, from the sums at that moment
                slots = np.flatnonzero(avail)
                xs = x[slots].astype(np.float64)
                table = xs @ sums.T
                xn = (xs * xs).sum(axis=1)
                pend.clear()
            apply_pending()
            live = np.flatnonzero(avail[slots])
            den = (counts.astype(F) + F(1e-5)).astype(np.float64)
            q = (sums * sums).sum(axis=1)
            rare = int(np.argmin(counts))
            mi = np.flatnonzero(maj)
            xl = xn[live]
            tm = table[np.ix_(live, mi)]             # dist() in place: (xn - 2 t / den) + q / den^2
            tm *= 2.0
            tm /= den[mi]
            np.subtract(xl[:, None], tm, out=tm)
            tm += q[mi] / (den[mi] * den[mi])
            far = tm.max(axis=1)
            near = np.ones(len(xl)) if counts[rare] == 0 else dist(xl, table[live, rare], den[rare], q[rare])
            with np.errstate(invalid="ignore", divide="ignore"):
                ratio = near / far
            key = ord32(ratio.astype(F) + F(0.0))
            i = int(np.argmin(key))                  # first (lowest row) among equal keys
            pick = int(slots[live[i]])
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
        sums[y] += x[pick].astype(np.float64)
        if table is not None:
            pend.append(pick)
    if table is not None:
        apply_pending()
    out.update(state=rng.state(), outputs=rng.outputs, slots=slots, table=table, sums=sums)
    return out
