"""NumPy twin of the decisions K6's parallel BASE route makes (alq_base_select with candidate lists, csrc/alq_mase.cu):

  * base_candidates_kernel: for every class with cnt > 0, the (key, row) pairs packed like base_pack (+0.0 canonical,
    ties by row).  Thread t of 1024 owns the rows with row % 1024 == t, keeps its 3 smallest pairs and remembers the
    smallest pair it dropped.  The list is the len = min(cnt + 32, 64) smallest kept pairs; fail[class] is set iff some
    thread's dropped pair sorts before the list's last entry.
  * base_resolve_kernel + the host loop: the classes in order against the set of taken rows.  A class stops the walk
    iff fail, or iff fewer than cnt of its list's entries are free with a finite key; otherwise it takes the first cnt
    such entries.  A class that stops gets the ordinary sequential step (the stable cnt smallest keys, taken rows at
    +inf) and the walk resumes at the next class.

Not the arithmetic: the keys are whatever the caller built.  With the same keys the picks must equal
oracle.al_oracle.base_select, and the fallback classes say which launches the device route makes.

The constructors build a key matrix K [n, C] (K[r, c] is row r's key for class c) aimed at one branch each, and
`split_keys` turns it into the (min_margin, radius, pred) triple base_select takes: pred[r] picks the column that comes
from min_margin, the radius entry there is +inf as mase_margins writes it."""
import numpy as np

THREADS, KEEP, LIST, MAX_CNT = 1024, 3, 64, 32
GROUP = 8                                   # classes per candidates CTA
EMPTY = np.uint64(0xFFFFFFFFFFFFFFFF)
ORD_INF = 0xFF800000                        # ord(+inf)


def counts(budget, c):
    """base_sampler.py:24-25: picks per class."""
    return np.array([budget // c + (1 if k < budget % c else 0) for k in range(c)], dtype=np.int64)


def list_len(cnt):
    return int(min(cnt + 32, LIST))


def ord32(key):
    """Order-preserving uint32 of a float32 key, -0.0 folded onto +0.0 (alq_ord(key + 0.0f))."""
    u = (np.asarray(key, dtype=np.float32) + np.float32(0.0)).view(np.uint32).astype(np.uint64)
    neg = (u >> np.uint64(31)).astype(bool)
    return np.where(neg, ~u & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))


def pack(key):
    """(ord(key) << 32) | row for rows 0 .. n-1."""
    return (ord32(key) << np.uint64(32)) | np.arange(len(key), dtype=np.uint64)


def class_candidates(key, cnt):
    """(list [64] uint64, EMPTY past len; fail) of one class."""
    w = pack(key)
    n = len(w)
    m = max((n + THREADS - 1) // THREADS, KEEP + 1)
    col = np.full(m * THREADS, EMPTY, dtype=np.uint64)
    col[:n] = w
    col = np.sort(col.reshape(m, THREADS), axis=0)            # column t: thread t's pairs, ascending
    kept, dropped = col[:KEEP].ravel(), col[KEEP]
    ln = list_len(cnt)
    lst = np.full(LIST, EMPTY, dtype=np.uint64)
    lst[:ln] = np.sort(kept)[:ln]
    return lst, bool((dropped < lst[ln - 1]).any())


def candidates(key_of, c, budget):
    """Lists [c, 64] and fail [c] of every class with cnt > 0 (classes with cnt == 0: EMPTY lists, fail False)."""
    cnt = counts(budget, c)
    lists = np.full((c, LIST), EMPTY, dtype=np.uint64)
    fail = np.zeros(c, dtype=bool)
    for k in range(c):
        if cnt[k]:
            lists[k], fail[k] = class_candidates(key_of(k), cnt[k])
    return lists, fail


def resolve(lists, fail, key_of, n, c, budget):
    """The in-order walk with the sequential step at every stop: (picks int64 in pick order, fallback classes,
    rows selected twice)."""
    cnt = counts(budget, c)
    taken = np.zeros(n, dtype=bool)
    picks, fallbacks, dup = [], [], 0
    for k in range(c):
        if cnt[k] == 0:
            continue
        ln = list_len(cnt[k])
        ent = lists[k, :ln]
        rows = (ent & np.uint64(0xFFFFFFFF)).astype(np.int64)
        real = (ent >> np.uint64(32)) < np.uint64(ORD_INF)
        free = np.zeros(ln, dtype=bool)
        free[real] = ~taken[rows[real]]
        if fail[k] or free.sum() < cnt[k]:
            fallbacks.append(k)
            key = np.array(key_of(k), dtype=np.float32)
            key[taken] = np.inf
            got = np.argsort(key, kind="stable")[:cnt[k]]
            dup += int(taken[got].sum())
        else:
            got = rows[free][:cnt[k]]
        taken[got] = True
        picks += got.tolist()
    return np.asarray(picks, dtype=np.int64), fallbacks, dup


def key_fn(K):
    return lambda k: K[:, k]


def twin_select(K, budget):
    """The parallel route on the key matrix K [n, C]: (picks, fallback classes, fail flags, rows selected twice)."""
    n, c = K.shape
    lists, fail = candidates(key_fn(K), c, budget)
    picks, fallbacks, dup = resolve(lists, fail, key_fn(K), n, c, budget)
    return picks, fallbacks, fail, dup


def launch_delta(fallbacks, c, budget, sel_launches):
    """Launches of one parallel base_select call: candidates, the first resolve, and per fallback class one keys
    launch, select_smallest's launches (sel_launches[cnt]) and one mark launch, plus the resolve that resumes after it
    unless the walk is already past the last class."""
    cnt = counts(budget, c)
    d = 2
    for k in fallbacks:
        d += 2 + sel_launches[int(cnt[k])] + (1 if k + 1 < c else 0)
    return d


def sequential_delta(c, budget, sel_launches):
    cnt = counts(budget, c)
    return sum(2 + sel_launches[int(x)] for x in cnt if x)


# ---------------------------------------------------------------------------------------------------------------
# key matrices aimed at one branch each
# ---------------------------------------------------------------------------------------------------------------
def split_keys(K, seed=0):
    """(min_margin [n], radius [n, C], pred [n] int32) whose base_select keys are K."""
    n, c = K.shape
    pred = np.random.default_rng(seed).integers(0, c, size=n).astype(np.int32)
    mm = K[np.arange(n), pred].astype(np.float32)
    radius = K.astype(np.float32, copy=True)
    radius[np.arange(n), pred] = np.inf
    return mm, radius, pred


def random_keys(n, c, seed, quantise=False):
    rng = np.random.default_rng(seed)
    K = rng.uniform(0.05, 3.0, size=(n, c)).astype(np.float32)
    if quantise:
        K = np.round(K * 4) / 4
    return K.astype(np.float32)


def fail_row(k):
    """The thread (row % 1024) that holds class k's four smallest keys in forced_fail."""
    return (37 * k + 11) % THREADS


def force_fail(K, targets):
    """Class k's 4 smallest keys at rows r, r + 1024, r + 2048, r + 3072 (one thread): the thread keeps 3 and drops the
    4th, which belongs in any list of 33 or more entries."""
    n = K.shape[0]
    for k in targets:
        r = fail_row(k)
        assert r + 3 * THREADS < n
        for j in range(4):
            K[r + j * THREADS, k] = np.float32(1e-3 * (j + 1))
    return K


def forced_fail(n, c, targets, seed):
    return force_fail(random_keys(n, c, seed), targets)


def exhausted(n, c, seed):
    """Every class sorts the same key column: class k's list is the rows earlier classes already took."""
    col = np.random.default_rng(seed).uniform(0.05, 3.0, size=n).astype(np.float32)
    return np.repeat(col[:, None], c, axis=1)


def exhausted_at(n, c, cnt, seed):
    """Only the last class runs out: classes 0..4 take 10 planted rows each, and the last class's 5 * cnt smallest keys
    are exactly those rows (more than its list holds), all taken."""
    K = random_keys(n, c, seed)
    rows = np.random.default_rng(seed + 1).permutation(n)[:5 * cnt]
    for k in range(5):
        K[rows[k * cnt:(k + 1) * cnt], k] = np.float32(1e-3) * np.arange(1, cnt + 1, dtype=np.float32)
    K[rows, c - 1] = np.float32(1e-4) * np.arange(1, 5 * cnt + 1, dtype=np.float32)
    return K


def ties(n, c, seed, short_class=None, short_finite=0):
    """Four key values shared by every class: thousands of equal keys per class, the list's last entry inside a run of
    ties.  A band of rows is +inf for every third class; `short_class` keeps only `short_finite` finite keys."""
    rng = np.random.default_rng(seed)
    K = (rng.integers(0, 4, size=(n, c)) * 0.25).astype(np.float32)
    K[: n // 10, ::3] = np.inf
    if short_class is not None:
        K[:, short_class] = np.inf
        K[rng.permutation(n)[:short_finite], short_class] = np.float32(0.5)
    return K
