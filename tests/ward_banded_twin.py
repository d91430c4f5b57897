"""NumPy twin of K8's banded layout (alq_ward_nn_chain_banded): scipy's condensed vector cut into bands of rows, each its
own array, and tests/ward_oracle.py's nn_chain reading and writing every entry through the kernel's addressing:

  * (i, j), i < j, lives in the band of row i, at cidx(i, j) - cidx(cut[b], cut[b] + 1);
  * the band of row r is the number of cut[1 .. 8) that are <= r, with the cuts past the last band equal to n
    (ward_chain_kernel's band_of);
  * a scan of row x reads (j, x), j < x, from j's band and (x, j), j > x, from x's; a merge stores (i, y) in the band of
    min(i, y).

With bands that cover [0, n) the merge list must be W.ward_nn_chain's over the square matrix, bit for bit."""
import numpy as np

MAX_BANDS = 8


def cidx(i, j, n):
    i, j = np.asarray(i, dtype=np.int64), np.asarray(j, dtype=np.int64)
    return n * i - i * (i + 1) // 2 + (j - i - 1)


def split_condensed(vec, cuts, n):
    """Copies of the bands [cuts[b], cuts[b + 1]) of a condensed vector (None for a band without pairs)."""
    out = []
    for lo, hi in zip(cuts, cuts[1:]):
        a, b = int(cidx(lo, lo + 1, n)), int(cidx(hi, hi + 1, n))
        out.append(np.array(vec[a:b], dtype=np.float64) if b > a else None)
    return out


class BandedD:
    """Entry access of the symmetric distance matrix through the banded layout."""

    def __init__(self, cuts, bands, n):
        cuts = [int(c) for c in cuts]
        assert 1 <= len(bands) == len(cuts) - 1 <= MAX_BANDS and cuts[0] == 0 and cuts[-1] == n
        assert all(a <= b for a, b in zip(cuts, cuts[1:]))
        self.n, self.bands = n, bands
        self.cut = np.asarray(cuts + [n] * (MAX_BANDS + 1 - len(cuts)), dtype=np.int64)
        self.start = cidx(self.cut[:-1], self.cut[:-1] + 1, n)

    def band_of(self, r):
        r = np.asarray(r, dtype=np.int64)
        return (self.cut[1:MAX_BANDS][None, :] <= r.reshape(-1, 1)).sum(axis=1)

    def _where(self, x, js):
        js = np.asarray(js, dtype=np.int64)
        lo, hi = np.minimum(js, x), np.maximum(js, x)
        b = self.band_of(lo)
        return b, cidx(lo, hi, self.n) - self.start[b]

    def get(self, x, js):
        b, off = self._where(x, js)
        out = np.empty(len(off), dtype=np.float64)
        for k in np.unique(b):
            m = b == k
            out[m] = self.bands[k][off[m]]
        return out

    def put(self, x, js, vals):
        b, off = self._where(x, js)
        for k in np.unique(b):
            m = b == k
            self.bands[k][off[m]] = vals[m]


def ward_nn_chain_banded(cuts, bands, n):
    """W.ward_nn_chain over the banded layout (the bands are consumed, as K8 consumes them): (merge_xy [n-1, 2] int64,
    merge_dist [n-1]) in discovery order."""
    D = BandedD(cuts, bands, n)
    size = np.ones(n, dtype=np.int64)
    xy = np.empty((n - 1, 2), dtype=np.int64)
    md = np.empty(n - 1, dtype=np.float64)
    chain = []
    for k in range(n - 1):
        if not chain:
            chain.append(int(np.flatnonzero(size > 0)[0]))
        while True:
            x = chain[-1]
            if len(chain) > 1:
                y = chain[-2]
                cur = D.get(x, [y])[0]               # ties go to the previous chain element
            else:
                y, cur = -1, np.inf
            live = np.flatnonzero(size > 0)
            live = live[live != x]
            row = np.full(n, np.inf)
            row[live] = D.get(x, live)
            row[np.isnan(row)] = np.inf
            i = int(np.argmin(row))
            if row[i] < cur:
                cur, y = row[i], i
            if len(chain) > 1 and y == chain[-2]:
                break
            chain.append(y)
        chain.pop()
        chain.pop()
        if x > y:
            x, y = y, x
        nx, ny = size[x], size[y]
        xy[k] = (x, y)
        md[k] = cur
        size[x] = 0
        size[y] = nx + ny
        live = np.flatnonzero(size > 0)
        live = live[live != y]
        ni = size[live]
        t = 1.0 / (nx + ny + ni)
        dx, dy = D.get(x, live), D.get(y, live)
        D.put(y, live, np.sqrt((ni + nx) * t * dx * dx + (ni + ny) * t * dy * dy - ni * t * cur * cur))
    return xy, md
