"""Edge tables shared by tests/test_rowref.py (oracle and pyoracle against tests/rowref.py, no GPU) and
tests/test_parity_edges.py (the CUDA path against both).  One constructor per family; each returns
(spec, rows, valid, queries) with `rows` / `valid` the raw add_rows calls rowref reads.

The values sit where the scan kernel's arithmetic branches: outside non-bounding IntInfo extents, next to 2^32,
on bucket and sub-range boundaries, on both sides of 0 on the time axis, at tile edges, and at the int64
extremes.  A query may carry `expect`: regular expressions its SG_PLAN_TRACE lines must match, so a GPU test
shows it reached the path it targets."""
import numpy as np

from tests.rowref import I64_MAX, I64_MIN, basic_layout, i64
from tests.util import INT, STR, Q, Spec

KT = [("g", STR), ("k", INT), ("w", INT), ("t", INT)] + [("v%d" % i, INT) for i in range(9)]


class _Table:
    def __init__(self, forms=None):
        self.spec = Spec(KT)
        self.spec.forms = forms
        self.rows, self.valid = [], []

    def add(self, cols, valid=None, block_rows=None, threshold=5000):
        cols = {k: (np.asarray(v, np.int64) if self.spec.KeyTypes[self.spec.KeyTable[k]] == INT else np.asarray(v))
                for k, v in cols.items()}
        self.spec.add_rows(cols, valid, threshold=threshold, block_rows=block_rows)
        self.rows.append((cols, block_rows, threshold))
        self.valid.append(valid or {})

    def extents(self, **info):
        # after add_rows, which widens an existing entry to cover the data
        self.spec.IntInfo.update(info)

    def done(self, queries):
        return self.spec, self.rows, self.valid, queries


def _q(spec, expect=(), **kw):
    q = Q(spec, **kw)
    q.expect = list(expect)
    return q


def _groups(rng, n, k=3):
    return np.array(["g%d" % x for x in rng.integers(0, k, n)])


# ---------------------------------------------------------------------------------------------------------------
# A. IntInfo extents that do not bound the data
# ---------------------------------------------------------------------------------------------------------------
A_EXTENTS = [(10, 50), (100, 1000), (-1000, -10), (-(1 << 40), 1 << 62), ((1 << 32) + 5, (1 << 32) + 5000),
             (-500, 500)]


def _around(lo, hi):
    vals = [lo - 1, lo, hi, hi + 1, i64(10 * hi), i64(10 * hi) + 1, (lo + hi) // 2, 0]
    return [v for v in vals if I64_MIN <= v <= I64_MAX]


def family_a(forms=None):
    rng = np.random.default_rng(1)
    t = _Table(forms)
    n = 30000
    cols = {"g": _groups(rng, n), "k": np.arange(n) % 25000, "w": rng.integers(1, 4, n)}
    valid = {}
    for i, (lo, hi) in enumerate(A_EXTENTS):
        cols["v%d" % i] = rng.choice(np.asarray(_around(lo, hi), np.int64), n)
        valid["v%d" % i] = rng.random(n) > 0.1
    t.add(cols, valid, block_rows=15000)  # few distinct values: bucket-encoded
    m = 20000  # the same values plus a spread of filler: value arrays with gaps reading 0
    cols = {"g": _groups(rng, m), "k": np.arange(m) % 25000, "w": rng.integers(1, 4, m)}
    valid = {}
    for i, (lo, hi) in enumerate(A_EXTENTS):
        pick = rng.choice(np.asarray(_around(lo, hi), np.int64), m)
        filler = rng.integers(min(lo, hi), max(lo, hi) + 1, m, dtype=np.int64)
        cols["v%d" % i] = np.where(rng.random(m) < 0.5, pick, filler)
        valid["v%d" % i] = rng.random(m) > 0.1
    t.add(cols, valid, block_rows=10000, threshold=50)
    t.extents(**{"v%d" % i: e for i, e in enumerate(A_EXTENTS)})
    s = t.spec
    aggs = ["v%d" % i for i in range(len(A_EXTENTS))]
    return t.done([
        _q(s, groups=["g"], aggs=aggs, op="avg"),
        _q(s, groups=["g"], aggs=aggs, op="hist"),
        _q(s, groups=["g"], aggs=aggs[:3] + aggs[4:], op="hist", loghist=True),
        _q(s, groups=["g"], aggs=aggs, op="avg", weight_col="w"),
        # more than 20k groups: accumulators in global memory
        _q(s, groups=["k"], aggs=aggs, op="avg", expect=[r"acc_repl=0 "]),
        _q(s, groups=["k"], aggs=aggs[:1], op="hist", expect=[r"acc_repl=0 "]),
        _q(s, int_filters=[("v2", "lt", -10)], groups=["g"], aggs=aggs, op="hist"),
    ])


# ---------------------------------------------------------------------------------------------------------------
# B. The 32-bit path and its carries
# ---------------------------------------------------------------------------------------------------------------
def family_b_carry(forms=None):
    """Full blocks of values just below 2^32, nearly all in one group, so that every replica's low limb carries;
    then a block holding exactly {0, 2^32-1} and one with a value one past the 32-bit path."""
    rng = np.random.default_rng(2)
    t = _Table(forms)
    n = 3 * 65536
    v = rng.integers((1 << 32) - (1 << 20), 1 << 32, n, dtype=np.int64)
    g = np.where(rng.random(n) < 0.95, "a", "b")
    t.add({"g": g, "v0": v, "v1": v - (1 << 31)}, block_rows=65536)
    t.add({"g": np.array(["a", "b"]), "v0": [0, (1 << 32) - 1], "v1": [0, (1 << 32) - 1]})
    t.add({"g": np.array(["a", "a", "b"]), "v0": [1 << 32, (1 << 32) - 1, 1], "v1": [1 << 32, 5, 1]})
    t.extents(v0=(0, (1 << 32) - 1), v1=(-(1 << 31), (1 << 32) - 1))
    s = t.spec
    return t.done([
        _q(s, groups=["g"], aggs=["v0", "v1"], op="avg", expect=[r"agg0=\[fmin=0 fmax=4294967295 hist32=\d nocarry=0\]"]),
        _q(s, groups=["g"], aggs=["v0", "v1"], op="hist", expect=[r"hist32=1 nocarry=0"]),
        _q(s, int_filters=[("v0", "gt", (1 << 32) - (1 << 19))], groups=["g"], aggs=["v0"], op="avg"),
    ])


# fmax for R = 32 replicas (2048 rows of a full block per replica): the no-carry bound fmax * 2048 * fold_every
# against 2^32, just below and just above, and two with room for the deferred fold (4 and 3 blocks: a bound
# twice too loose would fold 4 blocks of 600000 and overflow a low limb)
B_FOLD = {"below": 2097151, "above": 2097152, "fold": 524287, "fold3": 600000}


def family_b_fold(which, forms=None):
    """Four consecutive full blocks of one group with every row at fmax: each replica's low limb receives
    exactly fmax * 65536/R per block, folded over fold_every blocks ("above": exactly 2^32 per block)."""
    fmax = B_FOLD[which]
    t = _Table(forms)
    n = 4 * 65536
    # threshold 0: value arrays even with one distinct value (a bin would be summed as value x count)
    t.add({"g": np.full(n, "a"), "v0": np.full(n, fmax)}, block_rows=65536, threshold=0)
    t.extents(v0=(0, fmax))
    s = t.spec
    expect = {"below": [r"acc_repl=32 fold_every=1 .*nocarry=1"], "above": [r"acc_repl=32 fold_every=4 .*nocarry=0"],
              "fold": [r"acc_repl=32 fold_every=4 .*nocarry=1"],
              "fold3": [r"acc_repl=32 fold_every=3 .*nocarry=1"]}[which]
    return t.done([_q(s, groups=["g"], aggs=["v0"], op="avg", expect=expect),
                   _q(s, aggs=["v0"], op="hist", expect=expect)])


# ---------------------------------------------------------------------------------------------------------------
# C. Bucket boundaries
# ---------------------------------------------------------------------------------------------------------------
C_SIZES = [1, 2, 3, 7, 1000, (1 << 31) - 1, (1 << 32) - 1, 1 << 32]


def _c_extents(i, bs):
    lo = [0, -3000, 7, -5, 10 ** 6, -(1 << 33), 0, -(1 << 40)][i]  # (2^32-1 from 0: x reaches 2^32-1 in the fast path)
    return (lo, lo + 50) if bs == 1 else (lo, lo + 1000 * bs)


def c_values(lo, hi, bs):
    """lo + k*bs - 1, lo + k*bs, lo + k*bs + 1 for every slot k, the last slot, and beyond the extents."""
    nslots = basic_layout(lo, hi, 0)[1]
    vals = [lo + k * bs + d for k in range(nslots) for d in (-1, 0, 1)]
    vals += [hi, hi + 1, i64(10 * hi), i64(10 * hi) + 1, lo - 1]
    return sorted({v for v in vals if I64_MIN <= v <= I64_MAX})


def family_c(forms=None):
    rng = np.random.default_rng(4)
    t = _Table(forms)
    cols, ext = {}, {}
    for i, bs in enumerate(C_SIZES):
        ext["v%d" % i] = _c_extents(i, bs)
    lists = {c: c_values(lo, hi, C_SIZES[int(c[1:])]) for c, (lo, hi) in ext.items()}
    n = max(len(v) for v in lists.values())
    for c, vals in lists.items():  # every column holds its whole list (the shorter ones repeat)
        cols[c] = rng.permutation(np.resize(np.asarray(vals, np.int64), n))
    cols["g"] = _groups(rng, n, 2)
    cols["k"] = np.arange(n) % 90  # (bucket-encoded in both blocks: a value-array group column takes the hash path)
    t.add(cols)  # bucket-encoded
    t.add({k: v[::-1] for k, v in cols.items()}, threshold=100)  # value arrays
    t.extents(**ext)
    s = t.spec
    aggs = ["v%d" % i for i in range(8)]
    # the same values under HIST_BUCKET overrides (an int32 field: up to 2^31-1); 1 clamps nearly every value
    t2 = _Table(forms)
    m = 4000
    w = rng.integers(0, 10 ** 6, m)
    w[:300] = np.arange(300) * 7 - 1
    t2.add({"g": _groups(rng, m, 2), "k": np.arange(m) % 200, "v0": w, "v1": w - 500000})
    t2.extents(v0=(0, 10 ** 6), v1=(-500000, 500000))
    s2 = t2.spec
    # MultiHist: each sub-range's own Min and Max, +-1; positive and negative extents
    t3 = _Table(forms)
    from tests.rowref import multi_layout
    mext = {"v0": (0, 1 << 20), "v1": (-(1 << 20), -1000), "v2": (-70000, 70000)}
    mc = {}
    for c, (lo, hi) in mext.items():
        vals = sorted({x + d for a, b in multi_layout(lo, hi) for x in (a, b) for d in (-1, 0, 1)} |
                      {lo - 1, hi + 1, i64(10 * hi), i64(10 * hi) + 1})
        mc[c] = np.asarray(vals, np.int64)
    mn = max(len(v) for v in mc.values())
    mc = {c: np.resize(v, mn) for c, v in mc.items()}
    mc["g"] = _groups(rng, mn, 2)
    t3.add(mc)
    t3.add({c: v[::-1] for c, v in mc.items()}, threshold=10)
    t3.extents(**mext)
    s3 = t3.spec
    qs = [
        _q(s, groups=["g"], aggs=aggs, op="hist"),
        # slot count below / above the shared-memory histogram cache's rows (a 1002-counter row per slot)
        _q(s, groups=["g"], aggs=["v4"], op="hist", expect=[r"hist_rows=(\d+) lslots=\1 "]),
        _q(s, groups=["k"], aggs=["v4"], op="hist", expect=[r"acc_repl=[1-9]\d* .*hist_rows=([1-8]?\d) lslots=(9\d|1\d\d) "]),
        _q(s, groups=["g"], aggs=aggs[:5], op="hist", loghist=True),
    ]
    qs2 = [_q(s2, groups=["g"], aggs=["v0", "v1"], op="hist", hist_bucket=hb) for hb in (1, 7, 1000, (1 << 31) - 1)]
    qs3 = [_q(s3, groups=["g"], aggs=list(mext), op="hist", loghist=True)]
    return [t.done(qs), t2.done(qs2), t3.done(qs3)]


# ---------------------------------------------------------------------------------------------------------------
# D. The time axis
# ---------------------------------------------------------------------------------------------------------------
def family_d(forms=None):
    """Times below 0, across 0 (Go's truncating division makes bucket 0 span (-B, B)), at and above 2^32, and far
    below 0; blocks inside one bucket and across a bucket edge; the time column bucket-encoded and as a value
    array.  One table per range, so that each query's time axis stays small."""
    rng = np.random.default_rng(5)
    out = []
    for segs in (((-6000, 2, 5000), (-2500, 1, 100)), (((1 << 32) - 3000, 1, 5000), ((1 << 32) - 1000, 1, 100)),
                 ((-(1 << 33) - 1500, 1, 100),)):
        t = _Table(forms)
        n = 6000
        for base, step, thr in segs:
            # bucket-encoded: 4 rows per time value, some rows without one; value arrays: a time in every row (a
            # gap would read time 0, outside the table's time extents: refused, DESIGN.md §7)
            bucketed = thr == 5000
            tt = base + step * (np.arange(n) // (4 if bucketed else 1))
            valid = {"t": rng.random(n) > (0.02 if bucketed else 0), "v0": rng.random(n) > 0.1}
            t.add({"g": _groups(rng, n), "t": tt, "v0": rng.integers(0, 100, n)}, valid, block_rows=250, threshold=thr)
        t.extents(v0=(0, 100))
        s = t.spec
        qs = []
        for b in (1000, 700, 1 << 32):
            qs.append(_q(s, groups=["g"], aggs=["v0"], op="hist", time_col="t", time_bucket=b))
            qs.append(_q(s, groups=["g"], aggs=[], op="avg", time_col="t", time_bucket=b))
        qs.append(_q(s, int_filters=[("t", "lt", 0)], groups=["g"], aggs=["v0"], op="avg", time_col="t",
                     time_bucket=1000))
        out.append(t.done(qs))
    return out


# ---------------------------------------------------------------------------------------------------------------
# E. Tile and encoding geometry
# ---------------------------------------------------------------------------------------------------------------
E_SIZES = [1, 31, 32, 33, 511, 512, 513, 1023, 1024, 1025, 65535, 65536]


# len(Values) of v0 / v8 in the value-array pass: at a 512-row tile edge +-1, or the block's last row
E_END = {1: 1, 31: 31, 32: 32, 33: 33, 511: 511, 512: 511, 513: 512, 1023: 513, 1024: 1023, 1025: 1024,
         65535: 65023, 65536: 65535}


def family_e(forms=None):
    """Every size twice: bucket-encoded (threshold 1200: the bins below) and as value arrays (threshold 4)."""
    rng = np.random.default_rng(6)
    t = _Table(forms)
    for n in E_SIZES:
        for threshold in (1200, 4):
            r = np.arange(n)
            # v0 (wide values) and v8 (just below 2^32: the 32-bit scan, value_base near 2^32) end at row E_END[n]
            end = E_END[n]
            v0 = rng.integers(-(1 << 40), 1 << 40, n)
            va0 = np.zeros(n, bool)
            va0[:end] = rng.random(end) > 0.2
            va0[end - 1] = True
            v8 = (1 << 32) - 1 - np.abs(np.cumsum(rng.integers(-3, 4, n)))
            # v1: bins: one crossing a tile edge (rows 1000..1100), one per row over the first full tile, the rest
            v1 = np.where((r >= 1000) & (r <= 1100), 777, np.where(r < 1024, r, 5))
            # v2: one bin holding every row; v3: a bin holding rows 0 and n-1 only (narrow gap 65535 in a full block)
            v2 = np.full(n, 42)
            v3 = np.where((r == 0) | (r == n - 1), -9, 3 + (r % 3))
            # v4 / v5: int16 deltas at -32768 / 32767, int32 deltas at -2^31 / 2^31-1
            d4 = rng.choice(np.asarray([-32768, 32767, 1, -1, 12]), n)
            d5 = rng.choice(np.asarray([-(1 << 31), (1 << 31) - 1, 3, -7]), n)
            v4 = 100 + np.cumsum(d4)
            v5 = np.cumsum(d5)
            # v6: value_base just below 2^32, decoded values crossing it; v7: a negative base rising through 0
            v6 = (1 << 32) - 700 + np.cumsum(rng.integers(0, 3, n))
            v7 = -min(n, 3000) + r
            g = np.where(r % 97 == 0, "x", np.where(r % 2 == 0, "a", "b"))
            t.add({"g": g, "v0": v0, "v1": v1, "v2": v2, "v3": v3, "v4": v4, "v5": v5, "v6": v6, "v7": v7, "v8": v8},
                  {"v0": va0, "v8": va0}, threshold=threshold)
    s = t.spec
    aggs = ["v%d" % i for i in range(9)]
    return t.done([
        _q(s, groups=["g"], aggs=aggs, op="avg"),
        # (v6 and v8 stay out of hist mode: a spread of a few hundred around 2^32 leaves the stddev to the last
        # bits of the mean)
        _q(s, groups=["g", "v3"], aggs=["v1", "v7"], op="hist"),
        _q(s, int_filters=[("v7", "gt", -1)], str_filters=[("g", "neq", "x")], groups=["g"], aggs=aggs, op="avg"),
        _q(s, int_filters=[("v1", "eq", 777)], groups=["v2"], aggs=["v6", "v0", "v8"], op="avg"),
    ])


# ---------------------------------------------------------------------------------------------------------------
# F. int64 wrap and extremes
# ---------------------------------------------------------------------------------------------------------------
F_LITERALS = [I64_MIN, I64_MAX, 0, -1]


def family_f(forms=None):
    rng = np.random.default_rng(7)
    t = _Table(forms)
    big = I64_MAX // 10  # Max * 10 = 2^63 - 8: accepts up to there, rejects INT64_MAX
    n = 3000
    for blk, pool in enumerate(([I64_MIN, I64_MAX, 1 << 62, big * 10, -5], [1 << 62, (1 << 62) + 1, 7],
                                [I64_MIN, -(1 << 62), 0], [I64_MAX, I64_MAX - 1])):
        v0 = rng.choice(np.asarray(pool, np.int64), n)
        v1 = np.where(rng.random(n) < 0.5, -(1 << 62), rng.integers(-(1 << 62), big, n))
        v1[:4] = [I64_MIN, I64_MAX, -(1 << 62), big]
        g = np.where(rng.random(n) < 0.7, "a", "b")
        t.add({"g": g, "v0": v0, "v1": v1}, {"v1": rng.random(n) > 0.05}, threshold=5000 if blk % 2 else 2)
    t.extents(v0=(I64_MIN, big), v1=(-(1 << 62), big))
    s = t.spec
    qs = [_q(s, groups=["g"], aggs=["v0", "v1"], op="avg"),
          _q(s, groups=["g"], aggs=["v1"], op="hist")]
    for lit in F_LITERALS:
        for op in ("lt", "gt", "eq", "neq"):
            qs.append(_q(s, int_filters=[("v0", op, lit)], groups=["g"], aggs=["v0"], op="avg"))
    return t.done(qs)


def all_tables(forms=None):
    """(name, (spec, rows, valid, queries)) of every family."""
    out = [("A", family_a(forms))]
    out += [("B-carry", family_b_carry(forms))] + [("B-fold-" + w, family_b_fold(w, forms)) for w in B_FOLD]
    out += [("C%d" % i, x) for i, x in enumerate(family_c(forms))]
    out += [("D%d" % i, x) for i, x in enumerate(family_d(forms))]
    out += [("E", family_e(forms)), ("F", family_f(forms))]
    return out
