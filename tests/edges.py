"""Edge tables shared by tests/test_rowref.py (oracle and pyoracle against tests/rowref.py, no GPU) and
tests/test_parity_edges.py (the CUDA path against both).  One constructor per family; each returns
(spec, rows, valid, queries) with `rows` / `valid` the raw add_rows calls rowref reads.

The values sit where the scan kernel's arithmetic branches: outside non-bounding IntInfo extents, next to 2^32,
on bucket and sub-range boundaries, on both sides of 0 on the time axis, at tile edges, and at the int64
extremes.  A query may carry `expect`: regular expressions its SG_PLAN_TRACE lines must match, so a GPU test
shows it reached the path it targets."""
import numpy as np

from tests.rowref import I64_MAX, I64_MIN, basic_layout, i64
from tests.util import INT, SET, STR, Q, Spec

KT = [("g", STR), ("k", INT), ("w", INT), ("t", INT)] + [("v%d" % i, INT) for i in range(9)]


class _Table:
    def __init__(self, forms=None, kt=KT):
        self.spec = Spec(kt)
        self.spec.forms = forms
        self.rows, self.valid = [], []

    def add(self, cols, valid=None, block_rows=None, threshold=5000):
        def arr(k, v):
            typ = self.spec.KeyTypes[self.spec.KeyTable[k]]
            return np.asarray(v, np.int64) if typ == INT else (list(v) if typ == SET else np.asarray(v))
        cols = {k: arr(k, v) for k, v in cols.items()}
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


# ---------------------------------------------------------------------------------------------------------------
# G. Key identity and rendering
# ---------------------------------------------------------------------------------------------------------------
# The key side of the scan: a row's group key becomes a dictionary code, the codes a mixed-radix slot, the slot a
# rendered GroupByKey.  An int -1 is uint64(-1) = MISSING_VALUE in the reference (aggregate.go:125-143), so it is
# the missing group; INT64_MIN is the device value set's empty marker; values above 2^32 do not fit a 32-bit code.
G_KEYS = [-1, 0, I64_MIN, I64_MAX, (1 << 32) + 7, (1 << 40) + 1, -2]
# rows per key in each bucket-encoded block (None: rows without the column).  Missing and -1 are one group of 250
# rows, the largest; apart they would sort fifth (-1) and sixth (missing)
G_COUNTS = {None: 120, -1: 130, 0: 240, I64_MIN: 230, I64_MAX: 220, (1 << 32) + 7: 210, (1 << 40) + 1: 60, -2: 50}
KT_KEYS = ([("g", STR), ("s", STR), ("s2", STR), ("k", INT), ("t", INT), ("v0", INT), ("f", INT), ("f2", INT), ("tags", SET)] +
           [(c, INT) for c in "abcdeqrp"])


def _g_block(rng):
    keys = [k for k, c in G_COUNTS.items() for _ in range(c)]
    keys = [keys[i] for i in rng.permutation(len(keys))]
    k = np.array([0 if x is None else x for x in keys], np.int64)
    return k, np.array([x is not None for x in keys])


def _g_queries(s, expect, radix=()):
    # radix: (lslots of ["k"], of ["g", "k"]) when the dictionaries are known: k's 7 keys + missing, g's 2 strings +
    # the "" staging interns + missing
    e0, e1 = ([r"lslots=%d " % radix[0]], [r"lslots=%d " % radix[1]]) if radix else ([], [])
    return [
        _q(s, groups=["k"], aggs=["v0"], op="avg", expect=expect + e0),
        _q(s, groups=["g", "k"], aggs=["v0"], op="hist", expect=expect + e1),
        _q(s, groups=["k", "g"], aggs=["v0"], op="avg", expect=expect),
        _q(s, groups=["k"], aggs=["v0"], op="avg", time_col="t", time_bucket=500, expect=expect),
        _q(s, groups=["g", "k"], aggs=[], op="avg", time_col="t", time_bucket=1 << 20, expect=expect),
        # the merge of -1 into the missing group must come before the top-K: merged it is the first group
        _q(s, groups=["k"], aggs=["v0"], op="avg", limit=3, expect=expect),
        _q(s, int_filters=[("v0", "gt", 10)], groups=["k"], aggs=["v0"], op="avg", limit=2, expect=expect),
    ]


def family_g_int(mixed, forms=None):
    """The int keys of G_KEYS next to missing rows.  Bucket-encoded only (dictionary codes from the bins), or
    mixed with value-array blocks (the device value dictionary: distinct_kernel + vh_keys) that hold the same keys,
    a spread of filler keys, gaps that read 0 and are populated, and rows past len(Values)."""
    rng = np.random.default_rng(20 + mixed)
    t = _Table(forms, KT_KEYS)
    for _ in range(2):
        k, valid = _g_block(rng)
        n = len(k)
        t.add({"g": _groups(rng, n, 2), "k": k, "t": rng.integers(0, 1500, n), "v0": rng.integers(0, 100, n)},
              {"k": valid})
    if mixed:
        n = 3000
        k = np.where(rng.random(n) < 0.5, rng.choice(np.asarray(G_KEYS, np.int64), n), 1000 + np.arange(n))
        valid = rng.random(n) > 0.05  # the gaps read 0
        valid[-100:] = False  # past len(Values): missing
        k[0] = -1
        t.add({"g": _groups(rng, n, 2), "k": k, "t": rng.integers(0, 1500, n), "v0": rng.integers(0, 100, n)},
              {"k": valid}, threshold=50, block_rows=1500)
    t.extents(v0=(0, 100))
    return t.done(_g_queries(t.spec, [r"hashg=1"] if mixed else [r"hashg=0 .*gbits=\d"], () if mixed else (8, 32)))


def family_g_str(forms=None):
    """A str column holding "" next to rows without it, bucket-encoded and as value arrays (whose gaps read the
    block's first string, here "").  The reference renders both as "" and then keeps one of the two groups per
    block, whichever its map iteration visits last (translate_group_by, aggregate.go:284-324), so its answer is
    not deterministic; the engine merges them, as tests/rowref.py and pyoracle do.  These queries carry
    oracle=False: the C++ oracle, which keeps one of the two like the reference, is not compared."""
    rng = np.random.default_rng(23)
    t = _Table(forms, KT_KEYS)
    n = 1200
    for thr in (5000, 40):
        s = rng.choice(np.asarray(["", "a", "b"]), n)
        if thr < 5000:
            s = np.where(rng.random(n) < 0.5, s, np.asarray(["x%d" % i for i in range(n)]))
            s[0] = ""
        valid = rng.random(n) > 0.1
        valid[0] = True
        t.add({"g": _groups(rng, n, 2), "s": s, "t": rng.integers(0, 1500, n), "v0": rng.integers(0, 100, n)},
              {"s": valid}, threshold=thr)
    t.extents(v0=(0, 100))
    s = t.spec
    dense = [r"hashed=0 hashg=0 "]
    qs = [_q(s, groups=["s"], aggs=["v0"], op="avg", expect=dense),
          _q(s, groups=["g", "s"], aggs=["v0"], op="hist", expect=dense),
          _q(s, groups=["s"], aggs=["v0"], op="avg", time_col="t", time_bucket=500, expect=dense + [r"tbit=1"]),
          _q(s, groups=["s"], aggs=["v0"], op="avg", limit=2, expect=dense)]
    for q in qs:
        q.oracle = False
    return t.done(qs)


# ---------------------------------------------------------------------------------------------------------------
# H. Slot-word widths
# ---------------------------------------------------------------------------------------------------------------
# int group columns of a given number of distinct values (radix = that + 1, code 0 missing): radices 16, 16, 17,
# 256, 256, 8, 8, 2.  Every block holds every value, and one row sits on every axis' highest code at once
H_DISTINCT = {"a": 15, "b": 15, "c": 16, "d": 255, "e": 255, "q": 7, "r": 7, "p": 1}
H_TAGS = ["t%d" % i for i in range(14)]


def _h_word(gbits, fbits, tbit, nbytes):
    return r"slot_bytes=%d .*gbits=%d fbits=%d tbit=%d" % (nbytes, gbits, fbits, tbit)


def family_h(forms=None):
    """Group axes whose radix products put gbits + fbits + tbit on 8 / 9, 16 / 17 and 32 bits: no filter, fail mode
    (f is in every row), count mode with 1, 3 and 4 counting filters (f2 misses rows), IN / NIN sticky bits, with and
    without the time bit (every block inside one time bucket: a window of one code, so lslots = 2 x the group slots).
    The widest query passes the slot word 0xFFFFFFFF for legitimate rows in blocks whose v0 array ends early."""
    rng = np.random.default_rng(24)
    t = _Table(forms, KT_KEYS)
    n = 4096
    for blk in range(3):
        cols, valid = {}, {}
        for c, m in H_DISTINCT.items():
            v = rng.integers(0, m, n)
            v[:m] = np.arange(m)  # every value in every block
            v[300:364] = m - 1  # rows on the highest code of every axis
            cols[c] = v
            va = rng.random(n) > 0.02
            va[:364] = True
            va[-3:] = False  # rows on code 0 of every axis
            valid[c] = va
        cols["f"] = rng.integers(0, 10, n)
        cols["f2"] = rng.integers(0, 10, n)
        valid["f2"] = rng.random(n) > 0.1
        valid["f2"][:1024] = True
        tags = [list(H_TAGS) if i < 512 or rng.random() < 0.3 else list(rng.choice(H_TAGS, 3, replace=False))
                for i in range(n)]
        cols["tags"] = tags
        valid["tags"] = rng.random(n) > 0.05
        valid["tags"][:1024] = True
        cols["t"] = np.full(n, 1000 * blk + 10)
        # v0 a value array (threshold 300 < its distinct values) whose len(Values) ends 40 rows before the block
        cols["v0"] = rng.integers(0, 1000, n)
        valid["v0"] = np.ones(n, bool)
        valid["v0"][-40:] = False
        t.add(cols, valid, threshold=300)
    t.extents(v0=(0, 1000))
    s = t.spec
    ins = [("tags", "in", x) for x in H_TAGS]
    f1, f2 = [("f", "gt", -1)], [("f2", "gt", -1)]
    f3 = f2 + [("f2", "lt", 9), ("f2", "neq", 5)]
    f4 = f3 + [("f2", "neq", 7)]
    tm = dict(time_col="t", time_bucket=1000)
    avg = dict(aggs=["v0"], op="avg")
    qs = [
        _q(s, groups=["a", "b"], expect=[_h_word(8, 0, 0, 1)], **avg),
        _q(s, groups=["a", "c"], expect=[_h_word(9, 0, 0, 2)], **avg),
        _q(s, groups=["d", "e"], expect=[_h_word(16, 0, 0, 2)], **avg),
        _q(s, groups=["d", "e", "p"], expect=[_h_word(17, 0, 0, 4)], **avg),
        _q(s, int_filters=f1, groups=["a", "q"], expect=[_h_word(7, 1, 0, 1), "fail_mode=1"], **avg),
        _q(s, int_filters=f1, groups=["a", "b"], expect=[_h_word(8, 1, 0, 2), "fail_mode=1"], **avg),
        _q(s, int_filters=f1, groups=["d", "a"], expect=[_h_word(12, 1, 0, 2), "fail_mode=1"], **avg),
        _q(s, int_filters=f2, groups=["a", "q"], expect=[_h_word(7, 1, 0, 1), "fail_mode=0"], **avg),
        _q(s, int_filters=f2, groups=["a", "b"], expect=[_h_word(8, 1, 0, 2), "fail_mode=0"], **avg),
        _q(s, int_filters=f3, groups=["q", "r"], expect=[_h_word(6, 2, 0, 1)], **avg),
        _q(s, int_filters=f3, groups=["a", "q"], expect=[_h_word(7, 2, 0, 2)], **avg),
        _q(s, int_filters=f4, groups=["d", "a", "p"], expect=[_h_word(13, 3, 0, 2)], **avg),
        _q(s, int_filters=f4, groups=["d", "c", "p"], expect=[_h_word(14, 3, 0, 4)], **avg),
        _q(s, set_filters=ins[:1], groups=["a", "q"], expect=[_h_word(7, 1, 0, 1)], **avg),
        _q(s, set_filters=[("tags", "nin", "zz")], groups=["a", "q"], expect=[_h_word(7, 2, 0, 2)], **avg),
        _q(s, set_filters=[("tags", "nin", "t3")], groups=["q", "r"], expect=[_h_word(6, 2, 0, 1)], **avg),
        _q(s, groups=["q", "r"], expect=[_h_word(7, 0, 1, 1)], **avg, **tm),
        _q(s, groups=["a", "q"], expect=[_h_word(8, 0, 1, 2)], **avg, **tm),
        _q(s, int_filters=f1, groups=["a", "r"], expect=[_h_word(8, 1, 1, 2)], **avg, **tm),
        # 17 group bits + 1 pass-counter bit + 14 IN bits: the highest slot's passing rows have the word 0xFFFFFFFF
        _q(s, int_filters=f2, set_filters=ins, groups=["d", "e", "p"], expect=[_h_word(17, 15, 0, 4)], **avg),
        _q(s, int_filters=f2, set_filters=ins, groups=["d", "e", "p"], op="hist", aggs=["v0"],
           expect=[_h_word(17, 15, 0, 4)]),
    ]
    return t.done(qs)


def h_refused(spec):
    """The widest H layout plus the time bit: 33 bits, refused ("slot word wider than 32 bits")."""
    return _q(spec, int_filters=[("f2", "gt", -1)], set_filters=[("tags", "in", x) for x in H_TAGS],
              groups=["d", "e", "p"], aggs=["v0"], op="avg", time_col="t", time_bucket=1000)


# ---------------------------------------------------------------------------------------------------------------
# K. Thresholds inside the pass
# ---------------------------------------------------------------------------------------------------------------
K_BINS = [1023, 1024, 1025]  # per-bin payload: in shared memory up to SMEM_BINS = 1024 bins, then in gbinpay


def family_k(forms=None):
    """A bucket-encoded group column and filter column with 1,023 / 1,024 / 1,025 bins in one block each, and a
    group column in every row of its blocks (count from bin sizes, COL_FULL) next to the same with one row missing."""
    rng = np.random.default_rng(25)
    t = _Table(forms, KT_KEYS)
    for nb in K_BINS:
        n = 8192
        k = rng.integers(0, nb, n)
        k[:nb] = np.arange(nb)
        f = rng.integers(0, nb, n)
        f[:nb] = np.arange(nb)
        t.add({"g": _groups(rng, n, 2), "k": k * 7 - 3000, "f": f, "v0": rng.integers(0, 100, n)},
              threshold=nb)
    for miss in (False, True):
        n = 5000
        a = rng.integers(0, 40, n)
        va = np.ones(n, bool)
        va[1234] = not miss
        t.add({"g": _groups(rng, n, 3), "a": a, "v0": rng.integers(0, 100, n)}, {"a": va})
    t.extents(v0=(0, 100))
    s = t.spec
    return t.done([
        # count_bins: the blocks whose Count comes from bin sizes (the three k blocks list every row once)
        _q(s, groups=["k"], aggs=["v0"], op="avg", expect=[r"count_bins=3\b"]),
        _q(s, int_filters=[("f", "gt", 100)], groups=["k"], aggs=["v0"], op="avg", expect=[r"count_bins=0\b"]),
        _q(s, int_filters=[("f", "lt", 1000)], groups=["g", "k"], aggs=["v0"], op="hist", expect=[r"count_bins=0\b"]),
        # the a block without a missing row takes the shortcut, the one with a missing row does not
        _q(s, groups=["a"], aggs=["v0"], op="avg", expect=[r"count_bins=1\b"]),
        _q(s, groups=["a"], aggs=[], op="avg", expect=[r"count_bins=1\b"]),
    ])


# ---------------------------------------------------------------------------------------------------------------
# I. The dense / hashed switch and the code ceiling
# ---------------------------------------------------------------------------------------------------------------
def slot_hash(x):
    """sybil_b200/csrc/sg_internal.h slot_hash, restated over uint32 numpy arrays: the hashed slot space probes
    from slot_hash(code + 1) & hmask.  The collision chains of family_i_ceiling depend on this function."""
    x = np.asarray(x, np.uint32)
    with np.errstate(over="ignore"):
        x = x ^ (x >> np.uint32(16))
        x = x * np.uint32(0x7feb352d)
        x = x ^ (x >> np.uint32(15))
        x = x * np.uint32(0x846ca68b)
        x = x ^ (x >> np.uint32(16))
    return x


def _strs(prefix, n):
    return np.array(["%s%05d" % (prefix, i) for i in range(n)])


def family_i_dense(plus, forms=None):
    """Two str axes of radix 8192 each: 8,189 strings in a first block (then the "" staging interns) and one more
    in a second block, whose row sits on the last slot of the 2^26 dense slots.  plus: a third block adds one more s
    string, radix 8192 x 8193 = 2^26 + 8192 codes: hashed, its table at the 2^16 minimum.  (2^26 + 1 = 5 x
    13,421,773 would need 13M strings on one axis; 8192 x 8193 is the smallest product of these axes past 2^26.)"""
    rng = np.random.default_rng(26)
    t = _Table(forms, KT_KEYS)
    n = 8189
    g, s = _strs("a", n + 2), _strs("b", n + 2)
    t.add({"g": g[:n], "s": rng.permutation(s[:n]), "v0": rng.integers(0, 100, n)})
    # the last slot on 3 rows, the largest group (a tie-free top-1)
    t.add({"g": np.array([g[n], g[n], g[n], g[0]]), "s": np.array([s[n]] * 4), "v0": [7, 8, 9, 10]})
    if plus:
        t.add({"g": np.array([g[n]]), "s": np.array([s[n + 1]]), "v0": [9]})
    t.extents(v0=(0, 100))
    sp = t.spec
    expect = ([r"lslots=65536 nslots=65536 hashed=1 hashg=0 gbits=27 fbits=0 tbit=0 "] if plus else
              [r"lslots=67108864 nslots=67108864 hashed=0 hashg=0 gbits=26 fbits=0 tbit=0 "])
    return t.done([_q(sp, groups=["g", "s"], aggs=[], op="avg", expect=expect),
                   _q(sp, groups=["s", "g"], aggs=[], op="avg", limit=1, expect=expect)])


def i_dense_hist(spec):
    """A histogram over the 2^26 dense slots: 1,002 counters per slot, far past the 24 GiB accumulator limit."""
    return _q(spec, groups=["g", "s"], aggs=["v0"], op="hist")


I_CEIL = (42964, 49979)  # strings of g and s: radices 42,966 x 49,981 = 2^31 - 2 = MAX_CODE_SPACE


def family_i_ceiling(forms=None):
    """The 31-bit code ceiling.  A first block (f = 0) holds every string: g's 42,964, s's 49,979 and s2's 49,980
    (radix 49,982: g x s2 is past 2^31 - 2).  Queries filter on f with eq, so zone maps drop that block and the
    hashed table is sized by the rows of the blocks they list:
    - f = 1: 160 rows on codes whose slot_hash lands on the last entries of the 2^16-entry table or on its first
      ones, so probe chains wrap from hmask to 0 (each such key on 3 rows), plus random codes;
    - f = 2 / 3: 32,768 / 32,769 random rows, 2 x rows just at / just past 2^16: tables of 2^16 / 2^17 entries.
    With one filter in fail mode the slot word is 31 group bits + 1: exactly 32, accepted."""
    rng = np.random.default_rng(31)
    t = _Table(forms, KT_KEYS)
    ng, ns = I_CEIL
    n = ns + 1
    g, s, s2 = _strs("a", ng), _strs("b", ns), _strs("c", n)
    t.add({"g": np.resize(g, n), "s": np.resize(s, n), "s2": s2, "f": np.zeros(n, np.int64)})
    # global ids follow first sight: g[i] -> i, s[i] -> i ("" comes after them); code = (ig + 1) + (is + 1) * 42966
    ig = np.arange(ng, dtype=np.int64)
    pick = []
    for js in rng.choice(ns, 400, replace=False):
        code = (ig + 1) + (int(js) + 1) * (ng + 2)
        h = slot_hash((code + 1).astype(np.uint32)) & np.uint32(0xFFFF)
        for want in (0xFFFF, 0xFFFE, 0xFFFD, 0, 1):
            pick += [(int(i), int(js)) for i in np.nonzero(h == want)[0][:1]]
    pick = pick[:40]
    rows = [p for p in pick for _ in range(3)] + [(int(rng.integers(ng)), int(rng.integers(ns))) for _ in range(40)]
    a, b = np.array([r[0] for r in rows]), np.array([r[1] for r in rows])
    t.add({"g": g[a], "s": s[b], "f": np.ones(len(rows), np.int64), "v0": rng.integers(0, 100, len(rows))})
    for f, m in ((2, 32768), (3, 32769)):
        t.add({"g": g[rng.integers(0, ng, m)], "s": s[rng.integers(0, ns, m)], "f": np.full(m, f),
               "v0": rng.integers(0, 100, m)})
    t.extents(v0=(0, 100))
    sp = t.spec
    word = r"hashed=1 hashg=0 gbits=31 fbits=1 tbit=0 "
    qs = [_q(sp, int_filters=[("f", "eq", 1)], groups=["g", "s"], aggs=["v0"], op="avg",
             expect=[r"fail_mode=1 .*nslots=65536 " + word]),
          _q(sp, int_filters=[("f", "eq", 2)], groups=["g", "s"], aggs=[], op="avg",
             expect=[r"nslots=65536 " + word]),
          _q(sp, int_filters=[("f", "eq", 3)], groups=["s", "g"], aggs=[], op="avg",
             expect=[r"nslots=131072 " + word])]
    qs[0].wraps = pick  # (ig, is) of the keys whose probe chains wrap, for the test that checks they are there
    return t.done(qs)


def i_refused(spec):
    """Queries the planner must refuse on the ceiling table: the 2^31 - 2 codes with a time bit (33 bits), and a
    product past 2^31 - 2."""
    return [_q(spec, int_filters=[("f", "eq", 1)], groups=["g", "s"], aggs=[], op="avg", time_col="f",
               time_bucket=1),
            _q(spec, int_filters=[("f", "eq", 1)], groups=["g", "s2"], aggs=[], op="avg")]


# ---------------------------------------------------------------------------------------------------------------
# L, W, R. Result shaping: order, limit and ties; weights; StrReplace
# ---------------------------------------------------------------------------------------------------------------
# Every query of these families carries `expect` patterns for its `sg_select:` trace line (build_result's choice
# of selection path).  Ties break by the rendered GroupByKey as bytes: a leading byte below '\t' sorts before the
# missing field, an embedded tab compares against the next field's bytes.
KT_ORDER = [("s", STR), ("s2", STR), ("k", INT), ("k2", INT), ("t", INT), ("w", INT), ("f", INT), ("v0", INT),
            ("v1", INT)]
V0_HI = I64_MAX // 10  # 10 * V0_HI = INT64_MAX - 7: values up to there are accepted
# str key, rows, v0 values, v1 values (the other rows lack the column).  Counts tie on purpose: six groups of 6
# (missing, the control-byte and the tab keys), four of 3, two of 2.  Means: 1/3 and 2/6, -7.5 twice, 2^53 and
# 2^53 + 1 (one double), INT64_MAX - 7 twice (the sum wraps to -16), and no v0 / v1 histogram on many groups
L_STR = [(None, 6, [1, 0, 0], [5]),
         ("\x01", 6, [1, 1, 0, 0, 0, 0], []),
         ("\x08z", 6, [-7, -8], [5]),
         ("a\tb", 6, [1 << 53], [-3]),
         ("a", 6, [(1 << 53) + 1], []),
         ("\t", 6, [], [5]),
         ("a\tc", 3, [V0_HI * 10, V0_HI * 10], []),
         ("é", 3, [-8, -7], []),
         ("日本", 3, [], []),
         ("z", 3, [], [-1]),
         ("b", 2, [], []),
         ("c", 2, [1, 2], [])]
L_INT = [9, 10, -5, I64_MIN, -1, 100]  # -1 renders (and groups) as missing


def _sel(path, threads=None):
    return [r"^sg_select: path=%s threads=%s$" % (path, threads if threads is not None else r"\d+")]


def _l_rows(t, block_split=True):
    """The L_STR groups as rows: k cycles over L_INT and the missing value, t over two time buckets."""
    s, sv, v0, v0v, v1, v1v = [], [], [], [], [], []
    for key, n, a, b in L_STR:
        for i in range(n):
            s.append(key or "")
            sv.append(key is not None)
            v0.append(a[i] if i < len(a) else 0)
            v0v.append(i < len(a))
            v1.append(b[i] if i < len(b) else 0)
            v1v.append(i < len(b))
    n = len(s)
    kk = [L_INT[i % 7] if i % 7 < len(L_INT) else 0 for i in range(n)]
    cols = {"s": np.asarray(s, dtype=object).astype(str), "k": kk, "t": [(i * 37) % 2000 for i in range(n)],
            "v0": v0, "v1": v1}
    valid = {"s": np.asarray(sv), "k": np.asarray([i % 7 < len(L_INT) for i in range(n)]),
             "v0": np.asarray(v0v), "v1": np.asarray(v1v)}
    # first half bucket-encoded, second half as value arrays
    h = n // 2
    t.add({c: v[:h] for c, v in cols.items()}, {c: v[:h] for c, v in valid.items()})
    t.add({c: v[h:] for c, v in cols.items()}, {c: v[h:] for c, v in valid.items()}, threshold=2)


def _live(spec, rows, valid, q):
    from tests import rowref
    return len(rowref.run(spec, rows, valid, q).Results)


def _l_queries(t, groups_list, limits_of, orders=("$COUNT", "v0", "v1"), time=False, expect=None):
    s = t.spec
    qs = []
    for groups in groups_list:
        live = _live(s, t.rows, t.valid, Q(s, groups=groups, aggs=["v0", "v1"], op="avg"))
        for ob in orders:
            for asc in (False, True):
                for limit in limits_of(live):
                    kw = dict(time_col="t", time_bucket=1000) if time else {}
                    qs.append(_q(s, groups=groups, aggs=["v0", "v1"], op="avg", order_by=ob, order_asc=asc,
                                 limit=limit, expect=expect(ob, asc, limit, live) if expect else _sel("host", 1),
                                 **kw))
        for limit in (0, 2):  # OrderBy "": any `limit` groups
            qs.append(_q(s, groups=groups, aggs=["v0", "v1"], op="avg", order_by="", limit=limit,
                         expect=_sel("host", 1)))
    return qs


def family_l_small(forms=None):
    """Fewer than 2^17 slots: the lazy host path on one thread, and time mode."""
    t = _Table(forms, KT_ORDER)
    _l_rows(t)
    t.extents(v0=(-(1 << 62), V0_HI), v1=(-100, 100))
    qs = _l_queries(t, [["s"], ["k"], ["s", "k"], ["k", "s"]], lambda live: (0, 1, 3, live - 1, live, live + 1))
    qs += _l_queries(t, [["s"], ["s", "k"]], lambda live: (0, 3), time=True)
    return t.done(qs)


L_LIMIT = 100  # the device path's cap is L_LIMIT + 8192 candidates
L_TIED = L_LIMIT + 8192 - (L_LIMIT - 1)  # groups tied at the cut that fill the cap exactly


def family_l_large(forms=None):
    """More than 2^17 slots (s: 64 codes x k2: 5,000) with accumulators too large to come back behind the scan:
    the device top-K, its fall-back to the host and the host's many-thread selection.  L_LIMIT - 1 groups of 3
    rows, L_TIED + 1 groups of 2 (the last one's rows have f = 1: without them the candidates at the cut number
    L_LIMIT + 8192 exactly, with them one more) and filler groups of 1 row.  The groups of 2 include every
    control-byte, tab and missing key, so which of them make the cut depends on full-key byte order."""
    rng = np.random.default_rng(40)
    t = _Table(forms, KT_ORDER)
    strs = [k for k, _, _, _ in L_STR if k is not None] + ["s%02d" % i for i in range(51)]  # 63 strings + missing
    n3, n2, n1 = L_LIMIT - 1, L_TIED + 1, 2000
    tied = [(a, b) for a in [None] + strs[:12] for b in range(5)]  # control / tab / missing keys among the tied
    others = [(a, b) for b in range(5, 4999) for a in [None] + strs]  # every other (s, k2) group
    sel = [others[i] for i in rng.permutation(len(others))[:n3 + n2 - len(tied) + n1]]
    top, tied, filler = sel[:n3], tied + sel[n3:n3 + n2 - len(tied)], sel[n3 + n2 - len(tied):]
    groups = [(p, 3, 0) for p in top] + [(p, 2, 0) for p in tied[:-1]] + [(tied[-1], 2, 1)] + [(p, 1, 0) for p in filler]
    rows = [(p, f) for p, c, f in groups for _ in range(c)]
    rows = [rows[i] for i in rng.permutation(len(rows))]
    n = len(rows)
    cols = {"s": np.asarray([p[0] or "" for p, _ in rows]), "k2": [p[1] for p, _ in rows],
            "f": [f for _, f in rows], "t": rng.integers(0, 2000, n),
            "v0": rng.integers(-50, 50, n), "v1": rng.integers(-5, 5, n)}
    cols["v0"][:4] = [1 << 53, (1 << 53) + 1, V0_HI * 10, -7]
    valid = {"s": np.asarray([p[0] is not None for p, _ in rows]), "v1": rng.random(n) < 0.3}
    t.add(cols, valid, block_rows=8192)
    t.extents(v0=(-(1 << 62), V0_HI), v1=(-100, 100))
    s = t.spec
    big = dict(groups=["s", "k2"], aggs=["v0", "v1"], op="avg")
    cap = [("f", "neq", 1)]
    qs = [_q(s, int_filters=cap, order_by="$COUNT", limit=L_LIMIT, expect=_sel("device", 1), **big),
          _q(s, order_by="$COUNT", limit=L_LIMIT, expect=_sel("device-fallback"), **big)]
    live = len(groups)

    def expect(ob, asc, limit, live):
        return _sel("device", 1) if not asc and 1 <= limit <= 65536 else _sel("host")
    for ob in ("$COUNT", "v0", "v1"):
        for asc in (False, True):
            for limit in (1, live - 1, live, live + 1, 65536, 65537):
                qs.append(_q(s, order_by=ob, order_asc=asc, limit=limit, expect=expect(ob, asc, limit, live), **big))
    qs.append(_q(s, order_by="", limit=3, expect=_sel("host"), **big))
    qs.append(_q(s, order_by="$COUNT", limit=5, time_col="t", time_bucket=1000, expect=_sel("host", 1), **big))
    for q in qs:
        q.live = live
    return t.done(qs)


def family_w(forms=None):
    """Weights: 0, -1 (a weight, not the missing alias), negative, +w / -w pairs in one group, 2^62 x 4 rows (Count
    wraps to 0), values next to INT64_MAX.  Groups made only of weight-0 rows; the weight column bucket-encoded in
    one block and a value array in the other."""
    t = _Table(forms, KT_ORDER)
    groups = [("zero", [0, 0, 0]), ("neg1", [-1, -1]), ("neg", [-5, -5, 3]), ("cancel", [7, -7]),
              ("wrap", [1 << 62] * 4), ("big", [I64_MAX, 1]), ("max", [I64_MAX - 1]), ("plain", [1, 2, 3]),
              (None, [2, 0]), ("zero2", [0]), ("one", [1])]
    s, sv, w, v0 = [], [], [], []
    for key, ws in groups:
        for i, x in enumerate(ws):
            s.append(key or "")
            sv.append(key is not None)
            w.append(x)
            v0.append((len(s) * 13) % 101)
    n = len(s)
    for thr in (5000, 3):
        t.add({"s": s, "w": w, "t": [(i * 211) % 1500 for i in range(n)], "v0": v0, "v1": v0[::-1]},
              {"s": np.asarray(sv), "v1": np.arange(n) % 3 > 0}, threshold=thr)
    t.extents(v0=(0, 100), v1=(0, 100))
    sp = t.spec
    qs = []
    for op, loghist in (("avg", False), ("hist", False), ("avg", True)):
        for time in (False, True):
            kw = dict(time_col="t", time_bucket=500) if time else {}
            for ob, limit in (("$COUNT", 0), ("v0", 0), ("v1", 4), ("$COUNT", 3)):
                qs.append(_q(sp, groups=["s"], aggs=["v0", "v1"], op=op, loghist=loghist, weight_col="w",
                             order_by=ob, limit=limit, expect=_sel("host", 1), **kw))
    for q in qs:
        # the reference drops a block's group result whose Count is 0 when it combines blocks, unless that block
        # is the first to hold the group (query_spec.go:143-145, DESIGN.md §7); the oracle and pyoracle restate that
        q.oracle = q.pyoracle = False
    return t.done(qs)


def family_r(forms=None):
    """StrReplace with order and limit: merging rewrites whose merged groups decide the cut, rewrites to "" and
    to strings with a leading control byte or a tab, rewrites on both group columns, a rewrite with weights, and
    a filter on the rewritten column."""
    t = _Table(forms, KT_ORDER)
    # s: ab1..ab4 merge into "ab" (4 groups of 2 rows -> one of 8, above every other group), cd -> "\x01c",
    # xy -> "\tx", zz -> "" (the missing group)
    counts = {"ab1": 2, "ab2": 2, "ab3": 2, "ab4": 2, "ab": 1, "cd": 5, "xy": 5, "zz": 3, "m": 5, "n": 6, None: 2}
    s = [k for k, c in counts.items() for _ in range(c)]
    n = len(s)
    s2 = ["q%d" % (i % 3) if i % 4 else "r" for i in range(n)]
    cols = {"s": np.asarray([x or "" for x in s]), "s2": np.asarray(s2), "w": [1 + i % 3 for i in range(n)],
            "t": [(i * 97) % 1000 for i in range(n)], "v0": [(i * 7) % 50 for i in range(n)]}
    valid = {"s": np.asarray([x is not None for x in s])}
    t.add({c: v[:n // 2] for c, v in cols.items()}, {c: v[:n // 2] for c, v in valid.items()})
    t.add({c: v[n // 2:] for c, v in cols.items()}, {c: v[n // 2:] for c, v in valid.items()}, threshold=3)
    t.extents(v0=(0, 50))
    sp = t.spec
    merge = {"s": (r"^(ab)\d$", "$1")}
    ctrl = {"s": (r"^cd$", "\x01c")}
    tab = {"s": (r"^x(y)$", "\t$1")}
    empty = {"s": (r"^zz$", "")}
    both = {"s": (r"^(ab)\d$", "$1"), "s2": (r"^q\d$", "q")}
    allr = {**merge, **ctrl, **tab, **empty}
    qs = []
    for rep in (merge, ctrl, tab, empty, both, allr):
        for ob, asc, limit in (("$COUNT", False, 1), ("$COUNT", False, 3), ("$COUNT", True, 2), ("v0", False, 3),
                               ("$COUNT", False, 0), ("", False, 2)):
            groups = ["s", "s2"] if rep is both else ["s"]
            q = _q(sp, groups=groups, aggs=["v0"], op="avg", order_by=ob, order_asc=asc, limit=limit,
                   str_replace=rep, expect=_sel("host", 1))
            # the C++ oracle keeps one of "" and missing (family_g_str): not compared under rewrites to ""
            q.oracle = rep is not empty and rep is not allr
            qs.append(q)
    qs.append(_q(sp, groups=["s"], aggs=["v0"], op="hist", weight_col="w", order_by="$COUNT", limit=3,
                 str_replace=merge, expect=_sel("host", 1)))
    qs.append(_q(sp, groups=["s"], aggs=["v0"], op="avg", order_by="$COUNT", limit=2, time_col="t", time_bucket=500,
                 str_replace=allr, expect=_sel("host", 1)))
    qs[-1].oracle = False
    # a filter on the rewritten column: "ab" is a present literal, but under the merging rewrite the reference's
    # lookup maps it to one of the merged ids (DESIGN.md §7), so the oracle is not compared
    q = _q(sp, str_filters=[("s", "eq", "ab")], groups=["s", "s2"], aggs=["v0"], op="avg", order_by="$COUNT",
           limit=2, str_replace=merge, expect=_sel("host", 1))
    q.oracle = False
    qs.append(q)
    return t.done(qs)


ORDER_TABLES = {"L-small": family_l_small, "L-large": family_l_large, "W": family_w, "R": family_r}


KEY_TABLES = {"G-int": lambda forms=None: family_g_int(False, forms),
              "G-mixed": lambda forms=None: family_g_int(True, forms),
              "G-str": family_g_str, "H": family_h, "K": family_k,
              "I-dense": lambda forms=None: family_i_dense(False, forms),
              "I-hashed": lambda forms=None: family_i_dense(True, forms), "I-ceiling": family_i_ceiling}


def all_tables(forms=None):
    """(name, (spec, rows, valid, queries)) of every family."""
    out = [("A", family_a(forms))]
    out += [("B-carry", family_b_carry(forms))] + [("B-fold-" + w, family_b_fold(w, forms)) for w in B_FOLD]
    out += [("C%d" % i, x) for i, x in enumerate(family_c(forms))]
    out += [("D%d" % i, x) for i, x in enumerate(family_d(forms))]
    out += [("E", family_e(forms)), ("F", family_f(forms))]
    out += [(name, build(forms)) for name, build in KEY_TABLES.items()]
    out += [(name, build(forms)) for name, build in ORDER_TABLES.items()]
    return out
