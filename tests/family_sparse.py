"""Sparse group accumulators (sg_query_set_sparse_groups): group-by histograms whose accumulators, one row of
bucket counters per slot of the dense slot space or of the hashed table, pass 24 GiB while few groups occur.
Used by tests/test_parity_sparse.py.

Each constructor returns (spec, rows, valid, queries) like tests/edges.py.  A query's `ref` says what it is
checked against: "rowref" (tests/rowref.py, bit for bit) where the table is small enough for it, "oracle" (the
C++ oracle, tests.util.compare) otherwise.

Per slot, a BasicHist aggregation takes 1 + 3 + 1,002 words, so past about 3.2M slots its accumulators pass
24 GiB; a MultiHist (`loghist`) over extents of 10^6 takes 11 sub-ranges of about 1,000 counters each, so past
about 290k slots.  A hashed plan's table gets 2 x the listed rows' entries, rounded up to a power of two: past
2^20 listed rows (2^22 entries) for BasicHist, past 2^17 (2^19 entries) for MultiHist."""
import numpy as np

from tests.edges import _q, _strs, _Table
from tests.util import INT, STR

KT = [("g", STR), ("s", STR), ("k", INT), ("t", INT), ("f", INT), ("v", INT)]
V_HI = 1_000_000


def _pairs(rng, na, nb, n):
    """n distinct (a, b) index pairs drawn from na x nb."""
    flat = rng.choice(na * nb, n, replace=False)
    return flat // nb, flat % nb


def family_dense_axes(forms=None):
    """Two str axes of 2,000 x 1,700 strings (3.4M dense slots, within 2^26) with 1,500 live (g, s) pairs on
    30,000 rows, every string of both axes in the dictionaries; 3% of the rows lack s (the missing key), 5% lack v.
    BasicHist and MultiHist (`-op hist -loghist`) over v are both past 24 GiB dense; avg is not."""
    rng = np.random.default_rng(71)
    t = _Table(forms, KT)
    ng, ns = 2000, 1700
    g, s = _strs("a", ng), _strs("b", ns)
    # every string once (f = 1), then the live pairs (f = 0)
    t.add({"g": np.resize(g, ns), "s": s, "f": np.ones(ns, np.int64), "v": rng.integers(0, V_HI, ns)})
    t.add({"g": g[:300], "s": s[:300], "f": np.ones(300, np.int64), "v": rng.integers(0, V_HI, 300)})
    t.add({"g": g[300:], "s": np.resize(s, ng - 300), "f": np.ones(ng - 300, np.int64), "v": rng.integers(0, V_HI, ng - 300)})
    a, b = _pairs(rng, ng, ns, 1500)
    n = 30000
    pick = rng.integers(0, len(a), n)
    t.add({"g": g[a[pick]], "s": s[b[pick]], "f": np.zeros(n, np.int64), "k": rng.integers(0, 50, n),
           "v": rng.integers(0, V_HI, n)},
          {"s": rng.random(n) > 0.03, "v": rng.random(n) > 0.05}, block_rows=8192)
    t.extents(v=(0, V_HI))
    sp = t.spec
    qs = [_q(sp, groups=["g", "s"], aggs=["v"], op="hist"),
          _q(sp, groups=["s", "g"], aggs=["v"], op="hist", loghist=True),
          _q(sp, int_filters=[("k", "lt", 25)], str_filters=[("g", "neq", g[a[0]])], groups=["g", "s"], aggs=["v"],
             op="hist", order_by="v", limit=10),
          _q(sp, int_filters=[("f", "eq", 0)], groups=["g", "s"], aggs=["v"], op="hist", order_by="", limit=0)]
    for q in qs:
        q.ref = "rowref"
    return t.done(qs)


def family_time(forms=None):
    """Time mode: 1,200 g strings x 3,000 time buckets (3.6M dense (time, group) slots) with a BasicHist of 1,002
    counters (extents [0, 10^6]), past 24 GiB; 40 live g values on 6,000 rows whose times fall into 60 buckets, 2% of
    the rows without a time."""
    rng = np.random.default_rng(72)
    t = _Table(forms, KT)
    g = _strs("a", 1200)
    t.add({"g": g, "t": np.zeros(1200, np.int64), "v": rng.integers(0, V_HI, 1200), "f": np.ones(1200, np.int64)})
    n = 6000
    live = rng.choice(1200, 40, replace=False)
    tb = rng.choice(3000, 60, replace=False)
    t.add({"g": g[live[rng.integers(0, 40, n)]], "t": tb[rng.integers(0, 60, n)] * 100 + rng.integers(0, 100, n),
           "v": rng.integers(0, V_HI, n), "f": np.zeros(n, np.int64)},
          {"t": rng.random(n) > 0.02}, block_rows=2000)
    t.add({"g": g[:1], "t": np.array([299_999]), "v": np.array([5]), "f": np.ones(1, np.int64)})
    t.extents(v=(0, V_HI), t=(0, 299_999))
    sp = t.spec
    qs = [_q(sp, groups=["g"], aggs=["v"], op="hist", time_col="t", time_bucket=100),
          _q(sp, int_filters=[("f", "eq", 0)], groups=["g"], aggs=["v"], op="hist", time_col="t", time_bucket=100,
             order_by="v", limit=5)]
    for q in qs:
        q.ref = "rowref"
    return t.done(qs)


def family_hashed(rows, loghist, forms=None):
    """Two str axes of 5,000 x 20,000 strings (1e8 codes: hashed) with `rows` listed rows on 5,000 live pairs.
    A first block holds every string with f = 1; the queries filter f == 0, so the zone map drops it and the
    table is sized by the listed rows alone."""
    rng = np.random.default_rng(73 + rows)
    t = _Table(forms, KT)
    ng, ns = 5000, 20000
    g, s = _strs("a", ng), _strs("b", ns)
    t.add({"g": np.resize(g, ns), "s": s, "f": np.ones(ns, np.int64), "v": rng.integers(0, V_HI, ns),
           "k": rng.integers(0, 100, ns)})
    a, b = _pairs(rng, ng, ns, 5000)
    pick = rng.integers(0, len(a), rows)
    t.add({"g": g[a[pick]], "s": s[b[pick]], "f": np.zeros(rows, np.int64), "k": rng.integers(0, 100, rows),
           "v": rng.integers(0, V_HI, rows)},
          {"v": rng.random(rows) > 0.02}, block_rows=65536)
    t.extents(v=(0, V_HI))
    sp = t.spec
    f0 = [("f", "eq", 0)]
    kw = dict(aggs=["v"], op="hist", loghist=loghist)
    qs = [_q(sp, int_filters=f0, groups=["g", "s"], **kw),
          _q(sp, int_filters=f0 + [("k", "lt", 60)], str_filters=[("g", "neq", g[a[0]])], groups=["s", "g"],
             order_by="v", limit=20, **kw)]
    for q in qs:
        q.ref = "oracle"
    return t.done(qs)


def family_broken(forms=None):
    """A table whose second block holds keys of its own and whose NumRecords shrank under its row ids: the block
    is dropped whole ("BLOCK SIZE CHANGED"), so its keys must not become groups.  Its columns are bucket-encoded,
    with string tables no longer than the block, so staging accepts it and the scan itself finds the row ids past
    NumRecords: first in the discovery launch, whose table then holds the block's keys, then in the aggregation
    launch, which reports the block; the engine then discovers again without it."""
    rng = np.random.default_rng(74)
    t = _Table(forms, KT)
    for i in range(3):
        n = 3000
        t.add({"g": np.array(["b%d_%d" % (i, x) for x in rng.integers(0, 40, n)]), "s": _strs("s", 50)[rng.integers(0, 50, n)],
               "v": rng.integers(0, 1000, n)})
    t.spec.blocks[1].num_records = 1000
    t.extents(v=(0, 1000))
    sp = t.spec
    return t.done([_q(sp, groups=["g", "s"], aggs=["v"], op="hist")])
