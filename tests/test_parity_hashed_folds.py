"""Weighted and StrReplace group-bys over hashed and sparse group keys, folded on the device
(sg_query_set_hashed_folds, engine.FLAGS.HASHED_FOLDS).  Every folded result is checked bit for bit against the
row-level reference tests/rowref.py and, where the same query runs on a dense plan (folded on the host by
dense_fold), against that run's complete listing.  Tables: tests/edges.py (families W and R),
tests/test_parity_weight_carry.py and tables built here in the shape of tests/family_sparse.py."""
import ctypes as C
import re

import numpy as np
import pytest

from sybil_b200 import _ffi as F
from sybil_b200 import engine as E
from tests import edges, family_sparse as FS, rowref
from tests import test_parity_weight_carry as WC
from tests.test_parity_sparse import _check as check_sparse
from tests.util import INT, STR, Q, run_gpu

pytestmark = pytest.mark.gpu

_TABLES = {}


def _table(name, build):
    if name not in _TABLES:
        _TABLES[name] = build()
    return _TABLES[name]


@pytest.fixture(autouse=True)
def _reset_flags():
    """engine.FLAGS is process-wide: no test of another module may inherit HASHED_FOLDS / SPARSE_GROUPS."""
    yield
    E.FLAGS.reset()


def flags(q, folds=True, sparse=False):
    """q with engine.FLAGS.HASHED_FOLDS / SPARSE_GROUPS set whenever it builds its QuerySpec."""
    base = type(q).set_flags

    def set_flags():
        base(q)
        E.FLAGS.HASHED_FOLDS = folds
        E.FLAGS.SPARSE_GROUPS = sparse
    q.set_flags = set_flags
    return q


def _status(fn):
    try:
        fn()
    except E.SybilGpuError as e:
        return e.status
    return F.SG_OK


def _staged(spec):
    table = E.Table("t", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    for b in spec.blocks:
        table.add_block(b)
    return table


def _lines(capfd, prefix):
    return [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith(prefix)]


def _traces(capfd):
    err = capfd.readouterr().err.splitlines()
    return ([ln for ln in err if ln.startswith("sg_plan:")], [ln for ln in err if ln.startswith("sg_fold:")],
            [ln for ln in err if ln.startswith("sg_sparse:")])


def _canon(fold_line):
    return int(re.search(r"canon=(\d+)", fold_line).group(1))


# ---- 1. existing families through the fold ---------------------------------------------------------------------
MODES = [("dense", {}, dict(folds=False)),
         ("hashed", {"SG_FORCE_HASHED_SLOTS": "1"}, dict(folds=True)),
         ("sparse", {"SG_FORCE_SPARSE_GROUPS": "1"}, dict(folds=True, sparse=True))]


def _three_ways(spec, rows, valid, queries, monkeypatch, capfd, variant, where0):
    """Each query dense, forced hashed and forced sparse: one listing, equal to rowref."""
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    table = _staged(spec)
    try:
        for i, q in enumerate(queries):
            where = where0 + (i,)
            ref = rowref.run(spec, rows, valid, q)
            listings = []
            for mode, env, fl in MODES:
                for k in ("SG_FORCE_HASHED_SLOTS", "SG_FORCE_SPARSE_GROUPS"):
                    monkeypatch.delenv(k, raising=False)
                for k, v in env.items():
                    monkeypatch.setenv(k, v)
                capfd.readouterr()
                g = run_gpu(spec, flags(q, **fl), table)
                plans, folds, _ = _traces(capfd)
                w = where + (mode,)
                assert plans, w
                if mode == "dense":
                    assert " hashed=0 " in plans[-1] and " fold=1" not in plans[-1] and not folds, (w, plans[-1])
                else:
                    assert " hashed=1 " in plans[-1] and plans[-1].endswith(" fold=1"), (w, plans[-1])
                    assert (" sparse=1 " in plans[-1]) == (mode == "sparse"), (w, plans[-1])
                    assert len(folds) == 1, (w, folds)
                    if not q.time_col:
                        assert _canon(folds[0]) == g.NumGroups, (w, folds[0], g.NumGroups)
                rowref.check(ref, g, q, where=w)
                listings.append(_listing(g, q))
            assert listings[1] == listings[0] and listings[2] == listings[0], where
    finally:
        table.close()


def _listing(g, q):
    """WC._listing; with OrderBy "" the groups come in no set order, and under a limit any `limit` of them do (each
    is checked against rowref), so only the rest of the listing is compared then."""
    sorted_, *rest = WC._listing(g)
    if not q.order_by:
        sorted_ = None if q.limit else sorted(sorted_)
    return [sorted_] + rest


def _folded(queries):
    return [q for q in queries if q.weight_col or q.str_replace]


@pytest.mark.parametrize("name,forms,variant", [(n, f, v) for n in ("W", "R") for f in ("narrow", "wide")
                                                for v in (8, 16)])
def test_order_families_through_the_fold(name, forms, variant, monkeypatch, capfd):
    """Weights 0, -1, negative, cancelling and wrapping; rewrites that merge, that go to "", to control bytes or
    tabs and that apply to both group columns; time mode; order by Count or a mean with a limit; avg / hist /
    loghist."""
    spec, rows, valid, queries = _table((name, forms), lambda: edges.ORDER_TABLES[name](forms))
    _three_ways(spec, rows, valid, _folded(queries), monkeypatch, capfd, variant, (name, forms, variant))


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("kind", ["codes", "walk", "values", "mixed", "signed"])
def test_weight_carry_tables_through_the_fold(kind, variant, monkeypatch, capfd):
    """Rows without the weight column carry the previous row's weight (weight code 0 under wcarry: weight 1)."""
    spec, rows, valid = _table(("wc", kind), lambda: WC.table(kind))
    _three_ways(spec, rows, valid, _folded(WC.queries(spec)), monkeypatch, capfd, variant, (kind, variant))


# ---- 2. hashed because of the weight axis ----------------------------------------------------------------------
KT2 = [("g", STR), ("s", STR), ("w", INT), ("v", INT)]
WEIGHTS = (1, 2, 3, 5, 8, 13, 21, 34)


def _weight_axis_table():
    """g and s of 3,000 strings each (9M dense codes unweighted), 8 distinct weights (81M codes weighted: hashed)."""
    rng = np.random.default_rng(91)
    t = edges._Table(None, KT2)
    n = 3000
    g, s = edges._strs("a", n), edges._strs("b", n)
    t.add({"g": g, "s": s[rng.permutation(n)], "w": rng.choice(WEIGHTS, n), "v": rng.integers(0, 1000, n)})
    m = 20000
    a, b = rng.integers(0, 400, m), rng.integers(0, 300, m)
    t.add({"g": g[a * 7], "s": s[b * 9], "w": rng.choice(WEIGHTS, m), "v": rng.integers(0, 1000, m)},
          {"v": rng.random(m) > 0.05}, block_rows=8192)
    t.extents(v=(0, 1000))
    return t.spec, t.rows, t.valid


def test_hashed_because_of_the_weight_axis(monkeypatch, capfd):
    spec, rows, valid = _table("waxis", _weight_axis_table)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    table = _staged(spec)
    try:
        plain = Q(spec, groups=["g", "s"], aggs=["v"], op="avg")
        capfd.readouterr()
        rowref.check(rowref.run(spec, rows, valid, plain), run_gpu(spec, plain, table), plain, where="unweighted")
        assert " hashed=0 " in _lines(capfd, "sg_plan:")[0]
        merge = {"g": (r"^(a\d\d\d)\d$", "$1")}
        for op in ("avg", "hist"):
            for rep in (None, merge):
                q = Q(spec, groups=["g", "s"], aggs=["v"], op=op, weight_col="w", str_replace=rep, order_by="v",
                      limit=50)
                assert _status(lambda: run_gpu(spec, flags(q, False), table)) == F.SG_ERR_UNSUPPORTED, (op, rep)
                capfd.readouterr()
                g = run_gpu(spec, flags(q), table)
                plans, folds, _ = _traces(capfd)
                assert " hashed=1 " in plans[0] and plans[0].endswith(" fold=1"), plans
                assert _canon(folds[0]) == g.NumGroups, (folds, g.NumGroups)
                rowref.check(rowref.run(spec, rows, valid, q), g, q, where=(op, rep))
    finally:
        table.close()


# ---- 3. sparse past 24 GiB --------------------------------------------------------------------------------------
KT3 = FS.KT + [("w", INT)]


def _dense_axes_weighted():
    """family_sparse.family_dense_axes with a weight column of 8 values, 4% of the rows without it."""
    rng = np.random.default_rng(92)
    t = edges._Table(None, KT3)
    ng, ns = 2000, 1700
    g, s = edges._strs("a", ng), edges._strs("b", ns)
    t.add({"g": np.resize(g, ns), "s": s, "w": rng.choice(WEIGHTS, ns), "v": rng.integers(0, FS.V_HI, ns)})
    t.add({"g": g[300:], "s": np.resize(s, ng - 300), "w": rng.choice(WEIGHTS, ng - 300),
           "v": rng.integers(0, FS.V_HI, ng - 300)})
    a, b = FS._pairs(rng, ng, ns, 1500)
    n = 30000
    pick = rng.integers(0, len(a), n)
    t.add({"g": g[a[pick]], "s": s[b[pick]], "w": rng.choice(WEIGHTS, n), "v": rng.integers(0, FS.V_HI, n)},
          {"s": rng.random(n) > 0.03, "v": rng.random(n) > 0.05, "w": rng.random(n) > 0.04}, block_rows=8192)
    t.extents(v=(0, FS.V_HI))
    sp = t.spec
    qs = [WC.CQ(sp, groups=["g", "s"], aggs=["v"], op="hist", weight_col="w"),
          WC.CQ(sp, groups=["s", "g"], aggs=["v"], op="hist", loghist=True, weight_col="w", order_by="v", limit=10)]
    return sp, t.rows, t.valid, qs


def _hashed_weighted(rows):
    """family_sparse.family_hashed's shape (5,000 x 20,000 strings, 5,000 live pairs) with 8 weights: 9e8 codes, and
    a MultiHist table of 2 x `rows` entries past 24 GiB.  Checked against the oracle (every weight positive)."""
    rng = np.random.default_rng(93)
    t = edges._Table(None, KT3)
    ng, ns = 5000, 20000
    g, s = edges._strs("a", ng), edges._strs("b", ns)
    t.add({"g": np.resize(g, ns), "s": s, "f": np.ones(ns, np.int64), "w": rng.choice(WEIGHTS, ns),
           "v": rng.integers(0, FS.V_HI, ns)})
    a, b = FS._pairs(rng, ng, ns, 5000)
    pick = rng.integers(0, len(a), rows)
    t.add({"g": g[a[pick]], "s": s[b[pick]], "f": np.zeros(rows, np.int64), "w": rng.choice(WEIGHTS, rows),
           "v": rng.integers(0, FS.V_HI, rows)}, {"v": rng.random(rows) > 0.02}, block_rows=65536)
    t.extents(v=(0, FS.V_HI))
    sp = t.spec
    q = Q(sp, int_filters=[("f", "eq", 0)], groups=["g", "s"], aggs=["v"], op="hist", loghist=True, weight_col="w")
    q.ref = "oracle"
    return sp, t.rows, t.valid, [q]


@pytest.mark.parametrize("name", ["dense-axes", "hashed"])
def test_sparse_past_24_gib(name, monkeypatch, capfd):
    """Refused with sparse group accumulators alone, answered with both settings."""
    build = _dense_axes_weighted if name == "dense-axes" else (lambda: _hashed_weighted((1 << 17) + 1000))
    spec, rows, valid, queries = _table(name, build)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    table = _staged(spec)
    try:
        for i, q in enumerate(queries):
            assert _status(lambda: run_gpu(spec, flags(q, False, True), table)) == F.SG_ERR_UNSUPPORTED, (name, i)
            assert _status(lambda: run_gpu(spec, flags(q, True, False), table)) == F.SG_ERR_UNSUPPORTED, (name, i)
            capfd.readouterr()
            g = run_gpu(spec, flags(q, True, True), table)
            plans, folds, found = _traces(capfd)
            assert " sparse=1 " in plans[0] and plans[0].endswith(" fold=1"), plans
            live = int(re.search(r"live=(\d+)", found[0]).group(1))
            assert _canon(folds[0]) == g.NumGroups < live, (folds, g.NumGroups, live)
            check_sparse(spec, rows, valid, q, g, (name, i))
    finally:
        table.close()


# ---- 4. refusals that stay --------------------------------------------------------------------------------------
def test_rows_without_weights_stay_refused(monkeypatch):
    """weight_carry = 0 over rows without the weight column: today's refusal on hashed and sparse plans with the
    setting on; the next query on the context answers."""
    spec, rows, valid = _table(("wc", "mixed"), lambda: WC.table("mixed"))
    table = _staged(spec)
    try:
        for _, env, fl in MODES[1:]:
            for k, v in env.items():
                monkeypatch.setenv(k, v)
            q = flags(WC.queries(spec)[0], **fl)
            q.carry = False
            assert _status(lambda: run_gpu(spec, q, table)) == F.SG_ERR_UNSUPPORTED, env
            assert "rows without the weight column" in table.ctx.err(), env
            q.carry = True
            rowref.check(rowref.run(spec, rows, valid, q), run_gpu(spec, q, table), q, where=("after", env))
            for k in env:
                monkeypatch.delenv(k)
    finally:
        table.close()


def test_table_filled_by_canonical_inserts(monkeypatch):
    """A 16-entry table (SG_HASH_CAP_LOG2=4) holds the scan's 10 (s, weight) entries; their 7 canonical keys do not
    fit.  Refused, and the same query answers with a table of the usual size."""
    t = edges._Table(None, [("s", STR), ("w", INT), ("v", INT)])
    strs = ["s%d" % i for i in range(7)]
    t.add({"s": strs + strs[:3], "w": [1] * 7 + [2] * 3, "v": list(range(10))})
    t.extents(v=(0, 10))
    spec = t.spec
    q = flags(Q(spec, groups=["s"], aggs=["v"], op="avg", weight_col="w"))
    table = _staged(spec)
    monkeypatch.setenv("SG_FORCE_HASHED_SLOTS", "1")
    try:
        monkeypatch.setenv("SG_HASH_CAP_LOG2", "4")
        assert _status(lambda: run_gpu(spec, q, table)) == F.SG_ERR_UNSUPPORTED
        assert "filled up" in table.ctx.err()
        monkeypatch.delenv("SG_HASH_CAP_LOG2")
        rowref.check(rowref.run(spec, t.rows, t.valid, q), run_gpu(spec, q, table), q, where="after")
    finally:
        table.close()


def test_setter_values():
    spec, rows, valid = _table(("wc", "codes"), lambda: WC.table("codes"))
    table = _staged(spec)
    try:
        q = WC.queries(spec)[0]
        d, keep = q.desc()
        lib, ctx = table.lib, table.ctx
        h = lib.sg_query_begin(ctx.h, table.h, C.byref(d))
        assert h
        try:
            for bad in (2, -1, 1 << 30):
                assert lib.sg_query_set_hashed_folds(h, bad) == F.SG_ERR_INVALID
            assert lib.sg_query_set_hashed_folds(h, 1) == F.SG_OK
            assert lib.sg_query_run(h) == F.SG_OK  # (a dense plan: folded on the host as with 0)
            assert lib.sg_query_set_hashed_folds(h, 0) == F.SG_OK
            assert lib.sg_query_run(h) == F.SG_OK
        finally:
            lib.sg_query_free(h)
    finally:
        table.close()


# ---- 5. read-back and launches ---------------------------------------------------------------------------------
def test_read_back_and_launches(monkeypatch, capfd):
    """d2h_bytes: the scalars and the L' canonical groups' accumulator rows, keys and rows; nothing sized by the
    table or the (group, weight) entries.  Launches: the discovery scan, the canonical insert, two id passes
    (canonical entries first), the MAX region's fill, the aggregation scan and the fold."""
    spec, rows, valid, queries = _table("dense-axes", _dense_axes_weighted)
    q = flags(queries[0], True, True)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    capfd.readouterr()
    g = run_gpu(spec, q)
    _, folds, found = _traces(capfd)
    canon = _canon(folds[0])
    assert canon == g.NumGroups < int(re.search(r"live=(\d+)", found[0]).group(1))
    row_words = 1 + 3 * len(q.aggs) + 1002 * len(q.aggs)
    bound = 16 * 8 + canon * (row_words * 8 + 4 + 8) + 1024
    assert g.stats.d2h_bytes <= bound, (g.stats.d2h_bytes, bound, canon)
    assert g.stats.kernel_launches == 7, g.stats.kernel_launches


# ---- 6. prepared and streaming runs ----------------------------------------------------------------------------
def test_prepared_sparse_rerun_with_new_keys_and_weights(monkeypatch):
    """A prepared weighted sparse query re-runs; blocks with new keys and new weight values (a larger weight axis)
    are staged, and it runs again."""
    t = edges._Table(None, KT3)
    rng = np.random.default_rng(94)
    g, s = edges._strs("a", 300), edges._strs("b", 200)
    t.add({"g": g[rng.integers(0, 300, 3000)], "s": s[rng.integers(0, 200, 3000)], "w": rng.choice(WEIGHTS, 3000),
           "v": rng.integers(0, 1000, 3000)})
    t.extents(v=(0, 1000))
    spec = t.spec
    q = flags(Q(spec, groups=["g", "s"], aggs=["v"], op="hist", weight_col="w"), True, True)
    monkeypatch.setenv("SG_FORCE_SPARSE_GROUPS", "1")
    table = _staged(spec)
    try:
        pq = table.Prepare(None, q.query_spec())
        try:
            for step in range(2):
                ref = rowref.run(spec, t.rows, t.valid, q)
                for rerun in range(2):
                    qs = q.query_spec()
                    pq.Run(qs)
                    rowref.check(ref, qs, q, where=("prepared", step, rerun))
                before = len(spec.blocks)
                n = 500
                t.add({"g": np.array(["new%d_%d" % (step, x) for x in rng.integers(0, 30, n)]),
                       "s": s[rng.integers(0, 200, n)], "w": rng.integers(100, 140, n), "v": rng.integers(0, 1000, n)})
                for b in spec.blocks[before:]:
                    table.add_block(b)
        finally:
            pq.Close()
    finally:
        table.close()


def test_streaming_forced_hashed(monkeypatch):
    """sg_query_submit_block + sg_query_finish over a forced-hashed weighted query: the fold runs in finish."""
    spec, rows, valid = _table(("wc", "mixed"), lambda: WC.table("mixed"))
    monkeypatch.setenv("SG_FORCE_HASHED_SLOTS", "1")
    for q in WC.queries(spec)[:4]:
        ref = rowref.run(spec, rows, valid, q)
        t = E.Table("stream", spec.key_table)
        t.IntInfo = dict(spec.IntInfo)
        try:
            qs = q.query_spec()
            d, keep = E.make_query_desc(spec.KeyTable, spec.KeyTypes, spec.IntInfo, qs)
            qh = t.lib.sg_query_begin(t.ctx.h, t.h, C.byref(d))
            assert qh
            try:
                t.ctx.check(t.lib.sg_query_set_hashed_folds(qh, 1))
                for b in spec.blocks:
                    bd = b.desc()
                    t.ctx.check(t.lib.sg_query_submit_block(qh, C.byref(bd)))
                rp = C.c_void_p()
                t.ctx.check(t.lib.sg_query_finish(qh, C.byref(rp)))
                t._fill(qs, rp)
                t.lib.sg_result_free(rp)
            finally:
                t.lib.sg_query_free(qh)
            rowref.check(ref, qs, q, where="streaming")
        finally:
            t.close()
