"""Sparse group accumulators on the GPU (sg_query_set_sparse_groups, engine.FLAGS.SPARSE_GROUPS): group-by
histograms past the 24 GiB accumulator limit, dense and hashed, answer with the flag on and are refused with it
off; existing key and order families run through the sparse path (SG_FORCE_SPARSE_GROUPS) and give what the
row-level reference gives.  Tables: tests/family_sparse.py and tests/edges.py."""
import ctypes as C
import re

import numpy as np
import pytest

from sybil_b200 import _ffi as F
from sybil_b200 import engine as E
from tests import edges, family_sparse as FS, rowref
from tests.test_parity_edges import _mean_comparable
from tests.util import compare, compare_group, run_gpu, run_oracle

pytestmark = pytest.mark.gpu

_TABLES = {}


def _table(name, build):
    if name not in _TABLES:
        _TABLES[name] = build()
    return _TABLES[name]


@pytest.fixture(autouse=True)
def _reset_flags():
    """engine.FLAGS is process-wide: no test of another module may inherit SPARSE_GROUPS from one of these."""
    yield
    E.FLAGS.reset()


def sparse(q, on=True):
    """q with engine.FLAGS.SPARSE_GROUPS set whenever it builds its QuerySpec (Q.set_flags resets the flags)."""
    base = type(q).set_flags

    def set_flags():
        base(q)
        E.FLAGS.SPARSE_GROUPS = on
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


def _plan_lines(capfd):
    err = capfd.readouterr().err
    return ([ln for ln in err.splitlines() if ln.startswith("sg_plan:")],
            [ln for ln in err.splitlines() if ln.startswith("sg_sparse:")])


def _check(spec, rows, valid, q, g, where):
    assert g.BrokenBlocks == 0, where
    if getattr(q, "ref", "rowref") == "rowref":
        rowref.check(rowref.run(spec, rows, valid, q), g, q, where=where)
        return
    o = run_oracle(spec, q, nthreads=8)
    if q.order_by in ("$COUNT", ""):
        compare(g, o, q, mean=_mean_comparable)
        return
    # ordered by a mean: the oracle's order is its float running mean, so the expected list is made here from its
    # exact sums (descending, ties by the rendered key), and every group is compared with the oracle's
    ai = q.aggs.index(q.order_by)

    def mean(r):
        h = r.Hists.get(q.aggs[ai])
        return float(h.ExactSum) / float(h.Count) if h is not None and h.Count else float("-inf")
    want = sorted(o.Results.values(), key=lambda r: (-mean(r), r.GroupByKey.encode("utf-8", "surrogateescape")))
    want = want[:q.limit] if q.limit else want
    assert g.NumGroups == len(o.Results) and g.MatchedCount == o.MatchedCount, where
    assert [r.GroupByKey for r in g.Sorted] == [r.GroupByKey for r in want], where
    for r in g.Sorted:
        compare_group(r, o.Results[r.GroupByKey], q.aggs, q.op == "hist", (where, r.GroupByKey), q.loghist,
                      _mean_comparable)


def _run_family(name, build, monkeypatch, capfd, variant=16):
    """Every query: refused without the flag, answered with it on the sparse path, checked against its reference."""
    spec, rows, valid, queries = _table(name, build)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    table = _staged(spec)
    try:
        for i, q in enumerate(queries):
            where = (name, variant, i)
            sparse(q, False)
            assert _status(lambda: run_gpu(spec, q, table)) == F.SG_ERR_UNSUPPORTED, where
            sparse(q)
            capfd.readouterr()
            g = run_gpu(spec, q, table)
            plans, found = _plan_lines(capfd)
            assert len(plans) == 1 and re.search(r"hashed=1 .* sparse=1 live=\d+ ", plans[0]), (where, plans)
            assert plans[0].startswith("sg_plan: build=w%d " % variant), (where, plans)
            live = int(re.search(r"live=(\d+)", plans[0]).group(1))
            assert len(found) == 1 and ("live=%d " % live) in found[0], (where, found)
            assert g.stats.kernel_launches >= 3, where  # discovery, ids, aggregation
            _check(spec, rows, valid, q, g, where)
            if not q.time_col and not q.int_filters and not q.str_filters:
                assert g.NumGroups == live, (where, g.NumGroups, live)
    finally:
        table.close()


def test_dense_hist_over_the_2p26_slots(monkeypatch, capfd):
    """edges.i_dense_hist (1,002 counters on each of 2^26 dense slots) is refused without the flag and answers
    with it; the context keeps answering between the two."""
    spec, rows, valid, queries = edges.family_i_dense(False)
    table = _staged(spec)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    try:
        for loghist in (False, True):
            q = edges.i_dense_hist(spec)
            q.loghist = loghist  # (op hist: bucket counters of a MultiHist)
            ref = rowref.run(spec, rows, valid, q)
            assert _status(lambda: run_gpu(spec, sparse(q, False), table)) == F.SG_ERR_UNSUPPORTED
            capfd.readouterr()
            g = run_gpu(spec, sparse(q), table)
            plans, _ = _plan_lines(capfd)
            assert re.search(r"sparse=1 live=%d table=65536\b" % len(ref.Results), plans[0]), plans
            rowref.check(ref, g, q, where=("i_dense_hist", loghist))
            assert _status(lambda: run_gpu(spec, sparse(q, False), table)) == F.SG_ERR_UNSUPPORTED
            plain = queries[-1]
            rowref.check(rowref.run(spec, rows, valid, plain), run_gpu(spec, plain, table), plain, where="after")
    finally:
        table.close()


@pytest.mark.parametrize("variant", [8, 16])
def test_dense_str_axes(variant, monkeypatch, capfd):
    _run_family("dense", FS.family_dense_axes, monkeypatch, capfd, variant)


def test_time_mode(monkeypatch, capfd):
    _run_family("time", FS.family_time, monkeypatch, capfd)


@pytest.mark.parametrize("rows,loghist", [((1 << 20) + 1000, False), ((1 << 17) + 1000, True)])
def test_hashed_past_the_limit(rows, loghist, monkeypatch, capfd):
    """Key products past 2^26 whose table (2 x the listed rows) would carry 24 GiB of histograms; checked against
    the oracle, with int and str filters and order by a mean with a limit."""
    _run_family("hashed-%d" % rows, lambda: FS.family_hashed(rows, loghist), monkeypatch, capfd)


# ---- existing families through the sparse path ---------------------------------------------------------------
_REF = {}


@pytest.mark.parametrize("name,forms,variant", [(n, f, v) for n in ("G-int", "G-mixed", "G-str", "H", "K")
                                                for f in ("narrow", "wide") for v in (8, 16)] +
                         [("L-small", None, 8), ("L-small", None, 16), ("L-large", None, 16)])
def test_forced_sparse(name, forms, variant, monkeypatch, capfd):
    """SG_FORCE_SPARSE_GROUPS=1 takes the sparse path for any plan while the flag is set: what it gives must be
    what the row-level reference gives (weighted and StrReplace queries are refused on that path)."""
    build = edges.KEY_TABLES.get(name) or edges.ORDER_TABLES[name]
    spec, rows, valid, queries = _table((name, forms), lambda: build(forms))
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    monkeypatch.setenv("SG_FORCE_SPARSE_GROUPS", "1")
    table = _staged(spec)
    try:
        for i, q in enumerate(queries):
            if q.weight_col or q.str_replace:
                continue
            where = (name, forms, variant, i)
            capfd.readouterr()
            g = run_gpu(spec, sparse(q), table)
            plans, found = _plan_lines(capfd)
            assert plans and all(" sparse=1 " in ln for ln in plans), (where, plans)
            assert all(ln.startswith("sg_plan: build=w%d " % variant) for ln in plans), (where, plans)
            if (name, forms, i) not in _REF:
                _REF[name, forms, i] = rowref.run(spec, rows, valid, q)
            rowref.check(_REF[name, forms, i], g, q, where=where)
            if not q.time_col:
                assert g.NumGroups == int(re.search(r"live=(\d+)", found[-1]).group(1)), where
    finally:
        table.close()


def test_forced_sparse_refuses_weights_and_str_replace(monkeypatch):
    spec, rows, valid, queries = _table(("R", None), edges.family_r)
    monkeypatch.setenv("SG_FORCE_SPARSE_GROUPS", "1")
    table = _staged(spec)
    try:
        picked = [q for q in queries if q.weight_col][:1] + [q for q in queries if q.str_replace and not q.weight_col][:1]
        assert len(picked) == 2
        for q in picked:
            assert _status(lambda: run_gpu(spec, sparse(q), table)) == F.SG_ERR_UNSUPPORTED
            rowref.check(rowref.run(spec, rows, valid, q), run_gpu(spec, sparse(q, False), table), q, where="flag off")
    finally:
        table.close()


# ---- prepared queries, broken blocks ---------------------------------------------------------------------------
def test_prepared_query_rediscovers_new_keys(monkeypatch, capfd):
    """A prepared sparse query run twice over an unchanged table (the plan is reused, discovery runs again and the
    accumulators are laid out again for the same live groups), then again after blocks with new keys are staged:
    discovery runs again and the new groups appear."""
    t = edges._Table(None, FS.KT)
    rng = np.random.default_rng(75)
    g, s = edges._strs("a", 2000), edges._strs("b", 1700)
    t.add({"g": np.resize(g, 1700), "s": s, "v": rng.integers(0, 1000, 1700)})
    t.add({"g": g[1700:], "s": s[:300], "v": rng.integers(0, 1000, 300)})
    t.extents(v=(0, 1000))
    spec = t.spec
    q = sparse(edges._q(spec, groups=["g", "s"], aggs=["v"], op="hist"))
    table = _staged(spec)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    try:
        pq = table.Prepare(None, q.query_spec())
        try:
            for step in range(3):
                ref = rowref.run(spec, t.rows, t.valid, q)
                for rerun in range(2):
                    qs = q.query_spec()
                    capfd.readouterr()
                    pq.Run(qs)
                    _, found = _plan_lines(capfd)
                    assert len(found) == 1 and "live=%d " % len(ref.Results) in found[0], (step, rerun, found)
                    assert qs.NumGroups == len(ref.Results), (step, rerun)
                    rowref.check(ref, qs, q, where=("prepared", step, rerun))
                before = len(spec.blocks)
                n = 500
                t.add({"g": np.array(["new%d_%d" % (step, x) for x in rng.integers(0, 30, n)]),
                       "s": s[rng.integers(0, 1700, n)], "v": rng.integers(0, 1000, n)})
                for b in spec.blocks[before:]:
                    table.add_block(b)
        finally:
            pq.Close()
    finally:
        table.close()


def test_broken_block_keys_are_not_groups(monkeypatch, capfd):
    """The scan finds the broken block in the discovery launch, which puts its keys into the table and numbers them;
    the aggregation launch reports the block, and the query runs again without it: the second discovery's live
    groups exclude the block's keys, and none of them is a group."""
    spec, rows, valid, queries = FS.family_broken()
    q = sparse(queries[0])
    monkeypatch.setenv("SG_FORCE_SPARSE_GROUPS", "1")
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    capfd.readouterr()
    g = run_gpu(spec, q)
    plans, found = _plan_lines(capfd)
    o = run_oracle(spec, q)
    assert g.BrokenBlocks == 1
    lives = [int(re.search(r"live=(\d+)", ln).group(1)) for ln in found]
    assert len(lives) == 2 and len(plans) == 2, (found, plans)
    # the first discovery saw the broken block's keys, the second did not
    assert lives[0] > lives[1] == g.NumGroups == len(o.Results), (lives, g.NumGroups, len(o.Results))
    assert not [k for k in g.Results if k.startswith("b1_")]
    assert {k.split("_")[0] for k in g.Results} == {"b0", "b2"}
    compare(g, o, q, mean=_mean_comparable)


# ---- refusals, setter, read-back ---------------------------------------------------------------------------------
def test_live_groups_past_the_budget_are_refused(monkeypatch, capfd):
    """SG_SPARSE_BUDGET_MIB lowers the 24 GiB budget for the live groups' accumulators: past it the query is
    refused with a message naming the live groups, and the same query answers once the budget fits."""
    spec, rows, valid, queries = _table("dense", FS.family_dense_axes)
    q = sparse(queries[0])
    ref = rowref.run(spec, rows, valid, q)
    live = len(ref.Results)
    per_group = (1 + 3 + 1002) * 8
    table = _staged(spec)
    try:
        monkeypatch.setenv("SG_SPARSE_BUDGET_MIB", str(max(1, live * per_group // (2 << 20))))
        assert _status(lambda: run_gpu(spec, q, table)) == F.SG_ERR_UNSUPPORTED
        assert ("for %d live groups" % live).encode() in table.lib.sg_last_error(table.ctx.h)
        monkeypatch.setenv("SG_SPARSE_BUDGET_MIB", str(live * per_group // (1 << 20) + 2))
        rowref.check(ref, run_gpu(spec, q, table), q, where="within the budget")
    finally:
        table.close()


def test_setter_values_and_streaming_path():
    spec, rows, valid, queries = _table("dense", FS.family_dense_axes)
    table = _staged(spec)
    try:
        q = queries[0]
        d, keep = q.desc()
        lib, ctx = table.lib, table.ctx
        h = lib.sg_query_begin(ctx.h, table.h, C.byref(d))
        assert h
        try:
            for bad in (2, -1, 1 << 30):
                assert lib.sg_query_set_sparse_groups(h, bad) == F.SG_ERR_INVALID
            assert lib.sg_query_run(h) == F.SG_ERR_UNSUPPORTED  # still 0: past 24 GiB
            assert lib.sg_query_set_sparse_groups(h, 1) == F.SG_OK
            assert lib.sg_query_submit_block(h, C.byref(spec.blocks[0].desc())) == F.SG_ERR_UNSUPPORTED
            assert lib.sg_query_run(h) == F.SG_OK
            assert lib.sg_query_set_sparse_groups(h, 0) == F.SG_OK
            assert lib.sg_query_run(h) == F.SG_ERR_UNSUPPORTED
        finally:
            lib.sg_query_free(h)
    finally:
        table.close()


@pytest.mark.parametrize("name", ["dense", "hashed-1049576"])
def test_read_back_is_bounded_by_the_live_groups(name, monkeypatch, capfd):
    """d2h_bytes: the scalars, L rows of the accumulators, the L-entry id -> key array and the discovery's
    scalars and live count; nothing sized by the table or the dense space."""
    build = FS.family_dense_axes if name == "dense" else (lambda: FS.family_hashed((1 << 20) + 1000, False))
    spec, rows, valid, queries = _table(name, build)
    q = sparse(queries[0])
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    capfd.readouterr()
    g = run_gpu(spec, q)
    _, found = _plan_lines(capfd)
    live = int(re.search(r"live=(\d+)", found[0]).group(1))
    row_words = 1 + 3 * len(q.aggs) + 1002 * len(q.aggs)
    bound = 16 * 8 + live * (row_words * 8 + 4) + 64 + 8 + 1024
    assert g.NumGroups == live
    assert g.stats.d2h_bytes <= bound, (g.stats.d2h_bytes, bound, live)
    # the scan twice (discovery, aggregation), the id kernel, and the MAX region's fill
    assert g.stats.kernel_launches == 4, g.stats.kernel_launches
