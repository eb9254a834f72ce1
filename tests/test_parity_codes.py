"""Bucket columns of at most 255 bins read through per-row codes (COL_CODES, DESIGN.md §4) on the GPU.  Every query
is checked against the row-level reference tests/rowref.py and the oracle, and against the same run staged with
SG_NO_CODES=1 (every column walked through its ids), field for field and bit for bit.  SG_PLAN_TRACE's `codes=`
shows how many plan columns had codes.  Columns that must keep their ids (a row listed twice, a row >= NumRecords,
a gap >= 65,536) are built by editing the encoded blocks; they are compared with the oracle and the ids-only run."""
import re

import numpy as np
import pytest

from sybil_b200 import engine as E
from tests import edges, rowref
from tests.test_parity_edges import _mean_comparable
from tests.util import INT, SET, STR, compare, run_gpu, run_oracle

pytestmark = pytest.mark.gpu

KT_CODES = [("s", STR), ("s2", STR), ("k", INT), ("b1", INT), ("b2", INT), ("b254", INT), ("b255", INT),
            ("b256", INT), ("f", INT), ("v", INT), ("t", INT), ("w", INT), ("tags", SET)]
K_VALUES = [-1, 0, 5, -7, (1 << 32) + 3, 1 << 40, 123456789, -(1 << 33)]  # -1 renders as missing; < 0 and > 2^32
SIZES = [65536, 65536, 40001]  # the last block partial, NumRecords not a multiple of 16


def _rows(rng, n, sprefix="s"):
    s = np.array(["%s%d" % (sprefix, x) for x in rng.integers(0, 16, n)])
    s[rng.random(n) < 0.02] = ""  # "" groups with the missing rows
    tags = [["a", "b", "c"][: int(x)] for x in rng.integers(0, 4, n)]
    cols = {"s": s, "s2": np.array(["x%d" % x for x in rng.integers(0, 12, n)]),
            "k": np.array(K_VALUES, np.int64)[rng.integers(0, len(K_VALUES), n)],
            "b1": np.full(n, 7), "b2": rng.integers(0, 2, n) * 1000, "b254": rng.integers(0, 254, n) - 100,
            "b255": rng.integers(0, 255, n), "b256": rng.integers(0, 256, n), "f": rng.integers(0, 1000, n),
            "v": rng.integers(-50, 1 << 20, n), "t": rng.integers(0, 40, n) * 3600, "w": rng.integers(-3, 10, n),
            "tags": tags}
    # partial columns: unlisted rows read code 0xFF
    valid = {"k": rng.random(n) > 0.05, "s2": rng.random(n) > 0.1}
    return cols, valid


_TABLES = {}


def _codes_table(forms):
    if forms not in _TABLES:
        t = edges._Table(forms, KT_CODES)
        rng = np.random.default_rng(41)
        for n in SIZES:
            cols, valid = _rows(rng, n)
            t.add(cols, valid)
        _TABLES[forms] = t.done(_queries(t.spec))
    return _TABLES[forms]


def _no_oracle(q):
    q.oracle = False  # weighted: the reference drops a block result whose weighted Count is 0 (DESIGN.md §7)
    return q


def _queries(s):
    q = edges._q
    return [
        # count mode (s2 and k are partial): int and str filters of every op, first and second group with aliases
        q(s, int_filters=[("b255", "gt", 100), ("b254", "lt", 120)], str_filters=[("s2", "neq", "x3")],
          groups=["s", "k"], aggs=["v"], op="hist", expect=[r"fail_mode=0 ", r"codes=5\b"]),
        q(s, int_filters=[("k", "eq", 5), ("b2", "neq", 0)], str_filters=[("s2", "re", "^x1")], groups=["k", "s2"],
          aggs=["v"], op="avg", expect=[r"codes=5\b"]),
        # fail mode over full code columns, next to a 1,000-bin push-down filter and value arrays (the bench shape)
        q(s, int_filters=[("f", "gt", 100), ("v", "lt", 900000)], str_filters=[("s", "neq", "s3")], groups=["s", "b2"],
          aggs=["v"], op="hist", expect=[r"fail_mode=1 ", r"codes=3\b"]),
        q(s, int_filters=[("b255", "eq", 3), ("b254", "neq", 0), ("b1", "lt", 8)], str_filters=[("s", "nre", "^s1")],
          groups=["b254"], aggs=["v"], op="avg", expect=[r"fail_mode=1 ", r"codes=5\b"]),
        q(s, int_filters=[("b255", "lt", 200), ("b1", "eq", 7)], str_filters=[("s", "eq", "s4")], groups=["b255"],
          aggs=["v"], op="avg", expect=[r"fail_mode=1 ", r"codes=4\b"]),
        # 1 / 2 / 254 / 255 bins read through codes, 256 through ids
        q(s, groups=["b1", "b255"], aggs=["v"], op="avg", expect=[r"codes=2\b"]),
        q(s, groups=["b256"], aggs=["v"], op="avg", expect=[r"codes=0\b"]),
        q(s, str_filters=[("s", "eq", "s5")], groups=["b256", "b2"], aggs=["v"], op="hist", expect=[r"codes=2\b"]),
        # the aggregation column itself through codes: values below 0 and above 2^32, avg / hist / loghist
        q(s, groups=["s2"], aggs=["k"], op="avg", expect=[r"codes=2\b"]),
        q(s, int_filters=[("b256", "gt", 17)], groups=["b2"], aggs=["k", "v"], op="hist", expect=[r"codes=2\b"]),
        q(s, groups=["s"], aggs=["k"], op="hist", loghist=True, expect=[r"codes=2\b"]),
        # a bucket-encoded time column
        q(s, groups=["s2"], aggs=["v"], op="avg", time_col="t", time_bucket=7200, expect=[r"codes=2\b"]),
        q(s, str_filters=[("s", "neq", "s1")], groups=["b2"], aggs=["v"], op="hist", time_col="t", time_bucket=36000,
          expect=[r"codes=3\b"]),
        # a set filter on another column
        q(s, set_filters=[("tags", "in", "b")], groups=["s", "b255"], aggs=["v"], op="avg", expect=[r"codes=2\b"]),
        q(s, set_filters=[("tags", "nin", "c")], int_filters=[("b254", "gt", 0)], groups=["s"], aggs=["v"], op="avg",
          expect=[r"codes=2\b"]),
        # weights (a code column) and StrReplace on a code column
        _no_oracle(q(s, groups=["s2"], aggs=["v"], op="hist", weight_col="w", expect=[r"codes=2\b"])),
        q(s, str_filters=[("s", "neq", "zz")], groups=["s"], aggs=["v"], op="avg", str_replace={"s": ("^s1", "q")},
          expect=[r"codes=2\b"]),
    ]


def _hist(gh):
    vals = getattr(gh, "Values", None)
    return (gh.TotalCount(), gh.Sum(), gh.Min(), gh.Max(), repr(gh.Mean()),
            None if vals is None else np.asarray(vals).tolist())


def _fingerprint(g):
    """Everything a result holds, in order: two runs that match here match bit for bit."""
    def grp(r):
        return (r.GroupByKey, r.Count, r.Samples, sorted((a, _hist(h)) for a, h in r.Hists.items()))
    return (g.MatchedCount, g.NumGroups, g.BrokenBlocks, g.SkippedBlocks, [grp(r) for r in g.Sorted],
            sorted((tb, sorted(grp(r) for r in m.values())) for tb, m in g.TimeResults.items()))


def _gpu(spec, q, monkeypatch, capfd, no_codes):
    if no_codes:
        monkeypatch.setenv("SG_NO_CODES", "1")
    else:
        monkeypatch.delenv("SG_NO_CODES", raising=False)
    capfd.readouterr()
    g = run_gpu(spec, q)
    trace = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("sg_plan:")]
    assert trace, "no SG_PLAN_TRACE line"
    return g, trace


_REF, _ORC = {}, {}


def _run(forms, monkeypatch, capfd, variant, env=()):
    spec, rows, valid, queries = _codes_table(forms)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    for k in env:
        monkeypatch.setenv(k, "1")
    for i, q in enumerate(queries):
        if "SG_FORCE_HASHED_SLOTS" in env and (q.weight_col or q.str_replace):
            continue  # (weights and StrReplace over a hashed slot space are refused)
        if i not in _REF:  # (neither depends on the array form, the build or the switches)
            _REF[i] = rowref.run(spec, rows, valid, q)
            _ORC[i] = run_oracle(spec, q) if getattr(q, "oracle", True) else None
        where = (forms, variant, env, i)
        g, trace = _gpu(spec, q, monkeypatch, capfd, False)
        assert g.BrokenBlocks == 0, where
        rowref.check(_REF[i], g, q, where=where)
        if _ORC[i] is not None:
            compare(g, _ORC[i], q, mean=_mean_comparable)
        for pat in q.expect:
            assert any(re.search(pat, ln) for ln in trace), (where, pat, trace)
        ids, trace_ids = _gpu(spec, q, monkeypatch, capfd, True)
        assert all(re.search(r"codes=0\b", ln) for ln in trace_ids), (where, trace_ids)
        assert _fingerprint(g) == _fingerprint(ids), where


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("forms", ["narrow", "wide"])
def test_codes(forms, variant, monkeypatch, capfd):
    _run(forms, monkeypatch, capfd, variant)


@pytest.mark.parametrize("env", [("SG_FORCE_HASHED_SLOTS",), ("SG_FORCE_TAIL_SPLIT",), ("SG_NO_TMA",)])
def test_codes_switches(env, monkeypatch, capfd):
    _run(None, monkeypatch, capfd, 16, env)


@pytest.mark.parametrize("variant", [8, 16])
def test_codes_slot_words(variant, monkeypatch, capfd):
    """Family H's 8-, 16- and 32-bit slot words (up to 255 distinct values per column: every key through codes)."""
    spec, rows, valid, queries = edges.family_h()
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    for i, q in enumerate(queries):
        g, trace = _gpu(spec, q, monkeypatch, capfd, False)
        rowref.check(rowref.run(spec, rows, valid, q), g, q, where=(variant, i))
        for pat in getattr(q, "expect", []):
            assert any(re.search(pat, ln) for ln in trace), (variant, i, pat, trace)
        assert any(not re.search(r"codes=0\b", ln) for ln in trace), (variant, i, trace)
        ids, _ = _gpu(spec, q, monkeypatch, capfd, True)
        assert _fingerprint(g) == _fingerprint(ids), (variant, i)


# ---------------------------------------------------------------------------------------------------------------
# columns that keep their ids: the statistics kernel finds a row listed twice, a row >= NumRecords or a gap of
# 65,536 or more while it builds the codes, and the column is scanned through its ids as before
# ---------------------------------------------------------------------------------------------------------------
def _edited(kind):
    t = edges._Table("wide", KT_CODES)
    rng = np.random.default_rng(43)
    for n in SIZES:
        cols, valid = _rows(rng, n)
        t.add(cols, valid)
    spec = t.spec
    blk = spec.blocks[1]
    col = next(c for c in blk.cols if c.col_slot == spec.KeyTable["b2"])
    ids, offs = col.record_ids.copy(), col.bin_offsets
    if kind == "twice":  # bin 1's first row is also in bin 0 (its own first row is then unlisted)
        ids[offs[1]] = ids[offs[0]]
    elif kind == "past":  # the last row of bin 1 lands at NumRecords
        ids[offs[2] - 1] += blk.num_records - int(np.sum(ids[offs[1]:offs[2]], dtype=np.int64))
    else:  # a gap of 65,536 inside bin 1
        ids[offs[1] + 1] = 65536
    col.record_ids = ids
    return spec


@pytest.mark.parametrize("kind", ["twice", "past", "gap"])
def test_columns_that_keep_their_ids(kind, monkeypatch, capfd):
    spec = _edited(kind)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    for q in (edges._q(spec, int_filters=[("b2", "eq", 1000)], groups=["s"], aggs=["v"], op="avg"),
              edges._q(spec, groups=["b2", "s"], aggs=["v"], op="hist")):
        g, trace = _gpu(spec, q, monkeypatch, capfd, False)
        assert any(re.search(r"codes=2\b", ln) for ln in trace), trace  # b2 has codes in the blocks left alone
        ids, _ = _gpu(spec, q, monkeypatch, capfd, True)
        assert _fingerprint(g) == _fingerprint(ids), kind
        if kind != "twice":  # broken: counted and skipped as the oracle does
            assert g.BrokenBlocks == 1, kind
            compare(g, run_oracle(spec, q), q, mean=_mean_comparable)


def test_restage_and_growing_dictionary(monkeypatch, capfd):
    """Codes are bin indices within a block: blocks that bring new strings and values (the dictionaries grow between
    blocks) keep answering, and a table cleared and staged again answers as before."""
    t = edges._Table(None, KT_CODES)
    rng = np.random.default_rng(47)
    cols, valid = _rows(rng, 65536)
    t.add(cols, valid)
    spec = t.spec
    q = edges._q(spec, str_filters=[("s", "neq", "s2")], groups=["s", "k"], aggs=["v"], op="hist")
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    table = E.Table("t", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    for b in spec.blocks:
        table.add_block(b)
    try:
        rowref.check(rowref.run(spec, t.rows, t.valid, q), run_gpu(spec, q, table), q, where="first block")
        before = len(spec.blocks)
        cols, valid = _rows(rng, 30000, sprefix="n")
        cols["k"] = cols["k"] + 11
        t.add(cols, valid)
        table.IntInfo = dict(spec.IntInfo)
        for b in spec.blocks[before:]:
            table.add_block(b)
        capfd.readouterr()
        g = run_gpu(spec, q, table)
        trace = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("sg_plan:")]
        assert any(re.search(r"codes=3\b", ln) for ln in trace), trace
        ref = rowref.run(spec, t.rows, t.valid, q)
        rowref.check(ref, g, q, where="grown dictionary")
        table.ctx.check(table.lib.sg_table_clear(table.h))
        for b in spec.blocks:
            table.add_block(b)
        rowref.check(ref, run_gpu(spec, q, table), q, where="re-staged")
    finally:
        table.close()
