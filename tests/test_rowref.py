"""The oracle (oracle/oracle.cpp) and its Python restatement (oracle/pyoracle.py) against the row-level reference
tests/rowref.py on the edge tables of tests/edges.py.  No GPU: this pins the oracle itself at the values where
the scan kernel branches, so a misreading the oracle shares with the kernel cannot pass the GPU parity tests."""
import numpy as np
import pytest

from tests import edges, rowref
from tests.test_oracle_vs_py import py_query
from tests.util import run_oracle

TABLES = edges.all_tables()
SMALL = 30000  # rows: pyoracle's per-row loops are run on tables up to this size


class _Py:
    """pyoracle's tuple result in the shape rowref.check reads."""

    def __init__(self, spec, q):
        self.Results, self.TimeResults, self.Cumulative, self.MatchedCount, _ = py_query(spec, q)


def _nrows(rows):
    return sum(len(next(iter(cols.values()))) for cols, _, _ in rows)


@pytest.mark.parametrize("name", [n for n, _ in TABLES])
def test_oracle_matches_rowref(name):
    spec, rows, valid, queries = dict(TABLES)[name]
    for i, q in enumerate(queries):
        ref = rowref.run(spec, rows, valid, q)
        # (the C++ oracle keeps one of "" and missing, as the reference does: edges.family_g_str; pyoracle merges)
        if getattr(q, "oracle", True):
            o = run_oracle(spec, q)
            assert o.SkippedBlocks == ref.SkippedBlocks, (name, i, "skipped blocks")
            assert o.BrokenBlocks == 0
            # the oracle orders by its float running mean (DESIGN.md §7): the order is compared for Count only
            rowref.check(ref, o, q, where=(name, i, "oracle"), order=q.order_by == "$COUNT")
        if _nrows(rows) <= SMALL and getattr(q, "pyoracle", True):
            rowref.check(ref, _Py(spec, q), q, where=(name, i, "pyoracle"))


def test_edges_reach_their_values():
    """The tables hold what their families claim: a sum beyond int64, values outside the extents on both sides,
    values next to 2^32, negative and >= 2^32 times."""
    t = dict(TABLES)
    spec, rows, valid, qs = t["F"]
    assert rowref.wrapped(rowref.run(spec, rows, valid, qs[0]))
    spec, rows, valid, qs = t["A"]
    r = rowref.run(spec, rows, valid, qs[0])
    assert not rowref.wrapped(r)
    for a, (lo, hi) in zip(qs[0].aggs, edges.A_EXTENTS):
        vals = set(int(x) for cols, _, _ in rows for x in cols[a])
        assert {lo - 1, hi + 1} <= vals, a
    times = set(int(x) for d in ("D0", "D1", "D2") for cols, _, _ in t[d][1] for x in cols["t"])
    assert min(times) < -(1 << 32) and max(times) >= 1 << 32 and 0 in times


def test_c_tables_hold_every_boundary():
    """Every bucket size's column holds lo + k*bs - 1 / + 0 / + 1 for every slot k, the last slot and the values
    past the extents (10*Max and 10*Max + 1 included)."""
    spec, rows, valid, qs = dict(TABLES)["C0"]
    for i, bs in enumerate(edges.C_SIZES):
        lo, hi = spec.IntInfo["v%d" % i]
        have = set(int(x) for cols, _, _ in rows for x in cols["v%d" % i])
        assert set(edges.c_values(lo, hi, bs)) <= have, bs
        assert {lo + (rowref.basic_layout(lo, hi, 0)[1] - 1) * bs, hi + 1} <= have, bs
    lo, hi = spec.IntInfo["v6"]
    assert lo == 0 and {(1 << 32) - 2, (1 << 32) - 1} <= set(int(x) for cols, _, _ in rows for x in cols["v6"])


def test_e_tables_end_value_arrays_mid_tile():
    """The value-array pass of family E stores v0 and v8 as value arrays whose length ends at a tile edge +-1,
    short of NumRecords where E_END says so; v8 stays inside the 32-bit range."""
    from sybil_b200 import _ffi as F
    spec, rows, valid, qs = dict(TABLES)["E"]
    got = {}
    for b in spec.blocks:
        for c in b.cols:
            name = spec.key_table[c.col_slot][0]
            if name in ("v0", "v8") and c.encoding == F.SG_ENC_VALUES:
                got.setdefault(name, set()).add((b.num_records, len(c.values_i64)))
    want = {(n, e) for n, e in edges.E_END.items() if n >= 31}
    assert want <= got["v0"] and want <= got["v8"]
    assert any(e < n for n, e in want)
    v8 = [int(x) for cols, _, _ in rows for x in cols["v8"]]
    assert (1 << 32) - (1 << 20) < min(v8) and max(v8) < 1 << 32


def test_key_tables_hold_their_keys():
    """Family G holds every key of G_KEYS next to missing rows, in bucket-encoded and value-array blocks, and its
    value arrays have gaps and rows past len(Values); G-str holds "" next to missing rows in both encodings."""
    from sybil_b200 import _ffi as F
    t = dict(TABLES)
    spec, rows, valid, qs = t["G-mixed"]
    slot = spec.KeyTable["k"]
    encs = {c.encoding for b in spec.blocks for c in b.cols if c.col_slot == slot}
    assert encs == {F.SG_ENC_BUCKET, F.SG_ENC_VALUES}
    for (cols, _, _), va in zip(rows, valid):
        held = set(int(x) for x in cols["k"][va["k"]])
        assert set(edges.G_KEYS) <= held and not va["k"].all()
    assert any(len(c.values_i64) < b.num_records for b in spec.blocks for c in b.cols
               if c.col_slot == slot and c.encoding == F.SG_ENC_VALUES)
    spec, rows, valid, qs = t["G-str"]
    slot = spec.KeyTable["s"]
    assert {c.encoding for b in spec.blocks for c in b.cols if c.col_slot == slot} == {F.SG_ENC_BUCKET,
                                                                                       F.SG_ENC_VALUES}
    for (cols, _, _), va in zip(rows, valid):
        assert "" in set(cols["s"][va["s"]]) and not va["s"].all()
    # merged, -1 and the missing rows are the largest group: first under the top-K queries
    spec, rows, valid, qs = t["G-int"]
    r = rowref.run(spec, rows, valid, qs[0])
    assert max(r.Results, key=lambda k: r.Results[k].Count) == "\t"


def test_k_and_i_tables_reach_their_boundaries():
    """Family K's k / f blocks are bucket-encoded with 1,023 / 1,024 / 1,025 bins; family I's ceiling table puts
    keys on the last entries of the 2^16-entry hashed table and on its first ones, so probe chains wrap."""
    from sybil_b200 import _ffi as F
    spec, rows, valid, qs = dict(TABLES)["K"]
    for name in ("k", "f"):
        bins = [len(c.bin_values) for b in spec.blocks for c in b.cols
                if c.col_slot == spec.KeyTable[name] and c.encoding == F.SG_ENC_BUCKET]
        assert bins == edges.K_BINS, name
    spec, rows, valid, qs = dict(TABLES)["I-ceiling"]
    radix = edges.I_CEIL[0] + 2
    h = edges.slot_hash([(a + 1) + (b + 1) * radix + 1 for a, b in qs[0].wraps]) & 0xFFFF
    assert (h >= 0xFFFD).sum() >= 10 and (h <= 1).sum() >= 10


def test_rowref_set_filters_match_pyoracle():
    """rowref's SetFilter against pyoracle's on random set columns, both encodings of the set column."""
    from tests.util import INT, SET, Q, Spec
    for threshold in (5000, 4):
        rng = np.random.default_rng(threshold)
        n = 1500
        tags = [["t%d" % v for v in rng.choice(9, int(k), replace=False)] for k in rng.integers(0, 4, n)]
        va = {"tags": rng.random(n) > 0.1, "age": np.ones(n, bool)}
        s = Spec([("age", INT), ("tags", SET)])
        cols = {"age": rng.integers(10, 30, n), "tags": tags}
        s.add_rows(cols, va, threshold=threshold, block_rows=500)
        rows, valid = [(cols, 500, threshold)], [va]
        for f in ([("tags", "in", "t3")], [("tags", "nin", "t3")], [("tags", "nin", "zz")],
                  [("tags", "in", "t1"), ("tags", "nin", "t2")]):
            q = Q(s, set_filters=f, groups=["age"], aggs=[], op="avg")
            ref = rowref.run(s, rows, valid, q)
            rowref.check(ref, _Py(s, q), q, where=(threshold, f))
            rowref.check(ref, run_oracle(s, q), q, where=(threshold, f, "oracle"))


def test_rowref_rules():
    """The hand-restated rules at a few points worked out from the Go sources."""
    assert rowref.tdiv(-1999, 1000) == -1 and rowref.tdiv(1999, 1000) == 1 and rowref.tdiv(-999, 1000) == 0
    assert rowref.i64(10 * (1 << 62)) == rowref.I64_MIN
    assert rowref.rejects(-50, -1000, -10)  # 10 * Max = -100 < -50
    assert not rowref.rejects(-100, -1000, -10)
    assert rowref.basic_layout(0, 50, 0) == (1, 52)
    assert rowref.basic_layout(0, 990, 0) == (9, 112)
    assert rowref.basic_layout(0, 23470, 0) == (23, 1002)  # the reference's golden layout
    assert rowref.basic_layout(0, 10 ** 6, 7) == (7, 1002)
    subs = rowref.multi_layout(0, 1 << 20)
    assert subs[0] == ((1 << 19), 1 << 20) and subs[-1][0] == 0 and len(subs) == 12
