"""The oracle (oracle/oracle.cpp) and its Python restatement (oracle/pyoracle.py) against the row-level reference
tests/rowref.py on the edge tables of tests/edges.py.  No GPU: this pins the oracle itself at the values where
the scan kernel branches, so a misreading the oracle shares with the kernel cannot pass the GPU parity tests."""
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
        o = run_oracle(spec, q)
        assert o.SkippedBlocks == ref.SkippedBlocks, (name, i, "skipped blocks")
        assert o.BrokenBlocks == 0
        rowref.check(ref, o, q, where=(name, i, "oracle"))
        if _nrows(rows) <= SMALL:
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
