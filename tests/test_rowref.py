"""The oracle (oracle/oracle.cpp) and its Python restatement (oracle/pyoracle.py) against the row-level reference
tests/rowref.py on the edge tables of tests/edges.py.  No GPU: this pins the oracle itself at the values where
the scan kernel branches, so a misreading the oracle shares with the kernel cannot pass the GPU parity tests."""
import numpy as np
import pytest

from tests import edges, family_p, rowref
from tests.test_oracle_vs_py import py_query
from tests.util import run_oracle

TABLES = edges.all_tables() + [(name, build()) for name, build in family_p.P_TABLES.items()]
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
    # StrFilter re / nre (filter.go:199-250): MatchString is an unanchored search on the decoded string
    assert rowref._str_pass("re", "", "^$") and not rowref._str_pass("nre", "", "^$")
    assert rowref._str_pass("re", "", "") and not rowref._str_pass("re", "", ".")
    assert rowref._str_pass("re", "s12", "^s1") and not rowref._str_pass("re", "xs1", "^s1")
    assert rowref._str_pass("re", "s21", "1$") and not rowref._str_pass("re", "s12", "1$")
    assert rowref._str_pass("re", "s33", "^(s3|s33)$") and not rowref._str_pass("re", "s333", "^(s3|s33)$")
    # a row without the column fails re and nre alike, whatever the pattern
    from tests.util import STR, Q, Spec
    s = Spec([("g", STR)])
    cols, va = {"g": np.array(["", "s1", "x", "s1"])}, {"g": np.array([True, True, True, False])}
    s.add_rows(cols, va)
    rows, valid = [(cols, None, 5000)], [va]
    for op, pat, want in (("re", "^$", 1), ("nre", "^$", 2), ("re", "", 3), ("nre", "", 0), ("nre", "zz", 3),
                          ("re", "1$", 1)):
        q = Q(s, str_filters=[("g", op, pat)], groups=["g"])
        assert rowref.run(s, rows, valid, q).MatchedCount == want, (op, pat)


def _global_dict(spec, name):
    """A str column's global dictionary as staging builds it: each block's string table in order, then "" (interned
    for every block's str column, sg_table_add_block)."""
    d = {}
    for b in spec.blocks:
        for c in b.cols:
            if c.col_slot == spec.KeyTable[name]:
                for s in c.string_table + [b""]:
                    d.setdefault(s, len(d))
    return list(d)


def test_p_tables_hold_their_forms():
    """Family P's columns are in the forms the family claims: a partial bucket column, full code columns, full
    bucket columns of 256 to 1,025 bins straddling 1,024-entry tiles, value arrays on the 32-bit path with int16 and
    int32 deltas on a base near 2^32, value arrays with negatives and values past 2^32, value arrays shorter than
    their block, a column absent from some blocks, and str dictionaries of 33 and 65 strings whose last string is the
    only one its pattern matches."""
    import re
    from sybil_b200 import _ffi as F
    U32 = family_p.U32
    spec, rows, valid, qs = family_p.family_p_sweep("narrow")
    gspec = dict(TABLES)["P-geom"][0]

    def cols(sp, name, enc=None):
        out = [(b, c) for b in sp.blocks for c in b.cols if c.col_slot == sp.KeyTable[name]]
        return [(b, c) for b, c in out if enc is None or c.encoding == enc]

    def nlisted(c):
        return len(c.record_ids)

    bucket = F.SG_ENC_BUCKET
    values = F.SG_ENC_VALUES
    assert any(nlisted(c) < b.num_records for b, c in cols(spec, "bp", bucket))
    for name in ["bc", "sc"] + family_p.P_CODES:
        bc = cols(spec, name, bucket)
        assert bc and all(nlisted(c) == b.num_records and len(c.bin_values) <= 255 for b, c in bc), name
    for sp in (spec, gspec):
        bd = [(b, c) for b, c in cols(sp, "bd", bucket) if b.num_records >= 1024]
        assert bd and all(nlisted(c) == b.num_records and 256 <= len(c.bin_values) <= 1025 for b, c in bd)
    big = [c for b, c in cols(gspec, "bd", bucket) if b.num_records >= 65535]
    assert len(big) == 2 and all(any(int(o0) >> 10 != (int(o1) - 1) >> 10 for o0, o1 in
                                     zip(c.bin_offsets[:-1], c.bin_offsets[1:])) for c in big)
    assert any(len(c.bin_values) > 255 for b, c in cols(spec, "sm", bucket))
    v32 = cols(spec, "v32", values)
    assert {np.asarray(c.values_i64).dtype for b, c in v32 if b.num_records > 1} == {np.dtype(np.int16),
                                                                                     np.dtype(np.int32)}
    assert all(U32 - (1 << 24) <= c.value_base < U32 for b, c in v32 if b.num_records > 1)
    v = [int(x) for cl, _, _ in rows for x in cl["v32"]]
    assert min(v) >= 0 and max(v) == U32 - 1
    v = set(int(x) for cl, _, _ in rows for x in cl["v64"])
    assert min(v) < 0 and max(v) > U32
    for name in ("vs", "sv"):
        short = cols(spec, name, values)
        arr = (lambda c: c.values_i64) if name == "vs" else (lambda c: c.values_i32)
        assert any(len(arr(c)) < b.num_records for b, c in short), name
    assert 0 < len(cols(spec, "ab")) < len(spec.blocks)
    for name, size, last, pat in (("d33", 33, "pz", "^p"), ("d65", 65, "qz", "^q")):
        d = _global_dict(spec, name)
        assert len(d) == size and d[-1] == last.encode(), (name, len(d), d[-3:])
        assert [s for s in d if re.search(pat, s.decode())] == [last.encode()], name
        assert any(last in set(cl[name][va[name]]) for (cl, _, _), va in zip(rows, valid) if name in va)
