"""Shared helpers of the parity tests: random tables in sybil's block format, the
query description given identically to the oracle and to the CUDA path, and the
field-by-field comparison (bit-exact fields and float-tolerance fields)."""
import math

import numpy as np

from sybil_b200 import _ffi as F
from sybil_b200 import engine as E
import os

from sybil_b200.blocks import encode_block, narrow_column

INT, STR, SET = F.SG_COL_INT, F.SG_COL_STR, F.SG_COL_SET

# tolerances of SURVEY.md §8(d): mean |d| <= 1e-9*max(1,|mean|); stddev rel <= 1e-9
MEAN_TOL = 1e-9
STD_TOL = 1e-9


# Which columns of the test tables are handed over in their narrow form (uint16 ids, int16/int32 value deltas,
# sybilgpu.h): "mixed" (default) = column c of block b when b + c is even, so one table — even one block —
# mixes both forms and every test exercises both; "narrow" / "wide" = all / none (SG_TEST_FORMS).
FORMS = os.environ.get("SG_TEST_FORMS", "mixed")


def pick_narrow(block_index, col_slot, forms=None):
    forms = forms or FORMS
    return forms == "narrow" or (forms == "mixed" and (block_index + col_slot) % 2 == 0)


class Spec:
    """A table: key_table [(name, type)], IntInfo, and SavedBlocks."""

    forms = None  # None: the module default (FORMS)

    def __init__(self, key_table):
        self.key_table = key_table
        self.KeyTable = {n: i for i, (n, _) in enumerate(key_table)}
        self.KeyTypes = {i: t for i, (_, t) in enumerate(key_table)}
        self.IntInfo = {}
        self.blocks = []

    def add_rows(self, cols, valid=None, threshold=5000, block_rows=None):
        """cols: {name: array/list}; valid: {name: bool array}.  Splits into blocks of block_rows."""
        n = len(next(iter(cols.values())))
        block_rows = block_rows or n
        valid = valid or {}
        for start in range(0, n, block_rows):
            end = min(n, start + block_rows)
            cl = []
            for name, vals in cols.items():
                slot = self.KeyTable[name]
                v = vals[start:end]
                va = valid.get(name)
                cl.append((slot, self.KeyTypes[slot], v, None if va is None else va[start:end]))
            blk = encode_block(len(self.blocks), end - start, cl, threshold)
            blk.cols = [narrow_column(c) if pick_narrow(blk.block_index, c.col_slot, self.forms) else c for c in blk.cols]
            self.blocks.append(blk)
        for name, vals in cols.items():
            slot = self.KeyTable[name]
            if self.KeyTypes[slot] == INT:
                va = valid.get(name)
                v = np.asarray(vals, np.int64)
                if va is not None:
                    v = v[np.asarray(va, bool)]
                if len(v):
                    mn, mx = int(v.min()), int(v.max())
                    if name in self.IntInfo:
                        mn, mx = min(mn, self.IntInfo[name][0]), max(mx, self.IntInfo[name][1])
                    self.IntInfo[name] = (mn, mx)


class Q:
    """A query in the reference's vocabulary, buildable without a GPU."""

    def __init__(self, spec, int_filters=(), str_filters=(), groups=(), aggs=(), op="avg", loghist=False,
                 time_col=None, time_bucket=0, hist_bucket=0, order_by="$COUNT", order_asc=False, limit=0,
                 set_filters=(), str_replace=None, weight_col=None):
        self.spec = spec
        self.weight_col = weight_col  # FLAGS.WEIGHT_COL
        self.set_filters = list(set_filters)      # (column, "in" | "nin", tag)
        self.str_replace = dict(str_replace or {})  # column -> (pattern, replacement): FLAGS.STR_REPLACE
        self.order_by, self.order_asc, self.limit = order_by, order_asc, limit
        self.int_filters, self.str_filters = list(int_filters), list(str_filters)
        self.groups, self.aggs = list(groups), list(aggs)
        self.op, self.loghist, self.time_col, self.time_bucket, self.hist_bucket = op, loghist, time_col, time_bucket, hist_bucket

    def set_flags(self):
        E.FLAGS.reset()
        E.FLAGS.OP = self.op
        E.FLAGS.LOG_HIST = self.loghist
        E.FLAGS.HIST_BUCKET = self.hist_bucket
        if self.time_col:
            E.FLAGS.TIME_COL = self.time_col
            E.FLAGS.TIME_BUCKET = self.time_bucket
        E.FLAGS.WEIGHT_COL = self.weight_col or ""

    def query_spec(self):
        s = self.spec
        self.set_flags()
        filters = [E.IntFilter(c, s.KeyTable[c], op, v) for c, op, v in self.int_filters]
        filters += [E.StrFilter(c, s.KeyTable[c], op, v) for c, op, v in self.str_filters]
        filters += [E.SetFilter(c, s.KeyTable[c], op, v) for c, op, v in self.set_filters]
        groups = [E.Grouping(c, s.KeyTable[c]) for c in self.groups]
        aggs = [E.Aggregation(c, s.KeyTable[c], self.op) for c in self.aggs]
        return E.QuerySpec(Filters=filters, Groups=groups, Aggregations=aggs, TimeBucket=self.time_bucket if self.time_col else 0,
                           OrderBy=self.order_by, OrderAsc=self.order_asc, Limit=self.limit,
                           StrReplace={c: E.StrReplace(p, r) for c, (p, r) in self.str_replace.items()})

    def desc(self):
        qs = self.query_spec()
        return E.make_query_desc(self.spec.KeyTable, self.spec.KeyTypes, self.spec.IntInfo, qs)


def run_oracle(spec, q, nthreads=1):
    from oracle.oracle_ffi import OracleTable
    ot = OracleTable(spec.key_table)
    for b in spec.blocks:
        ot.add_block(b)
    for c, (pat, rep) in q.str_replace.items():
        ot.set_str_replace(spec.KeyTable[c], pat, rep)
    d, keep = q.desc()
    try:
        return ot.query(d, q.aggs, nthreads=nthreads)
    finally:
        ot.close()


def run_gpu(spec, q, table=None):
    """The CUDA path through the C ABI.  Returns the filled QuerySpec."""
    own = table is None
    if own:
        table = E.Table("t", spec.key_table)
        table.IntInfo = dict(spec.IntInfo)
        for b in spec.blocks:
            table.add_block(b)
    try:
        qs = q.query_spec()
        ls = table.NewLoadSpec()
        for c, _, _ in q.int_filters:
            ls.Int(c)
        for c, _, _ in q.str_filters:
            ls.Str(c)
        for c, _, _ in q.set_filters:
            ls.Set(c)
        for c in q.groups + q.aggs + ([q.weight_col] if q.weight_col else []):
            ls.Int(c)
        table.LoadAndQueryRecords(ls, qs)
        return qs
    finally:
        if own:
            table.close()


def close(a, b, tol):
    if math.isnan(a) and math.isnan(b):
        return True
    return abs(a - b) <= tol * max(1.0, abs(a), abs(b))


def compare_group(g, o, aggs, op_hist, where, loghist=False, mean=True):
    assert g.GroupByKey == o.GroupByKey, where
    assert g.Count == o.Count, (where, "Count")
    assert g.Samples == o.Samples, (where, "Samples")
    for a in aggs:
        oh = o.Hists.get(a)
        gh = g.Hists.get(a)
        if oh is None or oh.Count == 0:
            assert gh is None, (where, a, "unexpected hist")
            continue
        assert gh is not None, (where, a, "missing hist")
        assert gh.TotalCount() == oh.Count, (where, a, "hist Count")
        assert gh.Sum() == oh.ExactSum, (where, a, "exact int64 sum")
        check_mean = mean(oh) if callable(mean) else mean
        if check_mean:
            assert close(gh.Mean(), oh.Avg, MEAN_TOL), (where, a, "mean", gh.Mean(), oh.Avg)
        if op_hist or loghist:
            assert gh.Min() == oh.Min, (where, a, "Min")
            assert gh.Max() == oh.Max, (where, a, "Max")
        if op_hist:
            assert np.array_equal(gh.Values, oh.Values), (where, a, "bucket counters")
            # oh.Percentiles / IntBuckets / StdDev come from the oracle's merged view when the
            # first-seen block result still held Outliers (Q9, oracle_ffi._group)
            assert gh.GetPercentiles() == oh.Percentiles, (where, a, "percentiles")
            assert gh.GetIntBuckets() == oh.IntBuckets, (where, a, "sparse buckets")
            if check_mean:  # (the stddev is taken around the mean)
                assert close(gh.StdDev(), oh.StdDev, STD_TOL), (where, a, "stddev", gh.StdDev(), oh.StdDev)


def compare(qs, oq, q, mean=True):
    """GPU QuerySpec vs oracle result: keys, Count, Samples, hist Count, exact sums, Min/Max, bucket
    counters and percentiles bit-exact; mean / stddev within the stated tolerance.  mean=False, or a predicate
    on the oracle's histogram that is false, skips the mean and stddev of those histograms (DESIGN.md §7: the
    mean diverges where the sum left int64, and the reference's turns NaN in some groups)."""
    op_hist = q.op == "hist"
    assert qs.MatchedCount == oq.MatchedCount, "MatchedCount"
    assert qs.BrokenBlocks == oq.BrokenBlocks, "broken blocks"
    assert qs.SkippedBlocks == oq.SkippedBlocks, "skipped blocks"
    assert qs.NumGroups == len(oq.Results), "number of groups"
    want = list(oq.Sorted)
    if q.limit:  # only the first `limit` groups of the sorted list are materialised (FLAGS.LIMIT)
        want = want[:q.limit]
    if q.order_by:
        assert [r.GroupByKey for r in qs.Sorted] == [r.GroupByKey for r in want], "Sorted order"
    else:  # OrderBy == "": no sort (aggregate.go:499) — the same groups in whatever order
        assert sorted(r.GroupByKey for r in qs.Sorted) == sorted(r.GroupByKey for r in want), "groups"
    assert set(qs.Results) == set(r.GroupByKey for r in want), "group keys"
    for k in qs.Results:
        compare_group(qs.Results[k], oq.Results[k], q.aggs if not q.time_col else [], op_hist, ("Results", k), q.loghist, mean)
    c, oc = qs.Cumulative, oq.Cumulative
    assert c.GroupByKey == oc.GroupByKey
    assert c.Count == oc.Count and c.Samples == oc.Samples, "Cumulative counts"
    if not q.time_col:
        compare_group(c, oc, q.aggs, op_hist, ("Cumulative",), q.loghist, mean)
    assert set(qs.TimeResults) == set(oq.TimeResults), "time buckets"
    for tb, m in oq.TimeResults.items():
        assert set(qs.TimeResults[tb]) == set(m), ("time groups", tb)
        for k, o in m.items():
            compare_group(qs.TimeResults[tb][k], o, q.aggs, op_hist, ("TimeResults", tb, k), q.loghist, mean)


def random_spec(seed, nrows=3000, block_rows=1000, nulls=True, threshold=5000, wide=False, sets=False):
    """A small random table exercising both encodings, missing values and several string columns
    (sets: plus a set column `tags`, 0-3 of 9 tags per row, some rows without the column)."""
    rng = np.random.default_rng(seed)
    kt = [("age", INT), ("lat", INT), ("big", INT), ("host", STR), ("state", STR), ("time", INT), ("uid", STR)]
    if sets:
        kt.append(("tags", SET))
    s = Spec(kt)
    cols = {
        "age": rng.integers(10, 30, nrows),
        "lat": (rng.integers(0, 65536, (nrows, 4)).sum(1) * 23470 // (4 * 65535) + 30),
        "big": rng.integers(-(1 << 40), 1 << 50, nrows) if wide else rng.integers(0, 1000000, nrows),
        "host": np.array(["h%d" % v for v in rng.integers(0, 5, nrows)]),
        "state": np.array(["s%d" % v for v in rng.integers(0, 12, nrows)]),
        "time": 1500000000 + np.sort(rng.integers(0, 7200, nrows)),
        "uid": np.array(["u%d" % v for v in rng.integers(0, nrows * 4, nrows)]),
    }
    valid = {}
    if sets:
        ntag = rng.integers(0, 4, nrows)
        cols["tags"] = [["t%d" % v for v in rng.choice(9, int(k), replace=False)] for k in ntag]
    if nulls:
        for name in ("age", "lat", "host", "state", "big"):
            valid[name] = rng.random(nrows) > 0.07
    s.add_rows(cols, valid, threshold=threshold, block_rows=block_rows)
    return s
