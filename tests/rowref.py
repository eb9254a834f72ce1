"""An exact reference over raw rows: evaluates a `tests.util.Q` on the columns handed to `Spec.add_rows`,
without the block encoding, the decoder, the oracle or sg_hist.h.  Every rule is restated from the Go sources
of logv/sybil (cited as file:line under src/lib) with Python integers, so a rule that the oracle and the CUDA
path both misread shows up as a difference here.

Only order-independent fields are produced: Count, Samples, the accepted-value Count, the sum (modulo 2^64 and
unwrapped), Min / Max and the bucket counters.  Percentiles, stddev and sparse buckets depend on which block
result is adopted first (Q9) and stay compared against the oracle through `tests.util.compare`.  Counters are
kept as Python integers and compared wrapped to int64, as Go's `+= weight` leaves them.

The result shaping (`ordered`: SortResults, OrderAsc, Limit) is restated as the engine's documented rule, see
there.  StrReplace rewrites every decoded string of its column before filters and keys.

`rows` is the list of `Spec.add_rows` calls as `(cols, block_rows, threshold)` and `valid` the parallel list of
their validity masks ({name: bool array}; an absent name is fully valid)."""
import math
import re

import numpy as np

from tests.util import INT, SET, STR

NUM_BUCKETS = 1000  # hist.go:3
I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1

# The regular expressions the tests give re / nre filters: patterns on which Go's RE2 (the reference), Python's re
# (the engine's host builds the match bitset with it) and ECMAScript std::regex (the C++ oracle) agree, so that a
# difference between them is never a difference between dialects.  rowref refuses any other pattern.
PORTABLE_PATTERNS = ("^s1", "^x1", "1$", "^$", ".", "", "zz", "^(s3|s33)$", "^p", "2$", "^q")


def i64(x):
    """x wrapped to int64, as Go's int64 arithmetic does."""
    return ((x - I64_MIN) % (1 << 64)) + I64_MIN


def tdiv(a, b):
    """Go's integer division: truncates toward zero."""
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b > 0) else -q


def basic_layout(lo, hi, hist_bucket):
    """SetupBuckets, hist_basic.go:34-70: (BucketSize, len(Values))."""
    size = i64(hi - lo)
    nb = NUM_BUCKETS
    bs = tdiv(size, nb)
    if hist_bucket > 0:
        bs = hist_bucket
    if bs == 0:
        if size < 100:
            bs, nb = 1, size
        else:
            bs = tdiv(size, 100)
            nb = tdiv(size, bs)
    nb += 1
    return bs, nb + 1


def multi_layout(lo, hi):
    """MultiHist.TrackPercentiles, hist_multi.go:223-257: the sub-ranges [(Min, Max)] in lookup order."""
    bs = i64(hi - lo)
    n, t = 0, bs
    while t > NUM_BUCKETS:
        n += 1
        t >>= 1
    subs, right = [], hi
    for _ in range(n):
        bs >>= 1
        left = i64(right - bs)
        subs.append((left, right))
        right = left
    subs.append((lo, right))
    return subs


def rejects(v, lo, hi):
    """hist_basic.go:104 / hist_multi.go:50: `value > Info.Max*10 || value < Info.Min`, Max*10 wrapping."""
    return v > i64(hi * 10) or v < lo


class Basic:
    """BasicHist (hist_basic.go:72-151) with the exact sum of the accepted values added."""

    def __init__(self, lo, hi, pct, hist_bucket):
        self.lo, self.hi = lo, hi
        self.Count = self.Samples = 0
        self.Sum = 0  # unwrapped
        # SetupBuckets runs only in percentile mode; without it Min/Max start at 0 (not compared then)
        self.Min, self.Max = (lo, hi) if pct else (0, 0)
        self.Values = None
        if pct:
            self.bs, nvals = basic_layout(lo, hi, hist_bucket)
            self.Values = [0] * nvals

    def add(self, v, w, weighted):
        if rejects(v, self.lo, self.hi):
            return
        if weighted or w > 1:  # aggregate.go:100-102 via hist_basic.go:113-118
            self.Samples += 1
        self.Count += w if (weighted or w > 1) else 1
        self.Sum += v * w
        self.Max, self.Min = max(self.Max, v), min(self.Min, v)
        if self.Values is None:
            return
        # hist_basic.go:132-141: (value - Min) in int64, truncated, outliers to the last slot, underliers to 0
        b = tdiv(i64(v - self.Min), self.bs)
        b = min(b, len(self.Values) - 1)
        b = max(b, 0)
        self.Values[b] += w


class Multi:
    """MultiHist (hist_multi.go:22-88): the first sub-range holding the value takes it, under its own reject rule."""

    def __init__(self, lo, hi, pct, hist_bucket):
        self.lo, self.hi = lo, hi
        self.Count = self.Samples = 0
        self.Sum = 0
        self.Min, self.Max = lo, hi
        # every sub-range is a BasicHist of its own, HIST_BUCKET override included
        self.subs = [Basic(a, b, True, hist_bucket) for a, b in multi_layout(lo, hi)] if pct else []

    @property
    def Values(self):
        return [x for s in self.subs for x in s.Values] if self.subs else None

    def add(self, v, w, weighted):
        if rejects(v, self.lo, self.hi):
            return
        if weighted or w > 1:
            self.Samples += 1
        self.Count += w if (weighted or w > 1) else 1
        self.Sum += v * w
        self.Max, self.Min = max(self.Max, v), min(self.Min, v)
        for s in self.subs:
            if s.lo <= v <= s.hi:
                s.add(v, w, weighted)
                break


class Group:
    def __init__(self):
        self.Count = self.Samples = 0
        self.Hists = {}


class Result:
    def __init__(self):
        self.MatchedCount = self.SkippedBlocks = 0
        self.Results, self.TimeResults = {}, {}
        self.Cumulative = Group()


def decode(n, typ, vals, va, threshold):
    """What a block's column file holds once read back (column_store_io.go:82-113 writes it, :493-609,690-780 read
    it): (values, populated) over the block's n rows, or None when no row has the column (no file is written).
    Few distinct values: one bin per value, only the listed rows are populated.  Many: a Values array up to the
    last valid row, whose gaps read int 0 or string id 0 — the block's first string.
    A set column (SaveSetsToColumns, column_store_io.go:139-217; unpackSetCol :611-688): (per-row tag sets,
    populated).  Without any tag in the block no file is written.  Few distinct tags: bins, so a row is populated
    when its set is not empty.  Many: Values [][]int32 up to the last row holding a tag, every row below populated."""
    if typ == SET:
        tags = [frozenset(str(x) for x in s) if ok else frozenset() for s, ok in zip(vals, va)]
        held = [r for r, s in enumerate(tags) if s]
        if not held:
            return None
        pop = np.array([bool(s) for s in tags])
        if len(set().union(*tags)) > threshold:
            pop[:held[-1] + 1] = True
        out = np.empty(n, object)
        out[:] = tags
        return out, pop
    idx = np.nonzero(va)[0]
    if not len(idx):
        return None
    if typ == INT:
        v = np.asarray(vals, np.int64)
        distinct = len(np.unique(v[va]))
        gap = 0
    else:
        v = np.asarray([str(x) for x in vals], object)
        distinct = len(set(v[va].tolist()))
        gap = v[idx[0]]
    if distinct <= threshold:
        return v, va.copy()
    pop = np.zeros(n, bool)
    pop[:idx[-1] + 1] = True
    out = v.copy()
    out[~va] = gap
    return out, pop


def blocks(spec, rows, valid):
    """The blocks add_rows made, as {name: (values, populated)} plus the block's IntInfoMap (zone map)."""
    for (cols, block_rows, threshold), vmask in zip(rows, valid):
        n = len(next(iter(cols.values())))
        block_rows = block_rows or n
        for start in range(0, n, block_rows):
            end = min(n, start + block_rows)
            cells, info = {}, {}
            for name, vals in cols.items():
                typ = spec.KeyTypes[spec.KeyTable[name]]
                va = vmask.get(name)
                va = np.ones(end - start, bool) if va is None else np.asarray(va[start:end], bool)
                d = decode(end - start, typ, vals[start:end], va, threshold)
                if d is not None:
                    cells[name] = d
                if typ == INT and va.any():
                    v = np.asarray(vals[start:end], np.int64)[va]
                    info[name] = (int(v.min()), int(v.max()))
            yield end - start, cells, info


def should_load(q, info):
    """ShouldLoadBlockFromDir, table_block_io.go:110-182: a block is skipped when its min and max both fail a gt/lt
    filter, or an eq literal lies outside them or the block has no IntInfo for the column."""
    if not info:
        return True
    for c, op, v in q.int_filters:
        mm = info.get(c)
        if op in ("gt", "lt"):
            ok = mm is not None and any((x > v) if op == "gt" else (x < v) for x in mm)
            if not ok:
                return False
        if op == "eq" and (mm is None or mm[0] > v or mm[1] < v):
            return False
    return True


def _int_pass(op, x, v):
    return {"gt": x > v, "lt": x < v, "eq": x == v, "neq": x != v}[op]  # filter.go:171-195


def _str_pass(op, x, v):
    """StrFilter.Filter on a populated row's decoded string (filter.go:199-250): eq / neq compare the string, re /
    nre are MatchString, an unanchored search."""
    if op in ("re", "nre"):
        assert v in PORTABLE_PATTERNS, ("a pattern outside PORTABLE_PATTERNS", v)
        return (re.search(v, x) is not None) == (op == "re")
    return (x == v) if op == "eq" else (x != v)


def run(spec, rows, valid, q):
    """LoadAndQueryRecords + CombineResults over the raw rows (aggregate.go:56-282,414-467)."""
    out = Result()
    weighted = bool(q.weight_col)
    pct = q.op == "hist"
    infos = {a: spec.IntInfo.get(a, (0, 0)) for a in q.aggs}

    def new_hist(a):
        lo, hi = infos[a]
        return Multi(lo, hi, pct, q.hist_bucket) if q.loghist else Basic(lo, hi, pct, q.hist_bucket)

    # StrReplace (column_store_io.go:529-547 rewrites the block's string table): Go's $1 is Python's \g<1>
    repl = {c: (re.compile(p), re.sub(r"\$(\d+)", r"\\g<\1>", r)) for c, (p, r) in q.str_replace.items()}
    for n, cells, info in blocks(spec, rows, valid):
        if not should_load(q, info):
            out.SkippedBlocks += 1
            continue
        # per column: values as Python objects, populated flags
        cv = {k: (v.tolist(), p.tolist()) for k, (v, p) in cells.items()}
        for c, (pat, r) in repl.items():
            if c in cv:  # a string rewritten to "" renders, and so groups, like a missing value
                cv[c] = ([pat.sub(r, x) for x in cv[c][0]], cv[c][1])
        empty = ([0] * n, [False] * n)
        weight = 1  # declared per block, carried over rows without the weight column (Q13)
        for i in range(n):
            if weighted:
                wv, wp = cv.get(q.weight_col, empty)
                if wp[i]:
                    weight = wv[i]
            ok = True
            for c, op, v in q.int_filters:
                xv, xp = cv.get(c, empty)
                if not (xp[i] and _int_pass(op, xv[i], v)):
                    ok = False
                    break
            if ok:
                for c, op, v in q.str_filters:  # on the decoded string, after StrReplace; unpopulated fails
                    xv, xp = cv.get(c, empty)
                    if not (xp[i] and _str_pass(op, xv[i], v)):
                        ok = False
                        break
            if ok:
                for c, op, v in q.set_filters:  # filter.go:252-285: a row without a set fails in and nin
                    xv, xp = cv.get(c, empty)
                    if not (xp[i] and ((v in xv[i]) if op == "in" else (v not in xv[i]))):
                        ok = False
                        break
            if not ok:
                continue
            out.MatchedCount += 1
            # translate_group_by (aggregate.go:284-324): the value, "" when missing; an int -1 is the
            # MISSING_VALUE bit pattern and renders as missing too
            key = "".join(("" if not cv.get(g, empty)[1][i] or cv[g][0][i] == -1 else str(cv[g][0][i])) + "\t"
                          for g in q.groups) if q.groups else "total"
            target = out.Results
            if q.time_col:
                tv, tp = cv.get(q.time_col, empty)
                if not tp[i]:
                    continue  # matched, but no time value: counted, then skipped (aggregate.go:146-175)
                g = out.Results.setdefault(key, Group())
                g.Samples += 1
                g.Count += weight
                tb = tdiv(tv[i], q.time_bucket) * q.time_bucket  # Go's int64 division truncates (Q14)
                target = out.TimeResults.setdefault(tb, {})
            g = target.setdefault(key, Group())
            g.Samples += 1
            g.Count += weight
            for a in q.aggs:
                av, ap = cv.get(a, empty)
                if ap[i]:
                    h = g.Hists.get(a)
                    if h is None:
                        h = g.Hists[a] = new_hist(a)
                    h.add(av[i], weight, weighted)
    # the cumulative row combines every group's histograms (query_spec.go:138-193); with a time column the
    # groups hold none
    cum = out.Cumulative
    for g in out.Results.values():
        cum.Samples += g.Samples
        cum.Count += g.Count
        for a, h in g.Hists.items():
            ch = cum.Hists.get(a)
            if ch is None:
                ch = cum.Hists[a] = new_hist(a)
            merge(ch, h)
    return out


def merge(into, h):
    """Combine (hist_basic.go:259-279, hist_multi.go:202-221) restricted to the order-independent fields."""
    into.Count += h.Count
    into.Samples += h.Samples
    into.Sum += h.Sum
    into.Min, into.Max = min(into.Min, h.Min), max(into.Max, h.Max)
    if isinstance(into, Multi):
        for s, t in zip(into.subs, h.subs):
            merge(s, t)
    elif into.Values is not None:
        into.Values = [x + y for x, y in zip(into.Values, h.Values)]


def hist_fields(h):
    """A hist of any source as (Count, Sum mod 2^64, Min, Max, Values): rowref, oracle (OHist), pyoracle or the
    engine's HistCompat."""
    if isinstance(h, (Basic, Multi)):
        return h.Count, i64(h.Sum), h.Min, h.Max, h.Values
    if hasattr(h, "TotalCount"):
        return h.TotalCount(), h.Sum(), h.Min(), h.Max(), list(h.Values) if h.Values is not None else None
    return h.Count, h.ExactSum, h.Min, h.Max, list(h.Values)


def mean_value(g, a):
    """The mean SortResults orders by, as the engine documents it: float(int64 Sum) / float(int64 hist Count), each
    operand converted on its own as `(double)sum / (double)hc` does (not Python's correctly rounded int / int, which
    differs above 2^53); -inf when the group has no histogram for `a` or its Count is 0."""
    h = g.Hists.get(a)
    hc = i64(h.Count) if h is not None else 0
    return -math.inf if hc == 0 else float(i64(h.Sum)) / float(hc)


def ordered(groups, q):
    """SortResults + OrderAsc (aggregate.go:497-525) over {GroupByKey: Group}: the keys by Count (int64) or by
    mean_value of aggregation q.order_by, descending, ties by GroupByKey ascending (Python str order, which is
    UTF-8 byte order); OrderAsc reverses the whole list.  None for OrderBy "": any order is right.
    The reference's own order is a float running mean under Go's unstable sort, so its ties fall either way
    (aggregate.go:43-54,497-525; Q18/Q20): this restates the rule the engine and the oracle implement."""
    if not q.order_by:
        return None
    if q.order_by == "$COUNT":
        val = {k: i64(g.Count) for k, g in groups.items()}
    else:
        val = {k: mean_value(g, q.order_by) for k, g in groups.items()}
    keys = sorted(sorted(groups), key=lambda k: val[k], reverse=True)  # (stable: ties keep key order)
    return keys[::-1] if q.order_asc else keys


def wrapped(r):
    """True when some group's sum left int64 (its mean is then a documented divergence, DESIGN.md §7)."""
    groups = list(r.Results.values()) + [r.Cumulative] + [g for m in r.TimeResults.values() for g in m.values()]
    return any(h.Sum != i64(h.Sum) for g in groups for h in g.Hists.values())


def check(ref, got, q, hists_of=lambda g: g.Hists, where="", order=True):
    """got (oracle, pyoracle or engine result) against ref on every field rowref produces.  The engine (a result
    with NumGroups) keeps the first `limit` groups of the sorted list; the oracle and pyoracle keep every group.
    order=False compares the groups but not their order (the oracle's mean order is its float running mean)."""
    hist_mode = q.op == "hist" or q.loghist

    def grp(rg, gg, w):
        assert (i64(gg.Count), gg.Samples) == (i64(rg.Count), rg.Samples), (w, "Count/Samples", (gg.Count, gg.Samples),
                                                                            (rg.Count, rg.Samples))
        gh = hists_of(gg)
        for ai, a in enumerate(q.aggs if not (q.time_col and w[1] == "Results") else []):
            rh = rg.Hists.get(a)
            h = gh.get(a, gh.get(ai)) if isinstance(gh, dict) else None
            if rh is None or i64(rh.Count) == 0:
                assert h is None or i64(hist_fields(h)[0]) == 0, (w, a, "unexpected hist")
                continue
            assert h is not None, (w, a, "missing hist")
            c, s, mn, mx, vals = hist_fields(h)
            rc, rs, rmn, rmx, rvals = hist_fields(rh)
            assert i64(c) == i64(rc), (w, a, "hist Count", c, rc)
            assert s == rs, (w, a, "sum mod 2^64", s, rs)
            if hist_mode:
                assert (mn, mx) == (rmn, rmx), (w, a, "Min/Max", (mn, mx), (rmn, rmx))
            if q.op == "hist":
                vals, rvals = [i64(int(x)) for x in vals], [i64(x) for x in rvals]
                assert vals == rvals, (w, a, "bucket counters",
                                       [(k, x, y) for k, (x, y) in enumerate(zip(vals, rvals)) if x != y][:8])

    def keys_in_order(got_keys, groups, w):
        """got_keys (a result list's keys in its order) against `groups` shaped by ordered() and the limit."""
        assert len(got_keys) == len(set(got_keys)), (w, "groups sharing a key",
                                                     sorted(k for k in set(got_keys) if got_keys.count(k) > 1)[:8])
        want = ordered(groups, q)
        cut = q.limit if q.limit and hasattr(got, "NumGroups") and w[-1] == "Sorted" else None
        if want is None:  # OrderBy "": any `limit` of the groups, each exact
            assert len(got_keys) == len(list(groups)[:cut]), (w, "groups", len(got_keys), len(groups))
            assert set(got_keys) <= set(groups), (w, "group keys", sorted(set(got_keys) - set(groups))[:8])
            return
        want = want[:cut]
        if order and hasattr(got, "Sorted"):  # (pyoracle's Results have no order)
            i = next((i for i, (x, y) in enumerate(zip(got_keys, want)) if x != y), min(len(got_keys), len(want)))
            assert got_keys == want, (w, "order", len(got_keys), len(want), "first difference at", i,
                                      got_keys[i:i + 4], want[i:i + 4])
        else:
            assert set(got_keys) == set(want), (w, "group keys", sorted(set(got_keys) ^ set(want))[:8])

    assert got.MatchedCount == ref.MatchedCount, (where, "MatchedCount", got.MatchedCount, ref.MatchedCount)
    # Results is a dict keyed by the rendered key: two groups with one key would hide each other there, so the
    # group counts are checked on the lists the dicts were built from.  NumGroups counts every group, limit or not
    if hasattr(got, "NumGroups"):
        assert got.NumGroups == len(ref.Results), (where, "NumGroups", got.NumGroups, len(ref.Results))
    keys = [r.GroupByKey for r in getattr(got, "Sorted", None) or got.Results.values()]
    keys_in_order(keys, ref.Results, (where, "Sorted"))
    assert set(got.Results) == set(keys), (where, "Results against Sorted")
    for k in got.Results:
        grp(ref.Results[k], got.Results[k], (where, "Results", k))
    if q.time_col:
        assert ((i64(got.Cumulative.Count), got.Cumulative.Samples) ==
                (i64(ref.Cumulative.Count), ref.Cumulative.Samples)), (where, "Cumulative")
    else:
        grp(ref.Cumulative, got.Cumulative, (where, "Cumulative"))
    assert set(got.TimeResults) == set(ref.TimeResults), (where, "time buckets",
                                                          sorted(set(got.TimeResults) ^ set(ref.TimeResults))[:8])
    for tb, m in ref.TimeResults.items():
        n = getattr(got, "TimeNumGroups", {}).get(tb, len(got.TimeResults[tb]))
        assert n == len(m), (where, "time groups", tb, "groups sharing a key")
        if hasattr(got, "TimeNumGroups"):  # the engine's slices are dicts built from its sorted lists
            keys_in_order(list(got.TimeResults[tb]), m, (where, "TimeResults", tb))
        assert set(got.TimeResults[tb]) == set(m), (where, "time groups", tb)
        for k, rg in m.items():
            grp(rg, got.TimeResults[tb][k], (where, "TimeResults", tb, k))
