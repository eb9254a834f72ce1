"""pyoracle.py — a second, independent restatement of the reference's query path in
plain Python (TEST INFRASTRUCTURE; small inputs only).

It exists to cross-check oracle/oracle.cpp: the two were written separately from
the Go sources and must agree on every field.  Same citations as oracle.cpp:
unpack*Col column_store_io.go:493-609,690-780; filters filter.go:171-250;
FilterAndAggRecords aggregate.go:56-282; BasicHist hist_basic.go:34-279; MultiHist
hist_multi.go:22-257; Result.Combine query_spec.go:138-193; CombineResults
aggregate.go:414-467; unpackSetCol column_store_io.go:611-688; SetFilter filter.go:252-285;
weights aggregate.go:68,100-102,202-203 + AddWeightedValue; StrReplace
column_store_io.go:515-549.
"""
import math
import re

from sybil_b200 import _ffi as F
from sybil_b200.blocks import decode_column

M64 = (1 << 64) - 1


def _i64(x):
    x &= M64
    return x - (1 << 64) if x >= (1 << 63) else x


def _fdiv(a, b):  # Go float64 division: x/0 is +-Inf or NaN, never a panic
    if b == 0.0:
        return float("nan") if a == 0.0 or a != a else math.copysign(float("inf"), a)
    return a / b


def _tdiv(a, b):  # Go integer division truncates toward zero
    q = abs(a) // abs(b)
    return q if (a >= 0) == (b >= 0) else -q


class PyBasicHist:
    def __init__(self, mn, mx, hist_mode, hist_bucket=0):
        self.info = (mn, mx)
        self.Min, self.Max = 0, 0
        self.Count, self.Avg, self.ExactSum = 0, 0.0, 0
        self.pm = hist_mode
        self.Values, self.Outliers, self.Underliers = [], [], []
        if hist_mode:
            self.Min, self.Max = mn, mx
            size = _i64(mx - mn)
            nb, bs = 1000, _tdiv(size, 1000)
            if hist_bucket > 0:
                bs = hist_bucket
            if bs == 0:
                if size < 100:
                    bs, nb = 1, size
                else:
                    bs = _tdiv(size, 100)
                    nb = _tdiv(size, bs)
            nb += 1
            self.NumBuckets, self.BucketSize = nb, bs
            self.Values = [0] * (nb + 1)

    def add(self, v, weight=1, weight_col=False):  # AddWeightedValue, hist_basic.go:101-151
        if v > _i64(self.info[1] * 10) or v < self.info[0]:
            return
        self.Count += weight if (weight_col or weight > 1) else 1
        self.ExactSum = _i64(self.ExactSum + v * weight)
        self.Avg = self.Avg + _fdiv(float(v) - self.Avg, float(self.Count)) * float(weight)
        self.Max = max(self.Max, v)
        self.Min = min(self.Min, v)
        if not self.pm:
            return
        b = _tdiv(_i64(v - self.Min), self.BucketSize)
        if b >= len(self.Values):
            self.Outliers.append(v)
            b = len(self.Values) - 1
        if b < 0:
            self.Underliers.append(v)
            b = 0
        self.Values[b] += weight

    def combine(self, o):
        for k, v in enumerate(o.Values):
            self.Values[k] += v
        tot = self.Count + o.Count
        self.Avg = self.Avg * _fdiv(float(self.Count), float(tot)) + o.Avg * _fdiv(float(o.Count), float(tot))
        self.Min, self.Max = min(self.Min, o.Min), max(self.Max, o.Max)
        self.Count = tot
        self.ExactSum = _i64(self.ExactSum + o.ExactSum)

    def fresh(self, hist_bucket=0):
        return PyBasicHist(self.info[0], self.info[1], self.pm, hist_bucket)

    def sparse(self):
        m = {}
        for k, c in enumerate(self.Values):
            if c > 0:
                m[k * self.BucketSize + self.Min] = c
        for v in self.Outliers + self.Underliers:
            m[v] = m.get(v, 0) + 1
        return m

    def percentiles(self):
        if self.Count == 0:
            return []
        p = [0] * 101
        p[0] = self.Min
        cnt = prev = 0
        for k, c in enumerate(self.Values):
            cnt += c
            q = (100 * cnt) // self.Count
            for ip in range(prev, q + 1):
                p[ip] = k * self.BucketSize + self.Min
            p[q] = k
            prev = q
        return p[:100]

    def stddev(self):
        s = 0.0
        for b, c in enumerate(self.Values):
            d = float(b * self.BucketSize + self.Min) - self.Avg
            s += (d * d) * (float(c) / float(self.Count))
        for v in self.Outliers + self.Underliers:
            s += math.pow(float(v) - self.Avg, 2) * (1 / float(self.Count))
        return math.sqrt(s)


class PyMultiHist:
    def __init__(self, mn, mx, hist_mode):
        self.info = (mn, mx)
        self.Min, self.Max = mn, mx
        self.Count, self.Avg, self.ExactSum = 0, 0.0, 0
        self.pm = hist_mode
        self.subs = []
        if hist_mode:
            size = _i64(mx - mn)
            n, t = 0, size
            while t > 1000:
                n += 1
                t >>= 1
            right = mx
            for _ in range(n):
                size >>= 1
                self.subs.append(PyBasicHist(right - size, right, True))
                right = right - size
            self.subs.append(PyBasicHist(mn, right, True))

    def add(self, v, weight=1, weight_col=False):  # hist_multi.go:48-88
        if v > _i64(self.info[1] * 10) or v < self.info[0]:
            return
        self.Count += weight if (weight_col or weight > 1) else 1
        self.ExactSum = _i64(self.ExactSum + v * weight)
        self.Avg = self.Avg + _fdiv(float(v) - self.Avg, float(self.Count)) * float(weight)
        self.Max, self.Min = max(self.Max, v), min(self.Min, v)
        for sh in self.subs:
            if sh.info[0] <= v <= sh.info[1]:
                sh.add(v, weight, weight_col)
                break

    def combine(self, o):
        for a, b in zip(self.subs, o.subs):
            a.combine(b)
        tot = self.Count + o.Count
        self.Avg = self.Avg * _fdiv(float(self.Count), float(tot)) + o.Avg * _fdiv(float(o.Count), float(tot))
        self.Min, self.Max = min(self.Min, o.Min), max(self.Max, o.Max)
        self.Count = tot
        self.ExactSum = _i64(self.ExactSum + o.ExactSum)

    def fresh(self, hist_bucket=0):
        return PyMultiHist(self.info[0], self.info[1], self.pm)

    @property
    def Values(self):
        return [v for sh in self.subs for v in sh.Values]

    def sparse(self):
        m = {}
        for sh in self.subs:
            for k, c in sh.sparse().items():
                m[k] = m.get(k, 0) + c
        return m

    def percentiles(self):
        if self.Count == 0:
            return []
        m = self.sparse()
        ks = sorted(k for k in m if m[k] > 0)
        tot = sum(m[k] for k in ks)
        p = [0] * 101
        prev = cnt = 0
        for k in ks:
            cnt += m[k]
            q = (100 * cnt) // tot
            for ip in range(prev, q + 1):
                if ip <= 100:
                    p[ip] = k
            if q <= 100:
                p[q] = k
            prev = q
        return p[:100]

    def stddev(self):
        s = 0.0
        for k, c in sorted(self.sparse().items()):
            d = float(k) - self.Avg
            s += (d * d) * (float(c) / float(self.Count))
        return math.sqrt(s)


class PyResult:
    def __init__(self):
        self.Count = self.Samples = 0
        self.Hists = {}
        self.GroupByKey = ""


def _combine(into, r):
    if r.Count == 0:
        return
    for k, h in r.Hists.items():
        if k not in into.Hists:
            nh = h.fresh()
            nh.combine(h)
            into.Hists[k] = nh
        else:
            into.Hists[k].combine(h)
    into.Count += r.Count
    into.Samples += r.Samples


def _set_rows(c, n):
    """unpackSetCol (column_store_io.go:611-688): per row the tag strings and whether the row has a set; None when
    the block is broken (a row id beyond the block)."""
    import numpy as np
    tags = [[] for _ in range(n)]
    pop = [False] * n
    for b in range(len(c.bin_values)):
        ids = np.asarray(c.record_ids[c.bin_offsets[b]:c.bin_offsets[b + 1]]).astype(np.int64)
        rows = np.cumsum(ids) if c.delta_ids else ids
        for r in rows:
            if r >= n:
                return None
            tags[int(r)].append(c.string_table[int(c.bin_values[b])])
            pop[int(r)] = True
    nv = int(getattr(c, "set_nvalues", 0))
    if nv > n:
        return None
    for r in range(nv):  # the non-bucketed file form lists the row: populated, empty set or not
        pop[r] = True
    return tags, pop


def query(blocks, key_types, filters, groups, aggs, op_hist=False, log_hist=False, time_col=None, time_bucket=0,
          hist_bucket=0, weight_col=None, str_replace=None):
    """blocks: list of sybil_b200.blocks.SavedBlock.  filters: (slot, 'int'|'str'|'set', op, value);
    groups: slots; aggs: (slot, info_min, info_max); weight_col: slot (OPTS.WEIGHT_COL); str_replace: {slot:
    (pattern, python replacement template)} — the rewritten strings are what filters and keys see.  A merging rewrite
    is restated by its INTENT only for literals the rewritten table holds (see DESIGN.md §7 for the reference's id
    aliasing with other literals).  Returns (results, time_results, cumulative, matched, broken)."""
    str_replace = str_replace or {}
    master, tmaster = {}, {}
    cumulative = PyResult()
    cumulative.GroupByKey = "TOTAL" + "\t" * max(len(groups) - 1, 0)
    matched_total = broken = 0
    wanted = set([f[0] for f in filters] + list(groups) + [a[0] for a in aggs] + ([time_col] if time_col is not None else []) +
                 ([weight_col] if weight_col is not None else []))
    for blk in blocks:
        n = blk.num_records
        cols, bad = {}, False
        for c in blk.cols:
            if c.col_slot not in wanted:
                continue
            if c.col_type == F.SG_COL_STR and len(c.string_table) > n:
                bad = True
            if c.encoding == F.SG_ENC_VALUES and max(len(c.values_i64), len(c.values_i32)) > n:
                bad = True
            if c.encoding == F.SG_ENC_BUCKET:
                import numpy as np
                for b in range(len(c.bin_values)):
                    ids = c.record_ids[c.bin_offsets[b]:c.bin_offsets[b + 1]].astype(np.int64)
                    rows = np.cumsum(ids) if c.delta_ids else ids
                    if len(rows) and rows.max() >= n:
                        bad = True
            if bad:
                break
            if c.col_type == F.SG_COL_SET:
                sr = _set_rows(c, n)
                if sr is None:
                    bad = True
                    break
                cols[c.col_slot] = (sr, c)
                continue
            if c.col_slot in str_replace:  # re.ReplaceAllString over the block's string table (:529-531)
                import copy
                pat, rep = str_replace[c.col_slot]
                c = copy.copy(c)
                c.string_table = [re.sub(pat, rep, t.decode()).encode() for t in c.string_table]
            cols[c.col_slot] = (decode_column(c, n), c)
        if bad:
            broken += 1
            continue
        res, tres = {}, {}
        matched = 0
        weight = 1  # declared outside the row loop: a row without the weight column reuses the last one (Q13)
        for r in range(n):
            if weight_col is not None and weight_col in cols and cols[weight_col][0][1][r]:
                weight = int(cols[weight_col][0][0][r])
            ok = True
            for slot, kind, op, val in filters:
                if kind == "set":  # SetFilter, filter.go:252-285
                    if slot not in cols or not cols[slot][0][1][r]:
                        ok = False
                        break
                    lit = val if isinstance(val, bytes) else val.encode()
                    has = lit in cols[slot][0][0][r]
                    ok = has if op == "in" else not has
                    if not ok:
                        break
                    continue
                if slot not in cols or not cols[slot][0][1][r]:
                    ok = False
                    break
                v = int(cols[slot][0][0][r])
                if kind == "int":
                    ok = {"gt": v > val, "lt": v < val, "eq": v == val, "neq": v != val}.get(op, False)
                else:
                    tab = cols[slot][1].string_table
                    s = tab[v] if 0 <= v < len(tab) else b""
                    lit = val if isinstance(val, bytes) else val.encode()
                    if op == "eq":
                        ok = s == lit and lit in tab
                    elif op == "neq":
                        ok = not (s == lit and lit in tab)
                    else:
                        m = re.search(val, s.decode()) is not None
                        ok = m if op == "re" else not m
                if not ok:
                    break
            if not ok:
                continue
            matched += 1
            key = []
            for slot in groups:
                if slot in cols and cols[slot][0][1][r]:
                    v = int(cols[slot][0][0][r])
                    if key_types[slot] == F.SG_COL_STR:
                        tab = cols[slot][1].string_table
                        key.append((tab[v] if 0 <= v < len(tab) else b"").decode())
                    else:  # uint64(-1) is MISSING_VALUE: -1 renders as missing (aggregate.go:125-143,306)
                        key.append("" if v == -1 else str(v))
                else:
                    key.append("")
            skey = "".join(k + "\t" for k in key) if groups else "total"
            target = res
            if time_bucket > 0:
                if time_col not in cols or not cols[time_col][0][1][r]:
                    continue
                big = res.setdefault(skey, PyResult())
                big.GroupByKey = skey
                big.Count += weight
                big.Samples += 1
                tv = int(cols[time_col][0][0][r])
                target = tres.setdefault(_tdiv(tv, time_bucket) * time_bucket, {})
            rec = target.setdefault(skey, PyResult())
            rec.GroupByKey = skey
            rec.Count += weight
            rec.Samples += 1
            for ai, (slot, mn, mx) in enumerate(aggs):
                if slot in cols and cols[slot][0][1][r] and key_types[slot] == F.SG_COL_INT:
                    if ai not in rec.Hists:
                        rec.Hists[ai] = PyMultiHist(mn, mx, op_hist) if log_hist else PyBasicHist(mn, mx, op_hist, hist_bucket)
                    rec.Hists[ai].add(int(cols[slot][0][0][r]), weight, weight_col is not None)
        matched_total += matched
        for k, r in res.items():
            if k not in master:
                master[k] = r
            else:
                _combine(master[k], r)
            _combine(cumulative, r)
        for tb, m in tres.items():
            mm = tmaster.setdefault(tb, {})
            for k, r in m.items():
                if k not in mm:
                    mm[k] = r
                else:
                    _combine(mm[k], r)
    return master, tmaster, cumulative, matched_total, broken
