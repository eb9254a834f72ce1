"""Family P: predicates.  Int and str filter columns in every form the planner and the scan kernel tell apart, swept
over the literals where their arithmetic branches.  Shared by tests/test_rowref.py (oracle and pyoracle against
tests/rowref.py, no GPU) and tests/test_parity_filters.py (the CUDA path against both, under each plan switch).

The kernel evaluates a filter in one of three ways (DESIGN.md §4): count mode (a row adds the pass increment per
filter it passes), fail mode (every filter column lists every row of every listed block: a failing row ORs in a
sticky bit, and a bucket column walks only the 1,024-entry tiles that hold its failing bins) and the per-row code
pass (bucket columns of at most 255 bins).  Within each, a column is bucket bins, a value array on the 32-bit path
(its range clipped to [0, 2^32)), a value array on the 64-bit path, an array shorter than its block, or absent.

Every block size comes twice: bucket-form (threshold P_BUCKET: every column with few enough distinct values is
bucket-encoded) and value-form (threshold 0: every column is a value array).  Each query's `expect` holds patterns
for its SG_PLAN_TRACE line (fail_mode=, codes=) that show which path it reached."""
import numpy as np

from tests.edges import _q, _Table
from tests.util import INT, STR

U32 = 1 << 32
P_INT = ["bp", "bc", "bd", "v32", "v64", "vs", "ab"]
P_STR = ["sp", "sc", "sm", "sv", "d33", "d65"]
P_CODES = ["c%d" % i for i in range(9)]
KT_P = [("g", STR), ("v", INT)] + [(c, INT) for c in P_INT] + [(c, STR) for c in P_STR] + [(c, INT) for c in P_CODES]
P_BUCKET = 1100  # bucket-form threshold: above every bucket column's bins (bd: up to 1,025)
SWEEP_SIZES = [1025, 1024, 1, 1500]  # 1,025 / 1,024: one row past / at a tile; 1,500: a partial last tile
GEOM_SIZES = [65536, 65535]
BP_POOL = [-(1 << 33), -7, -1, 0, 3, 77, U32 - 1, U32, U32 + 9]
V64_POOL = [-(1 << 40), -(1 << 33), -5, -1, 0, 1, U32 - 1, U32, U32 + 1, 1 << 40]
# the global dictionaries of d33 / d65: the first block holds D33[:-1] / D65[:-1], staging then interns "" (a block's
# str column always has it, sg_table_add_block), and later blocks bring the last string: it has the largest id, and
# the patterns "^p" / "^q" match it alone
D33 = ["d%02d" % i for i in range(31)] + ["pz"]
D65 = ["e%02d" % i for i in range(63)] + ["qz"]
# literals and patterns per str column: a present literal, one in the dictionary but not in every block, one absent
# from the dictionary, and ""; patterns from rowref.PORTABLE_PATTERNS
STR_LITERALS = {"sp": ["s1", "only0", "zz", ""], "sc": ["s1", "s59", "zz", ""], "sm": ["m001", "m599", "zz", ""],
                "sv": ["s1", "s1999", "zz", ""], "d33": ["d05", "pz", "zz", ""], "d65": ["e05", "qz", "zz", ""]}
STR_PATTERNS = {"sp": ["^s1", "1$", "^$", "", "zz", "^(s3|s33)$"], "sc": ["^s1", "1$", "^$", ".", "^(s3|s33)$"],
                "sm": ["1$", "zz", "."], "sv": ["^s1", "2$", "^$", "."], "d33": ["^p", "."], "d65": ["^q", ""]}


def _walk(rng, n, lo, hi, step):
    """A random walk inside [lo, hi] whose steps stay below `step` in size."""
    v = np.empty(n, np.int64)
    x = int(rng.integers(lo, hi + 1))
    for i in range(n):
        v[i] = x
        x = min(hi, max(lo, x + int(rng.integers(-step + 1, step))))
    return v


def _strs(rng, prefix, k, n, fmt="%s%d"):
    return np.array([fmt % (prefix, x) for x in rng.integers(0, k, n)])


def _block(rng, n, form, blk):
    """One block's columns and validity.  `form` "bucket" or "values"; blk: its index in the table."""
    bucket = form == "bucket"
    r = np.arange(n)
    full = np.ones(n, bool)

    def gappy(p, tail=0):
        """rows without the column: in the value form only (gaps read 0 / the block's first string), and the last
        `tail` rows (the value array ends early); the bucket form lists every row."""
        if bucket or n == 1:
            return full.copy()
        va = rng.random(n) > p
        va[0] = True  # (the first string, which the gaps read, is a real one)
        if tail:
            va[-tail:] = False
        return va

    cols, valid = {}, {}
    cols["g"] = _strs(rng, "g", 3, n)
    cols["v"] = rng.integers(0, 1000, n)
    cols["bp"] = rng.choice(np.asarray(BP_POOL, np.int64), n)
    valid["bp"] = rng.random(n) > 0.15 if n > 1 else full.copy()  # partial in both forms (count mode)
    cols["bc"] = rng.integers(0, 200, n) * 3 - 100
    # bd: even values, so an odd literal inside the extents fails every bin; 400 / 900 bins in 1,024+ rows
    nb = 1 if n == 1 else (400 if n < 2048 else 900)
    k = rng.integers(0, nb, n)
    k[:nb] = np.arange(nb)
    cols["bd"] = 1000 + 2 * rng.permutation(k)
    # v32: a walk just below 2^32 through 2^32 - 1, all rows: value_base near 2^32, int16 deltas in even blocks,
    # int32 deltas in odd ones
    if blk % 2 == 0:
        cols["v32"] = _walk(rng, n, U32 - 30000, U32 - 1, 500)
    else:
        cols["v32"] = _walk(rng, n, U32 - (1 << 24), U32 - 1, 1 << 20)
    cols["v32"][n // 2] = U32 - 1
    # v64: negatives and values past 2^32, with a spread (value arrays past the 32-bit range)
    cols["v64"] = np.where(rng.random(n) < 0.7, rng.choice(np.asarray(V64_POOL, np.int64), n),
                           rng.integers(-(1 << 35), 1 << 35, n))
    valid["v64"] = gappy(0.1)
    cols["vs"] = np.where(rng.random(n) < 0.1, rng.choice(np.asarray([-1, 0, U32 - 1, U32], np.int64), n),
                          rng.integers(-3, 300, n))
    valid["vs"] = gappy(0.1, tail=min(n // 10, 100))
    if blk % 2 == 0:  # absent from every odd block
        cols["ab"] = rng.integers(-50, 50, n)
    cols["sp"] = _strs(rng, "s", 40, n)
    cols["sp"][r % 50 == 7] = ""
    cols["sp"][n // 3] = "only%d" % blk
    valid["sp"] = rng.random(n) > 0.15 if n > 1 else full.copy()
    cols["sc"] = _strs(rng, "s", 60, n)
    cols["sc"][r % 40 == 3] = ""
    cols["sm"] = _strs(rng, "m", 600, n, "%s%03d")
    cols["sv"] = _strs(rng, "s", 2000, n)
    valid["sv"] = gappy(0.1, tail=min(n // 10, 100))
    if blk == 0:  # every string but the last, in the first block
        d33, d65 = np.resize(np.asarray(D33[:-1]), n), np.resize(np.asarray(D65[:-1]), n)
    else:
        d33, d65 = rng.choice(np.asarray(D33[:-1]), n), rng.choice(np.asarray(D65[:-1]), n)
        if blk >= 2:
            d33[r % 7 == 1], d65[r % 5 == 2] = D33[-1], D65[-1]
            d33[0], d65[0] = D33[-1], D65[-1]
    cols["d33"], cols["d65"] = d33, d65
    valid["d33"] = valid["d65"] = rng.random(n) > 0.05 if n > 1 else full.copy()
    for i, c in enumerate(P_CODES):
        cols[c] = rng.integers(0, 20, n) + 10 * i
    return cols, valid


def _table(sizes, forms, seed):
    rng = np.random.default_rng(seed)
    t = _Table(forms, KT_P)
    plan = [(n, f) for n in sizes for f in ("bucket", "values")]
    for blk, (n, f) in enumerate(plan):
        cols, valid = _block(rng, n, f, blk)
        t.add(cols, valid, threshold=P_BUCKET if f == "bucket" else 0)
    t.extents(v=(0, 1000))
    return t


def sweep_literals(spec, c):
    lo, hi = spec.IntInfo[c]
    return sorted({lo - 1, lo, hi, hi + 1, -1, 0, U32 - 1, U32})


FAIL = {c: "fail_mode=%d " % (0 if c == "bp" else 1) for c in P_INT}


def _int_sweep(s):
    qs = []
    for c in P_INT:
        for op in ("gt", "lt", "eq", "neq"):
            for lit in sweep_literals(s, c):
                qs.append(_q(s, int_filters=[(c, op, lit)], groups=[c], aggs=["v"], op="avg", expect=[FAIL[c]]))
    return qs


def _str_sweep(s):
    qs = []
    for c in P_STR:
        for op in ("eq", "neq"):
            for lit in STR_LITERALS[c]:
                qs.append(_q(s, str_filters=[(c, op, lit)], groups=[c], aggs=["v"], op="avg"))
        for op in ("re", "nre"):
            for pat in STR_PATTERNS[c]:
                qs.append(_q(s, str_filters=[(c, op, pat)], groups=[c], aggs=["v"], op="avg"))
    return qs


def _shapes(s):
    bd_lo, bd_hi = s.IntInfo["bd"]
    odd = bd_lo + 301  # inside the extents, no row holds it: every bin fails
    avg = dict(aggs=["v"], op="avg")
    code5 = [("c0", "neq", 3), ("c1", "gt", 12), ("c2", "lt", 37), ("c3", "neq", 41), ("c4", "gt", 40)]
    code9 = code5 + [("c5", "lt", 66), ("c6", "neq", 70), ("c7", "gt", 70), ("c8", "neq", 95)]
    # count mode (bp lists some rows only): the pass counter is 1, 2, 3 or 4 bits wide
    count = [("bp", "neq", 77)] + code9 + [("bc", "gt", -100), ("bd", "neq", bd_lo + 2), ("v32", "gt", 0),
                                           ("v64", "neq", 1), ("vs", "lt", 299)]
    qs = [
        _q(s, int_filters=[("bd", "gt", bd_lo + 100), ("bd", "lt", bd_hi - 100)], groups=["bd"], expect=["fail_mode=1 "],
           **avg),
        _q(s, int_filters=[("v32", "gt", U32 - 20000), ("v32", "lt", U32 - 1)], groups=["g"], expect=["fail_mode=1 "],
           **avg),
        _q(s, int_filters=[("v64", "gt", -2), ("v64", "lt", U32 + 1)], groups=["v64"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bc", "eq", 200), ("bc", "neq", 200)], groups=["g"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bp", "eq", 77), ("bp", "neq", 77)], groups=["g"], expect=["fail_mode=0 "], **avg),
        _q(s, str_filters=[("sc", "eq", "s1"), ("sc", "neq", "s1")], groups=["g"], **avg),
        _q(s, str_filters=[("sv", "re", "^s1"), ("sv", "nre", "^s1")], groups=["g"], **avg),
        _q(s, int_filters=[("bd", "gt", bd_lo + 50)] * 2, groups=["bd"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("vs", "lt", 100)] * 2, str_filters=[("sp", "nre", "^s1")] * 2, groups=["g"],
           expect=["fail_mode=0 "], **avg),
        # the filter column is also the group, the aggregation and the time column
        _q(s, int_filters=[("bc", "gt", 10)], groups=["bc"], aggs=["bc"], op="avg", time_col="bc", time_bucket=50,
           expect=["fail_mode=1 "]),
        _q(s, int_filters=[("v32", "lt", U32 - 100)], groups=["g"], aggs=["v32"], op="avg", time_col="v32",
           time_bucket=1 << 21, expect=["fail_mode=1 "]),
        _q(s, int_filters=[("bd", "neq", bd_lo + 4)], groups=["bd"], aggs=["bd"], op="hist", expect=["fail_mode=1 "]),
        _q(s, int_filters=[("v64", "gt", -1)], groups=["g"], aggs=["v64"], op="avg", expect=["fail_mode=1 "]),
        # code-column filters only: 5 and 9 code pass tables, those after the fourth in global memory
        _q(s, int_filters=code5, expect=["fail_mode=1 ", r"codes=5\b"], aggs=[], op="avg"),
        _q(s, int_filters=code9, expect=["fail_mode=1 ", r"codes=9\b"], aggs=[], op="avg"),
        _q(s, int_filters=code9, str_filters=[("sc", "nre", "^s1")], groups=["g"], expect=["fail_mode=1 "], **avg),
        # fail mode where every bin fails (an odd literal: the zone maps keep every block) and where none does
        _q(s, int_filters=[("bd", "eq", odd)], groups=["g"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bd", "neq", odd)], groups=["g"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bd", "gt", bd_lo - 1), ("bc", "neq", 1)], groups=["bd"], expect=["fail_mode=1 "], **avg),
    ]
    for nf in (1, 3, 4, 7, 8, 15):
        qs.append(_q(s, int_filters=count[:nf], groups=["g"], expect=["fail_mode=0 "], **avg))
    qs.append(_q(s, int_filters=count[:14], str_filters=[("d33", "nre", "^p")], groups=["g"], expect=["fail_mode=0 "],
                 **avg))
    return qs


def _zone_maps(s):
    """Literals equal to a block's own min and max (IntInfo of one block), next to the table's."""
    qs = []
    for c in ("bp", "v64", "bd"):
        lits = set()
        for b in s.blocks[:4]:
            mm = b.info.get(s.KeyTable[c])
            if mm:
                lits |= set(mm)
        for lit in sorted(lits):
            for op in ("gt", "lt", "eq"):
                qs.append(_q(s, int_filters=[(c, op, lit)], groups=["g"], aggs=["v"], op="avg", expect=[FAIL[c]]))
    return qs


def _replace(s):
    """StrReplace on sc: s1<x> -> q<x> (merging s1 with s1x...), s3 -> "" (the "" of the dictionary).  The C++ oracle
    looks eq / neq literals up in the rewritten table as the reference does, keeping one of the merged ids
    (DESIGN.md §7): it is not compared."""
    qs = []
    for rep in ({"sc": ("^s1", "q")}, {"sc": ("^s3$", "")}):
        for op, lit in (("eq", "q"), ("neq", "q"), ("eq", ""), ("neq", ""), ("re", "^q"), ("nre", "^q"),
                        ("re", "^$"), ("nre", "^$")):
            q = _q(s, str_filters=[("sc", op, lit)], groups=["g"], aggs=["v"], op="avg", str_replace=rep)
            q.oracle = False
            qs.append(q)
    return qs


def family_p_sweep(forms=None):
    t = _table(SWEEP_SIZES, forms, 71)
    s = t.spec
    return t.done(_int_sweep(s) + _str_sweep(s) + _shapes(s) + _zone_maps(s) + _replace(s))


def family_p_geom(forms=None):
    """Full blocks (65,536 and 65,535 rows) in both forms: bd's 900 bins straddle the 1,024-entry tiles, so a failing
    bin pushes down to the tiles that hold it."""
    t = _table(GEOM_SIZES, forms, 72)
    s = t.spec
    bd_lo, bd_hi = s.IntInfo["bd"]
    avg = dict(aggs=["v"], op="avg")
    return t.done([
        _q(s, int_filters=[("bd", "neq", bd_lo + 900)], groups=["g"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bd", "gt", bd_lo + 20)], groups=["bd"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bd", "lt", bd_hi - 20)], str_filters=[("sm", "neq", "m001")], groups=["g"],
           expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bd", "eq", bd_lo + 2), ("v32", "lt", U32 - 1)], groups=["g"], expect=["fail_mode=1 "],
           **avg),
        _q(s, int_filters=[("v32", "eq", U32 - 1)], groups=["g"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("vs", "lt", 1), ("v64", "gt", -1)], groups=["g"], expect=["fail_mode=1 "], **avg),
        _q(s, int_filters=[("bp", "gt", 0), ("bc", "lt", 50)], groups=["bc"], expect=["fail_mode=0 "], **avg),
        _q(s, str_filters=[("sc", "re", "1$"), ("sv", "nre", "^s1")], groups=["g"], expect=["fail_mode=1 "], **avg),
        _q(s, str_filters=[("sp", "eq", "s3"), ("sc", "neq", "")], groups=["sc"], expect=["fail_mode=0 "], **avg),
        _q(s, int_filters=[("c0", "neq", 3), ("c1", "gt", 12), ("c2", "lt", 37), ("c3", "neq", 41), ("c4", "gt", 40),
                           ("c5", "lt", 66)], expect=["fail_mode=1 ", r"codes=6\b"], aggs=[], op="avg"),
    ])


P_TABLES = {"P-sweep": family_p_sweep, "P-geom": family_p_geom}
