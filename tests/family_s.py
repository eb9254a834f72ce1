"""Family S: set columns listing more than 65,536 (tag, row) pairs in one block, which the engine stages in segments
of whole bins (DESIGN.md §4, "Set filters").  Shared by tests/test_rowref_sets.py (oracle and pyoracle against
tests/rowref.py, no GPU) and tests/test_parity_sets.py (the CUDA path against both).

Every table is built from raw per-row tag lists (`blocks.encode_set_column` through `Spec.add_rows`, or
`blocks.set_values_to_bins`), so rowref sees the rows and not the encoding.  Each constructor returns
(spec, rows, valid, queries) like tests/edges.py; a query's `expect` holds patterns for its SG_PLAN_TRACE line, and
`oracle = False` marks a table where the oracle restates a documented divergence (DESIGN.md §7)."""
import numpy as np

from sybil_b200 import blocks as B
from tests.edges import _q, _Table
from tests.util import INT, SET, STR

KT = [("tags", SET), ("g", STR), ("k", INT), ("u", INT), ("v", INT), ("t", INT)]
SEGS_ONE = r"set_segs=1\b"
SEGS_MANY = r"set_segs=([2-9]|\d\d+)\b"


def _tags_with_total(rng, n, ntags, pairs):
    """n rows whose sets hold `pairs` tags in all, drawn without repetition from t0 .. t<ntags-1>."""
    k = np.full(n, pairs // n)
    k[:pairs % n] += 1
    assert k.max() <= ntags
    names = np.array(["t%d" % i for i in range(ntags)])
    return [list(names[rng.permutation(ntags)[:int(x)]]) for x in k]


def _other_cols(rng, n, t0):
    return {"g": np.array(["g%d" % x for x in rng.integers(0, 4, n)]), "k": rng.integers(0, 300, n),
            "u": rng.integers(0, 1 << 20, n), "v": rng.integers(0, 10000, n), "t": t0 + np.sort(rng.integers(0, 3000, n))}


def _add(t, rng, tags, t0, tag_valid=None, threshold=5000):
    n = len(tags)
    cols = _other_cols(rng, n, t0)
    cols["tags"] = tags
    valid = {"k": rng.random(n) > 0.05}
    if tag_valid is not None:
        valid["tags"] = tag_valid
    t.add(cols, valid, threshold=threshold)


def _queries(s, first, mid, last, expect, n_u=True):
    """IN / NIN on a present literal (its bin in the first, a middle and the last segment) and an absent one, two set
    filters on one column, set filters next to int / str filters, group-by, hist, loghist, time buckets and limit,
    and slot words of 8, 16 and 32 bits."""
    e = list(expect)
    avg = dict(aggs=["v"], op="avg")
    qs = [
        _q(s, set_filters=[("tags", "in", first)], groups=["g"], expect=e + [r"slot_bytes=1 "], **avg),
        _q(s, set_filters=[("tags", "nin", first)], groups=["g"], expect=e + [r"slot_bytes=1 "], **avg),
        _q(s, set_filters=[("tags", "in", mid)], groups=["g"], expect=e, **avg),
        _q(s, set_filters=[("tags", "nin", mid)], expect=e, **avg),
        _q(s, set_filters=[("tags", "in", last)], groups=["g"], expect=e, **avg),
        _q(s, set_filters=[("tags", "nin", last)], groups=["g"], expect=e, **avg),
        _q(s, set_filters=[("tags", "in", "absent")], groups=["g"], expect=e, **avg),
        _q(s, set_filters=[("tags", "nin", "absent")], groups=["g"], expect=e, **avg),
        _q(s, set_filters=[("tags", "in", mid), ("tags", "nin", last)], groups=["g"], expect=e, **avg),
        _q(s, int_filters=[("v", "gt", 2000)], str_filters=[("g", "neq", "g1")], set_filters=[("tags", "in", last)],
           groups=["g", "k"], aggs=["v"], op="hist", expect=e + [r"slot_bytes=2 "]),
        _q(s, set_filters=[("tags", "nin", first)], groups=["g"], aggs=["v"], op="hist", loghist=True, expect=e),
        _q(s, set_filters=[("tags", "in", mid)], groups=["g"], aggs=["v"], op="avg", time_col="t", time_bucket=1000,
           expect=e),
        _q(s, set_filters=[("tags", "nin", mid)], groups=["k"], aggs=["v"], op="avg", order_by="v", limit=5, expect=e),
    ]
    if n_u:
        qs.append(_q(s, set_filters=[("tags", "in", first), ("tags", "nin", "absent")], groups=["u"], aggs=["v"],
                     op="avg", limit=20, expect=e + [r"slot_bytes=4 "]))
    return qs


def _bin_order(spec):
    """The tags of the first block's set column in bin order (first-seen order of encode_set_column)."""
    c = next(c for c in spec.blocks[0].cols if c.col_slot == spec.KeyTable["tags"])
    return [c.string_table[int(v)].decode() for v in c.bin_values]


def family_s_at(forms=None):
    """65,535 and 65,536 pairs in one block: one segment, the path of the parent build."""
    rng = np.random.default_rng(61)
    t = _Table(forms, KT)
    for i, pairs in enumerate((65535, 65536)):
        _add(t, rng, _tags_with_total(rng, 8192, 12, pairs), 1000000 + 5000 * i)
    order = _bin_order(t.spec)
    return t.done(_queries(t.spec, order[0], order[len(order) // 2], order[-1], [SEGS_ONE]))


def family_s_past(forms=None):
    """65,537 and 131,072 +- 1 pairs in one block (two and three segments), a partial block of 80,000 pairs and a
    block without the column."""
    rng = np.random.default_rng(62)
    t = _Table(forms, KT)
    for i, pairs in enumerate((65537, 131071, 131072, 131073)):
        _add(t, rng, _tags_with_total(rng, 16384, 24, pairs), 1000000 + 5000 * i)
    _add(t, rng, _tags_with_total(rng, 5000, 24, 80000), 1030000)
    _add(t, rng, [[] for _ in range(3000)], 1040000, tag_valid=np.zeros(3000, bool))
    order = _bin_order(t.spec)
    return t.done(_queries(t.spec, order[0], order[len(order) // 2], order[-1], [SEGS_MANY]))


def family_s_full(forms=None):
    """One tag on every row of a full block (a bin of exactly 65,536 entries) next to small bins: in the first block
    that bin fills the first segment exactly, in the second one a bin of one entry comes first, so the segment edge
    lies one entry past a bin edge."""
    rng = np.random.default_rng(63)
    t = _Table(forms, KT)
    n = 65536
    for first in (None, "x0"):
        tags = [["all"] + (["x%d" % (1 + int(rng.integers(0, 9)))] if rng.random() < 0.05 else []) for _ in range(n)]
        if first:
            tags[0] = [first, "all"]
        _add(t, rng, tags, 1000000)
    # (NIN "all" matches no row: every row's set holds it)
    return t.done(_queries(t.spec, "all", "x3", "x9", [SEGS_MANY], n_u=False))


def family_s_heavy(forms=None):
    """Full blocks with 2-40 tags per row drawn from 200 (bucket form, about 1.4M pairs per block, some 20
    segments), and a partial one."""
    rng = np.random.default_rng(64)
    t = _Table(forms, KT)
    names = np.array(["tag%03d" % i for i in range(200)])
    for n in (65536, 20000):
        tags = [list(names[rng.permutation(200)[:int(k)]]) for k in rng.integers(2, 41, n)]
        _add(t, rng, tags, 1000000)
    order = _bin_order(t.spec)
    return t.done(_queries(t.spec, order[0], order[len(order) // 2], order[-1], [SEGS_MANY]))


def family_s_values(forms=None):
    """The Values file form (more than 5,000 distinct tags): 6,000 distinct tags in one block, more than 65,536 in
    another (one segment then holds more than SMEM_BINS bins, whose payload spills to global scratch), rows below
    len(Values) with empty sets — populated all the same."""
    rng = np.random.default_rng(65)
    t = _Table(forms, KT)
    for n, ntags in ((30000, 6000), (40000, 200000)):
        k = rng.integers(1, 5, n)
        k[rng.random(n) < 0.1] = 0  # empty sets below the last row holding a tag
        tags = [["w%d" % x for x in set(rng.integers(0, ntags, int(m)).tolist())] for m in k]
        # literals whose bins come first, in the middle and last (bins follow the tags' first-seen order)
        tags[0] = ["m-first", "w1"]
        tags[n // 2] = ["m-mid"]
        tags[-1] = ["w2", "m-last"]
        _add(t, rng, tags, 1000000)
    return t.done(_queries(t.spec, "m-first", "m-mid", "m-last", [SEGS_MANY]))


def family_s_dup(forms=None):
    """A string listed twice in the set column's string table, its two bins in different segments (the non-bucketed
    form through set_values_to_bins).  The reference keeps the later id and never matches rows stored under the
    earlier one; the engine and rowref map both to the string (DESIGN.md §7), so the oracle is not compared."""
    from tests.util import pick_narrow
    rng = np.random.default_rng(66)
    t = _Table(forms, KT)
    n = 16384
    table = ["dup"] + ["d%d" % i for i in range(1, 11)] + ["dup"]
    ids = [sorted(set([0 if r % 2 == 0 else 11] + [int(x) for x in rng.integers(1, 11, 5)])) for r in range(n)]
    tags = [[table[i] for i in row] for row in ids]
    cols = _other_cols(rng, n, 1000000)
    cols["tags"] = tags
    # rowref reads every table through add_rows' rule: the other columns are fully valid, so the threshold
    # only decides the set column's file form (the Values form set_values_to_bins restates)
    t.spec.add_rows({k: v for k, v in cols.items() if k != "tags"}, threshold=5000)
    blk = t.spec.blocks[-1]
    c = B.set_values_to_bins(t.spec.KeyTable["tags"], ids, table)
    blk.cols.append(B.narrow_column(c) if pick_narrow(blk.block_index, c.col_slot, forms) else c)
    t.rows.append((cols, None, 0))
    t.valid.append({})
    qs = _queries(t.spec, "dup", "d5", "d10", [SEGS_MANY], n_u=False)
    for q in qs:
        q.oracle = False
    return t.done(qs)


S_TABLES = {"S-at": family_s_at, "S-past": family_s_past, "S-full": family_s_full, "S-heavy": family_s_heavy,
            "S-values": family_s_values, "S-dup": family_s_dup}
