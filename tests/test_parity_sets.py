"""Set columns with more than 65,536 (tag, row) pairs per block on the GPU (tests/family_s.py): every query against
the row-level reference tests/rowref.py and the oracle, in both kernel builds, with narrow and wide ids, dense and
through the hashed slot space, with and without tensor-map tile loads; SG_PLAN_TRACE shows whether the multi-segment
path was reached.  Then broken blocks, the staging buffer's bound, the pinned zero-copy staging path, a block near
the top of the range and block directories through the native reader."""
import ctypes as C
import re

import numpy as np
import pytest

from sybil_b200 import _ffi as F
from sybil_b200 import blocks as B
from sybil_b200 import engine as E
from tests import family_s, rowref
from tests.test_parity_edges import _mean_comparable
from tests.util import INT, SET, STR, Q, Spec, compare, run_gpu, run_oracle

pytestmark = pytest.mark.gpu

_REF, _ORC, _TABLES = {}, {}, {}


def _table(name, forms):
    if (name, forms) not in _TABLES:
        _TABLES[name, forms] = family_s.S_TABLES[name](forms)
    return _TABLES[name, forms]


def _run(name, forms, monkeypatch, capfd, variant, env=()):
    spec, rows, valid, queries = _table(name, forms)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    for k in env:
        monkeypatch.setenv(k, "1")
    hashed = "SG_FORCE_HASHED_SLOTS" in env
    for i, q in enumerate(queries):
        if (name, i) not in _REF:  # (neither depends on the array form, the build or the slot space)
            _REF[name, i] = rowref.run(spec, rows, valid, q)
            _ORC[name, i] = run_oracle(spec, q) if getattr(q, "oracle", True) else None
        ref, o = _REF[name, i], _ORC[name, i]
        capfd.readouterr()
        g = run_gpu(spec, q)
        trace = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("sg_plan:")]
        where = (name, forms, variant, env, i)
        assert g.BrokenBlocks == 0, where
        assert g.SkippedBlocks == ref.SkippedBlocks, (where, "skipped blocks")
        rowref.check(ref, g, q, where=where)
        if o is not None:
            compare(g, o, q, mean=_mean_comparable)
        assert trace, (where, "no SG_PLAN_TRACE line")
        # the slot-word patterns describe the dense layout; the hashed one always takes 32-bit words
        pats = [p for p in q.expect if not (hashed and p.startswith("slot_bytes"))] + ([r"hashed=1 "] if hashed else [])
        for pat in pats:
            assert any(re.search(pat, ln) for ln in trace), (where, pat, trace)


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("forms", ["narrow", "wide"])
@pytest.mark.parametrize("name", list(family_s.S_TABLES))
def test_heavy_set_columns(name, forms, variant, monkeypatch, capfd):
    _run(name, forms, monkeypatch, capfd, variant)


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("env", [("SG_FORCE_HASHED_SLOTS",), ("SG_NO_TMA",)])
@pytest.mark.parametrize("name", list(family_s.S_TABLES))
def test_heavy_set_columns_hashed_and_plain_loads(name, env, variant, monkeypatch, capfd):
    _run(name, None, monkeypatch, capfd, variant, env)


# ---------------------------------------------------------------------------------------------------------------
# broken blocks: a row >= NumRecords only in the last segment, a bin longer than a block, a bin longer than a
# partial block.  Each such block is reported broken and skipped, as the oracle does; the others answer.
# ---------------------------------------------------------------------------------------------------------------
def _set_spec(nblocks, n, ntags, per_row, seed, forms="wide"):
    rng = np.random.default_rng(seed)
    s = Spec([("tags", SET), ("v", INT)])
    s.forms = forms
    names = np.array(["t%d" % i for i in range(ntags)])
    for _ in range(nblocks):
        s.add_rows({"tags": [list(names[rng.permutation(ntags)[:per_row]]) for _ in range(n)],
                    "v": rng.integers(0, 1000, n)})
    s.IntInfo["v"] = (0, 999)
    return s


def _set_col(blk):
    return next(c for c in blk.cols if c.col_slot == 0)


def _first_tag(blk):
    c = _set_col(blk)
    return c.string_table[int(c.bin_values[0])].decode()


def _check_broken(s, nbroken, queries):
    t = E.Table("t", s.key_table)
    t.IntInfo = dict(s.IntInfo)
    try:
        for b in s.blocks:
            t.add_block(b)
        for q, want in queries:
            g, o = run_gpu(s, q, table=t), run_oracle(s, q)
            assert g.BrokenBlocks == o.BrokenBlocks == want, (g.BrokenBlocks, o.BrokenBlocks, want)
            compare(g, o, q)
            assert g.MatchedCount > 0
    finally:
        t.close()


@pytest.mark.parametrize("forms", ["narrow", "wide"])
def test_row_past_the_block_in_the_last_segment(forms):
    s = _set_spec(3, 16384, 16, 8, 71, forms)  # 131,072 pairs per block: two segments
    c = _set_col(s.blocks[1])
    c.record_ids = np.array(c.record_ids, copy=True)
    c.record_ids[-1] += 16384  # the last entry of the last bin, in the last segment: row >= NumRecords
    first = _first_tag(s.blocks[1])
    _check_broken(s, 1, [(Q(s, set_filters=[("tags", "in", first)], aggs=["v"], op="avg"), 1),
                         (Q(s, set_filters=[("tags", "nin", first)], aggs=["v"], op="hist"), 1),
                         (Q(s, aggs=["v"], op="avg"), 0)])


def test_bins_longer_than_their_block():
    """A bin of 65,537 entries in a full block (multi-segment staging refuses to cut it) and a bin of 1,500 entries
    in a 1,000-row block, once next to few pairs (one segment: the scan finds it) and once next to more than 65,536
    (the staging finds it)."""
    s = _set_spec(2, 4096, 8, 3, 72)
    full = B.SavedBlock(2, 65536)
    col = B.SavedColumn(0, SET, F.SG_ENC_BUCKET)
    col.delta_ids = True
    col.string_table = [b"t0", b"t1"]
    col.bin_values = np.array([0, 1], np.int64)
    long_bin = np.ones(65537, np.uint32)  # rows 0 .. 65,536
    long_bin[0] = 0
    every3 = np.full(20000, 3, np.uint32)  # rows 0, 3, ..., 59,997
    every3[0] = 0
    col.record_ids = np.concatenate([long_bin, every3])
    col.bin_offsets = np.array([0, 65537, 85537], np.uint32)
    full.cols = [col, B.encode_int_column(1, np.arange(65536) % 1000, np.ones(65536, bool))]
    s.blocks.append(full)
    for i, npairs in enumerate((3000, 70000)):
        part = B.SavedBlock(3 + i, 1000)
        col = B.SavedColumn(0, SET, F.SG_ENC_BUCKET)
        col.delta_ids = True
        nb = npairs // 1000
        col.string_table = [b"t%d" % k for k in range(nb)]
        col.bin_values = np.arange(nb, dtype=np.int64)
        per = np.ones(1000, np.uint32)
        per[0] = 0
        long_bin = np.ones(1500, np.uint32)
        long_bin[0] = 0
        col.record_ids = np.concatenate([long_bin] + [per] * (nb - 1))
        col.bin_offsets = np.concatenate([[0], 1500 + 1000 * np.arange(nb)]).astype(np.uint32)
        part.cols = [col, B.encode_int_column(1, np.arange(1000), np.ones(1000, bool))]
        s.blocks.append(part)
    _check_broken(s, 3, [(Q(s, set_filters=[("tags", "in", "t1")], aggs=["v"], op="avg"), 3),
                         (Q(s, set_filters=[("tags", "nin", "t2")], aggs=["v"], op="avg"), 3),
                         (Q(s, aggs=["v"], op="avg"), 0)])


def _giant_block(index, ntags, skip_mod, wide=True):
    """65,536 rows; bin j lists every row r with (r * 7 + j) % skip_mod != 0 (delta ids built with numpy).  Returns
    (block, membership matrix [ntags][rows] as bool)."""
    n = 65536
    r = np.arange(n)
    member = np.array([(r * 7 + j) % skip_mod != 0 for j in range(ntags)])
    col = B.SavedColumn(0, SET, F.SG_ENC_BUCKET)
    col.delta_ids = True
    col.string_table = [b"g%d" % j for j in range(ntags)]
    col.bin_values = np.arange(ntags, dtype=np.int64)
    parts, offs = [], [0]
    for j in range(ntags):
        rows = r[member[j]]
        gaps = np.diff(rows, prepend=0)
        parts.append(gaps)
        offs.append(offs[-1] + len(rows))
    col.record_ids = np.concatenate(parts).astype(np.uint32 if wide else np.uint16)
    col.bin_offsets = np.array(offs, np.uint32)
    blk = B.SavedBlock(index, n)
    blk.cols = [col, B.encode_int_column(1, r % 1000, np.ones(n, bool))]
    return blk, member


def test_block_past_the_staging_buffer_keeps_its_error():
    big, _ = _giant_block(0, 256, 1 << 30)  # 256 tags on every row: 16,777,216 wide ids = the whole 64 MiB buffer
    s = _set_spec(1, 2000, 8, 2, 73)
    s.blocks[0].block_index = 1
    t = E.Table("t", s.key_table)
    t.IntInfo = dict(s.IntInfo)
    try:
        with pytest.raises(E.SybilGpuError) as ei:
            t.add_block(big)
        assert ei.value.status == F.SG_ERR_INVALID and "staging buffer" in str(ei.value)
        t.add_block(s.blocks[0])
        q = Q(s, set_filters=[("tags", "in", "t3")], aggs=["v"], op="avg")
        compare(run_gpu(s, q, table=t), run_oracle(s, q), q)
    finally:
        t.close()


@pytest.mark.parametrize("wide", [True, False])
def test_near_the_top_of_the_range(wide):
    """About 200 tags on every row: some 13M pairs (52 MiB of wide ids) in one block, one segment per bin.  IN and NIN
    counts against numpy."""
    blk, member = _giant_block(0, 200, 97, wide)
    assert 12_000_000 < len(_set_col(blk).record_ids) and (not wide or _set_col(blk).record_ids.nbytes > 48 << 20)
    s = Spec([("tags", SET), ("v", INT)])
    s.blocks.append(blk)
    s.IntInfo["v"] = (0, 999)
    t = E.Table("t", s.key_table)
    t.IntInfo = dict(s.IntInfo)
    try:
        t.add_block(blk)
        has = member.any(0)
        for j in (0, 99, 199):
            for op, want in (("in", member[j].sum()), ("nin", (has & ~member[j]).sum())):
                g = run_gpu(s, Q(s, set_filters=[("tags", op, "g%d" % j)]), table=t)
                assert g.BrokenBlocks == 0 and g.MatchedCount == want, (j, op, g.MatchedCount, want)
        g = run_gpu(s, Q(s, set_filters=[("tags", "in", "g0"), ("tags", "nin", "g5")]), table=t)
        assert g.MatchedCount == (member[0] & ~member[5]).sum()
        assert run_gpu(s, Q(s, set_filters=[("tags", "nin", "zz")]), table=t).MatchedCount == has.sum()
        assert run_gpu(s, Q(s, set_filters=[("tags", "in", "zz")]), table=t).MatchedCount == 0
    finally:
        t.close()


def test_pinned_record_ids_stage_like_bounced_ones():
    """sg_table_add_blocks with every record_ids array inside one sg_pinned_alloc region (the span is mirrored into
    the arena and single-segment columns are read in place) answers like sg_table_add_block from pageable memory."""
    spec, rows, valid, queries = _table("S-heavy", None)
    t = E.Table("pin", spec.key_table)
    t.IntInfo = dict(spec.IntInfo)
    descs = [b.desc() for b in spec.blocks]
    sizes = [(bi, k, d.cols[k].nrecord_ids * (2 if d.cols[k].id_bits == 16 else 4))
             for bi, d in enumerate(descs) for k in range(d.ncols) if d.cols[k].encoding == F.SG_ENC_BUCKET]
    total = sum((sz + 127) // 128 * 128 for _, _, sz in sizes)
    arena = t.lib.sg_pinned_alloc(t.ctx.h, total)
    assert arena
    try:
        off = 0
        for bi, k, sz in sizes:
            C.memmove(arena + off, descs[bi].cols[k].record_ids, sz)
            descs[bi].cols[k].record_ids = arena + off
            off += (sz + 127) // 128 * 128
        ptrs = (C.POINTER(F.sg_block_desc) * len(descs))(*[C.pointer(d) for d in descs])
        t.add_blocks(ptrs, len(descs))
        t.sync()
        for i, q in enumerate(queries[:6]):
            rowref.check(rowref.run(spec, rows, valid, q), run_gpu(spec, q, table=t), q, where=("pinned", i))
    finally:
        t.close()
        t.lib.sg_pinned_free(t.ctx.h, arena)


@pytest.mark.parametrize("narrow", [False, True])
def test_heavy_set_block_directories_through_the_native_reader(tmp_path, narrow):
    """write_block_dir (set_tags.db in the bucket form and in the Values form) -> sgob_read_block_dir -> the C ABI,
    against the oracle over the blocks the directories were written from."""
    from sybil_b200 import blockdir
    rng = np.random.default_rng(74)
    s = Spec([("tags", SET), ("v", INT), ("g", STR)])
    s.forms = "wide"
    for n, ntags in ((20000, 30), (12000, 8000)):  # ~120k pairs in bins; ~72k pairs, > 5,000 tags: Values
        s.add_rows({"tags": [["x%d" % x for x in set(rng.integers(0, ntags, 6).tolist())] for _ in range(n)],
                    "v": rng.integers(0, 1000, n), "g": np.array(["g%d" % x for x in rng.integers(0, 3, n)])})
    assert [int(getattr(_set_col(b), "set_nvalues", 0)) > 0 for b in s.blocks] == [False, True]
    g = F.gobread()
    g.sgob_set_narrow(1 if narrow else 0)
    names = (C.c_char_p * len(s.key_table))(*[nm.encode() for nm, _ in s.key_table])
    types = (C.c_int32 * len(s.key_table))(*[ty for _, ty in s.key_table])
    t = E.Table("dirs", s.key_table)
    t.IntInfo = dict(s.IntInfo)
    handles = []
    try:
        for i, b in enumerate(s.blocks):
            d = str(tmp_path / ("block%d" % i))
            blockdir.write_block_dir(d, b, s.key_table, compress=(i % 2 == 1))
            err = C.create_string_buffer(512)
            h = g.sgob_read_block_dir(d.encode(), names, types, len(s.key_table), None, b.block_index, err, len(err))
            assert h, err.value.decode()
            handles.append(h)
            t.add_block_desc_ptr(g.sgob_block_desc(h))
        for q in (Q(s, set_filters=[("tags", "in", "x3")], groups=["g"], aggs=["v"], op="avg"),
                  Q(s, set_filters=[("tags", "nin", "x3")], groups=["g"], aggs=["v"], op="hist"),
                  Q(s, set_filters=[("tags", "in", "x7"), ("tags", "nin", "x1")], aggs=["v"], op="avg")):
            gq = run_gpu(s, q, table=t)
            assert gq.MatchedCount > 0
            compare(gq, run_oracle(s, q), q)
    finally:
        g.sgob_set_narrow(0)
        t.close()
        for h in handles:
            g.sgob_block_free(h)
