"""The oracle (oracle/oracle.cpp) and its Python restatement (oracle/pyoracle.py) against the row-level reference
tests/rowref.py on the heavy set-column tables of tests/family_s.py.  No GPU."""
import numpy as np
import pytest

from sybil_b200 import _ffi as F
from tests import family_s, rowref
from tests.test_rowref import _Py
from tests.util import run_oracle

# pyoracle walks every (tag, row) pair in Python: it is run on the first queries of each table
PY_QUERIES = 3


@pytest.mark.parametrize("name", list(family_s.S_TABLES))
def test_oracles_match_rowref_on_heavy_set_columns(name):
    spec, rows, valid, queries = family_s.S_TABLES[name]()
    for i, q in enumerate(queries):
        ref = rowref.run(spec, rows, valid, q)
        if getattr(q, "oracle", True):
            o = run_oracle(spec, q)
            assert o.SkippedBlocks == ref.SkippedBlocks and o.BrokenBlocks == 0, (name, i)
            rowref.check(ref, o, q, where=(name, i, "oracle"), order=q.order_by == "$COUNT")
        if i < PY_QUERIES:
            rowref.check(ref, _Py(spec, q), q, where=(name, i, "pyoracle"))


def _pairs(spec, name="tags"):
    slot = spec.KeyTable[name]
    return [len(c.record_ids) if c.col_slot == slot else None for b in spec.blocks for c in b.cols if c.col_slot == slot]


def test_s_tables_reach_their_shapes():
    """The pair counts, the exact-fit bin, the Values form with more than SMEM_BINS bins per segment and more than
    65,536 distinct tags, the duplicated string with its two bins more than 65,536 entries apart."""
    spec = family_s.family_s_at()[0]
    assert _pairs(spec) == [65535, 65536]
    spec = family_s.family_s_past()[0]
    assert _pairs(spec) == [65537, 131071, 131072, 131073, 80000]
    assert spec.blocks[-1].num_records == 3000 and not any(c.col_slot == 0 for c in spec.blocks[-1].cols)
    spec = family_s.family_s_full()[0]
    for b, lead in zip(spec.blocks, ([65536], [1, 65536])):
        c = next(c for c in b.cols if c.col_slot == 0)
        assert list(np.diff(c.bin_offsets.astype(np.int64))[:len(lead)]) == lead
    spec = family_s.family_s_heavy()[0]
    assert _pairs(spec)[0] > 20 * 65536
    spec = family_s.family_s_values()[0]
    for b, more in zip(spec.blocks, (5000, 65536)):
        c = next(c for c in b.cols if c.col_slot == 0)
        assert len(c.string_table) > more and c.set_nvalues == b.num_records and len(c.record_ids) > 65536
    spec = family_s.family_s_dup()[0]
    c = next(c for c in spec.blocks[0].cols if c.col_slot == 0)
    assert c.string_table[0] == c.string_table[-1] == b"dup"
    assert c.bin_offsets[-2] - c.bin_offsets[1] > 65536 and int(c.bin_values[0]) == 0 and int(c.bin_values[-1]) == 11


def test_native_reader_keeps_long_set_bins(tmp_path):
    """The block writer and the native gob reader pass a set column of more than 65,536 pairs through unchanged in
    both file forms (wide and narrow ids), with a bin longer than a block in the bucket form (the reader does not
    judge NumRecords; staging does) and one of a whole block in the Values form (which the reader bounds by a
    block)."""
    import ctypes as C
    from sybil_b200 import blockdir
    from sybil_b200 import blocks as B
    rng = np.random.default_rng(67)
    for form, threshold, n in (("bucket", 5000, 70000), ("values", 1, 65536)):
        tags = [["a"] + (["b%d" % rng.integers(0, 3)] if r % 4 == 0 else []) for r in range(n)]
        blk = B.SavedBlock(0, n)
        blk.cols.append(B.encode_set_column(0, tags, np.ones(n, bool), threshold=threshold))
        d = str(tmp_path / form)
        blockdir.write_block_dir(d, blk, [("tags", F.SG_COL_SET)])
        g = F.gobread()
        names = (C.c_char_p * 1)(b"tags")
        types = (C.c_int32 * 1)(F.SG_COL_SET)
        for narrow in (0, 1):
            g.sgob_set_narrow(narrow)
            err = C.create_string_buffer(512)
            h = g.sgob_read_block_dir(d.encode(), names, types, 1, None, 0, err, len(err))
            assert h, err.value.decode()
            try:
                cd = g.sgob_block_desc(h).contents.cols[0]
                src = blk.cols[0]
                assert cd.nrecord_ids == len(src.record_ids) > 65536 and cd.nbins == len(src.bin_values)
                w = 2 if cd.id_bits == 16 else 4
                assert (cd.id_bits == 16) == bool(narrow)
                got = np.frombuffer(C.string_at(cd.record_ids, cd.nrecord_ids * w), np.uint16 if w == 2 else np.uint32)
                assert np.array_equal(got.astype(np.int64), src.record_ids.astype(np.int64))
                offs = np.frombuffer(C.string_at(cd.bin_offsets, (cd.nbins + 1) * 4), np.uint32)
                assert np.array_equal(offs.astype(np.int64), src.bin_offsets.astype(np.int64))
                assert max(np.diff(offs.astype(np.int64))) == n
                assert cd.nvalues == (n if form == "values" else 0)
            finally:
                g.sgob_block_free(h)
        g.sgob_set_narrow(0)
