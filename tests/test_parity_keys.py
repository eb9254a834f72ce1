"""The key side of the scan on the GPU: group keys, the slot-word layout and the thresholds inside the pass
(tests/edges.py families G, H and K) against the row-level reference tests/rowref.py and the oracle.  Both kernel
builds; narrow and wide array forms where the key columns are decoded; every family also through the hashed slot
space (SG_FORCE_HASHED_SLOTS), which must give what the dense one gives.  Refusals are checked by status."""
import re

import numpy as np
import pytest

from sybil_b200 import _ffi as F
from sybil_b200 import engine as E
from tests import edges, rowref
from tests.test_parity_edges import _mean_comparable
from tests.util import compare, run_gpu, run_oracle

pytestmark = pytest.mark.gpu

_REF, _ORC = {}, {}


def _run(name, forms, monkeypatch, capfd, variant, env=()):
    spec, rows, valid, queries = edges.KEY_TABLES[name](forms)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    for k in env:
        monkeypatch.setenv(k, "1")
    hashed = "SG_FORCE_HASHED_SLOTS" in env
    for i, q in enumerate(queries):
        if (name, i) not in _REF:
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
        for pat in [r"hashed=1 "] if hashed else getattr(q, "expect", []):
            assert any(re.search(pat, ln) for ln in trace), (where, pat, trace)


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("forms", ["narrow", "wide"])
@pytest.mark.parametrize("name", ["G-int", "G-mixed", "G-str"])
def test_keys(name, forms, variant, monkeypatch, capfd):
    _run(name, forms, monkeypatch, capfd, variant)


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("name", ["H", "K"])
def test_slot_words(name, variant, monkeypatch, capfd):
    _run(name, None, monkeypatch, capfd, variant)


@pytest.mark.parametrize("name", ["G-int", "G-mixed", "G-str", "H", "K"])
def test_hashed_slot_space(name, monkeypatch, capfd):
    _run(name, None, monkeypatch, capfd, 16, env=("SG_FORCE_HASHED_SLOTS",))


def _status(fn):
    try:
        fn()
    except E.SybilGpuError as e:
        return e.status
    return F.SG_OK


def test_refusals_leave_the_context_usable(monkeypatch, capfd):
    """A slot word wider than 32 bits is refused, and a hashed table that fills up fails the query instead of
    returning part of it; the next query on the same table answers."""
    spec, rows, valid, queries = edges.family_h()
    table = E.Table("t", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    for b in spec.blocks:
        table.add_block(b)
    try:
        q = queries[0]
        ref = rowref.run(spec, rows, valid, q)
        monkeypatch.setenv("SG_PLAN_TRACE", "1")
        capfd.readouterr()
        st = _status(lambda: run_gpu(spec, edges.h_refused(spec), table))
        assert st == F.SG_ERR_UNSUPPORTED, (st, capfd.readouterr().err[-2000:])
        rowref.check(ref, run_gpu(spec, q, table), q, where="after the 33-bit refusal")
        # [d, e] has 65,536 slots and rows on more than 256 of them: a 256-entry table fills up
        wide = queries[2]
        monkeypatch.setenv("SG_FORCE_HASHED_SLOTS", "1")
        monkeypatch.setenv("SG_HASH_CAP_LOG2", "8")
        assert _status(lambda: run_gpu(spec, wide, table)) == F.SG_ERR_UNSUPPORTED
        monkeypatch.delenv("SG_HASH_CAP_LOG2")
        rowref.check(rowref.run(spec, rows, valid, wide), run_gpu(spec, wide, table), wide, where="hashed, after full")
        monkeypatch.delenv("SG_FORCE_HASHED_SLOTS")
        rowref.check(ref, run_gpu(spec, q, table), q, where="after the full table")
    finally:
        table.close()


def test_value_dictionary_grows_between_runs():
    """Family J: a value-array int group column queried, then blocks with new key values (and -1) staged, then
    queried again, both by a fresh query and by re-running the prepared one.  No block may be dropped for a value
    the device dictionary did not hold yet."""
    spec, rows, valid, queries = edges.family_g_int(True)
    t = edges._Table(None, edges.KT_KEYS)
    t.spec, t.rows, t.valid = spec, list(rows), list(valid)
    q = queries[0]
    table = E.Table("t", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    for b in spec.blocks:
        table.add_block(b)
    try:
        pq = table.Prepare(None, q.query_spec())
        try:
            qs = q.query_spec()
            pq.Run(qs)
            rowref.check(rowref.run(spec, t.rows, t.valid, q), qs, q, where="before")
            rng = np.random.default_rng(30)
            n = 2000
            before = len(spec.blocks)
            k = 50000 + rng.integers(0, 900, n)
            k[:3] = [-1, -7, 1 << 50]
            t.add({"g": edges._groups(rng, n, 2), "k": k, "t": rng.integers(0, 1500, n),
                   "v0": rng.integers(0, 100, n)}, {"k": rng.random(n) > 0.05}, threshold=50)
            for b in spec.blocks[before:]:
                table.add_block(b)
            ref = rowref.run(spec, t.rows, t.valid, q)
            qs = q.query_spec()
            pq.Run(qs)
            assert qs.BrokenBlocks == 0
            rowref.check(ref, qs, q, where="prepared query re-run")
        finally:
            pq.Close()
        g = run_gpu(spec, q, table)
        assert g.BrokenBlocks == 0
        rowref.check(ref, g, q, where="fresh query")
    finally:
        table.close()


@pytest.mark.parametrize("name", ["I-dense", "I-hashed", "I-ceiling"])
def test_dense_hashed_switch_and_code_ceiling(name, monkeypatch, capfd):
    _run(name, None, monkeypatch, capfd, 16)


def test_slot_space_refusals(monkeypatch):
    """Past the code ceiling (a time axis on 2^31 - 2 codes, a product past it) and past the 24 GiB accumulator
    limit (histograms over 2^26 dense slots) the planner refuses; the next query on the same table answers."""
    for build, refused in ((edges.family_i_ceiling, edges.i_refused),
                           (lambda: edges.family_i_dense(False), lambda s: [edges.i_dense_hist(s)])):
        spec, rows, valid, queries = build()
        table = E.Table("t", spec.key_table)
        table.IntInfo = dict(spec.IntInfo)
        for b in spec.blocks:
            table.add_block(b)
        try:
            for bad in refused(spec):
                assert _status(lambda: run_gpu(spec, bad, table)) == F.SG_ERR_UNSUPPORTED
                q = queries[-1]
                rowref.check(rowref.run(spec, rows, valid, q), run_gpu(spec, q, table), q, where="after a refusal")
        finally:
            table.close()


def test_value_dictionary_at_its_cap():
    """Family J at INT_DICT_CAP: 2^22 distinct values of a value-array group column (64 full blocks) are accepted,
    with every group's Count equal to np.unique's over the rows the filter keeps; a block adding more refuses the
    next query."""
    from tests.util import INT, Q, Spec
    spec = Spec([("k", INT), ("f", INT)])
    n = 1 << 22
    vals = np.arange(n, dtype=np.int64) * 3 + 5
    rng = np.random.default_rng(22)
    k = rng.permutation(vals)
    spec.add_rows({"k": k, "f": np.arange(n) % 4096}, threshold=1000, block_rows=65536)
    q = Q(spec, int_filters=[("f", "eq", 2)], groups=["k"], aggs=[], op="avg")
    table = E.Table("t", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    for b in spec.blocks:
        table.add_block(b)
    try:
        qs = run_gpu(spec, q, table)
        keep = k[np.arange(n) % 4096 == 2]
        u, c = np.unique(keep, return_counts=True)
        assert qs.BrokenBlocks == 0 and qs.NumGroups == len(u) and qs.MatchedCount == len(keep)
        got = {int(key.rstrip("\t")): r.Count for key, r in qs.Results.items()}
        assert got == dict(zip(u.tolist(), c.tolist()))
        before = len(spec.blocks)
        spec.add_rows({"k": np.arange(100, dtype=np.int64) * 3 + 3 * n + 5, "f": np.full(100, 2)}, threshold=10)
        for b in spec.blocks[before:]:
            table.add_block(b)
        assert _status(lambda: run_gpu(spec, q, table)) == F.SG_ERR_UNSUPPORTED
    finally:
        table.close()


def test_str_replace_to_empty_joins_the_missing_group():
    """On a StrReplace column the strings rewritten to "" render like a missing value and are the missing group,
    as pyoracle (which groups by the rendered key) has them; no two groups may share a key."""
    from tests.test_oracle_vs_py import py_query
    spec, rows, valid, queries = edges.family_g_str()
    for pat in ("^a$", "^[ab]$"):
        q = edges._q(spec, groups=["s"], aggs=["v0"], op="avg", str_replace={"s": (pat, "")})
        g = run_gpu(spec, q)
        want, _, _, matched, _ = py_query(spec, q)
        assert g.NumGroups == len(g.Sorted) == len(want), (pat, g.NumGroups, len(want))
        assert g.MatchedCount == matched
        assert {k: r.Count for k, r in g.Results.items()} == {k: r.Count for k, r in want.items()}, pat
