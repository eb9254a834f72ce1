"""Filters on the GPU: family P (tests/family_p.py) against the row-level reference tests/rowref.py, the oracle and
SkippedBlocks, with each query's SG_PLAN_TRACE `expect` patterns, on both kernel builds and both array forms; then
every query again under each plan switch, which must give the same result field for field.

Then regex filters over a dictionary that grows after the match bitset was set (sg_query_set_str_lut): a prepared
query, the raw ABI and the streaming path.  A string interned later has no bit, so a stale bitset would drop its
rows under re and keep them under nre; planning refuses such a bitset and a prepared query sets it again."""
import ctypes as C
import re

import numpy as np
import pytest

from sybil_b200 import _ffi as F
from sybil_b200 import engine as E
from tests import edges, family_p, rowref
from tests.test_parity_codes import _fingerprint
from tests.test_parity_edges import _mean_comparable
from tests.util import INT, STR, compare, run_gpu, run_oracle

pytestmark = pytest.mark.gpu

SWITCHES = ["SG_NO_FAIL_MODE", "SG_NO_PUSHDOWN", "SG_NO_CODES", "SG_NO_TMA", "SG_FORCE_HASHED_SLOTS"]
_TABLES, _REF, _ORC, _DEFAULT = {}, {}, {}, {}


def _table(name, forms):
    if (name, forms) not in _TABLES:
        _TABLES[name, forms] = family_p.P_TABLES[name](forms)
    return _TABLES[name, forms]


def _staged(spec):
    table = E.Table("p", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    for b in spec.blocks:
        table.add_block(b)
    return table


def _runs(name, forms, monkeypatch, capfd, variant, env=()):
    """Every query of table `name` on one staged table: yields (index, query, result, plan trace lines)."""
    spec, rows, valid, queries = _table(name, forms)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    for k in env:
        monkeypatch.setenv(k, "1")
    table = _staged(spec)  # (staging reads SG_NO_CODES and SG_NO_TMA)
    try:
        for i, q in enumerate(queries):
            if "SG_FORCE_HASHED_SLOTS" in env and q.str_replace:
                continue  # (StrReplace over a hashed slot space is refused)
            capfd.readouterr()
            g = run_gpu(spec, q, table)
            trace = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("sg_plan:")]
            yield i, q, g, trace
    finally:
        table.close()


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("forms", ["narrow", "wide"])
@pytest.mark.parametrize("name", list(family_p.P_TABLES))
def test_filters(name, forms, variant, monkeypatch, capfd):
    spec, rows, valid, queries = _table(name, forms)
    nblocks = len(spec.blocks)
    for i, q, g, trace in _runs(name, forms, monkeypatch, capfd, variant):
        # rowref and the oracle depend on neither the array form nor the build: computed once per query
        if (name, i) not in _REF:
            _REF[name, i] = rowref.run(spec, rows, valid, q)
            _ORC[name, i] = run_oracle(spec, q) if getattr(q, "oracle", True) else None
        ref, o = _REF[name, i], _ORC[name, i]
        where = (name, forms, variant, i, q.int_filters, q.str_filters)
        assert g.BrokenBlocks == 0, where
        assert g.SkippedBlocks == ref.SkippedBlocks, (where, "skipped blocks")
        rowref.check(ref, g, q, where=where)
        if o is not None:
            compare(g, o, q, mean=_mean_comparable)
        if ref.SkippedBlocks < nblocks:  # (a query whose blocks the zone maps all drop launches nothing)
            assert trace, (where, "no SG_PLAN_TRACE line")
            for pat in q.expect:
                assert any(re.search(pat, ln) for ln in trace), (where, pat, trace)


@pytest.mark.parametrize("env", SWITCHES)
@pytest.mark.parametrize("name", list(family_p.P_TABLES))
def test_filters_switches(name, env, monkeypatch, capfd):
    """The same answers with fail mode off, push-down off (every tile walked), without per-row codes, without TMA
    loads and over the hashed slot space."""
    if name not in _DEFAULT:
        _DEFAULT[name] = {i: _fingerprint(g) for i, _, g, _ in _runs(name, None, monkeypatch, capfd, 16)}
    for i, q, g, trace in _runs(name, None, monkeypatch, capfd, 16, (env,)):
        where = (name, env, i, q.int_filters, q.str_filters)
        assert _fingerprint(g) == _DEFAULT[name][i], where
        if env == "SG_NO_FAIL_MODE":
            assert all("fail_mode=0 " in ln for ln in trace), (where, trace)
        if env == "SG_NO_CODES":
            assert all(re.search(r"codes=0\b", ln) for ln in trace), (where, trace)


# ---------------------------------------------------------------------------------------------------------------
# a dictionary that grows after the regex bitset was set
# ---------------------------------------------------------------------------------------------------------------
KT_GROW = [("s", STR), ("v", INT)]


def _grow_table():
    """A first block of s0..s9, then blocks that bring s1new / s1z (matching ^s1) and x5 / x6 (not matching)."""
    t = edges._Table(None, KT_GROW)
    rng = np.random.default_rng(81)
    n = 2000
    t.add({"s": np.array(["s%d" % x for x in rng.integers(0, 10, n)]), "v": rng.integers(0, 100, n)},
          {"s": rng.random(n) > 0.05})
    first = len(t.spec.blocks)
    for new in (["s1new", "x5"], ["s1z", "x6"]):
        s = np.where(rng.random(n) < 0.5, rng.choice(np.asarray(new), n),
                     np.array(["s%d" % x for x in rng.integers(0, 10, n)]))
        t.add({"s": s, "v": rng.integers(0, 100, n)}, {"s": rng.random(n) > 0.05}, threshold=5)
    t.extents(v=(0, 100))
    return t, first


def _upto(t, nblocks):
    """rowref's (rows, valid) for the first add() calls holding `nblocks` blocks (one block per call here)."""
    return t.rows[:nblocks], t.valid[:nblocks]


GROW_FILTERS = [("s", "re", "^s1"), ("s", "nre", "^s1"), ("s", "eq", "s1new")]


@pytest.mark.parametrize("flt", GROW_FILTERS, ids=lambda f: f[1])
def test_prepared_query_over_a_growing_dictionary(flt):
    t, first = _grow_table()
    spec = t.spec
    q = edges._q(spec, str_filters=[flt], groups=["s"], aggs=["v"], op="avg")
    table = E.Table("grow", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    try:
        for b in spec.blocks[:first]:
            table.add_block(b)
        qs = q.query_spec()
        ls = table.NewLoadSpec()
        ls.Str("s")
        ls.Int("v")
        pq = table.Prepare(ls, qs)
        try:
            pq.Run(qs)
            rowref.check(rowref.run(spec, *_upto(t, first), q), qs, q, where=(flt, "first block"))
            for b in spec.blocks[first:]:
                table.add_block(b)
            qs = q.query_spec()
            pq.Run(qs)
            rowref.check(rowref.run(spec, t.rows, t.valid, q), qs, q, where=(flt, "after the new strings"))
        finally:
            pq.Close()
    finally:
        table.close()


def _bits(strs, pattern):
    rx = re.compile(pattern)
    bits = np.zeros((len(strs) + 31) // 32 + 1, np.uint32)
    for gid, s in enumerate(strs):
        if rx.search(s.decode()):
            bits[gid >> 5] |= np.uint32(1 << (gid & 31))
    return bits


def _set_lut(lib, ctx, qh, table, pattern):
    strs = table.dict_strings("s")
    bits = _bits(strs, pattern)
    ctx.check(lib.sg_query_set_str_lut(qh, 0, bits.ctypes.data, len(strs)))


def _finish(table, qh, qs):
    rp = C.c_void_p()
    table.ctx.check(table.lib.sg_query_finish(qh, C.byref(rp)))
    try:
        table._fill(qs, rp)
    finally:
        table.lib.sg_result_free(rp)
    return qs


def _refused(ctx, rc):
    assert rc == F.SG_ERR_STATE, ("a bitset older than the dictionary must be refused", rc)
    assert "filter 0" in ctx.err(), ctx.err()


@pytest.mark.parametrize("op", ["re", "nre"])
def test_raw_abi_stale_regex_bitset(op):
    """sg_query_run after blocks brought new strings: refused with the stale bitset, right once it is set again."""
    t, first = _grow_table()
    spec = t.spec
    q = edges._q(spec, str_filters=[("s", op, "^s1")], groups=["s"], aggs=["v"], op="avg")
    table = E.Table("grow", spec.key_table)
    table.IntInfo = dict(spec.IntInfo)
    lib, ctx = table.lib, table.ctx
    try:
        for b in spec.blocks[:first]:
            table.add_block(b)
        d, keep = q.desc()
        qh = lib.sg_query_begin(ctx.h, table.h, C.byref(d))
        assert qh, ctx.err()
        try:
            _set_lut(lib, ctx, qh, table, "^s1")
            ctx.check(lib.sg_query_run(qh))
            rowref.check(rowref.run(spec, *_upto(t, first), q), _finish(table, qh, q.query_spec()), q, where="first")
            for b in spec.blocks[first:]:
                table.add_block(b)
            _refused(ctx, lib.sg_query_run(qh))
            _set_lut(lib, ctx, qh, table, "^s1")
            ctx.check(lib.sg_query_run(qh))
            rowref.check(rowref.run(spec, t.rows, t.valid, q), _finish(table, qh, q.query_spec()), q, where="re-set")
        finally:
            lib.sg_query_free(qh)
    finally:
        table.close()


@pytest.mark.parametrize("op", ["re", "nre"])
def test_streaming_stale_regex_bitset(op):
    """sg_query_submit_block stages blocks that bring new strings: a bitset set before the submits is refused at
    sg_query_finish, one set after them answers over every block."""
    t, first = _grow_table()
    spec = t.spec
    q = edges._q(spec, str_filters=[("s", op, "^s1")], groups=["s"], aggs=["v"], op="avg")
    for lut_after in (False, True):
        table = E.Table("grow", spec.key_table)
        table.IntInfo = dict(spec.IntInfo)
        lib, ctx = table.lib, table.ctx
        try:
            for b in spec.blocks[:first]:
                table.add_block(b)
            d, keep = q.desc()
            qh = lib.sg_query_begin(ctx.h, table.h, C.byref(d))
            assert qh, ctx.err()
            try:
                if not lut_after:
                    _set_lut(lib, ctx, qh, table, "^s1")
                descs = [b.desc() for b in spec.blocks[first:]]
                for dd in descs:
                    ctx.check(lib.sg_query_submit_block(qh, C.byref(dd)))
                if lut_after:
                    _set_lut(lib, ctx, qh, table, "^s1")
                    got = _finish(table, qh, q.query_spec())
                    rowref.check(rowref.run(spec, t.rows, t.valid, q), got, q, where="bitset after the submits")
                else:
                    rp = C.c_void_p()
                    _refused(ctx, lib.sg_query_finish(qh, C.byref(rp)))
            finally:
                lib.sg_query_free(qh)
        finally:
            table.close()
