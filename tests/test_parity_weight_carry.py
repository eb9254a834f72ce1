"""Weighted queries over rows without the weight column (sg_query_desc.weight_carry = 1, engine.FLAGS.WEIGHT_CARRY):
such a row takes the weight of the nearest earlier row of its block that has the column, or 1 (aggregate.go:68,
100-102).  The CUDA path against the row-level reference tests/rowref.py, integer fields bit for bit, and against
the oracle where no group's weighted Count can fold to 0 (DESIGN.md §7).  Weight columns in every form a block can
hold them: per-row codes, bins walked by id, a short value array, no file at all; 8-, 16- and 32-bit slot words;
both kernel builds; the streaming path and a prepared re-run.  With the flag off the same tables are refused."""
import ctypes as C
import re

import numpy as np
import pytest

from sybil_b200 import _ffi as F
from sybil_b200 import engine as E
from tests import edges, rowref
from tests.test_parity_edges import _mean_comparable
from tests.util import INT, STR, Q, compare, run_gpu, run_oracle

KT = [("g", STR), ("h", STR), ("w", INT), ("f", INT), ("v", INT), ("t", INT)]


class CQ(Q):
    """A Q that also sets the engine's WEIGHT_CARRY flag (carry=True by default)."""

    def __init__(self, spec, carry=True, **kw):
        super().__init__(spec, **kw)
        self.carry = carry

    def set_flags(self):
        super().set_flags()
        E.FLAGS.WEIGHT_CARRY = self.carry


def _add(t, rng, n, wvals, wvalid, block_rows=None, threshold=5000, fcorr=False):
    """n rows; w drawn from wvals where wvalid.  fcorr: f >= 50 exactly on the rows that list w.  The time column
    lacks rows only in bucket form: the gaps of a value array read 0, off the planned time axis."""
    f = rng.integers(0, 100, n)
    if fcorr:
        f = np.where(wvalid, 50 + rng.integers(0, 50, n), rng.integers(0, 50, n))
    t.add({"g": edges._groups(rng, n, 3), "h": np.array(["h%d" % x for x in rng.integers(0, 12, n)]),
           "w": rng.choice(np.asarray(wvals), n), "f": f, "v": rng.integers(0, 5000, n),
           "t": 1500000000 + np.sort(rng.integers(0, 7200, n))},
          {"w": wvalid, "t": rng.random(n) > (0.05 if threshold >= 5000 else 0.0), "v": rng.random(n) > 0.03},
          block_rows=block_rows, threshold=threshold)


def _gaps(rng, n, p):
    return rng.random(n) > p


def table(kind, forms=None, seed=0):
    """(spec, rows, valid).  kind "codes": <= 255 distinct weights (per-row codes, 8-bit slot words without filters);
    "walk": 256..5,000 distinct weights (bins walked by id, 16-bit words); "values": weight value arrays shorter than
    their blocks (32-bit words); "mixed": all of them in one table; "signed": weights -3..5 with 0; "full": every row
    has the weight."""
    rng = np.random.default_rng({"codes": 1, "walk": 2, "values": 3, "mixed": 4, "signed": 5, "full": 6}[kind] + 10 * seed)
    t = edges._Table(forms, KT)
    small = (1, 2, 3, 5)
    if kind == "full":
        _add(t, rng, 9000, (1, 2, 7, 10), np.ones(9000, bool), block_rows=4000)
        return t.spec, t.rows, t.valid
    wv = {"codes": small, "signed": (-3, -1, 0, 2, 5), "walk": tuple(range(1, 3001)),
          "values": tuple(range(1, 400)), "mixed": tuple(range(1, 41))}[kind]
    thr = 50 if kind == "values" else 5000
    _add(t, rng, 1500, wv, np.zeros(1500, bool), threshold=thr)                          # leading block without w
    v = _gaps(rng, 9000, 0.25)
    v[:700] = False                                                                        # row 0, long leading run
    v[4000] = False                                                                        # row 0 of the next block
    v[6000:6300] = False
    _add(t, rng, 9000, wv, v, block_rows=4000, threshold=thr, fcorr=True)                 # partial last block
    _add(t, rng, 2500, wv, np.zeros(2500, bool), threshold=thr)                          # middle block without w
    v = np.zeros(2000, bool)
    v[-1] = True
    _add(t, rng, 2000, wv, v, threshold=thr)                                               # only the last row listed
    _add(t, rng, 3000, wv, _gaps(rng, 3000, 0.05), threshold=thr)
    if kind == "values":  # value arrays cut short: every row past the last valid one lacks w
        v = _gaps(rng, 5000, 0.1)
        v[3500:] = False
        _add(t, rng, 5000, wv, v, threshold=thr)
    if kind == "mixed":
        _add(t, rng, 6000, tuple(range(1, 3001)), _gaps(rng, 6000, 0.1))                 # id walk
        v = _gaps(rng, 5000, 0.1)
        v[4000:] = False
        _add(t, rng, 5000, tuple(range(1, 400)), v, threshold=50)                          # short value array
    _add(t, rng, 3000, wv, np.ones(3000, bool), threshold=thr)                            # fully populated
    return t.spec, t.rows, t.valid


def queries(spec, oracle=True, no_oracle=()):
    """no_oracle: queries whose weighted Count folds to 0 in some block's group (value-array gaps read weight 0 there),
    where the reference drops that block result (DESIGN.md §7)."""
    qs = [CQ(spec, groups=["g"], aggs=["v"], op="hist", weight_col="w"),
          CQ(spec, groups=["g", "w"], aggs=["w", "v"], op="avg", weight_col="w", int_filters=[("w", "gt", 2)]),
          CQ(spec, groups=["g"], aggs=["v"], op="avg", weight_col="w", int_filters=[("f", "lt", 50)]),
          CQ(spec, groups=["g"], aggs=["v"], op="hist", weight_col="w", time_col="t", time_bucket=900),
          CQ(spec, groups=["h"], aggs=["v"], op="hist", loghist=True, weight_col="w"),
          CQ(spec, groups=["h"], aggs=["v"], op="avg", weight_col="w", order_by="v", limit=5),
          CQ(spec, aggs=["v"], op="avg", weight_col="w")]
    for i, q in enumerate(qs):
        q.oracle = oracle and i not in no_oracle
    return qs


def _trace(capfd):
    return [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("sg_plan:")]


def _expected_wcarry(spec, rows, valid):
    """Blocks whose weight column leaves rows out (a block without the column needs no carry)."""
    return sum(1 for _, cells, _ in rowref.blocks(spec, rows, valid) if "w" in cells and not cells["w"][1].all())


def _check(spec, rows, valid, q, g, where):
    assert g.BrokenBlocks == 0, where
    rowref.check(rowref.run(spec, rows, valid, q), g, q, where=where)
    if q.oracle and q.order_by == "$COUNT":
        # (a block group of weighted hist Count 0 leaves the reference's running mean NaN, DESIGN.md §7)
        compare(g, run_oracle(spec, q), q, mean=_mean_comparable)


def _run_table(kind, monkeypatch, capfd, variant=16, forms=None, slot_bytes=None, oracle=True):
    spec, rows, valid = table(kind, forms)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    want = _expected_wcarry(spec, rows, valid)
    assert want > 0
    # the "values" table's value-array gaps read weight 0: its filter (f < 50 keeps just the rows without w) and its
    # time buckets find block groups whose Count folds to 0
    for i, q in enumerate(queries(spec, oracle, (2, 3) if kind == "values" else ())):
        capfd.readouterr()
        g = run_gpu(spec, q)
        trace = _trace(capfd)
        assert trace, (kind, i, "no SG_PLAN_TRACE line")
        where = (kind, variant, forms, i)
        if i == 0:  # (no filter: every block is listed)
            assert "wcarry=%d " % want in trace[0] + " ", (where, trace[0])
        if slot_bytes is not None and i == 0:
            assert "slot_bytes=%d " % slot_bytes in trace[0], (where, trace[0])
        _check(spec, rows, valid, q, g, where)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("kind,slot_bytes", [("codes", 1), ("walk", 2), ("values", 4)])
def test_weight_forms_and_slot_words(kind, slot_bytes, variant, monkeypatch, capfd):
    _run_table(kind, monkeypatch, capfd, variant, slot_bytes=slot_bytes)


@pytest.mark.gpu
@pytest.mark.parametrize("forms", ["narrow", "wide"])
@pytest.mark.parametrize("variant", [8, 16])
def test_mixed_weight_forms(forms, variant, monkeypatch, capfd):
    _run_table("mixed", monkeypatch, capfd, variant, forms)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", [8, 16])
def test_zero_and_negative_carried_weights(variant, monkeypatch, capfd):
    # a group's weighted Count can fold to 0 here: the reference's float mean then stays NaN and it drops such block
    # results when combining (DESIGN.md §7), so only the row-level reference is compared
    _run_table("signed", monkeypatch, capfd, variant, oracle=False)


def _listing(g):
    def grp(r):
        return (r.GroupByKey, r.Count, r.Samples, sorted((a, h.TotalCount(), h.Sum(), list(h.Values) if h.Values is not None
                                                           else None) for a, h in r.Hists.items()))
    tr = sorted((tb, sorted(grp(r) for r in m.values())) for tb, m in g.TimeResults.items())
    return [grp(r) for r in g.Sorted], g.NumGroups, grp(g.Cumulative), g.MatchedCount, tr


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["codes", "mixed"])
def test_without_codes_bit_for_bit(kind, monkeypatch, capfd):
    """SG_NO_CODES=1 (every column walked by its ids) gives exactly what the per-row codes give."""
    spec, rows, valid = table(kind)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    for q in queries(spec):
        monkeypatch.delenv("SG_NO_CODES", raising=False)
        capfd.readouterr()
        a = run_gpu(spec, q)
        ta = _trace(capfd)
        monkeypatch.setenv("SG_NO_CODES", "1")
        b = run_gpu(spec, q)
        tb = _trace(capfd)
        assert re.search(r" codes=[1-9]", ta[0]) and " codes=0" in tb[0], (ta[0], tb[0])
        assert _listing(a) == _listing(b)
        rowref.check(rowref.run(spec, rows, valid, q), b, q)


@pytest.mark.gpu
def test_fully_populated_tables_do_not_carry(monkeypatch, capfd):
    """wcarry=0 in the plan trace, and the carry flag changes nothing."""
    spec, rows, valid = table("full")
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    for q in queries(spec):
        capfd.readouterr()
        on = run_gpu(spec, q)
        trace = _trace(capfd)
        assert trace and all(" wcarry=0" in ln for ln in trace), trace
        q.carry = False
        off = run_gpu(spec, q)
        assert _listing(on) == _listing(off)
        _check(spec, rows, valid, q, off, "full")


@pytest.mark.gpu
def test_refused_without_the_flag_and_invalid_values(monkeypatch, capfd):
    """weight_carry = 0 keeps SG_ERR_UNSUPPORTED on the same tables, and the next query on the context answers;
    a weight_carry other than 0 or 1 is refused by sg_query_begin."""
    spec, rows, valid = table("mixed")
    t = E.Table("t", spec.key_table)
    t.IntInfo = dict(spec.IntInfo)
    for b in spec.blocks:
        t.add_block(b)
    try:
        for q in [queries(spec)[i] for i in (0, 2, 4)]:  # (1 filters the rows without w away: nothing to refuse)
            q.carry = False
            with pytest.raises(E.SybilGpuError) as e:
                run_gpu(spec, q, t)
            assert e.value.status == F.SG_ERR_UNSUPPORTED
            q.carry = True
            _check(spec, rows, valid, q, run_gpu(spec, q, t), "after the refusal")
        q = queries(spec)[0]
        d, keep = q.desc()
        assert d.weight_carry == 1
        d.weight_carry = 2
        assert not t.lib.sg_query_begin(t.ctx.h, t.h, C.byref(d))
        assert "weight_carry" in t.ctx.err()
    finally:
        t.close()


@pytest.mark.gpu
def test_streaming_and_prepared_rerun():
    """sg_query_submit_block (blocks staged one by one inside the query) and a prepared query run twice."""
    spec, rows, valid = table("mixed")
    for q in queries(spec)[:4]:
        ref = rowref.run(spec, rows, valid, q)
        t = E.Table("stream", spec.key_table)
        t.IntInfo = dict(spec.IntInfo)
        try:
            qs = q.query_spec()
            d, keep = E.make_query_desc(spec.KeyTable, spec.KeyTypes, spec.IntInfo, qs)
            assert d.weight_carry == 1
            qh = t.lib.sg_query_begin(t.ctx.h, t.h, C.byref(d))
            assert qh
            try:
                for b in spec.blocks:
                    bd = b.desc()
                    t.ctx.check(t.lib.sg_query_submit_block(qh, C.byref(bd)))
                rp = C.c_void_p()
                t.ctx.check(t.lib.sg_query_finish(qh, C.byref(rp)))
                t._fill(qs, rp)
                t.lib.sg_result_free(rp)
            finally:
                t.lib.sg_query_free(qh)
            rowref.check(ref, qs, q, where="streaming")
        finally:
            t.close()
        t = E.Table("prepared", spec.key_table)
        t.IntInfo = dict(spec.IntInfo)
        for b in spec.blocks:
            t.add_block(b)
        try:
            pq = t.Prepare(None, q.query_spec())
            try:
                for k in range(2):
                    qs = q.query_spec()
                    pq.Run(qs)
                    rowref.check(ref, qs, q, where=("prepared", k))
            finally:
                pq.Close()
        finally:
            t.close()


# ---- without a GPU ------------------------------------------------------------------------------------------------
def test_query_desc_writes_the_carry_flag():
    spec = edges._Table(None, KT).spec
    d, _ = Q(spec, aggs=["v"], weight_col="w").desc()
    assert d.weight_carry == 0  # default, and reset with the other flags
    d, _ = CQ(spec, aggs=["v"], weight_col="w").desc()
    assert d.weight_carry == 1 and E.FLAGS.WEIGHT_CARRY
    E.FLAGS.reset()
    assert E.FLAGS.WEIGHT_CARRY is False


def test_the_flag_takes_the_former_padding():
    # the layout of ABI version 4 is unchanged: weight_carry sits where the padding word was
    S = F.sg_query_desc
    assert F.SG_ABI_VERSION == 4
    assert C.sizeof(S) == 104
    assert (S.order_asc.offset, S.weight_carry.offset, S.limit.offset, S.filters.offset) == (64, 68, 72, 80)
