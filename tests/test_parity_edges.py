"""The CUDA path on the edge tables of tests/edges.py, against the row-level reference tests/rowref.py and the
oracle.  Both kernel builds (SG_VARIANT 8 and 16); narrow and wide array forms where a family exercises
decoding; SG_PLAN_TRACE lines checked against each query's `expect`, so a test that targets a path shows it
reached it."""
import re

import pytest

from tests import edges, rowref
from tests.util import compare, run_gpu, run_oracle

pytestmark = pytest.mark.gpu

_REF, _ORC = {}, {}


def _tables(name, forms):
    builders = {"A": edges.family_a, "B-carry": edges.family_b_carry, "E": edges.family_e, "F": edges.family_f}
    if name.startswith("B-fold-"):
        return edges.family_b_fold(name[len("B-fold-"):], forms)
    if name[0] in "CD":
        return (edges.family_c if name[0] == "C" else edges.family_d)(forms)[int(name[1:])]
    return builders[name](forms)


def _mean_comparable(oh):
    """Whether this histogram's mean is compared (DESIGN.md §7): not where the reference's mean is NaN (the group
    combined a block whose values were all rejected) nor where the true sum left int64.  Count and the sum are
    compared bit-exact either way, against rowref and the oracle."""
    return oh.Avg == oh.Avg and abs(oh.Avg * oh.Count) < 2.0 ** 63


def _run(name, forms, monkeypatch, capfd, variant, env=()):
    spec, rows, valid, queries = _tables(name, forms)
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    for k in env:
        monkeypatch.setenv(k, "1")
    for i, q in enumerate(queries):
        # rowref and the oracle do not depend on the array form or the build: computed once per query
        if (name, i) not in _REF:
            _REF[name, i] = rowref.run(spec, rows, valid, q)
            _ORC[name, i] = run_oracle(spec, q)
        ref, o = _REF[name, i], _ORC[name, i]
        capfd.readouterr()
        g = run_gpu(spec, q)
        trace = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("sg_plan:")]
        where = (name, forms, variant, env, i)
        assert g.SkippedBlocks == ref.SkippedBlocks, (where, "skipped blocks")
        rowref.check(ref, g, q, where=where)
        compare(g, o, q, mean=_mean_comparable)
        # then the path: values first, so a wrong plan that also gives wrong values reports the values
        assert trace, (where, "no SG_PLAN_TRACE line")
        for pat in getattr(q, "expect", []):
            if "SG_NO_DEFER_FOLD" in env:
                pat = re.sub(r"fold_every=\d", "fold_every=1", pat)
            assert any(re.search(pat, ln) for ln in trace), (where, pat, trace)


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("name", ["A", "C0", "C1", "C2", "F"])
def test_edges(name, variant, monkeypatch, capfd):
    _run(name, None, monkeypatch, capfd, variant)


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("forms", ["narrow", "wide"])
@pytest.mark.parametrize("name", ["B-carry", "B-fold-below", "B-fold-above", "B-fold-fold", "B-fold-fold3", "E"])
def test_edges_decoding(name, forms, variant, monkeypatch, capfd):
    _run(name, forms, monkeypatch, capfd, variant)


@pytest.mark.parametrize("variant", [8, 16])
def test_fold_without_deferral(variant, monkeypatch, capfd):
    _run("B-fold-above", None, monkeypatch, capfd, variant, env=("SG_NO_DEFER_FOLD",))


@pytest.mark.parametrize("variant", [8, 16])
@pytest.mark.parametrize("env", [(), ("SG_NO_TIME_WINDOW",)])
@pytest.mark.parametrize("name", ["D0", "D1", "D2"])
def test_time_axis(name, env, variant, monkeypatch, capfd):
    _run(name, None, monkeypatch, capfd, variant, env)


def test_geometry_without_tma(monkeypatch, capfd):
    _run("E", "narrow", monkeypatch, capfd, 16, env=("SG_NO_TMA",))
