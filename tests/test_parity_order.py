"""Result shaping on the GPU: order, limit and ties (tests/edges.py family L), weights (W) and StrReplace (R)
against the row-level reference tests/rowref.py and, where comparable, the oracle.  Every query asserts which
selection built its result from the `sg_select:` trace line.  L runs dense and through the hashed slot space;
where one query can take two selection paths (the device top-K or the host, the host on one thread or many)
the lists must be identical."""
import re

import pytest

from tests import edges, rowref
from tests.test_parity_edges import _mean_comparable
from tests.util import compare, run_gpu, run_oracle

pytestmark = pytest.mark.gpu

_TABLES, _REF, _ORC = {}, {}, {}


def _table(name):
    if name not in _TABLES:
        _TABLES[name] = edges.ORDER_TABLES[name]()
    return _TABLES[name]


def _listing(g):
    """The whole result as a comparable value: Sorted with every group's counters, NumGroups, Cumulative."""
    def grp(r):
        return (r.GroupByKey, r.Count, r.Samples,
                sorted((a, h.TotalCount(), h.Sum()) for a, h in r.Hists.items()))
    return [grp(r) for r in g.Sorted], g.NumGroups, grp(g.Cumulative)


def _run_one(name, i, monkeypatch, capfd, env=()):
    spec, rows, valid, queries = _table(name)
    q = queries[i]
    if (name, i) not in _REF:
        _REF[name, i] = rowref.run(spec, rows, valid, q)
        _ORC[name, i] = run_oracle(spec, q) if getattr(q, "oracle", True) else None
    ref, o = _REF[name, i], _ORC[name, i]
    for k in env:
        monkeypatch.setenv(k, env[k] if isinstance(env, dict) else "1")
    capfd.readouterr()
    g = run_gpu(spec, q)
    trace = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("sg_select:")]
    for k in env:
        monkeypatch.delenv(k)
    where = (name, i, tuple(env))
    assert g.BrokenBlocks == 0, where
    rowref.check(ref, g, q, where=where)
    # the oracle's mean order is its float running mean, and without an order its first `limit` groups are any
    if o is not None and (q.order_by == "$COUNT" or not q.order_by and not q.limit):
        compare(g, o, q, mean=_mean_comparable)
    assert len(trace) == 1, (where, trace)
    return g, trace[0]


def _run(name, monkeypatch, capfd, variant=16, env=()):
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    monkeypatch.setenv("SG_VARIANT", str(variant))
    hashed = "SG_FORCE_HASHED_SLOTS" in env
    for i, q in enumerate(_table(name)[3]):
        _, line = _run_one(name, i, monkeypatch, capfd, env)
        # the hashed slot space has no device top-K (its keys come from the table read-back)
        pats = [r"^sg_select: path=host "] if hashed else q.expect
        assert any(re.search(p, line) for p in pats), ((name, i, env), pats, line)


@pytest.mark.parametrize("name", ["L-small", "L-large"])
def test_order_limit_ties(name, monkeypatch, capfd):
    _run(name, monkeypatch, capfd)


@pytest.mark.parametrize("name", ["L-small", "L-large"])
def test_order_limit_ties_hashed(name, monkeypatch, capfd):
    _run(name, monkeypatch, capfd, env=("SG_FORCE_HASHED_SLOTS",))


def test_selection_paths_agree(monkeypatch, capfd):
    """The L-large queries the device selects: the same lists from the host on many threads (SG_NO_GPU_TOPK) and
    on one (SG_HOST_THREADS=1); the cap / cap + 1 pair reaches the device and its fall-back."""
    monkeypatch.setenv("SG_PLAN_TRACE", "1")
    queries = _table("L-large")[3]
    paths = set()
    for i, q in enumerate(queries):
        g, line = _run_one("L-large", i, monkeypatch, capfd)
        paths.add(line.split()[1])
        if "path=device" not in line and "path=device-fallback" not in line:
            continue
        many = _run_one("L-large", i, monkeypatch, capfd, {"SG_NO_GPU_TOPK": "1"})
        one = _run_one("L-large", i, monkeypatch, capfd, {"SG_NO_GPU_TOPK": "1", "SG_HOST_THREADS": "1"})
        assert re.search(r"path=host threads=([2-9]|1\d)$", many[1]), many[1]
        assert one[1] == "sg_select: path=host threads=1", one[1]
        assert _listing(g) == _listing(many[0]) == _listing(one[0]), (i, "paths disagree")
    assert {"path=device", "path=device-fallback", "path=host"} <= paths, paths


@pytest.mark.parametrize("variant", [8, 16])
def test_weights(variant, monkeypatch, capfd):
    _run("W", monkeypatch, capfd, variant)


def test_str_replace_order_limit(monkeypatch, capfd):
    _run("R", monkeypatch, capfd)
