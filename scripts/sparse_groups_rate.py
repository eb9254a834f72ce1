"""Kernel time, live groups, accumulator bytes and read-back of sparse group accumulators
(sg_query_set_sparse_groups), with the card's name and power limit read in the same call.

    both     a group-by histogram both paths answer: 200 x 500 str keys (201 x 501 = 100,701 dense slots), `--both-blocks`
             copies of one 65,536-row block.  The dense plan and the same plan forced onto the sparse path
             (SG_FORCE_SPARSE_GROUPS=1) run alternately; their results must be identical.
    hashed   a group-by histogram refused without the flag: 5,000 x 20,000 str keys (a 1e8 key product, hashed),
             `--hashed-blocks` blocks (two 65,536-row blocks alternating, 100,000 live pairs in all).

Kernel times are the library's CUDA-event times: discovery and the id kernel from the `sg_sparse:` trace line
(SG_PLAN_TRACE), aggregation = sg_query_kernel_ms minus both.  Medians over `--runs` runs after `--warmup`.
Writes only into --out (the JSON line, and the captured trace lines while it runs).

    python scripts/sparse_groups_rate.py --out DIR [--both-blocks 1526] [--hashed-blocks 3052]
"""
import argparse
import contextlib
import ctypes as C
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N = 65536


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1])}
    except Exception:
        return {"gpu": None, "power_limit_w": None}


@contextlib.contextmanager
def stderr_to(path):
    """fd 2 (the library's trace lines) into `path` while the block runs."""
    sys.stderr.flush()
    saved = os.dup(2)
    fd = os.open(path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
    os.dup2(fd, 2)
    try:
        yield
    finally:
        sys.stderr.flush()
        os.dup2(saved, 2)
        os.close(fd)
        os.close(saved)


def make_specs(ng, ns, pairs_of_block, rng):
    """One Spec per block: columns g, s (str) and v (int 0..10^6, a histogram); block i's rows take the (g, s)
    pairs pairs_of_block[i]."""
    from tests.util import INT, STR, Spec
    g = np.array(["a%05d" % i for i in range(ng)])
    s = np.array(["b%05d" % i for i in range(ns)])
    specs = []
    for gi, si in pairs_of_block:
        sp = Spec([("g", STR), ("s", STR), ("v", INT)])
        sp.forms = "wide"
        sp.add_rows({"g": g[gi], "s": s[si], "v": rng.integers(0, 1_000_000, N)})
        sp.IntInfo["v"] = (0, 1_000_000)
        specs.append(sp)
    return specs


def stage(E, specs, nblocks):
    t = E.Table("t", specs[0].key_table)
    t.IntInfo = dict(specs[0].IntInfo)
    descs = [sp.blocks[0].desc() for sp in specs]
    for i in range(nblocks):
        d = descs[i % len(descs)]
        d.block_index = i
        t.add_block_desc_ptr(C.byref(d))
    t.sync()
    return t


def prepare(E, t, q, sparse, forced=False):
    qs = q.query_spec()
    E.FLAGS.SPARSE_GROUPS = sparse
    p = t.Prepare(None, qs)
    p.forced = forced  # SG_FORCE_SPARSE_GROUPS is read when the query plans, at its first run
    return p


def run(E, t, p, trace_path, keep=False):
    """One sg_query_run + finish: (kernel ms, launches, d2h bytes, discovery ms, ids ms, live, result or None)."""
    with stderr_to(trace_path):
        if p.forced:
            os.environ["SG_FORCE_SPARSE_GROUPS"] = "1"
        try:
            t.ctx.check(t.lib.sg_query_run(p.q))
        finally:
            os.environ.pop("SG_FORCE_SPARSE_GROUPS", None)
        ms = float(t.lib.sg_query_kernel_ms(p.q))
        rp = C.c_void_p()
        t.ctx.check(t.lib.sg_query_finish(p.q, C.byref(rp)))
    st = p.table.lib.sg_query_stats
    from sybil_b200 import _ffi as F
    stats = F.sg_stats()
    st(p.q, C.byref(stats))
    res = None
    try:
        if keep:
            from sybil_b200.engine import QuerySpec
            qs = QuerySpec(Filters=[], Groups=[E.Grouping("g", 0), E.Grouping("s", 1)],
                           Aggregations=[E.Aggregation("v", 2, "hist")])
            t._fill(qs, rp)
            res = sorted((k, r.Count, r.Hists["v"].TotalCount(), r.Hists["v"].Sum(), tuple(r.Hists["v"].Values))
                         for k, r in qs.Results.items())
    finally:
        t.lib.sg_result_free(rp)
    disc = ids = 0.0
    live = None
    for ln in open(trace_path):
        m = re.match(r"sg_sparse: live=(\d+) table=\d+ discover_ms=([\d.]+) ids_ms=([\d.]+)", ln)
        if m:
            live, disc, ids = int(m.group(1)), float(m.group(2)), float(m.group(3))
    return ms, int(stats.kernel_launches), int(stats.d2h_bytes), disc, ids, live, res


def acc_bytes(nslots, nvals):
    # scalars | count | sum | hist Count | buckets | max (one aggregation)
    return (16 + nslots * (4 + nvals)) * 8


def summary(samples):
    out = {}
    for k in ("kernel_ms", "discover_ms", "ids_ms", "aggregate_ms"):
        v = sorted(x[k] for x in samples)
        out[k + "_median"] = v[len(v) // 2]
        out[k + "_min"], out[k + "_max"] = v[0], v[-1]
    last = samples[-1]
    out.update({k: last[k] for k in ("live", "launches", "d2h_bytes", "acc_bytes")})
    return out


def sample(r, nslots, nvals):
    ms, launches, d2h, disc, ids, live, _ = r
    return {"kernel_ms": ms, "discover_ms": disc, "ids_ms": ids, "aggregate_ms": ms - disc - ids, "live": live,
            "launches": launches, "d2h_bytes": d2h, "acc_bytes": acc_bytes(live if live is not None else nslots, nvals)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--both-blocks", type=int, default=1526)
    ap.add_argument("--hashed-blocks", type=int, default=3052)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    trace = os.path.join(a.out, "sparse_groups_trace.txt")
    os.environ["SG_PLAN_TRACE"] = "1"
    from sybil_b200 import engine as E
    from tests.util import Q
    res = {"config": vars(a)}
    res.update(card())
    rng = np.random.default_rng(5)
    nvals = 1002  # BasicHist over [0, 10^6]

    # ---- both paths: 200 x 500 keys -------------------------------------------------------------------------
    specs = make_specs(200, 500, [(rng.integers(0, 200, N), rng.integers(0, 500, N))], rng)
    t = stage(E, specs, a.both_blocks)
    try:
        q = Q(specs[0], groups=["g", "s"], aggs=["v"], op="hist")
        preps = {"dense": prepare(E, t, q, False), "sparse": prepare(E, t, q, True, forced=True)}
        try:
            got = {k: [] for k in preps}
            first = {}
            for i in range(a.warmup + a.runs):
                for k, p in preps.items():
                    r = run(E, t, p, trace, keep=i == 0)
                    if i == 0:
                        first[k] = r[6]
                    if i >= a.warmup:
                        got[k].append(sample(r, 201 * 501, nvals))
            assert first["dense"] == first["sparse"], "dense and sparse results differ"
            res["both"] = {"rows": N * a.both_blocks, "dense_slots": 201 * 501, "identical": True,
                           "dense": summary(got["dense"]), "sparse": summary(got["sparse"])}
        finally:
            for p in preps.values():
                p.Close()
    finally:
        t.close()

    # ---- hashed, refused without the flag: 5,000 x 20,000 keys, 100,000 live pairs ------------------------------
    pairs = np.arange(100_000)
    blocks = [pairs[:N], pairs[100_000 - N:]]
    specs = make_specs(5000, 20000, [(b % 5000, b // 5) for b in (rng.permutation(x) for x in blocks)], rng)
    t = stage(E, specs, a.hashed_blocks)
    try:
        q = Q(specs[0], groups=["g", "s"], aggs=["v"], op="hist")
        off = prepare(E, t, q, False)
        try:
            with stderr_to(trace):
                refused = t.lib.sg_query_run(off.q)
        finally:
            off.Close()
        p = prepare(E, t, q, True)
        try:
            got = []
            for i in range(a.warmup + a.runs):
                r = run(E, t, p, trace)
                if i >= a.warmup:
                    got.append(sample(r, 0, nvals))
            res["hashed"] = {"rows": N * a.hashed_blocks, "key_product": 5001 * 20001, "status_without_flag": int(refused),
                             "table_entries": 1 << 26, "table_acc_bytes": acc_bytes(1 << 26, nvals), "sparse": summary(got)}
        finally:
            p.Close()
    finally:
        t.close()
    line = json.dumps(res)
    print(line)
    with open(os.path.join(a.out, "sparse_groups_rate.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
