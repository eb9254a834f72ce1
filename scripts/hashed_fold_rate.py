"""Kernel times, groups, accumulator bytes and read-back of device folds (sg_query_set_hashed_folds), with the
card's name and power limit read in the same call.

One table: 5,000 x 20,000 str keys (a 1e8 key product: hashed), a histogram column v over [0, 10^6] and a weight
column w of 8 values, `--blocks` blocks (two 65,536-row blocks alternating, 100,000 live (g, s) pairs in all).
Three prepared queries run alternately:

    weighted     -op hist -weight-col w, grouped by g, s: sparse group accumulators (the hashed table's histograms
                 pass 24 GiB) over the (group, weight) entries the rows make (each row position repeats its weight in
                 every copy of its block: about 227,000), folded onto the 100,000 groups
    unweighted   the same histogram without the weight: sparse, no fold
    hashed_avg   -op avg -weight-col w: a hashed plan (2^26 entries), folded

Kernel times are the library's CUDA-event times: discovery and the id kernel from the `sg_sparse:` trace line, the
canonical insert and the fold from `sg_fold:` (SG_PLAN_TRACE), aggregation = sg_query_kernel_ms minus those.
L is the table's occupied entries (the sparse plan's accumulator rows), L' the canonical ones (the groups).
Medians over `--runs` runs after `--warmup`.  Writes only into --out.

    python scripts/hashed_fold_rate.py --out DIR [--blocks 1526]
"""
import argparse
import ctypes as C
import json
import os
import re
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import sparse_groups_rate as S  # noqa: E402  (card, stderr_to, stage)

N = S.N
WEIGHTS = (1, 2, 3, 5, 8, 13, 21, 34)


def make_specs(pairs_of_block, rng):
    from tests.util import INT, STR, Spec
    g = np.array(["a%05d" % i for i in range(5000)])
    s = np.array(["b%05d" % i for i in range(20000)])
    specs = []
    for gi, si in pairs_of_block:
        sp = Spec([("g", STR), ("s", STR), ("v", INT), ("w", INT)])
        sp.forms = "wide"
        sp.add_rows({"g": g[gi], "s": s[si], "v": rng.integers(0, 1_000_000, N), "w": rng.choice(WEIGHTS, N)})
        sp.IntInfo["v"] = (0, 1_000_000)
        specs.append(sp)
    return specs


def run(E, F, t, p, trace_path):
    with S.stderr_to(trace_path):
        t.ctx.check(t.lib.sg_query_run(p.q))
        ms = float(t.lib.sg_query_kernel_ms(p.q))
        rp = C.c_void_p()
        t.ctx.check(t.lib.sg_query_finish(p.q, C.byref(rp)))
        ngroups = int(t.lib.sg_result_num_groups_total(rp))
        t.lib.sg_result_free(rp)
    stats = F.sg_stats()
    t.lib.sg_query_stats(p.q, C.byref(stats))
    r = {"kernel_ms": ms, "launches": int(stats.kernel_launches), "d2h_bytes": int(stats.d2h_bytes),
         "discover_ms": 0.0, "ids_ms": 0.0, "insert_ms": 0.0, "fold_ms": 0.0, "L": None, "L_canon": None,
         "groups": ngroups}
    for ln in open(trace_path):
        m = re.match(r"sg_sparse: live=(\d+) table=\d+ discover_ms=([\d.]+) ids_ms=([\d.]+)", ln)
        if m:
            r["L"], r["discover_ms"], r["ids_ms"] = int(m.group(1)), float(m.group(2)), float(m.group(3))
        m = re.match(r"sg_fold: entries=(\d+) canon=(\d+) insert_ms=([\d.]+) fold_ms=([\d.]+)", ln)
        if m:
            r["L"], r["L_canon"] = int(m.group(1)), int(m.group(2))
            r["insert_ms"], r["fold_ms"] = float(m.group(3)), float(m.group(4))
    r["aggregate_ms"] = ms - r["discover_ms"] - r["ids_ms"] - r["insert_ms"] - r["fold_ms"]
    return r


def summary(samples, acc_words_per_row, acc_rows=None):
    out = {}
    for k in ("kernel_ms", "discover_ms", "ids_ms", "insert_ms", "fold_ms", "aggregate_ms"):
        v = sorted(x[k] for x in samples)
        out[k + "_median"] = v[len(v) // 2]
        out[k + "_min"], out[k + "_max"] = v[0], v[-1]
    last = samples[-1]
    out.update({k: last.get(k) for k in ("L", "L_canon", "launches", "d2h_bytes", "groups")})
    rows = acc_rows if acc_rows is not None else last["L"]  # (a hashed plan's accumulators: one row per table entry)
    out["acc_bytes"] = (16 + rows * acc_words_per_row) * 8
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--blocks", type=int, default=1526)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    trace = os.path.join(a.out, "hashed_fold_trace.txt")
    os.environ["SG_PLAN_TRACE"] = "1"
    from sybil_b200 import _ffi as F
    from sybil_b200 import engine as E
    from tests.util import Q
    res = {"config": vars(a)}
    res.update(S.card())
    rng = np.random.default_rng(6)
    pairs = np.arange(100_000)
    blocks = [pairs[:N], pairs[100_000 - N:]]
    specs = make_specs([(b % 5000, b // 5) for b in (rng.permutation(x) for x in blocks)], rng)
    t = S.stage(E, specs, a.blocks)
    sp = specs[0]
    queries = {"weighted": (Q(sp, groups=["g", "s"], aggs=["v"], op="hist", weight_col="w"), 4 + 1002, None),
               "unweighted": (Q(sp, groups=["g", "s"], aggs=["v"], op="hist"), 4 + 1002, None),
               "hashed_avg": (Q(sp, groups=["g", "s"], aggs=["v"], op="avg", weight_col="w"), 4, 1 << 26)}
    preps = {}
    try:
        for k, (q, _, _) in queries.items():
            qs = q.query_spec()
            E.FLAGS.SPARSE_GROUPS = True
            E.FLAGS.HASHED_FOLDS = True
            preps[k] = t.Prepare(None, qs)
        got = {k: [] for k in preps}
        for i in range(a.warmup + a.runs):
            for k, p in preps.items():
                r = run(E, F, t, p, trace)
                if i >= a.warmup:
                    got[k].append(r)
        res["rows"] = N * a.blocks
        res["key_product"] = 5001 * 20001
        res["weights"] = len(WEIGHTS)
        for k, (_, words, rows) in queries.items():
            res[k] = summary(got[k], words, rows)
    finally:
        for p in preps.values():
            p.Close()
        t.close()
    line = json.dumps(res)
    print(line)
    with open(os.path.join(a.out, "hashed_fold_rate.json"), "w") as f:
        f.write(line + "\n")


if __name__ == "__main__":
    main()
