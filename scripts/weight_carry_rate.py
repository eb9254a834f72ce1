"""Scan time of weighted queries whose weight column leaves rows out, with the carry of the previous row's weight
(sg_query_desc.weight_carry = 1) and without it.

One generated block (65,536 rows: a str group column `g` of `--groups` strings, an int column `v` with a histogram,
and the weight column `w`) is staged `--blocks` times, once per weight column form:

    full          every row listed, <= 255 distinct weights (per-row codes): no block needs the carry
    codes_gaps    10% of the rows unlisted, <= 255 distinct weights (per-row codes)
    walk_gaps     10% of the rows unlisted, 2,000 distinct weights (bins walked by id)
    short_values  a value array covering the first 90% of the rows (32-bit slot words)

`g` grouped with op hist on `v`, timed with the library's CUDA-event kernel time (sg_query_kernel_ms, read before
sg_query_finish) over `--runs` runs per mode after `--warmup`, carry on and off alternating.  With the carry off the
kernel is the same and the query is refused only at finish, so the difference is the carry pass itself.  The card's
name and power limit are read in the same call.

    python scripts/weight_carry_rate.py [--blocks 1526] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N = 65536
FORMS = ("full", "codes_gaps", "walk_gaps", "short_values")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1])}
    except Exception:
        return {"gpu": None, "power_limit_w": None}


def make_spec(form, ngroups, rng):
    from tests.util import INT, STR, Spec
    s = Spec([("g", STR), ("v", INT), ("w", INT)])
    s.forms = "wide"
    wvals = {"full": 200, "codes_gaps": 200, "walk_gaps": 2000, "short_values": 2000}[form]
    valid = np.ones(N, bool)
    if form in ("codes_gaps", "walk_gaps"):
        valid = rng.random(N) > 0.1
    elif form == "short_values":
        valid[int(N * 0.9):] = False
    cols = {"g": np.array(["g%d" % x for x in rng.integers(0, ngroups, N)]), "v": rng.integers(0, 100000, N),
            "w": rng.integers(1, wvals + 1, N)}
    s.add_rows(cols, {"w": valid}, threshold=1000 if form == "short_values" else 5000)
    return s


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1526)
    ap.add_argument("--groups", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON line into this directory")
    a = ap.parse_args()
    from sybil_b200 import _ffi as F
    from sybil_b200 import engine as E
    from tests.util import Q
    res = {"config": vars(a), "rows": N * a.blocks}
    for form in FORMS:
        rng = np.random.default_rng(7)
        s = make_spec(form, a.groups, rng)
        t = E.Table(form, s.key_table)
        t.IntInfo = dict(s.IntInfo)
        r = {}
        try:
            desc = s.blocks[0].desc()
            for i in range(a.blocks):
                desc.block_index = i
                t.add_block_desc_ptr(C.byref(desc))
            t.sync()
            preps = {}
            for carry in (True, False):
                q = Q(s, groups=["g"], aggs=["v"], op="hist", weight_col="w")
                qs = q.query_spec()
                E.FLAGS.WEIGHT_CARRY = carry
                preps[carry] = t.Prepare(None, qs)
            ms = {True: [], False: []}
            status = {}
            try:
                for k in range(a.warmup + a.runs):
                    for carry in (True, False):
                        p = preps[carry]
                        t.ctx.check(t.lib.sg_query_run(p.q))
                        if k >= a.warmup:
                            ms[carry].append(float(t.lib.sg_query_kernel_ms(p.q)))
                        rp = C.c_void_p()
                        st = t.lib.sg_query_finish(p.q, C.byref(rp))
                        if st == F.SG_OK:
                            t.lib.sg_result_free(rp)
                        status[carry] = int(st)
            finally:
                for p in preps.values():
                    p.Close()
            for carry in (True, False):
                v = sorted(ms[carry])
                r["carry_on" if carry else "carry_off"] = {
                    "kernel_ms_median": v[len(v) // 2], "kernel_ms_min": v[0], "kernel_ms_max": v[-1],
                    "rows_per_s": N * a.blocks / (v[len(v) // 2] * 1e-3), "finish_status": status[carry]}
        finally:
            t.close()
        res[form] = r
    res.update(card())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "weight_carry_rate.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
