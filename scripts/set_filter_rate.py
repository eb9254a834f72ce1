"""Scan rate of set filters (IN / NIN) over set columns of more than 65,536 (tag, row) pairs per block.

One generated block (65,536 rows, `--tags-per-row` distinct tags per row drawn from `--tags`, delta-encoded ids in
bins) is staged `--blocks` times; IN and NIN on one tag are timed with the library's CUDA-event kernel time
(sg_query_kernel_ms) over `--runs` runs after `--warmup`.  Reported per query: kernel ms, (tag, row) pairs of the
table per second, and the encoded bytes the filter pass reads — every id for NIN, the ids of the segments holding
the literal's bin for IN (DESIGN.md §4, "Set filters") — with the card's name and power limit.

    python scripts/set_filter_rate.py [--blocks 1526] [--narrow] [--out DIR]
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

SEG = 65536  # entries per segment at most (SG_BLOCK_ROWS)


def make_block(rng, ntags, per_row, narrow):
    from sybil_b200 import _ffi as F
    from sybil_b200 import blocks as B
    n = 65536
    # per row `per_row` distinct tags: a random permutation's first entries, drawn as argsort of random keys
    choice = np.argsort(rng.random((n, ntags)), axis=1)[:, :per_row]
    tag = choice.ravel()
    row = np.repeat(np.arange(n), per_row)
    order = np.lexsort((row, tag))
    tag, row = tag[order], row[order]
    uniq, starts = np.unique(tag, return_index=True)
    gaps = np.diff(row, prepend=0)
    gaps[starts] = row[starts]  # a bin's first id is absolute
    col = B.SavedColumn(0, F.SG_COL_SET, F.SG_ENC_BUCKET)
    col.delta_ids = True
    col.string_table = [b"tag%d" % i for i in range(ntags)]
    col.bin_values = uniq.astype(np.int64)
    col.bin_offsets = np.append(starts, len(row)).astype(np.uint32)
    col.record_ids = gaps.astype(np.uint16 if narrow else np.uint32)
    blk = B.SavedBlock(0, n)
    blk.cols = [col]
    return blk, col


def segments(offs):
    """The staging's greedy cut (sg_runtime.cu, cut_set_segments): the first bin of every segment."""
    segs = [0]
    for b in range(len(offs) - 1):
        if offs[b + 1] - offs[segs[-1]] > SEG:
            segs.append(b)
    return segs


def card():
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": out[0], "power_limit_w": float(out[1])}
    except Exception:
        return {"gpu": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1526)
    ap.add_argument("--tags", type=int, default=64)
    ap.add_argument("--tags-per-row", type=int, default=4)
    ap.add_argument("--narrow", action="store_true", help="uint16 ids (id_bits 16) instead of uint32")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--out", default=None, help="also write the JSON line into this directory")
    a = ap.parse_args()
    from sybil_b200 import engine as E
    from tests.util import SET, Q, Spec
    rng = np.random.default_rng(5)
    blk, col = make_block(rng, a.tags, a.tags_per_row, a.narrow)
    offs = col.bin_offsets.astype(np.int64)
    cut = segments(offs) + [len(offs) - 1]
    literal = 0  # the first bin's tag: its segment is the first
    seg_of = next(s for s in range(len(cut) - 1) if cut[s] <= literal < cut[s + 1])
    id_bytes = col.record_ids.itemsize
    pairs = len(col.record_ids)
    spec = Spec([("tags", SET)])
    t = E.Table("sets", spec.key_table)
    res = {"config": vars(a), "pairs_per_block": pairs, "segments_per_block": len(cut) - 1, "rows": 65536 * a.blocks}
    try:
        desc = blk.desc()
        for i in range(a.blocks):
            desc.block_index = i
            t.add_block_desc_ptr(C.byref(desc))
        t.sync()
        res["encoded_bytes_resident"] = int(t.lib.sg_table_encoded_bytes(t.h))
        for op in ("in", "nin"):
            q = Q(spec, set_filters=[("tags", op, "tag%d" % literal)])
            qs = q.query_spec()
            ls = t.NewLoadSpec()
            ls.Set("tags")
            p = t.Prepare(ls, qs)
            try:
                for _ in range(a.warmup):
                    p.Run(qs)
                ms = []
                for _ in range(a.runs):
                    p.Run(qs)
                    ms.append(float(t.lib.sg_query_kernel_ms(p.q)))
            finally:
                p.Close()
            ms.sort()
            med = ms[len(ms) // 2]
            if op == "in":
                walked = offs[cut[seg_of + 1]] - offs[cut[seg_of]]
            else:
                walked = pairs
            read = a.blocks * (walked * id_bytes + (len(offs) + len(cut)) * 4 + (len(offs) - 1) * 8)
            res[op] = {"kernel_ms_median": med, "kernel_ms_min": ms[0], "matched": int(qs.MatchedCount),
                       "table_pairs_per_s": pairs * a.blocks / (med * 1e-3),
                       "pairs_read_per_block": int(walked), "encoded_bytes_read": int(read),
                       "bytes_read_per_s": read / (med * 1e-3)}
    finally:
        t.close()
    res.update(card())
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "set_filter_rate%s.json" % ("_narrow" if a.narrow else "")), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
