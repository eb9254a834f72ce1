"""Parity tests proper: the CUDA path, called through the C ABI (libsybilgpu.so), against the CPU
oracle on the same seeded inputs.  Bit-exact: group keys, Count, Samples, hist Count, exact int64
sums, Min/Max, every bucket counter, percentiles, MatchedCount.  Float tolerance (stated in
tests/util.py): mean 1e-9, stddev 1e-9."""
import json
import os

import numpy as np
import pytest

from sybil_b200 import _ffi as F
from tests.util import compare_group, INT, SET, STR, Q, Spec, compare, random_spec, run_gpu, run_oracle

pytestmark = pytest.mark.gpu


def both(spec, q):
    o = run_oracle(spec, q)
    g = run_gpu(spec, q)
    compare(g, o, q)
    return g, o


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_group_by_avg(seed):
    s = random_spec(seed, nrows=5000, block_rows=1500)
    both(s, Q(s, groups=["host"], aggs=["age", "lat", "big"], op="avg"))


def test_int_filters_like_filter_test_go():
    # filter_test.go:9-150: eq / neq / lt / gt on an int column
    s = random_spec(11, nrows=4000, block_rows=1000)
    for op in ("eq", "neq", "lt", "gt"):
        both(s, Q(s, int_filters=[("age", op, 20)], groups=["age"], aggs=["age"], op="avg"))


def test_str_filters_eq_neq_re_nre_and_absent_literal():
    s = random_spec(12, nrows=4000, block_rows=1000)
    for op, lit in (("eq", "s3"), ("neq", "s3"), ("re", "^s1"), ("nre", "^s1"), ("eq", "nope"), ("neq", "nope")):
        both(s, Q(s, str_filters=[("state", op, lit)], groups=["state"], aggs=["age"], op="avg"))


def test_three_filters_two_groups_hist_like_config3():
    s = random_spec(13, nrows=6000, block_rows=2000)
    g, o = both(s, Q(s, int_filters=[("age", "gt", 12), ("big", "lt", 900000)], str_filters=[("state", "neq", "s3")],
                     groups=["host", "age"], aggs=["lat"], op="hist"))
    assert len(g.Results) > 50


def test_histogram_percentiles_like_aggregate_test_go():
    # aggregate_test.go:102-208: per-group percentiles equal the key when every value of a group is the key
    n = 3000
    rng = np.random.default_rng(5)
    age = rng.integers(10, 30, n)
    s = Spec([("age", INT), ("age_str", STR)])
    s.add_rows({"age": age, "age_str": np.array([str(a) for a in age])}, block_rows=700)
    q = Q(s, groups=["age_str"], aggs=["age"], op="hist")
    g, o = both(s, q)
    for k, r in g.Results.items():
        p = r.Hists["age"].GetPercentiles()
        key = int(k.strip("\t"))
        assert p[25] == key and p[50] == key and p[75] == key


def test_loghist_multihist():
    s = random_spec(14, nrows=5000, block_rows=1700)
    both(s, Q(s, groups=["host"], aggs=["big", "lat"], op="hist", loghist=True))
    both(s, Q(s, groups=["host"], aggs=["big"], op="avg", loghist=True))


def test_hist_bucket_override():
    s = random_spec(15, nrows=3000, block_rows=1000)
    both(s, Q(s, groups=["host"], aggs=["lat"], op="hist", hist_bucket=100))


def test_time_series_like_aggregate_test_go():
    # aggregate_test.go:211-279: at least one bucket, none empty
    s = random_spec(16, nrows=6000, block_rows=2000)
    g, o = both(s, Q(s, groups=["host"], aggs=["lat"], op="hist", time_col="time", time_bucket=600))
    assert len(g.TimeResults) >= 1 and all(len(m) > 0 for m in g.TimeResults.values())
    both(s, Q(s, aggs=["age"], op="avg", time_col="time", time_bucket=3600))


def test_value_array_encodings_and_values_above_2_pow_32():
    # table_query_test.go (CHUNK_SIZE = CARDINALITY_THRESHOLD+1) and column_store_test.go:143-211
    s = random_spec(17, nrows=4000, block_rows=1300, threshold=50, wide=True)
    both(s, Q(s, int_filters=[("big", "gt", 0)], groups=["host"], aggs=["big", "lat"], op="avg"))
    both(s, Q(s, int_filters=[("big", "lt", 1 << 45)], groups=["host", "state"], aggs=["big"], op="hist"))
    both(s, Q(s, groups=["uid"], aggs=["age", "big"], op="avg"))  # high-cardinality str key, value-array ids


def test_no_groups_and_no_aggs():
    s = random_spec(18, nrows=2000, block_rows=800)
    g, o = both(s, Q(s, aggs=["age"], op="hist"))
    assert list(g.Results) == ["total"]
    both(s, Q(s, int_filters=[("age", "gt", 20)]))  # count(*) + one IntFilter (config 1's query shape)


def test_filter_matching_nothing():
    s = random_spec(19, nrows=1500, block_rows=500)
    g, o = both(s, Q(s, int_filters=[("age", "gt", 1000)], groups=["host"], aggs=["age"], op="avg"))
    assert g.MatchedCount == 0 and len(g.Results) == 0


def test_missing_columns_and_group_on_missing_values():
    # a column absent from some blocks; rows lacking the group column render an empty field (Q4)
    rng = np.random.default_rng(20)
    s = Spec([("a", INT), ("b", INT), ("h", STR)])
    n = 1200
    s.add_rows({"a": rng.integers(0, 10, n), "b": rng.integers(0, 100, n), "h": np.array(["x%d" % v for v in rng.integers(0, 4, n)])},
               valid={"h": rng.random(n) > 0.3, "b": rng.random(n) > 0.5}, block_rows=400)
    s.add_rows({"a": rng.integers(0, 10, n)}, block_rows=400)  # blocks without b and h at all
    both(s, Q(s, groups=["h"], aggs=["b"], op="hist"))
    both(s, Q(s, groups=["h", "a"], aggs=["b", "a"], op="avg"))
    both(s, Q(s, int_filters=[("b", "neq", 5)], groups=["a"], aggs=["b"], op="avg"))


def test_single_row_and_full_size_blocks():
    rng = np.random.default_rng(21)
    s = Spec([("v", INT), ("g", STR)])
    s.add_rows({"v": np.array([42]), "g": np.array(["only"])})
    n = F.SG_BLOCK_ROWS
    s.add_rows({"v": rng.integers(0, 1 << 20, n), "g": np.array(["g%d" % x for x in rng.integers(0, 7, n)])})
    s.add_rows({"v": rng.integers(0, 3000, n - 1), "g": np.array(["g%d" % x for x in rng.integers(0, 7, n - 1)])})
    both(s, Q(s, groups=["g"], aggs=["v"], op="hist"))
    both(s, Q(s, int_filters=[("v", "lt", 2000)], groups=["g"], aggs=["v"], op="avg"))


def test_broken_block_is_skipped_like_table_query_test_go():
    # table_query_test.go:11-158: a block whose NumRecords shrank under its row ids is dropped
    # whole ("BLOCK SIZE CHANGED DURING QUERY") and the other blocks still answer
    s = random_spec(22, nrows=3000, block_rows=1000)
    s.blocks[1].num_records = 400
    g, o = both(s, Q(s, groups=["host"], aggs=["age"], op="hist"))
    assert g.BrokenBlocks == 1
    s2 = random_spec(23, nrows=3000, block_rows=1000, threshold=50)
    s2.blocks[2].num_records = 500  # value arrays longer than the block
    g, o = both(s2, Q(s2, groups=["host"], aggs=["big"], op="avg"))
    assert g.BrokenBlocks == 1


def test_zone_map_pruning():
    # ShouldLoadBlockFromDir (table_block_io.go:110-182): blocks whose [min,max] cannot match are skipped
    rng = np.random.default_rng(24)
    s = Spec([("t", INT), ("v", INT)])
    for b in range(4):
        s.add_rows({"t": rng.integers(b * 1000, b * 1000 + 1000, 500), "v": rng.integers(0, 50, 500)})
    g, o = both(s, Q(s, int_filters=[("t", "gt", 2500)], groups=["v"], aggs=["t"], op="avg"))
    assert g.SkippedBlocks == 2
    g, o = both(s, Q(s, int_filters=[("t", "eq", 1200)], aggs=["v"], op="avg"))
    assert g.SkippedBlocks == 3


def test_negative_values_and_exact_sums():
    rng = np.random.default_rng(25)
    n = 5000
    s = Spec([("x", INT), ("g", STR)])
    # magnitudes whose true sum stays inside int64: the engine's sums are exact modulo 2^64
    # (Go int64 wrapping); a mean derived from a wrapped sum is a documented divergence
    s.add_rows({"x": rng.integers(-(1 << 50), 1 << 50, n), "g": np.array(["g%d" % v for v in rng.integers(0, 3, n)])},
               threshold=10, block_rows=2000)
    s.IntInfo["x"] = (-(1 << 50), (1 << 50) // 10)
    both(s, Q(s, groups=["g"], aggs=["x"], op="avg"))
    s2 = Spec([("x", INT), ("g", STR)])
    s2.add_rows({"x": rng.integers(-500, 500, n), "g": np.array(["g%d" % v for v in rng.integers(0, 3, n)])}, block_rows=2000)
    both(s2, Q(s2, groups=["g"], aggs=["x"], op="hist"))


def test_many_groups_spills_accumulators_to_global_memory():
    rng = np.random.default_rng(26)
    n = 20000
    s = Spec([("a", INT), ("b", INT), ("v", INT)])
    s.add_rows({"a": rng.integers(0, 300, n), "b": rng.integers(0, 200, n), "v": rng.integers(0, 100000, n)}, block_rows=7000)
    g, o = both(s, Q(s, groups=["a", "b"], aggs=["v"], op="avg"))
    assert len(g.Results) > 10000


def test_golden_rows_reproduce_reference_buckets():
    # the reference's golden result (decoding_test.go fixture) through the CUDA path
    from tests.test_oracle_golden import G, dense, golden_table
    s = golden_table()
    q = Q(s, groups=["browser", "device"], aggs=["pageload"], op="hist")
    g = run_gpu(s, q)
    assert g.MatchedCount == G["MatchedCount"]
    assert [r.GroupByKey for r in g.Sorted] == G["Sorted"]
    assert g.Cumulative.GroupByKey == "TOTAL\t"
    assert np.array_equal(g.Cumulative.Hists["pageload"].Values, dense(G["Cumulative"]["hist"]))
    for k, gold in G["Results"].items():
        r = g.Results[k]
        h = r.Hists["pageload"]
        assert (r.Count, r.Samples, h.TotalCount()) == (gold["Count"], gold["Samples"], gold["hist"]["Count"])
        assert (h.Min(), h.Max()) == (gold["hist"]["Min"], gold["hist"]["Max"])
        assert (h.NumBuckets, h.BucketSize, len(h.Values)) == (1001, 23, 1002)
        assert np.array_equal(h.Values, dense(gold["hist"]))


@pytest.mark.parametrize("narrow", [True, False])
@pytest.mark.parametrize("cfg,rows", [("c2", 300_000), ("c3", 400_000), ("c4", 300_000), ("c5", 300_000)])
def test_benchmark_configs_at_reduced_size(cfg, rows, narrow):
    """BASELINE.json configs 2-5 generated by the C++ generator at a size the oracle finishes in seconds, with
    the arrays in their narrow form (uint16 ids, int16 / int32 value deltas: 2 KiB / 1 KiB TMA tiles) and in Go's
    decoded types (4 KiB tiles)."""
    from sybil_b200 import engine as E
    from sybil_b200 import synth
    from oracle.oracle_ffi import OracleTable
    spec = synth.config(cfg, total_rows=rows)
    spec.narrow = narrow
    store = synth.generate(spec)
    qd = synth.query_for(spec)
    s = Spec(spec.key_table)
    s.IntInfo = dict(spec.IntInfo)
    q = Q(s, **qd)
    t = E.Table(cfg, spec.key_table)
    t.IntInfo = dict(spec.IntInfo)
    ot = OracleTable(spec.key_table)
    try:
        for i in range(store.num_blocks()):
            t.add_block_desc_ptr(store.block(i))
            ot.add_block(store.block(i))
        d, keep = q.desc()
        o = ot.query(d, q.aggs, nthreads=4)
        g = run_gpu(s, q, table=t)
        compare(g, o, q)
        assert g.MatchedCount > 0
    finally:
        t.close()
        ot.close()
        store.close()


def test_tma_and_plain_load_paths_agree(monkeypatch):
    """The TMA-staged tile feed and the plain 256-bit load path must give the same result: a table created
    while SG_NO_TMA is set has no tensor maps, so the same kernel reads with vector loads."""
    s = random_spec(31, nrows=9000, block_rows=4000, threshold=50, wide=True)
    q = Q(s, int_filters=[("big", "gt", 5)], str_filters=[("state", "neq", "s3")], groups=["host"], aggs=["lat", "big"], op="hist")
    o = run_oracle(s, q)
    compare(run_gpu(s, q), o, q)
    monkeypatch.setenv("SG_NO_TMA", "1")
    compare(run_gpu(s, q), o, q)


def test_batch_staging_restaging_and_streaming_submit():
    """sg_table_add_blocks (batch staging), sg_table_clear + re-staging into the same arena, and
    sg_query_submit_block (zone-map pruning before staging) all give the oracle's answer."""
    import ctypes as C
    from sybil_b200 import engine as E
    from sybil_b200 import synth
    from oracle.oracle_ffi import OracleTable
    spec = synth.config("c3", total_rows=5 * 20000, block_rows=20000)
    store = synth.generate(spec)
    s = Spec(spec.key_table)
    s.IntInfo = dict(spec.IntInfo)
    q = Q(s, **synth.query_for(spec))
    ot = OracleTable(spec.key_table)
    for i in range(store.num_blocks()):
        ot.add_block(store.block(i))
    d, keep = q.desc()
    o = ot.query(d, q.aggs, nthreads=2)
    t = E.Table("b", spec.key_table)
    t.IntInfo = dict(spec.IntInfo)
    try:
        ptrs, n = store.block_ptrs()
        for _ in range(2):  # stage, query, clear, stage again into the recycled arena
            t.add_blocks(ptrs, n)
            compare(run_gpu(s, q, table=t), o, q)
            t.ctx.check(t.lib.sg_table_clear(t.h))
        # streaming: blocks submitted to a query one by one
        qs = q.query_spec()
        dd, keep2 = E.make_query_desc(s.KeyTable, s.KeyTypes, s.IntInfo, qs)
        qh = t.lib.sg_query_begin(t.ctx.h, t.h, C.byref(dd))
        assert qh
        for i in range(n):
            t.ctx.check(t.lib.sg_query_submit_block(qh, store.block(i)))
        rp = C.c_void_p()
        t.ctx.check(t.lib.sg_query_finish(qh, C.byref(rp)))
        assert t.lib.sg_result_matched_count(rp) == o.MatchedCount
        assert t.lib.sg_result_num_groups(rp) == len(o.Results)
        t.lib.sg_result_free(rp)
        t.lib.sg_query_free(qh)
    finally:
        t.close()
        ot.close()
        store.close()


def test_staging_statistics_pick_the_right_paths():
    """Values inside [0, 2^32) take the 32-bit scan; negative / wide values, values outside the table's
    extents (rejected, hist_basic.go:104) and values above info_max (Max tracking) take the complete rule."""
    rng = np.random.default_rng(33)
    n = 6000
    s = Spec([("g", STR), ("small", INT), ("neg", INT), ("wide", INT)])
    s.add_rows({"g": np.array(["g%d" % v for v in rng.integers(0, 5, n)]),
                "small": rng.integers(0, 1 << 22, n), "neg": rng.integers(-100000, 100000, n),
                "wide": rng.integers(0, 1 << 40, n)}, threshold=10, block_rows=2500)
    s.IntInfo["small"] = (1000, 1 << 20)  # values below Min are rejected, values up to 10*Max accepted
    for op in ("avg", "hist"):
        both(s, Q(s, groups=["g"], aggs=["small", "neg", "wide"], op=op))
        both(s, Q(s, int_filters=[("small", "lt", 1 << 21), ("neg", "gt", -5)], groups=["g"], aggs=["small"], op=op))


def test_result_json_contract_like_printer_go():
    """Result.toResultJSON (printer.go:109-152), the reference's -json output per group, rebuilt from the
    engine's result and from the oracle's: same keys, bit-equal integers, floats within tolerance."""
    from sybil_b200.engine import toResultJSON
    from tests.util import close, MEAN_TOL, STD_TOL
    s = random_spec(41, nrows=5000, block_rows=1800)
    for op in ("hist", "avg"):
        q = Q(s, int_filters=[("age", "gt", 11)], groups=["host", "state"], aggs=["lat", "age"], op=op)
        g = run_gpu(s, q)
        o = run_oracle(s, q)
        q.set_flags()
        qs = q.query_spec()
        for k, r in g.Results.items():
            j = toResultJSON(r, qs)
            orr = o.Results[k]
            assert j["Count"] == orr.Count and j["Samples"] == orr.Samples
            assert (j["host"], j["state"]) == tuple(k.split("\t")[:2])
            for a in q.aggs:
                oh = orr.Hists.get(a)
                if op == "avg":
                    assert (j[a] is None) == (oh is None)
                    if oh is not None:
                        assert close(j[a], oh.Avg, MEAN_TOL)
                elif oh is not None and oh.Count:
                    assert j[a]["percentiles"] == oh.Percentiles
                    assert j[a]["buckets"] == {str(e): c for e, c in oh.IntBuckets.items() if c > 0}
                    assert j[a]["samples"] == oh.Count
                    assert close(j[a]["avg"], oh.Avg, MEAN_TOL) and close(j[a]["stddev"], oh.StdDev, STD_TOL)
                    assert close(j[a]["sum"], oh.Avg * oh.Count, 1e-9)


def test_tail_blocks_split_per_aggregation(monkeypatch):
    """Blocks of the last partial wave are split into one work item per subset of the aggregations;
    SG_FORCE_TAIL_SPLIT splits every block so that small tables exercise the path."""
    monkeypatch.setenv("SG_FORCE_TAIL_SPLIT", "1")
    s = random_spec(51, nrows=9000, block_rows=2000, threshold=50)
    both(s, Q(s, int_filters=[("age", "gt", 11)], groups=["host"], aggs=["age", "lat", "big"], op="avg"))
    both(s, Q(s, groups=["host", "state"], aggs=["lat", "age"], op="hist"))
    both(s, Q(s, groups=["host"], aggs=["lat", "big"], op="hist", time_col="time", time_bucket=600))
    s.blocks[1].num_records = 700  # a broken block must still vanish whole
    both(s, Q(s, groups=["host"], aggs=["age", "lat"], op="hist"))


def test_group_by_value_array_int_column():
    """Group-by on an int column that is value-array encoded (more distinct values per block than the
    cardinality threshold, column_store_io.go:82-113): the engine collects the blocks' distinct values on
    the GPU, joins them into the table-wide value dictionary and maps value -> dense code through a hash
    table.  Bit-exact against the oracle: keys, counts, sums, histogram buckets."""
    rng = np.random.default_rng(77)
    n = 6000
    s = Spec([("k", INT), ("v", INT), ("host", STR), ("lat", INT), ("time", INT)])
    keys = rng.integers(-(1 << 45), 1 << 45, 300)  # 300 distinct values, negative and above 2^32
    keys[0] = -(1 << 63)                           # the hash set's "empty" marker is a legal value
    s.add_rows({"k": keys[rng.integers(0, 300, n)], "v": rng.integers(0, 1000, n),
                "host": np.array(["h%d" % x for x in rng.integers(0, 4, n)]),
                "lat": rng.integers(0, 5000, n), "time": 1500000000 + np.sort(rng.integers(0, 7200, n))},
               {"k": rng.random(n) > 0.05, "v": rng.random(n) > 0.05}, threshold=50, block_rows=1700)
    both(s, Q(s, groups=["k"], aggs=["v"], op="avg"))
    both(s, Q(s, int_filters=[("v", "gt", 100)], str_filters=[("host", "neq", "h2")], groups=["host", "k"], aggs=["lat"], op="hist"))
    both(s, Q(s, groups=["k"], aggs=["v"], op="avg", time_col="time", time_bucket=1800))
    both(s, Q(s, groups=["k"]))  # count only


def test_group_by_int_column_with_mixed_encodings():
    """The same int column bucket-encoded in one block (few distinct values there) and value-array
    encoded in another: bin values and array values share one dictionary."""
    rng = np.random.default_rng(78)
    s = Spec([("k", INT), ("v", INT)])
    s.add_rows({"k": rng.integers(0, 20, 1500), "v": rng.integers(0, 100, 1500)}, threshold=50, block_rows=1500)
    s.add_rows({"k": rng.integers(0, 400, 1500), "v": rng.integers(0, 100, 1500)}, threshold=50, block_rows=1500)
    s.add_rows({"k": rng.integers(10, 30, 1500), "v": rng.integers(0, 100, 1500)}, threshold=50, block_rows=1500)
    g, o = both(s, Q(s, groups=["k"], aggs=["v"], op="avg"))
    assert len(g.Results) == len(o.Results) and len(g.Results) > 300
    both(s, Q(s, int_filters=[("k", "lt", 200)], groups=["k"], aggs=["v"], op="hist"))


def _splitmix64_np(x):
    with np.errstate(over="ignore"):
        x = x + np.uint64(0x9E3779B97F4A7C15)
        x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return x ^ (x >> np.uint64(31))


def test_full_size_c2_checksums_and_block_additivity():
    """BASELINE.json's metric configuration at FULL size (100M rows; the oracle would need minutes), through
    size-independent properties:
      * per-group Count and exact Sum of every aggregated column equal an independent numpy evaluation of the
        counter-based generator (no encoder, no decoder, no block structure: a checksum of the whole decode +
        filter-free group-by + aggregation path, bit-exact);
      * block additivity (CombineResults): the result over all blocks equals the merge of the results over
        the first and the second half of the blocks, staged as two separate tables."""
    from sybil_b200 import engine as E
    from sybil_b200 import synth
    spec = synth.config("c2")
    rows = spec.total_rows
    assert rows == 100_000_000
    store = synth.generate(spec)
    s = Spec(spec.key_table)
    s.IntInfo = dict(spec.IntInfo)
    q = Q(s, **synth.query_for(spec))
    nb = store.num_blocks()
    tabs = [E.Table("c2_all", spec.key_table), E.Table("c2_a", spec.key_table), E.Table("c2_b", spec.key_table)]
    try:
        for t in tabs:
            t.IntInfo = dict(spec.IntInfo)
        for i in range(nb):
            tabs[0].add_block_desc_ptr(store.block(i))
            tabs[1 if i < nb // 2 else 2].add_block_desc_ptr(store.block(i))
        res = [run_gpu(s, q, table=t) for t in tabs]
        g = res[0]
        assert g.MatchedCount == rows and sum(r.Count for r in g.Sorted) == rows and len(g.Results) == 64
        # --- independent evaluation of the generator, 10M rows at a time
        cnt = np.zeros(64, np.int64)
        sums = {c.name: np.zeros(64, np.float64) for c in spec.cols[1:]}
        gcol = spec.cols[0]
        for lo in range(0, rows, 10_000_000):
            r = np.arange(lo, min(lo + 10_000_000, rows), dtype=np.uint64)
            key = (_splitmix64_np(np.uint64(spec.seed) ^ (np.uint64(gcol.col_slot) << np.uint64(40)) ^ r) % np.uint64(gcol.span)).astype(np.int64)
            cnt += np.bincount(key, minlength=64)
            for c in spec.cols[1:]:
                v = (_splitmix64_np(np.uint64(spec.seed) ^ (np.uint64(c.col_slot) << np.uint64(40)) ^ r) % np.uint64(c.span)).astype(np.float64) + c.lo
                sums[c.name] += np.bincount(key, weights=v, minlength=64)  # exact: every partial sum < 2^53
        for k in range(64):
            r = g.Results["k%d\t" % k]
            assert r.Count == cnt[k]
            for c in spec.cols[1:]:
                assert r.Hists[c.name].Count == cnt[k]
                assert r.Hists[c.name].Sum() == int(sums[c.name][k]), (k, c.name)
        # --- additivity
        a, b = res[1], res[2]
        assert a.MatchedCount + b.MatchedCount == rows
        for key, r in g.Results.items():
            ra, rb = a.Results[key], b.Results[key]
            assert r.Count == ra.Count + rb.Count
            for c in spec.cols[1:]:
                assert r.Hists[c.name].Sum() == ra.Hists[c.name].Sum() + rb.Hists[c.name].Sum()
    finally:
        for t in tabs:
            t.close()
        store.close()


# ---------------------------------------------------------------------------------------------------
# round 2: predicate push-down into the inverted index (fail mode), slot windows over the time axis,
# the shared-memory histogram cache, full-size parity against the generator's row values
# ---------------------------------------------------------------------------------------------------
def _shuffle_bins(spec, seed):
    """Go writes a column's bins in map-iteration order: permute the bins of every bucket column (the id
    lists move with their bins) so that failing and passing bins interleave inside the warp tiles."""
    rng = np.random.default_rng(seed)
    for blk in spec.blocks:
        for col in blk.cols:
            if col.encoding != F.SG_ENC_BUCKET or len(col.bin_values) < 2:
                continue
            perm = rng.permutation(len(col.bin_values))
            offs = np.asarray(col.bin_offsets, np.int64)
            ids = [np.asarray(col.record_ids[offs[b]:offs[b + 1]]) for b in perm]
            col.bin_values = np.asarray(col.bin_values)[perm]
            col.record_ids = np.concatenate(ids).astype(np.asarray(col.record_ids).dtype)  # (uint16 stays uint16)
            col.bin_offsets = np.concatenate([[0], np.cumsum([len(x) for x in ids])]).astype(np.uint32)


def _wide_spec(seed, nrows, block_rows, nulls=False, shuffle=True):
    rng = np.random.default_rng(seed)
    s = Spec([("f0", INT), ("f1", INT), ("s0", STR), ("s1", STR), ("d", INT), ("lat", INT), ("time", INT)])
    cols = {
        "f0": rng.integers(0, 1000, nrows), "f1": rng.integers(0, 1000000, nrows),
        "s0": np.array(["v%d" % v for v in rng.integers(0, 16, nrows)]),
        "s1": np.array(["g%d" % v for v in rng.integers(0, 12, nrows)]),
        "d": rng.integers(0, 8, nrows),
        "lat": (rng.integers(0, 65536, (nrows, 4)).sum(1) * 23470 // (4 * 65535) + 30),
        "time": 1500000000 + np.sort(rng.integers(0, 40 * 3600, nrows)),
    }
    valid = {"f0": rng.random(nrows) > 0.01} if nulls else None
    s.add_rows(cols, valid, block_rows=block_rows)
    if shuffle:
        _shuffle_bins(s, seed + 1)
    return s


@pytest.mark.parametrize("nulls", [False, True])
def test_filter_push_down_on_fully_populated_columns(nulls, monkeypatch):
    """Filters over bucket columns that list every row (COL_FULL) run in fail mode and walk only the tiles of
    their failing bins; bins in arbitrary (Go map) order; full 65,536-row blocks so a column spans 64 tiles.
    With nulls in a filter column the plan falls back to counting passes.  Both must equal the oracle, and
    fail mode with every tile walked (SG_NO_PUSHDOWN) must agree too."""
    s = _wide_spec(41, 3 * 65536 + 12345, 65536, nulls=nulls)
    qs_ = [
        Q(s, int_filters=[("f0", "gt", 100), ("f1", "lt", 900000)], str_filters=[("s0", "neq", "v3")], groups=["s1", "d"], aggs=["lat"], op="hist"),
        Q(s, int_filters=[("f0", "eq", 7)], groups=["s1"], aggs=["lat"], op="avg"),
        Q(s, int_filters=[("f0", "neq", 7), ("d", "lt", 5)], str_filters=[("s1", "eq", "g4")], groups=["s0"], aggs=["f1"], op="avg"),
        Q(s, int_filters=[("f0", "lt", 0)], groups=["s1"], aggs=["lat"], op="avg"),   # every bin fails
        Q(s, int_filters=[("f0", "gt", -1)], groups=["s1"], aggs=["lat"], op="avg"),  # no bin fails: no tile is read
    ]
    for q in qs_:
        o = run_oracle(s, q, nthreads=4)
        compare(run_gpu(s, q), o, q)
        monkeypatch.setenv("SG_NO_PUSHDOWN", "1")
        compare(run_gpu(s, q), o, q)
        monkeypatch.delenv("SG_NO_PUSHDOWN")


def test_time_window_and_histogram_cache(monkeypatch):
    """Time rollup over a sorted time column: slot words hold block-relative time codes (the window comes
    from the column's exact extents), blocks inside one bucket do not read the column, the bucket counters
    live in the shared-memory cache and are flushed when the window moves.  Same answer with the window,
    the cache and both switched off."""
    s = _wide_spec(43, 4 * 65536 + 999, 65536, shuffle=False)
    for q in (Q(s, aggs=["lat"], op="hist", time_col="time", time_bucket=3600),
              Q(s, groups=["d"], aggs=["lat", "f1"], op="hist", time_col="time", time_bucket=7200),
              Q(s, int_filters=[("f0", "gt", 500)], groups=["s1"], aggs=["lat"], op="avg", time_col="time", time_bucket=600)):
        o = run_oracle(s, q, nthreads=4)
        compare(run_gpu(s, q), o, q)
        for env in ("SG_NO_TIME_WINDOW", "SG_NO_HIST_CACHE"):
            monkeypatch.setenv(env, "1")
            compare(run_gpu(s, q), o, q)
            monkeypatch.delenv(env)


@pytest.mark.parametrize("cfg,rows", [("c3", 100_000_000), ("c4", 100_000_000)])
def test_full_size_against_row_values(cfg, rows):
    """The histogram configs at a size where tail splitting, deferred folds, window moves and cache flushes
    all engage (1,526 blocks): every group's Count, hist Count, exact sum and every bucket counter equal
    the query evaluated directly on the generator's row values (synth.Expected: no encoder, no decoder)."""
    from sybil_b200 import engine as E
    from sybil_b200 import synth
    spec = synth.config(cfg, total_rows=rows)
    store = synth.generate(spec)
    s = Spec(spec.key_table)
    s.IntInfo = dict(spec.IntInfo)
    q = Q(s, **synth.query_for(spec))
    t = E.Table(cfg, spec.key_table)
    t.IntInfo = dict(spec.IntInfo)
    try:
        ptrs, n = store.block_ptrs()
        t.add_blocks(ptrs, n)
        g = run_gpu(s, q, table=t)
        exp = synth.Expected(spec)
        assert exp.check(g) > 1000
        assert g.MatchedCount > rows // 2
    finally:
        t.close()
        store.close()


def test_streaming_submit_gives_the_full_result():
    """sg_query_submit_block + sg_query_finish: the complete result (not only the counts) equals the oracle's."""
    import ctypes as C
    from sybil_b200 import engine as E
    from sybil_b200 import synth
    from oracle.oracle_ffi import OracleTable
    spec = synth.config("c3", total_rows=4 * 30000, block_rows=30000)
    store = synth.generate(spec)
    s = Spec(spec.key_table)
    s.IntInfo = dict(spec.IntInfo)
    q = Q(s, **synth.query_for(spec))
    ot = OracleTable(spec.key_table)
    for i in range(store.num_blocks()):
        ot.add_block(store.block(i))
    d, keep = q.desc()
    o = ot.query(d, q.aggs, nthreads=2)
    t = E.Table("stream", spec.key_table)
    t.IntInfo = dict(spec.IntInfo)
    try:
        qs = q.query_spec()
        dd, keep2 = E.make_query_desc(s.KeyTable, s.KeyTypes, s.IntInfo, qs)
        qh = t.lib.sg_query_begin(t.ctx.h, t.h, C.byref(dd))
        assert qh
        for i in range(store.num_blocks()):
            t.ctx.check(t.lib.sg_query_submit_block(qh, store.block(i)))
        rp = C.c_void_p()
        t.ctx.check(t.lib.sg_query_finish(qh, C.byref(rp)))
        t._fill(qs, rp)
        t.lib.sg_result_free(rp)
        t.lib.sg_query_free(qh)
        compare(qs, o, q)
    finally:
        t.close()
        ot.close()
        store.close()


def test_histogram_cache_misses_and_hot_counters():
    """More slots than the shared-memory histogram cache holds: the rows beyond the cache are reduced into L2
    directly.  One group takes 90% of the rows and almost every row has the same value, so a single counter
    takes tens of thousands of increments inside one block — in the cache for one query, in L2 for the other."""
    rng = np.random.default_rng(47)
    n = 2 * 65536 + 777
    g = np.where(rng.random(n) < 0.9, 39, rng.integers(0, 40, n))
    g[:40] = np.arange(40)  # every value shows up before the hot one: its slot lies beyond the cache rows
    lat = np.where(rng.random(n) < 0.95, 5000, rng.integers(30, 23500, n))
    s = Spec([("g", STR), ("lat", INT), ("f", INT)])
    s.add_rows({"g": np.array(["z%d" % v for v in g]), "lat": lat, "f": rng.integers(0, 100000, n)}, block_rows=65536, threshold=50)
    s.IntInfo["lat"] = (30, 23500)
    for q in (Q(s, groups=["g"], aggs=["lat"], op="hist"),
              Q(s, int_filters=[("f", "lt", 70000)], groups=["g"], aggs=["lat", "f"], op="hist")):
        compare(run_gpu(s, q), run_oracle(s, q, nthreads=4), q)


def _age_spec(seed, n=6000):
    rng = np.random.default_rng(seed)
    age = rng.integers(10, 30, n)
    s = Spec([("id", INT), ("age", INT), ("age_str", STR), ("w", INT)])
    s.add_rows({"id": np.arange(n), "age": age, "age_str": np.array([str(a) for a in age]), "w": rng.integers(0, 1000, n)},
               block_rows=n // 3 + 1)
    return s


def test_order_by_like_aggregate_test_go():
    """aggregate_test.go:281-413 (TestOrderBy / TestOrderByDesc): OrderBy = an aggregation's name sorts the
    groups by Hists[col].Mean() descending, OrderAsc reverses the list; also $COUNT ascending, Limit, and
    OrderBy == "" (no sort).  The CUDA path's Sorted list equals the oracle's, group for group."""
    s = _age_spec(51)
    for kw in (dict(order_by="age"), dict(order_by="age", order_asc=True), dict(order_by="$COUNT", order_asc=True),
               dict(order_by="w"), dict(order_by="age", limit=5), dict(order_by="$COUNT", limit=7),
               dict(order_by="$COUNT", order_asc=True, limit=4), dict(order_by="")):
        q = Q(s, groups=["age_str"], aggs=["age", "w"], op="avg", **kw)
        g, o = both(s, q)
        if kw.get("order_by") == "age":
            means = [r.Hists["age"].Mean() for r in g.Sorted]
            assert means == sorted(means, reverse=not kw.get("order_asc", False))  # the reference test's own check
        if kw.get("limit"):
            assert len(g.Sorted) == kw["limit"] and g.NumGroups == 20
            assert g.Cumulative.Count == 6000  # Cumulative still covers every group
    # hist mode, two group columns, mean order with ties broken by the rendered key
    q = Q(s, groups=["age_str", "age"], aggs=["w"], op="hist", order_by="w", limit=10)
    both(s, q)


def test_top_groups_of_a_high_cardinality_result():
    """300k distinct keys (accumulators in global memory), Limit = 100: the materialised top of the sorted list,
    NumGroups and Cumulative equal the oracle's full result; with ties broken by the rendered key."""
    rng = np.random.default_rng(53)
    n = 400_000
    s = Spec([("k", STR), ("m", INT)])
    s.add_rows({"k": np.array(["key%d" % v for v in rng.integers(0, 300_000, n)]), "m": rng.integers(0, 10000, n)},
               block_rows=65536)
    for kw in (dict(limit=100), dict(limit=100, order_by="m"), dict(limit=50, order_asc=True)):
        both(s, Q(s, groups=["k"], aggs=["m"], op="avg", **kw))
    # The first `limit` groups of such a result are selected on the device (radix descent over the order keys,
    # sg_runtime.cu build_result_topk).  Uniform keys above: thousands of groups tie at the cut for $COUNT, the
    # selection gives up and the host sorts (same answer).  Skewed keys here: distinct counts at the top, few ties
    # at the cut — the device path end to end, for Count, for a mean, with and without a second aggregation.
    keys = (rng.pareto(1.1, n) * 40).astype(np.int64) % 300_000
    s2 = Spec([("k", STR), ("m", INT), ("w", INT)])
    s2.add_rows({"k": np.array(["key%d" % v for v in keys]), "m": rng.integers(0, 10000, n), "w": rng.integers(-500, 500, n)},
                block_rows=65536)
    both(s2, Q(s2, groups=["k"], aggs=["m", "w"], op="avg", limit=100))
    # Ordered by a mean, groups of thousands of rows: the reference's float running mean and the engine's exact
    # sum / count differ in the last bits (DESIGN.md §7), so two groups whose means agree to 1e-12 may swap places.
    # Checked instead: the list is ordered by the engine's own means, it holds `limit` groups, none of them lies
    # below the oracle's cut by more than the tolerance, and every listed group matches the oracle's group.
    for ob, limit in (("w", 1000), ("m", 7)):
        q = Q(s2, groups=["k"], aggs=["m", "w"], op="avg", order_by=ob, limit=limit)
        g = run_gpu(s2, q)
        o = run_oracle(s2, Q(s2, groups=["k"], aggs=["m", "w"], op="avg", order_by=ob))
        means = [r.Hists[ob].Mean() for r in g.Sorted]
        assert len(means) == limit and means == sorted(means, reverse=True)
        assert g.NumGroups == len(o.Results) and g.MatchedCount == o.MatchedCount
        cut = o.Sorted[limit - 1].Hists[ob].Avg
        for r in g.Sorted:
            assert o.Results[r.GroupByKey].Hists[ob].Avg >= cut - 1e-9 * max(1.0, abs(cut)), ("below the cut", r.GroupByKey)
            compare_group(r, o.Results[r.GroupByKey], q.aggs, False, ("Results", r.GroupByKey))


# ---------------------------------------------------------------------------------------------------
# SURVEY §8(f) N1 / N2 on the hot path: block directories in sybil's on-disk format -> native (C++) gob
# reader -> sg_table_add_block -> CUDA scan, against the oracle over the blocks the directories were
# written from
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("narrow", [False, True])
def test_block_directories_through_the_native_reader(tmp_path, narrow):
    """write_block_dir (gob int_*.db / str_*.db / info.db, one gzipped) -> sgob_read_block_dir -> the C ABI.
    narrow: the reader keeps the file's varints narrow (uint16 ids, int16 / int32 deltas) instead of widening
    them to Go's decoded types; both must give the oracle's result."""
    import ctypes as C
    from sybil_b200 import blockdir
    from sybil_b200 import engine as E
    rng = np.random.default_rng(77)
    n = 9000
    s = Spec([("age", INT), ("big", INT), ("lat", INT), ("host", STR), ("uid", STR), ("time", INT)])
    s.forms = "wide"  # the directories are written from Go's decoded types; the READER decides what it hands over
    s.add_rows({"age": rng.integers(10, 30, n), "big": rng.integers(-(1 << 40), 1 << 45, n),
                "lat": (rng.integers(0, 65536, (n, 4)).sum(1) * 23470 // (4 * 65535) + 30),
                "host": np.array(["h%d" % x for x in rng.integers(0, 5, n)]),
                "uid": np.array(["u%d" % x for x in rng.integers(0, 4 * n, n)]),
                "time": 1500000000 + np.sort(rng.integers(0, 7200, n))},
               {"age": rng.random(n) > 0.1, "host": rng.random(n) > 0.1}, threshold=50, block_rows=4000)
    g = F.gobread()
    g.sgob_set_narrow(1 if narrow else 0)
    names = (C.c_char_p * len(s.key_table))(*[nm.encode() for nm, _ in s.key_table])
    types = (C.c_int32 * len(s.key_table))(*[t for _, t in s.key_table])
    t = E.Table("dirs", s.key_table)
    t.IntInfo = dict(s.IntInfo)
    handles = []
    try:
        saw_narrow = False
        for i, b in enumerate(s.blocks):
            d = str(tmp_path / ("block%d" % i))
            blockdir.write_block_dir(d, b, s.key_table, compress=(i % 2 == 1))
            err = C.create_string_buffer(512)
            h = g.sgob_read_block_dir(d.encode(), names, types, len(s.key_table), None, b.block_index, err, len(err))
            assert h, err.value.decode()
            handles.append(h)
            desc = g.sgob_block_desc(h)
            for k in range(desc.contents.ncols):
                cd = desc.contents.cols[k]
                saw_narrow = saw_narrow or cd.id_bits == 16 or cd.value_bits in (16, 32) and cd.col_type == INT
            t.add_block_desc_ptr(desc)
        assert saw_narrow == narrow
        for q in (Q(s, groups=["host"], aggs=["lat", "big"], op="hist"),
                  Q(s, int_filters=[("age", "gt", 15), ("big", "lt", 1 << 44)], str_filters=[("host", "neq", "h3")],
                    groups=["age"], aggs=["lat"], op="avg"),
                  Q(s, groups=["uid"], aggs=["age"], op="avg", limit=50),
                  Q(s, aggs=["lat"], op="hist", time_col="time", time_bucket=600)):
            compare(run_gpu(s, q, table=t), run_oracle(s, q), q)
    finally:
        g.sgob_set_narrow(0)
        t.close()
        for h in handles:
            g.sgob_block_free(h)


def test_pinned_buffer_reuse_needs_sync():
    """The zero-copy staging path (arrays inside a region from sg_pinned_alloc are DMA'd in place): a host that
    recycles one pinned buffer for successive batches calls sg_table_sync before it overwrites the buffer
    (INTEGRATION.md §3).  Two batches generated into the SAME pinned arena, one after the other; the table must
    hold both, bit for bit (oracle over all blocks)."""
    from sybil_b200 import engine as E
    from sybil_b200 import synth
    from oracle.oracle_ffi import OracleTable
    spec = synth.config("c3", total_rows=6 * 30000, block_rows=30000)
    s = Spec(spec.key_table)
    s.IntInfo = dict(spec.IntInfo)
    q = Q(s, **synth.query_for(spec))
    ot = OracleTable(spec.key_table)
    t = E.Table("pin", spec.key_table)
    t.IntInfo = dict(spec.IntInfo)
    nbytes = 64 << 20
    arena = t.lib.sg_pinned_alloc(t.ctx.h, nbytes)
    assert arena
    try:
        for first in (0, 3):
            store = synth.generate(spec, first, 3, nthreads=2, arena_ptr=arena, arena_bytes=nbytes)
            for i in range(store.num_blocks()):
                ot.add_block(store.block(i))  # (the oracle copies the arrays)
            ptrs, n = store.block_ptrs()
            t.add_blocks(ptrs, n)
            t.sync()  # the DMA out of the arena has finished: the next batch may overwrite it
            store.close()
        d, keep = q.desc()
        compare(run_gpu(s, q, table=t), ot.query(d, q.aggs, nthreads=2), q)
    finally:
        t.lib.sg_pinned_free(t.ctx.h, arena)
        t.close()
        ot.close()


@pytest.mark.parametrize("variant", ["8", "16"])
def test_both_kernel_builds_agree_with_the_oracle(variant, monkeypatch):
    """The library holds two builds of the scan kernel (16-warp CTAs, one per SM; 8-warp CTAs, two per SM) and
    picks one per plan; SG_VARIANT forces either.  Both must give the oracle's result on plans of every shape:
    filters + two group columns + histogram (the C3 shape, whose default is the 8-warp build), time rollup with
    the histogram cache, high-cardinality group-by with global accumulators, MultiHist."""
    monkeypatch.setenv("SG_VARIANT", variant)
    s = _wide_spec(5, 70000, 35000, nulls=False)
    for q in (Q(s, int_filters=[("f0", "gt", 100), ("f1", "lt", 900000)], str_filters=[("s0", "neq", "v3")],
                groups=["s1", "d"], aggs=["lat"], op="hist"),
              Q(s, aggs=["lat"], op="hist", time_col="time", time_bucket=3600),
              Q(s, groups=["s1"], aggs=["f1", "lat"], op="avg")):
        compare(run_gpu(s, q), run_oracle(s, q), q)
    r = random_spec(6, nrows=12000, block_rows=5000, threshold=40)
    for q in (Q(r, groups=["uid"], aggs=["age", "lat"], op="avg"),
              Q(r, int_filters=[("age", "gt", 12)], groups=["host", "age"], aggs=["lat", "big"], op="hist", loghist=True),
              Q(r, str_filters=[("state", "re", "^s1")], groups=["state"], aggs=["big"], op="hist")):
        compare(run_gpu(r, q), run_oracle(r, q), q)


def test_set_filters_in_nin_like_filter_go():
    # SetFilter (filter.go:252-285) over set columns (unpackSetCol, column_store_io.go:611-688): sticky bits in
    # the slot word; alone, two at once, mixed with pass-counting int / str filters, with groups, hist and time
    s = random_spec(31, nrows=6000, block_rows=1700, sets=True)
    for op, tag in (("in", "t3"), ("nin", "t3"), ("in", "nope"), ("nin", "nope")):
        g, o = both(s, Q(s, set_filters=[("tags", op, tag)], groups=["host"], aggs=["lat"], op="avg"))
    assert g.MatchedCount > 0
    both(s, Q(s, set_filters=[("tags", "in", "t1"), ("tags", "nin", "t2")], groups=["state"], aggs=["lat"], op="hist"))
    g, o = both(s, Q(s, int_filters=[("age", "gt", 12)], str_filters=[("state", "neq", "s3")],
                     set_filters=[("tags", "nin", "t5"), ("tags", "in", "t0")], groups=["host", "age"], aggs=["lat", "big"],
                     op="hist"))
    assert 0 < g.MatchedCount < 6000
    both(s, Q(s, set_filters=[("tags", "in", "t4")], groups=["host"], aggs=["lat"], op="hist", time_col="time", time_bucket=600))
    both(s, Q(s, set_filters=[("tags", "nin", "t4")]))


def test_set_column_values_form_and_many_tags():
    # the non-bucketed file form (more than `threshold` distinct tags): rows below len(Values) count as populated
    # even with an empty set; and a set column next to fail-mode-capable filters keeps the query in count mode
    from sybil_b200 import blocks as B
    n = 3000
    rng = np.random.default_rng(9)
    s = Spec([("v", INT), ("tags", SET)])
    s.forms = "wide"
    vals = [list(rng.choice(400, int(k), replace=False)) if k else ([] if i % 2 else None)
            for i, k in enumerate(rng.integers(0, 5, n - 500))]
    blk = B.SavedBlock(0, n)
    blk.cols.append(B.encode_int_column(0, rng.integers(0, 100000, n), np.ones(n, bool), threshold=10))
    blk.cols.append(B.set_values_to_bins(1, vals, ["tag%d" % i for i in range(400)]))
    s.blocks.append(blk)
    s.IntInfo["v"] = (0, 99999)
    for op, tag in (("in", "tag7"), ("nin", "tag7"), ("nin", "zzz")):
        g, o = both(s, Q(s, int_filters=[("v", "lt", 50000)], set_filters=[("tags", op, tag)], aggs=["v"], op="hist"))
    assert g.MatchedCount > 0


def test_set_column_limits_and_misuse():
    from sybil_b200 import engine as E
    s = random_spec(33, nrows=500, block_rows=500, sets=True)
    with pytest.raises(E.SybilGpuError):  # a set column cannot be grouped by (aggregate.go:125-143)
        run_gpu(s, Q(s, groups=["tags"]))
    with pytest.raises(E.SybilGpuError):  # IN / NIN are set ops
        run_gpu(s, Q(s, str_filters=[("host", "in", "h1")]))


def test_str_replace_like_table_query_go():
    # FLAGS.STR_REPLACE (table_query.go:34-50, column_store_io.go:515-549): group keys and filters see the
    # rewritten strings; strings that rewrite to the same text are one group
    s = random_spec(41, nrows=6000, block_rows=1700)
    rep = {"state": (r"^s(\d)\d*$", "S$1")}  # s0..s11 -> S0, S1 (s1, s10, s11), S2 ... S9
    g, o = both(s, Q(s, groups=["state"], aggs=["lat", "big"], op="hist", str_replace=rep))
    assert "S1\t" in g.Results and len(g.Results) == 11  # 10 rewritten names + the rows without the column
    both(s, Q(s, groups=["host", "state"], aggs=["lat"], op="avg", str_replace=rep, order_by="lat", limit=5))
    both(s, Q(s, groups=["state", "age"], aggs=["lat"], op="hist", str_replace=rep, time_col="time", time_bucket=900))
    # Filters see the rewritten strings.  Under a MERGING rewrite the reference's get_val_id hands a string it does
    # not know — an absent literal, and for re / nre the pattern text itself (filter.go:205) — the id
    # len(StringTable), which then is some other string's id, and overwrites that string in the lookup
    # (table_column.go:27-48): a reference bug the oracle restates (tests/test_oracle_sets_replace.py) and this
    # engine does not (DESIGN.md §7).  So: present literals under the merging rewrite, every op under a 1:1 one.
    for op, lit in (("eq", "S1"), ("neq", "S1")):
        both(s, Q(s, str_filters=[("state", op, lit)], groups=["state"], aggs=["lat"], op="avg", str_replace=rep))
    ren = {"state": ("^s", "S")}
    for op, lit in (("eq", "S1"), ("neq", "S1"), ("eq", "s1"), ("re", "^S1[01]?$"), ("nre", "^S1[01]?$")):
        both(s, Q(s, str_filters=[("state", op, lit)], groups=["state"], aggs=["lat"], op="avg", str_replace=ren))
    # a high-cardinality value-array column folded onto few keys, two rewritten columns at once
    rep2 = {"uid": (r"^u(\d).*$", "U$1"), "host": ("h", "node-")}
    g, o = both(s, Q(s, groups=["uid", "host"], aggs=["lat"], op="avg", str_replace=rep2))
    assert len(g.Results) <= 9 * 6 + 6


def _weighted_spec(seed, n=6000, block_rows=1700, threshold=5000, wvals=(1, 2, 5, 10, 100)):
    rng = np.random.default_rng(seed)
    s = Spec([("lat", INT), ("big", INT), ("host", STR), ("state", STR), ("time", INT), ("w", INT)])
    s.add_rows({"lat": rng.integers(0, 65536, (n, 4)).sum(1) * 23470 // (4 * 65535) + 30,
                "big": rng.integers(-(1 << 30), 1 << 40, n),  # (x weight x rows stays inside int64: the exact sum does not wrap)
                "host": np.array(["h%d" % v for v in rng.integers(0, 5, n)]),
                "state": np.array(["s%d" % v for v in rng.integers(0, 12, n)]),
                "time": 1500000000 + np.sort(rng.integers(0, 7200, n)),
                "w": rng.choice(np.asarray(wvals), n)},
               {"lat": rng.random(n) > 0.07, "host": rng.random(n) > 0.07}, threshold=threshold, block_rows=block_rows)
    return s


def test_weighted_queries_like_aggregate_go():
    # OPTS.WEIGHT_COL (aggregate.go:100-102,202-203; hist_basic.go:111-151): Count / hist Count / bucket counters /
    # sums weighted, Samples = rows, MatchedCount = rows.  Weight column fully populated.
    s = _weighted_spec(51)
    g, o = both(s, Q(s, groups=["host"], aggs=["lat", "big"], op="hist", weight_col="w"))
    assert g.Cumulative.Count > g.Cumulative.Samples == 6000
    both(s, Q(s, int_filters=[("lat", "gt", 9000)], str_filters=[("state", "neq", "s3")], groups=["host", "state"],
              aggs=["lat"], op="avg", weight_col="w", order_by="lat", limit=7))
    both(s, Q(s, aggs=["lat"], op="hist", weight_col="w"))                       # no group column
    both(s, Q(s, groups=["state"], aggs=["lat"], op="hist", weight_col="w", time_col="time", time_bucket=900))
    both(s, Q(s, groups=["host"], aggs=["lat"], op="hist", loghist=True, weight_col="w"))
    # a weight column stored as a value array (more distinct weights than the threshold).  Zero and negative
    # weights, and groups whose Count folds to 0, are pinned to the row-level reference by family W of
    # tests/edges.py (tests/test_parity_order.py): the reference's running float mean divides by a Count of 0 and
    # stays NaN (hist_basic.go:117), and it drops a block's group result whose Count is 0 when it combines blocks
    # (query_spec.go:143-145), so the oracle is not compared there.
    s2 = _weighted_spec(52, threshold=3, wvals=(1, 3, 7, 12, 40, 1000))
    both(s2, Q(s2, groups=["host"], aggs=["lat", "big"], op="hist", weight_col="w"))


def test_weighted_query_refuses_rows_without_a_weight():
    # Q13: a row lacking the weight column reuses the previous row's weight in the reference — not reproduced
    from sybil_b200 import engine as E
    rng = np.random.default_rng(5)
    n = 2000
    s = Spec([("lat", INT), ("w", INT)])
    s.add_rows({"lat": rng.integers(0, 100, n), "w": rng.integers(1, 4, n)}, {"w": rng.random(n) > 0.1})
    with pytest.raises(E.SybilGpuError) as e:
        run_gpu(s, Q(s, aggs=["lat"], weight_col="w"))
    assert e.value.status == F.SG_ERR_UNSUPPORTED


def test_hashed_slot_space_for_group_by_products_beyond_the_dense_space():
    # two group columns of 9,000 distinct strings each: 81M codes > 2^26 dense slots.  The scan keys an open-addressing
    # table on the device with the row's mixed-radix code (the reference's Go map over the key bytes,
    # aggregate.go:186-203) and the accumulators are indexed by the table index.
    rng = np.random.default_rng(61)
    n = 30000
    s = Spec([("a", STR), ("b", STR), ("v", INT), ("f", INT), ("time", INT)])
    s.add_rows({"a": np.array(["a%d" % x for x in rng.integers(0, 9000, n)]),
                "b": np.array(["b%d" % x for x in rng.integers(0, 9000, n)]),
                "v": rng.integers(0, 100000, n), "f": rng.integers(0, 100, n),
                "time": 1500000000 + np.sort(rng.integers(0, 3600, n))},
               {"a": rng.random(n) > 0.05, "v": rng.random(n) > 0.05}, block_rows=10000)
    # (8,648 and 8,713 of the 9,000 strings are drawn: with the missing-value code and "" that is 75.4M codes)
    g, o = both(s, Q(s, groups=["a", "b"], aggs=["v"], op="avg"))
    assert g.NumGroups > 25000
    both(s, Q(s, int_filters=[("f", "lt", 50)], str_filters=[("a", "neq", "a7")], groups=["a", "b"], aggs=["v", "f"], op="avg",
              order_by="v", limit=20))
    both(s, Q(s, groups=["b", "a"], aggs=["v"], op="avg", time_col="time", time_bucket=1800))


def test_hashed_slot_space_with_histograms():
    rng = np.random.default_rng(62)
    n = 12000
    s = Spec([("a", STR), ("b", STR), ("c", INT), ("v", INT)])
    s.add_rows({"a": np.array(["a%d" % x for x in rng.integers(0, 8300, n)]),
                "b": np.array(["b%d" % x for x in rng.integers(0, 8300, n)]),
                "c": rng.integers(0, 4, n), "v": rng.integers(0, 5000, n)}, block_rows=6000)
    # ~6,300 x 6,300 x 5 codes: three axes, one of them a bucket-encoded int column
    g, o = both(s, Q(s, groups=["a", "c", "b"], aggs=["v"], op="hist", limit=50))
    assert g.NumGroups > 11000
