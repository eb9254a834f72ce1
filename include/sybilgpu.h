/*
 * sybilgpu.h — C ABI of libsybilgpu.so, the H100 (sm_90a) scan-and-aggregate
 * engine that replaces sybil's per-block Go loop behind
 *
 *     func (t *Table) LoadAndQueryRecords(loadSpec *LoadSpec, querySpec *QuerySpec) int
 *                                                   (src/lib/table_query.go:18)
 *
 * The reference has no FFI; the seam is that Go method.  A cgo shim keeps gob
 * decoding, QuerySpec construction and printing in Go and hands the library the
 * post-gob flat arrays of SavedIntColumn / SavedStrColumn
 * (src/lib/column_store.go:46-64).  Every entry point below names the reference
 * code it stands in for.  Plain pointers and sizes only; no C++ or torch types.
 *
 * Conventions: every function returns an sg_status (0 = OK, <0 = error) unless it
 * returns a handle; nothing throws or aborts across the boundary; the message for
 * the last error on a context is sg_last_error().  All handles are owned by the
 * library and released by the matching *_free / *_destroy.  Host arrays passed in
 * descriptors are only read during the call (cgo rule: C never retains Go memory).
 */
#ifndef SYBILGPU_H
#define SYBILGPU_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SG_ABI_VERSION 4 /* 2: order_by_agg / order_asc / limit in sg_query_desc; 3: narrow arrays (id_bits / value_bits); \
                            4: set columns + SetFilter (SG_COL_SET, SG_OP_IN / SG_OP_NIN), sg_query_set_str_replace */

/* limits of one query (reference has none; beyond these -> SG_ERR_UNSUPPORTED).  Group keys: the product of the
 * group columns' distinct-value counts (x time buckets) may reach 2^31; up to 2^26 it is a dense array, beyond that
 * a hash table on the device keyed by the combined code (single GPU; at most 2^25 distinct groups per query).
 * Accumulators (count, sums, histogram counters per slot of that array or table) may take up to 24 GiB; with
 * sg_query_set_sparse_groups(q, 1) a plan past that holds accumulators for the groups that occur only, and the
 * 24 GiB limit applies to those (single GPU, sg_query_run only).  Weights and StrReplace over the hash table, or
 * over sparse accumulators, need sg_query_set_hashed_folds(q, 1). */
#define SG_MAX_FILTERS 15
#define SG_MAX_GROUPS 8
#define SG_MAX_AGGS 16
#define SG_MAX_COLS 64
/* CHUNK_SIZE, src/lib/table.go:44: rows per block never exceed this */
#define SG_BLOCK_ROWS 65536
/* MISSING_VALUE, src/lib/aggregate.go:31 */
#define SG_MISSING_KEY UINT64_MAX

typedef enum sg_status {
  SG_OK = 0,
  SG_ERR_INVALID = -1,     /* malformed descriptor / argument */
  SG_ERR_CUDA = -2,        /* CUDA runtime error, or no usable device */
  SG_ERR_UNSUPPORTED = -3, /* query shape outside this build (see DESIGN.md) */
  SG_ERR_NOMEM = -4,
  SG_ERR_NCCL = -5,
  SG_ERR_STATE = -6        /* call out of order */
} sg_status;

/* record.go:14-19 (INT_VAL = 1, STR_VAL = 2, SET_VAL = 3).  A set column (SavedSetColumn, column_store.go:66-74)
 * can be filtered on (SetFilter); like the reference it cannot be grouped by or aggregated. */
typedef enum sg_coltype { SG_COL_INT = 1, SG_COL_STR = 2, SG_COL_SET = 3 } sg_coltype;

/* SavedIntColumn.BucketEncoded / Values (column_store.go:46-64) */
typedef enum sg_encoding {
  SG_ENC_ABSENT = 0, /* no file for this column in the block: every row unpopulated */
  SG_ENC_BUCKET = 1, /* Bins[]{Value, Records[]} (inverted index) */
  SG_ENC_VALUES = 2  /* Values[] (one per row, rows >= len unpopulated) */
} sg_encoding;

/* filter.go:171-250 ops; RE/NRE are evaluated by the host into a bitset */
typedef enum sg_filter_op {
  SG_OP_GT = 0,
  SG_OP_LT = 1,
  SG_OP_EQ = 2,
  SG_OP_NEQ = 3,
  SG_OP_RE = 4,  /* str only: matches iff lut bit of the value's global id is set */
  SG_OP_NRE = 5, /* str only: populated and lut bit clear */
  SG_OP_IN = 6,  /* set only (SetFilter "in", filter.go:252-285): the row's set holds str_value */
  SG_OP_NIN = 7  /* set only ("nin"): the row has a set and it does not hold str_value */
} sg_filter_op;

/* FLAGS.OP (hist_basic.go:79) and FLAGS.LOG_HIST (hist.go:29) */
typedef enum sg_op_mode { SG_MODE_AVG = 0, SG_MODE_HIST = 1 } sg_op_mode;
typedef enum sg_hist_kind { SG_HIST_BASIC = 0, SG_HIST_MULTI = 1 } sg_hist_kind;
/* sg_query_desc.order_by_agg */
#define SG_ORDER_COUNT (-1)
#define SG_ORDER_NONE (-2)

typedef struct sg_ctx sg_ctx;
typedef struct sg_table sg_table;
typedef struct sg_query sg_query;
typedef struct sg_result sg_result;

/* ---- descriptors -------------------------------------------------------- */

/* IntFilter / StrFilter / SetFilter (filter.go:143-169). */
typedef struct sg_filter_desc {
  int32_t col_slot;
  int32_t col_type;      /* sg_coltype */
  int32_t op;            /* sg_filter_op */
  int32_t _pad;
  int64_t int_value;     /* IntFilter.Value */
  const char* str_value; /* StrFilter.Value for EQ/NEQ, SetFilter.Value for IN/NIN (not NUL-terminated) */
  int64_t str_len;
} sg_filter_desc;

/* Grouping (query_spec.go:73-76) + KeyTypes of the column */
typedef struct sg_group_desc {
  int32_t col_slot;
  int32_t col_type;
} sg_group_desc;

/* Aggregation (query_spec.go:78-83) + the table-level IntInfo{Min,Max}
 * the histogram is built from (table_column_info.go:18-24, hist.go:27-38). */
typedef struct sg_agg_desc {
  int32_t col_slot;
  int32_t _pad;
  int64_t info_min;
  int64_t info_max;
} sg_agg_desc;

/* QueryParams (query_spec.go:25-41) + the globals the hot path reads. */
typedef struct sg_query_desc {
  int32_t abi_version; /* SG_ABI_VERSION */
  int32_t op_mode;     /* sg_op_mode: FLAGS.OP == "hist" turns bucket tracking on */
  int32_t hist_kind;   /* sg_hist_kind: FLAGS.LOG_HIST */
  int32_t hist_bucket; /* FLAGS.HIST_BUCKET (hist_basic.go:51-53), 0 = unset */
  int32_t nfilters;
  int32_t ngroups;
  int32_t naggs;
  int32_t time_col_slot;   /* OPTS.TIME_COL_ID, -1 = no time series */
  int64_t time_bucket;     /* QuerySpec.TimeBucket, 0 = no time series */
  int64_t time_min;        /* table IntInfo of the time column: bounds the */
  int64_t time_max;        /*   dense time-bucket axis (rows outside are counted in overflow) */
  int32_t weight_col_slot; /* OPTS.WEIGHT_COL_ID, -1 = unweighted.  Count / hist Count / bucket counters / sums are
                            * weighted, Samples and MatchedCount count rows (aggregate.go:100-102,202-203).  A scanned
                            * row WITHOUT the column (an unlisted row of a bucket column, a row past a short value
                            * array, a block without the file) is what weight_carry decides */
  /* SortResults (aggregate.go:43-54,497-525): QuerySpec.OrderBy = "$COUNT" (SG_ORDER_COUNT), the name of an
   * aggregation (its index: groups ordered by Hists[col].Mean(), descending) or "" (SG_ORDER_NONE: no sort,
   * groups come in slot order); OrderAsc reverses the sorted list.  Ties (Go's sort is unstable): GroupByKey
   * ascending before the reversal.  A group without the histogram sorts as mean = -inf (Go would panic). */
  int32_t order_by_agg;
  int32_t order_asc;
  /* Rows without the weight column of a weighted query (weight_col_slot >= 0; ignored otherwise):
   *   0 = the query fails at sg_query_finish with SG_ERR_UNSUPPORTED when a scanned row lacks the column;
   *   1 = such a row takes the weight of the nearest earlier row of its block that has the column, or 1 when
   *       none does (aggregate.go:68,100-102: `weight` starts at 1 per block and is overwritten by every row
   *       holding the column, before the filters run).  Blocks never carry into each other.  This is what
   *       LoadAndQueryRecords computes.
   * Any other value is SG_ERR_INVALID. */
  int32_t weight_carry;
  /* FLAGS.LIMIT (printer.go): > 0 = only the first `limit` groups of the sorted list are materialised
   * (sg_result_num_groups); Cumulative and sg_result_num_groups_total still cover every group.  0 = all. */
  int64_t limit;
  const sg_filter_desc* filters;
  const sg_group_desc* groups;
  const sg_agg_desc* aggs;
} sg_query_desc;

/* One column of one block: the post-gob form of SavedIntColumn / SavedStrColumn / SavedSetColumn.
 *
 * Set columns (col_type SG_COL_SET, unpackSetCol column_store_io.go:611-688) come in the bucket form only:
 * Bins[i].Value = local string id of a tag, Bins[i].Records = the rows whose set holds it (a row may be listed
 * in several bins, never twice in one).  A bin lists at most NumRecords rows (a longer one, or a row >= NumRecords,
 * makes the block broken for queries that read the column, as the reference's "BLOCK SIZE CHANGED" does), and the
 * block's arrays must fit the 64 MiB staging buffer (SG_ERR_INVALID otherwise); a column may list any number of
 * (bin,row) pairs within those bounds.  The host turns the non-bucketed file form (Values [][]int32, written for more
 * than 5,000 distinct tags, column_store_io.go:183-192) into bins and passes len(Values) as `nvalues`: the
 * reference marks every row below it as populated, even with an empty set (column_store_io.go:672-682).
 *
 * Narrow arrays.  On disk the arrays are gob varints (1-3 bytes per small gap, SURVEY.md App. A); a decoder
 * that keeps them narrow instead of widening every element to Go's uint32 / int64 moves 2-3x fewer bytes
 * over PCIe and HBM.  The library takes them as they are and widens in the scan kernel:
 *   id_bits    0 / 32: record_ids is uint32_t[];  16: it points to uint16_t[] (a row id or gap is < 65,536 in
 *              every valid block, so this form always exists);
 *   value_bits 0 / 64 (int) or 0 / 32 (str): values_i64 is int64_t[] / values_i32 is int32_t[];
 *              int, 32 or 16: values_i64 points to int32_t[] / int16_t[] DELTAS (delta_values must be 1):
 *              decoded value k = value_base + deltas[0] + ... + deltas[k] (wrapping int64 arithmetic, like the
 *              reference's running sum, column_store_io.go:760-767);
 *              str, 16: values_i32 points to uint16_t[] local string ids (ids < len(StringTable) <= 65,536). */
typedef struct sg_column_desc {
  int32_t col_slot;
  int32_t col_type;     /* sg_coltype */
  int32_t encoding;     /* sg_encoding */
  int32_t delta_ids;    /* DeltaEncodedIDs: Records[] hold gaps (first absolute) */
  int32_t delta_values; /* ValueEncoded: Values[] hold gaps (int columns only) */
  uint32_t nbins;
  uint32_t nrecord_ids;        /* sum of len(Bins[i].Records) */
  uint32_t nvalues;            /* len(Values) */
  const int64_t* bin_values;   /* int: Bins[i].Value; str: Bins[i].Value widened */
  const uint32_t* bin_offsets; /* nbins+1 offsets into record_ids */
  const uint32_t* record_ids;  /* concatenated Bins[i].Records */
  const int64_t* values_i64;   /* int VALUES */
  const int32_t* values_i32;   /* str VALUES (local string ids) */
  /* SavedStrColumn.StringTable as one byte buffer + ndict+1 offsets */
  uint32_t ndict;
  int32_t id_bits;
  const char* dict_bytes;
  const uint32_t* dict_offsets;
  int32_t value_bits;
  int32_t _pad;
  int64_t value_base;
} sg_column_desc;

/* Block info.db IntInfoMap entry (column_store.go:39-44) for zone-map pruning */
typedef struct sg_int_info {
  int32_t col_slot;
  int32_t _pad;
  int64_t min;
  int64_t max;
} sg_int_info;

typedef struct sg_block_desc {
  int64_t block_index;
  int32_t num_records; /* SavedColumnInfo.NumRecords, 1..SG_BLOCK_ROWS */
  int32_t ncols;
  const sg_column_desc* cols;
  int32_t ninfo; /* may be 0: then the block is never pruned */
  int32_t _pad;
  const sg_int_info* info;
} sg_block_desc;

/* ---- context ------------------------------------------------------------ */

/* One context per process and GPU (one process per GPU under a launcher). */
sg_ctx* sg_create(int device, int* status_out);
void sg_destroy(sg_ctx* ctx);
const char* sg_last_error(sg_ctx* ctx);
int sg_abi_version(void);
/* number of SMs / device name of the context's GPU (0 / "" without one) */
int sg_device_sm_count(sg_ctx* ctx);

/* cudaHostAlloc'd staging the Go side fills (gob decodes straight into it). */
void* sg_pinned_alloc(sg_ctx* ctx, size_t bytes);
void sg_pinned_free(sg_ctx* ctx, void* p);

/* ---- resident table: blocks staged once into HBM -------------------------
 * Stands in for LoadBlockFromDir + unpackIntCol/unpackStrCol
 * (table_block_io.go:225-310, column_store_io.go:493-609,690-780): the encoded
 * arrays are copied to HBM as they are; decoding happens inside the query kernel. */
sg_table* sg_table_create(sg_ctx* ctx, int32_t num_col_slots, const int32_t* col_types);
void sg_table_free(sg_table* t);
/* Copies the block's arrays host->device (async on the table's copy stream),
 * interns its string tables into the table's global dictionary and its int bin
 * values into the per-column value dictionary.  Returns SG_ERR_INVALID for a
 * malformed descriptor (the block is not added).
 * Lifetime of the descriptor's arrays: everything is read during the call EXCEPT record_ids / values that lie
 * inside a region from sg_pinned_alloc — those are DMA'd in place (no bounce copy) and must stay untouched
 * until sg_table_sync (or the next sg_query_run) returns. */
int sg_table_add_block(sg_table* t, const sg_block_desc* block);
/* Batch form.  Arrays that lie inside one region from sg_pinned_alloc are mirrored into HBM with a
 * few large copies instead of one per array (full PCIe rate); otherwise as n calls above. */
int sg_table_add_blocks(sg_table* t, const sg_block_desc* const* blocks, int64_t n);
int sg_table_sync(sg_table* t); /* wait for staged copies */
/* forget the staged blocks, keep arena + dictionaries (re-staging without reallocation) */
int sg_table_clear(sg_table* t);
int64_t sg_table_num_blocks(sg_table* t);
int64_t sg_table_num_rows(sg_table* t);
int64_t sg_table_device_bytes(sg_table* t);
/* global string dictionary of a str column slot (for host-side regex LUTs and
 * rendering keys): number of strings / i-th string */
int64_t sg_table_dict_size(sg_table* t, int32_t col_slot);
int sg_table_dict_get(sg_table* t, int32_t col_slot, int64_t id, const char** bytes, int64_t* len);
/* value dictionary of a bucket-encoded int column (dense group-by axis) */
int64_t sg_table_intdict_size(sg_table* t, int32_t col_slot);
int sg_table_intdict_get(sg_table* t, int32_t col_slot, int64_t id, int64_t* value);
/* Multi-GPU fast path: when every rank numbers group keys identically the dense
 * partials merge with two all-reduces and no dictionary exchange.  Seed the
 * dictionaries (e.g. with the table's StrInfo) BEFORE staging blocks; later strings
 * append after the seed.  Optional: sg_query_allreduce detects differing
 * dictionaries and exchanges them itself. */
int sg_table_dict_seed_str(sg_table* t, int32_t col_slot, const char* bytes, const uint32_t* offsets, int64_t n);
int sg_table_dict_seed_int(sg_table* t, int32_t col_slot, const int64_t* values, int64_t n);
int64_t sg_table_encoded_bytes(sg_table* t); /* bytes of encoded column arrays resident */
int64_t sg_table_h2d_bytes(sg_table* t);     /* bytes copied host->device while staging */

/* ---- query ---------------------------------------------------------------
 * sg_query_begin .. sg_query_finish bracket what LoadAndQueryRecords does between
 * table_query.go:96 (block loop) and :415 (final combine + sort). */
sg_query* sg_query_begin(sg_ctx* ctx, sg_table* t, const sg_query_desc* desc);
void sg_query_free(sg_query* q);
/* host-evaluated regex for filter #filter_index (filter.go:215-237): bitset over the
 * GLOBAL string ids of that column, nbits = sg_table_dict_size at call time.  Blocks staged
 * later (sg_table_add_block, sg_query_submit_block) may add strings; planning then refuses the
 * query with SG_ERR_STATE until the bitset is set again over the grown dictionary. */
int sg_query_set_str_lut(sg_query* q, int32_t filter_index, const uint32_t* bits, int64_t nbits);
/* StrReplace (FLAGS.STR_REPLACE "col:pattern:replacement", table_query.go:34-50): the reference rewrites a str
 * column's string table with regexp.ReplaceAllString while it unpacks a block (column_store_io.go:515-549), so
 * filters and group keys see the rewritten strings and rows whose strings rewrite to the same text fall into
 * one group.  As for RE/NRE the regexp runs on the host, once per distinct string: bytes/offsets hold the
 * rewritten text of every string of the column's GLOBAL dictionary (n == sg_table_dict_size at call time, n+1
 * offsets).  Group keys of that column are then rendered from the rewritten strings and groups that rewrite to
 * the same key are combined (their str id in sg_result_group is the smallest global id of the class).  Filters
 * on a rewritten column must be sent by the host as RE / NRE with a bitset evaluated on the rewritten strings
 * (EQ "x" = RE bitset of the strings that rewrite to "x").  Call between sg_query_begin and sg_query_finish;
 * n == 0 removes the rewrite.  Not combinable with a cross-GPU merge over differing dictionaries. */
int sg_query_set_str_replace(sg_query* q, int32_t col_slot, const char* bytes, const uint32_t* offsets, int64_t n);
/* Sparse group accumulators (the Go reference's result map holds only the groups that occur, aggregate.go:186-203).
 *   0 (default) = a plan whose accumulators pass 24 GiB (groups x histogram counters) fails with SG_ERR_UNSUPPORTED;
 *   1 = such a plan scans twice: a discovery pass collects the group keys of every row that passes into a table on
 *       the device and numbers them, then the aggregation pass accumulates into arrays sized by those L live
 *       groups, and only those are read back.  It fails with SG_ERR_UNSUPPORTED when the L groups' accumulators
 *       pass 24 GiB, for weighted queries and StrReplace unless sg_query_set_hashed_folds(q, 1), and under
 *       sg_query_allreduce.  Plans within the limit run as with 0.  The streaming path needs every block staged
 *       before the first pass: sg_query_submit_block fails with SG_ERR_UNSUPPORTED while the setting is 1.
 * Any other value is SG_ERR_INVALID.  Takes effect at the next sg_query_run (a prepared query plans again). */
int sg_query_set_sparse_groups(sg_query* q, int32_t on);
/* Weights and StrReplace over hashed group keys (the Go reference's result map holds the keys that occur, and every
 * row adds its weight, aggregate.go:100-102,186-203).  A weighted query groups by the weight value as a hidden axis,
 * and StrReplace groups by the original strings; both are then folded: every (group, weight value, original string)
 * entry's accumulators are combined onto the group it belongs to, multiplied by its weight.
 *   0 (default) = a weighted or StrReplace query whose group keys go through the hashed table (past 2^26 codes) fails
 *       with SG_ERR_UNSUPPORTED after the scan, and with sparse group accumulators it is refused when planned;
 *   1 = such a query is folded on the device, behind the scan and before anything is read back, on hashed plans and,
 *       with sg_query_set_sparse_groups(q, 1), on sparse ones (single GPU).  Rows without the weight column still
 *       need weight_carry; a table the folded keys fill up still fails with SG_ERR_UNSUPPORTED.
 * Dense plans fold on the host with either value.  Any other value is SG_ERR_INVALID.  Takes effect at the next
 * sg_query_run (a prepared query plans again). */
int sg_query_set_hashed_folds(sg_query* q, int32_t on);
/* ShouldLoadBlockFromDir (table_block_io.go:110-182): 1 = load, 0 = pruned */
int sg_query_should_load(sg_query* q, const sg_block_desc* block);
/* Resident path: run the scan over every staged block of the table
 * (zone-map pruning applied from the info each block was staged with). */
int sg_query_run(sg_query* q);
/* Streaming path (end to end from host buffers): stage + scan one block; blocks
 * are batched internally, H2D overlaps the previous batch's kernel. */
int sg_query_submit_block(sg_query* q, const sg_block_desc* block);
/* CombineResults (aggregate.go:414-467) across GPUs: NCCL all-reduce of the dense
 * per-group partials (sum region + max region).  Ranks whose dictionaries / time
 * axes differ first all-gather them and re-lay their partials by the union, after
 * which the str ids of sg_result_group index that union (use sg_result_group_key
 * for the strings).  Collective: every rank must call it.  No-op without a
 * communicator. */
int sg_query_allreduce(sg_query* q);
/* sync, D2H, build the result (CombineResults + Cumulative + SortResults) */
int sg_query_finish(sg_query* q, sg_result** out);
/* device time of the scan kernels of this query so far (CUDA events), ms */
double sg_query_kernel_ms(sg_query* q);
int64_t sg_query_kernel_launches(sg_query* q);

/* ---- multi-GPU -----------------------------------------------------------
 * One process per GPU; the host exchanges the 128-byte NCCL id by its own means. */
int sg_comm_unique_id(sg_ctx* ctx, char id_out[128]);
int sg_comm_init(sg_ctx* ctx, const char id[128], int rank, int nranks);

/* ---- result --------------------------------------------------------------
 * QueryResults (query_spec.go:14-22).  Groups come sorted as sg_query_desc.order_by_agg / order_asc say
 * (SortResults made deterministic, aggregate.go:43-54,497-525). */
void sg_result_free(sg_result* r);
int64_t sg_result_matched_count(sg_result* r); /* QueryResults.MatchedCount */
int64_t sg_result_num_groups(sg_result* r);    /* groups materialised: min(len(Results), limit) */
int64_t sg_result_num_groups_total(sg_result* r); /* len(Results) */
int64_t sg_result_num_broken(sg_result* r);    /* blocks dropped: "BLOCK SIZE CHANGED" */
int64_t sg_result_num_skipped(sg_result* r);   /* blocks pruned by the zone map */
/* i-th group (0-based, sorted).  key_out: ngroups u64 (ints two's complement,
 * strs GLOBAL string id, missing = SG_MISSING_KEY); Result.Count / Result.Samples */
int sg_result_group(sg_result* r, int64_t i, uint64_t* key_out, int64_t* count, int64_t* samples);
/* rendered GroupByKey "a\tb\t" (translate_group_by, aggregate.go:284-324) */
int sg_result_group_key(sg_result* r, int64_t i, const char** bytes, int64_t* len);

/* histogram state of aggregation #agg of group i (i = -1: Cumulative "TOTAL"):
 * BasicHistCachedInfo (hist_basic.go:10-26) without Averages/Outliers. */
typedef struct sg_hist_view {
  int64_t count;       /* hist Count: values accepted (hist_basic.go:104-116) */
  int64_t sum;         /* exact int64 sum of accepted values (wrapping) */
  int64_t min, max;    /* hist Min / Max as the reference tracks them */
  double avg;          /* sum / count */
  int32_t num_buckets; /* NumBuckets (basic) */
  int32_t bucket_size; /* BucketSize (basic) */
  int32_t nvalues;     /* len(Values) (basic) or total counters (multi) */
  int32_t nsubhists;   /* 0 for basic */
  const int64_t* values; /* bucket counters, nvalues entries */
} sg_hist_view;
int sg_result_hist(sg_result* r, int64_t i, int32_t agg, sg_hist_view* out);
/* GetPercentiles (hist_basic.go:153-183 / hist_multi.go:90-131): out100[100];
 * returns the number written (0 when the hist is empty) */
int sg_result_percentiles(sg_result* r, int64_t i, int32_t agg, int64_t* out100);
/* GetStdDev (hist_basic.go:192-219 / hist_multi.go:144-158) */
double sg_result_stddev(sg_result* r, int64_t i, int32_t agg);
/* GetSparseBuckets: edge -> count for count > 0; call with edges == NULL to size */
int64_t sg_result_sparse_buckets(sg_result* r, int64_t i, int32_t agg, int64_t* edges,
                                 int64_t* counts, int64_t cap);

/* time series (QueryResults.TimeResults): distinct buckets ascending, and the
 * per-(bucket, group) results as a second result object with the same accessors */
int64_t sg_result_num_time_buckets(sg_result* r);
int64_t sg_result_time_bucket(sg_result* r, int64_t b);
sg_result* sg_result_time_slice(sg_result* r, int64_t b); /* owned by r */

/* device-side numbers for bench.py */
typedef struct sg_stats {
  double kernel_ms;       /* sum of scan-kernel durations (CUDA events) */
  double h2d_ms;          /* staged copies, streaming path */
  int64_t kernel_launches;
  int64_t h2d_bytes;
  int64_t d2h_bytes;
  int64_t rows_scanned;
  int64_t blocks_scanned;
  int64_t encoded_bytes;  /* bytes of encoded column arrays the kernels read */
} sg_stats;
int sg_query_stats(sg_query* q, sg_stats* out);

#ifdef __cplusplus
}
#endif
#endif /* SYBILGPU_H */
