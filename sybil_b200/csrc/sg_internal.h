// sg_internal.h — structures shared by the host runtime (sg_runtime.cu) and the
// scan kernels (sg_kernels.cu).  Not part of the C ABI.
#pragma once
#include <cstdint>

#include "../../include/sybilgpu.h"

namespace sg {

// ---- device-resident block format ---------------------------------------------
// One DevCol per (block, column slot).  The encoded arrays are the reference's
// post-gob arrays copied verbatim into HBM (16-byte aligned); decode happens in
// the scan kernel.
enum : uint32_t {
  COL_DELTA_IDS = 1u,     // SavedIntColumn.DeltaEncodedIDs
  COL_DELTA_VALUES = 2u,  // SavedIntColumn.ValueEncoded
  COL_IS_STR = 4u,
  COL_BROKEN = 8u,        // "BLOCK SIZE CHANGED DURING QUERY" found at staging
  COL_STATS = 16u,        // vmin/vmax hold the exact extents of the decoded int values
  COL_TMA = 32u,          // data_chunk/data_row locate `data` inside an arena tensor map
  COL_FULL = 64u,         // bucket column: the bins list every row of [0, NumRecords) exactly once (checked by
                          // the staging statistics kernel), so no row is unpopulated for this column
  // narrow arrays (sybilgpu.h, sg_column_desc::id_bits / value_bits): `data` holds
  COL_ID16 = 128u,        //   uint16 record ids / gaps
  COL_VAL32 = 256u,       //   int32 deltas relative to vbase (int VALUES)
  COL_VAL16 = 512u,       //   int16 deltas relative to vbase (int VALUES) / uint16 local string ids (str VALUES)
  COL_SET = 1024u,        // set column (SavedSetColumn): bucket form, a row may sit in several bins; vmin holds the
                          // number of leading rows that are populated whatever the bins say (len(Values) of the
                          // non-bucketed file form, column_store_io.go:672-682)
  COL_SEGS = 2048u,       // set column listing more than SG_BLOCK_ROWS (tag,row) pairs: this DevCol is its first segment,
                          // vmax holds (number of further segments << 32) | index of the first of them in
                          // LaunchParams::segs.  Every segment is a self-contained bucket column of whole bins (at most
                          // SG_BLOCK_ROWS entries); none carries COL_TMA, so all are read with plain loads
  COL_CODES = 4096u,      // bucket int / str column of at most 255 bins whose rows the staging statistics kernel checked
                          // (each listed once, all < NumRecords): `codes` holds every row's bin index as one byte in row
                          // order, 0xFF for a row the column does not list, padded to 16 bytes.  The scan reads the
                          // codes instead of walking the ids (no COL_TMA: the union below no longer locates the ids)
};
// log2(4-byte-id or 8-byte-value width / stored width): the row pitch of the arena view a column's tiles are
// fetched through is 128 >> shift bytes, so a warp tile always holds 1024 ids / 512 values
__host__ __device__ static inline uint32_t col_shift(uint32_t flags) {
  return (flags & (COL_ID16 | COL_VAL32)) ? 1u : ((flags & COL_VAL16) ? 2u : 0u);
}

struct DevCol {
  uint32_t enc;     // sg_encoding
  uint32_t flags;   // COL_*
  uint32_t nbins;   // non-empty bins (BUCKET)
  uint32_t nitems;  // record ids (BUCKET) or values (VALUES)
  uint32_t nremap;  // str: dictionary size; int BUCKET: nbins
  int32_t oob_gid;  // str: global id used for a local id outside the dictionary
  union {
    const int64_t* bin_values;  // BUCKET: [nbins] int value, or local string id widened
    int64_t vbase;              // VALUES with narrow deltas: decoded value k = vbase + deltas[0..k] (0 otherwise)
  };
  const uint32_t* bin_offsets;  // [nbins+1]
  const void* data;             // record ids u32[] | values i64[] | values i32[]
  const int32_t* remap;         // str: local id -> global id; int BUCKET: bin -> value-dict code
  // exact extents of the decoded values (int columns), computed by the engine when the block is
  // staged (bucket columns: on the host from the bin values; value arrays: stats kernel)
  int64_t vmin, vmax;
  union {
    // COL_TMA: `data` as a coordinate of the arena chunk's tensor map ({128 B, rows}): row = byte offset / 128
    struct {
      uint32_t data_chunk, data_row;
    };
    const uint8_t* codes;  // COL_CODES: per-row bin indices (see there)
  };
};
static_assert(sizeof(DevCol) == 80, "DevCol layout");

// A block's weight column leaves rows of its nrec rows unlisted, so they carry an earlier row's weight: a bucket
// column not checked to list every row, or a value array shorter than the block.  An absent column lists no row:
// every row keeps weight 1 without a carry.
__host__ __device__ static inline bool weight_needs_carry(const DevCol& c, uint32_t nrec) {
  return (c.enc == SG_ENC_BUCKET && !(c.flags & COL_FULL)) || (c.enc == SG_ENC_VALUES && c.nitems < nrec);
}

struct DevBlock {
  int64_t block_index;
  uint32_t num_records;
  uint32_t _pad;
};

// ---- query plan (device copy read by the kernels) ---------------------------------
constexpr int MAX_SUBHISTS = 64;

// The scalar words that open the accumulator array (Plan::scalars).  All of them lie in the region a cross-GPU merge
// sums.  A nonzero time overflow, rows on weight code 0, table full or sparse key missing fails the query.
enum : uint32_t {
  SC_MATCHED = 0,         // rows that passed every filter (scan)
  SC_BROKEN = 1,          // blocks the scan found broken (scan)
  SC_TIME_OVERFLOW = 2,   // rows outside the planned time axis (scan)
  SC_NO_WEIGHT = 3,       // weighted folds: rows left on weight code 0 without weight_carry
  SC_TABLE_FULL = 4,      // hashed slot space: inserts that found the table full (scan, fold_insert)
  SC_SPARSE_MISSING = 5,  // sparse plans: rows whose key the aggregation launch did not find (scan)
  SC_FOLD_ENTRIES = 6,    // device folds: the table's occupied entries (fold_rows)
  SC_FOLD_CANON = 7,      // ... the canonical ones among them (fold_rows)
  // the cross-GPU merge header (sg_query_allreduce, cleared again after the merge): broken staged blocks, skipped
  // blocks, rows scanned, blocks scanned, then four words that check the ranks' axes agree
  SC_MERGE = 8,
  SC_MERGE_AXES = 12,
  SCALAR_WORDS = 16,
  // a sparse plan's discovery launch writes its scalars to an array of its own, followed by two counters (assign_ids):
  DISC_LIVE = SCALAR_WORDS,  // the table's occupied entries, which get the ids 0..live-1
  DISC_CANON,                // device folds: the canonical entries among them (ids 0..canon-1)
  DISC_WORDS
};

struct KFilter {
  int32_t col;
  int32_t is_str;
  int32_t op;       // sg_filter_op
  int32_t str_gid;  // EQ/NEQ literal as a global id (-1: not in the dictionary)
  int64_t ival;
  const uint32_t* lut;  // RE/NRE: bitset over global ids
  int64_t lut_bits;
  // SetFilter (IN / NIN, filter.go:252-285): sticky bits of the slot word, already shifted into place.  Every bin of
  // the set column ORs set_pbit ("the row has a set"; 0 for IN) into its rows, the bin of the literal also set_tbit
  // ("the set holds the literal"); the plan's filt_target asks for pbit set and tbit set (IN) / clear (NIN).
  uint32_t set_pbit, set_tbit;
};

struct KGroup {
  int32_t col;
  int32_t is_str;
  uint32_t stride;  // slot += (code + 1) * stride ; code 0 is "missing"
  uint32_t radix;
  // value-array encoded int group column: value -> dense code through an open-addressing table
  // (ids == 0xffffffff: empty) over the column's table-wide value dictionary
  const long long* vh_keys;
  const uint32_t* vh_ids;
  uint32_t vh_mask;  // capacity - 1
  // the global id (str) / value-dictionary code (int) whose key renders like a missing value and so takes code 0
  // with the missing rows: the int -1 (uint64(-1) is MISSING_VALUE, aggregate.go:125-143) and the string "";
  // -1 when the dictionary holds neither
  int32_t alias;
};

struct KSubHist {  // one BasicHist bucket layout (hist_basic.go:34-70)
  int64_t lo, hi;  // Info.Min / Info.Max of this (sub)hist
  int64_t reject_hi;  // Info.Max * 10, wrapping (hist_basic.go:104)
  int64_t bsize;      // BucketSize
  uint32_t nvals;     // len(Values)
  uint32_t base;      // offset of its counters inside the agg's counter row
  uint64_t magic;     // floor(2^64 / bsize) + 1 for bsize in [2, 2^32): x / bsize == umul64hi(x, magic), x < 2^32
                      // (0: bsize == 1 or bsize >= 2^32, no magic)
};

struct KAgg {
  int32_t col;
  int32_t nsub;  // number of bucket layouts: 0 in avg mode, 1 for a BasicHist, the sub-ranges of a MultiHist
  int64_t info_min, info_max;
  int64_t reject_hi;
  uint32_t nvals_total;
  uint32_t _pad;      // bit 0: the plan proved hist Count == Count for every scanned block (the
                      // kernel then skips the hist-Count reductions; accumulators-in-global plans only)
  uint32_t hrow_off;  // offset of this aggregation's counters inside a slot's row of the shared-memory
                      // histogram cache (HROW_NONE: its buckets go straight to L2)
  uint32_t multi;     // a MultiHist: a value outside every sub-range takes no bucket (also with one sub-range)
  uint64_t* buckets;  // [nslots][nvals_total]
  uint64_t* hcount;   // [nslots]
  uint64_t* sum;      // [nslots]
  int64_t* vmax;      // [nslots] max accepted value above info_max (INT64_MIN if none)
  int64_t* vmin;      // [nslots] (avg-mode min tracking; unused in v1)
  KSubHist sub[MAX_SUBHISTS];
};

struct Plan {
  int32_t nfilters, ngroups, naggs;
  int32_t ncolslots;
  int32_t time_col;  // -1 none
  int32_t hist_mode; // op_mode == HIST
  int64_t time_bucket;
  int64_t time_first;  // trunc(time_min / bucket)
  uint32_t time_radix;  // number of dense time buckets + 1 (0 = unused code)
  uint32_t time_stride;
  uint32_t gbits;       // low bits of a slot word holding the group slot
  uint32_t pass_target; // value of (slot >> gbits) for a row that passed everything
  uint32_t finc;        // 1 << gbits : added per passed filter
  uint32_t time_ok;     // bit added when the time column is a populated int
  uint32_t filt_target; // (slot >> gbits) & filt_mask == filt_target : passed all filters
  uint32_t filt_mask;
  uint32_t nslots;      // dense group slots
  uint32_t acc_words;   // replicated smem words per slot: 1 + 2*naggs (count; per agg word0, sum low limb);
                        // the sum high limbs (rarely touched) follow unreplicated
  uint32_t acc_repl;    // replication (power of two, <= 32); 0 = accumulate in global memory
  uint32_t fail_mode;   // filters set a sticky FAIL bit (finc) instead of counting passes: every filter column
                        // of every listed block populates every row (value array, or a bucket column with
                        // COL_FULL), so only the FAILING bins of a bucket column need to be walked
  uint32_t wcarry;      // weighted query with sg_query_desc.weight_carry: a row without the weight column (digit
                        // 0 on the last group axis) takes the digit of the nearest earlier row of its block
  // ---- slot window.  The slot words, the replicated accumulators and the histogram cache index a
  // LOCAL slot space: the group part plus a block-relative time code (1..time_win; 0 = no time).  The
  // global slot of local slot l is l + tbase, tbase = (first time code of the block - 1) * time_stride
  // from the time column's exact extents (staging statistics).  Without a time column, or when some
  // listed block has no extents, the window is the whole axis and tbase = 0.
  uint32_t lslots;      // local slots (== nslots when the window is the whole axis)
  uint32_t time_win;    // time codes a block may span (== time_radix - 1 for the whole axis)
  uint64_t time_magic;  // floor(2^64 / time_bucket) + 1 when time_bucket < 2^32 (0: none); see div_magic
  // ---- shared-memory histogram cache: hist_rows local slots x hist_row_words 32-bit counters, flushed
  // to the 64-bit bucket arrays in L2 when the window moves and when the CTA runs out of work
  uint32_t hist_rows;
  uint32_t hist_row_words;
  uint64_t* count;      // [nslots]
  uint64_t* scalars;    // [SCALAR_WORDS] (SC_*)
  uint32_t* block_status;  // per table block: 1 = broken in this query
  KFilter filters[SG_MAX_FILTERS];
  KGroup groups[SG_MAX_GROUPS];
  KAgg aggs[SG_MAX_AGGS];
};

struct LaunchParams {
  const Plan* plan;
  const DevBlock* blocks;
  const DevCol* cols;         // [nblocks_table][ncolslots]
  const DevCol* segs;         // continuation segments of COL_SEGS set columns (table-wide)
  const uint4* items;         // work items {block, mask, NumRecords, -}; mask bits 0..15 = aggregations this
                              // item computes, bit 31 = the item owns the block's Count / MatchedCount
  uint32_t nlist;
  uint32_t slot_bytes;        // 1, 2 (shared memory) or 4 (global scratch)
  uint32_t* work_counter;
  uint32_t* gslots;           // slot_bytes == 4: [grid][SG_BLOCK_ROWS]
  uint32_t* gbinpay;          // [grid][SG_BLOCK_ROWS] per-bin payload spill
  unsigned long long* gdummy; // [grid][32] sink for histogram reductions of rows that did not pass
  uint32_t smem_bytes;
  uint32_t acc_smem;          // accumulators replicated in shared memory (plan.acc_repl > 0)
  const void* tmaps;          // CUtensorMap[chunks][3] in global memory: row pitch 128 / 64 / 32 bytes (nullptr: plain
                              // vector loads)
  uint32_t stage_units;       // TMA staging per warp in units of 2 KiB (0 none; 2 = one 4 KiB tile; 4 = two)
  unsigned long long* dbg;    // optional [grid][16] cycle counters per phase (SG_PHASE_TIMING=1)
  uint32_t fold_every;        // blocks whose shared accumulators may be folded together (>= 1)
  uint32_t hashg;             // a group column is a value-array int column (hash lookup path; slot_bytes == 4)
  // Hashed slot space (group-by products beyond the dense 2^26 slots): after the group / time passes a row's
  // mixed-radix code (< 2^31) is looked up / inserted in this open-addressing table (key = code + 1, 0 = empty) and the
  // slot word's group bits are replaced by the table index, which is what the accumulators are indexed by
  // (plan.nslots == hmask + 1; a sparse plan's accumulators are indexed by hids below, plan.nslots == its live groups,
  // and the table has hmask + 1 entries all the same).  nullptr: the slot space is dense.  SC_TABLE_FULL counts rows that
  // found the table full.
  uint32_t* hkeys;
  uint32_t hmask;
  // Sparse group accumulators (sg_query_set_sparse_groups): the same table is filled by a discovery launch
  // (hdisc = 1: codes are inserted, nothing is counted or aggregated), then each occupied entry gets a dense id
  // (assign_ids), then the aggregation launch (hids != nullptr) looks every code up without inserting and writes
  // hids[index] into the slot word's group bits.  The accumulators are indexed by that id.  SC_SPARSE_MISSING counts rows
  // whose code the aggregation launch did not find (an internal inconsistency that fails the query).
  const uint32_t* hids;
  uint32_t hdisc;
};
__host__ __device__ static inline uint32_t slot_hash(uint32_t x) {
  x ^= x >> 16;
  x *= 0x7feb352du;
  x ^= x >> 15;
  x *= 0x846ca68bu;
  x ^= x >> 16;
  return x;
}

// the hash both sides of the value -> code table use
__host__ __device__ static inline uint32_t vh_hash(long long v) {
  unsigned long long x = (unsigned long long)v;
  x ^= x >> 33;
  x *= 0xff51afd7ed558ccdull;
  x ^= x >> 33;
  return (uint32_t)x;
}

// host-callable launchers (sg_kernels.cu).  The kernel unit is compiled twice, into two namespaces:
//   w16: CTAs of 16 warps, one per SM (up to 227 KiB of shared memory: 16-bit slot words, big accumulator sets);
//   w8:  CTAs of 8 warps, two per SM (113 KiB each).  Two independent CTAs hide each other's barriers, look-back
//        waits and the L2-bound histogram pass (the runtime picks the build per plan).
#define SG_DECLARE_VARIANT(ns)                                                                                          \
  namespace ns {                                                                                                        \
  int launch_scan(const LaunchParams& lp, int grid, void* stream);                                                      \
  /* extents of value-array int columns, COL_FULL and COL_CODES of bucket columns: items[i] = index into cols[]       \
   * (block * ncolslots + slot), codes[i] = where item i's per-row codes go (0: none) */                               \
  int launch_stats(DevCol* cols, const DevBlock* blocks, const uint32_t* items, const unsigned long long* codes,       \
                   uint32_t nitems, uint32_t ncolslots, void* stream);                                                  \
  /* distinct values of value-array int columns: keys[cap] (pre-filled with INT64_MIN = empty) receives every          \
   * distinct decoded value of the listed (block, column) items; counters[0] += new keys, counters[1] = 1 if          \
   * INT64_MIN itself occurred, counters[2] = 1 if the set filled up (more than cap/2 keys) */                          \
  int launch_distinct(const DevCol* cols, const DevBlock* blocks, const uint32_t* items, uint32_t nitems,               \
                      uint32_t ncolslots, long long* keys, uint32_t cap_mask, unsigned int* counters, void* stream);    \
  int scan_threads();                                                                                                   \
  /* shared memory the kernel needs besides slots and accumulators (stage_units: per-warp TMA staging, 2 KiB units) */ \
  uint32_t scan_fixed_smem(uint32_t stage_units);                                                                       \
  int scan_ctas_per_sm();   /* CTAs the kernel is built to co-reside per SM */                                          \
  uint32_t scan_max_smem(); /* dynamic shared memory one CTA may use then */                                            \
  }
SG_DECLARE_VARIANT(w16)
SG_DECLARE_VARIANT(w8)
constexpr uint32_t HROW_NONE = 0xffffffffu;
constexpr uint32_t SMEM_BINS = 1024;  // per-bin payload entries kept in shared memory (more: global scratch)
constexpr uint32_t TMA_TILE_BYTES = 4096;  // one warp tile: 32 rows of 128 bytes

}  // namespace sg
