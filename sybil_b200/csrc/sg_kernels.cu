// sg_kernels.cu — the fused decode + filter + group-by + aggregate scan kernel
// for sm_90a (H100).
//
// What it replaces in the reference, per 65,536-row block:
//   unpackIntCol / unpackStrCol     src/lib/column_store_io.go:690-780 / :493-609
//   IntFilter.Filter / StrFilter    src/lib/filter.go:171-250
//   FilterAndAggRecords             src/lib/aggregate.go:56-282
//   BasicHist/MultiHist.AddWeightedValue   src/lib/hist_basic.go:101-151, hist_multi.go:48-88
//
// Shape of the kernel (DESIGN.md §3):
//   * persistent grid, one CTA of 16 warps per SM; CTAs pull 65,536-row blocks from
//     an atomic work counter;
//   * per block the CTA keeps ONE word per row in shared memory ("slot": dense group
//     index in the low bits, number of filters passed above them) and walks the
//     referenced columns one after another.  The encoded arrays are streamed from
//     HBM exactly once with 32-byte-per-lane loads; nothing decoded is written back;
//   * a column is cut into warp tiles (1024 row ids / 512 int64 values).  A warp
//     loads its tile into registers, scans it (lane-serial + one warp scan), publishes
//     the tile total in shared memory and picks up the totals of the 15 tiles between
//     its previous tile and this one ("look-back"): there is no block-wide barrier in
//     the streaming loops and the 16 warps' loads overlap each other's arithmetic;
//   * bucket-encoded columns (value -> delta-encoded row-id list) use a segmented
//     prefix sum (segment heads = bin starts, a 65,536-bit mask in shared memory) and
//     scatter into the slot words with plain byte/halfword stores;
//   * count / sum accumulators live in shared memory, replicated per lane so the
//     32-bit shared atomics of a warp never collide (64-bit shared atomics are CAS
//     loops on this architecture); sums are exact in two 32-bit limbs with explicit
//     carry.  Histogram bucket counters go to L2/HBM with 64-bit reductions.
// No tensor cores: this is integer / indexing work bound by HBM bandwidth.
#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

#include "sg_internal.h"

#ifndef SG_THREADS
#define SG_THREADS 512
#endif
// the variant this compilation builds (see sg_internal.h): 16 warps x 1 CTA per SM, or 8 warps x 2
#if SG_THREADS == 256
#define SG_VNS w8
#else
#define SG_VNS w16
#endif

namespace sg {
namespace SG_VNS {

constexpr int THREADS = SG_THREADS;
constexpr int NWARPS = THREADS / 32;
constexpr uint32_t FLAG = 0x80000000u;
constexpr uint32_t HEAD_WORDS = SG_BLOCK_ROWS / 32;  // 2048
constexpr uint32_t FULL = 0xffffffffu;
constexpr int BE = 32;  // row ids per lane in a bucket tile  (tile = 1024 ids, 4 KB)
constexpr int VE = 16;  // int64 values per lane in a value tile (tile = 512 rows, 4 KB)
constexpr int SE = 8;   // int32 string ids per lane (tile = 256 rows)
constexpr uint32_t MAX_TILES = 128;
// the code pass (COL_CODES columns): how a column's payload joins the row's slot word, and its payload table (one
// entry per code; code 0xFF, an unlisted row, reads 0)
enum : uint32_t { CODE_ADD = 0, CODE_OR = 1, CODE_TIME = 2 };
constexpr uint32_t CODE_BINS = 256;
constexpr uint32_t CODE_BATCH = SMEM_BINS / CODE_BINS;  // code columns whose loads are issued together (4)

int scan_threads() { return THREADS; }

// shared-memory carve-out (bytes).  The dynamic window is declared 1 KiB aligned (so every address
// below is a link-time constant plus at most the staging depth); first come
// the per-warp TMA staging tiles (128B-swizzled, must sit on 1 KiB boundaries), then the fixed part
// below, then the slot words and the accumulators.
constexpr uint32_t OFF_HEADBITS = 0;                                   // u32[2048]
constexpr uint32_t OFF_HEADPREFIX = OFF_HEADBITS + HEAD_WORDS * 4;     // u16[2048]
constexpr uint32_t OFF_BINPAY = OFF_HEADPREFIX + HEAD_WORDS * 2;       // u32[SMEM_BINS]
constexpr uint32_t OFF_PUBA = OFF_BINPAY + SMEM_BINS * 4;              // u64[MAX_TILES]
constexpr uint32_t OFF_PUBB = OFF_PUBA + MAX_TILES * 8;                // u64[MAX_TILES]
constexpr uint32_t OFF_MBAR = OFF_PUBB + MAX_TILES * 8;                // u64[NWARPS][2] mbarriers
constexpr uint32_t OFF_MISC = OFF_MBAR + NWARPS * 2 * 8;               // u32[128]
constexpr uint32_t PL_MAX = 48;                                        // TMA-fed column passes of one block
constexpr uint32_t OFF_PLIST = OFF_MISC + 128 * 4;                     // u32[PL_MAX][4]
constexpr uint32_t OFF_PCAND = OFF_PLIST + PL_MAX * 16;                // u32[PL_MAX] candidate passes of the plan
constexpr uint32_t OFF_PTMP = OFF_PCAND + PL_MAX * 4;                  // u32[PL_MAX][4] per-block scratch
constexpr uint32_t OFF_COLCACHE = OFF_PTMP + PL_MAX * 16;               // DevCol[PL_MAX]: the block's candidate columns
constexpr uint32_t FIXED_SMEM = OFF_COLCACHE + PL_MAX * 80;
// stage_units: per-warp TMA staging in units of 2 KiB (0 none, 1, 2 = one 4 KiB tile, 4 = two)
uint32_t scan_fixed_smem(uint32_t stage_units) { return NWARPS * (TMA_TILE_BYTES / 2) * stage_units + FIXED_SMEM; }
// CTAs of THREADS threads the kernel is built to co-reside per SM (launch bounds), and the dynamic shared
// memory each may then ask for (228 KiB per SM, 1 KiB reserved per CTA)
#ifndef SG_CTAS_PER_SM
#define SG_CTAS_PER_SM (SG_THREADS <= 256 ? 2 : 1)
#endif
constexpr int CTAS_PER_SM = SG_CTAS_PER_SM;
int scan_ctas_per_sm() { return CTAS_PER_SM; }
uint32_t scan_max_smem() { return CTAS_PER_SM >= 2 ? (228u * 1024u / CTAS_PER_SM - 1024u) : 227u * 1024u; }

struct Ctx {
  uint32_t* headbits;
  uint16_t* headprefix;
  uint32_t* binpay_s;
  volatile unsigned long long* pubA;
  volatile unsigned long long* pubB;
  volatile uint32_t* misc;  // [0] next block, [1] broken flag, [16..16+NWARPS) warp totals, [64..95] per-lane sinks
  uint32_t* acc;
  int tid, lane, warp;
  uint32_t epoch;  // one per column pass; tags the published tile totals
  // TMA staging of this warp: stage_bytes (a multiple of 2 KiB) + two mbarriers (shared-window addresses)
  const unsigned char* tmaps;
  uint32_t stage_bytes;
  uint32_t buf0, buf1, mbar0, mbar1, par0, par1;
  // the TMA-fed column passes of the current block, in execution order: {chunk, row0, ntiles, -};
  // a pass requests the first tiles of the NEXT pass before its end-of-pass barrier, so the HBM
  // latency at the head of a pass overlaps the tail of the previous one
  const uint32_t* plist;
  uint32_t npass, pass_idx, pref_idx;
  uint32_t zero;  // 0 at run time, opaque to the compiler (see staged_reads_done)
#ifdef SG_FINE_TIMING
  volatile unsigned long long* tacc;  // thread 0 only: [9..15] fine-grained marks
  bool t0;
  __device__ __forceinline__ void tmark(int i) {
    if (t0) {
      const unsigned long long now = (unsigned long long)clock64();
      tacc[i] += now - tacc[8];
      tacc[8] = now;
    }
  }
#else
  __device__ __forceinline__ void tmark(int) {}
#endif
  // SG_PHASE_TIMING: cycles warp 0 spent waiting for TMA tiles / for look-back totals
  bool timing;
  unsigned long long t_tma, t_lb;
  __device__ __forceinline__ uint32_t buf(uint32_t st) const { return st ? buf1 : buf0; }
  // narrow arrays (col_shift > 0): a tile is 2 KiB or 1 KiB, so a 4 KiB buffer holds two of them
  // a tile of a column with col_shift s is 4 KiB >> s: as many stages (at most two) as the warp's buffer holds;
  // 0 = the column's tiles do not fit (plain loads)
  __device__ __forceinline__ uint32_t stages(uint32_t shift) const { return min(2u, stage_bytes / (TMA_TILE_BYTES >> shift)); }
  __device__ __forceinline__ uint32_t bufx(uint32_t st, uint32_t shift) const { return buf0 + st * (TMA_TILE_BYTES >> shift); }
  __device__ __forceinline__ uint32_t mbar(uint32_t st) const { return st ? mbar1 : mbar0; }
  __device__ __forceinline__ uint32_t take_parity(uint32_t st) {
    const uint32_t p = st ? par1 : par0;
    if (st)
      par1 ^= 1u;
    else
      par0 ^= 1u;
    return p;
  }
};

// ---- TMA / mbarrier primitives (sm_90+ PTX; SASS: UTMALDG, SYNCS) -----------------------------
__device__ __forceinline__ void mbar_init(uint32_t mbar_s, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar_s), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t mbar_s, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar_s), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar_s, uint32_t parity) {
  // try_wait suspends for a hardware-defined interval; a transfer that never completes (bad tensor
  // map) traps instead of hanging the GPU
  for (uint32_t spins = 0;; spins++) {
    uint32_t done;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(done)
        : "r"(mbar_s), "r"(parity)
        : "memory");
    if (done) return;
    if (spins > (1u << 24)) __trap();
  }
}
// one 4 KiB tile = 32 rows x 128 bytes at row `row` of the arena chunk's tensor map
__device__ __forceinline__ void tma_load_tile(uint32_t dst_s, const void* tmap, uint32_t row, uint32_t mbar_s) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          dst_s),
      "l"(tmap), "r"(0), "r"(row), "r"(mbar_s)
      : "memory");
}
// the same tile, only as far as L2 (no shared memory, no barrier): issued a few tiles ahead of the
// staged load so that the load finds its lines in L2 instead of waiting out the HBM latency — the
// bytes in flight per SM are no longer capped by the staging buffers
__device__ __forceinline__ void tma_prefetch_tile(const void* tmap, uint32_t row) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(0), "r"(row) : "memory");
}
// this lane's 128-byte row of a staged tile (32 words), undoing the 128B swizzle:
// 16-byte chunk j of row r sits at chunk position j ^ (r & 7)
__device__ __forceinline__ void read_staged_row(uint32_t buf_s, int lane, uint32_t (&w)[32]) {
  const uint32_t rowbase = buf_s + (uint32_t)lane * 128u;
  const uint32_t x = (uint32_t)(lane & 7);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint32_t addr = rowbase + ((((uint32_t)j) ^ x) << 4);
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(w[4 * j + 0]), "=r"(w[4 * j + 1]), "=r"(w[4 * j + 2]), "=r"(w[4 * j + 3])
                 : "r"(addr));
  }
}
// The low 32-bit limbs of this lane's 16 staged int64 values.  The loads stay 16 bytes wide on
// purpose: a lane-per-row 32-bit load of a swizzled tile is a 4-way bank conflict, and ptxas narrows
// a vector load whose high words are dead — so the high limbs are folded into `hix`, which the
// caller keeps alive.
__device__ __forceinline__ void read_staged_row_lo(uint32_t buf_s, int lane, uint32_t (&lo)[16], uint32_t& hix) {
  const uint32_t rowbase = buf_s + (uint32_t)lane * 128u;
  const uint32_t x = (uint32_t)(lane & 7);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint32_t addr = rowbase + ((((uint32_t)j) ^ x) << 4);
    asm volatile(
        "{\n"
        ".reg .b32 h0, h1;\n"
        "ld.shared.v4.u32 {%0,h0,%1,h1}, [%3];\n"
        "lop3.b32 %2, %2, h0, h1, 0x96;\n"
        "}\n"
        : "=r"(lo[2 * j + 0]), "=r"(lo[2 * j + 1]), "+r"(hix)
        : "r"(addr));
  }
}
// The same for the narrow views (64 / 32 byte rows, 64B / 32B swizzle): chunk j of row r sits at
// j ^ ((r >> 1) & 3) resp. j ^ ((r >> 2) & 1) — the address bits the hardware XORs are bits 7.. of the shared
// address, i.e. the 128-byte line the row lies in.  A quarter warp's 16-byte loads still cover all 32 banks.
__device__ __forceinline__ void read_staged_row64(uint32_t buf_s, int lane, uint32_t (&w)[16]) {
  const uint32_t rowbase = buf_s + (uint32_t)lane * 64u;
  const uint32_t x = (uint32_t)(lane >> 1) & 3u;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const uint32_t addr = rowbase + ((((uint32_t)j) ^ x) << 4);
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(w[4 * j + 0]), "=r"(w[4 * j + 1]), "=r"(w[4 * j + 2]), "=r"(w[4 * j + 3])
                 : "r"(addr));
  }
}
__device__ __forceinline__ void read_staged_row32(uint32_t buf_s, int lane, uint32_t (&w)[8]) {
  const uint32_t rowbase = buf_s + (uint32_t)lane * 32u;
  const uint32_t x = (uint32_t)(lane >> 2) & 1u;
#pragma unroll
  for (int j = 0; j < 2; j++) {
    const uint32_t addr = rowbase + ((((uint32_t)j) ^ x) << 4);
    asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(w[4 * j + 0]), "=r"(w[4 * j + 1]), "=r"(w[4 * j + 2]), "=r"(w[4 * j + 3])
                 : "r"(addr));
  }
}
// After a warp has read a staged tile with ordinary shared loads, the next TMA write into the same
// buffer must not overtake those loads (they can sit in the load/store queue behind reductions for
// microseconds).  A proxy fence would do, but it compiles to MEMBAR.ALL.CTA, which also waits for
// every reduction in flight.  Instead the re-issue is made DATA dependent on the loads: `dep` is
// computed from a word of every load of the lane, the ballot needs every lane's `dep`, and its
// result (always 0: cx.zero is a zero the compiler cannot see) is added to the TMA coordinate.  A
// load whose value has reached a register has been performed; the copy cannot start before that.
__device__ __forceinline__ uint32_t staged_reads_done(const Ctx& cx, uint32_t dep) {
  uint32_t b;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.u32 p, %1, 0;\n"
      "vote.sync.ballot.b32 %0, p, 0xffffffff;\n"
      "}\n"
      : "=r"(b)
      : "r"(dep & cx.zero)
      : "memory");
  return b;
}
__device__ __forceinline__ uint32_t dep_of(const uint32_t (&w)[32]) {
  return (w[0] ^ w[4] ^ w[8]) ^ (w[12] ^ w[16] ^ w[20]) ^ (w[24] ^ w[28]);
}
// the tile feed of one column pass: issue(tile) by lane 0, take(stage) by the whole warp
struct Feed {
  const void* tmap;
  uint32_t row0;   // first row of the column's data in the view `tmap` describes (rows of 128 >> shift bytes)
  uint32_t shift;  // col_shift of the column
  uint32_t ns;     // stages this pass runs with
  bool on;
  // L2 prefetch distance bookkeeping: this warp's tile count in this pass, and the next fed pass
  uint32_t mine;
  const void* ntmap;
  uint32_t nrow0, nnt;
};
#ifndef SG_PF_AHEAD
#define SG_PF_AHEAD 0  // measured on C2: 0 -> 0.677 ms, 2 -> 0.708 ms, 4 -> 0.731 ms (the scan is bandwidth-, not latency-bound)
#endif
constexpr uint32_t PF_AHEAD = SG_PF_AHEAD;  // L2 prefetch runs this many of the warp's tiles ahead of its staged loads (0: off)
__device__ __forceinline__ Feed make_feed(const Ctx& cx, const DevCol& c) {
  Feed f;
  f.shift = col_shift(c.flags);
  f.ns = cx.stages(f.shift);
  f.on = cx.tmaps != nullptr && (c.flags & COL_TMA) != 0 && f.ns != 0u;
  f.tmap = cx.tmaps + ((size_t)c.data_chunk * 3u + f.shift) * 128;
  f.row0 = c.data_row << f.shift;
  f.mine = 0;
  f.ntmap = nullptr;
  f.nrow0 = f.nnt = 0;
  return f;
}
__device__ __forceinline__ void feed_issue(const Ctx& cx, const Feed& f, uint32_t tile, uint32_t st, uint32_t after = 0u) {
  if (cx.lane == 0) {
    mbar_expect_tx(cx.mbar(st), TMA_TILE_BYTES >> f.shift);
    tma_load_tile(cx.bufx(st, f.shift), f.tmap, f.row0 + tile * 32u + after, cx.mbar(st));
  }
}
// L2 prefetch of this warp's v-th tile counted from the start of the pass; past the end of the pass
// it runs on into the warp's first tiles of the next fed pass of the block
__device__ __forceinline__ void feed_prefetch(const Ctx& cx, const Feed& f, uint32_t v) {
  if (PF_AHEAD == 0 || cx.lane != 0) return;
  if (v < f.mine) {
    tma_prefetch_tile(f.tmap, f.row0 + (cx.warp + v * NWARPS) * 32u);
  } else {
    const uint32_t t = cx.warp + (v - f.mine) * NWARPS;
    if (t < f.nnt) tma_prefetch_tile(f.ntmap, f.nrow0 + t * 32u);
  }
}
// start of a fed pass: request this warp's first tile(s) unless the previous pass already did
__device__ __forceinline__ void feed_prologue(Ctx& cx, Feed& f, uint32_t ntiles) {
  if (!f.on) return;
  const uint32_t* e = cx.plist + 4 * cx.pass_idx;
  if (cx.pass_idx >= cx.npass || e[1] != f.row0 || e[2] != ntiles) __trap();  // pass list out of step
  f.mine = (uint32_t)cx.warp < ntiles ? (ntiles - (uint32_t)cx.warp + NWARPS - 1u) / NWARPS : 0u;
  if (cx.pass_idx + 1 < cx.npass) {
    f.ntmap = cx.tmaps + (size_t)e[4] * 128;
    f.nrow0 = e[5];
    f.nnt = e[6];
  }
  if (cx.pref_idx != cx.pass_idx)
    for (uint32_t st = 0; st < f.ns; st++)
      if (cx.warp + st * NWARPS < ntiles) feed_issue(cx, f, cx.warp + st * NWARPS, st);
  // the first pass of a block has nobody before it to prefetch its head
  if (cx.pass_idx == 0)
    for (uint32_t v = f.ns; v < f.ns + PF_AHEAD; v++) feed_prefetch(cx, f, v);
}
// end of a fed pass (all of this warp's tiles consumed, both staging buffers free): request the
// first tile(s) of the next fed pass of the block
__device__ __forceinline__ void feed_epilogue(Ctx& cx, const Feed& f) {
  if (!f.on) return;
  cx.pass_idx++;
  if (cx.pass_idx < cx.npass) {
    const uint32_t* e = cx.plist + 4 * cx.pass_idx;
    Feed nf;
    nf.on = true;
    nf.tmap = cx.tmaps + (size_t)e[0] * 128;  // e[0] = chunk * 3 + shift: the view's index
    nf.row0 = e[1];
    nf.shift = e[0] % 3u;
    nf.ns = cx.stages(nf.shift);
    const uint32_t nt = e[2];
    for (uint32_t st = 0; st < nf.ns; st++)
      if (cx.warp + st * NWARPS < nt) feed_issue(cx, nf, cx.warp + st * NWARPS, st);
    cx.pref_idx = cx.pass_idx;
  }
}

// 32 contiguous bytes (32-byte aligned) per lane.  sm_90 has no 256-bit load, so this is two 128-bit loads
// back to back: a warp still covers whole 1 KiB spans, and both halves of a lane's sector pair are in flight together
__device__ __forceinline__ void ldg256(const void* p, uint32_t* r) {
  asm volatile(
      "ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%8];\n"
      "ld.global.nc.L1::no_allocate.v4.u32 {%4,%5,%6,%7}, [%8+16];"
      : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
      : "l"(p));
}
__device__ __forceinline__ void ldg256(const void* p, unsigned long long* r) {
  asm volatile(
      "ld.global.nc.L1::no_allocate.v2.u64 {%0,%1}, [%4];\n"
      "ld.global.nc.L1::no_allocate.v2.u64 {%2,%3}, [%4+16];"
      : "=l"(r[0]), "=l"(r[1]), "=l"(r[2]), "=l"(r[3])
      : "l"(p));
}

// shared-memory accumulators are addressed in the shared window (32-bit addresses): a generic
// pointer would cost a window conversion per atomic
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void sred_add(uint32_t addr, uint32_t v) {
  asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// global reductions spelled out in the global state space: a plain atomicAdd() on a pointer the
// compiler cannot prove global becomes a generic ATOM that returns a predicate (round trip to L2)
__device__ __forceinline__ void gred_add(unsigned long long* p, unsigned long long v) {
  asm volatile("red.global.add.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// predicated forms (one instruction each, no branch): the bucket step of the histogram hot path
__device__ __forceinline__ void sred_inc_if(uint32_t pred, uint32_t addr) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.u32 p, %0, 0;\n"
      "@p red.shared.add.u32 [%1], 1;\n"
      "}\n" ::"r"(pred),
      "r"(addr)
      : "memory");
}
__device__ __forceinline__ void gred_inc_if(uint32_t pred, unsigned long long* p) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.u32 p, %0, 0;\n"
      "@p red.global.add.u64 [%1], 1;\n"
      "}\n" ::"r"(pred),
      "l"(p)
      : "memory");
}
__device__ __forceinline__ void gred_max(long long* p, long long v) {
  asm volatile("red.global.max.s64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
// a 64-bit constant parked in shared memory, re-read once per tile: under register pressure the
// compiler otherwise keeps such a constant in local memory or re-reads it from the plan in global
// memory, a long-scoreboard wait per use (the multiply-high of the bucket division showed 10% of all
// stall samples of the C3 kernel waiting for its magic constant)
__device__ __forceinline__ unsigned long long lds_u64(uint32_t addr) {
  unsigned long long v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t satom_add(uint32_t addr, uint32_t v) {
  uint32_t o;
  asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(o) : "r"(addr), "r"(v) : "memory");
  return o;
}

// ---------------------------------------------------------------------------
// look-back over the tile totals other warps published for tiles t-15 .. t-1
// ---------------------------------------------------------------------------
// segmented u32 flavour: returns the running segment sum entering tile t
__device__ __forceinline__ uint32_t lookback_seg(const Ctx& cx, uint32_t t, uint32_t prev_incl) {
  const int tt = (int)t - (NWARPS - 1) + cx.lane;
  const bool valid = cx.lane < NWARPS - 1 && tt >= 0;
  uint32_t a = 0;
  if (valid) {
    unsigned long long w;
    do {
      w = cx.pubA[tt];
    } while ((uint32_t)(w >> 32) != cx.epoch);
    a = (uint32_t)w;
  }
  const uint32_t m = __ballot_sync(FULL, valid && (a & FLAG));
  uint32_t contrib = valid ? (a & ~FLAG) : 0u;
  uint32_t base = prev_incl;
  if (m) {
    const int js = 31 - __clz(m);
    if (cx.lane < js) contrib = 0u;
    base = 0u;
  }
  return base + __reduce_add_sync(FULL, contrib);
}
// plain u64 flavour: returns the sum of the totals of tiles t-15 .. t-1
__device__ __forceinline__ unsigned long long lookback_sum(const Ctx& cx, uint32_t t) {
  const int tt = (int)t - (NWARPS - 1) + cx.lane;
  unsigned long long v = 0;
  if (cx.lane < NWARPS - 1 && tt >= 0) {
    unsigned long long lo, hi;
    do {
      lo = cx.pubA[tt];
    } while ((uint32_t)(lo >> 32) != cx.epoch);
    do {
      hi = cx.pubB[tt];
    } while ((uint32_t)(hi >> 32) != cx.epoch);
    v = (lo & 0xffffffffull) | (hi << 32);
  }
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
  return v;
}

// ---------------------------------------------------------------------------
// bucket-encoded column: on_row(row, pay_of(bin)) for every (bin,row) pair; pay_of(bin) is
// evaluated once per run of entries of the same bin inside a lane
// `need`: bit t set = warp tile t (1024 flat entries) holds entries of a bin the caller cares about; the
// other tiles are not read at all (predicate push-down into the inverted index: a filter in fail mode
// only has to mark the rows of the FAILING bins).  A skipped tile publishes "segment restarts here": a
// needed tile that starts inside a bin has that bin's head in an earlier, therefore also needed, tile.
// Passes with skipped tiles use plain loads (`use_tma` false): their tiles are not in the block's pass list.
template <class PayT, class PayOf, class OnRow>
__device__ __forceinline__ void scan_bucket(Ctx& cx, const DevCol& c, const uint32_t nrec, PayOf pay_of, OnRow on_row,
                                            const unsigned long long need = ~0ull, const bool use_tma = true) {
  const uint32_t n = c.nitems;
  const uint32_t nbins = c.nbins;
  const uint32_t* __restrict__ ids = reinterpret_cast<const uint32_t*>(c.data);
  const bool delta = (c.flags & COL_DELTA_IDS) != 0;
  const bool ids16 = (c.flags & COL_ID16) != 0;  // narrow ids: 1024 of them are 2 KiB (64-byte rows)
  const int tid = cx.tid, lane = cx.lane, warp = cx.warp;
#ifndef SG_FINE_FLUSH
  cx.tmark(9);  // since the previous mark: the caller's per-bin payload build
#endif
  // request this warp's first tile(s) right away: the HBM latency overlaps the head-bit build
  const uint32_t ntiles = (n + (32 * BE - 1)) / (32 * BE);
  Feed feed = make_feed(cx, c);
  if (!use_tma) feed.on = false;
  feed_prologue(cx, feed, ntiles);

  // segment heads: one bit per flat entry that starts a (non-empty) bin
  for (uint32_t i = tid; i < HEAD_WORDS; i += THREADS) cx.headbits[i] = 0;
  __syncthreads();
  {
    const uint32_t* __restrict__ offs = c.bin_offsets;
    for (uint32_t b = tid; b < nbins; b += THREADS) {
      const uint32_t o = offs[b];
      if (o < n) atomicOr(&cx.headbits[o >> 5], 1u << (o & 31));
    }
  }
  __syncthreads();
  {  // exclusive prefix popcount per 32-entry word: THREADS x 4 words per step
    uint32_t running = 0;
    for (uint32_t i0 = 0; i0 < HEAD_WORDS / 4; i0 += THREADS) {
      const uint32_t i = i0 + (uint32_t)tid;
      const uint4 w = i < HEAD_WORDS / 4 ? reinterpret_cast<const uint4*>(cx.headbits)[i] : make_uint4(0, 0, 0, 0);
      const uint32_t p0 = __popc(w.x), p1 = __popc(w.y), p2 = __popc(w.z), p3 = __popc(w.w);
      const uint32_t tot = p0 + p1 + p2 + p3;
      uint32_t inc = tot;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(FULL, inc, d);
        if (lane >= d) inc += t;
      }
      if (i0) __syncthreads();  // the previous step's warp totals have been read
      if (lane == 31) cx.misc[16 + warp] = inc;
      __syncthreads();
      uint32_t base = running;
      for (int k = 0; k < NWARPS; k++) {
        const uint32_t wt = cx.misc[16 + k];
        if (k < warp) base += wt;
        running += wt;
      }
      const uint32_t ex = base + inc - tot;
      if (i < HEAD_WORDS / 4) {
        cx.headprefix[i * 4 + 0] = (uint16_t)ex;
        cx.headprefix[i * 4 + 1] = (uint16_t)(ex + p0);
        cx.headprefix[i * 4 + 2] = (uint16_t)(ex + p0 + p1);
        cx.headprefix[i * 4 + 3] = (uint16_t)(ex + p0 + p1 + p2);
      }
    }
  }
  cx.epoch++;
  if (need != ~0ull)
    for (uint32_t t = tid; t < ntiles; t += THREADS)
      if (!((need >> t) & 1ull)) cx.pubA[t] = (unsigned long long)FLAG | ((unsigned long long)cx.epoch << 32);
  __syncthreads();

#ifndef SG_FINE_FLUSH
  cx.tmark(10);  // head bits + prefix popcounts
#endif
  uint32_t prev_incl = 0;  // running segment sum through this warp's previous tile
  uint32_t it = 0;
  for (uint32_t t = warp; t < ntiles; t += NWARPS, it++) {
    if (!((need >> t) & 1ull)) continue;  // (65,536 ids = at most 64 tiles)
    const uint32_t idx0 = t * (32 * BE) + lane * BE;
    uint32_t a[BE];
    if (feed.on) {
      // the tile was requested one (or two) iterations ago: TMA wrote it into this warp's staging
      // buffer while the previous tile was being processed
      const uint32_t st = it & (feed.ns - 1u);
      mbar_wait(cx.mbar(st), cx.take_parity(st));
      uint32_t dep;
      if (ids16) {
        uint32_t h[BE / 2];
        read_staged_row64(cx.bufx(st, 1u), lane, h);
        dep = (h[0] ^ h[4]) ^ (h[8] ^ h[12]);
#pragma unroll
        for (int k = 0; k < BE / 2; k++) {
          a[2 * k] = h[k] & 0xffffu;
          a[2 * k + 1] = h[k] >> 16;
        }
      } else {
        read_staged_row(cx.bufx(st, 0u), lane, a);
        dep = dep_of(a);
      }
      const uint32_t after = staged_reads_done(cx, dep);
      if (t + feed.ns * NWARPS < ntiles) feed_issue(cx, feed, t + feed.ns * NWARPS, st, after);
      feed_prefetch(cx, feed, it + feed.ns + PF_AHEAD);
      if (idx0 + BE > n) {
#pragma unroll
        for (int k = 0; k < BE; k++)
          if (idx0 + k >= n) a[k] = 0u;
      }
    } else if (ids16) {
      const uint16_t* __restrict__ ids_h = reinterpret_cast<const uint16_t*>(c.data);
      if (idx0 + BE <= n) {
        uint32_t h[BE / 2];
#pragma unroll
        for (int j = 0; j < BE / 16; j++) ldg256(ids_h + idx0 + 16 * j, h + 8 * j);
#pragma unroll
        for (int k = 0; k < BE / 2; k++) {
          a[2 * k] = h[k] & 0xffffu;
          a[2 * k + 1] = h[k] >> 16;
        }
      } else {
#pragma unroll
        for (int k = 0; k < BE; k++) a[k] = (idx0 + k < n) ? (uint32_t)ids_h[idx0 + k] : 0u;
      }
    } else if (idx0 + BE <= n) {
#pragma unroll
      for (int j = 0; j < BE / 8; j++) ldg256(ids + idx0 + 8 * j, a + 8 * j);
    } else {
#pragma unroll
      for (int k = 0; k < BE; k++) a[k] = (idx0 + k < n) ? ids[idx0 + k] : 0u;
    }
    const uint32_t word = (idx0 < n) ? cx.headbits[idx0 >> 5] : 0u;
    const uint32_t segw = delta ? word : FULL;  // absolute ids: every entry is its own segment
    {
      // a valid gap is < 65,536; anything larger marks the block broken and is masked so
      // the packed (sum | flag) scan word cannot overflow into the flag bit
      uint32_t orv = 0;
#pragma unroll
      for (int k = 0; k < BE; k++) orv |= a[k];
      if (orv >= 0x10000u) {
        cx.misc[1] = 1;
#pragma unroll
        for (int k = 0; k < BE; k++) a[k] &= 0xFFFFu;
      }
    }
    const uint32_t lastrow = nrec - 1u;
    // Fast path (warp-uniform): a full tile of delta-encoded ids in which no lane sees more than one
    // bin head.  The lane's 32 gaps become in-place prefix sums P_k; with the head at entry h the
    // row of entry k is P_k + carry for k < h and P_k - P_{h-1} for k >= h, the payload likewise one
    // of two values: no per-entry head test, bin step or payload lookup.
    if (delta && idx0 - lane * BE + 32 * BE <= n && !__any_sync(FULL, (word & (word - 1u)) != 0u)) {
      const uint32_t below = word ? ((word & (0u - word)) - 1u) : FULL;  // entries before the head (all if none)
#pragma unroll
      for (int k = 1; k < BE; k++) a[k] += a[k - 1];
      const uint32_t tot_all = a[BE - 1];
      // pre = P_{h-1}: a 5-level select over the register array (h = 0 or no head: unused / tot_all)
      uint32_t pre = 0;
      {
        const uint32_t hm1 = (uint32_t)__popc(below) - 1u;  // h - 1 (31 when there is no head)
        uint32_t l1[16], l2[8], l3[4], l4[2];
#pragma unroll
        for (int j = 0; j < 16; j++) l1[j] = (hm1 & 1u) ? a[2 * j + 1] : a[2 * j];
#pragma unroll
        for (int j = 0; j < 8; j++) l2[j] = (hm1 & 2u) ? l1[2 * j + 1] : l1[2 * j];
#pragma unroll
        for (int j = 0; j < 4; j++) l3[j] = (hm1 & 4u) ? l2[2 * j + 1] : l2[2 * j];
#pragma unroll
        for (int j = 0; j < 2; j++) l4[j] = (hm1 & 8u) ? l3[2 * j + 1] : l3[2 * j];
        pre = (hm1 & 16u) ? l4[1] : l4[0];
        if (below == 0u) pre = 0u;  // head at entry 0
      }
      const uint32_t tot = word ? tot_all - pre : tot_all;
      uint32_t incl = tot | (word ? FLAG : 0u);
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(FULL, incl, d);
        if (lane >= d && !(incl & FLAG)) incl += v;
      }
      uint32_t excl = __shfl_up_sync(FULL, incl, 1);
      if (lane == 0) excl = 0;
      const uint32_t tile_tot = __shfl_sync(FULL, incl, 31);
      if (lane == 0) cx.pubA[t] = (unsigned long long)tile_tot | ((unsigned long long)cx.epoch << 32);
      const uint32_t carry = lookback_seg(cx, t, prev_incl);
      prev_incl = (tile_tot & FLAG) ? (tile_tot & ~FLAG) : ((carry + tile_tot) & ~FLAG);
      const uint32_t offA = (excl & FLAG) ? (excl & ~FLAG) : ((excl + carry) & ~FLAG);
      const uint32_t offB = 0u - pre;
      int binA = (int)cx.headprefix[idx0 >> 5] - 1, binB = binA + 1;
      if ((binA < 0 && below != 0u) || (word && (uint32_t)binB >= nbins)) cx.misc[1] = 1;
      if (binA < 0) binA = 0;
      if ((uint32_t)binB >= nbins) binB = 0;
      const PayT payA = pay_of((uint32_t)binA);
      const PayT payB = word ? pay_of((uint32_t)binB) : payA;
      // rows grow inside a segment: the lane's largest is the last one of either segment
      const uint32_t lastA = (below ? pre : 0u) + offA, lastB = tot_all + (word ? offB : offA);
      if (max(below ? lastA : 0u, lastB) > lastrow) cx.misc[1] = 1;
#pragma unroll
      for (int k = 0; k < BE; k++) {
        const bool lo = (below >> k) & 1u;
        on_row(min(a[k] + (lo ? offA : offB), lastrow), lo ? payA : payB);
      }
      continue;
    }
    // pass 1: lane total since the last head in the lane
    uint32_t tot = 0;
#pragma unroll
    for (int k = 0; k < BE; k++) tot = ((segw >> k) & 1u) ? a[k] : tot + a[k];
    uint32_t incl = tot | (segw ? FLAG : 0u);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t v = __shfl_up_sync(FULL, incl, d);
      if (lane >= d && !(incl & FLAG)) incl += v;
    }
    uint32_t excl = __shfl_up_sync(FULL, incl, 1);
    if (lane == 0) excl = 0;
    const uint32_t tile_tot = __shfl_sync(FULL, incl, 31);
    if (lane == 0) cx.pubA[t] = (unsigned long long)tile_tot | ((unsigned long long)cx.epoch << 32);
    const uint32_t carry = lookback_seg(cx, t, prev_incl);
    prev_incl = (tile_tot & FLAG) ? (tile_tot & ~FLAG) : ((carry + tile_tot) & ~FLAG);
    uint32_t run = (excl & FLAG) ? (excl & ~FLAG) : ((excl + carry) & ~FLAG);
    // pass 2: rows and bins.  A row id >= NumRecords marks the block broken
    // ("BLOCK SIZE CHANGED DURING QUERY", column_store_io.go:733); ids are clamped so the
    // scatter stays in range and the whole block is dropped at the end.
    int bin = (int)((idx0 < n) ? cx.headprefix[idx0 >> 5] : 0) - 1;
    const uint32_t cnt = (idx0 >= n) ? 0u : ((n - idx0 < BE) ? n - idx0 : BE);
    uint32_t maxrow = 0;
    PayT cur = PayT();
    auto step = [&](int k) {
      const bool head = (word >> k) & 1u;
      if (head) bin++;
      run = ((segw >> k) & 1u) ? a[k] : run + a[k];
      if (head || k == 0) {
        if ((uint32_t)bin >= nbins) {
          cx.misc[1] = 1;
          bin = 0;
        }
        cur = pay_of((uint32_t)bin);
      }
      maxrow = max(maxrow, run);
      on_row(min(run, lastrow), cur);
    };
    if (cnt == BE) {
#pragma unroll
      for (int k = 0; k < BE; k++) step(k);
    } else {
#pragma unroll
      for (int k = 0; k < BE; k++)
        if (k < cnt) step(k);
    }
    if (maxrow > lastrow) cx.misc[1] = 1;
  }
#ifndef SG_FINE_FLUSH
  cx.tmark(11);  // this thread's tiles
#endif
  feed_epilogue(cx, feed);
  __syncthreads();
#ifndef SG_FINE_FLUSH
  cx.tmark(12);  // waiting for the slowest warp
#endif
}

// ---------------------------------------------------------------------------
// value-array int column (delta-encoded int64): visit(row, value) in row order
// ---------------------------------------------------------------------------
template <class TileVisit>
__device__ __forceinline__ void scan_values_i64(Ctx& cx, const DevCol& c, const uint32_t nrec, TileVisit tile_visit) {
  uint32_t n = c.nitems;
  if (n > nrec) n = nrec;  // staging already flags len(Values) > NumRecords as broken
  const unsigned long long* __restrict__ vals = reinterpret_cast<const unsigned long long*>(c.data);
  const bool delta = (c.flags & COL_DELTA_VALUES) != 0;
  const uint32_t vw = col_shift(c.flags);  // 0: int64 values; 1 / 2: int32 / int16 deltas on top of c.vbase
  const int lane = cx.lane, warp = cx.warp;
  cx.epoch++;
  const uint32_t ntiles = (n + (32 * VE - 1)) / (32 * VE);
  unsigned long long prev_incl = vw ? (unsigned long long)c.vbase : 0ull;
  Feed feed = make_feed(cx, c);
  feed_prologue(cx, feed, ntiles);
  uint32_t it = 0;
  for (uint32_t t = warp; t < ntiles; t += NWARPS, it++) {
    const uint32_t idx0 = t * (32 * VE) + lane * VE;
    unsigned long long a[VE];
    if (feed.on) {
      const uint32_t st = it & (feed.ns - 1u);
      mbar_wait(cx.mbar(st), cx.take_parity(st));
      uint32_t dep;
      if (vw == 0u) {
        uint32_t raw[32];
        read_staged_row(cx.bufx(st, 0u), lane, raw);
        dep = dep_of(raw);
#pragma unroll
        for (int k = 0; k < VE; k++) a[k] = (unsigned long long)raw[2 * k] | ((unsigned long long)raw[2 * k + 1] << 32);
      } else if (vw == 1u) {
        uint32_t raw[16];
        read_staged_row64(cx.bufx(st, 1u), lane, raw);
        dep = (raw[0] ^ raw[4]) ^ (raw[8] ^ raw[12]);
#pragma unroll
        for (int k = 0; k < VE; k++) a[k] = (unsigned long long)(long long)(int32_t)raw[k];
      } else {
        uint32_t raw[8];
        read_staged_row32(cx.bufx(st, 2u), lane, raw);
        dep = raw[0] ^ raw[4];
#pragma unroll
        for (int k = 0; k < VE / 2; k++) {
          a[2 * k] = (unsigned long long)(long long)(int16_t)(raw[k] & 0xffffu);
          a[2 * k + 1] = (unsigned long long)(long long)((int32_t)raw[k] >> 16);
        }
      }
      const uint32_t after = staged_reads_done(cx, dep);
      if (t + feed.ns * NWARPS < ntiles) feed_issue(cx, feed, t + feed.ns * NWARPS, st, after);
      feed_prefetch(cx, feed, it + feed.ns + PF_AHEAD);
      if (idx0 + VE > n) {
#pragma unroll
        for (int k = 0; k < VE; k++)
          if (idx0 + k >= n) a[k] = 0ull;
      }
    } else if (vw == 1u) {
      const int32_t* __restrict__ v32 = reinterpret_cast<const int32_t*>(c.data);
      if (idx0 + VE <= n) {
        uint32_t raw[16];
        ldg256(v32 + idx0, raw);
        ldg256(v32 + idx0 + 8, raw + 8);
#pragma unroll
        for (int k = 0; k < VE; k++) a[k] = (unsigned long long)(long long)(int32_t)raw[k];
      } else {
#pragma unroll
        for (int k = 0; k < VE; k++) a[k] = (idx0 + k < n) ? (unsigned long long)(long long)v32[idx0 + k] : 0ull;
      }
    } else if (vw == 2u) {
      const int16_t* __restrict__ v16 = reinterpret_cast<const int16_t*>(c.data);
      if (idx0 + VE <= n) {
        uint32_t raw[8];
        ldg256(v16 + idx0, raw);
#pragma unroll
        for (int k = 0; k < VE / 2; k++) {
          a[2 * k] = (unsigned long long)(long long)(int16_t)(raw[k] & 0xffffu);
          a[2 * k + 1] = (unsigned long long)(long long)((int32_t)raw[k] >> 16);
        }
      } else {
#pragma unroll
        for (int k = 0; k < VE; k++) a[k] = (idx0 + k < n) ? (unsigned long long)(long long)v16[idx0 + k] : 0ull;
      }
    } else if (idx0 + VE <= n) {
#pragma unroll
      for (int j = 0; j < VE / 4; j++) ldg256(vals + idx0 + 4 * j, a + 4 * j);
    } else {
#pragma unroll
      for (int k = 0; k < VE; k++) a[k] = (idx0 + k < n) ? vals[idx0 + k] : 0ull;
    }
    if (delta) {
#pragma unroll
      for (int k = 1; k < VE; k++) a[k] += a[k - 1];
      const unsigned long long tot = a[VE - 1];
      unsigned long long incl = tot;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long v = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += v;
      }
      const unsigned long long tile_tot = __shfl_sync(FULL, incl, 31);
      if (lane == 0) {
        cx.pubA[t] = (tile_tot & 0xffffffffull) | ((unsigned long long)cx.epoch << 32);
        cx.pubB[t] = (tile_tot >> 32) | ((unsigned long long)cx.epoch << 32);
      }
      const unsigned long long carry = prev_incl + lookback_sum(cx, t);
      prev_incl = carry + tile_tot;
      const unsigned long long base = incl - tot + carry;
#pragma unroll
      for (int k = 0; k < VE; k++) a[k] += base;
    }
    const uint32_t nvalid = (idx0 >= n) ? 0u : ((n - idx0 < VE) ? n - idx0 : (uint32_t)VE);
    tile_visit(idx0, a, nvalid);
  }
  feed_epilogue(cx, feed);
  __syncthreads();
}

// exact x / d for x < 2^32 with the host-computed magic M = floor(2^64 / d) + 1 (d < 2^32):
// x*M/2^64 = x/d + x*e/(d*2^64) with 0 < e <= d, and x*e < 2^64, so the floor is unchanged
__device__ __forceinline__ uint32_t div_magic(uint32_t x, unsigned long long M) {
  return (uint32_t)__umul64hi((unsigned long long)x, M);
}

// value-array int column whose decoded values are known (COL_STATS) to lie in [0, 2^32): the same
// tiles and look-back, in 32-bit arithmetic.  tile_visit(idx0, a[VE] (uint32), nvalid)
// `pf`: when not null, the tile's 32-bit slot words (global scratch, one per row) are prefetched into L1 before
// the tile is waited for, so that the loads behind the scan find them there (high-cardinality plans)
template <class TileVisit>
__device__ __forceinline__ void scan_values_u32(Ctx& cx, const DevCol& c, const uint32_t nrec, TileVisit tile_visit,
                                                const uint32_t* pf = nullptr) {
  uint32_t n = c.nitems;
  if (n > nrec) n = nrec;
  const unsigned long long* __restrict__ vals = reinterpret_cast<const unsigned long long*>(c.data);
  const bool delta = (c.flags & COL_DELTA_VALUES) != 0;
  const uint32_t vw = col_shift(c.flags);  // 0: int64 values; 1 / 2: int32 / int16 deltas on top of c.vbase
  const int lane = cx.lane, warp = cx.warp;
  cx.epoch++;
  const uint32_t ntiles = (n + (32 * VE - 1)) / (32 * VE);
  uint32_t prev_incl = vw ? (uint32_t)(unsigned long long)c.vbase : 0u;  // decoded values are exact mod 2^32
  uint32_t hix = 0;  // xor of the high limbs read (keeps the staged loads 16 bytes wide)
  Feed feed = make_feed(cx, c);
  feed_prologue(cx, feed, ntiles);
  uint32_t it = 0;
  for (uint32_t t = warp; t < ntiles; t += NWARPS, it++) {
    const uint32_t idx0 = t * (32 * VE) + lane * VE;
    uint32_t a[VE];
    if (pf != nullptr && idx0 < n) asm volatile("prefetch.global.L1 [%0];" ::"l"(pf + idx0));  // 16 words = 64 bytes
    if (feed.on) {
      const uint32_t st = it & (feed.ns - 1u);
#ifdef SG_WAIT_TIMING
      const long long tw0 = cx.timing ? clock64() : 0;
#endif
      mbar_wait(cx.mbar(st), cx.take_parity(st));
#ifdef SG_WAIT_TIMING
      if (cx.timing) cx.t_tma += (unsigned long long)(clock64() - tw0);
#endif
      uint32_t dep;
      if (vw == 0u) {
        read_staged_row_lo(cx.bufx(st, 0u), lane, a, hix);  // low limbs: exact mod 2^32
        dep = hix;
      } else if (vw == 1u) {
        read_staged_row64(cx.bufx(st, 1u), lane, a);  // int32 deltas: as they are (mod 2^32)
        dep = (a[0] ^ a[4]) ^ (a[8] ^ a[12]);
      } else {
        uint32_t raw[8];
        read_staged_row32(cx.bufx(st, 2u), lane, raw);
        dep = raw[0] ^ raw[4];
#pragma unroll
        for (int k = 0; k < VE / 2; k++) {
          a[2 * k] = (uint32_t)(int32_t)(int16_t)(raw[k] & 0xffffu);
          a[2 * k + 1] = (uint32_t)((int32_t)raw[k] >> 16);
        }
      }
      const uint32_t after = staged_reads_done(cx, dep);
      if (t + feed.ns * NWARPS < ntiles) feed_issue(cx, feed, t + feed.ns * NWARPS, st, after);
      feed_prefetch(cx, feed, it + feed.ns + PF_AHEAD);
      if (idx0 + VE > n) {
#pragma unroll
        for (int k = 0; k < VE; k++)
          if (idx0 + k >= n) a[k] = 0u;
      }
    } else if (vw == 1u) {
      const uint32_t* __restrict__ v32 = reinterpret_cast<const uint32_t*>(c.data);
      if (idx0 + VE <= n) {
        ldg256(v32 + idx0, a);
        ldg256(v32 + idx0 + 8, a + 8);
      } else {
#pragma unroll
        for (int k = 0; k < VE; k++) a[k] = (idx0 + k < n) ? v32[idx0 + k] : 0u;
      }
    } else if (vw == 2u) {
      const int16_t* __restrict__ v16 = reinterpret_cast<const int16_t*>(c.data);
      if (idx0 + VE <= n) {
        uint32_t raw[8];
        ldg256(v16 + idx0, raw);
#pragma unroll
        for (int k = 0; k < VE / 2; k++) {
          a[2 * k] = (uint32_t)(int32_t)(int16_t)(raw[k] & 0xffffu);
          a[2 * k + 1] = (uint32_t)((int32_t)raw[k] >> 16);
        }
      } else {
#pragma unroll
        for (int k = 0; k < VE; k++) a[k] = (idx0 + k < n) ? (uint32_t)(int32_t)v16[idx0 + k] : 0u;
      }
    } else if (idx0 + VE <= n) {
#pragma unroll
      for (int j = 0; j < VE / 4; j++) {
        unsigned long long q[4];
        ldg256(vals + idx0 + 4 * j, q);
#pragma unroll
        for (int i = 0; i < 4; i++) a[4 * j + i] = (uint32_t)q[i];  // values < 2^32: the low limb is exact mod 2^32
      }
    } else {
#pragma unroll
      for (int k = 0; k < VE; k++) a[k] = (idx0 + k < n) ? (uint32_t)vals[idx0 + k] : 0u;
    }
    if (delta) {
#pragma unroll
      for (int k = 1; k < VE; k++) a[k] += a[k - 1];
      const uint32_t tot = a[VE - 1];
      uint32_t incl = tot;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const uint32_t v = __shfl_up_sync(FULL, incl, d);
        if (lane >= d) incl += v;
      }
      const uint32_t tile_tot = __shfl_sync(FULL, incl, 31);
      if (lane == 0) cx.pubA[t] = (unsigned long long)tile_tot | ((unsigned long long)cx.epoch << 32);
      // totals of tiles t-15 .. t-1 (other warps) on top of this warp's previous inclusive prefix
      const int tt = (int)t - (NWARPS - 1) + lane;
      uint32_t contrib = 0;
#ifdef SG_WAIT_TIMING
      const long long tl0 = cx.timing ? clock64() : 0;
#endif
      if (lane < NWARPS - 1 && tt >= 0) {
        unsigned long long w;
        do {
          w = cx.pubA[tt];
        } while ((uint32_t)(w >> 32) != cx.epoch);
        contrib = (uint32_t)w;
      }
      const uint32_t carry = prev_incl + __reduce_add_sync(FULL, contrib);
#ifdef SG_WAIT_TIMING
      if (cx.timing) cx.t_lb += (unsigned long long)(clock64() - tl0);
#endif
      prev_incl = carry + tile_tot;
      const uint32_t base = incl - tot + carry;
#pragma unroll
      for (int k = 0; k < VE; k++) a[k] += base;
    }
    const uint32_t nvalid = (idx0 >= n) ? 0u : ((n - idx0 < VE) ? n - idx0 : (uint32_t)VE);
    tile_visit(idx0, a, nvalid);
  }
  if (hix == 0x5bd1e995u) cx.misc[4] = hix;  // never read: the use that keeps hix (and the wide loads) alive
  feed_epilogue(cx, feed);
  __syncthreads();
}

// the slot words of VE consecutive rows starting at idx0 (idx0 % VE == 0), as 32-bit values
template <typename SlotT>
__device__ __forceinline__ void load_slots(const SlotT* slot, uint32_t idx0, uint32_t (&sw)[VE]) {
  if (sizeof(SlotT) == 1) {
    const uint4 q = *reinterpret_cast<const uint4*>(slot + idx0);
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < VE; k++) sw[k] = __byte_perm(w[k >> 2], 0u, 0x4440u | (uint32_t)(k & 3));
  } else if (sizeof(SlotT) == 2) {
    const uint4 q0 = *reinterpret_cast<const uint4*>(slot + idx0);
    const uint4 q1 = *reinterpret_cast<const uint4*>(slot + idx0 + 8);
    const uint32_t w[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
    for (int k = 0; k < VE; k++) sw[k] = __byte_perm(w[k >> 1], 0u, (k & 1) ? 0x4432u : 0x4410u);
  } else {
#pragma unroll
    for (int j = 0; j < VE / 4; j++) {
      const uint4 q = *reinterpret_cast<const uint4*>(slot + idx0 + 4 * j);
      sw[4 * j + 0] = q.x;
      sw[4 * j + 1] = q.y;
      sw[4 * j + 2] = q.z;
      sw[4 * j + 3] = q.w;
    }
  }
}
// add inc[k] (already positioned in the slot word's field) to the slot words of VE consecutive rows
template <typename SlotT>
__device__ __forceinline__ void add_slots(SlotT* slot, uint32_t idx0, const uint32_t (&inc)[VE]) {
  if (sizeof(SlotT) == 1) {
    uint4* p = reinterpret_cast<uint4*>(slot + idx0);
    uint4 q = *p;
    uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < VE; k++) w[k >> 2] += inc[k] << (8 * (k & 3));
    *p = make_uint4(w[0], w[1], w[2], w[3]);
  } else if (sizeof(SlotT) == 2) {
    uint4* p = reinterpret_cast<uint4*>(slot + idx0);
    uint4 q0 = p[0], q1 = p[1];
    uint32_t w[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
    for (int k = 0; k < VE; k++) w[k >> 1] += inc[k] << (16 * (k & 1));
    p[0] = make_uint4(w[0], w[1], w[2], w[3]);
    p[1] = make_uint4(w[4], w[5], w[6], w[7]);
  } else {
#pragma unroll
    for (int k = 0; k < VE; k++) slot[idx0 + k] = (SlotT)(slot[idx0 + k] + inc[k]);
  }
}

// OR inc[k] (already positioned in the slot word's field) into the slot words of VE consecutive rows
template <typename SlotT>
__device__ __forceinline__ void or_slots(SlotT* slot, uint32_t idx0, const uint32_t (&inc)[VE]) {
  if (sizeof(SlotT) == 1) {
    uint4* p = reinterpret_cast<uint4*>(slot + idx0);
    uint4 q = *p;
    uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int k = 0; k < VE; k++) w[k >> 2] |= inc[k] << (8 * (k & 3));
    *p = make_uint4(w[0], w[1], w[2], w[3]);
  } else if (sizeof(SlotT) == 2) {
    uint4* p = reinterpret_cast<uint4*>(slot + idx0);
    uint4 q0 = p[0], q1 = p[1];
    uint32_t w[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
#pragma unroll
    for (int k = 0; k < VE; k++) w[k >> 1] |= inc[k] << (16 * (k & 1));
    p[0] = make_uint4(w[0], w[1], w[2], w[3]);
    p[1] = make_uint4(w[4], w[5], w[6], w[7]);
  } else {
#pragma unroll
    for (int k = 0; k < VE; k++) slot[idx0 + k] = (SlotT)(slot[idx0 + k] | inc[k]);
  }
}

// One row's slot word += v / |= v from the scattered (bucket) passes.  In shared memory the update is a
// 32-bit reduction on the word that holds the row's byte / halfword (v shifted into its lane; a slot word
// never overflows its field, so nothing carries into the neighbour): no load, hence no dependent
// shared-memory round trip per row (the read-modify-write version spent its time in short-scoreboard
// stalls).  32-bit slot words live in L2: plain read-modify-write there.
template <typename SlotT>
__device__ __forceinline__ void slot_add(SlotT* slot, uint32_t slot_s, uint32_t row, uint32_t v) {
  if (sizeof(SlotT) == 1)
    sred_add(slot_s + (row & ~3u), v << ((row & 3u) << 3));
  else if (sizeof(SlotT) == 2)
    sred_add(slot_s + ((row & ~1u) << 1), v << ((row & 1u) << 4));
  else
    slot[row] = (SlotT)(slot[row] + v);
}
template <typename SlotT>
__device__ __forceinline__ void slot_or(SlotT* slot, uint32_t slot_s, uint32_t row, uint32_t v) {
  if (sizeof(SlotT) == 1)
    asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(slot_s + (row & ~3u)), "r"(v << ((row & 3u) << 3)) : "memory");
  else if (sizeof(SlotT) == 2)
    asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(slot_s + ((row & ~1u) << 1)), "r"(v << ((row & 1u) << 4)) : "memory");
  else  // atomic too: a set column lists a row in as many bins as its set has tags, walked by different threads
    atomicOr(reinterpret_cast<unsigned int*>(slot) + row, v);
}

// value-array str column (raw int32 local ids): visit(row, local_id)
template <class Visit>
__device__ __forceinline__ void scan_values_i32(Ctx& cx, const DevCol& c, const uint32_t nrec, Visit visit) {
  uint32_t n = c.nitems;
  if (n > nrec) n = nrec;
  const uint32_t* __restrict__ vals = reinterpret_cast<const uint32_t*>(c.data);
  if (c.flags & COL_VAL16) {  // narrow form: uint16 local ids, 16 per lane and step
    const uint16_t* __restrict__ v16 = reinterpret_cast<const uint16_t*>(c.data);
    for (uint32_t idx0 = cx.tid * 2 * SE; idx0 < n; idx0 += THREADS * 2 * SE) {
      if (idx0 + 2 * SE <= n) {
        uint32_t a[SE];
        ldg256(v16 + idx0, a);
#pragma unroll
        for (int k = 0; k < SE; k++) {
          visit(idx0 + 2 * k, (int32_t)(a[k] & 0xffffu));
          visit(idx0 + 2 * k + 1, (int32_t)(a[k] >> 16));
        }
      } else {
#pragma unroll
        for (int k = 0; k < 2 * SE; k++)
          if (idx0 + k < n) visit(idx0 + k, (int32_t)v16[idx0 + k]);
      }
    }
    __syncthreads();
    return;
  }
  for (uint32_t idx0 = cx.tid * SE; idx0 < n; idx0 += THREADS * SE) {
    uint32_t a[SE];
    if (idx0 + SE <= n) {
      ldg256(vals + idx0, a);
#pragma unroll
      for (int k = 0; k < SE; k++) visit(idx0 + k, (int32_t)a[k]);
    } else {
#pragma unroll
      for (int k = 0; k < SE; k++)
        if (idx0 + k < n) visit(idx0 + k, (int32_t)vals[idx0 + k]);
    }
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// predicates
// ---------------------------------------------------------------------------
// IntFilter (filter.go:177-189) as one unsigned range test: pass <=> ((v - lo) <=u span) != inv
struct IntRange {
  unsigned long long lo, span;
  bool inv;   // NEQ: complement of the EQ range
  bool none;  // empty range (e.g. "gt INT64_MAX")
  __device__ __forceinline__ bool operator()(long long v) const {
    return !none && ((((unsigned long long)v - lo) <= span) != inv);
  }
};
__device__ __forceinline__ IntRange int_range(int op, long long lit) {
  IntRange r;
  r.lo = 0;
  r.span = 0;
  r.inv = false;
  r.none = false;
  const long long mn = -0x7fffffffffffffffll - 1, mx = 0x7fffffffffffffffll;
  switch (op) {
    case SG_OP_GT:
      if (lit == mx) r.none = true;
      r.lo = (unsigned long long)(lit + (lit == mx ? 0 : 1));
      r.span = (unsigned long long)mx - r.lo;
      break;
    case SG_OP_LT:
      if (lit == mn) r.none = true;
      r.lo = (unsigned long long)mn;
      r.span = (unsigned long long)(lit - (lit == mn ? 0 : 1)) - r.lo;
      break;
    case SG_OP_EQ:
      r.lo = (unsigned long long)lit;
      break;
    case SG_OP_NEQ:
      r.lo = (unsigned long long)lit;
      r.inv = true;
      break;
    default: r.none = true; break;
  }
  return r;
}
__device__ __forceinline__ bool int_pred(int op, long long v, long long lit) {
  // filter.go:177-189
  switch (op) {
    case SG_OP_GT: return v > lit;
    case SG_OP_LT: return v < lit;
    case SG_OP_EQ: return v == lit;
    case SG_OP_NEQ: return v != lit;
    default: return false;
  }
}
struct StrPred {  // filter.go:199-250 on global ids (registers, not plan memory)
  int op;
  int32_t gid;
  const uint32_t* lut;
  long long lut_bits;
  __device__ __forceinline__ bool operator()(int32_t g) const {
    switch (op) {
      case SG_OP_EQ: return g == gid;  // a literal absent from the dictionary matches nothing (Q3)
      case SG_OP_NEQ: return g != gid;
      case SG_OP_RE:
      case SG_OP_NRE: {
        bool m = false;
        if (g >= 0 && (long long)g < lut_bits) m = (lut[g >> 5] >> (g & 31)) & 1u;
        return op == SG_OP_RE ? m : !m;
      }
      default: return false;
    }
  }
};
__device__ __forceinline__ int32_t str_gid(const DevCol& c, long long local) {
  if (local < 0 || local >= (long long)c.nremap) return c.oob_gid;
  return c.remap[local];
}

// time bucket code (aggregate.go:177: int(val)/TimeBucket*TimeBucket, truncating):
// dense index 1.. of trunc(val/bucket) - first; 0 = outside the planned range
__device__ __forceinline__ uint32_t time_code(long long v, long long bucket, long long first, uint32_t radix) {
  const long long q = v / bucket - first;
  if (q < 0 || q >= (long long)(radix - 1)) return 0u;
  return (uint32_t)q + 1u;
}

// ---------------------------------------------------------------------------
// aggregation of one value: hot path inline in the kernel, everything rare out of line
// ---------------------------------------------------------------------------
struct AggSlow {  // what the out-of-line paths need (lives in local memory)
  long long info_min, info_max, reject_hi;
  int nsub, multi;
  uint32_t nvals_total;
  unsigned long long* buckets;
  unsigned long long* hcount;
  unsigned long long* sum;
  long long* vmax;
  const KSubHist* sub;
  uint32_t acc_w0_s;  // shared address of word0 of this aggregation for slot 0, this lane's replica
  unsigned long long* csum;  // this aggregation's sum in the CTA's 64-bit totals (shared memory), slot 0
  uint32_t ctw;              // words per slot of those totals
  uint32_t gstride_b;  // bytes between two slots' accumulators
  int acc_smem;
  uint32_t tb;         // global slot of local slot 0 (slot window of the block; 0 without a time window)
};

// BasicHist with a 64-bit bucket size, or MultiHist: first sub-range containing v (hist_multi.go:81-86)
__device__ __noinline__ void hist_bucket_general(const AggSlow* A, uint32_t g, long long v) {
  for (int s = 0; s < A->nsub; s++) {
    const KSubHist S = A->sub[s];
    if (A->multi) {  // a value in (Max, 10*Max] passes the MultiHist's reject rule but lies in no sub-range
      if (v < S.lo || v > S.hi) continue;
      if (v > S.reject_hi || v < S.lo) break;  // the subhist's own reject rule
    }
    long long b = (long long)((unsigned long long)v - (unsigned long long)S.lo) / S.bsize;
    if (b >= (long long)S.nvals) b = (long long)S.nvals - 1;  // outlier: last slot (hist_basic.go:134-137)
    if (b < 0) b = 0;
    gred_add(A->buckets + ((size_t)(g + A->tb) * A->nvals_total + S.base + (uint32_t)b), 1ull);
    break;
  }
}

// A value outside the fast range [max(info_min,0), min(info_max, 2^32-1)] of a row that passed:
// the complete AddWeightedValue (hist_basic.go:101-151).  count_accepted: word0 counts accepted
// values (bucket columns); otherwise it counts the NON-accepted ones (value arrays).
__device__ __noinline__ void agg_slow(const AggSlow* A, uint32_t g, long long v, int count_accepted) {
  if (v > A->reject_hi || v < A->info_min) {  // hist_basic.go:104
    if (A->acc_smem && !count_accepted) sred_add(A->acc_w0_s + g * A->gstride_b, 1u);
    return;
  }
  if (A->acc_smem) {
    if (count_accepted) sred_add(A->acc_w0_s + g * A->gstride_b, 1u);
    // the value goes straight to the CTA's 64-bit total of the slot (shared memory; the fold between blocks
    // runs between barriers): in the replicated low limb its low word (up to 2^32-1 for a negative value)
    // would void the `nocarry` bound, and a later hot-path add would drop its carry
    atomicAdd(A->csum + (size_t)(g + A->tb) * A->ctw, (unsigned long long)v);
  } else {
    gred_add(A->hcount + g + A->tb, 1ull);
    gred_add(A->sum + g + A->tb, (unsigned long long)v);
  }
  if (v > A->info_max) gred_max(A->vmax + g + A->tb, v);
  if (A->nsub > 0) hist_bucket_general(A, g, v);
}

// Weights carried over rows without the weight column (Plan::wcarry; aggregate.go:68,100-102).  After the group
// passes such a row's digit on the weight axis (the last group axis: stride, radix) is 0; it takes the digit of the
// nearest earlier row of the block whose digit is not 0, or keeps 0 (weight 1) when there is none.  That is a
// "last non-zero" scan over the block's rows.  Each warp owns a contiguous run of rows: it finds its run's last
// non-zero digit walking back from the end (one 32-row step unless the run's tail lacks the column), the warps
// exchange those once through `xw` (NWARPS words of shared memory), and each warp then walks its run forward
// 32 rows a step, a ballot and two shuffles per step.  Every digit is read back from the slot word, whichever
// pass wrote it.  Inlined: as an out-of-line call it moved the caller's register allocation (spill loads of the
// shared-accumulator instantiations +260 bytes, the C3 bench kernel 0.2% slower on H100); inlined, the unweighted
// instantiations spill within 20 bytes of what they did without it.
template <typename SlotT>
__device__ __forceinline__ void carry_weight(SlotT* slot, uint32_t nrec, uint32_t gmask, uint32_t stride, uint32_t radix,
                                          uint32_t* xw) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  const uint32_t per = (nrec + 32u * NWARPS - 1u) / (32u * NWARPS) * 32u;  // rows per warp, whole steps
  const uint32_t r0 = min(warp * per, nrec), r1 = min(r0 + per, nrec);
  auto digit = [&](uint32_t r) -> uint32_t { return r < r1 ? (((uint32_t)slot[r] & gmask) / stride) % radix : 0u; };
  uint32_t last = 0;
  if (r1 > r0) {
    for (uint32_t b = r0 + (r1 - 1u - r0) / 32u * 32u;; b -= 32u) {
      const uint32_t d = digit(b + lane);
      const uint32_t m = __ballot_sync(FULL, d != 0u);
      if (m) {
        last = __shfl_sync(FULL, d, 31 - __clz(m));
        break;
      }
      if (b == r0) break;
    }
  }
  if (lane == 0) xw[warp] = last;
  __syncthreads();
  uint32_t carry = 0;
  for (uint32_t w = 0; w < warp; w++)
    if (xw[w]) carry = xw[w];
  for (uint32_t b = r0; b < r1; b += 32u) {
    const uint32_t r = b + lane, d = digit(r);
    const uint32_t below = __ballot_sync(FULL, d != 0u) & (FULL >> (31u - lane));  // lanes <= this one with a digit
    const uint32_t src = __shfl_sync(FULL, d, below ? 31 - __clz(below) : 0);
    const uint32_t v = below ? src : carry;
    if (d == 0u && v != 0u && r < r1) slot[r] = (SlotT)(slot[r] + v * stride);
    carry = __shfl_sync(FULL, v, 31);
  }
  __syncthreads();
}

// ---------------------------------------------------------------------------
// the kernel
// ---------------------------------------------------------------------------
template <typename SlotT, bool ACC_SMEM, bool HASHG = false>
__global__ void __launch_bounds__(THREADS, CTAS_PER_SM) scan_kernel(const LaunchParams lp) {
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  const Plan* __restrict__ PP = lp.plan;
  Ctx cx;
  cx.tid = threadIdx.x;
  cx.lane = threadIdx.x & 31;
  cx.warp = threadIdx.x >> 5;
  cx.epoch = 0;
  // the 128B swizzle pattern of the staged tiles repeats every 1 KiB: the window must start on one
  unsigned char* const stage_base = smem_raw;
  if (smem_u32(smem_raw) & 1023u) __trap();
  cx.stage_bytes = lp.stage_units * (TMA_TILE_BYTES / 2);  // 0 when the table has no tensor maps
  cx.zero = lp.nlist >> 31;  // nlist < 2^31
  cx.tmaps = reinterpret_cast<const unsigned char*>(lp.tmaps);
  unsigned char* const smem = stage_base + NWARPS * cx.stage_bytes;
  cx.headbits = reinterpret_cast<uint32_t*>(smem + OFF_HEADBITS);
  cx.headprefix = reinterpret_cast<uint16_t*>(smem + OFF_HEADPREFIX);
  cx.binpay_s = reinterpret_cast<uint32_t*>(smem + OFF_BINPAY);
  cx.pubA = reinterpret_cast<volatile unsigned long long*>(smem + OFF_PUBA);
  cx.pubB = reinterpret_cast<volatile unsigned long long*>(smem + OFF_PUBB);
  cx.misc = reinterpret_cast<volatile uint32_t*>(smem + OFF_MISC);
  uint32_t* const plist_w = reinterpret_cast<uint32_t*>(smem + OFF_PLIST);
  cx.plist = plist_w;
  cx.timing = lp.dbg != nullptr && cx.warp == 0;
  cx.t_tma = cx.t_lb = 0;
  cx.npass = cx.pass_idx = 0;
  cx.pref_idx = 0xffffffffu;
  {
    cx.buf0 = smem_u32(stage_base) + (uint32_t)cx.warp * cx.stage_bytes;
    cx.buf1 = cx.buf0 + TMA_TILE_BYTES;
    cx.mbar0 = smem_u32(smem + OFF_MBAR) + (uint32_t)cx.warp * 16u;
    cx.mbar1 = cx.mbar0 + 8u;
    cx.par0 = cx.par1 = 0;
  }
  if (cx.stage_bytes && cx.lane == 0) {
    mbar_init(cx.mbar0, 1);
    mbar_init(cx.mbar1, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  SlotT* slot;
  uint32_t acc_off = FIXED_SMEM;
  if (sizeof(SlotT) == 4) {
    slot = reinterpret_cast<SlotT*>(lp.gslots + (size_t)blockIdx.x * SG_BLOCK_ROWS);
  } else {
    slot = reinterpret_cast<SlotT*>(smem + FIXED_SMEM);
    acc_off = FIXED_SMEM + SG_BLOCK_ROWS * sizeof(SlotT);
  }
  cx.acc = reinterpret_cast<uint32_t*>(smem + acc_off);
  const uint32_t slot_s = sizeof(SlotT) < 4 ? smem_u32(smem + FIXED_SMEM) : 0u;  // slot words in the shared window
  uint32_t* const gbinpay = lp.gbinpay + (size_t)blockIdx.x * SG_BLOCK_ROWS;

  // ---- plan scalars into registers (the plan lives in global memory; every shared
  // atomic would otherwise force the compiler to reload it) -------------------------------
  const int nfilters = PP->nfilters, ngroups = PP->ngroups, naggs = PP->naggs, ncolslots = PP->ncolslots;
  const int time_col = PP->time_col;
  const uint32_t gbits = PP->gbits, pass_target = PP->pass_target, finc = PP->finc, time_ok = PP->time_ok;
  const uint32_t filt_target = PP->filt_target, filt_mask = PP->filt_mask, nslots = PP->nslots;
  // local slot space (see Plan): slot words, replicated accumulators and the histogram cache index it
  const uint32_t lslots = PP->lslots;
  const bool fail_mode = PP->fail_mode != 0;
  const uint32_t acc_words = PP->acc_words, R = ACC_SMEM ? PP->acc_repl : 1u;
  const uint32_t gmask = (1u << gbits) - 1u;
  const uint32_t gstride = acc_words * R;       // words between two slots' accumulators
  const uint32_t lane_off = cx.lane & (R - 1);  // this lane's replica
  unsigned long long* const g_count = reinterpret_cast<unsigned long long*>(PP->count);
  unsigned long long* const g_scalars = reinterpret_cast<unsigned long long*>(PP->scalars);

  // replicated words of (lslots + trash) local slots, then one unreplicated high limb per (slot, aggregation)
  const uint32_t acc_rep = ACC_SMEM ? (lslots + 1u) * gstride : 0u;
  const uint32_t tw_magic = 0xffffffffu / (1u + 2u * (uint32_t)naggs) + 1u;  // x / tw == umulhi(x, magic), x * tw < 2^32
  const uint32_t acc_total = ACC_SMEM ? acc_rep + (lslots + 1u) * (uint32_t)naggs : 0u;
  for (uint32_t i = cx.tid; i < acc_total; i += THREADS) cx.acc[i] = 0;
  // the CTA's running totals (64-bit, one per GLOBAL slot) behind the replicated accumulators
  unsigned long long* const ctot = reinterpret_cast<unsigned long long*>(cx.acc + ((acc_total + 1u) & ~1u));
  const uint32_t ctot_n = ACC_SMEM ? nslots * (1u + 2u * (uint32_t)naggs) : 0u;
  for (uint32_t i = cx.tid; i < ctot_n; i += THREADS) ctot[i] = 0;
  // the histogram cache: 32-bit bucket counters of the first hist_rows local slots (DESIGN.md §4).  A
  // row in the cache costs one shared reduction instead of one 64-bit reduction to L2.
  const uint32_t hist_rows = ACC_SMEM ? PP->hist_rows : 0u, hrw = PP->hist_row_words;
  uint32_t* const hist = reinterpret_cast<uint32_t*>(ctot + ((ctot_n + 1u) & ~1u));
  const uint32_t hist_s = smem_u32(hist);
  for (uint32_t i = cx.tid; i < hist_rows * hrw; i += THREADS) hist[i] = 0;
  uint32_t hist_tb = 0;      // global slot of the cache's row 0
  uint32_t hist_blocks = 0;  // blocks counted into the cache since its last flush (32-bit counters: < 65,536)
  auto hist_flush = [&]() {
    __syncthreads();
    const uint32_t nw = hist_rows * hrw;
    for (uint32_t i = cx.tid; i < nw; i += THREADS) {
      const uint32_t v = hist[i];
      if (!v) continue;
      hist[i] = 0;
      const uint32_t row = i / hrw, off = i - row * hrw;
      for (int a = 0; a < naggs; a++) {
        const uint32_t ho = PP->aggs[a].hrow_off, nv = PP->aggs[a].nvals_total;
        if (ho != HROW_NONE && off >= ho && off - ho < nv) {
          gred_add(reinterpret_cast<unsigned long long*>(PP->aggs[a].buckets) + ((size_t)(row + hist_tb) * nv + (off - ho)),
                   (unsigned long long)v);
          break;
        }
      }
    }
    hist_blocks = 0;
    __syncthreads();
  };
  for (uint32_t i = cx.tid; i < MAX_TILES; i += THREADS) {
    cx.pubA[i] = 0;
    cx.pubB[i] = 0;
  }
  // candidate passes of the plan, in execution order: column | kind << 16 (0 filter, 1 group, 2 time,
  // 3 aggregation) | (string filter) << 24.  Built once; each block only looks its columns up.
  uint32_t* const pcand = reinterpret_cast<uint32_t*>(smem + OFF_PCAND);
  uint32_t* const ptmp = reinterpret_cast<uint32_t*>(smem + OFF_PTMP);
  // the block's column descriptors, one per candidate pass (same order as pcand): each pass would
  // otherwise start with two dependent global loads (plan -> column slot -> descriptor)
  DevCol* const colcache = reinterpret_cast<DevCol*>(smem + OFF_COLCACHE);
  if (cx.tid == 0) {
    uint32_t nc = 0;
    for (int fi = 0; fi < nfilters; fi++)
      pcand[nc++] = (uint32_t)PP->filters[fi].col | (0u << 16) | (PP->filters[fi].is_str ? 1u << 24 : 0u);
    for (int gi = 0; gi < ngroups; gi++) pcand[nc++] = (uint32_t)PP->groups[gi].col | (1u << 16);
    if (time_col >= 0) pcand[nc++] = (uint32_t)time_col | (2u << 16);
    for (int ai = 0; ai < naggs; ai++) pcand[nc++] = (uint32_t)PP->aggs[ai].col | ((uint32_t)ai << 8) | (3u << 16);
    cx.misc[3] = nc;
  }
  __syncthreads();
  const uint32_t ncand = cx.misc[3];
  unsigned long long matched = 0;
  // optional phase timing (thread 0 of each CTA): 0 init, 1 filters, 2 groups, 3 time, 4 count+aggs, 5 flush, 6 fetch
  unsigned long long* const dbg = lp.dbg ? lp.dbg + (size_t)blockIdx.x * 16 : nullptr;
  // phase counters live in shared memory (only thread 0 touches them): no registers spent on them
  volatile unsigned long long* const tacc = reinterpret_cast<volatile unsigned long long*>(cx.misc + 96);  // [0..6] + [7] last stamp
  if (dbg && cx.tid == 0) {
    for (int i = 0; i < 16; i++) tacc[i] = 0;
    tacc[7] = (unsigned long long)clock64();
  }
#ifndef SG_FINE_TIMING
  // SG_PHASE_TIMING also splits the block by column pass: dbg[9 + p] for the p-th pass of the plan (first 7)
  auto pass_mark = [&](int p) {
    if (dbg && cx.tid == 0) {
      const unsigned long long now = (unsigned long long)clock64();
      if (p >= 0 && p < 7) tacc[9 + p] += now - tacc[8];
      tacc[8] = now;
    }
  };
#else
  auto pass_mark = [&](int) {};
#endif
  auto phase = [&](int i) {
    if (dbg && cx.tid == 0) {
      const unsigned long long now = (unsigned long long)clock64();
      tacc[i] += now - tacc[7];
      tacc[7] = now;
    }
#ifdef SG_FINE_TIMING
    cx.tmark(13);  // everything outside the marked regions
#endif
  };
#ifdef SG_FINE_TIMING
  cx.tacc = tacc;
  cx.t0 = dbg && cx.tid == 0;
  if (cx.t0) {
    for (int i = 8; i < 16; i++) tacc[i] = 0;
    tacc[8] = (unsigned long long)clock64();
  }
#endif

#ifdef SG_STAGGER
  {  // experiment: desynchronise the CTAs' phases
    const long long until = clock64() + (long long)(blockIdx.x % 16u) * SG_STAGGER;
    while (clock64() < until) {
    }
  }
#endif
  // pending-fold state: bits 0-7 blocks accumulated since the last fold, 8 discard, 9 fold right away
  // (aggregation-subset item), 10 the item owns the Count, 16+ word0 semantics per aggregation
  uint32_t fstate = 0;
  uint32_t fold_tb = 0;  // slot window base of the block(s) waiting to be folded
  for (;;) {
    __syncthreads();
    if (cx.tid == 0) {
      cx.misc[0] = atomicAdd(lp.work_counter, 1u);
      cx.misc[1] = 0;
    }
    __syncthreads();
    const uint32_t wi = cx.misc[0];
    const bool done = wi >= lp.nlist;
    // work item = {block, aggregation mask | owner bit, NumRecords, -}: one load behind the counter.
    // Tail blocks may be split into several items, one per subset of the aggregations
    const uint4 item = done ? make_uint4(0u, 0x8000ffffu, 0u, 0u) : lp.items[wi];
    const uint32_t next_imask = item.y;
    // ---- deferred fold.  The replicated 32-bit accumulators of up to lp.fold_every consecutive blocks
    // are folded together (the planner bounds that number so that the no-carry proof of the hot path
    // still holds); always before an item that computes a subset of the aggregations, after one,
    // after a broken block (whose partial sums — and the pending blocks' — are discarded: the host
    // reruns the launch without that block) and when the CTA runs out of work.
    if (ACC_SMEM && (fstate & 0xffu) != 0u &&
        (done || (fstate & 0xffu) >= lp.fold_every || (fstate & 0x300u) != 0u || next_imask != 0x8000ffffu)) {
      const bool broken = (fstate & 0x100u) != 0u, owner = (fstate & 0x400u) != 0u;
      const uint32_t agg_mode_bits = fstate >> 16;
      fstate = 0;
      // Fold the R replicas of every accumulator word into the CTA's running 64-bit totals (shared
      // memory, no atomics) and zero them for the next block.  A row = the R replicas of one
      // (slot, word).  R >= 4: every lane takes 16 bytes, R/4 lanes share a row, 128/R rows per warp
      // step — consecutive addresses across the warp (no bank conflicts) — and the lanes of a row
      // combine with xor-shuffles.  The totals reach the global accumulators once, when the CTA runs
      // out of blocks: per-block global reductions from one CTA per SM in lockstep serialise on the same
      // few hundred L2 addresses right in front of a barrier.
      const uint32_t tw = 1u + 2u * (uint32_t)naggs;  // words per slot: count, then (word0, low limb) per agg
      const uint32_t nrows = lslots * tw, nrows_all = (lslots + 1u) * tw;  // + the trash slot (zeroed only)
      auto fold_row = [&](uint32_t row, unsigned long long t) {
        const uint32_t g = tw == 1u ? row : __umulhi(row, tw_magic), w = row - g * tw;  // exact: row * tw < 2^32
        if (w == 0) {
          // this block's count of slot g: parked in the (zeroed) row for the second step below
          cx.acc[row * R] = (uint32_t)t;
          if (R > 1) cx.acc[row * R + 1] = (uint32_t)(t >> 32);
          if (!broken && owner) ctot[(g + fold_tb) * tw] += t;
        } else if (!broken) {
          // word0 of a value-array aggregation counts the NON-accepted rows: hist count = count - word0
          const bool neg = (w & 1u) && ((agg_mode_bits >> ((w - 1u) >> 1)) & 1u);
          ctot[(g + fold_tb) * tw + w] += neg ? (0ull - t) : t;
        }
      };
      if (R >= 4) {
        const uint32_t lpr = R >> 2;  // lanes per row
        const uint32_t lg = 31u - (uint32_t)__clz(lpr);
        const uint32_t rps = 32u >> lg;
        const uint32_t sub = (uint32_t)cx.lane & (lpr - 1u), grp = (uint32_t)cx.lane >> lg;
        uint4* const acc4 = reinterpret_cast<uint4*>(cx.acc);
        for (uint32_t r0 = (uint32_t)cx.warp * rps; r0 < nrows_all; r0 += NWARPS * rps) {
#ifdef SG_FINE_FLUSH
          cx.tmark(12);
#endif
          const uint32_t row = r0 + grp;
          uint4 q = make_uint4(0, 0, 0, 0);
          if (row < nrows_all) {
            q = acc4[row * lpr + sub];
            acc4[row * lpr + sub] = make_uint4(0, 0, 0, 0);
          }
          unsigned long long t = ((unsigned long long)q.x + q.y) + ((unsigned long long)q.z + q.w);
#ifdef SG_FINE_FLUSH
          if (t == 0x123456789ull) cx.misc[5] = 1;
          cx.tmark(11);
#endif
          for (uint32_t d = lpr >> 1; d > 0; d >>= 1) t += __shfl_xor_sync(FULL, t, d);
#ifdef SG_FINE_FLUSH
          if (t == 0x123456789ull) cx.misc[5] = 1;
          cx.tmark(10);
#endif
          if (sub == 0 && row < nrows) fold_row(row, t);
        }
      } else {
        for (uint32_t row = cx.tid; row < nrows_all; row += THREADS) {
          unsigned long long t = cx.acc[row * R];
          cx.acc[row * R] = 0;
          if (R == 2) {
            t += cx.acc[row * R + 1];
            cx.acc[row * R + 1] = 0;
          }
          if (row < nrows) fold_row(row, t);
        }
      }
      cx.tmark(14);  // fold loop
      __syncthreads();
      // second step, one thread per (slot, aggregation): the unreplicated high limbs and "+ count"
      for (uint32_t i = cx.tid; i < (lslots + 1u) * (uint32_t)naggs; i += THREADS) {
        const uint32_t g = i / (uint32_t)naggs, a = i - g * (uint32_t)naggs;
        const unsigned long long hi = cx.acc[acc_rep + i];
        cx.acc[acc_rep + i] = 0;
        if (g < lslots && !broken) {
          unsigned long long cnt = cx.acc[g * gstride];  // R == 1: a block's count fits one word
          if (R > 1) cnt |= (unsigned long long)cx.acc[g * gstride + 1] << 32;
          if (hi) ctot[(g + fold_tb) * tw + 2 + 2 * a] += hi << 32;
          if ((agg_mode_bits >> a) & 1u) ctot[(g + fold_tb) * tw + 1 + 2 * a] += cnt;
        }
      }
      __syncthreads();
      for (uint32_t g = cx.tid; g < lslots; g += THREADS) {
        cx.acc[g * gstride] = 0;
        if (R > 1) cx.acc[g * gstride + 1] = 0;
      }
    }
    // (the block below starts behind the barrier that ends the pass-list build)

    if (done) break;
    phase(6);
    const uint32_t bid = item.x, imask = item.y, nrec = item.z;
    // (a discovery launch of the sparse path aggregates nothing: no aggregation pass enters the block's pass list)
    const uint32_t aggmask = (sizeof(SlotT) == 4 && lp.hdisc) ? 0u : imask & 0xffffu;
    const bool owner = (imask >> 31) != 0;
    const DevCol* __restrict__ cols = lp.cols + (size_t)bid * ncolslots;

    // the block's TMA-fed passes in execution order (mirrors the pass sequence below): one thread
    // per candidate looks its column up, warp 0 compacts after the barrier.  ptmp[4 * i]: bit 0 TMA-fed,
    // bit 1 read in the code pass (COL_CODES filter / group / time column), bits 2.. its CODE_* role
    bool my_code = false;
    if ((uint32_t)cx.tid < ncand) {
      const uint32_t pc = pcand[cx.tid];
      const uint32_t kind = (pc >> 16) & 0xffu;
      const DevCol c = cols[pc & 0xffu];
      bool on = cx.tmaps != nullptr && (c.flags & COL_TMA) && cx.stages(col_shift(c.flags)) != 0u;
      bool bucket = c.enc == SG_ENC_BUCKET;
      const bool coded = bucket && (c.flags & COL_CODES);
      uint32_t role = CODE_ADD;
      if (kind == 0) {
        // (a bucket filter in fail mode walks only the tiles of its failing bins, with plain loads)
        on = on && ((bucket && !fail_mode) || (c.enc == SG_ENC_VALUES && !(pc >> 24)));
        my_code = coded && PP->filters[cx.tid].op < SG_OP_IN;
        if (fail_mode) role = CODE_OR;
      } else if (kind == 1) {
        on = on && (bucket || (HASHG && c.enc == SG_ENC_VALUES && !(c.flags & COL_IS_STR)));
        my_code = coded;
      } else {
        on = on && !(c.flags & COL_IS_STR) && (bucket || c.enc == SG_ENC_VALUES);
        if (kind == 3) on = on && ((aggmask >> ((pc >> 8) & 0xffu)) & 1u);
        bool cconst = false;
        if (kind == 2 && (c.enc == SG_ENC_VALUES || (bucket && (c.flags & COL_FULL))) && (c.flags & COL_STATS) &&
            !(c.flags & COL_IS_STR)) {
          // a fully populated time column whose extents fall into one time bucket is not read at all
          const uint32_t clo = time_code(c.vmin, PP->time_bucket, PP->time_first, PP->time_radix);
          cconst = clo != 0u && clo == time_code(c.vmax, PP->time_bucket, PP->time_first, PP->time_radix);
        }
        if (cconst) on = false;
        my_code = kind == 2 && coded && !(c.flags & COL_IS_STR) && !cconst;
        role = CODE_TIME;
      }
      uint32_t n = c.nitems;
      if (!bucket && n > nrec) n = nrec;
      colcache[cx.tid] = c;
      ptmp[4 * cx.tid + 0] = (on ? 1u : 0u) | (my_code ? 2u | (role << 2) : 0u);
      ptmp[4 * cx.tid + 1] = c.data_chunk * 3u + col_shift(c.flags);  // which view of the chunk (see make_feed)
      ptmp[4 * cx.tid + 2] = c.data_row << col_shift(c.flags);
      ptmp[4 * cx.tid + 3] = bucket ? (n + (32 * BE - 1)) / (32 * BE) : (n + (32 * VE - 1)) / (32 * VE);
    }
    const bool code_pass = __syncthreads_or(my_code) != 0;
    // every row starts as: group slot 0, no filter passed (the code pass, when there is one, stores every row's word)
    if (!code_pass) {
      if (sizeof(SlotT) < 4) {
        uint4* s4 = reinterpret_cast<uint4*>(slot);
        const uint32_t n16 = (nrec * (uint32_t)sizeof(SlotT) + 15u) / 16u;
        for (uint32_t i = cx.tid; i < n16; i += THREADS) s4[i] = make_uint4(0, 0, 0, 0);
      } else {
        for (uint32_t r = cx.tid; r < nrec; r += THREADS) slot[r] = 0;
      }
    }
    if (cx.warp == 0) {
      uint32_t np = 0;
      for (uint32_t b0 = 0; b0 < ncand; b0 += 32) {
        const uint32_t i = b0 + cx.lane;
        const bool on = i < ncand && (ptmp[4 * i] & 1u) != 0;
        const uint32_t m = __ballot_sync(FULL, on);
        if (on) {
          const uint32_t pos = np + __popc(m & ((1u << cx.lane) - 1u));
          plist_w[4 * pos + 0] = ptmp[4 * i + 1];
          plist_w[4 * pos + 1] = ptmp[4 * i + 2];
          plist_w[4 * pos + 2] = ptmp[4 * i + 3];
        }
        np += __popc(m);
      }
      if (cx.lane == 0) cx.misc[2] = np;
    }
    __syncthreads();
    cx.npass = cx.misc[2];
    cx.pass_idx = 0;
    cx.pref_idx = 0xffffffffu;
    // ---- slot window of this block: first time code from the time column's exact extents -------------
    const long long tbk = PP->time_bucket, tfirst = PP->time_first;
    const uint32_t tradix = PP->time_radix, tstride = PP->time_stride, twin = PP->time_win;
    uint32_t tcode0 = 1u;
    if (time_col >= 0 && twin + 1u < tradix) {
      const DevCol& tc = colcache[nfilters + ngroups];
      if (tc.enc != SG_ENC_ABSENT && !(tc.flags & COL_IS_STR) && (tc.flags & COL_STATS)) {
        const uint32_t c0 = time_code(tc.vmin, tbk, tfirst, tradix);
        if (c0) tcode0 = min(c0, tradix - twin);  // the window stays inside the axis
      }
    }
    const uint32_t tb = (tcode0 - 1u) * tstride;
    if (hist_rows && (tb != hist_tb || hist_blocks >= 65535u)) {
      hist_flush();
      hist_tb = tb;
    }
    hist_blocks++;
    auto rel_of = [&](uint32_t code) -> uint32_t {  // global time code (0 = off the axis) -> window-relative, 0 = bad
      const uint32_t r = code - tcode0 + 1u;
      return (code != 0u && r >= 1u && r <= twin) ? r : 0u;
    };
    // Count without touching a row: with no filter, no time column and ONE group column whose bins list every
    // row of the block exactly once (COL_FULL), a group's Count in this block is the size of its bin
    const bool count_in_group = ACC_SMEM && nfilters == 0 && time_col < 0 && ngroups == 1 &&
                                colcache[0].enc == SG_ENC_BUCKET && (colcache[0].flags & COL_FULL) != 0u;
    phase(0);
    pass_mark(-1);
    int pass_no = 0;

    // ---- code pass: every COL_CODES filter, group and time column of the block in ONE row-ordered loop -------
    // A column's per-bin payload is what its own pass below would give the rows of that bin; each lane then reads
    // 16 consecutive rows' codes of every such column (16 bytes each), looks the payloads up and stores the 16 slot
    // words: the first writer of every row (the zeroing above is skipped), no head bits, no look-back, no atomics.
    if (code_pass) {
      uint32_t ncode = 0;
      const SlotT fincS = (SlotT)finc;
      for (uint32_t i = 0; i < ncand; i++) {
        const uint32_t f = ptmp[4 * i];
        if (!(f & 2u)) continue;
        const DevCol& c = colcache[i];
        const uint32_t kind = (pcand[i] >> 16) & 0xffu;
        uint32_t* const pay = (ncode + 1u) * CODE_BINS <= SMEM_BINS ? cx.binpay_s + ncode * CODE_BINS : gbinpay + ncode * CODE_BINS;
        for (uint32_t b = cx.tid; b < CODE_BINS; b += THREADS) {
          uint32_t p = 0;
          if (b < c.nbins) {
            if (kind == 0) {
              const KFilter& F = PP->filters[i];
              StrPred sp;
              sp.op = F.op;
              sp.gid = F.str_gid;
              sp.lut = F.lut;
              sp.lut_bits = F.lut_bits;
              const long long bv = c.bin_values[b];
              const bool pass = F.is_str ? sp(str_gid(c, bv)) : int_pred(F.op, bv, F.ival);
              p = (pass != fail_mode) ? (uint32_t)fincS : 0u;  // count mode: finc = passes; fail mode: finc = fails
            } else if (kind == 1) {
              const KGroup& G = PP->groups[i - (uint32_t)nfilters];
              const int32_t code = G.is_str ? str_gid(c, c.bin_values[b]) : c.remap[b];
              p = code == G.alias ? 0u : ((uint32_t)code + 1u) * G.stride;
              if (count_in_group)
                sred_add(smem_u32(cx.acc + p * gstride + lane_off), c.bin_offsets[b + 1] - c.bin_offsets[b]);
            } else {
              const uint32_t rc = rel_of(time_code(c.bin_values[b], tbk, tfirst, tradix));
              p = rc ? rc * tstride + time_ok : 0u;  // 0: counted into SC_TIME_OVERFLOW below
            }
          }
          pay[b] = p;
        }
        if (cx.tid == 0) ptmp[4 * ncode + 1] = i | ((f >> 2) << 8);  // (ncode <= i: no flag word is overwritten)
        ncode++;
      }
      __syncthreads();
      unsigned long long ovf = 0;  // listed rows outside the time window
      const uint32_t pay_s = smem_u32(cx.binpay_s);
      for (uint32_t idx0 = (uint32_t)cx.tid * 16u; idx0 < nrec; idx0 += THREADS * 16u) {
        uint32_t w[16];
#pragma unroll
        for (int k = 0; k < 16; k++) w[k] = 0u;
        // columns in groups of CODE_BATCH: their loads are in flight together (the first group's tables are in
        // shared memory, any further ones in gbinpay)
        for (uint32_t j0 = 0; j0 < ncode; j0 += CODE_BATCH) {
          uint4 q[CODE_BATCH];
          uint32_t role[CODE_BATCH];
#pragma unroll
          for (uint32_t jj = 0; jj < CODE_BATCH; jj++) {
            q[jj] = make_uint4(FULL, FULL, FULL, FULL);
            role[jj] = CODE_ADD;
            if (j0 + jj < ncode) {
              const uint32_t e = ptmp[4 * (j0 + jj) + 1];
              role[jj] = e >> 8;
              q[jj] = __ldg(reinterpret_cast<const uint4*>(colcache[e & 0xffu].codes + idx0));
            }
          }
#pragma unroll
          for (uint32_t jj = 0; jj < CODE_BATCH; jj++) {
            if (j0 + jj >= ncode) break;
            const uint32_t cw[4] = {q[jj].x, q[jj].y, q[jj].z, q[jj].w};
#pragma unroll
            for (int k = 0; k < 16; k++) {
              const uint32_t code = (cw[k >> 2] >> (8 * (k & 3))) & 0xffu;
              uint32_t v;
              if (j0 == 0)
                asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(pay_s + (jj * CODE_BINS + code) * 4u));
              else
                v = gbinpay[(j0 + jj) * CODE_BINS + code];
              w[k] = role[jj] == CODE_OR ? (w[k] | v) : (w[k] + v);
              if (role[jj] == CODE_TIME && v == 0u && code != 0xffu) ovf++;
            }
          }
        }
        if (sizeof(SlotT) == 1) {
          uint32_t p[4];
#pragma unroll
          for (int j = 0; j < 4; j++) p[j] = w[4 * j] | (w[4 * j + 1] << 8) | (w[4 * j + 2] << 16) | (w[4 * j + 3] << 24);
          *reinterpret_cast<uint4*>(slot + idx0) = make_uint4(p[0], p[1], p[2], p[3]);
        } else if (sizeof(SlotT) == 2) {
          uint32_t p[8];
#pragma unroll
          for (int j = 0; j < 8; j++) p[j] = w[2 * j] | (w[2 * j + 1] << 16);
          reinterpret_cast<uint4*>(slot + idx0)[0] = make_uint4(p[0], p[1], p[2], p[3]);
          reinterpret_cast<uint4*>(slot + idx0)[1] = make_uint4(p[4], p[5], p[6], p[7]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; j++)
            reinterpret_cast<uint4*>(slot + idx0)[j] = make_uint4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
        }
      }
      if (ovf) gred_add(g_scalars + SC_TIME_OVERFLOW, ovf);
      __syncthreads();
      pass_mark(pass_no++);
    }

    // ---- filters (aggregate.go:105-112; unpopulated -> false, Q1) -----------------
    // Count mode: a row collects finc per filter it passes (an unpopulated row passes none).  Fail mode
    // (the plan proved every filter column populates every row of every listed block): a row that fails
    // a filter gets the sticky FAIL bit (finc) OR-ed in — a bucket column then only walks the tiles
    // that hold entries of its FAILING bins.
    for (int fi = 0; fi < nfilters; fi++) {
      if (ptmp[4 * fi] & 2u) continue;  // read in the code pass
      const KFilter F = PP->filters[fi];
      const DevCol c = colcache[fi];
      const SlotT fincS = (SlotT)finc;
      StrPred sp;
      sp.op = F.op;
      sp.gid = F.str_gid;
      sp.lut = F.lut;
      sp.lut_bits = F.lut_bits;
      if (F.op >= SG_OP_IN) {
        // SetFilter (filter.go:252-285) over a set column in its bucket form (unpackSetCol, column_store_io.go:641-668):
        // sticky bits instead of a pass count — a row may be listed in several bins.  The planner keeps such a query
        // in count mode (fail_mode == 0).
        if (c.enc == SG_ENC_BUCKET) {
          // A column with more than SG_BLOCK_ROWS pairs comes in segments of whole bins (COL_SEGS), each walked like
          // a column of its own; the bits are ORed, so the order does not matter.  Under IN only the literal's bins
          // set bits: a segment without one is not read at all (its rows were range-checked at staging).
          const uint32_t nseg = (c.flags & COL_SEGS) ? 1u + (uint32_t)((unsigned long long)c.vmax >> 32) : 1u;
          for (uint32_t s = 0; s < nseg; s++) {
            const DevCol sc = s ? lp.segs[(uint32_t)c.vmax + s - 1u] : c;
            uint32_t* pay = sc.nbins <= SMEM_BINS ? cx.binpay_s : gbinpay;
            uint32_t any = 0;
            for (uint32_t b = cx.tid; b < sc.nbins; b += THREADS) {
              const uint32_t p = F.set_pbit | (str_gid(sc, sc.bin_values[b]) == F.str_gid ? F.set_tbit : 0u);
              pay[b] = p;
              any |= p;
            }
            if (!__syncthreads_or(any) && nseg > 1u) continue;
            scan_bucket<SlotT>(
                cx, sc, nrec, [&](uint32_t bin) { return (SlotT)pay[bin]; },
                [&](uint32_t row, SlotT cur) {
                  if (cur) slot_or(slot, slot_s, row, (uint32_t)cur);
                });
          }
        }
        // rows the non-bucketed file form listed (even with an empty set) are populated (a column of nothing but
        // empty sets is staged as ABSENT + COL_SET)
        const uint32_t npop = (c.flags & COL_SET) ? (uint32_t)min((long long)nrec, max(0ll, (long long)c.vmin)) : 0u;
        if (F.set_pbit && npop) {
          for (uint32_t r = cx.tid; r < npop; r += THREADS) slot_or(slot, slot_s, r, F.set_pbit);
          __syncthreads();
        }
        pass_mark(pass_no++);
        continue;
      }
      if (c.enc == SG_ENC_BUCKET) {
        uint32_t* pay = c.nbins <= SMEM_BINS ? cx.binpay_s : gbinpay;
        const bool push_down = PP->fail_mode == 1u;
        if (push_down) {
          if (!(c.flags & COL_FULL)) __trap();  // the planner only picks fail mode over fully populated columns
          if (cx.tid < 2) cx.misc[6 + cx.tid] = 0;
          __syncthreads();
        }
        for (uint32_t b = cx.tid; b < c.nbins; b += THREADS) {
          const long long bv = c.bin_values[b];
          const bool pass = F.is_str ? sp(str_gid(c, bv)) : int_pred(F.op, bv, F.ival);
          pay[b] = (pass != fail_mode) ? 1u : 0u;  // count mode: 1 = passes; fail mode: 1 = fails
          if (push_down && !pass) {
            const uint32_t o0 = c.bin_offsets[b], o1 = c.bin_offsets[b + 1];
            for (uint32_t t = o0 >> 10; t <= ((o1 - 1u) >> 10) && t < 64u; t++)
              atomicOr(const_cast<uint32_t*>(&cx.misc[6 + (t >> 5)]), 1u << (t & 31));
          }
        }
        __syncthreads();
        // (a warp-per-failing-bin walk without head bits was tried here: 2.4x slower — every bin costs its
        // warp a round trip to HBM, and one long bin serialises on a single warp)
        {
          // one instantiation serves both modes: rows of bins with a zero payload are left alone (with skipped
          // tiles the entries of such a bin may decode to rows that are not theirs); count mode adds finc to
          // the rows of passing bins, fail mode ORs it into the rows of failing bins
          const unsigned long long need =
              push_down ? ((unsigned long long)cx.misc[6] | ((unsigned long long)cx.misc[7] << 32)) : ~0ull;
          scan_bucket<SlotT>(
              cx, c, nrec, [&](uint32_t bin) { return pay[bin] ? fincS : (SlotT)0; },
              [&](uint32_t row, SlotT cur) {
                if (cur) {
                  if (fail_mode)
                    slot_or(slot, slot_s, row, (uint32_t)cur);
                  else
                    slot_add(slot, slot_s, row, (uint32_t)cur);
                }
              },
              need, !fail_mode);
        }
      } else if (c.enc == SG_ENC_VALUES) {
        uint32_t nval = c.nitems < nrec ? c.nitems : nrec;
        if (F.is_str) {
          scan_values_i32(cx, c, nrec, [&](uint32_t row, int32_t local) {
            const bool pass = sp(str_gid(c, local));
            if (fail_mode) {
              if (!pass) slot[row] = (SlotT)(slot[row] | fincS);
            } else if (pass) {
              slot[row] = (SlotT)(slot[row] + fincS);
            }
          });
        } else {
          const IntRange rg = int_range(F.op, F.ival);
          const bool u32ok = (c.flags & COL_STATS) && c.vmin >= 0 && c.vmax <= 0xffffffffll;
          // clip the range to [0, 2^32) for the 32-bit scan
          const unsigned long long hi64 = rg.lo + rg.span;  // inclusive upper end (signed order = unsigned order
                                                            // after the bias below)
          const long long rlo = (long long)rg.lo, rhi = (long long)hi64;
          const bool none32 = rg.none || rhi < 0 || rlo > 0xffffffffll;
          const uint32_t lo32 = rlo < 0 ? 0u : (uint32_t)rlo;
          const uint32_t span32 = none32 ? 0u : ((rhi > 0xffffffffll ? 0xffffffffu : (uint32_t)rhi) - lo32);
          // the word a row gets: count mode finc when it passes, fail mode finc when it fails
          const uint32_t on_pass = fail_mode ? 0u : finc, on_fail = fail_mode ? finc : 0u;
          if (u32ok) {
            scan_values_u32(cx, c, nrec, [&](uint32_t idx0, const uint32_t(&a)[VE], uint32_t nvalid) {
              uint32_t inc[VE];
#pragma unroll
              for (int k = 0; k < VE; k++)
                inc[k] = k < nvalid ? ((!rg.none && ((!none32 && (a[k] - lo32) <= span32) != rg.inv)) ? on_pass : on_fail) : 0u;
              if (fail_mode)
                or_slots(slot, idx0, inc);
              else
                add_slots(slot, idx0, inc);
            });
          } else {
            scan_values_i64(cx, c, nrec, [&](uint32_t idx0, const unsigned long long(&a)[VE], uint32_t nvalid) {
              uint32_t inc[VE];
#pragma unroll
              for (int k = 0; k < VE; k++) inc[k] = k < nvalid ? (rg((long long)a[k]) ? on_pass : on_fail) : 0u;
              if (fail_mode)
                or_slots(slot, idx0, inc);
              else
                add_slots(slot, idx0, inc);
            });
          }
        }
        if (fail_mode && nval < nrec) {  // rows past len(Values) are unpopulated: they fail (Q1)
          for (uint32_t r = nval + cx.tid; r < nrec; r += THREADS) slot[r] = (SlotT)(slot[r] | fincS);
          __syncthreads();
        }
      } else if (fail_mode) {  // column absent from the block: no row passes
        for (uint32_t r = cx.tid; r < nrec; r += THREADS) slot[r] = (SlotT)(slot[r] | fincS);
        __syncthreads();
      }
      pass_mark(pass_no++);
    }

    phase(1);
    // ---- group key (aggregate.go:125-143) as a dense mixed-radix index ---------------
    // (the first pass to touch the slot words, when there is no filter and no code pass, stores instead of adding)
    for (int gi = 0; gi < ngroups; gi++) {
      if (ptmp[4 * (nfilters + gi)] & 2u) continue;  // read in the code pass
      const KGroup G = PP->groups[gi];
      const DevCol c = colcache[nfilters + gi];
      const bool first = nfilters == 0 && gi == 0 && !code_pass;
      if (c.enc == SG_ENC_BUCKET) {
        uint32_t* pay = c.nbins <= SMEM_BINS ? cx.binpay_s : gbinpay;
        for (uint32_t b = cx.tid; b < c.nbins; b += THREADS) {
          const int32_t code = G.is_str ? str_gid(c, c.bin_values[b]) : c.remap[b];
          pay[b] = code == G.alias ? 0u : ((uint32_t)code + 1u) * G.stride;
          if (count_in_group)
            sred_add(smem_u32(cx.acc + pay[b] * gstride + lane_off), c.bin_offsets[b + 1] - c.bin_offsets[b]);
        }
        __syncthreads();
        if (first) {
          // first pass to touch the (zeroed) slot words: a plain store (measured on C2: 20% faster than the
          // reduction for this pass)
          scan_bucket<SlotT>(
              cx, c, nrec, [&](uint32_t bin) { return (SlotT)pay[bin]; },
              [&](uint32_t row, SlotT cur) { slot[row] = cur; });
        } else {
          scan_bucket<SlotT>(
              cx, c, nrec, [&](uint32_t bin) { return (SlotT)pay[bin]; },
              [&](uint32_t row, SlotT cur) { slot_add(slot, slot_s, row, (uint32_t)cur); });
        }
      } else if (c.enc == SG_ENC_VALUES && G.is_str) {
        const uint32_t stride = G.stride;
        const int32_t alias = G.alias;
        auto word = [&](int32_t local) {
          const int32_t gid = str_gid(c, local);
          return gid == alias ? 0u : ((uint32_t)gid + 1u) * stride;
        };
        if (first) {
          // first pass to touch the zeroed slot words: a store, not a read-modify-write (with the slot words in
          // the global scratch the load was the top stall of the high-cardinality plan)
          scan_values_i32(cx, c, nrec, [&](uint32_t row, int32_t local) { slot[row] = (SlotT)word(local); });
        } else {
          scan_values_i32(cx, c, nrec, [&](uint32_t row, int32_t local) { slot[row] = (SlotT)(slot[row] + word(local)); });
        }
      }
      else if (HASHG && c.enc == SG_ENC_VALUES && !G.is_str) {
        // value-array int group column: decoded value -> dense code through the table-wide value
        // dictionary's open-addressing table (L2-resident); a value the table does not hold can
        // only come from a block staged after the table was built: the block is dropped
        const uint32_t stride = G.stride, vmask = G.vh_mask;
        const long long* __restrict__ vk = G.vh_keys;
        const uint32_t* __restrict__ vi = G.vh_ids;
        scan_values_i64(cx, c, nrec, [&](uint32_t idx0, const unsigned long long(&a)[VE], uint32_t nvalid) {
          uint32_t inc[VE];
#pragma unroll
          for (int k = 0; k < VE; k++) {
            inc[k] = 0u;
            if (k < nvalid) {
              const long long v = (long long)a[k];
              uint32_t h = vh_hash(v) & vmask, id;
              for (;;) {
                id = vi[h];
                if (id == 0xffffffffu || vk[h] == v) break;
                h = (h + 1u) & vmask;
              }
              if (id == 0xffffffffu) {
                cx.misc[1] = 1;
                id = 0u;
              }
              inc[k] = id == (uint32_t)G.alias ? 0u : (id + 1u) * stride;
            }
          }
          add_slots(slot, idx0, inc);
        });
      }
      pass_mark(pass_no++);
    }

    phase(2);
    // ---- time bucket (aggregate.go:146-183) ------------------------------------------
    // The slot word takes the code relative to the block's window (1..twin; see Plan).  A row outside
    // the planned axis — or outside the window, which the exact extents rule out — is counted in
    // SC_TIME_OVERFLOW and fails the query on the host.
    const bool time_pass = time_col >= 0 && !(ptmp[4 * (nfilters + ngroups)] & 2u);  // (else read in the code pass)
    if (time_pass) {
      const DevCol c = colcache[nfilters + ngroups];
      const SlotT tok = (SlotT)time_ok;
      const long long tb64 = tbk, tf = tfirst;
      const uint32_t tr = tradix, ts = tstride;
      // every populated row of the block in ONE time bucket (exact extents): the column is not read
      const bool all_rows = c.enc == SG_ENC_VALUES || (c.enc == SG_ENC_BUCKET && (c.flags & COL_FULL));
      uint32_t cconst = 0;
      if (all_rows && !(c.flags & COL_IS_STR) && (c.flags & COL_STATS)) {
        const uint32_t clo = time_code(c.vmin, tb64, tf, tr);
        if (clo != 0u && clo == time_code(c.vmax, tb64, tf, tr)) cconst = clo;
      }
      if (cconst) {
        const uint32_t nval = c.enc == SG_ENC_VALUES ? (c.nitems < nrec ? c.nitems : nrec) : nrec;
        const uint32_t w = rel_of(cconst) * ts + time_ok;
        if (sizeof(SlotT) < 4) {
          const uint32_t per = 16u / (uint32_t)sizeof(SlotT);
          uint32_t rep = w;
          if (sizeof(SlotT) == 1) rep = w * 0x01010101u;
          if (sizeof(SlotT) == 2) rep = w * 0x00010001u;
          uint4* s4 = reinterpret_cast<uint4*>(slot);
          const uint32_t nfull = nval / per;
          for (uint32_t i = cx.tid; i < nfull; i += THREADS) {
            uint4 q = s4[i];
            q.x += rep;
            q.y += rep;
            q.z += rep;
            q.w += rep;
            s4[i] = q;
          }
          for (uint32_t r = nfull * per + cx.tid; r < nval; r += THREADS) slot[r] = (SlotT)(slot[r] + w);
        } else {
          for (uint32_t r = cx.tid; r < nval; r += THREADS) slot[r] = (SlotT)(slot[r] + w);
        }
        // (the pass list built at block start leaves this pass out: same test there)
        __syncthreads();
      } else if (c.enc == SG_ENC_BUCKET && !(c.flags & COL_IS_STR)) {
        uint32_t* pay = c.nbins <= SMEM_BINS ? cx.binpay_s : gbinpay;
        for (uint32_t b = cx.tid; b < c.nbins; b += THREADS) pay[b] = rel_of(time_code(c.bin_values[b], tb64, tf, tr));
        __syncthreads();
        scan_bucket<uint32_t>(
            cx, c, nrec, [&](uint32_t bin) { return pay[bin]; },
            [&](uint32_t row, uint32_t cur) {
              if (cur)
                slot_add(slot, slot_s, row, cur * ts + (uint32_t)tok);
              else
                gred_add(g_scalars + SC_TIME_OVERFLOW, 1ull);
            });
      } else if (c.enc == SG_ENC_VALUES && !(c.flags & COL_IS_STR)) {
        const bool stats = (c.flags & COL_STATS) != 0;
        const unsigned long long tmagic_p = PP->time_magic;
        const uint32_t magic_s = smem_u32(const_cast<uint32_t*>(cx.misc) + 8);
        if (cx.tid == 0) *reinterpret_cast<volatile unsigned long long*>(cx.misc + 8) = tmagic_p;
        __syncthreads();
        if (stats && c.vmin >= 0 && c.vmax <= 0xffffffffll && tmagic_p != 0ull && tf >= 0) {
          // 32-bit scan; v / bucket by multiply-high (exact for v < 2^32, see div_magic)
          scan_values_u32(cx, c, nrec, [&](uint32_t idx0, const uint32_t(&a)[VE], uint32_t nvalid) {
            uint32_t inc[VE];
            const unsigned long long tmagic = lds_u64(magic_s);
#pragma unroll
            for (int k = 0; k < VE; k++) {
              inc[k] = 0u;
              if (k < nvalid) {
                const long long q = (long long)div_magic(a[k], tmagic) - tf;
                const uint32_t code = (q < 0 || q >= (long long)(tr - 1u)) ? 0u : (uint32_t)q + 1u;
                const uint32_t rc = rel_of(code);
                if (rc)
                  inc[k] = rc * ts + time_ok;
                else
                  gred_add(g_scalars + SC_TIME_OVERFLOW, 1ull);
              }
            }
            add_slots(slot, idx0, inc);
          });
        } else {
          scan_values_i64(cx, c, nrec, [&](uint32_t idx0, const unsigned long long(&a)[VE], uint32_t nvalid) {
            uint32_t inc[VE];
#pragma unroll
            for (int k = 0; k < VE; k++) {
              inc[k] = 0u;
              if (k < nvalid) {
                const uint32_t rc = rel_of(time_code((long long)a[k], tb64, tf, tr));
                if (rc)
                  inc[k] = rc * ts + time_ok;
                else
                  gred_add(g_scalars + SC_TIME_OVERFLOW, 1ull);
              }
            }
            add_slots(slot, idx0, inc);
          });
        }
      }
    }
    __syncthreads();
    if (time_pass) pass_mark(pass_no++);

    // ---- weights carried over the block's rows without the weight column (see carry_weight); the group passes
    // above wrote every row, including rows that already failed a filter, so each row holds its own digit.
    // (count_in_group needs COL_FULL on its one group column, so it never meets a block that carries.)
    if (PP->wcarry && weight_needs_carry(colcache[nfilters + ngroups - 1], nrec)) {
      const KGroup& WG = PP->groups[ngroups - 1];
      carry_weight<SlotT>(slot, nrec, gmask, WG.stride, WG.radix, cx.binpay_s);
    }

    // ---- hashed slot space (LaunchParams::hkeys): code -> index of an open-addressing table in global memory.
    // Only rows that passed every filter (and carry a time code in time mode) take a slot.  The reference keys a Go
    // map with the row's key bytes (aggregate.go:186-203); this is that map, shared by all blocks.
    if (sizeof(SlotT) == 4 && lp.hkeys != nullptr) {
      uint32_t* const hk = lp.hkeys;
      const uint32_t hmask = lp.hmask;
      const uint32_t* const hids = lp.hids;
      for (uint32_t r = cx.tid; r < nrec; r += THREADS) {
        const uint32_t s = (uint32_t)slot[r];
        if ((s >> gbits) != pass_target) continue;
        const uint32_t key = (s & gmask) + 1u;
        uint32_t idx = slot_hash(key) & hmask, probes = 0;
        if (hids != nullptr) {
          // sparse aggregation launch: the table is complete and read-only; the accumulators are indexed by id
          for (;;) {
            const uint32_t k = __ldg(hk + idx);
            if (k == key) {
              idx = __ldg(hids + idx);
              break;
            }
            if (k == 0u || ++probes > hmask) {  // not discovered: the host fails the query (SC_SPARSE_MISSING)
              gred_add(g_scalars + SC_SPARSE_MISSING, 1ull);
              idx = 0u;
              break;
            }
            idx = (idx + 1u) & hmask;
          }
        } else {
          for (;;) {
            const uint32_t old = atomicCAS(hk + idx, 0u, key);
            if (old == 0u || old == key) break;
            idx = (idx + 1u) & hmask;
            if (++probes > hmask) {  // table full: the host fails the query (SC_TABLE_FULL)
              gred_add(g_scalars + SC_TABLE_FULL, 1ull);
              idx = 0u;
              break;
            }
          }
        }
        slot[r] = (SlotT)((s & ~gmask) | idx);
      }
      __syncthreads();
      if (lp.hdisc) continue;  // discovery launch: the table is all it fills
    }

    phase(3);
    // ---- Count / Samples (aggregate.go:202-203), MatchedCount (:117), aggregations
    // (:246-261).  The count is taken inside the first aggregation pass when that column
    // is a value array covering every row; otherwise in its own pass over the slot words.
    unsigned long long my_matched = 0;
    // MatchedCount differs from the sum of the group counts only in time mode (rows lacking
    // the time column are matched but not counted, aggregate.go:117,146-154)
    const bool count_matched = time_col >= 0;
    bool counted = false;
    uint32_t agg_mode_bits = 0;  // bit a: word0 of agg a counts NON-accepted rows (value arrays)

    const int agg_cand0 = nfilters + ngroups + (time_col >= 0 ? 1 : 0);  // candidate index of aggregation 0
    for (int ai = -1; ai < naggs; ai++) {
      if (ai >= 0 && !((aggmask >> ai) & 1u)) continue;  // another work item of this block computes it
      if (ai < 0) {
        // decide whether the first value-array aggregation (of this item) can carry the count
        bool fuse = false;
        const int ai0 = __ffs((int)(aggmask & ((naggs >= 32 ? 0xffffffffu : (1u << naggs)) - 1u))) - 1;
        if (ai0 >= 0) {
          const DevCol c0 = colcache[agg_cand0 + ai0];
          fuse = c0.enc == SG_ENC_VALUES && !(c0.flags & COL_IS_STR);
        }
        if (count_in_group) {  // the group pass added the bin sizes
          counted = true;
          continue;
        }
        if (fuse) continue;
        for (uint32_t r = cx.tid; r < nrec; r += THREADS) {
          const uint32_t s = (uint32_t)slot[r];
          const uint32_t hi = s >> gbits;
          if (count_matched && (hi & filt_mask) == filt_target) my_matched++;
          if (hi == pass_target) {
            const uint32_t g = s & gmask;
            if (ACC_SMEM)
              sred_add(smem_u32(cx.acc + g * gstride + lane_off), 1u);
            else
              gred_add(g_count + g + tb, 1ull);
          }
        }
        counted = true;
        continue;
      }
      const KAgg* __restrict__ KA = &PP->aggs[ai];
      const DevCol c = colcache[agg_cand0 + ai];
      if (c.flags & COL_IS_STR) continue;  // Populated != INT_VAL: no update
      const uint32_t w0 = 1u + 2u * (uint32_t)ai;  // word0 of this aggregation inside a slot's replicated words
      const bool do_count = !counted;              // only reachable for ai == 0 on a value array
      const uint32_t acc_s = smem_u32(cx.acc);
      const uint32_t gstride_b = gstride * 4u, R_b = R * 4u;
      const uint32_t cnt_s = acc_s + lane_off * 4u;            // + g*gstride_b: the slot's count word
      const uint32_t w0_s = acc_s + (w0 * R + lane_off) * 4u;  // + g*gstride_b: this aggregation's word0
      const uint32_t dummy_s = smem_u32(const_cast<uint32_t*>(cx.misc) + 64 + cx.lane);  // per-lane sink
      AggSlow AS;
      AS.info_min = KA->info_min;
      AS.info_max = KA->info_max;
      AS.reject_hi = KA->reject_hi;
      AS.nsub = KA->nsub;
      AS.multi = (int)KA->multi;
      AS.nvals_total = KA->nvals_total;
      AS.buckets = reinterpret_cast<unsigned long long*>(KA->buckets);
      AS.hcount = reinterpret_cast<unsigned long long*>(KA->hcount);
      AS.sum = reinterpret_cast<unsigned long long*>(KA->sum);
      AS.vmax = reinterpret_cast<long long*>(KA->vmax);
      AS.sub = KA->sub;
      AS.acc_w0_s = w0_s;
      AS.csum = ctot + 2u + 2u * (uint32_t)ai;
      AS.ctw = 1u + 2u * (uint32_t)naggs;
      const uint32_t hi_s = acc_s + (acc_rep + (uint32_t)ai) * 4u;  // + e * naggs * 4: this aggregation's high limb
      const uint32_t hi_stride_b = (uint32_t)naggs * 4u;
      AS.gstride_b = gstride_b;
      AS.acc_smem = ACC_SMEM ? 1 : 0;
      AS.tb = tb;
      // fast range: values the hot path takes — accepted (>= info_min, <= info_max <= reject_hi),
      // not above the table's max, and with a zero high limb
      const long long fmin = AS.info_min > 0 ? AS.info_min : 0;
      long long fmax = AS.info_max < 0xffffffffll ? AS.info_max : 0xffffffffll;
      if (AS.reject_hi < fmax) fmax = AS.reject_hi;
      const bool fast_any = ACC_SMEM && fmax >= fmin;
      const unsigned long long fspan = fast_any ? (unsigned long long)(fmax - fmin) : 0ull;
      // BasicHist with a 32-bit bucket size: bucket index in the hot path
      const bool hist32 = KA->nsub == 1 && KA->sub[0].bsize > 0 && KA->sub[0].bsize < 0x100000000ll &&
                          KA->sub[0].lo == AS.info_min && fast_any &&
                          (unsigned long long)fmax - (unsigned long long)AS.info_min < 0x100000000ull;
      const uint32_t bsize0 = (uint32_t)KA->sub[0].bsize, nvals0 = KA->sub[0].nvals;
      const uint32_t hdelta = (uint32_t)(fmin - AS.info_min);  // fast values: v - info_min = (v - fmin) + hdelta
      unsigned long long* const bkt = AS.buckets;
      const uint32_t nvt = AS.nvals_total;
      const int nsub = AS.nsub;

      // Hot path (ACC_SMEM).  A row that did not pass, or whose value is outside the fast
      // range, is steered to the TRASH slot (an extra accumulator row nobody reads) so that the
      // shared atomics run unconditionally: no branch per row.  Carries out of the low limb and
      // values that need the complete rule are collected in per-lane bit masks and handled
      // after the tile.
      const uint32_t trash = lslots;
      const uint32_t passbits = pass_target << gbits;
      const uint32_t fmin32 = (uint32_t)fmin, fspan32 = (uint32_t)fspan;
      // no carry can leave a low limb inside one block when every hot-path value is below
      // 2^32 / (rows one replica can receive per block): then the adds need no return value
      const bool nocarry = fast_any && (unsigned long long)fmax * (unsigned long long)(SG_BLOCK_ROWS / R) * lp.fold_every < 0x100000000ull;
      // one bucket increment of local slot e (may be TRASH): into the shared-memory histogram cache when
      // the slot's row lives there, else a 64-bit reduction to L2
      const uint32_t hoff = KA->hrow_off;
      const uint32_t hrows = (hist32 && hoff != HROW_NONE) ? hist_rows : 0u;
      const uint32_t hcache_s = hist_s + hoff * 4u, hrw_b = hrw * 4u;
      unsigned long long* const bkt_w = bkt + (size_t)tb * nvt;  // the window's first row of bucket counters
      auto hist_add = [&](uint32_t e, uint32_t b) {
        if (e < hrows)
          sred_add(hcache_s + e * hrw_b + b * 4u, 1u);
        else if (e != trash)
          gred_add(bkt_w + ((size_t)e * nvt + b), 1ull);
      };

      // one populated value of a row whose slot word is s (bucket columns: row order is scattered)
      auto accept_one = [&](uint32_t s, long long v) {
        const uint32_t e = min(s ^ passbits, trash);
        if (e == trash) return;
        if (ACC_SMEM) {
          const uint32_t vlo = (uint32_t)(unsigned long long)v, vhi = (uint32_t)((unsigned long long)v >> 32);
          const bool fr = fast_any && vhi == 0u && (vlo - fmin32) <= fspan32;
          if (fr) {
            const uint32_t w = w0_s + e * gstride_b;
            sred_add(w, 1u);
            const uint32_t old = satom_add(w + R_b, vlo);
            if (old > ~vlo) sred_add(hi_s + e * hi_stride_b, 1u);
            if (nsub > 0) {
              if (hist32) {
                uint32_t b = (vlo - fmin32 + hdelta) / bsize0;
                if (b >= nvals0) b = nvals0 - 1;
                hist_add(e, b);
              } else {
                hist_bucket_general(&AS, e, v);
              }
            }
            return;
          }
        }
        agg_slow(&AS, e, v, 1);
      };

      if (c.enc == SG_ENC_BUCKET && (c.flags & COL_CODES)) {
        // per-row codes: the rows in order, each with its bin's value
        const int64_t* __restrict__ bv = c.bin_values;
        for (uint32_t idx0 = (uint32_t)cx.tid * 16u; idx0 < nrec; idx0 += THREADS * 16u) {
          const uint4 q = __ldg(reinterpret_cast<const uint4*>(c.codes + idx0));
          const uint32_t cw[4] = {q.x, q.y, q.z, q.w};
          uint32_t sw[VE];
          load_slots(slot, idx0, sw);
#pragma unroll
          for (int k = 0; k < 16; k++) {
            const uint32_t code = (cw[k >> 2] >> (8 * (k & 3))) & 0xffu;
            if (code != 0xffu) accept_one(sw[k], bv[code]);
          }
        }
        __syncthreads();
      } else if (c.enc == SG_ENC_BUCKET) {
        scan_bucket<long long>(
            cx, c, nrec, [&](uint32_t bin) { return (long long)c.bin_values[bin]; },
            [&](uint32_t row, long long curv) { accept_one((uint32_t)slot[row], curv); });
      } else if (c.enc == SG_ENC_VALUES && ACC_SMEM && fast_any && (c.flags & COL_STATS) && c.vmin >= 0 &&
                 c.vmax <= 0xffffffffll) {
        // ---- value array whose decoded values provably fit 32 bits (staging statistics) ----
        agg_mode_bits |= 1u << ai;
        // every value inside the fast range and no carry possible: no per-row checks at all
        const bool allfast = nocarry && c.vmin >= fmin && c.vmax <= fmax;
        const uint32_t magic_s = smem_u32(const_cast<uint32_t*>(cx.misc) + 8);  // misc[8..9]: this aggregation's division magic
        if (cx.tid == 0) *reinterpret_cast<volatile unsigned long long*>(cx.misc + 8) = KA->sub[0].magic;
        __syncthreads();
        auto tile32 = [&](uint32_t idx0, const uint32_t(&a)[VE], uint32_t nvalid, auto do_count_tag, auto allfast_tag,
                          auto nofilt_tag) {
          constexpr bool DO_COUNT = decltype(do_count_tag)::value;
          constexpr bool ALLFAST = decltype(allfast_tag)::value;
          // NOFILT: no filters, no time column, at most one group column — every slot word IS a valid
          // slot (stored from the per-bin payload), so the pass test and the clamp to TRASH drop out
          constexpr bool NOFILT = decltype(nofilt_tag)::value;
          uint32_t sw[VE];
          load_slots(slot, idx0, sw);
          const unsigned long long magic0 = nsub > 0 ? lds_u64(magic_s) : 0ull;
          if (nvalid < VE) {
#pragma unroll
            for (int k = 0; k < VE; k++)
              if (k >= nvalid) sw[k] = NOFILT ? trash : ~passbits;  // rows past len(Values): handled by the tail loop below
          }
          if (DO_COUNT && count_matched) {
#pragma unroll
            for (int k = 0; k < VE; k++)
              if (k < (int)nvalid && ((sw[k] >> gbits) & filt_mask) == filt_target) my_matched++;
          }
          uint32_t cmask = 0, slow_any = 0;
#pragma unroll
          for (int k = 0; k < VE; k++) {
            const uint32_t e = NOFILT ? sw[k] : min(sw[k] ^ passbits, trash);  // passing row: its slot, else trash
            if (DO_COUNT) sred_add(cnt_s + e * gstride_b, 1u);
            if (ALLFAST) {
              sred_add(w0_s + R_b + e * gstride_b, a[k]);
            } else {
              const bool fr = (a[k] - fmin32) <= fspan32;
              const uint32_t e2 = fr ? e : trash;
              slow_any |= e ^ e2;
              const uint32_t old = satom_add(w0_s + R_b + e2 * gstride_b, a[k]);
              cmask |= (old > ~a[k]) ? (1u << k) : 0u;
            }
          }
          if (!ALLFAST && (cmask | slow_any)) {  // rare
#pragma unroll
            for (int k = 0; k < VE; k++) {
              const uint32_t e = NOFILT ? sw[k] : min(sw[k] ^ passbits, trash);
              const bool fr = (a[k] - fmin32) <= fspan32;
              if ((cmask >> k) & 1u) sred_add(hi_s + (fr ? e : trash) * hi_stride_b, 1u);  // carry
              if (!fr && e != trash) agg_slow(&AS, e, (long long)a[k], 0);
            }
          }
          if (nsub > 0 && hist32) {
            // Straight-line bucket step: x / BucketSize by multiply-high (BucketSize 1 has no magic: b = x), then
            // ONE predicated shared reduction (the slot's row is in the cache) and, unless every row is, ONE
            // predicated 64-bit reduction to L2.  (With `magic ? mulhi : x / bsize` and if / else-if the compiler
            // kept a software division and five branches per row: the loop was branch- and fetch-bound.)
            const bool unit = bsize0 == 1u;
            const uint32_t nv1 = nvals0 - 1u;
            if (hrows >= lslots) {
#pragma unroll
              for (int k = 0; k < VE; k++) {
                const uint32_t e = NOFILT ? sw[k] : min(sw[k] ^ passbits, trash);
                const bool fr = ALLFAST || (a[k] - fmin32) <= fspan32;
                const uint32_t e2 = fr ? e : trash;
                const uint32_t x = a[k] - fmin32 + hdelta;
                const uint32_t q = div_magic(x, magic0);
                const uint32_t b = min(unit ? x : q, nv1);  // outlier: clamped into the last slot (hist_basic.go:134-137)
                sred_inc_if(e2 < hrows ? 1u : 0u, hcache_s + e2 * hrw_b + b * 4u);
              }
            } else {
#pragma unroll
              for (int k = 0; k < VE; k++) {
                const uint32_t e = NOFILT ? sw[k] : min(sw[k] ^ passbits, trash);
                const bool fr = ALLFAST || (a[k] - fmin32) <= fspan32;
                const uint32_t e2 = fr ? e : trash;
                const uint32_t x = a[k] - fmin32 + hdelta;
                const uint32_t q = div_magic(x, magic0);
                const uint32_t b = min(unit ? x : q, nv1);
                sred_inc_if(e2 < hrows ? 1u : 0u, hcache_s + e2 * hrw_b + b * 4u);
                gred_inc_if((e2 >= hrows && e2 != trash) ? 1u : 0u, bkt_w + ((size_t)e2 * nvt + b));
              }
            }
          } else if (nsub > 0) {
#pragma unroll
            for (int k = 0; k < VE; k++) {
              const uint32_t e = NOFILT ? sw[k] : min(sw[k] ^ passbits, trash);
              const bool fr = ALLFAST || (a[k] - fmin32) <= fspan32;
              const uint32_t e2 = fr ? e : trash;
              if (e2 != trash) hist_bucket_general(&AS, e2, (long long)a[k]);
            }
          }
        };
        auto run32 = [&](auto dc, auto af, auto nf) {
          scan_values_u32(cx, c, nrec, [&](uint32_t idx0, const uint32_t(&a)[VE], uint32_t nvalid) {
            tile32(idx0, a, nvalid, dc, af, nf);
          });
        };
        const bool nofilt = allfast && nfilters == 0 && time_col < 0 && ngroups <= 1;
        if (do_count) {
          if (nofilt)
            run32(std::true_type(), std::true_type(), std::true_type());
          else if (allfast)
            run32(std::true_type(), std::true_type(), std::false_type());
          else
            run32(std::true_type(), std::false_type(), std::false_type());
        } else {
          if (nofilt)
            run32(std::false_type(), std::true_type(), std::true_type());
          else if (allfast)
            run32(std::false_type(), std::true_type(), std::false_type());
          else
            run32(std::false_type(), std::false_type(), std::false_type());
        }
        // rows past len(Values) are unpopulated for this column (Q6): they still count
        const uint32_t nv = c.nitems < nrec ? c.nitems : nrec;
        for (uint32_t r = nv + cx.tid; r < nrec; r += THREADS) {
          const uint32_t s = (uint32_t)slot[r];
          const uint32_t hi = s >> gbits;
          if (do_count && count_matched && (hi & filt_mask) == filt_target) my_matched++;
          if (hi == pass_target) {
            const uint32_t g = s & gmask;
            if (do_count) sred_add(cnt_s + g * gstride_b, 1u);
            sred_add(w0_s + g * gstride_b, 1u);
          }
        }
        counted = true;
      } else if (c.enc == SG_ENC_VALUES && !ACC_SMEM && (c.flags & COL_STATS) && c.vmin >= 0 &&
                 c.vmax <= 0xffffffffll) {
        // ---- high-cardinality plan (accumulators in L2/HBM), 32-bit values: one RED per row for the
        // count, one (two unless the plan proved hist Count == Count) per aggregation
        const long long amin = AS.info_min, amax = AS.reject_hi < AS.info_max ? AS.reject_hi : AS.info_max;
        const bool allin = c.vmin >= amin && c.vmax <= amax;  // every value accepted and not above info_max
        const bool skip_hc = (KA->_pad & 1u) != 0;             // plan: hist Count == Count for this aggregation
        unsigned long long* const g_hc = AS.hcount;
        unsigned long long* const g_sum = AS.sum;
        auto tile32g = [&](uint32_t idx0, const uint32_t(&a)[VE], uint32_t nvalid) {
          uint32_t sw[VE];
          load_slots(slot, idx0, sw);
#pragma unroll
          for (int k = 0; k < VE; k++) {
            if (k >= nvalid) continue;
            const uint32_t e = min(sw[k] ^ passbits, trash);
            if (do_count && count_matched && ((sw[k] >> gbits) & filt_mask) == filt_target) my_matched++;
            if (e == trash) continue;
            if (do_count) gred_add(g_count + e + tb, 1ull);
            const long long v = (long long)a[k];
            if (allin || (v >= amin && v <= amax)) {
              if (!skip_hc) gred_add(g_hc + e + tb, 1ull);
              gred_add(g_sum + e + tb, (unsigned long long)a[k]);
              if (nsub > 0) hist_bucket_general(&AS, e, v);
            } else {
              agg_slow(&AS, e, v, 0);
            }
          }
        };
        scan_values_u32(cx, c, nrec, tile32g, sizeof(SlotT) == 4 ? reinterpret_cast<const uint32_t*>(slot) : nullptr);
        const uint32_t nv = c.nitems < nrec ? c.nitems : nrec;
        for (uint32_t r = nv + cx.tid; r < nrec; r += THREADS) {
          const uint32_t s = (uint32_t)slot[r];
          const uint32_t hi = s >> gbits;
          if (do_count && count_matched && (hi & filt_mask) == filt_target) my_matched++;
          if (hi == pass_target && do_count) gred_add(g_count + (s & gmask) + tb, 1ull);
        }
        counted = true;
      } else if (c.enc == SG_ENC_VALUES) {
        agg_mode_bits |= 1u << ai;
        auto tile = [&](uint32_t idx0, const unsigned long long(&a)[VE], uint32_t nvalid, auto do_count_tag,
                        auto nocarry_tag) {
          constexpr bool DO_COUNT = decltype(do_count_tag)::value;
          constexpr bool NOCARRY = decltype(nocarry_tag)::value;
          uint32_t sw[VE];
          load_slots(slot, idx0, sw);
          if (nvalid < VE) {
#pragma unroll
            for (int k = 0; k < VE; k++)
              // rows past len(Values), handled by the tail loop below, take a word that maps to trash and fails the
              // filters (~0 would not: it is the highest slot's passing word when the slot word fills 32 bits)
              if (k >= nvalid) sw[k] = ~passbits;
          }
          if (DO_COUNT && count_matched) {
#pragma unroll
            for (int k = 0; k < VE; k++)
              if (k < (int)nvalid && ((sw[k] >> gbits) & filt_mask) == filt_target) my_matched++;
          }
          if (ACC_SMEM && fast_any) {
            uint32_t cmask = 0, slow_any = 0;
#pragma unroll
            for (int k = 0; k < VE; k++) {
              const uint32_t e = min(sw[k] ^ passbits, trash);  // passing row: its slot, else trash
              if (DO_COUNT) sred_add(cnt_s + e * gstride_b, 1u);
              const uint32_t vlo = (uint32_t)a[k], vhi = (uint32_t)(a[k] >> 32);
              const bool fr = vhi == 0u && (vlo - fmin32) <= fspan32;
              const uint32_t e2 = fr ? e : trash;
              slow_any |= e ^ e2;  // non-zero: a passing row whose value needs the complete rule
              if (NOCARRY) {
                sred_add(w0_s + R_b + e2 * gstride_b, vlo);
              } else {
                const uint32_t old = satom_add(w0_s + R_b + e2 * gstride_b, vlo);
                cmask |= (old > ~vlo) ? (1u << k) : 0u;
              }
              if (hist32) {
                uint32_t b = (vlo - fmin32 + hdelta) / bsize0;
                if (b >= nvals0) b = nvals0 - 1;  // outlier: clamped into the last slot (hist_basic.go:134-137)
                hist_add(e2, b);
              }
            }
            if (cmask | slow_any) {  // rare
#pragma unroll
              for (int k = 0; k < VE; k++) {
                const uint32_t e = min(sw[k] ^ passbits, trash);
                const uint32_t vlo = (uint32_t)a[k], vhi = (uint32_t)(a[k] >> 32);
                const bool fr = vhi == 0u && (vlo - fmin32) <= fspan32;
                if ((cmask >> k) & 1u) sred_add(hi_s + (fr ? e : trash) * hi_stride_b, 1u);  // carry
                if (!fr && e != trash) agg_slow(&AS, e, (long long)a[k], 0);
              }
            }
            if (nsub > 0 && !hist32) {  // MultiHist / wide buckets: per-row general path
#pragma unroll
              for (int k = 0; k < VE; k++) {
                const uint32_t e = min(sw[k] ^ passbits, trash);
                const uint32_t vlo = (uint32_t)a[k], vhi = (uint32_t)(a[k] >> 32);
                if (e != trash && fast_any && vhi == 0u && (vlo - fmin32) <= fspan32)
                  hist_bucket_general(&AS, e, (long long)a[k]);
              }
            }
          } else {
#pragma unroll
            for (int k = 0; k < VE; k++) {
              const uint32_t e = min(sw[k] ^ passbits, trash);
              if (e != trash) {
                if (DO_COUNT) {
                  if (ACC_SMEM)
                    sred_add(cnt_s + e * gstride_b, 1u);
                  else
                    gred_add(g_count + e + tb, 1ull);
                }
                agg_slow(&AS, e, (long long)a[k], 0);
              }
            }
          }
        };
        auto run = [&](auto dc, auto nc) {
          scan_values_i64(cx, c, nrec, [&](uint32_t idx0, const unsigned long long(&a)[VE], uint32_t nvalid) {
            tile(idx0, a, nvalid, dc, nc);
          });
        };
        if (do_count) {
          if (nocarry)
            run(std::true_type(), std::true_type());
          else
            run(std::true_type(), std::false_type());
        } else {
          if (nocarry)
            run(std::false_type(), std::true_type());
          else
            run(std::false_type(), std::false_type());
        }
        // rows past len(Values) are unpopulated for this column (Q6): they still count
        const uint32_t nv = c.nitems < nrec ? c.nitems : nrec;
        for (uint32_t r = nv + cx.tid; r < nrec; r += THREADS) {
          const uint32_t s = (uint32_t)slot[r];
          const uint32_t hi = s >> gbits;
          if (do_count && count_matched && (hi & filt_mask) == filt_target) my_matched++;
          if (hi == pass_target) {
            const uint32_t g = s & gmask;
            if (do_count) {
              if (ACC_SMEM)
                sred_add(cnt_s + g * gstride_b, 1u);
              else
                gred_add(g_count + g + tb, 1ull);
            }
            if (ACC_SMEM) sred_add(w0_s + g * gstride_b, 1u);
          }
        }
        counted = true;
      }
      if (ai >= 0) pass_mark(pass_no++);
    }
    __syncthreads();

    phase(4);
    cx.tmark(15);
    // ---- end of block: publish or discard ------------------------------------------------
    const bool broken = cx.misc[1] != 0;
    if (broken) {
      if (cx.tid == 0) {
        PP->block_status[bid] = 1;
        gred_add(g_scalars + SC_BROKEN, 1ull);
      }
    } else {
      if (owner) matched += my_matched;
    }
    if (ACC_SMEM) {
      // the replicated accumulators are folded at the top of a later iteration (see there): remember
      // what that fold must know about the blocks it covers
      fstate = ((fstate & 0xffu) + 1u) | (broken || (fstate & 0x100u) ? 0x100u : 0u) |
               (imask != 0x8000ffffu ? 0x200u : 0u) | (owner ? 0x400u : 0u) | (agg_mode_bits << 16);
      // a moving slot window: fold before the next block (the runtime launches such plans with fold_every 1)
      if (twin + 1u < tradix) fstate |= 0x200u;
      fold_tb = tb;
    }
    phase(5);
  }

  if (dbg && cx.tid == 0) {
    for (int i = 0; i < 7; i++) dbg[i] = tacc[i];
    dbg[7] = cx.t_tma;
    dbg[8] = cx.t_lb;
    for (int i = 9; i < 16; i++) dbg[i] = tacc[i];  // per column pass (or the -DSG_FINE_TIMING marks)
  }
  if (hist_rows) hist_flush();
  if (ACC_SMEM) {
    __syncthreads();
    const uint32_t tw = 1u + 2u * (uint32_t)naggs;
    for (uint32_t i = cx.tid; i < ctot_n; i += THREADS) {
      const unsigned long long v = ctot[i];
      if (!v) continue;
      const uint32_t g = i / tw, k = i - g * tw;
      if (k == 0) {
        gred_add(g_count + g, v);
      } else {
        const KAgg* KA = &PP->aggs[(k - 1u) >> 1];
        gred_add(reinterpret_cast<unsigned long long*>(((k - 1u) & 1u) ? KA->sum : KA->hcount) + g, v);
      }
    }
  }
  // MatchedCount
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) matched += __shfl_xor_sync(FULL, matched, d);
  if (cx.lane == 0 && matched) gred_add(g_scalars + SC_MATCHED, matched);
}

// ---------------------------------------------------------------------------
// staging-time statistics: exact min / max of the decoded values of value-array int
// columns (one CTA per column of a block).  They let the scan kernel pick 32-bit
// arithmetic and drop per-row range checks when a column provably needs neither.
// Bucket columns get COL_FULL and, when the host reserved room for them, their per-row codes
// (COL_CODES) from the same walk.
// ---------------------------------------------------------------------------
constexpr uint32_t STATS_DYN_SMEM = SG_BLOCK_ROWS;  // the per-row codes of one block, built in shared memory
__global__ void __launch_bounds__(THREADS, 1) stats_kernel(DevCol* cols, const DevBlock* blocks,
                                                           const uint32_t* items, const unsigned long long* codes,
                                                           uint32_t nitems, uint32_t ncolslots) {
  __shared__ __align__(16) unsigned char smem_s[FIXED_SMEM];
  __shared__ long long red_min[NWARPS], red_max[NWARPS];
  __shared__ uint32_t rowbits[HEAD_WORDS];  // bucket columns: one bit per listed row
  extern __shared__ uint4 codes_s4[];       // [STATS_DYN_SMEM / 16]
  uint8_t* const codes_s = reinterpret_cast<uint8_t*>(codes_s4);
  Ctx cx;
  cx.tid = threadIdx.x;
  cx.lane = threadIdx.x & 31;
  cx.warp = threadIdx.x >> 5;
  cx.epoch = 0;
  cx.headbits = reinterpret_cast<uint32_t*>(smem_s + OFF_HEADBITS);
  cx.headprefix = reinterpret_cast<uint16_t*>(smem_s + OFF_HEADPREFIX);
  cx.binpay_s = reinterpret_cast<uint32_t*>(smem_s + OFF_BINPAY);
  cx.pubA = reinterpret_cast<volatile unsigned long long*>(smem_s + OFF_PUBA);
  cx.pubB = reinterpret_cast<volatile unsigned long long*>(smem_s + OFF_PUBB);
  cx.misc = reinterpret_cast<volatile uint32_t*>(smem_s + OFF_MISC);
  cx.acc = nullptr;
  cx.tmaps = nullptr;
  cx.stage_bytes = 0;
  cx.zero = 0;
  cx.buf0 = cx.buf1 = cx.mbar0 = cx.mbar1 = cx.par0 = cx.par1 = 0;
  cx.plist = nullptr;
  cx.timing = false;
  cx.t_tma = cx.t_lb = 0;
  cx.npass = cx.pass_idx = 0;
  cx.pref_idx = 0xffffffffu;
  for (uint32_t i = cx.tid; i < MAX_TILES; i += THREADS) {
    cx.pubA[i] = 0;
    cx.pubB[i] = 0;
  }
  __syncthreads();
  for (uint32_t it = blockIdx.x; it < nitems; it += gridDim.x) {
    const uint32_t ci = items[it];
    const DevCol c = cols[ci];
    const uint32_t nrec = blocks[ci / ncolslots].num_records;
    if (c.enc == SG_ENC_BUCKET) {
      // COL_FULL: the bins list every row of [0, NumRecords) exactly once — as many entries as rows,
      // every decoded id in range, no id twice.  Then no row is unpopulated for this column and a
      // filter may reason about the complement of a set of bins.
      // COL_CODES (the host reserved `codes[it]`, nbins <= 255): the bin index of every row, 0xFF for an
      // unlisted one.  Kept only when the walk found no row listed twice, no row >= NumRecords, no gap
      // >= 65,536 and no bad bin index; otherwise the column stays with its ids alone.
      uint8_t* const dst = reinterpret_cast<uint8_t*>(codes[it]);
      if (c.nitems != nrec && !dst) continue;
      for (uint32_t i = cx.tid; i < HEAD_WORDS; i += THREADS) rowbits[i] = 0;
      if (dst)
        for (uint32_t i = cx.tid; i < SG_BLOCK_ROWS / 16; i += THREADS) codes_s4[i] = make_uint4(FULL, FULL, FULL, FULL);
      if (cx.tid == 0) {
        cx.misc[1] = 0;
        cx.misc[2] = 0;  // a row listed twice
      }
      __syncthreads();
      scan_bucket<uint32_t>(
          cx, c, nrec, [&](uint32_t bin) { return bin; },
          [&](uint32_t row, uint32_t bin) {
            const uint32_t bit = 1u << (row & 31);
            if (atomicOr(&rowbits[row >> 5], bit) & bit) cx.misc[2] = 1;
            if (dst) codes_s[row] = (uint8_t)bin;
          });
      uint32_t pc = 0;
      for (uint32_t i = cx.tid; i < HEAD_WORDS; i += THREADS) pc += (uint32_t)__popc(rowbits[i]);
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) pc += __shfl_xor_sync(FULL, pc, d);
      if (cx.lane == 0) red_min[cx.warp] = (long long)pc;
      __syncthreads();
      const bool clean = cx.misc[1] == 0 && cx.misc[2] == 0;
      if (dst && clean) {
        uint4* const d4 = reinterpret_cast<uint4*>(dst);
        for (uint32_t i = cx.tid; i < (nrec + 15u) / 16u; i += THREADS) d4[i] = codes_s4[i];
      }
      if (cx.tid == 0) {
        long long tot = 0;
        for (int w = 0; w < NWARPS; w++) tot += red_min[w];
        uint32_t fl = c.flags;
        if (c.nitems == nrec && tot == (long long)nrec && cx.misc[1] == 0) fl |= COL_FULL;
        if (dst && clean) {
          fl = (fl | COL_CODES) & ~COL_TMA;
          cols[ci].codes = dst;
        }
        cols[ci].flags = fl;
      }
      __syncthreads();
      continue;
    }
    long long mn = 0x7fffffffffffffffll, mx = -0x7fffffffffffffffll - 1;
    scan_values_i64(cx, c, nrec, [&](uint32_t idx0, const unsigned long long(&a)[VE], uint32_t nvalid) {
#pragma unroll
      for (int k = 0; k < VE; k++)
        if (k < nvalid) {
          const long long v = (long long)a[k];
          mn = v < mn ? v : mn;
          mx = v > mx ? v : mx;
        }
    });
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      const long long omn = __shfl_xor_sync(FULL, mn, d), omx = __shfl_xor_sync(FULL, mx, d);
      mn = omn < mn ? omn : mn;
      mx = omx > mx ? omx : mx;
    }
    if (cx.lane == 0) {
      red_min[cx.warp] = mn;
      red_max[cx.warp] = mx;
    }
    __syncthreads();
    if (cx.tid == 0) {
      for (int w = 1; w < NWARPS; w++) {
        mn = red_min[w] < mn ? red_min[w] : mn;
        mx = red_max[w] > mx ? red_max[w] : mx;
      }
      cols[ci].vmin = mn;
      cols[ci].vmax = mx;
      cols[ci].flags = c.flags | COL_STATS;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// distinct values of value-array int columns (group-by on such a column needs a table-wide
// value dictionary; built on demand, once per staged block)
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS, 1) distinct_kernel(const DevCol* cols, const DevBlock* blocks,
                                                              const uint32_t* items, uint32_t nitems, uint32_t ncolslots,
                                                              long long* keys, uint32_t cap_mask, unsigned int* counters) {
  __shared__ __align__(16) unsigned char smem_s[FIXED_SMEM];
  Ctx cx;
  cx.tid = threadIdx.x;
  cx.lane = threadIdx.x & 31;
  cx.warp = threadIdx.x >> 5;
  cx.epoch = 0;
  cx.headbits = reinterpret_cast<uint32_t*>(smem_s + OFF_HEADBITS);
  cx.headprefix = reinterpret_cast<uint16_t*>(smem_s + OFF_HEADPREFIX);
  cx.binpay_s = reinterpret_cast<uint32_t*>(smem_s + OFF_BINPAY);
  cx.pubA = reinterpret_cast<volatile unsigned long long*>(smem_s + OFF_PUBA);
  cx.pubB = reinterpret_cast<volatile unsigned long long*>(smem_s + OFF_PUBB);
  cx.misc = reinterpret_cast<volatile uint32_t*>(smem_s + OFF_MISC);
  cx.acc = nullptr;
  cx.tmaps = nullptr;
  cx.stage_bytes = 0;
  cx.zero = 0;
  cx.buf0 = cx.buf1 = cx.mbar0 = cx.mbar1 = cx.par0 = cx.par1 = 0;
  cx.plist = nullptr;
  cx.timing = false;
  cx.t_tma = cx.t_lb = 0;
  cx.npass = cx.pass_idx = 0;
  cx.pref_idx = 0xffffffffu;
  for (uint32_t i = cx.tid; i < MAX_TILES; i += THREADS) {
    cx.pubA[i] = 0;
    cx.pubB[i] = 0;
  }
  __syncthreads();
  const long long EMPTY = -0x7fffffffffffffffll - 1;
  const unsigned int limit = (cap_mask + 1u) / 2u;
  for (uint32_t it = blockIdx.x; it < nitems; it += gridDim.x) {
    const uint32_t ci = items[it];
    const DevCol c = cols[ci];
    const uint32_t nrec = blocks[ci / ncolslots].num_records;
    scan_values_i64(cx, c, nrec, [&](uint32_t idx0, const unsigned long long(&a)[VE], uint32_t nvalid) {
      long long prev = EMPTY;
#pragma unroll
      for (int k = 0; k < VE; k++)
        if (k < nvalid) {
          const long long v = (long long)a[k];
          if (v == prev) continue;  // runs of equal values are common in sorted / low-entropy columns
          prev = v;
          if (v == EMPTY) {
            counters[1] = 1u;
            continue;
          }
          if (counters[2]) continue;  // the set is full: the host reports the overflow
          uint32_t h = vh_hash(v) & cap_mask;
          for (;;) {
            const long long cur = keys[h];
            if (cur == v) break;
            if (cur == EMPTY) {
              const long long old = (long long)atomicCAS(reinterpret_cast<unsigned long long*>(keys + h),
                                                         (unsigned long long)EMPTY, (unsigned long long)v);
              if (old == EMPTY) {
                if (atomicAdd(&counters[0], 1u) + 1u > limit) counters[2] = 1u;
                break;
              }
              if (old == v) break;
            }
            h = (h + 1u) & cap_mask;
          }
        }
    });
  }
}

int launch_distinct(const DevCol* cols, const DevBlock* blocks, const uint32_t* items, uint32_t nitems, uint32_t ncolslots,
                    long long* keys, uint32_t cap_mask, unsigned int* counters, void* stream) {
  if (nitems == 0) return 0;
  int dev = 0, sms = 148;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const uint32_t grid = nitems < (uint32_t)sms * 2 ? nitems : (uint32_t)sms * 2;
  distinct_kernel<<<grid, THREADS, 0, (cudaStream_t)stream>>>(cols, blocks, items, nitems, ncolslots, keys, cap_mask, counters);
  return (int)cudaGetLastError();
}

int launch_stats(DevCol* cols, const DevBlock* blocks, const uint32_t* items, const unsigned long long* codes,
                 uint32_t nitems, uint32_t ncolslots, void* stream) {
  if (nitems == 0) return 0;
  int dev = 0, sms = 148;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const uint32_t grid = nitems < (uint32_t)sms * 2 ? nitems : (uint32_t)sms * 2;
  const cudaError_t e = cudaFuncSetAttribute(stats_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)STATS_DYN_SMEM);
  if (e != cudaSuccess) return (int)e;
  stats_kernel<<<grid, THREADS, STATS_DYN_SMEM, (cudaStream_t)stream>>>(cols, blocks, items, codes, nitems, ncolslots);
  return (int)cudaGetLastError();
}

template <typename SlotT, bool ACC_SMEM, bool HASHG = false>
static int launch_one(const LaunchParams& lp, int grid, cudaStream_t st) {
  auto k = scan_kernel<SlotT, ACC_SMEM, HASHG>;
  cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lp.smem_bytes);
  if (e != cudaSuccess) return (int)e;
  k<<<grid, THREADS, lp.smem_bytes, st>>>(lp);
  return (int)cudaGetLastError();
}

int launch_scan(const LaunchParams& lp, int grid, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  const bool acc_smem = lp.acc_smem != 0;
  const uint32_t sb = lp.slot_bytes;
  if (lp.hashg) {
    // the planner gives plans with a hashed group column 32-bit slot words and global accumulators
    if (sb != 4 || acc_smem) return (int)cudaErrorInvalidValue;
    return launch_one<uint32_t, false, true>(lp, grid, st);
  }
  if (sb == 1) return acc_smem ? launch_one<uint8_t, true>(lp, grid, st) : launch_one<uint8_t, false>(lp, grid, st);
  if (sb == 2) return acc_smem ? launch_one<uint16_t, true>(lp, grid, st) : launch_one<uint16_t, false>(lp, grid, st);
  return acc_smem ? launch_one<uint32_t, true>(lp, grid, st) : launch_one<uint32_t, false>(lp, grid, st);
}

}  // namespace SG_VNS
}  // namespace sg
