// sg_runtime.cu — host runtime of libsybilgpu.so: context, HBM-resident tables,
// query planning, kernel launches, NCCL merge, result finalisation, C ABI.
//
// Mirrors the host half of Table.LoadAndQueryRecords (src/lib/table_query.go:18-422):
//   block enumeration + zone-map skip   table_query.go:96-131, table_block_io.go:110-182
//   LoadBlockFromDir                    table_block_io.go:225-310   -> sg_table_add_block (staging)
//   per-block FilterAndAggRecords       aggregate.go:56-282         -> scan kernel (sg_kernels.cu)
//   CombineResults / SortResults        aggregate.go:414-467,497-525 -> device accumulators shared by
//                                        all blocks (+ NCCL all-reduce across GPUs) and build_result()
//   translate_group_by                  aggregate.go:284-324        -> render_key() over the global dictionary
#include <cuda.h>
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "sg_hist.h"
#include "sg_internal.h"

using namespace sg;

// ---------------------------------------------------------------------------
// NCCL, bound lazily so the library loads on machines without it
// ---------------------------------------------------------------------------
namespace {
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclUint8 = 1, ncclInt64 = 4, ncclUint64 = 5 };  // nccl.h ncclDataType_t
enum { ncclSum = 0, ncclMax = 2 };       // nccl.h ncclRedOp_t
struct NcclApi {
  void* lib = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool load() {
    if (lib) return true;
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (auto n : names) {
      lib = dlopen(n, RTLD_NOW | RTLD_GLOBAL);
      if (lib) break;
    }
    if (!lib) return false;
    GetUniqueId = (decltype(GetUniqueId))dlsym(lib, "ncclGetUniqueId");
    CommInitRank = (decltype(CommInitRank))dlsym(lib, "ncclCommInitRank");
    CommDestroy = (decltype(CommDestroy))dlsym(lib, "ncclCommDestroy");
    AllReduce = (decltype(AllReduce))dlsym(lib, "ncclAllReduce");
    AllGather = (decltype(AllGather))dlsym(lib, "ncclAllGather");
    GetErrorString = (decltype(GetErrorString))dlsym(lib, "ncclGetErrorString");
    return GetUniqueId && CommInitRank && CommDestroy && AllReduce && AllGather;
  }
};
NcclApi g_nccl;

// cuTensorMapEncodeTiled through the runtime's driver entry point query (no link against libcuda)
typedef CUresult (*TmapEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                 const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                 CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
TmapEncodeFn tmap_encode_fn() {
  static TmapEncodeFn fn = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess &&
        qr == cudaDriverEntryPointSuccess)
      fn = (TmapEncodeFn)p;
  }
  return fn;
}

constexpr size_t ARENA_CHUNK = (size_t)512 << 20;
constexpr size_t STAGE_BYTES = (size_t)64 << 20;
// the two builds of the kernel unit (sg_internal.h)
struct Variant {
  const char* name;
  int warps, ctas;
  uint32_t max_smem;  // dynamic shared memory of one CTA
  uint32_t (*fixed_smem)(uint32_t);
  int (*launch)(const LaunchParams&, int, void*);
};
static const Variant V16 = {"w16", 16, w16::scan_ctas_per_sm(), w16::scan_max_smem(), w16::scan_fixed_smem, w16::launch_scan};
static const Variant V8 = {"w8", 8, w8::scan_ctas_per_sm(), w8::scan_max_smem(), w8::scan_fixed_smem, w8::launch_scan};
constexpr int64_t MAX_SLOTS = (int64_t)1 << 26;
constexpr uint64_t MAX_CODE_SPACE = ((uint64_t)1 << 31) - 2;  // codes of a hashed slot space (key = code + 1 in 32 bits)
constexpr int64_t INT_DICT_CAP = (int64_t)1 << 22;

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) & ~(a - 1); }
}  // namespace

struct sg_ctx {
  int device = -1;
  bool has_device = false;
  int sm_count = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t copy_stream = nullptr;
  std::string err;
  std::mutex mu;
  ncclComm_t comm = nullptr;
  int rank = 0, nranks = 1;
  char devname[256] = {0};
  std::vector<std::pair<const char*, size_t>> pinned;  // sg_pinned_alloc ranges (DMA without a bounce copy)
  // query-lifetime device buffers are recycled: cudaMalloc/cudaFree per query cost milliseconds
  std::vector<std::pair<void*, size_t>> pool_free;
  std::unordered_map<void*, size_t> pool_live;
  // pinned host scratch for the per-query parameter uploads and the accumulator read-back: copies
  // from/to pageable memory are staged by the driver and block the caller
  char* hpin = nullptr;
  size_t hpin_cap = 0;
  char* scratch(size_t bytes) {
    if (bytes > hpin_cap) {
      if (hpin) cudaFreeHost(hpin);
      hpin = nullptr;
      hpin_cap = 0;
      size_t cap = std::max<size_t>(bytes * 2, (size_t)1 << 20);
      if (cudaHostAlloc((void**)&hpin, cap, cudaHostAllocDefault) != cudaSuccess) return nullptr;
      hpin_cap = cap;
    }
    return hpin;
  }
  // pinned buffers large results are read back into (and read from: no copy to pageable memory); recycled,
  // because cudaHostAlloc of tens of megabytes costs milliseconds
  std::vector<std::pair<char*, size_t>> pin_free;
  char* pin_get(size_t bytes, size_t* got) {
    {
      std::lock_guard<std::mutex> lk(mu);
      for (size_t i = 0; i < pin_free.size(); i++)
        if (pin_free[i].second >= bytes && pin_free[i].second <= bytes * 2 + ((size_t)1 << 20)) {
          char* p = pin_free[i].first;
          *got = pin_free[i].second;
          pin_free.erase(pin_free.begin() + (long)i);
          return p;
        }
    }
    char* p = nullptr;
    if (cudaHostAlloc((void**)&p, bytes, cudaHostAllocDefault) != cudaSuccess) return nullptr;
    *got = bytes;
    return p;
  }
  void pin_put(char* p, size_t bytes) {
    if (!p) return;
    std::lock_guard<std::mutex> lk(mu);
    if (pin_free.size() >= 4) {
      cudaFreeHost(pin_free.front().first);
      pin_free.erase(pin_free.begin());
    }
    pin_free.emplace_back(p, bytes);
  }
  void set_err(const std::string& s) { err = s; }
  bool is_pinned(const void* p, size_t n) const {
    const char* c = (const char*)p;
    for (auto& r : pinned)
      if (c >= r.first && c + n <= r.first + r.second) return true;
    return false;
  }
};

static cudaError_t pool_alloc(sg_ctx* c, void** out, size_t bytes);
static void pool_release(sg_ctx* c, void* p);

#define CUDA_TRY(ctx, expr)                                                                   \
  do {                                                                                        \
    cudaError_t _e = (expr);                                                                  \
    if (_e != cudaSuccess) {                                                                  \
      (ctx)->set_err(std::string(#expr) + ": " + cudaGetErrorString(_e));                     \
      return SG_ERR_CUDA;                                                                     \
    }                                                                                         \
  } while (0)

// a temporary pool buffer that goes back to the pool on every exit path
struct PoolTmp {
  sg_ctx* c;
  void* p = nullptr;
  explicit PoolTmp(sg_ctx* ctx) : c(ctx) {}
  ~PoolTmp() {
    if (p) pool_release(c, p);
  }
  PoolTmp(const PoolTmp&) = delete;
  PoolTmp& operator=(const PoolTmp&) = delete;
};

static cudaError_t pool_alloc(sg_ctx* c, void** out, size_t bytes) {
  std::lock_guard<std::mutex> lk(c->mu);
  size_t best = (size_t)-1;
  for (size_t i = 0; i < c->pool_free.size(); i++)
    if (c->pool_free[i].second >= bytes && (best == (size_t)-1 || c->pool_free[i].second < c->pool_free[best].second))
      best = i;
  if (best != (size_t)-1 && c->pool_free[best].second <= bytes * 2 + (1 << 20)) {
    *out = c->pool_free[best].first;
    c->pool_live[*out] = c->pool_free[best].second;
    c->pool_free.erase(c->pool_free.begin() + (long)best);
    return cudaSuccess;
  }
  cudaError_t e = cudaMalloc(out, bytes);
  if (e == cudaSuccess) c->pool_live[*out] = bytes;
  return e;
}
static void pool_release(sg_ctx* c, void* p) {
  if (!p) return;
  std::lock_guard<std::mutex> lk(c->mu);
  auto it = c->pool_live.find(p);
  if (it == c->pool_live.end()) {
    cudaFree(p);
    return;
  }
  c->pool_free.emplace_back(p, it->second);
  c->pool_live.erase(it);
  // keep the cache bounded: drop the largest buffers beyond 16 entries
  while (c->pool_free.size() > 16) {
    size_t big = 0;
    for (size_t i = 1; i < c->pool_free.size(); i++)
      if (c->pool_free[i].second > c->pool_free[big].second) big = i;
    cudaFree(c->pool_free[big].first);
    c->pool_free.erase(c->pool_free.begin() + (long)big);
  }
}

namespace {

// String -> dense id.  Open addressing over (hash, id); lookups hash the caller's bytes in place
// (a block of a high-cardinality column interns ~65,000 strings, a 1B-row table ~10^9 in all)
struct StrDict {
  std::vector<std::string> strs;
  std::vector<uint64_t> slots;  // (hash & ~0xffffffff) | (id + 1); 0 = empty
  size_t mask = 0;
  static uint64_t hash_bytes(const char* p, size_t n) {
    uint64_t h = 0x9E3779B97F4A7C15ull ^ (n * 0xff51afd7ed558ccdull);
    while (n >= 8) {
      uint64_t w;
      memcpy(&w, p, 8);
      h = (h ^ w) * 0xff51afd7ed558ccdull;
      h ^= h >> 32;
      p += 8;
      n -= 8;
    }
    uint64_t w = 0;
    memcpy(&w, p, n);
    h = (h ^ w) * 0xc4ceb9fe1a85ec53ull;
    h ^= h >> 29;
    return h;
  }
  void grow() {
    size_t cap = slots.empty() ? 1024 : slots.size() * 2;
    std::vector<uint64_t> ns(cap, 0);
    size_t m = cap - 1;
    for (size_t id = 0; id < strs.size(); id++) {
      uint64_t h = hash_bytes(strs[id].data(), strs[id].size());
      size_t i = (size_t)h & m;
      while (ns[i]) i = (i + 1) & m;
      ns[i] = (h & ~0xffffffffull) | (uint64_t)(id + 1);
    }
    slots.swap(ns);
    mask = m;
  }
  int32_t lookup(const char* p, size_t n, uint64_t h) const {
    if (slots.empty()) return -1;
    size_t i = (size_t)h & mask;
    while (slots[i]) {
      if ((slots[i] & ~0xffffffffull) == (h & ~0xffffffffull)) {
        const std::string& s = strs[(size_t)(slots[i] & 0xffffffffull) - 1];
        if (s.size() == n && memcmp(s.data(), p, n) == 0) return (int32_t)((slots[i] & 0xffffffffull) - 1);
      }
      i = (i + 1) & mask;
    }
    return -1;
  }
  int32_t intern(const char* p, size_t n) {
    const uint64_t h = hash_bytes(p, n);
    int32_t id = lookup(p, n, h);
    if (id >= 0) return id;
    if ((strs.size() + 1) * 2 > slots.size()) grow();
    id = (int32_t)strs.size();
    strs.emplace_back(p, n);
    size_t i = (size_t)h & mask;
    while (slots[i]) i = (i + 1) & mask;
    slots[i] = (h & ~0xffffffffull) | (uint64_t)(id + 1);
    return id;
  }
  int32_t find(const std::string& s) const { return lookup(s.data(), s.size(), hash_bytes(s.data(), s.size())); }
};
struct IntDict {
  std::unordered_map<int64_t, int32_t> map;
  std::vector<int64_t> vals;
  bool overflow = false;
  int32_t intern(int64_t v) {
    auto it = map.find(v);
    if (it != map.end()) return it->second;
    if ((int64_t)vals.size() >= INT_DICT_CAP) {
      overflow = true;
      return 0;
    }
    int32_t id = (int32_t)vals.size();
    map.emplace(v, id);
    vals.push_back(v);
    return id;
  }
};

struct HostBlock {
  int64_t block_index = 0;
  uint32_t num_records = 0;
  std::vector<sg_int_info> info;
};

struct Stage {
  char* host = nullptr;
  size_t used = 0;
  cudaEvent_t done = nullptr;
  bool pending = false;
};

}  // namespace

struct sg_table {
  sg_ctx* ctx = nullptr;
  int ncols = 0;
  std::vector<int32_t> types;
  std::vector<HostBlock> blocks;
  std::vector<DevCol> cols;  // [nblocks][ncols] host mirror (device pointers inside)
  std::vector<DevCol> segs;  // continuation segments of COL_SEGS set columns (sg_internal.h), host mirror
  std::vector<StrDict> sdict;
  std::vector<IntDict> idict;
  // entries each dictionary held after its last sg_table_dict_seed_* call (-1: never seeded).  A dictionary that
  // is still exactly its seed has the same size and numbering on every rank that seeded it alike.
  std::vector<int64_t> sseed, iseed;
  // the previous block's string table / bin values of each column and the global ids they interned to: blocks of one
  // table mostly repeat them (the same 12 strings, the same 1,000 bin values), and then the per-block hash lookups
  // — the host-side cost of staging once the arrays are narrow — shrink to one memcmp
  struct LastDict {
    std::string bytes;
    std::vector<uint32_t> offsets;
    std::vector<int32_t> remap;
  };
  struct LastBins {
    std::vector<int64_t> values;
    std::vector<int32_t> remap;
    int64_t mn = 0, mx = 0;
  };
  std::vector<LastDict> last_dict;
  std::vector<LastBins> last_bins;
  std::vector<char> has_values_int;  // an int column that is value-array encoded somewhere
  // group-by on such a column: its value-array blocks' distinct values join the column's IntDict
  // (on demand, kernel-side distinct set) and a device open-addressing table maps value -> code
  struct ValueHash {
    size_t blocks_done = 0;      // blocks [0, blocks_done) have contributed their values
    size_t dict_size = 0;        // IntDict size the device table was built from
    long long* d_keys = nullptr;
    uint32_t* d_ids = nullptr;
    uint32_t mask = 0;
  };
  std::vector<ValueHash> vhash;
  std::vector<uint32_t> pending_stats;  // value-array int columns whose extents are not computed yet
  std::vector<unsigned long long> pending_codes;  // parallel to pending_stats: where the item's per-row codes go (0: none)
  // The per-row codes of COL_CODES columns (sg_internal.h) are written on the device by the statistics kernel, so they
  // get a bump allocator of their own: in the arena they would sit between the slabs of consecutive blocks and split
  // the slabs' merged copies (and a merged copy over them would send their bytes over PCIe for nothing)
  std::vector<std::pair<char*, size_t>> code_chunks;
  size_t code_idx = 0, code_used = 0;
  // sort ranks of the dictionaries' rendered fields (ties of SortResults break by GroupByKey ascending):
  // rank[id] over the strings (resp. the decimal renderings of the int values) + '\t'; rebuilt when a
  // dictionary has grown.  splain[col]: no string of srank[col]'s dictionary holds a byte <= '\t' (the ranks
  // then give GroupByKey order field by field)
  std::vector<std::vector<uint32_t>> srank, irank;
  std::vector<uint8_t> splain;
  std::vector<std::pair<char*, size_t>> chunks;  // device arena chunks (ptr, capacity)
  size_t chunk_idx = 0, chunk_used = 0;
  Stage stage[2];
  int cur_stage = 0;
  int64_t total_rows = 0;
  int64_t device_bytes = 0;
  int64_t encoded_bytes = 0;
  int64_t h2d_bytes = 0;
  int64_t stats_launches = 0;
  // one tensor map per arena chunk ({128 B, rows} bytes view, 128B swizzle, 32-row boxes)
  std::vector<CUtensorMap> tmaps;
  void* d_tmaps = nullptr;
  size_t d_tmaps_cap = 0;
  bool tmaps_dirty = false;
  bool tma_ok = true;
  // device mirrors of blocks / cols, refreshed when dirty
  DevBlock* d_blocks = nullptr;
  DevCol* d_cols = nullptr;
  size_t d_blocks_cap = 0;
  DevCol* d_segs = nullptr;
  size_t d_segs_cap = 0;
  bool dirty = true;
  uint64_t version = 1;  // bumped whenever blocks or dictionaries change: a query's plan is reused while it stands
  // Small arrays of consecutive blocks (bin values, offsets, remap tables: a few KB per block) sit back to back both in
  // the pinned staging buffer and in the arena (both bump-allocated with the same 256-byte rounding): their copies
  // are merged into one cudaMemcpyAsync per run of blocks instead of one per block (15,259 driver calls per staged
  // C3 table otherwise).  Flushed before a staging buffer is handed over, and when a public staging call returns.
  char* pend_dev = nullptr;
  const char* pend_host = nullptr;
  size_t pend_len = 0;
};
static int flush_pending_copy(sg_table* t) {
  if (!t->pend_len) return SG_OK;
  sg_ctx* c = t->ctx;
  const size_t n = t->pend_len;
  t->pend_len = 0;
  CUDA_TRY(c, cudaMemcpyAsync(t->pend_dev, t->pend_host, n, cudaMemcpyHostToDevice, c->copy_stream));
  return SG_OK;
}

namespace {

int arena_alloc(sg_table* t, size_t bytes, char** out) {
  bytes = align_up(bytes, 256);
  while (t->chunk_idx < t->chunks.size() && t->chunk_used + bytes > t->chunks[t->chunk_idx].second) {
    t->chunk_idx++;
    t->chunk_used = 0;
  }
  if (t->chunk_idx >= t->chunks.size()) {
    size_t cap = std::max(ARENA_CHUNK, bytes);
    char* p = nullptr;
    cudaError_t e = cudaMalloc(&p, cap);
    if (e != cudaSuccess) {
      t->ctx->set_err(std::string("cudaMalloc arena: ") + cudaGetErrorString(e));
      return SG_ERR_NOMEM;
    }
    t->chunks.emplace_back(p, cap);
    t->chunk_idx = t->chunks.size() - 1;
    t->chunk_used = 0;
    t->device_bytes += (int64_t)cap;
    // three views of the chunk, row pitch 128 / 64 / 32 bytes (wide / 2x / 4x narrow arrays, see col_shift):
    // a box is always 32 rows = one warp tile, swizzled so that a lane reading its own row is conflict-free
    TmapEncodeFn enc = getenv("SG_NO_TMA") ? nullptr : tmap_encode_fn();  // SG_NO_TMA=1: plain vector loads (A/B)
    for (uint32_t sh = 0; sh < 3; sh++) {
      CUtensorMap tm;
      memset(&tm, 0, sizeof(tm));
      if (enc && t->tma_ok) {
        const cuuint32_t pitch = 128u >> sh;
        const cuuint64_t gdim[2] = {pitch, (cuuint64_t)(cap / pitch)};
        const cuuint64_t gstr[1] = {pitch};
        const cuuint32_t box[2] = {pitch, 32};
        const cuuint32_t estr[2] = {1, 1};
        const CUtensorMapSwizzle swz = sh == 0 ? CU_TENSOR_MAP_SWIZZLE_128B : (sh == 1 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
        if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, p, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swz,
                CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
          t->tma_ok = false;
      } else {
        t->tma_ok = false;
      }
      t->tmaps.push_back(tm);
    }
    t->tmaps_dirty = true;
  }
  *out = t->chunks[t->chunk_idx].first + t->chunk_used;
  t->chunk_used += bytes;
  return SG_OK;
}

constexpr size_t CODE_CHUNK = (size_t)64 << 20;
int code_alloc(sg_table* t, size_t bytes, char** out) {
  bytes = align_up(bytes, 128);
  while (t->code_idx < t->code_chunks.size() && t->code_used + bytes > t->code_chunks[t->code_idx].second) {
    t->code_idx++;
    t->code_used = 0;
  }
  if (t->code_idx >= t->code_chunks.size()) {
    char* p = nullptr;
    cudaError_t e = cudaMalloc(&p, CODE_CHUNK);
    if (e != cudaSuccess) {
      t->ctx->set_err(std::string("cudaMalloc codes: ") + cudaGetErrorString(e));
      return SG_ERR_NOMEM;
    }
    t->code_chunks.emplace_back(p, CODE_CHUNK);
    t->code_idx = t->code_chunks.size() - 1;
    t->code_used = 0;
    t->device_bytes += (int64_t)CODE_CHUNK;
  }
  *out = t->code_chunks[t->code_idx].first + t->code_used;
  t->code_used += bytes;
  return SG_OK;
}

// One block's arrays are packed into a slab: host copy in pinned staging, same
// layout in the device arena, one cudaMemcpyAsync per block.
struct SlabWriter {
  std::vector<std::pair<const void*, size_t>> parts;  // source, bytes
  std::vector<size_t> offs;
  std::vector<char> direct;  // source already pinned: DMA straight from the caller's buffer
  size_t total = 0;
  size_t staged = 0;
  size_t add(const void* src, size_t bytes, bool is_direct = false) {
    size_t off = total;
    parts.emplace_back(src, bytes);
    offs.push_back(off);
    direct.push_back(is_direct ? 1 : 0);
    total = align_up(total + bytes, 128);
    if (!is_direct) staged = total;
    return off;
  }
};

}  // namespace

// ===========================================================================
// context
// ===========================================================================
extern "C" {

int sg_abi_version(void) { return SG_ABI_VERSION; }

sg_ctx* sg_create(int device, int* status_out) {
  sg_ctx* c = new sg_ctx();
  c->device = device;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) {
    c->set_err(e != cudaSuccess ? std::string("cudaGetDeviceCount: ") + cudaGetErrorString(e)
                                : std::string("no such CUDA device"));
    if (status_out) *status_out = SG_ERR_CUDA;
    // the context is still returned so the message can be read; every call that
    // needs the GPU fails loudly (there is no CPU fallback)
    return c;
  }
  cudaSetDevice(device);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, device);
  c->sm_count = prop.multiProcessorCount;
  snprintf(c->devname, sizeof(c->devname), "%s", prop.name);
  if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking) != cudaSuccess) {
    c->set_err("cudaStreamCreate failed");
    if (status_out) *status_out = SG_ERR_CUDA;
    return c;
  }
  c->has_device = true;
  if (status_out) *status_out = SG_OK;
  return c;
}

void sg_destroy(sg_ctx* c) {
  if (!c) return;
  if (c->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(c->comm);
  for (auto& p : c->pool_free) cudaFree(p.first);
  for (auto& p : c->pool_live) cudaFree(p.first);  // buffers an error path did not hand back
  if (c->hpin) cudaFreeHost(c->hpin);
  for (auto& p : c->pin_free) cudaFreeHost(p.first);
  if (c->stream) cudaStreamDestroy(c->stream);
  if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
  delete c;
}
const char* sg_last_error(sg_ctx* c) { return c ? c->err.c_str() : "null context"; }
int sg_device_sm_count(sg_ctx* c) { return c ? c->sm_count : 0; }

void* sg_pinned_alloc(sg_ctx* c, size_t bytes) {
  if (!c || !c->has_device) return nullptr;
  void* p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
    c->set_err("cudaHostAlloc failed");
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(c->mu);
  c->pinned.emplace_back((const char*)p, bytes);
  return p;
}
void sg_pinned_free(sg_ctx* c, void* p) {
  if (!p) return;
  if (c) {
    std::lock_guard<std::mutex> lk(c->mu);
    for (size_t i = 0; i < c->pinned.size(); i++)
      if (c->pinned[i].first == (const char*)p) {
        c->pinned.erase(c->pinned.begin() + (long)i);
        break;
      }
  }
  cudaFreeHost(p);
}

int sg_comm_unique_id(sg_ctx* c, char id_out[128]) {
  if (!c) return SG_ERR_INVALID;
  if (!g_nccl.load()) {
    c->set_err("libnccl.so.2 not found");
    return SG_ERR_NCCL;
  }
  ncclUniqueId id;
  ncclResult_t r = g_nccl.GetUniqueId(&id);
  if (r != 0) {
    c->set_err("ncclGetUniqueId failed");
    return SG_ERR_NCCL;
  }
  memcpy(id_out, id.internal, 128);
  return SG_OK;
}
int sg_comm_init(sg_ctx* c, const char id[128], int rank, int nranks) {
  if (!c || !c->has_device) return SG_ERR_CUDA;
  if (!g_nccl.load()) {
    c->set_err("libnccl.so.2 not found");
    return SG_ERR_NCCL;
  }
  cudaSetDevice(c->device);
  ncclUniqueId uid;
  memcpy(uid.internal, id, 128);
  ncclResult_t r = g_nccl.CommInitRank(&c->comm, nranks, uid, rank);
  if (r != 0) {
    c->set_err(std::string("ncclCommInitRank: ") + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"));
    c->comm = nullptr;
    return SG_ERR_NCCL;
  }
  c->rank = rank;
  c->nranks = nranks;
  return SG_OK;
}

// ===========================================================================
// table
// ===========================================================================
sg_table* sg_table_create(sg_ctx* c, int32_t num_col_slots, const int32_t* col_types) {
  if (!c) return nullptr;
  if (!c->has_device) {
    c->set_err("sg_table_create: no CUDA device (libsybilgpu has no CPU path)");
    return nullptr;
  }
  if (num_col_slots <= 0 || num_col_slots > SG_MAX_COLS) {
    c->set_err("sg_table_create: num_col_slots out of range");
    return nullptr;
  }
  sg_table* t = new sg_table();
  t->ctx = c;
  t->ncols = num_col_slots;
  t->types.assign(col_types, col_types + num_col_slots);
  t->sdict.resize((size_t)num_col_slots);
  t->idict.resize((size_t)num_col_slots);
  t->has_values_int.assign((size_t)num_col_slots, 0);
  t->vhash.assign((size_t)num_col_slots, sg_table::ValueHash());
  t->last_dict.assign((size_t)num_col_slots, sg_table::LastDict());
  t->last_bins.assign((size_t)num_col_slots, sg_table::LastBins());
  t->sseed.assign((size_t)num_col_slots, -1);
  t->iseed.assign((size_t)num_col_slots, -1);
  t->srank.assign((size_t)num_col_slots, std::vector<uint32_t>());
  t->irank.assign((size_t)num_col_slots, std::vector<uint32_t>());
  t->splain.assign((size_t)num_col_slots, 1);
  cudaSetDevice(c->device);
  for (int i = 0; i < 2; i++) {
    if (cudaHostAlloc((void**)&t->stage[i].host, STAGE_BYTES, cudaHostAllocDefault) != cudaSuccess ||
        cudaEventCreateWithFlags(&t->stage[i].done, cudaEventDisableTiming) != cudaSuccess) {
      c->set_err("sg_table_create: staging allocation failed");
      delete t;
      return nullptr;
    }
  }
  return t;
}

void sg_table_free(sg_table* t) {
  if (!t) return;
  cudaSetDevice(t->ctx->device);
  cudaStreamSynchronize(t->ctx->copy_stream);
  for (auto& p : t->chunks) cudaFree(p.first);
  for (auto& p : t->code_chunks) cudaFree(p.first);
  for (int i = 0; i < 2; i++) {
    if (t->stage[i].host) cudaFreeHost(t->stage[i].host);
    if (t->stage[i].done) cudaEventDestroy(t->stage[i].done);
  }
  if (t->d_blocks) cudaFree(t->d_blocks);
  if (t->d_cols) cudaFree(t->d_cols);
  if (t->d_segs) cudaFree(t->d_segs);
  for (auto& vh : t->vhash) {
    if (vh.d_keys) cudaFree(vh.d_keys);
    if (vh.d_ids) cudaFree(vh.d_ids);
  }
  if (t->d_tmaps) cudaFree(t->d_tmaps);
  delete t;
}

}  // extern "C"

namespace {
// A span of the caller's pinned memory mirrored into the arena by one large copy
// (sg_table_add_blocks): arrays inside it are addressed in place, not copied again.
struct Premap {
  const char* host = nullptr;
  char* dev = nullptr;
  size_t bytes = 0;
  size_t chunk = 0;
  bool has(const void* p, size_t n) const {
    const char* c = (const char*)p;
    return host && c >= host && c + n <= host + bytes && ((size_t)(c - host) % 128) == 0;
  }
};

// One segment of a set column cut at bin boundaries: its first bin, its bin offsets rebased to its own ids, and
// where its two arrays sit in the block's slab.
struct SetSeg {
  uint32_t b0 = 0;
  std::vector<uint32_t> bo;
  size_t off_bo = 0, off_data = 0;
};

// A set column listing more than SG_BLOCK_ROWS (tag,row) pairs is cut greedily into segments of whole bins, each of
// at most SG_BLOCK_ROWS entries.  A bin's first id is absolute even with delta-encoded ids, so every segment is a
// bucket column of its own.  `offs` are the offsets of the column's non-empty bins into record_ids (nbins + 1).
// Returns false when the block is broken for this column: some row >= NumRecords, or a bin longer than
// SG_BLOCK_ROWS (never two entries for one row in a bin, so it holds such a row).  The rows are checked here and
// not only by the scan: an IN filter does not read the segments that lack its tag.
static bool cut_set_segments(const sg_column_desc& cd, size_t id_size, uint32_t nrec, const std::vector<uint32_t>& offs,
                             std::vector<SetSeg>& segs) {
  auto rows_ok = [&](auto ids) {
    for (size_t b = 0; b + 1 < offs.size(); b++) {
      uint64_t row = 0;
      for (uint32_t j = offs[b]; j < offs[b + 1]; j++) {
        row = (cd.delta_ids && j > offs[b]) ? row + ids[j] : (uint64_t)ids[j];
        if (row >= nrec) return false;
      }
    }
    return true;
  };
  segs.clear();  // (left empty when the block is broken)
  for (size_t b = 0; b + 1 < offs.size(); b++)
    if (offs[b + 1] - offs[b] > SG_BLOCK_ROWS) return false;
  if (!(id_size == 2 ? rows_ok((const uint16_t*)cd.record_ids) : rows_ok((const uint32_t*)cd.record_ids))) return false;
  for (size_t b = 0; b + 1 < offs.size(); b++) {
    if (segs.empty() || offs[b + 1] - offs[segs.back().b0] > SG_BLOCK_ROWS) {
      segs.emplace_back();
      segs.back().b0 = (uint32_t)b;
    }
  }
  for (size_t s = 0; s < segs.size(); s++) {
    const uint32_t b0 = segs[s].b0, b1 = s + 1 < segs.size() ? segs[s + 1].b0 : (uint32_t)offs.size() - 1u;
    for (uint32_t b = b0; b <= b1; b++) segs[s].bo.push_back(offs[b] - offs[b0]);
  }
  return true;
}
}  // namespace

static int add_block_impl(sg_table* t, const sg_block_desc* b, const Premap& pm) {
  if (!t || !b) return SG_ERR_INVALID;
  sg_ctx* c = t->ctx;
  if (b->num_records <= 0 || b->num_records > SG_BLOCK_ROWS) {
    c->set_err("add_block: num_records out of range");
    return SG_ERR_INVALID;
  }
  if (b->ncols < 0 || (b->ncols > 0 && !b->cols)) {
    c->set_err("add_block: bad column list");
    return SG_ERR_INVALID;
  }
  cudaSetDevice(c->device);
  const uint32_t nrec = (uint32_t)b->num_records;
  std::vector<DevCol> dcs((size_t)t->ncols);
  memset(dcs.data(), 0, sizeof(DevCol) * dcs.size());
  // host-side temporaries that must live until the slab is packed
  struct Tmp {
    std::vector<int64_t> bin_values;
    std::vector<uint32_t> bin_offsets;
    std::vector<int32_t> remap;
    size_t off_bv = 0, off_bo = 0, off_data = 0, off_remap = 0;
    bool has_bv = false, has_bo = false, has_data = false, has_remap = false;
    char* premapped = nullptr;  // the data array already sits in the arena (mirrored span)
    std::vector<SetSeg> segs;   // a set column cut into segments (COL_SEGS)
  };
  std::vector<Tmp> tmp((size_t)b->ncols);
  SlabWriter sw;
  int64_t enc_bytes = 0;
  std::vector<uint32_t> stats_slots;
  std::vector<unsigned long long> stats_codes;  // parallel: where the column's per-row codes go (0: none)

  for (int ci = 0; ci < b->ncols; ci++) {
    const sg_column_desc& cd = b->cols[ci];
    if (cd.col_slot < 0 || cd.col_slot >= t->ncols) {
      c->set_err("add_block: col_slot out of range");
      return SG_ERR_INVALID;
    }
    if (cd.col_type != t->types[(size_t)cd.col_slot]) {
      c->set_err("add_block: column type differs from the table's KeyTypes");
      return SG_ERR_INVALID;
    }
    if (cd.col_type != SG_COL_INT && cd.col_type != SG_COL_STR && cd.col_type != SG_COL_SET) {
      c->set_err("add_block: unknown column type");
      return SG_ERR_INVALID;
    }
    DevCol& dc = dcs[(size_t)cd.col_slot];
    Tmp& tm = tmp[(size_t)ci];
    // a set column (SavedSetColumn) is staged like a bucket-encoded str column: tags are strings of the column's
    // global dictionary, bins list the rows whose set holds the tag (unpackSetCol, column_store_io.go:611-688)
    const bool is_set = cd.col_type == SG_COL_SET;
    const bool is_str = cd.col_type == SG_COL_STR || is_set;
    if (is_set && cd.encoding == SG_ENC_VALUES) {
      c->set_err("add_block: a set column comes in the bucket form (sybilgpu.h); nvalues carries len(Values)");
      return SG_ERR_INVALID;
    }
    dc.enc = (uint32_t)cd.encoding;
    dc.flags = (cd.delta_ids ? COL_DELTA_IDS : 0u) | (cd.delta_values ? COL_DELTA_VALUES : 0u) |
               (is_str ? COL_IS_STR : 0u) | (is_set ? COL_SET : 0u);
    dc.oob_gid = -1;
    if (cd.encoding == SG_ENC_ABSENT) continue;
    // narrow arrays (sybilgpu.h): element sizes of record_ids / values
    size_t id_size = 4, val_size = is_str ? 4 : 8;
    if (cd.encoding == SG_ENC_BUCKET) {
      if (cd.id_bits == 16) {
        id_size = 2;
        dc.flags |= COL_ID16;
      } else if (cd.id_bits != 0 && cd.id_bits != 32) {
        c->set_err("add_block: id_bits must be 0, 16 or 32");
        return SG_ERR_INVALID;
      }
    } else if (cd.encoding == SG_ENC_VALUES) {
      const int vb = cd.value_bits;
      if (is_str) {
        if (vb == 16) {
          val_size = 2;
          dc.flags |= COL_VAL16;
        } else if (vb != 0 && vb != 32) {
          c->set_err("add_block: value_bits of a str column must be 0, 16 or 32");
          return SG_ERR_INVALID;
        }
      } else if (vb == 32 || vb == 16) {
        if (!cd.delta_values) {
          c->set_err("add_block: narrow int values are deltas (delta_values must be set)");
          return SG_ERR_INVALID;
        }
        val_size = vb == 32 ? 4 : 2;
        dc.flags |= vb == 32 ? COL_VAL32 : COL_VAL16;
      } else if (vb != 0 && vb != 64) {
        c->set_err("add_block: value_bits of an int column must be 0, 16, 32 or 64");
        return SG_ERR_INVALID;
      }
    }
    if (is_str) {
      // unpackStrCol: a string table longer than the block is "BLOCK SIZE CHANGED" (:524); unpackSetCol has no
      // such check
      if (cd.ndict > nrec && !is_set) dc.flags |= COL_BROKEN;
      if (cd.ndict > 0 && (!cd.dict_bytes || !cd.dict_offsets)) {
        c->set_err("add_block: string table missing");
        return SG_ERR_INVALID;
      }
      StrDict& sd = t->sdict[(size_t)cd.col_slot];
      sg_table::LastDict& ld = t->last_dict[(size_t)cd.col_slot];
      const size_t nbytes = cd.ndict ? cd.dict_offsets[cd.ndict] : 0;
      if (cd.ndict > 0 && ld.offsets.size() == (size_t)cd.ndict + 1 && ld.bytes.size() == nbytes &&
          memcmp(ld.offsets.data(), cd.dict_offsets, ((size_t)cd.ndict + 1) * 4) == 0 &&
          memcmp(ld.bytes.data(), cd.dict_bytes, nbytes) == 0) {
        tm.remap = ld.remap;  // the same string table as the column's previous block
      } else {
        tm.remap.resize(cd.ndict);
        // duplicate strings inside one table keep the first id (bucket_replace, :536-545)
        for (uint32_t k = 0; k < cd.ndict; k++) {
          uint32_t o0 = cd.dict_offsets[k], o1 = cd.dict_offsets[k + 1];
          if (o1 < o0) {
            c->set_err("add_block: string offsets not monotone");
            return SG_ERR_INVALID;
          }
          tm.remap[k] = sd.intern(cd.dict_bytes + o0, o1 - o0);
        }
        if (cd.ndict > 0 && cd.ndict <= 4096) {  // (a 60,000-string table is not worth a copy per block)
          ld.offsets.assign(cd.dict_offsets, cd.dict_offsets + cd.ndict + 1);
          ld.bytes.assign(cd.dict_bytes, nbytes);
          ld.remap = tm.remap;
        }
      }
      dc.oob_gid = sd.intern("", 0);
      dc.nremap = cd.ndict;
    }
    if (cd.encoding == SG_ENC_BUCKET) {
      if (cd.nbins > 0 && (!cd.bin_values || !cd.bin_offsets)) {
        c->set_err("add_block: bucket arrays missing");
        return SG_ERR_INVALID;
      }
      if (cd.nrecord_ids > 0 && !cd.record_ids) {
        c->set_err("add_block: record ids missing");
        return SG_ERR_INVALID;
      }
      if (cd.nbins > 0 && (cd.bin_offsets[0] != 0 || cd.bin_offsets[cd.nbins] != cd.nrecord_ids)) {
        c->set_err("add_block: bin_offsets do not span record_ids");
        return SG_ERR_INVALID;
      }
      if (cd.nrecord_ids > SG_BLOCK_ROWS && !is_set) {
        // more (bin,row) pairs than a block has rows: some row would be listed twice
        c->set_err("add_block: more record ids than rows in a block");
        return SG_ERR_INVALID;
      }
      // drop empty bins (the kernel's head-bit scheme needs non-empty bins)
      tm.bin_values.reserve(cd.nbins);
      tm.bin_offsets.reserve(cd.nbins + 1);
      for (uint32_t k = 0; k < cd.nbins; k++) {
        uint32_t o0 = cd.bin_offsets[k], o1 = cd.bin_offsets[k + 1];
        if (o1 < o0) {
          c->set_err("add_block: bin_offsets not monotone");
          return SG_ERR_INVALID;
        }
        if (o1 == o0) continue;
        int64_t v = cd.bin_values[k];
        // a string bin whose id is outside the table decodes to id 0 in the
        // reference (Go map zero value, column_store_io.go:557-562)
        if (is_str && (v < 0 || v >= (int64_t)cd.ndict)) v = 0;
        tm.bin_values.push_back(v);
        tm.bin_offsets.push_back(o0);
      }
      tm.bin_offsets.push_back(cd.nrecord_ids);
      dc.nbins = (uint32_t)tm.bin_values.size();
      dc.nitems = cd.nrecord_ids;
      if (is_set) dc.vmin = (int64_t)std::min<uint32_t>(cd.nvalues, nrec);  // rows populated whatever the bins say
      if (dc.nbins == 0) {
        dc.enc = SG_ENC_ABSENT;  // (a set column of nothing but empty sets keeps COL_SET + vmin: see the kernel)
        continue;
      }
      if (!is_str) {
        IntDict& id = t->idict[(size_t)cd.col_slot];
        sg_table::LastBins& lb = t->last_bins[(size_t)cd.col_slot];
        int64_t mn = INT64_MAX, mx = INT64_MIN;
        if (lb.values.size() == tm.bin_values.size() && !id.overflow &&
            memcmp(lb.values.data(), tm.bin_values.data(), tm.bin_values.size() * 8) == 0) {
          tm.remap = lb.remap;  // the same bin values as the column's previous block
          mn = lb.mn;
          mx = lb.mx;
        } else {
          tm.remap.resize(dc.nbins);
          for (uint32_t k = 0; k < dc.nbins; k++) {
            tm.remap[k] = id.intern(tm.bin_values[k]);
            mn = std::min(mn, tm.bin_values[k]);
            mx = std::max(mx, tm.bin_values[k]);
          }
          lb.values = tm.bin_values;
          lb.remap = tm.remap;
          lb.mn = mn;
          lb.mx = mx;
        }
        dc.nremap = dc.nbins;
        dc.vmin = mn;
        dc.vmax = mx;
        dc.flags |= COL_STATS;
      }
      if (cd.nrecord_ids > SG_BLOCK_ROWS) {  // (a set column: int / str columns were refused above)
        if (!cut_set_segments(cd, id_size, nrec, tm.bin_offsets, tm.segs)) {
          // a row >= NumRecords: "BLOCK SIZE CHANGED DURING QUERY" (column_store_io.go:654-656), nothing to stage
          dc.enc = SG_ENC_ABSENT;
          dc.flags |= COL_BROKEN;
          continue;
        }
        dc.flags |= COL_SEGS;
        tm.off_bv = sw.add(tm.bin_values.data(), tm.bin_values.size() * 8);
        // every segment's ids are a part of their own (128-byte aligned, as the tile loads assume): never a pointer
        // into the middle of the caller's array, premapped or not
        const char* ids = (const char*)cd.record_ids;
        for (size_t s = 0; s < tm.segs.size(); s++) {
          auto& sg = tm.segs[s];
          const size_t e0 = tm.bin_offsets[sg.b0], n = sg.bo.back();
          sg.off_bo = sw.add(sg.bo.data(), sg.bo.size() * 4);
          sg.off_data = sw.add(ids + e0 * id_size, n * id_size, c->is_pinned(ids + e0 * id_size, n * id_size));
          enc_bytes += (int64_t)(sg.bo.size() * 4);
        }
        tm.has_bv = true;
        enc_bytes += (int64_t)(tm.bin_values.size() * 8 + (size_t)cd.nrecord_ids * id_size);
      } else {
        tm.off_bv = sw.add(tm.bin_values.data(), tm.bin_values.size() * 8);
        tm.off_bo = sw.add(tm.bin_offsets.data(), tm.bin_offsets.size() * 4);
        if (pm.has(cd.record_ids, (size_t)cd.nrecord_ids * id_size))
          tm.premapped = pm.dev + ((const char*)cd.record_ids - pm.host);
        else
          tm.off_data = sw.add(cd.record_ids, (size_t)cd.nrecord_ids * id_size, c->is_pinned(cd.record_ids, (size_t)cd.nrecord_ids * id_size));
        tm.has_bv = tm.has_bo = tm.has_data = true;
        enc_bytes += (int64_t)(tm.bin_values.size() * 8 + tm.bin_offsets.size() * 4 + (size_t)cd.nrecord_ids * id_size);
        // candidate for COL_FULL, and for COL_CODES: room for one byte per row, which the statistics kernel fills
        // when the walk finds every listed row once and in range (SG_NO_CODES=1: no codes, for A/B and tests)
        char* codes = nullptr;
        if (!is_set && dc.nbins <= 255 && cd.nrecord_ids <= nrec && !(dc.flags & COL_BROKEN) && !getenv("SG_NO_CODES")) {
          const int rc = code_alloc(t, align_up(nrec, 16), &codes);
          if (rc != SG_OK) return rc;
          enc_bytes += (int64_t)align_up(nrec, 16);
        }
        if (codes || (cd.nrecord_ids == nrec && !is_set)) {
          stats_slots.push_back((uint32_t)cd.col_slot);
          stats_codes.push_back((unsigned long long)(uintptr_t)codes);
        }
      }
    } else if (cd.encoding == SG_ENC_VALUES) {
      dc.nitems = cd.nvalues;
      if (cd.nvalues > nrec) {
        dc.flags |= COL_BROKEN;  // unpackIntCol :752 / unpackStrCol :592
        dc.nitems = 0;
      } else if (cd.nvalues > 0) {
        if (is_str) {
          if (!cd.values_i32) {
            c->set_err("add_block: values_i32 missing");
            return SG_ERR_INVALID;
          }
          if (pm.has(cd.values_i32, (size_t)cd.nvalues * val_size))
            tm.premapped = pm.dev + ((const char*)cd.values_i32 - pm.host);
          else
            tm.off_data = sw.add(cd.values_i32, (size_t)cd.nvalues * val_size, c->is_pinned(cd.values_i32, (size_t)cd.nvalues * val_size));
          enc_bytes += (int64_t)cd.nvalues * (int64_t)val_size;
        } else {
          if (!cd.values_i64) {
            c->set_err("add_block: values_i64 missing");
            return SG_ERR_INVALID;
          }
          if (pm.has(cd.values_i64, (size_t)cd.nvalues * val_size))
            tm.premapped = pm.dev + ((const char*)cd.values_i64 - pm.host);
          else
            tm.off_data = sw.add(cd.values_i64, (size_t)cd.nvalues * val_size, c->is_pinned(cd.values_i64, (size_t)cd.nvalues * val_size));
          enc_bytes += (int64_t)cd.nvalues * (int64_t)val_size;
          if (val_size != 8) dc.vbase = cd.value_base;
          t->has_values_int[(size_t)cd.col_slot] = 1;
          stats_slots.push_back((uint32_t)cd.col_slot);
          stats_codes.push_back(0ull);
        }
        tm.has_data = true;
      }
    } else {
      c->set_err("add_block: unknown encoding");
      return SG_ERR_INVALID;
    }
    if (!tm.remap.empty()) {
      tm.off_remap = sw.add(tm.remap.data(), tm.remap.size() * 4);
      tm.has_remap = true;
    }
  }

  // ---- stage + copy ------------------------------------------------------------
  char* dev = nullptr;
  if (sw.total > 0) {
    if (sw.total > STAGE_BYTES) {
      c->set_err("add_block: block larger than the staging buffer");
      return SG_ERR_INVALID;
    }
    int rc = arena_alloc(t, sw.total, &dev);
    if (rc != SG_OK) return rc;
    Stage* st = &t->stage[t->cur_stage];
    if (st->used + sw.total > STAGE_BYTES) {
      rc = flush_pending_copy(t);  // (the event below must cover every copy that reads this staging buffer)
      if (rc != SG_OK) return rc;
      CUDA_TRY(c, cudaEventRecord(st->done, c->copy_stream));
      st->pending = true;
      t->cur_stage ^= 1;
      st = &t->stage[t->cur_stage];
      if (st->pending) {
        CUDA_TRY(c, cudaEventSynchronize(st->done));
        st->pending = false;
      }
      st->used = 0;
    }
    // staged parts: contiguous runs of non-direct parts are bounced through pinned
    // staging and copied run by run; direct parts go straight from the caller's memory
    char* hostp = st->host + st->used;
    size_t i = 0;
    bool any_direct = false;
    for (char d : sw.direct) any_direct = any_direct || d;
    if (!any_direct) {
      // the whole slab is staged: extend the pending merged copy when this slab continues it on both sides
      for (size_t j = 0; j < sw.parts.size(); j++) memcpy(hostp + sw.offs[j], sw.parts[j].first, sw.parts[j].second);
      if (t->pend_len && dev >= t->pend_dev && (size_t)(dev - t->pend_dev) == (size_t)(hostp - t->pend_host) &&
          (size_t)(dev - t->pend_dev) >= t->pend_len && (size_t)(dev - t->pend_dev) <= t->pend_len + 256) {
        t->pend_len = (size_t)(dev - t->pend_dev) + sw.total;
      } else {
        rc = flush_pending_copy(t);
        if (rc != SG_OK) return rc;
        t->pend_dev = dev;
        t->pend_host = hostp;
        t->pend_len = sw.total;
      }
      i = sw.parts.size();
    } else {
      rc = flush_pending_copy(t);
      if (rc != SG_OK) return rc;
    }
    while (i < sw.parts.size()) {
      if (sw.direct[i]) {
        CUDA_TRY(c, cudaMemcpyAsync(dev + sw.offs[i], sw.parts[i].first, sw.parts[i].second, cudaMemcpyHostToDevice,
                                    c->copy_stream));
        i++;
        continue;
      }
      size_t j = i, run_begin = sw.offs[i], run_end = sw.offs[i];
      while (j < sw.parts.size() && !sw.direct[j]) {
        memcpy(hostp + sw.offs[j], sw.parts[j].first, sw.parts[j].second);
        run_end = sw.offs[j] + sw.parts[j].second;
        j++;
      }
      CUDA_TRY(c, cudaMemcpyAsync(dev + run_begin, hostp + run_begin, run_end - run_begin, cudaMemcpyHostToDevice,
                                  c->copy_stream));
      i = j;
    }
    st->used += align_up(sw.total, 256);
    t->h2d_bytes += (int64_t)sw.total;
  }
  for (int ci = 0; ci < b->ncols; ci++) {
    const sg_column_desc& cd = b->cols[ci];
    DevCol& dc = dcs[(size_t)cd.col_slot];
    Tmp& tm = tmp[(size_t)ci];
    if (tm.has_bv) dc.bin_values = (const int64_t*)(dev + tm.off_bv);  // (VALUES columns keep vbase in the same field)
    if (tm.has_bo) dc.bin_offsets = (const uint32_t*)(dev + tm.off_bo);
    if (tm.has_data) {
      const size_t chunk = tm.premapped ? pm.chunk : t->chunk_idx;
      char* dptr = tm.premapped ? tm.premapped : dev + tm.off_data;
      dc.data = dptr;
      if (t->tma_ok) {
        dc.data_chunk = (uint32_t)chunk;
        dc.data_row = (uint32_t)((size_t)(dptr - t->chunks[chunk].first) / 128);
        dc.flags |= COL_TMA;
      }
    }
    if (tm.has_remap) dc.remap = (const int32_t*)(dev + tm.off_remap);
    if (!tm.segs.empty()) {
      // the slot's DevCol is the first segment, the others follow in the table-wide segment array
      const uint64_t first = t->segs.size();
      for (size_t s = 0; s < tm.segs.size(); s++) {
        const SetSeg& sg = tm.segs[s];
        DevCol sc = dc;
        sc.flags &= ~COL_SEGS;
        sc.nbins = (uint32_t)sg.bo.size() - 1u;
        sc.nitems = sg.bo.back();
        sc.bin_values = (const int64_t*)(dev + tm.off_bv) + sg.b0;
        sc.bin_offsets = (const uint32_t*)(dev + sg.off_bo);
        sc.data = dev + sg.off_data;
        if (s == 0) {
          sc.flags |= COL_SEGS;
          sc.vmax = (int64_t)(((uint64_t)(tm.segs.size() - 1) << 32) | first);
          dc = sc;
        } else {
          t->segs.push_back(sc);
        }
      }
    }
  }
  HostBlock hb;
  hb.block_index = b->block_index;
  hb.num_records = nrec;
  for (int i = 0; i < b->ninfo; i++) hb.info.push_back(b->info[i]);
  t->blocks.push_back(std::move(hb));
  for (uint32_t sl : stats_slots) t->pending_stats.push_back((uint32_t)(t->blocks.size() - 1) * (uint32_t)t->ncols + sl);
  t->pending_codes.insert(t->pending_codes.end(), stats_codes.begin(), stats_codes.end());
  t->cols.insert(t->cols.end(), dcs.begin(), dcs.end());
  t->total_rows += nrec;
  t->encoded_bytes += enc_bytes;
  t->dirty = true;
  t->version++;
  return SG_OK;
}

extern "C" {

int sg_table_add_block(sg_table* t, const sg_block_desc* b) {
  int rc = add_block_impl(t, b, Premap());
  const int rf = t ? flush_pending_copy(t) : SG_OK;
  return rc != SG_OK ? rc : rf;
}

int sg_table_add_blocks(sg_table* t, const sg_block_desc* const* blocks, int64_t n) {
  // Batch staging.  When the big arrays of the batch lie densely inside one region from
  // sg_pinned_alloc, the whole span is mirrored into the arena with a few large copies (full PCIe
  // rate, one DMA setup per 64 MiB instead of one per array) and the per-block work below only
  // handles dictionaries and the small per-bin arrays while that copy is in flight.
  if (!t || (n > 0 && !blocks)) return SG_ERR_INVALID;
  sg_ctx* c = t->ctx;
  cudaSetDevice(c->device);
  Premap pm;
  const char* lo = nullptr;
  const char* hi = nullptr;
  size_t payload = 0;
  auto see = [&](const void* p, size_t bytes) {
    if (!p || !bytes || !c->is_pinned(p, bytes)) return;
    const char* q = (const char*)p;
    if (!lo || q < lo) lo = q;
    if (!hi || q + bytes > hi) hi = q + bytes;
    payload += bytes;
  };
  for (int64_t i = 0; i < n; i++) {
    const sg_block_desc* b = blocks[i];
    if (!b || b->ncols < 0 || (b->ncols > 0 && !b->cols)) continue;
    for (int ci = 0; ci < b->ncols; ci++) {
      const sg_column_desc& cd = b->cols[ci];
      if (cd.encoding == SG_ENC_BUCKET)
        see(cd.record_ids, (size_t)cd.nrecord_ids * (cd.id_bits == 16 ? 2 : 4));
      else if (cd.encoding == SG_ENC_VALUES)
        see(cd.col_type == SG_COL_STR ? (const void*)cd.values_i32 : (const void*)cd.values_i64,
            (size_t)cd.nvalues * (cd.col_type == SG_COL_STR ? (cd.value_bits == 16 ? 2 : 4)
                                                            : (cd.value_bits == 32 ? 4 : (cd.value_bits == 16 ? 2 : 8))));
    }
  }
  if (lo && payload >= ((size_t)1 << 20)) {
    const char* base = (const char*)((uintptr_t)lo & ~(uintptr_t)127);
    size_t span = (size_t)(hi - base);
    if (span <= payload + payload / 2 + ((size_t)8 << 20)) {
      char* dev = nullptr;
      int rc = arena_alloc(t, span, &dev);
      if (rc != SG_OK) return rc;
      pm.host = base;
      pm.dev = dev;
      pm.bytes = span;
      pm.chunk = t->chunk_idx;
      const size_t piece = (size_t)64 << 20;
      for (size_t off = 0; off < span; off += piece) {
        size_t nb = std::min(piece, span - off);
        CUDA_TRY(c, cudaMemcpyAsync(dev + off, base + off, nb, cudaMemcpyHostToDevice, c->copy_stream));
      }
      t->h2d_bytes += (int64_t)span;
    }
  }
  for (int64_t i = 0; i < n; i++) {
    int rc = add_block_impl(t, blocks[i], pm);
    if (rc != SG_OK) {
      flush_pending_copy(t);
      return rc;
    }
  }
  return flush_pending_copy(t);
}

int sg_table_clear(sg_table* t) {
  // drop the staged blocks but keep the device arena, the staging buffers and the
  // dictionaries: the next sg_table_add_block reuses the memory
  if (!t) return SG_ERR_INVALID;
  cudaSetDevice(t->ctx->device);
  CUDA_TRY(t->ctx, cudaStreamSynchronize(t->ctx->copy_stream));
  CUDA_TRY(t->ctx, cudaStreamSynchronize(t->ctx->stream));
  t->blocks.clear();
  t->cols.clear();
  t->segs.clear();
  t->pending_stats.clear();
  t->pending_codes.clear();
  for (auto& vh : t->vhash) vh.blocks_done = 0;
  t->chunk_idx = 0;
  t->chunk_used = 0;
  t->code_idx = 0;
  t->code_used = 0;
  t->stage[0].pending = t->stage[1].pending = false;
  t->stage[0].used = t->stage[1].used = 0;
  t->total_rows = 0;
  t->encoded_bytes = 0;
  t->h2d_bytes = 0;
  t->dirty = true;
  t->version++;
  return SG_OK;
}

int sg_table_sync(sg_table* t) {
  if (!t) return SG_ERR_INVALID;
  cudaSetDevice(t->ctx->device);
  CUDA_TRY(t->ctx, cudaStreamSynchronize(t->ctx->copy_stream));
  t->stage[0].pending = t->stage[1].pending = false;
  t->stage[0].used = t->stage[1].used = 0;
  return SG_OK;
}
int64_t sg_table_num_blocks(sg_table* t) { return t ? (int64_t)t->blocks.size() : 0; }
int64_t sg_table_num_rows(sg_table* t) { return t ? t->total_rows : 0; }
int64_t sg_table_device_bytes(sg_table* t) { return t ? t->device_bytes : 0; }
int64_t sg_table_dict_size(sg_table* t, int32_t col) {
  if (!t || col < 0 || col >= t->ncols) return -1;
  return (int64_t)t->sdict[(size_t)col].strs.size();
}
int sg_table_dict_get(sg_table* t, int32_t col, int64_t id, const char** bytes, int64_t* len) {
  if (!t || col < 0 || col >= t->ncols) return SG_ERR_INVALID;
  auto& sd = t->sdict[(size_t)col];
  if (id < 0 || id >= (int64_t)sd.strs.size()) return SG_ERR_INVALID;
  *bytes = sd.strs[(size_t)id].data();
  *len = (int64_t)sd.strs[(size_t)id].size();
  return SG_OK;
}

int sg_table_dict_seed_str(sg_table* t, int32_t col, const char* bytes, const uint32_t* offsets, int64_t n) {
  if (!t || col < 0 || col >= t->ncols || n < 0 || (n > 0 && (!bytes || !offsets))) return SG_ERR_INVALID;
  for (int64_t i = 0; i < n; i++) t->sdict[(size_t)col].intern(bytes + offsets[i], offsets[i + 1] - offsets[i]);
  t->sseed[(size_t)col] = (int64_t)t->sdict[(size_t)col].strs.size();
  t->version++;
  return SG_OK;
}
int sg_table_dict_seed_int(sg_table* t, int32_t col, const int64_t* values, int64_t n) {
  if (!t || col < 0 || col >= t->ncols || n < 0 || (n > 0 && !values)) return SG_ERR_INVALID;
  for (int64_t i = 0; i < n; i++) t->idict[(size_t)col].intern(values[i]);
  t->iseed[(size_t)col] = (int64_t)t->idict[(size_t)col].vals.size();
  t->version++;
  return SG_OK;
}
int64_t sg_table_intdict_size(sg_table* t, int32_t col) {
  if (!t || col < 0 || col >= t->ncols) return -1;
  return (int64_t)t->idict[(size_t)col].vals.size();
}
int sg_table_intdict_get(sg_table* t, int32_t col, int64_t id, int64_t* value) {
  if (!t || col < 0 || col >= t->ncols || !value) return SG_ERR_INVALID;
  auto& d = t->idict[(size_t)col];
  if (id < 0 || id >= (int64_t)d.vals.size()) return SG_ERR_INVALID;
  *value = d.vals[(size_t)id];
  return SG_OK;
}
int64_t sg_table_encoded_bytes(sg_table* t) { return t ? t->encoded_bytes : 0; }
int64_t sg_table_h2d_bytes(sg_table* t) { return t ? t->h2d_bytes : 0; }

}  // extern "C"

// ===========================================================================
// query
// ===========================================================================
namespace {

struct GroupDim {  // one axis of the dense slot space
  int col = -1;
  bool is_str = false;
  bool is_time = false;
  bool is_weight = false;  // the hidden axis of a weighted query (OPTS.WEIGHT_COL): folded away before the result
  uint32_t radix = 1, stride = 1;
};

// The canonical key of a group code (canon_code), the one definition of the weight and StrReplace folds: the code
// with the weight digit set to 0 and each rewritten axis' digit replaced by its class representative's (0 when the
// string rewrites to "": the missing group, DESIGN.md §7); every other digit, time included, unchanged.  Dense plans
// fold their slots on the host (dense_fold), hashed and sparse plans their table entries on the device (fold_rows);
// build_fold_key fills it, with the tables in host vectors the caller points it at.
struct FoldKey {
  uint32_t naxes = 0;  // rewritten (StrReplace) axes
  uint32_t stride[SG_MAX_GROUPS] = {}, radix[SG_MAX_GROUPS] = {};
  uint32_t lut[SG_MAX_GROUPS] = {};  // offset of the axis' table in luts
  uint32_t wstride = 0, wradix = 0;  // the weight axis (wradix 0: unweighted)
  uint32_t wcarry = 0;
  const int64_t* wmul = nullptr;     // per weight code its multiplier (code 0: weight 1 under wcarry)
  const uint32_t* luts = nullptr;    // per rewritten axis, radix entries: digit -> canonical digit
};

// One region of the accumulator array after the scalars (layout_accumulators): per row `per_row` words at `off`,
// merged and folded by addition, or by max (the MAX region)
struct AccRegion {
  size_t off;
  uint32_t per_row;
  bool is_max;
};

struct ResultGroup {
  std::vector<uint64_t> key;
  std::string skey;
  int64_t count = 0;
  int64_t samples = -1;  // Result.Samples when it differs from Count (weighted queries); -1: == count
  // per aggregation a: agg[3a] = hist Count, agg[3a+1] = exact sum, agg[3a+2] = max above info_max
  // (one allocation per group: a high-cardinality result holds a million of these)
  std::vector<int64_t> agg;
  std::vector<std::vector<int64_t>> values;  // bucket counters per aggregation (hist mode only)
  int64_t& hc(int a) { return agg[(size_t)a * 3]; }
  int64_t& sm(int a) { return agg[(size_t)a * 3 + 1]; }
  int64_t& vx(int a) { return agg[(size_t)a * 3 + 2]; }
  int64_t hc(int a) const { return agg[(size_t)a * 3]; }
  int64_t sm(int a) const { return agg[(size_t)a * 3 + 1]; }
  int64_t vx(int a) const { return agg[(size_t)a * 3 + 2]; }
  const std::vector<int64_t>* vals(int a) const {
    return (size_t)a < values.size() && !values[(size_t)a].empty() ? &values[(size_t)a] : nullptr;
  }
};

// Words [0, words) of the accumulator array on the host (read_acc fills it): in a pinned buffer of the context's
// pool, which goes back to the pool with the object, or in a vector.  Move-only: a result takes over its query's.
struct HostAcc {
  sg_ctx* c = nullptr;
  char* pin = nullptr;
  size_t pin_bytes = 0;
  std::vector<uint64_t> vec;
  size_t words = 0;  // 0: no copy (a pinned buffer may still be held for the next read)
  HostAcc() = default;
  HostAcc& operator=(HostAcc&& o) noexcept {
    unpin();
    c = o.c;
    pin = std::exchange(o.pin, nullptr);
    pin_bytes = std::exchange(o.pin_bytes, 0);
    vec = std::move(o.vec);
    words = std::exchange(o.words, 0);
    return *this;
  }
  ~HostAcc() { unpin(); }
  uint64_t* data() { return pin ? (uint64_t*)pin : vec.data(); }
  void unpin() {
    if (pin) c->pin_put(pin, pin_bytes);
    pin = nullptr;
  }
  // a copy made on the host: n words, zeroed, in the vector
  uint64_t* host(size_t n) {
    unpin();
    vec.assign(n, 0);
    words = n;
    return vec.data();
  }
};

}  // namespace

struct sg_result {
  sg_query* q = nullptr;  // not owned
  std::vector<HistLayout> layouts;
  bool hist_mode = false;
  int ngroups_cols = 0;
  int naggs = 0;
  std::vector<ResultGroup> groups;  // sorted
  ResultGroup total;                // Cumulative
  int64_t matched = 0, broken = 0, skipped = 0;
  std::vector<int64_t> time_keys;
  std::vector<std::unique_ptr<sg_result>> time_slices;
  bool has_total_hists = true;
  // Results without a time axis are materialised on demand: the accumulators stay as read back, `order`
  // lists the (limit) slots in sorted order and a ResultGroup is built the first time it is asked for — a
  // 1M-group result no longer renders and sorts a million keys on the host per query
  bool lazy = false;
  HostAcc acc;
  std::vector<uint32_t> order;
  int64_t ngroups_total = 0;
  std::unordered_map<int64_t, std::unique_ptr<ResultGroup>> cache;
  // weighted queries: rows (Result.Samples) per dense slot — Count holds the weights' sum (aggregate.go:202-203)
  std::vector<uint64_t> samples;
};

struct sg_query {
  sg_ctx* ctx = nullptr;
  sg_table* table = nullptr;
  bool own_table = false;
  // copied descriptor
  sg_query_desc d;
  std::vector<sg_filter_desc> filters;
  std::vector<std::string> filter_strs;
  std::vector<sg_group_desc> groups;
  // the group columns the PLAN scans: `groups`, plus the weight column of a weighted query as a last, hidden axis
  std::vector<sg_group_desc> pgroups;
  std::vector<sg_agg_desc> aggs;
  std::vector<std::vector<uint32_t>> luts;  // per filter (host copy)
  std::vector<int64_t> lut_bits;
  // plan
  bool planned = false;
  Plan plan;
  std::vector<GroupDim> dims;
  std::vector<HistLayout> layouts;
  uint32_t slot_bytes = 2;
  uint32_t smem_bytes = 0;
  uint32_t nstage = 0;
  const Variant* variant = &V16;  // which build of the kernel runs the plan (make_plan)
  // device state
  Plan* d_plan = nullptr;
  uint64_t* d_acc = nullptr;  // one allocation: scalars | count | per agg hcount,sum,vmax | buckets
  size_t acc_words = 0;
  size_t sum_words = 0;  // leading words merged by SUM; the rest (vmax) by MAX
  size_t prefix_words = 0;  // scalars | count | sums
  size_t off_count = 0;
  std::vector<size_t> off_hcount, off_sum, off_vmax, off_buckets;
  std::vector<AccRegion> regions;  // the regions above in layout order (bucket counters of no width left out)
  uint32_t* d_block_status = nullptr;
  uint32_t* d_block_list = nullptr;
  uint32_t* d_item_mask = nullptr;
  uint32_t* d_work = nullptr;
  uint32_t* d_gslots = nullptr;
  uint32_t* d_gbinpay = nullptr;
  unsigned long long* d_gdummy = nullptr;
  std::vector<uint32_t*> d_luts;
  size_t block_cap = 0;
  int grid = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  // stats
  double kernel_ms = 0;
  int64_t launches = 0;
  int64_t skipped = 0, broken_staged = 0, stream_skipped = 0;
  int64_t rows_scanned = 0, blocks_scanned = 0;
  int64_t d2h_bytes = 0;
  bool ran = false;
  double host_plan_ms = 0, host_run_ms = 0;  // SG_HOST_TIMING
  // a prepared query run again over an unchanged table keeps its block list, plan and uploaded work items
  uint64_t plan_version = 0;
  std::vector<uint32_t> plan_list;
  int64_t plan_skipped = 0, plan_broken = 0, plan_rows = 0;
  std::vector<uint32_t> items_up, masks_up;  // work items as they sit in d_block_list
  uint64_t fold_version = 0;
  uint32_t fold_every = 1;
  std::vector<uint32_t> last_list;
  std::vector<char> hc_is_count;
  // cross-GPU merge under differing per-rank dictionaries: the union dictionaries the merged
  // accumulators are laid out by (per entry of dims; empty for the time axis)
  bool merged = false;
  bool hashg = false;  // a group column goes through the value -> code hash table
  // hashed slot space: the product of the group axes exceeds the dense slot space; accumulators are indexed by
  // the index of the row's mixed-radix code in an open-addressing table on the device (LaunchParams::hkeys)
  bool hashed = false;
  uint64_t code_space = 0;  // product of the axes' radices
  uint32_t* d_hkeys = nullptr;
  uint32_t hcap = 0;              // entries of the device table (LaunchParams::hkeys)
  std::vector<uint32_t> h_hkeys;  // read back for the result: slot -> code + 1 (0: empty)
  // sparse group accumulators (sg_query_set_sparse_groups): a hashed plan whose table is filled by a discovery
  // launch first; the accumulators then hold the live groups only, indexed by the dense id of their table entry
  int32_t sparse_req = 0;        // the setter's value, applied by the next plan
  bool sparse = false;           // this plan takes the path
  uint32_t* d_hids = nullptr;    // [hcap] table entry -> dense id, then [hcap] dense id -> key (code + 1)
  uint64_t* d_disc = nullptr;    // [DISC_WORDS] the discovery launch's scalars, then the live and canonical counts
  double disc_ms = 0;            // the last discovery launch (SG_PLAN_TRACE)
  // device folds (sg_query_set_hashed_folds): a hashed or sparse plan with weights or StrReplace combines the
  // accumulators of every table entry onto its canonical entry on the device (fold_insert, fold_rows)
  int32_t hfold_req = 0;           // the setter's value, applied by the next plan
  bool dfold = false;              // this plan folds on the device
  FoldKey fkey;                    // its device pointers name d_fold
  void* d_fold = nullptr;          // the weight multipliers (int64 per weight code), then the rewrite tables (uint32)
  uint64_t* d_samples = nullptr;   // [n] rows per accumulator row after the fold, then [n] each row's own rows
  uint32_t canon_live = 0;         // sparse: canonical entries, which hold ids 0..canon_live-1
  double insert_ms = 0, fold_ms = 0;
  cudaEvent_t ev2 = nullptr, ev3 = nullptr;
  // the whole accumulator array as read back right behind the last launch or merge (arrays up to 4 MiB: a C3-shaped
  // one is 0.94 MB): spares build_result a blocking copy, and its result takes the copy over
  HostAcc acc;
  uint64_t scal[SC_MERGE] = {};  // the scalars of the last launch (run_list)
  uint64_t axes_sig = 0, axes_sig_version = 0;  // axes_signature(): valid for table version axes_sig_version - 1
  size_t axes_size = 0;
  // multi-GPU: aggregations whose hist Count the kernel skipped on THIS rank (== Count here); the count array is
  // copied over the hist-Count array behind the scan so that the element-wise merge sums real values
  std::vector<char> hc_fill;
  std::vector<std::vector<std::string>> m_strs;
  std::vector<std::vector<int64_t>> m_ints;
  // StrReplace (sg_query_set_str_replace): per str column slot the rewritten text of every global string and the
  // smallest global id that rewrites to the same text (the class representative the groups are folded onto)
  struct Replace {
    std::vector<std::string> strs;
    std::vector<uint32_t> canon;
  };
  std::map<int, Replace> repl;
};

namespace {

// Reads words [0, words) of the accumulator array into h: the one place that picks pinned or pageable storage for it.
// An array of pin_from bytes or more lands in a pinned buffer of the context's pool (h's own when large enough) that
// h then holds, so nothing is copied out afterwards (that copy cost as much as the read itself).  A smaller one, or
// one no pinned buffer can be had for, lands in `stage` and is copied to a vector; without a stage the pinned buffer
// is required (a pageable destination is staged by the driver at a fraction of the PCIe rate).  `stage` is pinned
// scratch (sg_ctx::scratch) that copies queued earlier on c->stream may still read, and that the next query reuses:
// the copies into it queue behind those, and it is read only after the stream is synchronised.  copy(dst) queues the
// device-to-host copies on c->stream.
template <class Copy>
int read_acc(sg_query* q, HostAcc& h, size_t words, size_t pin_from, char* stage, Copy copy) {
  sg_ctx* c = q->ctx;
  const size_t bytes = words * 8;
  h.c = c;
  h.words = 0;
  char* dst = nullptr;
  if (bytes >= pin_from) {
    if (h.pin && h.pin_bytes < bytes) h.unpin();
    if (!h.pin) h.pin = c->pin_get(bytes, &h.pin_bytes);
    dst = h.pin;
  }
  if (!dst) dst = stage;
  if (!dst) {
    c->set_err("cudaHostAlloc (result buffer) failed");
    return SG_ERR_CUDA;
  }
  CUDA_TRY(c, copy((uint64_t*)dst));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  if (dst == stage) {
    h.unpin();
    h.vec.assign((const uint64_t*)stage, (const uint64_t*)stage + words);
  }
  h.words = words;
  return SG_OK;
}
int read_acc(sg_query* q, HostAcc& h, const uint64_t* src, size_t words, size_t pin_from, char* stage) {
  return read_acc(q, h, words, pin_from, stage, [&](uint64_t* dst) {
    return cudaMemcpyAsync(dst, src, words * 8, cudaMemcpyDeviceToHost, q->ctx->stream);
  });
}
// whole arrays from this size on are read into a pinned buffer of the pool rather than through the scratch area
constexpr size_t PIN_WHOLE_FROM = (size_t)32 << 10;

void free_device(sg_query* q) {
  sg_ctx* c = q->ctx;
  pool_release(c, q->d_plan);
  pool_release(c, q->d_acc);
  pool_release(c, q->d_block_status);
  pool_release(c, q->d_block_list);
  pool_release(c, q->d_item_mask);
  q->d_item_mask = nullptr;
  pool_release(c, q->d_work);
  pool_release(c, q->d_gslots);
  pool_release(c, q->d_hkeys);
  q->d_hkeys = nullptr;
  pool_release(c, q->d_hids);
  q->d_hids = nullptr;
  pool_release(c, q->d_disc);
  q->d_disc = nullptr;
  pool_release(c, q->d_fold);
  q->d_fold = nullptr;
  pool_release(c, q->d_samples);
  q->d_samples = nullptr;
  pool_release(c, q->d_gbinpay);
  pool_release(c, q->d_gdummy);
  for (auto p : q->d_luts) pool_release(c, p);
  q->d_luts.clear();
  q->d_plan = nullptr;
  q->d_acc = nullptr;
  q->d_gdummy = nullptr;
  q->d_block_status = q->d_block_list = q->d_work = q->d_gslots = q->d_gbinpay = nullptr;
}

uint32_t bits_for(uint64_t n) {  // bits to hold values 0..n-1
  uint32_t b = 0;
  while (((uint64_t)1 << b) < n) b++;
  return b;
}

// ShouldLoadBlockFromDir (table_block_io.go:110-182) over the staged block info
bool should_load(const sg_query* q, const std::vector<sg_int_info>& info) {
  if (info.empty()) return true;
  bool add = true;
  for (auto& f : q->filters) {
    if (f.col_type != SG_COL_INT) continue;
    const sg_int_info* fi = nullptr;
    for (auto& i : info)
      if (i.col_slot == f.col_slot) fi = &i;
    if (f.op == SG_OP_GT || f.op == SG_OP_LT) {
      bool pmin = false, pmax = false;
      if (fi) {
        pmin = f.op == SG_OP_GT ? fi->min > f.int_value : fi->min < f.int_value;
        pmax = f.op == SG_OP_GT ? fi->max > f.int_value : fi->max < f.int_value;
      }
      if (!pmin && !pmax) add = false;
    } else if (f.op == SG_OP_EQ) {
      if (!fi || fi->min > f.int_value || fi->max < f.int_value) add = false;
    }
  }
  return add;
}

int upload_table(sg_table* t) {
  sg_ctx* c = t->ctx;
  if (t->tmaps_dirty && t->tma_ok && !t->tmaps.empty()) {
    if (t->tmaps.size() > t->d_tmaps_cap) {
      if (t->d_tmaps) cudaFree(t->d_tmaps);
      t->d_tmaps = nullptr;
      size_t cap = t->tmaps.size() * 2 + 8;
      CUDA_TRY(c, cudaMalloc(&t->d_tmaps, cap * sizeof(CUtensorMap)));
      t->d_tmaps_cap = cap;
    }
    CUDA_TRY(c, cudaMemcpyAsync(t->d_tmaps, t->tmaps.data(), t->tmaps.size() * sizeof(CUtensorMap), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // (H2D on the stream the kernels run on: see remap_to_union)
    t->tmaps_dirty = false;
  }
  if (!t->dirty && t->d_blocks) return SG_OK;
  size_t nb = t->blocks.size();
  if (nb > t->d_blocks_cap) {
    if (t->d_blocks) cudaFree(t->d_blocks);
    if (t->d_cols) cudaFree(t->d_cols);
    t->d_blocks = nullptr;
    t->d_cols = nullptr;
    size_t cap = std::max<size_t>(nb * 2, 1024);
    CUDA_TRY(c, cudaMalloc(&t->d_blocks, cap * sizeof(DevBlock)));
    CUDA_TRY(c, cudaMalloc(&t->d_cols, cap * (size_t)t->ncols * sizeof(DevCol)));
    t->d_blocks_cap = cap;
  }
  std::vector<DevBlock> hb(nb);
  for (size_t i = 0; i < nb; i++) {
    hb[i].block_index = t->blocks[i].block_index;
    hb[i].num_records = t->blocks[i].num_records;
    hb[i]._pad = 0;
  }
  if (nb) {
    CUDA_TRY(c, cudaMemcpyAsync(t->d_blocks, hb.data(), nb * sizeof(DevBlock), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // (H2D on the stream the kernels run on: see remap_to_union)
    CUDA_TRY(c, cudaMemcpyAsync(t->d_cols, t->cols.data(), nb * (size_t)t->ncols * sizeof(DevCol), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // (H2D on the stream the kernels run on: see remap_to_union)
  }
  if (!t->segs.empty()) {
    if (t->segs.size() > t->d_segs_cap) {
      if (t->d_segs) cudaFree(t->d_segs);
      t->d_segs = nullptr;
      const size_t cap = std::max<size_t>(t->segs.size() * 2, 256);
      CUDA_TRY(c, cudaMalloc(&t->d_segs, cap * sizeof(DevCol)));
      t->d_segs_cap = cap;
    }
    CUDA_TRY(c, cudaMemcpyAsync(t->d_segs, t->segs.data(), t->segs.size() * sizeof(DevCol), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  }
  if (!t->pending_stats.empty()) {
    // exact extents of the newly staged value-array int columns (one more read of those
    // arrays from HBM, once per staging): they select the 32-bit / check-free kernel paths
    uint32_t* d_items = nullptr;
    size_t n = t->pending_stats.size();
    // items (u32) then, 8-byte aligned, where each item's codes go
    const size_t codes_off = align_up(n * 4, 8);
    CUDA_TRY(c, pool_alloc(c, (void**)&d_items, codes_off + n * 8));
    const unsigned long long* d_codes = reinterpret_cast<const unsigned long long*>(reinterpret_cast<char*>(d_items) + codes_off);
    CUDA_TRY(c, cudaMemcpyAsync(d_items, t->pending_stats.data(), n * 4, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync((void*)d_codes, t->pending_codes.data(), n * 8, cudaMemcpyHostToDevice, c->stream));
    int rc = w16::launch_stats(t->d_cols, t->d_blocks, d_items, d_codes, (uint32_t)n, (uint32_t)t->ncols, c->stream);
    if (rc != 0) {
      c->set_err(std::string("stats kernel launch: ") + cudaGetErrorString((cudaError_t)rc));
      pool_release(c, d_items);
      return SG_ERR_CUDA;
    }
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    CUDA_TRY(c, cudaMemcpy(t->cols.data(), t->d_cols, nb * (size_t)t->ncols * sizeof(DevCol), cudaMemcpyDeviceToHost));
    pool_release(c, d_items);
    t->pending_stats.clear();
    t->pending_codes.clear();
    t->stats_launches++;
  }
  t->dirty = false;
  return SG_OK;
}

// Build the dense slot space and the device plan from the table's dictionaries.
// accumulator layout for `nslots` dense slots: one SUM region (scalars | count | per agg hcount,
// sum | per agg buckets) followed by one MAX region (per agg vmax): the cross-GPU merge is two
// all-reduces
__global__ void fill_ll(long long* p, size_t n, long long v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// Group-by on an int column that is value-array encoded in some blocks (more than
// CARDINALITY_THRESHOLD distinct values there, column_store_io.go:82-113): the dense slot space needs
// a table-wide value dictionary.  The blocks' distinct values are collected on the GPU (one pass over
// each such block's array, once), joined into the column's IntDict (ascending, so the numbering does
// not depend on the hash order), and a device open-addressing table value -> code is (re)built.
int ensure_value_dict(sg_table* t, int col) {
  sg_ctx* c = t->ctx;
  auto& vh = t->vhash[(size_t)col];
  IntDict& D = t->idict[(size_t)col];
  const size_t nb = t->blocks.size();
  std::vector<uint32_t> items;
  for (size_t b = vh.blocks_done; b < nb; b++) {
    const DevCol& dc = t->cols[b * (size_t)t->ncols + (size_t)col];
    if (dc.enc == SG_ENC_VALUES && !(dc.flags & (COL_IS_STR | COL_BROKEN))) items.push_back((uint32_t)(b * (size_t)t->ncols + (size_t)col));
  }
  if (!items.empty()) {
    const uint32_t cap = (uint32_t)(INT_DICT_CAP * 2);  // load factor <= 1/2 at the dictionary's size limit
    PoolTmp tk(c), ti(c), tc(c);
    CUDA_TRY(c, pool_alloc(c, &tk.p, (size_t)cap * 8));
    CUDA_TRY(c, pool_alloc(c, &ti.p, items.size() * 4));
    CUDA_TRY(c, pool_alloc(c, &tc.p, 16));
    long long* d_keys = (long long*)tk.p;
    uint32_t* d_items = (uint32_t*)ti.p;
    unsigned int* d_cnt = (unsigned int*)tc.p;
    fill_ll<<<(unsigned)(((size_t)cap + 255) / 256), 256, 0, c->stream>>>(d_keys, cap, INT64_MIN);
    CUDA_TRY(c, cudaMemsetAsync(d_cnt, 0, 16, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(d_items, items.data(), items.size() * 4, cudaMemcpyHostToDevice, c->stream));
    int rc = w16::launch_distinct(t->d_cols, t->d_blocks, d_items, (uint32_t)items.size(), (uint32_t)t->ncols, d_keys, cap - 1u, d_cnt,
                             c->stream);
    if (rc != 0) {
      c->set_err(std::string("distinct kernel launch: ") + cudaGetErrorString((cudaError_t)rc));
      return SG_ERR_CUDA;
    }
    unsigned int cnt[4] = {0, 0, 0, 0};
    CUDA_TRY(c, cudaMemcpyAsync(cnt, d_cnt, 16, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    std::vector<int64_t> found;
    if (!cnt[2]) {
      std::vector<long long> keys(cap);
      CUDA_TRY(c, cudaMemcpy(keys.data(), d_keys, (size_t)cap * 8, cudaMemcpyDeviceToHost));
      found.reserve(cnt[0] + 1);
      for (uint32_t i = 0; i < cap; i++)
        if (keys[i] != INT64_MIN) found.push_back(keys[i]);
      if (cnt[1]) found.push_back(INT64_MIN);
    }
    if (cnt[2]) {
      D.overflow = true;
    } else {
      std::sort(found.begin(), found.end());
      for (int64_t v : found) D.intern(v);
    }
    vh.blocks_done = nb;
  }
  if (D.overflow) {
    c->set_err("query: group-by int column has more distinct values than the dense slot space holds");
    return SG_ERR_UNSUPPORTED;
  }
  if (vh.dict_size != D.vals.size() || !vh.d_keys) {
    uint32_t cap = 1024;
    while ((size_t)cap < D.vals.size() * 2 + 2) cap <<= 1;
    std::vector<long long> keys(cap, 0);
    std::vector<uint32_t> ids(cap, 0xffffffffu);
    for (size_t i = 0; i < D.vals.size(); i++) {
      uint32_t h = vh_hash((long long)D.vals[i]) & (cap - 1u);
      while (ids[h] != 0xffffffffu) h = (h + 1u) & (cap - 1u);
      keys[h] = (long long)D.vals[i];
      ids[h] = (uint32_t)i;
    }
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // no query is using the old table
    if (vh.d_keys) cudaFree(vh.d_keys);
    if (vh.d_ids) cudaFree(vh.d_ids);
    vh.d_keys = nullptr;
    vh.d_ids = nullptr;
    CUDA_TRY(c, cudaMalloc((void**)&vh.d_keys, (size_t)cap * 8));
    CUDA_TRY(c, cudaMalloc((void**)&vh.d_ids, (size_t)cap * 4));
    CUDA_TRY(c, cudaMemcpyAsync(vh.d_keys, keys.data(), (size_t)cap * 8, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // (H2D on the stream the kernels run on: see remap_to_union)
    CUDA_TRY(c, cudaMemcpyAsync(vh.d_ids, ids.data(), (size_t)cap * 4, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // (H2D on the stream the kernels run on: see remap_to_union)
    vh.mask = cap - 1u;
    vh.dict_size = D.vals.size();
  }
  return SG_OK;
}

// The accumulator array: SCALAR_WORDS scalars (SC_* in sg_internal.h), then per slot regions in this order: count,
// the exact sums, the hist Counts, the bucket counters (all added when merged or folded: the SUM region), then the
// max above info_max (the MAX region).  q->regions lists them; the off_* members name them one by one.
constexpr uint64_t ACC_LIMIT_BYTES = (uint64_t)24 << 30;
// bytes of the SUM region (scalars | count | sums | hist Counts | bucket counters) for nslots slots: what the
// 24 GiB limit of layout_accumulators is taken on
static uint64_t sum_region_bytes(const sg_query* q, uint64_t nslots) {
  uint64_t per_slot = 1 + 2 * (uint64_t)q->layouts.size();
  for (const auto& L : q->layouts) per_slot += L.nvals_total;
  return (SCALAR_WORDS + nslots * per_slot) * 8;
}
int layout_accumulators(sg_query* q, uint32_t nslots) {
  const int naggs = (int)q->layouts.size();
  size_t words = SCALAR_WORDS;
  q->off_hcount.clear();
  q->off_sum.clear();
  q->off_vmax.clear();
  q->off_buckets.clear();
  q->regions.clear();
  auto region = [&](uint32_t per_row, bool is_max) {
    const size_t off = words;
    if (per_row) q->regions.push_back({off, per_row, is_max});
    words += (size_t)nslots * per_row;
    return off;
  };
  q->off_count = region(1, false);
  // all sums, then all hist Counts: when every hist Count equals Count (hc_is_count) and no buckets exist,
  // scalars | count | sums is all a result needs and it is one contiguous prefix of the array
  for (int i = 0; i < naggs; i++) q->off_sum.push_back(region(1, false));
  q->prefix_words = words;
  for (int i = 0; i < naggs; i++) q->off_hcount.push_back(region(1, false));
  for (int i = 0; i < naggs; i++) {
    q->off_buckets.push_back(region(q->layouts[(size_t)i].nvals_total, false));
    if (words * 8 > ACC_LIMIT_BYTES) {
      q->ctx->set_err("query: accumulators exceed 24 GiB (groups x histogram buckets); needs sparse group "
                      "accumulators (sg_query_set_sparse_groups)");
      return SG_ERR_UNSUPPORTED;
    }
  }
  q->sum_words = words;
  for (int i = 0; i < naggs; i++) q->off_vmax.push_back(region(1, true));
  q->acc_words = words;
  return SG_OK;
}

// time bucket code of the kernel (sg_kernels.cu time_code): 1.. dense index, 0 = off the planned axis
static uint32_t host_time_code(const Plan& P, int64_t v) {
  const int64_t qv = v / P.time_bucket - P.time_first;
  if (qv < 0 || qv >= (int64_t)(P.time_radix - 1)) return 0u;
  return (uint32_t)qv + 1u;
}

// `list`: the blocks the launch will scan (zone-map pruned); the slot window, the filters' fail mode
// and the histogram cache are chosen from their column descriptors
int make_plan(sg_query* q, const std::vector<uint32_t>& list) {
  sg_ctx* c = q->ctx;
  sg_table* t = q->table;
  Plan& P = q->plan;
  memset(&P, 0, sizeof(P));
  q->hashg = false;
  P.nfilters = (int32_t)q->filters.size();
  // Weighted queries (OPTS.WEIGHT_COL, aggregate.go:68,100-102,202-203; hist_basic.go:111-151): Count += weight,
  // hist Count += weight, Values[bucket] += weight, mean weighted.  All of these are linear in the weight, so the
  // scan groups by the weight VALUE as one more (hidden, last) axis — the ordinary int group-by — and the host
  // folds that axis away with a multiplication per slot (dense_fold).  Rows WITHOUT the weight column reuse the
  // previous row's weight in the reference (Q13): with weight_carry the scan fills their digit of the weight axis
  // forward from the nearest earlier row of the block (a row with no such row keeps code 0: weight 1); without it
  // such a query is refused when the result is built.
  q->pgroups = q->groups;
  const bool weighted = q->d.weight_col_slot >= 0;
  P.wcarry = weighted && q->d.weight_carry == 1 ? 1u : 0u;
  if (weighted) {
    if (q->d.weight_col_slot >= t->ncols || t->types[(size_t)q->d.weight_col_slot] != SG_COL_INT) {
      c->set_err("query: the weight column must be an int column");
      return SG_ERR_INVALID;
    }
    if (q->pgroups.size() >= SG_MAX_GROUPS) {
      c->set_err("query: a weighted query takes one group axis: at most SG_MAX_GROUPS - 1 group columns");
      return SG_ERR_UNSUPPORTED;
    }
    sg_group_desc wg;
    wg.col_slot = q->d.weight_col_slot;
    wg.col_type = SG_COL_INT;
    q->pgroups.push_back(wg);
  }
  P.ngroups = (int32_t)q->pgroups.size();
  P.naggs = (int32_t)q->aggs.size();
  P.ncolslots = t->ncols;
  P.hist_mode = q->d.op_mode == SG_MODE_HIST;
  const bool time_mode = q->d.time_col_slot >= 0 && q->d.time_bucket > 0;
  P.time_col = time_mode ? q->d.time_col_slot : -1;

  auto col_ok = [&](int col) { return col >= 0 && col < t->ncols; };
  // ---- slot space ------------------------------------------------------------
  q->dims.clear();
  uint64_t stride = 1;
  for (size_t i = 0; i < q->pgroups.size(); i++) {
    GroupDim gd;
    gd.col = q->pgroups[i].col_slot;
    gd.is_weight = weighted && i + 1 == q->pgroups.size();
    if (!col_ok(gd.col)) {
      c->set_err("query: group column out of range");
      return SG_ERR_INVALID;
    }
    if (t->types[(size_t)gd.col] == SG_COL_SET) {
      c->set_err("query: a set column cannot be grouped by (aggregate.go:125-143 reads Ints / Strs only)");
      return SG_ERR_INVALID;
    }
    gd.is_str = t->types[(size_t)gd.col] == SG_COL_STR;
    if (!gd.is_str && t->has_values_int[(size_t)gd.col]) {
      int rc = ensure_value_dict(t, gd.col);
      if (rc != SG_OK) return rc;
      const auto& vh = t->vhash[(size_t)gd.col];
      P.groups[i].vh_keys = vh.d_keys;
      P.groups[i].vh_ids = vh.d_ids;
      P.groups[i].vh_mask = vh.mask;
      q->hashg = true;
    } else if (!gd.is_str && t->idict[(size_t)gd.col].overflow) {
      c->set_err("query: group-by int column has more distinct values than the dense slot space holds");
      return SG_ERR_UNSUPPORTED;
    }
    uint64_t card = gd.is_str ? t->sdict[(size_t)gd.col].strs.size() : t->idict[(size_t)gd.col].vals.size();
    gd.radix = (uint32_t)(card + 1);
    gd.stride = (uint32_t)stride;
    stride *= gd.radix;
    if (stride > MAX_CODE_SPACE) {
      c->set_err("query: group-by cardinality product exceeds 2^31 (the hashed slot space keys 31-bit codes)");
      return SG_ERR_UNSUPPORTED;
    }
    q->dims.push_back(gd);
    P.groups[i].col = gd.col;
    P.groups[i].is_str = gd.is_str;
    P.groups[i].stride = gd.stride;
    P.groups[i].radix = gd.radix;
    // a key that renders like a missing value is the missing group (DESIGN.md §7): the int -1 and the string ""
    // take code 0.  Not on the weight axis (a weight of -1 multiplies), nor on a StrReplace column (its rewritten
    // strings are folded on the host)
    P.groups[i].alias = -1;
    if (gd.is_str && !gd.is_weight && !q->repl.count(gd.col)) {
      P.groups[i].alias = t->sdict[(size_t)gd.col].find(std::string());
    } else if (!gd.is_str && !gd.is_weight) {
      const auto& m = t->idict[(size_t)gd.col].map;
      const auto it = m.find(-1);
      if (it != m.end()) P.groups[i].alias = it->second;
    }
  }
  if (time_mode) {
    if (!col_ok(P.time_col) || t->types[(size_t)P.time_col] != SG_COL_INT) {
      c->set_err("query: time column must be an int column");
      return SG_ERR_INVALID;
    }
    // extents: the query's table IntInfo widened by the staged block infos
    int64_t tmin = q->d.time_min, tmax = q->d.time_max;
    for (auto& hb : t->blocks)
      for (auto& ii : hb.info)
        if (ii.col_slot == P.time_col) {
          tmin = std::min(tmin, ii.min);
          tmax = std::max(tmax, ii.max);
        }
    if (tmax < tmin) {
      c->set_err("query: time_max < time_min");
      return SG_ERR_INVALID;
    }
    P.time_bucket = q->d.time_bucket;
    P.time_first = tmin / P.time_bucket;
    int64_t nb = tmax / P.time_bucket - P.time_first + 1;
    if (nb <= 0 || nb > (int64_t)MAX_SLOTS || (uint64_t)nb * stride > MAX_CODE_SPACE) {
      c->set_err("query: time axis too large for the slot space");
      return SG_ERR_UNSUPPORTED;
    }
    P.time_radix = (uint32_t)nb + 1;
    P.time_stride = (uint32_t)stride;
    GroupDim gd;
    gd.col = P.time_col;
    gd.is_time = true;
    gd.radix = P.time_radix;
    gd.stride = P.time_stride;
    q->dims.push_back(gd);
    stride *= P.time_radix;
  }
  P.nslots = (uint32_t)stride;

  // ---- aggregations ----------------------------------------------------------------
  // accumulator layout: one SUM region (scalars | count | per agg hcount, sum | per agg buckets)
  // followed by one MAX region (per agg vmax): the cross-GPU merge is two all-reduces
  q->layouts.clear();
  for (int i = 0; i < P.naggs; i++) {
    const sg_agg_desc& a = q->aggs[(size_t)i];
    if (!col_ok(a.col_slot)) {
      c->set_err("query: aggregation column out of range");
      return SG_ERR_INVALID;
    }
    HistLayout L;
    if (!make_layout(a.info_min, a.info_max, P.hist_mode != 0, q->d.hist_kind == SG_HIST_MULTI, q->d.hist_bucket, L)) {
      c->set_err("query: IntInfo extents give no usable histogram layout");
      return SG_ERR_INVALID;
    }
    q->layouts.push_back(L);
    KAgg& ka = P.aggs[i];
    ka.col = a.col_slot;
    ka.info_min = a.info_min;
    ka.info_max = a.info_max;
    ka.reject_hi = wmul10(a.info_max);
    ka.nsub = (int32_t)L.subs.size();
    ka.multi = q->d.hist_kind == SG_HIST_MULTI ? 1u : 0u;
    ka.nvals_total = L.nvals_total;
    for (size_t s = 0; s < L.subs.size(); s++) ka.sub[s] = L.subs[s];
  }

  // ---- hashed slot space: more codes than dense slots.  The table gets twice as many entries as rows can make
  // groups (every scanned row its own group at worst), within [2^16, 2^26]; a table that fills up fails the query.
  q->code_space = stride;
  // tests: SG_FORCE_HASHED_SLOTS=1 takes the hashed slot space at any size (it must give what the dense one gives);
  // SG_HASH_CAP_LOG2=n caps its table at 2^n entries, so that a table that fills up can be reached with few rows
  bool hashed = (stride > (uint64_t)MAX_SLOTS || getenv("SG_FORCE_HASHED_SLOTS")) && !getenv("SG_NO_HASHED_SLOTS");
  uint64_t cap = 0;
  {
    uint64_t rows = 0;
    for (uint32_t b : list) rows += t->blocks[b].num_records;
    uint64_t cap_max = (uint64_t)MAX_SLOTS;
    if (const char* e = getenv("SG_HASH_CAP_LOG2")) cap_max = (uint64_t)1 << std::min(std::max(atoi(e), 4), 26);
    cap = std::min<uint64_t>((uint64_t)1 << 16, cap_max);
    while (cap < 2 * std::min<uint64_t>(rows, stride) && cap < cap_max) cap <<= 1;
  }
  // ---- sparse group accumulators (sg_query_set_sparse_groups): a plan whose accumulators, dense or hashed, pass the
  // 24 GiB limit keys the same table by the row's code, and its accumulators hold only the groups a discovery
  // launch finds.  Plans within the limit are planned as without the flag.
  // tests: SG_FORCE_SPARSE_GROUPS=1 takes the sparse path for every plan while the flag is set
  q->sparse = q->sparse_req == 1 &&
              (getenv("SG_FORCE_SPARSE_GROUPS") || sum_region_bytes(q, hashed ? cap : stride) > ACC_LIMIT_BYTES);
  if (q->sparse) {
    if ((weighted || !q->repl.empty()) && q->hfold_req != 1) {
      c->set_err("query: weights / StrReplace are not combined with sparse group accumulators in this build");
      return SG_ERR_UNSUPPORTED;
    }
    hashed = true;
  }
  q->hashed = hashed;
  // ---- device folds (sg_query_set_hashed_folds): a hashed slot space has no slot per code for dense_fold, so its
  // weight axis and rewritten strings are folded over the table's entries on the device (fold_insert, fold_rows)
  q->dfold = hashed && q->hfold_req == 1 && (weighted || !q->repl.empty());
  if (stride > (uint64_t)MAX_SLOTS && !q->hashed) {
    c->set_err("query: group-by cardinality product exceeds the dense slot space");
    return SG_ERR_UNSUPPORTED;
  }
  q->hcap = 0;
  if (q->hashed) {
    P.nslots = (uint32_t)cap;
    q->hcap = (uint32_t)cap;
  }
  // ---- fail mode: every filter column populates every row of every listed block (value array, or a
  // bucket column whose bins were checked to list each row once) -> one sticky FAIL bit instead of a
  // pass count, and bucket filters walk the failing bins only
  bool fail_mode = P.nfilters > 0 && !getenv("SG_NO_FAIL_MODE");
  // SetFilters (IN / NIN) do not count passes: each owns sticky bits above the pass counter (one for IN: "the set
  // holds the literal"; two for NIN: "the row has a set", "the set holds the literal"); they keep the query in
  // count mode
  uint32_t nset_in = 0, nset_nin = 0;
  for (auto& f : q->filters) {
    if (f.op == SG_OP_IN) nset_in++;
    if (f.op == SG_OP_NIN) nset_nin++;
  }
  const uint32_t ncount = (uint32_t)P.nfilters - nset_in - nset_nin;  // filters that count passes
  const uint32_t sbits = nset_in + 2u * nset_nin;
  if (sbits) fail_mode = false;
  for (size_t i = 0; i < q->filters.size() && fail_mode; i++) {
    const int col = q->filters[i].col_slot;
    if (!col_ok(col)) break;  // reported below
    for (uint32_t b : list) {
      const DevCol& dc = t->cols[(size_t)b * (size_t)t->ncols + (size_t)col];
      if (dc.enc == SG_ENC_BUCKET && !(dc.flags & COL_FULL)) {
        fail_mode = false;
        break;
      }
    }
  }
  P.fail_mode = fail_mode ? (getenv("SG_NO_PUSHDOWN") ? 2u : 1u) : 0u;  // 2: fail bits, but every tile is walked (A/B)
  // ---- slot window over the time axis (see Plan): widest span of time codes inside one listed block
  const uint32_t group_slots = time_mode ? P.time_stride : P.nslots;
  auto window_for = [&](bool windowed) {
    uint32_t win = time_mode ? P.time_radix - 1u : 0u;
    if (time_mode && windowed && !getenv("SG_NO_TIME_WINDOW")) {
      bool ok = true;
      uint32_t w = 1;
      for (uint32_t b : list) {
        const DevCol& dc = t->cols[(size_t)b * (size_t)t->ncols + (size_t)P.time_col];
        if (dc.enc == SG_ENC_ABSENT) continue;
        if (!(dc.flags & COL_STATS) || (dc.flags & COL_IS_STR)) {
          ok = false;
          break;
        }
        const uint32_t c0 = host_time_code(P, dc.vmin), c1 = host_time_code(P, dc.vmax);
        if (!c0 || !c1) {  // rows off the planned axis: the query fails in the kernel's own check
          ok = false;
          break;
        }
        w = std::max(w, c1 - c0 + 1u);
      }
      if (ok && w < win) win = w;
    }
    P.time_win = win;
    P.lslots = time_mode ? group_slots * (win + 1u) : P.nslots;
    P.gbits = bits_for(P.lslots);
  };
  window_for(!q->hashed);
  if (q->hashed) {  // the slot word carries the whole code, then the table index the accumulators are indexed by
    P.lslots = P.nslots;
    P.gbits = bits_for(std::max<uint64_t>(q->code_space, P.nslots));  // (the table outgrows a forced small space)
  }
  P.time_magic = 0;
  if (time_mode && P.time_bucket >= 2 && P.time_bucket < 0x100000000ll)
    P.time_magic = (uint64_t)(((unsigned __int128)1 << 64) / (unsigned __int128)P.time_bucket) + 1u;
  uint32_t fbits = 0, cbits = 0;
  uint32_t sticky_target = 0;  // the sticky bits (relative to gbits + cbits) a passing row shows
  auto slot_layout = [&]() -> int {
    cbits = fail_mode ? 1u : (ncount ? bits_for((uint64_t)ncount + 1) : 0u);
    fbits = cbits + sbits;
    sticky_target = 0;
    for (uint32_t i = 0, k = 0; i < (uint32_t)P.nfilters && P.gbits + fbits <= 32; i++) {
      KFilter& kf = P.filters[i];
      const int op = q->filters[i].op;
      kf.set_pbit = kf.set_tbit = 0;
      if (op == SG_OP_IN) {
        kf.set_tbit = 1u << (P.gbits + cbits + k);
        sticky_target |= 1u << k;
        k += 1;
      } else if (op == SG_OP_NIN) {
        kf.set_pbit = 1u << (P.gbits + cbits + k);
        kf.set_tbit = 1u << (P.gbits + cbits + k + 1);
        sticky_target |= 1u << k;
        k += 2;
      }
    }
    const uint32_t tbit = time_mode ? 1u : 0u;
    const uint32_t total_bits = P.gbits + fbits + tbit;
    if (total_bits > 32) {
      c->set_err("query: slot word wider than 32 bits");
      return SG_ERR_UNSUPPORTED;
    }
    q->slot_bytes = total_bits <= 8 ? 1u : (total_bits <= 16 ? 2u : 4u);
    if (q->hashg || q->hashed) q->slot_bytes = 4;  // these passes exist for 32-bit slot words + global accumulators only
    P.finc = 1u << P.gbits;
    P.filt_mask = (uint32_t)(((uint64_t)1 << fbits) - 1u);
    P.filt_target = fail_mode ? 0u : (ncount | (sticky_target << cbits));
    P.time_ok = time_mode ? (1u << (P.gbits + fbits)) : 0u;
    P.pass_target = P.filt_target | (time_mode ? (1u << fbits) : 0u);
    return SG_OK;
  };
  {
    int rc = slot_layout();
    if (rc != SG_OK) return rc;
  }

  // ---- filters -----------------------------------------------------------------
  for (int i = 0; i < P.nfilters; i++) {
    const sg_filter_desc& f = q->filters[(size_t)i];
    if (!col_ok(f.col_slot)) {
      c->set_err("query: filter column out of range");
      return SG_ERR_INVALID;
    }
    KFilter& kf = P.filters[i];
    kf.col = f.col_slot;
    kf.is_str = t->types[(size_t)f.col_slot] != SG_COL_INT;
    if (f.col_type != t->types[(size_t)f.col_slot]) {
      c->set_err("query: filter type does not match the column's KeyTypes");
      return SG_ERR_INVALID;
    }
    kf.op = f.op;
    kf.ival = f.int_value;
    kf.str_gid = -1;
    kf.lut = nullptr;
    kf.lut_bits = 0;
    if (f.col_type == SG_COL_SET) {
      if (f.op != SG_OP_IN && f.op != SG_OP_NIN) {
        c->set_err("query: op not valid for a set filter");
        return SG_ERR_INVALID;
      }
      // a literal absent from the dictionary is in no row's set (get_val_id hands out a fresh id, filter.go:264)
      kf.str_gid = t->sdict[(size_t)f.col_slot].find(q->filter_strs[(size_t)i]);
      // (its sticky bits: slot_layout)
    } else if (f.op == SG_OP_IN || f.op == SG_OP_NIN) {
      c->set_err("query: IN / NIN are set filter ops");
      return SG_ERR_INVALID;
    } else if (kf.is_str) {
      if (f.op == SG_OP_EQ || f.op == SG_OP_NEQ) {
        kf.str_gid = t->sdict[(size_t)f.col_slot].find(q->filter_strs[(size_t)i]);
      } else if (f.op == SG_OP_RE || f.op == SG_OP_NRE) {
        if (q->lut_bits[(size_t)i] < 0) {
          c->set_err("query: regex filter without sg_query_set_str_lut");
          return SG_ERR_STATE;
        }
        // strings interned after the bitset was built have no bit: the kernel would read them as "no match"
        // (RE drops their rows, NRE keeps them), so a dictionary that grew since needs the bitset set again
        if (q->lut_bits[(size_t)i] < (int64_t)t->sdict[(size_t)f.col_slot].strs.size()) {
          c->set_err("query: filter " + std::to_string(i) + ": the regex bitset covers " +
                     std::to_string(q->lut_bits[(size_t)i]) + " strings, the column's dictionary now holds " +
                     std::to_string(t->sdict[(size_t)f.col_slot].strs.size()) + " (sg_query_set_str_lut again)");
          return SG_ERR_STATE;
        }
        kf.lut = q->d_luts[(size_t)i];
        kf.lut_bits = q->lut_bits[(size_t)i];
      } else {
        c->set_err("query: op not valid for a str filter");
        return SG_ERR_INVALID;
      }
    } else if (f.op > SG_OP_NEQ) {
      c->set_err("query: op not valid for an int filter");
      return SG_ERR_INVALID;
    }
  }

  {
    // sparse plans are laid out for their live groups once the discovery launch has counted them
    int rc = layout_accumulators(q, q->sparse ? 0u : P.nslots);
    if (rc != SG_OK) return rc;
  }

  // ---- histogram cache candidates: BasicHist aggregations the kernel's 32-bit bucket path serves
  // (same test as `hist32` in scan_kernel)
  uint32_t hrow_words = 0;
  for (int i = 0; i < P.naggs; i++) {
    KAgg& ka = P.aggs[i];
    ka.hrow_off = HROW_NONE;
    if (!P.hist_mode || ka.nsub != 1 || getenv("SG_NO_HIST_CACHE")) continue;
    const long long fmin = ka.info_min > 0 ? ka.info_min : 0;
    long long fmax = ka.info_max < 0xffffffffll ? ka.info_max : 0xffffffffll;
    if (ka.reject_hi < fmax) fmax = ka.reject_hi;
    const KSubHist& S = ka.sub[0];
    if (fmax < fmin || S.bsize <= 0 || S.bsize >= 0x100000000ll || S.lo != ka.info_min ||
        (unsigned long long)fmax - (unsigned long long)ka.info_min >= 0x100000000ull)
      continue;
    ka.hrow_off = hrow_words;
    hrow_words += ka.nvals_total;
  }
  P.hist_row_words = hrow_words;

  // ---- shared memory budget ----------------------------------------------------------
  // TMA staging (per warp 4 KiB tiles, 1 or 2 deep) competes with the accumulator replicas and the
  // histogram cache: two stages while 32 replicas and every cache row still fit, else one, else plain loads
  P.acc_words = 1 + 2 * (uint32_t)P.naggs;
  uint32_t slots_b = 0;
  auto acc_bytes = [&](uint32_t repl) -> uint64_t {  // replicas (+ trash slot), high limbs, CTA totals (global slots)
    return ((uint64_t)P.lslots + 1) * P.acc_words * repl * 4 + ((uint64_t)P.lslots + 1) * (uint64_t)P.naggs * 4 + 8 +
           (uint64_t)P.nslots * (1 + 2 * (uint64_t)P.naggs) * 8 + 16;
  };
  const Variant* V = &V16;  // the budget below is taken for this build of the kernel
  auto repl_for = [&](uint32_t nstage) -> uint32_t {
    const uint32_t fixed = V->fixed_smem(nstage) + slots_b;
    if (fixed > V->max_smem) return 0;
    const uint32_t avail = V->max_smem - fixed;
    uint32_t repl = 32;
    while (repl >= 1 && acc_bytes(repl) > avail) repl >>= 1;
    return repl;
  };
  auto hist_rows_for = [&](uint32_t nstage, uint32_t repl) -> uint32_t {
    if (!hrow_words || !repl) return 0;
    const uint64_t used = (uint64_t)V->fixed_smem(nstage) + slots_b + acc_bytes(repl);
    if (used >= V->max_smem) return 0;
    return (uint32_t)std::min<uint64_t>(P.lslots, (V->max_smem - used) / ((uint64_t)hrow_words * 4));
  };
  // (nstage below counts 2 KiB units per warp: 4 = two 4 KiB tiles, 2 = one — or two tiles of a narrow column —,
  // 1 = 2 KiB: one tile of a uint16 / int32 column, two of an int16 one; wide columns then use plain loads)
  bool all_narrow = true;  // every TMA-feedable column the plan reads is stored narrow in every listed block
  {
    std::vector<int> pcols;
    for (int i = 0; i < P.nfilters; i++) pcols.push_back(q->filters[(size_t)i].col_slot);
    for (int i = 0; i < P.ngroups; i++) pcols.push_back(q->pgroups[(size_t)i].col_slot);
    for (int i = 0; i < P.naggs; i++) pcols.push_back(q->aggs[(size_t)i].col_slot);
    if (time_mode) pcols.push_back(P.time_col);
    for (uint32_t b : list) {
      for (int col : pcols) {
        if (col < 0 || col >= t->ncols) continue;
        const DevCol& dc = t->cols[(size_t)b * (size_t)t->ncols + (size_t)col];
        if (dc.enc == SG_ENC_ABSENT || !(dc.flags & COL_TMA)) continue;
        if (dc.enc == SG_ENC_VALUES && (dc.flags & COL_IS_STR)) continue;  // read with plain loads anyway
        if (col_shift(dc.flags) == 0u) all_narrow = false;
      }
      if (!all_narrow) break;
    }
  }
  const char* force_units = getenv("SG_STAGE_UNITS");  // A/B: 0, 1, 2 or 4
  auto pick_units = [&]() -> uint32_t {
    uint32_t u = 0;
    if (t->tma_ok && t->d_tmaps) {
      auto fits = [&](uint32_t x) { return repl_for(x) >= 2 || (repl_for(x) >= 1 && repl_for(0) <= 1); };
      if (repl_for(4) >= 32 && hist_rows_for(4, 32) >= std::min<uint32_t>(P.lslots, hrow_words ? P.lslots : 0u))
        u = 4;
      else if (fits(2))
        u = 2;
      else if (all_narrow && fits(1))
        u = 1;
      // accumulators that cannot live in shared memory at any size (high-cardinality plans): nothing competes
      // with the staging buffers — take the deepest that fits (round 1 left such plans on plain loads)
      if (u == 0 && (q->hashg || repl_for(0) == 0))
        for (uint32_t x : {4u, 2u, 1u})
          if (V->fixed_smem(x) + slots_b <= V->max_smem && (x >= 2 || all_narrow)) {
            u = x;
            break;
          }
      if (force_units) u = (uint32_t)atoi(force_units);
    }
    if (V->fixed_smem(u) + slots_b > V->max_smem) u = 0;
    return u;
  };
  uint32_t nstage = 0, repl = 0;
  for (int attempt = 0; attempt < 2; attempt++) {
    slots_b = q->slot_bytes < 4 ? SG_BLOCK_ROWS * q->slot_bytes : 0u;
    nstage = pick_units();
    repl = (q->hashg || q->hashed) ? 0u : repl_for(nstage);
    if (repl == 0 && time_mode && P.lslots != P.nslots) {
      // accumulators in global memory: no slot window (the kernel's global paths index whole-axis slots)
      window_for(false);
      int rc = slot_layout();
      if (rc != SG_OK) return rc;
      continue;
    }
    break;
  }
  // cache rows are worth more than replicas beyond 4 (a shared reduction costs 2-3 cycles per warp
  // instruction at any replication; a bucket increment that misses the cache costs ~45)
  uint32_t hrows = hist_rows_for(nstage, repl);
  while (hrow_words && repl > 4 && hrows < P.lslots) {
    repl >>= 1;
    hrows = hist_rows_for(nstage, repl);
  }
  // ---- which build runs it.  Two 8-warp CTAs per SM (113 KiB each) beat one 16-warp CTA whenever their
  // shared-memory diet costs nothing that matters: 8-bit (or global) slot words, narrow arrays (2 KiB staging per
  // warp), at least two accumulator replicas, and no histogram row lost that the big CTA would have cached —
  // unless most rows go to L2 either way (then the second CTA overlaps that LSU-bound pass with its own scans).
  q->variant = &V16;
  {
    const char* fv = getenv("SG_VARIANT");  // A/B: 8 or 16
    const uint32_t nstage16 = nstage, repl16 = repl, hrows16 = hrows;
    V = &V8;
    const uint32_t u8 = pick_units();
    const uint32_t r8 = q->hashg ? 0u : repl_for(u8);
    uint32_t rr = r8;
    uint32_t h8 = hist_rows_for(u8, rr);
    while (hrow_words && rr > 2 && h8 < P.lslots) {
      rr >>= 1;
      h8 = hist_rows_for(u8, rr);
    }
    const bool feasible = q->slot_bytes != 2 && V8.ctas >= 2 && V8.fixed_smem(u8) + slots_b <= V8.max_smem &&
                          (repl16 == 0 ? rr == 0 || !P.lslots : rr >= 2) && (u8 >= 1 || !(t->tma_ok && t->d_tmaps));
    const bool hist_l2_bound = hrow_words != 0 && hrows16 < P.lslots;
    bool use8 = feasible && all_narrow && repl16 != 0 && hist_l2_bound;
    if (fv) use8 = feasible && atoi(fv) == 8;
    if (use8) {
      q->variant = &V8;
      nstage = u8;
      repl = repl16 == 0 ? 0u : rr;
      hrows = repl ? h8 : 0u;
    } else {
      V = &V16;
      nstage = nstage16;
      repl = repl16;
      hrows = hrows16;
    }
  }
  q->nstage = nstage;
  P.acc_repl = repl;  // 0: accumulate straight into global memory
  P.hist_rows = hrows;
  q->smem_bytes = V->fixed_smem(nstage) + slots_b + (repl ? (uint32_t)acc_bytes(repl) + hrows * hrow_words * 4 + 16 : 0u);
  return SG_OK;
}

void point_plan(sg_query* q);
int upload_fold(sg_query* q);

int alloc_device(sg_query* q) {
  sg_ctx* c = q->ctx;
  sg_table* t = q->table;
  cudaSetDevice(c->device);
  pool_release(c, q->d_acc);
  q->d_acc = nullptr;
  CUDA_TRY(c, pool_alloc(c, (void**)&q->d_acc, q->acc_words * 8));
  if (!q->d_plan) CUDA_TRY(c, pool_alloc(c, (void**)&q->d_plan, sizeof(Plan)));
  if (!q->d_work) CUDA_TRY(c, pool_alloc(c, (void**)&q->d_work, 64));
  size_t nb = std::max<size_t>(t->blocks.size(), 1);
  q->grid = (c->sm_count > 0 ? c->sm_count : 1) * q->variant->ctas;
  const size_t grid_cap = (size_t)(c->sm_count > 0 ? c->sm_count : 1) * 2;  // per-CTA scratch: sized for either build
  if (nb > q->block_cap) {
    pool_release(c, q->d_block_status);
    pool_release(c, q->d_block_list);
    pool_release(c, q->d_item_mask);
    q->d_block_status = q->d_block_list = q->d_item_mask = nullptr;
    const size_t items_cap = nb + grid_cap * SG_MAX_AGGS;  // tail blocks may split per aggregation
    CUDA_TRY(c, pool_alloc(c, (void**)&q->d_block_status, nb * 4));
    CUDA_TRY(c, pool_alloc(c, (void**)&q->d_block_list, items_cap * 16));  // uint4 {block, mask, NumRecords, -}
    q->block_cap = nb;
  }
  if (!q->d_gbinpay) CUDA_TRY(c, pool_alloc(c, (void**)&q->d_gbinpay, grid_cap * SG_BLOCK_ROWS * 4));
  if (!q->d_gdummy) CUDA_TRY(c, pool_alloc(c, (void**)&q->d_gdummy, grid_cap * 32 * 8));
  if (q->slot_bytes == 4 && !q->d_gslots)
    CUDA_TRY(c, pool_alloc(c, (void**)&q->d_gslots, grid_cap * SG_BLOCK_ROWS * 4));
  pool_release(c, q->d_hkeys);
  q->d_hkeys = nullptr;
  pool_release(c, q->d_hids);
  q->d_hids = nullptr;
  if (q->hashed) CUDA_TRY(c, pool_alloc(c, (void**)&q->d_hkeys, (size_t)q->hcap * 4));
  if (q->sparse) {
    CUDA_TRY(c, pool_alloc(c, (void**)&q->d_hids, (size_t)q->hcap * 8));
    if (!q->d_disc) CUDA_TRY(c, pool_alloc(c, (void**)&q->d_disc, DISC_WORDS * 8));
  }
  if (!q->ev0) {
    CUDA_TRY(c, cudaEventCreate(&q->ev0));
    CUDA_TRY(c, cudaEventCreate(&q->ev1));
  }
  pool_release(c, q->d_samples);
  q->d_samples = nullptr;
  if (q->dfold) {
    int rc = upload_fold(q);
    if (rc != SG_OK) return rc;
    // (a sparse plan's rows are counted by its discovery launch: discover_groups allocates them)
    if (!q->sparse) CUDA_TRY(c, pool_alloc(c, (void**)&q->d_samples, (size_t)q->hcap * 16));
    if (!q->ev2) {
      CUDA_TRY(c, cudaEventCreate(&q->ev2));
      CUDA_TRY(c, cudaEventCreate(&q->ev3));
    }
  }
  point_plan(q);
  return SG_OK;
}

// The plan's canonical key (FoldKey) without its table pointers: the weight axis' multipliers (wmul: code 0 -> 1, then
// the weight dictionary, the union one after a cross-GPU merge) and each rewritten axis' digit -> canonical digit map
// (luts), from the dictionaries and StrReplace classes as they are now.  Refused if those no longer match the plan.
static int build_fold_key(sg_query* q, FoldKey* F, std::vector<int64_t>* wmul, std::vector<uint32_t>* luts) {
  sg_ctx* c = q->ctx;
  *F = FoldKey();
  F->wcarry = q->plan.wcarry;
  for (size_t di = 0; di < q->dims.size(); di++) {
    const GroupDim& d = q->dims[di];
    if (d.is_weight) {
      const std::vector<int64_t>& vals = q->merged ? q->m_ints[di] : q->table->idict[(size_t)d.col].vals;
      if (vals.size() + 1 != (size_t)d.radix) {
        c->set_err("query: the weight column's value dictionary changed under the query");
        return SG_ERR_STATE;
      }
      F->wstride = d.stride;
      F->wradix = d.radix;
      wmul->push_back(1);
      wmul->insert(wmul->end(), vals.begin(), vals.end());
    } else if (d.is_str && q->repl.count(d.col)) {
      const auto& R = q->repl.at(d.col);
      if (R.canon.size() + 1 != (size_t)d.radix || R.strs.size() != R.canon.size()) {
        c->set_err("query: the dictionary of a StrReplace column grew after sg_query_set_str_replace");
        return SG_ERR_STATE;
      }
      F->stride[F->naxes] = d.stride;
      F->radix[F->naxes] = d.radix;
      F->lut[F->naxes] = (uint32_t)luts->size();
      F->naxes++;
      luts->push_back(0);
      for (size_t i = 0; i < R.canon.size(); i++) luts->push_back(R.strs[i].empty() ? 0u : R.canon[i] + 1u);
    }
  }
  return SG_OK;
}

// the device fold's key, its tables copied to d_fold
int upload_fold(sg_query* q) {
  sg_ctx* c = q->ctx;
  FoldKey& F = q->fkey;
  std::vector<int64_t> wmul;
  std::vector<uint32_t> luts;
  const int rc = build_fold_key(q, &F, &wmul, &luts);
  if (rc != SG_OK) return rc;
  const size_t wbytes = wmul.size() * 8, bytes = wbytes + luts.size() * 4;
  pool_release(c, q->d_fold);
  q->d_fold = nullptr;
  CUDA_TRY(c, pool_alloc(c, &q->d_fold, std::max<size_t>(bytes, 8)));
  char* hp = c->scratch(std::max<size_t>(bytes, 8));
  if (!hp) {
    c->set_err("cudaHostAlloc (query scratch) failed");
    return SG_ERR_CUDA;
  }
  memcpy(hp, wmul.data(), wbytes);
  memcpy(hp + wbytes, luts.data(), luts.size() * 4);
  CUDA_TRY(c, cudaMemcpyAsync(q->d_fold, hp, bytes, cudaMemcpyHostToDevice, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // (the scratch is reused by the next launch)
  F.wmul = wmul.empty() ? nullptr : (const int64_t*)q->d_fold;
  F.luts = luts.empty() ? nullptr : (const uint32_t*)((char*)q->d_fold + wbytes);
  return SG_OK;
}

// point the plan at the accumulators
void point_plan(sg_query* q) {
  Plan& P = q->plan;
  P.scalars = q->d_acc;
  P.count = q->d_acc + q->off_count;
  P.block_status = q->d_block_status;
  for (int i = 0; i < P.naggs; i++) {
    P.aggs[i].hcount = q->d_acc + q->off_hcount[(size_t)i];
    P.aggs[i].sum = q->d_acc + q->off_sum[(size_t)i];
    P.aggs[i].vmax = (int64_t*)(q->d_acc + q->off_vmax[(size_t)i]);
    P.aggs[i].vmin = nullptr;
    P.aggs[i].buckets = q->d_acc + q->off_buckets[(size_t)i];
  }
}

// ---- top-K selection on the device (results with very many groups and a limit) ------------------------------
// The order value of a slot as a 64-bit key whose unsigned order is the value's order: Count, or the mean of
// one aggregation (the IEEE double the host computes: sum / hist Count, -inf without a histogram).
struct TopkArgs {
  const uint64_t* acc;
  size_t off_count, off_hc, off_sum;  // of the ordering aggregation (off_hc unused when hc_is_count)
  int order_by;                       // < 0: Count
  int hc_is_count;
  uint32_t nslots;
};
struct TopkTotals {
  unsigned long long live, count, max_key;
  unsigned long long hc[SG_MAX_AGGS], sum[SG_MAX_AGGS];
  unsigned int n_out, overflow;
};
__device__ __forceinline__ unsigned long long topk_key(const TopkArgs& A, uint32_t s, unsigned long long cnt) {
  if (A.order_by < 0) return cnt;
  const unsigned long long hc = A.hc_is_count ? cnt : A.acc[A.off_hc + s];
  const double v = hc ? (double)(long long)A.acc[A.off_sum + s] / (double)(long long)hc : -INFINITY;
  const long long b = __double_as_longlong(v);
  return b < 0 ? ~(unsigned long long)b : ((unsigned long long)b | 0x8000000000000000ull);
}
// pass 0: Cumulative totals of every live slot and the largest key
__global__ void topk_totals(TopkArgs A, int naggs, const size_t* off_hc_all, const size_t* off_sum_all, const int* hc_is_count_all,
                            TopkTotals* tot) {
  unsigned long long live = 0, count = 0, mx = 0;
  unsigned long long hc[SG_MAX_AGGS], sm[SG_MAX_AGGS];
  for (int a = 0; a < naggs; a++) hc[a] = sm[a] = 0;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < A.nslots; s += gridDim.x * blockDim.x) {
    const unsigned long long c = A.acc[A.off_count + s];
    if (!c) continue;
    live++;
    count += c;
    const unsigned long long k = topk_key(A, s, c);
    mx = k > mx ? k : mx;
    for (int a = 0; a < naggs; a++) {
      const unsigned long long h = hc_is_count_all[a] ? c : A.acc[off_hc_all[a] + s];
      if (!h) continue;
      hc[a] += h;
      sm[a] += A.acc[off_sum_all[a] + s];
    }
  }
  for (int d = 16; d > 0; d >>= 1) {
    live += __shfl_xor_sync(0xffffffffu, live, d);
    count += __shfl_xor_sync(0xffffffffu, count, d);
    const unsigned long long o = __shfl_xor_sync(0xffffffffu, mx, d);
    mx = o > mx ? o : mx;
    for (int a = 0; a < naggs; a++) {
      hc[a] += __shfl_xor_sync(0xffffffffu, hc[a], d);
      sm[a] += __shfl_xor_sync(0xffffffffu, sm[a], d);
    }
  }
  if ((threadIdx.x & 31) == 0 && live) {
    atomicAdd(&tot->live, live);
    atomicAdd(&tot->count, count);
    atomicMax(&tot->max_key, mx);
    for (int a = 0; a < naggs; a++) {
      atomicAdd(&tot->hc[a], hc[a]);
      atomicAdd(&tot->sum[a], sm[a]);
    }
  }
}
// one radix digit (`bits` wide at `shift`) of the keys whose higher bits equal `prefix`
__global__ void topk_hist(TopkArgs A, unsigned long long prefix, int shift, int bits, int has_prefix, unsigned int* hist) {
  __shared__ unsigned int sh[2048];
  for (int i = threadIdx.x; i < 2048; i += blockDim.x) sh[i] = 0;
  __syncthreads();
  const unsigned long long mask = (1ull << bits) - 1ull;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < A.nslots; s += gridDim.x * blockDim.x) {
    const unsigned long long c = A.acc[A.off_count + s];
    if (!c) continue;
    const unsigned long long k = topk_key(A, s, c);
    if (has_prefix && (k >> (shift + bits)) != prefix) continue;
    atomicAdd(&sh[(k >> shift) & mask], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 2048; i += blockDim.x)
    if (sh[i]) atomicAdd(&hist[i], sh[i]);
}
// every live slot whose key is >= lower: {slot, count, (hist Count, sum) per aggregation} appended to `rows`
__global__ void topk_emit(TopkArgs A, unsigned long long lower, int naggs, const size_t* off_hc_all, const size_t* off_sum_all,
                          const int* hc_is_count_all, unsigned long long* rows, unsigned int cap, TopkTotals* tot) {
  const int w = 2 + 2 * naggs;
  for (uint32_t s = blockIdx.x * blockDim.x + threadIdx.x; s < A.nslots; s += gridDim.x * blockDim.x) {
    const unsigned long long c = A.acc[A.off_count + s];
    if (!c || topk_key(A, s, c) < lower) continue;
    const unsigned int i = atomicAdd(&tot->n_out, 1u);
    if (i >= cap) {
      tot->overflow = 1u;
      continue;
    }
    unsigned long long* r = rows + (size_t)i * w;
    r[0] = s;
    r[1] = c;
    for (int a = 0; a < naggs; a++) {
      r[2 + 2 * a] = hc_is_count_all[a] ? c : A.acc[off_hc_all[a] + s];
      r[3 + 2 * a] = A.acc[off_sum_all[a] + s];
    }
  }
}

__global__ void fill_i64(int64_t* p, size_t n, int64_t v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

int reset_accumulators(sg_query* q) {
  sg_ctx* c = q->ctx;
  CUDA_TRY(c, cudaMemsetAsync(q->d_acc, 0, q->sum_words * 8, c->stream));
  // (a sparse plan's table was filled by its discovery launch, which cleared it first)
  if (q->hashed && !q->sparse && q->d_hkeys) CUDA_TRY(c, cudaMemsetAsync(q->d_hkeys, 0, (size_t)q->hcap * 4, c->stream));
  if (q->acc_words > q->sum_words) {
    size_t n = q->acc_words - q->sum_words;
    fill_i64<<<(unsigned)((n + 255) / 256), 256, 0, c->stream>>>((int64_t*)(q->d_acc + q->sum_words), n, INT64_MIN);
  }
  CUDA_TRY(c, cudaGetLastError());
  q->launches += (q->acc_words > q->sum_words) ? 1 : 0;
  return SG_OK;
}

int device_fold(sg_query* q, bool discover);

// one launch of the scan kernel over `list`.  discover: the discovery launch of a sparse plan (its scalars go to
// d_disc and are what comes back)
int run_list(sg_query* q, const std::vector<uint32_t>& list, bool discover = false) {
  sg_ctx* c = q->ctx;
  sg_table* t = q->table;
  // Work items.  The blocks of the last, partial wave (n mod #SMs) would leave most SMs idle for a
  // whole block time; when the plan has several aggregations they are split into one item per subset
  // of the aggregations (every item redoes the cheap filter/group passes, one owns the Count).
  std::vector<uint32_t> items(list), masks(list.size(), 0x8000ffffu);
  {
    const size_t grid = (size_t)q->grid, n = list.size();
    const int na = q->plan.naggs;
    const bool force = getenv("SG_FORCE_TAIL_SPLIT") != nullptr;  // tests: split every block
    const size_t r = force ? n : n % grid;
    if (q->plan.acc_repl > 0 && na >= 2 && r > 0 &&
        (force || (n > grid && r * 2 <= grid && !getenv("SG_NO_TAIL_SPLIT")))) {
      const int k = force ? na : (int)std::min<size_t>((size_t)na, grid / r);
      items.resize(n - r);
      masks.resize(n - r);
      for (size_t i = n - r; i < n; i++)
        for (int j = 0; j < k; j++) {
          uint32_t m = 0;
          for (int a = j; a < na; a += k) m |= 1u << a;
          items.push_back(list[i]);
          masks.push_back(m | (j == 0 ? 0x80000000u : 0u));
        }
    }
  }
  // parameters go up from pinned scratch (truly asynchronous); the same scratch later receives the
  // accumulators when they are small
  // small accumulator arrays come back right behind the scan (build_result then needs no further copy) — unless a
  // cross-GPU merge follows, which reads the MERGED array back itself: then only the scalars (broken blocks) do
  const bool merge_follows = c->comm != nullptr && c->nranks > 1;
  // (a folded sparse plan: build_result reads the canonical groups' rows alone)
  const bool whole_back = !discover && !merge_follows && !(q->sparse && q->dfold);
  const size_t acc_back = (whole_back && q->acc_words * 8 <= ((size_t)4 << 20)) ? q->acc_words * 8 : 64;
  const size_t off_items = (sizeof(Plan) + 255) & ~(size_t)255;
  const size_t off_acc = off_items + ((items.size() * 16 + 255) & ~(size_t)255);
  char* hp = c->scratch(off_acc + acc_back);
  if (!hp) {
    c->set_err("cudaHostAlloc (query scratch) failed");
    return SG_ERR_CUDA;
  }
  memcpy(hp, &q->plan, sizeof(Plan));
  const bool items_same = items == q->items_up && masks == q->masks_up && q->fold_version == t->version;
  if (!items.empty() && !items_same) {
    uint32_t* w = (uint32_t*)(hp + off_items);
    for (size_t i = 0; i < items.size(); i++) {
      w[4 * i + 0] = items[i];
      w[4 * i + 1] = masks[i];
      w[4 * i + 2] = (uint32_t)t->blocks[items[i]].num_records;
      w[4 * i + 3] = 0;
    }
    CUDA_TRY(c, cudaMemcpyAsync(q->d_block_list, hp + off_items, items.size() * 16, cudaMemcpyHostToDevice, c->stream));
    q->items_up = items;
    q->masks_up = masks;
  }
  CUDA_TRY(c, cudaMemsetAsync(q->d_work, 0, 64, c->stream));
  CUDA_TRY(c, cudaMemsetAsync(q->d_block_status, 0, std::max<size_t>(t->blocks.size(), 1) * 4, c->stream));
  CUDA_TRY(c, cudaMemcpyAsync(q->d_plan, hp, sizeof(Plan), cudaMemcpyHostToDevice, c->stream));
  LaunchParams lp;
  memset(&lp, 0, sizeof(lp));
  lp.plan = q->d_plan;
  lp.blocks = t->d_blocks;
  lp.cols = t->d_cols;
  lp.segs = t->d_segs;
  lp.items = reinterpret_cast<const uint4*>(q->d_block_list);
  lp.nlist = (uint32_t)items.size();
  lp.slot_bytes = q->slot_bytes;
  lp.work_counter = q->d_work;
  lp.gslots = q->d_gslots;
  lp.gbinpay = q->d_gbinpay;
  lp.gdummy = q->d_gdummy;
  lp.smem_bytes = q->smem_bytes;
  lp.acc_smem = q->plan.acc_repl > 0 ? 1u : 0u;
  lp.stage_units = t->d_tmaps ? q->nstage : 0u;
  lp.dbg = nullptr;
  lp.hashg = q->hashg ? 1u : 0u;
  lp.hkeys = q->hashed ? q->d_hkeys : nullptr;
  lp.hmask = q->hashed ? q->hcap - 1u : 0u;
  lp.hids = q->sparse && !discover ? q->d_hids : nullptr;
  lp.hdisc = discover ? 1u : 0u;
  // Deferred fold: the replicated 32-bit accumulators of up to fold_every consecutive blocks are
  // folded together.  Needs one encoding per aggregation column across the listed blocks (word0
  // counts accepted rows for bucket columns, rejected ones for value arrays) and keeps the hot
  // path's no-carry proof: fast-range max x rows one replica can receive x fold_every < 2^32.
  lp.fold_every = 1;
  if (items_same) {
    lp.fold_every = q->fold_every;
  } else if (q->plan.acc_repl > 0 && !list.empty() && !getenv("SG_NO_DEFER_FOLD")) {
    bool uniform = true;
    for (int a = 0; a < q->plan.naggs && uniform; a++) {
      const size_t col = (size_t)q->plan.aggs[a].col;
      const uint32_t enc0 = t->cols[(size_t)list[0] * (size_t)t->ncols + col].enc;
      for (uint32_t b : list)
        if (t->cols[(size_t)b * (size_t)t->ncols + col].enc != enc0) {
          uniform = false;
          break;
        }
    }
    if (q->plan.lslots != q->plan.nslots) uniform = false;  // a moving slot window folds block by block
    if (uniform) {
      const unsigned long long rows = (unsigned long long)SG_BLOCK_ROWS / q->plan.acc_repl;
      unsigned long long k = 4;
      for (int a = 0; a < q->plan.naggs; a++) {
        const KAgg& ka = q->plan.aggs[a];
        const long long fmin = ka.info_min > 0 ? ka.info_min : 0;
        long long fmax = ka.info_max < 0xffffffffll ? ka.info_max : 0xffffffffll;
        if (ka.reject_hi < fmax) fmax = ka.reject_hi;
        if (fmax < fmin || fmax <= 0) continue;
        const unsigned long long per_block = (unsigned long long)fmax * rows;
        if (per_block >= 0x100000000ull) continue;  // never carry-free: the carry path is exact for any k
        k = std::min<unsigned long long>(k, 0xffffffffull / per_block);
      }
      lp.fold_every = (uint32_t)std::max<unsigned long long>(k, 1);
    }
  }
  q->fold_every = lp.fold_every;
  q->fold_version = t->version;
  static const bool phase_timing = getenv("SG_PHASE_TIMING") != nullptr;
  unsigned long long* d_dbg = nullptr;
  if (phase_timing) {
    if (pool_alloc(c, (void**)&d_dbg, (size_t)q->grid * 16 * 8) == cudaSuccess) {
      cudaMemsetAsync(d_dbg, 0, (size_t)q->grid * 16 * 8, c->stream);
      lp.dbg = d_dbg;
    }
  }
  lp.tmaps = lp.stage_units ? t->d_tmaps : nullptr;
  // SG_PLAN_TRACE=1: one line per launch on stderr, so a test can see which path it reached (a sparse plan: one per
  // aggregation launch)
  if (getenv("SG_PLAN_TRACE") && !discover) {
    const Plan& P = q->plan;
    // (the slot word: gbits group bits, fbits pass-counter / fail and set-filter bits, tbit time bit)
    // count_bins: listed blocks whose group Count the kernel takes from bin sizes (its count_in_group conditions)
    uint32_t count_bins = 0;
    if (P.acc_repl > 0 && P.nfilters == 0 && P.time_col < 0 && P.ngroups == 1)
      for (uint32_t b : list) {
        const DevCol& dc = t->cols[(size_t)b * (size_t)t->ncols + (size_t)P.groups[0].col];
        count_bins += dc.enc == SG_ENC_BUCKET && (dc.flags & COL_FULL) ? 1u : 0u;
      }
    // codes: plan columns (filters, groups, the time column, aggregations) with per-row codes (COL_CODES) in some listed block
    std::vector<int32_t> pcols;
    for (int i = 0; i < P.nfilters; i++) pcols.push_back(P.filters[i].col);
    for (int i = 0; i < P.ngroups; i++) pcols.push_back(P.groups[i].col);
    if (P.time_col >= 0) pcols.push_back(P.time_col);
    for (int i = 0; i < P.naggs; i++) pcols.push_back(P.aggs[i].col);
    uint32_t ncodes = 0;
    for (int32_t col : pcols) {
      bool any = false;
      for (uint32_t b : list) any = any || (t->cols[(size_t)b * (size_t)t->ncols + (size_t)col].flags & COL_CODES) != 0u;
      ncodes += any ? 1u : 0u;
    }
    // wcarry: listed blocks whose weight column the kernel fills forward over unlisted rows
    uint32_t wcarry = 0;
    if (P.wcarry)
      for (uint32_t b : list)
        wcarry += weight_needs_carry(t->cols[(size_t)b * (size_t)t->ncols + (size_t)P.groups[P.ngroups - 1].col],
                                     (uint32_t)t->blocks[b].num_records) ? 1u : 0u;
    fprintf(stderr, "sg_plan: build=%s slot_bytes=%u acc_repl=%u fold_every=%u fail_mode=%u hist_rows=%u lslots=%u nslots=%u hashed=%d"
            " hashg=%d gbits=%u fbits=%d tbit=%d count_bins=%u codes=%u wcarry=%u",
            q->variant->name, q->slot_bytes, P.acc_repl, lp.fold_every, P.fail_mode, P.hist_rows, P.lslots, P.nslots,
            q->hashed ? 1 : 0, q->hashg ? 1 : 0, P.gbits, __builtin_popcount(P.filt_mask), P.time_ok ? 1 : 0, count_bins, ncodes,
            wcarry);
    for (int i = 0; i < P.nfilters; i++) {  // per set filter: the most segments its column has in a listed block
      if (P.filters[i].op != SG_OP_IN && P.filters[i].op != SG_OP_NIN) continue;
      uint32_t segs = 0;
      for (uint32_t b : list) {
        const DevCol& dc = t->cols[(size_t)b * (size_t)t->ncols + (size_t)P.filters[i].col];
        if (dc.enc == SG_ENC_BUCKET)
          segs = std::max(segs, (dc.flags & COL_SEGS) ? 1u + (uint32_t)((uint64_t)dc.vmax >> 32) : 1u);
      }
      fprintf(stderr, " set_segs=%u", segs);
    }
    for (int a = 0; a < P.naggs; a++) {
      // the same expressions as scan_kernel's fast range, `hist32` and `nocarry` (R = acc_repl there)
      const KAgg& ka = P.aggs[a];
      const long long fmin = ka.info_min > 0 ? ka.info_min : 0;
      long long fmax = ka.info_max < 0xffffffffll ? ka.info_max : 0xffffffffll;
      if (ka.reject_hi < fmax) fmax = ka.reject_hi;
      const bool fast_any = P.acc_repl > 0 && fmax >= fmin;
      const bool hist32 = ka.nsub == 1 && ka.sub[0].bsize > 0 && ka.sub[0].bsize < 0x100000000ll && ka.sub[0].lo == ka.info_min &&
                          fast_any && (unsigned long long)fmax - (unsigned long long)ka.info_min < 0x100000000ull;
      const bool nocarry = fast_any && (unsigned long long)fmax * (unsigned long long)(SG_BLOCK_ROWS / P.acc_repl) * lp.fold_every <
                                           0x100000000ull;
      fprintf(stderr, " agg%d=[fmin=%lld fmax=%lld hist32=%d nocarry=%d]", a, fmin, fmax, hist32 ? 1 : 0, nocarry ? 1 : 0);
    }
    if (q->sparse) fprintf(stderr, " sparse=1 live=%u table=%u", P.nslots, q->hcap);
    if (q->dfold) fprintf(stderr, " fold=1");
    fprintf(stderr, "\n");
  }
  int grid = (int)std::min<size_t>((size_t)q->grid, std::max<size_t>(items.size(), 1));
  CUDA_TRY(c, cudaEventRecord(q->ev0, c->stream));
  int rc = q->variant->launch(lp, grid, c->stream);
  if (rc != 0) {
    c->set_err(std::string("scan kernel launch: ") + cudaGetErrorString((cudaError_t)rc));
    return SG_ERR_CUDA;
  }
  CUDA_TRY(c, cudaEventRecord(q->ev1, c->stream));
  if (q->dfold) {  // after the last scan of the run and before anything is read back
    rc = device_fold(q, discover);
    if (rc != SG_OK) return rc;
  }
  if (acc_back == q->acc_words * 8) {
    rc = read_acc(q, q->acc, q->d_acc, q->acc_words, PIN_WHOLE_FROM, hp + off_acc);
    if (rc != SG_OK) return rc;
    memcpy(q->scal, q->acc.data(), sizeof(q->scal));
  } else {
    q->acc.words = 0;
    CUDA_TRY(c, cudaMemcpyAsync(hp + off_acc, discover ? q->d_disc : q->d_acc, acc_back, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    memcpy(q->scal, hp + off_acc, sizeof(q->scal));
  }
  q->d2h_bytes += (int64_t)acc_back;
  float ms = 0;
  CUDA_TRY(c, cudaEventElapsedTime(&ms, q->ev0, q->ev1));
  q->kernel_ms += ms;
  if (discover) q->disc_ms = ms;
  q->launches += 1;
  if (q->dfold) {
    float ims = 0, fms = 0;
    CUDA_TRY(c, cudaEventElapsedTime(&ims, q->ev1, q->ev2));
    CUDA_TRY(c, cudaEventElapsedTime(&fms, q->ev2, q->ev3));
    q->kernel_ms += ims + fms;
    if (discover || !q->sparse) q->insert_ms = ims;
    q->fold_ms = fms;
    if (!discover && getenv("SG_PLAN_TRACE"))
      fprintf(stderr, "sg_fold: entries=%llu canon=%llu insert_ms=%.4f fold_ms=%.4f\n",
              (unsigned long long)q->scal[SC_FOLD_ENTRIES], (unsigned long long)q->scal[SC_FOLD_CANON], q->insert_ms,
              q->fold_ms);
  }
  if (d_dbg) {
    std::vector<unsigned long long> hd((size_t)q->grid * 16);
    cudaMemcpy(hd.data(), d_dbg, hd.size() * 8, cudaMemcpyDeviceToHost);
    unsigned long long tot[16] = {0}, mx = 0;
    for (int g = 0; g < q->grid; g++) {
      unsigned long long sum = 0;
      for (int i = 0; i < 16; i++) {
        tot[i] += hd[(size_t)g * 16 + i];
        if (i < 7) sum += hd[(size_t)g * 16 + i];
      }
      mx = std::max(mx, sum);
    }
    fprintf(stderr, "[sg phase cycles avg/CTA] init %llu filters %llu groups %llu time %llu aggs %llu flush %llu fetch %llu | warp0 value-pass waits: tma %llu lookback %llu | max CTA total %llu (kernel %.3f ms)\n",
            tot[0] / q->grid, tot[1] / q->grid, tot[2] / q->grid, tot[3] / q->grid, tot[4] / q->grid, tot[5] / q->grid,
            tot[6] / q->grid, tot[7] / q->grid, tot[8] / q->grid, mx, ms);
    if (tot[9] | tot[10] | tot[11] | tot[12] | tot[13])  // per column pass in plan order (filters, groups, time, aggregations)
      fprintf(stderr, "[sg pass cycles avg/CTA] %llu %llu %llu %llu %llu %llu %llu\n", tot[9] / q->grid, tot[10] / q->grid,
              tot[11] / q->grid, tot[12] / q->grid, tot[13] / q->grid, tot[14] / q->grid, tot[15] / q->grid);
    pool_release(c, d_dbg);
  }
  return SG_OK;
}

__host__ __device__ __forceinline__ uint32_t canon_code(const FoldKey& F, uint32_t code) {
  uint32_t out = code;
#pragma unroll
  for (uint32_t a = 0; a < SG_MAX_GROUPS; a++) {  // (unrolled: the parameter arrays stay out of local memory)
    if (a >= F.naxes) break;
    const uint32_t d = (code / F.stride[a]) % F.radix[a];
    out += (F.luts[F.lut[a] + d] - d) * F.stride[a];  // (mod 2^32: the result is a code again)
  }
  if (F.wradix) out -= ((code / F.wstride) % F.wradix) * F.wstride;
  return out;
}

// Dense ids of the sparse path: every occupied entry of the table gets an id in 0..L-1 (in no set order: the result
// orders its groups itself), id2key[id] = the entry's key (code + 1), *live = L.  One warp-aggregated atomic per warp
// and step; the launch runs after every insert of the discovery launch is done.  pick (device folds): 1 numbers the
// canonical entries only, 2 the others, continuing from *live; 0 every entry.
__global__ void assign_ids(const uint32_t* __restrict__ keys, uint32_t cap, uint32_t* __restrict__ ids,
                           uint32_t* __restrict__ id2key, unsigned int* live, FoldKey F, int pick) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t base = blockIdx.x * blockDim.x; base < cap; base += stride) {
    const uint32_t i = base + threadIdx.x;
    uint32_t k = i < cap ? keys[i] : 0u;
    if (k != 0u && pick != 0 && (canon_code(F, k - 1u) == k - 1u) != (pick == 1)) k = 0u;
    const unsigned m = __ballot_sync(0xffffffffu, k != 0u);
    if (!m) continue;
    const int lane = (int)(threadIdx.x & 31u);
    unsigned first = 0;
    if (lane == __ffs((int)m) - 1) first = atomicAdd(live, (unsigned)__popc(m));
    first = __shfl_sync(0xffffffffu, first, __ffs((int)m) - 1);
    if (k != 0u) {
      const uint32_t id = first + (uint32_t)__popc(m & ((1u << lane) - 1u));
      ids[i] = id;
      id2key[id] = k;
    }
  }
}

// ---- device folds (sg_query_set_hashed_folds) ------------------------------------------------------------------
// Canonical insert: every occupied entry whose key is not canonical inserts its canonical key into the same table,
// with the scan's probing (a hashed plan: after the scan; a sparse plan: after discovery, so that the canonical
// entries get ids and accumulator rows).  An entry read while another thread inserts it is canonical: nothing to
// do.  SC_TABLE_FULL counts inserts that found the table full, as the scan does.
__global__ void fold_insert(uint32_t* hk, uint32_t hmask, FoldKey F, unsigned long long* scalars) {
  const uint32_t stride = gridDim.x * blockDim.x;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i <= hmask; i += stride) {
    const uint32_t k = hk[i];
    if (k == 0u) continue;
    const uint32_t key = canon_code(F, k - 1u) + 1u;
    if (key == k) continue;
    uint32_t idx = slot_hash(key) & hmask, probes = 0;
    for (;;) {
      const uint32_t old = atomicCAS(hk + idx, 0u, key);
      if (old == 0u || old == key) break;
      idx = (idx + 1u) & hmask;
      if (++probes > hmask) {
        atomicAdd(scalars + SC_TABLE_FULL, 1ull);
        break;
      }
    }
  }
}

// the accumulator regions a fold combines, as offsets into the accumulator array
struct FoldAcc {
  uint64_t* acc;
  const uint32_t* hk;
  uint32_t hmask;
  const uint32_t* ids;         // sparse plans: table entry -> accumulator row; nullptr: the entry itself
  const unsigned long long* own;  // each row's own rows (the count array as the scan left it)
  unsigned long long* samples;    // rows per row after the fold (zeroed)
  unsigned long long* scalars;
  uint32_t nadd, nmax, nbk;
  size_t add_off[1 + 2 * SG_MAX_AGGS];  // one word per row, added: count, exact sums, hist Counts
  size_t max_off[SG_MAX_AGGS];          // one word per row, max: the MAX region
  size_t bk_off[SG_MAX_AGGS];           // bk_nv words per row, added: bucket counters
  uint32_t bk_nv[SG_MAX_AGGS];
};

// Fold: every non-canonical entry e with canonical entry c and weight multiplier w adds acc[e] * w into acc[c]
// (uint64, wrapping: dense_fold's arithmetic) and takes the max into the MAX region unmultiplied, then clears e; its
// rows go to samples[c], where a canonical entry's own rows also land.  Integer sums in any order: the result is
// the dense path's bit for bit.  Each warp reads 32 entries, then folds its sources one after the other with the
// lanes striding over the source's words.  Scalars: SC_NO_WEIGHT, SC_FOLD_ENTRIES, SC_FOLD_CANON.
__global__ void fold_rows(FoldAcc A, FoldKey F) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  constexpr uint32_t NONE = 0xffffffffu;
  for (uint32_t base = warp * 32u; base <= A.hmask; base += nwarps * 32u) {
    const uint32_t i = base + lane;
    const uint32_t k = i <= A.hmask ? A.hk[i] : 0u;
    uint32_t src = NONE, dst = 0u;
    unsigned long long mul = 1ull;
    bool canon = false;
    if (k != 0u) {
      const uint32_t code = k - 1u, cc = canon_code(F, code);
      const uint32_t row = A.ids ? A.ids[i] : i;
      const unsigned long long own = A.own[row];
      uint32_t to = row;
      if (F.wradix) {
        const uint32_t wd = (code / F.wstride) % F.wradix;
        if (wd == 0u && !F.wcarry && own) atomicAdd(A.scalars + SC_NO_WEIGHT, own);
        mul = (unsigned long long)F.wmul[wd];
      }
      canon = cc == code;
      if (!canon) {
        uint32_t j = slot_hash(cc + 1u) & A.hmask;
        for (uint32_t probes = 0;; probes++) {
          const uint32_t kk = A.hk[j];
          if (kk == cc + 1u) break;
          if (kk == 0u || probes >= A.hmask) {  // (only after the insert found the table full: refused)
            j = NONE;
            break;
          }
          j = (j + 1u) & A.hmask;
        }
        if (j != NONE) {
          to = A.ids ? A.ids[j] : j;
          src = row;
          dst = to;
        }
      }
      if (own) atomicAdd(A.samples + to, own);
    }
    const unsigned occ = __ballot_sync(0xffffffffu, k != 0u), can = __ballot_sync(0xffffffffu, canon);
    if (lane == 0 && occ) {
      atomicAdd(A.scalars + SC_FOLD_ENTRIES, (unsigned long long)__popc(occ));
      if (can) atomicAdd(A.scalars + SC_FOLD_CANON, (unsigned long long)__popc(can));
    }
    for (unsigned m = __ballot_sync(0xffffffffu, src != NONE); m; m &= m - 1u) {
      const int l = __ffs((int)m) - 1;
      const uint32_t s = __shfl_sync(0xffffffffu, src, l), d = __shfl_sync(0xffffffffu, dst, l);
      const unsigned long long w = __shfl_sync(0xffffffffu, mul, l);
      for (uint32_t r = lane; r < A.nadd; r += 32u) {
        unsigned long long* p = (unsigned long long*)A.acc + A.add_off[r];
        const unsigned long long v = p[s];
        if (v) {
          atomicAdd(p + d, v * w);
          p[s] = 0ull;
        }
      }
      for (uint32_t r = lane; r < A.nmax; r += 32u) {
        long long* p = (long long*)A.acc + A.max_off[r];
        const long long v = p[s];
        if (v != INT64_MIN) {
          atomicMax(p + d, v);
          p[s] = INT64_MIN;
        }
      }
      for (uint32_t b = 0; b < A.nbk; b++) {
        const size_t nv = A.bk_nv[b];
        unsigned long long* p = (unsigned long long*)A.acc + A.bk_off[b];
        for (size_t x = lane; x < nv; x += 32u) {
          const unsigned long long v = p[(size_t)s * nv + x];
          if (v) {
            atomicAdd(p + (size_t)d * nv + x, v * w);
            p[(size_t)s * nv + x] = 0ull;
          }
        }
      }
    }
  }
}

// The device fold of a run, queued behind its scan launch: the canonical insert (a hashed plan, or a sparse plan's
// discovery launch), then the fold (every launch that aggregates).  ev1 -> ev2 times the insert, ev2 -> ev3 the fold.
int device_fold(sg_query* q, bool discover) {
  sg_ctx* c = q->ctx;
  const Plan& P = q->plan;
  const uint32_t cap = q->hcap;
  const unsigned grid = (unsigned)std::min<uint64_t>(((uint64_t)cap + 255) / 256, (uint64_t)std::max(c->sm_count, 1) * 8);
  unsigned long long* const scalars = (unsigned long long*)(discover ? q->d_disc : q->d_acc);
  if (discover || !q->sparse) {
    fold_insert<<<grid, 256, 0, c->stream>>>(q->d_hkeys, cap - 1u, q->fkey, scalars);
    CUDA_TRY(c, cudaGetLastError());
    q->launches += 1;
  }
  CUDA_TRY(c, cudaEventRecord(q->ev2, c->stream));
  if (!discover) {
    const size_t n = P.nslots;  // accumulator rows: the table's entries, or a sparse plan's live groups
    FoldAcc A;
    memset(&A, 0, sizeof(A));
    A.acc = q->d_acc;
    A.hk = q->d_hkeys;
    A.hmask = cap - 1u;
    A.ids = q->sparse ? q->d_hids : nullptr;
    A.samples = (unsigned long long*)q->d_samples;
    A.own = (const unsigned long long*)(q->d_samples + n);
    A.scalars = scalars;
    // (the one-word added regions, count, sums and hist Counts, come first and fit add_off; a bucket region
    // that is one word wide may follow them there while room is left)
    for (const AccRegion& R : q->regions) {
      if (R.is_max) {
        A.max_off[A.nmax++] = R.off;
      } else if (R.per_row == 1 && A.nadd < 1 + 2 * SG_MAX_AGGS) {
        A.add_off[A.nadd++] = R.off;
      } else {
        A.bk_off[A.nbk] = R.off;
        A.bk_nv[A.nbk++] = R.per_row;
      }
    }
    CUDA_TRY(c, cudaMemsetAsync(q->d_samples, 0, n * 8, c->stream));
    CUDA_TRY(c, cudaMemcpyAsync(q->d_samples + n, q->d_acc + q->off_count, n * 8, cudaMemcpyDeviceToDevice, c->stream));
    fold_rows<<<grid, 256, 0, c->stream>>>(A, q->fkey);
    CUDA_TRY(c, cudaGetLastError());
    q->launches += 1;
  }
  CUDA_TRY(c, cudaEventRecord(q->ev3, c->stream));
  return SG_OK;
}

// Sparse group accumulators, before the aggregation launch: the discovery launch fills the table with the code of
// every row that passes, assign_ids numbers the entries, and the accumulators are laid out for the L live groups.
// Refuses when L groups' accumulators pass 24 GiB (tests: SG_SPARSE_BUDGET_MIB=n lowers that budget); the query's
// device state stays valid for another run.
int discover_groups(sg_query* q, const std::vector<uint32_t>& list) {
  sg_ctx* c = q->ctx;
  Plan& P = q->plan;
  CUDA_TRY(c, cudaMemsetAsync(q->d_hkeys, 0, (size_t)q->hcap * 4, c->stream));
  CUDA_TRY(c, cudaMemsetAsync(q->d_disc, 0, DISC_WORDS * 8, c->stream));
  uint64_t* const acc_scalars = P.scalars;
  P.scalars = q->d_disc;
  int rc = run_list(q, list, true);
  P.scalars = acc_scalars;
  if (rc != SG_OK) return rc;
  const uint64_t* scal = q->scal;
  if (scal[SC_TIME_OVERFLOW] != 0) {
    c->set_err("query: rows fall outside the planned time axis (time_min/time_max too narrow)");
    return SG_ERR_INVALID;
  }
  if (scal[SC_TABLE_FULL] != 0) {
    c->set_err("query: the hashed slot space filled up (more distinct group keys than its table holds)");
    return SG_ERR_UNSUPPORTED;
  }
  uint32_t* const d_ids = q->d_hids;
  uint32_t* const d_id2key = q->d_hids + q->hcap;
  unsigned int* const d_live = reinterpret_cast<unsigned int*>(q->d_disc + DISC_LIVE);
  cudaEvent_t e0 = q->ev0, e1 = q->ev1;
  CUDA_TRY(c, cudaEventRecord(e0, c->stream));
  const unsigned grid = (unsigned)std::min<uint64_t>(((uint64_t)q->hcap + 255) / 256, (uint64_t)std::max(c->sm_count, 1) * 8);
  // a folded plan numbers its canonical entries first (ids 0..L'-1: the rows its result reads back), then the others
  const int npass = q->dfold ? 2 : 1;
  for (int pass = 0; pass < npass; pass++) {
    assign_ids<<<grid, 256, 0, c->stream>>>(q->d_hkeys, q->hcap, d_ids, d_id2key, d_live, q->fkey, q->dfold ? pass + 1 : 0);
    CUDA_TRY(c, cudaGetLastError());
    if (q->dfold && pass == 0)
      CUDA_TRY(c, cudaMemcpyAsync(q->d_disc + DISC_CANON, q->d_disc + DISC_LIVE, 8, cudaMemcpyDeviceToDevice, c->stream));
  }
  CUDA_TRY(c, cudaEventRecord(e1, c->stream));
  uint64_t counts[2] = {0, 0};  // L, L'
  CUDA_TRY(c, cudaMemcpyAsync(counts, q->d_disc + DISC_LIVE, (size_t)npass * 8, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  const uint64_t live = counts[0];
  q->canon_live = (uint32_t)counts[1];
  q->d2h_bytes += npass * 8;
  q->launches += npass;
  float ids_ms = 0;
  CUDA_TRY(c, cudaEventElapsedTime(&ids_ms, e0, e1));
  q->kernel_ms += ids_ms;
  uint64_t budget = ACC_LIMIT_BYTES;
  if (const char* e = getenv("SG_SPARSE_BUDGET_MIB")) budget = (uint64_t)std::max(atoll(e), 0ll) << 20;
  if (getenv("SG_PLAN_TRACE"))
    fprintf(stderr, "sg_sparse: live=%llu table=%u discover_ms=%.4f ids_ms=%.4f\n", (unsigned long long)live, q->hcap,
            q->disc_ms, (double)ids_ms);
  if (sum_region_bytes(q, live) > budget) {
    c->set_err("query: sparse group accumulators for " + std::to_string(live) + " live groups exceed " +
               std::to_string(budget >> 20) + " MiB");
    return SG_ERR_UNSUPPORTED;
  }
  // accumulators for the live groups (a run over a table with more live groups needs a larger array)
  P.nslots = (uint32_t)live;
  rc = layout_accumulators(q, P.nslots);
  if (rc != SG_OK) return rc;
  pool_release(c, q->d_acc);
  q->d_acc = nullptr;
  CUDA_TRY(c, pool_alloc(c, (void**)&q->d_acc, q->acc_words * 8));
  if (q->dfold) {
    pool_release(c, q->d_samples);
    q->d_samples = nullptr;
    CUDA_TRY(c, pool_alloc(c, (void**)&q->d_samples, std::max<size_t>(live, 1) * 16));
  }
  point_plan(q);
  return SG_OK;
}

std::string render_key(const sg_query* q, const std::vector<uint64_t>& key) {
  // translate_group_by (aggregate.go:284-324)
  std::string s;
  const sg_table* t = q->table;
  if (q->groups.empty()) return "total";
  for (size_t i = 0; i < q->groups.size(); i++) {
    uint64_t v = key[i];
    if (v != SG_MISSING_KEY) {
      int col = q->groups[i].col_slot;
      if (t->types[(size_t)col] == SG_COL_INT)
        s += std::to_string((int64_t)v);
      else if (q->merged) {
        if (v < q->m_strs[i].size()) s += q->m_strs[i][(size_t)v];
      } else if (q->repl.count(col)) {  // StrReplace: the rewritten text (column_store_io.go:529-547)
        const auto& rs = q->repl.at(col).strs;
        if (v < rs.size()) s += rs[(size_t)v];
      } else if (v < t->sdict[(size_t)col].strs.size())
        s += t->sdict[(size_t)col].strs[(size_t)v];
    }
    s += "\t";
  }
  return s;
}

// g's Count, hist Counts, sums, maxima and bucket counters added into `into`; an aggregation whose hist Count is 0 in
// g adds nothing
void merge_group(ResultGroup& into, const ResultGroup& g, int naggs, const std::vector<HistLayout>& L) {
  into.count += g.count;
  for (int a = 0; a < naggs; a++) {
    if (g.hc(a) == 0) continue;
    into.hc(a) += g.hc(a);
    into.sm(a) = (int64_t)((uint64_t)into.sm(a) + (uint64_t)g.sm(a));
    into.vx(a) = std::max(into.vx(a), g.vx(a));
    if (L[(size_t)a].nvals_total) {
      if (into.values.size() < (size_t)naggs) into.values.resize((size_t)naggs);
      if (into.values[(size_t)a].empty()) into.values[(size_t)a].assign(L[(size_t)a].nvals_total, 0);
      if (const auto* gv = g.vals(a))
        for (uint32_t k = 0; k < L[(size_t)a].nvals_total; k++) into.values[(size_t)a][k] += (*gv)[k];
    }
  }
}

void init_group(ResultGroup& g, int naggs) {
  g.agg.assign((size_t)naggs * 3, 0);
  for (int a = 0; a < naggs; a++) g.vx(a) = INT64_MIN;
}

// ---- SortResults (aggregate.go:43-54,497-525) -------------------------------------------------------
// the value groups are ordered by: Count, or the mean of one aggregation (-inf without its histogram)
static inline double order_value(const sg_query* q, int64_t count, int64_t hc, int64_t sum) {
  const int ob = q->d.order_by_agg;
  if (ob < 0) return (double)count;
  return hc == 0 ? -INFINITY : (double)sum / (double)hc;
}
void sort_groups(const sg_query* q, std::vector<ResultGroup>& v) {
  // descending by the order value; Go's sort is unstable, ties are broken by the rendered key ascending;
  // OrderAsc reverses the sorted list; OrderBy == "" leaves the groups in slot order
  const int ob = q->d.order_by_agg;
  if (ob == SG_ORDER_NONE) return;
  auto val = [&](const ResultGroup& g) { return ob < 0 ? (double)g.count : order_value(q, g.count, g.hc(ob), g.sm(ob)); };
  std::sort(v.begin(), v.end(), [&](const ResultGroup& a, const ResultGroup& b) {
    const double va = val(a), vb = val(b);
    if (va != vb) return va > vb;
    return a.skey < b.skey;
  });
  if (q->d.order_asc) std::reverse(v.begin(), v.end());
}

// Ties of SortResults break by the rendered GroupByKey, the fields joined with '\t', compared as bytes.  When no
// string of an axis holds a byte <= '\t', the order of its fields f + '\t' is the byte order of the strings, the
// missing field ("") comes first, and comparing whole keys is comparing field by field: a per-axis rank gives
// the order.  Otherwise ("\x01" sorts before missing; "a\tb" against "a" depends on the next field) the keys
// themselves are compared (slot_key).
static bool ranks_of(const std::vector<std::string>& strs, std::vector<uint32_t>& rank) {
  bool plain = true;
  for (const auto& s : strs)
    for (unsigned char ch : s) plain = plain && ch > (unsigned char)'\t';
  std::vector<uint32_t> idx(strs.size());
  for (size_t i = 0; i < idx.size(); i++) idx[i] = (uint32_t)i;
  std::sort(idx.begin(), idx.end(), [&](uint32_t x, uint32_t y) { return strs[x] < strs[y]; });
  rank.resize(strs.size());
  for (size_t i = 0; i < idx.size(); i++) rank[idx[i]] = (uint32_t)i;
  return plain;
}
// rank of every code of one slot-space axis in the order of its rendered field (code 0 = missing = "" first);
// *plain is cleared when the ranks do not give that order (a string holds a byte <= '\t')
static const std::vector<uint32_t>& axis_ranks(sg_query* q, size_t di, std::vector<uint32_t>& scratch, bool* plain) {
  const GroupDim& d = q->dims[di];
  sg_table* t = q->table;
  if (q->merged) {  // union dictionaries of a cross-GPU merge: per query
    if (d.is_str) {
      if (!ranks_of(q->m_strs[di], scratch)) *plain = false;
    } else {
      std::vector<std::string> r;
      for (int64_t v : q->m_ints[di]) r.push_back(std::to_string(v));
      ranks_of(r, scratch);
    }
    return scratch;
  }
  if (d.is_str && q->repl.count(d.col)) {
    if (!ranks_of(q->repl.at(d.col).strs, scratch)) *plain = false;
    return scratch;
  }
  if (d.is_str) {
    auto& cache = t->srank[(size_t)d.col];
    if (cache.size() != t->sdict[(size_t)d.col].strs.size())
      t->splain[(size_t)d.col] = ranks_of(t->sdict[(size_t)d.col].strs, cache) ? 1 : 0;
    if (!t->splain[(size_t)d.col]) *plain = false;
    return cache;
  }
  auto& cache = t->irank[(size_t)d.col];
  const auto& vals = t->idict[(size_t)d.col].vals;
  if (cache.size() != vals.size()) {
    std::vector<std::string> r;
    r.reserve(vals.size());
    for (int64_t v : vals) r.push_back(std::to_string(v));
    ranks_of(r, cache);
  }
  return cache;
}

// the mixed-radix code of accumulator slot s: the slot itself in a dense slot space, the table's key otherwise
static inline uint32_t slot_code(const sg_query* q, uint32_t s) {
  if (!q->hashed) return s;
  return s < q->h_hkeys.size() && q->h_hkeys[s] ? q->h_hkeys[s] - 1u : 0u;
}
// one group's ResultGroup from the accumulators of dense slot s (h: words [0, have))
// key words and rendered key of dense slot s
static void group_key(const sg_query* q, uint32_t s, ResultGroup& g, int64_t* tbucket) {
  const Plan& P = q->plan;
  const uint32_t cs = slot_code(q, s);
  for (size_t di = 0; di < q->dims.size(); di++) {
    const GroupDim& d = q->dims[di];
    uint32_t code = (cs / d.stride) % d.radix;
    if (d.is_time) {
      if (tbucket) *tbucket = (P.time_first + (int64_t)code - 1) * P.time_bucket;
      continue;
    }
    if (d.is_weight) continue;  // (folded away: every live slot has code 0 here)
    if (code == 0)
      g.key.push_back(SG_MISSING_KEY);
    else if (d.is_str)
      g.key.push_back((uint64_t)(code - 1));
    else if (q->merged)
      g.key.push_back((uint64_t)q->m_ints[di][code - 1]);
    else
      g.key.push_back((uint64_t)q->table->idict[(size_t)d.col].vals[code - 1]);
  }
  g.skey = render_key(q, g.key);
}
// the rendered GroupByKey of slot s (ties between keys whose fields hold bytes <= '\t', axis_ranks)
static std::string slot_key(const sg_query* q, uint32_t s) {
  ResultGroup g;
  group_key(q, s, g, nullptr);
  return std::move(g.skey);
}

// The order of the slots of a result without a time axis, as sort_groups orders rendered keys: order value
// descending, ties by the rendered GroupByKey ascending.  That is lexicographic over the axes' field ranks when they
// are `plain`; otherwise tied entries compare their rendered keys (`keys` by Ent::row when the caller rendered them
// once, slot_key otherwise).
struct GroupOrder {
  struct Ent {
    double v;
    uint64_t tie;
    uint32_t slot;
    uint32_t row;  // the device top-K: the candidate's row
  };
  const sg_query* q;
  std::vector<std::vector<uint32_t>> scratch;
  std::vector<const std::vector<uint32_t>*> ranks;
  bool plain = true;
  std::vector<std::string> keys;
  // ranked false: the groups stay in slot order (OrderBy ""), nothing to rank
  GroupOrder(sg_query* q, bool ranked) : q(q), scratch(q->dims.size()), ranks(q->dims.size(), nullptr) {
    if (ranked)
      for (size_t di = 0; di < q->dims.size(); di++) ranks[di] = &axis_ranks(q, di, scratch[di], &plain);
  }
  // the tie rank of a code (the missing value's digit 0 first on every axis)
  uint64_t tie(uint32_t code) const {
    uint64_t t = 0;
    for (size_t di = 0; di < q->dims.size(); di++) {
      const GroupDim& d = q->dims[di];
      const uint32_t digit = (code / d.stride) % d.radix;
      t = t * d.radix + (digit ? (uint64_t)(*ranks[di])[digit - 1] + 1u : 0u);
    }
    return t;
  }
  bool before(const Ent& a, const Ent& b) const {
    if (a.v != b.v) return a.v > b.v;
    if (plain) return a.tie < b.tie;
    return keys.empty() ? slot_key(q, a.slot) < slot_key(q, b.slot) : keys[a.row] < keys[b.row];
  }
};

// A result of q without groups: the header every result of the query carries and an empty Cumulative.  scal: the
// scalars of the accumulators it is built from, for the broken blocks; a time slice (nullptr) carries no block
// counters and its Cumulative no key.
static std::unique_ptr<sg_result> new_result(sg_query* q, bool hist_mode, const uint64_t* scal) {
  std::unique_ptr<sg_result> r(new sg_result());
  r->q = q;
  r->layouts = q->layouts;
  r->hist_mode = hist_mode;
  r->ngroups_cols = (int)q->groups.size();
  r->naggs = q->plan.naggs;
  init_group(r->total, r->naggs);
  if (scal) {
    r->broken = q->broken_staged + (int64_t)scal[SC_BROKEN];
    r->skipped = q->skipped;
    r->total.skey = "TOTAL";
    for (int i = 1; i < (int)q->groups.size(); i++) r->total.skey += "\t";
  }
  return r;
}
static void make_group(const sg_query* q, const uint64_t* h, uint32_t s, ResultGroup& g, int64_t* tbucket,
                       const std::vector<uint64_t>* samples = nullptr) {
  const Plan& P = q->plan;
  const int naggs = P.naggs;
  init_group(g, naggs);
  g.count = (int64_t)h[q->off_count + s];
  if (samples && s < samples->size()) g.samples = (int64_t)(*samples)[s];
  group_key(q, s, g, tbucket);
  const bool want_max = P.hist_mode || q->d.hist_kind == SG_HIST_MULTI;
  for (int a = 0; a < naggs; a++) {
    g.hc(a) = (size_t)a < q->hc_is_count.size() && q->hc_is_count[(size_t)a] ? g.count : (int64_t)h[q->off_hcount[(size_t)a] + s];
    g.sm(a) = (int64_t)h[q->off_sum[(size_t)a] + s];
    g.vx(a) = want_max ? (int64_t)h[q->off_vmax[(size_t)a] + s] : INT64_MIN;
    uint32_t nv = q->layouts[(size_t)a].nvals_total;
    if (nv && g.hc(a)) {
      const uint64_t* src = h + q->off_buckets[(size_t)a] + (size_t)s * nv;
      if (g.values.size() < (size_t)naggs) g.values.resize((size_t)naggs);
      g.values[(size_t)a].assign(src, src + nv);
    }
  }
}

// run fn(thread index, first slot, end slot) over [0, n) on up to `want` host threads
template <class Fn>
static void parallel_slots(uint32_t n, int want, Fn fn) {
  int nt = n >= (1u << 17) ? want : 1;
  if (nt <= 1) {
    fn(0, 0u, n);
    return;
  }
  std::vector<std::thread> th;
  const uint32_t per = (n + (uint32_t)nt - 1) / (uint32_t)nt;
  for (int i = 0; i < nt; i++) {
    const uint32_t a = std::min(n, per * (uint32_t)i), b = std::min(n, a + per);
    th.emplace_back(fn, i, a, b);
  }
  for (auto& x : th) x.join();
}

// Results with very many groups and a limit (the 1M-key group-by: `-limit 100`): the first `limit` groups of
// the sorted list are selected on the device — Cumulative totals + largest key, a radix descent over the order
// keys (11 bits a pass, from the top set bit down) to the key of the limit-th group, then every slot at or above
// it with its values — instead of reading a 40 MB accumulator array back and scanning a million slots on the
// host.  Ties at the cut are all emitted and broken on the host exactly as sort_groups does.
// Returns SG_OK with *out set, 1 when the query is not of that shape (or the tie group is huge, *fell_back set):
// host path.
static int build_result_topk(sg_query* q, sg_result** out, bool* fell_back) {
  sg_ctx* c = q->ctx;
  const Plan& P = q->plan;
  const int naggs = P.naggs, ob = q->d.order_by_agg;
  const int64_t limit = q->d.limit;
  if (P.time_col >= 0 || P.hist_mode || q->d.hist_kind == SG_HIST_MULTI) return 1;
  if (!q->repl.empty() || q->d.weight_col_slot >= 0) return 1;  // StrReplace / weights fold slots on the host first
  if (q->hashed) return 1;                                       // keys come from the table read-back (build_result)
  if (limit <= 0 || limit > 65536 || ob == SG_ORDER_NONE || q->d.order_asc) return 1;
  if (P.nslots < (1u << 17) || getenv("SG_NO_GPU_TOPK")) return 1;
  // a query holding a host copy answers from it: after the small-plan cross-GPU merge only that copy is merged, the
  // device array is still this rank's own
  if (q->acc.words) return 1;
  const unsigned cap = (unsigned)limit + 8192u;
  const size_t w = 2 + 2 * (size_t)naggs;
  const size_t off_tot = 0, off_hist = 512, off_offs = off_hist + 8192, off_scal = off_offs + 512, off_rows = off_scal + 128;
  const size_t total = off_rows + (size_t)cap * w * 8;
  char* hp = c->scratch(total);
  PoolTmp dev(c);
  if (!hp || pool_alloc(c, &dev.p, total) != cudaSuccess) {
    cudaGetLastError();
    return 1;
  }
  char* dp = (char*)dev.p;
  size_t* h_offs = (size_t*)(hp + off_offs);
  int* h_hcic = (int*)(h_offs + 2 * SG_MAX_AGGS);
  for (int a = 0; a < naggs; a++) {
    h_offs[a] = q->off_hcount[(size_t)a];
    h_offs[SG_MAX_AGGS + a] = q->off_sum[(size_t)a];
    h_hcic[a] = (size_t)a < q->hc_is_count.size() && q->hc_is_count[(size_t)a] ? 1 : 0;
  }
  TopkArgs A;
  A.acc = q->d_acc;
  A.off_count = q->off_count;
  A.order_by = ob;
  A.off_hc = ob >= 0 ? q->off_hcount[(size_t)ob] : 0;
  A.off_sum = ob >= 0 ? q->off_sum[(size_t)ob] : 0;
  A.hc_is_count = ob >= 0 ? h_hcic[ob] : 1;
  A.nslots = P.nslots;
  const size_t* d_off_hc = (const size_t*)(dp + off_offs);
  const size_t* d_off_sum = d_off_hc + SG_MAX_AGGS;
  const int* d_hcic = (const int*)(d_off_hc + 2 * SG_MAX_AGGS);
  TopkTotals* d_tot = (TopkTotals*)(dp + off_tot);
  unsigned int* d_hist = (unsigned int*)(dp + off_hist);
  unsigned long long* d_rows = (unsigned long long*)(dp + off_rows);
  const int grid = std::max(1, c->sm_count) * 4;
  static_assert(sizeof(TopkTotals) <= 512, "TopkTotals");
  CUDA_TRY(c, cudaMemsetAsync(dp, 0, off_offs, c->stream));
  CUDA_TRY(c, cudaMemcpyAsync(dp + off_offs, hp + off_offs, 512, cudaMemcpyHostToDevice, c->stream));
  topk_totals<<<grid, 256, 0, c->stream>>>(A, naggs, d_off_hc, d_off_sum, d_hcic, d_tot);
  CUDA_TRY(c, cudaMemcpyAsync(hp + off_tot, d_tot, sizeof(TopkTotals), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaMemcpyAsync(hp + off_scal, q->d_acc, SCALAR_WORDS * 8, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  q->launches += 1;
  TopkTotals T = *(const TopkTotals*)(hp + off_tot);
  if (T.live == 0 || T.max_key == 0) return 1;
  // radix descent to the key of the limit-th group
  int hi = 64 - __builtin_clzll(T.max_key);  // keys have no bit at or above `hi`
  unsigned long long prefix = 0, lower = 0;
  int has_prefix = 0;
  uint64_t need = (uint64_t)limit;
  for (;;) {
    const int bits = std::min(11, hi), shift = hi - bits;
    CUDA_TRY(c, cudaMemsetAsync(d_hist, 0, 8192, c->stream));
    topk_hist<<<grid, 256, 0, c->stream>>>(A, prefix, shift, bits, has_prefix, d_hist);
    CUDA_TRY(c, cudaMemcpyAsync(hp + off_hist, d_hist, 8192, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    q->launches += 1;
    const unsigned int* hist = (const unsigned int*)(hp + off_hist);
    uint64_t cum = 0;
    int b = (1 << bits) - 1;
    for (; b > 0; b--) {
      if (cum + hist[b] >= need) break;
      cum += hist[b];
    }
    // (b == 0 also when fewer than `need` keys exist under this prefix: then everything under it qualifies)
    const unsigned long long np = (prefix << bits) | (unsigned long long)b;
    if (hist[b] <= 8192u - 1u || shift == 0 || cum + hist[b] < need) {
      lower = np << shift;
      break;
    }
    need -= cum;
    prefix = np;
    has_prefix = 1;
    hi = shift;
  }
  topk_emit<<<grid, 256, 0, c->stream>>>(A, lower, naggs, d_off_hc, d_off_sum, d_hcic, d_rows, cap, d_tot);
  CUDA_TRY(c, cudaMemcpyAsync(hp + off_tot, d_tot, sizeof(TopkTotals), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  q->launches += 1;
  T = *(const TopkTotals*)(hp + off_tot);
  if (T.overflow || T.n_out > cap) {  // a huge group of ties at the cut: the host path sorts them all
    *fell_back = true;
    return 1;
  }
  const size_t n = T.n_out;
  CUDA_TRY(c, cudaMemcpyAsync(hp + off_rows, d_rows, n * w * 8, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  q->d2h_bytes += (int64_t)(n * w * 8 + 8192 + 1024);
  const unsigned long long* rows = (const unsigned long long*)(hp + off_rows);
  const uint64_t* scal = (const uint64_t*)(hp + off_scal);

  // exact order of the candidates (keys rendered once each when the ranks do not give it)
  GroupOrder O(q, true);
  std::vector<GroupOrder::Ent> ents(n);
  if (!O.plain) O.keys.resize(n);
  for (size_t i = 0; i < n; i++) {
    const unsigned long long* r = rows + i * w;
    const uint32_t sl = (uint32_t)r[0];
    ents[i].v = order_value(q, (int64_t)r[1], ob >= 0 ? (int64_t)r[2 + 2 * ob] : 0, ob >= 0 ? (int64_t)r[3 + 2 * ob] : 0);
    ents[i].tie = O.tie(sl);
    ents[i].slot = sl;
    ents[i].row = (uint32_t)i;
    if (!O.plain) O.keys[i] = slot_key(q, sl);
  }
  std::sort(ents.begin(), ents.end(), [&](const GroupOrder::Ent& a, const GroupOrder::Ent& b) { return O.before(a, b); });
  if ((int64_t)ents.size() > limit) ents.resize((size_t)limit);

  std::unique_ptr<sg_result> r = new_result(q, false, scal);
  r->total.count = (int64_t)T.count;
  for (int a = 0; a < naggs; a++) {
    r->total.hc(a) = (int64_t)T.hc[a];
    r->total.sm(a) = (int64_t)T.sum[a];
  }
  r->matched = (int64_t)T.count;  // no time column: every matched row is counted in exactly one group
  r->ngroups_total = (int64_t)T.live;
  r->groups.resize(ents.size());
  for (size_t i = 0; i < ents.size(); i++) {
    const unsigned long long* rw = rows + (size_t)ents[i].row * w;
    ResultGroup& g = r->groups[i];
    init_group(g, naggs);
    g.count = (int64_t)rw[1];
    group_key(q, (uint32_t)rw[0], g, nullptr);
    for (int a = 0; a < naggs; a++) {
      g.hc(a) = (int64_t)rw[2 + 2 * a];
      g.sm(a) = (int64_t)rw[3 + 2 * a];
      g.vx(a) = INT64_MIN;
    }
  }
  *out = r.release();
  return SG_OK;
}

// The folds of the accumulators before the result is built (canon_code: dense_fold here, fold_rows on the device).
//
// StrReplace: strings of a group column that rewrite to the same text are one group in the reference (the block's
// string table is rewritten before any row is read, column_store_io.go:529-547).  The scan grouped by the original
// global ids; every group whose code on a rewritten axis is not its class representative is added onto the
// representative's group (counts, hist counts, sums, bucket counters: +; max: max) and cleared.  A string that
// rewrites to "" goes onto code 0 instead: it renders like a missing value, and is the missing group (DESIGN.md §7).
//
// Weights (OPTS.WEIGHT_COL): the scan grouped by the weight value as a hidden last axis (make_plan); the groups of
// weight w are multiplied by w and added onto code 0 of that axis — Count / hist Count / Values[] += weight
// (aggregate.go:203, hist_basic.go:111-116,146), exact sum += value * weight; Result.Samples keeps the rows.
// A row without the weight column reuses the previous row's weight (Q13, aggregate.go:68,100-102).  With
// weight_carry the scan has already given such a row that weight's code, and a row left on code 0 had no earlier
// row with the column in its block: weight 1, so the slot stays in place.  Without weight_carry it is refused.
static const char* const NO_WEIGHT_MSG =
    "query: rows without the weight column (the reference reuses the previous row's weight, aggregate.go:68,100-102): "
    "not reproduced by this engine";

// The dense plans' fold (the device's is fold_rows, over table entries): every slot s moves onto its canonical slot
// c = canon_code(F, s) with its weight multiplier w: acc[s] * w is added into acc[c] (uint64, wrapping, like the
// reference's int64 arithmetic), the MAX region takes the max unmultiplied, and s is cleared.  canon_code is
// idempotent, so every source is non-canonical and every destination canonical: no source changes before it is read,
// in any order.  A slot without rows holds nothing to move.  Weighted, each slot's rows go to samples[c] first and the
// rows left on weight code 0 without weight_carry are counted into SC_NO_WEIGHT.  Regions past `have` were not read
// back: the result does not use them.
static void dense_fold(sg_query* q, const FoldKey& F, uint64_t* h, size_t have, sg_result* r) {
  const uint32_t ns = q->plan.nslots;
  const uint64_t* cnt = h + q->off_count;
  if (F.wradix) {
    r->samples.assign(ns, 0);
    for (uint32_t s = 0; s < ns; s++) {
      if (!cnt[s]) continue;
      if ((s / F.wstride) % F.wradix == 0 && !F.wcarry) h[SC_NO_WEIGHT] += cnt[s];
      r->samples[canon_code(F, s)] += cnt[s];
    }
  }
  std::vector<AccRegion> regions;
  for (const AccRegion& R : q->regions)
    if (R.off + (size_t)ns * R.per_row <= have) regions.push_back(R);
  for (uint32_t s = 0; s < ns; s++) {
    const uint32_t to = canon_code(F, s);
    if (to == s || !cnt[s]) continue;
    const uint64_t w = F.wradix ? (uint64_t)F.wmul[(s / F.wstride) % F.wradix] : 1u;
    for (const AccRegion& R : regions) {
      uint64_t* src = h + R.off + (size_t)s * R.per_row;
      uint64_t* dst = h + R.off + (size_t)to * R.per_row;
      for (uint32_t k = 0; k < R.per_row; k++) {
        if (R.is_max)
          dst[k] = (uint64_t)std::max((int64_t)dst[k], (int64_t)src[k]), src[k] = (uint64_t)INT64_MIN;
        else
          dst[k] += src[k] * w, src[k] = 0;
      }
    }
  }
}

// A folded sparse plan's read-back: the scalars and, of every accumulator region, the rows of the L' canonical
// groups (ids 0..L'-1), into a pinned buffer, laid out for L' rows.  The query's layout becomes that one (the next
// run lays the accumulators out again after its discovery).
static int read_canonical_rows(sg_query* q, HostAcc& h) {
  sg_ctx* c = q->ctx;
  const uint32_t n = q->canon_live;
  const std::vector<AccRegion> old = q->regions;
  int rc = layout_accumulators(q, n);
  if (rc != SG_OK) return rc;
  q->plan.nslots = n;
  rc = read_acc(q, h, q->acc_words, 0, nullptr, [&](uint64_t* dst) {
    auto back = [&](size_t to, size_t from, size_t words) {
      return words ? cudaMemcpyAsync(dst + to, q->d_acc + from, words * 8, cudaMemcpyDeviceToHost, c->stream) : cudaSuccess;
    };
    cudaError_t e = back(0, 0, SCALAR_WORDS);
    for (size_t i = 0; i < old.size() && e == cudaSuccess; i++) e = back(q->regions[i].off, old[i].off, (size_t)n * old[i].per_row);
    return e;
  });
  if (rc != SG_OK) return rc;
  q->d2h_bytes += (int64_t)q->acc_words * 8;
  return SG_OK;
}

int build_result(sg_query* q, sg_result** out) {
  sg_ctx* c = q->ctx;
  const Plan& P = q->plan;
  // SG_PLAN_TRACE=1: which selection built the result ("sg_select: path=device|device-fallback|host threads=N")
  // (device-fallback: the device found more ties at the cut than it keeps, and the host selected)
  const bool trace = getenv("SG_PLAN_TRACE") != nullptr;
  bool fell_back = false;
  {
    const int rc = build_result_topk(q, out, &fell_back);
    if (rc != 1) {
      if (trace && rc == SG_OK) fprintf(stderr, "sg_select: path=device threads=1\n");
      return rc;
    }
  }
  const bool time_mode = P.time_col >= 0;
  const int naggs = P.naggs;
  // what the result reads: without bucket counters, without hist Min/Max tracking and with every hist Count
  // equal to Count, the contiguous prefix scalars | count | sums is enough
  bool all_hc = true;
  for (int a = 0; a < naggs; a++) all_hc = all_hc && (size_t)a < q->hc_is_count.size() && q->hc_is_count[(size_t)a];
  const bool want_max = P.hist_mode || q->d.hist_kind == SG_HIST_MULTI;
  size_t have = q->acc_words;
  if (!want_max) have = q->sum_words;
  if (!want_max && !P.hist_mode && all_hc) have = q->prefix_words;
  HostAcc acc;
  if (q->sparse && q->dfold) {
    // a folded sparse plan: the canonical groups hold ids 0..L'-1, and only their rows come back, laid out for L'
    const int rc = read_canonical_rows(q, acc);
    if (rc != SG_OK) return rc;
    have = q->acc_words;
  } else if (q->acc.words == q->acc_words) {  // read back behind the kernel or the merge: the result takes it over
    acc = std::move(q->acc);
    have = q->acc_words;
  } else {
    const int rc = read_acc(q, acc, q->d_acc, have, 0, nullptr);
    if (rc != SG_OK) return rc;
    q->d2h_bytes += (int64_t)have * 8;
  }
  std::unique_ptr<sg_result> r = new_result(q, P.hist_mode != 0, acc.data());
  r->acc = std::move(acc);
  uint64_t* const h = r->acc.data();  // (this result's own copy: the folds below change it)
  if (q->hashed) {
    if (h[SC_TABLE_FULL] != 0) {
      c->set_err("query: the hashed slot space filled up (more distinct group keys than its table holds)");
      return SG_ERR_UNSUPPORTED;
    }
    if ((!q->repl.empty() || q->d.weight_col_slot >= 0) && !q->dfold) {
      c->set_err("query: StrReplace / weights over a hashed slot space are not in this build");
      return SG_ERR_UNSUPPORTED;
    }
    // slot -> key: the table itself, or for a sparse plan its id -> key array (L entries, nothing sized by the table)
    q->h_hkeys.resize(P.nslots);
    const uint32_t* keys = q->sparse ? q->d_hids + q->hcap : q->d_hkeys;
    if (P.nslots) CUDA_TRY(c, cudaMemcpyAsync(q->h_hkeys.data(), keys, (size_t)P.nslots * 4, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    q->d2h_bytes += (int64_t)P.nslots * 4;
  }
  if (q->dfold) {
    // folded on the device: a weighted result takes the rows per group the fold counted
    if (q->d.weight_col_slot >= 0) {
      r->samples.resize(P.nslots);
      if (P.nslots)
        CUDA_TRY(c, cudaMemcpyAsync(r->samples.data(), q->d_samples, (size_t)P.nslots * 8, cudaMemcpyDeviceToHost, c->stream));
      CUDA_TRY(c, cudaStreamSynchronize(c->stream));
      q->d2h_bytes += (int64_t)P.nslots * 8;
    }
  } else if (!q->repl.empty() || q->d.weight_col_slot >= 0) {
    if (q->merged && !q->repl.empty()) {
      c->set_err("query: StrReplace cannot follow a cross-GPU merge over differing dictionaries (seed them)");
      return SG_ERR_UNSUPPORTED;
    }
    FoldKey F;
    std::vector<int64_t> wmul;
    std::vector<uint32_t> luts;
    const int rc = build_fold_key(q, &F, &wmul, &luts);
    if (rc != SG_OK) return rc;
    F.wmul = wmul.data();
    F.luts = luts.data();
    dense_fold(q, F, h, have, r.get());
  }
  if (h[SC_NO_WEIGHT] != 0) {
    c->set_err(NO_WEIGHT_MSG);
    return SG_ERR_UNSUPPORTED;
  }
  int64_t w_rows = -1;  // weighted queries: matched ROWS (MatchedCount counts records, aggregate.go:117)
  if (q->d.weight_col_slot >= 0) {
    w_rows = 0;
    for (uint64_t n : r->samples) w_rows += (int64_t)n;
  }
  r->matched = (int64_t)h[SC_MATCHED];
  r->has_total_hists = !time_mode;
  const uint64_t* cnt = h + q->off_count;
  // a group is a slot that rows were scanned into.  Weighted, its Count is the sum of the rows' weights and can
  // be 0 (weight 0, +w / -w, wrapped): the rows per slot (r->samples) decide then, as in the reference, where
  // every row creates its group (aggregate.go:156-203)
  const uint64_t* rows_of = r->samples.empty() ? cnt : (const uint64_t*)r->samples.data();
  const bool weighted = !r->samples.empty();

  if (!time_mode) {
    // ---- lazy result: live slots, Cumulative, order -------------------------------------------------
    const uint32_t ns = P.nslots;
    const int ob = q->d.order_by_agg;
    const int64_t limit = q->d.limit;
    int hw = (int)std::thread::hardware_concurrency();
    int nt = std::max(1, std::min(hw > 0 ? hw : 1, 16));
    if (const char* e = getenv("SG_HOST_THREADS")) nt = std::max(1, std::min(atoi(e), 16));  // tests: 1 vs many
    const GroupOrder O(q, ob != SG_ORDER_NONE);
    using Ent = GroupOrder::Ent;
    auto before = [&](const Ent& a, const Ent& b) { return O.before(a, b); };
    struct Part {
      std::vector<Ent> ents;
      ResultGroup tot;
      int64_t live = 0;
    };
    std::vector<Part> parts((size_t)nt);
    for (auto& p : parts) init_group(p.tot, naggs);
    const bool keep_all = ob == SG_ORDER_NONE || limit <= 0 || q->d.order_asc;  // ascending: the END of the list
    parallel_slots(ns, nt, [&](int ti, uint32_t s0, uint32_t s1) {
      Part& p = parts[(size_t)ti];
      double thr = -INFINITY;  // top-`limit` only: order values below the part's limit-th best cannot make the list
      const size_t trim_at = keep_all ? (size_t)-1 : (size_t)limit * 4 + 64;
      if (P.hist_mode) {
        p.tot.values.resize((size_t)naggs);
        for (int a = 0; a < naggs; a++) p.tot.values[(size_t)a].assign(q->layouts[(size_t)a].nvals_total, 0);
      }
      for (uint32_t s = s0; s < s1; s++) {
        if (rows_of[s] == 0) continue;
        const int64_t n = (int64_t)cnt[s];
        p.live++;
        p.tot.count += n;
        int64_t hc_o = 0, sm_o = 0;
        for (int a = 0; a < naggs; a++) {
          const int64_t hc = q->hc_is_count[(size_t)a] ? n : (int64_t)h[q->off_hcount[(size_t)a] + s];
          if (hc == 0 && !weighted) continue;  // (weighted, a histogram whose Count folds to 0 still has a sum)
          const int64_t sm = (int64_t)h[q->off_sum[(size_t)a] + s];
          p.tot.hc(a) += hc;
          p.tot.sm(a) = (int64_t)((uint64_t)p.tot.sm(a) + (uint64_t)sm);
          if (want_max) p.tot.vx(a) = std::max(p.tot.vx(a), (int64_t)h[q->off_vmax[(size_t)a] + s]);
          const uint32_t nv = q->layouts[(size_t)a].nvals_total;
          if (nv) {
            const uint64_t* src = h + q->off_buckets[(size_t)a] + (size_t)s * nv;
            int64_t* dst = p.tot.values[(size_t)a].data();
            for (uint32_t k = 0; k < nv; k++) dst[k] += (int64_t)src[k];
          }
          if (a == ob) {
            hc_o = hc;
            sm_o = sm;
          }
        }
        Ent e;
        e.slot = s;
        e.row = 0;
        e.v = ob == SG_ORDER_NONE ? 0.0 : order_value(q, n, hc_o, sm_o);
        if (e.v < thr) continue;
        e.tie = ob == SG_ORDER_NONE ? 0 : O.tie(slot_code(q, s));
        p.ents.push_back(e);
        if (p.ents.size() >= trim_at) {
          std::nth_element(p.ents.begin(), p.ents.begin() + limit, p.ents.end(), before);
          p.ents.resize((size_t)limit);
          thr = p.ents[0].v;
          for (auto& x : p.ents) thr = std::min(thr, x.v);
        }
      }
      if (!keep_all && (int64_t)p.ents.size() > limit) {  // only this part's best `limit` can make the list
        std::nth_element(p.ents.begin(), p.ents.begin() + limit, p.ents.end(), before);
        p.ents.resize((size_t)limit);
      }
    });
    std::vector<Ent> all;
    int64_t live = 0;
    for (auto& p : parts) {
      live += p.live;
      all.insert(all.end(), p.ents.begin(), p.ents.end());
      merge_group(r->total, p.tot, naggs, q->layouts);  // Cumulative (aggregate.go:422-436): every group combined
    }
    if (ob != SG_ORDER_NONE) {
      std::sort(all.begin(), all.end(), before);
      if (q->d.order_asc) std::reverse(all.begin(), all.end());
    }
    if (limit > 0 && (int64_t)all.size() > limit) all.resize((size_t)limit);
    r->order.reserve(all.size());
    for (auto& e : all) r->order.push_back(e.slot);
    r->ngroups_total = live;
    // without a time column every matched row is counted in exactly one group, so the kernel does not
    // count matches separately (MatchedCount, aggregate.go:117)
    r->matched = w_rows >= 0 ? w_rows : r->total.count;
    if (w_rows >= 0) r->total.samples = w_rows;
    r->lazy = true;
    if (trace)
      fprintf(stderr, "sg_select: path=%s threads=%d\n", fell_back ? "device-fallback" : "host", ns >= (1u << 17) ? nt : 1);
    *out = r.release();
    return SG_OK;
  }

  // ---- time mode: Results[key] (counts), TimeResults[bucket][key] ----------------------------------
  std::map<std::vector<uint64_t>, size_t> by_key;                    // Results in time mode
  std::map<int64_t, std::unique_ptr<sg_result>> slices;              // TimeResults
  for (uint32_t s = 0; s < P.nslots; s++) {
    if (rows_of[s] == 0) continue;
    ResultGroup g;
    int64_t tbucket = 0;
    make_group(q, h, s, g, &tbucket, r->samples.empty() ? nullptr : &r->samples);
    // Results[key]: Count/Samples only (aggregate.go:156-171); hists live per bucket
    auto it = by_key.find(g.key);
    if (it == by_key.end()) {
      ResultGroup base;
      init_group(base, naggs);
      base.key = g.key;
      base.skey = g.skey;
      by_key[g.key] = r->groups.size();
      r->groups.push_back(std::move(base));
      it = by_key.find(g.key);
    }
    r->groups[it->second].count += g.count;
    r->total.count += g.count;
    if (g.samples >= 0) {  // weighted: Samples are rows
      ResultGroup& bg = r->groups[it->second];
      bg.samples = (bg.samples < 0 ? 0 : bg.samples) + g.samples;
      r->total.samples = (r->total.samples < 0 ? 0 : r->total.samples) + g.samples;
    }
    auto& sl = slices[tbucket];
    if (!sl) sl = new_result(q, r->hist_mode, nullptr);
    sl->groups.push_back(std::move(g));
  }
  sort_groups(q, r->groups);
  r->ngroups_total = (int64_t)r->groups.size();
  if (q->d.limit > 0 && (int64_t)r->groups.size() > q->d.limit) r->groups.resize((size_t)q->d.limit);
  for (auto& kv : slices) {
    sort_groups(q, kv.second->groups);
    kv.second->ngroups_total = (int64_t)kv.second->groups.size();
    r->time_keys.push_back(kv.first);
    r->time_slices.push_back(std::move(kv.second));
  }
  if (trace) fprintf(stderr, "sg_select: path=host threads=1\n");
  *out = r.release();
  return SG_OK;
}

}  // namespace

extern "C" {

sg_query* sg_query_begin(sg_ctx* c, sg_table* t, const sg_query_desc* d) {
  if (!c || !d) return nullptr;
  if (!c->has_device) {
    c->set_err("sg_query_begin: no CUDA device (libsybilgpu has no CPU path)");
    return nullptr;
  }
  if (d->abi_version != SG_ABI_VERSION) {
    c->set_err("sg_query_begin: ABI version mismatch");
    return nullptr;
  }
  if (d->nfilters < 0 || d->nfilters > SG_MAX_FILTERS || d->ngroups < 0 || d->ngroups > SG_MAX_GROUPS ||
      d->naggs < 0 || d->naggs > SG_MAX_AGGS) {
    c->set_err("sg_query_begin: too many filters / groups / aggregations for this build");
    return nullptr;
  }
  if (d->weight_carry != 0 && d->weight_carry != 1) {
    c->set_err("sg_query_begin: weight_carry must be 0 or 1");
    return nullptr;
  }
  if (!t) {
    c->set_err("sg_query_begin: table is NULL");
    return nullptr;
  }
  sg_query* q = new sg_query();
  q->ctx = c;
  q->table = t;
  q->d = *d;
  if (d->nfilters) q->filters.assign(d->filters, d->filters + d->nfilters);
  if (d->ngroups) q->groups.assign(d->groups, d->groups + d->ngroups);
  if (d->naggs) q->aggs.assign(d->aggs, d->aggs + d->naggs);
  q->filter_strs.resize(q->filters.size());
  for (size_t i = 0; i < q->filters.size(); i++) {
    if (q->filters[i].str_value && q->filters[i].str_len > 0)
      q->filter_strs[i].assign(q->filters[i].str_value, (size_t)q->filters[i].str_len);
    q->filters[i].str_value = nullptr;
  }
  q->luts.resize(q->filters.size());
  q->lut_bits.assign(q->filters.size(), -1);
  q->d_luts.assign(q->filters.size(), nullptr);
  q->d.filters = nullptr;
  q->d.groups = nullptr;
  q->d.aggs = nullptr;
  return q;
}

void sg_query_free(sg_query* q) {
  if (!q) return;
  cudaSetDevice(q->ctx->device);
  free_device(q);
  if (q->ev0) cudaEventDestroy(q->ev0);
  if (q->ev1) cudaEventDestroy(q->ev1);
  if (q->ev2) cudaEventDestroy(q->ev2);
  if (q->ev3) cudaEventDestroy(q->ev3);
  delete q;
}

int sg_query_set_str_lut(sg_query* q, int32_t fi, const uint32_t* bits, int64_t nbits) {
  if (!q || fi < 0 || (size_t)fi >= q->filters.size() || nbits < 0) return SG_ERR_INVALID;
  sg_ctx* c = q->ctx;
  cudaSetDevice(c->device);
  size_t words = (size_t)((nbits + 31) / 32);
  q->luts[(size_t)fi].assign(bits, bits + words);
  q->lut_bits[(size_t)fi] = nbits;
  pool_release(c, q->d_luts[(size_t)fi]);
  q->d_luts[(size_t)fi] = nullptr;
  CUDA_TRY(c, pool_alloc(c, (void**)&q->d_luts[(size_t)fi], std::max<size_t>(words, 1) * 4));
  if (words) CUDA_TRY(c, cudaMemcpyAsync(q->d_luts[(size_t)fi], bits, words * 4, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));  // (H2D on the stream the kernels run on: see remap_to_union)
  q->planned = false;
  return SG_OK;
}

int sg_query_set_str_replace(sg_query* q, int32_t col, const char* bytes, const uint32_t* offsets, int64_t n) {
  if (!q || n < 0) return SG_ERR_INVALID;
  sg_ctx* c = q->ctx;
  sg_table* t = q->table;
  if (col < 0 || col >= t->ncols || t->types[(size_t)col] != SG_COL_STR) {
    c->set_err("sg_query_set_str_replace: not a str column");
    return SG_ERR_INVALID;
  }
  if (n == 0) {
    q->repl.erase(col);
    return SG_OK;
  }
  if (!bytes || !offsets || (size_t)n != t->sdict[(size_t)col].strs.size()) {
    c->set_err("sg_query_set_str_replace: one rewritten string per entry of the column's dictionary is needed");
    return SG_ERR_INVALID;
  }
  sg_query::Replace R;
  R.strs.reserve((size_t)n);
  R.canon.resize((size_t)n);
  std::unordered_map<std::string, uint32_t> first;
  for (int64_t i = 0; i < n; i++) {
    if (offsets[i + 1] < offsets[i]) {
      c->set_err("sg_query_set_str_replace: offsets not monotone");
      return SG_ERR_INVALID;
    }
    R.strs.emplace_back(bytes + offsets[i], offsets[i + 1] - offsets[i]);
    R.canon[(size_t)i] = first.emplace(R.strs.back(), (uint32_t)i).first->second;
  }
  q->repl[col] = std::move(R);
  return SG_OK;
}

int sg_query_set_sparse_groups(sg_query* q, int32_t on) {
  if (!q) return SG_ERR_INVALID;
  if (on != 0 && on != 1) {
    q->ctx->set_err("sg_query_set_sparse_groups: on must be 0 or 1");
    return SG_ERR_INVALID;
  }
  if (on != q->sparse_req) q->planned = false;  // the next sg_query_run plans again
  q->sparse_req = on;
  return SG_OK;
}

int sg_query_set_hashed_folds(sg_query* q, int32_t on) {
  if (!q) return SG_ERR_INVALID;
  if (on != 0 && on != 1) {
    q->ctx->set_err("sg_query_set_hashed_folds: on must be 0 or 1");
    return SG_ERR_INVALID;
  }
  if (on != q->hfold_req) q->planned = false;  // the next sg_query_run plans again
  q->hfold_req = on;
  return SG_OK;
}

int sg_query_should_load(sg_query* q, const sg_block_desc* b) {
  if (!q || !b) return SG_ERR_INVALID;
  std::vector<sg_int_info> info(b->info, b->info + b->ninfo);
  return should_load(q, info) ? 1 : 0;
}

int sg_query_run(sg_query* q) {
  if (!q) return SG_ERR_INVALID;
  sg_ctx* c = q->ctx;
  sg_table* t = q->table;
  cudaSetDevice(c->device);
  const auto t_begin = std::chrono::steady_clock::now();
  int rc = sg_table_sync(t);
  if (rc != SG_OK) return rc;
  rc = upload_table(t);
  if (rc != SG_OK) return rc;
  const bool reuse = q->planned && q->plan_version == t->version && !q->merged && !getenv("SG_NO_PLAN_REUSE");
  q->merged = false;
  q->kernel_ms = 0;  // statistics are per run
  q->launches = 0;
  q->d2h_bytes = 0;
  std::vector<uint32_t> list;
  if (reuse) {
    list = q->plan_list;
    q->skipped = q->plan_skipped;
    q->broken_staged = q->plan_broken;
    q->rows_scanned = q->plan_rows;
  } else {
  // block list: zone-map pruning + blocks already known broken for a referenced column
  std::vector<char> wanted((size_t)t->ncols, 0);
  auto want = [&](int col) {
    if (col >= 0 && col < t->ncols) wanted[(size_t)col] = 1;  // (make_plan reports columns out of range)
  };
  for (auto& f : q->filters) want(f.col_slot);
  for (auto& g : q->groups) want(g.col_slot);
  if (q->d.weight_col_slot >= 0) want(q->d.weight_col_slot);
  for (auto& a : q->aggs) want(a.col_slot);
  if (q->d.time_col_slot >= 0 && q->d.time_bucket > 0) want(q->d.time_col_slot);
  q->skipped = q->stream_skipped;
  q->broken_staged = 0;
  q->rows_scanned = 0;
  for (size_t i = 0; i < t->blocks.size(); i++) {
    if (!should_load(q, t->blocks[i].info)) {
      q->skipped++;
      continue;
    }
    bool broken = false;
    for (int cidx = 0; cidx < t->ncols; cidx++)
      if (wanted[(size_t)cidx] && (t->cols[i * (size_t)t->ncols + (size_t)cidx].flags & COL_BROKEN)) broken = true;
    if (broken) {
      q->broken_staged++;
      continue;
    }
    list.push_back((uint32_t)i);
    q->rows_scanned += t->blocks[i].num_records;
  }
  q->blocks_scanned = (int64_t)list.size();
  rc = make_plan(q, list);
  if (rc != SG_OK) return rc;
  rc = alloc_device(q);
  if (rc != SG_OK) return rc;
  q->planned = true;
  // hist Count == Count for an aggregation when, in every scanned block, its column is a value
  // array covering every row whose exact extents lie inside the accepted range: the kernel then
  // skips that reduction (accumulators-in-global plans) and the result takes Count
  q->hc_is_count.assign((size_t)q->plan.naggs, 0);
  q->hc_fill.assign((size_t)q->plan.naggs, 0);
  const bool multi = c->comm != nullptr && c->nranks > 1;
  if (q->plan.acc_repl == 0) {  // (multi-GPU: the proof is per rank — see hc_fill)
    for (int a = 0; a < q->plan.naggs; a++) {
      const KAgg& ka = q->plan.aggs[a];
      const int64_t amax = std::min(ka.reject_hi, ka.info_max);
      bool ok = !list.empty();
      for (uint32_t b : list) {
        const DevCol& dc = t->cols[(size_t)b * (size_t)t->ncols + (size_t)ka.col];
        if (dc.enc != SG_ENC_VALUES || (dc.flags & COL_IS_STR) || !(dc.flags & COL_STATS) ||
            dc.nitems < t->blocks[b].num_records || dc.vmin < ka.info_min || dc.vmax > amax) {
          ok = false;
          break;
        }
      }
      q->hc_is_count[(size_t)a] = ok && !multi ? 1 : 0;
      q->hc_fill[(size_t)a] = ok && multi ? 1 : 0;
      q->plan.aggs[a]._pad = ok ? 1u : 0u;
    }
  }
  q->plan_version = t->version;
  q->plan_list = list;
  q->plan_skipped = q->skipped;
  q->plan_broken = q->broken_staged;
  q->plan_rows = q->rows_scanned;
  }  // !reuse

  const auto t_planned = std::chrono::steady_clock::now();
  q->host_plan_ms = std::chrono::duration<double, std::milli>(t_planned - t_begin).count();
  // a block found broken by the kernel ("BLOCK SIZE CHANGED", row id >= NumRecords)
  // must contribute nothing: rerun without it (rare path)
  for (int attempt = 0; attempt < 8; attempt++) {
    if (q->sparse) {  // (every attempt rediscovers: the keys of a dropped block get no id)
      rc = discover_groups(q, list);
      if (rc != SG_OK) return rc;
    }
    rc = reset_accumulators(q);
    if (rc != SG_OK) return rc;
    rc = run_list(q, list);
    if (rc != SG_OK) return rc;
    const uint64_t* scal = q->scal;  // read back behind the kernel by run_list
    if (scal[SC_TIME_OVERFLOW] != 0) {
      c->set_err("query: rows fall outside the planned time axis (time_min/time_max too narrow)");
      return SG_ERR_INVALID;
    }
    if (q->sparse && scal[SC_SPARSE_MISSING] != 0) {
      c->set_err("query: " + std::to_string(scal[SC_SPARSE_MISSING]) + " rows' group keys were missing from the discovered sparse groups");
      return SG_ERR_STATE;
    }
    if (scal[SC_BROKEN] == 0) break;
    std::vector<uint32_t> status(t->blocks.size());
    CUDA_TRY(c, cudaMemcpy(status.data(), q->d_block_status, status.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<uint32_t> next;
    for (uint32_t b : list) {
      if (status[b]) {
        q->broken_staged++;
        q->rows_scanned -= t->blocks[b].num_records;
      } else {
        next.push_back(b);
      }
    }
    list.swap(next);
  }
  // multi-GPU: hist Counts this rank's kernel did not accumulate (they equal Count on this rank) are filled in
  // from the count array, so that every rank's array holds real values for the element-wise merge
  for (int a = 0; a < q->plan.naggs; a++)
    if ((size_t)a < q->hc_fill.size() && q->hc_fill[(size_t)a])
      CUDA_TRY(c, cudaMemcpyAsync(q->d_acc + q->off_hcount[(size_t)a], q->d_acc + q->off_count, (size_t)q->plan.nslots * 8,
                                  cudaMemcpyDeviceToDevice, c->stream));
  q->last_list = list;
  q->ran = true;
  q->host_run_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_planned).count();
  return SG_OK;
}

int sg_query_submit_block(sg_query* q, const sg_block_desc* b) {
  // streaming path: the block is staged into the query's table (H2D on the copy
  // stream) and scanned by sg_query_finish; zone-map pruning happens before staging
  if (!q || !b) return SG_ERR_INVALID;
  if (q->sparse_req) {
    q->ctx->set_err("sg_query_submit_block: sparse group accumulators scan every block twice (discovery, then "
                    "aggregation); stage the blocks with sg_table_add_block(s) and use sg_query_run");
    return SG_ERR_UNSUPPORTED;
  }
  std::vector<sg_int_info> info(b->info, b->info + b->ninfo);
  if (!should_load(q, info)) {
    q->stream_skipped++;
    return SG_OK;
  }
  return sg_table_add_block(q->table, b);
}

// ---- cross-GPU merge ---------------------------------------------------------------------------
// CombineResults across GPUs (table_query.go:155-170 across processes).  Each rank scanned its
// shard into dense accumulators laid out by ITS dictionaries.  When every rank's dictionaries
// (and time axis) agree — seeded tables, or shards that saw the same values in the same order —
// the merge is two element-wise all-reduces.  Otherwise the ranks first exchange their
// dictionaries (all-gather), build the same union dictionary in rank order, re-lay their
// accumulators by it, and then all-reduce.
static int nccl_fail(sg_ctx* c, const char* what, ncclResult_t r) {
  c->set_err(std::string(what) + ": " + (g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "?"));
  return SG_ERR_NCCL;
}

static int comm_allreduce_host(sg_ctx* c, uint64_t* v, size_t n, int dtype, int op) {
  uint64_t* d = nullptr;
  CUDA_TRY(c, pool_alloc(c, (void**)&d, n * 8));
  CUDA_TRY(c, cudaMemcpyAsync(d, v, n * 8, cudaMemcpyHostToDevice, c->stream));
  ncclResult_t r = g_nccl.AllReduce(d, d, n, dtype, op, c->comm, c->stream);
  if (r != 0) return nccl_fail(c, "ncclAllReduce", r);
  CUDA_TRY(c, cudaMemcpyAsync(v, d, n * 8, cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  pool_release(c, d);
  return SG_OK;
}

// every rank contributes `each` bytes; all[r*each ...] holds rank r's
static int comm_allgather_host(sg_ctx* c, const void* mine, size_t each, std::vector<uint8_t>& all) {
  uint8_t *ds = nullptr, *dr = nullptr;
  all.resize(each * (size_t)c->nranks);
  CUDA_TRY(c, pool_alloc(c, (void**)&ds, each));
  CUDA_TRY(c, pool_alloc(c, (void**)&dr, all.size()));
  CUDA_TRY(c, cudaMemcpyAsync(ds, mine, each, cudaMemcpyHostToDevice, c->stream));
  ncclResult_t r = g_nccl.AllGather(ds, dr, each, ncclUint8, c->comm, c->stream);
  if (r != 0) return nccl_fail(c, "ncclAllGather", r);
  CUDA_TRY(c, cudaMemcpyAsync(all.data(), dr, all.size(), cudaMemcpyDeviceToHost, c->stream));
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  pool_release(c, ds);
  pool_release(c, dr);
  return SG_OK;
}

static inline uint64_t fnv64(uint64_t h, const void* p, size_t n) {
  const uint8_t* b = (const uint8_t*)p;
  for (size_t i = 0; i < n; i++) h = (h ^ b[i]) * 0x100000001b3ull;
  return h;
}

// this rank's group axes, serialised: per axis  time: [i64 first][u64 radix]
//                                                str:  [u64 n] n x ([u32 len] bytes)
//                                                int:  [u64 n] n x i64
static void serialise_axes(const sg_query* q, std::vector<uint8_t>& out) {
  auto put = [&](const void* p, size_t n) { out.insert(out.end(), (const uint8_t*)p, (const uint8_t*)p + n); };
  const sg_table* t = q->table;
  for (auto& d : q->dims) {
    if (d.is_time) {
      int64_t first = q->plan.time_first;
      uint64_t radix = d.radix;
      put(&first, 8);
      put(&radix, 8);
    } else if (d.is_str) {
      const auto& strs = t->sdict[(size_t)d.col].strs;
      uint64_t n = d.radix - 1;  // the entries the plan was laid out by
      put(&n, 8);
      for (uint64_t i = 0; i < n; i++) {
        uint32_t len = (uint32_t)strs[(size_t)i].size();
        put(&len, 4);
        put(strs[(size_t)i].data(), len);
      }
    } else {
      const auto& vals = t->idict[(size_t)d.col].vals;
      uint64_t n = d.radix - 1;
      put(&n, 8);
      put(vals.data(), (size_t)n * 8);
    }
  }
}

static int remap_to_union(sg_query* q) {
  sg_ctx* c = q->ctx;
  Plan& P = q->plan;
  const int nr = c->nranks;
  std::vector<uint8_t> mine;
  serialise_axes(q, mine);
  uint64_t maxlen = mine.size();
  int rc = comm_allreduce_host(c, &maxlen, 1, ncclUint64, ncclMax);
  if (rc != SG_OK) return rc;
  const size_t each = (size_t)((maxlen + 15) & ~7ull) + 8;
  std::vector<uint8_t> padded(each, 0), all;
  uint64_t mylen = mine.size();
  memcpy(padded.data(), &mylen, 8);
  memcpy(padded.data() + 8, mine.data(), mine.size());
  rc = comm_allgather_host(c, padded.data(), each, all);
  if (rc != SG_OK) return rc;

  // union per axis, ranks in order; remap[axis][local code] -> union code
  const size_t nd = q->dims.size();
  std::vector<std::vector<std::string>> u_strs(nd);
  std::vector<std::vector<int64_t>> u_ints(nd);
  std::vector<std::unordered_map<std::string, uint32_t>> s_ids(nd);
  std::vector<std::unordered_map<int64_t, uint32_t>> i_ids(nd);
  std::vector<std::vector<uint32_t>> remap(nd);
  int64_t g_first = 0, g_last = 0;
  bool have_time = false;
  for (int r = 0; r < nr; r++) {
    const uint8_t* p = all.data() + (size_t)r * each;
    uint64_t len;
    memcpy(&len, p, 8);
    p += 8;
    const uint8_t* end = p + len;
    auto need = [&](size_t n) { return (size_t)(end - p) >= n; };
    for (size_t di = 0; di < nd; di++) {
      const GroupDim& d = q->dims[di];
      if (!need(8)) goto corrupt;
      if (d.is_time) {
        int64_t first;
        uint64_t radix;
        if (!need(16)) goto corrupt;
        memcpy(&first, p, 8);
        memcpy(&radix, p + 8, 8);
        p += 16;
        int64_t last = first + (int64_t)radix - 2;
        if (!have_time) {
          g_first = first;
          g_last = last;
          have_time = true;
        } else {
          g_first = std::min(g_first, first);
          g_last = std::max(g_last, last);
        }
        continue;
      }
      uint64_t n;
      memcpy(&n, p, 8);
      p += 8;
      if (r == c->rank) remap[di].assign((size_t)n + 1, 0);
      for (uint64_t i = 0; i < n; i++) {
        uint32_t uid;
        if (d.is_str) {
          uint32_t l;
          if (!need(4)) goto corrupt;
          memcpy(&l, p, 4);
          p += 4;
          if (!need(l)) goto corrupt;
          std::string sv((const char*)p, l);
          p += l;
          auto it = s_ids[di].find(sv);
          if (it == s_ids[di].end()) {
            uid = (uint32_t)u_strs[di].size();
            s_ids[di].emplace(sv, uid);
            u_strs[di].push_back(std::move(sv));
          } else {
            uid = it->second;
          }
        } else {
          int64_t v;
          if (!need(8)) goto corrupt;
          memcpy(&v, p, 8);
          p += 8;
          auto it = i_ids[di].find(v);
          if (it == i_ids[di].end()) {
            uid = (uint32_t)u_ints[di].size();
            i_ids[di].emplace(v, uid);
            u_ints[di].push_back(v);
          } else {
            uid = it->second;
          }
        }
        if (r == c->rank) remap[di][(size_t)i + 1] = uid + 1;
      }
    }
  }
  {
    // union slot space
    std::vector<GroupDim> ndims = q->dims;
    uint64_t stride = 1;
    for (size_t di = 0; di < nd; di++) {
      GroupDim& d = ndims[di];
      if (d.is_time) {
        const int64_t shift = P.time_first - g_first;
        remap[di].assign(d.radix, 0);
        for (uint32_t code = 1; code < d.radix; code++) remap[di][code] = (uint32_t)((int64_t)code + shift);
        d.radix = (uint32_t)(g_last - g_first + 2);
      } else {
        d.radix = (uint32_t)((d.is_str ? u_strs[di].size() : u_ints[di].size()) + 1);
      }
      d.stride = (uint32_t)stride;
      stride *= d.radix;
      if (stride > (uint64_t)MAX_SLOTS) {
        c->set_err("allreduce: union of the ranks' group keys exceeds the dense slot space");
        return SG_ERR_UNSUPPORTED;
      }
    }
    const uint32_t old_slots = P.nslots, new_slots = (uint32_t)stride;
    // old accumulators to the host, re-laid by the union, back to the device
    std::vector<uint64_t> h_old(q->acc_words);
    // (on the query's own stream: it does not synchronise with the legacy default stream, and a pageable
    // cudaMemcpy may return before its DMA has landed)
    CUDA_TRY(c, cudaMemcpyAsync(h_old.data(), q->d_acc, q->acc_words * 8, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    q->d2h_bytes += (int64_t)q->acc_words * 8;
    const size_t o_count = q->off_count;
    const std::vector<AccRegion> old = q->regions;
    rc = layout_accumulators(q, new_slots);
    if (rc != SG_OK) return rc;
    std::vector<uint64_t> h_new(q->acc_words, 0);
    for (size_t w = q->sum_words; w < q->acc_words; w++) h_new[w] = (uint64_t)INT64_MIN;
    for (size_t w = 0; w < SCALAR_WORDS; w++) h_new[w] = h_old[w];
    for (uint32_t s = 0; s < old_slots; s++) {
      if (h_old[o_count + s] == 0) continue;
      uint64_t ns = 0;
      for (size_t di = 0; di < nd; di++) {
        const GroupDim& od = q->dims[di];
        uint32_t code = (s / od.stride) % od.radix;
        ns += (uint64_t)remap[di][code] * ndims[di].stride;
      }
      for (size_t i = 0; i < old.size(); i++) {
        const size_t w = old[i].per_row;
        memcpy(&h_new[q->regions[i].off + (size_t)ns * w], &h_old[old[i].off + (size_t)s * w], w * 8);
      }
    }
    pool_release(c, q->d_acc);
    q->d_acc = nullptr;
    CUDA_TRY(c, pool_alloc(c, (void**)&q->d_acc, q->acc_words * 8));
    CUDA_TRY(c, cudaMemcpyAsync(q->d_acc, h_new.data(), q->acc_words * 8, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    q->dims = ndims;
    P.nslots = new_slots;
    if (have_time) P.time_first = g_first;
    q->m_strs = std::move(u_strs);
    q->m_ints = std::move(u_ints);
    q->merged = true;
  }
  return SG_OK;
corrupt:
  c->set_err("allreduce: malformed dictionary exchange");
  return SG_ERR_NCCL;
}

// signature (and serialised size) of the query's axes; hashing a 1M-string dictionary costs ~15 ms, so it is kept
// per (table version) — the axes of an un-merged query only change when blocks are staged
static uint64_t axes_signature(sg_query* q, size_t* size_out) {
  if (!q->merged && q->axes_sig_version == q->table->version + 1) {
    if (size_out) *size_out = q->axes_size;
    return q->axes_sig;
  }
  std::vector<uint8_t> axes;
  serialise_axes(q, axes);
  const uint64_t sig = fnv64(0xcbf29ce484222325ull, axes.data(), axes.size());
  if (!q->merged) {
    q->axes_sig = sig;
    q->axes_size = axes.size();
    q->axes_sig_version = q->table->version + 1;
  }
  if (size_out) *size_out = axes.size();
  return sig;
}

int sg_query_allreduce(sg_query* q) {
  if (!q || !q->ran) return SG_ERR_STATE;
  sg_ctx* c = q->ctx;
  if (!c->comm || c->nranks <= 1) return SG_OK;
  cudaSetDevice(c->device);
  if (q->hashed) {
    c->set_err("allreduce: a hashed slot space (group-by product beyond 2^26) is merged on one GPU only in this build");
    return SG_ERR_UNSUPPORTED;
  }
  q->acc.words = 0;  // the device copy is about to change
  // Small plans (the usual case: a few hundred groups): ONE collective.  Every rank writes a header
  // (block counters, signature of its axes) into its scalars and all-gathers its whole accumulator
  // array; each rank then reduces the gathered copies on the host (sum region, max region) — or, if
  // the signatures differ, falls through to the dictionary exchange below with its own copy intact.
  static const bool force_allreduce = getenv("SG_MERGE_ALLREDUCE") != nullptr;  // (tests: the large-plan path at any size)
  // (larger plans, such as C3's 0.94 MB per rank, go through the all-reduce path below: the host-reduce path is kept
  // for plans whose gathered copies are a few pages)
  if (q->acc_words * 8 * (size_t)c->nranks <= ((size_t)256 << 10) && !force_allreduce) {
    size_t axes_size = 0;
    const uint64_t sig = axes_signature(q, &axes_size);
    const size_t aw = q->acc_words, nr = (size_t)c->nranks;
    char* hp = c->scratch(64 + aw * 8 * nr);
    uint64_t* d_all = nullptr;
    if (!hp) {
      c->set_err("cudaHostAlloc (merge scratch) failed");
      return SG_ERR_CUDA;
    }
    CUDA_TRY(c, pool_alloc(c, (void**)&d_all, aw * 8 * nr));
    uint64_t* hdr = (uint64_t*)hp;  // the merge header: words SC_MERGE.. of the scalars
    hdr[0] = (uint64_t)q->broken_staged;
    hdr[1] = (uint64_t)q->skipped;
    hdr[2] = (uint64_t)q->rows_scanned;
    hdr[3] = (uint64_t)q->blocks_scanned;
    hdr[4] = sig;
    hdr[5] = (uint64_t)axes_size;
    hdr[6] = hdr[7] = 0;
    CUDA_TRY(c, cudaMemcpyAsync(q->d_acc + SC_MERGE, hdr, 64, cudaMemcpyHostToDevice, c->stream));
    ncclResult_t r = g_nccl.AllGather(q->d_acc, d_all, aw * 8, ncclUint8, c->comm, c->stream);
    if (r != 0) return nccl_fail(c, "ncclAllGather", r);
    uint64_t* all = (uint64_t*)(hp + 64);
    CUDA_TRY(c, cudaMemcpyAsync(all, d_all, aw * 8 * nr, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(c, cudaStreamSynchronize(c->stream));
    pool_release(c, d_all);
    q->d2h_bytes += (int64_t)(aw * 8 * nr);
    bool agree = true;
    for (size_t k = 0; k < nr; k++) agree = agree && all[k * aw + SC_MERGE_AXES] == sig && all[k * aw + SC_MERGE_AXES + 1] == (uint64_t)axes_size;
    // the counters are job totals on either path
    uint64_t tot[4] = {0, 0, 0, 0};
    for (size_t k = 0; k < nr; k++)
      for (int j = 0; j < 4; j++) tot[j] += all[k * aw + SC_MERGE + (size_t)j];
    if (agree) {
      uint64_t* h = q->acc.host(aw);  // build_result reads the merged host copy (the device copy stays per-rank)
      for (size_t w = 0; w < q->sum_words; w++) {
        uint64_t v = 0;
        for (size_t k = 0; k < nr; k++) v += all[k * aw + w];
        h[w] = v;
      }
      for (size_t w = q->sum_words; w < aw; w++) {
        int64_t v = INT64_MIN;
        for (size_t k = 0; k < nr; k++) v = std::max(v, (int64_t)all[k * aw + w]);
        h[w] = (uint64_t)v;
      }
      q->broken_staged = (int64_t)tot[0];
      q->skipped = (int64_t)tot[1];
      q->rows_scanned = (int64_t)tot[2];
      q->blocks_scanned = (int64_t)tot[3];
      return SG_OK;
    }
    // differing axes: every rank sees that in the same gathered data and takes the exchange path
    CUDA_TRY(c, cudaMemsetAsync(q->d_acc + SC_MERGE, 0, 64, c->stream));
  }
  // ---- larger plans: element-wise all-reduces (sums: scalars, count, hcount, sum, buckets; max: vmax) --------
  const uint64_t sig = axes_signature(q, nullptr);
  const uint64_t sa = sig & 0x3fffffffull, sb = (sig >> 32) & 0x3fffffffull;
  const uint64_t n = (uint64_t)c->nranks;
  auto ar = [&](const uint64_t* src, uint64_t* dst, size_t cnt, int dtype, int op) -> int {
    ncclResult_t r = g_nccl.AllReduce(src, dst, cnt, dtype, op, c->comm, c->stream);
    return r != 0 ? nccl_fail(c, "ncclAllReduce", r) : (int)SG_OK;
  };
  const bool whole = q->acc_words * 8 <= ((size_t)4 << 20);  // small enough to read back right behind the merge
  int rc = SG_OK;
  // ... which is only safe when every rank's accumulator array has the same length BY CONSTRUCTION (an element-wise
  // collective with different counts on different ranks is undefined): every group axis is a dictionary still
  // exactly as the host seeded it (sg_table_dict_seed_*) or the time axis (planned from the query's IntInfo).
  // Otherwise a small host-synchronous collective compares the signatures first, as before.
  bool sized_alike = !q->merged;
  for (const GroupDim& d : q->dims) {
    if (d.is_time) continue;
    const sg_table* t = q->table;
    const int64_t have = d.is_str ? (int64_t)t->sdict[(size_t)d.col].strs.size() : (int64_t)t->idict[(size_t)d.col].vals.size();
    const int64_t seeded = d.is_str ? t->sseed[(size_t)d.col] : t->iseed[(size_t)d.col];
    if (seeded < 0 || seeded != have) sized_alike = false;
  }
  if (getenv("SG_MERGE_ONE_STEP")) sized_alike = true;  // (diagnostics: the caller vouches for equal sizes)
  if (c->nranks <= 8 && sized_alike && !getenv("SG_MERGE_TWO_STEP")) {
    // The job-wide block counters and the answer to "do the ranks agree on the slot space?" ride in spare scalar
    // words of the SUM all-reduce itself: with two independent 30-bit signatures s of the serialised axes, every
    // rank checks  sum(s) == n*s_mine  and  sum(s^2) == n*s_mine^2  (exact in 64 bits for n <= 8) on the merged
    // copy; if the signatures differ the variance is positive and the test fails on EVERY rank, so all ranks take
    // the same branch.  The reduction is out of place: a rank's own accumulators survive for the dictionary
    // exchange of that (rare) case.  No host-synchronous collective ahead of the merge (it cost ~80 us a query).
    char* hp = c->scratch(64 + (whole ? q->acc_words * 8 : 128));
    uint64_t* d_merged = nullptr;
    if (!hp) {
      c->set_err("cudaHostAlloc (merge scratch) failed");
      return SG_ERR_CUDA;
    }
    CUDA_TRY(c, pool_alloc(c, (void**)&d_merged, q->acc_words * 8));
    uint64_t* hc = (uint64_t*)hp;  // the merge header: words SC_MERGE.. of the scalars
    hc[0] = (uint64_t)q->broken_staged;
    hc[1] = (uint64_t)q->skipped;
    hc[2] = (uint64_t)q->rows_scanned;
    hc[3] = (uint64_t)q->blocks_scanned;
    hc[4] = sa;
    hc[5] = sa * sa;
    hc[6] = sb;
    hc[7] = sb * sb;
    cudaError_t ce = cudaMemcpyAsync(q->d_acc + SC_MERGE, hc, 64, cudaMemcpyHostToDevice, c->stream);
    if (ce == cudaSuccess) {
      rc = ar(q->d_acc, d_merged, q->sum_words, ncclUint64, ncclSum);
      if (rc == SG_OK && q->acc_words > q->sum_words)
        rc = ar(q->d_acc + q->sum_words, d_merged + q->sum_words, q->acc_words - q->sum_words, ncclInt64, ncclMax);
    }
    if (ce == cudaSuccess && rc == SG_OK) ce = cudaMemsetAsync(q->d_acc + SC_MERGE, 0, 64, c->stream);  // own copy as it was
    // the merged array comes back whole into the query's host copy when small enough, else its scalars alone
    uint64_t* hm = (uint64_t*)(hp + 64);
    if (ce == cudaSuccess && rc == SG_OK) {
      if (whole) {
        rc = read_acc(q, q->acc, d_merged, q->acc_words, PIN_WHOLE_FROM, hp + 64);
        hm = q->acc.data();
      } else {
        ce = cudaMemcpyAsync(hm, d_merged, 128, cudaMemcpyDeviceToHost, c->stream);
        if (ce == cudaSuccess) ce = cudaStreamSynchronize(c->stream);
      }
    }
    if (ce != cudaSuccess || rc != SG_OK) {
      pool_release(c, d_merged);
      if (rc != SG_OK) return rc;
      c->set_err(std::string("merge: ") + cudaGetErrorString(ce));
      return SG_ERR_CUDA;
    }
    const uint64_t* m = hm + SC_MERGE;
    const bool agree = m[4] == n * sa && m[5] == n * sa * sa && m[6] == n * sb && m[7] == n * sb * sb;
    q->broken_staged = (int64_t)m[0];
    q->skipped = (int64_t)m[1];
    q->rows_scanned = (int64_t)m[2];
    q->blocks_scanned = (int64_t)m[3];
    if (agree) {
      // the merged copy becomes the query's accumulator array (the plan's device pointers name q->d_acc)
      ce = cudaMemsetAsync(d_merged + SC_MERGE, 0, 64, c->stream);
      if (ce == cudaSuccess) ce = cudaMemcpyAsync(q->d_acc, d_merged, q->acc_words * 8, cudaMemcpyDeviceToDevice, c->stream);
      if (ce == cudaSuccess && !whole) ce = cudaStreamSynchronize(c->stream);
      pool_release(c, d_merged);  // (stream-ordered pool: reuse waits for the copy queued above)
      if (ce != cudaSuccess) {
        q->acc.words = 0;
        c->set_err(std::string("merge: ") + cudaGetErrorString(ce));
        return SG_ERR_CUDA;
      }
      if (whole) {
        for (int k = SC_MERGE; k < SCALAR_WORDS; k++) hm[k] = 0;
        q->d2h_bytes += (int64_t)q->acc_words * 8;
      }
      return SG_OK;
    }
    q->acc.words = 0;  // (this rank's layout differs from others': the copy is no merge)
    pool_release(c, d_merged);
    rc = remap_to_union(q);  // differing dictionaries / time axes: re-lay this rank's accumulators by the union
    if (rc != SG_OK) return rc;
  } else {
    uint64_t hc[8] = {(uint64_t)q->broken_staged, (uint64_t)q->skipped, (uint64_t)q->rows_scanned, (uint64_t)q->blocks_scanned,
                      sa, sa * sa, sb, sb * sb};
    if (c->nranks <= 8) {
      rc = comm_allreduce_host(c, hc, 8, ncclUint64, ncclSum);
      if (rc != SG_OK) return rc;
    } else {
      // more ranks than the exact-moment test covers: max of sig and of ~sig (equal iff all equal)
      uint64_t pr[2] = {sig, ~sig};
      rc = comm_allreduce_host(c, pr, 2, ncclUint64, ncclMax);
      if (rc != SG_OK) return rc;
      rc = comm_allreduce_host(c, hc, 4, ncclUint64, ncclSum);
      if (rc != SG_OK) return rc;
      const bool same = pr[0] == ~pr[1];
      hc[4] = same ? sa * n : ~0ull;
      hc[5] = sa * sa * n;
      hc[6] = sb * n;
      hc[7] = sb * sb * n;
    }
    const bool agree = hc[4] == n * sa && hc[5] == n * sa * sa && hc[6] == n * sb && hc[7] == n * sb * sb;
    q->broken_staged = (int64_t)hc[0];
    q->skipped = (int64_t)hc[1];
    q->rows_scanned = (int64_t)hc[2];
    q->blocks_scanned = (int64_t)hc[3];
    if (!agree) {
      rc = remap_to_union(q);
      if (rc != SG_OK) return rc;
    }
  }
  // in place (after a dictionary exchange, or the two-step path): the counters are already job totals
  rc = ar(q->d_acc, q->d_acc, q->sum_words, ncclUint64, ncclSum);
  if (rc == SG_OK && q->acc_words > q->sum_words)
    rc = ar(q->d_acc + q->sum_words, q->d_acc + q->sum_words, q->acc_words - q->sum_words, ncclInt64, ncclMax);
  if (rc != SG_OK) return rc;
  // read the merged accumulators back behind the all-reduces (small plans, through the scratch area into a vector):
  // build_result then needs no further copy
  if (whole) {
    char* hp = c->scratch(q->acc_words * 8);
    if (hp) {
      rc = read_acc(q, q->acc, q->d_acc, q->acc_words, SIZE_MAX, hp);
      if (rc != SG_OK) return rc;
      q->d2h_bytes += (int64_t)q->acc_words * 8;
      return SG_OK;
    }
  }
  CUDA_TRY(c, cudaStreamSynchronize(c->stream));
  return SG_OK;
}

int sg_query_finish(sg_query* q, sg_result** out) {
  if (!q || !out) return SG_ERR_INVALID;
  if (!q->ran) {
    int rc = sg_query_run(q);
    if (rc != SG_OK) return rc;
  }
  cudaSetDevice(q->ctx->device);
  static const bool host_timing = getenv("SG_HOST_TIMING") != nullptr;
  const auto t0 = std::chrono::steady_clock::now();
  int rc = build_result(q, out);
  if (host_timing)
    fprintf(stderr, "[sg host] build_result %.3f ms (run: plan+list %.3f, launch+wait %.3f)\n",
            std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count(), q->host_plan_ms, q->host_run_ms);
  return rc;
}

double sg_query_kernel_ms(sg_query* q) { return q ? q->kernel_ms : 0; }
int64_t sg_query_kernel_launches(sg_query* q) { return q ? q->launches : 0; }

int sg_query_stats(sg_query* q, sg_stats* s) {
  if (!q || !s) return SG_ERR_INVALID;
  memset(s, 0, sizeof(*s));
  s->kernel_ms = q->kernel_ms;
  s->kernel_launches = q->launches;
  s->h2d_bytes = q->table->h2d_bytes;
  s->d2h_bytes = q->d2h_bytes;
  s->rows_scanned = q->rows_scanned;
  s->blocks_scanned = q->blocks_scanned;
  s->encoded_bytes = q->table->encoded_bytes;
  return SG_OK;
}

// ===========================================================================
// result accessors
// ===========================================================================
void sg_result_free(sg_result* r) { delete r; }
int64_t sg_result_matched_count(sg_result* r) { return r ? r->matched : 0; }
int64_t sg_result_num_groups(sg_result* r) { return r ? (int64_t)(r->lazy ? r->order.size() : r->groups.size()) : 0; }
int64_t sg_result_num_groups_total(sg_result* r) { return r ? r->ngroups_total : 0; }
int64_t sg_result_num_broken(sg_result* r) { return r ? r->broken : 0; }
int64_t sg_result_num_skipped(sg_result* r) { return r ? r->skipped : 0; }

static ResultGroup* pick_group(sg_result* r, int64_t i) {
  if (!r) return nullptr;
  if (i == -1) return &r->total;
  if (r->lazy) {
    if (i < 0 || (size_t)i >= r->order.size()) return nullptr;
    auto it = r->cache.find(i);
    if (it == r->cache.end()) {
      std::unique_ptr<ResultGroup> g(new ResultGroup());
      make_group(r->q, r->acc.data(), r->order[(size_t)i], *g, nullptr, r->samples.empty() ? nullptr : &r->samples);
      it = r->cache.emplace(i, std::move(g)).first;
    }
    return it->second.get();
  }
  if (i < 0 || (size_t)i >= r->groups.size()) return nullptr;
  return &r->groups[(size_t)i];
}

int sg_result_group(sg_result* r, int64_t i, uint64_t* key_out, int64_t* count, int64_t* samples) {
  ResultGroup* g = pick_group(r, i);
  if (!g) return SG_ERR_INVALID;
  if (key_out)
    for (size_t k = 0; k < g->key.size(); k++) key_out[k] = g->key[k];
  if (count) *count = g->count;
  if (samples) *samples = g->samples >= 0 ? g->samples : g->count;  // unweighted: Samples == Count (aggregate.go:202-203)
  return SG_OK;
}
int sg_result_group_key(sg_result* r, int64_t i, const char** bytes, int64_t* len) {
  ResultGroup* g = pick_group(r, i);
  if (!g) return SG_ERR_INVALID;
  *bytes = g->skey.data();
  *len = (int64_t)g->skey.size();
  return SG_OK;
}

// hist Min/Max as the reference tracks them (hist_basic.go:34-41,120-126;
// hist_multi.go:31-33): hist mode and MultiHist start at the table extents;
// BasicHist in avg mode starts at 0 and is not tracked by this build.
static void hist_minmax(sg_result* r, const ResultGroup* g, int a, int64_t* mn, int64_t* mx) {
  const HistLayout& L = r->layouts[(size_t)a];
  if (L.tracked || L.multi) {
    *mn = L.info_min;
    *mx = std::max(L.info_max, g->vx(a));
  } else {
    *mn = 0;
    *mx = 0;
  }
}

int sg_result_hist(sg_result* r, int64_t i, int32_t a, sg_hist_view* out) {
  ResultGroup* g = pick_group(r, i);
  if (!g || a < 0 || a >= r->naggs || !out) return SG_ERR_INVALID;
  memset(out, 0, sizeof(*out));
  if (i == -1 && !r->has_total_hists) return 0;
  if (g->hc(a) == 0) return 0;  // no hist for this aggregation (Q7)
  const HistLayout& L = r->layouts[(size_t)a];
  out->count = g->hc(a);
  out->sum = g->sm(a);
  hist_minmax(r, g, a, &out->min, &out->max);
  out->avg = (double)out->sum / (double)out->count;
  out->num_buckets = (int32_t)L.num_buckets;
  out->bucket_size = L.subs.size() == 1 ? (int32_t)L.subs[0].bsize : 0;
  out->nvalues = (int32_t)L.nvals_total;
  out->nsubhists = L.multi ? (int32_t)L.subs.size() : 0;
  out->values = g->vals(a) ? g->vals(a)->data() : nullptr;
  return 1;
}

int sg_result_percentiles(sg_result* r, int64_t i, int32_t a, int64_t* out100) {
  ResultGroup* g = pick_group(r, i);
  if (!g || a < 0 || a >= r->naggs) return SG_ERR_INVALID;
  if (g->hc(a) == 0 || !g->vals(a)) return 0;
  int64_t mn, mx;
  hist_minmax(r, g, a, &mn, &mx);
  return percentiles(r->layouts[(size_t)a], g->vals(a)->data(), g->hc(a), mn, out100);
}

double sg_result_stddev(sg_result* r, int64_t i, int32_t a) {
  ResultGroup* g = pick_group(r, i);
  if (!g || a < 0 || a >= r->naggs || g->hc(a) == 0 || !g->vals(a)) return NAN;
  int64_t mn, mx;
  hist_minmax(r, g, a, &mn, &mx);
  double avg = (double)g->sm(a) / (double)g->hc(a);
  return stddev(r->layouts[(size_t)a], g->vals(a)->data(), g->hc(a), avg, mn);
}

int64_t sg_result_sparse_buckets(sg_result* r, int64_t i, int32_t a, int64_t* edges, int64_t* counts, int64_t cap) {
  ResultGroup* g = pick_group(r, i);
  if (!g || a < 0 || a >= r->naggs) return SG_ERR_INVALID;
  if (g->hc(a) == 0 || !g->vals(a)) return 0;
  auto m = sparse_buckets(r->layouts[(size_t)a], g->vals(a)->data());
  int64_t n = 0;
  for (auto& kv : m) {
    if (edges && n < cap) {
      edges[n] = kv.first;
      counts[n] = kv.second;
    }
    n++;
  }
  return n;
}

int64_t sg_result_num_time_buckets(sg_result* r) { return r ? (int64_t)r->time_keys.size() : 0; }
int64_t sg_result_time_bucket(sg_result* r, int64_t b) {
  if (!r || b < 0 || (size_t)b >= r->time_keys.size()) return 0;
  return r->time_keys[(size_t)b];
}
sg_result* sg_result_time_slice(sg_result* r, int64_t b) {
  if (!r || b < 0 || (size_t)b >= r->time_slices.size()) return nullptr;
  return r->time_slices[(size_t)b].get();
}

}  // extern "C"
