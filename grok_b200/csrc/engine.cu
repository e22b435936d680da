/*
 * grok_b200/csrc/engine.cu -- the tile engine behind include/grok_b200.h.
 *
 * Replaces, for the tiles it is given, the per-tile pipeline of the reference
 *   encode: TileProcessorCompress::preCompressTile / buildCompressDAG / doCompress
 *           (tile_processor/TileProcessorCompress.cpp L104-254, L347-531, L539-)  up to, not
 *           including, rate allocation and T2;
 *   decode: TileProcessor::scheduleAndRunDecompress (tile_processor/TileProcessor.cpp L1272-)
 *           after the T2 parse.
 * The Taskflow DAG (dcShift -> MCT -> per-level vert/horiz -> T1) becomes stream-ordered kernel
 * launches over ALL selected tiles at once: one launch per decomposition level, one for the
 * block coder.  Buffers are image-shaped planes in HBM addressed by canvas coordinate, so a
 * tile is a view, tiles of every size batch into the same launch, and the engine never copies
 * a tile out of the image (the reference's preCompressTile row copy disappears).
 *
 * Product code: fails loudly (negative return + b2k_last_error) without a CUDA device; there is
 * no CPU fallback here -- the host (Grok) owns that decision via the >0 return convention.
 */
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <map>
#include <mutex>
#include <unordered_map>
#include <string>
#include <vector>

#include "b2k_internal.h"
#include "geometry.h"
#include "t2_device.h"
#include "t2_decode.h"
#include "t2_parse.h"
#include "t2_plan.h"

using namespace b2k;

static thread_local std::string g_err;
static std::atomic<uint64_t> g_launches{0};
static std::atomic<int> g_pack_policy{-1}; /* host packing: -1 auto (PackTuner), 0 never, 1 always */
static std::atomic<int> g_last_pack[2]{{-1}, {-1}};
void b2k_count_launch(void) { g_launches.fetch_add(1, std::memory_order_relaxed); }

#define CUDA_TRY(expr)                                                                             \
  do                                                                                               \
  {                                                                                                \
    cudaError_t _e = (expr);                                                                       \
    if(_e != cudaSuccess)                                                                          \
    {                                                                                              \
      g_err = std::string(#expr) + ": " + cudaGetErrorString(_e);                                  \
      return -1;                                                                                   \
    }                                                                                              \
  } while(0)

struct b2k_engine
{
  int device = 0;
  cudaStream_t stream = nullptr, copy_stream = nullptr, h2d_stream = nullptr;
  cudaStream_t aux[4] = {nullptr, nullptr, nullptr, nullptr}; /* latency-bound side kernels run concurrently here */
  cudaDeviceProp prop{};
  /* b2k_encode / b2k_decode keep the job (device buffers, plans) of the last coding they saw.  The cache and its lock
     belong to the engine: calls on one engine are serialised, engines (one per GPU) run side by side */
  std::mutex mu;
  b2k_device_job* cached = nullptr;
  cudaEvent_t caller_ev = nullptr; /* b2k_encode_device / b2k_decode_device: orders the engine's streams after the caller's */
  uint8_t* d_cs = nullptr;         /* b2k_encode_codestream_device: the last code stream */
  uint64_t cs_cap = 0;
  /* b2k_codestream_window_device_stats: the last windowed device parse's wanted tiles and the bytes its arena takes */
  bool have_window_stats = false;
  uint32_t window_tiles = 0;
  uint64_t window_bytes = 0;
  /* b2k_decode_codestreams_device: the batch job (beside `cached`, so that single and batch calls alternate without
     replanning), each stream's text of the last call, and the gather tables and header staging of a call */
  b2k_device_job* batch = nullptr;
  std::vector<std::string> batch_errors;
  CopyEntry* d_copy = nullptr;
  CopyEntry* h_copy = nullptr;     /* pinned */
  uint32_t copy_cap = 0;
  uint8_t* d_hdr = nullptr;        /* the header prefixes, end to end */
  uint8_t* h_hdr = nullptr;        /* pinned */
  uint64_t hdr_cap = 0;
  /* b2k_encode_codestreams_device: the code streams of the last call (not d_cs: a batch leaves the single call's stream
     alone) and each image's text */
  uint8_t* d_bcs = nullptr;
  uint64_t bcs_cap = 0;
  std::vector<std::string> enc_batch_errors;
  /* b2k_codestream_parse_device_stats: the plan of the last device parse (single, window or batch); cleared when a job
     drops that plan */
  T2Parse* last_parse = nullptr;
};

/* ---- device memory cache --------------------------------------------------------------------------------------
 * Jobs come and go with the coding (every windowed decode is a new virtual image, SURVEY 8f N3) and cudaMalloc /
 * cudaFree synchronise the device and cost milliseconds per gigabyte.  Freed job buffers are kept per device and
 * handed out again to requests of about the same size (best fit, at most 25 % slack); the cache is trimmed, largest
 * first, above B2K_DEV_CACHE_GB (default 16: a fifth of an H100's 80 GB, more than config 4's job needs). */
namespace {
struct DevCache
{
  std::mutex mu;
  std::multimap<size_t, void*> free_;
  std::unordered_map<void*, size_t> live;
  size_t cached = 0;
};
DevCache g_devcache[32];
size_t dev_cache_limit()
{
  static const size_t v = [] {
    const char* e = getenv("B2K_DEV_CACHE_GB");
    return (size_t)(e ? atof(e) : 16.0) << 30;
  }();
  return v;
}
cudaError_t dev_alloc(void** p, size_t n)
{
  int dev = 0;
  cudaGetDevice(&dev);
  DevCache& C = g_devcache[dev & 31];
  const size_t gran = std::max<size_t>(256u << 10, n >> 4);
  const size_t want = (n + gran - 1) / gran * gran;
  {
    std::lock_guard<std::mutex> lk(C.mu);
    auto it = C.free_.lower_bound(want);
    if(it != C.free_.end() && it->first <= want + want / 4)
    {
      *p = it->second;
      C.live[*p] = it->first;
      C.cached -= it->first;
      C.free_.erase(it);
      return cudaSuccess;
    }
  }
  cudaError_t e = cudaMalloc(p, want);
  if(e != cudaSuccess)
  { /* give the cache back and try once more */
    (void)cudaGetLastError();
    std::vector<void*> drop;
    {
      std::lock_guard<std::mutex> lk(C.mu);
      for(auto& kv : C.free_)
        drop.push_back(kv.second);
      C.free_.clear();
      C.cached = 0;
    }
    for(void* q : drop)
      cudaFree(q);
    e = cudaMalloc(p, want);
  }
  if(e == cudaSuccess)
  {
    std::lock_guard<std::mutex> lk(C.mu);
    C.live[*p] = want;
  }
  return e;
}
cudaError_t dev_free(void* p)
{
  if(!p)
    return cudaSuccess;
  int dev = 0;
  cudaGetDevice(&dev);
  DevCache& C = g_devcache[dev & 31];
  std::vector<void*> drop;
  {
    std::lock_guard<std::mutex> lk(C.mu);
    auto it = C.live.find(p);
    if(it == C.live.end())
      drop.push_back(p); /* not ours (or another device's): plain free */
    else
    {
      C.free_.insert({it->second, p});
      C.cached += it->second;
      C.live.erase(it);
      while(C.cached > dev_cache_limit() && !C.free_.empty())
      {
        auto big = std::prev(C.free_.end());
        drop.push_back(big->second);
        C.cached -= big->first;
        C.free_.erase(big);
      }
    }
  }
  for(void* q : drop)
    cudaFree(q);
  return cudaSuccess;
}
} // namespace
template <class T>
static inline cudaError_t dev_alloc_t(T** p, size_t n) { return dev_alloc(reinterpret_cast<void**>(p), n); }

/* the same for pinned host memory (descriptor tables, staging rings): cudaHostAlloc / cudaFreeHost are slower still */
namespace {
struct HostCache
{
  std::mutex mu;
  std::multimap<size_t, void*> free_;
  std::unordered_map<void*, size_t> live;
  size_t cached = 0;
} g_hostcache;
cudaError_t host_alloc(void** p, size_t n)
{
  const size_t gran = std::max<size_t>(64u << 10, n >> 4);
  const size_t want = (n + gran - 1) / gran * gran;
  {
    std::lock_guard<std::mutex> lk(g_hostcache.mu);
    auto it = g_hostcache.free_.lower_bound(want);
    if(it != g_hostcache.free_.end() && it->first <= want + want / 4)
    {
      *p = it->second;
      g_hostcache.live[*p] = it->first;
      g_hostcache.cached -= it->first;
      g_hostcache.free_.erase(it);
      return cudaSuccess;
    }
  }
  const cudaError_t e = cudaHostAlloc(p, want, cudaHostAllocDefault);
  if(e == cudaSuccess)
  {
    std::lock_guard<std::mutex> lk(g_hostcache.mu);
    g_hostcache.live[*p] = want;
  }
  return e;
}
cudaError_t host_free(void* p)
{
  if(!p)
    return cudaSuccess;
  std::vector<void*> drop;
  {
    std::lock_guard<std::mutex> lk(g_hostcache.mu);
    auto it = g_hostcache.live.find(p);
    if(it == g_hostcache.live.end())
      drop.push_back(p);
    else
    {
      g_hostcache.free_.insert({it->second, p});
      g_hostcache.cached += it->second;
      g_hostcache.live.erase(it);
      while(g_hostcache.cached > ((size_t)8 << 30) && !g_hostcache.free_.empty())
      {
        auto big = std::prev(g_hostcache.free_.end());
        drop.push_back(big->second);
        g_hostcache.cached -= big->first;
        g_hostcache.free_.erase(big);
      }
    }
  }
  for(void* q : drop)
    cudaFreeHost(q);
  return cudaSuccess;
}
} // namespace
template <class T>
static inline cudaError_t host_alloc_t(T** p, size_t n) { return host_alloc(reinterpret_cast<void**>(p), n); }
/* from here on the engine's device and pinned buffers come from the caches */
#define cudaMalloc(p, n) dev_alloc_t((p), (n))
#define cudaFree(p) dev_free((void*)(p))
#define cudaHostAlloc(p, n, flags) host_alloc_t((p), (n))
#define cudaFreeHost(p) host_free((void*)(p))

/* ---- a plane set: `n` image-shaped 32-bit planes addressed by canvas coordinate ------------- */
struct Planes
{
  int32_t* base = nullptr;
  uint32_t pitch = 0, rows = 0; /* elements, rows */
  uint32_t X0 = 0, Y0 = 0;      /* canvas coordinate stored at column 0 / row 0 */
  int n = 0;
  size_t plane_elems() const { return (size_t)pitch * rows; }
  int32_t* at(int c, uint32_t x, uint32_t y) const { return base + (size_t)c * plane_elems() + (size_t)(y - Y0) * pitch + (x - X0); }
};

static int alloc_planes(Planes& p, int n, uint32_t cx0, uint32_t cy0, uint32_t cx1, uint32_t cy1)
{
  p.n = n;
  p.X0 = cx0 & ~31u; /* 128-byte aligned canvas columns */
  p.Y0 = cy0;
  p.pitch = ((cx1 - p.X0) + 31u + 32u) & ~31u; /* slack: vector loads of halo lanes stay inside */
  p.rows = (cy1 - cy0) + 2;
  CUDA_TRY(cudaMalloc(&p.base, (size_t)n * p.plane_elems() * sizeof(int32_t)));
  CUDA_TRY(cudaMemset(p.base, 0, (size_t)n * p.plane_elems() * sizeof(int32_t)));
  return 0;
}

struct LevelLaunch
{
  std::vector<DwtLevelDesc> descs;
  DwtLevelDesc* d_descs = nullptr;
  int nc = 1, max_jobs = 0;
  bool point = false;              /* numres = 1: no wavelet level, the launch is the point transform alone */
  uint32_t max_w = 0, max_h = 0;   /* point launches: largest tile component */
  uint64_t alg_bytes = 0; /* one read + one write of every sample of the level */
  std::vector<uint32_t> tile_first; /* descs of selected tile ti are [tile_first[ti], tile_first[ti+1]) */
};

/* Whether the int32 entry points should narrow to 16-bit containers on the host is a property of the
   machine at that moment: it halves the PCIe bytes but triples the host DRAM traffic, so it wins while
   PCIe is the bound (one or two GPUs per socket, or unpinned caller memory) and loses once several
   ranks share a socket's DRAM.  Default policy: time both ways on the first calls, keep the faster,
   look at the other one again every 64 calls. */
/* pipeline chunks per call (tile granular) and their events: purpose 0 chunk done on its stream, 1 chunk's
   upload done, 2 side-stream / scan done, 3 misc */
#define B2K_MAX_CHUNKS 32
#define CEV(purpose, k) ((purpose) * (B2K_MAX_CHUNKS + 1) + (int)(k))

struct PackTuner
{
  int calls = 0;
  double best[2] = {1e30, 1e30}; /* [0] direct, [1] packed: best wall ms seen while probing */
  double recent = 0;             /* EMA of the chosen mode */
  int choice = -1;
  bool probing_other = false;
  bool next_mode()
  {
    if(choice < 0)
      return (calls & 1) == 0; /* packed, direct, packed, direct, packed, direct */
    probing_other = (calls % 64) == 63;
    return probing_other ? !choice : (choice != 0);
  }
  void record(bool packed, double ms)
  {
    ++calls;
    if(choice < 0)
    {
      if(calls > 1 || !packed) /* the very first packed call allocates the staging buffer */
        best[packed ? 1 : 0] = std::min(best[packed ? 1 : 0], ms);
      if(calls >= 6)
      {
        choice = best[1] < best[0] ? 1 : 0;
        recent = best[choice];
      }
      return;
    }
    if(probing_other)
    {
      if(ms < 0.9 * recent)
      {
        choice = packed ? 1 : 0;
        recent = ms;
      }
      probing_other = false;
      return;
    }
    recent = 0.9 * recent + 0.1 * ms;
  }
};

struct b2k_device_job
{
  b2k_engine* eng = nullptr;
  b2k_coding cp{};
  uint32_t tile_mod = 1, tile_rem = 0;
  TileGrid grid{};
  std::vector<uint32_t> tiles;
  std::vector<Rect> tile_rects;
  /* a batch job (b2k_decode_codestreams_device) holds `slots` images of one coding: slot s of component c is plane
     s * numcomps + c of img, coef and ll[], and the selected tiles are slot 0's tiles, then slot 1's, ...  slot_tiles per
     slot; tile_slot[ti] is selected tile ti's slot.  A single image is one slot. */
  uint32_t slots = 1, slot_tiles = 0;
  std::vector<uint32_t> tile_slot;
  BatchDst* d_batch_dst = nullptr; /* the conversion's table: per component (or one for interleaved images), per slot */
  BatchDst* h_batch_dst = nullptr; /* pinned */
  BatchSrc* d_batch_src = nullptr; /* b2k_encode_codestreams_device's conversion table, laid out likewise */
  BatchSrc* h_batch_src = nullptr; /* pinned */
  std::vector<std::vector<BandQuant>> quant; /* [comp][band] */
  std::vector<b2k_block> blocks;       /* every block, enumeration order */
  std::vector<uint32_t> coded_index;   /* blocks with area, index into `blocks` */
  std::vector<float> dec_quant;        /* per coded block: decoder step / 2^(31-Kmax) */
  std::vector<uint32_t> coded_first;   /* coded blocks of selected tile ti are [coded_first[ti], coded_first[ti+1]) */
  std::vector<uint32_t> chunk_tile;    /* pipeline chunks: selected tiles [chunk_tile[k], chunk_tile[k+1]) */
  cudaEvent_t chunk_ev[4 * (B2K_MAX_CHUNKS + 1)]{}; /* [purpose][chunk], see CEV() */
  uint32_t max_cblk_w = 0;
  HtEncodeLimits enc_limits{0, 0};     /* shared-memory sizing of the HT encoder launches */

  Planes img, coef, ll[2];
  uint16_t* d_stage = nullptr;         /* 16-bit containers crossing PCIe, planar or pixel-interleaved (stage_container), lazily */
  std::vector<LevelLaunch> fwd, inv;   /* launch order */
  HtBlockDesc* d_enc_desc = nullptr;
  HtBlockDesc* d_dec_desc = nullptr;
  std::vector<HtBlockDesc> h_enc_desc;
  HtBlockDesc* h_dec_desc = nullptr;   /* pinned staging */
  HtBlockOut* d_out = nullptr;
  uint64_t* d_offsets = nullptr;
  uint32_t* d_recs = nullptr;     /* decode: per-quad records between the two decode phases */
  float* d_dec_quant = nullptr;
  HtBlockOut* d_dec_status = nullptr;
  uint64_t total_quads = 0, group_quads = 0; /* record scratch: closed groups / largest block of the open group */
  uint8_t* d_scratch = nullptr;
  uint64_t scratch_bytes = 0;
  uint8_t* d_bytes = nullptr;
  uint64_t bytes_cap = 0, bytes_used = 0;
  /* the arena was sized from a coding of the image the job holds: the round trips skip their sizing pass.  A new image
     (b2k_job_upload, or b2k_job_inverse of the coefficient planes) or a caller's arena (b2k_job_t1_decode_blocks) clears it */
  bool arena_sized = false;
  int* d_err = nullptr;
  /* pinned host staging for results */
  HtBlockOut* h_out = nullptr;
  uint64_t* h_offsets = nullptr;
  cudaEvent_t ev[8]{};
  float last_level1_ms = 0.f, last_inv_level1_ms = 0.f;
  uint64_t level1_alg_bytes = 0;
  /* host packing (host_pack.cpp): a few MB-sized pinned slots, narrowed into / widened out of while still cache-resident,
     so that the 16-bit copy of the image never round-trips through host DRAM */
  uint16_t* h_ring = nullptr;
  uint32_t ring_slots = 0;
  uint64_t ring_slot_elems = 0, ring_elems = 0;
  cudaEvent_t ring_ev[16]{};
  PackTuner tune_enc, tune_dec;
  std::vector<cudaEvent_t> q_ev;   /* per-step timing events of the round trips (roundtrip_begin) */
  std::vector<cudaEvent_t> p_ev;   /* per-chunk events of b2k_job_roundtrip_pipelined_n (scan done, chunk done) */
  std::vector<cudaStream_t> p_streams; /* its block-coder streams */
  bool dec_has_refinement = false; /* the block table of the current decode carries SigProp / MagRef passes */
  T2Job* t2 = nullptr;             /* b2k_encode_codestream_device: the code stream's plan for the flags of the last call */
  T2Parse* t2p = nullptr;          /* b2k_decode_codestream_device: the packet plan for the last stream's progression / SOP / EPH */
  T2Parse* t2w = nullptr;          /* b2k_decode_codestream_window_device: the box coding's plan (this job's coding is the virtual one) */
};

/* -------------------------------------------------------------------------------------------- */
extern "C" const char* b2k_last_error(void) { return g_err.c_str(); }
void b2k_set_error(const char* msg) { g_err = msg ? msg : ""; } /* for the other translation units */
extern "C" uint64_t b2k_launch_count(void) { return g_launches.load(); }

extern "C" int32_t b2k_engine_create(int32_t device, b2k_engine** out)
{
  if(!out)
    return -1;
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if(e != cudaSuccess || n == 0)
  {
    g_err = std::string("no CUDA device: ") + cudaGetErrorString(e) +
            " (this engine has no CPU path; the host keeps its own)";
    return -1;
  }
  if(device < 0 || device >= n)
  {
    g_err = "device index out of range";
    return -1;
  }
  CUDA_TRY(cudaSetDevice(device));
  b2k_engine* eng = new b2k_engine();
  eng->device = device;
  CUDA_TRY(cudaGetDeviceProperties(&eng->prop, device));
  CUDA_TRY(cudaStreamCreateWithFlags(&eng->stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&eng->copy_stream, cudaStreamNonBlocking));
  CUDA_TRY(cudaStreamCreateWithFlags(&eng->h2d_stream, cudaStreamNonBlocking));
  for(cudaStream_t& a : eng->aux)
    CUDA_TRY(cudaStreamCreateWithFlags(&a, cudaStreamNonBlocking));
  CUDA_TRY(cudaEventCreateWithFlags(&eng->caller_ev, cudaEventDisableTiming));
  *out = eng;
  return 0;
}

extern "C" void b2k_engine_destroy(b2k_engine* e)
{
  if(!e)
    return;
  cudaSetDevice(e->device);
  if(e->cached)
  {
    b2k_job_destroy(e->cached);
    e->cached = nullptr;
  }
  if(e->batch)
  {
    b2k_job_destroy(e->batch);
    e->batch = nullptr;
  }
  cudaFree(e->d_copy);
  cudaFreeHost(e->h_copy);
  cudaFree(e->d_hdr);
  cudaFreeHost(e->h_hdr);
  if(e->stream)
    cudaStreamDestroy(e->stream);
  if(e->copy_stream)
    cudaStreamDestroy(e->copy_stream);
  if(e->h2d_stream)
    cudaStreamDestroy(e->h2d_stream);
  for(cudaStream_t a : e->aux)
    if(a)
      cudaStreamDestroy(a);
  if(e->caller_ev)
    cudaEventDestroy(e->caller_ev);
  cudaFree(e->d_cs);
  cudaFree(e->d_bcs);
  delete e;
}

extern "C" void* b2k_host_alloc(size_t bytes)
{
  void* p = nullptr;
  if(cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess)
    return nullptr;
  return p;
}
extern "C" int32_t b2k_set_host_threads(int32_t n)
{
  b2k_host_set_threads(n);
  g_pack_policy.store(n < 0 ? -1 : n == 0 ? 0 : 1);
  return b2k_host_threads();
}

extern "C" int32_t b2k_host_pack_last(int32_t decode) { return g_last_pack[decode ? 1 : 0].load(); }

extern "C" void b2k_host_free(void* p)
{
  if(p)
    cudaFreeHost(p);
}

extern "C" int64_t b2k_enumerate(const b2k_coding* cp, uint32_t tile_mod, uint32_t tile_rem, b2k_block* out, uint64_t cap)
{
  if(!cp || tile_mod == 0)
    return -1;
  if(const char* why = unsupported_reason(*cp))
  {
    g_err = why;
    return -1;
  }
  const TileGrid g = tile_grid(*cp);
  const std::vector<std::vector<BandQuant>> q = component_quant(*cp);
  std::vector<b2k_block> v;
  for(uint32_t t = 0; t < g.nx * g.ny; ++t)
    if(t % tile_mod == tile_rem)
      enumerate_tile_blocks(*cp, t, tile_rect(*cp, g, t), q, v);
  for(uint64_t i = 0; i < v.size() && i < cap; ++i)
    out[i] = v[i];
  return (int64_t)v.size();
}

/* -------------------------------------------------------------------------------------------- */
/* Column strips of one warp job each.  5/3 (whole_warp): 256 columns, all 32 lanes own 8 of them and the neighbours
   outside the warp arrive as ghost columns (dwt.cu); only the last strip may be narrower.  9/7: lanes 0 and 31 are
   halo lanes, so a strip owns at most 240 columns, and the span is cut into strips of equal width. */
static void fill_strips(DwtLevelDesc& d, int pairs_per_seg, bool whole_warp)
{
  const int span = d.u1 - (d.u0 & ~7);
  const int nstrips = std::max(1, whole_warp ? (span + 255) / 256 : (span + 239) / 240);
  int sw = whole_warp ? 256 : (span + nstrips - 1) / nstrips;
  sw = (sw + 7) & ~7;
  d.nstrips = (uint16_t)nstrips;
  d.strip_w = (uint16_t)sw;
  const int npairs = ((d.v1 - 1) >> 1) - (d.v0 >> 1) + 1;
  d.pairs_per_seg = (uint16_t)pairs_per_seg;
  d.nsegs = (uint16_t)((npairs + pairs_per_seg - 1) / pairs_per_seg);
}

static int upload_descs(LevelLaunch& L)
{
  L.max_jobs = 0;
  for(const DwtLevelDesc& d : L.descs)
    L.max_jobs = std::max(L.max_jobs, (int)d.nstrips * (int)d.nsegs);
  if(L.descs.empty())
    return 0;
  CUDA_TRY(cudaMalloc(&L.d_descs, L.descs.size() * sizeof(DwtLevelDesc)));
  CUDA_TRY(cudaMemcpy(L.d_descs, L.descs.data(), L.descs.size() * sizeof(DwtLevelDesc), cudaMemcpyHostToDevice));
  return 0;
}

static int build_dwt_plan(b2k_device_job* J)
{
  const b2k_coding& cp = J->cp;
  const int L = cp.numres - 1;
  const int ncomp = cp.numcomps;
  const int pairs53 = 32, pairs97 = 32;
  const int P = cp.irreversible ? pairs97 : pairs53;
  const int32_t dc = cp.sgnd ? 0 : -(1 << (cp.prec - 1));
  const int32_t lo = cp.sgnd ? -(1 << (cp.prec - 1)) : 0, hi = cp.sgnd ? (1 << (cp.prec - 1)) - 1 : (1 << cp.prec) - 1;

  if(L == 0)
  { /* one resolution: the tile is its own LL band; what is left is DC shift + colour transform (dwt.cu k_point_transform) */
    for(int dir = 0; dir < 2; ++dir)
    {
      std::vector<LevelLaunch>& out = dir == 0 ? J->fwd : J->inv;
      LevelLaunch mctL, sglL;
      mctL.nc = 3;
      sglL.nc = 1;
      mctL.point = sglL.point = true;
      for(size_t ti = 0; ti < J->tiles.size(); ++ti)
      {
        mctL.tile_first.push_back((uint32_t)mctL.descs.size());
        sglL.tile_first.push_back((uint32_t)sglL.descs.size());
        const Rect tc = J->tile_rects[ti];
        if(tc.empty())
          continue;
        const int sc = (int)J->tile_slot[ti] * ncomp; /* the slot's first plane */
        for(int c = 0; c < ncomp;)
        {
          const bool group = cp.mct && c == 0;
          const int nc = group ? 3 : 1;
          LevelLaunch& LL = group ? mctL : sglL;
          DwtLevelDesc d{};
          d.u0 = (int32_t)tc.x0; d.v0 = (int32_t)tc.y0; d.u1 = (int32_t)tc.x1; d.v1 = (int32_t)tc.y1;
          d.first_level = 1;
          d.comp0 = (uint8_t)c;
          for(int k = 0; k < nc; ++k)
          {
            d.in[k] = J->img.at(sc + c + k, tc.x0, tc.y0);
            d.in_pitch = J->img.pitch;
            d.out_c[k] = J->coef.at(sc + c + k, tc.x0, tc.y0);
            d.out_ll[k] = d.out_c[k];
            d.c_pitch = d.ll_pitch = J->coef.pitch;
            d.shift[k] = dc;
            d.lo[k] = lo;
            d.hi[k] = hi;
          }
          LL.descs.push_back(d);
          LL.max_w = std::max(LL.max_w, tc.w());
          LL.max_h = std::max(LL.max_h, tc.h());
          LL.alg_bytes += (uint64_t)tc.w() * tc.h() * nc * 8;
          c += nc;
        }
      }
      mctL.tile_first.push_back((uint32_t)mctL.descs.size());
      sglL.tile_first.push_back((uint32_t)sglL.descs.size());
      if(!mctL.descs.empty()) out.push_back(std::move(mctL));
      if(!sglL.descs.empty()) out.push_back(std::move(sglL));
      for(LevelLaunch& Lh : out)
      {
        Lh.max_jobs = 1;
        if(upload_descs(Lh))
          return -1;
      }
    }
    return 0;
  }
  /* forward: level 1 (MCT group, then the rest), then levels 2..L component-wise */
  for(int dir = 0; dir < 2; ++dir)
  {
    std::vector<LevelLaunch>& out = dir == 0 ? J->fwd : J->inv;
    for(int lvl = 1; lvl <= L; ++lvl)
    {
      const int resno = cp.numres - lvl; /* resolution being split / rebuilt */
      LevelLaunch mctL, sglL;
      mctL.nc = 3;
      sglL.nc = 1;
      for(size_t ti = 0; ti < J->tiles.size(); ++ti)
      {
        mctL.tile_first.push_back((uint32_t)mctL.descs.size());
        sglL.tile_first.push_back((uint32_t)sglL.descs.size());
        const Rect tc = J->tile_rects[ti];
        const Rect r = resolution_rect(tc, cp.numres, resno);
        if(r.empty())
          continue;
        const int sc = (int)J->tile_slot[ti] * ncomp; /* the slot's first plane */
        for(int c = 0; c < ncomp;)
        {
          const bool group = (lvl == 1 && cp.mct && c == 0);
          const int nc = group ? 3 : 1;
          DwtLevelDesc d{};
          d.u0 = (int32_t)r.x0; d.v0 = (int32_t)r.y0; d.u1 = (int32_t)r.x1; d.v1 = (int32_t)r.y1;
          d.first_level = lvl == 1;
          d.comp0 = (uint8_t)c;
          const uint32_t llx = (r.x0 + 1) >> 1, lly = (r.y0 + 1) >> 1;
          for(int k = 0; k < nc; ++k)
          {
            const int cc = sc + c + k;
            /* finer side: image at level 1, else LL scratch written by level lvl-1 */
            const Planes& fine = (lvl == 1) ? J->img : J->ll[(lvl - 1) & 1];
            d.in[k] = fine.at(cc, r.x0, r.y0);
            d.in_pitch = fine.pitch;
            d.out_c[k] = J->coef.at(cc, tc.x0, tc.y0);
            d.c_pitch = J->coef.pitch;
            if(lvl == L)
            {
              d.out_ll[k] = d.out_c[k];
              d.ll_pitch = J->coef.pitch;
            }
            else
            {
              const Planes& coarse = J->ll[lvl & 1];
              d.out_ll[k] = coarse.at(cc, llx, lly);
              d.ll_pitch = coarse.pitch;
            }
            d.shift[k] = dc;
            d.lo[k] = lo;
            d.hi[k] = hi;
          }
          fill_strips(d, P, !cp.irreversible);
          (group ? mctL : sglL).descs.push_back(d);
          const uint64_t samples = (uint64_t)r.w() * r.h() * nc;
          (group ? mctL : sglL).alg_bytes += samples * 8;
          c += nc;
        }
      }
      mctL.tile_first.push_back((uint32_t)mctL.descs.size());
      sglL.tile_first.push_back((uint32_t)sglL.descs.size());
      /* Coarse levels have few rows: with 32 row pairs per warp-job the whole level is a handful of long serial
         chains on an almost empty GPU (level 3 of config 2: 34.7 us for 64 MB).  Cut the segments until the level
         offers about two warp-jobs per resident warp (or segments of 8 pairs, where the recomputed halo rows start
         to dominate): the work is L2-resident there, parallelism is what it lacks. */
      for(LevelLaunch* LL : {&mctL, &sglL})
      {
        int Pl = P;
        auto jobs = [&] {
          uint64_t n = 0;
          for(const DwtLevelDesc& d : LL->descs)
            n += (uint64_t)d.nstrips * d.nsegs;
          return n;
        };
        while(!LL->descs.empty() && Pl > 8 && jobs() < 3552)
        {
          Pl >>= 1;
          for(DwtLevelDesc& d : LL->descs)
            fill_strips(d, Pl, !cp.irreversible);
        }
      }
      if(dir == 0)
      {
        if(!mctL.descs.empty()) out.push_back(std::move(mctL));
        if(!sglL.descs.empty()) out.push_back(std::move(sglL));
      }
      else
      {
        if(!sglL.descs.empty()) out.insert(out.begin(), std::move(sglL));
        if(!mctL.descs.empty()) out.insert(out.begin(), std::move(mctL));
      }
    }
    for(LevelLaunch& Lh : out)
      if(upload_descs(Lh))
        return -1;
  }
  return 0;
}

static uint32_t slot_capacity(uint32_t w, uint32_t h, uint32_t kmax)
{
  /* MagSgn: <= (kmax+2) bits per sample, 8/7 stuffing; VLC: <= 15 bits per quad, 8/7; MEL 256 */
  const uint64_t samples = (uint64_t)w * h, quads = (uint64_t)((w + 1) / 2) * ((h + 1) / 2);
  const uint64_t ms = (samples * (kmax + 2) + 6) / 7 + 16;
  const uint64_t vlc = (quads * 15 + 6) / 7 + 16;
  return (uint32_t)((ms + vlc + 256 + 15) & ~15ull);
}

static int build_block_plan(b2k_device_job* J)
{
  const b2k_coding& cp = J->cp;
  J->blocks.clear();
  /* the enumeration is one slot's: every slot has the same blocks, and coded block k of slot s is descriptor
     s * coded_index.size() + k */
  for(size_t ti = 0; ti < J->slot_tiles; ++ti)
    enumerate_tile_blocks(cp, J->tiles[ti], J->tile_rects[ti], J->quant, J->blocks);
  /* map tile index -> rect */
  std::vector<Rect> rect_of(J->grid.nx * J->grid.ny);
  for(size_t ti = 0; ti < J->slot_tiles; ++ti)
    rect_of[J->tiles[ti]] = J->tile_rects[ti];
  uint64_t off = 0;
  std::vector<uint32_t> sel_of(J->grid.nx * J->grid.ny, 0);
  for(size_t ti = 0; ti < J->slot_tiles; ++ti)
    sel_of[J->tiles[ti]] = (uint32_t)ti;
  J->coded_first.assign(J->tiles.size() + 1, 0);
  for(uint32_t s = 0; s < J->slots; ++s)
  for(uint32_t i = 0; i < J->blocks.size(); ++i)
  {
    const b2k_block& b = J->blocks[i];
    if(b.x1 <= b.x0 || b.y1 <= b.y0)
      continue;
    J->coded_first[s * J->slot_tiles + sel_of[b.tile] + 1] = (uint32_t)J->h_enc_desc.size() + 1;
    const Rect& tr = rect_of[b.tile];
    const BandQuant& bq = J->quant[b.comp][band_quant_index(b.resno, b.orient)];
    HtBlockDesc d{};
    d.coef = J->coef.at((int)(s * cp.numcomps) + b.comp, tr.x0 + b.buf_x, tr.y0 + b.buf_y);
    d.pitch = J->coef.pitch;
    d.w = (uint16_t)(b.x1 - b.x0);
    d.h = (uint16_t)(b.y1 - b.y0);
    d.kmax = bq.kmax;
    d.irreversible = cp.irreversible;
    d.quant = 1.0f / bq.step_enc; /* CompressScheduler.cpp L131: inv_step_ht */
    d.slot_cap = slot_capacity(d.w, d.h, bq.kmax);
    d.slot_off = off;
    off += d.slot_cap;
    { /* per-quad records of 32 consecutive coded blocks are interleaved word by word (ht_dec.cu phase A): a group of 32
         takes 32 x its largest block's quads; entry k of block j of the group sits at group_base + 32 k + j */
      const size_t j = J->h_enc_desc.size() & 31u;
      const uint64_t quads = (uint64_t)((d.w + 1) / 2) * ((d.h + 1) / 2);
      if(j == 0)
      {
        J->total_quads += 32 * J->group_quads; /* close the previous group */
        J->group_quads = 0;
      }
      J->group_quads = std::max(J->group_quads, quads);
      d.rec_off = (uint32_t)(J->total_quads + j);
    }
    J->max_cblk_w = std::max<uint32_t>(J->max_cblk_w, d.w);
    J->enc_limits.stage_words = std::max(J->enc_limits.stage_words, b2k_ht_encode_stage_words(d.w));
    J->enc_limits.max_kmax = std::max<uint32_t>(J->enc_limits.max_kmax, d.kmax);
    J->h_enc_desc.push_back(d);
    J->dec_quant.push_back(bq.step_dec / (float)(1u << (31 - bq.kmax)));
    if(s == 0)
      J->coded_index.push_back(i);
  }
  J->scratch_bytes = off;
  /* descriptor indices, coded_first and the per-quad record offsets (rec_off) are 32-bit: a batch job of too many slots
     is refused rather than left to wrap */
  if(J->h_enc_desc.size() >= UINT32_MAX || J->total_quads + 32 * J->group_quads + 64 > UINT32_MAX)
  {
    g_err = "too many code blocks for one job (" + std::to_string(J->h_enc_desc.size()) + " blocks, " +
            std::to_string(J->total_quads + 32 * J->group_quads) + " quad records; at most 2^32 - 1 of each)";
    return -1;
  }
  for(size_t ti = 1; ti <= J->tiles.size(); ++ti) /* tiles without coded blocks inherit the running count */
    J->coded_first[ti] = std::max(J->coded_first[ti], J->coded_first[ti - 1]);
  {
    const uint32_t nt = (uint32_t)J->tiles.size();
    uint32_t want = 8;
    if(const char* ev = getenv("B2K_CHUNKS"))
      want = (uint32_t)std::max(1, std::min(B2K_MAX_CHUNKS, atoi(ev)));
    const uint32_t nchunks = std::max(1u, std::min(want, nt));
    J->chunk_tile.clear();
    for(uint32_t k = 0; k <= nchunks; ++k)
      J->chunk_tile.push_back((uint32_t)((uint64_t)k * nt / nchunks));
  }
  const size_t n = J->h_enc_desc.size();
  if(n)
  {
    CUDA_TRY(cudaMalloc(&J->d_enc_desc, n * sizeof(HtBlockDesc)));
    CUDA_TRY(cudaMemcpy(J->d_enc_desc, J->h_enc_desc.data(), n * sizeof(HtBlockDesc), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaMalloc(&J->d_dec_desc, n * sizeof(HtBlockDesc)));
    CUDA_TRY(cudaMalloc(&J->d_out, n * sizeof(HtBlockOut)));
    CUDA_TRY(cudaMalloc(&J->d_offsets, (n + 1) * sizeof(uint64_t)));
    CUDA_TRY(cudaMemset(J->d_offsets, 0, (n + 1) * sizeof(uint64_t))); /* offsets[0] stays 0: the scan's base */
    CUDA_TRY(cudaMalloc(&J->d_scratch, J->scratch_bytes + 64));
    CUDA_TRY(cudaMalloc(&J->d_recs, (J->total_quads + 32 * J->group_quads + 64) * sizeof(uint32_t)));
    CUDA_TRY(cudaMalloc(&J->d_dec_status, n * sizeof(HtBlockOut)));
    CUDA_TRY(cudaMalloc(&J->d_dec_quant, n * sizeof(float)));
    CUDA_TRY(cudaMemcpy(J->d_dec_quant, J->dec_quant.data(), n * sizeof(float), cudaMemcpyHostToDevice));
    CUDA_TRY(cudaHostAlloc(&J->h_out, n * sizeof(HtBlockOut), cudaHostAllocDefault));
    CUDA_TRY(cudaHostAlloc(&J->h_dec_desc, n * sizeof(HtBlockDesc), cudaHostAllocDefault));
    CUDA_TRY(cudaHostAlloc(&J->h_offsets, (n + 1) * sizeof(uint64_t), cudaHostAllocDefault));
  }
  CUDA_TRY(cudaMalloc(&J->d_err, J->slots * sizeof(int)));
  CUDA_TRY(cudaMemset(J->d_err, 0, J->slots * sizeof(int)));
  return 0;
}

static int job_create(b2k_engine* e, const b2k_coding* cp, uint32_t tile_mod, uint32_t tile_rem, uint32_t slots, b2k_device_job** out);

extern "C" int32_t b2k_job_create(b2k_engine* e, const b2k_coding* cp, uint32_t tile_mod, uint32_t tile_rem,
                                  b2k_device_job** out)
{
  return job_create(e, cp, tile_mod, tile_rem, 1, out);
}

/* b2k_job_create with `slots` images of the coding (a batch job) */
static int job_create(b2k_engine* e, const b2k_coding* cp, uint32_t tile_mod, uint32_t tile_rem, uint32_t slots, b2k_device_job** out)
{
  if(!e || !cp || !out || tile_mod == 0 || slots == 0)
    return -1;
  *out = nullptr;
  if(const char* why = unsupported_reason(*cp))
  {
    g_err = why;
    return 1; /* not handled: the host keeps its CPU path (plugin_accelerate.h L32-36) */
  }
  CUDA_TRY(cudaSetDevice(e->device));
  b2k_device_job* J = new b2k_device_job();
  J->eng = e;
  J->cp = *cp;
  J->tile_mod = tile_mod;
  J->tile_rem = tile_rem;
  J->grid = tile_grid(*cp);
  J->quant = component_quant(*cp);
  J->slots = slots;
  for(uint32_t s = 0; s < slots; ++s)
    for(uint32_t t = 0; t < J->grid.nx * J->grid.ny; ++t)
      if(t % tile_mod == tile_rem)
      {
        const Rect r = tile_rect(*cp, J->grid, t);
        if(r.empty())
          continue;
        J->tiles.push_back(t);
        J->tile_rects.push_back(r);
        J->tile_slot.push_back(s);
      }
  J->slot_tiles = (uint32_t)(J->tiles.size() / slots);
  const int nc = cp->numcomps * (int)slots;
  if(alloc_planes(J->img, nc, cp->x0, cp->y0, cp->x1, cp->y1) || alloc_planes(J->coef, nc, cp->x0, cp->y0, cp->x1, cp->y1))
  {
    b2k_job_destroy(J);
    return -1;
  }
  /* LL scratch, canvas origin (0,0): ll[1] receives the LL of odd levels (1/2, 1/8, ... resolution),
     ll[0] of even levels (1/4, 1/16, ...); a level reads one and writes the other */
  if(alloc_planes(J->ll[1], nc, 0, 0, ((cp->x1 + 1) >> 1) + 1, ((cp->y1 + 1) >> 1) + 1) ||
     alloc_planes(J->ll[0], nc, 0, 0, ((cp->x1 + 3) >> 2) + 1, ((cp->y1 + 3) >> 2) + 1))
  {
    b2k_job_destroy(J);
    return -1;
  }
  if(build_dwt_plan(J) || build_block_plan(J))
  {
    b2k_job_destroy(J);
    return -1;
  }
  for(cudaEvent_t& ev : J->ev)
    CUDA_TRY(cudaEventCreate(&ev));
  for(cudaEvent_t& ev : J->chunk_ev)
    CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  *out = J;
  return 0;
}

/* one of J's parse plans goes: b2k_codestream_parse_device_stats no longer reports it */
static void drop_parse(b2k_device_job* J, T2Parse*& p)
{
  if(J->eng->last_parse == p)
    J->eng->last_parse = nullptr;
  b2k_t2_parse_destroy(p);
  p = nullptr;
}

extern "C" void b2k_job_destroy(b2k_device_job* J)
{
  if(!J)
    return;
  cudaSetDevice(J->eng->device);
  cudaStreamSynchronize(J->eng->stream);
  b2k_t2_destroy(J->t2);
  drop_parse(J, J->t2p);
  drop_parse(J, J->t2w);
  cudaFree(J->img.base);
  cudaFree(J->d_stage);
  cudaFree(J->coef.base);
  cudaFree(J->ll[0].base);
  cudaFree(J->ll[1].base);
  for(LevelLaunch& L : J->fwd) cudaFree(L.d_descs);
  for(LevelLaunch& L : J->inv) cudaFree(L.d_descs);
  cudaFree(J->d_enc_desc);
  cudaFree(J->d_dec_desc);
  cudaFree(J->d_out);
  cudaFree(J->d_offsets);
  cudaFree(J->d_scratch);
  cudaFree(J->d_recs);
  cudaFree(J->d_dec_quant);
  cudaFree(J->d_dec_status);
  cudaFree(J->d_bytes);
  cudaFree(J->d_err);
  cudaFree(J->d_batch_dst);
  cudaFreeHost(J->h_batch_dst);
  cudaFree(J->d_batch_src);
  cudaFreeHost(J->h_batch_src);
  cudaFreeHost(J->h_out);
  cudaFreeHost(J->h_dec_desc);
  cudaFreeHost(J->h_offsets);
  cudaFreeHost(J->h_ring);
  for(cudaEvent_t ev : J->q_ev)
    cudaEventDestroy(ev);
  for(cudaEvent_t ev : J->p_ev)
    cudaEventDestroy(ev);
  for(cudaStream_t ps : J->p_streams)
    cudaStreamDestroy(ps);
  for(cudaEvent_t& ev : J->ring_ev)
    if(ev)
      cudaEventDestroy(ev);
  for(cudaEvent_t& ev : J->ev)
    if(ev)
      cudaEventDestroy(ev);
  for(cudaEvent_t& ev : J->chunk_ev)
    if(ev)
      cudaEventDestroy(ev);
  delete J;
}

extern "C" uint64_t b2k_job_num_blocks(const b2k_device_job* J) { return J ? J->blocks.size() : 0; }

/* ---- sample transport: the caller's containers <-> the engine's int32 planes ---------------------------------------
   Every container samples cross is described as a b2k_device_planes: component c of canvas pixel (x, y) is at
   comp[c] + ((y - oy) * row_pitch[c] + (x - ox) * col_step[c]) * sample_bytes, (ox, oy) being the canvas position of its
   first sample (the image's, the window's, or the staging's own origin). */
struct Container
{
  b2k_device_planes d{};
  uint32_t ox = 0, oy = 0;
  bool device = false;      /* device memory (the engine's buffers, the caller's device image), else host memory */
  bool interleaved = false; /* pixel-interleaved: comp[c] = comp[0] + c samples, col_step = numcomps */
  uint8_t* at(int c, uint32_t x, uint32_t y) const
  {
    return static_cast<uint8_t*>(d.comp[c]) +
           ((size_t)(y - oy) * d.row_pitch[c] + (size_t)(x - ox) * d.col_step[c]) * d.sample_bytes;
  }
};

/* planar: the caller's host planes, or the engine's int32 planes */
static Container planar_container(int nc, void* const* comp, const uint32_t* pitch, uint32_t sample_bytes, uint32_t ox, uint32_t oy,
                                  bool device)
{
  Container C;
  for(int c = 0; c < nc && c < 4; ++c)
  {
    C.d.comp[c] = comp[c];
    C.d.row_pitch[c] = pitch[c];
    C.d.col_step[c] = 1;
  }
  C.d.sample_bytes = sample_bytes;
  C.ox = ox;
  C.oy = oy;
  C.device = device;
  return C;
}
static Container interleaved_container(int nc, void* base, uint32_t pitch, uint32_t sample_bytes, uint32_t ox, uint32_t oy, bool device)
{
  Container C;
  for(int c = 0; c < nc && c < 4; ++c)
  {
    C.d.comp[c] = static_cast<uint8_t*>(base) + (size_t)c * sample_bytes;
    C.d.row_pitch[c] = pitch;
    C.d.col_step[c] = (uint32_t)nc;
  }
  C.d.sample_bytes = sample_bytes;
  C.ox = ox;
  C.oy = oy;
  C.device = device;
  C.interleaved = true;
  return C;
}
static Container plane_container(const Planes& P)
{
  void* comp[4];
  uint32_t pitch[4];
  for(int c = 0; c < P.n && c < 4; ++c)
  {
    comp[c] = P.at(c, P.X0, P.Y0);
    pitch[c] = P.pitch;
  }
  return planar_container(P.n, comp, pitch, 4, P.X0, P.Y0, true);
}

/* The 16-bit containers that cross PCIe land in (and leave from) one device buffer, J->d_stage, in one of two layouts:
   planar, canvas column x0 & ~63 at column 0, rows of the image's width rounded up to 8 samples (a full-width tile row is one
   contiguous block) and two rows of slack; or pixel-interleaved, the image's rows as they are, rounded up to 8 samples. */
static uint32_t stage_pitch(const b2k_coding& cp, bool interleaved)
{
  return interleaved ? ((cp.x1 - cp.x0) * cp.numcomps + 7u) & ~7u : ((cp.x1 - (cp.x0 & ~63u)) + 7u) & ~7u;
}
static size_t stage_plane_elems(const b2k_coding& cp) { return (size_t)stage_pitch(cp, false) * (cp.y1 - cp.y0 + 2); }
static Container stage_container(const b2k_device_job* J, bool interleaved)
{
  const b2k_coding& cp = J->cp;
  const uint32_t pitch = stage_pitch(cp, interleaved);
  if(interleaved)
    return interleaved_container(cp.numcomps, J->d_stage, pitch, 2, cp.x0, cp.y0, true);
  void* comp[4];
  const uint32_t pitches[4] = {pitch, pitch, pitch, pitch};
  for(int c = 0; c < cp.numcomps; ++c)
    comp[c] = J->d_stage + c * stage_plane_elems(cp);
  return planar_container(cp.numcomps, comp, pitches, 2, cp.x0 & ~63u, cp.y0, true);
}
static int ensure_stage(b2k_device_job* J)
{
  if(J->d_stage)
    return 0;
  const b2k_coding& cp = J->cp;
  const size_t bytes = std::max(cp.numcomps * stage_plane_elems(cp), (size_t)stage_pitch(cp, true) * (cp.y1 - cp.y0)) * sizeof(uint16_t);
  CUDA_TRY(cudaMalloc(&J->d_stage, bytes));
  CUDA_TRY(cudaMemset(J->d_stage, 0, bytes));
  /* cudaMemset runs on the legacy default stream, which the engine's non-blocking streams do not wait for: without this
     wait the zeroing could land after the first chunk of the call that allocated the staging had been copied into it */
  CUDA_TRY(cudaStreamSynchronize(0));
  return 0;
}

/* fn(r) for every run of horizontally adjacent selected tiles of [t0, t1) in one tile row, merged into one rectangle; with a
   window, r is clipped to it and runs outside it are skipped */
template <typename F>
static void for_tile_row_runs(const b2k_device_job* J, size_t t0, size_t t1, const Rect* window, F&& fn)
{
  t1 = std::min(t1, J->tiles.size());
  for(size_t ti = t0; ti < t1;)
  {
    Rect r = J->tile_rects[ti];
    size_t tj = ti + 1;
    while(tj < t1 && J->tile_rects[tj].y0 == r.y0 && J->tile_rects[tj].y1 == r.y1 && J->tile_rects[tj].x0 == r.x1)
    {
      r.x1 = J->tile_rects[tj].x1;
      ++tj;
    }
    ti = tj;
    if(window)
    {
      r.x0 = std::max(r.x0, window->x0); r.y0 = std::max(r.y0, window->y0);
      r.x1 = std::min(r.x1, window->x1); r.y1 = std::min(r.y1, window->y1);
      if(r.empty())
        continue;
    }
    fn(r);
  }
}

/* `rows` rows of `row` bytes: one linear copy where they abut on both sides, else one 2-D copy */
static cudaError_t copy_rows(void* dst, size_t dpitch, const void* src, size_t spitch, size_t row, uint32_t rows, cudaMemcpyKind kind,
                             cudaStream_t st)
{
  if(dpitch == row && spitch == row)
    return cudaMemcpyAsync(dst, src, row * rows, kind, st);
  return cudaMemcpy2DAsync(dst, dpitch, src, spitch, row, rows, kind, st);
}

/* the selected tiles [t0, t1), clipped to `window`, from one container to another of the same sample size and layout: host to
   device, device to host or device to device, per run one copy per component, or one for all of them when pixel-interleaved */
static int copy_runs(const b2k_device_job* J, const Container& dst, const Container& src, cudaStream_t st, size_t t0, size_t t1,
                     const Rect* window)
{
  const int nc = J->cp.numcomps, group = src.interleaved ? nc : 1;
  const size_t sb = src.d.sample_bytes;
  const cudaMemcpyKind kind = !src.device ? cudaMemcpyHostToDevice : dst.device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
  cudaError_t err = cudaSuccess;
  for_tile_row_runs(J, t0, t1, window, [&](const Rect& r) {
    for(int c = 0; c < nc; c += group)
    {
      const cudaError_t e = copy_rows(dst.at(c, r.x0, r.y0), dst.d.row_pitch[c] * sb, src.at(c, r.x0, r.y0), src.d.row_pitch[c] * sb,
                                      (size_t)r.w() * group * sb, r.h(), kind, st);
      if(e != cudaSuccess)
        err = e;
    }
  });
  CUDA_TRY(err);
  return 0;
}

extern "C" int32_t b2k_job_upload(b2k_device_job* J, const int32_t* const* planes, const uint32_t* strides)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  const Container host = planar_container(J->cp.numcomps, (void* const*)planes, strides, 4, J->cp.x0, J->cp.y0, false);
  J->arena_sized = false;
  if(copy_runs(J, plane_container(J->img), host, J->eng->stream, 0, J->tiles.size(), nullptr)) return -1;
  CUDA_TRY(cudaStreamSynchronize(J->eng->stream));
  return 0;
}
extern "C" int32_t b2k_job_download(b2k_device_job* J, int32_t* const* planes, const uint32_t* strides)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  const Container host = planar_container(J->cp.numcomps, (void* const*)planes, strides, 4, J->cp.x0, J->cp.y0, false);
  if(copy_runs(J, host, plane_container(J->img), J->eng->stream, 0, J->tiles.size(), nullptr)) return -1;
  CUDA_TRY(cudaStreamSynchronize(J->eng->stream));
  return 0;
}
extern "C" int32_t b2k_job_download_coeffs(b2k_device_job* J, int32_t* const* planes, const uint32_t* strides)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  const Container host = planar_container(J->cp.numcomps, (void* const*)planes, strides, 4, J->cp.x0, J->cp.y0, false);
  if(copy_runs(J, host, plane_container(J->coef), J->eng->stream, 0, J->tiles.size(), nullptr)) return -1;
  CUDA_TRY(cudaStreamSynchronize(J->eng->stream));
  return 0;
}
extern "C" int32_t b2k_job_upload_coeffs(b2k_device_job* J, const int32_t* const* planes, const uint32_t* strides)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  const Container host = planar_container(J->cp.numcomps, (void* const*)planes, strides, 4, J->cp.x0, J->cp.y0, false);
  if(copy_runs(J, plane_container(J->coef), host, J->eng->stream, 0, J->tiles.size(), nullptr)) return -1;
  CUDA_TRY(cudaStreamSynchronize(J->eng->stream));
  return 0;
}

/* ---- images the caller keeps in device memory (b2k_encode_device / b2k_decode_device) ------------------------------ */
/* 0 usable, 1 not handled, -1 bad input; b2k_last_error says why */
static int check_device_planes(const b2k_engine* e, const b2k_coding* cp, const b2k_device_planes* img)
{
  if(!img)
  {
    g_err = "no device image";
    return -1;
  }
  if(img->sample_bytes != 1 && img->sample_bytes != 2 && img->sample_bytes != 4)
  {
    g_err = "sample_bytes must be 1, 2 or 4";
    return -1;
  }
  if(cp->numcomps > 4)
  {
    g_err = "a device image holds at most 4 components";
    return 1;
  }
  if(img->sample_bytes * 8 < cp->prec)
  {
    g_err = std::to_string(img->sample_bytes * 8) + "-bit containers cannot hold " + std::to_string(cp->prec) + "-bit samples";
    return 1;
  }
  for(int c = 0; c < cp->numcomps; ++c)
  {
    const std::string comp = "device image component " + std::to_string(c) + ": ";
    cudaPointerAttributes a{};
    const cudaError_t err = img->comp[c] ? cudaPointerGetAttributes(&a, img->comp[c]) : cudaErrorInvalidValue;
    if(err != cudaSuccess)
      (void)cudaGetLastError();
    if(err != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != e->device)
    {
      g_err = comp + "not device or managed memory of the engine's device (" + std::to_string(e->device) + ")";
      return -1;
    }
    if(reinterpret_cast<uintptr_t>(img->comp[c]) % img->sample_bytes)
    {
      g_err = comp + "address not a multiple of sample_bytes";
      return -1;
    }
    if(!img->col_step[c])
    {
      g_err = comp + "col_step is 0";
      return -1;
    }
  }
  return 0;
}

/* components one conversion launch covers: all of them when they are pixel-interleaved (comp[c] = comp[0] + c samples, one
   pitch and one step), else one */
static int device_group(const b2k_device_planes& img, int nc)
{
  const uint8_t* base = static_cast<const uint8_t*>(img.comp[0]);
  for(int c = 1; c < nc; ++c)
    if(static_cast<const uint8_t*>(img.comp[c]) != base + (size_t)c * img.sample_bytes || img.row_pitch[c] != img.row_pitch[0] ||
       img.col_step[c] != img.col_step[0])
      return 1;
  return nc;
}

/* a device container -> the engine's planes (to_planes) or back, selected tiles [t0, t1) clipped to `window`, on stream st:
   conversion launches, or device-to-device copies for int32 planes */
static int device_convert(b2k_device_job* J, const Container& img, bool to_planes, cudaStream_t st, size_t t0, size_t t1,
                          const Rect* window)
{
  const b2k_coding& cp = J->cp;
  const int nc = cp.numcomps;
  bool planar32 = img.d.sample_bytes == 4;
  for(int c = 0; c < nc; ++c)
    planar32 = planar32 && img.d.col_step[c] == 1;
  if(planar32) /* int32 planes: nothing to convert */
  {
    const Container planes = plane_container(J->img);
    return to_planes ? copy_runs(J, planes, img, st, t0, t1, window) : copy_runs(J, img, planes, st, t0, t1, window);
  }
  const int group = device_group(img.d, nc);
  for_tile_row_runs(J, t0, t1, window, [&](const Rect& r) {
    for(int c = 0; c < nc; c += group)
    {
      int32_t* planes[4];
      for(int k = 0; k < group; ++k)
        planes[k] = J->img.at(c + k, r.x0, r.y0);
      if(to_planes)
        b2k_launch_container_to_planes(img.at(c, r.x0, r.y0), img.d.row_pitch[c], img.d.col_step[c], img.d.sample_bytes, planes, group,
                                       J->img.pitch, r.w(), r.h(), cp.sgnd, st);
      else
        b2k_launch_planes_to_container(planes, group, J->img.pitch, img.at(c, r.x0, r.y0), img.d.row_pitch[c], img.d.col_step[c],
                                       img.d.sample_bytes, r.w(), r.h(), st);
    }
  });
  CUDA_TRY(cudaGetLastError());
  return 0;
}

/* int32 entry points with samples of <= 16 bits: the PCIe legs carry 16-bit containers, converted
   chunk by chunk on host threads (host_pack.cpp) while the neighbouring chunk is on the bus */
static bool host_pack_eligible(const b2k_device_job* J)
{
  const b2k_coding& cp = J->cp;
  const uint64_t samples = (uint64_t)(cp.x1 - cp.x0) * (cp.y1 - cp.y0) * cp.numcomps;
  return cp.prec <= 16 && samples >= (1u << 22) && J->chunk_tile.size() > 2 && b2k_host_threads() > 0;
}

/* ---- ring staging ---------------------------------------------------------------------------- */
struct StagePiece
{
  uint32_t chunk, comp, x0, y0, w, rows; /* canvas coordinates */
};
struct RingGeom
{
  uint32_t slot_mb, slots;
};
/* B2K_RING_ENC / B2K_RING_DEC = "<slot MB>,<slots>": slots of at least 1 MB, 2 to 16 of them */
static RingGeom ring_geom(bool decode)
{
  auto parse = [](const char* name, RingGeom r) {
    if(const char* e = getenv(name))
    {
      r.slot_mb = (uint32_t)std::max(1, atoi(e));
      if(const char* c = strchr(e, ','))
        r.slots = (uint32_t)std::max(2, std::min(16, atoi(c + 1)));
    }
    return r;
  };
  static const RingGeom g[2] = {parse("B2K_RING_ENC", {8, 4}), parse("B2K_RING_DEC", {16, 4})};
  return g[decode ? 1 : 0];
}
static int ensure_ring(b2k_device_job* J, bool decode)
{
  const RingGeom g = ring_geom(decode);
  const uint64_t min_elems = (uint64_t)(J->cp.x1 - J->cp.x0) * 4;
  const uint64_t slot_elems = std::max<uint64_t>((uint64_t)g.slot_mb * (1u << 20) / sizeof(uint16_t), min_elems);
  const uint64_t need = slot_elems * g.slots;
  if(need > J->ring_elems)
  {
    if(J->h_ring)
      cudaFreeHost(J->h_ring);
    J->h_ring = nullptr;
    CUDA_TRY(cudaHostAlloc(&J->h_ring, need * sizeof(uint16_t), cudaHostAllocDefault));
    J->ring_elems = need;
  }
  for(uint32_t i = 0; i < g.slots; ++i)
    if(!J->ring_ev[i])
      CUDA_TRY(cudaEventCreateWithFlags(&J->ring_ev[i], cudaEventDisableTiming));
  J->ring_slots = g.slots;
  J->ring_slot_elems = slot_elems;
  return 0;
}
static void chunk_pieces(const b2k_device_job* J, uint32_t chunk, std::vector<StagePiece>& out)
{
  for_tile_row_runs(J, J->chunk_tile[chunk], J->chunk_tile[chunk + 1], nullptr, [&](const Rect& r) {
    const uint32_t rows_per = (uint32_t)std::max<uint64_t>(1, J->ring_slot_elems / r.w());
    for(uint32_t y = r.y0; y < r.y1; y += rows_per)
      for(uint32_t c = 0; c < J->cp.numcomps; ++c)
        out.push_back({chunk, c, r.x0, y, r.w(), std::min(rows_per, r.y1 - y)});
  });
}
/* narrow one chunk of the caller's int32 planes piece by piece into the ring and send each piece on its way to the staging */
static int ring_upload_chunk(b2k_device_job* J, const Container& user, const Container& stage, uint32_t chunk, cudaStream_t cs,
                             uint64_t& counter, const std::function<int()>& between_pieces)
{
  std::vector<StagePiece> pcs;
  chunk_pieces(J, chunk, pcs);
  for(const StagePiece& pc : pcs)
  {
    const uint32_t slot = (uint32_t)(counter % J->ring_slots);
    if(counter >= J->ring_slots)
      CUDA_TRY(cudaEventSynchronize(J->ring_ev[slot])); /* the slot's previous piece has left */
    uint16_t* sp = J->h_ring + (uint64_t)slot * J->ring_slot_elems;
    const b2k_host_rect hr{user.at(pc.comp, pc.x0, pc.y0), sp, user.d.row_pitch[pc.comp], pc.w, pc.w, pc.rows};
    b2k_host_convert(&hr, 1, false, J->cp.sgnd != 0, true);
    CUDA_TRY(copy_rows(stage.at(pc.comp, pc.x0, pc.y0), (size_t)stage.d.row_pitch[pc.comp] * 2, sp, (size_t)pc.w * 2,
                       (size_t)pc.w * 2, pc.rows, cudaMemcpyHostToDevice, cs));
    CUDA_TRY(cudaEventRecord(J->ring_ev[slot], cs));
    ++counter;
    if(between_pieces())
      return -1;
  }
  return 0;
}
/* bring every chunk's pixels down from the staging through the ring and widen them into the caller's int32 planes; chunk
   k's pixels are ready on the device when chunk_ev[CEV(0, k)] fires */
static int ring_download_all(b2k_device_job* J, const Container& user, const Container& stage, cudaStream_t cs)
{
  std::vector<StagePiece> pcs;
  for(uint32_t k = 0; k + 1 < J->chunk_tile.size(); ++k)
    chunk_pieces(J, k, pcs);
  const size_t N = pcs.size(), S = J->ring_slots;
  auto issue = [&](size_t p) -> int {
    const StagePiece& pc = pcs[p];
    const uint32_t slot = (uint32_t)(p % S);
    uint16_t* sp = J->h_ring + (uint64_t)slot * J->ring_slot_elems;
    if(p == 0 || pcs[p - 1].chunk != pc.chunk)
      CUDA_TRY(cudaStreamWaitEvent(cs, J->chunk_ev[CEV(0, pc.chunk)], 0));
    CUDA_TRY(copy_rows(sp, (size_t)pc.w * 2, stage.at(pc.comp, pc.x0, pc.y0), (size_t)stage.d.row_pitch[pc.comp] * 2,
                       (size_t)pc.w * 2, pc.rows, cudaMemcpyDeviceToHost, cs));
    CUDA_TRY(cudaEventRecord(J->ring_ev[slot], cs));
    return 0;
  };
  for(size_t p = 0; p < std::min(S, N); ++p)
    if(issue(p)) return -1;
  for(size_t p = 0; p < N; ++p)
  {
    const StagePiece& pc = pcs[p];
    const uint32_t slot = (uint32_t)(p % S);
    CUDA_TRY(cudaEventSynchronize(J->ring_ev[slot]));
    const uint16_t* sp = J->h_ring + (uint64_t)slot * J->ring_slot_elems;
    const b2k_host_rect hr{sp, user.at(pc.comp, pc.x0, pc.y0), pc.w, user.d.row_pitch[pc.comp], pc.w, pc.rows};
    b2k_host_convert(&hr, 1, true, J->cp.sgnd != 0);
    if(p + S < N)
      if(issue(p + S)) return -1;
  }
  return 0;
}

/* ---- one call's transport -------------------------------------------------------------------------------------- */
/* How the samples of one b2k_encode* / b2k_decode* call travel between the caller and the engine's planes; settled before the
   chunk pipeline starts (resolve_transport), so that the pipeline only asks for chunk k to be brought in or sent out */
struct Transport
{
  Container user;               /* the caller's samples: host planes or pixels, or a device image */
  const Rect* window = nullptr; /* b2k_decode_window / b2k_decode_device: only these pixels go back, and `user` holds them */
  Container stage;              /* the 16-bit staging, when `staged` */
  bool staged = false;          /* host copies go to / come from the staging, converted to / from the planes on the device */
  bool ring = false;            /* int32 host planes packed on host threads, through the pinned ring into the staging */
  uint64_t ring_pieces = 0;     /* pieces sent through the ring so far */
  PackTuner* tuner = nullptr;   /* the tuner chose whether to pack; it hears how long the call took */
  Transport() = default;
  Transport(const Transport&) = delete;
  ~Transport()
  {
    if(ring)
      b2k_host_session(false);
  }
};

/* T.user (and T.window) given: whether the call packs on host threads, by policy or tuner, and whether it goes through the
   staging, which 16-bit host samples and packed ones do */
static int resolve_transport(b2k_device_job* J, Transport& T, bool decode)
{
  if(T.user.device)
    return 0;
  if(T.user.d.sample_bytes == 4)
  { /* several ranks on one host share its DRAM and CPU quota: measured (DESIGN.md section 4) packing loses there,
       so the automatic policy only considers it for a process that has the host to itself */
    const bool eligible = !T.window && host_pack_eligible(J);
    const bool tuned = eligible && g_pack_policy.load() < 0 && b2k_host_local_peers() == 1;
    PackTuner& tuner = decode ? J->tune_dec : J->tune_enc;
    const bool pack = eligible && (tuned ? tuner.next_mode() : g_pack_policy.load() > 0);
    g_last_pack[decode ? 1 : 0].store(pack ? 1 : 0);
    T.tuner = tuned ? &tuner : nullptr;
    if(!pack)
      return 0;
    if(ensure_ring(J, decode))
      return -1;
    T.ring = true;
    b2k_host_session(true);
  }
  if(ensure_stage(J))
    return -1;
  T.stage = stage_container(J, T.user.interleaved);
  T.staged = true;
  return 0;
}

/* chunk k of the caller's host samples onto the device on the copy stream cs, and the compute stream st waits for it: packed
   through the ring, or copied as they are into the staging or the planes.  between_pieces: host work slotted in between ring
   pieces */
static int upload_chunk(b2k_device_job* J, Transport& T, size_t k, cudaStream_t st, cudaStream_t cs,
                        const std::function<int()>& between_pieces)
{
  if(T.ring ? ring_upload_chunk(J, T.user, T.stage, (uint32_t)k, cs, T.ring_pieces, between_pieces)
            : copy_runs(J, T.staged ? T.stage : plane_container(J->img), T.user, cs, J->chunk_tile[k], J->chunk_tile[k + 1], nullptr))
    return -1;
  CUDA_TRY(cudaEventRecord(J->chunk_ev[CEV(0, k)], cs));
  CUDA_TRY(cudaStreamWaitEvent(st, J->chunk_ev[CEV(0, k)], 0));
  return 0;
}

/* chunk k's pixels out of the planes, once the compute stream st has them: into a device image by conversion on st; to the
   host narrowed into the staging on st (when staged), then copied on the copy stream cs, or through the ring once every chunk
   is queued (ring_download_all) */
static int download_chunk(b2k_device_job* J, const Transport& T, size_t k, cudaStream_t st, cudaStream_t cs)
{
  const size_t t0 = J->chunk_tile[k], t1 = J->chunk_tile[k + 1];
  if(T.user.device)
    return device_convert(J, T.user, false, st, t0, t1, T.window);
  if(T.staged && device_convert(J, T.stage, false, st, t0, t1, T.window))
    return -1;
  CUDA_TRY(cudaEventRecord(J->chunk_ev[CEV(0, k)], st));
  if(T.ring)
    return 0;
  CUDA_TRY(cudaStreamWaitEvent(cs, J->chunk_ev[CEV(0, k)], 0));
  return copy_runs(J, T.user, T.staged ? T.stage : plane_container(J->img), cs, t0, t1, T.window);
}

/* ---- bookkeeping every entry point shares ------------------------------------------------------- */
/* The coded-byte arena holds `bytes` and the 64 the HT decoder reads past a block's end, or is replaced by one of bytes +
   headroom + 4096.  Nothing queued still uses the old arena when it is freed.  A failed allocation leaves the job without
   an arena (d_bytes NULL, bytes_cap 0): the next call allocates again, and b2k_job_destroy has nothing to free twice. */
static int arena_reserve(b2k_device_job* J, uint64_t bytes, uint64_t headroom)
{
  if(bytes + 64 <= J->bytes_cap)
    return 0;
  CUDA_TRY(cudaStreamSynchronize(J->eng->stream));
  cudaFree(J->d_bytes);
  J->d_bytes = nullptr;
  J->bytes_cap = 0;
  const uint64_t cap = bytes + headroom + 4096;
  CUDA_TRY(cudaMalloc(&J->d_bytes, cap));
  J->bytes_cap = cap;
  return 0;
}

/* what the HT decoder said of the blocks decoded since d_err was cleared: 0, or -2 and how many it rejected */
static int decoder_verdict(b2k_device_job* J)
{
  int herr = 0;
  CUDA_TRY(cudaMemcpy(&herr, J->d_err, sizeof(int), cudaMemcpyDeviceToHost));
  if(herr)
  {
    g_err = "HT decoder rejected " + std::to_string(herr) + " block(s)";
    return -2;
  }
  return 0;
}

/* what is queued on `next` from here on runs after what is queued on `first` now: the engine's stream after the caller's on
   the way in, the caller's after the engine's on the way out */
static int queue_after(b2k_engine* e, cudaStream_t first, cudaStream_t next)
{
  CUDA_TRY(cudaEventRecord(e->caller_ev, first));
  CUDA_TRY(cudaStreamWaitEvent(next, e->caller_ev, 0));
  return 0;
}

/* a stage hook's frame: enqueue(stream) between ev[0] and ev[1] on the engine's stream, one synchronisation, the time
   between the two */
template <class Enqueue>
static int timed_stage(b2k_device_job* J, float* ms, Enqueue enqueue)
{
  cudaStream_t st = J->eng->stream;
  CUDA_TRY(cudaEventRecord(J->ev[0], st));
  if(enqueue(st)) return -1;
  CUDA_TRY(cudaEventRecord(J->ev[1], st));
  CUDA_TRY(cudaEventSynchronize(J->ev[1]));
  float t = 0;
  CUDA_TRY(cudaEventElapsedTime(&t, J->ev[0], J->ev[1]));
  if(ms) *ms = t;
  return 0;
}

/* ---- stages ----------------------------------------------------------------------------------- */
static int enqueue_forward(b2k_device_job* J, cudaStream_t st, bool time_level1, size_t t0 = 0, size_t t1 = (size_t)-1,
                           cudaEvent_t l1_begin = nullptr, cudaEvent_t l1_end = nullptr)
{
  if(!l1_begin) l1_begin = J->ev[4];
  if(!l1_end) l1_end = J->ev[5];
  t1 = std::min(t1, J->tiles.size());
  bool first = true;
  for(size_t li = 0; li < J->fwd.size(); ++li)
  {
    LevelLaunch& L = J->fwd[li];
    const uint32_t d0 = L.tile_first[t0], d1 = L.tile_first[t1];
    if(first && time_level1)
      CUDA_TRY(cudaEventRecord(l1_begin, st));
    if(d1 > d0 && L.point)
      b2k_launch_point_transform(L.d_descs + d0, (int)(d1 - d0), L.max_w, L.max_h, L.nc, J->cp.irreversible, true, st);
    else if(d1 > d0)
      b2k_launch_dwt_fwd(L.d_descs + d0, (int)(d1 - d0), L.max_jobs, L.nc, J->cp.irreversible, st);
    if(first && time_level1)
    {
      CUDA_TRY(cudaEventRecord(l1_end, st));
      J->level1_alg_bytes = L.alg_bytes;
    }
    first = false;
  }
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int enqueue_inverse(b2k_device_job* J, cudaStream_t st, size_t t0 = 0, size_t t1 = (size_t)-1)
{
  t1 = std::min(t1, J->tiles.size());
  for(size_t li = 0; li < J->inv.size(); ++li)
  {
    LevelLaunch& L = J->inv[li];
    const uint32_t d0 = L.tile_first[t0], d1 = L.tile_first[t1];
    if(d1 > d0 && L.point)
      b2k_launch_point_transform(L.d_descs + d0, (int)(d1 - d0), L.max_w, L.max_h, L.nc, J->cp.irreversible, false, st);
    else if(d1 > d0)
      b2k_launch_dwt_inv(L.d_descs + d0, (int)(d1 - d0), L.max_jobs, L.nc, J->cp.irreversible, st);
  }
  CUDA_TRY(cudaGetLastError());
  return 0;
}

/* block coder over the coded blocks of selected tiles [t0, t1) */
static int enqueue_t1_blocks(b2k_device_job* J, cudaStream_t st, size_t t0, size_t t1)
{
  t1 = std::min(t1, J->tiles.size());
  const uint32_t b0 = J->coded_first[t0], b1 = J->coded_first[t1];
  if(b1 > b0)
    b2k_launch_ht_encode(J->d_enc_desc + b0, J->d_out + b0, J->d_scratch, b1 - b0, J->enc_limits, J->cp.irreversible, st);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

static int enqueue_t1_encode(b2k_device_job* J, cudaStream_t st)
{
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  b2k_launch_ht_encode(J->d_enc_desc, J->d_out, J->d_scratch, n, J->enc_limits, J->cp.irreversible, st);
  b2k_launch_scan_lengths(J->d_out, J->d_offsets, n, st);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

/* total size known -> (re)allocate the arena, compact */
static int finish_t1_encode(b2k_device_job* J, cudaStream_t st)
{
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  uint64_t total = 0;
  CUDA_TRY(cudaMemcpyAsync(&J->h_offsets[n], J->d_offsets + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  total = J->h_offsets[n];
  if(arena_reserve(J, total, total / 8)) return -1;
  J->bytes_used = total;
  J->arena_sized = true;
  b2k_launch_ht_gather(J->d_enc_desc, J->d_out, J->d_offsets, J->d_scratch, J->d_bytes, n, J->bytes_cap, st);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int32_t b2k_job_forward(b2k_device_job* J, float* ms)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  if(timed_stage(J, ms, [&](cudaStream_t st) { return enqueue_forward(J, st, true); })) return -1;
  CUDA_TRY(cudaEventElapsedTime(&J->last_level1_ms, J->ev[4], J->ev[5]));
  return 0;
}

extern "C" int32_t b2k_job_inverse(b2k_device_job* J, float* ms)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  J->arena_sized = false; /* the image planes now hold whatever the coefficient planes make */
  return timed_stage(J, ms, [&](cudaStream_t st) { return enqueue_inverse(J, st); });
}

extern "C" int32_t b2k_job_t1_encode(b2k_device_job* J, float* ms, uint64_t* total_bytes)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  if(timed_stage(J, ms, [&](cudaStream_t st) { return enqueue_t1_encode(J, st) || finish_t1_encode(J, st); })) return -1;
  if(total_bytes) *total_bytes = J->bytes_used;
  return 0;
}

/* decode descriptors from (length, offset, numbps) per coded block, for coded blocks [k0, k1) */
static int prepare_decode(b2k_device_job* J, const b2k_block* blocks, uint64_t num_blocks, cudaStream_t st, size_t k0 = 0,
                          size_t k1 = (size_t)-1)
{
  const size_t n = J->h_enc_desc.size();
  k1 = std::min(k1, n);
  if(num_blocks != J->blocks.size())
  {
    g_err = "block count does not match this coding's enumeration";
    return -1;
  }
  for(size_t k = k0; k < k1; ++k)
  {
    const b2k_block& b = blocks[J->coded_index[k]];
    HtBlockDesc d = J->h_enc_desc[k];
    d.length = b.length;
    d.slot_off = b.offset;
    if(b.numpasses > 3)
    {
      g_err = "an HT code block with more than 3 coding passes";
      return 1;
    }
    const t2::ParsedBlock pb{b.offset, b.length, b.length2, b.numbps, b.numpasses, {}};
    t2::block_decode_fields(pb, d.kmax, &d.mmsbs, &d.passes, &d.length2);
    if(d.passes > 1)
      J->dec_has_refinement = true;
    d.quant = J->dec_quant[k]; /* stepsize / 2^(31-Kmax), PostDecodeFiltersOJPH.h L103 */
    J->h_dec_desc[k] = d;
  }
  if(k1 > k0)
    CUDA_TRY(cudaMemcpyAsync(J->d_dec_desc + k0, J->h_dec_desc + k0, (k1 - k0) * sizeof(HtBlockDesc), cudaMemcpyHostToDevice, st));
  return 0;
}

static int enqueue_t1_decode_own(b2k_device_job* J, cudaStream_t st)
{
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  b2k_launch_build_dec_desc(J->d_enc_desc, J->d_out, J->d_offsets, J->d_dec_quant, J->d_dec_desc, n, J->bytes_cap, st);
  b2k_launch_ht_decode(J->d_dec_desc, J->d_bytes, J->d_recs, J->d_dec_status, n, J->max_cblk_w, J->d_err, J->cp.irreversible, 0, st);
  CUDA_TRY(cudaGetLastError());
  return 0;
}

extern "C" int32_t b2k_job_t1_decode(b2k_device_job* J, float* ms)
{
  if(!J) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  CUDA_TRY(cudaMemsetAsync(J->d_err, 0, sizeof(int), J->eng->stream));
  if(timed_stage(J, ms, [&](cudaStream_t st) { return enqueue_t1_decode_own(J, st); })) return -1;
  return decoder_verdict(J);
}

/* stage hook: block-decode a caller-supplied block table (what the host's T2 parse produced, or a foreign
   stream's blocks with SigProp / MagRef passes) into the job's coefficient planes */
extern "C" int32_t b2k_job_t1_decode_blocks(b2k_device_job* J, const b2k_block* blocks, uint64_t num_blocks,
                                            const uint8_t* bytes, uint64_t num_bytes, float* ms)
{
  if(!J || !blocks || (!bytes && num_bytes)) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  cudaStream_t st = J->eng->stream;
  J->arena_sized = false;
  if(arena_reserve(J, num_bytes, 0)) return -1;
  J->dec_has_refinement = false;
  if(int prc = prepare_decode(J, blocks, num_blocks, st)) return prc;
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  for(uint32_t k = 0; k < n; ++k)
    if((uint64_t)J->h_dec_desc[k].slot_off + J->h_dec_desc[k].length + J->h_dec_desc[k].length2 > num_bytes)
    {
      g_err = "block offsets exceed the byte arena";
      return -1;
    }
  CUDA_TRY(cudaMemsetAsync(J->d_err, 0, sizeof(int), st));
  if(num_bytes)
    CUDA_TRY(cudaMemcpyAsync(J->d_bytes, bytes, num_bytes, cudaMemcpyHostToDevice, st));
  auto decode = [&](cudaStream_t) {
    b2k_launch_ht_decode(J->d_dec_desc, J->d_bytes, J->d_recs, J->d_dec_status, n, J->max_cblk_w, J->d_err, J->cp.irreversible,
                         J->dec_has_refinement, st);
    if(J->dec_has_refinement)
      b2k_launch_ht_decode_refine(J->d_dec_desc, J->d_bytes, J->d_dec_status, n, (J->cp.cblk_sty & 0x08) != 0, st);
    return 0;
  };
  if(timed_stage(J, ms, decode)) return -1;
  CUDA_TRY(cudaGetLastError());
  return decoder_verdict(J);
}

/* One device-resident round trip, enqueued back to back with a single synchronisation at the end:
   forward (DC shift + MCT + DWT) -> block encode -> scan + compact -> block decode -> inverse.
   stage_ms[4] (optional) = forward, encode (incl. scan/compact), decode, inverse from CUDA events.  The arena is sized by
   one synchronising pass over each newly uploaded image; a 9/7 step codes the previous step's reconstruction, whose size
   can drift past that estimate's slack: then the call returns 2 with the arena grown, and the image planes hold the
   reconstruction of a partial decode, so the caller uploads the image again before calling again. */
extern "C" int32_t b2k_job_roundtrip(b2k_device_job* J, float* ms_total, float* stage_ms, uint64_t* total_bytes)
{
  return b2k_job_roundtrip_n(J, 1, ms_total, stage_ms, nullptr, total_bytes);
}

/* The frame the round trips share.  Each step owns `per` timing events of q_ev: e[0] its start, e[1] and e[2] around the
   level-1 transform, e[3 + i] the end of its stage i.  Before the first step: the device, the arena sized by one
   synchronising pass over a newly uploaded image, `events` events, the decoder's error count cleared. */
static int roundtrip_begin(b2k_device_job* J, size_t events)
{
  CUDA_TRY(cudaSetDevice(J->eng->device));
  if(!J->arena_sized)
  {
    if(int rc = b2k_job_forward(J, nullptr)) return rc;
    if(int rc = b2k_job_t1_encode(J, nullptr, nullptr)) return rc;
  }
  while(J->q_ev.size() < events)
  {
    cudaEvent_t ev;
    CUDA_TRY(cudaEventCreate(&ev));
    J->q_ev.push_back(ev);
  }
  CUDA_TRY(cudaMemsetAsync(J->d_err, 0, sizeof(int), J->eng->stream));
  return 0;
}

/* After the last step: the one synchronisation (on the end of the last step's last stage), the arena against the coded
   size, the times (each stage's and level 1's summed over the steps), the decoder's verdict. */
static int roundtrip_end(b2k_device_job* J, uint32_t steps, size_t per, int stages, float* ms_total, float* stage_ms, float* level1_ms,
                         uint64_t* total_bytes)
{
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  cudaEvent_t last = J->q_ev[per * (steps - 1) + 2 + stages];
  CUDA_TRY(cudaEventSynchronize(last));
  CUDA_TRY(cudaGetLastError());
  if(J->h_offsets[n] > J->bytes_cap)
  { /* arena estimate too small (a 9/7 step drifted past its slack): grow; the caller uploads again and repeats */
    if(arena_reserve(J, J->h_offsets[n], J->h_offsets[n] / 8)) return -1;
    g_err = "coded size grew past the arena: arena resized; the image planes hold a partial decode, upload again";
    return 2;
  }
  J->bytes_used = J->h_offsets[n];
  J->arena_sized = true;
  float sums[4] = {0, 0, 0, 0}, l1 = 0, tot = 0;
  for(uint32_t s = 0; s < steps; ++s)
  {
    cudaEvent_t* e = J->q_ev.data() + per * s;
    float t = 0;
    for(int i = 0; i < stages; ++i)
    {
      cudaEventElapsedTime(&t, e[i ? 2 + i : 0], e[3 + i]);
      sums[i] += t;
    }
    cudaEventElapsedTime(&t, e[1], e[2]);
    l1 += t;
  }
  cudaEventElapsedTime(&tot, J->q_ev[0], last);
  J->last_level1_ms = l1 / steps;
  if(ms_total) *ms_total = tot;
  if(stage_ms)
    for(int i = 0; i < stages; ++i)
      stage_ms[i] = sums[i];
  if(level1_ms) *level1_ms = l1;
  if(total_bytes) *total_bytes = J->bytes_used;
  return decoder_verdict(J);
}

/* n device-resident round trips queued back to back on the stream, ONE synchronisation after the last: what a
   benchmark step loop should cost when the host is not in the way (several ranks on one box).  Times come from
   events recorded per step: ms_total = first step's start to last step's end; stage_ms[4] and level1_ms are sums
   over the steps.  Returns 2 if the coded size outgrew the arena, as b2k_job_roundtrip does (arena resized, image planes
   no longer the input: upload again before calling again). */
extern "C" int32_t b2k_job_roundtrip_n(b2k_device_job* J, uint32_t steps, float* ms_total, float* stage_ms, float* level1_ms,
                                       uint64_t* total_bytes)
{
  if(!J || !steps) return -1;
  cudaStream_t st = J->eng->stream;
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  const size_t per = 7; /* start, l1 begin, l1 end, after forward, after encode, after decode, end */
  if(int rc = roundtrip_begin(J, per * steps)) return rc;
  for(uint32_t s = 0; s < steps; ++s)
  {
    cudaEvent_t* e = J->q_ev.data() + per * s;
    CUDA_TRY(cudaEventRecord(e[0], st));
    if(enqueue_forward(J, st, true, 0, (size_t)-1, e[1], e[2])) return -1;
    CUDA_TRY(cudaEventRecord(e[3], st));
    if(enqueue_t1_encode(J, st)) return -1;
    b2k_launch_ht_gather(J->d_enc_desc, J->d_out, J->d_offsets, J->d_scratch, J->d_bytes, n, J->bytes_cap, st);
    if(s + 1 == steps)
      CUDA_TRY(cudaMemcpyAsync(&J->h_offsets[n], J->d_offsets + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(e[4], st));
    if(enqueue_t1_decode_own(J, st)) return -1;
    CUDA_TRY(cudaEventRecord(e[5], st));
    if(enqueue_inverse(J, st)) return -1;
    CUDA_TRY(cudaEventRecord(e[6], st));
  }
  return roundtrip_end(J, steps, per, 4, ms_total, stage_ms, level1_ms, total_bytes);
}

/* The same n round trips with the BLOCK-CODER stage software-pipelined over tile-independent block ranges: the forward
   transform of the whole image runs alone on the main stream (its kernels are HBM-bound and are timed as such), then the
   coded blocks are cut into `chunks` ranges (0: 2) and each range goes encode -> scan -> compact -> parse (phase A) -> MagSgn
   (phase B) on one of `streams` side streams, so that the latency-bound kernels of one range (phase A is a serial chain
   per block, the scan a single CTA) run under the issue-bound kernels of its neighbours; the inverse transform again
   runs alone after all ranges have joined.  Ranges are independent except for the byte offsets of the compacted arena,
   which chain from one range's scan to the next (event per range).  stage_ms[3] = forward, block coder (encode + decode
   together), inverse.  Same results as b2k_job_roundtrip_n, byte for byte, return code 2 included. */
extern "C" int32_t b2k_job_roundtrip_pipelined_n(b2k_device_job* J, uint32_t steps, uint32_t chunks, uint32_t streams, float* ms_total,
                                                 float* stage_ms, float* level1_ms, uint64_t* total_bytes)
{
  if(!J || !steps) return -1;
  cudaStream_t st = J->eng->stream;
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  const size_t per = 5; /* start, l1 begin, l1 end, after forward, after the block coder; the next step's start ends the inverse */
  if(int rc = roundtrip_begin(J, per * steps + 1)) return rc;
  /* measured on config 2 (tools/stage_times.py, DESIGN.md section 6): 2 ranges on 2 streams 2.62 ms against 2.82 ms back to
     back; more ranges per stream lose (phase A's serial chain is a ~0.35 ms floor per launch, the persistent encoder grid
     fills every SM's shared memory), and so does a dedicated encoder stream with a capped grid */
  chunks = std::max(1u, std::min(chunks ? chunks : 2u, 64u));
  streams = std::max(1u, std::min(streams ? streams : 2u, 8u));
  /* ranges start on multiples of 128 blocks: whole CTAs of both decode kernels, whole record-interleave groups */
  const uint32_t per_chunk = std::max(128u, (((n + chunks - 1) / chunks) + 127u) & ~127u);
  const uint32_t nch = n ? (n + per_chunk - 1) / per_chunk : 0;
  while(J->p_streams.size() < streams)
  {
    cudaStream_t ps;
    CUDA_TRY(cudaStreamCreateWithFlags(&ps, cudaStreamNonBlocking));
    J->p_streams.push_back(ps);
  }
  while(J->p_ev.size() < 2 * (size_t)nch)
  {
    cudaEvent_t ev;
    CUDA_TRY(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    J->p_ev.push_back(ev);
  }
  for(uint32_t s = 0; s < steps; ++s)
  {
    cudaEvent_t* e = J->q_ev.data() + per * s;
    CUDA_TRY(cudaEventRecord(e[0], st));
    if(enqueue_forward(J, st, true, 0, (size_t)-1, e[1], e[2])) return -1;
    CUDA_TRY(cudaEventRecord(e[3], st));
    for(uint32_t k = 0; k < streams && k < nch; ++k)
      CUDA_TRY(cudaStreamWaitEvent(J->p_streams[k], e[3], 0));
    for(uint32_t c = 0; c < nch; ++c)
    {
      cudaStream_t ps = J->p_streams[c % streams];
      const uint32_t b0 = c * per_chunk, b1 = std::min(n, b0 + per_chunk), nb = b1 - b0;
      b2k_launch_ht_encode(J->d_enc_desc + b0, J->d_out + b0, J->d_scratch, nb, J->enc_limits, J->cp.irreversible, ps);
      if(c > 0)
        CUDA_TRY(cudaStreamWaitEvent(ps, J->p_ev[2 * (c - 1)], 0)); /* the previous range's end offset */
      b2k_launch_scan_lengths(J->d_out + b0, J->d_offsets + b0, nb, ps);
      CUDA_TRY(cudaEventRecord(J->p_ev[2 * c], ps));
      b2k_launch_ht_gather(J->d_enc_desc + b0, J->d_out + b0, J->d_offsets + b0, J->d_scratch, J->d_bytes, nb, J->bytes_cap, ps);
      b2k_launch_build_dec_desc(J->d_enc_desc + b0, J->d_out + b0, J->d_offsets + b0, J->d_dec_quant + b0, J->d_dec_desc + b0, nb,
                                J->bytes_cap, ps);
      b2k_launch_ht_decode(J->d_dec_desc + b0, J->d_bytes, J->d_recs, J->d_dec_status + b0, nb, J->max_cblk_w, J->d_err,
                           J->cp.irreversible, 0, ps);
      CUDA_TRY(cudaEventRecord(J->p_ev[2 * c + 1], ps));
    }
    for(uint32_t c = 0; c < nch; ++c)
      CUDA_TRY(cudaStreamWaitEvent(st, J->p_ev[2 * c + 1], 0));
    if(s + 1 == steps)
      CUDA_TRY(cudaMemcpyAsync(&J->h_offsets[n], J->d_offsets + n, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaEventRecord(e[4], st));
    if(enqueue_inverse(J, st)) return -1;
  }
  CUDA_TRY(cudaEventRecord(J->q_ev[per * steps], st)); /* the last step's e[per]: the end of its inverse */
  return roundtrip_end(J, steps, per, 3, ms_total, stage_ms, level1_ms, total_bytes);
}

extern "C" int32_t b2k_job_last_kernel_stats(const b2k_device_job* J, int which, float* ms, uint64_t* alg_bytes)
{
  if(!J) return -1;
  if(which == 0)
  {
    if(ms) *ms = J->last_level1_ms;
    if(alg_bytes) *alg_bytes = J->level1_alg_bytes;
    return 0;
  }
  return 1;
}

/* ---- results ---------------------------------------------------------------------------------- */
/* pinned result arenas are recycled: cudaHostAlloc of ~150 MB costs more than the whole encode */
struct PinnedPool
{
  std::mutex mu;
  std::vector<std::pair<uint8_t*, uint64_t>> free_list;
  std::vector<std::pair<uint8_t*, uint64_t>> live;
  std::vector<uint8_t*> heap; /* arenas that had to come from malloc (no CUDA device: b2k_result_merge on a writer-only host) */
};
static PinnedPool g_pool;
static uint8_t* pool_get(uint64_t bytes)
{
  std::lock_guard<std::mutex> lock(g_pool.mu);
  for(size_t i = 0; i < g_pool.free_list.size(); ++i)
    if(g_pool.free_list[i].second >= bytes)
    {
      auto e = g_pool.free_list[i];
      g_pool.free_list.erase(g_pool.free_list.begin() + i);
      g_pool.live.push_back(e);
      return e.first;
    }
  uint8_t* p = nullptr;
  const uint64_t cap = bytes + bytes / 4 + 4096;
  if(cudaHostAlloc(&p, cap, cudaHostAllocDefault) != cudaSuccess)
    return nullptr;
  g_pool.live.push_back({p, cap});
  return p;
}
static void pool_put(uint8_t* p)
{
  std::lock_guard<std::mutex> lock(g_pool.mu);
  for(size_t i = 0; i < g_pool.heap.size(); ++i)
    if(g_pool.heap[i] == p)
    {
      g_pool.heap.erase(g_pool.heap.begin() + i);
      free(p);
      return;
    }
  for(size_t i = 0; i < g_pool.live.size(); ++i)
    if(g_pool.live[i].first == p)
    {
      g_pool.free_list.push_back(g_pool.live[i]);
      g_pool.live.erase(g_pool.live.begin() + i);
      while(g_pool.free_list.size() > 16) /* streams keep depth-many results alive per direction; re-pinning 150 MB costs tens of ms */
      {
        cudaFreeHost(g_pool.free_list.front().first);
        g_pool.free_list.erase(g_pool.free_list.begin());
      }
      return;
    }
  cudaFreeHost(p);
}

/* the part of a result that does not depend on the device: the block table in enumeration order */
static b2k_result* result_shell(b2k_device_job* J)
{
  b2k_result* R = new b2k_result();
  memset(R, 0, sizeof(*R));
  R->num_blocks = J->blocks.size();
  R->blocks = (b2k_block*)malloc(sizeof(b2k_block) * std::max<size_t>(1, J->blocks.size()));
  memcpy(R->blocks, J->blocks.data(), sizeof(b2k_block) * J->blocks.size());
  R->num_tiles = (uint32_t)J->tiles.size();
  return R;
}

/* host_bytes: the caller already brought the byte arena home (chunk by chunk); meta_on_host: also the per-block
   lengths / offsets (h_out, h_offsets) are on their way on a stream that `st` waits for */
static int fetch_result(b2k_device_job* J, cudaStream_t st, b2k_result** out, uint8_t* host_bytes = nullptr,
                        b2k_result* shell = nullptr, bool meta_on_host = false)
{
  const uint32_t n = (uint32_t)J->h_enc_desc.size();
  b2k_result* R = shell ? shell : result_shell(J);
  R->num_bytes = J->bytes_used;
  R->bytes = host_bytes ? host_bytes : pool_get(std::max<uint64_t>(64, J->bytes_used));
  if(!R->bytes)
  {
    g_err = "cudaHostAlloc(result bytes) failed";
    free(R->blocks);
    delete R;
    return -1;
  }
  struct ResultGuard /* a failing CUDA call below must not leak the result and its pinned arena */
  {
    b2k_result* r;
    ~ResultGuard() { if(r) b2k_result_free(r); }
  } guard{R};
  if(!host_bytes)
    CUDA_TRY(cudaMemcpyAsync(R->bytes, J->d_bytes, J->bytes_used, cudaMemcpyDeviceToHost, st));
  if(!meta_on_host)
  {
    CUDA_TRY(cudaMemcpyAsync(J->h_out, J->d_out, n * sizeof(HtBlockOut), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(J->h_offsets, J->d_offsets, (n + 1) * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  int bad = 0;
  for(uint32_t k = 0; k < n; ++k)
  {
    b2k_block& b = R->blocks[J->coded_index[k]];
    if(J->h_out[k].total == 0xFFFFFFFFu)
    {
      bad++;
      continue;
    }
    b.length = J->h_out[k].total;
    b.offset = J->h_offsets[k];
    b.numbps = 1;    /* CoderOJPH.cpp L203-206 */
    b.numpasses = 1;
  }
  if(bad)
  {
    g_err = std::to_string(bad) + " code block(s) overflowed the coder's buffers";
    return -2;
  }
  guard.r = nullptr;
  *out = R;
  return 0;
}

extern "C" int32_t b2k_job_fetch_result(b2k_device_job* J, b2k_result** out)
{
  if(!J || !out) return -1;
  CUDA_TRY(cudaSetDevice(J->eng->device));
  return fetch_result(J, J->eng->stream, out);
}

extern "C" void b2k_result_free(b2k_result* r)
{
  if(!r) return;
  free(r->blocks);
  if(r->bytes) pool_put(r->bytes);
  delete r;
}

/* Merge the results of ranks that each coded the tiles t with t % nshards == rank (tile_mod / tile_rem of b2k_encode)
   into one result in full enumeration order -- what the writer rank needs for b2k_codestream_write after gathering the
   shards' block tables and byte arenas (SURVEY.md 8e).  The shards are not modified; free the merged result with
   b2k_result_free. */
extern "C" int32_t b2k_result_merge(const b2k_coding* cp, const b2k_result* const* shards, uint32_t nshards, b2k_result** out)
{
  if(!cp || !shards || !nshards || !out)
    return -1;
  if(const char* why = unsupported_reason(*cp))
  {
    g_err = why;
    return -1;
  }
  const TileGrid g = tile_grid(*cp);
  const uint32_t ntiles = g.nx * g.ny;
  const std::vector<std::vector<BandQuant>> q = component_quant(*cp);
  std::vector<b2k_block> all;
  for(uint32_t t = 0; t < ntiles; ++t)
    enumerate_tile_blocks(*cp, t, tile_rect(*cp, g, t), q, all);
  uint64_t total_bytes = 0;
  std::vector<uint64_t> base(nshards, 0);
  for(uint32_t s = 0; s < nshards; ++s)
  {
    if(!shards[s])
    {
      g_err = "missing shard";
      return -1;
    }
    base[s] = total_bytes;
    total_bytes += shards[s]->num_bytes;
  }
  b2k_result* R = new b2k_result();
  memset(R, 0, sizeof(*R));
  R->num_blocks = all.size();
  R->num_tiles = ntiles;
  R->num_bytes = total_bytes;
  R->blocks = (b2k_block*)malloc(sizeof(b2k_block) * std::max<size_t>(1, all.size()));
  /* recycled pinned arena (pinning a gigabyte costs hundreds of milliseconds); plain memory on a writer-only host */
  uint8_t* arena = pool_get(std::max<uint64_t>(64, total_bytes));
  if(!arena)
  {
    (void)cudaGetLastError();
    arena = (uint8_t*)malloc(std::max<uint64_t>(64, total_bytes));
    std::lock_guard<std::mutex> lock(g_pool.mu);
    g_pool.heap.push_back(arena);
  }
  R->bytes = arena;
  if(!R->blocks || !arena)
  {
    b2k_result_free(R);
    g_err = "out of memory";
    return -1;
  }
  std::vector<uint64_t> next(nshards, 0);
  for(size_t i = 0; i < all.size(); ++i)
  {
    const uint32_t s = all[i].tile % nshards;
    const b2k_result* S = shards[s];
    if(next[s] >= S->num_blocks)
    {
      b2k_result_free(R);
      g_err = "a shard holds fewer blocks than its tiles have";
      return -1;
    }
    const b2k_block& b = S->blocks[next[s]++];
    if(b.tile != all[i].tile || b.comp != all[i].comp || b.resno != all[i].resno || b.band_index != all[i].band_index ||
       b.precno != all[i].precno || b.cblkno != all[i].cblkno)
    {
      b2k_result_free(R);
      g_err = "a shard's block table is not the enumeration of the tiles t % nshards == shard";
      return -1;
    }
    R->blocks[i] = b;
    R->blocks[i].offset = b.offset + base[s];
  }
  for(uint32_t s = 0; s < nshards; ++s)
  {
    if(next[s] != shards[s]->num_blocks)
    {
      b2k_result_free(R);
      g_err = "a shard holds more blocks than its tiles have";
      return -1;
    }
  }
  { /* the arenas, 8 MB pieces on the host pool */
    struct Piece { uint8_t* dst; const uint8_t* src; size_t n; };
    std::vector<Piece> pieces;
    const size_t step = (size_t)8 << 20;
    for(uint32_t s = 0; s < nshards; ++s)
      for(size_t o = 0; o < shards[s]->num_bytes; o += step)
        pieces.push_back({arena + base[s] + o, shards[s]->bytes + o, std::min<size_t>(step, shards[s]->num_bytes - o)});
    b2k_host_parallel(pieces.size(), [&](size_t i) { memcpy(pieces[i].dst, pieces[i].src, pieces[i].n); });
  }
  *out = R;
  return 0;
}

/* ---- one-call host paths ---------------------------------------------------------------------- */
static bool dbg_timing()
{
  static const bool v = getenv("B2K_DEBUG_TIMING") != nullptr;
  return v;
}
#define DBG_T(label)                                                                                              \
  do                                                                                                              \
  {                                                                                                               \
    if(dbg_timing())                                                                                              \
      fprintf(stderr, "[b2k] %-28s %8.3f ms\n", label,                                                            \
              std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count());       \
  } while(0)

static b2k_device_job* cached_job(b2k_engine* e, const b2k_coding* cp, uint32_t mod, uint32_t rem, int* rc)
{
  b2k_device_job*& J = e->cached;
  cudaSetDevice(e->device);
  if(J && (memcmp(&J->cp, cp, sizeof(b2k_coding)) != 0 || J->tile_mod != mod || J->tile_rem != rem))
  {
    b2k_job_destroy(J);
    J = nullptr;
  }
  if(!J)
    *rc = b2k_job_create(e, cp, mod, rem, &J);
  else
    *rc = 0;
  return J;
}

/* T.user: the caller's samples.  A device image (b2k_encode_device) is read after the work queued on `caller`. */
static int32_t encode_common(b2k_engine* e, const b2k_coding* cp, uint32_t mod, uint32_t rem, b2k_result** out, Transport& T,
                             cudaStream_t caller = nullptr)
{
  if(!e || !cp || !out)
    return -1;
  std::lock_guard<std::mutex> lock(e->mu);
  int rc = 0;
  b2k_device_job* J = cached_job(e, cp, mod, rem, &rc);
  if(rc)
    return rc;
  CUDA_TRY(cudaSetDevice(e->device));
  const auto wall0 = std::chrono::steady_clock::now();
  if(resolve_transport(J, T, false))
    return -1;
  const bool dev = T.user.device;
  cudaStream_t st = e->stream;
  /* software pipeline over tile chunks: chunk k+1 crosses PCIe on the copy stream while chunk k
     is transformed and block-coded on the compute stream */
  cudaStream_t cs = e->copy_stream;
  /* what the caller queued before the call (the kernel that made the frame) comes first */
  if(dev && queue_after(e, caller, st)) return -1;
  CUDA_TRY(cudaEventRecord(J->ev[0], st));
  CUDA_TRY(cudaStreamWaitEvent(cs, J->ev[0], 0));
  const size_t nchunks = J->chunk_tile.size() - 1;
  /* the arena size of the previous call is the estimate: scan + compact + return every chunk's bytes while later
     chunks are still arriving (the D2H direction of PCIe is otherwise idle) */
  const bool streamed = J->bytes_cap > 0 && nchunks > 1;
  uint8_t* hb = nullptr;
  struct ArenaGuard /* the pinned arena goes back to the pool on every early return until a result owns it */
  {
    uint8_t*& p;
    ~ArenaGuard() { if(p) pool_put(p); }
  } arena_guard{hb};
  if(streamed)
  {
    hb = pool_get(J->bytes_cap);
    if(!hb)
    {
      g_err = "cudaHostAlloc(result bytes) failed";
      return -1;
    }
  }
  cudaStream_t ds = e->h2d_stream; /* third stream: device-to-host here */
  size_t next_out = 0, enqueued = 0;
  uint64_t total = 0;
  bool overflow = false;
  /* send finished chunks' bytes home; non-blocking while the host still has chunks to feed */
  auto return_chunks = [&](bool block) -> int {
    while(next_out < enqueued)
    {
      const size_t k = next_out;
      if(block)
        CUDA_TRY(cudaEventSynchronize(J->chunk_ev[CEV(2, k)]));
      else if(cudaEventQuery(J->chunk_ev[CEV(2, k)]) != cudaSuccess)
        break;
      const uint32_t b0 = J->coded_first[J->chunk_tile[k]], b1 = J->coded_first[J->chunk_tile[k + 1]];
      const uint64_t lo = k == 0 ? 0 : J->h_offsets[b0], hi = J->h_offsets[b1];
      total = hi;
      if(hi > J->bytes_cap)
        overflow = true;
      else if(hi > lo)
      {
        CUDA_TRY(cudaStreamWaitEvent(ds, J->chunk_ev[CEV(2, k)], 0));
        CUDA_TRY(cudaMemcpyAsync(hb + lo, J->d_bytes + lo, hi - lo, cudaMemcpyDeviceToHost, ds));
      }
      if(b1 > b0)
      { /* per-block lengths and offsets of the chunk ride along (h_offsets[b1] is already here) */
        CUDA_TRY(cudaStreamWaitEvent(ds, J->chunk_ev[CEV(2, k)], 0));
        CUDA_TRY(cudaMemcpyAsync(J->h_out + b0, J->d_out + b0, (size_t)(b1 - b0) * sizeof(HtBlockOut), cudaMemcpyDeviceToHost, ds));
        CUDA_TRY(cudaMemcpyAsync(J->h_offsets + b0, J->d_offsets + b0, (size_t)(b1 - b0) * sizeof(uint64_t),
                                 cudaMemcpyDeviceToHost, ds));
      }
      ++next_out;
    }
    (void)cudaGetLastError(); /* cudaEventQuery's cudaErrorNotReady is not an error */
    return 0;
  };
  for(size_t k = 0; k < nchunks; ++k)
  {
    const size_t t0 = J->chunk_tile[k], t1 = J->chunk_tile[k + 1];
    /* a device image's chunk is converted on the compute stream in place of its upload */
    if(dev ? device_convert(J, T.user, true, st, t0, t1, nullptr) : upload_chunk(J, T, k, st, cs, [&] { return return_chunks(false); }))
      return -1;
    if(k == nchunks - 1)
      CUDA_TRY(cudaEventRecord(J->ev[1], st)); /* all planes on the device */
    if(T.staged && device_convert(J, T.stage, true, st, t0, t1, nullptr)) return -1;
    if(enqueue_forward(J, st, k == 0, t0, t1)) return -1;
    if(enqueue_t1_blocks(J, st, t0, t1)) return -1;
    if(streamed)
    {
      const uint32_t b0 = J->coded_first[t0], b1 = J->coded_first[t1];
      if(b1 > b0)
      {
        b2k_launch_scan_lengths(J->d_out + b0, J->d_offsets + b0, b1 - b0, st);
        b2k_launch_ht_gather(J->d_enc_desc + b0, J->d_out + b0, J->d_offsets + b0, J->d_scratch, J->d_bytes, b1 - b0,
                             J->bytes_cap, st);
      }
      CUDA_TRY(cudaMemcpyAsync(&J->h_offsets[b1], J->d_offsets + b1, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
      CUDA_TRY(cudaEventRecord(J->chunk_ev[CEV(2, k)], st));
      enqueued = k + 1;
      if(return_chunks(false)) return -1;
    }
  }
  CUDA_TRY(cudaEventRecord(J->ev[2], st));
  /* the caller's stream goes on once every chunk of its image has been read */
  if(dev && queue_after(e, st, caller)) return -1;
  DBG_T("encode: chunks enqueued");
  b2k_result* R = nullptr;
  const uint32_t nb_all = (uint32_t)J->h_enc_desc.size();
  b2k_result* shell = result_shell(J); /* host work while the device finishes the last chunks */
  if(streamed)
  {
    if(return_chunks(true)) return -1;
    CUDA_TRY(cudaEventRecord(J->chunk_ev[CEV(3, 0)], ds));
    CUDA_TRY(cudaStreamWaitEvent(st, J->chunk_ev[CEV(3, 0)], 0));
    DBG_T("encode: last chunk coded");
    J->bytes_used = total;
    if(overflow)
    { /* estimate too small: grow, compact everything again from the scratch slots, plain copy */
      pool_put(hb);
      hb = nullptr;
      if(arena_reserve(J, total, total / 8)) return -1;
      b2k_launch_ht_gather(J->d_enc_desc, J->d_out, J->d_offsets, J->d_scratch, J->d_bytes, nb_all, J->bytes_cap, st);
      CUDA_TRY(cudaEventRecord(J->ev[3], st));
      if(int frc = fetch_result(J, st, &R, nullptr, shell)) return frc;
    }
    else
    {
      CUDA_TRY(cudaEventRecord(J->ev[3], st));
      uint8_t* owned = hb;
      hb = nullptr; /* fetch_result hands it to the result, or frees it with the result on failure */
      if(int frc = fetch_result(J, st, &R, owned, shell, true)) return frc;
    }
  }
  if(!streamed)
  {
    b2k_launch_scan_lengths(J->d_out, J->d_offsets, nb_all, st);
    if(finish_t1_encode(J, st)) return -1;
    CUDA_TRY(cudaEventRecord(J->ev[3], st));
    if(int frc = fetch_result(J, st, &R, nullptr, shell)) return frc;
  }
  DBG_T("encode: result fetched");
  CUDA_TRY(cudaEventRecord(J->ev[6], st));
  CUDA_TRY(cudaEventSynchronize(J->ev[6]));
  DBG_T("encode: done");
  float a = 0, b = 0, c = 0, d = 0;
  cudaEventElapsedTime(&a, J->ev[0], J->ev[1]);
  cudaEventElapsedTime(&b, J->ev[1], J->ev[2]);
  cudaEventElapsedTime(&c, J->ev[2], J->ev[3]);
  cudaEventElapsedTime(&d, J->ev[3], J->ev[6]);
  cudaEventElapsedTime(&J->last_level1_ms, J->ev[4], J->ev[5]);
  R->ms_h2d = a; R->ms_dwt = b; R->ms_t1 = c; R->ms_d2h = d; R->ms_total = a + b + c + d;
  if(T.tuner)
    T.tuner->record(T.ring, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count());
  *out = R;
  return 0;
}

/* the caller's planes in host memory, samples of 4 or 2 bytes, the first one at canvas (x0, y0) */
static int32_t host_samples(Transport& T, const b2k_coding* cp, const void* const* planes, const uint32_t* strides, uint32_t sample_bytes,
                            uint32_t x0, uint32_t y0)
{
  if(!planes || !strides)
    return -1;
  T.user = planar_container(cp->numcomps, const_cast<void* const*>(planes), strides, sample_bytes, x0, y0, false);
  return 0;
}
/* the caller's device image, the first sample at canvas (x0, y0) */
static void device_samples(Transport& T, const b2k_device_planes& img, uint32_t x0, uint32_t y0)
{
  T.user.d = img;
  T.user.ox = x0;
  T.user.oy = y0;
  T.user.device = true;
}

extern "C" int32_t b2k_encode(b2k_engine* e, const b2k_coding* cp, const int32_t* const* planes, const uint32_t* strides,
                              uint32_t tile_mod, uint32_t tile_rem, b2k_result** out)
{
  Transport T;
  if(!cp || host_samples(T, cp, (const void* const*)planes, strides, 4, cp->x0, cp->y0))
    return -1;
  return encode_common(e, cp, tile_mod, tile_rem, out, T);
}

extern "C" int32_t b2k_encode16(b2k_engine* e, const b2k_coding* cp, const uint16_t* const* planes, const uint32_t* strides,
                                uint32_t tile_mod, uint32_t tile_rem, b2k_result** out)
{
  Transport T;
  if(!cp || host_samples(T, cp, (const void* const*)planes, strides, 2, cp->x0, cp->y0))
    return -1;
  return encode_common(e, cp, tile_mod, tile_rem, out, T);
}

extern "C" int32_t b2k_encode16_interleaved(b2k_engine* e, const b2k_coding* cp, const uint16_t* pixels, uint32_t stride,
                                            uint32_t tile_mod, uint32_t tile_rem, b2k_result** out)
{
  if(!cp || !pixels || stride < (uint32_t)(cp->x1 - cp->x0) * cp->numcomps)
    return -1;
  Transport T;
  T.user = interleaved_container(cp->numcomps, const_cast<uint16_t*>(pixels), stride, 2, cp->x0, cp->y0, false);
  return encode_common(e, cp, tile_mod, tile_rem, out, T);
}

static int32_t decode_common(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                             const uint8_t* bytes, uint64_t num_bytes, uint32_t tile_mod, uint32_t tile_rem, double* ms_total,
                             Transport& T, const uint32_t* window = nullptr, cudaStream_t caller = nullptr);

extern "C" int32_t b2k_decode(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                              const uint8_t* bytes, uint64_t num_bytes, int32_t* const* planes, const uint32_t* strides,
                              uint32_t tile_mod, uint32_t tile_rem, double* ms_total)
{
  Transport T;
  if(!cp || host_samples(T, cp, (const void* const*)planes, strides, 4, cp->x0, cp->y0))
    return -1;
  return decode_common(e, cp, blocks, num_blocks, bytes, num_bytes, tile_mod, tile_rem, ms_total, T);
}
extern "C" int32_t b2k_decode16(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                                const uint8_t* bytes, uint64_t num_bytes, uint16_t* const* planes, const uint32_t* strides,
                                uint32_t tile_mod, uint32_t tile_rem, double* ms_total)
{
  Transport T;
  if(!cp || host_samples(T, cp, (const void* const*)planes, strides, 2, cp->x0, cp->y0))
    return -1;
  return decode_common(e, cp, blocks, num_blocks, bytes, num_bytes, tile_mod, tile_rem, ms_total, T);
}

/* b2k_decode / b2k_decode16 with only `window` (x0, y0, x1, y1 in cp's canvas coordinates) of the pixels returned: planes[c]
   holds window rows of strides[c] samples.  With b2k_codestream_parse_window this is the windowed decode of SURVEY 8f N3: the
   tiles the window touches are decoded, the window's pixels alone cross PCIe. */
extern "C" int32_t b2k_decode_window(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                                     const uint8_t* bytes, uint64_t num_bytes, void* const* planes, const uint32_t* strides,
                                     const uint32_t* window, uint32_t sample_bytes, double* ms_total)
{
  Transport T;
  if(!cp || !window || (sample_bytes != 2 && sample_bytes != 4) ||
     host_samples(T, cp, (const void* const*)planes, strides, sample_bytes, window[0], window[1]))
    return -1;
  return decode_common(e, cp, blocks, num_blocks, bytes, num_bytes, 1, 0, ms_total, T, window);
}

/* NULL is the legacy default stream, as the CUDA Array Interface assumes */
static cudaStream_t caller_stream(void* s) { return s ? static_cast<cudaStream_t>(s) : cudaStreamLegacy; }

extern "C" int32_t b2k_encode_device(b2k_engine* e, const b2k_coding* cp, const b2k_device_planes* img, uint32_t tile_mod,
                                     uint32_t tile_rem, void* cuda_stream, b2k_result** out)
{
  if(!e || !cp || !out)
    return -1;
  if(int rc = check_device_planes(e, cp, img))
    return rc;
  Transport T;
  device_samples(T, *img, cp->x0, cp->y0);
  return encode_common(e, cp, tile_mod, tile_rem, out, T, caller_stream(cuda_stream));
}

extern "C" int32_t b2k_decode_device(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                                     const uint8_t* bytes, uint64_t num_bytes, const b2k_device_planes* img, const uint32_t* window,
                                     uint32_t tile_mod, uint32_t tile_rem, void* cuda_stream, double* ms_total)
{
  if(!e || !cp)
    return -1;
  if(window && tile_mod != 1)
  {
    g_err = "a windowed decode takes every tile: tile_mod must be 1";
    return -1;
  }
  if(int rc = check_device_planes(e, cp, img))
    return rc;
  Transport T;
  device_samples(T, *img, window ? window[0] : cp->x0, window ? window[1] : cp->y0);
  return decode_common(e, cp, blocks, num_blocks, bytes, num_bytes, tile_mod, tile_rem, ms_total, T, window, caller_stream(cuda_stream));
}

/* the block decoder over chunk k's coded blocks, from the descriptors in d_dec_desc and the bytes in d_bytes: phase A
   (serial VLC/MEL parse, one thread per block) is latency-bound and leaves the SMs nearly empty, so the chunks' parses run
   concurrently on side streams once `ready` (this chunk's descriptors + bytes are on the device) has happened, ahead of st */
static int enqueue_block_decode(b2k_engine* e, b2k_device_job* J, size_t k, cudaEvent_t ready, cudaStream_t st,
                                size_t t0 = (size_t)-1, size_t t1 = (size_t)-1)
{
  /* chunk k's tiles, or selected tiles [t0, t1) (a batch's chunk k over the slots it uses) */
  const uint32_t b0 = J->coded_first[t0 == (size_t)-1 ? J->chunk_tile[k] : t0];
  const uint32_t b1 = J->coded_first[t1 == (size_t)-1 ? J->chunk_tile[k + 1] : t1];
  if(b1 <= b0)
    return 0;
  cudaStream_t ax = e->aux[k & 3];
  if(ready)
    CUDA_TRY(cudaStreamWaitEvent(ax, ready, 0));
  b2k_launch_ht_decode_vlc(J->d_dec_desc + b0, J->d_bytes, J->d_recs, J->d_dec_status + b0, b1 - b0, J->max_cblk_w, ax);
  CUDA_TRY(cudaEventRecord(J->chunk_ev[CEV(2, k)], ax));
  CUDA_TRY(cudaStreamWaitEvent(st, J->chunk_ev[CEV(2, k)], 0));
  /* a batch counts the blocks the HT decoder rejects per slot */
  b2k_launch_ht_decode_magsgn(J->d_dec_desc + b0, J->d_bytes, J->d_recs, J->d_dec_status + b0, b1 - b0, J->max_cblk_w, J->d_err,
                              J->cp.irreversible, J->dec_has_refinement, st, b0, J->slots > 1 ? (uint32_t)J->coded_index.size() : 0);
  if(J->dec_has_refinement)
    b2k_launch_ht_decode_refine(J->d_dec_desc + b0, J->d_bytes, J->d_dec_status + b0, b1 - b0, (J->cp.cblk_sty & 0x08) != 0, st);
  return 0;
}

/* T.user: the caller's samples, which hold only `window` (x0, y0, x1, y1) of the pixels when there is one.  A device image
   (b2k_decode_device) is written after the work queued on `caller` */
static int32_t decode_common(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                             const uint8_t* bytes, uint64_t num_bytes, uint32_t tile_mod, uint32_t tile_rem, double* ms_total,
                             Transport& T, const uint32_t* window, cudaStream_t caller)
{
  if(!e || !cp || !blocks)
    return -1;
  if(window &&
     (window[0] >= window[2] || window[1] >= window[3] || window[0] < cp->x0 || window[1] < cp->y0 || window[2] > cp->x1 || window[3] > cp->y1))
  {
    g_err = "window outside the image";
    return -1;
  }
  std::lock_guard<std::mutex> lock(e->mu);
  int rc = 0;
  b2k_device_job* J = cached_job(e, cp, tile_mod, tile_rem, &rc);
  if(rc)
    return rc;
  CUDA_TRY(cudaSetDevice(e->device));
  const Rect win = window ? Rect{window[0], window[1], window[2], window[3]} : Rect{};
  T.window = window ? &win : nullptr;
  const auto wall0 = std::chrono::steady_clock::now();
  if(resolve_transport(J, T, true))
    return -1;
  const bool dev = T.user.device;
  cudaStream_t st = e->stream;
  if(arena_reserve(J, num_bytes, 0)) return -1;
  /* what the caller queued before the call (e.g. the last reader of its buffer) comes first */
  if(dev && queue_after(e, caller, st)) return -1;
  CUDA_TRY(cudaEventRecord(J->ev[0], st));
  CUDA_TRY(cudaMemsetAsync(J->d_err, 0, sizeof(int), st));
  J->dec_has_refinement = false;
  cudaStream_t cs = e->copy_stream;
  const size_t nchunks = J->chunk_tile.size() - 1;
  CUDA_TRY(cudaStreamWaitEvent(cs, J->ev[0], 0));
  CUDA_TRY(cudaStreamWaitEvent(e->h2d_stream, J->ev[0], 0));
  /* Pipeline over tile chunks.  Host: build chunk k's descriptors while the device works on chunk
     k-1.  PCIe in: chunk k's coded bytes (one contiguous range when the arena is in block order,
     which ours always is; otherwise the whole arena goes up once).  Compute: block decode +
     inverse transform.  PCIe out: chunk k-1's pixels -- both directions stay busy. */
  bool all_uploaded = false;
  uint64_t prev_end = 0;
  for(size_t k = 0; k < nchunks; ++k)
  {
    const size_t t0 = J->chunk_tile[k], t1 = J->chunk_tile[k + 1];
    const uint32_t b0 = J->coded_first[t0], b1 = J->coded_first[t1];
    /* descriptors travel on the upload stream with the chunk's bytes, so the side-stream parse of
       chunk k+1 depends on nothing the main stream is still doing for chunk k */
    if(int prc = prepare_decode(J, blocks, num_blocks, e->h2d_stream, b0, b1)) return prc;
    uint64_t lo = UINT64_MAX, hi = 0;
    for(uint32_t b = b0; b < b1; ++b)
    {
      const HtBlockDesc& d = J->h_dec_desc[b];
      if(!d.length)
        continue;
      lo = std::min<uint64_t>(lo, d.slot_off);
      hi = std::max<uint64_t>(hi, d.slot_off + d.length + d.length2);
    }
    if(hi > num_bytes)
    {
      g_err = "block offsets exceed the byte arena";
      return -1;
    }
    if(!all_uploaded && lo != UINT64_MAX)
    {
      if(lo < prev_end)
      { /* arena not in block order (a foreign codestream whose tile parts are out of tile order, a caller arena laid
           out some other way): ranges below prev_end that no earlier chunk covered may be needed now, so the whole
           arena goes up once; bytes already on the device are simply written again with the same values */
        CUDA_TRY(cudaMemcpyAsync(J->d_bytes, bytes, num_bytes, cudaMemcpyHostToDevice, e->h2d_stream));
        all_uploaded = true;
      }
      else
      {
        CUDA_TRY(cudaMemcpyAsync(J->d_bytes + lo, bytes + lo, hi - lo, cudaMemcpyHostToDevice, e->h2d_stream));
        prev_end = hi;
      }
    }
    CUDA_TRY(cudaEventRecord(J->chunk_ev[CEV(1, k)], e->h2d_stream));
    CUDA_TRY(cudaStreamWaitEvent(st, J->chunk_ev[CEV(1, k)], 0));
    if(enqueue_block_decode(e, J, k, J->chunk_ev[CEV(1, k)], st)) return -1;
    if(enqueue_inverse(J, st, t0, t1)) return -1;
    if(download_chunk(J, T, k, st, cs)) return -1;
  }
  DBG_T("decode: chunks enqueued");
  if(T.ring && ring_download_all(J, T.user, T.stage, cs)) return -1;
  CUDA_TRY(cudaEventRecord(J->chunk_ev[CEV(0, nchunks)], cs));
  CUDA_TRY(cudaStreamWaitEvent(st, J->chunk_ev[CEV(0, nchunks)], 0));
  CUDA_TRY(cudaEventRecord(J->ev[1], st));
  /* the caller's stream goes on once its image is written */
  if(dev && queue_after(e, st, caller)) return -1;
  CUDA_TRY(cudaEventSynchronize(J->ev[1]));
  CUDA_TRY(cudaGetLastError());
  DBG_T("decode: done");
  float t = 0;
  cudaEventElapsedTime(&t, J->ev[0], J->ev[1]);
  if(ms_total) *ms_total = t;
  if(T.tuner)
    T.tuner->record(T.ring, std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - wall0).count());
  return decoder_verdict(J);
}

/* ---- code streams in device memory (b2k_decode_codestream_device / b2k_codestream_parse_device) ----------------------
 * The main header is read on the host from a prefix of the stream, by b2k_codestream_parse's own code; the tile parts and
 * packets are parsed on the device (t2_decode.cu) from a copy of the stream in the job's arena, which also gives the HT
 * decoder the slack it reads past a block.  A single stream is a batch of one (b2k_decode_codestreams_device below): the
 * same header read, arena copy, parse and image write, in slot 0 of the engine's single-image job.  Synchronisations: the
 * header, the parse status, the end of the decode. */
static int check_device_bytes(const b2k_engine* e, const uint8_t* cs, uint64_t len)
{
  if(len == 0)
  { /* no bytes, whatever the pointer (an empty tensor's is often NULL): what the host parser says of them */
    g_err = "no SOC marker";
    return -1;
  }
  cudaPointerAttributes a{};
  const cudaError_t err = cs ? cudaPointerGetAttributes(&a, cs) : cudaErrorInvalidValue;
  if(err != cudaSuccess)
    (void)cudaGetLastError();
  if(err != cudaSuccess || (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != e->device)
  {
    g_err = "code stream: not device or managed memory of the engine's device (" + std::to_string(e->device) + ")";
    return -1;
  }
  return 0;
}

static int grow_copy_table(b2k_engine* e, uint32_t n)
{
  if(n <= e->copy_cap)
    return 0;
  cudaFree(e->d_copy);
  cudaFreeHost(e->h_copy);
  e->d_copy = nullptr;
  e->h_copy = nullptr;
  e->copy_cap = 0;
  CUDA_TRY(cudaMalloc(&e->d_copy, n * sizeof(CopyEntry)));
  CUDA_TRY(cudaHostAlloc(&e->h_copy, n * sizeof(CopyEntry), cudaHostAllocDefault));
  e->copy_cap = n;
  return 0;
}

/* h_copy[0, m) into out on st: the table to the device and one gather launch, or for one entry a plain device-to-device
   copy */
static int gather_streams(b2k_engine* e, uint32_t m, uint64_t max_len, uint8_t* out, cudaStream_t st)
{
  if(m == 1)
  {
    CUDA_TRY(cudaMemcpyAsync(out + e->h_copy[0].dst, e->h_copy[0].src, e->h_copy[0].len, cudaMemcpyDeviceToDevice, st));
    return 0;
  }
  if(!m)
    return 0;
  CUDA_TRY(cudaMemcpyAsync(e->d_copy, e->h_copy, m * sizeof(CopyEntry), cudaMemcpyHostToDevice, st));
  return b2k_copy_table(e->d_copy, m, max_len, out, st);
}

/* the main headers h[i] of the n streams whose status is 0, read on st by b2k_parse_main_header from prefixes of `prefix`
   bytes gathered into one copy; the streams whose header runs past its prefix go round again together with twice the
   prefix.  A stream whose header fails gets its status and, with `errors`, its text there.  0, or -1 for a failure of the
   call. */
static int read_batch_headers(b2k_engine* e, uint32_t n, const uint8_t* const* cs, const uint64_t* len, uint64_t prefix, cudaStream_t st,
                              int32_t* status, b2k::t2::MainHeader* h, std::string* errors)
{
  std::vector<uint64_t> want(n, 0);
  for(uint32_t i = 0; i < n; ++i)
    want[i] = status[i] ? 0 : std::min<uint64_t>(len[i], prefix);
  for(;;)
  {
    uint32_t m = 0;
    uint64_t total = 0, longest = 0;
    if(grow_copy_table(e, n)) return -1;
    for(uint32_t i = 0; i < n; ++i)
      if(want[i])
      {
        e->h_copy[m++] = CopyEntry{cs[i], want[i], total};
        total += want[i];
        longest = std::max(longest, want[i]);
      }
    if(!m)
      return 0;
    if(total > e->hdr_cap)
    {
      cudaFree(e->d_hdr);
      cudaFreeHost(e->h_hdr);
      e->d_hdr = nullptr;
      e->h_hdr = nullptr;
      e->hdr_cap = 0;
      CUDA_TRY(cudaMalloc(&e->d_hdr, total));
      CUDA_TRY(cudaHostAlloc(&e->h_hdr, total, cudaHostAllocDefault));
      e->hdr_cap = total;
    }
    if(m == 1) /* one prefix goes to the host as it is */
      CUDA_TRY(cudaMemcpyAsync(e->h_hdr, e->h_copy[0].src, total, cudaMemcpyDeviceToHost, st));
    else
    {
      if(gather_streams(e, m, longest, e->d_hdr, st)) return -1;
      CUDA_TRY(cudaMemcpyAsync(e->h_hdr, e->d_hdr, total, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    uint64_t at = 0;
    for(uint32_t i = 0; i < n; ++i)
    {
      if(!want[i])
        continue;
      const uint64_t got = want[i];
      const int rc = b2k_parse_main_header(e->h_hdr + at, got, h[i]);
      at += got;
      want[i] = 0;
      if(rc && h[i].short_read && got < len[i])
        want[i] = std::min<uint64_t>(len[i], 2 * got);
      else if(rc)
      {
        status[i] = rc;
        if(errors)
          errors[i] = g_err;
      }
    }
  }
}

/* one stream's main header, read after the work queued on `caller` from a 64 KiB prefix, so that a large TLM costs no
   second round trip: 0, or b2k_codestream_parse's code with its text */
static int read_main_header(b2k_engine* e, const uint8_t* cs, uint64_t len, cudaStream_t caller, b2k::t2::MainHeader& h)
{
  CUDA_TRY(cudaSetDevice(e->device));
  if(queue_after(e, caller, e->stream)) return -1;
  int32_t status = 0;
  if(read_batch_headers(e, 1, &cs, &len, 64u << 10, e->stream, &status, &h, nullptr)) return -1;
  return status;
}

/* the parse on st of the streams i < n whose status is 0 (main headers h[i], progression and SOP / EPH `flags`) in slots i
   of J: the streams laid out in the arena at 256-byte boundaries (with headroom for a larger batch when n > 1), then
   the five parse kernels and, with dec, the decoder's descriptors.  One synchronisation; a stream that fails gets its
   status and, with `errors`, its text there.  *refinement: a stream has refinement passes.  0, or -1 for a failure of
   the call. */
static int parse_streams(b2k_engine* e, b2k_device_job* J, uint32_t n, const uint8_t* const* cs, const uint64_t* len,
                         const b2k::t2::MainHeader* h, uint32_t flags, bool dec, int32_t* status, std::string* errors, bool* refinement)
{
  cudaStream_t st = e->stream;
  if(!J->t2p || b2k_t2_parse_flags(J->t2p) != flags || b2k_t2_parse_streams(J->t2p) != J->slots)
  { /* geometry and progression only: planned once for every stream or batch of this coding */
    drop_parse(J, J->t2p);
    if(b2k_t2_parse_create(J->cp, flags, J->blocks.data(), J->blocks.size(), J->slot_tiles, J->coded_index.data(), J->coded_index.size(),
                           &J->t2p, J->slots))
      return -1;
  }
  /* the arena: stream i at a 256-byte boundary, the decoder's read-past slack after the last one; one gather */
  std::vector<uint64_t> at(n, 0), plen(n, 0), sot(n, 0);
  uint64_t total = 0, longest = 0;
  uint32_t m = 0;
  if(grow_copy_table(e, n)) return -1;
  for(uint32_t i = 0; i < n; ++i)
  {
    if(status[i])
      continue;
    at[i] = total;
    plen[i] = len[i];
    sot[i] = h[i].sot;
    e->h_copy[m++] = CopyEntry{cs[i], len[i], total};
    longest = std::max(longest, len[i]);
    total = b2k::t2::batch_arena_next(total, len[i]);
  }
  if(arena_reserve(J, total, n > 1 ? total / 8 : 0)) return -1;
  J->arena_sized = false; /* the arena now holds callers' streams, not this job's coding of its image */
  e->last_parse = J->t2p;
  CUDA_TRY(cudaEventRecord(J->ev[0], st));
  if(gather_streams(e, m, longest, J->d_bytes, st)) return -1;
  if(b2k_t2_batch_enqueue(J->t2p, J->d_bytes, n, at.data(), plen.data(), sot.data(), J->d_enc_desc, J->d_dec_quant,
                          dec ? J->d_dec_desc : nullptr, st))
    return -1;
  CUDA_TRY(cudaStreamSynchronize(st));
  bool any = false;
  for(uint32_t i = 0; i < n; ++i)
  {
    if(status[i])
      continue;
    bool r = false;
    if(int prc = b2k_t2_batch_result(J->t2p, i, &r))
    {
      status[i] = prc;
      if(errors)
        errors[i] = g_err;
    }
    any = any || r;
  }
  if(refinement)
    *refinement = any;
  return 0;
}

/* after a parse into J's descriptors: block decode -> inverse -> images, chunk by chunk over the (slot, tile) ranges of the
   n slots used (as many chunks as the job's pipeline has, whatever its slot count).  After the chunk that holds slot i's
   last tile, rects[i] of its planes (the whole canvas, or a window on the virtual canvas) goes to imgs[i] when status[i]
   is 0, in one launch per component group.  With write_rejected the image of a slot whose blocks the HT decoder rejected
   is written too (as b2k_decode_device writes it), else it is left alone.  The caller's stream then waits for the
   writes.  A slot with rejected blocks gets -2 and, with `errors`, its text there.  0, or -1 for a failure of the call. */
static int decode_slots(b2k_engine* e, b2k_device_job* J, uint32_t n, const b2k_device_planes* imgs, const Rect* rects, bool refinement,
                        bool write_rejected, cudaStream_t caller, double* ms_total, int32_t* status, std::string* errors)
{
  cudaStream_t st = e->stream;
  /* the conversion's tables: one per component, or one for all when every image written is pixel-interleaved */
  const int nc = J->cp.numcomps;
  bool interleaved = nc > 1;
  for(uint32_t i = 0; i < n; ++i)
    if(!status[i])
      interleaved = interleaved && device_group(imgs[i], nc) == nc;
  const int group = interleaved ? nc : 1, tables = nc / group;
  uint32_t max_w = 0, max_h = 0;
  if(!J->h_batch_dst)
  {
    CUDA_TRY(cudaMalloc(&J->d_batch_dst, (size_t)J->slots * 4 * sizeof(BatchDst)));
    CUDA_TRY(cudaHostAlloc(&J->h_batch_dst, (size_t)J->slots * 4 * sizeof(BatchDst), cudaHostAllocDefault));
  }
  for(int t = 0; t < tables; ++t)
    for(uint32_t i = 0; i < n; ++i)
    {
      BatchDst& D = J->h_batch_dst[(size_t)t * n + i];
      D = BatchDst{};
      if(status[i])
        continue;
      const int c0 = t * group;
      const Rect& r = rects[i];
      for(int k = 0; k < group; ++k)
        D.src[k] = J->img.at((int)i * nc + c0 + k, r.x0, r.y0);
      D.dst = imgs[i].comp[c0];
      D.err = write_rejected ? nullptr : J->d_err + i;
      D.dpitch = imgs[i].row_pitch[c0];
      D.step = imgs[i].col_step[c0];
      D.w = r.w();
      D.h = r.h();
      max_w = std::max(max_w, D.w);
      max_h = std::max(max_h, D.h);
    }
  CUDA_TRY(cudaMemcpyAsync(J->d_batch_dst, J->h_batch_dst, (size_t)tables * n * sizeof(BatchDst), cudaMemcpyHostToDevice, st));
  CUDA_TRY(cudaMemsetAsync(J->d_err, 0, n * sizeof(int), st));
  J->dec_has_refinement = refinement;
  const size_t used = (size_t)n * J->slot_tiles, T = J->slot_tiles;
  const size_t nchunks = std::min<size_t>(J->chunk_tile.size() - 1, used);
  const uint32_t sb = imgs[0].sample_bytes;
  for(size_t k = 0; k < nchunks; ++k)
  {
    const size_t t0 = k * used / nchunks, t1 = (k + 1) * used / nchunks;
    if(t1 <= t0)
      continue;
    if(enqueue_block_decode(e, J, k, nullptr, st, t0, t1)) return -1;
    if(enqueue_inverse(J, st, t0, t1)) return -1;
    const uint32_t s0 = (uint32_t)(t0 / T), s1 = (uint32_t)(t1 / T);
    for(int t = 0; t < tables && s1 > s0; ++t)
      b2k_launch_planes_to_containers(J->d_batch_dst + (size_t)t * n + s0, s1 - s0, group, J->img.pitch, sb, max_w, max_h, st);
  }
  CUDA_TRY(cudaEventRecord(J->ev[1], st));
  /* the caller's stream goes on once its images are written */
  if(queue_after(e, st, caller)) return -1;
  CUDA_TRY(cudaEventSynchronize(J->ev[1]));
  CUDA_TRY(cudaGetLastError());
  float t = 0;
  cudaEventElapsedTime(&t, J->ev[0], J->ev[1]);
  if(ms_total) *ms_total = t;
  /* the HT decoder's verdict, per slot */
  std::vector<int> herr(n, 0);
  CUDA_TRY(cudaMemcpy(herr.data(), J->d_err, n * sizeof(int), cudaMemcpyDeviceToHost));
  for(uint32_t i = 0; i < n; ++i)
    if(!status[i] && herr[i])
    {
      g_err = "HT decoder rejected " + std::to_string(herr[i]) + " block(s)";
      status[i] = -2;
      if(errors)
        errors[i] = g_err;
    }
  return 0;
}

/* the single-stream calls' job (of h's coding) and the stream's parse in its slot 0, with dec the decoder's descriptors
   too; the caller's block table is checked first, as the host parser checks it before it looks at a tile part.  0, or
   b2k_codestream_parse's code with its text.  *out: the job, once there is one. */
static int parse_single(b2k_engine* e, const uint8_t* cs, uint64_t len, const b2k::t2::MainHeader& h, b2k_device_job** out, bool dec,
                        bool* refinement, uint64_t cap_blocks = UINT64_MAX)
{
  int rc = 0;
  b2k_device_job* J = cached_job(e, &h.cp, 1, 0, &rc);
  if(rc)
    return rc;
  *out = J;
  if(cap_blocks < J->blocks.size())
  {
    g_err = "block table too small";
    return -1;
  }
  int32_t status = 0;
  if(parse_streams(e, J, 1, &cs, &len, &h, h.flags(), dec, &status, nullptr, refinement)) return -1;
  return status;
}

extern "C" int64_t b2k_codestream_parse_device(b2k_engine* e, const uint8_t* cs, uint64_t len, void* cuda_stream, b2k_coding* cp_out,
                                               b2k_block* blocks, uint64_t cap_blocks)
{
  if(!e || !cp_out)
    return -1;
  if(check_device_bytes(e, cs, len))
    return -1;
  std::lock_guard<std::mutex> lock(e->mu);
  b2k::t2::MainHeader h;
  if(int rc = read_main_header(e, cs, len, caller_stream(cuda_stream), h))
    return rc;
  if(!blocks)
  {
    *cp_out = h.cp;
    return b2k_enumerate(&h.cp, 1, 0, nullptr, 0);
  }
  b2k_device_job* J = nullptr;
  int rc = parse_single(e, cs, len, h, &J, false, nullptr, cap_blocks);
  if(J)
    *cp_out = h.cp;
  if(rc)
    return rc;
  const uint64_t n = J->blocks.size();
  if(b2k_t2_parse_blocks(J->t2p, blocks, e->stream))
    return -1;
  return (int64_t)n;
}

extern "C" int32_t b2k_decode_codestream_device(b2k_engine* e, const uint8_t* cs, uint64_t len, const b2k_device_planes* img,
                                                void* cuda_stream, b2k_coding* cp_out, double* ms_total)
{
  if(!e || !cp_out)
    return -1;
  if(check_device_bytes(e, cs, len))
    return -1;
  std::lock_guard<std::mutex> lock(e->mu);
  const auto wall0 = std::chrono::steady_clock::now();
  cudaStream_t caller = caller_stream(cuda_stream);
  b2k::t2::MainHeader h;
  if(int rc = read_main_header(e, cs, len, caller, h))
    return rc;
  b2k_device_job* J = nullptr;
  bool refinement = false;
  if(int rc = parse_single(e, cs, len, h, &J, true, &refinement))
    return rc;
  *cp_out = h.cp;
  DBG_T("device decode: parsed");
  if(int rc = check_device_planes(e, &h.cp, img))
    return rc;
  int32_t status = 0;
  const Rect whole{h.cp.x0, h.cp.y0, h.cp.x1, h.cp.y1};
  if(decode_slots(e, J, 1, img, &whole, refinement, true, caller, ms_total, &status, nullptr))
    return -1;
  DBG_T("device decode: done");
  return status;
}

/* ---- windows of code streams in device memory (b2k_codestream_parse_window_device / b2k_decode_codestream_window_device)
 * The host reads the main header and derives the virtual coding as b2k_codestream_parse_window does (b2k_window_coding);
 * the device parses the wanted tiles' packets in place from cs against the box coding's plan, then one gather copies only
 * those tiles' packet data into the virtual job's arena.  A window that covers every tile at full resolution is the
 * stream's own coding: the whole-stream path.  Synchronisations: the header, the parse status, the end of the decode. */
struct DeviceWindow
{
  b2k::t2::MainHeader h;
  b2k::t2::WindowCoding wc;
  Rect rect{}; /* the window's pixels at 1 / 2^reduce on the virtual canvas */
};

/* the window's coding of a stream whose main header w.h has been read, and the window's pixels: 0, or the host parser's
   code and text for the window errors */
static int window_coding(const uint32_t* window, uint32_t reduce, DeviceWindow& w)
{
  if(int rc = b2k_window_coding(w.h.cp, window, reduce, w.wc))
    return rc;
  const b2k_coding& v = w.wc.vcp;
  w.rect = Rect{v.x0, v.y0, v.x1, v.y1};
  if(window)
  {
    const uint32_t m = (1u << reduce) - 1u;
    w.rect = Rect{std::max((uint32_t)(((uint64_t)window[0] + m) >> reduce), v.x0), std::max((uint32_t)(((uint64_t)window[1] + m) >> reduce), v.y0),
                  std::min((uint32_t)(((uint64_t)window[2] + m) >> reduce), v.x1), std::min((uint32_t)(((uint64_t)window[3] + m) >> reduce), v.y1)};
  }
  return 0;
}

/* the header and the window's coding, read after the caller's queued work: 0 or the host parser's code and text */
static int device_window_coding(b2k_engine* e, const uint8_t* cs, uint64_t len, const uint32_t* window, uint32_t reduce,
                                cudaStream_t caller, DeviceWindow& w)
{
  if(int rc = read_main_header(e, cs, len, caller, w.h))
    return rc;
  return window_coding(window, reduce, w);
}

/* the windowed parse on e->stream of the streams i < n whose status is 0 (w[i]: their headers and window codings, all with
   w[ref]'s box coding, tile box and flags), read in place, in slots i of J: the five parse kernels and, with dec, the
   arena layout and the decoder's descriptors, then after the statuses the gather of the parsed streams' wanted packet
   data into the arena.  One synchronisation; a stream that fails gets its status and, with `errors`, its text there.
   *refinement: a stream has refinement passes.  0, or -1 for a failure of the call. */
static int parse_windows(b2k_engine* e, b2k_device_job* J, uint32_t n, const uint8_t* const* cs, const uint64_t* len, const DeviceWindow* w,
                         uint32_t ref, uint32_t reduce, bool dec, int32_t* status, std::string* errors, bool* refinement)
{
  cudaStream_t st = e->stream;
  const DeviceWindow& R = w[ref];
  const uint32_t flags = R.h.flags();
  if(!b2k_t2_window_matches(J->t2w, R.wc.box, flags, reduce, J->slots))
  { /* box geometry, progression and reduce: planned once for every window with the same tile box */
    drop_parse(J, J->t2w);
    if(b2k_t2_window_create(R.wc, flags, reduce, J->blocks.data(), J->blocks.size(), J->coded_index.data(), J->coded_index.size(), &J->t2w,
                            J->slots))
      return -1;
  }
  e->last_parse = J->t2w;
  J->arena_sized = false;
  std::vector<uint64_t> sot(n, 0);
  std::vector<const std::vector<Rect>*> need(n, nullptr);
  for(uint32_t i = 0; i < n; ++i)
    if(!status[i])
    {
      sot[i] = w[i].h.sot;
      need[i] = &w[i].wc.need;
    }
  const TileGrid g = tile_grid(R.h.cp);
  const b2k::t2::TileBox box{g.nx, R.wc.ta_x, R.wc.ta_y, R.wc.tb_x, R.wc.tb_y};
  CUDA_TRY(cudaEventRecord(J->ev[0], st));
  if(b2k_t2_window_enqueue(J->t2w, n, cs, len, sot.data(), need.data(), box, g.nx * g.ny, J->d_enc_desc, J->d_dec_quant,
                           dec ? J->d_dec_desc : nullptr, st))
    return -1;
  CUDA_TRY(cudaStreamSynchronize(st));
  bool any = false;
  for(uint32_t i = 0; i < n; ++i)
  {
    if(status[i])
      continue;
    bool r = false;
    if(int prc = b2k_t2_batch_result(J->t2w, i, &r))
    {
      status[i] = prc;
      if(errors)
        errors[i] = g_err;
    }
    any = any || r;
  }
  if(refinement)
    *refinement = any;
  if(!dec)
    return 0;
  const std::string err = g_err; /* a single stream's verdict outlives the gather */
  if(arena_reserve(J, b2k_t2_window_arena(J->t2w), 0)) return -1;
  if(b2k_t2_window_gather(J->t2w, J->d_bytes, st)) return -1;
  g_err = err;
  return 0;
}

/* the windowed parse of one stream in slot 0 of the single-image job of its virtual coding: 0, or the host parser's code
   and text.  *out: the job, once there is one. */
static int parse_device_window(b2k_engine* e, const uint8_t* cs, uint64_t len, const DeviceWindow& w, uint32_t reduce,
                               b2k_device_job** out, bool dec, bool* refinement, uint64_t cap_blocks)
{
  int rc = 0;
  b2k_device_job* J = cached_job(e, &w.wc.vcp, 1, 0, &rc);
  if(rc)
    return rc;
  *out = J;
  if(cap_blocks < J->blocks.size())
  {
    g_err = "block table too small";
    return -1;
  }
  int32_t status = 0;
  if(parse_windows(e, J, 1, &cs, &len, &w, 0, reduce, dec, &status, nullptr, refinement)) return -1;
  return status;
}

/* a windowed parse passed its status: its wanted tiles, and the bytes of the stream its decode copies into the arena (the
   wanted tiles' packet data; the whole stream when every tile is wanted at full resolution) */
static void note_window_stats(b2k_engine* e, const b2k_device_job* J, uint64_t bytes)
{
  e->have_window_stats = true;
  e->window_tiles = J->slot_tiles;
  e->window_bytes = bytes;
}

extern "C" int64_t b2k_codestream_parse_window_device(b2k_engine* e, const uint8_t* cs, uint64_t len, const uint32_t* window,
                                                      uint32_t reduce, void* cuda_stream, b2k_coding* cp_out, b2k_block* blocks,
                                                      uint64_t cap_blocks)
{
  if(!e || !cp_out)
    return -1;
  if(check_device_bytes(e, cs, len))
    return -1;
  std::lock_guard<std::mutex> lock(e->mu);
  cudaStream_t caller = caller_stream(cuda_stream);
  DeviceWindow w;
  if(int rc = device_window_coding(e, cs, len, window, reduce, caller, w))
    return rc;
  if(!blocks)
  {
    *cp_out = w.wc.vcp;
    return b2k_enumerate(&w.wc.vcp, 1, 0, nullptr, 0);
  }
  b2k_device_job* J = nullptr;
  e->have_window_stats = false;
  if(w.wc.whole)
  {
    int rc = parse_single(e, cs, len, w.h, &J, false, nullptr, cap_blocks);
    if(J)
      *cp_out = w.h.cp;
    if(rc)
      return rc;
    note_window_stats(e, J, len);
    if(b2k_t2_parse_blocks(J->t2p, blocks, e->stream))
      return -1;
    return (int64_t)J->blocks.size();
  }
  int rc = parse_device_window(e, cs, len, w, reduce, &J, false, nullptr, cap_blocks);
  if(J)
    *cp_out = w.wc.vcp;
  if(rc)
    return rc;
  note_window_stats(e, J, b2k_t2_window_bytes(J->t2w));
  if(b2k_t2_window_blocks(J->t2w, J->blocks.data(), J->blocks.size(), w.wc.need, blocks, e->stream))
    return -1;
  return (int64_t)J->blocks.size();
}

extern "C" int32_t b2k_decode_codestream_window_device(b2k_engine* e, const uint8_t* cs, uint64_t len, const uint32_t* window,
                                                       uint32_t reduce, const b2k_device_planes* img, void* cuda_stream,
                                                       b2k_coding* cp_out, uint32_t* rect_out, double* ms_total)
{
  if(!e || !cp_out)
    return -1;
  if(check_device_bytes(e, cs, len))
    return -1;
  std::lock_guard<std::mutex> lock(e->mu);
  const auto wall0 = std::chrono::steady_clock::now();
  cudaStream_t caller = caller_stream(cuda_stream);
  DeviceWindow w;
  if(int rc = device_window_coding(e, cs, len, window, reduce, caller, w))
    return rc;
  b2k_device_job* J = nullptr;
  bool refinement = false;
  e->have_window_stats = false;
  int rc = w.wc.whole ? parse_single(e, cs, len, w.h, &J, true, &refinement)
                      : parse_device_window(e, cs, len, w, reduce, &J, true, &refinement, UINT64_MAX);
  if(rc)
    return rc;
  note_window_stats(e, J, w.wc.whole ? len : b2k_t2_window_bytes(J->t2w));
  *cp_out = w.wc.vcp;
  if(rect_out)
  {
    rect_out[0] = w.rect.x0;
    rect_out[1] = w.rect.y0;
    rect_out[2] = w.rect.x1;
    rect_out[3] = w.rect.y1;
  }
  DBG_T("device window decode: parsed");
  if(int crc = check_device_planes(e, &w.wc.vcp, img))
    return crc;
  int32_t status = 0;
  if(decode_slots(e, J, 1, img, &w.rect, refinement, true, caller, ms_total, &status, nullptr))
    return -1;
  DBG_T("device window decode: done");
  return status;
}

extern "C" int32_t b2k_codestream_window_device_stats(b2k_engine* e, uint32_t* tiles_wanted, uint64_t* arena_bytes)
{
  if(!e || !tiles_wanted || !arena_bytes)
    return -1;
  std::lock_guard<std::mutex> lock(e->mu);
  if(!e->have_window_stats)
  {
    g_err = "no windowed code stream parse has been made on the device";
    return -1;
  }
  *tiles_wanted = e->window_tiles;
  *arena_bytes = e->window_bytes;
  return 0;
}

extern "C" int32_t b2k_codestream_parse_device_stats(b2k_engine* e, uint32_t* tiles_indexed, uint32_t* tiles_walked)
{
  if(!e || !tiles_indexed || !tiles_walked)
    return -1;
  std::lock_guard<std::mutex> lock(e->mu);
  if(!e->last_parse)
  {
    g_err = "no code stream has been parsed on the device";
    return -1;
  }
  b2k_t2_parse_stats(e->last_parse, tiles_indexed, tiles_walked);
  return 0;
}

/* ---- batches of code streams in device memory (b2k_decode_codestreams_device) --------------------------------------
 * n streams of one coding go through one launch chain: the batch job holds n images as slots of its planes and
 * descriptors, the parse kernels run over (stream, item), one gather lays the streams out in the arena and one conversion
 * launch per chunk and component group writes the images.  Each stream keeps the single call's checks, in its order, and
 * its verdict; a stream that fails is parsed no further, decodes as all-zero blocks in its own slot and is not written
 * out, so it cannot change another stream's pixels or verdict.  Synchronisations: the header prefixes (one more round for
 * the streams whose header runs past its prefix, all together), the parse statuses, the end. */

/* the batch job of coding cp for n streams: the cached one when its coding matches and it has n slots or more, but not
   more than 4 n (its planes take memory in proportion to its slots: a large batch's job is not kept for small ones) */
static b2k_device_job* cached_batch_job(b2k_engine* e, const b2k_coding& cp, uint32_t n, int* rc)
{
  b2k_device_job*& J = e->batch;
  if(J && (memcmp(&J->cp, &cp, sizeof(b2k_coding)) != 0 || J->slots < n || J->slots > 4ull * n))
  {
    b2k_job_destroy(J);
    J = nullptr;
  }
  *rc = J ? 0 : job_create(e, &cp, 1, 0, n, &J);
  return J;
}

extern "C" int32_t b2k_decode_codestreams_device(b2k_engine* e, uint32_t n, const uint8_t* const* cs, const uint64_t* len,
                                                 const b2k_device_planes* imgs, void* cuda_stream, b2k_coding* cp_out, int32_t* status,
                                                 double* ms_total)
{
  if(!e || !cs || !len || !cp_out || !status)
  {
    g_err = "b2k_decode_codestreams_device: NULL argument";
    return -1;
  }
  if(n == 0)
  {
    g_err = "b2k_decode_codestreams_device: no code streams";
    return -1;
  }
  if(imgs)
    for(uint32_t i = 1; i < n; ++i)
      if(imgs[i].sample_bytes != imgs[0].sample_bytes)
      {
        g_err = "b2k_decode_codestreams_device: the images' sample_bytes differ";
        return -1;
      }
  std::lock_guard<std::mutex> lock(e->mu);
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t caller = caller_stream(cuda_stream), st = e->stream;
  e->batch_errors.assign(n, std::string());
  auto fail = [&](uint32_t i, int32_t rc) {
    status[i] = rc;
    e->batch_errors[i] = g_err;
  };
  auto failures = [&] {
    int32_t f = 0;
    for(uint32_t i = 0; i < n; ++i)
      f += status[i] != 0;
    return f;
  };
  /* each stream's checks in the single call's order: its memory, its main header, the batch's coding */
  for(uint32_t i = 0; i < n; ++i)
  {
    status[i] = 0;
    if(check_device_bytes(e, cs[i], len[i]))
      fail(i, -1);
  }
  /* what the caller queued before the call (the kernels, receives or reads that produced the streams) comes first */
  if(queue_after(e, caller, st)) return -1;
  std::vector<b2k::t2::MainHeader> h(n);
  if(read_batch_headers(e, n, cs, len, b2k::t2::BATCH_HEADER_PREFIX, st, status, h.data(), e->batch_errors.data())) return -1;
  uint32_t ref = n;
  for(uint32_t i = 0; i < n && ref == n; ++i)
    if(!status[i])
      ref = i;
  if(ref == n)
    return failures();
  const b2k_coding cp = h[ref].cp;
  *cp_out = cp;
  for(uint32_t i = ref + 1; i < n; ++i)
    if(!status[i] && b2k_batch_coding_check(h[ref], ref, h[i], i))
      fail(i, 1);
  if(!imgs)
    return failures();
  /* the job of the batch's coding; a coding the engine declines is every such stream's verdict, as in the single call */
  int jrc = 0;
  b2k_device_job* J = cached_batch_job(e, cp, n, &jrc);
  if(jrc < 0)
    return -1;
  if(jrc)
  {
    for(uint32_t i = 0; i < n; ++i)
      if(!status[i])
        fail(i, jrc);
    return failures();
  }
  bool refinement = false;
  if(parse_streams(e, J, n, cs, len, h.data(), h[ref].flags(), true, status, e->batch_errors.data(), &refinement)) return -1;
  /* the image descriptors; a stream whose image is unusable is decoded (its slot is its own) but not written out */
  for(uint32_t i = 0; i < n; ++i)
    if(!status[i])
      if(int rc = check_device_planes(e, &cp, &imgs[i]))
        fail(i, rc);
  /* an image the HT decoder rejected blocks of is not written */
  const std::vector<Rect> whole(n, Rect{cp.x0, cp.y0, cp.x1, cp.y1});
  if(decode_slots(e, J, n, imgs, whole.data(), refinement, false, caller, ms_total, status, e->batch_errors.data()))
    return -1;
  return failures();
}

extern "C" const char* b2k_decode_codestreams_error(b2k_engine* e, uint32_t i)
{
  if(!e)
    return "";
  std::lock_guard<std::mutex> lock(e->mu);
  return i < e->batch_errors.size() ? e->batch_errors[i].c_str() : "";
}

/* ---- windows of batches of code streams in device memory (b2k_decode_codestreams_window_device) ------------------------
 * The batch of b2k_decode_codestreams_device with each stream's window and a shared reduce: the batch job is that of the
 * virtual coding, and the windowed parse runs over (stream, item) in place from the callers' buffers, one gather copying
 * only the wanted tiles' packet data of every stream into the arena.  When the virtual coding is the streams' own (every
 * tile at reduce 0), the batch parse of whole streams runs instead; only the rectangles written out differ. */

extern "C" int32_t b2k_decode_codestreams_window_device(b2k_engine* e, uint32_t n, const uint8_t* const* cs, const uint64_t* len,
                                                        const uint32_t* windows, uint32_t reduce, const b2k_device_planes* imgs,
                                                        void* cuda_stream, b2k_coding* cp_out, uint32_t* rects_out, int32_t* status,
                                                        double* ms_total)
{
  if(!e || !cs || !len || !cp_out || !rects_out || !status)
  {
    g_err = "b2k_decode_codestreams_window_device: NULL argument";
    return -1;
  }
  if(n == 0)
  {
    g_err = "b2k_decode_codestreams_window_device: no code streams";
    return -1;
  }
  if(imgs)
    for(uint32_t i = 1; i < n; ++i)
      if(imgs[i].sample_bytes != imgs[0].sample_bytes)
      {
        g_err = "b2k_decode_codestreams_window_device: the images' sample_bytes differ";
        return -1;
      }
  std::lock_guard<std::mutex> lock(e->mu);
  CUDA_TRY(cudaSetDevice(e->device));
  cudaStream_t caller = caller_stream(cuda_stream), st = e->stream;
  e->batch_errors.assign(n, std::string());
  auto fail = [&](uint32_t i, int32_t rc) {
    status[i] = rc;
    e->batch_errors[i] = g_err;
  };
  auto failures = [&] {
    int32_t f = 0;
    for(uint32_t i = 0; i < n; ++i)
      f += status[i] != 0;
    return f;
  };
  /* each stream's checks in the single call's order: its memory, its main header, its window, the batch's coding */
  for(uint32_t i = 0; i < n; ++i)
  {
    status[i] = 0;
    memset(rects_out + 4 * (size_t)i, 0, 4 * sizeof(uint32_t));
    if(check_device_bytes(e, cs[i], len[i]))
      fail(i, -1);
  }
  if(queue_after(e, caller, st)) return -1;
  std::vector<b2k::t2::MainHeader> h(n);
  if(read_batch_headers(e, n, cs, len, b2k::t2::BATCH_HEADER_PREFIX, st, status, h.data(), e->batch_errors.data())) return -1;
  std::vector<DeviceWindow> w(n);
  uint32_t ref = n;
  for(uint32_t i = 0; i < n; ++i)
  {
    if(status[i])
      continue;
    w[i].h = h[i];
    if(int rc = window_coding(windows ? windows + 4 * (size_t)i : nullptr, reduce, w[i]))
    {
      fail(i, rc);
      continue;
    }
    const Rect& r = w[i].rect;
    const uint32_t q[4] = {r.x0, r.y0, r.x1, r.y1};
    memcpy(rects_out + 4 * (size_t)i, q, sizeof(q));
    if(ref == n)
      ref = i;
    else if(b2k_batch_window_check(w[ref].h, w[ref].wc, ref, w[i].h, w[i].wc, i))
      fail(i, 1);
  }
  if(ref == n)
    return failures();
  const b2k_coding cp = w[ref].wc.vcp;
  *cp_out = cp;
  if(!imgs)
    return failures();
  int jrc = 0;
  b2k_device_job* J = cached_batch_job(e, cp, n, &jrc);
  if(jrc < 0)
    return -1;
  if(jrc)
  {
    for(uint32_t i = 0; i < n; ++i)
      if(!status[i])
        fail(i, jrc);
    return failures();
  }
  e->have_window_stats = false;
  bool refinement = false;
  const bool whole = w[ref].wc.whole;
  if(whole ? parse_streams(e, J, n, cs, len, h.data(), h[ref].flags(), true, status, e->batch_errors.data(), &refinement)
           : parse_windows(e, J, n, cs, len, w.data(), ref, reduce, true, status, e->batch_errors.data(), &refinement))
    return -1;
  uint64_t bytes = 0;
  for(uint32_t i = 0; i < n && whole; ++i)
    bytes += status[i] ? 0 : len[i];
  note_window_stats(e, J, whole ? bytes : b2k_t2_window_bytes(J->t2w));
  std::vector<Rect> rects(n);
  for(uint32_t i = 0; i < n; ++i)
  {
    rects[i] = w[i].rect;
    if(!status[i])
      if(int rc = check_device_planes(e, &cp, &imgs[i]))
        fail(i, rc);
  }
  if(decode_slots(e, J, n, imgs, rects.data(), refinement, false, caller, ms_total, status, e->batch_errors.data()))
    return -1;
  return failures();
}

/* ---- images in device memory to code streams (b2k_encode_codestream_device / b2k_encode_codestreams_device) -----------
 * n images of one coding become n code streams in one launch chain.  The images that pass their checks take slots
 * 0..m-1 of the batch job, in image order; chunk by chunk over the (slot, tile) ranges, one conversion launch per
 * component group brings the images whose first tile the chunk holds into their planes, then the forward transform and
 * the block coder run over the chunk.  The device writer (t2_device.cu) then writes the m streams behind each other.
 * A failed image takes no slot, so none of its samples is coded.  A stream the coder or the writer gives a verdict is
 * neither placed nor gathered, and the other streams' places depend only on their own lengths: no image can change
 * another stream's bytes.  A single image is a batch of one in the engine's single-image job, written into its own
 * buffer.  Synchronisations: one, and a second when the output buffer has to grow. */

/* the images imgs[image_of[s]], which passed check_device_planes, in slots s of J, after the work queued on `caller`:
   coded and written as code streams with `flags` into buf[0, cap), which grows as they need.  Image i's stream is
   buf[offset[i], offset[i] + length[i]) when its status[i] stays 0; a stream the coder or writer gives a verdict gets
   that status and, with `errors`, its text there.  0; 1 when the writer declines the flags (b2k_last_error says why, no
   status is set); -1 for a failure of the call. */
static int encode_images(b2k_engine* e, b2k_device_job* J, const b2k_device_planes* imgs, const std::vector<uint32_t>& image_of,
                         uint32_t flags, cudaStream_t caller, uint8_t*& buf, uint64_t& cap, int32_t* status, uint64_t* offset,
                         uint64_t* length, std::string* errors, double* ms_total)
{
  const b2k_coding& cp = J->cp;
  cudaStream_t st = e->stream;
  const uint32_t m = (uint32_t)image_of.size();
  if(!J->t2 || b2k_t2_flags(J->t2) != flags || b2k_t2_streams(J->t2) != J->slots)
  { /* geometry and flags only: planned once for every image or batch of this coding */
    b2k_t2_destroy(J->t2);
    J->t2 = nullptr;
    if(int trc = b2k_t2_create(cp, flags, J->blocks.data(), J->blocks.size(), J->slot_tiles, J->coded_index.data(),
                               J->coded_index.size(), &J->t2, J->slots))
      return trc < 0 ? -1 : 1;
  }
  /* the conversion's tables: one per component, or one for all when every image is pixel-interleaved */
  const int nc = cp.numcomps;
  bool interleaved = nc > 1;
  for(uint32_t i : image_of)
    interleaved = interleaved && device_group(imgs[i], nc) == nc;
  const int group = interleaved ? nc : 1, tables = nc / group;
  if(!J->h_batch_src)
  {
    CUDA_TRY(cudaMalloc(&J->d_batch_src, (size_t)J->slots * 4 * sizeof(BatchSrc)));
    CUDA_TRY(cudaHostAlloc(&J->h_batch_src, (size_t)J->slots * 4 * sizeof(BatchSrc), cudaHostAllocDefault));
  }
  for(int t = 0; t < tables; ++t)
    for(uint32_t s = 0; s < m; ++s)
    {
      const b2k_device_planes& img = imgs[image_of[s]];
      const int c0 = t * group;
      BatchSrc& E = J->h_batch_src[(size_t)t * m + s];
      E = BatchSrc{};
      E.src = img.comp[c0];
      E.spitch = img.row_pitch[c0];
      E.step = img.col_step[c0];
      E.dst = J->img.at((int)s * nc + c0, cp.x0, cp.y0);
    }
  /* what the caller queued before the call (the kernels that made the images) comes first */
  if(queue_after(e, caller, st)) return -1;
  CUDA_TRY(cudaEventRecord(J->ev[0], st));
  CUDA_TRY(cudaMemcpyAsync(J->d_batch_src, J->h_batch_src, (size_t)tables * m * sizeof(BatchSrc), cudaMemcpyHostToDevice, st));
  /* conversion -> forward transform -> block coder, chunk by chunk over the (slot, tile) ranges of the m slots used (as
     many chunks as the job's pipeline has, whatever its slot count); an image is converted in the chunk of its first tile */
  const size_t T = J->slot_tiles, used = (size_t)m * T;
  const size_t nchunks = std::min<size_t>(J->chunk_tile.size() - 1, used);
  const uint32_t w = cp.x1 - cp.x0, hgt = cp.y1 - cp.y0, sb = imgs[image_of[0]].sample_bytes;
  for(size_t k = 0; k < nchunks; ++k)
  {
    const size_t t0 = k * used / nchunks, t1 = (k + 1) * used / nchunks;
    if(t1 <= t0)
      continue;
    const uint32_t s0 = (uint32_t)((t0 + T - 1) / T), s1 = (uint32_t)((t1 + T - 1) / T);
    for(int t = 0; t < tables && s1 > s0; ++t)
      b2k_launch_containers_to_planes(J->d_batch_src + (size_t)t * m + s0, s1 - s0, group, J->img.pitch, J->img.plane_elems(), sb, w,
                                      hgt, cp.sgnd, st);
    if(enqueue_forward(J, st, false, t0, t1)) return -1;
    if(enqueue_t1_blocks(J, st, t0, t1)) return -1;
  }
  CUDA_TRY(cudaGetLastError());
  /* the caller's stream goes on once every image has been read */
  if(queue_after(e, st, caller)) return -1;
  /* the m code streams into buf; the call's one synchronisation reads their statuses and places */
  for(;;)
  {
    if(b2k_t2_enqueue(J->t2, J->d_enc_desc, J->d_out, J->d_scratch, buf, cap, st, m))
      return -1;
    CUDA_TRY(cudaEventRecord(J->ev[1], st));
    CUDA_TRY(cudaEventSynchronize(J->ev[1]));
    const uint64_t need = b2k_t2_used(J->t2);
    if(need <= cap)
      break;
    cudaFree(buf);
    buf = nullptr;
    cap = 0;
    CUDA_TRY(cudaMalloc(&buf, need + need / 8 + 4096));
    cap = need + need / 8 + 4096;
  }
  float t = 0;
  cudaEventElapsedTime(&t, J->ev[0], J->ev[1]);
  if(ms_total) *ms_total = t;
  for(uint32_t s = 0; s < m; ++s)
  {
    const uint32_t i = image_of[s];
    const int64_t r = b2k_t2_result(J->t2, s);
    if(r < 0)
    {
      status[i] = (int32_t)r;
      if(errors)
        errors[i] = g_err;
    }
    else
    {
      offset[i] = b2k_t2_offset(J->t2, s);
      length[i] = (uint64_t)r;
    }
  }
  return 0;
}

extern "C" int64_t b2k_encode_codestream_device(b2k_engine* e, const b2k_coding* cp, const b2k_device_planes* img, uint32_t flags,
                                                void* cuda_stream, const uint8_t** cs)
{
  if(!e || !cp || !cs)
    return -1;
  if(int rc = check_device_planes(e, cp, img))
    return rc;
  std::lock_guard<std::mutex> lock(e->mu);
  int rc = 0;
  b2k_device_job* J = cached_job(e, cp, 1, 0, &rc);
  if(rc)
    return rc;
  CUDA_TRY(cudaSetDevice(e->device));
  int32_t status = 0;
  uint64_t offset = 0, length = 0;
  if(encode_images(e, J, img, {0}, flags, caller_stream(cuda_stream), e->d_cs, e->cs_cap, &status, &offset, &length, nullptr, nullptr))
    return -1;
  if(status)
    return status;
  *cs = e->d_cs;
  return (int64_t)length;
}

extern "C" int32_t b2k_encode_codestreams_device(b2k_engine* e, const b2k_coding* cp, uint32_t n, const b2k_device_planes* imgs,
                                                 uint32_t flags, void* cuda_stream, const uint8_t** cs, uint64_t* offset,
                                                 uint64_t* length, int32_t* status, double* ms_total)
{
  if(!e || !cp || !imgs || !cs || !offset || !length || !status)
  {
    g_err = "b2k_encode_codestreams_device: NULL argument";
    return -1;
  }
  if(n == 0)
  {
    g_err = "b2k_encode_codestreams_device: no images";
    return -1;
  }
  for(uint32_t i = 1; i < n; ++i)
    if(imgs[i].sample_bytes != imgs[0].sample_bytes)
    {
      g_err = "b2k_encode_codestreams_device: the images' sample_bytes differ";
      return -1;
    }
  std::lock_guard<std::mutex> lock(e->mu);
  CUDA_TRY(cudaSetDevice(e->device));
  e->enc_batch_errors.assign(n, std::string());
  *cs = nullptr;
  auto fail = [&](uint32_t i, int32_t rc) {
    status[i] = rc;
    e->enc_batch_errors[i] = g_err;
  };
  auto failures = [&] {
    int32_t f = 0;
    for(uint32_t i = 0; i < n; ++i)
      f += status[i] != 0;
    return f;
  };
  /* each image's descriptor, as the single call checks it first; the images that pass take the slots in order */
  std::vector<uint32_t> image_of;
  for(uint32_t i = 0; i < n; ++i)
  {
    status[i] = 0;
    offset[i] = length[i] = 0;
    if(int rc = check_device_planes(e, cp, &imgs[i]))
      fail(i, rc);
    else
      image_of.push_back(i);
  }
  const uint32_t m = (uint32_t)image_of.size();
  if(!m)
    return failures();
  /* a verdict of the coding or the flags alone is every remaining image's, as in the single call */
  auto fail_all = [&](int32_t rc) {
    for(uint32_t i : image_of)
      fail(i, rc);
    return failures();
  };
  int jrc = 0;
  b2k_device_job* J = cached_batch_job(e, *cp, m, &jrc);
  if(jrc < 0)
    return -1;
  if(jrc)
    return fail_all(jrc);
  const int rc = encode_images(e, J, imgs, image_of, flags, caller_stream(cuda_stream), e->d_bcs, e->bcs_cap, status, offset, length,
                               e->enc_batch_errors.data(), ms_total);
  if(rc < 0)
    return -1;
  if(rc)
    return fail_all(-1);
  *cs = e->d_bcs;
  return failures();
}

extern "C" const char* b2k_encode_codestreams_error(b2k_engine* e, uint32_t i)
{
  if(!e)
    return "";
  std::lock_guard<std::mutex> lock(e->mu);
  return i < e->enc_batch_errors.size() ? e->enc_batch_errors[i].c_str() : "";
}
