/*
 * grok_b200/csrc/t2_decode.cu -- T2 parse on the device: a code stream in device memory becomes the block table and the
 * HT decoder's descriptors, with no byte of it crossing PCIe.  The host reads the main header (b2k_parse_main_header) and
 * builds the packet plan once per coding and progression (b2k_t2_plan, the writer's own, one tile part per tile); then
 * five launches per call, however many tiles:
 *   1. k_t2_locate   one thread: the host parser's SOT walk (Psot hops, tile-part header segments up to SOD), in stream
 *                    order, into a table of tile parts chained per tile.  The first failure in stream order is the verdict.
 *   2. k_t2_plt      a thread per tile: clears the tile's blocks; decodes the Iplt entries of its tile parts into packet
 *                    starts.  The tile is indexed when they account for exactly its packets and its packet data.
 *   3. k_t2_packets  a thread per packet of an indexed tile: its header parsed at its PLT start, its body laid out; any
 *                    anomaly (a header error, an end other than PLT's) marks the tile instead of failing the call.
 *   4. k_t2_walk     a thread per tile that is not indexed or is marked: the tile's packets over its tile parts in order,
 *                    with the host's parse_tile_packets semantics.  Its verdict is final, so PLT changes only the speed:
 *                    an indexed, unmarked tile is one whose every packet the walk would have met at its PLT start and
 *                    parsed exactly as kernel 3 did.  The lowest failing tile's reason is kept.
 *   5. k_t2_desc     a thread per coded block: prepare_decode's rule into the decoder's descriptors; whether any block
 *                    has refinement passes.
 * Tag trees live in global scratch sized by the plan (packet_tag_nodes per packet, so every packet has its own); a walking
 * thread reuses its tile's share for every packet of the tile.
 *
 * A windowed parse runs the same five launches against the plan of the box coding (the wanted tiles at full resolution,
 * whose packets are those of the stream's tiles), reading cs in place: k_t2_locate checks every SOT but reads and records
 * only the wanted tiles' parts, under their box index, and lays their packet data end to end; k_t2_desc maps each coded
 * block of the virtual coding to its box block, leaves the blocks outside the window's need rectangles uncoded and points
 * the descriptors into that layout.  After the status read, k_t2_gather copies just those bytes into the job's arena.
 */
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "b2k_internal.h"
#include "t2_packet.h"
#include "t2_plan.h"
#include "t2_parse.h"
#include "t2_decode.h"
#include "geometry.h"

using namespace b2k;
using namespace b2k::t2;
static_assert(WINDOW_MAX_RES == B2K_MAX_RES, "a need rectangle per resolution");

void b2k_set_error(const char* msg); /* engine.cu */

namespace
{
/* Every kernel runs over the n streams of a batch (n = 1 for a single stream), one thread per item; the threads' bodies
   are t2_parse.h's batch_* functions, which tests/t2_batch_check.cpp runs on the host */
__global__ void k_t2_locate(const uint8_t* __restrict__ cs, const StreamDesc* __restrict__ sd, uint32_t n, uint32_t ntiles, TileBox box,
                            PartRange* __restrict__ parts, uint32_t* __restrict__ head, uint32_t* __restrict__ last,
                            uint32_t* __restrict__ count, uint64_t* __restrict__ body_at, ParseStatus* status)
{
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if(s < n)
    batch_locate(cs, sd, s, ntiles, box, parts, head, last, count, body_at, status);
}

__global__ void k_t2_plt(const uint8_t* __restrict__ cs, const StreamDesc* __restrict__ sd, uint32_t n, const PartRange* __restrict__ parts,
                         const uint32_t* __restrict__ head, const DevPart* __restrict__ tiles, uint32_t ntiles,
                         const uint64_t* __restrict__ tile_first, uint64_t nblocks, uint64_t np, ParsedBlock* __restrict__ blk,
                         uint64_t* __restrict__ start, uint64_t* __restrict__ end, uint64_t* __restrict__ part_end,
                         uint32_t* __restrict__ indexed, uint32_t* __restrict__ marked, ParseStatus* status)
{
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(g < (uint64_t)n * ntiles)
    batch_plt(cs, sd, g, parts, head, tiles, ntiles, tile_first, nblocks, np, blk, start, end, part_end, indexed, marked, status);
}

__global__ void k_t2_packets(const uint8_t* __restrict__ cs, const StreamDesc* __restrict__ sd, uint32_t n,
                             const DevPacket* __restrict__ packets, uint64_t np, const uint32_t* __restrict__ pkt_tile, uint32_t ntiles,
                             uint64_t nblocks, uint64_t tag_nodes, const uint32_t* __restrict__ indexed,
                             const uint64_t* __restrict__ start, const uint64_t* __restrict__ end, const uint64_t* __restrict__ part_end,
                             const uint8_t* __restrict__ kmax, ParsedBlock* __restrict__ blk, TagNode* __restrict__ tags,
                             uint32_t* __restrict__ marked, bool sop, bool eph, const ParseStatus* status)
{
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(g < n * np)
    batch_packet(cs, sd, g, packets, np, pkt_tile, ntiles, nblocks, tag_nodes, indexed, start, end, part_end, kmax, blk, tags, marked, sop,
                 eph, status);
}

__global__ void k_t2_walk(const uint8_t* __restrict__ cs, const StreamDesc* __restrict__ sd, uint32_t n, const PartRange* __restrict__ parts,
                          const uint32_t* __restrict__ head, const DevPart* __restrict__ tiles, uint32_t ntiles,
                          const DevPacket* __restrict__ packets, const uint8_t* __restrict__ kmax, const uint64_t* __restrict__ tile_first,
                          uint64_t nblocks, uint64_t tag_nodes, ParsedBlock* __restrict__ blk, TagNode* __restrict__ tags,
                          const uint32_t* __restrict__ indexed, const uint32_t* __restrict__ marked, bool sop, bool eph,
                          ParseStatus* status)
{
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(g < (uint64_t)n * ntiles)
    batch_walk(cs, sd, g, parts, head, tiles, ntiles, packets, kmax, tile_first, nblocks, tag_nodes, blk, tags, indexed, marked, sop, eph,
               status);
}

/* a thread per (stream, coded block): descriptor s * ncoded + k from template enc[s * ncoded + k], pointing into the arena.
   A stream whose parse failed (or was skipped) gets length-0 descriptors, which decode as all-zero blocks.  win != NULL (a
   windowed batch): t2_parse.h's window_block, the need filter and the address of the block's gathered bytes */
__global__ void k_t2_desc(const StreamDesc* __restrict__ sd, uint32_t n, const ParsedBlock* __restrict__ blk, uint64_t nblocks,
                          const uint32_t* __restrict__ coded, uint32_t ncoded, const HtBlockDesc* __restrict__ enc,
                          const float* __restrict__ quant, HtBlockDesc* __restrict__ dec, const WinBlock* __restrict__ win,
                          const NeedRects* __restrict__ need, const PartRange* __restrict__ parts, const uint32_t* __restrict__ head,
                          uint32_t bt, const uint64_t* __restrict__ body_at, ParseStatus* status)
{
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(g >= (uint64_t)n * ncoded)
    return;
  uint32_t s = 0;
  uint64_t slot_off = 0;
  ParsedBlock b;
  if(win)
    b = window_block(blk, nblocks, coded, g, ncoded, status, sd, win, need, parts, head, bt, body_at, &s, &slot_off);
  else
  {
    b = batch_block(blk, nblocks, coded, g, ncoded, status, &s);
    slot_off = sd[s].at + b.offset;
  }
  HtBlockDesc d = enc[g];
  d.length = b.length;
  d.slot_off = slot_off;
  block_decode_fields(b, d.kmax, &d.mmsbs, &d.passes, &d.length2);
  d.quant = quant[g]; /* stepsize / 2^(31-Kmax) */
  dec[g] = d;
  if(d.passes > 1)
    status[s].refinement = 1;
}

/* a windowed batch's arena layout, one CTA: sd[s].at for every stream (window_arena_at), each thread a run of streams
   whose start is the scan of the runs before it */
__global__ void __launch_bounds__(1024) k_t2_window_at(StreamDesc* __restrict__ sd, const ParseStatus* __restrict__ status, uint32_t n)
{
  __shared__ uint64_t sum[1024];
  const uint32_t per = (n + 1023) / 1024, s0 = min(n, threadIdx.x * per), s1 = min(n, s0 + per);
  uint64_t mine = 0;
  for(uint32_t s = s0; s < s1; ++s)
    mine += window_gathered_bytes(status[s]);
  sum[threadIdx.x] = mine;
  __syncthreads();
  for(uint32_t d = 1; d < 1024; d <<= 1)
  {
    const uint64_t v = threadIdx.x >= d ? sum[threadIdx.x - d] : 0;
    __syncthreads();
    sum[threadIdx.x] += v;
    __syncthreads();
  }
  window_arena_at(sd, status, s0, s1, sum[threadIdx.x] - mine);
}

/* one copy per entry of a (source, length, destination) table: entry e (blockIdx.y strided) by a strip of CTAs along x;
   16 bytes per thread and step where source and destination are both 16-byte aligned (the arena's streams start on
   256-byte boundaries, and CUDA allocations on 256-byte ones), the bytes after the last whole 16 one by one */
__global__ void k_copy_table(const CopyEntry* __restrict__ tab, uint32_t n, uint8_t* __restrict__ out)
{
  const uint64_t first = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (uint64_t)gridDim.x * blockDim.x;
  for(uint32_t e = blockIdx.y; e < n; e += gridDim.y)
  {
    const CopyEntry E = tab[e];
    uint8_t* dst = out + E.dst;
    uint64_t done = 0;
    if(((reinterpret_cast<uintptr_t>(E.src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0)
    {
      const uint64_t v = E.len / 16;
      const uint4* s4 = reinterpret_cast<const uint4*>(E.src);
      uint4* d4 = reinterpret_cast<uint4*>(dst);
      for(uint64_t i = first; i < v; i += stride)
        d4[i] = s4[i];
      done = v * 16;
    }
    for(uint64_t i = done + first; i < E.len; i += stride)
      dst[i] = E.src[i];
  }
}

/* a windowed batch's gather: item g (blockIdx.y strided) of window_gather_part, over (stream, part), by a strip of CTAs
   along x */
__global__ void k_t2_gather(const StreamDesc* __restrict__ sd, const PartRange* __restrict__ parts, const uint64_t* __restrict__ body_at,
                            const ParseStatus* __restrict__ status, uint64_t items, uint64_t per, uint8_t* __restrict__ out)
{
  for(uint64_t g = blockIdx.y; g < items; g += gridDim.y)
  {
    const uint8_t* src = nullptr;
    uint64_t dst = 0, len = 0;
    if(!window_gather_part(sd, parts, body_at, status, g, per, &src, &dst, &len))
      continue;
    for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < len; i += (uint64_t)gridDim.x * blockDim.x)
      out[dst + i] = src[i];
  }
}

template <class T>
T* carve(uint8_t*& p, uint64_t n)
{
  T* r = reinterpret_cast<T*>(p);
  p += (n * sizeof(T) + 255) & ~(uint64_t)255;
  return r;
}
} // namespace

struct T2Parse
{
  Plan plan;
  uint32_t flags = 0, ntiles = 0;
  uint64_t nblocks = 0, ncoded = 0;
  uint32_t streams = 1;            /* stream capacity: the per-stream slices below are allocated for this many */
  uint32_t last_n = 1;             /* streams of the last enqueue */
  std::vector<b2k_block> blocks; /* the enumeration, into which the parsed fields are merged */
  uint8_t* d_mem = nullptr;
  DevPacket* d_packets = nullptr;
  DevPart* d_tiles = nullptr;
  uint8_t* d_kmax = nullptr;
  uint64_t* d_tile_first = nullptr;
  uint32_t* d_coded = nullptr;
  /* per stream (slice s of `streams`) */
  TagNode* d_tags = nullptr;
  ParsedBlock* d_blk = nullptr;
  uint32_t *d_head = nullptr, *d_last = nullptr, *d_count = nullptr;
  uint32_t *d_pkt_tile = nullptr, *d_indexed = nullptr, *d_marked = nullptr;
  uint64_t *d_start = nullptr, *d_end = nullptr, *d_part_end = nullptr; /* per packet, from PLT */
  ParseStatus* d_status = nullptr; /* streams statuses, then streams StreamDescs: one upload */
  StreamDesc* d_sd = nullptr;
  ParseStatus* h_status = nullptr; /* pinned, the same layout */
  StreamDesc* h_sd = nullptr;
  PartRange* d_parts = nullptr;    /* grown with the code streams' lengths */
  uint64_t parts_cap = 0;
  /* a windowed parse: the plan is the box coding's; coded block k of the virtual coding is box block d_coded[k] */
  bool window = false;
  b2k_coding box{};
  uint32_t reduce = 0;
  std::vector<uint32_t> vmap;      /* every virtual block -> its box block */
  WinBlock* d_win = nullptr;
  NeedRects* d_need = nullptr;     /* per stream */
  NeedRects* h_need = nullptr;     /* pinned */
  uint64_t* d_body_at = nullptr;   /* per recorded part, parts_cap of them */
  uint32_t* d_wcount = nullptr;    /* tile parts seen per stream tile, per stream */
  uint64_t wcount_cap = 0;
};

#define T2P_TRY(expr)                                                                                                          \
  do                                                                                                                           \
  {                                                                                                                            \
    cudaError_t _e = (expr);                                                                                                   \
    if(_e != cudaSuccess)                                                                                                      \
    {                                                                                                                          \
      b2k_set_error((std::string(#expr) + ": " + cudaGetErrorString(_e)).c_str());                                            \
      return -1;                                                                                                               \
    }                                                                                                                          \
  } while(0)

int b2k_t2_parse_create(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles,
                        const uint32_t* coded_index, uint64_t ncoded, T2Parse** out, uint32_t streams)
{
  *out = nullptr;
  T2Parse* J = new T2Parse();
  struct Guard
  {
    T2Parse*& j;
    ~Guard() { b2k_t2_parse_destroy(j); }
  } guard{J};
  /* the writer's plan with one tile part per tile: plan.parts[t] holds tile t's packets in code-stream order */
  if(b2k_t2_plan(cp, flags & ~(uint32_t)(B2K_CS_TPARTS_R | B2K_CS_TLM), blocks, nblocks, num_tiles, J->plan))
    return -1;
  const Plan& P = J->plan;
  if(P.parts.size() != num_tiles)
  {
    b2k_set_error("internal: the parse plan does not hold one tile part per tile");
    return -1;
  }
  J->flags = flags;
  J->ntiles = num_tiles;
  J->nblocks = nblocks;
  J->ncoded = ncoded;
  J->streams = streams = std::max(streams, 1u);
  J->blocks.assign(blocks, blocks + nblocks);
  std::vector<uint8_t> kmax(nblocks);
  std::vector<uint64_t> tile_first(num_tiles + 1, nblocks);
  for(uint64_t i = nblocks; i-- > 0;)
  {
    kmax[i] = blocks[i].kmax;
    tile_first[blocks[i].tile] = i;
  }
  for(uint32_t t = num_tiles; t-- > 0;) /* a tile without blocks starts where the next one does */
    tile_first[t] = std::min(tile_first[t], tile_first[t + 1]);
  const uint64_t np = P.packets.size(), S = streams;
  auto bytes = [](uint64_t n, size_t sz) { return (n * sz + 255) & ~(uint64_t)255; };
  const uint64_t total = bytes(np, sizeof(DevPacket)) + bytes(num_tiles, sizeof(DevPart)) + bytes(nblocks, 1) +
                         bytes(num_tiles + 1, sizeof(uint64_t)) + bytes(ncoded, sizeof(uint32_t)) + bytes(S * P.tag_nodes, sizeof(TagNode)) +
                         bytes(S * nblocks, sizeof(ParsedBlock)) + 5 * bytes(S * num_tiles, sizeof(uint32_t)) + bytes(np, sizeof(uint32_t)) +
                         3 * bytes(S * np, sizeof(uint64_t)) + bytes(S, sizeof(ParseStatus) + sizeof(StreamDesc));
  T2P_TRY(cudaMalloc(&J->d_mem, total));
  uint8_t* p = J->d_mem;
  J->d_packets = carve<DevPacket>(p, np);
  J->d_tiles = carve<DevPart>(p, num_tiles);
  J->d_kmax = carve<uint8_t>(p, nblocks);
  J->d_tile_first = carve<uint64_t>(p, num_tiles + 1);
  J->d_coded = carve<uint32_t>(p, ncoded);
  J->d_tags = carve<TagNode>(p, S * P.tag_nodes);
  J->d_blk = carve<ParsedBlock>(p, S * nblocks);
  J->d_head = carve<uint32_t>(p, S * num_tiles);
  J->d_last = carve<uint32_t>(p, S * num_tiles);
  J->d_count = carve<uint32_t>(p, S * num_tiles);
  J->d_indexed = carve<uint32_t>(p, S * num_tiles);
  J->d_marked = carve<uint32_t>(p, S * num_tiles);
  J->d_pkt_tile = carve<uint32_t>(p, np);
  J->d_start = carve<uint64_t>(p, S * np);
  J->d_end = carve<uint64_t>(p, S * np);
  J->d_part_end = carve<uint64_t>(p, S * np);
  J->d_status = reinterpret_cast<ParseStatus*>(p);
  J->d_sd = reinterpret_cast<StreamDesc*>(J->d_status + S);
  T2P_TRY(cudaMemcpy(J->d_packets, P.packets.data(), np * sizeof(DevPacket), cudaMemcpyHostToDevice));
  T2P_TRY(cudaMemcpy(J->d_tiles, P.parts.data(), num_tiles * sizeof(DevPart), cudaMemcpyHostToDevice));
  T2P_TRY(cudaMemcpy(J->d_kmax, kmax.data(), nblocks, cudaMemcpyHostToDevice));
  T2P_TRY(cudaMemcpy(J->d_tile_first, tile_first.data(), (num_tiles + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice));
  T2P_TRY(cudaMemcpy(J->d_coded, coded_index, ncoded * sizeof(uint32_t), cudaMemcpyHostToDevice));
  std::vector<uint32_t> pkt_tile(np);
  for(uint32_t t = 0; t < num_tiles; ++t)
    for(uint64_t k = P.parts[t].p0; k < P.parts[t].p1; ++k)
      pkt_tile[k] = t;
  T2P_TRY(cudaMemcpy(J->d_pkt_tile, pkt_tile.data(), np * sizeof(uint32_t), cudaMemcpyHostToDevice));
  T2P_TRY(cudaHostAlloc(&J->h_status, S * (sizeof(ParseStatus) + sizeof(StreamDesc)), cudaHostAllocDefault));
  J->h_sd = reinterpret_cast<StreamDesc*>(J->h_status + S);
  *out = J;
  guard.j = nullptr;
  return 0;
}

int b2k_t2_window_create(const b2k::t2::WindowCoding& wc, uint32_t flags, uint32_t reduce, const b2k_block* vblocks, uint64_t nv,
                         const uint32_t* coded_index, uint64_t ncoded, T2Parse** out, uint32_t streams)
{
  *out = nullptr;
  std::vector<b2k_block> box_blocks;
  std::vector<uint32_t> vmap;
  if(b2k_window_blocks(wc, vblocks, nv, box_blocks, vmap))
    return -1;
  const TileGrid bg = tile_grid(wc.box);
  std::vector<uint32_t> coded_box(ncoded);
  std::vector<WinBlock> win(ncoded);
  for(uint64_t k = 0; k < ncoded; ++k)
  {
    const b2k_block& v = vblocks[coded_index[k]];
    coded_box[k] = vmap[coded_index[k]];
    win[k] = WinBlock{v.tile, v.resno ? v.resno - 1u : 0u, v.x0, v.y0, v.x1, v.y1};
  }
  T2Parse* J = nullptr;
  if(b2k_t2_parse_create(wc.box, flags, box_blocks.data(), box_blocks.size(), bg.nx * bg.ny, coded_box.data(), ncoded, &J, streams))
    return -1;
  struct Guard
  {
    T2Parse*& j;
    ~Guard() { b2k_t2_parse_destroy(j); }
  } guard{J};
  J->window = true;
  J->box = wc.box;
  J->reduce = reduce;
  J->vmap.swap(vmap);
  T2P_TRY(cudaMalloc(&J->d_win, std::max<uint64_t>(ncoded, 1) * sizeof(WinBlock) + J->streams * sizeof(NeedRects)));
  J->d_need = reinterpret_cast<NeedRects*>(J->d_win + std::max<uint64_t>(ncoded, 1));
  T2P_TRY(cudaMemcpy(J->d_win, win.data(), ncoded * sizeof(WinBlock), cudaMemcpyHostToDevice));
  T2P_TRY(cudaHostAlloc(&J->h_need, J->streams * sizeof(NeedRects), cudaHostAllocDefault));
  *out = J;
  J = nullptr;
  return 0;
}

bool b2k_t2_window_matches(const T2Parse* J, const b2k_coding& box, uint32_t flags, uint32_t reduce, uint32_t streams)
{
  return J && J->window && J->flags == flags && J->reduce == reduce && J->streams == streams && memcmp(&J->box, &box, sizeof(box)) == 0;
}

void b2k_t2_parse_destroy(T2Parse* J)
{
  if(!J)
    return;
  cudaFree(J->d_mem);
  cudaFree(J->d_parts);
  cudaFree(J->d_body_at);
  cudaFree(J->d_win);
  cudaFree(J->d_wcount);
  cudaFreeHost(J->h_status);
  cudaFreeHost(J->h_need);
  delete J;
}

uint32_t b2k_t2_parse_flags(const T2Parse* J) { return J->flags; }

/* the five launches over the plan's tiles, which are the tiles of `box` among each stream's ntiles, for the n streams whose
   h_sd[s].at / len / sot / base the caller filled in (sot = 0: not parsed); the part table is laid out here.  A windowed
   batch lays its arena out on the device (k_t2_window_at) before the descriptors point into it */
static int enqueue_parse(T2Parse* J, const uint8_t* cs, uint32_t n, uint32_t ntiles, const TileBox& box, uint32_t* d_count,
                         const HtBlockDesc* d_enc, const float* d_quant, HtBlockDesc* d_dec, cudaStream_t st)
{
  uint64_t need = 0;
  for(uint32_t s = 0; s < n; ++s)
  {
    StreamDesc& D = J->h_sd[s];
    D.parts0 = need;
    D.parts_cap = D.sot ? part_capacity(D.len, J->ntiles) : 0;
    need += D.parts_cap;
  }
  if(need > J->parts_cap)
  {
    cudaFree(J->d_parts);
    cudaFree(J->d_body_at);
    J->d_parts = nullptr;
    J->d_body_at = nullptr;
    J->parts_cap = 0;
    const uint64_t cap = need + need / 4 + 16;
    T2P_TRY(cudaMalloc(&J->d_parts, cap * sizeof(PartRange)));
    if(J->window)
      T2P_TRY(cudaMalloc(&J->d_body_at, cap * sizeof(uint64_t)));
    J->parts_cap = cap;
  }
  for(uint32_t s = 0; s < n; ++s)
    J->h_status[s] = ParseStatus{NO_TILE_ERROR, J->h_sd[s].sot ? (uint32_t)PR_NONE : (uint32_t)PR_SKIPPED, 0, 0, 0, 0, 0};
  J->last_n = n;
  const uint64_t S = J->streams;
  /* statuses and stream table in one copy */
  T2P_TRY(cudaMemcpyAsync(J->d_status, J->h_status, S * sizeof(ParseStatus) + n * sizeof(StreamDesc), cudaMemcpyHostToDevice, st));
  if(J->window)
    T2P_TRY(cudaMemcpyAsync(J->d_need, J->h_need, n * sizeof(NeedRects), cudaMemcpyHostToDevice, st));
  const uint32_t tpb = 32; /* streams, tiles and packets are few and each thread is a long serial chain: spread them over the SMs */
  auto grid = [&](uint64_t items) { return (unsigned)((items + tpb - 1) / tpb); };
  k_t2_locate<<<grid(n), tpb, 0, st>>>(cs, J->d_sd, n, ntiles, box, J->d_parts, J->d_head, J->d_last, d_count, J->d_body_at, J->d_status);
  b2k_count_launch();
  const bool sop = (J->flags & B2K_CS_SOP) != 0, eph = (J->flags & B2K_CS_EPH) != 0;
  const uint64_t np = J->plan.packets.size(), tags = J->plan.tag_nodes;
  k_t2_plt<<<grid((uint64_t)n * J->ntiles), tpb, 0, st>>>(cs, J->d_sd, n, J->d_parts, J->d_head, J->d_tiles, J->ntiles, J->d_tile_first,
                                                          J->nblocks, np, J->d_blk, J->d_start, J->d_end, J->d_part_end, J->d_indexed,
                                                          J->d_marked, J->d_status);
  b2k_count_launch();
  if(np)
  {
    k_t2_packets<<<grid(n * np), tpb, 0, st>>>(cs, J->d_sd, n, J->d_packets, np, J->d_pkt_tile, J->ntiles, J->nblocks, tags, J->d_indexed,
                                               J->d_start, J->d_end, J->d_part_end, J->d_kmax, J->d_blk, J->d_tags, J->d_marked, sop, eph,
                                               J->d_status);
    b2k_count_launch();
  }
  k_t2_walk<<<grid((uint64_t)n * J->ntiles), tpb, 0, st>>>(cs, J->d_sd, n, J->d_parts, J->d_head, J->d_tiles, J->ntiles, J->d_packets,
                                                           J->d_kmax, J->d_tile_first, J->nblocks, tags, J->d_blk, J->d_tags, J->d_indexed,
                                                           J->d_marked, sop, eph, J->d_status);
  b2k_count_launch();
  if(d_dec && J->window)
  {
    k_t2_window_at<<<1, 1024, 0, st>>>(J->d_sd, J->d_status, n);
    b2k_count_launch();
  }
  if(d_dec && J->ncoded)
  {
    k_t2_desc<<<(unsigned)((n * J->ncoded + 127) / 128), 128, 0, st>>>(J->d_sd, n, J->d_blk, J->nblocks, J->d_coded, (uint32_t)J->ncoded,
                                                                       d_enc, d_quant, d_dec, J->d_win, J->d_need, J->d_parts, J->d_head,
                                                                       box.tiles(), J->d_body_at, J->d_status);
    b2k_count_launch();
  }
  T2P_TRY(cudaMemcpyAsync(J->h_status, J->d_status, n * sizeof(ParseStatus), cudaMemcpyDeviceToHost, st));
  T2P_TRY(cudaGetLastError());
  return 0;
}

int b2k_t2_batch_enqueue(T2Parse* J, const uint8_t* arena, uint32_t n, const uint64_t* at, const uint64_t* len, const uint64_t* sot,
                         const HtBlockDesc* d_enc, const float* d_quant, HtBlockDesc* d_dec, cudaStream_t st)
{
  if(n > J->streams)
  {
    b2k_set_error("internal: more code streams than the parse was made for");
    return -1;
  }
  for(uint32_t s = 0; s < n; ++s)
    J->h_sd[s] = StreamDesc{at[s], len[s], sot[s], 0, 0, nullptr};
  return enqueue_parse(J, arena, n, J->ntiles, TileBox{J->ntiles, 0, 0, J->ntiles, 1}, J->d_count, d_enc, d_quant, d_dec, st);
}

uint32_t b2k_t2_parse_streams(const T2Parse* J) { return J->streams; }

int b2k_t2_window_enqueue(T2Parse* J, uint32_t n, const uint8_t* const* cs, const uint64_t* len, const uint64_t* sot,
                          const std::vector<Rect>* const* need, const TileBox& box, uint32_t ntiles, const HtBlockDesc* d_enc,
                          const float* d_quant, HtBlockDesc* d_dec, cudaStream_t st)
{
  if(n > J->streams)
  {
    b2k_set_error("internal: more code streams than the parse was made for");
    return -1;
  }
  if((uint64_t)n * ntiles > J->wcount_cap)
  {
    cudaFree(J->d_wcount);
    J->d_wcount = nullptr;
    J->wcount_cap = 0;
    const uint64_t cap = (uint64_t)J->streams * ntiles;
    T2P_TRY(cudaMalloc(&J->d_wcount, cap * sizeof(uint32_t)));
    J->wcount_cap = cap;
  }
  for(uint32_t s = 0; s < n; ++s)
  {
    NeedRects& N = J->h_need[s];
    N.n = need[s] ? (uint32_t)std::min<size_t>(need[s]->size(), WINDOW_MAX_RES) : 0;
    for(uint32_t r = 0; r < N.n; ++r)
    {
      const Rect& R = (*need[s])[r];
      N.r[r][0] = R.x0;
      N.r[r][1] = R.y0;
      N.r[r][2] = R.x1;
      N.r[r][3] = R.y1;
    }
    J->h_sd[s] = StreamDesc{0, len[s], sot[s], 0, 0, cs[s]};
  }
  return enqueue_parse(J, nullptr, n, ntiles, box, J->d_wcount, d_enc, d_quant, d_dec, st);
}

uint64_t b2k_t2_window_bytes(const T2Parse* J)
{
  uint64_t bytes = 0;
  for(uint32_t s = 0; s < J->last_n; ++s)
    if(status_reason(J->h_status[s]) == PR_NONE)
      bytes += J->h_status[s].bytes;
  return bytes;
}

uint64_t b2k_t2_window_arena(const T2Parse* J)
{
  uint64_t bytes = 0;
  for(uint32_t s = 0; s < J->last_n; ++s)
    bytes += window_gathered_bytes(J->h_status[s]);
  return bytes;
}

int b2k_t2_window_gather(const T2Parse* J, uint8_t* out, cudaStream_t st)
{
  uint64_t per = 0, bytes = 0, parts = 0;
  for(uint32_t s = 0; s < J->last_n; ++s)
    if(status_reason(J->h_status[s]) == PR_NONE)
    {
      per = std::max<uint64_t>(per, J->h_status[s].nparts);
      bytes += J->h_status[s].bytes;
      parts += J->h_status[s].nparts;
    }
  if(!parts || !bytes)
    return 0;
  const uint64_t items = J->last_n * per;
  const unsigned gx = (unsigned)std::min<uint64_t>(256, bytes / parts / (256 * 16) + 1);
  k_t2_gather<<<dim3(gx, (unsigned)std::min<uint64_t>(items, 65535)), 256, 0, st>>>(J->d_sd, J->d_parts, J->d_body_at, J->d_status, items,
                                                                                     per, out);
  b2k_count_launch();
  T2P_TRY(cudaGetLastError());
  return 0;
}

int b2k_t2_window_blocks(const T2Parse* J, const b2k_block* vblocks, uint64_t nv, const std::vector<Rect>& need, b2k_block* out,
                         cudaStream_t st)
{
  std::vector<ParsedBlock> pb(J->nblocks);
  T2P_TRY(cudaMemcpyAsync(pb.data(), J->d_blk, J->nblocks * sizeof(ParsedBlock), cudaMemcpyDeviceToHost, st));
  T2P_TRY(cudaStreamSynchronize(st));
  for(uint64_t i = 0; i < nv; ++i)
  {
    b2k_block b = vblocks[i];
    const ParsedBlock& p = pb[J->vmap[i]];
    bool wanted = true;
    if(!need.empty())
    {
      const Rect& n = need[b.resno ? b.resno - 1 : 0];
      const uint32_t r[4] = {n.x0, n.y0, n.x1, n.y1};
      wanted = window_needs(r, b.x0, b.y0, b.x1, b.y1);
    }
    if(wanted)
    {
      b.offset = p.offset;
      b.length = p.length;
      b.length2 = p.length2;
      b.numbps = p.numbps;
      b.numpasses = p.numpasses;
    }
    out[i] = b;
  }
  return 0;
}

int b2k_t2_batch_result(const T2Parse* J, uint32_t s, bool* refinement)
{
  const ParseStatus& st = J->h_status[s];
  const uint32_t r = status_reason(st);
  if(refinement)
    *refinement = st.refinement != 0;
  if(r == PR_NONE)
    return 0;
  b2k_set_error(parse_reason_text(r));
  return parse_reason_rc(r);
}

int b2k_t2_parse_result(const T2Parse* J, bool* refinement) { return b2k_t2_batch_result(J, 0, refinement); }

void b2k_t2_parse_stats(const T2Parse* J, uint32_t* indexed, uint32_t* walked)
{
  *indexed = *walked = 0;
  for(uint32_t s = 0; s < J->last_n; ++s)
  {
    *indexed += J->h_status[s].indexed;
    *walked += J->h_status[s].walked;
  }
}

int b2k_copy_table(const CopyEntry* d_tab, uint32_t n, uint64_t max_len, uint8_t* out, cudaStream_t st)
{
  if(!n || !max_len)
    return 0;
  const unsigned gx = (unsigned)std::min<uint64_t>(256, max_len / (256 * 16 * 4) + 1);
  k_copy_table<<<dim3(gx, std::min<uint32_t>(n, 65535)), 256, 0, st>>>(d_tab, n, out);
  b2k_count_launch();
  T2P_TRY(cudaGetLastError());
  return 0;
}

int b2k_t2_parse_blocks(const T2Parse* J, b2k_block* out, cudaStream_t st)
{
  std::vector<ParsedBlock> pb(J->nblocks);
  T2P_TRY(cudaMemcpyAsync(pb.data(), J->d_blk, J->nblocks * sizeof(ParsedBlock), cudaMemcpyDeviceToHost, st));
  T2P_TRY(cudaStreamSynchronize(st));
  for(uint64_t i = 0; i < J->nblocks; ++i)
  {
    b2k_block b = J->blocks[i];
    b.offset = pb[i].offset;
    b.length = pb[i].length;
    b.length2 = pb[i].length2;
    b.numbps = pb[i].numbps;
    b.numpasses = pb[i].numpasses;
    out[i] = b;
  }
  return 0;
}
