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
 */
#include <algorithm>
#include <string>
#include <vector>

#include "b2k_internal.h"
#include "t2_packet.h"
#include "t2_plan.h"
#include "t2_parse.h"
#include "t2_decode.h"

using namespace b2k;
using namespace b2k::t2;

void b2k_set_error(const char* msg); /* engine.cu */

namespace
{
constexpr unsigned long long NO_ERROR = ~0ull;
struct ParseStatus
{
  unsigned long long tile_err; /* (tile << 8) | reason of the lowest failing tile, NO_ERROR when none */
  uint32_t locate;             /* the tile-part walk's reason */
  uint32_t nparts;
  uint32_t refinement;         /* some block has refinement passes to decode */
  uint32_t walked;             /* tiles with data parsed by the walk */
  uint32_t indexed;            /* tiles whose packets were parsed from their PLT starts */
};

__global__ void k_t2_locate(const uint8_t* __restrict__ cs, uint64_t len, uint64_t sot, uint32_t ntiles, PartRange* __restrict__ parts,
                            uint64_t cap, uint32_t* __restrict__ head, uint32_t* __restrict__ last, uint32_t* __restrict__ count,
                            ParseStatus* status)
{
  uint32_t n = 0;
  status->locate = locate_tile_parts(cs, len, sot, ntiles, parts, cap, head, last, count, &n);
  status->nparts = n;
}

__global__ void k_t2_plt(const uint8_t* __restrict__ cs, const PartRange* __restrict__ parts, const uint32_t* __restrict__ head,
                         const DevPart* __restrict__ tiles, uint32_t ntiles, const uint64_t* __restrict__ tile_first,
                         ParsedBlock* __restrict__ blk, uint64_t* __restrict__ start, uint64_t* __restrict__ end,
                         uint64_t* __restrict__ part_end, uint32_t* __restrict__ indexed, uint32_t* __restrict__ marked,
                         ParseStatus* status)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if(t >= ntiles || status->locate != PR_NONE)
    return;
  for(uint64_t i = tile_first[t]; i < tile_first[t + 1]; ++i)
    blk[i] = ParsedBlock{};
  const DevPart T = tiles[t];
  const bool ix = plt_index(cs, parts, head[t], T.p1 - T.p0, start + T.p0, end + T.p0, part_end + T.p0);
  indexed[t] = ix;
  marked[t] = 0;
  if(ix && T.p1 > T.p0)
    atomicAdd(&status->indexed, 1u);
}

__global__ void k_t2_packets(const uint8_t* __restrict__ cs, const DevPacket* __restrict__ packets, uint64_t np,
                             const uint32_t* __restrict__ pkt_tile, const uint32_t* __restrict__ indexed,
                             const uint64_t* __restrict__ start, const uint64_t* __restrict__ end, const uint64_t* __restrict__ part_end,
                             const uint8_t* __restrict__ kmax, ParsedBlock* __restrict__ blk, TagNode* __restrict__ tags,
                             uint32_t* __restrict__ marked, bool sop, bool eph, const ParseStatus* status)
{
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(g >= np || status->locate != PR_NONE)
    return;
  const uint32_t t = pkt_tile[g];
  if(!indexed[t])
    return;
  uint64_t at = start[g];
  const DevPacket& P = packets[g];
  if(parse_packet(cs, P, &at, part_end[g], kmax, blk, tags + P.tag_at, sop, eph) != PR_NONE || at != end[g])
    marked[t] = 1; /* the walk decides */
}

__global__ void k_t2_walk(const uint8_t* __restrict__ cs, const PartRange* __restrict__ parts, const uint32_t* __restrict__ head,
                          const DevPart* __restrict__ tiles, uint32_t ntiles, const DevPacket* __restrict__ packets,
                          const uint8_t* __restrict__ kmax, const uint64_t* __restrict__ tile_first, ParsedBlock* __restrict__ blk,
                          TagNode* __restrict__ tags, const uint32_t* __restrict__ indexed, const uint32_t* __restrict__ marked,
                          bool sop, bool eph, ParseStatus* status)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if(t >= ntiles || status->locate != PR_NONE || (indexed[t] && !marked[t]))
    return;
  const DevPart T = tiles[t];
  if(T.p1 == T.p0)
    return;
  if(marked[t]) /* the packets parsed from PLT may have left fields behind */
    for(uint64_t i = tile_first[t]; i < tile_first[t + 1]; ++i)
      blk[i] = ParsedBlock{};
  if(head[t] != PART_NONE)
    atomicAdd(&status->walked, 1u);
  const uint32_t r = parse_tile(cs, parts, head[t], packets + T.p0, T.p1 - T.p0, kmax, blk, tags + packets[T.p0].tag_at, sop, eph);
  if(r != PR_NONE)
    atomicMin(&status->tile_err, ((unsigned long long)t << 8) | r);
}

__global__ void k_t2_desc(const ParsedBlock* __restrict__ blk, const uint32_t* __restrict__ coded, uint32_t ncoded,
                          const HtBlockDesc* __restrict__ enc, const float* __restrict__ quant, HtBlockDesc* __restrict__ dec,
                          ParseStatus* status)
{
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if(k >= ncoded || status->locate != PR_NONE || status->tile_err != NO_ERROR)
    return;
  const ParsedBlock b = blk[coded[k]];
  HtBlockDesc d = enc[k];
  d.length = b.length;
  d.slot_off = b.offset;
  block_decode_fields(b, d.kmax, &d.mmsbs, &d.passes, &d.length2);
  d.quant = quant[k]; /* stepsize / 2^(31-Kmax) */
  dec[k] = d;
  if(d.passes > 1)
    status->refinement = 1;
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
  std::vector<b2k_block> blocks; /* the enumeration, into which the parsed fields are merged */
  uint8_t* d_mem = nullptr;
  DevPacket* d_packets = nullptr;
  DevPart* d_tiles = nullptr;
  uint8_t* d_kmax = nullptr;
  uint64_t* d_tile_first = nullptr;
  uint32_t* d_coded = nullptr;
  TagNode* d_tags = nullptr;
  ParsedBlock* d_blk = nullptr;
  uint32_t *d_head = nullptr, *d_last = nullptr, *d_count = nullptr;
  uint32_t *d_pkt_tile = nullptr, *d_indexed = nullptr, *d_marked = nullptr;
  uint64_t *d_start = nullptr, *d_end = nullptr, *d_part_end = nullptr; /* per packet, from PLT */
  ParseStatus* d_status = nullptr;
  ParseStatus* h_status = nullptr; /* pinned */
  PartRange* d_parts = nullptr;    /* grown with the code stream's length */
  uint64_t parts_cap = 0;
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
                        const uint32_t* coded_index, uint64_t ncoded, T2Parse** out)
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
  const uint64_t np = P.packets.size();
  auto bytes = [](uint64_t n, size_t sz) { return (n * sz + 255) & ~(uint64_t)255; };
  const uint64_t total = bytes(np, sizeof(DevPacket)) + bytes(num_tiles, sizeof(DevPart)) + bytes(nblocks, 1) +
                         bytes(num_tiles + 1, sizeof(uint64_t)) + bytes(ncoded, sizeof(uint32_t)) + bytes(P.tag_nodes, sizeof(TagNode)) +
                         bytes(nblocks, sizeof(ParsedBlock)) + 5 * bytes(num_tiles, sizeof(uint32_t)) + bytes(np, sizeof(uint32_t)) +
                         3 * bytes(np, sizeof(uint64_t)) + bytes(1, sizeof(ParseStatus));
  T2P_TRY(cudaMalloc(&J->d_mem, total));
  uint8_t* p = J->d_mem;
  J->d_packets = carve<DevPacket>(p, np);
  J->d_tiles = carve<DevPart>(p, num_tiles);
  J->d_kmax = carve<uint8_t>(p, nblocks);
  J->d_tile_first = carve<uint64_t>(p, num_tiles + 1);
  J->d_coded = carve<uint32_t>(p, ncoded);
  J->d_tags = carve<TagNode>(p, P.tag_nodes);
  J->d_blk = carve<ParsedBlock>(p, nblocks);
  J->d_head = carve<uint32_t>(p, num_tiles);
  J->d_last = carve<uint32_t>(p, num_tiles);
  J->d_count = carve<uint32_t>(p, num_tiles);
  J->d_indexed = carve<uint32_t>(p, num_tiles);
  J->d_marked = carve<uint32_t>(p, num_tiles);
  J->d_pkt_tile = carve<uint32_t>(p, np);
  J->d_start = carve<uint64_t>(p, np);
  J->d_end = carve<uint64_t>(p, np);
  J->d_part_end = carve<uint64_t>(p, np);
  J->d_status = carve<ParseStatus>(p, 1);
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
  T2P_TRY(cudaHostAlloc(&J->h_status, sizeof(ParseStatus), cudaHostAllocDefault));
  *out = J;
  guard.j = nullptr;
  return 0;
}

void b2k_t2_parse_destroy(T2Parse* J)
{
  if(!J)
    return;
  cudaFree(J->d_mem);
  cudaFree(J->d_parts);
  cudaFreeHost(J->h_status);
  delete J;
}

uint32_t b2k_t2_parse_flags(const T2Parse* J) { return J->flags; }

int b2k_t2_parse_enqueue(T2Parse* J, const uint8_t* cs, uint64_t len, uint64_t sot, const HtBlockDesc* d_enc, const float* d_quant,
                         HtBlockDesc* d_dec, cudaStream_t st)
{
  /* every tile part takes at least the 12 bytes of its SOT, and a tile has at most 256 */
  const uint64_t need = std::min<uint64_t>(len / 12 + 1, 256ull * J->ntiles);
  if(need > J->parts_cap)
  {
    cudaFree(J->d_parts);
    J->d_parts = nullptr;
    J->parts_cap = 0;
    const uint64_t cap = need + need / 4 + 16;
    T2P_TRY(cudaMalloc(&J->d_parts, cap * sizeof(PartRange)));
    J->parts_cap = cap;
  }
  ParseStatus init{NO_ERROR, 0, 0, 0, 0, 0};
  *J->h_status = init;
  T2P_TRY(cudaMemcpyAsync(J->d_status, J->h_status, sizeof(ParseStatus), cudaMemcpyHostToDevice, st));
  k_t2_locate<<<1, 1, 0, st>>>(cs, len, sot, J->ntiles, J->d_parts, J->parts_cap, J->d_head, J->d_last, J->d_count, J->d_status);
  b2k_count_launch();
  const uint32_t tpb = 32; /* tiles and packets are few and each thread is a long serial chain: spread them over the SMs */
  const bool sop = (J->flags & B2K_CS_SOP) != 0, eph = (J->flags & B2K_CS_EPH) != 0;
  const uint64_t np = J->plan.packets.size();
  const unsigned tile_grid = (J->ntiles + tpb - 1) / tpb;
  k_t2_plt<<<tile_grid, tpb, 0, st>>>(cs, J->d_parts, J->d_head, J->d_tiles, J->ntiles, J->d_tile_first, J->d_blk, J->d_start, J->d_end,
                                      J->d_part_end, J->d_indexed, J->d_marked, J->d_status);
  b2k_count_launch();
  if(np)
  {
    k_t2_packets<<<(unsigned)((np + tpb - 1) / tpb), tpb, 0, st>>>(cs, J->d_packets, np, J->d_pkt_tile, J->d_indexed, J->d_start, J->d_end,
                                                                   J->d_part_end, J->d_kmax, J->d_blk, J->d_tags, J->d_marked, sop, eph,
                                                                   J->d_status);
    b2k_count_launch();
  }
  k_t2_walk<<<tile_grid, tpb, 0, st>>>(cs, J->d_parts, J->d_head, J->d_tiles, J->ntiles, J->d_packets, J->d_kmax, J->d_tile_first,
                                       J->d_blk, J->d_tags, J->d_indexed, J->d_marked, sop, eph, J->d_status);
  b2k_count_launch();
  if(d_dec && J->ncoded)
  {
    k_t2_desc<<<(unsigned)((J->ncoded + 127) / 128), 128, 0, st>>>(J->d_blk, J->d_coded, (uint32_t)J->ncoded, d_enc, d_quant, d_dec,
                                                                   J->d_status);
    b2k_count_launch();
  }
  T2P_TRY(cudaMemcpyAsync(J->h_status, J->d_status, sizeof(ParseStatus), cudaMemcpyDeviceToHost, st));
  T2P_TRY(cudaGetLastError());
  return 0;
}

int b2k_t2_parse_result(const T2Parse* J, bool* refinement)
{
  const ParseStatus& s = *J->h_status;
  uint32_t r = s.locate;
  if(r == PR_NONE && s.tile_err != NO_ERROR)
    r = (uint32_t)(s.tile_err & 0xFF);
  if(refinement)
    *refinement = s.refinement != 0;
  if(r == PR_NONE)
    return 0;
  b2k_set_error(parse_reason_text(r));
  return parse_reason_rc(r);
}

void b2k_t2_parse_stats(const T2Parse* J, uint32_t* indexed, uint32_t* walked)
{
  *indexed = J->h_status->indexed;
  *walked = J->h_status->walked;
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
