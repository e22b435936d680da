/*
 * grok_b200/csrc/t2_device.cu -- T2 on the device: the block coder's output (per-block lengths, bytes in the encoder's
 * scratch slots) becomes a complete code stream in device memory, byte-identical to b2k_codestream_write's.
 *
 * With one quality layer every packet is independent: its header depends on its own blocks alone.  The plan (t2_plan.h)
 * fixes everything geometry decides; per frame six launches, however many tiles:
 *   1. k_t2_headers  a thread per packet: SOP, header bits (t2_packet.h, shared with the host writer), EPH into the
 *                    packet's slot of the header scratch; header and body lengths; each block's place in the body
 *   2. k_t2_parts    a thread per tile part: PLT size and tile-part length
 *   3. k_t2_scan     one CTA: tile-part offsets, the code-stream length; main header and EOC
 *   4. k_t2_emit     a thread per tile part: SOT, PLT, SOD, TLM entry, every packet's offset
 *   5. k_t2_packets  a warp per packet: its header to its place; its blocks' absolute offsets
 *   6. the encoder's gather (ht_enc.cu): each block's bytes straight from its scratch slot to its place in the file
 * A thread per packet: a header is a sequential bit string with tag-tree state, and packets outnumber the threads one
 * packet's blocks could keep busy (config 2: 1152 packets of at most 192 blocks).
 * Kernels 3-6 write only when the code stream fits the caller's buffer; otherwise the caller grows it and runs them all
 * again from the same scratch slots.
 */
#include <algorithm>
#include <cstring>
#include <string>

#include "b2k_internal.h"
#include "t2_packet.h"
#include "t2_plan.h"
#include "t2_device.h"

using namespace b2k;
using namespace b2k::t2;

void b2k_set_error(const char* msg); /* engine.cu */

namespace
{
enum : uint32_t
{
  ERR_RANGE = 1,      /* a block outside the writer's range */
  ERR_PACKET = 2,     /* a packet of 4 GiB or more */
  ERR_PART = 4,       /* a tile part of 4 GiB or more */
  ERR_HDR_BOUND = 8,  /* a header longer than its bound */
};

__global__ void k_t2_headers(const DevPacket* __restrict__ packets, uint64_t np, const int32_t* __restrict__ coded,
                             const uint8_t* __restrict__ kmax, const HtBlockOut* __restrict__ outs, uint8_t* __restrict__ hdr,
                             TagNode* __restrict__ tags, uint32_t* __restrict__ hdr_len, uint64_t* __restrict__ body_len,
                             uint64_t* __restrict__ dst, T2Status* status, bool sop, bool eph)
{
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(p >= np)
    return;
  const DevPacket P = packets[p];
  /* a coded block as b2k_encode reports it: one pass, one bit plane (CoderOJPH), length = the coder's total */
  auto code = [&](uint32_t i) {
    const int32_t c = coded[i];
    uint32_t len = c >= 0 ? outs[c].total : 0u;
    len = len == 0xFFFFFFFFu ? 0u : len;
    return BlockCode{len, 0u, (uint8_t)(c >= 0 ? 1 : 0), 1, kmax[i]};
  };
  BitWriter bw;
  bw.init(hdr + P.hdr_at, P.hdr_cap);
  uint32_t err = 0;
  if(packet_header(bw, P.band, (int)P.nbands, code, tags + P.tag_at, P.sop, sop, eph))
    err |= ERR_RANGE;
  if(bw.n > bw.cap)
    err |= ERR_HDR_BOUND;
  uint64_t rel = 0;
  uint32_t bad = 0;
  for(uint32_t b = 0; b < P.nbands; ++b)
  {
    const uint32_t n = P.band[b].gw * P.band[b].gh;
    for(uint32_t k = 0; k < n; ++k)
    {
      const int32_t c = coded[P.band[b].first + k];
      if(c < 0)
        continue;
      const uint32_t t = outs[c].total;
      if(t == 0xFFFFFFFFu)
      {
        ++bad;
        continue;
      }
      dst[c] = rel; /* relative to the body; k_t2_packets adds the body's offset */
      rel += t;
    }
  }
  if(bw.n + rel > 0xFFFFFFFFull)
    err |= ERR_PACKET;
  hdr_len[p] = (uint32_t)bw.n;
  body_len[p] = rel;
  if(bad)
    atomicAdd(&status->bad_blocks, bad);
  if(err)
    atomicOr(&status->errors, err);
}

struct PacketLen
{
  const uint32_t* hdr_len;
  const uint64_t* body_len;
  __device__ uint32_t operator()(uint64_t k) const { return (uint32_t)(hdr_len[k] + body_len[k]); }
};

__global__ void k_t2_parts(const DevPart* __restrict__ parts, uint64_t nparts, const uint32_t* __restrict__ hdr_len,
                           const uint64_t* __restrict__ body_len, uint64_t* __restrict__ part_plt, uint64_t* __restrict__ part_bytes,
                           T2Status* status, bool plt)
{
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(t >= nparts)
    return;
  const DevPart D = parts[t];
  uint64_t body = 0;
  for(uint64_t k = D.p0; k < D.p1; ++k)
    body += hdr_len[k] + body_len[k];
  const uint64_t pl = plt ? plt_segments(PacketLen{hdr_len, body_len}, D.p0, D.p1, nullptr) : 0;
  const uint64_t bytes = 12 + pl + 2 + body;
  part_plt[t] = pl;
  part_bytes[t] = bytes;
  if(bytes > 0xFFFFFFFFull)
    atomicOr(&status->errors, (uint32_t)ERR_PART);
}

/* exclusive scan of the tile-part lengths behind the main header; then, if the code stream fits, the main header and EOC */
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS) k_t2_scan(const uint64_t* __restrict__ part_bytes, uint64_t nparts,
                                                          uint64_t* __restrict__ part_at, const uint8_t* __restrict__ head,
                                                          uint64_t head_len, uint8_t* __restrict__ cs, uint64_t cap, T2Status* status)
{
  __shared__ uint64_t warp_sum[32];
  __shared__ uint64_t carry_s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if(threadIdx.x == 0)
    carry_s = head_len;
  __syncthreads();
  for(uint64_t base = 0; base < nparts; base += SCAN_THREADS)
  {
    const uint64_t i = base + threadIdx.x;
    const uint64_t v = i < nparts ? part_bytes[i] : 0;
    uint64_t incl = v;
#pragma unroll
    for(int o = 1; o < 32; o <<= 1)
    {
      const uint64_t y = __shfl_up_sync(0xffffffffu, incl, o);
      if(lane >= o)
        incl += y;
    }
    if(lane == 31)
      warp_sum[warp] = incl;
    const uint64_t carry = carry_s;
    __syncthreads();
    if(warp == 0)
    {
      const uint64_t w = warp_sum[lane];
      uint64_t wi = w;
#pragma unroll
      for(int o = 1; o < 32; o <<= 1)
      {
        const uint64_t y = __shfl_up_sync(0xffffffffu, wi, o);
        if(lane >= o)
          wi += y;
      }
      warp_sum[lane] = wi - w;
      if(lane == 31)
        carry_s = carry + wi;
    }
    __syncthreads();
    if(i < nparts)
      part_at[i] = carry + warp_sum[warp] + incl - v;
    __syncthreads();
  }
  const uint64_t total = carry_s + 2;
  if(threadIdx.x == 0)
    status->total = total;
  if(total > cap)
    return;
  for(uint64_t i = threadIdx.x; i < head_len; i += SCAN_THREADS)
    cs[i] = head[i];
  if(threadIdx.x == 0)
  {
    cs[total - 2] = 0xFF; /* EOC */
    cs[total - 1] = 0xD9;
  }
}

__global__ void k_t2_emit(const DevPart* __restrict__ parts, uint64_t nparts, const uint64_t* __restrict__ part_at,
                          const uint64_t* __restrict__ part_plt, const uint64_t* __restrict__ part_bytes,
                          const uint32_t* __restrict__ hdr_len, const uint64_t* __restrict__ body_len, uint64_t* __restrict__ pkt_at,
                          uint8_t* __restrict__ cs, uint64_t cap, const T2Status* status, bool plt, bool tlm, uint64_t tlm_at)
{
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if(t >= nparts || status->total > cap)
    return;
  const DevPart D = parts[t];
  uint8_t* w = cs + part_at[t];
  put_sot(w, D.tile, (uint32_t)part_bytes[t], D.index, D.count);
  w += 12;
  if(plt)
    plt_segments(PacketLen{hdr_len, body_len}, D.p0, D.p1, w);
  w += part_plt[t];
  w[0] = 0xFF; /* SOD */
  w[1] = 0x93;
  uint64_t at = part_at[t] + 12 + part_plt[t] + 2;
  for(uint64_t k = D.p0; k < D.p1; ++k)
  {
    pkt_at[k] = at;
    at += hdr_len[k] + body_len[k];
  }
  if(tlm)
    put_tlm_entry(cs + tlm_at, t, D.tile, (uint32_t)part_bytes[t]);
}

__global__ void k_t2_packets(const DevPacket* __restrict__ packets, uint64_t np, const int32_t* __restrict__ coded,
                             const HtBlockOut* __restrict__ outs, const uint8_t* __restrict__ hdr, const uint32_t* __restrict__ hdr_len,
                             const uint64_t* __restrict__ pkt_at, uint64_t* __restrict__ dst, uint8_t* __restrict__ cs, uint64_t cap,
                             const T2Status* status)
{
  const uint64_t p = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t lane = threadIdx.x & 31;
  if(p >= np || status->total > cap)
    return;
  const DevPacket P = packets[p];
  const uint64_t at = pkt_at[p];
  const uint32_t hn = hdr_len[p];
  for(uint32_t i = lane; i < hn; i += 32)
    cs[at + i] = hdr[P.hdr_at + i];
  for(uint32_t b = 0; b < P.nbands; ++b)
  {
    const uint32_t n = P.band[b].gw * P.band[b].gh;
    for(uint32_t k = lane; k < n; k += 32)
    {
      const int32_t c = coded[P.band[b].first + k];
      if(c >= 0 && outs[c].total != 0xFFFFFFFFu)
        dst[c] += at + hn;
    }
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

struct T2Job
{
  Plan plan;
  uint64_t ncoded = 0;
  uint8_t* d_mem = nullptr;
  DevPacket* d_packets = nullptr;
  DevPart* d_parts = nullptr;
  uint8_t* d_head = nullptr;
  int32_t* d_coded = nullptr;
  uint8_t* d_kmax = nullptr;
  uint8_t* d_hdr = nullptr;
  TagNode* d_tags = nullptr;
  uint32_t* d_hdr_len = nullptr;
  uint64_t *d_body_len = nullptr, *d_pkt_at = nullptr, *d_part_plt = nullptr, *d_part_bytes = nullptr, *d_part_at = nullptr, *d_dst = nullptr;
  T2Status* d_status = nullptr;
  T2Status* h_status = nullptr; /* pinned */
};

#define T2_TRY(expr)                                                                                                           \
  do                                                                                                                           \
  {                                                                                                                            \
    cudaError_t _e = (expr);                                                                                                   \
    if(_e != cudaSuccess)                                                                                                      \
    {                                                                                                                          \
      b2k_set_error((std::string(#expr) + ": " + cudaGetErrorString(_e)).c_str());                                            \
      return -1;                                                                                                               \
    }                                                                                                                          \
  } while(0)

int b2k_t2_create(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles,
                  const uint32_t* coded_index, uint64_t ncoded, T2Job** out)
{
  *out = nullptr;
  T2Job* J = new T2Job();
  struct Guard
  {
    T2Job*& j;
    ~Guard() { b2k_t2_destroy(j); }
  } guard{J};
  if(b2k_t2_plan(cp, flags, blocks, nblocks, num_tiles, J->plan))
    return -1;
  const Plan& P = J->plan;
  J->ncoded = ncoded;
  std::vector<int32_t> coded(nblocks, -1);
  std::vector<uint8_t> kmax(nblocks);
  for(uint64_t k = 0; k < ncoded; ++k)
    coded[coded_index[k]] = (int32_t)k;
  for(uint64_t i = 0; i < nblocks; ++i)
    kmax[i] = blocks[i].kmax;
  const uint64_t np = P.packets.size(), nparts = P.parts.size();
  auto bytes = [](uint64_t n, size_t sz) { return (n * sz + 255) & ~(uint64_t)255; };
  const uint64_t total = bytes(np, sizeof(DevPacket)) + bytes(nparts, sizeof(DevPart)) + bytes(P.head.size(), 1) +
                         bytes(nblocks, sizeof(int32_t)) + bytes(nblocks, 1) + bytes(P.hdr_bytes, 1) + bytes(P.tag_nodes, sizeof(TagNode)) +
                         bytes(np, sizeof(uint32_t)) + 2 * bytes(np, sizeof(uint64_t)) + 3 * bytes(nparts, sizeof(uint64_t)) +
                         bytes(ncoded, sizeof(uint64_t)) + bytes(1, sizeof(T2Status));
  T2_TRY(cudaMalloc(&J->d_mem, total));
  uint8_t* p = J->d_mem;
  J->d_packets = carve<DevPacket>(p, np);
  J->d_parts = carve<DevPart>(p, nparts);
  J->d_head = carve<uint8_t>(p, P.head.size());
  J->d_coded = carve<int32_t>(p, nblocks);
  J->d_kmax = carve<uint8_t>(p, nblocks);
  J->d_hdr = carve<uint8_t>(p, P.hdr_bytes);
  J->d_tags = carve<TagNode>(p, P.tag_nodes);
  J->d_hdr_len = carve<uint32_t>(p, np);
  J->d_body_len = carve<uint64_t>(p, np);
  J->d_pkt_at = carve<uint64_t>(p, np);
  J->d_part_plt = carve<uint64_t>(p, nparts);
  J->d_part_bytes = carve<uint64_t>(p, nparts);
  J->d_part_at = carve<uint64_t>(p, nparts);
  J->d_dst = carve<uint64_t>(p, ncoded);
  J->d_status = carve<T2Status>(p, 1);
  T2_TRY(cudaMemcpy(J->d_packets, P.packets.data(), np * sizeof(DevPacket), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_parts, P.parts.data(), nparts * sizeof(DevPart), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_head, P.head.data(), P.head.size(), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_coded, coded.data(), nblocks * sizeof(int32_t), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_kmax, kmax.data(), nblocks, cudaMemcpyHostToDevice));
  T2_TRY(cudaHostAlloc(&J->h_status, sizeof(T2Status), cudaHostAllocDefault));
  *out = J;
  guard.j = nullptr;
  return 0;
}

void b2k_t2_destroy(T2Job* J)
{
  if(!J)
    return;
  cudaFree(J->d_mem);
  cudaFreeHost(J->h_status);
  delete J;
}

uint32_t b2k_t2_flags(const T2Job* J) { return J->plan.flags; }

int b2k_t2_enqueue(T2Job* J, const HtBlockDesc* d_enc, const HtBlockOut* d_out, const uint8_t* d_scratch, uint8_t* cs, uint64_t cap,
                   cudaStream_t st)
{
  const Plan& P = J->plan;
  const uint64_t np = P.packets.size(), nparts = P.parts.size();
  const bool plt = (P.flags & B2K_CS_PLT) != 0, tlm = (P.flags & B2K_CS_TLM) != 0;
  T2_TRY(cudaMemsetAsync(J->d_status, 0, sizeof(T2Status), st));
  const uint32_t tpb = 64; /* packets and tile parts are few: small CTAs spread them over the SMs */
  auto grid = [](uint64_t n, uint32_t per) { return (unsigned)std::max<uint64_t>(1, (n + per - 1) / per); };
  k_t2_headers<<<grid(np, tpb), tpb, 0, st>>>(J->d_packets, np, J->d_coded, J->d_kmax, d_out, J->d_hdr, J->d_tags,
                                                                 J->d_hdr_len, J->d_body_len, J->d_dst, J->d_status,
                                                                 (P.flags & B2K_CS_SOP) != 0, (P.flags & B2K_CS_EPH) != 0);
  b2k_count_launch();
  k_t2_parts<<<grid(nparts, tpb), tpb, 0, st>>>(J->d_parts, nparts, J->d_hdr_len, J->d_body_len, J->d_part_plt,
                                                                   J->d_part_bytes, J->d_status, plt);
  b2k_count_launch();
  k_t2_scan<<<1, SCAN_THREADS, 0, st>>>(J->d_part_bytes, nparts, J->d_part_at, J->d_head, P.head.size(), cs, cap, J->d_status);
  b2k_count_launch();
  k_t2_emit<<<grid(nparts, tpb), tpb, 0, st>>>(J->d_parts, nparts, J->d_part_at, J->d_part_plt, J->d_part_bytes,
                                                                  J->d_hdr_len, J->d_body_len, J->d_pkt_at, cs, cap, J->d_status, plt,
                                                                  tlm, P.tlm_at);
  b2k_count_launch();
  const uint32_t wpb = 8; /* warps per CTA */
  k_t2_packets<<<grid(np, wpb), wpb * 32, 0, st>>>(J->d_packets, np, J->d_coded, d_out, J->d_hdr, J->d_hdr_len,
                                                                      J->d_pkt_at, J->d_dst, cs, cap, J->d_status);
  b2k_count_launch();
  b2k_launch_ht_gather(d_enc, d_out, J->d_dst, d_scratch, cs, (uint32_t)J->ncoded, cap, st);
  T2_TRY(cudaMemcpyAsync(J->h_status, J->d_status, sizeof(T2Status), cudaMemcpyDeviceToHost, st));
  T2_TRY(cudaGetLastError());
  return 0;
}

int64_t b2k_t2_result(const T2Job* J)
{
  const T2Status& s = *J->h_status;
  if(s.bad_blocks)
  {
    b2k_set_error((std::to_string(s.bad_blocks) + " code block(s) overflowed the coder's buffers").c_str());
    return -2;
  }
  const char* why = (s.errors & ERR_RANGE)       ? "code block outside the writer's range (bit planes / passes)"
                    : (s.errors & ERR_PACKET)    ? "packet longer than 4 GiB"
                    : (s.errors & ERR_HDR_BOUND) ? "packet header longer than its bound"
                    : (s.errors & ERR_PART)      ? "tile part longer than 4 GiB"
                                                 : nullptr;
  if(why)
  {
    b2k_set_error(why);
    return -1;
  }
  return (int64_t)s.total;
}
