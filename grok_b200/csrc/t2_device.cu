/*
 * grok_b200/csrc/t2_device.cu -- T2 on the device: the block coder's output (per-block lengths, bytes in the encoder's
 * scratch slots) becomes n complete code streams in device memory, each byte-identical to b2k_codestream_write's.
 *
 * With one quality layer every packet is independent: its header depends on its own blocks alone.  The plan (t2_plan.h)
 * fixes everything geometry decides and is shared by the n streams of a batch; per call six launches, however many
 * tiles and streams.  The threads' work is t2_write.h's:
 *   1. k_t2_headers  a thread per (stream, packet): SOP, header bits (t2_packet.h, shared with the host writer), EPH into
 *                    the packet's slot of the stream's header scratch; header and body lengths; each block's place in the
 *                    body; the stream's verdict (overflowed blocks, writer limits)
 *   2. k_t2_parts    a thread per (stream, tile part): PLT size and tile-part length
 *   3. k_t2_scan     a CTA per stream: tile-part offsets and the stream's length (0 with a verdict); the last CTA places
 *                    the streams behind each other at 256-byte boundaries
 *   4. k_t2_emit     a thread per (stream, tile part): SOT, PLT, SOD, TLM entry, every packet's offset; the main header
 *                    and EOC in pieces shared out over the stream's parts
 *   5. k_t2_packets  a warp per (stream, packet): its header to its place; its blocks' absolute offsets
 *   6. the encoder's gather (ht_enc.cu): each block's bytes straight from its scratch slot to its place in the output
 * A thread per packet: a header is a sequential bit string with tag-tree state, and packets outnumber the threads one
 * packet's blocks could keep busy (config 2: 1152 packets of at most 192 blocks).
 * Kernels 3-6 write only when the streams fit the caller's buffer; otherwise the caller grows it and runs them all
 * again from the same scratch slots.  A single code stream is the batch of one.
 */
#include <algorithm>
#include <cstring>
#include <string>

#include "b2k_internal.h"
#include "t2_packet.h"
#include "t2_plan.h"
#include "t2_device.h"
#include "t2_write.h"

using namespace b2k;
using namespace b2k::t2;

void b2k_set_error(const char* msg); /* engine.cu */

namespace
{
/* threads over n streams of `per` items: g = s * per + i */
__device__ __forceinline__ uint64_t thread_item() { return (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; }

__global__ void k_t2_headers(const DevPacket* __restrict__ packets, uint64_t np, uint64_t items, const int32_t* __restrict__ coded,
                             const uint8_t* __restrict__ kmax, uint64_t ncoded, const HtBlockOut* __restrict__ outs,
                             uint8_t* __restrict__ hdr, uint64_t hdr_bytes, TagNode* __restrict__ tags, uint64_t tag_nodes,
                             uint32_t* __restrict__ hdr_len, uint64_t* __restrict__ body_len, uint64_t* __restrict__ dst,
                             WriteStatus* status, bool sop, bool eph)
{
  const uint64_t g = thread_item();
  if(g < items)
    write_header(g, packets, np, coded, kmax, ncoded, outs, hdr, hdr_bytes, tags, tag_nodes, hdr_len, body_len, dst, status, sop, eph);
}

__global__ void k_t2_parts(const DevPart* __restrict__ parts, uint64_t nparts, uint64_t items, uint64_t np,
                           const uint32_t* __restrict__ hdr_len, const uint64_t* __restrict__ body_len, uint64_t* __restrict__ part_plt,
                           uint64_t* __restrict__ part_bytes, WriteStatus* status, bool plt)
{
  const uint64_t g = thread_item();
  if(g < items)
    write_part(g, parts, nparts, np, hdr_len, body_len, part_plt, part_bytes, status, plt);
}

/* exclusive scan over count values of one CTA, in rounds of SCAN_THREADS, starting from carry: out(i, prefix); returns the
   sum of everything (carry included).  Every thread of the CTA calls it. */
constexpr int SCAN_THREADS = 1024;
template <class Val, class Out>
__device__ uint64_t cta_scan(uint64_t count, uint64_t carry, const Val& val, const Out& out)
{
  __shared__ uint64_t warp_sum[32];
  __shared__ uint64_t carry_s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if(threadIdx.x == 0)
    carry_s = carry;
  __syncthreads();
  for(uint64_t base = 0; base < count; base += SCAN_THREADS)
  {
    const uint64_t i = base + threadIdx.x;
    const uint64_t v = i < count ? val(i) : 0;
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
    const uint64_t c = carry_s;
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
        carry_s = c + wi;
    }
    __syncthreads();
    if(i < count)
      out(i, c + warp_sum[warp] + incl - v);
    __syncthreads();
  }
  const uint64_t total = carry_s;
  __syncthreads(); /* every thread has read carry_s before the next call sets it */
  return total;
}

/* a CTA per stream: the stream's tile-part offsets behind the main header and its total (write_total).  The last CTA to
   finish places the streams behind each other (WriteStatus::at, WritePlace::used).  write_scan_host is the same for the
   host. */
__global__ void __launch_bounds__(SCAN_THREADS) k_t2_scan(const uint64_t* __restrict__ part_bytes, uint64_t nparts, uint32_t n,
                                                          uint64_t* __restrict__ part_at, uint64_t head_len, WriteStatus* status,
                                                          WritePlace* place)
{
  __shared__ bool last;
  __shared__ unsigned long long used_s;
  for(uint32_t s = blockIdx.x; s < n; s += gridDim.x)
  {
    const uint64_t o = (uint64_t)s * nparts;
    const uint64_t end = cta_scan(
        nparts, head_len, [&](uint64_t i) { return part_bytes[o + i]; }, [&](uint64_t i, uint64_t x) { part_at[o + i] = x; });
    if(threadIdx.x == 0)
      status[s].total = write_total(status[s], end);
  }
  __threadfence();
  __syncthreads();
  if(threadIdx.x == 0)
  {
    last = atomicAdd(&place->done, 1u) == gridDim.x - 1;
    used_s = 0;
  }
  __syncthreads();
  if(!last)
    return;
  __threadfence();
  /* the streams behind each other, each at a 256-byte boundary; another CTA's totals are read through L2.  The bytes
     used end where the last stream with a length ends: the largest at + total, offsets growing with s */
  const volatile WriteStatus* vs = status;
  cta_scan(
      n, 0, [&](uint64_t s) { const uint64_t t = vs[s].total; return t ? batch_arena_next(0, t) : 0; },
      [&](uint64_t s, uint64_t x) {
        status[s].at = x;
        if(const uint64_t t = vs[s].total)
          atomicMax(&used_s, (unsigned long long)(x + t));
      });
  if(threadIdx.x == 0)
    place->used = used_s;
}

__global__ void k_t2_emit(const DevPart* __restrict__ parts, uint64_t nparts, uint64_t items, uint64_t np, const uint64_t* __restrict__ part_at,
                          const uint64_t* __restrict__ part_plt, const uint64_t* __restrict__ part_bytes,
                          const uint32_t* __restrict__ hdr_len, const uint64_t* __restrict__ body_len, uint64_t* __restrict__ pkt_at,
                          uint8_t* __restrict__ cs, uint64_t cap, const WriteStatus* status, const WritePlace* place,
                          const uint8_t* __restrict__ head, uint64_t head_len, bool plt, bool tlm, uint64_t tlm_at)
{
  const uint64_t g = thread_item();
  if(g < items)
    write_emit(g, parts, nparts, np, part_at, part_plt, part_bytes, hdr_len, body_len, pkt_at, cs, cap, status, place, head, head_len, plt,
               tlm, tlm_at);
}

/* a warp per packet */
__global__ void k_t2_packets(const DevPacket* __restrict__ packets, uint64_t np, uint64_t items, const int32_t* __restrict__ coded,
                             uint64_t ncoded, const HtBlockOut* __restrict__ outs, const uint8_t* __restrict__ hdr, uint64_t hdr_bytes,
                             const uint32_t* __restrict__ hdr_len, const uint64_t* __restrict__ pkt_at, uint64_t* __restrict__ dst,
                             uint8_t* __restrict__ cs, uint64_t cap, const WriteStatus* status, const WritePlace* place)
{
  const uint64_t g = thread_item() >> 5;
  if(g < items)
    write_packet(g, threadIdx.x & 31, 32, packets, np, coded, ncoded, outs, hdr, hdr_bytes, hdr_len, pkt_at, dst, cs, cap, status, place);
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
  uint32_t streams = 1;
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
  /* the streams' statuses and the batch's placement, side by side so that one copy brings them home */
  WriteStatus* d_status = nullptr;
  WritePlace* d_place = nullptr;
  WriteStatus* h_status = nullptr; /* pinned, likewise followed by the placement */
  WritePlace* h_place = nullptr;
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
                  const uint32_t* coded_index, uint64_t ncoded, T2Job** out, uint32_t streams)
{
  *out = nullptr;
  T2Job* J = new T2Job();
  struct Guard
  {
    T2Job*& j;
    ~Guard() { b2k_t2_destroy(j); }
  } guard{J};
  if(b2k_t2_plan(cp, flags, blocks, nblocks, num_tiles, J->plan))
    return 1;
  const Plan& P = J->plan;
  J->ncoded = ncoded;
  J->streams = streams;
  std::vector<int32_t> coded(nblocks, -1);
  std::vector<uint8_t> kmax(nblocks);
  for(uint64_t k = 0; k < ncoded; ++k)
    coded[coded_index[k]] = (int32_t)k;
  for(uint64_t i = 0; i < nblocks; ++i)
    kmax[i] = blocks[i].kmax;
  const uint64_t np = P.packets.size(), nparts = P.parts.size(), S = streams;
  const uint64_t status_bytes = S * sizeof(WriteStatus) + sizeof(WritePlace);
  auto bytes = [](uint64_t n, size_t sz) { return (n * sz + 255) & ~(uint64_t)255; };
  const uint64_t total = bytes(np, sizeof(DevPacket)) + bytes(nparts, sizeof(DevPart)) + bytes(P.head.size(), 1) +
                         bytes(nblocks, sizeof(int32_t)) + bytes(nblocks, 1) + bytes(S * P.hdr_bytes, 1) +
                         bytes(S * P.tag_nodes, sizeof(TagNode)) + bytes(S * np, sizeof(uint32_t)) + 2 * bytes(S * np, sizeof(uint64_t)) +
                         3 * bytes(S * nparts, sizeof(uint64_t)) + bytes(S * ncoded, sizeof(uint64_t)) + bytes(status_bytes, 1);
  T2_TRY(cudaMalloc(&J->d_mem, total));
  uint8_t* p = J->d_mem;
  J->d_packets = carve<DevPacket>(p, np);
  J->d_parts = carve<DevPart>(p, nparts);
  J->d_head = carve<uint8_t>(p, P.head.size());
  J->d_coded = carve<int32_t>(p, nblocks);
  J->d_kmax = carve<uint8_t>(p, nblocks);
  J->d_hdr = carve<uint8_t>(p, S * P.hdr_bytes);
  J->d_tags = carve<TagNode>(p, S * P.tag_nodes);
  J->d_hdr_len = carve<uint32_t>(p, S * np);
  J->d_body_len = carve<uint64_t>(p, S * np);
  J->d_pkt_at = carve<uint64_t>(p, S * np);
  J->d_part_plt = carve<uint64_t>(p, S * nparts);
  J->d_part_bytes = carve<uint64_t>(p, S * nparts);
  J->d_part_at = carve<uint64_t>(p, S * nparts);
  J->d_dst = carve<uint64_t>(p, S * ncoded);
  J->d_status = reinterpret_cast<WriteStatus*>(carve<uint8_t>(p, status_bytes));
  J->d_place = reinterpret_cast<WritePlace*>(J->d_status + S);
  T2_TRY(cudaMemcpy(J->d_packets, P.packets.data(), np * sizeof(DevPacket), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_parts, P.parts.data(), nparts * sizeof(DevPart), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_head, P.head.data(), P.head.size(), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_coded, coded.data(), nblocks * sizeof(int32_t), cudaMemcpyHostToDevice));
  T2_TRY(cudaMemcpy(J->d_kmax, kmax.data(), nblocks, cudaMemcpyHostToDevice));
  T2_TRY(cudaHostAlloc(&J->h_status, status_bytes, cudaHostAllocDefault));
  J->h_place = reinterpret_cast<WritePlace*>(J->h_status + S);
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
uint32_t b2k_t2_streams(const T2Job* J) { return J->streams; }

int b2k_t2_enqueue(T2Job* J, const HtBlockDesc* d_enc, const HtBlockOut* d_out, const uint8_t* d_scratch, uint8_t* cs, uint64_t cap,
                   cudaStream_t st, uint32_t n)
{
  const Plan& P = J->plan;
  const uint64_t np = P.packets.size(), nparts = P.parts.size();
  const bool plt = (P.flags & B2K_CS_PLT) != 0, tlm = (P.flags & B2K_CS_TLM) != 0;
  const size_t status_bytes = J->streams * sizeof(WriteStatus) + sizeof(WritePlace);
  T2_TRY(cudaMemsetAsync(J->d_status, 0, status_bytes, st));
  const uint32_t tpb = 64; /* packets and tile parts are few: small CTAs spread them over the SMs */
  auto grid = [](uint64_t n, uint32_t per) { return (unsigned)std::max<uint64_t>(1, (n + per - 1) / per); };
  k_t2_headers<<<grid(n * np, tpb), tpb, 0, st>>>(J->d_packets, np, n * np, J->d_coded, J->d_kmax, J->ncoded, d_out, J->d_hdr,
                                                  P.hdr_bytes, J->d_tags, P.tag_nodes, J->d_hdr_len, J->d_body_len, J->d_dst,
                                                  J->d_status, (P.flags & B2K_CS_SOP) != 0, (P.flags & B2K_CS_EPH) != 0);
  b2k_count_launch();
  k_t2_parts<<<grid(n * nparts, tpb), tpb, 0, st>>>(J->d_parts, nparts, n * nparts, np, J->d_hdr_len, J->d_body_len, J->d_part_plt,
                                                    J->d_part_bytes, J->d_status, plt);
  b2k_count_launch();
  k_t2_scan<<<std::min<uint32_t>(n, 65535u), SCAN_THREADS, 0, st>>>(J->d_part_bytes, nparts, n, J->d_part_at, P.head.size(),
                                                                    J->d_status, J->d_place);
  b2k_count_launch();
  k_t2_emit<<<grid(n * nparts, tpb), tpb, 0, st>>>(J->d_parts, nparts, n * nparts, np, J->d_part_at, J->d_part_plt, J->d_part_bytes,
                                                   J->d_hdr_len, J->d_body_len, J->d_pkt_at, cs, cap, J->d_status, J->d_place, J->d_head,
                                                   P.head.size(), plt, tlm, P.tlm_at);
  b2k_count_launch();
  const uint32_t wpb = 8; /* warps per CTA */
  k_t2_packets<<<grid(n * np, wpb), wpb * 32, 0, st>>>(J->d_packets, np, n * np, J->d_coded, J->ncoded, d_out, J->d_hdr, P.hdr_bytes,
                                                       J->d_hdr_len, J->d_pkt_at, J->d_dst, cs, cap, J->d_status, J->d_place);
  b2k_count_launch();
  b2k_launch_ht_gather(d_enc, d_out, J->d_dst, d_scratch, cs, (uint32_t)(n * J->ncoded), cap, st);
  T2_TRY(cudaMemcpyAsync(J->h_status, J->d_status, status_bytes, cudaMemcpyDeviceToHost, st)); /* statuses and placement */
  T2_TRY(cudaGetLastError());
  return 0;
}

int64_t b2k_t2_result(const T2Job* J, uint32_t s)
{
  std::string text;
  const int64_t r = write_verdict(J->h_status[s], &text);
  if(r < 0)
    b2k_set_error(text.c_str());
  return r;
}

uint64_t b2k_t2_offset(const T2Job* J, uint32_t s) { return J->h_status[s].at; }
uint64_t b2k_t2_used(const T2Job* J) { return J->h_place->used; }
