/*
 * grok_b200/csrc/t2_write.h -- the code-stream writer's steps over a batch of n code streams, as __host__ __device__
 * functions.  t2_device.cu runs them as kernels over the block coder's output; codestream.cpp runs them on the host pool
 * over a caller's block table (b2k_codestream_write and the per-rank writers, one stream); tests/t2_write_batch_check.cpp
 * runs the device's batch on the host, under the sanitizers.
 *
 * The plan (t2_plan.h: packets, tile parts, main header) is shared by every stream; everything else is sliced per stream:
 * header scratch (hdr_bytes each), tag-tree nodes (tag_nodes each), per-packet arrays (np each), per-part arrays (nparts
 * each), block destinations (the block source's slots each).  A thread of a launch over n streams of `per` items is
 * g = s * per + i.  The blocks come from a block source: CoderBlocks on the device, the caller's block table on the host.
 *
 * A stream's verdict is its WriteStatus: blocks the source marks failed, or a writer limit.  A stream with either gets
 * total 0: it takes no bytes of the output, and its blocks are not placed (dst = NOT_PLACED, which the gather skips).
 * Stream s starts at status[s].at: the streams lie in order, each at a 256-byte boundary (batch_arena_next, as a decode
 * batch lays out its arena).  When the streams do not fit the caller's buffer (place->used > cap) nothing is written
 * beyond the lengths; the caller grows the buffer and runs the steps again from the same coder output.
 */
#pragma once
#include <stdint.h>
#include <string>
#include "t2_packet.h"
#include "t2_parse.h"
#include "t2_plan.h"

namespace b2k
{
namespace t2
{
enum : uint32_t
{
  WERR_RANGE = 1,      /* a block outside the writer's range */
  WERR_PACKET = 2,     /* a packet of 4 GiB or more */
  WERR_PART = 4,       /* a tile part of 4 GiB or more */
  WERR_HDR_BOUND = 8,  /* a header longer than its bound */
  WERR_BLOCK = 16,     /* a block its source marks failed (per-packet error words only) */
};
/* a block the gather must leave alone: offset + length exceeds any buffer */
constexpr uint64_t NOT_PLACED = ~0ull >> 1;

struct WriteStatus /* one stream */
{
  uint64_t total;      /* code-stream length; 0 when the stream failed */
  uint32_t bad_blocks; /* blocks that overflowed the coder */
  uint32_t errors;     /* WERR_* */
  uint64_t at;         /* where the stream starts in the output */
};
struct WritePlace /* the batch */
{
  uint64_t used;       /* bytes the streams take, from the first to the end of the last */
  uint32_t done;       /* the scan's CTAs that have finished (the last one places the streams) */
  uint32_t pad;
};

/* the block coder's output (Out: HtBlockOut) as a block source: block i of the image is coded block coded[i] of the
   stream, or none (< 0); one pass, one bit plane (CoderOJPH), length = the coder's total, 0xFFFFFFFF when the block
   overflowed the coder's buffers.  A source gives block i's BlockCode (source(i)), the entry of dst its place goes to
   (slot(i), < 0 when the packet carries no bytes of it), and that slot's body length (bytes) or that it cannot give
   the bytes (failed). */
template <class Out>
struct CoderBlocks
{
  const int32_t* coded;
  const uint8_t* kmax;
  uint64_t slots;  /* coded blocks per stream */
  const Out* outs; /* stream 0's; stream(s) is stream s's */
  B2K_HD CoderBlocks stream(uint32_t s) const { return CoderBlocks{coded, kmax, slots, outs + (uint64_t)s * slots}; }
  B2K_HD BlockCode operator()(uint32_t i) const
  {
    const int32_t c = coded[i];
    uint32_t len = c >= 0 ? outs[c].total : 0u;
    len = len == 0xFFFFFFFFu ? 0u : len;
    return BlockCode{len, 0u, (uint8_t)(c >= 0 ? 1 : 0), 1, kmax[i]};
  }
  B2K_HD int64_t slot(uint32_t i) const { return coded[i]; }
  B2K_HD uint64_t bytes(int64_t c) const { return outs[c].total; }
  B2K_HD bool failed(int64_t c) const { return outs[c].total == 0xFFFFFFFFu; }
};

/* step 1, thread g = s * np + p: SOP, header bits and EPH of packet p of stream s into its header scratch; header and body
   lengths; each block's place in the body.  With pkt_err (the host's single stream) the packet's WERR_* word goes to
   pkt_err[g], WERR_BLOCK for a failed block, and the status is left alone; else failed blocks count in bad_blocks. */
template <class Blocks>
B2K_HD void write_header(uint64_t g, const DevPacket* packets, uint64_t np, const Blocks& blocks, uint8_t* hdr, uint64_t hdr_bytes,
                         TagNode* tags, uint64_t tag_nodes, uint32_t* hdr_len, uint64_t* body_len, uint64_t* dst, WriteStatus* status,
                         bool sop, bool eph, uint32_t* pkt_err = nullptr)
{
  const uint32_t s = (uint32_t)(g / np);
  const DevPacket P = packets[g % np];
  const Blocks B = blocks.stream(s);
  dst += (uint64_t)s * blocks.slots;
  BitWriter bw;
  bw.init(hdr + s * hdr_bytes + P.hdr_at, P.hdr_cap);
  uint32_t err = 0;
  if(packet_header(bw, P.band, (int)P.nbands, B, tags + s * tag_nodes + P.tag_at, P.sop, sop, eph))
    err |= WERR_RANGE;
  if(bw.n > bw.cap)
    err |= WERR_HDR_BOUND;
  uint64_t rel = 0;
  uint32_t bad = 0;
  for(uint32_t b = 0; b < P.nbands; ++b)
  {
    const uint32_t n = P.band[b].gw * P.band[b].gh;
    for(uint32_t k = 0; k < n; ++k)
    {
      const int64_t c = B.slot(P.band[b].first + k);
      if(c < 0)
        continue;
      if(B.failed(c))
      {
        ++bad;
        continue;
      }
      const uint64_t t = B.bytes(c);
      dst[c] = rel; /* relative to the body; write_packet adds the body's offset */
      rel += t;
    }
  }
  if(bw.n + rel > 0xFFFFFFFFull)
    err |= WERR_PACKET;
  hdr_len[g] = (uint32_t)bw.n;
  body_len[g] = rel;
  if(pkt_err)
    pkt_err[g] = err | (bad ? (uint32_t)WERR_BLOCK : 0u);
  else
  {
    if(bad)
      status_add(&status[s].bad_blocks, bad);
    if(err)
      status_or(&status[s].errors, err);
  }
}

/* step 1 over the block coder's output (CoderBlocks): the form the kernel and the batch harness call */
template <class Out>
B2K_HD void write_header(uint64_t g, const DevPacket* packets, uint64_t np, const int32_t* coded, const uint8_t* kmax, uint64_t ncoded,
                         const Out* outs, uint8_t* hdr, uint64_t hdr_bytes, TagNode* tags, uint64_t tag_nodes, uint32_t* hdr_len,
                         uint64_t* body_len, uint64_t* dst, WriteStatus* status, bool sop, bool eph)
{
  write_header(g, packets, np, CoderBlocks<Out>{coded, kmax, ncoded, outs}, hdr, hdr_bytes, tags, tag_nodes, hdr_len, body_len, dst,
               status, sop, eph);
}

/* packet k's length, header and body, for plt_segments */
struct PacketLen
{
  const uint32_t* hdr_len;
  const uint64_t* body_len;
  B2K_HD uint32_t operator()(uint64_t k) const { return (uint32_t)(hdr_len[k] + body_len[k]); }
};

/* step 2, thread g = s * nparts + t: PLT size and length of tile part t of stream s */
B2K_HD void write_part(uint64_t g, const DevPart* parts, uint64_t nparts, uint64_t np, const uint32_t* hdr_len, const uint64_t* body_len,
                       uint64_t* part_plt, uint64_t* part_bytes, WriteStatus* status, bool plt)
{
  const uint32_t s = (uint32_t)(g / nparts);
  const DevPart D = parts[g % nparts];
  hdr_len += (uint64_t)s * np;
  body_len += (uint64_t)s * np;
  uint64_t body = 0;
  for(uint64_t k = D.p0; k < D.p1; ++k)
    body += hdr_len[k] + body_len[k];
  const uint64_t pl = plt ? plt_segments(PacketLen{hdr_len, body_len}, D.p0, D.p1, nullptr) : 0;
  const uint64_t bytes = 12 + pl + 2 + body;
  part_plt[g] = pl;
  part_bytes[g] = bytes;
  if(bytes > 0xFFFFFFFFull)
    status_or(&status[s].errors, (uint32_t)WERR_PART);
}

/* step 3 ends with each stream's length (head, tile parts, EOC), or 0 for a stream with a verdict */
B2K_HD uint64_t write_total(const WriteStatus& st, uint64_t parts_end)
{
  return st.bad_blocks || st.errors ? 0 : parts_end + 2;
}

/* step 3 on the host: the exclusive scan of each stream's tile-part lengths behind the main header
   (part_at, relative to the stream), each stream's total, and the streams placed behind each other.  The kernel
   (t2_device.cu k_t2_scan) does the same with a CTA per stream. */
inline void write_scan_host(uint32_t n, const uint64_t* part_bytes, uint64_t nparts, uint64_t* part_at, uint64_t head_len,
                            WriteStatus* status, WritePlace* place)
{
  uint64_t at = 0, used = 0;
  for(uint32_t s = 0; s < n; ++s)
  {
    uint64_t carry = head_len;
    for(uint64_t i = 0; i < nparts; ++i)
    {
      part_at[s * nparts + i] = carry;
      carry += part_bytes[s * nparts + i];
    }
    status[s].total = write_total(status[s], carry);
    status[s].at = at;
    if(status[s].total)
      used = at + status[s].total;
    at = status[s].total ? batch_arena_next(at, status[s].total) : at;
  }
  place->used = used;
}

/* step 4, thread g = s * nparts + t: SOT, PLT, SOD and TLM entry of tile part t of stream s; every packet's offset in
   the output.  The main header (head) is written by the stream's threads too, in pieces no two threads share: part 0
   the markers before TLM, the first part of each TLM segment that segment's marker (the plan's, entries left to their
   parts), the last part the EOC.  Without a main header (head_len 0: a shard's tile parts) there is no EOC either. */
B2K_HD void write_emit(uint64_t g, const DevPart* parts, uint64_t nparts, uint64_t np, const uint64_t* part_at, const uint64_t* part_plt,
                       const uint64_t* part_bytes, const uint32_t* hdr_len, const uint64_t* body_len, uint64_t* pkt_at, uint8_t* cs,
                       uint64_t cap, const WriteStatus* status, const WritePlace* place, const uint8_t* head, uint64_t head_len,
                       bool plt, bool tlm, uint64_t tlm_at)
{
  const uint32_t s = (uint32_t)(g / nparts);
  const uint64_t t = g % nparts;
  if(place->used > cap || !status[s].total)
    return;
  const DevPart D = parts[t];
  hdr_len += (uint64_t)s * np;
  body_len += (uint64_t)s * np;
  pkt_at += (uint64_t)s * np;
  uint8_t* const base = cs + status[s].at;
  uint8_t* w = base + part_at[g];
  put_sot(w, D.tile, (uint32_t)part_bytes[g], D.index, D.count);
  w += 12;
  if(plt)
    plt_segments(PacketLen{hdr_len, body_len}, D.p0, D.p1, w);
  w += part_plt[g];
  w[0] = 0xFF; /* SOD */
  w[1] = 0x93;
  uint64_t at = status[s].at + part_at[g] + 12 + part_plt[g] + 2;
  for(uint64_t k = D.p0; k < D.p1; ++k)
  {
    pkt_at[k] = at;
    at += hdr_len[k] + body_len[k];
  }
  if(t == 0)
    for(uint64_t i = 0, e = tlm ? tlm_at : head_len; i < e; ++i)
      base[i] = head[i];
  if(tlm && t % TLM_PER_SEGMENT == 0)
    for(uint64_t i = tlm_at + tlm_entry_at(t) - 6, e = i + 6; i < e; ++i)
      base[i] = head[i];
  if(tlm)
    put_tlm_entry(base + tlm_at, t, D.tile, (uint32_t)part_bytes[g]);
  if(t == nparts - 1 && head_len)
  {
    base[status[s].total - 2] = 0xFF; /* EOC */
    base[status[s].total - 1] = 0xD9;
  }
}

/* step 5, packet g = s * np + p, worked by `lanes` threads of which this is `lane`: the packet's header to its place; its
   blocks' offsets in the output, or NOT_PLACED when the stream failed or the streams do not fit */
template <class Blocks>
B2K_HD void write_packet(uint64_t g, uint32_t lane, uint32_t lanes, const DevPacket* packets, uint64_t np, const Blocks& blocks,
                         const uint8_t* hdr, uint64_t hdr_bytes, const uint32_t* hdr_len, const uint64_t* pkt_at, uint64_t* dst,
                         uint8_t* cs, uint64_t cap, const WriteStatus* status, const WritePlace* place)
{
  const uint32_t s = (uint32_t)(g / np);
  const DevPacket P = packets[g % np];
  const Blocks B = blocks.stream(s);
  dst += (uint64_t)s * blocks.slots;
  const bool placed = place->used <= cap && status[s].total;
  const uint64_t at = placed ? pkt_at[g] : 0;
  const uint32_t hn = hdr_len[g];
  if(placed)
    for(uint32_t i = lane; i < hn; i += lanes)
      cs[at + i] = hdr[s * hdr_bytes + P.hdr_at + i];
  for(uint32_t b = 0; b < P.nbands; ++b)
  {
    const uint32_t n = P.band[b].gw * P.band[b].gh;
    for(uint32_t k = lane; k < n; k += lanes)
    {
      const int64_t c = B.slot(P.band[b].first + k);
      if(c >= 0 && !B.failed(c))
        dst[c] = placed ? dst[c] + at + hn : NOT_PLACED;
    }
  }
}
/* step 5 over the block coder's output (CoderBlocks) */
template <class Out>
B2K_HD void write_packet(uint64_t g, uint32_t lane, uint32_t lanes, const DevPacket* packets, uint64_t np, const int32_t* coded,
                         uint64_t ncoded, const Out* outs, const uint8_t* hdr, uint64_t hdr_bytes, const uint32_t* hdr_len,
                         const uint64_t* pkt_at, uint64_t* dst, uint8_t* cs, uint64_t cap, const WriteStatus* status,
                         const WritePlace* place)
{
  write_packet(g, lane, lanes, packets, np, CoderBlocks<Out>{coded, nullptr, ncoded, outs}, hdr, hdr_bytes, hdr_len, pkt_at, dst, cs, cap,
               status, place);
}
/* a stream's verdict as the single call reports it: its length, or -2 (blocks overflowed the coder) / -1 (the writer's
   limits) with the text b2k_encode_device / b2k_codestream_write give */
inline int64_t write_verdict(const WriteStatus& w, std::string* text)
{
  if(w.bad_blocks)
  {
    *text = std::to_string(w.bad_blocks) + " code block(s) overflowed the coder's buffers";
    return -2;
  }
  const char* why = (w.errors & WERR_RANGE)       ? "code block outside the writer's range (bit planes / passes)"
                    : (w.errors & WERR_PACKET)    ? "packet longer than 4 GiB"
                    : (w.errors & WERR_HDR_BOUND) ? "packet header longer than its bound"
                    : (w.errors & WERR_PART)      ? "tile part longer than 4 GiB"
                                                  : nullptr;
  if(why)
  {
    *text = why;
    return -1;
  }
  text->clear();
  return (int64_t)w.total;
}
} // namespace t2
} // namespace b2k
