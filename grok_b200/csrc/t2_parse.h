/*
 * grok_b200/csrc/t2_parse.h -- reading the tile parts and packet headers of an HTJ2K code stream, as __host__ __device__
 * code over a byte buffer: the tile-part walk (SOT / Psot / tile-part header segments up to SOD), the packet-header bit
 * reader (7 bits after 0xFF), the tag-tree decoder, pass count, Lblock and the HT segment lengths, SOP / EPH.
 * The device parser (t2_decode.cu) runs these functions in its kernels; tests/t2_parse_check.cpp runs them on the host in
 * the same order and compares with b2k_codestream_parse.
 *
 * The verdicts are those of the host parser (codestream.cpp, parse_impl / parse_tile_packets) for every input: the same
 * tile parts, the same blocks, the same first failure and its return code.  Written from ITU-T T.800 Annex A/B and T.814
 * Annex B; the packets of a tile and their blocks come from the code-stream plan (t2_plan.h).
 */
#pragma once
#include <stdint.h>
#include "t2_packet.h"

namespace b2k
{
namespace t2
{

/* why a parse failed; 0 = it did not */
enum ParseReason : uint32_t
{
  PR_NONE = 0,
  PR_EXPECTED_SOT,  /* -1 */
  PR_BAD_SOT,       /* -1 */
  PR_TP_ORDER,      /*  1 */
  PR_PSOT,          /* -1 */
  PR_TP_TRUNCATED,  /* -1 */
  PR_TP_SEGMENT,    /* -1 */
  PR_TP_MARKER,     /*  1 */
  PR_ZBP,           /* -1 */
  PR_PASSES,        /*  1 */
  PR_LBLOCK,        /* -1 */
  PR_ZBP_KMAX,      /* -1 */
  PR_SHORT_CLEANUP, /* -1 */
  PR_HEADER_RUN,    /* -1 */
  PR_EPH,           /* -1 */
  PR_BODY_RUN,      /* -1 */
  PR_PART_TABLE,    /* -1: more tile parts than the table holds (cannot happen: each takes at least 12 bytes) */
  PR_SKIPPED,       /* a stream of a batch that failed before its tile parts: not parsed, its blocks stay uncoded */
  PR_COUNT
};
B2K_HD int parse_reason_rc(uint32_t r) { return (r == PR_TP_ORDER || r == PR_TP_MARKER || r == PR_PASSES) ? 1 : -1; }
/* the host parser's text for each reason */
inline const char* parse_reason_text(uint32_t r)
{
  switch(r)
  {
    case PR_EXPECTED_SOT: return "expected SOT or EOC";
    case PR_BAD_SOT: return "bad SOT";
    case PR_TP_ORDER: return "tile parts out of order";
    case PR_PSOT: return "Psot exceeds the codestream";
    case PR_TP_TRUNCATED: return "truncated tile-part header";
    case PR_TP_SEGMENT: return "bad tile-part marker segment";
    case PR_TP_MARKER: return "tile-part COD / COC / QCD / QCC / RGN / POC / PPT are not handled";
    case PR_ZBP: return "corrupt packet header (zero bit planes)";
    case PR_PASSES: return "HT code blocks with placeholder passes or several HT sets are not handled";
    case PR_LBLOCK: return "corrupt packet header (Lblock)";
    case PR_ZBP_KMAX: return "more zero bit planes than the band has bit planes";
    case PR_SHORT_CLEANUP: return "HT cleanup segment shorter than 2 bytes";
    case PR_HEADER_RUN: return "packet header runs past the tile part";
    case PR_EPH: return "EPH marker missing after a packet header";
    case PR_BODY_RUN: return "packet body runs past the tile part";
    case PR_PART_TABLE: return "internal: tile-part table too small";
    default: return "";
  }
}

constexpr uint32_t PART_NONE = 0xFFFFFFFFu;
/* one tile part, in stream order: where its header starts, its packet data [begin, end) (offsets into the code stream; begin may exceed end when
   a tile-part header runs past Psot, exactly as on the host), its tile, the next tile part of the same tile */
struct PartRange
{
  uint64_t hdr;        /* the tile-part header's first segment (just after SOT) */
  uint64_t begin, end;
  uint32_t tile, next;
};
/* what the parse gives a block: the fields b2k_codestream_parse fills in (offset into the code stream) */
struct ParsedBlock
{
  uint64_t offset;
  uint32_t length, length2;
  uint8_t numbps, numpasses, pad[6];
};

/* big-endian reads with the host parser's sticky failure: a read past `end` fails and reads nothing */
struct ByteCursor
{
  const uint8_t* cs;
  uint64_t p, end;
  bool ok;
  B2K_HD uint32_t u8()
  {
    if(p + 1 > end)
    {
      ok = false;
      return 0;
    }
    return cs[p++];
  }
  B2K_HD uint32_t u16()
  {
    if(p + 2 > end)
    {
      ok = false;
      return 0;
    }
    const uint32_t v = ((uint32_t)cs[p] << 8) | cs[p + 1];
    p += 2;
    return v;
  }
  B2K_HD uint32_t u32()
  {
    const uint32_t a = u16();
    return (a << 16) | u16();
  }
};

/* the tiles a windowed parse wants: columns [x0, x1) and rows [y0, y1) of a grid nx tiles wide.  Box tile
   (ix - x0) + (iy - y0) * (x1 - x0) is the stream's tile ix + iy * nx. */
struct TileBox
{
  uint32_t nx, x0, y0, x1, y1;
  B2K_HD uint32_t tiles() const { return (x1 - x0) * (y1 - y0); }
};

/* The tile parts from the first SOT (at sot) to EOC or the end of the stream, in stream order, as the host parser walks
 * them (A.4.2): SOT, Psot hop, tile-part header segments up to SOD.  Every SOT is checked; a tile outside `box` is hopped
 * over through Psot without its tile-part header being read, and only the wanted tiles' parts are recorded, under their
 * box tile index.  head[t] / last[t] (box.tiles() each) and count[t] (ntiles) are scratch the walk initialises; parts holds
 * cap entries.  body_at (when not NULL) receives where each recorded part's packet data starts when the bodies are laid
 * end to end, *body_bytes their total.  Returns PR_NONE or the first failure in stream order. */
B2K_HD uint32_t locate_tile_parts_box(const uint8_t* cs, uint64_t len, uint64_t sot, uint32_t ntiles, const TileBox& box,
                                      PartRange* parts, uint64_t cap, uint32_t* head, uint32_t* last, uint32_t* count, uint32_t* nparts,
                                      uint64_t* body_at, uint64_t* body_bytes)
{
  for(uint32_t t = 0; t < box.tiles(); ++t)
    head[t] = last[t] = PART_NONE;
  for(uint32_t t = 0; t < ntiles; ++t)
    count[t] = 0;
  *nparts = 0;
  uint64_t bytes = 0;
  if(body_bytes)
    *body_bytes = 0;
  /* Psot = 0: the tile part runs to the end of the stream, before a final EOC */
  const uint64_t open_end = len - ((len >= 2 && cs[len - 2] == 0xFF && cs[len - 1] == 0xD9) ? 2 : 0);
  ByteCursor c{cs, sot, len, true};
  uint32_t n = 0;
  for(;;)
  {
    const uint64_t at = c.p;
    const uint32_t m = c.u16();
    if(!c.ok || m == 0xFFD9)
      break; /* a missing EOC is tolerated */
    if(m != 0xFF90)
      return PR_EXPECTED_SOT;
    const uint32_t lsot = c.u16(), isot = c.u16(), psot = c.u32(), tpsot = c.u8();
    c.u8(); /* TNsot */
    if(!c.ok || lsot != 10 || isot >= ntiles)
      return PR_BAD_SOT;
    if(tpsot != count[isot])
      return PR_TP_ORDER;
    ++count[isot];
    const uint64_t tp_end = psot ? at + psot : open_end;
    if(tp_end > len || tp_end < c.p)
      return PR_PSOT;
    const uint32_t ix = isot % box.nx, iy = isot / box.nx;
    if(ix < box.x0 || ix >= box.x1 || iy < box.y0 || iy >= box.y1)
    { /* not wanted: hop over it */
      c.p = tp_end;
      continue;
    }
    const uint32_t bt = (ix - box.x0) + (iy - box.y0) * (box.x1 - box.x0);
    for(;;)
    { /* tile-part header: PLT, COM and unknown segments are skipped */
      const uint32_t tm = c.u16();
      if(!c.ok)
        return PR_TP_TRUNCATED;
      if(tm == 0xFF93)
        break;
      const uint32_t L = c.u16();
      if(!c.ok || L < 2 || c.p + (L - 2) > tp_end)
        return PR_TP_SEGMENT;
      if(tm == 0xFF52 || tm == 0xFF53 || tm == 0xFF5C || tm == 0xFF5D || tm == 0xFF5E || tm == 0xFF5F || tm == 0xFF61)
        return PR_TP_MARKER;
      c.p += L - 2;
    }
    if(n >= cap)
      return PR_PART_TABLE;
    parts[n] = PartRange{at + 12, c.p, tp_end, bt, PART_NONE};
    if(body_at)
      body_at[n] = bytes;
    bytes += tp_end > c.p ? tp_end - c.p : 0;
    if(body_bytes)
      *body_bytes = bytes;
    if(last[bt] == PART_NONE)
      head[bt] = n;
    else
      parts[last[bt]].next = n;
    last[bt] = n;
    *nparts = ++n;
    c.p = tp_end;
  }
  return PR_NONE;
}

/* every tile wanted: the tile parts of the whole stream, under their own tile index */
B2K_HD uint32_t locate_tile_parts(const uint8_t* cs, uint64_t len, uint64_t sot, uint32_t ntiles, PartRange* parts, uint64_t cap,
                                  uint32_t* head, uint32_t* last, uint32_t* count, uint32_t* nparts)
{
  return locate_tile_parts_box(cs, len, sot, ntiles, TileBox{ntiles, 0, 0, ntiles, 1}, parts, cap, head, last, count, nparts, nullptr,
                               nullptr);
}

/* packet-header bits: MSB first, the byte after 0xFF carries 7 bits (T.800 B.10.1); reading past end gives 0 bits and
   sets overrun */
struct BitReader
{
  const uint8_t* cs;
  uint64_t p, end;
  uint32_t cur;
  int left;
  bool prev_ff, overrun;
  B2K_HD void init(const uint8_t* b, uint64_t at, uint64_t e)
  {
    cs = b;
    p = at;
    end = e;
    cur = 0;
    left = 0;
    prev_ff = overrun = false;
  }
  B2K_HD uint32_t get()
  {
    if(left == 0)
    {
      if(p >= end)
      {
        overrun = true;
        return 0;
      }
      cur = cs[p++];
      left = prev_ff ? 7 : 8;
      prev_ff = cur == 0xFF;
    }
    --left;
    return (cur >> left) & 1u;
  }
  B2K_HD uint32_t get_bits(int n)
  {
    uint32_t v = 0;
    for(int i = 0; i < n; ++i)
      v = (v << 1) | get();
    return v;
  }
  /* the header ends byte aligned; a final 0xFF is followed by one stuffed byte */
  B2K_HD uint64_t finish()
  {
    left = 0;
    if(prev_ff && p < end)
      ++p;
    prev_ff = false;
    return p;
  }
};

/* tag-tree decoder (T.800 B.10.2) over the node layout of tag_encode (leaves first, the root last), nodes initialised to
   {TAG_INF, 0}: true when leaf (x, y) is below threshold, its value then in *value */
B2K_HD bool tag_decode(BitReader& br, TagNode* nd, uint32_t w, uint32_t h, uint32_t nodes, int levels, uint32_t x, uint32_t y,
                       uint32_t threshold, uint32_t* value)
{
  uint32_t low = 0, base = nodes;
  TagNode* t = nullptr;
  for(int l = levels - 1; l >= 0; --l)
  {
    const uint32_t lw = tag_level_w(w, l);
    base -= lw * tag_level_w(h, l);
    t = &nd[base + (y >> l) * lw + (x >> l)];
    if(low > t->low)
      t->low = low;
    else
      low = t->low;
    uint32_t v = t->value;
    while(low < threshold && low < v)
    {
      if(br.get())
        v = low;
      else
        ++low;
    }
    t->value = v;
    t->low = low;
  }
  *value = t->value;
  return t->value < threshold;
}

/* One packet (one quality layer) at p of the tile part that ends at tp_end, as the host's parse_tile_packets reads it:
 * optional SOP, the header bits, EPH when COD asks for it, the body.  pk.band[].first index blk / kmax; tags holds
 * packet_tag_nodes(pk) nodes.  The packet's blocks in blk must be zero.  *p moves past the packet.  PR_NONE or the failure. */
template <class Packet>
B2K_HD uint32_t parse_packet(const uint8_t* cs, const Packet& pk, uint64_t* at, uint64_t tp_end, const uint8_t* kmax, ParsedBlock* blk,
                             TagNode* tags, bool sop, bool eph)
{
  uint64_t p = *at;
  if(sop && (int64_t)(tp_end - p) >= 6 && cs[p] == 0xFF && cs[p + 1] == 0x91)
    p += 6; /* SOP may be there when COD allows it (A.8.1) */
  BitReader br;
  br.init(cs, p, tp_end);
  if(br.get())
  {
    for(uint32_t b = 0; b < pk.nbands; ++b)
    {
      const uint32_t gw = pk.band[b].gw, gh = pk.band[b].gh, n = gw * gh;
      if(!n)
        continue;
      int levels = 0;
      const uint32_t nodes = tag_nodes(gw, gh, &levels);
      TagNode* incl = tags;
      TagNode* imsb = tags + nodes;
      for(uint32_t i = 0; i < 2 * nodes; ++i)
        tags[i] = TagNode{TAG_INF, 0};
      for(uint32_t i = 0; i < n; ++i)
      {
        const uint32_t x = i % gw, y = i / gw;
        uint32_t v = 0;
        if(!tag_decode(br, incl, gw, gh, nodes, levels, x, y, 1, &v))
          continue;
        uint32_t zbp = 0;
        for(uint32_t th = 1;; ++th)
        {
          if(tag_decode(br, imsb, gw, gh, nodes, levels, x, y, th, &v))
          {
            zbp = v;
            break;
          }
          if(th > 64 || br.overrun)
            return PR_ZBP;
        }
        uint32_t npass; /* number of passes, B.10.6 */
        if(!br.get())
          npass = 1;
        else if(!br.get())
          npass = 2;
        else
        {
          const uint32_t v2 = br.get_bits(2);
          if(v2 < 3)
            npass = 3 + v2;
          else
          {
            const uint32_t v5 = br.get_bits(5);
            npass = v5 < 31 ? 6 + v5 : 37 + br.get_bits(7);
          }
        }
        if(npass > 3)
          return PR_PASSES;
        int lblock = 3;
        while(br.get())
          if(++lblock > 32)
            return PR_LBLOCK;
        /* HT: the cleanup pass is one segment, the refinement passes another (T.814 B.10.7) */
        const uint32_t len1 = br.get_bits(lblock);
        const int l2 = lblock + floorlog2(npass - 1);
        const uint32_t len2 = npass > 1 ? br.get_bits(l2 < 32 ? l2 : 32) : 0;
        const uint32_t kb = kmax[pk.band[b].first + i];
        if(zbp > kb)
          return PR_ZBP_KMAX;
        if(len1 < 2)
          return PR_SHORT_CLEANUP;
        ParsedBlock& B = blk[pk.band[b].first + i];
        B.numbps = (uint8_t)(kb - zbp);
        B.numpasses = (uint8_t)npass;
        B.length = len1;
        B.length2 = len2;
      }
    }
  }
  if(br.overrun)
    return PR_HEADER_RUN;
  p = br.finish();
  if(eph)
  { /* EPH shall follow every packet header when COD says so (A.8.2) */
    if((int64_t)(tp_end - p) < 2 || cs[p] != 0xFF || cs[p + 1] != 0x92)
      return PR_EPH;
    p += 2;
  }
  /* the body: the included blocks' bytes in header order (a block is in one packet only, so numpasses marks it) */
  for(uint32_t b = 0; b < pk.nbands; ++b)
  {
    const uint32_t n = pk.band[b].gw * pk.band[b].gh;
    for(uint32_t i = 0; i < n; ++i)
    {
      ParsedBlock& B = blk[pk.band[b].first + i];
      if(!B.numpasses)
        continue;
      const uint32_t sz = B.length + B.length2; /* 32-bit, as the host parser adds them */
      if(tp_end - p < sz)
        return PR_BODY_RUN;
      B.offset = p;
      p += sz;
    }
  }
  *at = p;
  return PR_NONE;
}

/* One tile's packets from its tile parts, as the host's parse_tile_packets reads them.  packets[0, np) are the tile's
 * packets in code-stream order; tags: packet_tag_nodes of the largest of them.  blk must hold the tile's blocks cleared to
 * zero.  A packet never straddles tile parts; where the data ends the remaining packets stay uncoded.  PR_NONE or the
 * failure. */
template <class Packet>
B2K_HD uint32_t parse_tile(const uint8_t* cs, const PartRange* parts, uint32_t first_part, const Packet* packets, uint64_t np,
                           const uint8_t* kmax, ParsedBlock* blk, TagNode* tags, bool sop, bool eph)
{
  if(first_part == PART_NONE)
    return PR_NONE; /* a tile without a tile part decodes as all zero */
  uint32_t part = first_part;
  uint64_t p = parts[part].begin, tp_end = parts[part].end;
  for(uint64_t k = 0; k < np; ++k)
  {
    while(p == tp_end && parts[part].next != PART_NONE)
    {
      part = parts[part].next;
      p = parts[part].begin;
      tp_end = parts[part].end;
    }
    if(p == tp_end)
      break;
    if(const uint32_t r = parse_packet(cs, packets[k], &p, tp_end, kmax, blk, tags, sop, eph))
      return r;
  }
  return PR_NONE;
}

/* Packet starts from PLT (A.7.3).  A tile is indexed when every one of its tile parts carries PLT segments (Zplt 0, 1, ...
 * in its header), every Iplt entry is complete, at least 1 and at most 32 bits, the entries of each part add up to exactly
 * its packet data, and the parts hold exactly np entries together.  Then packet k of the tile starts at start[k], ends at
 * end[k] and lies in the tile part that ends at part_end[k] -- where the host's walk would meet it, provided each packet
 * before it ends where PLT says.  A PLT that is not understood only means "not indexed": the tile is walked. */
B2K_HD bool plt_index(const uint8_t* cs, const PartRange* parts, uint32_t first_part, uint64_t np, uint64_t* start, uint64_t* end,
                      uint64_t* part_end)
{
  if(first_part == PART_NONE)
    return false;
  uint64_t k = 0;
  for(uint32_t part = first_part; part != PART_NONE; part = parts[part].next)
  {
    const PartRange& R = parts[part];
    if(R.begin < R.hdr + 2 || R.begin > R.end)
      return false;
    uint64_t q = R.hdr, at = R.begin;
    const uint64_t sod = R.begin - 2;
    uint32_t z = 0;
    while(q + 4 <= sod)
    { /* the tile-part header's segments; their lengths were checked by locate_tile_parts */
      const uint32_t m = ((uint32_t)cs[q] << 8) | cs[q + 1], L = ((uint32_t)cs[q + 2] << 8) | cs[q + 3];
      const uint64_t seg_end = q + 2 + L;
      if(m == 0xFF58)
      {
        if(L < 3 || seg_end > sod || cs[q + 4] != z)
          return false;
        ++z;
        uint64_t v = 0;
        int nb = 0;
        for(uint64_t i = q + 5; i < seg_end; ++i)
        {
          v = (v << 7) | (cs[i] & 0x7F);
          if(++nb > 5 || v > 0xFFFFFFFFull)
            return false;
          if(cs[i] & 0x80)
            continue;
          if(v == 0 || k >= np || R.end - at < v)
            return false;
          start[k] = at;
          at += v;
          end[k] = at;
          part_end[k] = R.end;
          ++k;
          v = 0;
          nb = 0;
        }
        if(nb)
          return false; /* an entry that runs past its segment */
      }
      q = seg_end;
    }
    if(!z || at != R.end)
      return false;
  }
  return k == np;
}

/* which passes of one coded block are decoded: missing MSBs, passes and refinement length (passes > 1: it has refinement
   passes to decode).  The one statement of the rule: the device parser (k_t2_desc) and the host path (prepare_decode,
   engine.cu) both call it, so the decoder gets the same descriptor either way */
B2K_HD void block_decode_fields(const ParsedBlock& b, uint8_t kmax, uint8_t* mmsbs, uint8_t* passes, uint32_t* length2)
{
  const int nb = b.length ? b.numbps : 0;
  const int m = (int)kmax - nb;
  *mmsbs = (uint8_t)(m > 0 ? m : 0);
  /* ojph_block_decoder32.cpp L752-758, L790-803: no refinement bytes, or a cleanup pass already at bit-plane 1, leave
     nothing to refine */
  *passes = (b.length && b.numpasses > 1 && b.length2 > 0 && *mmsbs < 29) ? b.numpasses : 1;
  *length2 = *passes > 1 ? b.length2 : 0;
}

/* a windowed decode's rule for one block of the virtual coding: its rectangle (band coordinates) meets need = x0, y0, x1,
   y1 of resolution max(resno - 1, 0) (b2k_codestream_parse_window's need rectangles).  A block outside keeps length 0. */
B2K_HD bool window_needs(const uint32_t* need, uint32_t x0, uint32_t y0, uint32_t x1, uint32_t y1)
{
  return x0 < need[2] && x1 > need[0] && y0 < need[3] && y1 > need[1];
}

/* ---- batches: n code streams of one coding parsed by the same five launches -------------------------------------------
 * The plan (packets, tag-tree offsets, Kmax) is shared; every other piece of parse state is sliced per stream.  Stream s
 * lies at byte at of the arena (batch_arena_next) or, in a windowed batch, is read in place from its own buffer, its gathered
 * packet data going to byte at of the arena (window_arena_at); its tile parts in entries [parts0, parts0 + parts_cap) of the part
 * table (a prefix sum of part_capacity), and its blocks, packets, tiles and tag scratch in slice s of their arrays.
 * sot = 0: the stream failed before its tile parts and is not parsed. */
struct StreamDesc
{
  uint64_t at, len, sot, parts0, parts_cap;
  const uint8_t* base; /* the stream's own buffer, read in place (a windowed batch); NULL: the stream is byte `at` of the arena */
};
/* stream s's first byte: its own buffer, or its place in the arena */
B2K_HD const uint8_t* stream_bytes(const uint8_t* arena, const StreamDesc& D) { return D.base ? D.base : arena + D.at; }
/* item i of stream s in a launch over n streams of `per` items each, flattened as g = s * per + i */
struct StreamItem
{
  uint32_t s;
  uint64_t i;
};
B2K_HD StreamItem split_stream_item(uint64_t g, uint64_t per) { return StreamItem{(uint32_t)(g / per), g % per}; }
/* the tile-part table a stream of len bytes over ntiles tiles may need: every tile part takes at least the 12 bytes of its
   SOT, and a tile has at most 256 */
B2K_HD uint64_t part_capacity(uint64_t len, uint32_t ntiles)
{
  const uint64_t a = len / 12 + 1, b = 256ull * ntiles;
  return a < b ? a : b;
}
/* where the stream after one of len bytes at `at` starts in a batch arena: the next 256-byte boundary, the base alignment
   the single-stream decode gives its stream */
B2K_HD uint64_t batch_arena_next(uint64_t at, uint64_t len) { return (at + len + 255) & ~(uint64_t)255; }

/* the main-header prefix a batch first reads of each stream; a header that runs past it is read again with twice as many
   bytes, all such streams together */
constexpr uint64_t BATCH_HEADER_PREFIX = 4096;

/* one stream's parse status.  tile_err: (tile << 8) | reason of the lowest failing tile, NO_TILE_ERROR when none */
constexpr unsigned long long NO_TILE_ERROR = ~0ull;
struct ParseStatus
{
  unsigned long long tile_err;
  uint32_t locate;             /* the tile-part walk's reason (PR_SKIPPED: the stream is not parsed) */
  uint32_t nparts;
  uint32_t refinement;         /* some block has refinement passes to decode */
  uint32_t walked;             /* tiles with data parsed by the walk */
  uint32_t indexed;            /* tiles whose packets were parsed from their PLT starts */
  unsigned long long bytes;    /* packet data of the recorded tile parts */
};
/* the kernels' threads update a stream's counters together; the host runs them one after another */
B2K_HD void status_add(uint32_t* p, uint32_t v)
{
#ifdef __CUDA_ARCH__
  atomicAdd(p, v);
#else
  *p += v;
#endif
}
B2K_HD void status_or(uint32_t* p, uint32_t v)
{
#ifdef __CUDA_ARCH__
  atomicOr(p, v);
#else
  *p |= v;
#endif
}
B2K_HD void status_min(unsigned long long* p, unsigned long long v)
{
#ifdef __CUDA_ARCH__
  atomicMin(p, v);
#else
  if(v < *p)
    *p = v;
#endif
}
/* 0, or the stream's failure as parse_reason_* take it */
B2K_HD uint32_t status_reason(const ParseStatus& st)
{
  return st.locate != PR_NONE ? st.locate : st.tile_err != NO_TILE_ERROR ? (uint32_t)(st.tile_err & 0xFF) : (uint32_t)PR_NONE;
}

/* The five kernels' threads over a batch (t2_decode.cu runs them as kernels, tests/t2_batch_check.cpp on the host in the same
 * order).  cs is the arena; stream s is sd[s] (stream_bytes), its status status[s].  A stream whose status is set before the first step
 * (PR_SKIPPED) is left alone.  The per-stream arrays are sliced: head / last (bt = box.tiles() each), count (ntiles each),
 * indexed / marked (plan tiles each), blk (nblocks each), start / end / part_end (np each), tags (tag_nodes each). */
/* step 1, thread s: the tile-part walk of stream s */
B2K_HD void batch_locate(const uint8_t* cs, const StreamDesc* sd, uint32_t s, uint32_t ntiles, const TileBox& box, PartRange* parts,
                         uint32_t* head, uint32_t* last, uint32_t* count, uint64_t* body_at, ParseStatus* status)
{
  if(status[s].locate != PR_NONE)
    return;
  const StreamDesc D = sd[s];
  const uint64_t bt = box.tiles();
  uint32_t np = 0;
  uint64_t bytes = 0;
  status[s].locate = locate_tile_parts_box(stream_bytes(cs, D), D.len, D.sot, ntiles, box, parts + D.parts0, D.parts_cap, head + s * bt, last + s * bt,
                                           count + (uint64_t)s * ntiles, &np, body_at ? body_at + D.parts0 : nullptr, &bytes);
  status[s].nparts = np;
  status[s].bytes = bytes;
}

/* step 2, thread g = s * ntiles + t (ntiles: the plan's tiles): tile t's blocks cleared, its PLT packet starts */
template <class Part>
B2K_HD void batch_plt(const uint8_t* cs, const StreamDesc* sd, uint64_t g, const PartRange* parts, const uint32_t* head, const Part* tiles,
                      uint32_t ntiles, const uint64_t* tile_first, uint64_t nblocks, uint64_t np, ParsedBlock* blk, uint64_t* start,
                      uint64_t* end, uint64_t* part_end, uint32_t* indexed, uint32_t* marked, ParseStatus* status)
{
  const StreamItem it = split_stream_item(g, ntiles);
  const uint32_t s = it.s, t = (uint32_t)it.i;
  if(status[s].locate != PR_NONE)
    return;
  blk += s * nblocks;
  for(uint64_t i = tile_first[t]; i < tile_first[t + 1]; ++i)
    blk[i] = ParsedBlock{};
  const Part T = tiles[t];
  const uint64_t o = s * np;
  const bool ix = plt_index(stream_bytes(cs, sd[s]), parts + sd[s].parts0, head[g], T.p1 - T.p0, start + o + T.p0, end + o + T.p0, part_end + o + T.p0);
  indexed[g] = ix;
  marked[g] = 0;
  if(ix && T.p1 > T.p0)
    status_add(&status[s].indexed, 1u);
}

/* step 3, thread g = s * np + k: packet k of stream s from its PLT start, when its tile is indexed */
template <class Packet>
B2K_HD void batch_packet(const uint8_t* cs, const StreamDesc* sd, uint64_t g, const Packet* packets, uint64_t np, const uint32_t* pkt_tile,
                         uint32_t ntiles, uint64_t nblocks, uint64_t tag_nodes, const uint32_t* indexed, const uint64_t* start,
                         const uint64_t* end, const uint64_t* part_end, const uint8_t* kmax, ParsedBlock* blk, TagNode* tags,
                         uint32_t* marked, bool sop, bool eph, const ParseStatus* status)
{
  const StreamItem it = split_stream_item(g, np);
  const uint32_t s = it.s;
  if(status[s].locate != PR_NONE)
    return;
  const uint64_t t = (uint64_t)s * ntiles + pkt_tile[it.i];
  if(!indexed[t])
    return;
  uint64_t at = start[g];
  const Packet& P = packets[it.i];
  if(parse_packet(stream_bytes(cs, sd[s]), P, &at, part_end[g], kmax, blk + s * nblocks, tags + s * tag_nodes + P.tag_at, sop, eph) != PR_NONE ||
     at != end[g])
    marked[t] = 1; /* the walk decides */
}

/* step 4, thread g = s * ntiles + t: the walk of tile t of stream s when it is not indexed or is marked; the lowest failing
   tile's reason is kept */
template <class Part, class Packet>
B2K_HD void batch_walk(const uint8_t* cs, const StreamDesc* sd, uint64_t g, const PartRange* parts, const uint32_t* head, const Part* tiles,
                       uint32_t ntiles, const Packet* packets, const uint8_t* kmax, const uint64_t* tile_first, uint64_t nblocks,
                       uint64_t tag_nodes, ParsedBlock* blk, TagNode* tags, const uint32_t* indexed, const uint32_t* marked, bool sop,
                       bool eph, ParseStatus* status)
{
  const StreamItem it = split_stream_item(g, ntiles);
  const uint32_t s = it.s, t = (uint32_t)it.i;
  if(status[s].locate != PR_NONE || (indexed[g] && !marked[g]))
    return;
  const Part T = tiles[t];
  if(T.p1 == T.p0)
    return;
  blk += s * nblocks;
  if(marked[g]) /* the packets parsed from PLT may have left fields behind */
    for(uint64_t i = tile_first[t]; i < tile_first[t + 1]; ++i)
      blk[i] = ParsedBlock{};
  if(head[g] != PART_NONE)
    status_add(&status[s].walked, 1u);
  const uint32_t r = parse_tile(stream_bytes(cs, sd[s]), parts + sd[s].parts0, head[g], packets + T.p0, T.p1 - T.p0, kmax, blk,
                                tags + s * tag_nodes + packets[T.p0].tag_at, sop, eph);
  if(r != PR_NONE)
    status_min(&status[s].tile_err, ((unsigned long long)t << 8) | r);
}

/* step 5, thread g = s * ncoded + k: what descriptor g of coded block k (enumeration index coded[k]) of stream s decodes:
   the parsed block, or an empty one when the stream failed or was not parsed (all-zero coefficients) */
B2K_HD ParsedBlock batch_block(const ParsedBlock* blk, uint64_t nblocks, const uint32_t* coded, uint64_t g, uint64_t ncoded,
                               const ParseStatus* status, uint32_t* s_out)
{
  const StreamItem it = split_stream_item(g, ncoded);
  *s_out = it.s;
  return status_reason(status[it.s]) == PR_NONE ? blk[it.s * nblocks + coded[it.i]] : ParsedBlock{};
}

/* where stream offset off of a parsed block of the tile whose first part is first lies once the tile parts' packet data
   are laid end to end at body_at[part] (locate_tile_parts_box); a parsed block lies inside one of its tile's parts */
B2K_HD uint64_t gathered_offset(const PartRange* parts, uint32_t first, const uint64_t* body_at, uint64_t off)
{
  for(uint32_t p = first; p != PART_NONE; p = parts[p].next)
    if(off >= parts[p].begin && off < parts[p].end)
      return body_at[p] + (off - parts[p].begin);
  return 0;
}

/* ---- windowed batches: n streams parsed against the plan of one box coding, read in place -----------------------------
 * Every stream wants the same tile box; its tile parts are recorded under their box tile index (batch_locate with the box
 * and body_at), and only their packet data is gathered into the arena, stream s's at sd[s].at (window_arena_at). */
constexpr uint32_t WINDOW_MAX_RES = 33; /* resolutions of a coding (B2K_MAX_RES) */
/* a coded block of the virtual coding (the plan's, shared by every stream): its box tile, the need rectangle that applies
   to it (resolution max(resno - 1, 0)) and its rectangle in band coordinates */
struct WinBlock
{
  uint32_t tile, res, x0, y0, x1, y1;
};
/* one stream's need rectangles, one per resolution of the virtual coding; n = 0: no filter */
struct NeedRects
{
  uint32_t n;
  uint32_t r[WINDOW_MAX_RES][4];
};

/* the arena bytes stream s's gathered packet data takes: its wanted parts' packet data up to the next 256-byte boundary
   (batch_arena_next), none when its tile-part walk failed or it is not parsed */
B2K_HD uint64_t window_gathered_bytes(const ParseStatus& st) { return st.locate == PR_NONE ? batch_arena_next(0, st.bytes) : 0; }

/* where each stream's gathered data starts: sd[s].at for s in [s0, s1), from `at` on (the streams laid end to end) */
B2K_HD uint64_t window_arena_at(StreamDesc* sd, const ParseStatus* status, uint32_t s0, uint32_t s1, uint64_t at)
{
  for(uint32_t s = s0; s < s1; ++s)
  {
    sd[s].at = at;
    at += window_gathered_bytes(status[s]);
  }
  return at;
}

/* step 5 of a windowed batch, thread g = s * ncoded + k: batch_block's block, left uncoded when stream s's need rectangles
   leave it out, and *slot_off: where its bytes lie in the arena once k_t2_gather has put stream s's wanted parts' packet
   data end to end at sd[s].at.  win[k] is coded block k's; head is sliced per stream (bt box tiles each), parts and
   body_at from sd[s].parts0 */
B2K_HD ParsedBlock window_block(const ParsedBlock* blk, uint64_t nblocks, const uint32_t* coded, uint64_t g, uint64_t ncoded,
                                const ParseStatus* status, const StreamDesc* sd, const WinBlock* win, const NeedRects* need,
                                const PartRange* parts, const uint32_t* head, uint32_t bt, const uint64_t* body_at, uint32_t* s_out,
                                uint64_t* slot_off)
{
  ParsedBlock b = batch_block(blk, nblocks, coded, g, ncoded, status, s_out);
  const uint32_t s = *s_out;
  const WinBlock w = win[g % ncoded];
  const NeedRects& N = need[s];
  if(b.length && N.n && !window_needs(N.r[w.res], w.x0, w.y0, w.x1, w.y1))
    b = ParsedBlock{};
  const StreamDesc& D = sd[s];
  *slot_off = D.at + (b.length ? gathered_offset(parts + D.parts0, head[(uint64_t)s * bt + w.tile], body_at + D.parts0, b.offset) : 0);
  return b;
}

/* the gather of a windowed batch, item g = s * per + j (per: the most parts a stream recorded): part j of stream s, when
   stream s parsed and recorded it -- len bytes from *src to arena byte *dst.  False: nothing to copy */
B2K_HD bool window_gather_part(const StreamDesc* sd, const PartRange* parts, const uint64_t* body_at, const ParseStatus* status, uint64_t g,
                               uint64_t per, const uint8_t** src, uint64_t* dst, uint64_t* len)
{
  const StreamItem it = split_stream_item(g, per);
  const StreamDesc& D = sd[it.s];
  if(status_reason(status[it.s]) != PR_NONE || it.i >= status[it.s].nparts)
    return false;
  const PartRange R = parts[D.parts0 + it.i];
  if(R.end <= R.begin)
    return false;
  *src = D.base + R.begin;
  *dst = D.at + body_at[D.parts0 + it.i];
  *len = R.end - R.begin;
  return true;
}

} // namespace t2
} // namespace b2k
