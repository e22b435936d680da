/*
 * grok_b200/csrc/codestream.cpp -- HTJ2K codestream assembly and parsing on the host (SURVEY.md section 8f, row N1):
 * the T2 step between the block coder's output (b2k_result) and a file a JPEG 2000 decoder reads.
 *
 * Replaces (reference, CPU):
 *   main header   codestream/compress/CodeStreamCompress.cpp L1064-1098 (SOC, SIZ, CAP, COD, QCD, TLM order),
 *                 codestream/markers/SIZMarker.cpp, t2/quantizer/part15/QuantizerOJPH.cpp L259-330 (CAP, MAGB)
 *   tile parts    CodeStreamCompress::writeTilePart L1099-, codestream/markers/SOTMarker.cpp,
 *                 PLMarker.cpp (PLT), TLMMarker.cpp (TLM)
 *   packets       t2/T2Compress.cpp L261-489 (header: inclusion / zero-bit-plane tag trees, pass count, Lblock,
 *                 lengths; body), t2/TagTree.h, t1_t2 BitIO (bit stuffing after 0xFF)
 *   parsing       codestream/decompress/CodeStreamDecompress_ReadMarkers.cpp, t2/PacketParser.cpp,
 *                 t1/codeblock/CodeblockDecompressImpl.h L205-420 (HT segments: cleanup | refinement, T.814 B.10.7)
 * Scope: what this engine's path produces and consumes -- one quality layer, any of the five progression orders,
 * any number of tile parts per tile (in order), SOP / EPH markers, no COC/QCC/POC/RGN/PPM/PPT, HT code blocks with 1..3
 * passes, the HT quantiser's QCD.  Anything else parses as "not handled".
 * Written from the standard's rules (ITU-T T.800 Annex A/B, T.814 Annex A/B), not transcribed from the reference;
 * tests decode the output with an independent decoder (OpenJPEG via Pillow / OpenCV) -- tests/test_codestream.py.
 */
#include "geometry.h"
#include "b2k_internal.h"
#include "t2_packet.h"
#include "t2_plan.h"
#include "t2_write.h"

#include <algorithm>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

using namespace b2k;
using t2::floorlog2;

extern "C" const char* b2k_last_error(void);
void b2k_set_error(const char* msg); /* engine.cu */

namespace
{

/* ---- packet-header bit reader: MSB first, the byte after 0xFF carries 7 bits (T.800 B.10.1); the writer is
   t2::BitWriter ---------------------------------------------------------------------------------------------------- */
struct BitReader
{
  const uint8_t* p;
  const uint8_t* end;
  uint32_t cur = 0;
  int left = 0;
  bool prev_ff = false, overrun = false;
  BitReader(const uint8_t* b, const uint8_t* e) : p(b), end(e) {}
  uint32_t get()
  {
    if(left == 0)
    {
      if(p >= end)
      {
        overrun = true;
        return 0;
      }
      cur = *p++;
      left = prev_ff ? 7 : 8;
      prev_ff = (cur == 0xFF);
    }
    --left;
    return (cur >> left) & 1u;
  }
  uint32_t get_bits(int n)
  {
    uint32_t v = 0;
    for(int i = 0; i < n; ++i)
      v = (v << 1) | get();
    return v;
  }
  /* header ends byte aligned; a final 0xFF is followed by one stuffed byte */
  const uint8_t* finish()
  {
    left = 0;
    if(prev_ff && p < end)
      ++p;
    prev_ff = false;
    return p;
  }
};

/* ---- tag-tree decoder (T.800 B.10.2); the encoder is t2::tag_encode ---------------------------------------- */
struct TagTree
{
  struct Node
  {
    int parent;
    uint32_t value, low;
    bool known;
  };
  std::vector<Node> nodes;
  uint32_t w = 0, h = 0;
  static constexpr uint32_t INF = 0x7FFFFFFFu;
  void init(uint32_t w_, uint32_t h_)
  {
    w = w_;
    h = h_;
    nodes.clear();
    std::vector<std::pair<uint32_t, uint32_t>> dims;
    uint32_t lw = w, lh = h;
    for(;;)
    {
      dims.push_back({lw, lh});
      if(lw <= 1 && lh <= 1)
        break;
      lw = (lw + 1) / 2;
      lh = (lh + 1) / 2;
    }
    size_t total = 0;
    std::vector<size_t> base;
    for(auto& d : dims)
    {
      base.push_back(total);
      total += (size_t)d.first * d.second;
    }
    nodes.assign(total, Node{-1, INF, 0, false});
    for(size_t l = 0; l + 1 < dims.size(); ++l)
      for(uint32_t y = 0; y < dims[l].second; ++y)
        for(uint32_t x = 0; x < dims[l].first; ++x)
          nodes[base[l] + (size_t)y * dims[l].first + x].parent = (int)(base[l + 1] + (size_t)(y / 2) * dims[l + 1].first + x / 2);
  }
  /* true if the leaf's value is < threshold (then nodes[leaf].value holds it) */
  bool decode(BitReader& br, uint32_t leaf, uint32_t threshold)
  {
    int path[32], np = 0;
    for(int n = (int)leaf; n >= 0; n = nodes[n].parent)
      path[np++] = n;
    uint32_t low = 0;
    for(int i = np - 1; i >= 0; --i)
    {
      Node& nd = nodes[path[i]];
      if(low > nd.low)
        nd.low = low;
      else
        low = nd.low;
      while(low < threshold && low < nd.value)
      {
        if(br.get())
          nd.value = low;
        else
          ++low;
      }
      nd.low = low;
    }
    return nodes[leaf].value < threshold;
  }
};

/* ---- packets of a tile in LRCP order, with where their blocks sit in the tile's enumeration ---------------- */
typedef t2::BandGrid PacketBand; /* first block (index into the tile's blocks), code-block grid of the precinct */
struct Packet
{
  uint16_t comp;
  uint8_t resno, nbands;
  uint32_t precno;
  uint32_t xpos, ypos; /* where the position-driven progressions meet this precinct on the reference grid (B.12.1.3-5) */
  PacketBand band[3] = {};
};
/* prog: 0 LRCP, 1 RLCP, 2 RPCL, 3 PCRL, 4 CPRL (one layer, so the first two coincide) */
void tile_packets(const b2k_coding& cp, const Rect& tile, std::vector<Packet>& lrcp, uint32_t& nblocks, int prog = 0)
{
  const int numres = cp.numres;
  std::vector<std::vector<Packet>> per_res_comp((size_t)numres * cp.numcomps);
  nblocks = walk_precincts(cp, tile, [&](const PrecinctBand& pb) {
    std::vector<Packet>& pk = per_res_comp[(size_t)pb.resno * cp.numcomps + pb.comp];
    if(pb.band_index == 0)
      pk.push_back(Packet{pb.comp, pb.resno, pb.nbands, pb.precno, pb.xpos, pb.ypos});
    pk[pb.precno].band[pb.band_index] = PacketBand{pb.first, pb.gw, pb.gh};
  });
  lrcp.clear();
  for(int resno = 0; resno < numres; ++resno)
    for(uint16_t comp = 0; comp < cp.numcomps; ++comp)
      for(const Packet& p : per_res_comp[(size_t)resno * cp.numcomps + comp])
        lrcp.push_back(p);
  if(prog >= 2)
  { /* the position-driven orders are the nested loops of B.12.1.3-5 read as sort keys (stable: ties keep LRCP order) */
    auto key = [prog](const Packet& a) {
      struct K
      {
        uint64_t k[4];
      } k;
      if(prog == 2)
        k = {{a.resno, a.ypos, a.xpos, a.comp}};
      else if(prog == 3)
        k = {{a.ypos, a.xpos, a.comp, a.resno}};
      else
        k = {{a.comp, a.ypos, a.xpos, a.resno}};
      return k;
    };
    std::stable_sort(lrcp.begin(), lrcp.end(), [&](const Packet& a, const Packet& b) {
      const auto ka = key(a), kb = key(b);
      for(int i = 0; i < 4; ++i)
        if(ka.k[i] != kb.k[i])
          return ka.k[i] < kb.k[i];
      return false;
    });
  }
}

void put16(std::vector<uint8_t>& o, uint32_t v)
{
  o.push_back((uint8_t)(v >> 8));
  o.push_back((uint8_t)v);
}
void put32(std::vector<uint8_t>& o, uint32_t v)
{
  put16(o, v >> 16);
  put16(o, v & 0xFFFF);
}

/* Ccap15's magnitude bound from the quantiser (QuantizerOJPH::get_MAGBp L259-280, ::write L281-330); q[comp][band] */
uint32_t magb_code(const b2k_coding& cp, const std::vector<std::vector<BandQuant>>& qc)
{
  uint32_t B = 0;
  const int ndecomp = cp.numres - 1;
  /* Grok's own tables and a quality factor's: the reference computes MAGB from component 0's steps only (a quality
     factor's are pushed into its quantiser from component 0, CodeStreamCompress.cpp L617-626) */
  const bool quirk = cp.irreversible && (cp.qfactor || (!cp.qcd_explicit && !cp.qcc_mask));
  for(size_t c = 0; c < (quirk ? 1 : qc.size()); ++c)
  {
    const std::vector<BandQuant>& q = qc[c];
    for(size_t i = 0; i < q.size(); ++i)
    {
      if(!cp.irreversible)
        B = std::max<uint32_t>(B, (uint32_t)q[i].expn + cp.numgbits - 1u);
      else if(!quirk)
      { /* foreign step sizes: the bound T.814 asks for (the "scalar expounded" branch of get_MAGBp) */
        const int nb = ndecomp - (i ? (int)((i - 1) / 3) : 0);
        B = std::max<uint32_t>(B, (uint32_t)std::max(0, (int)q[i].expn + (int)cp.numgbits - nb));
      }
      else
      { /* What the reference actually writes: its Sqcd never carries the quantisation style (Quantizer.cpp L24), so
           get_MAGBp takes the reversible branch and scans the first 3*ndecomp+1 BYTES of the 16-bit (exponent << 11 |
           mantissa) array through the u8/u16 union (Quantizer.h L52-57, little endian).  A looser bound than the
           standard's, still a valid one; mirrored so that main headers stay byte-identical to grk_compress's. */
        if(i >= (size_t)(3 * ndecomp + 1))
          break;
        const BandQuant& w = q[i / 2];
        const uint32_t word = ((uint32_t)w.expn << 11) | (uint32_t)w.mant;
        const uint32_t byte = (i & 1) ? (word >> 8) & 0xFF : word & 0xFF;
        B = std::max<uint32_t>(B, (byte >> 3) + cp.numgbits - 1u);
      }
    }
  }
  if(B <= 8)
    return 0;
  if(B < 28)
    return B - 8;
  if(B < 48)
    return 13 + (B >> 2);
  return 31;
}

/* Sqcd / Sqcc and the band values of one component's table (A.6.4, A.6.5) */
void put_quant(const b2k_coding& cp, const std::vector<BandQuant>& q, std::vector<uint8_t>& o)
{
  o.push_back((uint8_t)((cp.numgbits << 5) | (cp.irreversible ? 2 : 0)));
  for(const BandQuant& b : q)
  {
    if(cp.irreversible)
      put16(o, ((uint32_t)b.expn << 11) | b.mant);
    else
      o.push_back((uint8_t)(b.expn << 3));
  }
}

void write_main_header(const b2k_coding& cp, const TileGrid& g, const std::vector<std::vector<BandQuant>>& q, std::vector<uint8_t>& o,
                       int prog, bool sop, bool eph)
{
  put16(o, 0xFF4F); /* SOC */
  put16(o, 0xFF51); /* SIZ (T.800 A.5.1) */
  put16(o, 38 + 3 * cp.numcomps);
  put16(o, 0x4000); /* Rsiz: bit 14 = Part 15 capabilities, detailed in CAP */
  put32(o, cp.x1);
  put32(o, cp.y1);
  put32(o, cp.x0);
  put32(o, cp.y0);
  put32(o, g.tw);
  put32(o, g.th);
  put32(o, g.tx0);
  put32(o, g.ty0);
  put16(o, cp.numcomps);
  for(int c = 0; c < cp.numcomps; ++c)
  {
    o.push_back((uint8_t)((cp.prec - 1) | (cp.sgnd ? 0x80 : 0)));
    o.push_back(1);
    o.push_back(1);
  }
  put16(o, 0xFF50); /* CAP (T.814 A.3) */
  put16(o, 8);
  put32(o, 0x00020000u);                                        /* Pcap: bit 15 -> Ccap15 follows */
  put16(o, (cp.irreversible ? 0x0020u : 0u) | magb_code(cp, q)); /* HTONLY, single HT set, RGN free, homogeneous */
  bool user_prec = false;
  for(int r = 0; r < cp.numres; ++r)
    user_prec |= (cp.prcw_exp[r] && cp.prcw_exp[r] != 15) || (cp.prch_exp[r] && cp.prch_exp[r] != 15);
  put16(o, 0xFF52); /* COD (A.6.1) */
  put16(o, 12 + (user_prec ? cp.numres : 0));
  o.push_back((uint8_t)((user_prec ? 1 : 0) | (sop ? 2 : 0) | (eph ? 4 : 0)));
  o.push_back((uint8_t)prog); /* progression order */
  put16(o, 1);    /* layers */
  o.push_back(cp.mct ? 1 : 0);
  o.push_back((uint8_t)(cp.numres - 1));
  o.push_back((uint8_t)(cp.cblkw_exp - 2));
  o.push_back((uint8_t)(cp.cblkh_exp - 2));
  o.push_back((uint8_t)(0x40 | (cp.cblk_sty & 0x08))); /* HT code blocks (+ stripe causal) */
  o.push_back(cp.irreversible ? 0 : 1);
  if(user_prec)
    for(int r = 0; r < cp.numres; ++r)
      o.push_back((uint8_t)(((cp.prch_exp[r] ? cp.prch_exp[r] : 15) << 4) | (cp.prcw_exp[r] ? cp.prcw_exp[r] : 15)));
  const uint32_t nb = (uint32_t)q[0].size(), vals = cp.irreversible ? 2 * nb : nb;
  put16(o, 0xFF5C); /* QCD (A.6.4): component 0's table */
  put16(o, 3 + vals);
  put_quant(cp, q[0], o);
  for(int c = 1; c < cp.numcomps; ++c)
    if(!same_quant(q[c], q[0]))
    { /* QCC (A.6.5) for every other component whose table differs, in component order; Cqcc is 8 bits (Csiz < 257) */
      put16(o, 0xFF5D);
      put16(o, 4 + vals);
      o.push_back((uint8_t)c);
      put_quant(cp, q[c], o);
    }
}

/* where a tile's tile parts end (packet indices): one part for the whole tile, or one per run of packets of the same
   resolution; a tile without packets still has one (empty) tile part */
std::vector<size_t> tile_part_ends(const std::vector<uint8_t>& res_of, bool split_res)
{
  std::vector<size_t> ends;
  const size_t np = res_of.size();
  size_t p = 0;
  do
  {
    const uint8_t r0 = np ? res_of[p] : 0;
    while(p < np && (!split_res || res_of[p] == r0))
      ++p;
    ends.push_back(p);
  } while(p < np);
  return ends;
}

/* the main header for `flags`, with the TLM segments of nparts tile parts (entries zero) behind it: where TLM starts */
uint64_t main_header(const b2k_coding& cp, uint32_t flags, uint64_t nparts, std::vector<uint8_t>& head)
{
  write_main_header(cp, tile_grid(cp), component_quant(cp), head, (int)((flags >> 8) & 7), (flags & B2K_CS_SOP) != 0, (flags & B2K_CS_EPH) != 0);
  const uint64_t at = head.size();
  if(flags & B2K_CS_TLM)
  {
    head.resize(at + t2::tlm_bytes(nparts), 0);
    for(uint64_t e0 = 0; e0 < nparts; e0 += t2::TLM_PER_SEGMENT)
      t2::put_tlm_segment(head.data() + at, e0, std::min<uint64_t>(t2::TLM_PER_SEGMENT, nparts - e0));
  }
  return at;
}

/* what b2k_codestream_write checks before it looks at a block: 0, or -1 with the error set */
int check_whole_image(const b2k_coding& cp, uint32_t num_tiles, uint32_t flags)
{
  if(const char* why = unsupported_reason(cp))
  {
    b2k_set_error(why);
    return -1;
  }
  const TileGrid g = tile_grid(cp);
  const uint32_t ntiles = g.nx * g.ny;
  if(num_tiles != ntiles)
  {
    b2k_set_error("the result does not hold every tile of the image (gather the shards first)");
    return -1;
  }
  if(ntiles > 65535)
  {
    b2k_set_error("more than 65535 tiles");
    return -1;
  }
  if(((flags >> 8) & 7) > 4)
  {
    b2k_set_error("unknown progression order");
    return -1;
  }
  return 0;
}

/* the plan of tiles t % tile_mod == tile_rem of cp, whose blocks `blocks` holds in tile order; the tiles are planned on the
   host pool.  0; 1 when the table is not those tiles' blocks in tile order (no error set); -1 with the error of the first
   tile the plan declines, `plan` then holding the packets and tile parts of the tiles before it. */
int plan_tiles(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t tile_mod, uint32_t tile_rem,
               t2::Plan& plan)
{
  plan = t2::Plan();
  plan.flags = flags;
  const TileGrid g = tile_grid(cp);
  std::vector<uint32_t> mine;
  for(uint32_t t = tile_rem; t < g.nx * g.ny; t += tile_mod)
    mine.push_back(t);
  std::vector<uint64_t> first(mine.size() + 1);
  uint64_t i = 0;
  for(size_t k = 0; k < mine.size(); ++k)
  {
    first[k] = i;
    while(i < nblocks && blocks[i].tile == mine[k])
      ++i;
  }
  first[mine.size()] = i;
  if(i != nblocks)
    return 1;
  const int prog = (int)((flags >> 8) & 7);
  const bool split_res = (flags & B2K_CS_TPARTS_R) != 0 && prog <= 2; /* a tile part per resolution needs a resolution-major order */
  struct TileSlice /* one tile's packets and parts, numbered within the tile */
  {
    std::vector<t2::DevPacket> packets;
    std::vector<t2::DevPart> parts;
    uint64_t hdr_bytes = 0, tag_nodes = 0;
    const char* err = nullptr;
  };
  std::vector<TileSlice> tiles(mine.size());
  b2k_host_parallel(mine.size(), [&](size_t k) {
    TileSlice& T = tiles[k];
    std::vector<Packet> pkts;
    uint32_t expect = 0;
    tile_packets(cp, tile_rect(cp, g, mine[k]), pkts, expect, prog);
    if(expect != first[k + 1] - first[k])
    {
      T.err = "block table does not match the tile's enumeration";
      return;
    }
    uint8_t kmax = 0;
    for(uint64_t b = first[k]; b < first[k + 1]; ++b)
      kmax = std::max(kmax, blocks[b].kmax);
    std::vector<uint8_t> res_of;
    for(size_t p = 0; p < pkts.size(); ++p)
    {
      const Packet& pk = pkts[p];
      t2::DevPacket d{};
      for(int b = 0; b < pk.nbands; ++b)
        d.band[b] = t2::BandGrid{(uint32_t)first[k] + pk.band[b].first, pk.band[b].gw, pk.band[b].gh};
      d.nbands = pk.nbands;
      d.sop = (uint32_t)(p & 0xFFFF);
      const uint64_t cap = t2::packet_header_bound(pk.band, pk.nbands, kmax);
      if(cap > 0xFFFFFFFFull)
      {
        T.err = "packet longer than 4 GiB";
        return;
      }
      d.hdr_cap = (uint32_t)cap;
      d.hdr_at = T.hdr_bytes;
      d.tag_at = T.tag_nodes;
      T.hdr_bytes += cap;
      T.tag_nodes += t2::packet_tag_nodes(pk.band, pk.nbands);
      T.packets.push_back(d);
      res_of.push_back(pk.resno);
    }
    const std::vector<size_t> ends = tile_part_ends(res_of, split_res);
    if(ends.size() > 255)
    {
      T.err = "more than 255 tile parts";
      return;
    }
    for(size_t j = 0, p0 = 0; j < ends.size(); p0 = ends[j++])
      T.parts.push_back(t2::DevPart{p0, ends[j], mine[k], (uint32_t)j, (uint32_t)ends.size()});
  });
  for(TileSlice& T : tiles)
  {
    if(T.err)
    {
      b2k_set_error(T.err);
      return -1;
    }
    const uint64_t p_first = plan.packets.size();
    for(t2::DevPacket& d : T.packets)
    {
      d.hdr_at += plan.hdr_bytes;
      d.tag_at += plan.tag_nodes;
      plan.packets.push_back(d);
    }
    for(t2::DevPart& d : T.parts)
      plan.parts.push_back(t2::DevPart{p_first + d.p0, p_first + d.p1, d.tile, d.index, d.count});
    plan.hdr_bytes += T.hdr_bytes;
    plan.tag_nodes += T.tag_nodes;
  }
  plan.tlm_at = main_header(cp, flags, plan.parts.size(), plan.head);
  return 0;
}

/* the caller's block table as the writer's block source (t2_write.h): a block is in its packet when it has passes and
   bytes; its body is the cleanup segment and, with more than one pass, the refinement segment, at `offset` in the arena */
struct TableBlocks
{
  const b2k_block* blk;
  uint64_t arena; /* bytes in the arena */
  uint64_t slots; /* dst has an entry per block */
  TableBlocks stream(uint32_t) const { return *this; }
  t2::BlockCode operator()(uint32_t i) const
  {
    const b2k_block& B = blk[i];
    return t2::BlockCode{B.length, B.length2, B.numpasses, B.numbps, B.kmax};
  }
  int64_t slot(uint32_t i) const { return blk[i].numpasses && blk[i].length ? (int64_t)i : -1; }
  uint64_t bytes(int64_t i) const { return (uint64_t)blk[i].length + (blk[i].numpasses > 1 ? blk[i].length2 : 0); }
  bool failed(int64_t i) const { return blk[i].offset + bytes(i) > arena; }
};

/* n elements, not cleared */
template <class T>
std::unique_ptr<T[]> scratch(uint64_t n)
{
  return std::unique_ptr<T[]>(new T[n]);
}

/* the text of a packet's error word: the first of its faults in the order the packet is written */
const char* packet_error(uint32_t e)
{
  return (e & t2::WERR_RANGE)       ? "code block outside the writer's range (bit planes / passes)"
         : (e & t2::WERR_HDR_BOUND) ? "packet header longer than its bound"
         : (e & t2::WERR_BLOCK)     ? "block offsets exceed the byte arena"
                                    : "packet longer than 4 GiB";
}

/* The host writer: the code stream of plan P and r's blocks, as one stream of the device writer's steps (t2_write.h) on the
   host pool; then each block's bytes copied once, from r's arena to the place write_packet gave it.  whole: main header,
   tile parts and EOC; else a shard's tile parts alone, at out + tile_at[k] when tile_at is given (tile_bytes[k] their
   lengths).  plan_rc: the plan's return code; a declined plan's error (already set) comes after the planned tiles' faults.
   Faults are reported for the first tile in tile order that has one: a packet's, in code-stream order, before its tile
   parts'.  Returns the length (also when out is NULL or, without tile_at, cap is too small), or -1 with the error set. */
int64_t write_plan(const t2::Plan& P, int plan_rc, const b2k_result* r, bool whole, uint8_t* out, uint64_t cap, uint64_t* tile_bytes,
                   const uint64_t* tile_at)
{
  using namespace t2;
  const uint64_t np = P.packets.size(), nparts = P.parts.size();
  const TableBlocks B{r->blocks, r->num_bytes, r->num_blocks};
  const bool sop = (P.flags & B2K_CS_SOP) != 0, eph = (P.flags & B2K_CS_EPH) != 0, plt = (P.flags & B2K_CS_PLT) != 0;
  const bool tlm = whole && (P.flags & B2K_CS_TLM) != 0;
  const uint64_t head_len = whole ? P.head.size() : 0;
  /* every entry is written before it is read, so none is cleared here: the pool's threads touch the pages first */
  const auto hdr = scratch<uint8_t>(P.hdr_bytes);
  const auto tags = scratch<TagNode>(P.tag_nodes);
  const auto hdr_len = scratch<uint32_t>(np), pkt_err = scratch<uint32_t>(np);
  const auto body_len = scratch<uint64_t>(np), pkt_at = scratch<uint64_t>(np), dst = scratch<uint64_t>(r->num_blocks);
  std::vector<uint64_t> part_plt(nparts), part_bytes(nparts), part_at(nparts);
  WriteStatus st{};
  WritePlace place{};
  b2k_host_parallel(nparts, [&](size_t t) {
    for(uint64_t p = P.parts[t].p0; p < P.parts[t].p1; ++p)
      write_header(p, P.packets.data(), np, B, hdr.get(), P.hdr_bytes, tags.get(), P.tag_nodes, hdr_len.get(), body_len.get(),
                   dst.get(), &st, sop, eph, pkt_err.get());
  });
  for(uint64_t t = 0; t < nparts; ++t)
    write_part(t, P.parts.data(), nparts, np, hdr_len.get(), body_len.get(), part_plt.data(), part_bytes.data(), &st, plt);
  for(uint64_t t0 = 0, t1; t0 < nparts; t0 = t1)
  {
    for(t1 = t0; t1 < nparts && P.parts[t1].tile == P.parts[t0].tile; ++t1)
    {
    }
    for(uint64_t p = P.parts[t0].p0; p < P.parts[t1 - 1].p1; ++p)
      if(pkt_err[p])
      {
        b2k_set_error(packet_error(pkt_err[p]));
        return -1;
      }
    for(uint64_t t = t0; t < t1; ++t)
      if(part_bytes[t] > 0xFFFFFFFFull)
      {
        b2k_set_error("tile part longer than 4 GiB");
        return -1;
      }
    if(tile_bytes)
      tile_bytes[t0] = part_bytes[t0]; /* a shard has a tile part per tile */
  }
  if(plan_rc)
    return -1;
  write_scan_host(1, part_bytes.data(), nparts, part_at.data(), head_len, &st, &place);
  const uint64_t total = whole ? st.total : st.total - 2; /* a shard's tile parts have no EOC */
  if(!out || (!tile_at && cap < total))
    return (int64_t)total;
  for(uint64_t k = 0; tile_at && k < nparts; ++k)
  {
    if(tile_at[k] + part_bytes[k] > cap)
    {
      b2k_set_error("a tile part would land outside the buffer");
      return -1;
    }
    part_at[k] = tile_at[k];
  }
  /* every place is inside the buffer: the steps write without a bound */
  b2k_host_parallel(nparts, [&](size_t t) {
    write_emit(t, P.parts.data(), nparts, np, part_at.data(), part_plt.data(), part_bytes.data(), hdr_len.get(), body_len.get(),
               pkt_at.get(), out, ~0ull, &st, &place, P.head.data(), head_len, plt, tlm, P.tlm_at);
    for(uint64_t p = P.parts[t].p0; p < P.parts[t].p1; ++p)
    {
      write_packet(p, 0, 1, P.packets.data(), np, B, hdr.get(), P.hdr_bytes, hdr_len.get(), pkt_at.get(), dst.get(), out, ~0ull, &st,
                   &place);
      const DevPacket& D = P.packets[p];
      uint64_t from = 0, to = 0, n = 0; /* blocks that are neighbours in the arena and in the packet: one copy */
      for(uint32_t b = 0; b < D.nbands; ++b)
        for(uint32_t i = D.band[b].first, e = i + D.band[b].gw * D.band[b].gh; i < e; ++i)
          if(B.slot(i) >= 0)
          {
            if(r->blocks[i].offset != from + n || dst[i] != to + n)
            {
              if(n)
                memcpy(out + to, r->bytes + from, n);
              from = r->blocks[i].offset, to = dst[i], n = 0;
            }
            n += B.bytes(i);
          }
      if(n)
        memcpy(out + to, r->bytes + from, n);
    }
  });
  return (int64_t)total;
}
} // namespace

/* ============================================================================================================ */
extern "C" __attribute__((visibility("default"))) int64_t b2k_codestream_write(const b2k_coding* cp, const b2k_result* r,
                                                                                uint32_t flags, uint8_t* out, uint64_t cap)
{
  if(!cp || !r)
    return -1;
  t2::Plan P;
  const int rc = b2k_t2_plan(*cp, flags, r->blocks, r->num_blocks, r->num_tiles, P);
  return write_plan(P, rc, r, true, out, cap, nullptr, nullptr);
}

int b2k_t2_plan(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles, t2::Plan& plan)
{
  if(check_whole_image(cp, num_tiles, flags))
    return -1;
  const int rc = plan_tiles(cp, flags, blocks, nblocks, 1, 0, plan);
  if(rc > 0)
    b2k_set_error("block table is not in tile order");
  return rc ? -1 : 0;
}

/* ---- per-rank writers (SURVEY.md 8e: "T2 can itself be sharded per tile; the writer concatenates in index order") ------
 * b2k_codestream_write_tiles: the finished tile parts (SOT [PLT] SOD packets, one tile part per tile) of the tiles a shard
 * holds (tile t with t % tile_mod == tile_rem, as b2k_encode returned them), consecutively in tile order; tile_bytes[k] =
 * length of the k-th of them.  b2k_codestream_write_header: SOC .. QCD [TLM] for the whole image from every tile's length.
 * A code stream = header + the tile parts in tile-index order + EOC (0xFFD9): byte-identical to b2k_codestream_write's. */
static int64_t write_tiles_impl(const b2k_coding* cp, const b2k_result* r, uint32_t flags, uint32_t tile_mod, uint32_t tile_rem, uint8_t* out,
                                uint64_t cap, uint64_t* tile_bytes, const uint64_t* tile_at)
{
  if(!cp || !r || !tile_mod || tile_rem >= tile_mod)
    return -1;
  if(const char* why = unsupported_reason(*cp))
  {
    b2k_set_error(why);
    return -1;
  }
  if(flags & B2K_CS_TPARTS_R)
  {
    b2k_set_error("per-rank writers emit one tile part per tile");
    return -1;
  }
  const TileGrid g = tile_grid(*cp);
  if(((flags >> 8) & 7) > 4 || g.nx * g.ny > 65535)
  {
    b2k_set_error("unknown progression order / too many tiles");
    return -1;
  }
  t2::Plan P;
  const int rc = plan_tiles(*cp, flags, r->blocks, r->num_blocks, tile_mod, tile_rem, P);
  if(rc > 0)
  {
    b2k_set_error("the block table is not the shard's tiles in tile order");
    return -1;
  }
  return write_plan(P, rc, r, false, out, cap, tile_bytes, tile_at);
}

extern "C" __attribute__((visibility("default"))) int64_t b2k_codestream_write_tiles(const b2k_coding* cp, const b2k_result* r, uint32_t flags,
                                                                                      uint32_t tile_mod, uint32_t tile_rem, uint8_t* out,
                                                                                      uint64_t cap, uint64_t* tile_bytes)
{
  return write_tiles_impl(cp, r, flags, tile_mod, tile_rem, out, cap, tile_bytes, nullptr);
}

/* the same, each of the shard's tiles written at out + tile_at[k] (the writer rank puts its own tiles straight into their
   places in the code stream once every tile's length is known) */
extern "C" __attribute__((visibility("default"))) int64_t b2k_codestream_write_tiles_at(const b2k_coding* cp, const b2k_result* r, uint32_t flags,
                                                                                         uint32_t tile_mod, uint32_t tile_rem, uint8_t* out,
                                                                                         uint64_t cap, const uint64_t* tile_at)
{
  if(!tile_at)
    return -1;
  return write_tiles_impl(cp, r, flags, tile_mod, tile_rem, out, cap, nullptr, tile_at);
}

extern "C" __attribute__((visibility("default"))) int64_t b2k_codestream_write_header(const b2k_coding* cp, uint32_t flags,
                                                                                       const uint64_t* tile_bytes, uint32_t ntiles_in,
                                                                                       uint8_t* out, uint64_t cap)
{
  if(!cp)
    return -1;
  if(const char* why = unsupported_reason(*cp))
  {
    b2k_set_error(why);
    return -1;
  }
  const TileGrid g = tile_grid(*cp);
  const uint32_t ntiles = g.nx * g.ny;
  if(((flags >> 8) & 7) > 4 || ((flags & B2K_CS_TLM) && (!tile_bytes || ntiles_in != ntiles)))
  {
    b2k_set_error("TLM needs the length of every tile's tile part");
    return -1;
  }
  std::vector<uint8_t> head;
  const uint64_t tlm_at = main_header(*cp, flags, ntiles, head);
  for(uint32_t t = 0; (flags & B2K_CS_TLM) && t < ntiles; ++t)
    t2::put_tlm_entry(head.data() + tlm_at, t, t, (uint32_t)tile_bytes[t]);
  if(out && cap >= head.size())
    memcpy(out, head.data(), head.size());
  return (int64_t)head.size();
}

namespace
{
/* packets of one tile part -> the tile's slice of the block table (offsets relative to `base`).
   0 ok, 1 outside this path's scope, -1 damaged; err says why. */
struct ByteRange
{
  const uint8_t *begin, *end;
};
int parse_tile_packets(const b2k_coding& cp, const Rect& tile, b2k_block* tb, const std::vector<ByteRange>& parts,
                       const uint8_t* base, int prog, bool sop, bool eph, std::string& err)
{
  std::vector<Packet> pkts;
  uint32_t nblk = 0;
  tile_packets(cp, tile, pkts, nblk, prog);
  size_t part = 0;
  const uint8_t* p = parts.empty() ? nullptr : parts[0].begin;
  const uint8_t* tp_end = parts.empty() ? nullptr : parts[0].end;
  TagTree incl, imsb;
  struct Seg
  {
    uint32_t blk, n;
  };
  std::vector<Seg> order;
  auto fail = [&](const char* m, int rc) {
    err = m;
    return rc;
  };
  for(const Packet& pk : pkts)
  {
    while(p == tp_end && part + 1 < parts.size())
    { /* a packet never straddles tile parts: continue in the next one */
      ++part;
      p = parts[part].begin;
      tp_end = parts[part].end;
    }
    if(p == tp_end)
      break; /* the tile's data ends here (truncated or resolution-progressive file): what follows stays uncoded */
    if(sop && tp_end - p >= 6 && p[0] == 0xFF && p[1] == 0x91)
      p += 6; /* SOP may be there when COD allows it (A.8.1) */
    BitReader br(p, tp_end);
    order.clear();
    if(br.get())
    {
      for(int b = 0; b < pk.nbands; ++b)
      {
        const PacketBand& pb = pk.band[b];
        const uint32_t n = pb.gw * pb.gh;
        if(!n)
          continue;
        incl.init(pb.gw, pb.gh);
        imsb.init(pb.gw, pb.gh);
        for(uint32_t k = 0; k < n; ++k)
        {
          b2k_block& B = tb[pb.first + k];
          if(!incl.decode(br, k, 1))
            continue;
          uint32_t zbp = 0;
          for(uint32_t th = 1;; ++th)
          {
            if(imsb.decode(br, k, th))
            {
              zbp = imsb.nodes[k].value;
              break;
            }
            if(th > 64 || br.overrun)
              return fail("corrupt packet header (zero bit planes)", -1);
          }
          uint32_t np; /* number of passes, B.10.6 */
          if(!br.get())
            np = 1;
          else if(!br.get())
            np = 2;
          else
          {
            const uint32_t v = br.get_bits(2);
            if(v < 3)
              np = 3 + v;
            else
            {
              const uint32_t v5 = br.get_bits(5);
              np = v5 < 31 ? 6 + v5 : 37 + br.get_bits(7);
            }
          }
          if(np > 3)
            return fail("HT code blocks with placeholder passes or several HT sets are not handled", 1);
          int lblock = 3;
          while(br.get())
            if(++lblock > 32)
              return fail("corrupt packet header (Lblock)", -1);
          /* HT: the cleanup pass is one segment, the refinement passes another (T.814 B.10.7) */
          const uint32_t len1 = br.get_bits(lblock);
          const uint32_t len2 = np > 1 ? br.get_bits(std::min(32, lblock + floorlog2(np - 1))) : 0;
          if(zbp > B.kmax)
            return fail("more zero bit planes than the band has bit planes", -1);
          if(len1 < 2)
            return fail("HT cleanup segment shorter than 2 bytes", -1);
          B.numbps = (uint8_t)(B.kmax - zbp);
          B.numpasses = (uint8_t)np;
          B.length = len1;
          B.length2 = len2;
          order.push_back({pb.first + k, len1 + len2});
        }
      }
    }
    if(br.overrun)
      return fail("packet header runs past the tile part", -1);
    p = br.finish();
    if(eph)
    { /* EPH shall follow every packet header when COD says so (A.8.2) */
      if(tp_end - p < 2 || p[0] != 0xFF || p[1] != 0x92)
        return fail("EPH marker missing after a packet header", -1);
      p += 2;
    }
    for(const Seg& sg : order)
    {
      if((uint64_t)(tp_end - p) < sg.n)
        return fail("packet body runs past the tile part", -1);
      tb[sg.blk].offset = (uint64_t)(p - base);
      p += sg.n;
    }
  }
  return 0;
}

} // namespace

/* ============================================================================================================ */
namespace
{
struct Cursor
{
  const uint8_t* p;
  const uint8_t* end;
  bool ok = true;
  uint32_t u8()
  {
    if(p + 1 > end) { ok = false; return 0; }
    return *p++;
  }
  uint32_t u16()
  {
    if(p + 2 > end) { ok = false; return 0; }
    const uint32_t v = ((uint32_t)p[0] << 8) | p[1];
    p += 2;
    return v;
  }
  uint32_t u32()
  {
    const uint32_t a = u16();
    return (a << 16) | u16();
  }
};
} // namespace

/* The main header of cs[0, len), SOC up to the first SOT: the coding, the progression order, SOP / EPH and where the first
   SOT starts.  0, or b2k_codestream_parse's return code and text for a main header it declines; h.short_read says the
   failure came from reaching `len`, so that a longer prefix of the same stream may parse (b2k_codestream_parse_device
   reads the header from a prefix). */
int b2k_batch_coding_check(const t2::MainHeader& ref, uint32_t ref_index, const t2::MainHeader& h, uint32_t index)
{
  std::string why;
  if(memcmp(&h.cp, &ref.cp, sizeof(b2k_coding)) != 0)
    why = "its coding differs from that of code stream ";
  else if(h.flags() != ref.flags())
    why = "its progression order, SOP or EPH differ from those of code stream ";
  if(why.empty())
    return 0;
  b2k_set_error(("code stream " + std::to_string(index) + ": " + why + std::to_string(ref_index) + ", which the batch takes its coding from")
                    .c_str());
  return 1;
}

int b2k_batch_window_check(const t2::MainHeader& ref, const t2::WindowCoding& rw, uint32_t ref_index, const t2::MainHeader& h,
                           const t2::WindowCoding& w, uint32_t index)
{
  const TileGrid a = tile_grid(ref.cp), b = tile_grid(h.cp);
  std::string why;
  if(memcmp(&rw.vcp, &w.vcp, sizeof(b2k_coding)) != 0 || memcmp(&rw.box, &w.box, sizeof(b2k_coding)) != 0 || rw.whole != w.whole ||
     a.nx != b.nx || a.ny != b.ny || rw.ta_x != w.ta_x || rw.ta_y != w.ta_y || rw.tb_x != w.tb_x || rw.tb_y != w.tb_y)
    why = "its window's coding (tile grid, wanted tiles or virtual coding) differs from that of code stream ";
  else if(h.flags() != ref.flags())
    why = "its progression order, SOP or EPH differ from those of code stream ";
  if(why.empty())
    return 0;
  b2k_set_error(("code stream " + std::to_string(index) + ": " + why + std::to_string(ref_index) + ", which the batch takes its coding from")
                    .c_str());
  return 1;
}

int b2k_parse_main_header(const uint8_t* cs, uint64_t len, t2::MainHeader& h)
{
  h = t2::MainHeader();
  auto fail = [&](const char* m, int rc) {
    b2k_set_error(m);
    return rc;
  };
  Cursor c{cs, cs + len};
  if(c.u16() != 0xFF4F)
    return fail("no SOC marker", -1);
  b2k_coding cp;
  memset(&cp, 0, sizeof(cp));
  bool have_siz = false, have_cod = false, have_qcd = false, have_cap = false;
  int progression = 0;
  bool use_sop = false, use_eph = false;
  std::vector<uint32_t> qcd_vals;
  uint32_t sqcd = 0;
  std::vector<uint32_t> qcc_vals[4]; /* per component named by a QCC, its Sqcc in qcc_sq */
  uint32_t qcc_sq[4] = {0, 0, 0, 0};
  uint8_t qcc_mask = 0;
  /* ---- main header ---- */
  for(;;)
  {
    const uint32_t m = c.u16();
    if(!c.ok)
    {
      h.short_read = true;
      return fail("truncated main header", -1);
    }
    if(m == 0xFF90)
    {
      c.p -= 2;
      break;
    }
    const uint32_t L = c.u16();
    if(!c.ok || L < 2 || c.p + (L - 2) > c.end)
    {
      h.short_read = !c.ok || (L >= 2 && c.p + (L - 2) > c.end);
      return fail("bad marker segment length", -1);
    }
    Cursor s{c.p, c.p + (L - 2)};
    c.p += L - 2;
    switch(m)
    {
      case 0xFF51: {
        const uint32_t rsiz = s.u16();
        (void)rsiz;
        cp.x1 = s.u32(); cp.y1 = s.u32(); cp.x0 = s.u32(); cp.y0 = s.u32();
        cp.tw = s.u32(); cp.th = s.u32(); cp.tx0 = s.u32(); cp.ty0 = s.u32();
        const uint32_t nc = s.u16();
        if(nc < 1 || nc > 4)
          return fail("1..4 components handled", 1);
        cp.numcomps = (uint16_t)nc;
        for(uint32_t i = 0; i < nc; ++i)
        {
          const uint32_t ssiz = s.u8(), dx = s.u8(), dy = s.u8();
          if(dx != 1 || dy != 1)
            return fail("sub-sampled components are not handled", 1);
          const uint8_t prec = (uint8_t)((ssiz & 0x7F) + 1), sg = (uint8_t)(ssiz >> 7);
          if(i && (prec != cp.prec || sg != cp.sgnd))
            return fail("components of different precision are not handled", 1);
          cp.prec = prec;
          cp.sgnd = sg;
        }
        have_siz = s.ok;
        break;
      }
      case 0xFF50: {
        const uint32_t pcap = s.u32();
        have_cap = (pcap & 0x00020000u) != 0;
        if(have_cap)
        {
          /* Ccap15 is the entry of the 15th capability bit among those set */
          uint32_t idx = 0;
          for(int b = 31; b > 17; --b)
            idx += (pcap >> b) & 1u;
          uint32_t ccap15 = 0;
          for(uint32_t i = 0; i <= idx; ++i)
            ccap15 = s.u16();
          if((ccap15 >> 14) != 0)
            return fail("only HTONLY codestreams are handled (no Part-1 or mixed code blocks)", 1);
          if(ccap15 & 0x2000)
            return fail("multiple HT sets per code block are not handled", 1);
        }
        break;
      }
      case 0xFF52: {
        const uint32_t scod = s.u8();
        use_sop = (scod & 0x02) != 0;
        use_eph = (scod & 0x04) != 0;
        const uint32_t prog = s.u8(), layers = s.u16(), mct = s.u8();
        cp.mct = (uint8_t)mct;
        const uint32_t nd = s.u8();
        cp.numres = (uint8_t)(nd + 1);
        cp.cblkw_exp = (uint8_t)(s.u8() + 2);
        cp.cblkh_exp = (uint8_t)(s.u8() + 2);
        const uint32_t sty = s.u8(), xf = s.u8();
        if(layers != 1)
          return fail("one quality layer handled", 1);
        if(prog > 4)
          return fail("unknown progression order", -1);
        progression = (int)prog;
        if(!(sty & 0x40) || (sty & ~0x48u))
          return fail("only HT code blocks (optionally stripe-causal) are handled", 1);
        cp.cblk_sty = (uint8_t)(sty & 0x08);
        if(xf > 1)
          return fail("unknown wavelet", 1);
        cp.irreversible = xf == 0;
        for(int r = 0; r < 33; ++r)
          cp.prcw_exp[r] = cp.prch_exp[r] = 15;
        if(scod & 1)
          for(uint32_t r = 0; r <= nd && r < 33; ++r)
          {
            const uint32_t v = s.u8();
            cp.prcw_exp[r] = (uint8_t)(v & 0xF);
            cp.prch_exp[r] = (uint8_t)(v >> 4);
            /* PPx / PPy = 0 (1-sample precincts, legal at resolution 0 only): b2k_coding reads exponent 0 as
               "default 15", so such a stream is declined rather than enumerated wrongly */
            if(s.ok && ((v & 0xF) == 0 || (v >> 4) == 0))
              return fail("precinct exponent 0 is not handled", 1);
          }
        have_cod = s.ok;
        break;
      }
      case 0xFF5C: {
        sqcd = s.u8();
        cp.numgbits = (uint8_t)(sqcd >> 5);
        const uint32_t style = sqcd & 0x1F;
        if(style > 2)
          return fail("unknown quantisation style", -1);
        while(s.ok && s.p < s.end) /* an odd byte left over in a 16-bit QCD ends the loop through s.ok */
          qcd_vals.push_back(style == 0 ? s.u8() : s.u16());
        have_qcd = s.ok;
        break;
      }
      case 0xFF5D: { /* QCC (A.6.5): Cqcc is one byte, as Csiz < 257 here */
        if(!have_siz)
          return fail("QCC before SIZ", -1);
        const uint32_t comp = s.u8(), sq = s.u8();
        if(!s.ok)
          return fail("truncated QCC", -1);
        if(comp >= cp.numcomps)
          return fail("QCC names a component the image does not have", -1);
        if((sq & 0x1F) > 2)
          return fail("unknown quantisation style", -1);
        qcc_vals[comp].clear();
        while(s.ok && s.p < s.end)
          qcc_vals[comp].push_back((sq & 0x1F) == 0 ? s.u8() : s.u16());
        if(!s.ok || qcc_vals[comp].empty())
          return fail("truncated QCC", -1);
        qcc_sq[comp] = sq;
        qcc_mask |= (uint8_t)(1u << comp);
        break;
      }
      case 0xFF64: /* COM */
      case 0xFF55: /* TLM: lengths are read from SOT */
      case 0xFF63: /* CRG */
        break;
      case 0xFF53: case 0xFF5E: case 0xFF5F: case 0xFF60: case 0xFF57:
        return fail("COC / RGN / POC / PPM / PLM marker segments are not handled", 1);
      default:
        if(m < 0xFF00)
          return fail("garbage in the main header", -1);
        break; /* unknown informative segment: skip */
    }
  }
  if(!have_siz || !have_cod || !have_qcd)
    return fail("SIZ, COD and QCD are required", -1);
  if(!have_cap)
    return fail("not an HTJ2K codestream (no Part-15 capability)", 1);
  if(cp.mct && cp.numcomps < 3)
    return fail("MCT with fewer than three components", -1);
  if(const char* why = unsupported_reason(cp))
    return fail(why, 1);
  /* band exponents / mantissas: Grok's HT quantiser tables when QCD agrees with them, or some quality factor's when QCD
     and every QCC agree with its tables, else QCD's and the QCCs' own values */
  {
    const size_t nbands = 3 * (size_t)(cp.numres - 1) + 1;
    /* one QCD / QCC: (exponent << 11 | mantissa) per band; 0, else the return code with the error set */
    auto band_values = [&](uint32_t sq, const std::vector<uint32_t>& raw, const char* none, const char* few,
                           std::vector<uint32_t>& vals) -> int {
      const uint32_t style = sq & 0x1F;
      if((style != 0) != (cp.irreversible != 0))
        return fail("quantisation style does not match the wavelet", 1);
      if((sq >> 5) != cp.numgbits)
        return fail("QCC with guard bits other than QCD's is not handled", 1);
      vals.assign(nbands, 0);
      if(style == 1)
      { /* scalar derived (A.6.4, E.1.1.1): (e_b, m_b) = (e_0 - N_L + n_b, m_0), n_b = decomposition level of the band */
        if(raw.empty())
          return fail(none, -1);
        const int e0 = (int)(raw[0] >> 11), m0 = (int)(raw[0] & 0x7FF), NL = cp.numres - 1;
        for(size_t i = 0; i < nbands; ++i)
        {
          const int nb = i == 0 ? NL : NL - (int)((i - 1) / 3);
          vals[i] = (uint32_t)(std::max(0, e0 - NL + nb) << 11) | (uint32_t)m0;
        }
      }
      else
      {
        if(raw.size() < nbands)
          return fail(few, -1);
        for(size_t i = 0; i < nbands; ++i)
          vals[i] = style == 0 ? (raw[i] >> 3) << 11 : raw[i];
      }
      return 0;
    };
    auto agrees = [&](const std::vector<uint32_t>& vals, const std::vector<BandQuant>& q) {
      bool same = true;
      for(size_t i = 0; i < nbands; ++i)
        same &= (vals[i] >> 11) == q[i].expn && (cp.irreversible ? (vals[i] & 0x7FF) == q[i].mant : true);
      return same;
    };
    std::vector<uint32_t> vals[5]; /* [0..3]: what each component uses, [4]: QCD */
    if(int rc = band_values(sqcd, qcd_vals, "QCD has no entry", "QCD has fewer entries than bands", vals[4]))
      return rc;
    for(int k = 0; k < cp.numcomps; ++k)
    {
      if(!((qcc_mask >> k) & 1))
        vals[k] = vals[4];
      else if(int rc = band_values(qcc_sq[k], qcc_vals[k], "QCC has no entry", "QCC has fewer entries than bands", vals[k]))
        return rc;
    }
    bool same = true;
    const std::vector<BandQuant> dflt = band_quant(cp); /* Grok's HT tables: the same for every component */
    for(int k = 0; k < cp.numcomps; ++k)
      same &= agrees(vals[k], dflt);
    /* some quality factor's tables?  Compared word for word with the cached tables, component 0 first, so that a stream
       that is none of them costs one short comparison per quality factor */
    for(int qf = 1; !same && cp.irreversible && (cp.numcomps == 1 || cp.numcomps == 3) && qf <= 100; ++qf)
    {
      same = true;
      for(int k = 0; k < cp.numcomps && same; ++k)
        same = vals[k] == qfactor_words(qf, cp.prec, cp.numres, k);
      if(same)
        cp.qfactor = (uint8_t)qf;
    }
    if(!same)
    {
      cp.qcd_explicit = 1;
      for(size_t i = 0; i < nbands && i < 97; ++i)
      {
        cp.qcd_expn[i] = (uint8_t)(vals[4][i] >> 11);
        cp.qcd_mant[i] = (uint16_t)(vals[4][i] & 0x7FF);
      }
      cp.qcc_mask = qcc_mask;
      for(int k = 0; k < cp.numcomps; ++k)
        if((qcc_mask >> k) & 1)
          for(size_t i = 0; i < nbands && i < 97; ++i)
          {
            cp.qcc_expn[k][i] = (uint8_t)(vals[k][i] >> 11);
            cp.qcc_mant[k][i] = (uint16_t)(vals[k][i] & 0x7FF);
          }
    }
  }
  if(const char* why = unsupported_reason(cp))
    return fail(why, 1);
  /* SIZ sanity (A.5.1) and a bound on what a damaged header can make us enumerate */
  if(cp.tw == 0 || cp.th == 0 || cp.tx0 > cp.x0 || cp.ty0 > cp.y0 || (uint64_t)cp.tx0 + cp.tw <= cp.x0 ||
     (uint64_t)cp.ty0 + cp.th <= cp.y0)
    return fail("tile grid does not cover the image origin", -1);
  if((uint64_t)(cp.x1 - cp.x0) * (cp.y1 - cp.y0) > (1ull << 32))
    return fail("image larger than 2^32 samples per component", 1);
  {
    const uint64_t nx = ceil_div(cp.x1 - cp.tx0, cp.tw), ny = ceil_div(cp.y1 - cp.ty0, cp.th);
    if(nx * ny > 65535)
      return fail("more than 65535 tiles", -1);
    uint64_t precincts = 0;
    for(int r = 0; r < cp.numres; ++r)
    { /* upper bound: precincts of resolution r over the whole image, plus one row / column per tile */
      const int nd = cp.numres - 1 - r;
      const uint64_t rw = (((uint64_t)(cp.x1 - cp.x0)) >> nd) + 2 * nx, rh = (((uint64_t)(cp.y1 - cp.y0)) >> nd) + 2 * ny;
      const uint32_t pw = cp.prcw_exp[r] ? cp.prcw_exp[r] : 15, ph = cp.prch_exp[r] ? cp.prch_exp[r] : 15;
      precincts += ((rw >> pw) + 2 * nx) * ((rh >> ph) + 2 * ny);
    }
    if(precincts * cp.numcomps > (1ull << 24))
      return fail("more than 2^24 precincts", 1);
    if((((uint64_t)(cp.x1 - cp.x0) * (cp.y1 - cp.y0) * cp.numcomps) >> (cp.cblkw_exp + cp.cblkh_exp)) > (1ull << 26))
      return fail("more than 2^26 code blocks", 1);
  }
  memcpy(&h.cp, &cp, sizeof(cp)); /* padding included: the engine compares codings bytewise */
  h.progression = progression;
  h.sop = use_sop;
  h.eph = use_eph;
  h.sot = (uint64_t)(c.p - cs);
  return 0;
}

int b2k_window_coding(const b2k_coding& cp, const uint32_t* window, uint32_t reduce, t2::WindowCoding& wc)
{
  auto fail = [&](const char* m, int rc) {
    b2k_set_error(m);
    return rc;
  };
  const std::vector<std::vector<BandQuant>> q = component_quant(cp);
  const TileGrid g = tile_grid(cp);
  /* ---- the tiles to deliver and the coding to decode them with ---------------------------------------------------
   * Whole image at full resolution: the stream's own coding.  Otherwise a VIRTUAL image: its area is the bounding box
   * of the tiles the window touches (clipped to the image), its tile grid is the stream's grid re-anchored at the first
   * of those tiles, and for reduce > 0 everything is divided by 2^reduce and the highest `reduce` resolutions are
   * dropped -- by the standard's own definitions (B.5: resolution r of a tile component is the tile rectangle
   * ceil-divided by 2^(N_L - r)) the remaining resolutions, precinct grids and code blocks of every tile are exactly
   * those of the original, so the parsed blocks carry over one to one
   * (cf. CodeStreamDecompress.cpp L670-870: tiles from the window, resolutions from `reduce`). */
  uint32_t ta_x = 0, ta_y = 0, tb_x = g.nx, tb_y = g.ny;
  if(window)
  {
    const uint32_t wx0 = std::max(window[0], cp.x0), wy0 = std::max(window[1], cp.y0), wx1 = std::min(window[2], cp.x1),
                   wy1 = std::min(window[3], cp.y1);
    if(wx0 >= wx1 || wy0 >= wy1)
      return fail("the window does not intersect the image", -1);
    ta_x = (wx0 - g.tx0) / g.tw;
    ta_y = (wy0 - g.ty0) / g.th;
    tb_x = (uint32_t)ceil_div(wx1 - g.tx0, g.tw);
    tb_y = (uint32_t)ceil_div(wy1 - g.ty0, g.th);
  }
  if((int)reduce >= cp.numres)
    return fail("reduce exceeds the number of decomposition levels", -1);
  const bool whole = ta_x == 0 && ta_y == 0 && tb_x == g.nx && tb_y == g.ny && reduce == 0;
  b2k_coding vcp = cp;
  if(!whole)
  {
    vcp.tx0 = g.tx0 + ta_x * g.tw;
    vcp.ty0 = g.ty0 + ta_y * g.th;
    vcp.tw = g.tw;
    vcp.th = g.th;
    vcp.x0 = std::max(cp.x0, vcp.tx0);
    vcp.y0 = std::max(cp.y0, vcp.ty0);
    vcp.x1 = (uint32_t)std::min<uint64_t>(cp.x1, (uint64_t)g.tx0 + (uint64_t)tb_x * g.tw);
    vcp.y1 = (uint32_t)std::min<uint64_t>(cp.y1, (uint64_t)g.ty0 + (uint64_t)tb_y * g.th);
    /* every component's band exponents are the stream's: spelled out, since the default and the quality factor's
       tables depend on the level count */
    vcp.qfactor = 0;
    vcp.qcd_explicit = 1;
    vcp.qcc_mask = 0;
    for(int k = 0; k < cp.numcomps; ++k)
    {
      if(k && !same_quant(q[k], q[0]))
        vcp.qcc_mask |= (uint8_t)(1u << k);
      for(size_t i = 0; i < q[k].size() && i < 97; ++i)
      {
        (k ? vcp.qcc_expn[k][i] : vcp.qcd_expn[i]) = q[k][i].expn;
        (k ? vcp.qcc_mant[k][i] : vcp.qcd_mant[i]) = q[k][i].mant;
      }
    }
    const bool one_tile = tb_x - ta_x == 1 && tb_y - ta_y == 1;
    if(one_tile)
      vcp.tx0 = vcp.ty0 = vcp.tw = vcp.th = 0; /* the tile is the (virtual) image: no grid to keep aligned */
    wc.box = vcp;
    if(reduce)
    {
      const uint32_t m = (1u << reduce) - 1u;
      if(!one_tile && ((vcp.tx0 & m) || (vcp.ty0 & m) || (vcp.tw & m) || (vcp.th & m)))
        return fail("reduced decode of several tiles needs a tile grid aligned to 2^reduce", 1);
      vcp.tx0 >>= reduce; vcp.ty0 >>= reduce; vcp.tw >>= reduce; vcp.th >>= reduce;
      vcp.x0 = (vcp.x0 + m) >> reduce; vcp.y0 = (vcp.y0 + m) >> reduce;
      vcp.x1 = (vcp.x1 + m) >> reduce; vcp.y1 = (vcp.y1 + m) >> reduce;
      vcp.numres = (uint8_t)(cp.numres - reduce);
      if(vcp.x1 <= vcp.x0 || vcp.y1 <= vcp.y0)
        return fail("nothing left at this resolution", -1);
    }
    if(const char* why = unsupported_reason(vcp))
      return fail(why, 1);
  }
  /* ---- which code blocks a window needs (SURVEY 8f N3: "only the code blocks ... an ROI needs") ----
   * need[r] = the samples of resolution r (canvas coordinates of the virtual coding) that the window's pixels depend on.
   * The top resolution needs the window itself; one synthesis step down, a sample at x depends on the low / high band
   * samples around x / 2: within 1 for the 5/3 filter pair (x[2n+1] uses L[n], L[n+1], H[n-1..n+1]), within 3 for the
   * four lifting steps of 9/7 -- taken as 2 and 5.  A block of resolution r >= 1 lives in band coordinates, i.e. those
   * of resolution r - 1.  Blocks outside are handed back with length 0 ("not in any packet": decoded as zeros): their
   * coefficients cannot reach the window. */
  std::vector<Rect>& need = wc.need;
  need.clear();
  if(window && !whole)
  {
    const uint32_t m = (1u << reduce) - 1u;
    Rect w{(std::max(window[0], cp.x0) + m) >> reduce, (std::max(window[1], cp.y0) + m) >> reduce,
           (std::min(window[2], cp.x1) + m) >> reduce, (std::min(window[3], cp.y1) + m) >> reduce};
    w.x0 = std::max(w.x0, vcp.x0); w.y0 = std::max(w.y0, vcp.y0);
    w.x1 = std::min(w.x1, vcp.x1); w.y1 = std::min(w.y1, vcp.y1);
    if(w.x1 > w.x0 && w.y1 > w.y0)
    {
      const uint32_t M = vcp.irreversible ? 5u : 2u;
      need.assign(vcp.numres, w);
      for(int r = (int)vcp.numres - 2; r >= 0; --r)
      {
        const Rect& f = need[r + 1];
        need[r] = Rect{(f.x0 >> 1) > M ? (f.x0 >> 1) - M : 0u, (f.y0 >> 1) > M ? (f.y0 >> 1) - M : 0u, ((f.x1 + 1) >> 1) + M,
                       ((f.y1 + 1) >> 1) + M};
      }
    }
  }
  wc.whole = whole;
  wc.ta_x = ta_x;
  wc.ta_y = ta_y;
  wc.tb_x = tb_x;
  wc.tb_y = tb_y;
  wc.vcp = vcp;
  if(whole)
    wc.box = cp;
  return 0;
}

int b2k_window_blocks(const t2::WindowCoding& wc, const b2k_block* vblocks, uint64_t nv, std::vector<b2k_block>& box_blocks,
                      std::vector<uint32_t>& vmap)
{
  const b2k_coding& box = wc.box;
  const TileGrid bg = tile_grid(box);
  const uint32_t nt = bg.nx * bg.ny;
  const std::vector<std::vector<BandQuant>> bq = component_quant(box);
  box_blocks.clear();
  vmap.assign(nv, 0);
  uint64_t k = 0;
  for(uint32_t t = 0; t < nt; ++t)
  {
    const size_t first = box_blocks.size();
    enumerate_tile_blocks(box, t, tile_rect(box, bg, t), bq, box_blocks);
    for(size_t i = first; i < box_blocks.size(); ++i)
    { /* the virtual tile's own enumeration: the box tile's blocks of the kept resolutions follow in the same order */
      const b2k_block& b = box_blocks[i];
      if(b.resno >= wc.vcp.numres)
        continue;
      const b2k_block* v = k < nv ? &vblocks[k] : nullptr;
      if(!v || v->tile != t || v->comp != b.comp || v->resno != b.resno || v->band_index != b.band_index || v->precno != b.precno ||
         v->cblkno != b.cblkno || v->x1 - v->x0 != b.x1 - b.x0 || v->y1 - v->y0 != b.y1 - b.y0)
      {
        b2k_set_error("internal: virtual and original block enumerations disagree");
        return -1;
      }
      vmap[k++] = (uint32_t)i;
    }
    if(k < nv && vblocks[k].tile == t)
    {
      b2k_set_error("internal: virtual tile holds a different number of blocks");
      return -1;
    }
  }
  if(k != nv || box_blocks.size() > 0xFFFFFFFFull)
  {
    b2k_set_error("internal: virtual tile holds a different number of blocks");
    return -1;
  }
  return 0;
}

/* window: x0,y0,x1,y1 on the full-resolution canvas, or NULL for the whole image; reduce: highest resolutions to drop.
   *cp_out is the coding to DECODE WITH: for a window / reduced decode a virtual image that holds exactly the tiles the
   window touches, at the reduced resolution (see b2k_codestream_parse_window below). */
static int64_t parse_impl(const uint8_t* cs, uint64_t len, const uint32_t* window, uint32_t reduce, b2k_coding* cp_out,
                          b2k_block* blocks, uint64_t cap_blocks)
{
  if(!cs || !cp_out)
    return -1;
  auto fail = [&](const char* m, int rc) {
    b2k_set_error(m);
    return (int64_t)rc;
  };
  t2::MainHeader mh;
  if(int rc = b2k_parse_main_header(cs, len, mh))
    return rc;
  Cursor c{cs + mh.sot, cs + len};
  const b2k_coding cp = mh.cp;
  const int progression = mh.progression;
  const bool use_sop = mh.sop, use_eph = mh.eph;
  const std::vector<std::vector<BandQuant>> q = component_quant(cp);
  const TileGrid g = tile_grid(cp);
  const uint32_t ntiles = g.nx * g.ny;
  t2::WindowCoding wc;
  if(int rc = b2k_window_coding(cp, window, reduce, wc))
    return rc;
  const bool whole = wc.whole;
  const uint32_t ta_x = wc.ta_x, ta_y = wc.ta_y, tb_x = wc.tb_x, tb_y = wc.tb_y;
  const b2k_coding& vcp = wc.vcp;
  const std::vector<Rect>& need = wc.need;
  const TileGrid vg = tile_grid(vcp);
  const uint32_t vnt = vg.nx * vg.ny;
  if(!whole && (vg.nx != tb_x - ta_x || vg.ny != tb_y - ta_y))
    return fail("internal: virtual tile grid", -1);
  const std::vector<std::vector<BandQuant>> vq = whole ? q : component_quant(vcp);
  /* block table of the virtual coding in enumeration order: sizes first, then every tile fills its own slice */
  std::vector<uint64_t> tile_first(vnt + 1, 0);
  for(uint32_t t = 0; t < vnt; ++t)
    tile_first[t + 1] = tile_first[t] + walk_precincts(vcp, tile_rect(vcp, vg, t), [](const PrecinctBand&) {});
  const uint64_t nblocks = tile_first[vnt];
  *cp_out = vcp;
  if(!blocks)
    return (int64_t)nblocks;
  if(cap_blocks < nblocks)
    return fail("block table too small", -1);

  /* ---- tile parts: locate them (SOT / Psot: one hop per tile part), then parse the packets of the wanted tiles on the
     host pool -- the other tiles' packets are never looked at ---- */
  std::vector<std::vector<ByteRange>> tile_parts(ntiles);
  std::vector<uint32_t> next_tp(ntiles, 0);
  for(;;)
  {
    const uint8_t* sot = c.p;
    const uint32_t m = c.u16();
    if(!c.ok)
      break; /* a missing EOC is tolerated */
    if(m == 0xFFD9)
      break;
    if(m != 0xFF90)
      return fail("expected SOT or EOC", -1);
    const uint32_t lsot = c.u16(), isot = c.u16();
    const uint32_t psot = c.u32();
    const uint32_t tpsot = c.u8(), tnsot = c.u8();
    (void)tnsot;
    if(!c.ok || lsot != 10 || isot >= ntiles)
      return fail("bad SOT", -1);
    if(tpsot != next_tp[isot])
      return fail("tile parts out of order", 1);
    ++next_tp[isot];
    const uint8_t* tp_end = psot ? sot + psot : c.end - ((len >= 2 && cs[len - 2] == 0xFF && cs[len - 1] == 0xD9) ? 2 : 0);
    if(tp_end > c.end || tp_end < c.p)
      return fail("Psot exceeds the codestream", -1);
    const uint32_t ix = isot % g.nx, iy = isot / g.nx;
    if(ix < ta_x || ix >= tb_x || iy < ta_y || iy >= tb_y)
    { /* not wanted: hop over it */
      c.p = tp_end;
      continue;
    }
    for(;;)
    { /* tile-part header */
      const uint32_t tm = c.u16();
      if(!c.ok)
        return fail("truncated tile-part header", -1);
      if(tm == 0xFF93)
        break;
      const uint32_t L = c.u16();
      if(!c.ok || L < 2 || c.p + (L - 2) > tp_end)
        return fail("bad tile-part marker segment", -1);
      if(tm == 0xFF52 || tm == 0xFF53 || tm == 0xFF5C || tm == 0xFF5D || tm == 0xFF5E || tm == 0xFF5F || tm == 0xFF61)
        return fail("tile-part COD / COC / QCD / QCC / RGN / POC / PPT are not handled", 1);
      c.p += L - 2; /* PLT, COM: skipped */
    }
    tile_parts[isot].push_back({c.p, tp_end});
    c.p = tp_end;
  }
  std::vector<int> rcs(vnt, 0);
  std::vector<std::string> errs(vnt);
  b2k_host_parallel(vnt, [&](size_t vt) {
    const uint32_t t = whole ? (uint32_t)vt : (ta_y + (uint32_t)vt / vg.nx) * g.nx + ta_x + (uint32_t)vt % vg.nx; /* the stream's tile */
    std::vector<b2k_block> tb;
    enumerate_tile_blocks(cp, t, tile_rect(cp, g, t), q, tb);
    if(!tile_parts[t].empty()) /* a tile without a tile part decodes as all zero (blocks stay uncoded) */
      rcs[vt] = parse_tile_packets(cp, tile_rect(cp, g, t), tb.data(), tile_parts[t], cs, progression, use_sop, use_eph, errs[vt]);
    if(whole)
    {
      memcpy(blocks + tile_first[vt], tb.data(), tb.size() * sizeof(b2k_block));
      return;
    }
    /* the virtual tile's own enumeration; the stream's blocks of the kept resolutions follow in the same order */
    std::vector<b2k_block> vb;
    enumerate_tile_blocks(vcp, (uint32_t)vt, tile_rect(vcp, vg, (uint32_t)vt), vq, vb);
    size_t k = 0;
    for(const b2k_block& b : tb)
    {
      if(b.resno >= vcp.numres)
        continue;
      if(k >= vb.size() || vb[k].comp != b.comp || vb[k].resno != b.resno || vb[k].band_index != b.band_index ||
         vb[k].precno != b.precno || vb[k].cblkno != b.cblkno || vb[k].x1 - vb[k].x0 != b.x1 - b.x0 || vb[k].y1 - vb[k].y0 != b.y1 - b.y0)
      {
        rcs[vt] = -1;
        errs[vt] = "internal: virtual and original block enumerations disagree";
        return;
      }
      bool wanted = true;
      if(!need.empty())
      { /* the block's rectangle is in band coordinates = those of resolution max(resno - 1, 0) */
        const Rect& n = need[vb[k].resno ? vb[k].resno - 1 : 0];
        wanted = vb[k].x0 < n.x1 && vb[k].x1 > n.x0 && vb[k].y0 < n.y1 && vb[k].y1 > n.y0;
      }
      if(wanted)
      {
        vb[k].length = b.length;
        vb[k].length2 = b.length2;
        vb[k].offset = b.offset;
        vb[k].numbps = b.numbps;
        vb[k].numpasses = b.numpasses;
      }
      ++k;
    }
    if(k != vb.size())
    {
      rcs[vt] = -1;
      errs[vt] = "internal: virtual tile holds a different number of blocks";
      return;
    }
    memcpy(blocks + tile_first[vt], vb.data(), vb.size() * sizeof(b2k_block));
  });
  for(uint32_t t = 0; t < vnt; ++t)
    if(rcs[t])
      return fail(errs[t].c_str(), rcs[t]);
  return (int64_t)nblocks;
}

extern "C" __attribute__((visibility("default"))) int64_t b2k_codestream_parse(const uint8_t* cs, uint64_t len, b2k_coding* cp_out,
                                                                                b2k_block* blocks, uint64_t cap_blocks)
{
  return parse_impl(cs, len, nullptr, 0, cp_out, blocks, cap_blocks);
}

/* Windowed / reduced-resolution parse (SURVEY.md 8f N3; reference: CodeStreamDecompress.cpp L670-870 window -> tiles,
 * t2/SelectiveFetchRanges.cpp, grk_decompress_parameters.core.reduce).  Tile-granular: *cp_out describes a virtual image
 * made of exactly the tiles the window touches, at 1 / 2^reduce of the resolution; decoding it with b2k_decode gives the
 * samples of that area, of which the window is a crop: window sample (x, y) at the reduced resolution -- x in
 * [ceil(wx0 / 2^reduce), ceil(wx1 / 2^reduce)) -- sits at column x - cp_out->x0 of the decoded planes.  Only the wanted
 * tiles' packet headers are parsed (tile parts are hopped over through Psot), only their code blocks are decoded. */
extern "C" __attribute__((visibility("default"))) int64_t b2k_codestream_parse_window(const uint8_t* cs, uint64_t len, const uint32_t* window,
                                                                                       uint32_t reduce, b2k_coding* cp_out, b2k_block* blocks,
                                                                                       uint64_t cap_blocks)
{
  return parse_impl(cs, len, window, reduce, cp_out, blocks, cap_blocks);
}

/* ============================================================================================================
 * JPH file format (T.814 Annex D: the JP2 box structure with brand 'jph '), the container Grok writes by default for
 * HT codestreams (fileformat/compress/FileFormatJP2Compress.cpp; brand selection in FileFormatJPHCompress).  Minimal
 * form: signature, file type, header (image header + enumerated colour space), contiguous codestream.
 * ============================================================================================================ */
namespace
{
void box(std::vector<uint8_t>& o, const char* type, const std::vector<uint8_t>& payload)
{
  put32(o, (uint32_t)payload.size() + 8);
  o.insert(o.end(), type, type + 4);
  o.insert(o.end(), payload.begin(), payload.end());
}
} // namespace

extern "C" __attribute__((visibility("default"))) int64_t b2k_jph_wrap(const b2k_coding* cp, const uint8_t* cs, uint64_t cs_len,
                                                                        uint8_t* out, uint64_t cap)
{
  if(!cp || (!cs && cs_len))
    return -1;
  std::vector<uint8_t> o;
  box(o, "jP  ", {0x0D, 0x0A, 0x87, 0x0A});
  {
    std::vector<uint8_t> p = {'j', 'p', 'h', ' ', 0, 0, 0, 0, 'j', 'p', 'h', ' '};
    box(o, "ftyp", p);
  }
  {
    std::vector<uint8_t> ihdr, colr, hdr;
    put32(ihdr, cp->y1 - cp->y0);
    put32(ihdr, cp->x1 - cp->x0);
    put16(ihdr, cp->numcomps);
    ihdr.push_back((uint8_t)((cp->prec - 1) | (cp->sgnd ? 0x80 : 0)));
    ihdr.push_back(7); /* compression type */
    ihdr.push_back(0); /* colour space known */
    ihdr.push_back(0); /* no IPR */
    colr = {1, 0, 0};  /* enumerated colour space */
    put32(colr, cp->numcomps >= 3 ? 16u : 17u); /* sRGB / greyscale */
    box(hdr, "ihdr", ihdr);
    box(hdr, "colr", colr);
    box(o, "jp2h", hdr);
  }
  const uint64_t total = o.size() + 8 + cs_len;
  if(total > 0xFFFFFFFFull)
  {
    b2k_set_error("file larger than 4 GiB: extended box lengths are not written");
    return -1;
  }
  if(!out || cap < total)
    return (int64_t)total;
  put32(o, (uint32_t)(cs_len + 8));
  o.insert(o.end(), {'j', 'p', '2', 'c'});
  memcpy(out, o.data(), o.size());
  memcpy(out + o.size(), cs, cs_len);
  return (int64_t)total;
}

/* locate the contiguous codestream inside a JP2 / JPH file (or accept a raw codestream): 0 + offset/length, <0 none */
extern "C" __attribute__((visibility("default"))) int32_t b2k_jph_codestream(const uint8_t* file, uint64_t len, uint64_t* off,
                                                                              uint64_t* n)
{
  if(!file || !off || !n)
    return -1;
  if(len >= 2 && file[0] == 0xFF && file[1] == 0x4F)
  {
    *off = 0;
    *n = len;
    return 0;
  }
  uint64_t p = 0;
  while(p + 8 <= len)
  {
    uint64_t L = ((uint64_t)file[p] << 24) | ((uint64_t)file[p + 1] << 16) | ((uint64_t)file[p + 2] << 8) | file[p + 3];
    uint64_t hdr = 8;
    if(L == 1)
    { /* extended length */
      if(p + 16 > len)
        break;
      L = 0;
      for(int i = 0; i < 8; ++i)
        L = (L << 8) | file[p + 8 + i];
      hdr = 16;
    }
    else if(L == 0)
      L = len - p; /* box runs to the end of the file */
    if(L < hdr || p + L > len)
      break;
    if(memcmp(file + p + 4, "jp2c", 4) == 0)
    {
      *off = p + hdr;
      *n = L - hdr;
      return 0;
    }
    p += L;
  }
  b2k_set_error("no contiguous codestream box");
  return -1;
}
