/*
 * grok_b200/csrc/t2_packet.h -- the byte format of packet headers and tile-part markers, for the host writer
 * (codestream.cpp) and the device writer (t2_device.cu) alike: bit writer with 0xFF stuffing, tag-tree encoder, pass
 * count / Lblock / lengths, SOP / EPH, SOT, PLT and TLM.  Everything works over buffers the caller provides.
 * Written from ITU-T T.800 Annex A/B and T.814 Annex B.
 */
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define B2K_HD __host__ __device__ __forceinline__
#else
#define B2K_HD inline
#endif

namespace b2k
{
namespace t2
{

B2K_HD int floorlog2(uint32_t v)
{
  int l = 0;
  while(v > 1)
  {
    v >>= 1;
    ++l;
  }
  return l;
}

/* ---- packet-header bits: MSB first, the byte after 0xFF carries 7 bits (T.800 B.10.1) ---------------------------------
 * Writes into out[0, cap); n counts every byte produced, so n > cap afterwards means the buffer was too small. */
struct BitWriter
{
  uint8_t* out;
  uint64_t cap, n;
  uint32_t acc;
  int bits, room; /* bits the current byte holds / still free */
  uint8_t last;
  B2K_HD void init(uint8_t* o, uint64_t c)
  {
    out = o;
    cap = c;
    n = 0;
    acc = 0;
    bits = room = 8;
    last = 0;
  }
  B2K_HD void byte(uint8_t v) /* a whole byte outside the bit stream (SOP, EPH) */
  {
    if(n < cap)
      out[n] = v;
    ++n;
    last = v;
  }
  B2K_HD void emit()
  {
    byte((uint8_t)acc);
    bits = room = (acc == 0xFF) ? 7 : 8;
    acc = 0;
  }
  B2K_HD void put(uint32_t bit)
  {
    --room;
    acc |= (bit & 1u) << room;
    if(room == 0)
      emit();
  }
  B2K_HD void put_bits(uint32_t v, int k)
  {
    for(int i = k - 1; i >= 0; --i)
      put((v >> i) & 1u);
  }
  B2K_HD void flush()
  {
    if(room != bits)
      emit();
    if(n && last == 0xFF)
      emit(); /* a header must not end on 0xFF: the stuffed byte follows */
  }
};

/* ---- tag-tree encoder (T.800 B.10.2) over caller storage ------------------------------------------------------------
 * Level l (0 = the leaves) holds ceil(w / 2^l) x ceil(h / 2^l) nodes; levels are stored leaves first, the root last. */
struct TagNode
{
  uint32_t value; /* minimum of the leaves below */
  uint32_t low;   /* lower bound signalled so far; bit 31: value signalled */
};
constexpr uint32_t TAG_INF = 0x7FFFFFFFu;
constexpr uint32_t TAG_KNOWN = 0x80000000u;

B2K_HD uint32_t tag_level_w(uint32_t w, int l) { return (uint32_t)(((uint64_t)w + (1ull << l) - 1) >> l); }
/* node count of a w x h tree (w, h >= 1); *levels = its number of levels */
B2K_HD uint32_t tag_nodes(uint32_t w, uint32_t h, int* levels)
{
  uint32_t total = 0;
  int l = 0;
  for(;; ++l)
  {
    const uint32_t lw = tag_level_w(w, l), lh = tag_level_w(h, l);
    total += lw * lh;
    if(lw <= 1 && lh <= 1)
      break;
  }
  if(levels)
    *levels = l + 1;
  return total;
}
/* leaf (x, y) takes value v: every node above it holds the minimum of its leaves */
B2K_HD void tag_set(TagNode* nd, uint32_t w, uint32_t h, uint32_t x, uint32_t y, uint32_t v)
{
  uint32_t base = 0;
  for(int l = 0;; ++l)
  {
    const uint32_t lw = tag_level_w(w, l), lh = tag_level_w(h, l);
    TagNode& t = nd[base + (y >> l) * lw + (x >> l)];
    if(t.value <= v)
      return;
    t.value = v;
    if(lw <= 1 && lh <= 1)
      return;
    base += lw * lh;
  }
}
/* the bits that tell whether leaf (x, y) is below `threshold`, and its value when it is; walks from the root down, where
   level l starts at the start of level l + 1 minus its own size */
B2K_HD void tag_encode(BitWriter& bw, TagNode* nd, uint32_t w, uint32_t h, uint32_t nodes, int levels, uint32_t x, uint32_t y,
                       uint32_t threshold)
{
  uint32_t low = 0, base = nodes;
  for(int l = levels - 1; l >= 0; --l)
  {
    const uint32_t lw = tag_level_w(w, l);
    base -= lw * tag_level_w(h, l);
    TagNode& t = nd[base + (y >> l) * lw + (x >> l)];
    bool known = (t.low & TAG_KNOWN) != 0;
    const uint32_t tl = t.low & ~TAG_KNOWN;
    if(low < tl)
      low = tl;
    while(low < threshold)
    {
      if(low >= t.value)
      {
        if(!known)
        {
          bw.put(1);
          known = true;
        }
        break;
      }
      bw.put(0);
      ++low;
    }
    t.low = low | (known ? TAG_KNOWN : 0u);
  }
}

/* ---- one packet (one quality layer, HT code blocks) ------------------------------------------------------------------ */
struct BandGrid
{
  uint32_t first, gw, gh; /* first block (index into the caller's block numbering), code-block grid of the precinct band */
};
struct BlockCode
{
  uint32_t length, length2; /* cleanup segment, refinement segment */
  uint8_t numpasses, numbps, kmax;
};

/* bytes one packet's header (SOP and EPH included) can take: per band, every tag-tree node signals at most 2 inclusion
   bits and kmax + 1 zero-bit-plane bits; per block at most 4 pass-count bits, 30 Lblock bits and 32 + 33 length bits;
   the non-empty bit; at least 7 bits per byte after stuffing, plus the byte a final 0xFF pulls in */
B2K_HD uint64_t packet_header_bound(const BandGrid* band, int nbands, uint32_t kmax)
{
  uint64_t bits = 1;
  for(int b = 0; b < nbands; ++b)
  {
    const uint64_t n = (uint64_t)band[b].gw * band[b].gh;
    if(n)
      bits += (uint64_t)tag_nodes(band[b].gw, band[b].gh, nullptr) * (kmax + 3u) + 100u * n;
  }
  return bits / 7 + 2 + 6 + 2;
}

/* the tag-tree scratch packet_header needs: two trees of the largest band */
B2K_HD uint32_t packet_tag_nodes(const BandGrid* band, int nbands)
{
  uint32_t m = 0;
  for(int b = 0; b < nbands; ++b)
    if(band[b].gw && band[b].gh)
    {
      const uint32_t n = tag_nodes(band[b].gw, band[b].gh, nullptr);
      m = n > m ? n : m;
    }
  return 2 * m;
}

/* SOP, the header bits and EPH of one packet (T.800 B.10, T.814 B.10.7): a block is included when it has passes and
   bytes.  get(i) is the BlockCode of block i; tags holds packet_tag_nodes(band, nbands) nodes.  0, or -1 when a block is
   outside the writer's range (more bit planes than Kmax, more than 3 passes). */
template <class Get>
B2K_HD int packet_header(BitWriter& bw, const BandGrid* band, int nbands, const Get& get, TagNode* tags, uint32_t sop_index,
                         bool sop, bool eph)
{
  if(sop)
  { /* SOP (A.8.1): marker, Lsop = 4, packet counter modulo 65536 */
    bw.byte(0xFF);
    bw.byte(0x91);
    bw.byte(0);
    bw.byte(4);
    bw.byte((uint8_t)(sop_index >> 8));
    bw.byte((uint8_t)sop_index);
  }
  bw.put(1); /* non-empty packet; also when it carries no block, as the reference writes it */
  for(int b = 0; b < nbands; ++b)
  {
    const uint32_t gw = band[b].gw, gh = band[b].gh, n = gw * gh;
    if(!n)
      continue;
    int levels = 0;
    const uint32_t nodes = tag_nodes(gw, gh, &levels);
    TagNode* incl = tags;
    TagNode* imsb = tags + nodes;
    for(uint32_t i = 0; i < 2 * nodes; ++i)
      tags[i] = TagNode{TAG_INF, 0};
    for(uint32_t k = 0; k < n; ++k)
    {
      const BlockCode B = get(band[b].first + k);
      if(B.numpasses && B.length)
      {
        if(B.numbps > B.kmax || B.numpasses > 3)
          return -1;
        tag_set(incl, gw, gh, k % gw, k / gw, 0);
        tag_set(imsb, gw, gh, k % gw, k / gw, (uint32_t)B.kmax - B.numbps);
      }
      else
        tag_set(incl, gw, gh, k % gw, k / gw, 1); /* never included in the only layer */
    }
    for(uint32_t k = 0; k < n; ++k)
    {
      const BlockCode B = get(band[b].first + k);
      tag_encode(bw, incl, gw, gh, nodes, levels, k % gw, k / gw, 1);
      if(!(B.numpasses && B.length))
        continue;
      tag_encode(bw, imsb, gw, gh, nodes, levels, k % gw, k / gw, TAG_INF);
      /* number of passes (B.10.6): 1 -> 0, 2 -> 10, 3 -> 1100 */
      if(B.numpasses == 1)
        bw.put(0);
      else if(B.numpasses == 2)
        bw.put_bits(2, 2);
      else
        bw.put_bits(12, 4);
      /* HT: the cleanup segment, then one segment for the refinement passes (T.814 B.10.7) */
      const uint32_t len1 = B.length, len2 = B.numpasses > 1 ? B.length2 : 0;
      const int extra2 = B.numpasses > 1 ? floorlog2((uint32_t)B.numpasses - 1) : 0;
      int lblock = 3, inc = 0;
      inc = inc > floorlog2(len1) + 1 - lblock ? inc : floorlog2(len1) + 1 - lblock;
      if(B.numpasses > 1)
      {
        const int need = floorlog2(len2 > 1 ? len2 : 1) + 1 - (lblock + extra2);
        inc = inc > need ? inc : need;
      }
      for(int i = 0; i < inc; ++i)
        bw.put(1);
      bw.put(0);
      lblock += inc;
      bw.put_bits(len1, lblock);
      if(B.numpasses > 1)
        bw.put_bits(len2, lblock + extra2);
    }
  }
  bw.flush();
  if(eph)
  { /* EPH (A.8.2) */
    bw.byte(0xFF);
    bw.byte(0x92);
  }
  return 0;
}

/* ---- tile-part markers ---------------------------------------------------------------------------------------------- */
/* SOT (A.4.2): tile index, Psot = bytes of the whole tile part, its index, the tile's number of tile parts */
B2K_HD void put_sot(uint8_t* w, uint32_t tile, uint32_t psot, uint32_t part, uint32_t nparts)
{
  w[0] = 0xFF;
  w[1] = 0x90;
  w[2] = 0;
  w[3] = 10; /* Lsot */
  w[4] = (uint8_t)(tile >> 8);
  w[5] = (uint8_t)tile;
  w[6] = (uint8_t)(psot >> 24);
  w[7] = (uint8_t)(psot >> 16);
  w[8] = (uint8_t)(psot >> 8);
  w[9] = (uint8_t)psot;
  w[10] = (uint8_t)part;
  w[11] = (uint8_t)nparts;
}

/* PLT marker segments (A.7.3) of the packets k in [p0, p1) whose lengths are len(k): 7 bits per byte, MSB = continuation;
   a segment is closed when the next length would take its Iplt bytes past 65532.  A tile part without packets still
   carries one empty segment.  Writes at out (NULL: counts only); returns the bytes. */
B2K_HD void put_plt_head(uint8_t* w, uint32_t iplt_bytes, uint8_t z)
{
  w[0] = 0xFF;
  w[1] = 0x58;
  w[2] = (uint8_t)((iplt_bytes + 3) >> 8);
  w[3] = (uint8_t)(iplt_bytes + 3);
  w[4] = z;
}
template <class Len>
B2K_HD uint64_t plt_segments(const Len& len, uint64_t p0, uint64_t p1, uint8_t* out)
{
  uint64_t seg_at = 0, n = 5;
  uint32_t seg = 0;
  uint8_t z = 0;
  for(uint64_t k = p0; k < p1; ++k)
  {
    const uint32_t L = len(k);
    int nb = 1;
    while(nb < 5 && (L >> (7 * nb)))
      ++nb;
    if(seg + nb > 65535 - 3)
    {
      if(out)
        put_plt_head(out + seg_at, seg, z);
      ++z;
      seg_at = n;
      n += 5;
      seg = 0;
    }
    for(int i = nb - 1; i >= 0; --i)
    {
      if(out)
        out[n] = (uint8_t)(((L >> (7 * i)) & 0x7F) | (i ? 0x80 : 0));
      ++n;
    }
    seg += (uint32_t)nb;
  }
  if(out)
    put_plt_head(out + seg_at, seg, z);
  return n;
}

/* TLM (A.7.1): segments of at most 10000 entries, each a 16-bit tile index and a 32-bit tile-part length */
constexpr uint64_t TLM_PER_SEGMENT = 10000;
B2K_HD uint64_t tlm_bytes(uint64_t entries) { return (entries + TLM_PER_SEGMENT - 1) / TLM_PER_SEGMENT * 6 + 6 * entries; }
B2K_HD uint64_t tlm_entry_at(uint64_t e) { return (e / TLM_PER_SEGMENT + 1) * 6 + 6 * e; }
/* the head of the segment that holds entries [e0, e0 + n), at its place in a buffer of tlm_bytes */
B2K_HD void put_tlm_segment(uint8_t* tlm, uint64_t e0, uint64_t n)
{
  uint8_t* w = tlm + tlm_entry_at(e0) - 6;
  const uint32_t L = (uint32_t)(4 + 6 * n);
  w[0] = 0xFF;
  w[1] = 0x55;
  w[2] = (uint8_t)(L >> 8);
  w[3] = (uint8_t)L;
  w[4] = (uint8_t)(e0 / TLM_PER_SEGMENT);
  w[5] = 0x60; /* ST = 2 (16-bit Ttlm), SP = 1 (32-bit Ptlm) */
}
B2K_HD void put_tlm_entry(uint8_t* tlm, uint64_t e, uint32_t tile, uint32_t len)
{
  uint8_t* w = tlm + tlm_entry_at(e);
  w[0] = (uint8_t)(tile >> 8);
  w[1] = (uint8_t)tile;
  w[2] = (uint8_t)(len >> 24);
  w[3] = (uint8_t)(len >> 16);
  w[4] = (uint8_t)(len >> 8);
  w[5] = (uint8_t)len;
}

} // namespace t2
} // namespace b2k
