/*
 * grok_b200/csrc/geometry.h -- host-side JPEG 2000 canvas geometry and quantiser tables.
 * Reproduces, for the tile engine, the rules Grok's canvas classes implement (all canvas
 * coordinates):
 *   tile / tile-component / resolution rects   tile_processor/TileProcessor.cpp L329-351
 *   band rects                                  canvas/resolution/ResSimple.h L81-109
 *   precinct partition, band precincts          canvas/resolution/Resolution.cpp L69-160, canvas/subband/Subband.cpp L66-78
 *   code-block grid                             canvas/precinct/PrecinctImpl.cpp L45-66
 *   Mallat buffer position of a block           canvas/tile/TileComponentWindow.h L241-264
 *   enumeration order comp->res->band->prec->cblk  scheduling/standard/CompressScheduler.cpp L84-139
 *   HT step sizes / exponents                   t2/quantizer/part15/QuantizerOJPH.cpp L150-259
 *   quality-factor step sizes (--qfactor)       CodeStreamCompress.cpp L591-630 (derived here from T.800 F / G)
 *   band step size and Kmax                     tile_processor/TileProcessor.cpp L398-419
 * Product code (no oracle/ dependency).
 */
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>
#include "../../include/grok_b200.h"

namespace b2k {

struct Rect
{
  uint32_t x0, y0, x1, y1;
  uint32_t w() const { return x1 > x0 ? x1 - x0 : 0; }
  uint32_t h() const { return y1 > y0 ? y1 - y0 : 0; }
  bool empty() const { return x1 <= x0 || y1 <= y0; }
};

inline uint32_t ceil_div_pow2(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a + ((1ull << b) - 1)) >> b); }
inline uint32_t ceil_div(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a + b - 1) / b); }

struct TileGrid
{
  uint32_t tw, th, nx, ny;
  uint32_t tx0, ty0;
};
TileGrid tile_grid(const b2k_coding& cp);
Rect tile_rect(const b2k_coding& cp, const TileGrid& g, uint32_t tile_index);
Rect resolution_rect(const Rect& tc, int numres, int resno);
Rect band_rect(const Rect& tc, int numres, int resno, int orient);

struct BandQuant
{
  uint8_t expn;
  uint16_t mant;
  uint8_t kmax;         /* maxBitPlanes_ */
  float step_enc;       /* encoder convention (sub-band gain included) */
  float step_dec;       /* decoder convention (gain 0 when irreversible) */
};
/* Component comp's band exponents, mantissas, Kmax and steps: the one place that chooses them -- Grok's HT tables, or
   QCD's (qcd_explicit), or the component's QCC (qcc_mask), or the quality factor's (qfactor), in rising precedence.
   index = 0 for LL, else 1 + 3*(resno-1) + (orient-1) */
std::vector<BandQuant> band_quant(const b2k_coding& cp, int comp = 0);
/* grk_compress --qfactor q's table for one component: (exponent << 11 | mantissa) per band, QCD order */
const std::vector<uint32_t>& qfactor_words(int q, int prec, int numres, int comp);
/* band_quant of every component, indexed [comp][band] */
std::vector<std::vector<BandQuant>> component_quant(const b2k_coding& cp);
/* the same exponents and mantissas (what QCC is written for when it differs from QCD) */
bool same_quant(const std::vector<BandQuant>& a, const std::vector<BandQuant>& b);
inline int band_quant_index(int resno, int orient) { return resno == 0 ? 0 : 1 + 3 * (resno - 1) + (orient - 1); }

/* ---- the precincts of a tile ---------------------------------------------------------------------------------------
 * The one place that partitions a tile's resolutions into precincts (T.800 B.6) and their bands into code blocks (B.7):
 * the block enumeration, the packets of the code-stream writers and parsers, and the plugin's gpup trees all take their
 * geometry from here. */
struct PrecinctGrid /* the precinct partition of one resolution of a tile component */
{
  Rect res;          /* the resolution */
  uint32_t pw, ph;   /* precinct exponents */
  uint32_t px0, py0; /* the partition's origin: res.x0, res.y0 rounded down to a precinct corner */
  uint32_t gw, gh;   /* precincts across and down; an empty resolution has none (B.6) */
};
PrecinctGrid precinct_grid(const b2k_coding& cp, const Rect& tile, int resno);

struct PrecinctBand /* one band of one precinct */
{
  uint16_t comp;
  uint8_t resno, band_index, orient, nbands;
  uint32_t precno;
  uint32_t xpos, ypos;     /* where the position-driven progressions meet the precinct on the reference grid (B.12.1.3-5) */
  Rect band;               /* the whole band */
  Rect rect;               /* the precinct's part of the band; may be empty */
  uint32_t cbw, cbh;       /* code-block exponents */
  uint32_t gx, gy, gw, gh; /* the code-block grid of rect; 0 x 0 when rect is empty */
  uint32_t first;          /* the index of its first block in the tile's enumeration */
};

/* visit(const PrecinctBand&) for every band of every precinct of the tile, empty ones included, in Grok's enumeration
   order: component -> resolution -> band -> precinct.  Returns the number of code blocks in the tile. */
template <class Visit>
uint32_t walk_precincts(const b2k_coding& cp, const Rect& tile, Visit&& visit)
{
  uint32_t first = 0;
  PrecinctBand pb{};
  for(uint16_t comp = 0; comp < cp.numcomps; ++comp)
    for(int resno = 0; resno < cp.numres; ++resno)
    {
      const PrecinctGrid g = precinct_grid(cp, tile, resno);
      /* a precinct of a resolution above 0 spans half as many samples in each of its three bands */
      const uint32_t bpw = resno ? g.pw - 1 : g.pw, bph = resno ? g.ph - 1 : g.ph;
      const uint32_t bpx0 = resno ? g.px0 >> 1 : g.px0, bpy0 = resno ? g.py0 >> 1 : g.py0;
      const uint32_t nd = (uint32_t)(cp.numres - 1 - resno);
      pb.comp = comp;
      pb.resno = (uint8_t)resno;
      pb.nbands = resno ? 3 : 1;
      pb.cbw = std::min<uint32_t>(cp.cblkw_exp, bpw);
      pb.cbh = std::min<uint32_t>(cp.cblkh_exp, bph);
      for(uint8_t b = 0; b < pb.nbands; ++b)
      {
        pb.band_index = b;
        pb.orient = resno ? b + 1 : 0;
        pb.band = band_rect(tile, cp.numres, resno, pb.orient);
        for(uint64_t p = 0; p < (uint64_t)g.gw * g.gh; ++p)
        {
          const uint32_t ix = (uint32_t)(p % g.gw), iy = (uint32_t)(p / g.gw);
          pb.precno = (uint32_t)p;
          /* a precinct is met where its corner lies on the reference grid; the first column / row of a resolution whose
             origin is not precinct aligned is met at the tile's edge instead */
          const uint64_t cx = ((uint64_t)(g.px0 >> g.pw) + ix) << (g.pw + nd), cy = ((uint64_t)(g.py0 >> g.ph) + iy) << (g.ph + nd);
          pb.xpos = (ix == 0 && g.px0 != g.res.x0) ? tile.x0 : (uint32_t)std::min<uint64_t>(cx, 0xFFFFFFFFull);
          pb.ypos = (iy == 0 && g.py0 != g.res.y0) ? tile.y0 : (uint32_t)std::min<uint64_t>(cy, 0xFFFFFFFFull);
          Rect& r = pb.rect;
          r.x0 = bpx0 + (ix << bpw);
          r.y0 = bpy0 + (iy << bph);
          r.x1 = (uint32_t)std::min<uint64_t>((uint64_t)r.x0 + (1ull << bpw), pb.band.x1);
          r.y1 = (uint32_t)std::min<uint64_t>((uint64_t)r.y0 + (1ull << bph), pb.band.y1);
          r.x0 = std::max(r.x0, pb.band.x0);
          r.y0 = std::max(r.y0, pb.band.y0);
          pb.gx = r.x0 >> pb.cbw;
          pb.gy = r.y0 >> pb.cbh;
          pb.gw = r.empty() ? 0 : ceil_div_pow2(r.x1, pb.cbw) - pb.gx;
          pb.gh = r.empty() ? 0 : ceil_div_pow2(r.y1, pb.cbh) - pb.gy;
          pb.first = first;
          visit(pb);
          first += pb.gw * pb.gh;
        }
      }
    }
  return first;
}

/* append the blocks of one tile (all components) in Grok's enumeration order; q[comp] = band_quant(cp, comp) */
void enumerate_tile_blocks(const b2k_coding& cp, uint32_t tile_index, const Rect& tile,
                           const std::vector<std::vector<BandQuant>>& q, std::vector<b2k_block>& out);
/* the same with one table for every component (a coding without QCC or quality factor) */
void enumerate_tile_blocks(const b2k_coding& cp, uint32_t tile_index, const Rect& tile,
                           const std::vector<BandQuant>& q, std::vector<b2k_block>& out);

/* the subset of a b2k_coding this engine handles; returns nullptr if fine, else the reason */
const char* unsupported_reason(const b2k_coding& cp);

} // namespace b2k
