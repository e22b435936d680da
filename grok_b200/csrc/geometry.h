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

/* append the blocks of one tile (all components) in Grok's enumeration order; q[comp] = band_quant(cp, comp) */
void enumerate_tile_blocks(const b2k_coding& cp, uint32_t tile_index, const Rect& tile,
                           const std::vector<std::vector<BandQuant>>& q, std::vector<b2k_block>& out);
/* the same with one table for every component (a coding without QCC or quality factor) */
void enumerate_tile_blocks(const b2k_coding& cp, uint32_t tile_index, const Rect& tile,
                           const std::vector<BandQuant>& q, std::vector<b2k_block>& out);

/* the subset of a b2k_coding this engine handles; returns nullptr if fine, else the reason */
const char* unsupported_reason(const b2k_coding& cp);

} // namespace b2k
