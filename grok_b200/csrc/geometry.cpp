/* see geometry.h for the reference citations */
#include "geometry.h"
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <map>
#include <mutex>

namespace b2k {

TileGrid tile_grid(const b2k_coding& cp)
{
  TileGrid g;
  if(cp.tw == 0 || cp.th == 0)
  { /* untiled: one tile covering the image, anchored at the image origin */
    g.tx0 = cp.x0;
    g.ty0 = cp.y0;
    g.tw = cp.x1 - cp.x0;
    g.th = cp.y1 - cp.y0;
    g.nx = g.ny = 1;
    return g;
  }
  g.tx0 = cp.tx0;
  g.ty0 = cp.ty0;
  g.tw = cp.tw;
  g.th = cp.th;
  g.nx = ceil_div(cp.x1 - cp.tx0, cp.tw);
  g.ny = ceil_div(cp.y1 - cp.ty0, cp.th);
  return g;
}

Rect tile_rect(const b2k_coding& cp, const TileGrid& g, uint32_t t)
{
  const uint32_t p = t % g.nx, q = t / g.nx;
  Rect r;
  r.x0 = std::max<uint64_t>((uint64_t)g.tx0 + (uint64_t)p * g.tw, cp.x0);
  r.y0 = std::max<uint64_t>((uint64_t)g.ty0 + (uint64_t)q * g.th, cp.y0);
  r.x1 = (uint32_t)std::min<uint64_t>((uint64_t)g.tx0 + (uint64_t)(p + 1) * g.tw, cp.x1);
  r.y1 = (uint32_t)std::min<uint64_t>((uint64_t)g.ty0 + (uint64_t)(q + 1) * g.th, cp.y1);
  return r;
}

Rect resolution_rect(const Rect& tc, int numres, int resno)
{
  const uint32_t n = (uint32_t)(numres - 1 - resno);
  return Rect{ceil_div_pow2(tc.x0, n), ceil_div_pow2(tc.y0, n), ceil_div_pow2(tc.x1, n), ceil_div_pow2(tc.y1, n)};
}

PrecinctGrid precinct_grid(const b2k_coding& cp, const Rect& tile, int resno)
{
  PrecinctGrid g;
  g.res = resolution_rect(tile, cp.numres, resno);
  g.pw = cp.prcw_exp[resno] ? cp.prcw_exp[resno] : 15;
  g.ph = cp.prch_exp[resno] ? cp.prch_exp[resno] : 15;
  g.px0 = (g.res.x0 >> g.pw) << g.pw;
  g.py0 = (g.res.y0 >> g.ph) << g.ph;
  g.gw = g.res.empty() ? 0 : ceil_div_pow2(g.res.x1, g.pw) - (g.res.x0 >> g.pw);
  g.gh = g.res.empty() ? 0 : ceil_div_pow2(g.res.y1, g.ph) - (g.res.y0 >> g.ph);
  return g;
}

static uint32_t band_coord(uint32_t c, uint32_t ndecomp, uint32_t high)
{
  if(ndecomp == 0)
    return c;
  const uint32_t off = (1u << (ndecomp - 1)) * high;
  return c <= off ? 0 : ceil_div_pow2(c - off, ndecomp);
}

Rect band_rect(const Rect& tc, int numres, int resno, int orient)
{
  const uint32_t level = resno == 0 ? (uint32_t)(numres - 1) : (uint32_t)(numres - resno);
  const uint32_t hx = orient & 1, hy = (orient >> 1) & 1;
  return Rect{band_coord(tc.x0, level, hx), band_coord(tc.y0, level, hy), band_coord(tc.x1, level, hx),
              band_coord(tc.y1, level, hy)};
}

/* ---- quantiser ------------------------------------------------------------------------------ */
static const float kBibo53L[34] = {
    1.0000e+00f, 1.5000e+00f, 1.6250e+00f, 1.6875e+00f, 1.6963e+00f, 1.7067e+00f, 1.7116e+00f, 1.7129e+00f,
    1.7141e+00f, 1.7145e+00f, 1.7151e+00f, 1.7152e+00f, 1.7155e+00f, 1.7155e+00f, 1.7156e+00f, 1.7156e+00f,
    1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f,
    1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f,
    1.7156e+00f, 1.7156e+00f};
static const float kBibo53H[34] = {
    2.0000e+00f, 2.5000e+00f, 2.7500e+00f, 2.8047e+00f, 2.8198e+00f, 2.8410e+00f, 2.8558e+00f, 2.8601e+00f,
    2.8628e+00f, 2.8656e+00f, 2.8662e+00f, 2.8667e+00f, 2.8669e+00f, 2.8670e+00f, 2.8671e+00f, 2.8671e+00f,
    2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f,
    2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f,
    2.8671e+00f, 2.8671e+00f};
/* sqrt energy gains of the 9/7 synthesis filters, per number of decompositions */
static const float kGain97L[34] = {
    1.0000e+00f, 1.4021e+00f, 2.0304e+00f, 2.9012e+00f, 4.1153e+00f, 5.8245e+00f, 8.2388e+00f, 1.1652e+01f,
    1.6479e+01f, 2.3304e+01f, 3.2957e+01f, 4.6609e+01f, 6.5915e+01f, 9.3217e+01f, 1.3183e+02f, 1.8643e+02f,
    2.6366e+02f, 3.7287e+02f, 5.2732e+02f, 7.4574e+02f, 1.0546e+03f, 1.4915e+03f, 2.1093e+03f, 2.9830e+03f,
    4.2185e+03f, 5.9659e+03f, 8.4371e+03f, 1.1932e+04f, 1.6874e+04f, 2.3864e+04f, 3.3748e+04f, 4.7727e+04f,
    6.7496e+04f, 9.5454e+04f};
static const float kGain97H[34] = {
    1.4425e+00f, 1.9669e+00f, 2.8839e+00f, 4.1475e+00f, 5.8946e+00f, 8.3472e+00f, 1.1809e+01f, 1.6701e+01f,
    2.3620e+01f, 3.3403e+01f, 4.7240e+01f, 6.6807e+01f, 9.4479e+01f, 1.3361e+02f, 1.8896e+02f, 2.6723e+02f,
    3.7792e+02f, 5.3446e+02f, 7.5583e+02f, 1.0689e+03f, 1.5117e+03f, 2.1378e+03f, 3.0233e+03f, 4.2756e+03f,
    6.0467e+03f, 8.5513e+03f, 1.2093e+04f, 1.7103e+04f, 2.4187e+04f, 3.4205e+04f, 4.8373e+04f, 6.8410e+04f,
    9.6747e+04f, 1.3682e+05f};

static void irrev_expn_mant(float delta_b, uint8_t& e, uint16_t& m)
{
  int exp = 0;
  while(delta_b < 1.0f)
  {
    exp++;
    delta_b *= 2.0f;
  }
  int mant = (int)std::round(delta_b * (float)(1 << 11)) - (1 << 11);
  mant = mant < (1 << 11) ? mant : 0x7FF;
  e = (uint8_t)exp;
  m = (uint16_t)mant;
}

/* ---- quality factor -------------------------------------------------------------------------
 * The JPEG-style quality model grk_compress --qfactor, Kakadu's Qfactor and OpenHTJ2K share: a reference step from the
 * quality factor, divided per band by the norm of the band's 9/7 synthesis basis function, a visual weight and the norm
 * of the component's inverse-ICT column.  Everything is double and evaluated in the order written (geometry.cpp is
 * compiled with -ffp-contract=off), so the tables do not depend on the target's FMA support. */

/* 9/7 synthesis low-pass (7 taps) and high-pass (9 taps) filters, T.800 Annex F (Table F.4, synthesis side) */
static const double kSyn97Lo[7] = {-0.091271763114250, -0.057543526228500, 0.591271763114250, 1.115087052457000,
                                   0.591271763114250,  -0.057543526228500, -0.091271763114250};
static const double kSyn97Hi[9] = {0.053497514821622,  0.033728236885750, -0.156446533057980, -0.533728236885750, 1.205898036472720,
                                   -0.533728236885750, -0.156446533057980, 0.033728236885750,  0.053497514821622};
/* Zeng, Daly and Lei, "An overview of the visual optimization tools in JPEG 2000" (2002), Table 2, square-root domain,
   4:4:4: five decomposition levels from the finest, HH, LH, HL within each.  Coarser bands and LL weigh 1. */
static const double kVisY[15] = {0.0901, 0.2758, 0.2758, 0.7018, 0.8378, 0.8378, 1.0000, 1.0000,
                                 1.0000, 1.0000, 1.0000, 1.0000, 1.0000, 1.0000, 1.0000};
static const double kVisCb[15] = {0.0263, 0.0863, 0.0863, 0.1362, 0.2564, 0.2564, 0.3346, 0.4691,
                                  0.4691, 0.5444, 0.6523, 0.6523, 0.7078, 0.7797, 0.7797};
static const double kVisCr[15] = {0.0773, 0.1835, 0.1835, 0.2598, 0.4130, 0.4130, 0.5040, 0.6464,
                                  0.6464, 0.7220, 0.8254, 0.8254, 0.8769, 0.9424, 0.9424};
/* norms of the columns of the inverse ICT (T.800 G.3, equation G-7), rounded to four places */
static const double kIctNorm[3] = {1.7321, 1.8051, 1.5734};

static double sum_squares(const std::vector<double>& f)
{
  double s = 0.0;
  for(double t : f)
    s += t * t;
  return s;
}

/* f(z) -> H0(z) f(z^2): the synthesis filter one decomposition level coarser */
static std::vector<double> coarser(const std::vector<double>& f)
{
  std::vector<double> r(7 + 2 * f.size() - 1, 0.0);
  for(size_t i = 0; i < 7; ++i)
    for(size_t j = 0; j < f.size(); ++j)
      r[i + 2 * j] += kSyn97Lo[i] * f[j];
  return r;
}

/* energies (sums of squared taps) of the low- and high-pass synthesis filters of decomposition level l + 1, l = 0..14;
   computed once, the level-15 filters having some 10^5 taps */
struct SynthesisEnergies
{
  double lo[15], hi[15];
  SynthesisEnergies()
  {
    std::vector<double> fl(kSyn97Lo, kSyn97Lo + 7), fh(kSyn97Hi, kSyn97Hi + 9);
    for(int l = 0; l < 15; ++l)
    {
      lo[l] = sum_squares(fl);
      hi[l] = sum_squares(fh);
      fl = coarser(fl);
      fh = coarser(fh);
    }
  }
};

/* the table of quality factor q: (exponent << 11 | mantissa) per band in QCD order */
static std::vector<uint32_t> derive_qfactor_words(int q, int prec, int D, int comp)
{
  /* m: the JPEG quality curve's scale; above the knee (65) the visual weights fade out, gone from the top (97) on */
  const double knee = 2.0 * (1.0 - 65 / 100.0), top = 2.0 * (1.0 - 97 / 100.0);
  const double m = q < 50 ? 50.0 / q : 2.0 * (1.0 - q / 100.0);
  double alpha = 0.04, wpow = 1.0;
  if(q >= 97)
  {
    wpow = 0.0;
    alpha = 0.10;
  }
  else if(q > 65)
  {
    wpow = (std::log(top) - std::log(m)) / (std::log(top) - std::log(knee));
    alpha = 0.10 * std::pow(0.04 / 0.10, wpow);
  }
  const double ref = (alpha * m + std::sqrt(0.5) * std::ldexp(1.0, -prec)) * kIctNorm[0];
  const double cgain = kIctNorm[comp < 3 ? comp : 0];
  const double* vis = comp == 0 ? kVisY : comp == 1 ? kVisCb : kVisCr;
  /* squared basis norms per band, finest level first (HH, LH, HL), then LL */
  static const SynthesisEnergies E;
  std::vector<double> norm2;
  for(int l = 0; l < D; ++l)
  {
    norm2.push_back(E.hi[l] * E.hi[l]);
    norm2.push_back(E.lo[l] * E.hi[l]);
    norm2.push_back(E.hi[l] * E.lo[l]);
  }
  norm2.push_back(D ? E.lo[D - 1] * E.lo[D - 1] : 1.0);
  const size_t nb = norm2.size();
  std::vector<uint32_t> words(nb);
  for(size_t k = 0; k < nb; ++k)
  {
    const double w = (k == nb - 1 || k >= 15) ? 1.0 : std::pow(vis[k], wpow);
    double step = ref / (std::sqrt(norm2[k]) * w * cgain);
    /* step = 2^-e (1 + mu / 2^11), T.800 E.1.1.1 */
    int e = 0;
    for(; step < 1.0; ++e)
      step *= 2.0;
    int mu = (int)std::floor((step - 1.0) * 2048.0 + 0.5);
    if(mu > 2047)
    {
      mu = 0;
      --e;
    }
    if(e > 31)
    {
      e = 31;
      mu = 0;
    }
    if(e < 0)
    {
      e = 0;
      mu = 2047;
    }
    words[nb - 1 - k] = ((uint32_t)e << 11) | (uint32_t)mu; /* QCD order: LL first, then HL, LH, HH from the coarsest */
  }
  return words;
}

/* derived once per (quality factor, precision, levels, component) and kept: the parser tries all 100 quality factors on
   every irreversible stream whose QCD is not Grok's default, and every band_quant of a quality-factor coding reads one */
const std::vector<uint32_t>& qfactor_words(int q, int prec, int numres, int comp)
{
  static std::mutex mu;
  static std::map<uint32_t, std::vector<uint32_t>> cache;
  const uint32_t key = (uint32_t)q | (uint32_t)prec << 8 | (uint32_t)(numres - 1) << 16 | (uint32_t)(comp < 3 ? comp : 0) << 24;
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find(key);
  if(it == cache.end())
    it = cache.emplace(key, derive_qfactor_words(q, prec, numres - 1, comp < 3 ? comp : 0)).first;
  return it->second; /* std::map nodes do not move: the reference stays valid */
}



std::vector<BandQuant> band_quant(const b2k_coding& cp, int comp)
{
  const int D = cp.numres - 1;
  std::vector<BandQuant> q(3 * D + 1);
  std::vector<uint8_t> expn(3 * D + 1);
  std::vector<uint16_t> mant(3 * D + 1, 0);
  int s = 0;
  if(!cp.irreversible)
  {
    const int B = cp.prec + (cp.mct ? 1 : 0);
    float bl = kBibo53L[D];
    int X = (int)std::ceil(std::log(bl * bl * 1.1f) / M_LN2);
    expn[s++] = (uint8_t)(B + X);
    for(int d = D - 1; d >= 0; --d)
    {
      bl = kBibo53L[d + 1];
      const float bh = kBibo53H[d];
      X = (int)std::ceil(std::log(bh * bl * 1.1f) / M_LN2);
      expn[s++] = (uint8_t)(B + X);
      expn[s++] = (uint8_t)(B + X);
      X = (int)std::ceil(std::log(bh * bh * 1.1f) / M_LN2);
      expn[s++] = (uint8_t)(B + X);
    }
  }
  else
  {
    const float base_delta = 1.0f / (float)(1 << (cp.prec + (cp.sgnd ? 1 : 0)));
    const float gl0 = kGain97L[D];
    irrev_expn_mant(base_delta / (gl0 * gl0), expn[s], mant[s]);
    s++;
    for(int d = D; d > 0; --d)
    {
      const float gl = kGain97L[d], gh = kGain97H[d - 1];
      irrev_expn_mant(base_delta / (gl * gh), expn[s], mant[s]);
      expn[s + 1] = expn[s];
      mant[s + 1] = mant[s];
      s += 2;
      irrev_expn_mant(base_delta / (gh * gh), expn[s], mant[s]);
      s++;
    }
  }
  const bool own = comp >= 0 && comp < 4 && ((cp.qcc_mask >> comp) & 1);
  if(cp.qfactor && cp.irreversible)
  {
    const std::vector<uint32_t>& w = qfactor_words(cp.qfactor, cp.prec, cp.numres, comp);
    for(int i = 0; i < 3 * D + 1; ++i)
    {
      expn[i] = (uint8_t)(w[i] >> 11);
      mant[i] = (uint16_t)(w[i] & 0x7FF);
    }
  }
  else if(own || cp.qcd_explicit)
    for(int i = 0; i < 3 * D + 1 && i < 97; ++i)
    { /* a foreign stream's QCD / QCC (or a caller's own choice) instead of the HT quantiser's tables */
      expn[i] = own ? cp.qcc_expn[comp][i] : cp.qcd_expn[i];
      mant[i] = cp.irreversible ? (uint16_t)((own ? cp.qcc_mant[comp][i] : cp.qcd_mant[i]) & 0x7FF) : 0;
    }
  for(int i = 0; i < 3 * D + 1; ++i)
  {
    const int orient = i == 0 ? 0 : ((i - 1) % 3) + 1;
    const int gain = orient == 0 ? 0 : (orient == 3 ? 2 : 1);
    BandQuant& b = q[i];
    b.expn = expn[i];
    b.mant = mant[i];
    const int k = (int)expn[i] + (int)cp.numgbits - 1;
    b.kmax = (uint8_t)(k > 0 ? k : 0);
    b.step_enc = (float)((1.0 + mant[i] / 2048.0) * std::pow(2.0, (double)((int)cp.prec + gain - (int)expn[i])));
    const int dgain = cp.irreversible ? 0 : gain;
    b.step_dec = (float)((1.0 + mant[i] / 2048.0) * std::pow(2.0, (double)((int)cp.prec + dgain - (int)expn[i])));
  }
  return q;
}

/* whether component c has a table of its own (its QCC's, or a quality factor's chroma table); the others share QCD's */
static bool own_table(const b2k_coding& cp, int c)
{
  return ((cp.qcc_mask >> c) & 1) || (c > 0 && cp.qfactor && cp.irreversible);
}

std::vector<std::vector<BandQuant>> component_quant(const b2k_coding& cp)
{
  std::vector<std::vector<BandQuant>> q;
  int shared = -1; /* the first component that takes QCD's table */
  for(int c = 0; c < cp.numcomps; ++c)
  {
    const bool own = own_table(cp, c);
    q.push_back(own || shared < 0 ? band_quant(cp, c) : q[shared]);
    if(!own && shared < 0)
      shared = c;
  }
  return q;
}

bool same_quant(const std::vector<BandQuant>& a, const std::vector<BandQuant>& b)
{
  if(a.size() != b.size())
    return false;
  for(size_t i = 0; i < a.size(); ++i)
    if(a[i].expn != b[i].expn || a[i].mant != b[i].mant)
      return false;
  return true;
}

const char* unsupported_reason(const b2k_coding& cp)
{
  if(cp.numcomps < 1 || cp.numcomps > 4)
    return "1..4 components supported";
  if(cp.numres < 1 || cp.numres > 16)
    return "1..16 resolutions supported";
  if(cp.prec < 1 || cp.prec > 16)
    return "precision 1..16 supported";
  if(cp.cblkw_exp < 2 || cp.cblkh_exp < 2 || cp.cblkw_exp > 10 || cp.cblkh_exp > 10 || cp.cblkw_exp + cp.cblkh_exp > 12)
    return "invalid code-block size";
  if(cp.mct && cp.numcomps < 3)
    return "MCT needs three components";
  if(cp.x1 <= cp.x0 || cp.y1 <= cp.y0)
    return "empty image";
  if(cp.qfactor > 100)
    return "quality factor 1..100 supported";
  if(cp.qfactor && !cp.irreversible)
    return "a quality factor needs the irreversible 9/7 transform";
  if(cp.qfactor && cp.numcomps != 1 && cp.numcomps != 3)
    return "a quality factor needs one or three components";
  if(cp.qcc_mask >> cp.numcomps)
    return "qcc_mask names a component the image does not have";
  bool shared_checked = false; /* the components without a table of their own share one */
  for(int c = 0; c < cp.numcomps; ++c)
  {
    if(!own_table(cp, c))
    {
      if(shared_checked)
        continue;
      shared_checked = true;
    }
    for(const BandQuant& b : band_quant(cp, c))
      if(b.kmax > 29 || b.kmax < 1)
      {
        if(cp.qfactor && b.kmax < 1)
        { /* the reference's T2 refuses such a band too ("exceeding band maximum"): its HT coder signals one bit plane */
          static thread_local char why[160];
          snprintf(why, sizeof why, "quality factor %u with %u guard bit(s) leaves a band without bit planes (Kmax 0): "
                   "use more guard bits or a higher quality factor", (unsigned)cp.qfactor, (unsigned)cp.numgbits);
          return why;
        }
        return "band bit planes outside the 32-bit HT coder's range";
      }
  }
  return nullptr;
}

void enumerate_tile_blocks(const b2k_coding& cp, uint32_t tile_index, const Rect& tile,
                           const std::vector<BandQuant>& quant, std::vector<b2k_block>& out)
{
  enumerate_tile_blocks(cp, tile_index, tile, std::vector<std::vector<BandQuant>>(cp.numcomps, quant), out);
}

void enumerate_tile_blocks(const b2k_coding& cp, uint32_t tile_index, const Rect& tile,
                           const std::vector<std::vector<BandQuant>>& quant, std::vector<b2k_block>& out)
{
  walk_precincts(cp, tile, [&](const PrecinctBand& pb) {
    const BandQuant& bq = quant[pb.comp][band_quant_index(pb.resno, pb.orient)];
    /* in the resolution's buffer the high-pass bands follow the lower resolution's samples */
    const Rect lower = resolution_rect(tile, cp.numres, pb.resno ? pb.resno - 1 : 0);
    const uint32_t bx = (pb.orient & 1) ? lower.w() : 0, by = (pb.orient & 2) ? lower.h() : 0;
    const Rect& prc = pb.rect;
    for(uint32_t k = 0; k < pb.gw * pb.gh; ++k)
    {
      b2k_block blk{};
      blk.tile = tile_index;
      blk.comp = pb.comp;
      blk.resno = pb.resno;
      blk.band_index = pb.band_index;
      blk.orient = pb.orient;
      blk.kmax = bq.kmax;
      blk.precno = pb.precno;
      blk.cblkno = k;
      blk.x0 = std::max((pb.gx + k % pb.gw) << pb.cbw, prc.x0);
      blk.y0 = std::max((pb.gy + k / pb.gw) << pb.cbh, prc.y0);
      blk.x1 = (uint32_t)std::min<uint64_t>(((uint64_t)(pb.gx + k % pb.gw) + 1) << pb.cbw, prc.x1);
      blk.y1 = (uint32_t)std::min<uint64_t>(((uint64_t)(pb.gy + k / pb.gw) + 1) << pb.cbh, prc.y1);
      blk.buf_x = blk.x0 - pb.band.x0 + bx;
      blk.buf_y = blk.y0 - pb.band.y0 + by;
      blk.length = 0;
      blk.offset = 0;
      blk.numbps = 0;
      blk.numpasses = 0;
      blk.stepsize = bq.step_enc;
      out.push_back(blk);
    }
  });
}

} // namespace b2k
