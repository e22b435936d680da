/*
 * oracle/j2k_oracle.c -- TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C, scalar, deliberately slow restatement of the JPEG 2000 tile-engine hot path of
 * GrokImageCompression/Grok (reference tree /root/reference, commit dfb9ad42).  It exists so
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg can CHECK the CUDA engine;
 * nothing in grok_b200/ may include, link or call it.
 *
 * Every function cites the reference file:line it restates.  Pinning status (see DESIGN.md):
 *   - HT cleanup encoder / decoder : byte-for-byte vs the reference's own OpenJPH sources
 *     compiled into oracle/_ref (tests/test_oracle.py), fixtures in tests/golden/.
 *   - HT SigProp / MagRef          : word-for-word vs the same decoders with 2 / 3 passes
 *     (tests/golden/ht_refine.npz), and decoded identically by OpenJPEG (tests/test_codestream.py).
 *   - forward 5/3 and 9/7 lifting  : vs grk::dwt53 / grk::dwt97 compiled from
 *     wavelet/WaveletFwd.cpp into oracle/_ref, fixtures in tests/golden/.
 *   - inverse 5/3                  : exact inverse of the pinned forward (perfect reconstruction).
 *   - RCT / ICT, inverse 9/7, quantiser tables, geometry: restatement of the cited lines (the
 *     reference classes need the whole Tile object graph, so there is no per-function pin against
 *     Grok).  They are pinned END TO END against an independent JPEG 2000 implementation instead:
 *     codestreams assembled from this oracle's blocks are decoded by OpenJPEG 2.5 (Pillow's and
 *     OpenCV's builds) exactly to the source on the reversible path -- which fixes RCT, DC shift,
 *     5/3, geometry, precinct / code-block partition, exponents and Kmax -- and to within one code of
 *     this oracle's own decode on the 9/7 + ICT path with default and with explicit step sizes --
 *     which fixes ICT, inverse 9/7 and the step-size formula (tests/test_codestream.py).
 */
#include <stdint.h>
#include <stddef.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

#include "t814_vlc_rows.h"

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------ */
/* small helpers                                                                               */
/* ------------------------------------------------------------------------------------------ */
static inline uint32_t ceildivpow2_u32(uint32_t a, uint32_t b)
{
  return (uint32_t)(((uint64_t)a + ((1ULL << b) - 1)) >> b);
}
static inline uint32_t floordivpow2_u32(uint32_t a, uint32_t b) { return a >> b; }
static inline int imax(int a, int b) { return a > b ? a : b; }
static inline int imin(int a, int b) { return a < b ? a : b; }

/* whole-sample symmetric extension index: periodic reflection about 0 and n-1 */
static inline int mirror_idx(int i, int n)
{
  if(n == 1)
    return 0;
  int period = 2 * (n - 1);
  i %= period;
  if(i < 0)
    i += period;
  return i < n ? i : period - i;
}

/* ------------------------------------------------------------------------------------------ */
/* MCT: point_transform/mct.cpp                                                                */
/* ------------------------------------------------------------------------------------------ */

/* CompressRev::transform, mct.cpp L497-531: add (negative) DC shift, then RCT, in place. */
ORC_API void orc_rct_fwd(int32_t* c0, int32_t* c1, int32_t* c2, size_t n, const int32_t shift[3])
{
  for(size_t i = 0; i < n; ++i)
  {
    int32_t r = c0[i] + shift[0], g = c1[i] + shift[1], b = c2[i] + shift[2];
    c0[i] = ((g + g) + b + r) >> 2;
    c1[i] = b - g;
    c2[i] = r - g;
  }
}

/* DecompressRev::transform, mct.cpp L201-256: inverse RCT, +shift, clamp. */
ORC_API void orc_rct_inv(int32_t* c0, int32_t* c1, int32_t* c2, size_t n, const int32_t shift[3],
                         const int32_t lo[3], const int32_t hi[3])
{
  for(size_t i = 0; i < n; ++i)
  {
    int32_t y = c0[i], u = c1[i], v = c2[i];
    int32_t g = y - ((u + v) >> 2);
    int32_t r = v + g, b = u + g;
    r += shift[0];
    g += shift[1];
    b += shift[2];
    c0[i] = r < lo[0] ? lo[0] : (r > hi[0] ? hi[0] : r);
    c1[i] = g < lo[1] ? lo[1] : (g > hi[1] ? hi[1] : g);
    c2[i] = b < lo[2] ? lo[2] : (b > hi[2] ? hi[2] : b);
  }
}

/* CompressIrrev::transform, mct.cpp L584-636: integer DC shift, ICT in fp32, float bits out. */
ORC_API void orc_ict_fwd(const int32_t* r_in, const int32_t* g_in, const int32_t* b_in, float* y_out,
                         float* cb_out, float* cr_out, size_t n, const int32_t shift[3])
{
  const float a_r = 0.299f, a_g = 0.587f, a_b = 0.114f;
  const float cb = 0.5f / (1.0f - a_b), cr = 0.5f / (1.0f - a_r);
  for(size_t i = 0; i < n; ++i)
  {
    float r = (float)(r_in[i] + shift[0]), g = (float)(g_in[i] + shift[1]),
          b = (float)(b_in[i] + shift[2]);
    /* libgrokj2k (gcc, Highway AVX2/AVX-512 targets) contracts this into fma(a_b,b, fma(a_g,g, a_r*r)); pinned against
       the real library's code-block bytes by tests/test_interop.py */
    float y = fmaf(a_b, b, fmaf(a_g, g, a_r * r));
    y_out[i] = y;
    cb_out[i] = cb * (b - y);
    cr_out[i] = cr * (r - y);
  }
}

/* DecompressIrrev::transform, mct.cpp L318-391: inverse ICT, NearestInt, +shift, clamp. */
ORC_API void orc_ict_inv(const float* y_in, const float* cb_in, const float* cr_in, int32_t* r_out,
                         int32_t* g_out, int32_t* b_out, size_t n, const int32_t shift[3],
                         const int32_t lo[3], const int32_t hi[3])
{
  for(size_t i = 0; i < n; ++i)
  {
    float y = y_in[i], u = cb_in[i], v = cr_in[i];
    /* as libgrokj2k's build contracts them (FMA / FNMA); pinned against the real library's decoded pixels by
       tests/test_interop.py */
    float fr = fmaf(v, 1.402f, y);
    float fg = fmaf(-v, 0.71414f, fmaf(-u, 0.34413f, y));
    float fb = fmaf(u, 1.772f, y);
    int32_t r = (int32_t)lrintf(fr) + shift[0];
    int32_t g = (int32_t)lrintf(fg) + shift[1];
    int32_t b = (int32_t)lrintf(fb) + shift[2];
    r_out[i] = r < lo[0] ? lo[0] : (r > hi[0] ? hi[0] : r);
    g_out[i] = g < lo[1] ? lo[1] : (g > hi[1] ? hi[1] : g);
    b_out[i] = b < lo[2] ? lo[2] : (b > hi[2] ? hi[2] : b);
  }
}

/* ------------------------------------------------------------------------------------------ */
/* 1-D lifting on an interleaved line a[0..n), sample i sits at canvas position i+parity, so   */
/* (i+parity) even = low-pass.  wavelet/WaveletFwd.cpp L139-439 (5/3), L441-876 (9/7);         */
/* wavelet/WaveletReverse.cpp L879-1397, WaveletReverse97.cpp L98-103, L837-857.               */
/* ------------------------------------------------------------------------------------------ */
#define AT(a, i, n) ((a)[mirror_idx((i), (n))])

static void fwd53_line(int32_t* a, int n, int parity)
{
  if(n == 1)
  {
    if(parity)
      a[0] = (int32_t)((uint32_t)a[0] << 1); /* WaveletFwd.cpp L146-156 */
    return;
  }
  /* predict: odd canvas positions */
  for(int i = !parity; i < n; i += 2)
    a[i] = (int32_t)((uint32_t)a[i] - (uint32_t)((AT(a, i - 1, n) + AT(a, i + 1, n)) >> 1));
  /* update: even canvas positions */
  for(int i = parity; i < n; i += 2)
    a[i] = (int32_t)((uint32_t)a[i] + (uint32_t)((AT(a, i - 1, n) + AT(a, i + 1, n) + 2) >> 2));
}

static void inv53_line(int32_t* a, int n, int parity)
{
  if(n == 1)
  {
    if(parity)
      a[0] = a[0] >> 1; /* WaveletReverse.cpp: lone odd sample is halved */
    return;
  }
  for(int i = parity; i < n; i += 2)
    a[i] = (int32_t)((uint32_t)a[i] - (uint32_t)((int32_t)((uint32_t)AT(a, i - 1, n) + (uint32_t)AT(a, i + 1, n) + 2u) >> 2));
  for(int i = !parity; i < n; i += 2)
    a[i] = (int32_t)((uint32_t)a[i] + (uint32_t)((int32_t)((uint32_t)AT(a, i - 1, n) + (uint32_t)AT(a, i + 1, n)) >> 1));
}

static const float F97_ALPHA = -1.586134342f, F97_BETA = -0.052980118f, F97_GAMMA = 0.882911075f,
                   F97_DELTA = 0.443506852f, F97_K = 1.230174105f;

/* The reference build (g++ -O3, Highway AVX2/AVX-512 targets) contracts `cur + (l + r) * c`
 * into one fused multiply-add; the trailing `* K` stays a separate multiply.  fmaf() states that
 * explicitly, which makes this restatement bit-identical to grk::dwt97 as built in oracle/_ref
 * (pinned by tests/test_oracle_pinning.py). */
static void fwd97_line(float* a, int n, int parity)
{
  if(n == 1)
  {
    if(parity)
      a[0] *= 2.0f; /* WaveletFwd.cpp L444-455 */
    return;
  }
  const float invK = (float)(1.0 / 1.230174105);
  const float delta_s = F97_DELTA * invK; /* WaveletFwd.cpp L565 */
  for(int i = !parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), F97_ALPHA, a[i]);
  for(int i = parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), F97_BETA, a[i]);
  for(int i = !parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), F97_GAMMA, a[i]) * F97_K;
  for(int i = parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), delta_s, a[i]) * invK;
}

static void inv97_line(float* a, int n, int parity)
{
  /* WaveletReverse97.cpp L837-857 (step_97) with constants L98-103; same contraction assumed
   * (this direction is not compiled into oracle/_ref: tolerance-tested, see DESIGN.md) */
  if(n == 1)
    return;
  const float K = 1.230174105f, twice_invK = 1.625732422f;
  for(int i = parity; i < n; i += 2)
    a[i] *= K;
  for(int i = !parity; i < n; i += 2)
    a[i] *= twice_invK;
  for(int i = parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), -0.443506852f, a[i]);
  for(int i = !parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), -0.882911075f, a[i]);
  for(int i = parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), 0.052980118f, a[i]);
  for(int i = !parity; i < n; i += 2)
    a[i] = fmaf(AT(a, i - 1, n) + AT(a, i + 1, n), 1.586134342f, a[i]);
}

/* exported 1-D entry points (used by the pinning tests against oracle/_ref) */
ORC_API void orc_fwd53_line(int32_t* a, int n, int parity) { fwd53_line(a, n, parity); }
ORC_API void orc_inv53_line(int32_t* a, int n, int parity) { inv53_line(a, n, parity); }
ORC_API void orc_fwd97_line(float* a, int n, int parity) { fwd97_line(a, n, parity); }
ORC_API void orc_inv97_line(float* a, int n, int parity) { inv97_line(a, n, parity); }

/* ------------------------------------------------------------------------------------------ */
/* 2-D multi-level transform, Mallat layout in place.                                          */
/* encode<T,DWT>, WaveletFwd.cpp L1337-1514: per level (finest first) all columns, then all    */
/* rows, on the top-left rw x rh of the buffer; parity = res.x0&1 / res.y0&1 (L1406-1407);     */
/* low band to [0,sn), high band to [sn,n) (deinterleave_v/h L77-137).                          */
/* tile_53/tile_97 (WaveletReverse.cpp L1347-1397): per resolution horizontal then vertical.   */
/* tc = tile-component rect in canvas coordinates.                                             */
/* ------------------------------------------------------------------------------------------ */
typedef struct
{
  uint32_t x0, y0, x1, y1;
} orc_rect;

static orc_rect res_rect(orc_rect tc, int numres, int resno)
{
  int n = numres - 1 - resno;
  orc_rect r = {ceildivpow2_u32(tc.x0, n), ceildivpow2_u32(tc.y0, n), ceildivpow2_u32(tc.x1, n),
                ceildivpow2_u32(tc.y1, n)};
  return r;
}

#define DEFINE_DWT2D(NAME, T, FWD, INV)                                                           \
  ORC_API void orc_##NAME##_fwd_2d(T* buf, uint32_t stride, uint32_t x0, uint32_t y0, uint32_t x1, \
                                   uint32_t y1, int numres)                                        \
  {                                                                                                \
    orc_rect tc = {x0, y0, x1, y1};                                                                \
    uint32_t maxdim = (x1 - x0) > (y1 - y0) ? (x1 - x0) : (y1 - y0);                               \
    T* line = (T*)malloc(sizeof(T) * (maxdim + 1));                                                \
    T* tmp = (T*)malloc(sizeof(T) * (maxdim + 1));                                                 \
    for(int resno = numres - 1; resno >= 1; --resno)                                               \
    {                                                                                              \
      orc_rect r = res_rect(tc, numres, resno), lo = res_rect(tc, numres, resno - 1);              \
      int rw = (int)(r.x1 - r.x0), rh = (int)(r.y1 - r.y0);                                        \
      int snx = (int)(lo.x1 - lo.x0), sny = (int)(lo.y1 - lo.y0);                                  \
      int px = r.x0 & 1, py = r.y0 & 1;                                                            \
      for(int x = 0; x < rw && rh > 0; ++x)                                                        \
      {                                                                                            \
        for(int y = 0; y < rh; ++y)                                                                \
          line[y] = buf[(size_t)y * stride + x];                                                   \
        FWD(line, rh, py);                                                                         \
        for(int y = 0; y < rh; ++y)                                                                \
        {                                                                                          \
          int low = ((y + py) & 1) == 0;                                                           \
          int k = (y + py) >> 1;                                                                   \
          int dst = low ? (k - py) : (sny + k);                                                    \
          buf[(size_t)dst * stride + x] = line[y];                                                 \
        }                                                                                          \
      }                                                                                            \
      for(int y = 0; y < rh && rw > 0; ++y)                                                        \
      {                                                                                            \
        T* row = buf + (size_t)y * stride;                                                         \
        memcpy(line, row, sizeof(T) * rw);                                                         \
        FWD(line, rw, px);                                                                         \
        for(int x = 0; x < rw; ++x)                                                                \
        {                                                                                          \
          int low = ((x + px) & 1) == 0;                                                           \
          int k = (x + px) >> 1;                                                                   \
          int dst = low ? (k - px) : (snx + k);                                                    \
          row[dst] = line[x];                                                                      \
        }                                                                                          \
      }                                                                                            \
    }                                                                                              \
    free(line);                                                                                    \
    free(tmp);                                                                                     \
  }                                                                                                \
  ORC_API void orc_##NAME##_inv_2d(T* buf, uint32_t stride, uint32_t x0, uint32_t y0, uint32_t x1, \
                                   uint32_t y1, int numres)                                        \
  {                                                                                                \
    orc_rect tc = {x0, y0, x1, y1};                                                                \
    uint32_t maxdim = (x1 - x0) > (y1 - y0) ? (x1 - x0) : (y1 - y0);                               \
    T* line = (T*)malloc(sizeof(T) * (maxdim + 1));                                                \
    for(int resno = 1; resno < numres; ++resno)                                                    \
    {                                                                                              \
      orc_rect r = res_rect(tc, numres, resno), lo = res_rect(tc, numres, resno - 1);              \
      int rw = (int)(r.x1 - r.x0), rh = (int)(r.y1 - r.y0);                                        \
      int snx = (int)(lo.x1 - lo.x0), sny = (int)(lo.y1 - lo.y0);                                  \
      int px = r.x0 & 1, py = r.y0 & 1;                                                            \
      for(int y = 0; y < rh && rw > 0; ++y)                                                        \
      {                                                                                            \
        T* row = buf + (size_t)y * stride;                                                         \
        for(int x = 0; x < rw; ++x)                                                                \
        {                                                                                          \
          int low = ((x + px) & 1) == 0;                                                           \
          int k = (x + px) >> 1;                                                                   \
          line[x] = row[low ? (k - px) : (snx + k)];                                               \
        }                                                                                          \
        INV(line, rw, px);                                                                         \
        memcpy(row, line, sizeof(T) * rw);                                                         \
      }                                                                                            \
      for(int x = 0; x < rw && rh > 0; ++x)                                                        \
      {                                                                                            \
        for(int y = 0; y < rh; ++y)                                                                \
        {                                                                                          \
          int low = ((y + py) & 1) == 0;                                                           \
          int k = (y + py) >> 1;                                                                   \
          line[y] = buf[(size_t)(low ? (k - py) : (sny + k)) * stride + x];                        \
        }                                                                                          \
        INV(line, rh, py);                                                                         \
        for(int y = 0; y < rh; ++y)                                                                \
          buf[(size_t)y * stride + x] = line[y];                                                   \
      }                                                                                            \
    }                                                                                              \
    free(line);                                                                                    \
  }

DEFINE_DWT2D(dwt53, int32_t, fwd53_line, inv53_line)
DEFINE_DWT2D(dwt97, float, fwd97_line, inv97_line)

/* ------------------------------------------------------------------------------------------ */
/* Quantiser tables: t2/quantizer/part15/QuantizerOJPH.cpp L150-259, pulled by                 */
/* t2/quantizer/part1/Quantizer.cpp L47-64; band step / Kmax: TileProcessor.cpp L398-419.      */
/* ------------------------------------------------------------------------------------------ */
/* the reference's tables in full (34 entries; emitted by tools/gen_gain_tables.py from QuantizerOJPH.cpp L103-185) */
static const float bibo_5x3_l[34] = {
    1.0000e+00f, 1.5000e+00f, 1.6250e+00f, 1.6875e+00f, 1.6963e+00f, 1.7067e+00f, 1.7116e+00f,
    1.7129e+00f, 1.7141e+00f, 1.7145e+00f, 1.7151e+00f, 1.7152e+00f, 1.7155e+00f, 1.7155e+00f,
    1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f,
    1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f,
    1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f, 1.7156e+00f
};
static const float bibo_5x3_h[34] = {
    2.0000e+00f, 2.5000e+00f, 2.7500e+00f, 2.8047e+00f, 2.8198e+00f, 2.8410e+00f, 2.8558e+00f,
    2.8601e+00f, 2.8628e+00f, 2.8656e+00f, 2.8662e+00f, 2.8667e+00f, 2.8669e+00f, 2.8670e+00f,
    2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f,
    2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f,
    2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f, 2.8671e+00f
};
static const float sqe_9x7_l[34] = {
    1.0000e+00f, 1.4021e+00f, 2.0304e+00f, 2.9012e+00f, 4.1153e+00f, 5.8245e+00f, 8.2388e+00f,
    1.1652e+01f, 1.6479e+01f, 2.3304e+01f, 3.2957e+01f, 4.6609e+01f, 6.5915e+01f, 9.3217e+01f,
    1.3183e+02f, 1.8643e+02f, 2.6366e+02f, 3.7287e+02f, 5.2732e+02f, 7.4574e+02f, 1.0546e+03f,
    1.4915e+03f, 2.1093e+03f, 2.9830e+03f, 4.2185e+03f, 5.9659e+03f, 8.4371e+03f, 1.1932e+04f,
    1.6874e+04f, 2.3864e+04f, 3.3748e+04f, 4.7727e+04f, 6.7496e+04f, 9.5454e+04f
};
static const float sqe_9x7_h[34] = {
    1.4425e+00f, 1.9669e+00f, 2.8839e+00f, 4.1475e+00f, 5.8946e+00f, 8.3472e+00f, 1.1809e+01f,
    1.6701e+01f, 2.3620e+01f, 3.3403e+01f, 4.7240e+01f, 6.6807e+01f, 9.4479e+01f, 1.3361e+02f,
    1.8896e+02f, 2.6723e+02f, 3.7792e+02f, 5.3446e+02f, 7.5583e+02f, 1.0689e+03f, 1.5117e+03f,
    2.1378e+03f, 3.0233e+03f, 4.2756e+03f, 6.0467e+03f, 8.5513e+03f, 1.2093e+04f, 1.7103e+04f,
    2.4187e+04f, 3.4205e+04f, 4.8373e+04f, 6.8410e+04f, 9.6747e+04f, 1.3682e+05f
};

/* expn[3*decomps+1], mant[...]; band order LL, then per level coarsest->finest HL,LH,HH.
 * decomps <= 32 (the tables' extent). */
ORC_API int orc_ht_stepsizes(int decomps, int prec, int mct, int sgnd, int reversible,
                             uint8_t* expn, uint16_t* mant)
{
  if(decomps > 32)
    return -1;
  int s = 0;
  if(reversible)
  { /* set_rev_quant L193-212 */
    int B = prec + (mct ? 1 : 0);
    float bl = bibo_5x3_l[decomps];
    int X = (int)ceil(log(bl * bl * 1.1f) / M_LN2);
    expn[s] = (uint8_t)(B + X);
    mant[s++] = 0;
    for(int d = decomps - 1; d >= 0; --d)
    {
      bl = bibo_5x3_l[d + 1];
      float bh = bibo_5x3_h[d];
      X = (int)ceil(log(bh * bl * 1.1f) / M_LN2);
      expn[s] = (uint8_t)(B + X);
      mant[s++] = 0;
      expn[s] = (uint8_t)(B + X);
      mant[s++] = 0;
      X = (int)ceil(log(bh * bh * 1.1f) / M_LN2);
      expn[s] = (uint8_t)(B + X);
      mant[s++] = 0;
    }
  }
  else
  { /* set_irrev_quant L213-259; base_delta L186-187 */
    float base_delta = 1.0f / (float)(1 << (prec + sgnd));
    float gl = sqe_9x7_l[decomps];
    float delta_b = base_delta / (gl * gl);
    int e = 0;
    while(delta_b < 1.0f)
    {
      e++;
      delta_b *= 2.0f;
    }
    int m = (int)round(delta_b * (float)(1 << 11)) - (1 << 11);
    m = m < (1 << 11) ? m : 0x7FF;
    expn[s] = (uint8_t)e;
    mant[s++] = (uint16_t)m;
    for(int d = decomps; d > 0; --d)
    {
      float g_l = sqe_9x7_l[d], g_h = sqe_9x7_h[d - 1];
      delta_b = base_delta / (g_l * g_h);
      e = 0;
      while(delta_b < 1.0f)
      {
        e++;
        delta_b *= 2.0f;
      }
      m = (int)round(delta_b * (float)(1 << 11)) - (1 << 11);
      m = m < (1 << 11) ? m : 0x7FF;
      expn[s] = (uint8_t)e;
      mant[s++] = (uint16_t)m;
      expn[s] = (uint8_t)e;
      mant[s++] = (uint16_t)m;
      delta_b = base_delta / (g_h * g_h);
      e = 0;
      while(delta_b < 1)
      {
        e++;
        delta_b *= 2.0f;
      }
      m = (int)round(delta_b * (float)(1 << 11)) - (1 << 11);
      m = m < (1 << 11) ? m : 0x7FF;
      expn[s] = (uint8_t)e;
      mant[s++] = (uint16_t)m;
    }
  }
  return s;
}

/* TileProcessor.cpp L398-419.  orient 0..3 = LL,HL,LH,HH. */
ORC_API float orc_band_stepsize(int prec, int orient, int expn, int mant, int is_compressor,
                                int reversible)
{
  int log2_gain = (!is_compressor && !reversible) ? 0 : (orient == 0) ? 0 : (orient == 3) ? 2 : 1;
  int numbps = prec + log2_gain;
  return (float)((1.0 + mant / 2048.0) * pow(2.0, (double)(numbps - expn)));
}
ORC_API int orc_band_kmax(int expn, int numgbits, int roishift)
{
  int v = expn + numgbits - 1;
  return roishift + (v > 0 ? v : 0);
}

/* ------------------------------------------------------------------------------------------ */
/* Geometry: TileProcessor.cpp L329-351, ResSimple.h L81-109, Resolution.cpp L69-160,          */
/* Subband.cpp L66-78, PrecinctImpl.cpp L45-66, TileComponentWindow.h L241-264,                */
/* CompressScheduler.cpp L84-139 (enumeration order comp->res->band->precinct->cblk).          */
/* ------------------------------------------------------------------------------------------ */
typedef struct
{
  uint8_t resno, orient, band_index;
  uint32_t precno, cblkno;  /* precinct index in the resolution grid, block raster index in it */
  uint32_t x0, y0, x1, y1;  /* band (canvas) coordinates */
  uint32_t buf_x, buf_y;    /* position in the Mallat tile-component buffer */
} orc_block;

static uint32_t band_coord(uint32_t c, int ndecomp, uint32_t high)
{
  if(ndecomp == 0)
    return c;
  uint32_t off = (1u << (ndecomp - 1)) * high;
  return c <= off ? 0 : ceildivpow2_u32(c - off, (uint32_t)ndecomp);
}

/* Enumerate every code block (including zero-area ones, flagged by x0==x1||y0==y1) of one
 * tile component.  Returns the count; writes at most cap entries. */
ORC_API int orc_enumerate_blocks(uint32_t tcx0, uint32_t tcy0, uint32_t tcx1, uint32_t tcy1,
                                 int numres, int cblkw_exp, int cblkh_exp, const uint8_t* prcw_exp,
                                 const uint8_t* prch_exp, orc_block* out, int cap)
{
  orc_rect tc = {tcx0, tcy0, tcx1, tcy1};
  int count = 0;
  for(int resno = 0; resno < numres; ++resno)
  {
    orc_rect res = res_rect(tc, numres, resno);
    int pw = prcw_exp ? prcw_exp[resno] : 15, ph = prch_exp ? prch_exp[resno] : 15;
    /* precinct partition of the resolution (Resolution.cpp L119-160) */
    uint32_t px0 = floordivpow2_u32(res.x0, pw) << pw, py0 = floordivpow2_u32(res.y0, ph) << ph;
    uint32_t px1 = ceildivpow2_u32(res.x1, pw) << pw, py1 = ceildivpow2_u32(res.y1, ph) << ph;
    uint32_t gridw = (res.x1 > res.x0) ? ((px1 - px0) >> pw) : 0;
    uint32_t gridh = (res.y1 > res.y0) ? ((py1 - py0) >> ph) : 0;
    /* TileProcessor.cpp: precinctGrid_ = partition.scaleDownPow2 */
    gridw = (ceildivpow2_u32(px1, pw)) - (px0 >> pw);
    gridh = (ceildivpow2_u32(py1, ph)) - (py0 >> ph);
    int nbands = resno == 0 ? 1 : 3;
    int level = resno == 0 ? numres - 1 : numres - resno;
    orc_rect lower = resno ? res_rect(tc, numres, resno - 1) : res;
    /* band precinct partition: halve for resno>0 (Resolution.cpp L78-93) */
    int bpw = resno ? pw - 1 : pw, bph = resno ? ph - 1 : ph;
    uint32_t bpx0 = resno ? (px0 >> 1) : px0, bpy0 = resno ? (py0 >> 1) : py0;
    int cbw = imin(cblkw_exp, bpw), cbh = imin(cblkh_exp, bph);
    for(int b = 0; b < nbands; ++b)
    {
      int orient = resno == 0 ? 0 : b + 1;
      orc_rect band = {band_coord(tc.x0, level, orient & 1), band_coord(tc.y0, level, orient >> 1),
                       band_coord(tc.x1, level, orient & 1), band_coord(tc.y1, level, orient >> 1)};
      for(uint32_t p = 0; p < gridw * gridh; ++p)
      {
        /* Subband.cpp L66-78 */
        uint32_t qx0 = bpx0 + ((p % gridw) << bpw), qy0 = bpy0 + ((p / gridw) << bph);
        uint32_t qx1 = qx0 + (1u << bpw), qy1 = qy0 + (1u << bph);
        if(qx0 < band.x0) qx0 = band.x0;
        if(qy0 < band.y0) qy0 = band.y0;
        if(qx1 > band.x1) qx1 = band.x1;
        if(qy1 > band.y1) qy1 = band.y1;
        if(qx1 < qx0) qx1 = qx0;
        if(qy1 < qy0) qy1 = qy0;
        /* PrecinctImpl.cpp L45-66 */
        uint32_t gx = floordivpow2_u32(qx0, cbw), gy = floordivpow2_u32(qy0, cbh);
        uint32_t gw = ceildivpow2_u32(qx1, cbw) - gx, gh = ceildivpow2_u32(qy1, cbh) - gy;
        if(qx1 == qx0 || qy1 == qy0)
          gw = gh = 0;
        for(uint32_t k = 0; k < gw * gh; ++k)
        {
          uint32_t cx0 = (gx + k % gw) << cbw, cy0 = (gy + k / gw) << cbh;
          uint32_t cx1 = cx0 + (1u << cbw), cy1 = cy0 + (1u << cbh);
          if(cx0 < qx0) cx0 = qx0;
          if(cy0 < qy0) cy0 = qy0;
          if(cx1 > qx1) cx1 = qx1;
          if(cy1 > qy1) cy1 = qy1;
          if(count < cap)
          {
            orc_block* o = out + count;
            o->resno = (uint8_t)resno;
            o->orient = (uint8_t)orient;
            o->band_index = (uint8_t)b;
            o->precno = p;
            o->cblkno = k;
            o->x0 = cx0; o->y0 = cy0; o->x1 = cx1; o->y1 = cy1;
            /* TileComponentWindow.h L241-264 */
            o->buf_x = cx0 - band.x0 + ((resno && (orient & 1)) ? (lower.x1 - lower.x0) : 0);
            o->buf_y = cy0 - band.y0 + ((resno && (orient & 2)) ? (lower.y1 - lower.y0) : 0);
          }
          ++count;
        }
      }
    }
  }
  return count;
}

/* ------------------------------------------------------------------------------------------ */
/* T1 pre/post: CoderOJPH.cpp L121-185 (preCompress), PostDecodeFiltersOJPH.h L48-66,L100-119  */
/* ------------------------------------------------------------------------------------------ */
ORC_API void orc_ht_pre_rev(const int32_t* tile, uint32_t tstride, uint32_t w, uint32_t h,
                            uint32_t k_msbs, uint32_t* out)
{
  int shift = 31 - (int)(k_msbs + 1);
  for(uint32_t y = 0; y < h; ++y)
    for(uint32_t x = 0; x < w; ++x)
    {
      int32_t v = tile[(size_t)y * tstride + x];
      uint32_t mag = v >= 0 ? (uint32_t)v : (uint32_t)0 - (uint32_t)v;
      out[y * w + x] = (v >= 0 ? 0u : 0x80000000u) | (mag << shift);
    }
}
ORC_API void orc_ht_pre_irrev(const float* tile, uint32_t tstride, uint32_t w, uint32_t h,
                              uint32_t k_msbs, float inv_step, uint32_t* out)
{
  int shift = 31 - (int)(k_msbs + 1);
  for(uint32_t y = 0; y < h; ++y)
    for(uint32_t x = 0; x < w; ++x)
    {
      int32_t t = (int32_t)(tile[(size_t)y * tstride + x] * inv_step * (float)(1 << shift));
      uint32_t mag = t >= 0 ? (uint32_t)t : (uint32_t)0 - (uint32_t)t;
      out[y * w + x] = (t >= 0 ? 0u : 0x80000000u) | mag;
    }
}
ORC_API void orc_ht_post_rev(const uint32_t* dec, uint32_t dstride, uint32_t w, uint32_t h,
                             uint32_t kmax, int32_t* tile, uint32_t tstride)
{
  uint32_t shift = 31u - kmax;
  for(uint32_t y = 0; y < h; ++y)
    for(uint32_t x = 0; x < w; ++x)
    {
      uint32_t v = dec[y * dstride + x];
      int32_t m = (int32_t)((v & 0x7FFFFFFFu) >> shift);
      tile[(size_t)y * tstride + x] = (v & 0x80000000u) ? -m : m;
    }
}
ORC_API void orc_ht_post_irrev(const uint32_t* dec, uint32_t dstride, uint32_t w, uint32_t h,
                               uint32_t kmax, float stepsize, float* tile, uint32_t tstride)
{
  float scale = stepsize / (float)(1u << (31 - kmax));
  for(uint32_t y = 0; y < h; ++y)
    for(uint32_t x = 0; x < w; ++x)
    {
      uint32_t v = dec[y * dstride + x];
      float f = (float)(int32_t)(v & 0x7FFFFFFFu) * scale;
      tile[(size_t)y * tstride + x] = (v & 0x80000000u) ? -f : f;
    }
}

/* ------------------------------------------------------------------------------------------ */
/* HT block coder tables, derived from the T.814 rows at first use                             */
/* (ojph_block_encoder.cpp L76-256, ojph_block_common.cpp L118-178)                            */
/* ------------------------------------------------------------------------------------------ */
static uint16_t enc_vlc[2][2048];
static uint16_t dec_vlc[2][1024]; /* rho | e_k<<4 | e_1<<8 | u_off<<12 | len<<13 */
static int tables_ready = 0;

static void unpack_row(uint32_t p, int* c_q, int* rho, int* u_off, int* e_k, int* e_1, int* cwd,
                       int* len)
{
  *c_q = p & 7; *rho = (p >> 3) & 0xF; *u_off = (p >> 7) & 1; *e_k = (p >> 8) & 0xF;
  *e_1 = (p >> 12) & 0xF; *cwd = (p >> 16) & 0x7F; *len = (p >> 23) & 7;
}

static void build_tables(void)
{
  if(tables_ready)
    return;
  const uint32_t* src[2] = {T814_VLC_ROWS0, T814_VLC_ROWS1};
  const size_t nsrc[2] = {sizeof(T814_VLC_ROWS0) / 4, sizeof(T814_VLC_ROWS1) / 4};
  for(int t = 0; t < 2; ++t)
  {
    for(int i = 0; i < 2048; ++i)
    {
      int cq = i >> 8, rho = (i >> 4) & 0xF, emb = i & 0xF;
      enc_vlc[t][i] = 0;
      if((emb & rho) != emb || (rho == 0 && cq == 0))
        continue;
      int best = -1, best_pop = -1;
      for(size_t j = 0; j < nsrc[t]; ++j)
      {
        int c, r, u, ek, e1, cwd, len;
        unpack_row(src[t][j], &c, &r, &u, &ek, &e1, &cwd, &len);
        if(c != cq || r != rho)
          continue;
        if(emb)
        {
          if(u == 1 && (emb & ek) == e1)
          {
            int pop = __builtin_popcount((unsigned)ek);
            if(pop >= best_pop)
            {
              best = (int)j;
              best_pop = pop;
            }
          }
        }
        else if(u == 0)
        {
          best = (int)j;
          break;
        }
      }
      int c, r, u, ek, e1, cwd, len;
      unpack_row(src[t][best], &c, &r, &u, &ek, &e1, &cwd, &len);
      enc_vlc[t][i] = (uint16_t)((cwd << 8) | (len << 4) | ek);
    }
    for(int i = 0; i < 1024; ++i)
    {
      int cq = i >> 7, bits = i & 0x7F;
      dec_vlc[t][i] = 0;
      for(size_t j = 0; j < nsrc[t]; ++j)
      {
        int c, r, u, ek, e1, cwd, len;
        unpack_row(src[t][j], &c, &r, &u, &ek, &e1, &cwd, &len);
        if(c == cq && cwd == (bits & ((1 << len) - 1)))
          dec_vlc[t][i] = (uint16_t)(r | (ek << 4) | (e1 << 8) | (u << 12) | (len << 13));
      }
    }
  }
  tables_ready = 1;
}

ORC_API const uint16_t* orc_ht_enc_table(int t) { build_tables(); return enc_vlc[t]; }
ORC_API const uint16_t* orc_ht_dec_table(int t) { build_tables(); return dec_vlc[t]; }

/* UVLC code for u (ojph_block_encoder.cpp L196-256): prefix then suffix, LSB first. */
static void uvlc_code(int u, int* pre, int* pre_len, int* suf, int* suf_len)
{
  if(u == 0) { *pre = 0; *pre_len = 0; *suf = 0; *suf_len = 0; }
  else if(u == 1) { *pre = 1; *pre_len = 1; *suf = 0; *suf_len = 0; }
  else if(u == 2) { *pre = 2; *pre_len = 2; *suf = 0; *suf_len = 0; }
  else if(u <= 4) { *pre = 4; *pre_len = 3; *suf = u - 3; *suf_len = 1; }
  else { *pre = 0; *pre_len = 3; *suf = u - 5; *suf_len = 5; } /* u <= 32 on the 32-bit path */
}

/* ---- the three byte streams (ojph_block_encoder.cpp L273-535) ---- */
typedef struct { uint8_t* buf; uint32_t pos, cap; int rem, tmp, run, k, thr; int err; } mel_w;
typedef struct { uint8_t* last; uint32_t pos, cap; int used, tmp, gt8f; int err; } vlc_w;
typedef struct { uint8_t* buf; uint32_t pos, cap; int maxb, used; uint32_t tmp; int err; } ms_w;

static const int MEL_EXP[13] = {0, 0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 4, 5};

static void mel_bit(mel_w* m, int v)
{
  m->tmp = (m->tmp << 1) + v;
  if(--m->rem == 0)
  {
    if(m->pos >= m->cap) { m->err = 1; return; }
    m->buf[m->pos++] = (uint8_t)m->tmp;
    m->rem = (m->tmp == 0xFF) ? 7 : 8;
    m->tmp = 0;
  }
}
static void mel_event(mel_w* m, int bit)
{
  if(!bit)
  {
    if(++m->run >= m->thr)
    {
      mel_bit(m, 1);
      m->run = 0;
      m->k = imin(12, m->k + 1);
      m->thr = 1 << MEL_EXP[m->k];
    }
  }
  else
  {
    mel_bit(m, 0);
    for(int t = MEL_EXP[m->k]; t > 0;)
      mel_bit(m, (m->run >> --t) & 1);
    m->run = 0;
    m->k = imax(0, m->k - 1);
    m->thr = 1 << MEL_EXP[m->k];
  }
}
static void vlc_put(vlc_w* v, int cwd, int len)
{
  while(len > 0)
  {
    if(v->pos >= v->cap) { v->err = 1; return; }
    int avail = 8 - v->gt8f - v->used;
    int t = imin(avail, len);
    v->tmp |= (cwd & ((1 << t) - 1)) << v->used;
    v->used += t; avail -= t; len -= t; cwd >>= t;
    if(avail == 0)
    {
      if(v->gt8f && v->tmp != 0x7F) { v->gt8f = 0; continue; }
      *(v->last - v->pos) = (uint8_t)v->tmp;
      v->pos++;
      v->gt8f = v->tmp > 0x8F;
      v->tmp = 0; v->used = 0;
    }
  }
}
static void ms_put(ms_w* s, uint32_t cwd, int len)
{
  while(len > 0)
  {
    if(s->pos >= s->cap) { s->err = 1; return; }
    int t = imin(s->maxb - s->used, len);
    s->tmp |= (cwd & ((1u << t) - 1)) << s->used;
    s->used += t; cwd >>= t; len -= t;
    if(s->used >= s->maxb)
    {
      s->buf[s->pos++] = (uint8_t)s->tmp;
      s->maxb = (s->tmp == 0xFF) ? 7 : 8;
      s->tmp = 0; s->used = 0;
    }
  }
}

typedef struct { int rho, emax, e[4]; uint32_t s[4]; } orc_quad;

static void load_quad(const uint32_t* buf, uint32_t stride, uint32_t w, uint32_t h, uint32_t x,
                      uint32_t y, uint32_t p, orc_quad* q)
{
  /* ojph_block_encoder.cpp L590-643: sample order (x,y),(x,y+1),(x+1,y),(x+1,y+1) */
  q->rho = 0; q->emax = 0;
  for(int i = 0; i < 4; ++i)
  {
    uint32_t xx = x + (uint32_t)(i >> 1), yy = y + (uint32_t)(i & 1);
    q->e[i] = 0; q->s[i] = 0;
    if(xx >= w || yy >= h)
      continue;
    uint32_t t = buf[(size_t)yy * stride + xx];
    uint32_t val = t + t;
    val >>= p;
    val &= ~1u;
    if(val)
    {
      q->rho |= 1 << i;
      --val;
      q->e[i] = 32 - __builtin_clz(val);
      q->emax = imax(q->emax, q->e[i]);
      q->s[i] = --val + (t >> 31);
    }
  }
}

/* The choices T.814 leaves to an encoder, as orc_ht_encode_foreign takes them (bit set).  orc_ht_encode makes none of
 * them: it codes like the reference.  Each one below is decoded by the reference decoder (oracle/_ref) to the source's
 * bin-centre values, pinned by tests/golden/ht_foreign.npz. */
enum
{
  ORC_FOREIGN_ROWS = 1,        /* any legal CxtVLC row of a u_off = 1 quad, not the one with the most e_k bits */
  ORC_FOREIGN_RAISE_U = 2,     /* exponent bound U_q above max(E_max, kappa), up to missing_msbs + 2 */
  ORC_FOREIGN_NO_FUSE = 4,     /* MEL and VLC terminated in separate bytes even where one byte could end both */
  ORC_FOREIGN_PAD_MAGSGN = 8,  /* bytes after the MagSgn data that the decoder never reads */
  ORC_FOREIGN_PAD_SCUP = 16,   /* bytes between the MEL and the VLC data (a larger Scup, at most 4079) */
};

/* per-call counts of the choices made, for the coverage tests: [0] quads whose U_q is the decoder's limit, [1] u_off = 1
 * quads coded with a row the max-popcount rule would not pick, [2] raises dropped for want of a row with e_1 = 0;
 * [3] the MEL bytes of the stream (where MEL ends and padding or VLC begins, for tests that edit streams) */
static int32_t foreign_stats[4];
ORC_API void orc_ht_encode_foreign_stats(int32_t* out) { memcpy(out, foreign_stats, sizeof(foreign_stats)); }

typedef struct { uint64_t s; } orc_lcg;
static uint32_t lcg_next(orc_lcg* g)
{
  g->s = g->s * 6364136223846793005ULL + 1442695040888963407ULL;
  return (uint32_t)(g->s >> 33);
}

/* the rows of table t (0: first quad row, 1: the others) a quad (c_q, rho) may be coded with when its u_off is 1 and
 * the samples whose exponent equals U_q are `emb`: e_1 == emb & e_k (an e_k sample has U_q - 1 bits and e_1 as its
 * implied top bit).  Writes up to 16 candidates as enc_vlc entries; returns their count and, in *best, the index of the
 * one orc_ht_encode's table holds (most e_k bits, the last of equals) */
static int legal_rows(int t, int cq, int rho, int emb, uint16_t* cand, int* best)
{
  const uint32_t* src = t ? T814_VLC_ROWS1 : T814_VLC_ROWS0;
  const size_t nsrc = t ? sizeof(T814_VLC_ROWS1) / 4 : sizeof(T814_VLC_ROWS0) / 4;
  int n = 0, best_pop = -1;
  *best = -1;
  for(size_t j = 0; j < nsrc && n < 16; ++j)
  {
    int c, r, u, ek, e1, cwd, len;
    unpack_row(src[j], &c, &r, &u, &ek, &e1, &cwd, &len);
    if(c != cq || r != rho || u != 1 || (emb & ek) != e1)
      continue;
    if(__builtin_popcount((unsigned)ek) >= best_pop)
    {
      best_pop = __builtin_popcount((unsigned)ek);
      *best = n;
    }
    cand[n++] = (uint16_t)((cwd << 8) | (len << 4) | ek);
  }
  return n;
}

/* HT cleanup-pass encoder: ojph_encode_codeblock32, ojph_block_encoder.cpp L542-1017, with the encoder's choices of
 * `choices` (ORC_FOREIGN_*) made by an LCG seeded with `seed`; choices = 0 is orc_ht_encode. */
static int ht_encode_core(const uint32_t* buf, uint32_t missing_msbs, uint32_t width, uint32_t height, uint32_t stride,
                          uint32_t choices, uint64_t seed, uint8_t* out, uint32_t out_cap)
{
  build_tables();
  orc_lcg rng = {seed ^ 0x9E3779B97F4A7C15ULL};
  memset(foreign_stats, 0, sizeof(foreign_stats));
  const int u_limit = (int)missing_msbs + 2; /* ojph_block_decoder32.cpp L846, L1114: U_q > missing_msbs + 2 is refused */
  enum { MS_CAP = (16384 * 16 + 14) / 15, MEL_CAP = 192, VLC_CAP = 3072 - 192 };
  uint8_t* ms_buf = (uint8_t*)malloc(MS_CAP);
  uint8_t mel_buf[MEL_CAP], vlc_buf[VLC_CAP];
  mel_w mel = {mel_buf, 0, MEL_CAP, 8, 0, 0, 0, 1, 0};
  vlc_w vlc = {vlc_buf + VLC_CAP - 1, 1, VLC_CAP, 4, 0xF, 1, 0};
  vlc_buf[VLC_CAP - 1] = 0xFF;
  ms_w ms = {ms_buf, 0, MS_CAP, 8, 0, 0, 0};
  const uint32_t p = 30 - missing_msbs;
  const uint32_t nq = (width + 1) / 2;

  /* exponent of the bottom sample row of the previous quad row, index x+1 (x=-1..width+1) */
  uint8_t* eab = (uint8_t*)calloc(width + 4, 1);
  uint8_t* enew = (uint8_t*)calloc(width + 4, 1);

  for(uint32_t y = 0; y < height; y += 2)
  {
    memset(enew, 0, width + 4);
    int rho_left = 0;
    for(uint32_t q0 = 0; q0 < nq; q0 += 2)
    {
      orc_quad Q[2];
      int cq[2] = {0, 0}, U[2] = {0, 0}, u[2] = {0, 0};
      uint16_t tuple[2] = {0, 0};
      int npair = (q0 + 1 < nq) ? 2 : 1;
      for(int j = 0; j < npair; ++j)
      {
        uint32_t q = q0 + (uint32_t)j, x = 2 * q;
        load_quad(buf, stride, width, height, x, y, p, &Q[j]);
        int kappa = 1;
        if(y == 0)
          cq[j] = (rho_left >> 1) | (rho_left & 1); /* L731, L788 */
        else
        {
          const uint8_t* E = eab + 1 + x; /* E[-1..2] */
          cq[j] = ((E[-1] | E[0]) ? 1 : 0) | ((rho_left & 0xC) ? 2 : 0) | ((E[1] | E[2]) ? 4 : 0);
          int max_e = imax(imax(E[-1], E[0]), imax(E[1], E[2])) - 1; /* L799, L862, L950 */
          kappa = (Q[j].rho & (Q[j].rho - 1)) ? imax(1, max_e) : 1;
        }
        U[j] = imax(Q[j].emax, kappa);
        uint16_t cand[16];
        int ncand = 0, best = -1;
        if((choices & ORC_FOREIGN_RAISE_U) && Q[j].rho && U[j] < u_limit)
        { /* with U_q above every exponent no sample is in EMB: a u_off = 1 row with e_1 = 0 is needed */
          const int raise = (lcg_next(&rng) & 3) == 0 ? u_limit - U[j] : (int)(lcg_next(&rng) % (uint32_t)(u_limit - U[j] + 1));
          if(raise > 0)
          {
            ncand = legal_rows(y ? 1 : 0, cq[j], Q[j].rho, 0, cand, &best);
            if(ncand)
              U[j] += raise;
            else
              foreign_stats[2]++;
          }
        }
        u[j] = U[j] - kappa;
        int eps = 0;
        if(u[j] > 0)
          for(int i = 0; i < 4; ++i)
            eps |= (Q[j].e[i] == U[j]) << i;
        tuple[j] = enc_vlc[y ? 1 : 0][(cq[j] << 8) + (Q[j].rho << 4) + eps];
        if(u[j] > 0 && (ncand || (choices & ORC_FOREIGN_ROWS)))
        {
          if(!ncand)
            ncand = legal_rows(y ? 1 : 0, cq[j], Q[j].rho, eps, cand, &best);
          const int pick = (choices & ORC_FOREIGN_ROWS) ? (int)(lcg_next(&rng) % (uint32_t)ncand) : best;
          tuple[j] = cand[pick];
          foreign_stats[1] += pick != best && (cand[pick] & 0xF) != (cand[best] & 0xF);
        }
        foreign_stats[0] += Q[j].rho && U[j] == u_limit;
        vlc_put(&vlc, tuple[j] >> 8, (tuple[j] >> 4) & 7);
        if(cq[j] == 0)
          mel_event(&mel, Q[j].rho != 0);
        for(int i = 0; i < 4; ++i)
        {
          int m = (Q[j].rho & (1 << i)) ? U[j] - ((tuple[j] >> i) & 1) : 0;
          ms_put(&ms, Q[j].s[i] & ((1u << m) - 1), m);
        }
        enew[1 + x] = (uint8_t)Q[j].e[1];
        if(x + 1 < width)
          enew[1 + x + 1] = (uint8_t)Q[j].e[3];
        rho_left = Q[j].rho;
      }
      int pre[2], prel[2], suf[2], sufl[2];
      if(y == 0)
      { /* L750-785 */
        if(u[0] > 0 && u[1] > 0)
          mel_event(&mel, imin(u[0], u[1]) > 2);
        if(u[0] > 2 && u[1] > 2)
        {
          uvlc_code(u[0] - 2, &pre[0], &prel[0], &suf[0], &sufl[0]);
          uvlc_code(u[1] - 2, &pre[1], &prel[1], &suf[1], &sufl[1]);
          vlc_put(&vlc, pre[0], prel[0]);
          vlc_put(&vlc, pre[1], prel[1]);
          vlc_put(&vlc, suf[0], sufl[0]);
          vlc_put(&vlc, suf[1], sufl[1]);
        }
        else if(u[0] > 2 && u[1] > 0)
        {
          uvlc_code(u[0], &pre[0], &prel[0], &suf[0], &sufl[0]);
          vlc_put(&vlc, pre[0], prel[0]);
          vlc_put(&vlc, u[1] - 1, 1);
          vlc_put(&vlc, suf[0], sufl[0]);
        }
        else
        {
          uvlc_code(u[0], &pre[0], &prel[0], &suf[0], &sufl[0]);
          uvlc_code(u[1], &pre[1], &prel[1], &suf[1], &sufl[1]);
          vlc_put(&vlc, pre[0], prel[0]);
          vlc_put(&vlc, pre[1], prel[1]);
          vlc_put(&vlc, suf[0], sufl[0]);
          vlc_put(&vlc, suf[1], sufl[1]);
        }
      }
      else
      { /* L985-988 */
        uvlc_code(u[0], &pre[0], &prel[0], &suf[0], &sufl[0]);
        uvlc_code(u[1], &pre[1], &prel[1], &suf[1], &sufl[1]);
        vlc_put(&vlc, pre[0], prel[0]);
        vlc_put(&vlc, pre[1], prel[1]);
        vlc_put(&vlc, suf[0], sufl[0]);
        vlc_put(&vlc, suf[1], sufl[1]);
      }
    }
    uint8_t* t = eab; eab = enew; enew = t;
  }

  /* terminate_mel_vlc L412-444 */
  if(mel.run > 0)
    mel_bit(&mel, 1);
  mel.tmp = mel.tmp << mel.rem;
  int mel_mask = (0xFF << mel.rem) & 0xFF;
  int vlc_mask = 0xFF >> (8 - vlc.used);
  if((mel_mask | vlc_mask) != 0)
  {
    int fuse = mel.tmp | vlc.tmp;
    if((((fuse ^ mel.tmp) & mel_mask) | ((fuse ^ vlc.tmp) & vlc_mask)) == 0 && fuse != 0xFF &&
       vlc.pos > 1 && !(choices & ORC_FOREIGN_NO_FUSE))
    {
      if(mel.pos >= mel.cap) mel.err = 1; else mel.buf[mel.pos++] = (uint8_t)fuse;
      if(choices & ORC_FOREIGN_PAD_SCUP)
      { /* bytes will come between the two: the fused byte ends each of them */
        if(vlc.pos >= vlc.cap) mel.err = 1;
        else
        {
          *(vlc.last - vlc.pos) = (uint8_t)fuse;
          vlc.pos++;
        }
      }
    }
    else
    {
      if(mel.pos >= mel.cap || vlc.pos >= vlc.cap) mel.err = 1;
      else
      {
        mel.buf[mel.pos++] = (uint8_t)mel.tmp;
        *(vlc.last - vlc.pos) = (uint8_t)vlc.tmp;
        vlc.pos++;
      }
    }
  }
  /* ms_terminate L516-535: a last byte of ones is left out, the decoder feeds 0xFF past the segment -- unless bytes
     follow it in the segment, which the decoder would read in its place */
  const int ms_pad = (choices & ORC_FOREIGN_PAD_MAGSGN) != 0;
  if(ms.used)
  {
    int t = ms.maxb - ms.used;
    ms.tmp |= (0xFFu & ((1u << t) - 1)) << ms.used;
    ms.used += t;
    if(ms.tmp != 0xFF || ms_pad)
    {
      if(ms.pos >= ms.cap) ms.err = 1; else ms.buf[ms.pos++] = (uint8_t)ms.tmp;
    }
  }
  else if(ms.maxb == 7 && !ms_pad)
    ms.pos--;
  /* padding: bytes below 0x80, so that no pair of bytes in the segment reads as a marker */
  const uint32_t npad_ms = ms_pad ? 1 + lcg_next(&rng) % 40 : 0;
  uint32_t npad_scup = 0;
  if(choices & ORC_FOREIGN_PAD_SCUP)
  {
    const uint32_t room = 4079 > mel.pos + vlc.pos ? 4079 - (mel.pos + vlc.pos) : 0;
    npad_scup = (lcg_next(&rng) & 7) == 0 ? room : imin((int)room, 1 + (int)(lcg_next(&rng) % 48));
  }

  int total = (int)(mel.pos + vlc.pos + ms.pos + npad_ms + npad_scup);
  int rc = total;
  if(mel.err || vlc.err || ms.err || (uint32_t)total > out_cap)
    rc = -1;
  else
  {
    uint8_t* o = out;
    memcpy(o, ms.buf, ms.pos);
    o += ms.pos;
    for(uint32_t i = 0; i < npad_ms; ++i)
      *o++ = (uint8_t)(lcg_next(&rng) & 0x7F);
    memcpy(o, mel.buf, mel.pos);
    o += mel.pos;
    foreign_stats[3] = (int32_t)mel.pos;
    for(uint32_t i = 0; i < npad_scup; ++i)
      *o++ = (uint8_t)(lcg_next(&rng) & 0x7F);
    memcpy(o, vlc.last - vlc.pos + 1, vlc.pos);
    uint32_t nb = mel.pos + npad_scup + vlc.pos; /* L1009-1014 */
    out[total - 1] = (uint8_t)(nb >> 4);
    out[total - 2] = (uint8_t)((out[total - 2] & 0xF0) | (nb & 0xF));
  }
  free(ms_buf); free(eab); free(enew);
  return rc;
}

/* buf: sign-magnitude words (sign bit 31, magnitude << (30 - missing_msbs)).
 * Returns the coded length, or -1 on a buffer overflow the reference would have reported. */
ORC_API int orc_ht_encode(const uint32_t* buf, uint32_t missing_msbs, uint32_t width, uint32_t height,
                          uint32_t stride, uint8_t* out, uint32_t out_cap)
{
  return ht_encode_core(buf, missing_msbs, width, height, stride, 0, 0, out, out_cap);
}

/* TEST INFRASTRUCTURE: the same cleanup pass as another HTJ2K encoder may write it, with the choices of `choices`
 * (ORC_FOREIGN_*) made by an LCG seeded with `seed` -- streams this project's own coders never write, for testing the
 * decoders on them.  choices = 0 gives orc_ht_encode's bytes. */
ORC_API int orc_ht_encode_foreign(const uint32_t* buf, uint32_t missing_msbs, uint32_t width, uint32_t height,
                                  uint32_t stride, uint32_t choices, uint64_t seed, uint8_t* out, uint32_t out_cap)
{
  return ht_encode_core(buf, missing_msbs, width, height, stride, choices, seed, out, out_cap);
}

/* ------------------------------------------------------------------------------------------ */
/* HT cleanup-pass decoder, ojph_decode_codeblock32 (ojph_block_decoder32.cpp L742-1317),      */
/* written from the T.814 procedure: bit readers work a bit at a time, so the byte-alignment   */
/* tricks of the reference (mel_init L226-258, rev_init L367-395, frwd_init L679-701) vanish.  */
/* ------------------------------------------------------------------------------------------ */
typedef struct { const uint8_t* d; int size, pos; int bits; uint32_t tmp; int unstuff; int k; int run; int have_run; } mel_r;

static int mel_getbit(mel_r* m)
{ /* mel_read L92-149: MSB first; after 0xFF the next byte carries 7 bits; the last byte of
     the MEL+VLC region has its low nibble forced to 1s; 0xFF fed when exhausted */
  if(m->bits == 0)
  {
    uint32_t v = 0xFF;
    if(m->pos < m->size)
    {
      v = m->d[m->pos];
      if(m->pos == m->size - 1)
        v |= 0xF;
      m->pos++;
    }
    m->bits = 8 - m->unstuff;
    m->tmp = v;
    m->unstuff = (v == 0xFF);
  }
  m->bits--;
  return (m->tmp >> m->bits) & 1;
}
/* returns next MEL symbol (0/1): mel_decode L168-206 */
static int mel_symbol(mel_r* m)
{
  if(!m->have_run)
  {
    int eval = MEL_EXP[m->k];
    if(mel_getbit(m))
    {
      m->run = 1 << eval; /* that many zeros, no terminating one */
      m->have_run = 1;    /* 1: run of zeros only */
      m->k = imin(12, m->k + 1);
    }
    else
    {
      int r = 0;
      for(int i = 0; i < eval; ++i)
        r = (r << 1) | mel_getbit(m);
      m->run = r;
      m->have_run = 2; /* 2: zeros then a one */
      m->k = imax(0, m->k - 1);
    }
  }
  if(m->run > 0)
  {
    m->run--;
    if(m->run == 0 && m->have_run == 1)
      m->have_run = 0;
    return 0;
  }
  /* run == 0 */
  if(m->have_run == 2)
  {
    m->have_run = 0;
    return 1;
  }
  m->have_run = 0;
  return mel_symbol(m);
}

typedef struct { const uint8_t* d; int pos; int lo; uint64_t tmp; int bits; int unstuff; } vlc_r;

static void vlc_fill(vlc_r* v)
{ /* rev_read L296-345: bytes consumed backwards, a byte that follows one > 0x8F and whose low
     7 bits are all ones contributes 7 bits; zeros once the segment is exhausted */
  while(v->bits <= 56)
  {
    uint32_t b = 0;
    if(v->pos >= v->lo)
      b = v->d[v->pos--];
    int nb = 8 - ((v->unstuff && ((b & 0x7F) == 0x7F)) ? 1 : 0);
    v->tmp |= (uint64_t)b << v->bits;
    v->bits += nb;
    v->unstuff = b > 0x8F;
  }
}
static uint32_t vlc_peek(vlc_r* v) { vlc_fill(v); return (uint32_t)v->tmp; }
static void vlc_skip(vlc_r* v, int n) { v->tmp >>= n; v->bits -= n; }

typedef struct { const uint8_t* d; int size, pos; uint64_t tmp; int bits; int unstuff; } ms_r;
static void ms_fill(ms_r* s)
{ /* frwd_read<0xFF> L628-669 */
  while(s->bits <= 56)
  {
    uint32_t b = s->pos < s->size ? s->d[s->pos] : 0xFF;
    s->pos++;
    s->tmp |= (uint64_t)b << s->bits;
    s->bits += 8 - s->unstuff;
    s->unstuff = (b == 0xFF);
  }
}
static uint32_t ms_peek(ms_r* s) { ms_fill(s); return (uint32_t)s->tmp; }
static void ms_skip(ms_r* s, int n) { s->tmp >>= n; s->bits -= n; }

/* decode one UVLC prefix from bits (LSB first): returns value class and length */
static int uvlc_prefix(uint32_t bits, int* len)
{
  if(bits & 1) { *len = 1; return 1; }
  if(bits & 2) { *len = 2; return 2; }
  if(bits & 4) { *len = 3; return 3; }
  *len = 3; return 5;
}
static int uvlc_suffix_len(int pfx) { return pfx == 3 ? 1 : (pfx == 5 ? 5 : 0); }

/* Decodes the cleanup pass only (num_passes == 1).  out: sign<<31 | (2*mu+1) << (p-1),
 * row stride `stride`.  Returns 0 on success, -1 on a malformed block. */
ORC_API int orc_ht_decode(const uint8_t* data, uint32_t lcup, uint32_t missing_msbs, uint32_t width,
                          uint32_t height, uint32_t stride, uint32_t* out)
{
  build_tables();
  for(uint32_t y = 0; y < height; ++y)
    memset(out + (size_t)y * stride, 0, sizeof(uint32_t) * width);
  if(missing_msbs > 29 || lcup < 2)
    return -1;
  const uint32_t p = 30 - missing_msbs;
  int scup = ((int)data[lcup - 1] << 4) + (data[lcup - 2] & 0xF);
  if(scup < 2 || scup > (int)lcup || scup > 4079)
    return -1;
  const uint32_t nq = (width + 1) / 2;
  const uint32_t mmsbp2 = missing_msbs + 2;

  mel_r mel = {data + lcup - scup, scup - 1, 0, 0, 0, 0, 0, 0, 0};
  /* rev_init L367-395: first (half) byte */
  vlc_r vlc = {data, (int)lcup - 3, (int)lcup - scup, 0, 0, 0};
  {
    uint32_t d = data[lcup - 2];
    vlc.tmp = d >> 4;
    vlc.bits = 4 - ((vlc.tmp & 7) == 7);
    vlc.unstuff = (d | 0xF) > 0x8F;
  }
  ms_r ms = {data, (int)lcup - scup, 0, 0, 0, 0};

  /* per-quad records of the previous quad row */
  uint8_t* rho_prev = (uint8_t*)calloc(nq + 2, 1);
  uint8_t* rho_cur = (uint8_t*)calloc(nq + 2, 1);
  uint32_t* vn_prev = (uint32_t*)calloc(width + 4, sizeof(uint32_t)); /* v_n of row y-1, idx x+1 */
  uint32_t* vn_cur = (uint32_t*)calloc(width + 4, sizeof(uint32_t));
  int rc = 0;

  for(uint32_t y = 0; y < height && rc == 0; y += 2)
  {
    memset(rho_cur, 0, nq + 2);
    memset(vn_cur, 0, (width + 4) * sizeof(uint32_t));
    int rho_left = 0;
    for(uint32_t q0 = 0; q0 < nq && rc == 0; q0 += 2)
    {
      int npair = (q0 + 1 < nq) ? 2 : 1;
      int rho[2] = {0, 0}, uoff[2] = {0, 0}, ek[2] = {0, 0}, e1[2] = {0, 0}, u[2] = {0, 0};
      for(int j = 0; j < npair; ++j)
      {
        uint32_t q = q0 + (uint32_t)j;
        int cq;
        if(y == 0)
          cq = (rho_left >> 1) | (rho_left & 1);
        else
        { /* L958-1010: nw/n | w,sw | ne/nf */
          int a = (q > 0 ? (rho_prev[q - 1] & 8) : 0) | (rho_prev[q] & 2);
          int b = (rho_prev[q] & 8) | (q + 1 < nq ? (rho_prev[q + 1] & 2) : 0);
          cq = (a ? 1 : 0) | ((rho_left & 0xC) ? 2 : 0) | (b ? 4 : 0);
        }
        uint16_t t = dec_vlc[y ? 1 : 0][(cq << 7) | (vlc_peek(&vlc) & 0x7F)];
        if(cq == 0 && !mel_symbol(&mel))
          t = 0;
        rho[j] = t & 0xF; ek[j] = (t >> 4) & 0xF; e1[j] = (t >> 8) & 0xF; uoff[j] = (t >> 12) & 1;
        vlc_skip(&vlc, t >> 13);
        rho_cur[q] = (uint8_t)rho[j];
        rho_left = rho[j];
      }
      /* UVLC (T.814 7.3.6; L903-941 and L1044-1062) */
      if(y == 0 && uoff[0] && uoff[1])
      {
        int len;
        if(mel_symbol(&mel))
        { /* both > 2 */
          uint32_t b = vlc_peek(&vlc);
          int p0 = uvlc_prefix(b, &len); vlc_skip(&vlc, len);
          b = vlc_peek(&vlc);
          int p1 = uvlc_prefix(b, &len); vlc_skip(&vlc, len);
          int l0 = uvlc_suffix_len(p0), l1 = uvlc_suffix_len(p1);
          b = vlc_peek(&vlc);
          u[0] = 2 + p0 + (int)(b & ((1u << l0) - 1)); vlc_skip(&vlc, l0);
          b = vlc_peek(&vlc);
          u[1] = 2 + p1 + (int)(b & ((1u << l1) - 1)); vlc_skip(&vlc, l1);
        }
        else
        {
          uint32_t b = vlc_peek(&vlc);
          int p0 = uvlc_prefix(b, &len); vlc_skip(&vlc, len);
          if(p0 > 2)
          {
            b = vlc_peek(&vlc);
            u[1] = 1 + (int)(b & 1); vlc_skip(&vlc, 1);
            int l0 = uvlc_suffix_len(p0);
            b = vlc_peek(&vlc);
            u[0] = p0 + (int)(b & ((1u << l0) - 1)); vlc_skip(&vlc, l0);
          }
          else
          {
            b = vlc_peek(&vlc);
            int p1 = uvlc_prefix(b, &len); vlc_skip(&vlc, len);
            int l1 = uvlc_suffix_len(p1);
            u[0] = p0;
            b = vlc_peek(&vlc);
            u[1] = p1 + (int)(b & ((1u << l1) - 1)); vlc_skip(&vlc, l1);
          }
        }
      }
      else
      {
        int len, pf[2] = {0, 0};
        for(int j = 0; j < 2; ++j)
          if(uoff[j])
          {
            pf[j] = uvlc_prefix(vlc_peek(&vlc), &len);
            vlc_skip(&vlc, len);
          }
        for(int j = 0; j < 2; ++j)
          if(uoff[j])
          {
            int l = uvlc_suffix_len(pf[j]);
            u[j] = pf[j] + (int)(vlc_peek(&vlc) & ((1u << l) - 1));
            vlc_skip(&vlc, l);
          }
      }
      /* MagSgn for the pair (L1108-1313) */
      for(int j = 0; j < npair; ++j)
      {
        uint32_t q = q0 + (uint32_t)j, x = 2 * q;
        int kappa = 1;
        if(y > 0)
        {
          const uint32_t* V = vn_prev + 1 + x;
          int gamma = (rho[j] & (rho[j] - 1)) != 0;
          uint32_t emax = V[-1] | V[0] | V[1] | V[2];
          int e = 31 - __builtin_clz(emax | 2);
          kappa = gamma ? e : 1;
        }
        uint32_t U = (uint32_t)(u[j] + kappa);
        if(U > mmsbp2) { rc = -1; break; }
        for(int i = 0; i < 4; ++i)
        {
          uint32_t xx = x + (uint32_t)(i >> 1), yy = y + (uint32_t)(i & 1);
          if(!(rho[j] & (1 << i)))
            continue;
          uint32_t msv = ms_peek(&ms);
          uint32_t m_n = U - ((ek[j] >> i) & 1);
          ms_skip(&ms, (int)m_n);
          uint32_t val = msv << 31;
          uint32_t v_n = msv & ((1u << m_n) - 1);
          v_n |= (uint32_t)((e1[j] >> i) & 1) << m_n;
          v_n |= 1;
          val |= (v_n + 2) << (p - 1);
          if(xx < width && yy < height)
            out[(size_t)yy * stride + xx] = val;
          if(i & 1) /* bottom row of the quad feeds the next row's exponent predictor */
            if(xx < width + 2)
              vn_cur[1 + xx] = v_n;
        }
      }
    }
    uint8_t* tr = rho_prev; rho_prev = rho_cur; rho_cur = tr;
    uint32_t* tv = vn_prev; vn_prev = vn_cur; vn_cur = tv;
  }
  free(rho_prev); free(rho_cur); free(vn_prev); free(vn_cur);
  return rc;
}

/* ================================================================================================
 * HT refinement passes (ITU-T T.814 SigProp + MagRef), the part of T1OJPH::decompress the reference
 * runs when a code block carries 2 or 3 passes: ojph_block_decoder32.cpp L1318-1616.
 *
 * The reference works on 4x4 nibble-packed significance words; this restatement keeps per-sample
 * state and the scan order only:
 *   stripes of 4 rows, inside a stripe groups of 4 columns, inside a group column by column,
 *   top to bottom.  sigma = significant after the cleanup pass (cleanup LSB plane p); the passes
 *   add bit-plane p-1.
 *   SigProp: a sample that is not in sigma is a member when any of its 8 neighbours is in sigma or
 *     became significant earlier in this pass; neighbours outside the block do not exist, and in
 *     stripe-causal mode neither do those in the stripe below (L1404-1407).  Each member costs one
 *     bit (1 = significant at plane p-1); the sign bits of a group's new samples follow the
 *     group's last membership bit (L1437-1543).  Forward stream, LSB first, a byte after 0xFF
 *     carries 7 bits (frwd_read<0>, L609-654); zeros once the segment is used up.
 *   MagRef: every sample in sigma (not the ones SigProp added) costs one bit = bit p-1 of its
 *     magnitude, same scan except that groups do not matter (L1562-1612).  Backward stream from
 *     the segment's last byte, LSB first, a byte whose 7 low bits are all ones and whose successor
 *     (in reading order: predecessor) was > 0x8F carries 7 bits, starting as if that were the case
 *     (rev_read_mrp / rev_init_mrp, L453-541).
 * Decoded magnitudes keep the reference's bin-centre convention: a half bit at plane p-2.
 * The encoder below is test infrastructure only (the reference's own encoder never emits these
 * passes); tests pin it by decoding its output with the reference decoder (oracle/_ref).
 * ============================================================================================== */
typedef struct { uint8_t* buf; int pos, cap, nbits, limit; uint32_t tmp; } spp_w;
static void spp_put(spp_w* s, int bit)
{
  s->tmp |= (uint32_t)(bit & 1) << s->nbits;
  if(++s->nbits == s->limit)
  {
    if(s->pos < s->cap) s->buf[s->pos] = (uint8_t)s->tmp;
    s->pos++;
    s->limit = (s->tmp == 0xFF) ? 7 : 8;
    s->tmp = 0; s->nbits = 0;
  }
}
static void spp_flush(spp_w* s)
{
  if(s->nbits)
  {
    uint32_t last = s->tmp;
    if(s->pos < s->cap) s->buf[s->pos] = (uint8_t)last;
    s->pos++;
    s->tmp = 0; s->nbits = 0;
    s->limit = (last == 0xFF) ? 7 : 8;
  }
  if(s->limit == 7)
  { /* never end a forward segment on 0xFF: what follows may be > 0x8F */
    if(s->pos < s->cap) s->buf[s->pos] = 0;
    s->pos++;
    s->limit = 8;
  }
}
typedef struct { uint8_t* buf; int pos, cap, nbits; uint32_t tmp; int prev_gt8f; } mrp_w; /* buf filled in writing order */
static void mrp_emit(mrp_w* m)
{
  if(m->pos < m->cap) m->buf[m->pos] = (uint8_t)m->tmp;
  m->pos++;
  m->prev_gt8f = m->tmp > 0x8F;
  m->tmp = 0; m->nbits = 0;
}
static void mrp_put(mrp_w* m, int bit)
{
  m->tmp |= (uint32_t)(bit & 1) << m->nbits;
  ++m->nbits;
  if(m->nbits == 7 && m->prev_gt8f && m->tmp == 0x7F) { mrp_emit(m); return; }
  if(m->nbits == 8) mrp_emit(m);
}

static int refine_neighbour(const uint8_t* sig, uint32_t w, uint32_t h, uint32_t x, uint32_t y, uint32_t y_limit)
{
  for(int dy = -1; dy <= 1; ++dy)
    for(int dx = -1; dx <= 1; ++dx)
    {
      if(!dx && !dy) continue;
      const int xx = (int)x + dx, yy = (int)y + dy;
      if(xx < 0 || yy < 0 || xx >= (int)w || yy >= (int)h || yy >= (int)y_limit) continue;
      if(sig[(size_t)yy * w + xx]) return 1;
    }
  return 0;
}

/* buf as for orc_ht_encode; the cleanup pass is assumed coded with the same missing_msbs (plane p =
 * 30 - missing_msbs, p >= 2).  num_passes 2 (SigProp) or 3 (SigProp + MagRef).  Writes the refinement
 * segment (SigProp bytes, then MagRef bytes) and returns its length, -1 if it does not fit. */
ORC_API int orc_ht_encode_refine(const uint32_t* buf, uint32_t missing_msbs, uint32_t num_passes, uint32_t width,
                                 uint32_t height, uint32_t stride, int stripe_causal, uint8_t* out, uint32_t out_cap)
{
  if(missing_msbs > 28 || num_passes < 2 || num_passes > 3) return -1;
  const uint32_t p = 30 - missing_msbs;
  uint8_t* sig = (uint8_t*)calloc((size_t)width * height, 1);   /* sigma, then sigma + new */
  uint8_t* cup = (uint8_t*)calloc((size_t)width * height, 1);
  const int cap = (int)(width * height / 4 + 64);
  uint8_t* sbuf = (uint8_t*)malloc((size_t)cap);
  uint8_t* mbuf = (uint8_t*)malloc((size_t)cap);
  spp_w sp = {sbuf, 0, cap, 0, 8, 0};
  mrp_w mr = {mbuf, 0, cap, 0, 0, 1};
  for(uint32_t y = 0; y < height; ++y)
    for(uint32_t x = 0; x < width; ++x)
      cup[(size_t)y * width + x] = sig[(size_t)y * width + x] = ((buf[(size_t)y * stride + x] & 0x7FFFFFFFu) >> p) != 0;
  for(uint32_t y0 = 0; y0 < height; y0 += 4)
  {
    const uint32_t y_limit = stripe_causal ? y0 + 4 : height;
    for(uint32_t gx = 0; gx < width; gx += 4)
    {
      int signs[16], ns = 0;
      for(uint32_t x = gx; x < gx + 4 && x < width; ++x)
        for(uint32_t y = y0; y < y0 + 4 && y < height; ++y)
        {
          if(cup[(size_t)y * width + x]) continue;
          if(!refine_neighbour(sig, width, height, x, y, y_limit)) continue;
          const uint32_t v = buf[(size_t)y * stride + x];
          const int bit = (int)(((v & 0x7FFFFFFFu) >> (p - 1)) & 1);
          spp_put(&sp, bit);
          if(bit)
          {
            sig[(size_t)y * width + x] = 1;
            signs[ns++] = (int)(v >> 31);
          }
        }
      for(int i = 0; i < ns; ++i) spp_put(&sp, signs[i]);
    }
  }
  spp_flush(&sp);
  if(num_passes == 3)
  {
    for(uint32_t y0 = 0; y0 < height; y0 += 4)
      for(uint32_t x = 0; x < width; ++x)
        for(uint32_t y = y0; y < y0 + 4 && y < height; ++y)
          if(cup[(size_t)y * width + x])
            mrp_put(&mr, (int)(((buf[(size_t)y * stride + x] & 0x7FFFFFFFu) >> (p - 1)) & 1));
    if(mr.nbits) mrp_emit(&mr);
  }
  int total = sp.pos + mr.pos;
  int rc = -1;
  if(sp.pos <= cap && mr.pos <= cap)
  {
    if(total == 0) { sbuf[0] = 0; sp.pos = 1; total = 1; } /* a refinement segment cannot be empty */
    if((uint32_t)total <= out_cap)
    {
      memcpy(out, sbuf, (size_t)sp.pos);
      for(int i = 0; i < mr.pos; ++i) out[total - 1 - i] = mbuf[i];
      rc = total;
    }
  }
  free(sig); free(cup); free(sbuf); free(mbuf);
  return rc;
}

/* Both readers place a 7-bit byte's top bit where the next byte's first bit goes, as frwd_read and rev_read_mrp
   (L609-654, L453-541) OR whole bytes into their bit buffers: in a valid segment that bit is 0, in a damaged one it is
   ORed into the next byte's lowest bit (`carry`). */
typedef struct { const uint8_t* data; int size, pos, unstuff; uint64_t tmp; int bits; uint32_t carry; } spp_r;
static int spp_get(spp_r* s)
{
  if(!s->bits)
  {
    const uint32_t b = s->pos < s->size ? s->data[s->pos] : 0;
    s->pos++;
    s->bits = 8 - s->unstuff;
    s->tmp = b | s->carry;
    s->carry = s->bits == 7 ? b >> 7 : 0;
    s->unstuff = (b == 0xFF);
  }
  const int v = (int)(s->tmp & 1);
  s->tmp >>= 1; s->bits--;
  return v;
}
typedef struct { const uint8_t* last; int size, pos, unstuff; uint64_t tmp; int bits; uint32_t carry; } mrp_r;
static int mrp_get(mrp_r* m)
{
  if(!m->bits)
  {
    const uint32_t b = m->pos < m->size ? *(m->last - m->pos) : 0;
    m->pos++;
    m->bits = 8 - ((m->unstuff && (b & 0x7F) == 0x7F) ? 1 : 0);
    m->tmp = b | m->carry;
    m->carry = m->bits == 7 ? b >> 7 : 0;
    m->unstuff = b > 0x8F;
  }
  const int v = (int)(m->tmp & 1);
  m->tmp >>= 1; m->bits--;
  return v;
}

/* Full block decode: cleanup (orc_ht_decode) + SigProp (+ MagRef).  `data` holds the cleanup segment
 * (lcup bytes) followed by the refinement segment (len2 bytes).  Mirrors the reference's leniency:
 * len2 == 0 or p == 1 drop the refinement passes (L752-758, L790-803); more than 3 passes fail. */
ORC_API int orc_ht_decode_passes(const uint8_t* data, uint32_t lcup, uint32_t len2, uint32_t num_passes,
                                 uint32_t missing_msbs, uint32_t width, uint32_t height, uint32_t stride,
                                 int stripe_causal, uint32_t* out)
{
  if(num_passes > 3) return -1;
  if(num_passes > 1 && len2 == 0) num_passes = 1;
  if(missing_msbs == 29) num_passes = 1;
  const int rc = orc_ht_decode(data, lcup, missing_msbs, width, height, stride, out);
  if(rc || num_passes <= 1) return rc;
  const uint32_t p = 30 - missing_msbs;
  uint8_t* sig = (uint8_t*)calloc((size_t)width * height, 1);
  uint8_t* cup = (uint8_t*)calloc((size_t)width * height, 1);
  for(uint32_t y = 0; y < height; ++y)
    for(uint32_t x = 0; x < width; ++x)
      cup[(size_t)y * width + x] = sig[(size_t)y * width + x] = out[(size_t)y * stride + x] != 0;
  spp_r sp = {data + lcup, (int)len2, 0, 0, 0, 0, 0};
  for(uint32_t y0 = 0; y0 < height; y0 += 4)
  {
    const uint32_t y_limit = stripe_causal ? y0 + 4 : height;
    for(uint32_t gx = 0; gx < width; gx += 4)
    {
      uint32_t nx[16], ny[16];
      int nn = 0;
      for(uint32_t x = gx; x < gx + 4 && x < width; ++x)
        for(uint32_t y = y0; y < y0 + 4 && y < height; ++y)
        {
          if(cup[(size_t)y * width + x]) continue;
          if(!refine_neighbour(sig, width, height, x, y, y_limit)) continue;
          if(spp_get(&sp))
          {
            sig[(size_t)y * width + x] = 1;
            nx[nn] = x; ny[nn] = y; ++nn;
          }
        }
      for(int i = 0; i < nn; ++i)
        out[(size_t)ny[i] * stride + nx[i]] = ((uint32_t)spp_get(&sp) << 31) | (3u << (p - 2));
    }
  }
  if(num_passes > 2)
  {
    mrp_r mr = {data + lcup + len2 - 1, (int)len2, 0, 1, 0, 0, 0};
    for(uint32_t y0 = 0; y0 < height; y0 += 4)
      for(uint32_t x = 0; x < width; ++x)
        for(uint32_t y = y0; y < y0 + 4 && y < height; ++y)
          if(cup[(size_t)y * width + x])
          {
            const uint32_t bit = (uint32_t)mrp_get(&mr);
            out[(size_t)y * stride + x] ^= ((1u - bit) << (p - 1)) | (1u << (p - 2));
          }
  }
  free(sig); free(cup);
  return 0;
}
