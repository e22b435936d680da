/*
 * grok_b200/csrc/dwt.cu -- forward / inverse lifting DWT (reversible 5/3, irreversible 9/7) for
 * sm_90a, one decomposition level per launch, with the DC level shift and the RCT / ICT
 * multi-component transform fused into the finest level.
 *
 * What it replaces in the reference (CPU, Highway SIMD + Taskflow):
 *   forward : Mct::compress_rev / compress_irrev      point_transform/mct.cpp L497-531, L584-636
 *             encode_53_v/h, encode_97_v/h, encode<>  wavelet/WaveletFwd.cpp L139-876, L1337-1514
 *   inverse : tile_53 / tile_97                       wavelet/WaveletReverse.cpp L1347-1397,
 *                                                     wavelet/WaveletReverse97.cpp L837-857, L950-
 *             DecompressRev / DecompressIrrev         point_transform/mct.cpp L201-256, L318-391
 *
 * Design (not a port of the column-strip SIMD loops):
 *   - one warp = one job = (tile component(s), column strip, row segment).  Each lane
 *     owns 8 consecutive canvas columns (two 128-bit loads per row).  The reference's
 *     "all columns, then all rows" double pass is fused: rows stream through a register
 *     sliding window for the vertical lifting, every finished vertical row is lifted
 *     horizontally with warp shuffles (predict/update need one neighbour each), and the four
 *     sub-bands are written once, de-interleaved, with 128-bit stores.  HBM traffic per level is
 *     one read + one write of every coefficient: the algorithmic minimum.
 *   - symmetric extension is implemented in the LOADS (mirrored addresses), so the lifting
 *     code has no boundary cases.  Neighbours outside the warp are recomputed instead of
 *     exchanged: 5/3 strips are 256 columns wide, all 32 lanes own, and the few columns the
 *     edge lanes need from outside arrive as ghost columns (GhostCol / GhostBand); 9/7 strips
 *     keep lanes 0 and 31 as halo lanes.  Row segments recompute 3 (5/3) or 7 (9/7) halo rows.
 *   - integer maths is bit-exact with the reference; 9/7 uses fmaf() where the reference build
 *     contracts to FMA (see oracle/j2k_oracle.c fwd97_line) and explicit _rn intrinsics elsewhere.
 */
#include "b2k_internal.h"

namespace {

__device__ __noinline__ int mirror_rel_slow(int t, int n)
{
  if(n == 1)
    return 0;
  const int period = 2 * (n - 1);
  t %= period;
  if(t < 0)
    t += period;
  return t < n ? t : period - t;
}
/* whole-sample symmetric extension index; one reflection covers every halo unless the line is
   shorter than the halo, which takes the (out-of-line) periodic path */
__device__ __forceinline__ int mirror_rel(int t, int n)
{
  if((unsigned)t < (unsigned)n)
    return t;
  const int r = t < 0 ? -t : 2 * (n - 1) - t;
  if((unsigned)r < (unsigned)n)
    return r;
  return mirror_rel_slow(t, n);
}

/* ---- 8-sample row loads ------------------------------------------------------------------ */
/* row points at the sample with relative index 0 (canvas u0); rel = first wanted index */
__device__ __forceinline__ void load8_w32(const int32_t* __restrict__ row, int rel, int n, int (&v)[8])
{
  const int32_t* p = row + rel;
  if(rel >= 0 && rel + 8 <= n && ((reinterpret_cast<uintptr_t>(p) & 15) == 0))
  {
    const int4 a = __ldg(reinterpret_cast<const int4*>(p));
    const int4 b = __ldg(reinterpret_cast<const int4*>(p) + 1);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
    v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  }
  else
  {
#pragma unroll
    for(int i = 0; i < 8; ++i)
      v[i] = __ldg(row + mirror_rel(rel + i, n));
  }
}

/* 4 consecutive band samples (inverse transform): idx0 = first band-relative index wanted,
 * mirrored per element through the interleaved domain when out of range */
__device__ __forceinline__ void load4_band(const int32_t* __restrict__ row, int k0, int kb0, int u0, int u1, int odd,
                                           int (&v)[4])
{
  /* sample i has canvas position u = 2*(k0+i)+odd ; band index = (u' >> 1) - kb0 */
  const int ufirst = 2 * k0 + odd, ulast = ufirst + 6;
  const int32_t* p = row + (k0 - kb0);
  if(ufirst >= u0 && ulast < u1 && ((reinterpret_cast<uintptr_t>(p) & 15) == 0))
  {
    const int4 a = __ldg(reinterpret_cast<const int4*>(p));
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  }
  else
  {
    const int n = u1 - u0;
#pragma unroll
    for(int i = 0; i < 4; ++i)
    {
      const int um = u0 + mirror_rel(ufirst + 2 * i - u0, n);
      /* a length-1 line mirrors onto a sample of the other parity: that band is empty */
      v[i] = ((um & 1) == odd) ? __ldg(row + ((um >> 1) - kb0)) : 0;
    }
  }
}

/* ---- job decoding ------------------------------------------------------------------------- */
struct Job
{
  int lane, ulane, jbeg, jend, wn, hn, nvalid;
  bool owner, need;
};
/* WHOLE (5/3): whole-warp strips of 256 columns, lane L owns columns x0 + 8L .. x0 + 8L + 7 and the neighbours outside the
   warp arrive as ghost columns.  Otherwise (9/7): lane 0 is the left halo lane, lanes 1 .. strip_w/8 own, the next is the
   right halo.  `need`: the lane's samples feed an owner (its own, or the right neighbour of the line's last owner). */
template <bool WHOLE>
__device__ __forceinline__ bool decode_job(const DwtLevelDesc& D, Job& J)
{
  J.lane = threadIdx.x & 31;
  const int job = blockIdx.x * B2K_WARPS_PER_CTA + (threadIdx.x >> 5);
  if(job >= (int)D.nstrips * (int)D.nsegs)
    return false;
  const int strip = job % D.nstrips, seg = job / D.nstrips;
  constexpr int halo = WHOLE ? 0 : 1;
  J.wn = D.u1 - D.u0;
  J.hn = D.v1 - D.v0;
  J.nvalid = D.strip_w >> 3;
  J.ulane = (D.u0 & ~7) + strip * (int)D.strip_w + (J.lane - halo) * 8;
  J.owner = J.lane >= halo && J.lane < J.nvalid + halo && J.ulane < D.u1;
  J.need = J.lane <= J.nvalid + halo && J.ulane < D.u1 + 8;
  const int jlo = D.v0 >> 1, jhi = (D.v1 - 1) >> 1;
  J.jbeg = jlo + seg * (int)D.pairs_per_seg;
  J.jend = min(J.jbeg + (int)D.pairs_per_seg, jhi + 1);
  return true;
}

/* =============================================================================================
 * DC shift + colour transforms of the finest level, for N sample positions of NC components (one
 * component: the DC shift alone).  The level-1 DWT kernels, their degenerate jobs and
 * k_point_transform all call these.  The irreversible ones spell out every rounding with _rn
 * intrinsics, in the reference build's operand order: that build contracts a_r*r + a_g*g + a_b*b
 * into two FMAs and the inverse ICT into FMA / FNMA, and the coded bytes are pinned against
 * libgrokj2k (tests/test_interop.py).
 * =========================================================================================== */
/* forward RCT: mct.cpp L497-531 */
template <int NC, int N>
__device__ __forceinline__ void rct_fwd(const DwtLevelDesc& D, int (&x)[NC][N])
{
#pragma unroll
  for(int i = 0; i < N; ++i)
  {
    if constexpr(NC == 3)
    {
      const int r = x[0][i] + D.shift[0], g = x[1][i] + D.shift[1], b = x[2][i] + D.shift[2];
      x[0][i] = ((g + g) + b + r) >> 2;
      x[1][i] = b - g;
      x[2][i] = r - g;
    }
    else
      x[0][i] += D.shift[0];
  }
}

/* forward ICT: mct.cpp L584-636 */
template <int NC, int N>
__device__ __forceinline__ void ict_fwd(const DwtLevelDesc& D, const int (&x)[NC][N], float (&out)[NC][N])
{
  const float a_r = 0.299f, a_g = 0.587f, a_b = 0.114f;
  const float cb = __fdiv_rn(0.5f, __fsub_rn(1.0f, a_b)), cr = __fdiv_rn(0.5f, __fsub_rn(1.0f, a_r));
#pragma unroll
  for(int i = 0; i < N; ++i)
  {
    if constexpr(NC == 3)
    {
      const float r = (float)(x[0][i] + D.shift[0]), g = (float)(x[1][i] + D.shift[1]), b = (float)(x[2][i] + D.shift[2]);
      const float y = __fmaf_rn(a_b, b, __fmaf_rn(a_g, g, __fmul_rn(a_r, r)));
      out[0][i] = y;
      out[1][i] = __fmul_rn(cb, __fsub_rn(b, y));
      out[2][i] = __fmul_rn(cr, __fsub_rn(r, y));
    }
    else
      out[0][i] = (float)(x[0][i] + D.shift[0]);
  }
}

/* inverse RCT, DC shift and clamp to the sample range: mct.cpp L201-256 */
template <int NC, int N>
__device__ __forceinline__ void rct_inv(const DwtLevelDesc& D, int (&x)[NC][N])
{
#pragma unroll
  for(int i = 0; i < N; ++i)
  {
    if constexpr(NC == 3)
    {
      const int y = x[0][i], u = x[1][i], w = x[2][i];
      const int gg = y - ((u + w) >> 2);
      x[0][i] = w + gg;
      x[1][i] = gg;
      x[2][i] = u + gg;
    }
#pragma unroll
    for(int c = 0; c < NC; ++c)
      x[c][i] = min(max(x[c][i] - D.shift[c], D.lo[c]), D.hi[c]);
  }
}

/* inverse ICT, rounding, DC shift and clamp to the sample range: mct.cpp L318-391 */
template <int NC, int N>
__device__ __forceinline__ void ict_inv(const DwtLevelDesc& D, const float (&x)[NC][N], int (&out)[NC][N])
{
#pragma unroll
  for(int i = 0; i < N; ++i)
  {
    float f[NC];
    if constexpr(NC == 3)
    {
      const float y = x[0][i], u = x[1][i], w = x[2][i];
      f[0] = __fmaf_rn(w, 1.402f, y);
      f[1] = __fmaf_rn(-w, 0.71414f, __fmaf_rn(-u, 0.34413f, y));
      f[2] = __fmaf_rn(u, 1.772f, y);
    }
    else
      f[0] = x[0][i];
#pragma unroll
    for(int c = 0; c < NC; ++c)
      out[c][i] = min(max(__float2int_rn(f[c]) - D.shift[c], D.lo[c]), D.hi[c]);
  }
}

/* =============================================================================================
 * forward sample fetch: integers from the image at the finest level (+ DC shift, + RCT / ICT),
 * the previous level's LL coefficients elsewhere
 * =========================================================================================== */
template <int NC>
__device__ __forceinline__ void fetch_int_rows(const DwtLevelDesc& D, const Job& J, int v, int (&out)[NC][8])
{
  const int r = mirror_rel(v - D.v0, J.hn);
#pragma unroll
  for(int c = 0; c < NC; ++c)
  {
    if(!J.need)
    {
#pragma unroll
      for(int i = 0; i < 8; ++i)
        out[c][i] = 0;
      continue;
    }
    load8_w32(reinterpret_cast<const int32_t*>(D.in[c]) + (size_t)r * D.in_pitch, J.ulane - D.u0, J.wn, out[c]);
  }
}

/* a fetched row -> the values the 5/3 lifting starts from */
template <int NC, int N>
__device__ __forceinline__ void to_coeffs53(const DwtLevelDesc& D, int (&x)[NC][N])
{
  if(D.first_level)
    rct_fwd<NC, N>(D, x);
}

/* a fetched row -> the values the 9/7 lifting starts from; the float conversion of the finest level
   is WaveletFwd.cpp L658-681, other levels hold float bits */
template <int NC>
__device__ __forceinline__ void to_coeffs97(const DwtLevelDesc& D, const int (&raw)[NC][8], float (&out)[NC][8])
{
  if(D.first_level)
    ict_fwd<NC>(D, raw, out);
  else
  {
#pragma unroll
    for(int c = 0; c < NC; ++c)
#pragma unroll
      for(int i = 0; i < 8; ++i)
        out[c][i] = __int_as_float(raw[c][i]);
  }
}

template <int NC>
__device__ __forceinline__ void fetch53(const DwtLevelDesc& D, const Job& J, int v, int (&out)[NC][8])
{
  fetch_int_rows<NC>(D, J, v, out);
  to_coeffs53<NC>(D, out);
}

/* ---- ghost columns of a whole-warp 5/3 strip (forward) ----------------------------------------------------------------
 * The horizontal lifting of lane 0 needs the vertically lifted columns x0-2 and x0-1, lane 31 needs x0+256 (x0 = the
 * strip's first column).  Lane 0 carries column x0-1, lane 1 column x0-2 and lane 31 column x0+256 through the same
 * vertical lifting as its body (one extra column per lane, mirrored address: the extension stays in the loads); a
 * shuffle hands lane 1's result to lane 0.  The other lanes carry a copy of their own first column, which nobody uses. */
struct GhostCol
{
  int col;    /* mirrored column, relative to u0 */
  int slot;   /* 0, 1, 2 for lanes 0, 1, 31; -1: no ghost */
};
__device__ __forceinline__ GhostCol ghost_col(const DwtLevelDesc& D, const Job& J)
{
  const int x0 = J.ulane - 8 * J.lane;
  GhostCol G;
  G.slot = J.lane == 0 ? 0 : J.lane == 1 ? 1 : J.lane == 31 ? 2 : -1;
  const int x = J.lane == 0 ? x0 - 1 : J.lane == 1 ? x0 - 2 : J.lane == 31 ? x0 + 256 : J.ulane;
  G.col = mirror_rel(x - D.u0, J.wn);
  return G;
}
/* the ghost column of canvas row v, unstaged (degenerate jobs and the first even row of a segment) */
template <int NC>
__device__ __forceinline__ void fetch_ghost53(const DwtLevelDesc& D, const Job& J, const GhostCol& G, int v, int (&out)[NC][1])
{
  const int r = mirror_rel(v - D.v0, J.hn);
#pragma unroll
  for(int c = 0; c < NC; ++c)
    out[c][0] = __ldg(reinterpret_cast<const int32_t*>(D.in[c]) + (size_t)r * D.in_pitch + G.col);
  to_coeffs53<NC>(D, out);
}

template <int NC>
__device__ __forceinline__ void fetch97(const DwtLevelDesc& D, const Job& J, int v, float (&out)[NC][8])
{
  int raw[NC][8];
  fetch_int_rows<NC>(D, J, v, raw);
  to_coeffs97<NC>(D, raw, out);
}

/* ---- sub-band row stores (Mallat layout: TileComponentWindow.h L241-264) -------------------- */
struct BandGeom
{
  int x0l, x0h, y0l, y0h, snx, sny;
};
__device__ __forceinline__ BandGeom band_geom(const DwtLevelDesc& D)
{
  BandGeom g;
  g.x0l = (D.u0 + 1) >> 1;
  g.x0h = D.u0 >> 1;
  g.y0l = (D.v0 + 1) >> 1;
  g.y0h = D.v0 >> 1;
  g.snx = ((D.u1 + 1) >> 1) - g.x0l;
  g.sny = ((D.v1 + 1) >> 1) - g.y0l;
  return g;
}

/* per-lane constants of the sub-band stores */
struct StoreCtx
{
  unsigned mlo, mhi;
  bool vec_ll, vec_lo, vec_hi; /* all four samples valid and the 16-byte store is aligned */
  int col_ll, col_lo, col_hi; /* column of the lane's first low sample in the LL plane / in the
                                 Mallat buffer, and of its first high sample */
};
__device__ __forceinline__ StoreCtx store_ctx(const DwtLevelDesc& D, const Job& J, const BandGeom& g)
{
  StoreCtx s;
  s.mlo = s.mhi = 0;
  if(J.owner)
  {
#pragma unroll
    for(int i = 0; i < 4; ++i)
    {
      const int ue = J.ulane + 2 * i;
      if(ue >= D.u0 && ue < D.u1)
        s.mlo |= 1u << i;
      if(ue + 1 >= D.u0 && ue + 1 < D.u1)
        s.mhi |= 1u << i;
    }
  }
  const int k0 = J.ulane >> 1;
  s.col_ll = k0 - g.x0l;
  s.col_lo = k0 - g.x0l;
  s.col_hi = g.snx + k0 - g.x0h;
  /* row pitches are multiples of 4 elements (engine allocates 128-byte multiples) */
  const bool pitch_ok = ((D.ll_pitch | D.c_pitch) & 3u) == 0;
  s.vec_ll = pitch_ok && s.mlo == 0xF && (((reinterpret_cast<uintptr_t>(D.out_ll[0]) >> 2) + (unsigned)s.col_ll) & 3u) == 0;
  s.vec_lo = pitch_ok && s.mlo == 0xF && (((reinterpret_cast<uintptr_t>(D.out_c[0]) >> 2) + (unsigned)s.col_lo) & 3u) == 0;
  s.vec_hi = pitch_ok && s.mhi == 0xF && (((reinterpret_cast<uintptr_t>(D.out_c[0]) >> 2) + (unsigned)s.col_hi) & 3u) == 0;
  return s;
}
__device__ __forceinline__ void store4v(int32_t* __restrict__ p, const int (&v)[4], unsigned mask, bool vec)
{
  if(vec)
    *reinterpret_cast<int4*>(p) = make_int4(v[0], v[1], v[2], v[3]);
  else
  {
#pragma unroll
    for(int i = 0; i < 4; ++i)
      if(mask & (1u << i))
        p[i] = v[i];
  }
}
/* lo[4]/hi[4]: horizontally transformed samples of one vertical row (vertical low if !vhigh) */
__device__ __forceinline__ void store_rows(const DwtLevelDesc& D, const BandGeom& g, const StoreCtx& S, int c, int j,
                                           bool vhigh, const int (&lo)[4], const int (&hi)[4])
{
  const int v = 2 * j + (vhigh ? 1 : 0);
  if(v < D.v0 || v >= D.v1 || (S.mlo | S.mhi) == 0)
    return;
  /* all components of a descriptor share the alignment of component 0 (planes are equally laid out) */
  if(!vhigh)
  {
    /* LL -> out_ll, HL -> Mallat top-right */
    const int r = j - g.y0l;
    store4v(reinterpret_cast<int32_t*>(D.out_ll[c]) + (r * (int)D.ll_pitch + S.col_ll), lo, S.mlo, S.vec_ll);
    store4v(reinterpret_cast<int32_t*>(D.out_c[c]) + (r * (int)D.c_pitch + S.col_hi), hi, S.mhi, S.vec_hi);
  }
  else
  {
    const int r = g.sny + j - g.y0h;
    int32_t* crow = reinterpret_cast<int32_t*>(D.out_c[c]) + r * (int)D.c_pitch;
    store4v(crow + S.col_lo, lo, S.mlo, S.vec_lo);
    store4v(crow + S.col_hi, hi, S.mhi, S.vec_hi);
  }
}

/* ---- horizontal lifting of one row held as 8 values per lane -------------------------------- */
/* g: the lane's ghost column of the same row (see GhostCol); lanes 0 and 31 take their outer neighbours from the ghosts
   by selects, so every lane runs the same instructions */
template <bool DEGEN = true>
__device__ __forceinline__ void hfwd53(const int (&r)[8], int g, int wn, int (&lo)[4], int (&hi)[4])
{
  const int lane = threadIdx.x & 31;
  const int g2 = __shfl_down_sync(0xffffffffu, g, 1); /* lane 0: column x0-2 */
  const int rn = __shfl_down_sync(0xffffffffu, r[0], 1);
  const int en = lane == 31 ? g : rn;
  hi[0] = r[1] - ((r[0] + r[2]) >> 1);
  hi[1] = r[3] - ((r[2] + r[4]) >> 1);
  hi[2] = r[5] - ((r[4] + r[6]) >> 1);
  hi[3] = r[7] - ((r[6] + en) >> 1);
  const int hp = __shfl_up_sync(0xffffffffu, hi[3], 1);
  const int dp = lane == 0 ? g - ((g2 + r[0]) >> 1) : hp;
  lo[0] = r[0] + ((dp + hi[0] + 2) >> 2);
  lo[1] = r[2] + ((hi[0] + hi[1] + 2) >> 2);
  lo[2] = r[4] + ((hi[1] + hi[2] + 2) >> 2);
  lo[3] = r[6] + ((hi[2] + hi[3] + 2) >> 2);
  if(DEGEN && wn == 1)
  { /* WaveletFwd.cpp L289-300: lone column, doubled when it sits on an odd coordinate */
#pragma unroll
    for(int i = 0; i < 4; ++i)
    {
      lo[i] = r[2 * i];
      hi[i] = r[2 * i + 1] << 1;
    }
  }
}

#define F97_ALPHA (-1.586134342f)
#define F97_BETA (-0.052980118f)
#define F97_GAMMA (0.882911075f)
#define F97_DELTA (0.443506852f)
#define F97_K (1.230174105f)

__device__ __forceinline__ void hfwd97(const float (&r)[8], int wn, float invK, float deltaS, int (&lo)[4],
                                       int (&hi)[4])
{
  float e[5], d[4], s[5];
#pragma unroll
  for(int i = 0; i < 4; ++i)
    e[i] = r[2 * i];
  e[4] = __shfl_down_sync(0xffffffffu, r[0], 1);
#pragma unroll
  for(int i = 0; i < 4; ++i)
    d[i] = fmaf(e[i] + e[i + 1], F97_ALPHA, r[2 * i + 1]);
  float dm = __shfl_up_sync(0xffffffffu, d[3], 1);
  s[0] = fmaf(dm + d[0], F97_BETA, e[0]);
#pragma unroll
  for(int i = 1; i < 4; ++i)
    s[i] = fmaf(d[i - 1] + d[i], F97_BETA, e[i]);
  s[4] = __shfl_down_sync(0xffffffffu, s[0], 1);
#pragma unroll
  for(int i = 0; i < 4; ++i)
    d[i] = __fmul_rn(fmaf(s[i] + s[i + 1], F97_GAMMA, d[i]), F97_K);
  dm = __shfl_up_sync(0xffffffffu, d[3], 1);
  float o0 = __fmul_rn(fmaf(dm + d[0], deltaS, s[0]), invK);
  lo[0] = __float_as_int(o0);
#pragma unroll
  for(int i = 1; i < 4; ++i)
    lo[i] = __float_as_int(__fmul_rn(fmaf(d[i - 1] + d[i], deltaS, s[i]), invK));
#pragma unroll
  for(int i = 0; i < 4; ++i)
    hi[i] = __float_as_int(d[i]);
  if(wn == 1)
  { /* WaveletFwd.cpp L444-455 */
#pragma unroll
    for(int i = 0; i < 4; ++i)
    {
      lo[i] = __float_as_int(r[2 * i]);
      hi[i] = __float_as_int(__fmul_rn(r[2 * i + 1], 2.0f));
    }
  }
}

/* ---- asynchronous copies into shared memory -------------------------------------------------
 * cp.async (LDGSTS): 16 or 4 bytes per lane and instruction, L1 bypass for the 16-byte ones;
 * completion is tracked per thread by commit groups. */
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src)
{
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src)
{
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait()
{
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

/* ---- bulk asynchronous copies (the TMA engine: SASS UBLKCP) completing on an mbarrier -------------------------
 * A warp whose 32 lanes all sit inside the line stages a whole 1 KB warp-row with ONE instruction issued by one lane
 * instead of 64 LDGSTS (two per lane): the copy engine generates the addresses, the LSU issue slots go back to the
 * lifting code.  The row lands linearly (no XOR swizzle -- a bulk copy is contiguous); the lanes' two 128-bit reads
 * are then 2-way bank conflicted, which costs nothing here: shared memory moves 16 B/clk/SM of the 128 it can. */
__device__ __forceinline__ void mbar_init(uint64_t* bar, unsigned count)
{
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, unsigned bytes)
{
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, unsigned bytes, uint64_t* bar)
{
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   (unsigned)__cvta_generic_to_shared(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, unsigned parity)
{
  asm volatile("{\n"
               ".reg .pred p;\n"
               "MBAR_WAIT_%=:\n"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
               "@p bra MBAR_DONE_%=;\n"
               "bra MBAR_WAIT_%=;\n"
               "MBAR_DONE_%=:\n"
               "}" ::"r"((unsigned)__cvta_generic_to_shared(bar)),
               "r"(parity)
               : "memory");
}

/* =============================================================================================
 * the per-warp staging pipeline of all four DWT kernels: each warp owns DWT_STAGES shared-memory
 * slots of one row pair (Stage::PAIRB bytes), plus one mbarrier per slot, so DWT_STAGES-1 row pairs
 * are in flight while one is lifted, without holding registers.  Pair t sits in slot
 * (t - tfirst) % DWT_STAGES.  A warp whose lanes are all interior (`bulk`) has lane 0 fill the
 * slot's body (its first Stage::BODYB bytes) with bulk copies that complete on the slot's mbarrier;
 * any other warp fills it with cp.async.  Stages with ghost columns (Stage::GHOSTS, the whole-warp
 * 5/3 strips) keep them after the body; every lane fills its own ghost words with cp.async
 * (fill_side) on both paths, and the bulk path waits for those too.
 * A commit group is closed on every step, filled or not, so that wait_group DWT_STAGES-1 always
 * leaves exactly the pair about to be read complete.
 * Stage::COOPERATIVE: the cp.async fill has each lane copy samples other lanes read, so the warp
 * syncs after the wait, and before every refill on both paths.  Otherwise each lane's cp.async
 * slot is private and only the bulk path (lane 0 writes every lane's samples) syncs before a refill.
 * =========================================================================================== */
constexpr int DWT_STAGES = 3;

struct NoSideFill
{
  __device__ __forceinline__ void operator()(uint8_t*, int) const {}
};

template <class Stage>
struct WarpPipe
{
  /* dynamic shared memory of a CTA: every warp's slots, then every warp's mbarriers */
  static constexpr size_t SLOT_BYTES = (size_t)B2K_WARPS_PER_CTA * DWT_STAGES * Stage::PAIRB;
  static constexpr size_t SMEM_BYTES = SLOT_BYTES + (size_t)B2K_WARPS_PER_CTA * DWT_STAGES * sizeof(uint64_t);

  uint8_t* slots;
  uint64_t* bars;
  int tfirst, tlast, tfill;
  bool bulk;

  __device__ __forceinline__ WarpPipe(uint8_t* smem, bool bulk_, int tfirst_, int tlast_)
      : slots(smem + (size_t)(threadIdx.x >> 5) * DWT_STAGES * Stage::PAIRB),
        bars(reinterpret_cast<uint64_t*>(smem + SLOT_BYTES) + (threadIdx.x >> 5) * DWT_STAGES), tfirst(tfirst_),
        tlast(tlast_), tfill(tfirst_), bulk(bulk_)
  {
  }
  /* fill_bulk(slot, t, bar) runs on lane 0 only; fill_async(slot, t) and fill_side(slot, t) on every lane */
  template <class Bulk, class Async, class Side = NoSideFill>
  __device__ __forceinline__ void refill(const Bulk& fill_bulk, const Async& fill_async, const Side& fill_side = Side())
  {
    if(tfill <= tlast)
    {
      const int slot = (tfill - tfirst) % DWT_STAGES;
      uint8_t* st = slots + (size_t)slot * Stage::PAIRB;
      if(bulk)
      {
        if((threadIdx.x & 31) == 0)
        {
          mbar_expect_tx(bars + slot, Stage::BODYB);
          fill_bulk(st, tfill, bars + slot);
        }
      }
      else
        fill_async(st, tfill);
      fill_side(st, tfill);
    }
    cp_async_commit();
    ++tfill;
  }
  template <class Bulk, class Async, class Side = NoSideFill>
  __device__ __forceinline__ void prime(const Bulk& fill_bulk, const Async& fill_async, const Side& fill_side = Side())
  {
    if(bulk)
    {
      if((threadIdx.x & 31) == 0)
      {
#pragma unroll
        for(int s = 0; s < DWT_STAGES; ++s)
          mbar_init(bars + s, 1);
        mbar_fence_init();
      }
      __syncwarp();
    }
#pragma unroll
    for(int s = 0; s < DWT_STAGES - 1; ++s)
      refill(fill_bulk, fill_async, fill_side);
  }
  /* starts the pair DWT_STAGES-1 ahead, waits for pair t and returns its slot */
  template <class Bulk, class Async, class Side = NoSideFill>
  __device__ __forceinline__ const uint8_t* acquire(int t, const Bulk& fill_bulk, const Async& fill_async,
                                                    const Side& fill_side = Side())
  {
    if(Stage::COOPERATIVE || bulk)
      __syncwarp(); /* every lane has read the slot that is refilled next */
    refill(fill_bulk, fill_async, fill_side);
    const int k = t - tfirst;
    if(bulk)
    {
      mbar_wait(bars + k % DWT_STAGES, (unsigned)((k / DWT_STAGES) & 1));
      if(Stage::GHOSTS)
        cp_async_wait<DWT_STAGES - 1>(); /* the lane's own ghost words: read by this lane only */
    }
    else
    {
      cp_async_wait<DWT_STAGES - 1>();
      if(Stage::COOPERATIVE)
        __syncwarp();
    }
    return slots + (size_t)(k % DWT_STAGES) * Stage::PAIRB;
  }
  __device__ __forceinline__ void drain() const { cp_async_wait<0>(); }
};

/* staged row fetch for the forward kernels: a slot holds the NC warp-rows of the two rows of a
   pair (odd row, next even row), the 8 samples of lane L at bytes [32L, 32L+32) of each.
   GHOSTS_ (whole-warp 5/3 strips): then a 16-byte group per row and component, whose words 0, 1, 2
   hold the ghost samples of lanes 0, 1, 31 (GhostCol) */
template <int NC, bool GHOSTS_ = false>
struct RowStage
{
  static constexpr int ROWB = 1024;           /* bytes of one warp-row of one component */
  static constexpr int BODYB = 2 * NC * ROWB; /* one row pair, all components */
  static constexpr bool GHOSTS = GHOSTS_;
  static constexpr int PAIRB = BODYB + (GHOSTS ? 2 * NC * 16 : 0);
  static constexpr bool COOPERATIVE = true;
  /* 16-byte chunk k of a warp-row (lane L owns chunks 2L, 2L+1) is stored at chunk slot
     k ^ ((k >> 3) & 1): the two 128-bit reads of a lane then hit disjoint banks per quarter warp */
  static __device__ __forceinline__ int swz(int k) { return k ^ ((k >> 3) & 1); }

  /* fill row `which` (0 = odd row, 1 = next even row) of a slot with canvas row v.
     Rows are copied COOPERATIVELY: one cp.async instruction moves 512 contiguous bytes
     (lane L copies chunks L and L+32), so every 32-byte DRAM sector is requested once.
     fastmask: ballot of the lanes whose 8 columns are interior and aligned.
     mcol(i): mirrored column of the lane's sample i (edge lanes only). */
  template <class MCol>
  static __device__ __forceinline__ void fill(uint8_t* stage, int which, const DwtLevelDesc& D, const Job& J, int v,
                                              bool fast, unsigned fastmask, const MCol& mcol)
  {
    const int r = mirror_rel(v - D.v0, J.hn);
    const int rel = J.ulane - D.u0;
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      uint8_t* dst = stage + (which * NC + c) * ROWB;
      const int32_t* row = reinterpret_cast<const int32_t*>(D.in[c]) + (size_t)r * D.in_pitch;
      const int rel0 = rel - 8 * J.lane; /* lane 0's first column */
#pragma unroll
      for(int h = 0; h < 2; ++h)
      {
        const int k = J.lane + 32 * h;
        if((fastmask >> (k >> 1)) & 1u)
          cp_async16(dst + swz(k) * 16, row + rel0 + 4 * k);
      }
      if(J.need && !fast)
      { /* edge lane: mirrored columns, still asynchronous (4-byte copies) */
        uint8_t* d0 = dst + swz(2 * J.lane) * 16;
        uint8_t* d1 = dst + swz(2 * J.lane + 1) * 16;
#pragma unroll
        for(int i = 0; i < 4; ++i)
        {
          cp_async4(d0 + 4 * i, row + mcol(i));
          cp_async4(d1 + 4 * i, row + mcol(4 + i));
        }
      }
    }
  }
  /* the lane's ghost sample of canvas row v into word G.slot of the row's ghost group (lanes 0, 1, 31) */
  static __device__ __forceinline__ void fill_ghost(uint8_t* stage, int which, const DwtLevelDesc& D, const Job& J, int v,
                                                    const GhostCol& G)
  {
    static_assert(GHOSTS, "stage without ghost columns");
    const int r = mirror_rel(v - D.v0, J.hn);
#pragma unroll
    for(int c = 0; c < NC; ++c)
      if(G.slot >= 0)
        cp_async4(stage + BODYB + (which * NC + c) * 16 + 4 * G.slot,
                  reinterpret_cast<const int32_t*>(D.in[c]) + (size_t)r * D.in_pitch + G.col);
  }
  /* byte offset, relative to row `which` = 0, component 0, and stride per (row, component) of the lane's ghost sample;
     a lane without a ghost reads its own first sample instead */
  static __device__ __forceinline__ int2 ghost_at(const Job& J, const GhostCol& G)
  {
    return G.slot >= 0 ? make_int2(BODYB + 4 * G.slot, 16) : make_int2(32 * J.lane, ROWB);
  }
  static __device__ __forceinline__ void read_ghost(const uint8_t* stage, int which, int2 at, int (&out)[NC][1])
  {
#pragma unroll
    for(int c = 0; c < NC; ++c)
      out[c][0] = *reinterpret_cast<const int*>(stage + at.x + (which * NC + c) * at.y);
  }
  /* bulk path (every lane fast): one lane asks the copy engine for the NC whole warp-rows of canvas
     row v; they land linearly in the slot and complete on `bar` (armed with expect_tx) */
  static __device__ __forceinline__ void fill_bulk(uint8_t* stage, int which, const DwtLevelDesc& D, const Job& J, int v, uint64_t* bar)
  {
    const int r = mirror_rel(v - D.v0, J.hn);
    const int rel0 = J.ulane - D.u0 - 8 * J.lane; /* lane 0's first column */
#pragma unroll
    for(int c = 0; c < NC; ++c)
      bulk_g2s(stage + (which * NC + c) * ROWB, reinterpret_cast<const int32_t*>(D.in[c]) + (size_t)r * D.in_pitch + rel0, ROWB, bar);
  }
  /* the lane's 8 samples of row `which`: linear after a bulk fill, swizzled after a cp.async one */
  static __device__ __forceinline__ void read(const uint8_t* stage, int which, const Job& J, bool linear, int (&out)[NC][8])
  {
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      const uint8_t* row = stage + (which * NC + c) * ROWB;
      int4 a, b;
      if(linear)
      {
        a = *reinterpret_cast<const int4*>(row + J.lane * 32);
        b = *reinterpret_cast<const int4*>(row + J.lane * 32 + 16);
      }
      else
      {
        a = *reinterpret_cast<const int4*>(row + swz(2 * J.lane) * 16);
        b = *reinterpret_cast<const int4*>(row + swz(2 * J.lane + 1) * 16);
      }
      out[c][0] = a.x; out[c][1] = a.y; out[c][2] = a.z; out[c][3] = a.w;
      out[c][4] = b.x; out[c][5] = b.y; out[c][6] = b.z; out[c][7] = b.w;
      /* lanes beyond the right halo hold stale shared memory: nothing they compute is stored */
    }
  }
  /* lane can use 16-byte async copies: its 8 columns are inside the line and 16-byte aligned */
  static __device__ __forceinline__ bool lane_fast(const DwtLevelDesc& D, const Job& J)
  {
    const int rel = J.ulane - D.u0;
    bool ok = J.need && rel >= 0 && rel + 8 <= J.wn && (D.in_pitch & 3u) == 0;
#pragma unroll
    for(int c = 0; c < NC; ++c)
      ok = ok && (((reinterpret_cast<uintptr_t>(D.in[c]) + (size_t)rel * 4) & 15) == 0);
    return ok;
  }
};

/* a tile component one sample wide or high at this level: straightforward, unpipelined path
   (WaveletFwd.cpp L146-156, L289-300 special cases live here, not in the hot loop).  The degenerate
   jobs build their store context at every store instead of keeping it live across the loop: held in
   registers it would raise the register count of the kernel that calls them. */
template <int NC>
__device__ __noinline__ void fwd53_degenerate_job(const DwtLevelDesc* __restrict__ dptr, const Job J)
{
  const DwtLevelDesc& D = *dptr; /* re-read from global memory: this path is cold */
  const BandGeom g = band_geom(D);
  const GhostCol G = ghost_col(D, J);
  /* column 8 of each row is the lane's ghost column */
  int E[NC][9], DP[NC][9];
  auto fetch = [&](int v, int (&x)[NC][9]) {
    int b[NC][8], gh[NC][1];
    fetch53<NC>(D, J, v, b);
    fetch_ghost53<NC>(D, J, G, v, gh);
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
#pragma unroll
      for(int i = 0; i < 8; ++i)
        x[c][i] = b[c][i];
      x[c][8] = gh[c][0];
    }
  };
  {
    int A[NC][9], B[NC][9];
    fetch(2 * J.jbeg - 2, A);
    fetch(2 * J.jbeg - 1, B);
    fetch(2 * J.jbeg, E);
#pragma unroll
    for(int c = 0; c < NC; ++c)
#pragma unroll
      for(int i = 0; i < 9; ++i)
        DP[c][i] = B[c][i] - ((A[c][i] + E[c][i]) >> 1);
  }
  for(int j = J.jbeg; j < J.jend; ++j)
  {
    int O[NC][9], E2[NC][9];
    fetch(2 * j + 1, O);
    fetch(2 * j + 2, E2);
#pragma unroll 1
    for(int c = 0; c < NC; ++c)
    {
      int s[9], d[9];
#pragma unroll
      for(int i = 0; i < 9; ++i)
      {
        d[i] = O[c][i] - ((E[c][i] + E2[c][i]) >> 1);
        s[i] = E[c][i] + ((DP[c][i] + d[i] + 2) >> 2);
        if(J.hn == 1)
        {
          s[i] = E[c][i];
          d[i] = O[c][i] << 1;
        }
        DP[c][i] = d[i];
        E[c][i] = E2[c][i];
      }
      int s8[8], d8[8], lo[4], hi[4];
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        s8[i] = s[i];
        d8[i] = d[i];
      }
      hfwd53<true>(s8, s[8], J.wn, lo, hi);
      store_rows(D, g, store_ctx(D, J, g), c, j, false, lo, hi);
      hfwd53<true>(d8, d[8], J.wn, lo, hi);
      store_rows(D, g, store_ctx(D, J, g), c, j, true, lo, hi);
    }
  }
}

/* =============================================================================================
 * forward 5/3
 * =========================================================================================== */
/* 3 CTAs (12 warps) per SM, as the shared memory allows: at most 168 registers per thread, without spills */
template <int NC>
__global__ void __launch_bounds__(B2K_WARPS_PER_CTA * 32, 3) k_dwt53_fwd(const DwtLevelDesc* __restrict__ descs)
{
  extern __shared__ __align__(16) uint8_t smem_dwt[];
  typedef RowStage<NC, true> RS;
  const DwtLevelDesc D = descs[blockIdx.y]; /* by value: fields live in (uniform) registers, not re-read after every store */
  Job J;
  if(!decode_job<true>(D, J))
    return;
  if(J.hn == 1 || J.wn == 1)
  {
    fwd53_degenerate_job<NC>(descs + blockIdx.y, J);
    return;
  }
  const BandGeom g = band_geom(D);
  const StoreCtx SC = store_ctx(D, J, g);
  const bool fast = RS::lane_fast(D, J);
  const unsigned fastmask = __ballot_sync(0xffffffffu, fast);
  const GhostCol G = ghost_col(D, J);
  const int2 gat = RS::ghost_at(J, G);

  /* pairs t = jbeg-1 .. jend-1 : rows (2t+1, 2t+2); the even row before them is fetched directly.
     A strip whose 256 columns lie inside the line gets its rows by bulk copy (TMA engine), any other (the ragged last
     strip, a first strip that starts left of the line) by LDGSTS with mirrored columns for the lanes at the line's ends
     (computed at the copy: only those strips pay for them).  The ghost columns always arrive by LDGSTS. */
  const int tfirst = J.jbeg - 1, tlast = J.jend - 1;
  WarpPipe<RS> pipe(smem_dwt, fastmask == 0xffffffffu, tfirst, tlast);
  auto fill_bulk = [&](uint8_t* st, int tf, uint64_t* bar) {
    RS::fill_bulk(st, 0, D, J, 2 * tf + 1, bar);
    RS::fill_bulk(st, 1, D, J, 2 * tf + 2, bar);
  };
  auto mcol = [&](int i) { return mirror_rel(J.ulane - D.u0 + i, J.wn); };
  auto fill_async = [&](uint8_t* st, int tf) {
    RS::fill(st, 0, D, J, 2 * tf + 1, fast, fastmask, mcol);
    RS::fill(st, 1, D, J, 2 * tf + 2, fast, fastmask, mcol);
  };
  auto fill_ghost = [&](uint8_t* st, int tf) {
    RS::fill_ghost(st, 0, D, J, 2 * tf + 1, G);
    RS::fill_ghost(st, 1, D, J, 2 * tf + 2, G);
  };
  pipe.prime(fill_bulk, fill_async, fill_ghost);
  int E[NC][8], DP[NC][8], gE[NC][1], gDP[NC];
  fetch53<NC>(D, J, 2 * tfirst, E);
  fetch_ghost53<NC>(D, J, G, 2 * tfirst, gE);
#pragma unroll
  for(int c = 0; c < NC; ++c)
  {
#pragma unroll
    for(int i = 0; i < 8; ++i)
      DP[c][i] = 0;
    gDP[c] = 0;
  }

  for(int t = tfirst; t <= tlast; ++t)
  {
    const uint8_t* st = pipe.acquire(t, fill_bulk, fill_async, fill_ghost);
    int O[NC][8], E2[NC][8], gO[NC][1], gE2[NC][1];
    RS::read(st, 0, J, pipe.bulk, O);
    RS::read(st, 1, J, pipe.bulk, E2);
    RS::read_ghost(st, 0, gat, gO);
    RS::read_ghost(st, 1, gat, gE2);
    to_coeffs53<NC>(D, O);
    to_coeffs53<NC>(D, E2);
    to_coeffs53<NC>(D, gO);
    to_coeffs53<NC>(D, gE2);
    const bool emit = t >= J.jbeg;
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      int s[8], d[8];
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        d[i] = O[c][i] - ((E[c][i] + E2[c][i]) >> 1);
        s[i] = E[c][i] + ((DP[c][i] + d[i] + 2) >> 2);
        DP[c][i] = d[i];
        E[c][i] = E2[c][i];
      }
      const int gd = gO[c][0] - ((gE[c][0] + gE2[c][0]) >> 1);
      const int gs = gE[c][0] + ((gDP[c] + gd + 2) >> 2);
      gDP[c] = gd;
      gE[c][0] = gE2[c][0];
      if(emit)
      { /* warp-uniform */
        int lo[4], hi[4];
        hfwd53<false>(s, gs, J.wn, lo, hi);
        store_rows(D, g, SC, c, t, false, lo, hi);
        hfwd53<false>(d, gd, J.wn, lo, hi);
        store_rows(D, g, SC, c, t, true, lo, hi);
      }
    }
  }
  pipe.drain();
}

/* =============================================================================================
 * forward 9/7: vertical pipeline  d1[t] -> s1[t] -> d2[t-1] -> s2[t-1]   (see DESIGN.md)
 * =========================================================================================== */
/* unpipelined path for lines of one sample (cold) */
template <int NC>
__device__ __noinline__ void fwd97_degenerate_job(const DwtLevelDesc* __restrict__ dptr, const Job J)
{
  const DwtLevelDesc& D = *dptr;
  const BandGeom g = band_geom(D);
  const float invK = (float)(1.0 / 1.230174105);
  const float deltaS = __fmul_rn(F97_DELTA, invK);

  float Ev[NC][8], D1[NC][8], S1[NC][8], D2[NC][8];
  fetch97<NC>(D, J, 2 * (J.jbeg - 2), Ev);
#pragma unroll
  for(int c = 0; c < NC; ++c)
#pragma unroll
    for(int i = 0; i < 8; ++i)
      D1[c][i] = S1[c][i] = D2[c][i] = 0.f;

  for(int t = J.jbeg - 2; t <= J.jend; ++t)
  {
    float O[NC][8], E2[NC][8];
    fetch97<NC>(D, J, 2 * t + 1, O);
    fetch97<NC>(D, J, 2 * t + 2, E2);
    const bool emit = (t - 1) >= J.jbeg;
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      float lowrow[8], highrow[8];
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        const float d1 = fmaf(Ev[c][i] + E2[c][i], F97_ALPHA, O[c][i]);
        const float s1 = fmaf(D1[c][i] + d1, F97_BETA, Ev[c][i]);
        const float d2 = __fmul_rn(fmaf(S1[c][i] + s1, F97_GAMMA, D1[c][i]), F97_K);
        const float s2 = __fmul_rn(fmaf(D2[c][i] + d2, deltaS, S1[c][i]), invK);
        lowrow[i] = s2;
        highrow[i] = d2;
        if(J.hn == 1)
        { /* WaveletFwd.cpp L639-654; the values of pair t-1 are asked for, every row mirrors
             to the single real one */
          lowrow[i] = Ev[c][i];
          highrow[i] = __fmul_rn(O[c][i], 2.0f);
        }
        D2[c][i] = d2;
        D1[c][i] = d1;
        S1[c][i] = s1;
        Ev[c][i] = E2[c][i];
      }
      /* shuffles are executed by every lane on every iteration */
      int lo[4], hi[4];
      hfwd97(lowrow, J.wn, invK, deltaS, lo, hi);
      if(emit)
        store_rows(D, g, store_ctx(D, J, g), c, t - 1, false, lo, hi);
      hfwd97(highrow, J.wn, invK, deltaS, lo, hi);
      if(emit)
        store_rows(D, g, store_ctx(D, J, g), c, t - 1, true, lo, hi);
    }
  }
}

template <int NC>
__global__ void __launch_bounds__(B2K_WARPS_PER_CTA * 32) k_dwt97_fwd(const DwtLevelDesc* __restrict__ descs)
{
  extern __shared__ __align__(16) uint8_t smem_dwt[];
  typedef RowStage<NC> RS;
  const DwtLevelDesc D = descs[blockIdx.y]; /* by value */
  Job J;
  if(!decode_job<false>(D, J))
    return;
  if(J.hn == 1 || J.wn == 1)
  {
    fwd97_degenerate_job<NC>(descs + blockIdx.y, J);
    return;
  }
  const BandGeom g = band_geom(D);
  const StoreCtx SC = store_ctx(D, J, g);
  const bool fast = RS::lane_fast(D, J);
  const unsigned fastmask = __ballot_sync(0xffffffffu, fast);
  int mcol[8];
#pragma unroll
  for(int i = 0; i < 8; ++i)
    mcol[i] = mirror_rel(J.ulane - D.u0 + i, J.wn);
  const float invK = (float)(1.0 / 1.230174105);
  const float deltaS = __fmul_rn(F97_DELTA, invK);

  /* pairs t = jbeg-2 .. jend : rows (2t+1, 2t+2); output pair t-1 from t = jbeg+1 on.
     Interior strip: rows by bulk copy (TMA engine), see k_dwt53_fwd */
  const int tfirst = J.jbeg - 2, tlast = J.jend;
  WarpPipe<RS> pipe(smem_dwt, fastmask == 0xffffffffu, tfirst, tlast);
  auto fill_bulk = [&](uint8_t* st, int tf, uint64_t* bar) {
    RS::fill_bulk(st, 0, D, J, 2 * tf + 1, bar);
    RS::fill_bulk(st, 1, D, J, 2 * tf + 2, bar);
  };
  auto mc = [&](int i) { return mcol[i]; };
  auto fill_async = [&](uint8_t* st, int tf) {
    RS::fill(st, 0, D, J, 2 * tf + 1, fast, fastmask, mc);
    RS::fill(st, 1, D, J, 2 * tf + 2, fast, fastmask, mc);
  };
  pipe.prime(fill_bulk, fill_async);
  float Ev[NC][8], D1[NC][8], S1[NC][8], D2[NC][8];
  fetch97<NC>(D, J, 2 * tfirst, Ev);
#pragma unroll
  for(int c = 0; c < NC; ++c)
#pragma unroll
    for(int i = 0; i < 8; ++i)
      D1[c][i] = S1[c][i] = D2[c][i] = 0.f;

  for(int t = tfirst; t <= tlast; ++t)
  {
    const uint8_t* st = pipe.acquire(t, fill_bulk, fill_async);
    float O[NC][8], E2[NC][8];
    {
      int raw[NC][8];
      RS::read(st, 0, J, pipe.bulk, raw);
      to_coeffs97<NC>(D, raw, O);
      RS::read(st, 1, J, pipe.bulk, raw);
      to_coeffs97<NC>(D, raw, E2);
    }
    const bool emit = (t - 1) >= J.jbeg;
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      float lowrow[8], highrow[8];
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        const float d1 = fmaf(Ev[c][i] + E2[c][i], F97_ALPHA, O[c][i]);
        const float s1 = fmaf(D1[c][i] + d1, F97_BETA, Ev[c][i]);
        const float d2 = __fmul_rn(fmaf(S1[c][i] + s1, F97_GAMMA, D1[c][i]), F97_K);
        const float s2 = __fmul_rn(fmaf(D2[c][i] + d2, deltaS, S1[c][i]), invK);
        lowrow[i] = s2;
        highrow[i] = d2;
        D2[c][i] = d2;
        D1[c][i] = d1;
        S1[c][i] = s1;
        Ev[c][i] = E2[c][i];
      }
      if(emit)
      { /* warp-uniform */
        int lo[4], hi[4];
        hfwd97(lowrow, 2, invK, deltaS, lo, hi);
        store_rows(D, g, SC, c, t - 1, false, lo, hi);
        hfwd97(highrow, 2, invK, deltaS, lo, hi);
        store_rows(D, g, SC, c, t - 1, true, lo, hi);
      }
    }
  }
  pipe.drain();
}

/* =============================================================================================
 * inverse: descriptor roles swap -- out_ll / out_c are the SOURCE (LL and HL/LH/HH), in[] the
 * destination (interleaved samples of the next finer resolution, or the image at the finest).
 * =========================================================================================== */
template <int NC>
__device__ __forceinline__ void fetch_band_rows(const DwtLevelDesc& D, const Job& J, const BandGeom& g, int j,
                                                bool vhigh, int (&lo)[NC][4], int (&hi)[NC][4])
{
  /* vertical mirror in the interleaved domain */
  const int vm = D.v0 + mirror_rel(2 * j + (vhigh ? 1 : 0) - D.v0, J.hn);
  const int jm = vm >> 1;
  const int k0 = J.ulane >> 1;
#pragma unroll
  for(int c = 0; c < NC; ++c)
  {
    if(!J.need || (vm & 1) != (vhigh ? 1 : 0))
    {
#pragma unroll
      for(int i = 0; i < 4; ++i)
        lo[c][i] = hi[c][i] = 0;
      continue;
    }
    const int32_t* lrow;
    const int32_t* hrow;
    if(!vhigh)
    {
      lrow = reinterpret_cast<const int32_t*>(D.out_ll[c]) + (size_t)(jm - g.y0l) * D.ll_pitch;
      hrow = reinterpret_cast<const int32_t*>(D.out_c[c]) + (size_t)(jm - g.y0l) * D.c_pitch + g.snx;
    }
    else
    {
      lrow = reinterpret_cast<const int32_t*>(D.out_c[c]) + (size_t)(g.sny + jm - g.y0h) * D.c_pitch;
      hrow = lrow + g.snx;
    }
    load4_band(lrow, k0, g.x0l, D.u0, D.u1, 0, lo[c]);
    load4_band(hrow, k0, g.x0h, D.u0, D.u1, 1, hi[c]);
  }
}

/* ---- ghost samples of a whole-warp 5/3 strip (inverse) ------------------------------------------------------------------
 * Lane 0's synthesis needs the high-band sample at column x0-1, lane 31's the low-band sample at x0+256 and the high-band
 * sample at x0+257, from each of the two band-row pairs (LL|HL, LH|HH) of a row pair; mirrored addresses, as for the body.
 * `a`: the high-band sample's column in the row that holds HL (or HH) at snx; `b`: the low-band sample's column in the row
 * of LL (or LH).  a is lane 0's x0-1 and lane 31's x0+257, b is lane 31's x0+256; other lanes use neither. */
struct GhostBand
{
  int a, b;
};
__device__ __forceinline__ GhostBand ghost_band(const DwtLevelDesc& D, const Job& J, const BandGeom& g)
{
  const int x0 = J.ulane - 8 * J.lane;
  const int ua = J.lane == 0 ? x0 - 1 : J.lane == 31 ? x0 + 257 : J.ulane + 1;
  const int ub = J.lane == 31 ? x0 + 256 : J.ulane;
  /* symmetric extension keeps a column's parity (wn >= 2) */
  const int uam = D.u0 + mirror_rel(ua - D.u0, J.wn), ubm = D.u0 + mirror_rel(ub - D.u0, J.wn);
  GhostBand G;
  G.a = g.snx + (uam >> 1) - g.x0h;
  G.b = (ubm >> 1) - g.x0l;
  return G;
}
/* the lane's ghost samples of the band rows of pair j (vertical low or high), unstaged (degenerate jobs; a line one
   sample wide has no horizontal lifting and no ghosts) */
template <int NC>
__device__ __forceinline__ void fetch_band_ghosts(const DwtLevelDesc& D, const Job& J, const BandGeom& g, const GhostBand& G,
                                                  int j, bool vhigh, int (&ga)[NC], int (&gb)[NC])
{
  const int vm = D.v0 + mirror_rel(2 * j + (vhigh ? 1 : 0) - D.v0, J.hn);
  const int jm = vm >> 1;
#pragma unroll
  for(int c = 0; c < NC; ++c)
  {
    ga[c] = gb[c] = 0;
    if(J.wn == 1 || (vm & 1) != (vhigh ? 1 : 0))
      continue;
    const int32_t* lrow = !vhigh ? reinterpret_cast<const int32_t*>(D.out_ll[c]) + (size_t)(jm - g.y0l) * D.ll_pitch
                                 : reinterpret_cast<const int32_t*>(D.out_c[c]) + (size_t)(g.sny + jm - g.y0h) * D.c_pitch;
    const int32_t* hrow = !vhigh ? reinterpret_cast<const int32_t*>(D.out_c[c]) + (size_t)(jm - g.y0l) * D.c_pitch : lrow;
    ga[c] = __ldg(hrow + G.a);
    gb[c] = __ldg(lrow + G.b);
  }
}

/* inverse horizontal 5/3: WaveletReverse.cpp L879-1072.  ga, gb: the lane's ghost samples of the same band row pair (see
   GhostBand); lanes 0 and 31 take their outer neighbours from them by selects */
template <bool DEGEN = true>
__device__ __forceinline__ void hinv53(const int (&lo)[4], const int (&hi)[4], int ga, int gb, int wn, int (&r)[8])
{
  const int lane = threadIdx.x & 31;
  const int hp = __shfl_up_sync(0xffffffffu, hi[3], 1);
  const int dm = lane == 0 ? ga : hp;
  int e[5];
  e[0] = lo[0] - ((dm + hi[0] + 2) >> 2);
  e[1] = lo[1] - ((hi[0] + hi[1] + 2) >> 2);
  e[2] = lo[2] - ((hi[1] + hi[2] + 2) >> 2);
  e[3] = lo[3] - ((hi[2] + hi[3] + 2) >> 2);
  const int en = __shfl_down_sync(0xffffffffu, e[0], 1);
  e[4] = lane == 31 ? gb - ((hi[3] + ga + 2) >> 2) : en;
#pragma unroll
  for(int i = 0; i < 4; ++i)
  {
    r[2 * i] = e[i];
    r[2 * i + 1] = hi[i] + ((e[i] + e[i + 1]) >> 1);
  }
  if(DEGEN && wn == 1)
  {
#pragma unroll
    for(int i = 0; i < 4; ++i)
    {
      r[2 * i] = lo[i];
      r[2 * i + 1] = hi[i] >> 1;
    }
  }
}

/* inverse horizontal 9/7: WaveletReverse97.cpp L837-857, constants L98-103 */
__device__ __forceinline__ void hinv97(const int (&loi)[4], const int (&hii)[4], int wn, float (&r)[8])
{
  const float K = 1.230174105f, twice_invK = 1.625732422f;
  float s[5], d[4];
#pragma unroll
  for(int i = 0; i < 4; ++i)
  {
    s[i] = __fmul_rn(__int_as_float(loi[i]), K);
    d[i] = __fmul_rn(__int_as_float(hii[i]), twice_invK);
  }
  float dm = __shfl_up_sync(0xffffffffu, d[3], 1);
  s[0] = fmaf(dm + d[0], -0.443506852f, s[0]);
#pragma unroll
  for(int i = 1; i < 4; ++i)
    s[i] = fmaf(d[i - 1] + d[i], -0.443506852f, s[i]);
  s[4] = __shfl_down_sync(0xffffffffu, s[0], 1);
#pragma unroll
  for(int i = 0; i < 4; ++i)
    d[i] = fmaf(s[i] + s[i + 1], -0.882911075f, d[i]);
  dm = __shfl_up_sync(0xffffffffu, d[3], 1);
  s[0] = fmaf(dm + d[0], 0.052980118f, s[0]);
#pragma unroll
  for(int i = 1; i < 4; ++i)
    s[i] = fmaf(d[i - 1] + d[i], 0.052980118f, s[i]);
  s[4] = __shfl_down_sync(0xffffffffu, s[0], 1);
#pragma unroll
  for(int i = 0; i < 4; ++i)
  {
    r[2 * i] = s[i];
    r[2 * i + 1] = fmaf(s[i] + s[i + 1], 1.586134342f, d[i]);
  }
  if(wn == 1)
  {
#pragma unroll
    for(int i = 0; i < 4; ++i)
    {
      r[2 * i] = __int_as_float(loi[i]);
      r[2 * i + 1] = __int_as_float(hii[i]);
    }
  }
}

/* per-lane constants of the reconstructed-row stores */
struct OutCtx
{
  unsigned m;
  bool vec;
  int col;
};
__device__ __forceinline__ OutCtx out_ctx(const DwtLevelDesc& D, const Job& J)
{
  OutCtx o;
  o.m = 0;
  if(J.owner)
  {
#pragma unroll
    for(int i = 0; i < 8; ++i)
      if(J.ulane + i >= D.u0 && J.ulane + i < D.u1)
        o.m |= 1u << i;
  }
  o.col = J.ulane - D.u0;
  o.vec = o.m == 0xFF && (D.in_pitch & 3u) == 0 && (((reinterpret_cast<uintptr_t>(D.in[0]) >> 2) + (unsigned)o.col) & 3u) == 0;
  return o;
}
/* write one reconstructed row (canvas row v) of NC components, already in its output form */
template <int NC>
__device__ __forceinline__ void store_out_rows(const DwtLevelDesc& D, const OutCtx& O, int v, const int (&x)[NC][8])
{
#pragma unroll
  for(int c = 0; c < NC; ++c)
  {
    int32_t* p = reinterpret_cast<int32_t*>(const_cast<void*>(D.in[c])) + ((v - D.v0) * (int)D.in_pitch + O.col);
    if(O.vec)
    {
      reinterpret_cast<int4*>(p)[0] = make_int4(x[c][0], x[c][1], x[c][2], x[c][3]);
      reinterpret_cast<int4*>(p)[1] = make_int4(x[c][4], x[c][5], x[c][6], x[c][7]);
    }
    else
    {
#pragma unroll
      for(int i = 0; i < 8; ++i)
        if(O.m & (1u << i))
          p[i] = x[c][i];
    }
  }
}
/* 5/3: at the finest level the samples go through the inverse RCT + DC shift + clamp (in place) */
template <int NC>
__device__ __forceinline__ void store_rows53(const DwtLevelDesc& D, const OutCtx& O, int v, int (&x)[NC][8])
{
  if(v < D.v0 || v >= D.v1 || O.m == 0)
    return;
  if(D.first_level)
    rct_inv<NC>(D, x);
  store_out_rows<NC>(D, O, v, x);
}
/* 9/7: at the finest level inverse ICT + rounding + DC shift + clamp, elsewhere the float bits */
template <int NC>
__device__ __forceinline__ void store_rows97(const DwtLevelDesc& D, const OutCtx& O, int v, const float (&x)[NC][8])
{
  if(v < D.v0 || v >= D.v1 || O.m == 0)
    return;
  int o[NC][8];
  if(D.first_level)
    ict_inv<NC>(D, x, o);
  else
  {
#pragma unroll
    for(int c = 0; c < NC; ++c)
#pragma unroll
      for(int i = 0; i < 8; ++i)
        o[c][i] = __float_as_int(x[c][i]);
  }
  store_out_rows<NC>(D, O, v, o);
}

/* a resolution one sample wide or high: straightforward, unpipelined path (cold) */
template <int NC>
__device__ __noinline__ void inv53_degenerate_job(const DwtLevelDesc* __restrict__ dptr, const Job J)
{
  const DwtLevelDesc& D = *dptr;
  const BandGeom g = band_geom(D);
  const GhostBand G = ghost_band(D, J, g);
  int DV[NC][8], EP[NC][8];
#pragma unroll
  for(int c = 0; c < NC; ++c)
#pragma unroll
    for(int i = 0; i < 8; ++i)
      DV[c][i] = EP[c][i] = 0;

  for(int t = J.jbeg - 1; t <= J.jend; ++t)
  {
    int lo[NC][4], hi[NC][4], ga[NC], gb[NC];
    int sv[NC][8], dv[NC][8];
    fetch_band_rows<NC>(D, J, g, t, false, lo, hi);
    fetch_band_ghosts<NC>(D, J, g, G, t, false, ga, gb);
#pragma unroll
    for(int c = 0; c < NC; ++c)
      hinv53(lo[c], hi[c], ga[c], gb[c], J.wn, sv[c]);
    fetch_band_rows<NC>(D, J, g, t, true, lo, hi);
    fetch_band_ghosts<NC>(D, J, g, G, t, true, ga, gb);
#pragma unroll
    for(int c = 0; c < NC; ++c)
      hinv53(lo[c], hi[c], ga[c], gb[c], J.wn, dv[c]);
    int Er[NC][8], Or[NC][8];
#pragma unroll
    for(int c = 0; c < NC; ++c)
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        const int e = sv[c][i] - ((DV[c][i] + dv[c][i] + 2) >> 2);
        Or[c][i] = DV[c][i] + ((EP[c][i] + e) >> 1);
        Er[c][i] = EP[c][i];
        EP[c][i] = e;
        DV[c][i] = dv[c][i];
      }
    if(J.hn == 1)
    { /* single row: pair t holds it (low unchanged, lone high halved) */
      if(t >= J.jbeg && t < J.jend)
      {
        int hv[NC][8];
#pragma unroll
        for(int c = 0; c < NC; ++c)
#pragma unroll
          for(int i = 0; i < 8; ++i)
            hv[c][i] = dv[c][i] >> 1;
        store_rows53<NC>(D, out_ctx(D, J), 2 * t, sv);
        store_rows53<NC>(D, out_ctx(D, J), 2 * t + 1, hv);
      }
    }
    else if(t - 1 >= J.jbeg)
    {
      store_rows53<NC>(D, out_ctx(D, J), 2 * (t - 1), Er);
      store_rows53<NC>(D, out_ctx(D, J), 2 * (t - 1) + 1, Or);
    }
  }
}


/* staged band-row fetch for the inverse kernels: per row pair four band rows (LL|HL, LH|HH) x NC,
   each lane owning 4 consecutive samples (16 bytes) of each -> one cp.async per lane per band row,
   512 contiguous bytes per instruction, private slots (no barrier).
   WHOLE (whole-warp 5/3 strips): a 16-byte group per band-row pair and component follows the body, word 0 holding lane 0's
   ghost sample a, words 2, 3 lane 31's a and b (GhostBand); the mirrored columns of edge lanes are computed at the copy
   instead of being held in registers */
template <int NC, bool WHOLE = false>
struct BandStage
{
  static constexpr int ROWB = 512;
  static constexpr int BODYB = 4 * NC * ROWB;
  static constexpr bool GHOSTS = WHOLE;
  static constexpr int PAIRB = BODYB + (GHOSTS ? 2 * NC * 16 : 0);
  static constexpr bool COOPERATIVE = false;
  struct Lane
  {
    bool need;
    bool fast[4];   /* LL, HL, LH, HH source: 4 samples interior and 16-byte aligned */
    int col[4];     /* band-relative column of the lane's first sample (low, high) per source */
    int mlo[4], mhi[4]; /* mirrored band-relative columns for edge lanes (!WHOLE) */
  };
  /* mirrored band-relative column of the lane's low (odd = 0) or high (odd = 1) sample i */
  static __device__ __forceinline__ int mirrored(const DwtLevelDesc& D, const Job& J, const BandGeom& g, int i, int odd)
  {
    const int u = D.u0 + mirror_rel(2 * ((J.ulane >> 1) + i) + odd - D.u0, J.wn);
    return (u >> 1) - (odd ? g.x0h : g.x0l);
  }
  static __device__ __forceinline__ void setup(const DwtLevelDesc& D, const Job& J, const BandGeom& g, Lane& L)
  {
    const int k0 = J.ulane >> 1;
    L.need = J.need;
    if(!WHOLE)
    {
#pragma unroll
      for(int i = 0; i < 4; ++i)
      {
        L.mlo[i] = mirrored(D, J, g, i, 0);
        L.mhi[i] = mirrored(D, J, g, i, 1);
      }
    }
    const bool in_lo = 2 * k0 >= D.u0 && 2 * k0 + 6 < D.u1, in_hi = 2 * k0 + 1 >= D.u0 && 2 * k0 + 7 < D.u1;
    const int clo = k0 - g.x0l, chi = k0 - g.x0h;
    L.col[0] = clo; L.col[1] = g.snx + chi; L.col[2] = clo; L.col[3] = g.snx + chi;
    const bool pitch_ok = ((D.ll_pitch | D.c_pitch) & 3u) == 0;
    L.fast[0] = J.need && pitch_ok && in_lo && (((reinterpret_cast<uintptr_t>(D.out_ll[0]) >> 2) + (unsigned)clo) & 3u) == 0;
    L.fast[1] = J.need && pitch_ok && in_hi && (((reinterpret_cast<uintptr_t>(D.out_c[0]) >> 2) + (unsigned)(g.snx + chi)) & 3u) == 0;
    L.fast[2] = J.need && pitch_ok && in_lo && (((reinterpret_cast<uintptr_t>(D.out_c[0]) >> 2) + (unsigned)clo) & 3u) == 0;
    L.fast[3] = L.fast[1];
  }
  /* band rows of pair t into the stage */
  static __device__ __forceinline__ void fill(uint8_t* stage, const DwtLevelDesc& D, const Job& J, const BandGeom& g,
                                              const Lane& L, int t)
  {
    if(!L.need)
      return;
    const int jl = ((D.v0 + mirror_rel(2 * t - D.v0, J.hn)) >> 1), jh = ((D.v0 + mirror_rel(2 * t + 1 - D.v0, J.hn)) >> 1);
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      const int32_t* src[4];
      src[0] = reinterpret_cast<const int32_t*>(D.out_ll[c]) + (jl - g.y0l) * (int)D.ll_pitch;
      src[1] = reinterpret_cast<const int32_t*>(D.out_c[c]) + (jl - g.y0l) * (int)D.c_pitch;
      src[2] = reinterpret_cast<const int32_t*>(D.out_c[c]) + (g.sny + jh - g.y0h) * (int)D.c_pitch;
      src[3] = src[2];
#pragma unroll
      for(int b = 0; b < 4; ++b)
      {
        uint8_t* dst = stage + (b * NC + c) * ROWB + J.lane * 16;
        if(L.fast[b])
          cp_async16(dst, src[b] + L.col[b]);
        else
        {
          const int base = (b & 1) ? g.snx : 0;
#pragma unroll
          for(int i = 0; i < 4; ++i)
          {
            const int m = WHOLE ? mirrored(D, J, g, i, b & 1) : ((b & 1) ? L.mhi[i] : L.mlo[i]);
            cp_async4(dst + 4 * i, src[b] + base + m);
          }
        }
      }
    }
  }
  /* the ghost samples of pair t: lane 0's a, lane 31's a and b, of both band-row pairs */
  static __device__ __forceinline__ void fill_ghost(uint8_t* stage, const DwtLevelDesc& D, const Job& J, const BandGeom& g,
                                                    const GhostBand& G, int t)
  {
    static_assert(GHOSTS, "stage without ghost samples");
    const int jl = ((D.v0 + mirror_rel(2 * t - D.v0, J.hn)) >> 1), jh = ((D.v0 + mirror_rel(2 * t + 1 - D.v0, J.hn)) >> 1);
    const bool right = J.lane == 31, on = J.lane == 0 || right;
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      const int32_t* lsrc[2];
      const int32_t* hsrc[2];
      lsrc[0] = reinterpret_cast<const int32_t*>(D.out_ll[c]) + (jl - g.y0l) * (int)D.ll_pitch;
      hsrc[0] = reinterpret_cast<const int32_t*>(D.out_c[c]) + (jl - g.y0l) * (int)D.c_pitch;
      lsrc[1] = hsrc[1] = reinterpret_cast<const int32_t*>(D.out_c[c]) + (g.sny + jh - g.y0h) * (int)D.c_pitch;
#pragma unroll
      for(int v = 0; v < 2; ++v)
      {
        uint8_t* dst = stage + BODYB + (v * NC + c) * 16;
        if(on)
          cp_async4(dst + (right ? 8 : 0), hsrc[v] + G.a);
        if(right)
          cp_async4(dst + 12, lsrc[v] + G.b);
      }
    }
  }
  /* byte offset, relative to band-row pair 0, component 0, and stride per (band-row pair, component) of the lane's
     ghost samples; a lane without them reads two of its own body samples instead */
  static __device__ __forceinline__ int2 ghost_at(const Job& J)
  {
    return J.lane == 0 ? make_int2(BODYB, 16) : J.lane == 31 ? make_int2(BODYB + 8, 16) : make_int2(16 * J.lane, ROWB);
  }
  static __device__ __forceinline__ int2 read_ghost(const uint8_t* stage, int2 at, int v, int c)
  {
    return *reinterpret_cast<const int2*>(stage + at.x + (v * NC + c) * at.y);
  }
  /* bulk path: every lane of the warp is `fast` on all four sources, so each band row of the pair is 512 contiguous,
     16-byte aligned bytes starting at lane 0's column: lane 0 asks the copy engine (TMA, UBLKCP) for the 4 x NC rows,
     which land in the same linear layout the per-lane cp.async path writes and complete on `bar` */
  static __device__ __forceinline__ void fill_bulk(uint8_t* stage, const DwtLevelDesc& D, const Job& J, const BandGeom& g,
                                                   const Lane& L, int t, uint64_t* bar)
  {
    const int jl = ((D.v0 + mirror_rel(2 * t - D.v0, J.hn)) >> 1), jh = ((D.v0 + mirror_rel(2 * t + 1 - D.v0, J.hn)) >> 1);
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      const int32_t* src[4];
      src[0] = reinterpret_cast<const int32_t*>(D.out_ll[c]) + (jl - g.y0l) * (int)D.ll_pitch;
      src[1] = reinterpret_cast<const int32_t*>(D.out_c[c]) + (jl - g.y0l) * (int)D.c_pitch;
      src[2] = reinterpret_cast<const int32_t*>(D.out_c[c]) + (g.sny + jh - g.y0h) * (int)D.c_pitch;
      src[3] = src[2];
#pragma unroll
      for(int b = 0; b < 4; ++b)
        bulk_g2s(stage + (b * NC + c) * ROWB, src[b] + L.col[b], ROWB, bar);
    }
  }
  static __device__ __forceinline__ bool all_fast(const Lane& L)
  {
    return __all_sync(0xffffffffu, L.fast[0] && L.fast[1] && L.fast[2] && L.fast[3]);
  }
  static __device__ __forceinline__ void read(const uint8_t* stage, const Job& J, int b, int c, int (&v)[4])
  {
    const int4 a = *reinterpret_cast<const int4*>(stage + (b * NC + c) * ROWB + J.lane * 16);
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w;
  }
};

/* 3 CTAs per SM, as k_dwt53_fwd */
template <int NC>
__global__ void __launch_bounds__(B2K_WARPS_PER_CTA * 32, 3) k_dwt53_inv(const DwtLevelDesc* __restrict__ descs)
{
  extern __shared__ __align__(16) uint8_t smem_dwt[];
  typedef BandStage<NC, true> BS;
  const DwtLevelDesc D = descs[blockIdx.y]; /* by value: fields live in (uniform) registers */
  Job J;
  if(!decode_job<true>(D, J))
    return;
  if(J.hn == 1 || J.wn == 1)
  {
    inv53_degenerate_job<NC>(descs + blockIdx.y, J);
    return;
  }
  const BandGeom g = band_geom(D);
  typename BS::Lane L;
  BS::setup(D, J, g, L);
  const OutCtx OC = out_ctx(D, J);
  const GhostBand G = ghost_band(D, J, g);
  const int2 gat = BS::ghost_at(J);

  /* a strip whose band quads all lie inside the line and are 16-byte aligned: band rows by bulk copy (TMA engine) on
     per-slot mbarriers; the ghost samples always arrive by LDGSTS */
  const int tfirst = J.jbeg - 1, tlast = J.jend;
  WarpPipe<BS> pipe(smem_dwt, BS::all_fast(L), tfirst, tlast);
  auto fill_bulk = [&](uint8_t* st, int tf, uint64_t* bar) { BS::fill_bulk(st, D, J, g, L, tf, bar); };
  auto fill_async = [&](uint8_t* st, int tf) { BS::fill(st, D, J, g, L, tf); };
  auto fill_ghost = [&](uint8_t* st, int tf) { BS::fill_ghost(st, D, J, g, G, tf); };
  pipe.prime(fill_bulk, fill_async, fill_ghost);
  int DV[NC][8], EP[NC][8];
#pragma unroll
  for(int c = 0; c < NC; ++c)
#pragma unroll
    for(int i = 0; i < 8; ++i)
      DV[c][i] = EP[c][i] = 0;

  for(int t = tfirst; t <= tlast; ++t)
  {
    const uint8_t* st = pipe.acquire(t, fill_bulk, fill_async, fill_ghost);
    int Er[NC][8], Or[NC][8];
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      int lo[4], hi[4], sv[8], dv[8];
      BS::read(st, J, 0, c, lo);
      BS::read(st, J, 1, c, hi);
      int2 gh = BS::read_ghost(st, gat, 0, c);
      hinv53<false>(lo, hi, gh.x, gh.y, J.wn, sv);
      BS::read(st, J, 2, c, lo);
      BS::read(st, J, 3, c, hi);
      gh = BS::read_ghost(st, gat, 1, c);
      hinv53<false>(lo, hi, gh.x, gh.y, J.wn, dv);
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        const int e = sv[i] - ((DV[c][i] + dv[i] + 2) >> 2);
        Or[c][i] = DV[c][i] + ((EP[c][i] + e) >> 1);
        Er[c][i] = EP[c][i];
        EP[c][i] = e;
        DV[c][i] = dv[i];
      }
    }
    if(t - 1 >= J.jbeg)
    {
      store_rows53<NC>(D, OC, 2 * (t - 1), Er);
      store_rows53<NC>(D, OC, 2 * (t - 1) + 1, Or);
    }
  }
  pipe.drain();
}

/* unpipelined path for lines of one sample (cold) */
template <int NC>
__device__ __noinline__ void inv97_degenerate_job(const DwtLevelDesc* __restrict__ dptr, const Job J)
{
  const DwtLevelDesc& D = *dptr;
  const BandGeom g = band_geom(D);
  const float K = 1.230174105f, twice_invK = 1.625732422f;
  /* state: d0[t-1], s1[t-1], d1[t-2], s2[t-2] */
  float D0[NC][8], S1[NC][8], D1[NC][8], S2[NC][8];
#pragma unroll
  for(int c = 0; c < NC; ++c)
#pragma unroll
    for(int i = 0; i < 8; ++i)
      D0[c][i] = S1[c][i] = D1[c][i] = S2[c][i] = 0.f;

  for(int t = J.jbeg - 2; t <= J.jend + 1; ++t)
  {
    int lo[NC][4], hi[NC][4];
    float sv[NC][8], dv[NC][8];
    fetch_band_rows<NC>(D, J, g, t, false, lo, hi);
#pragma unroll
    for(int c = 0; c < NC; ++c)
      hinv97(lo[c], hi[c], J.wn, sv[c]);
    fetch_band_rows<NC>(D, J, g, t, true, lo, hi);
#pragma unroll
    for(int c = 0; c < NC; ++c)
      hinv97(lo[c], hi[c], J.wn, dv[c]);
    float Er[NC][8], Or[NC][8];
#pragma unroll
    for(int c = 0; c < NC; ++c)
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        const float s0 = __fmul_rn(sv[c][i], K), d0 = __fmul_rn(dv[c][i], twice_invK);
        const float s1 = fmaf(D0[c][i] + d0, -0.443506852f, s0);            /* s1[t]   */
        const float d1 = fmaf(S1[c][i] + s1, -0.882911075f, D0[c][i]);      /* d1[t-1] */
        const float s2 = fmaf(D1[c][i] + d1, 0.052980118f, S1[c][i]);       /* s2[t-1] */
        const float d2 = fmaf(S2[c][i] + s2, 1.586134342f, D1[c][i]);       /* d2[t-2] */
        Er[c][i] = S2[c][i];
        Or[c][i] = d2;
        D0[c][i] = d0;
        S1[c][i] = s1;
        D1[c][i] = d1;
        S2[c][i] = s2;
      }
    if(J.hn == 1)
    {
      if(t >= J.jbeg && t < J.jend)
      {
        store_rows97<NC>(D, out_ctx(D, J), 2 * t, sv);
        store_rows97<NC>(D, out_ctx(D, J), 2 * t + 1, dv);
      }
    }
    else if(t - 2 >= J.jbeg)
    {
      store_rows97<NC>(D, out_ctx(D, J), 2 * (t - 2), Er);
      store_rows97<NC>(D, out_ctx(D, J), 2 * (t - 2) + 1, Or);
    }
  }
}

template <int NC>
__global__ void __launch_bounds__(B2K_WARPS_PER_CTA * 32) k_dwt97_inv(const DwtLevelDesc* __restrict__ descs)
{
  extern __shared__ __align__(16) uint8_t smem_dwt[];
  typedef BandStage<NC> BS;
  const DwtLevelDesc D = descs[blockIdx.y]; /* by value */
  Job J;
  if(!decode_job<false>(D, J))
    return;
  if(J.hn == 1 || J.wn == 1)
  {
    inv97_degenerate_job<NC>(descs + blockIdx.y, J);
    return;
  }
  const BandGeom g = band_geom(D);
  typename BS::Lane L;
  BS::setup(D, J, g, L);
  const OutCtx OC = out_ctx(D, J);
  const float K = 1.230174105f, twice_invK = 1.625732422f;

  /* interior strip: band rows by bulk copy (TMA engine) on per-slot mbarriers */
  const int tfirst = J.jbeg - 2, tlast = J.jend + 1;
  WarpPipe<BS> pipe(smem_dwt, BS::all_fast(L), tfirst, tlast);
  auto fill_bulk = [&](uint8_t* st, int tf, uint64_t* bar) { BS::fill_bulk(st, D, J, g, L, tf, bar); };
  auto fill_async = [&](uint8_t* st, int tf) { BS::fill(st, D, J, g, L, tf); };
  pipe.prime(fill_bulk, fill_async);
  /* state: d0[t-1], s1[t-1], d1[t-2], s2[t-2] */
  float D0[NC][8], S1[NC][8], D1[NC][8], S2[NC][8];
#pragma unroll
  for(int c = 0; c < NC; ++c)
#pragma unroll
    for(int i = 0; i < 8; ++i)
      D0[c][i] = S1[c][i] = D1[c][i] = S2[c][i] = 0.f;

  for(int t = tfirst; t <= tlast; ++t)
  {
    const uint8_t* st = pipe.acquire(t, fill_bulk, fill_async);
    float Er[NC][8], Or[NC][8];
#pragma unroll
    for(int c = 0; c < NC; ++c)
    {
      int lo[4], hi[4];
      float sv[8], dv[8];
      BS::read(st, J, 0, c, lo);
      BS::read(st, J, 1, c, hi);
      hinv97(lo, hi, 2, sv);
      BS::read(st, J, 2, c, lo);
      BS::read(st, J, 3, c, hi);
      hinv97(lo, hi, 2, dv);
#pragma unroll
      for(int i = 0; i < 8; ++i)
      {
        const float s0 = __fmul_rn(sv[i], K), d0 = __fmul_rn(dv[i], twice_invK);
        const float s1 = fmaf(D0[c][i] + d0, -0.443506852f, s0);
        const float d1 = fmaf(S1[c][i] + s1, -0.882911075f, D0[c][i]);
        const float s2 = fmaf(D1[c][i] + d1, 0.052980118f, S1[c][i]);
        const float d2 = fmaf(S2[c][i] + s2, 1.586134342f, D1[c][i]);
        Er[c][i] = S2[c][i];
        Or[c][i] = d2;
        D0[c][i] = d0;
        S1[c][i] = s1;
        D1[c][i] = d1;
        S2[c][i] = s2;
      }
    }
    if(t - 2 >= J.jbeg)
    {
      store_rows97<NC>(D, OC, 2 * (t - 2), Er);
      store_rows97<NC>(D, OC, 2 * (t - 2) + 1, Or);
    }
  }
  pipe.drain();
}

/* ---- sample containers <-> the engine's 32-bit planes ----------------------------------------------------------------
   A container holds S-byte samples (S = 1, 2 or 4); component c of pixel (x, y) is at  base + y * pitch + x * step + c
   samples.  Planar containers (step 1) take one launch per component; NC components that sit side by side in every pixel
   take one launch together (step == NC: RGB / RGBA rows; step > NC: e.g. the RGB of an RGBA buffer).  One rectangle (a
   merged tile row) per launch, 8 pixels per thread.  When the thread's 8 pixels are whole, step == NC and the addresses
   are aligned, the container side moves as one group of 8 * NC * S bytes in 128-bit accesses (64-bit ones when the group
   is not a multiple of 16 bytes: 8-bit samples with NC odd) and every plane as two 128-bit accesses; anything else goes
   sample by sample.  HBM traffic is S + 4 bytes per sample, which bounds these kernels.
   Widening sign-extends from the container width when the samples are signed; narrowing truncates (the inverse
   transforms have already clamped to the precision). */
template <int S> struct Sample;
template <> struct Sample<1> { typedef uint8_t U; typedef int8_t I; };
template <> struct Sample<2> { typedef uint16_t U; typedef int16_t I; };
template <> struct Sample<4> { typedef uint32_t U; typedef int32_t I; };

template <int S>
__device__ __forceinline__ int widen_sample(uint32_t u, int sgnd)
{
  if constexpr(S == 4)
    return (int)u;
  else
  {
    u &= (1u << (8 * S)) - 1;
    return sgnd ? (int)(typename Sample<S>::I)u : (int)u;
  }
}

/* a group of BYTES bytes (a multiple of 8) as 32-bit words, in 128-bit pieces when BYTES allows, else 64-bit ones */
template <int BYTES>
__device__ __forceinline__ void load_group(const void* p, uint32_t (&wd)[BYTES / 4])
{
  if constexpr(BYTES % 16 == 0)
  {
#pragma unroll
    for(int i = 0; i < BYTES / 16; ++i)
    {
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(p) + i);
      wd[4 * i] = a.x; wd[4 * i + 1] = a.y; wd[4 * i + 2] = a.z; wd[4 * i + 3] = a.w;
    }
  }
  else
  {
#pragma unroll
    for(int i = 0; i < BYTES / 8; ++i)
    {
      const uint2 a = __ldg(reinterpret_cast<const uint2*>(p) + i);
      wd[2 * i] = a.x; wd[2 * i + 1] = a.y;
    }
  }
}
template <int BYTES>
__device__ __forceinline__ void store_group(void* p, const uint32_t (&wd)[BYTES / 4])
{
  if constexpr(BYTES % 16 == 0)
  {
#pragma unroll
    for(int i = 0; i < BYTES / 16; ++i)
      reinterpret_cast<uint4*>(p)[i] = make_uint4(wd[4 * i], wd[4 * i + 1], wd[4 * i + 2], wd[4 * i + 3]);
  }
  else
  {
#pragma unroll
    for(int i = 0; i < BYTES / 8; ++i)
      reinterpret_cast<uint2*>(p)[i] = make_uint2(wd[2 * i], wd[2 * i + 1]);
  }
}

struct Ptr4
{
  int32_t* p[4];
};
struct CPtr4
{
  const int32_t* p[4];
};

/* container -> NC int32 planes, the rows blockIdx.y + k gridDim.y of the 8 pixels at x8 (b2k_encode16 /
   b2k_encode16_interleaved after the upload, b2k_encode_device, and each image of a batch) */
template <int S, int NC, class Dst>
__device__ __forceinline__ void container_to_planes_rows(const void* __restrict__ src, uint32_t spitch, uint32_t step, const Dst& dst,
                                                         uint32_t dpitch, uint32_t w, uint32_t h, int sgnd, uint32_t x8)
{
  typedef typename Sample<S>::U U;
  constexpr int BYTES = 8 * NC * S, V = BYTES % 16 == 0 ? 16 : 8;
  for(uint32_t y = blockIdx.y; y < h; y += gridDim.y)
  {
    const U* s = static_cast<const U*>(src) + (size_t)y * spitch + (size_t)x8 * step;
    const size_t doff = (size_t)y * dpitch + x8;
    bool vec = x8 + 8 <= w && step == NC && (reinterpret_cast<uintptr_t>(s) & (V - 1)) == 0;
#pragma unroll
    for(int c = 0; c < NC; ++c)
      vec = vec && (reinterpret_cast<uintptr_t>(dst(c) + doff) & 15) == 0;
    if(vec)
    {
      uint32_t wd[BYTES / 4];
      load_group<BYTES>(s, wd);
#pragma unroll
      for(int c = 0; c < NC; ++c)
      {
        int v[8];
#pragma unroll
        for(int i = 0; i < 8; ++i)
        {
          const int e = (i * NC + c) * S; /* byte of the sample within the group */
          v[i] = widen_sample<S>(wd[e >> 2] >> ((e & 3) * 8), sgnd);
        }
        int4* d = reinterpret_cast<int4*>(dst(c) + doff);
        d[0] = make_int4(v[0], v[1], v[2], v[3]);
        d[1] = make_int4(v[4], v[5], v[6], v[7]);
      }
    }
    else
    { /* a row's last pixels, or an unaligned / strided container */
      const uint32_t n = w - x8 < 8 ? w - x8 : 8;
#pragma unroll 1
      for(uint32_t i = 0; i < n; ++i)
#pragma unroll
        for(int c = 0; c < NC; ++c)
          dst(c)[doff + i] = widen_sample<S>(s[(size_t)i * step + c], sgnd);
    }
  }
}

template <int S, int NC>
__global__ void __launch_bounds__(128) k_container_to_planes(const void* __restrict__ src, uint32_t spitch, uint32_t step, Ptr4 dst,
                                                             uint32_t dpitch, uint32_t w, uint32_t h, int sgnd)
{
  const uint32_t x8 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if(x8 >= w)
    return;
  container_to_planes_rows<S, NC>(src, spitch, step, [&](int c) { return dst.p[c]; }, dpitch, w, h, sgnd, x8);
}

/* the images of a batch into its planes: image blockIdx.z from its table entry */
template <int S, int NC>
__global__ void __launch_bounds__(128) k_containers_to_planes(const BatchSrc* __restrict__ tab, uint32_t dpitch, size_t dplane, uint32_t w,
                                                              uint32_t h, int sgnd)
{
  const uint32_t x8 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  const BatchSrc* E = tab + blockIdx.z;
  if(x8 >= w)
    return;
  int32_t* const dst = E->dst;
  container_to_planes_rows<S, NC>(E->src, E->spitch, E->step, [=](int c) { return dst + c * dplane; }, dpitch, w, h, sgnd, x8);
}

/* NC int32 planes -> container, the rows blockIdx.y + k gridDim.y of the 8 pixels at x8 (b2k_decode16 before the download,
   b2k_decode_device, and each image of a batch) */
template <int S, int NC, class Src>
__device__ __forceinline__ void planes_to_container_rows(const Src& src, uint32_t spitch, void* __restrict__ dst, uint32_t dpitch,
                                                         uint32_t step, uint32_t w, uint32_t h, uint32_t x8)
{
  typedef typename Sample<S>::U U;
  constexpr int BYTES = 8 * NC * S, V = BYTES % 16 == 0 ? 16 : 8;
  constexpr uint32_t MASK = S == 4 ? 0xFFFFFFFFu : (1u << (8 * S)) - 1;
  for(uint32_t y = blockIdx.y; y < h; y += gridDim.y)
  {
    const size_t soff = (size_t)y * spitch + x8;
    U* d = static_cast<U*>(dst) + (size_t)y * dpitch + (size_t)x8 * step;
    bool vec = x8 + 8 <= w && step == NC && (reinterpret_cast<uintptr_t>(d) & (V - 1)) == 0;
#pragma unroll
    for(int c = 0; c < NC; ++c)
      vec = vec && (reinterpret_cast<uintptr_t>(src(c) + soff) & 15) == 0;
    if(vec)
    {
      uint32_t wd[BYTES / 4];
#pragma unroll
      for(int k = 0; k < BYTES / 4; ++k)
        wd[k] = 0;
#pragma unroll
      for(int c = 0; c < NC; ++c)
      {
        const int4 a = __ldg(reinterpret_cast<const int4*>(src(c) + soff)), b = __ldg(reinterpret_cast<const int4*>(src(c) + soff) + 1);
        const int v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for(int i = 0; i < 8; ++i)
        {
          const int e = (i * NC + c) * S;
          wd[e >> 2] |= ((uint32_t)v[i] & MASK) << ((e & 3) * 8);
        }
      }
      store_group<BYTES>(d, wd);
    }
    else
    { /* a row's last pixels, or an unaligned / strided container */
      const uint32_t n = w - x8 < 8 ? w - x8 : 8;
#pragma unroll 1
      for(uint32_t i = 0; i < n; ++i)
#pragma unroll
        for(int c = 0; c < NC; ++c)
          d[(size_t)i * step + c] = (U)src(c)[soff + i];
    }
  }
}

template <int S, int NC>
__global__ void __launch_bounds__(128) k_planes_to_container(CPtr4 src, uint32_t spitch, void* __restrict__ dst, uint32_t dpitch,
                                                             uint32_t step, uint32_t w, uint32_t h)
{
  const uint32_t x8 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  if(x8 >= w)
    return;
  planes_to_container_rows<S, NC>([&](int c) { return src.p[c]; }, spitch, dst, dpitch, step, w, h, x8);
}

/* the images of a batch: image blockIdx.z from its table entry, at its own size within the grid of the largest; an entry
   without a destination, or with a counter (of the blocks of its slot the HT decoder rejected, earlier on the stream)
   that is not 0, is skipped */
template <int S, int NC>
__global__ void __launch_bounds__(128) k_planes_to_containers(const BatchDst* __restrict__ tab, uint32_t spitch)
{
  const uint32_t x8 = (blockIdx.x * blockDim.x + threadIdx.x) * 8;
  const BatchDst* E = tab + blockIdx.z;
  void* dst = E->dst;
  const uint32_t w = E->w;
  if(x8 >= w || !dst || (E->err && *E->err))
    return;
  /* the plane pointers are read from the table where they are used */
  planes_to_container_rows<S, NC>([E](int c) { return E->src[c]; }, spitch, dst, E->dpitch, E->step, w, E->h, x8);
}

dim3 convert_grid(uint32_t w, uint32_t h) { return dim3((w + 8 * 128 - 1) / (8 * 128), h < 65535u ? h : 65535u); }

template <int S>
void launch_container_to_planes(const void* src, uint32_t spitch, uint32_t step, const Ptr4& P, int nc, uint32_t dpitch, uint32_t w,
                                uint32_t h, int sgnd, cudaStream_t st)
{
  const dim3 grid = convert_grid(w, h), block(128);
  switch(nc)
  {
    case 1: k_container_to_planes<S, 1><<<grid, block, 0, st>>>(src, spitch, step, P, dpitch, w, h, sgnd); break;
    case 2: k_container_to_planes<S, 2><<<grid, block, 0, st>>>(src, spitch, step, P, dpitch, w, h, sgnd); break;
    case 3: k_container_to_planes<S, 3><<<grid, block, 0, st>>>(src, spitch, step, P, dpitch, w, h, sgnd); break;
    default: k_container_to_planes<S, 4><<<grid, block, 0, st>>>(src, spitch, step, P, dpitch, w, h, sgnd); break;
  }
}
template <int S>
void launch_planes_to_container(const CPtr4& P, int nc, uint32_t spitch, void* dst, uint32_t dpitch, uint32_t step, uint32_t w,
                                uint32_t h, cudaStream_t st)
{
  const dim3 grid = convert_grid(w, h), block(128);
  switch(nc)
  {
    case 1: k_planes_to_container<S, 1><<<grid, block, 0, st>>>(P, spitch, dst, dpitch, step, w, h); break;
    case 2: k_planes_to_container<S, 2><<<grid, block, 0, st>>>(P, spitch, dst, dpitch, step, w, h); break;
    case 3: k_planes_to_container<S, 3><<<grid, block, 0, st>>>(P, spitch, dst, dpitch, step, w, h); break;
    default: k_planes_to_container<S, 4><<<grid, block, 0, st>>>(P, spitch, dst, dpitch, step, w, h); break;
  }
}

} /* namespace */

void b2k_launch_container_to_planes(const void* src, uint32_t spitch, uint32_t step, uint32_t sample_bytes, int32_t* const* dst, int nc,
                                    uint32_t dpitch, uint32_t w, uint32_t h, int sgnd, cudaStream_t st)
{
  if(!w || !h)
    return;
  Ptr4 P{};
  for(int c = 0; c < nc && c < 4; ++c)
    P.p[c] = dst[c];
  switch(sample_bytes)
  {
    case 1: launch_container_to_planes<1>(src, spitch, step, P, nc, dpitch, w, h, sgnd, st); break;
    case 2: launch_container_to_planes<2>(src, spitch, step, P, nc, dpitch, w, h, sgnd, st); break;
    default: launch_container_to_planes<4>(src, spitch, step, P, nc, dpitch, w, h, sgnd, st); break;
  }
  b2k_count_launch();
}
void b2k_launch_planes_to_container(const int32_t* const* src, int nc, uint32_t spitch, void* dst, uint32_t dpitch, uint32_t step,
                                    uint32_t sample_bytes, uint32_t w, uint32_t h, cudaStream_t st)
{
  if(!w || !h)
    return;
  CPtr4 P{};
  for(int c = 0; c < nc && c < 4; ++c)
    P.p[c] = src[c];
  switch(sample_bytes)
  {
    case 1: launch_planes_to_container<1>(P, nc, spitch, dst, dpitch, step, w, h, st); break;
    case 2: launch_planes_to_container<2>(P, nc, spitch, dst, dpitch, step, w, h, st); break;
    default: launch_planes_to_container<4>(P, nc, spitch, dst, dpitch, step, w, h, st); break;
  }
  b2k_count_launch();
}

namespace
{
/* a batch conversion's grid: the rows of every image, enough CTAs for the GPU without a grid of 65535 x 65535 */
dim3 batch_grid(uint32_t n, uint32_t w, uint32_t h)
{
  dim3 grid = convert_grid(w, h);
  grid.y = std::min<uint32_t>(grid.y, std::max<uint32_t>(1u, 16384u / std::max(1u, n)));
  grid.y = std::min<uint32_t>(std::max<uint32_t>(grid.y, 8u), std::max(1u, h));
  return grid;
}

template <int S>
void launch_planes_to_containers(const BatchDst* d_dst, uint32_t n, int nc, uint32_t spitch, uint32_t w, uint32_t h, cudaStream_t st)
{
  dim3 grid = batch_grid(n, w, h);
  const dim3 block(128);
  for(uint32_t i0 = 0; i0 < n; i0 += 65535u) /* one launch below 65536 images */
  {
    grid.z = std::min<uint32_t>(n - i0, 65535u);
    switch(nc)
    {
      case 1: k_planes_to_containers<S, 1><<<grid, block, 0, st>>>(d_dst + i0, spitch); break;
      case 2: k_planes_to_containers<S, 2><<<grid, block, 0, st>>>(d_dst + i0, spitch); break;
      case 3: k_planes_to_containers<S, 3><<<grid, block, 0, st>>>(d_dst + i0, spitch); break;
      default: k_planes_to_containers<S, 4><<<grid, block, 0, st>>>(d_dst + i0, spitch); break;
    }
    b2k_count_launch();
  }
}

template <int S>
void launch_containers_to_planes(const BatchSrc* d_src, uint32_t n, int nc, uint32_t dpitch, size_t dplane, uint32_t w, uint32_t h,
                                 int sgnd, cudaStream_t st)
{
  dim3 grid = batch_grid(n, w, h);
  const dim3 block(128);
  for(uint32_t i0 = 0; i0 < n; i0 += 65535u)
  {
    grid.z = std::min<uint32_t>(n - i0, 65535u);
    switch(nc)
    {
      case 1: k_containers_to_planes<S, 1><<<grid, block, 0, st>>>(d_src + i0, dpitch, dplane, w, h, sgnd); break;
      case 2: k_containers_to_planes<S, 2><<<grid, block, 0, st>>>(d_src + i0, dpitch, dplane, w, h, sgnd); break;
      case 3: k_containers_to_planes<S, 3><<<grid, block, 0, st>>>(d_src + i0, dpitch, dplane, w, h, sgnd); break;
      default: k_containers_to_planes<S, 4><<<grid, block, 0, st>>>(d_src + i0, dpitch, dplane, w, h, sgnd); break;
    }
    b2k_count_launch();
  }
}
} // namespace

void b2k_launch_planes_to_containers(const BatchDst* d_dst, uint32_t n, int nc, uint32_t spitch, uint32_t sample_bytes, uint32_t w,
                                     uint32_t h, cudaStream_t st)
{
  if(!n || !w || !h)
    return;
  switch(sample_bytes)
  {
    case 1: launch_planes_to_containers<1>(d_dst, n, nc, spitch, w, h, st); break;
    case 2: launch_planes_to_containers<2>(d_dst, n, nc, spitch, w, h, st); break;
    default: launch_planes_to_containers<4>(d_dst, n, nc, spitch, w, h, st); break;
  }
}

void b2k_launch_containers_to_planes(const BatchSrc* d_src, uint32_t n, int nc, uint32_t dpitch, size_t dplane, uint32_t sample_bytes,
                                     uint32_t w, uint32_t h, int sgnd, cudaStream_t st)
{
  if(!n || !w || !h)
    return;
  switch(sample_bytes)
  {
    case 1: launch_containers_to_planes<1>(d_src, n, nc, dpitch, dplane, w, h, sgnd, st); break;
    case 2: launch_containers_to_planes<2>(d_src, n, nc, dpitch, dplane, w, h, sgnd, st); break;
    default: launch_containers_to_planes<4>(d_src, n, nc, dpitch, dplane, w, h, sgnd, st); break;
  }
}

/* one launch of a DWT kernel whose warps stage through WarpPipe<Stage>; the shared-memory limit it needs is raised once
   per device for each kernel */
template <class Stage, void (*KERNEL)(const DwtLevelDesc*)>
static void launch_dwt(dim3 grid, dim3 block, cudaStream_t st, const DwtLevelDesc* d)
{
  const size_t smem = WarpPipe<Stage>::SMEM_BYTES;
  static DeviceOnce once; /* function attributes are per device */
  once.run([&] { cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); });
  KERNEL<<<grid, block, smem, st>>>(d);
}

void b2k_launch_dwt_fwd(const DwtLevelDesc* d, int ndesc, int max_jobs, int nc, bool irreversible, cudaStream_t st)
{
  if(ndesc <= 0 || max_jobs <= 0)
    return;
  dim3 grid((max_jobs + B2K_WARPS_PER_CTA - 1) / B2K_WARPS_PER_CTA), block(B2K_WARPS_PER_CTA * 32);
  for(int d0 = 0; d0 < ndesc; d0 += 65535) /* descriptor blockIdx.y: one launch per 65535 of them */
  {
    grid.y = (unsigned)std::min(ndesc - d0, 65535);
    if(!irreversible)
    {
      if(nc == 3) launch_dwt<RowStage<3, true>, k_dwt53_fwd<3>>(grid, block, st, d + d0);
      else launch_dwt<RowStage<1, true>, k_dwt53_fwd<1>>(grid, block, st, d + d0);
    }
    else
    {
      if(nc == 3) launch_dwt<RowStage<3>, k_dwt97_fwd<3>>(grid, block, st, d + d0);
      else launch_dwt<RowStage<1>, k_dwt97_fwd<1>>(grid, block, st, d + d0);
    }
    b2k_count_launch();
  }
}

/* ---- tiles with NO wavelet level (numres = 1): what is left of the stage is the point transform -- DC shift + RCT / ICT
 * forwards, its inverse + rounding + clamp backwards (with one resolution the tile itself is the LL band,
 * TileProcessor.cpp L366-425).  The arithmetic is the level-1 kernels' own (rct_fwd / ict_fwd, rct_inv / ict_inv), one
 * sample per thread; the descriptors reuse DwtLevelDesc: in = image samples of the tile component(s), out_c = the tile's
 * place in the coefficient planes. */
template <int NC, bool IRREV, bool FWD>
__global__ void k_point_transform(const DwtLevelDesc* __restrict__ descs, int ndesc)
{
  for(int di = blockIdx.z; di < ndesc; di += gridDim.z)
  {
  const DwtLevelDesc& D = descs[di];
  const int w = D.u1 - D.u0, h = D.v1 - D.v0;
  const int x = blockIdx.x * blockDim.x + threadIdx.x;
  if(x >= w)
    continue;
  for(int y = blockIdx.y; y < h; y += gridDim.y)
  {
  const size_t ii = (size_t)y * D.in_pitch + x, oi = (size_t)y * D.c_pitch + x;
  if(FWD)
  {
    int v[NC][1];
#pragma unroll
    for(int c = 0; c < NC; ++c)
      v[c][0] = static_cast<const int32_t*>(D.in[c])[ii];
    if(!IRREV)
    {
      rct_fwd<NC>(D, v);
#pragma unroll
      for(int c = 0; c < NC; ++c)
        static_cast<int32_t*>(D.out_c[c])[oi] = v[c][0];
    }
    else
    {
      float f[NC][1];
      ict_fwd<NC>(D, v, f);
#pragma unroll
      for(int c = 0; c < NC; ++c)
        static_cast<float*>(D.out_c[c])[oi] = f[c][0];
    }
  }
  else
  {
    int o[NC][1];
    if(!IRREV)
    {
#pragma unroll
      for(int c = 0; c < NC; ++c)
        o[c][0] = static_cast<const int32_t*>(D.out_c[c])[oi];
      rct_inv<NC>(D, o);
    }
    else
    {
      float f[NC][1];
#pragma unroll
      for(int c = 0; c < NC; ++c)
        f[c][0] = static_cast<const float*>(D.out_c[c])[oi];
      ict_inv<NC>(D, f, o);
    }
#pragma unroll
    for(int c = 0; c < NC; ++c)
      static_cast<int32_t*>(const_cast<void*>(D.in[c]))[ii] = o[c][0];
  }
  } /* rows */
  } /* descriptors */
}

void b2k_launch_point_transform(const DwtLevelDesc* d, int ndesc, uint32_t max_w, uint32_t max_h, int nc, bool irreversible,
                                bool forward, cudaStream_t st)
{
  if(ndesc <= 0 || !max_w || !max_h)
    return;
  dim3 grid((max_w + 127) / 128, std::min<uint32_t>(max_h, 65535u), (unsigned)std::min(ndesc, 65535)), block(128);
#define B2K_PT(NC_, IR_, FW_) k_point_transform<NC_, IR_, FW_><<<grid, block, 0, st>>>(d, ndesc)
  if(nc == 3)
  {
    if(irreversible) { if(forward) B2K_PT(3, true, true); else B2K_PT(3, true, false); }
    else { if(forward) B2K_PT(3, false, true); else B2K_PT(3, false, false); }
  }
  else
  {
    if(irreversible) { if(forward) B2K_PT(1, true, true); else B2K_PT(1, true, false); }
    else { if(forward) B2K_PT(1, false, true); else B2K_PT(1, false, false); }
  }
#undef B2K_PT
  b2k_count_launch();
}

void b2k_launch_dwt_inv(const DwtLevelDesc* d, int ndesc, int max_jobs, int nc, bool irreversible, cudaStream_t st)
{
  if(ndesc <= 0 || max_jobs <= 0)
    return;
  dim3 grid((max_jobs + B2K_WARPS_PER_CTA - 1) / B2K_WARPS_PER_CTA), block(B2K_WARPS_PER_CTA * 32);
  for(int d0 = 0; d0 < ndesc; d0 += 65535) /* descriptor blockIdx.y: one launch per 65535 of them */
  {
    grid.y = (unsigned)std::min(ndesc - d0, 65535);
    if(!irreversible)
    {
      if(nc == 3) launch_dwt<BandStage<3, true>, k_dwt53_inv<3>>(grid, block, st, d + d0);
      else launch_dwt<BandStage<1, true>, k_dwt53_inv<1>>(grid, block, st, d + d0);
    }
    else
    {
      if(nc == 3) launch_dwt<BandStage<3>, k_dwt97_inv<3>>(grid, block, st, d + d0);
      else launch_dwt<BandStage<1>, k_dwt97_inv<1>>(grid, block, st, d + d0);
    }
    b2k_count_launch();
  }
}
