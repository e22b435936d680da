/*
 * grok_b200/csrc/ht_enc.cu -- HTJ2K (ITU-T T.814) cleanup-pass block ENCODER for sm_90a,
 * one warp per code block, fused with the T1 pre-processing (sign-magnitude conversion and,
 * for the irreversible path, scalar quantisation).
 *
 * Replaces (reference, CPU): T1OJPH::preCompress + compress   t1/part15/CoderOJPH.cpp L121-211
 *                            ojph_encode_codeblock32          t1/part15/coding/ojph_block_encoder.cpp L542-1017
 * Output is byte-identical to that encoder (tests/test_gpu.py against oracle/ and oracle/_ref,
 * tests/test_interop.py against the real library's code streams).
 *
 * The reference walks quads serially and pushes bits into three byte streams as it goes.  Nothing
 * about a quad depends on coding STATE, only on neighbouring SAMPLES (significance and exponents
 * of the quad to the left and of the sample row above).  So the block is cut into UNITS -- runs
 * of <= 8 consecutive quads of one quad row, in coding order -- and every lane codes one unit
 * by itself, start to end, with no cross-lane traffic at all:
 *   stage    the warp loads the sample rows of 32 units (coalesced 128-byte rows), converts them
 *            to magnitude/sign once and parks them in shared memory (odd pitch + a one-word skew
 *            per 32 columns: lanes walking different rows hit different banks);
 *   code     lane = unit: per quad pair rho / exponents / context / kappa / U_q / EMB, CxtVLC and
 *            U-VLC codewords; MagSgn and VLC bits are appended to the lane's own bit strings in
 *            shared memory through 64-bit register accumulators, MEL events to a lane bitmask;
 *   join     the 32 bit strings are concatenated in coding order into per-warp bit rings
 *            (funnel-shifted word copies, plain stores) and the rings are drained into the
 *            byte streams: 128 bytes per round for MagSgn, 32 for VLC, with the streams'
 *            bit-stuffing rules resolved by speculate-and-fix iterations on ballots (a stuffing
 *            event only shifts what follows by one bit, events are rare); the MEL run-length
 *            coder is inherently serial but tiny: every lane replays the event masks
 *            redundantly (uniform code).
 * Round 1 mapped lane = quad COLUMN and stepped over quad rows: a warp scan, two shared-memory
 * atomicOr scatters, four reductions and two drain checks per 32 quads -- 26.8 k warp instructions
 * per 64x64 block, issue-bound.  Per-unit coding amortises all of that over 16 quads per lane.
 */
#include <algorithm>
#include "b2k_internal.h"
#define HT_TABLE_QUAL static __device__ const
#include "ht_tables.h"

namespace {

#ifndef ENC_WARPS_N
#define ENC_WARPS_N 20
#endif
#ifndef ENC_MIN_CTAS
#define ENC_MIN_CTAS 1
#endif
/* warps (= code blocks in flight) per CTA, at most: ONE persistent CTA per SM.  For 64-wide blocks a warp needs 9.3 KB of
   shared memory and the CTA 8.3 KB of tables: 20 warps = 194 KB of the 227 KB a block may opt into on sm_90, so one CTA
   per SM, its tables loaded once (several smaller CTAs per SM would each carry a copy of the tables and leave the L1
   its minimum).  ENC_WARPS_N / ENC_MIN_CTAS let tools/build_variant.py build other shapes for A/B runs.  Launches with
   wider blocks (more shared memory per warp) run with fewer warps per CTA: the kernel takes its warp count from blockDim. */
constexpr int ENC_WARPS = ENC_WARPS_N;
constexpr int UNIT_QUADS = 8;       /* quads per unit (even: the VLC stream codes quads in pairs) */
constexpr int MS_RING_WORDS = 128;  /* 4096 bits: < 1024 left by the last drain + one 2048-bit gather batch */
constexpr int VLC_RING_WORDS = 64;  /* 2048 bits: < 256 left over + one 1024-bit gather batch */
constexpr int VLC_UNIT_WORDS = 5;   /* 4 pairs * <= 30 bits = 120 bits -> 4 words, + 1 so that the pitch is odd */
constexpr int OFFS_WORDS = 34;      /* exclusive prefix sums of the 32 units' string lengths + the total */
constexpr int MEL_CAP = 256;        /* reference buffer is 192 bytes (L555); more is an error there */

#ifdef ENC_PHASE_CLOCKS
/* ENC_PHASE_CLOCKS (tools/enc_phases.py builds it with tools/build_variant.py): every warp adds the clock64() cycles it
   spends in each phase of k_ht_encode to g_enc_phase.  Lane p keeps phase p's sum in one register, so the instrumented
   kernel needs two more 64-bit registers, not one per phase (some instances then spill 8 bytes; the product has no spills).  Slots past the phases: blocks coded, warp cycles from start
   to exit and the same span in %globaltimer nanoseconds (their ratio is the SM clock while the kernel runs). */
enum
{
  PH_SETUP, PH_STAGE, PH_CODE, PH_MEL, PH_SCAN, PH_MS, PH_VLC, PH_TERM, PH_N,
  PH_BLOCKS = PH_N, PH_WARP_CYCLES, PH_WARP_NS, PH_SLOTS
};
__device__ unsigned long long g_enc_phase[PH_SLOTS];
__device__ __forceinline__ unsigned long long enc_globaltimer()
{
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define PHASE_MARK(p)                                                          \
  do                                                                           \
  {                                                                            \
    const long long t_ = clock64();                                            \
    ph_acc += lane == (p) ? (unsigned long long)(t_ - ph_t) : 0ull;            \
    ph_t = t_;                                                                 \
  } while(0)
#else
#define PHASE_MARK(p) do {} while(0)
#endif

__device__ __forceinline__ unsigned lanemask_lt()
{
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

/* pulls the 128-byte lines of [p, p + bytes) into L2: no registers held, no shared memory, nothing waits for it.  A plain
   per-thread prefetch, one line per instruction, because lanes prefetch different rows: the bulk form
   (cp.async.bulk.prefetch.L2) takes a warp-uniform address, so per-lane rows compile to a loop over the lanes, and it
   measured slower (1.94 against 1.90 ms per encode of config 2, H100 80GB HBM3 at 400 W). */
__device__ __forceinline__ void prefetch_l2(const void* p, uint32_t bytes)
{
  const uintptr_t a = reinterpret_cast<uintptr_t>(p);
  for(uintptr_t l = a & ~(uintptr_t)127; l < a + bytes; l += 128)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(l) : "memory");
}

/* 15 bits starting at absolute bit position pos; bits at or beyond `tail` read as `fill`
   (MASK = false: the caller guarantees pos + 15 <= tail) */
template <bool MASK = true>
__device__ __forceinline__ uint32_t ring_get15(const uint32_t* ring, int ring_words, uint32_t pos, uint32_t tail,
                                               uint32_t fill)
{
  const uint32_t w = pos >> 5;
  const int sh = pos & 31;
  const uint32_t lo = ring[w & (ring_words - 1)], hi = ring[(w + 1) & (ring_words - 1)];
  uint32_t v = __funnelshift_r(lo, hi, sh) & 0x7FFFu;
  const int avail = (int)(tail - pos);
  if(MASK && avail < 15)
  {
    const uint32_t keep = avail <= 0 ? 0u : ((1u << avail) - 1u);
    v = (v & keep) | ((fill ? 0x7FFFu : 0u) & ~keep);
  }
  return v;
}

/* 64 bits of the concatenation of the units' bit strings, starting `rel` bits into it (rel < 0: the result's low
   -rel bits stay zero, they belong to the previous round); zeros beyond `total`.  offs[0..32] are the exclusive
   prefix sums of the string lengths, string u lives at scr + u * pitch (whole words; the word after its end may
   hold anything).  Lanes run this independently -- no cross-lane traffic. */
__device__ __forceinline__ uint64_t gather64(const uint32_t* scr, uint32_t pitch, const uint32_t* offs, int rel, uint32_t total)
{
  uint64_t out = 0;
  int filled = 0;
  if(rel < 0)
  {
    filled = -rel;
    rel = 0;
  }
  uint32_t p = (uint32_t)rel;
  if(p >= total)
    return 0ull;
  int u = 0;
#pragma unroll
  for(int s = 16; s; s >>= 1)
    if(offs[u + s] <= p)
      u += s;
  uint32_t o = offs[u], n = offs[u + 1];
  while(filled < 64 && p < total)
  {
    if(n <= p)
    { /* string exhausted (or empty): on to the next one */
      ++u;
      o = n;
      n = offs[u + 1];
      continue;
    }
    const uint32_t bit = p - o;
    const uint32_t* src = scr + (size_t)u * pitch + (bit >> 5);
    const uint32_t s0 = src[0], s1 = src[1], s2 = src[2]; /* may run past the string: masked by `take` */
    uint64_t v = (uint64_t)__funnelshift_r(s0, s1, bit & 31u) | ((uint64_t)__funnelshift_r(s1, s2, bit & 31u) << 32);
    const int take = min(64 - filled, (int)min(n - p, 64u));
    if(take < 64)
      v &= (1ull << take) - 1ull;
    out |= v << filled;
    filled += take;
    p += (uint32_t)take;
  }
  return out;
}

/* ---------------------------------------------------------------------------------------------
 * Drain up to 32 bytes of the forward MagSgn stream (ms_encode, ojph_block_encoder.cpp L470-491):
 * a byte following 0xFF carries 7 bits.  Returns number of bytes written.
 * final: pad the tail with 1s and emit the last partial byte too (ms_terminate L516-535; the
 * caller drops a trailing 0xFF).
 * ------------------------------------------------------------------------------------------- */
template <bool FINAL>
__device__ __forceinline__ int ms_drain32(uint32_t* ring, uint32_t& head, uint32_t tail, bool& last_ff, uint8_t* out,
                                          int lane, uint32_t& last_byte)
{
  const bool final = FINAL;
  unsigned ffmask = 0;
  uint32_t byte = 0, start = 0;
  int nbits = 8;
  for(int it = 0; it < 34; ++it)
  {
    /* lanes below i that produced 0xFF each shift everything after them by one bit */
    const unsigned prevff = (ffmask << 1) | (last_ff ? 1u : 0u); /* bit i: byte i-1 is 0xFF */
    nbits = ((prevff >> lane) & 1u) ? 7 : 8;
    const int stuffed_before = __popc(prevff & lanemask_lt()) ; /* 7-bit bytes among lanes < i */
    start = head + 8u * lane - (uint32_t)stuffed_before;
    /* non-final drains run with >= 256 bits queued, but lane 31's window can still poke past the tail */
    const uint32_t raw = ring_get15<true>(ring, MS_RING_WORDS, start, tail, 1u);
    byte = raw & (nbits == 7 ? 0x7Fu : 0xFFu);
    const unsigned nf = __ballot_sync(0xffffffffu, byte == 0xFFu);
    if(nf == ffmask)
      break;
    ffmask = nf;
  }
  /* complete bytes: all bits available, or (final) at least one real bit */
  const bool complete = final ? (start < tail) : (start + nbits <= tail);
  const unsigned cm = __ballot_sync(0xffffffffu, complete);
  const int nb = (cm == 0xffffffffu) ? 32 : (__ffs(~cm) - 1);
  if(lane < nb)
    out[lane] = (uint8_t)byte;
  /* advance */
  const uint32_t endpos = start + nbits;
  const uint32_t new_head = nb ? __shfl_sync(0xffffffffu, endpos, nb - 1) : head;
  if(nb)
  {
    last_byte = __shfl_sync(0xffffffffu, byte, nb - 1);
    last_ff = (last_byte == 0xFFu);
  }
  head = new_head;
  return nb;
}

/* ---------------------------------------------------------------------------------------------
 * Drain exactly 128 bytes of the forward MagSgn stream, 4 bytes per lane (requires >= 1024 raw bits
 * queued).  A lane walks its own four bytes serially (a byte after 0xFF carries 7 bits); how many
 * stuffed bytes sit in the lanes below -- which shifts the lane's window one bit each -- is
 * resolved with the same speculate-and-fix iteration on ballots as the 32-byte drain.
 * ------------------------------------------------------------------------------------------- */
__device__ __forceinline__ void ms_drain128(const uint32_t* ring, uint32_t& head, bool& last_ff, uint8_t* out, int lane)
{
  unsigned m1 = 0, m2 = 0, lf = 0; /* lanes with >=1 / >=2 seven-bit bytes; lanes whose 4th byte is 0xFF */
  uint32_t word = 0;
  for(int it = 0; it < 34; ++it)
  {
    const unsigned below = lanemask_lt();
    const uint32_t start = head + 32u * lane - (uint32_t)(__popc(m1 & below) + __popc(m2 & below));
    const bool pff = lane == 0 ? last_ff : (((lf >> (lane - 1)) & 1u) != 0);
    const uint32_t wi = start >> 5;
    const int sh = start & 31;
    uint32_t raw = __funnelshift_r(ring[wi & (MS_RING_WORDS - 1)], ring[(wi + 1) & (MS_RING_WORDS - 1)], sh);
    int sev = 0;
    bool f = pff;
    word = 0;
#pragma unroll
    for(int j = 0; j < 4; ++j)
    {
      const uint32_t b = raw & (f ? 0x7Fu : 0xFFu);
      raw >>= f ? 7 : 8;
      sev += f ? 1 : 0;
      f = (b == 0xFFu);
      word |= b << (8 * j);
    }
    const unsigned n1 = __ballot_sync(0xffffffffu, sev >= 1), n2 = __ballot_sync(0xffffffffu, sev >= 2),
                   nf = __ballot_sync(0xffffffffu, f);
    if(n1 == m1 && n2 == m2 && nf == lf)
      break;
    m1 = n1; m2 = n2; lf = nf;
  }
  /* the slot is 16-byte aligned and ms_out advances in multiples of 128 here */
  *reinterpret_cast<uint32_t*>(out + 4 * lane) = word;
  head += 1024u - (uint32_t)(__popc(m1) + __popc(m2));
  last_ff = (lf >> 31) & 1u;
}

/* ---------------------------------------------------------------------------------------------
 * Drain up to 32 bytes of the backward VLC stream (vlc_encode L378-410): a byte that follows one
 * > 0x8F and whose first 7 bits are all ones is emitted as 0x7F and carries 7 bits.  Only
 * complete bytes are written; byte k of the stream goes to out_last[-k].
 * ------------------------------------------------------------------------------------------- */
__device__ __forceinline__ int vlc_drain32(uint32_t* ring, uint32_t& head, uint32_t tail, uint32_t& prev_byte,
                                           uint8_t* out_first, int lane)
{
  unsigned smask = 0; /* bit i: byte i is a 7-bit (stuffed) byte */
  uint32_t byte = 0, start = 0;
  int nbits = 8;
  for(int it = 0; it < 34; ++it)
  {
    const int before = __popc(smask & lanemask_lt());
    start = head + 8u * lane - (uint32_t)before;
    const uint32_t raw = ring_get15(ring, VLC_RING_WORDS, start, tail, 0u);
    const uint32_t b8 = raw & 0xFFu;
    /* tentative value of the previous byte */
    uint32_t pb = __shfl_up_sync(0xffffffffu, byte, 1);
    if(lane == 0)
      pb = prev_byte;
    const bool stuffed = (pb > 0x8Fu) && ((raw & 0x7Fu) == 0x7Fu);
    nbits = stuffed ? 7 : 8;
    const uint32_t nbyte = stuffed ? 0x7Fu : b8;
    const unsigned ns = __ballot_sync(0xffffffffu, stuffed);
    const bool same = __all_sync(0xffffffffu, nbyte == byte) && ns == smask;
    byte = nbyte;
    smask = ns;
    if(same && it > 0)
      break;
  }
  const bool complete = start + nbits <= tail;
  const unsigned cm = __ballot_sync(0xffffffffu, complete);
  const int nb = (cm == 0xffffffffu) ? 32 : (__ffs(~cm) - 1);
  if(lane < nb)
    *(out_first - lane) = (uint8_t)byte;
  const uint32_t endpos = start + nbits;
  const uint32_t new_head = nb ? __shfl_sync(0xffffffffu, endpos, nb - 1) : head;
  if(nb)
    prev_byte = __shfl_sync(0xffffffffu, byte, nb - 1);
  head = new_head;
  return nb;
}

/* ---------------------------------------------------------------------------------------------
 * Drain exactly 128 bytes of the backward VLC stream, 4 bytes per lane (requires >= 1024 raw bits
 * queued).  A lane walks its four bytes serially; what it needs from the lanes below -- how many
 * of their bytes were stuffed (each shifts its window by one bit) and the value of the byte just
 * before its first one -- is speculated and fixed up on ballots / shuffles until nothing moves.
 * A stuffed byte is 0x7F, so two stuffed bytes are never adjacent: at most two per lane.
 * ------------------------------------------------------------------------------------------- */
__device__ __forceinline__ void vlc_drain128(const uint32_t* ring, uint32_t& head, uint32_t& prev_byte, uint8_t* out_first, int lane)
{
  unsigned m1 = 0, m2 = 0; /* lanes with >= 1 / >= 2 stuffed bytes */
  uint32_t word = 0, last = 0;
  for(int it = 0; it < 40; ++it)
  {
    const unsigned below = lanemask_lt();
    const uint32_t start = head + 32u * lane - (uint32_t)(__popc(m1 & below) + __popc(m2 & below));
    uint32_t pb = __shfl_up_sync(0xffffffffu, last, 1);
    if(lane == 0)
      pb = prev_byte;
    const uint32_t wi = start >> 5;
    const int sh = start & 31;
    uint32_t raw = __funnelshift_r(ring[wi & (VLC_RING_WORDS - 1)], ring[(wi + 1) & (VLC_RING_WORDS - 1)], sh);
    int st = 0;
    uint32_t nword = 0;
#pragma unroll
    for(int j = 0; j < 4; ++j)
    {
      const bool stuffed = (pb > 0x8Fu) && ((raw & 0x7Fu) == 0x7Fu);
      const uint32_t b = stuffed ? 0x7Fu : (raw & 0xFFu);
      raw >>= stuffed ? 7 : 8;
      st += stuffed ? 1 : 0;
      pb = b;
      nword |= b << (8 * j);
    }
    const unsigned n1 = __ballot_sync(0xffffffffu, st >= 1), n2 = __ballot_sync(0xffffffffu, st >= 2);
    const bool same = __all_sync(0xffffffffu, nword == word) && n1 == m1 && n2 == m2;
    word = nword;
    last = pb;
    m1 = n1;
    m2 = n2;
    if(same && it > 0)
      break;
  }
  uint8_t* o = out_first - 4 * lane; /* byte k of the stream lives at out_first[-k] */
  o[0] = (uint8_t)word;
  o[-1] = (uint8_t)(word >> 8);
  o[-2] = (uint8_t)(word >> 16);
  o[-3] = (uint8_t)(word >> 24);
  head += 1024u - (uint32_t)(__popc(m1) + __popc(m2));
  prev_byte = __shfl_sync(0xffffffffu, last, 31);
}

/* ---- MEL coder state (mel_struct, L273-345), identical in every lane ------------------------ */
struct Mel
{
  int rem, tmp, run, k, thr, pos;
};
__device__ __forceinline__ int mel_exp(int k) { return (int)((0x58da489200ull >> (3 * k)) & 7ull); }
/* exponents {0,0,0,1,1,1,2,2,2,3,3,4,5}: 3 bits each, k=0 lowest */

__device__ __forceinline__ void mel_emit(Mel& m, int v, uint8_t* buf, int lane)
{
  m.tmp = (m.tmp << 1) + v;
  if(--m.rem == 0)
  {
    if(lane == 0 && m.pos < MEL_CAP)
      buf[m.pos] = (uint8_t)m.tmp;
    m.pos++;
    m.rem = (m.tmp == 0xFF) ? 7 : 8;
    m.tmp = 0;
  }
}
__device__ __forceinline__ void mel_zeros(Mel& m, int n, uint8_t* buf, int lane)
{
  while(n > 0)
  {
    const int need = m.thr - m.run;
    if(n >= need)
    {
      mel_emit(m, 1, buf, lane);
      m.run = 0;
      m.k = min(12, m.k + 1);
      m.thr = 1 << mel_exp(m.k);
      n -= need;
    }
    else
    {
      m.run += n;
      n = 0;
    }
  }
}
__device__ __forceinline__ void mel_one(Mel& m, uint8_t* buf, int lane)
{
  mel_emit(m, 0, buf, lane);
  for(int t = mel_exp(m.k); t > 0;)
    mel_emit(m, (m.run >> --t) & 1, buf, lane);
  m.run = 0;
  m.k = max(0, m.k - 1);
  m.thr = 1 << mel_exp(m.k);
}

/* UVLC codeword (uvlc_tbl, L196-256): prefix[2:0] | prefix_len<<3 | suffix<<6 | suffix_len<<11 for
   u = 0..32 (u==0: nothing; 1: "1"; 2: "01"; 3,4: "001"+1 bit; 5..32: "000"+5 bits).  Copied to shared memory by
   the kernel: lanes look up different u, which a __constant__ bank would serialise. */
__device__ const uint16_t UVLC_LUT[34] = {0x0000, 0x0009, 0x0012, 0x081C, 0x085C, 0x2818, 0x2858, 0x2898, 0x28D8, 0x2918, 0x2958, 0x2998, 0x29D8, 0x2A18, 0x2A58, 0x2A98, 0x2AD8, 0x2B18, 0x2B58, 0x2B98, 0x2BD8, 0x2C18, 0x2C58, 0x2C98, 0x2CD8, 0x2D18, 0x2D58, 0x2D98, 0x2DD8, 0x2E18, 0x2E58, 0x2E98, 0x2ED8, 0x2ED8};

/* append n (<= 32) bits to a lane's bit string: 64-bit register accumulator, whole words to shared memory */
__device__ __forceinline__ void bits_put(uint64_t& acc, int& cnt, uint32_t*& wp, uint32_t bits, int n)
{
  acc |= (uint64_t)bits << cnt;
  cnt += n;
  if(cnt >= 32)
  {
    *wp++ = (uint32_t)acc;
    acc >>= 32;
    cnt -= 32;
  }
}

/* staged sample word: (mu << 1) | sign, 0 for an insignificant sample */
__device__ __forceinline__ int sm_exponent(uint32_t sm) { return sm ? 32 - __clz((sm & ~1u) - 1u) : 0; } /* 2*mu - 1 */
/* exponent / value of a staged word: with PACK the exponent sits in the top 6 bits */
#define SM_E(wd) (PACK ? (int)((wd) >> 26) : sm_exponent(wd))
#define SM_V(wd) (PACK ? ((wd) & 0x03FFFFFFu) : (wd))

/* shared-memory geometry of one launch (filled in by b2k_launch_ht_encode) */
struct EncLayout
{
  uint32_t stage_words; /* per warp: the staged sample rows of one round */
  uint32_t ms_w;        /* per lane: words of its MagSgn bit string (odd) */
};

__host__ __device__ inline uint32_t enc_stage_pitch(uint32_t w)
{ /* columns -1 .. w+4, one skew word per 32 columns, odd */
  const uint32_t c = w + 6;
  return (c + (c >> 5)) | 1u;
}
__host__ __device__ inline uint32_t enc_rows_per_round(uint32_t w)
{ /* quad rows whose units fill (at most) the 32 lanes */
  const uint32_t upr = (((w + 1) >> 1) + UNIT_QUADS - 1) / UNIT_QUADS;
  return upr >= 32 ? 1u : 32u / upr;
}

/* PACK: Kmax <= 24 in the whole launch, so a staged word has room for the sample's exponent in its top 6 bits
   (computed once, at staging, instead of by every lane that looks at the sample) */
template <bool IRREV, bool PACK>
__global__ void __launch_bounds__(ENC_WARPS * 32, ENC_MIN_CTAS)
    k_ht_encode(const HtBlockDesc* __restrict__ blocks, HtBlockOut* __restrict__ outs, uint8_t* __restrict__ scratch,
                uint32_t nblocks, EncLayout lay)
{
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint16_t* tbl0 = reinterpret_cast<uint16_t*>(smem_raw);
  uint16_t* tbl1 = tbl0 + 2048;
  uint16_t* uvlc = tbl1 + 2048; /* 34 entries, padded to 64 */
  const uint32_t warp_words = lay.stage_words + 32u * lay.ms_w + 32u * VLC_UNIT_WORDS + MS_RING_WORDS + VLC_RING_WORDS + MEL_CAP / 4 + 2 * OFFS_WORDS;
  uint32_t* warp_base = reinterpret_cast<uint32_t*>(smem_raw + 2 * 2048 * sizeof(uint16_t) + 64 * sizeof(uint16_t));

  for(int i = threadIdx.x; i < 2048; i += blockDim.x)
  {
    tbl0[i] = HT_ENC_VLC0[i];
    tbl1[i] = HT_ENC_VLC1[i];
  }
  if(threadIdx.x < 34)
    uvlc[threadIdx.x] = UVLC_LUT[threadIdx.x];
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#ifdef ENC_PHASE_CLOCKS
  unsigned long long ph_acc = 0;
  long long ph_t = clock64();
  const long long ph_c0 = ph_t;
  const unsigned long long ph_g0 = enc_globaltimer();
#endif
  uint32_t* stage = warp_base + (size_t)warp * warp_words;
  uint32_t* ms_scr = stage + lay.stage_words;
  uint32_t* vlc_scr = ms_scr + 32u * lay.ms_w;
  uint32_t* ms_ring = vlc_scr + 32u * VLC_UNIT_WORDS;
  uint32_t* vlc_ring = ms_ring + MS_RING_WORDS;
  uint8_t* mel_buf = reinterpret_cast<uint8_t*>(vlc_ring + VLC_RING_WORDS);
  uint32_t* offs_m = vlc_ring + VLC_RING_WORDS + MEL_CAP / 4; /* [0..32]: where unit u's MagSgn string starts in the round */
  uint32_t* offs_v = offs_m + OFFS_WORDS;

  /* persistent CTAs: the tables above are loaded once per CTA, each warp then walks the block list with a fixed stride
     (a work counter instead was measured and changes nothing: 1.524 against 1.529 ms on config 2) */
  const uint32_t cta_warps = blockDim.x >> 5;
  for(uint32_t bidx = blockIdx.x * cta_warps + warp; bidx < nblocks; bidx += gridDim.x * cta_warps)
  {
  const HtBlockDesc B = blocks[bidx];
  __syncwarp();
  const int w = B.w, h = B.h;
  const int nq = (w + 1) >> 1;
  const int kmax = B.kmax;
  const int shift = 30 - kmax; /* CoderOJPH.cpp L131: 31 - (k_msbs + 1) */
  const int upr = (nq + UNIT_QUADS - 1) / UNIT_QUADS; /* units per quad row */
  const int R = upr >= 32 ? 1 : 32 / upr;             /* quad rows staged together */
  const int P = (int)enc_stage_pitch((uint32_t)w);
  uint8_t* slot = scratch + B.slot_off;
  uint8_t* slot_last = slot + B.slot_cap - 1; /* VLC byte k lives at slot_last[-k] (vlc_init L364-375) */

  /* stream states */
  uint32_t ms_head = 0, ms_tail = 0, ms_out = 0, ms_lastbyte = 0;
  bool ms_lastff = false;
  uint32_t vlc_head = 0, vlc_tail = 4, vlc_out = 1, vlc_prev = 0xFF; /* 4 one-bits, virtual previous byte > 0x8F */
  if(lane == 0)
  {
    ms_ring[0] = 0;
    vlc_ring[0] = 0xF;
    vlc_ring[1] = 0;
    *slot_last = 0xFF;
  }
  Mel mel = {8, 0, 0, 0, 1, 0};
  /* guard columns (x = -1 and x = w .. w+4) of every staged row read as insignificant samples */
  for(int i = lane; i < (2 * R + 1) * 6; i += 32)
  {
    const int rr = i / 6, g = i % 6;
    const int c = g == 0 ? 0 : w + g; /* column + 1 */
    stage[rr * P + c + (c >> 5)] = 0;
  }
  const float fscale = (float)(1u << shift);
  const uint32_t mu_mask = (kmax >= 31) ? 0xFFFFFFFFu : ((1u << (kmax + 1)) - 1u);

  for(int y0 = 0; y0 < h; y0 += 2 * R)
  {
    /* ---- stage: sample rows y0-1 .. y0+2R-1, converted to (mu << 1) | sign --------------------------- */
    PHASE_MARK(PH_SETUP);
    /* the rows the warp stages next -- the next round's, or in the last round the first round's rows of the warp's next
       block -- are pulled into L2 (one row per lane) while this round is coded: without it the staging loads go to HBM
       and staging took 40 % of a warp's cycles (tools/enc_phases.py).  The next block's descriptor is read here, the
       prefetch issued after staging, so that the staging loads overlap its latency. */
    const uint8_t* pf_row = nullptr;
    uint32_t pf_bytes = 0;
    if(y0 + 2 * R < h)
    {
      const int gy = y0 + 2 * R + lane;
      if(lane < 2 * R && gy < h)
      {
        pf_row = static_cast<const uint8_t*>(B.coef) + (size_t)gy * B.pitch * 4u;
        pf_bytes = 4u * (uint32_t)w;
      }
    }
    else
    {
      const uint32_t nxt = bidx + gridDim.x * cta_warps;
      if(nxt < nblocks)
      {
        const HtBlockDesc* N = blocks + nxt;
        const uint32_t nw = N->w, nh = N->h;
        if(lane < 2 * (int)enc_rows_per_round(nw) && lane < (int)nh)
        {
          pf_row = static_cast<const uint8_t*>(N->coef) + (size_t)lane * N->pitch * 4u;
          pf_bytes = 4u * nw;
        }
      }
    }
    __syncwarp();
    {
      const uint32_t* cbase = reinterpret_cast<const uint32_t*>(B.coef);
      auto convert = [&](uint32_t raw) -> uint32_t {

        uint32_t mu, sgn;
        if(!IRREV)
        {
          const int32_t v = (int32_t)raw;
          sgn = (uint32_t)v >> 31;
          /* bits of |v| above Kmax are shifted out by the reference's `mag << shift; t + t` */
          mu = (uint32_t)(v < 0 ? -v : v) & mu_mask;
        }
        else
        { /* CoderOJPH.cpp L166-180 */
          const int32_t t = __float2int_rz(__fmul_rn(__fmul_rn(__uint_as_float(raw), B.quant), fscale));
          sgn = (uint32_t)t >> 31;
          const uint32_t m = (uint32_t)(t < 0 ? -t : t);
          mu = ((m + m) >> shift) >> 1;
        }
        /* branch-free: a zero sample stages as 0 (selected, not branched around) */
        const uint32_t sm = (mu << 1) | sgn;
        const uint32_t wd = PACK ? (((uint32_t)(32 - __clz((int)(2u * mu - 1u))) << 26) | sm) : sm;
        return mu ? wd : 0u;
      };
      const bool vec = (((reinterpret_cast<uintptr_t>(cbase) | ((uintptr_t)B.pitch << 2)) & 7u) == 0) && !(w & 1);
      if(vec)
      { /* 8-byte loads, six rows per trip in flight (17 staged rows of a 64-wide block = 3 trips, one load per lane
           and row) */
        for(int rr0 = 0; rr0 <= 2 * R; rr0 += 6)
          for(int x = 2 * lane; x < w; x += 64)
          {
            uint2 raw[6];
#pragma unroll
            for(int k = 0; k < 6; ++k)
            {
              const int gy = y0 - 1 + rr0 + k;
              const bool ok = rr0 + k <= 2 * R && gy >= 0 && gy < h;
              raw[k] = ok ? __ldg(reinterpret_cast<const uint2*>(cbase + (size_t)gy * B.pitch + x)) : make_uint2(0u, 0u);
            }
            const int c0 = x + 1, c1 = x + 2;
            uint32_t* d0 = stage + rr0 * P + c0 + (c0 >> 5);
            uint32_t* d1 = stage + rr0 * P + c1 + (c1 >> 5);
#pragma unroll
            for(int k = 0; k < 6; ++k)
            { /* rows past 2R land in the buffer's spare rows (b2k_ht_encode_stage_words) */
              d0[k * P] = convert(raw[k].x);
              d1[k * P] = convert(raw[k].y);
            }
          }
      }
      else
      {
        /* four rows per trip: their loads are in flight together */
        for(int rr0 = 0; rr0 <= 2 * R; rr0 += 4)
          for(int x = lane; x < w; x += 32)
          {
            uint32_t raw[4];
#pragma unroll
            for(int k = 0; k < 4; ++k)
            {
              const int gy = y0 - 1 + rr0 + k;
              const bool ok = rr0 + k <= 2 * R && gy >= 0 && gy < h;
              raw[k] = ok ? __ldg(cbase + (size_t)gy * B.pitch + x) : 0u; /* 0 converts to 0 on both paths */
            }
            const int c = x + 1;
            uint32_t* dst = stage + rr0 * P + c + (c >> 5);
#pragma unroll
            for(int k = 0; k < 4; ++k)
              if(rr0 + k <= 2 * R)
                dst[k * P] = convert(raw[k]);
          }
      }
    }
    __syncwarp();
    if(pf_row)
      prefetch_l2(pf_row, pf_bytes);
    PHASE_MARK(PH_STAGE);

    /* ---- code: lane = unit; the staged rows hold R * upr units, 32 at a time (more than one trip only for
       blocks wider than 32 units, where R = 1) ------------------------------------------------------------ */
    for(int ub = 0; ub < R * upr; ub += 32)
    {
    const int unit = ub + lane;
    const int r_local = unit / upr, seg = unit - r_local * upr;
    const int y = y0 + 2 * r_local;
    const bool unit_ok = r_local < R && y < h;
    const int q0 = seg * UNIT_QUADS, q1 = min(nq, q0 + UNIT_QUADS);
    uint32_t* const ms_base = ms_scr + (size_t)lane * lay.ms_w;
    uint32_t* const vlc_base = vlc_scr + (size_t)lane * VLC_UNIT_WORDS;
    uint32_t mlen = 0, vlen = 0, mel_has = 0, mel_val = 0;
    if(unit_ok)
    {
      const bool first_row = (y == 0);
      const uint16_t* tbl = first_row ? tbl0 : tbl1;
      const uint32_t* r0 = stage + (1 + 2 * r_local) * P; /* sample row y; r0 - P = row above, r0 + P = row y + 1 */
      uint64_t macc = 0, vacc = 0;
      int mcnt = 0, vcnt = 0;
      uint32_t *mwp = ms_base, *vwp = vlc_base;
      /* quad to the left of the unit: its significance pattern */
      int rho_left = 0;
      int ea_m1 = 0, ea_0 = 0; /* exponents of the row above at columns x-1 and x */
      {
        const int x = 2 * q0;
        if(q0 > 0)
        {
          const int c0 = x - 1, c1 = x; /* (column + 1) of x-2 and x-1 */
          const int s0 = c0 + (c0 >> 5), s1 = c1 + (c1 >> 5);
          rho_left = (r0[s0] ? 1 : 0) | (r0[s0 + P] ? 2 : 0) | (r0[s1] ? 4 : 0) | (r0[s1 + P] ? 8 : 0);
        }
        if(!first_row)
        {
          const int c0 = x, c1 = x + 1; /* (column + 1) of x-1 and x */
          ea_m1 = SM_E(r0[c0 + (c0 >> 5) - P]);
          ea_0 = SM_E(r0[c1 + (c1 >> 5) - P]);
        }
      }
      for(int qa = q0, p = 0; qa < q1; qa += 2, ++p)
      {
        const int x = 2 * qa;
        const bool hasB = qa + 1 < q1;
        int sx[5];
#pragma unroll
        for(int k = 0; k < 5; ++k)
        {
          const int c = x + 1 + k;
          sx[k] = c + (c >> 5);
        }
        uint32_t sa[4], sb[4]; /* quad A: (x,y) (x,y+1) (x+1,y) (x+1,y+1); quad B two columns on */
        sa[0] = r0[sx[0]]; sa[1] = r0[sx[0] + P]; sa[2] = r0[sx[1]]; sa[3] = r0[sx[1] + P];
        sb[0] = r0[sx[2]]; sb[1] = r0[sx[2] + P]; sb[2] = r0[sx[3]]; sb[3] = r0[sx[3] + P];
        int ea1 = 0, ea2 = 0, ea3 = 0, ea4 = 0;
        if(!first_row)
        {
          ea1 = SM_E(r0[sx[1] - P]);
          ea2 = SM_E(r0[sx[2] - P]);
          ea3 = SM_E(r0[sx[3] - P]);
          ea4 = SM_E(r0[sx[4] - P]);
        }
        int uq2[2];
        uint32_t cw[2];
        int cwl[2];
#pragma unroll
        for(int j = 0; j < 2; ++j)
        {
          const uint32_t* sq = j ? sb : sa;
          const bool qv = j ? hasB : true;
          int rho = 0, emax = 0;
          int e[4];
#pragma unroll
          for(int i = 0; i < 4; ++i)
          {
            e[i] = SM_E(sq[i]);
            rho |= sq[i] ? (1 << i) : 0;
            emax = max(emax, e[i]);
          }
          /* ---- context and kappa (L731, L788, L799-802, L862-878, L950-967) ---- */
          const int em1 = j ? ea1 : ea_m1, e0 = j ? ea2 : ea_0, e1 = j ? ea3 : ea1, e2 = j ? ea4 : ea2;
          const int cq_first = (rho_left >> 1) | (rho_left & 1);
          const int cq_rest = ((em1 | e0) ? 1 : 0) | ((rho_left & 0xC) ? 2 : 0) | ((e1 | e2) ? 4 : 0);
          const int cq = first_row ? cq_first : cq_rest;
          const int max_e = max(max(em1, e0), max(e1, e2)) - 1;
          const int kappa = (!first_row && (rho & (rho - 1))) ? max(1, max_e) : 1;
          const int Uq = max(emax, kappa);
          const int uq = Uq - kappa;
          int eps = 0;
#pragma unroll
          for(int i = 0; i < 4; ++i)
            eps |= (e[i] == emax) << i;
          eps = uq > 0 ? eps : 0;
          const uint32_t tuple = qv ? (uint32_t)tbl[(cq << 8) + (rho << 4) + eps] : 0u;
          cw[j] = tuple >> 8;
          cwl[j] = (tuple >> 4) & 7;
          uq2[j] = qv ? uq : 0;
          /* ---- MagSgn bits (L667-674, L886-893): U_q - e_k low bits of 2(mu-1)+sign ---- */
#pragma unroll
          for(int i = 0; i < 4; ++i)
          {
            /* unconditional append: an insignificant (or absent) sample adds zero bits */
            const bool on = qv && sq[i] != 0;
            const int m = on ? Uq - (int)((tuple >> i) & 1u) : 0;
            bits_put(macc, mcnt, mwp, (SM_V(sq[i]) - 2u) & (m >= 32 ? 0xFFFFFFFFu : ((1u << m) - 1u)), m);
          }
          /* ---- MEL event of the quad (L664-665, L883-884) ---- */
          if(qv && cq == 0)
          {
            mel_has |= 1u << (3 * p + j);
            mel_val |= (rho ? 1u : 0u) << (3 * p + j);
          }
          if(qv)
            rho_left = rho;
        }
        ea_m1 = ea3;
        ea_0 = ea4;
        /* ---- VLC bits of the quad pair: cwd0 cwd1 prefix0 prefix1 suffix0 suffix1 (L750-785, L985-988) ---- */
        {
          const int u0 = uq2[0], u1 = uq2[1];
          const bool both2 = first_row && u0 > 2 && u1 > 2;
          const bool one2 = first_row && !both2 && u0 > 2 && u1 > 0;
          if(first_row && u0 > 0 && u1 > 0)
          {
            mel_has |= 1u << (3 * p + 2);
            mel_val |= (min(u0, u1) > 2 ? 1u : 0u) << (3 * p + 2);
          }
          const uint32_t t0 = uvlc[both2 ? u0 - 2 : min(u0, 33)], t1 = uvlc[both2 ? u1 - 2 : min(u1, 33)];
          uint32_t p0 = t0 & 7u, s0 = (t0 >> 6) & 31u, p1 = t1 & 7u, s1 = (t1 >> 6) & 31u;
          int pl0 = (int)((t0 >> 3) & 7u), sl0 = (int)(t0 >> 11), pl1 = (int)((t1 >> 3) & 7u), sl1 = (int)(t1 >> 11);
          if(one2)
          { /* u1 in {1, 2}: one bit */
            p1 = (uint32_t)(u1 - 1);
            pl1 = 1;
            s1 = 0;
            sl1 = 0;
          }
          uint32_t vb = cw[0];
          int vl = cwl[0];
          vb |= cw[1] << vl; vl += cwl[1];
          vb |= p0 << vl; vl += pl0;
          vb |= p1 << vl; vl += pl1;
          vb |= s0 << vl; vl += sl0;
          vb |= s1 << vl; vl += sl1;
          bits_put(vacc, vcnt, vwp, vb, vl);
        }
      }
      mlen = 32u * (uint32_t)(mwp - ms_base) + (uint32_t)mcnt;
      vlen = 32u * (uint32_t)(vwp - vlc_base) + (uint32_t)vcnt;
      if(mcnt)
        *mwp = (uint32_t)macc;
      if(vcnt)
        *vwp = (uint32_t)vacc;
    }
    __syncwarp();
    PHASE_MARK(PH_CODE);

    /* ---- join: MEL events, unit by unit in coding order: quad 2p, quad 2p+1, pair p ---- */
    if(__any_sync(0xffffffffu, mel_has != 0))
    {
      for(int u = 0; u < 32; ++u)
      {
        uint32_t has = __shfl_sync(0xffffffffu, mel_has, u);
        const uint32_t val = __shfl_sync(0xffffffffu, mel_val, u);
        while(has)
        {
          const uint32_t ones = has & val;
          if(ones == 0)
          {
            mel_zeros(mel, __popc(has), mel_buf, lane);
            break;
          }
          const int b = __ffs((int)ones) - 1;
          mel_zeros(mel, __popc(has & ((1u << b) - 1u)), mel_buf, lane);
          mel_one(mel, mel_buf, lane);
          has &= ~((2u << b) - 1u);
        }
      }
    }
    PHASE_MARK(PH_MEL);
    /* ---- join: where each unit's strings start (one scan for both: MagSgn < 2^17 bits per round, VLC < 2^14) ---- */
    {
      uint32_t x = mlen | (vlen << 17);
#pragma unroll
      for(int o = 1; o < 32; o <<= 1)
      {
        const uint32_t t = __shfl_up_sync(0xffffffffu, x, o);
        if(lane >= o)
          x += t;
      }
      const uint32_t ex = x - (mlen | (vlen << 17));
      offs_m[lane] = ex & 0x1FFFFu;
      offs_v[lane] = ex >> 17;
      if(lane == 31)
      {
        offs_m[32] = x & 0x1FFFFu;
        offs_v[32] = x >> 17;
      }
    }
    __syncwarp();
    PHASE_MARK(PH_SCAN);
    /* ---- join: MagSgn.  64 ring words (2048 bits) are gathered from the units' strings at a time, two words per
       lane, and 128 bytes leave whenever 1024 bits are queued. ---- */
    {
      const uint32_t total = offs_m[32], t0 = ms_tail;
      ms_tail += total;
      for(uint32_t wb = t0 >> 5; (wb << 5) < ms_tail; wb += 64)
      {
        const uint32_t W = wb + 2u * lane;
        if((W << 5) < ms_tail)
        {
          const int rel = (int)(W << 5) - (int)t0;
          uint64_t v = gather64(ms_scr, lay.ms_w, offs_m, rel, total);
          if(rel < 0)
            v |= ms_ring[W & (MS_RING_WORDS - 1)] & ((1u << (t0 & 31u)) - 1u);
          ms_ring[W & (MS_RING_WORDS - 1)] = (uint32_t)v;
          ms_ring[(W + 1) & (MS_RING_WORDS - 1)] = (uint32_t)(v >> 32);
        }
        __syncwarp();
        const uint32_t have = min(ms_tail, (wb + 64u) << 5);
        while(have - ms_head >= 1024u)
        {
          ms_drain128(ms_ring, ms_head, ms_lastff, slot + ms_out, lane);
          ms_out += 128u;
        }
        __syncwarp();
      }
    }
    PHASE_MARK(PH_MS);
    /* ---- join: VLC, 128 bytes out when 1024 bits are queued, else 32 whenever 256 are ---- */
    {
      const uint32_t total = offs_v[32], t0 = vlc_tail;
      vlc_tail += total;
      for(uint32_t wb = t0 >> 5; (wb << 5) < vlc_tail; wb += 32)
      {
        const uint32_t W = wb + 2u * lane;
        if(lane < 16 && (W << 5) < vlc_tail)
        {
          const int rel = (int)(W << 5) - (int)t0;
          uint64_t v = gather64(vlc_scr, VLC_UNIT_WORDS, offs_v, rel, total);
          if(rel < 0)
            v |= vlc_ring[W & (VLC_RING_WORDS - 1)] & ((1u << (t0 & 31u)) - 1u);
          vlc_ring[W & (VLC_RING_WORDS - 1)] = (uint32_t)v;
          vlc_ring[(W + 1) & (VLC_RING_WORDS - 1)] = (uint32_t)(v >> 32);
        }
        __syncwarp();
        const uint32_t have = min(vlc_tail, (wb + 32u) << 5);
        while(have - vlc_head >= 1024u)
        {
          vlc_drain128(vlc_ring, vlc_head, vlc_prev, slot_last - vlc_out, lane);
          vlc_out += 128u;
        }
        while(have - vlc_head >= 256u)
          vlc_out += (uint32_t)vlc_drain32(vlc_ring, vlc_head, have, vlc_prev, slot_last - vlc_out, lane);
        __syncwarp();
      }
    }
    PHASE_MARK(PH_VLC);
    } /* unit trips */
  }

  /* ---- terminate MagSgn (ms_terminate L516-535) ---- */
  while(ms_head < ms_tail)
    ms_out += (uint32_t)ms_drain32<true>(ms_ring, ms_head, ms_tail, ms_lastff, slot + ms_out, lane, ms_lastbyte);
  if(ms_out > 0 && ms_lastff)
    ms_out--; /* a final 0xFF is not written (padded partial byte) or is taken back (L533-534) */

  /* ---- VLC: flush complete bytes, keep the partial one for the MEL/VLC fusion ---- */
  for(;;)
  {
    const int n = vlc_drain32(vlc_ring, vlc_head, vlc_tail, vlc_prev, slot_last - vlc_out, lane);
    vlc_out += (uint32_t)n;
    if(n < 32)
      break;
  }
  const int vused = (int)(vlc_tail - vlc_head);
  const int vtmp = (int)ring_get15(vlc_ring, VLC_RING_WORDS, vlc_head, vlc_tail, 0u) & 0xFF;

  /* ---- terminate_mel_vlc (L412-444) ---- */
  if(mel.run > 0)
    mel_emit(mel, 1, mel_buf, lane);
  {
    const int mtmp = (mel.tmp << mel.rem) & 0xFFFF;
    const int mel_mask = (0xFF << mel.rem) & 0xFF;
    const int vlc_mask = vused ? (0xFF >> (8 - vused)) : 0;
    if((mel_mask | vlc_mask) != 0)
    {
      const int fuse = mtmp | vtmp;
      if(((((fuse ^ mtmp) & mel_mask) | ((fuse ^ vtmp) & vlc_mask)) == 0) && fuse != 0xFF && vlc_out > 1)
      {
        if(lane == 0 && mel.pos < MEL_CAP)
          mel_buf[mel.pos] = (uint8_t)fuse;
        mel.pos++;
      }
      else
      {
        if(lane == 0 && mel.pos < MEL_CAP)
          mel_buf[mel.pos] = (uint8_t)mtmp;
        mel.pos++;
        if(lane == 0)
          *(slot_last - vlc_out) = (uint8_t)vtmp;
        vlc_out++;
      }
    }
  }
  __syncwarp();
  /* MEL bytes follow the MagSgn bytes */
  for(int i = lane; i < mel.pos && i < MEL_CAP; i += 32)
    slot[ms_out + i] = mel_buf[i];
  /* interface locator word (L1009-1014) */
  const uint32_t scup = (uint32_t)mel.pos + vlc_out;
  __syncwarp();
  if(lane == 0)
  {
    slot_last[0] = (uint8_t)(scup >> 4);
    slot_last[-1] = (uint8_t)((slot_last[-1] & 0xF0) | (scup & 0xF));
    HtBlockOut o;
    o.ms_len = ms_out;
    o.mel_len = (uint32_t)mel.pos;
    o.vlc_len = vlc_out;
    o.total = ms_out + (uint32_t)mel.pos + vlc_out;
    if(mel.pos > 192 || o.total > B.slot_cap)
      o.total = 0xFFFFFFFFu; /* the reference raises "mel encoder's buffer is full" here */
    outs[bidx] = o;
  }
  PHASE_MARK(PH_TERM);
#ifdef ENC_PHASE_CLOCKS
  ph_acc += lane == PH_BLOCKS ? 1ull : 0ull;
#endif
  } /* block loop */
#ifdef ENC_PHASE_CLOCKS
  const unsigned long long ph_cycles = (unsigned long long)(clock64() - ph_c0), ph_ns = enc_globaltimer() - ph_g0;
  ph_acc += lane == PH_WARP_CYCLES ? ph_cycles : lane == PH_WARP_NS ? ph_ns : 0ull;
  if(lane < PH_SLOTS)
    atomicAdd(&g_enc_phase[lane], ph_acc);
#endif
}

/* lengths -> exclusive byte offsets.  One CTA of 1024 threads, SCAN_ITEMS consecutive blocks per thread and round:
   thread-local sums, a shuffle scan inside each warp, one more over the 32 warp totals; ~5e4 blocks take 7 rounds.
   offsets[0] is the running base: 0 for the first range, the previous range's end otherwise. */
constexpr int SCAN_ITEMS = 8;
__global__ void __launch_bounds__(1024) k_scan_lengths(const HtBlockOut* __restrict__ outs, uint64_t* __restrict__ offsets, uint32_t n)
{
  __shared__ uint64_t warp_sum[32];
  __shared__ uint64_t carry_s;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if(threadIdx.x == 0)
    carry_s = offsets[0];
  __syncthreads();
  for(uint32_t base = 0; base < n; base += 1024 * SCAN_ITEMS)
  {
    const uint32_t i0 = base + threadIdx.x * SCAN_ITEMS;
    uint32_t v[SCAN_ITEMS];
    uint64_t local = 0;
#pragma unroll
    for(int k = 0; k < SCAN_ITEMS; ++k)
    {
      uint32_t t = 0;
      if(i0 + k < n)
      {
        t = outs[i0 + k].total;
        t = (t == 0xFFFFFFFFu) ? 0u : t;
      }
      v[k] = t;
      local += t;
    }
    uint64_t incl = local;
#pragma unroll
    for(int o = 1; o < 32; o <<= 1)
    {
      const uint64_t y = __shfl_up_sync(0xffffffffu, incl, o);
      if(lane >= o)
        incl += y;
    }
    if(lane == 31)
      warp_sum[warp] = incl;
    const uint64_t carry = carry_s;
    __syncthreads();
    if(warp == 0)
    {
      uint64_t w = warp_sum[lane], wi = w;
#pragma unroll
      for(int o = 1; o < 32; o <<= 1)
      {
        const uint64_t y = __shfl_up_sync(0xffffffffu, wi, o);
        if(lane >= o)
          wi += y;
      }
      warp_sum[lane] = wi - w; /* exclusive */
      if(lane == 31)
        carry_s = carry + wi;
    }
    __syncthreads();
    uint64_t at = carry + warp_sum[warp] + (incl - local);
#pragma unroll
    for(int k = 0; k < SCAN_ITEMS; ++k)
      if(i0 + k < n)
      {
        offsets[i0 + k] = at;
        at += v[k];
      }
    __syncthreads(); /* warp_sum and carry_s are rewritten by the next round */
  }
  if(threadIdx.x == 0)
    offsets[n] = carry_s;
}

/* byte j of a block's coded bytes: MagSgn|MEL (slot[0, front)) followed by VLC (vsrc[0, ...)) */
__device__ __forceinline__ uint32_t coded_byte(const uint8_t* slot, const uint8_t* vsrc, uint32_t front, uint32_t j)
{
  return j < front ? slot[j] : vsrc[j - front];
}

/* bytes j .. j+3 of the same, little-endian.  Inside one of the two pieces: the two aligned words that hold them, funnel-
   shifted (both words hold at least one of the four bytes, so neither read leaves the piece's words); across the seam,
   byte by byte. */
__device__ __forceinline__ uint32_t coded_word(const uint8_t* slot, const uint8_t* vsrc, uint32_t front, uint32_t j)
{
  if(j + 4u <= front || j >= front)
  {
    const uintptr_t a = reinterpret_cast<uintptr_t>(j >= front ? vsrc + (j - front) : slot + j);
    const uint32_t* p = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t sh = (uint32_t)(a & 3u);
    const uint32_t lo = p[0];
    return sh ? __funnelshift_r(lo, p[1], 8u * sh) : lo;
  }
  uint32_t v = 0;
#pragma unroll
  for(int k = 0; k < 4; ++k)
    v |= coded_byte(slot, vsrc, front, j + k) << (8 * k);
  return v;
}

/* compaction: MagSgn|MEL from the slot head, VLC from the slot tail (warp per block).  The destination's whole 4-byte words
   are written as words, four per lane in flight (byte-wide copies left the kernel bound by load latency); the up to three
   bytes at each end share their words with the neighbouring blocks and are written as bytes. */
constexpr int GATHER_UNROLL = 4;
__global__ void k_ht_gather(const HtBlockDesc* __restrict__ blocks, const HtBlockOut* __restrict__ outs,
                            const uint64_t* __restrict__ offsets, const uint8_t* __restrict__ scratch,
                            uint8_t* __restrict__ bytes, uint32_t nblocks, uint64_t cap)
{
  const uint32_t bidx = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if(bidx >= nblocks)
    return;
  const HtBlockOut o = outs[bidx];
  if(o.total == 0xFFFFFFFFu || offsets[bidx] + o.total > cap)
    return; /* arena too small: the host notices from the offsets and re-gathers */
  const uint8_t* slot = scratch + blocks[bidx].slot_off;
  uint8_t* dst = bytes + offsets[bidx];
  const uint32_t front = o.ms_len + o.mel_len, total = front + o.vlc_len;
  const uint8_t* vsrc = slot + blocks[bidx].slot_cap - o.vlc_len;
  const uint32_t head = (uint32_t)(-reinterpret_cast<uintptr_t>(dst) & 3u); /* bytes before the first whole word */
  if(total < head + 4u)
  {
    for(uint32_t i = lane; i < total; i += 32)
      dst[i] = (uint8_t)coded_byte(slot, vsrc, front, i);
    return;
  }
  const uint32_t words = (total - head) >> 2, tail0 = head + 4u * words;
  if((uint32_t)lane < head)
    dst[lane] = (uint8_t)coded_byte(slot, vsrc, front, lane);
  if((uint32_t)lane < total - tail0)
    dst[tail0 + lane] = (uint8_t)coded_byte(slot, vsrc, front, tail0 + lane);
  uint32_t* dw = reinterpret_cast<uint32_t*>(dst + head);
  for(uint32_t w0 = lane; w0 < words; w0 += 32 * GATHER_UNROLL)
  {
    uint32_t v[GATHER_UNROLL];
#pragma unroll
    for(int k = 0; k < GATHER_UNROLL; ++k)
    {
      const uint32_t w = w0 + 32u * k;
      v[k] = w < words ? coded_word(slot, vsrc, front, head + 4u * w) : 0u;
    }
#pragma unroll
    for(int k = 0; k < GATHER_UNROLL; ++k)
      if(w0 + 32u * k < words)
        dw[w0 + 32u * k] = v[k];
  }
}

} /* namespace */

void b2k_launch_ht_encode(const HtBlockDesc* d_blocks, HtBlockOut* d_out, uint8_t* d_scratch, uint32_t nblocks,
                          const HtEncodeLimits& lim, bool irreversible, cudaStream_t st)
{
  if(!nblocks)
    return;
  EncLayout lay;
  lay.stage_words = lim.stage_words;
  /* a unit's MagSgn string: 4 * UNIT_QUADS samples of <= kmax + 2 bits each (m = U_q - e_k, U_q <= kmax + 2) */
  const uint32_t bits = 4u * UNIT_QUADS * std::min<uint32_t>(32u, lim.max_kmax + 2u);
  lay.ms_w = ((bits + 31u) / 32u) | 1u; /* odd pitch: lanes storing word k of their strings hit 32 different banks */
  const uint32_t warp_words = lay.stage_words + 32u * lay.ms_w + 32u * VLC_UNIT_WORDS + MS_RING_WORDS + VLC_RING_WORDS + MEL_CAP / 4 + 2 * OFFS_WORDS;
  const size_t table_bytes = 2 * 2048 * sizeof(uint16_t) + 64 * sizeof(uint16_t), smem_max = 227 * 1024;
  /* as many warps per CTA as the opt-in maximum of shared memory holds */
  uint32_t cta_warps = (uint32_t)std::max<size_t>(1, std::min<size_t>(ENC_WARPS, (smem_max - table_bytes) / (warp_words * sizeof(uint32_t))));
  int dev = 0, sms = 132, per_sm = 1;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if(nblocks < (uint32_t)sms * cta_warps) /* a small launch: fewer warps per CTA, every SM still gets one */
    cta_warps = std::max(1u, (nblocks + (uint32_t)sms - 1u) / (uint32_t)sms);
  const size_t smem = table_bytes + (size_t)cta_warps * warp_words * sizeof(uint32_t);
  typedef void (*Kernel)(const HtBlockDesc*, HtBlockOut*, uint8_t*, uint32_t, EncLayout);
  const Kernel variants[4] = {k_ht_encode<false, false>, k_ht_encode<false, true>, k_ht_encode<true, false>, k_ht_encode<true, true>};
  static DeviceOnce once; /* function attributes are per device */
  once.run([&] {
    for(Kernel k : variants)
    {
      cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024); /* the opt-in maximum of sm_90 */
      /* the kernel lives on shared memory (staged samples, per-lane bit strings): without this hint the driver may
         size the carve-out for fewer CTAs per SM than fit */
      cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    }
  });
  const Kernel kern = variants[(irreversible ? 2 : 0) + (lim.max_kmax <= 24 ? 1 : 0)];
  /* persistent grid: as many CTAs as fit on the device at once (the tables are loaded once per CTA) */
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, (int)cta_warps * 32, smem);
  const uint32_t want = (nblocks + cta_warps - 1) / cta_warps;
  const uint32_t grid = std::min<uint32_t>(want, (uint32_t)(sms * std::max(per_sm, 1)));
  kern<<<grid, cta_warps * 32, smem, st>>>(d_blocks, d_out, d_scratch, nblocks, lay);
  b2k_count_launch();
}

#ifdef ENC_PHASE_CLOCKS
/* copies up to n of the ENC_PHASE_CLOCKS counters (layout: the PH_ enum) to out, zeroes them, returns how many there are */
extern "C" B2K_API int32_t b2k_enc_phase_clocks(uint64_t* out, int32_t n)
{
  unsigned long long h[PH_SLOTS] = {};
  if(cudaMemcpyFromSymbol(h, g_enc_phase, sizeof(h)) != cudaSuccess)
    return -1;
  const unsigned long long zero[PH_SLOTS] = {};
  if(cudaMemcpyToSymbol(g_enc_phase, zero, sizeof(zero)) != cudaSuccess)
    return -1;
  for(int i = 0; i < n && i < PH_SLOTS; ++i)
    out[i] = h[i];
  return PH_SLOTS;
}
#endif

/* words of shared memory one warp needs to stage the sample rows of one round of a w-wide block */
uint32_t b2k_ht_encode_stage_words(uint32_t w)
{
  /* rows rounded up to the six of a staging trip: the trip's stores need no row test (the spare rows are never read) */
  return ((2u * enc_rows_per_round(w) + 1u + 5u) / 6u) * 6u * enc_stage_pitch(w);
}

void b2k_launch_scan_lengths(const HtBlockOut* d_out, uint64_t* d_offsets, uint32_t nblocks, cudaStream_t st)
{
  k_scan_lengths<<<1, 1024, 0, st>>>(d_out, d_offsets, nblocks);
  b2k_count_launch();
}

void b2k_launch_ht_gather(const HtBlockDesc* d_blocks, const HtBlockOut* d_out, const uint64_t* d_offsets,
                          const uint8_t* d_scratch, uint8_t* d_bytes, uint32_t nblocks, uint64_t cap, cudaStream_t st)
{
  if(!nblocks)
    return;
  const uint32_t threads = 256, wpb = threads / 32;
  k_ht_gather<<<(nblocks + wpb - 1) / wpb, threads, 0, st>>>(d_blocks, d_out, d_offsets, d_scratch, d_bytes, nblocks, cap);
  b2k_count_launch();
}
