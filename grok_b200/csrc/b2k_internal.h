/*
 * grok_b200/csrc/b2k_internal.h -- structures shared by the host engine and the CUDA kernels.
 * Product code: must not include anything under oracle/.
 */
#pragma once
#include <stdint.h>
#include <stddef.h>
#include <atomic>
#include <functional>
#include <cuda_runtime.h>
#include "../../include/grok_b200.h"

#define B2K_WARPS_PER_CTA 4

/* Runs `f` once per CUDA device (the device current at the call): cudaFuncSetAttribute settings belong to the
 * device, and one process may hold engines on several GPUs.  Threads racing on the first call may both run `f`
 * (the settings are idempotent); nobody launches before his own call to `f` has returned. */
struct DeviceOnce
{
  std::atomic<uint64_t> done{0};
  template <class F> void run(F&& f)
  {
    int dev = 0;
    cudaGetDevice(&dev);
    const uint64_t bit = 1ull << (dev & 63);
    if(!(done.load(std::memory_order_acquire) & bit))
    {
      f();
      done.fetch_or(bit, std::memory_order_release);
    }
  }
};
#define B2K_MAX_RES 33

/* ---- one DWT level of one tile-component (or of the 3 colour components together) ---------
 * All coordinates are canvas coordinates of the resolution being split (reference:
 * WaveletFwd.cpp L1398-1407: rw/rh/parity from currentRes).  Pointers are pre-offset so that
 * in[c] addresses the sample at canvas (u0,v0). */
struct DwtLevelDesc
{
  const void* in[3];   /* input planes (level 1: image samples; else previous LL) */
  void* out_c[3];      /* Mallat buffer of the tile component: element (0,0) of the tile */
  void* out_ll[3];     /* where the LL sample (ceil(u0/2), ceil(v0/2)) is stored */
  uint32_t in_pitch, c_pitch, ll_pitch; /* in elements */
  int32_t u0, v0, u1, v1;
  int32_t shift[3];    /* value ADDED to the samples on load at level 1 (= -2^(prec-1)) */
  int32_t lo[3], hi[3];/* inverse: clamp range after the shift is restored */
  uint16_t nstrips, nsegs, strip_w, pairs_per_seg;
  uint8_t first_level; /* 1: samples are integers from the image (apply shift / MCT) */
  uint8_t comp0;       /* first component this descriptor covers */
  uint8_t pad[2];
};

/* ---- one code block for the HT coder kernels ------------------------------------------------
 * reference: t1/BlockExec.h L62-153 (CompressBlockExec / DecompressBlockExec) */
struct HtBlockDesc
{
  void* coef;          /* first sample of the block inside the Mallat buffer */
  uint32_t pitch;      /* buffer row pitch in elements */
  uint16_t w, h;
  uint8_t kmax;        /* band maxBitPlanes_ == missing_msbs handed to the encoder */
  uint8_t irreversible;
  uint8_t mmsbs;       /* decode: missing MSBs = Kmax - numbps (DecompressScheduler.cpp L261-263) */
  uint8_t passes;      /* decode: 1 cleanup only, 2 + SigProp, 3 + SigProp + MagRef */
  float quant;         /* encode: inv_step_ht * 2^(30-kmax); decode: stepsize / 2^(31-kmax) */
  uint32_t slot_cap;   /* bytes reserved in the scratch slot */
  uint64_t slot_off;   /* byte offset of the scratch slot (encode) / of the coded bytes (decode) */
  uint32_t length;     /* decode: coded length */
  uint32_t rec_off;    /* decode: first entry of this block in the per-quad record scratch */
  uint32_t length2;    /* decode: bytes of the refinement segment that follows the cleanup segment */
};
static_assert(sizeof(HtBlockDesc) == 56, "HtBlockDesc layout");

struct HtBlockOut /* written by the encoder kernel */
{
  uint32_t ms_len, mel_len, vlc_len, total;
};

/* kernel launchers (dwt.cu, ht_enc.cu, ht_dec.cu) */
void b2k_launch_dwt_fwd(const DwtLevelDesc* d_descs, int ndesc, int max_jobs, int nc, bool irreversible, cudaStream_t st);
void b2k_launch_dwt_inv(const DwtLevelDesc* d_descs, int ndesc, int max_jobs, int nc, bool irreversible, cudaStream_t st);
/* numres = 1: DC shift + colour transform only (forward: image -> coefficient planes; else back, rounded and clamped) */
void b2k_launch_point_transform(const DwtLevelDesc* d_descs, int ndesc, uint32_t max_w, uint32_t max_h, int nc, bool irreversible,
                                bool forward, cudaStream_t st);
/* per-launch limits the encoder sizes its shared memory from (host: build_block_plan) */
struct HtEncodeLimits
{
  uint32_t stage_words; /* max over the launch's blocks of b2k_ht_encode_stage_words(w) */
  uint32_t max_kmax;    /* max Kmax over the launch's blocks */
};
uint32_t b2k_ht_encode_stage_words(uint32_t w);
void b2k_launch_ht_encode(const HtBlockDesc* d_blocks, HtBlockOut* d_out, uint8_t* d_scratch, uint32_t nblocks,
                          const HtEncodeLimits& lim, bool irreversible, cudaStream_t st);
void b2k_launch_ht_gather(const HtBlockDesc* d_blocks, const HtBlockOut* d_out, const uint64_t* d_offsets,
                          const uint8_t* d_scratch, uint8_t* d_bytes, uint32_t nblocks, uint64_t cap, cudaStream_t st);
void b2k_launch_scan_lengths(const HtBlockOut* d_out, uint64_t* d_offsets, uint32_t nblocks, cudaStream_t st);
void b2k_launch_ht_decode_refine(const HtBlockDesc* d_blocks, const uint8_t* d_bytes, const HtBlockOut* d_status,
                                 uint32_t nblocks, int stripe_causal, cudaStream_t st);
void b2k_launch_ht_decode(const HtBlockDesc* d_blocks, const uint8_t* d_bytes, uint32_t* d_recs, HtBlockOut* d_status,
                          uint32_t nblocks, uint32_t max_w, int* d_err, int irreversible, int any_refinement, cudaStream_t st);
void b2k_launch_ht_decode_vlc(const HtBlockDesc* d_blocks, const uint8_t* d_bytes, uint32_t* d_recs, HtBlockOut* d_status,
                              uint32_t nblocks, uint32_t max_w, cudaStream_t st);
/* rejected blocks are counted in d_err[(first_block + b) / blocks_per_slot] for block b of the launch (blocks_per_slot 0:
   all in d_err[0]); a batch's launch over its coded blocks from first_block on counts them per image */
void b2k_launch_ht_decode_magsgn(const HtBlockDesc* d_blocks, const uint8_t* d_bytes, const uint32_t* d_recs,
                                 const HtBlockOut* d_status, uint32_t nblocks, uint32_t max_w, int* d_err, int irreversible,
                                 int any_refinement, cudaStream_t st, uint32_t first_block = 0, uint32_t blocks_per_slot = 0);
void b2k_launch_build_dec_desc(const HtBlockDesc* d_enc, const HtBlockOut* d_out, const uint64_t* d_offsets,
                               const float* d_dec_quant, HtBlockDesc* d_dec, uint32_t n, uint64_t cap, cudaStream_t st);
/* sample containers (sample_bytes 1, 2 or 4) <-> int32 planes.  Component c of pixel (x, y) of the container is at
   base + y * pitch + x * step + c samples; the nc components go to / come from dst[c] / src[c] + y * plane pitch + x */
void b2k_launch_container_to_planes(const void* src, uint32_t spitch, uint32_t step, uint32_t sample_bytes, int32_t* const* dst, int nc,
                                    uint32_t dpitch, uint32_t w, uint32_t h, int sgnd, cudaStream_t st);
void b2k_launch_planes_to_container(const int32_t* const* src, int nc, uint32_t spitch, void* dst, uint32_t dpitch, uint32_t step,
                                    uint32_t sample_bytes, uint32_t w, uint32_t h, cudaStream_t st);
/* a batch's images out, one launch: for each of the n entries of the device table d_dst (BatchDst), its nc components
   (nc > 1: pixel-interleaved, step = nc) from the int32 planes src[c] to dst + y * dpitch + x * step + c samples, the
   entry's w x h pixels.  Entries with dst NULL, or with an err whose *err (the HT decoder's rejections in that image) is
   not 0, are skipped; an entry with err NULL is always written.  All share sample_bytes; max_w x max_h (the largest
   entry) sizes the grid. */
struct BatchDst
{
  const int32_t* src[4];
  void* dst;
  const int* err;
  uint32_t dpitch, step;
  uint32_t w, h;
};
void b2k_launch_planes_to_containers(const BatchDst* d_dst, uint32_t n, int nc, uint32_t spitch, uint32_t sample_bytes, uint32_t max_w,
                                     uint32_t max_h, cudaStream_t st);
/* a batch's images in, one launch: for each of the n entries of the device table d_src (BatchSrc), its nc components
   (nc > 1: pixel-interleaved, step = nc) from src + y * spitch + x * step + c samples to the int32 plane at
   dst + c * dplane + y * dpitch + x, w x h pixels, with the sign handling of b2k_launch_container_to_planes.  All share
   sample_bytes; int32 planes are sample_bytes 4. */
struct BatchSrc
{
  const void* src;
  int32_t* dst; /* the first component's plane */
  uint32_t spitch, step;
};
void b2k_launch_containers_to_planes(const BatchSrc* d_src, uint32_t n, int nc, uint32_t dpitch, size_t dplane, uint32_t sample_bytes,
                                     uint32_t w, uint32_t h, int sgnd, cudaStream_t st);
void b2k_count_launch(void);

/* host_pack.cpp: container conversion on a small host thread pool (int32 planes <-> pinned 16-bit staging) */
struct b2k_host_rect
{
  const void* src;
  void* dst;
  size_t src_stride, dst_stride; /* in elements */
  size_t w, h;
};
/* cached_dst: narrow with plain stores (the 16-bit destination is consumed right away) instead of streaming ones */
void b2k_host_convert(const b2k_host_rect* rects, size_t nrects, bool widen, bool sgnd, bool cached_dst = false);
void b2k_host_session(bool begin); /* between begin and end the pool's idle workers spin instead of sleeping */
void b2k_host_set_threads(int n); /* 0 disables host packing, <0 restores the default */
int b2k_host_threads(void);
int b2k_host_local_peers(void);
/* fn(i) for i in [0, n) on the host pool (plus the caller) */
void b2k_host_parallel(size_t n, const std::function<void(size_t)>& fn);
