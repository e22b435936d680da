/*
 * grok_b200/csrc/plugin_decode.cpp -- the stock decode entry point, plugin_decompress().
 *
 * Protocol (host side: CodeStreamDecompress.cpp L199-271, grok.cpp L1882-2015): the PLUGIN drives and
 * calls the host back four times with decompress_flags
 *   HEADER  -> host parses the main header, fills header_info + image, and calls OUR
 *              init_decompressors_func(header_info, image): we size the engine and allocate the tile tree
 *              (every code block gets a buffer the host will copy its bytes into);
 *   T2      -> host parses packets only and fills, per block, compressedData / compressedDataLength /
 *              numBitPlanes / numPasses (decompress_synch_plugin_with_host, TileProcessor.cpp L157-227);
 *   POST_T1 -> we have decoded: host copies the int32 planes out (pluginStoreDecodedImage L243-271);
 *   CLEAN   -> both sides drop per-tile state.
 * Return: 0 decoded, 1 not handled (host decodes on the CPU), <0 error (plugin_accelerate.h L32-36).
 * Eligibility mirrors the host's own (single tile, no reduce/window/layers: L199-205) plus: HT cleanup
 * pass only, one segment per block, this engine's quantiser (Grok's HT defaults).
 */
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <atomic>
#include <thread>
#include <vector>

#include "plugin_decode_abi.h"
#include "geometry.h"
#include "t2_packet.h"

using namespace b2k;

extern b2k_engine* b2k_plugin_engine(void); /* plugin.cpp: the engine plugin_init created (or creates it) */
extern void b2k_plugin_free_tree(gpup_tile* T);

namespace {

struct DecodeCtx
{
  b2k_coding cp{};
  bool ready = false;
  int32_t rc = 0;
  std::vector<b2k_block> blocks;
  std::vector<gpup_code_block*> cb_of; /* tree node of every enumerated block */
  std::vector<gpup_band*> bands;       /* comp-major, then resolution, then band */
  gpup_tile* tree = nullptr;
  uint8_t* slab = nullptr; /* host-visible block buffers the T2 callback fills */
  uint64_t slab_bytes = 0;
};
thread_local DecodeCtx* g_ctx = nullptr;

uint32_t block_capacity(uint32_t w, uint32_t h, uint32_t kmax)
{
  const uint64_t samples = (uint64_t)w * h, quads = (uint64_t)((w + 1) / 2) * ((h + 1) / 2);
  return (uint32_t)(((samples * (kmax + 2) + 6) / 7 + (quads * 15 + 6) / 7 + 256 + 64 + 15) & ~15ull);
}

/* HEADER callback -> host -> here */
int init_decompressors(gpup_header_info* h, gpup_image* image)
{
  DecodeCtx* C = g_ctx;
  if(!C || !h || !image || !image->comps)
    return -1;
  b2k_coding& cp = C->cp;
  memset(&cp, 0, sizeof(cp));
  C->rc = 1; /* "not handled" unless everything below fits */
  if(!(h->cblk_sty & GPUP_CBLKSTY_HT) || h->t_grid_width != 1 || h->t_grid_height != 1 || h->mct > 1)
    return 0;
  cp.x0 = image->x0; cp.y0 = image->y0; cp.x1 = image->x1; cp.y1 = image->y1;
  cp.numcomps = image->numcomps;
  if(cp.numcomps < 1 || cp.numcomps > 4)
    return 0;
  cp.prec = image->comps[0].prec;
  cp.sgnd = image->comps[0].sgnd;
  for(uint16_t c = 0; c < image->numcomps; ++c)
  {
    const gpup_image_comp& k = image->comps[c];
    if(k.dx != 1 || k.dy != 1 || k.prec != cp.prec || (k.sgnd ? 1 : 0) != cp.sgnd)
      return 0;
  }
  cp.numres = h->numresolutions;
  cp.cblkw_exp = (uint8_t)t2::floorlog2(h->cblockw_init);
  cp.cblkh_exp = (uint8_t)t2::floorlog2(h->cblockh_init);
  cp.irreversible = h->irreversible;
  cp.mct = h->mct;
  cp.numgbits = 1; /* Grok's HT setting (GrkCompress.cpp L849); checked per block against numBitPlanes */
  for(int r = 0; r < 33; ++r)
  {
    cp.prcw_exp[r] = r < h->numresolutions && h->prcw_init[r] ? (uint8_t)t2::floorlog2(h->prcw_init[r]) : 15;
    cp.prch_exp[r] = r < h->numresolutions && h->prch_init[r] ? (uint8_t)t2::floorlog2(h->prch_init[r]) : 15;
    /* the host hands 1 << PPx; PPx = 0 would read as "default" in b2k_coding -> leave such streams to the host */
    if(r < h->numresolutions && (h->prcw_init[r] == 1 || h->prch_init[r] == 1))
      return 0;
  }
  if(unsupported_reason(cp))
    return 0;
  /* enumerate, allocate the block buffers and the tree */
  const int64_t n = b2k_enumerate(&cp, 1, 0, nullptr, 0);
  if(n < 0)
    return 0;
  C->blocks.resize((size_t)n);
  b2k_enumerate(&cp, 1, 0, C->blocks.data(), (uint64_t)n);
  uint64_t off = 0;
  for(b2k_block& b : C->blocks)
  {
    b.offset = off;
    b.length = (b.x1 > b.x0 && b.y1 > b.y0) ? block_capacity(b.x1 - b.x0, b.y1 - b.y0, b.kmax) : 0;
    b.numbps = 0;
    b.numpasses = 0;
    off += b.length;
  }
  C->slab_bytes = off;
  C->slab = (uint8_t*)malloc(off + 64); /* pages are touched only where the host writes */
  if(!C->slab)
    return -1;
  b2k_result fake{};
  fake.num_blocks = (uint64_t)n;
  fake.blocks = C->blocks.data();
  fake.bytes = C->slab;
  fake.num_bytes = off;
  C->tree = b2k_result_to_gpup_tile(&cp, &fake, 0);
  if(!C->tree)
    return -1;
  /* remember the node of every block (same walk order as the builder), reset what T2 will fill */
  C->cb_of.clear();
  C->bands.clear();
  for(size_t c = 0; c < C->tree->numComponents; ++c)
  {
    gpup_tile_component* tc = C->tree->tileComponents[c];
    for(size_t r = 0; r < tc->numResolutions; ++r)
      for(size_t bi = 0; bi < tc->resolutions[r]->numBands; ++bi)
      {
        gpup_band* band = tc->resolutions[r]->band[bi];
        C->bands.push_back(band);
        for(uint64_t p = 0; p < band->numPrecincts; ++p)
          for(uint64_t k = 0; k < band->precincts[p]->numBlocks; ++k)
          {
            gpup_code_block* cb = band->precincts[p]->blocks[k];
            cb->compressedDataLength = 0;
            cb->numBitPlanes = 0;
            cb->numPasses = 0;
            C->cb_of.push_back(cb);
          }
      }
  }
  if(C->cb_of.size() != C->blocks.size())
    return -1;
  C->ready = true;
  C->rc = 0;
  return 0;
}

} // namespace

namespace {

/* One frame through the HEADER -> T2 -> POST_T1 -> CLEAN protocol.  `codestream` != NULL: a frame of an in-memory batch
   (the host reads it instead of a file: PluginDecodeCallbackInfo::codestream, plugin_interface.h L111-114); a failed
   batch frame still reaches the host's frame callback, with a NULL image (grok.h "NULL when this frame failed"). */
int32_t decode_frame(b2k_engine* eng, gpup_decompress_params* params, PLUGIN_DECODE_USER_CALLBACK cb, const uint8_t* codestream,
                     size_t codestream_length, void* frame_user)
{
  const bool batch = codestream != nullptr;
  DecodeCtx ctx;
  g_ctx = &ctx;
  PluginDecodeCallbackInfo info("", "", params, 1 /* J2K */, GPUP_DECODE_HEADER);
  info.init_decompressors_func = init_decompressors;
  info.deviceId = 0;
  info.codestream = codestream;
  info.codestreamLength = codestream_length;
  info.frameUser = frame_user;
  int32_t rc = -1;
  gpup_image* host_img = nullptr;
  bool delivered = false;
  std::vector<int32_t*> plane_ptrs;
  std::vector<uint32_t> strides;
  do
  {
    if(cb(&info) != 0 || !ctx.ready)
    {
      rc = ctx.rc ? ctx.rc : 1;
      break;
    }
    /* ---- T2: the host fills the tree ---- */
    info.tile = ctx.tree;
    info.decompress_flags = GPUP_DECODE_T2;
    ctx.tree->decompress_flags = GPUP_DECODE_T2;
    if(cb(&info) != 0)
    {
      rc = -1;
      break;
    }
    /* ---- gather what the host parsed; compact the used bytes for the upload ---- */
    const b2k_coding& cp = ctx.cp;
    const std::vector<std::vector<BandQuant>> q = component_quant(cp);
    uint64_t used = 0;
    bool ok = true;
    for(size_t i = 0; i < ctx.blocks.size() && ok; ++i)
    {
      const gpup_code_block* cbk = ctx.cb_of[i];
      b2k_block& b = ctx.blocks[i];
      const uint32_t cap = b.length;
      b.length = cbk->compressedDataLength;
      b.numbps = cbk->numBitPlanes;
      b.numpasses = (uint8_t)(cbk->numPasses > 255 ? 255 : cbk->numPasses);
      if(b.length > cap || (b.length && (b.numpasses != 1 || b.numbps > b.kmax || b.numbps < 1)))
        ok = false; /* refinement passes / other guard bits / overflow: leave it to the CPU */
      used += b.length;
    }
    if(ok && cp.irreversible)
    { /* host hands decoder-convention step / 2 (TileProcessor.cpp L183-184): it must be this engine's */
      size_t bi = 0;
      for(int c = 0; c < cp.numcomps && ok; ++c)
        for(int r = 0; r < cp.numres && ok; ++r)
          for(int b = 0; b < (r ? 3 : 1) && ok; ++b, ++bi)
          {
            const float mine = q[c][band_quant_index(r, r ? b + 1 : 0)].step_dec;
            const float theirs = ctx.bands[bi]->stepsize * 2.0f;
            if(std::fabs(mine - theirs) > 1e-6f * std::fabs(mine))
              ok = false;
          }
    }
    if(!ok)
    {
      rc = 1;
      break;
    }
    uint8_t* compact = (uint8_t*)b2k_host_alloc(used + 64);
    if(!compact)
    {
      rc = -1;
      break;
    }
    uint64_t at = 0;
    for(b2k_block& b : ctx.blocks)
    {
      if(b.length)
        memcpy(compact + at, ctx.slab + b.offset, b.length);
      b.offset = at;
      at += b.length;
    }
    /* ---- decode into pinned planes ---- */
    const uint32_t w = cp.x1 - cp.x0, hgt = cp.y1 - cp.y0;
    const uint32_t stride = (w + 15u) & ~15u; /* 64-byte aligned rows (gpu_plugin_shared.h L540-544) */
    plane_ptrs.resize(cp.numcomps);
    strides.assign(cp.numcomps, stride);
    bool alloc_ok = true;
    for(int c = 0; c < cp.numcomps; ++c)
    {
      plane_ptrs[c] = (int32_t*)b2k_host_alloc((size_t)stride * hgt * sizeof(int32_t));
      alloc_ok = alloc_ok && plane_ptrs[c];
    }
    double ms = 0;
    int32_t drc = alloc_ok ? b2k_decode(eng, &cp, ctx.blocks.data(), ctx.blocks.size(), compact, used, plane_ptrs.data(),
                                        strides.data(), 1, 0, &ms)
                           : -1;
    b2k_host_free(compact);
    if(drc != 0)
    {
      rc = drc > 0 ? 1 : -1;
      for(int32_t* p : plane_ptrs)
        b2k_host_free(p);
      plane_ptrs.clear();
      break;
    }
    /* ---- POST_T1: hand the planes over.  The image shell is made the way the host makes its own (grk_to_gpup_image,
       plugin_gpup_bridge.h L160-189: new + new[]): a batch host drops it with gpup_image_free_shell after its frame callback
       (grok.cpp L1992-1996), the per-call host leaves it to us. ---- */
    gpup_image* out_img = new gpup_image();
    memset(out_img, 0, sizeof(*out_img));
    out_img->comps = new gpup_image_comp[cp.numcomps]();
    for(int c = 0; c < cp.numcomps; ++c)
    {
      gpup_image_comp& k = out_img->comps[c];
      k.x0 = cp.x0; k.y0 = cp.y0; k.w = w; k.h = hgt; k.stride = stride;
      k.dx = k.dy = 1;
      k.prec = cp.prec;
      k.sgnd = cp.sgnd;
      k.data = plane_ptrs[c];
      k.owns_data = false;
    }
    out_img->x0 = cp.x0; out_img->y0 = cp.y0; out_img->x1 = cp.x1; out_img->y1 = cp.y1;
    out_img->numcomps = cp.numcomps;
    out_img->color_space = info.image ? info.image->color_space : 0;
    host_img = info.image;
    info.image = out_img;
    info.plugin_owns_image = true;
    info.decompress_flags = GPUP_DECODE_POST_T1;
    const int32_t prc = cb(&info);
    delivered = true;
    if(info.image == out_img)
    {
      delete[] out_img->comps;
      delete out_img;
    }
    info.image = host_img;
    host_img = nullptr;
    for(int32_t* p : plane_ptrs)
      b2k_host_free(p);
    plane_ptrs.clear();
    rc = prc == 0 ? 0 : -1;
  } while(false);
  if(batch && !delivered)
  { /* the frame's owner hears about it: NULL image */
    host_img = info.image;
    info.image = nullptr;
    info.decompress_flags = GPUP_DECODE_POST_T1;
    cb(&info);
    info.image = host_img;
  }
  /* ---- CLEAN ---- */
  info.decompress_flags = GPUP_DECODE_CLEAN;
  cb(&info);
  if(ctx.tree)
    b2k_plugin_free_tree(ctx.tree);
  free(ctx.slab);
  g_ctx = nullptr;
  return rc;
}

} // namespace

extern "C" int32_t plugin_decompress(gpup_decompress_params* params, PLUGIN_DECODE_USER_CALLBACK cb)
{
  if(!cb)
    return -1;
  b2k_engine* eng = b2k_plugin_engine();
  if(!eng)
    return -1;
  return decode_frame(eng, params, cb, nullptr, 0, nullptr);
}

/* ---- in-memory batch decompress (SURVEY 8f N2; host side grok.cpp L2023-2188) -------------------------------------------
 *   plugin_batch_decompress_memory_begin(gpup_batch_decompress_memory_info*, PLUGIN_DECODE_USER_CALLBACK)
 *       typedef plugin_interface.h L130-131; info gpu_plugin_shared.h L492-506
 *   plugin_batch_decompress_memory_end()          L133
 * The plugin's workers PULL code streams from the host (info->pull; false ends a worker), run each through the same
 * four-step protocol as plugin_decompress with the frame's bytes in PluginDecodeCallbackInfo::codestream, and the host's
 * frame callback runs inside POST_T1 on the worker's thread (batchDecompressMemoryCallback, grok.cpp L2052-2092).
 * Design: `depth` workers, each a host thread with its OWN engine (own streams, own cached job), so one frame's
 * host T2 parse and copies overlap its neighbours' kernels.  8-bit RGB output packing (srgb8_output / display_transform) is
 * not taken: rgb8_on_device stays false and the frames come back as planes, which the contract allows. */
namespace {
struct DecodeBatch
{
  bool running = false;
  gpup_decompress_params params{};
  PLUGIN_DECODE_USER_CALLBACK cb = nullptr;
  GPUP_BATCH_DECOMPRESS_PULL pull = nullptr;
  void* pull_user = nullptr;
  std::vector<b2k_engine*> engines;
  std::vector<std::thread> workers;
  std::atomic<int32_t> failures{0};
};
DecodeBatch g_dbatch;
} // namespace

extern int32_t b2k_plugin_device(void);

extern "C" int32_t plugin_batch_decompress_memory_begin(gpup_batch_decompress_memory_info* info, PLUGIN_DECODE_USER_CALLBACK cb)
{
  DecodeBatch& B = g_dbatch;
  if(!info || !cb || !info->pull || B.running)
    return -1;
  const gpup_header_info& h = info->header_info;
  /* the shape check plugin_decompress does per frame, up front: anything else stays on the host (return 1) */
  if(!(h.cblk_sty & GPUP_CBLKSTY_HT) || h.t_grid_width != 1 || h.t_grid_height != 1 || h.mct > 1 || !info->image ||
     info->image->numcomps < 1 || info->image->numcomps > 4)
    return 1;
  for(uint16_t c = 0; c < info->image->numcomps; ++c)
    if(info->image->comps[c].dx != 1 || info->image->comps[c].dy != 1 || info->image->comps[c].prec != info->image->comps[0].prec)
      return 1;
  if(info->decompress_parameters)
    B.params = *info->decompress_parameters;
  B.cb = cb;
  B.pull = info->pull;
  B.pull_user = info->pull_user;
  B.failures = 0;
  const uint32_t depth = 3;
  for(uint32_t i = 0; i < depth; ++i)
  {
    b2k_engine* e = nullptr;
    if(b2k_engine_create(b2k_plugin_device(), &e) != 0)
    {
      for(b2k_engine* x : B.engines)
        b2k_engine_destroy(x);
      B.engines.clear();
      return -1;
    }
    B.engines.push_back(e);
  }
  info->rgb8_on_device = false;
  B.running = true;
  for(uint32_t i = 0; i < depth; ++i)
    B.workers.emplace_back([&B, i] {
      for(;;)
      {
        const uint8_t* cs = nullptr;
        size_t len = 0;
        void* frame_user = nullptr;
        if(!B.pull(B.pull_user, &cs, &len, &frame_user))
          return;
        if(!cs || !len)
          continue;
        if(decode_frame(B.engines[i], &B.params, B.cb, cs, len, frame_user) != 0)
          B.failures++;
      }
    });
  return 0;
}

extern "C" bool plugin_batch_decompress_memory_end(void)
{
  DecodeBatch& B = g_dbatch;
  if(!B.running)
    return false;
  for(std::thread& t : B.workers)
    t.join(); /* the host's pull answers false from here on (grok.cpp L2173-2181) */
  B.workers.clear();
  for(b2k_engine* e : B.engines)
    b2k_engine_destroy(e);
  B.engines.clear();
  B.running = false;
  return true;
}
