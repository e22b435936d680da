/*
 * grok_b200/csrc/plugin.cpp -- the STOCK accelerator-plugin symbols (group 1 of
 * include/grok_b200.h) on top of the b2k engine.
 *
 *   minpf_post_load_plugin   minpf loader handshake           plugin/minpf_plugin_manager.cpp L136-238
 *   plugin_init              device selection                 grok.cpp L1344-1370
 *   gpup_encode_mem          whole image = one tile           grok.cpp L1302-1328, CodeStreamCompress.cpp L878-912
 *   gpup_tile_free           tree + coded bytes owned here    grok.cpp L1330, plugin_bridge.cpp L185-189
 *   gpup_encode_mem_tiles    multi-tile images, all tiles in one call -- the seam of the host patch
 *   gpup_tiles_free          baseline/patches/0001-multi-tile-plugin-encode-decode.patch (SURVEY.md 8b)
 *   plugin_decompress_codestream   multi-tile code streams held in memory (same patch, decode side)
 * Return convention plugin_accelerate.h L32-36: 0 handled, >0 not handled (CPU fallback), <0 error.
 * Messages go through the host's logger (minpf_platform_services::logger, minpf_plugin.h L98-107) once the
 * loader has handed it over; before that (or without a host) to stderr when verbose.
 */
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "../../include/grok_b200.h"
#include "geometry.h"
#include "t2_packet.h"

using namespace b2k;

/* The logger interface the host passes across the boundary (minpf_plugin.h L23-32: three variadic virtuals, no
 * virtual destructor) and the services struct it arrives in (L98-107). */
namespace gpup
{
struct ILogger
{
  virtual void info(const char* fmt, ...) = 0;
  virtual void warn(const char* fmt, ...) = 0;
  virtual void error(const char* fmt, ...) = 0;
};
} // namespace gpup
struct _minpf_platform_services
{
  struct { int32_t major, minor; } version;
  int32_t (*registerObject)(const char* nodeType, const void* params);
  int32_t (*invokeService)(const char* serviceName, void* serviceParams);
  const char* pluginPath;
  bool verbose;
  gpup::ILogger* logger;
};

static std::mutex g_mu;
static gpup::ILogger* g_logger = nullptr;

enum { LOG_INFO, LOG_WARN, LOG_ERROR };
void b2k_plugin_log(int level, const char* fmt, ...)
{
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  gpup::ILogger* L = g_logger;
  if(L)
  {
    if(level == LOG_ERROR)
      L->error("[grok_b200] %s", buf);
    else if(level == LOG_WARN)
      L->warn("[grok_b200] %s", buf);
    else
      L->info("[grok_b200] %s", buf);
  }
  else if(level != LOG_INFO || getenv("B2K_PLUGIN_VERBOSE"))
    fprintf(stderr, "[grok_b200] %s\n", buf);
}

static b2k_engine* g_engine = nullptr;
static int32_t g_device = 0;
static bool g_verbose = false;
/* tile -> result that owns its coded bytes */
static std::unordered_map<gpup_tile*, b2k_result*> g_owned;

static int32_t plugin_exit(void)
{
  std::lock_guard<std::mutex> lock(g_mu);
  if(g_engine)
  {
    b2k_engine_destroy(g_engine);
    g_engine = nullptr;
  }
  return 0;
}

extern "C" minpf_exit_func minpf_post_load_plugin(const minpf_platform_services* services)
{
  /* nothing to register: the host resolves our entry points by name (grok.cpp L1177-1186); the services carry
     the host's logger and verbosity (minpf_plugin_manager.cpp L225-238) */
  if(services && services->version.major == 1)
  {
    g_logger = services->logger;
    g_verbose = services->verbose;
  }
  return plugin_exit;
}

extern "C" bool plugin_init(gpup_init_info info)
{
  std::lock_guard<std::mutex> lock(g_mu);
  g_verbose = info.verbose;
  g_device = info.deviceId < 0 ? 0 : info.deviceId;
  if(!g_engine && b2k_engine_create(g_device, &g_engine) != 0)
  {
    b2k_plugin_log(LOG_ERROR, "plugin_init failed: %s", b2k_last_error());
    return false;
  }
  return true;
}

extern "C" uint32_t plugin_get_debug_state(void)
{ /* B2K_PLUGIN_DEBUG_STATE=1 asks the host to run its own T1 beside ours and diff every block (plugin_bridge.cpp L127-198) */
  static const uint32_t state = getenv("B2K_PLUGIN_DEBUG_STATE") ? (uint32_t)strtoul(getenv("B2K_PLUGIN_DEBUG_STATE"), nullptr, 0)
                                                                  : (uint32_t)GPUP_STATE_NO_DEBUG;
  return state;
}

/* gpup_compress_params + gpup_image -> b2k_coding; false if the engine does not cover it */
static bool coding_from_gpup(const gpup_compress_params* p, const gpup_image* im, b2k_coding* cp, bool allow_tiles = false)
{
  memset(cp, 0, sizeof(*cp));
  if(!p || !im || !im->comps || im->numcomps < 1 || im->numcomps > 4)
    return false;
  if(!(p->cblk_sty & GPUP_CBLKSTY_HT))
    return false; /* Part-1 MQ block coding stays on the host */
  if(p->numlayers > 1 || p->roi_compno >= 0 || p->numpocs)
    return false;
  cp->x0 = im->x0; cp->y0 = im->y0; cp->x1 = im->x1; cp->y1 = im->y1;
  const bool tiled = p->tile_size_on && (p->t_width < cp->x1 - p->tx0 || p->t_height < cp->y1 - p->ty0);
  if(tiled && !allow_tiles)
    return false; /* stock contract: one tile (CodeStreamCompress.cpp L908-912) */
  cp->tw = cp->th = 0;
  if(tiled)
  { /* tile grid as CodeStreamCompress::init sets it up from the parameters (SIZ: XTOsiz, YTOsiz, XTsiz, YTsiz) */
    cp->tx0 = p->tx0; cp->ty0 = p->ty0; cp->tw = p->t_width; cp->th = p->t_height;
    if(!cp->tw || !cp->th || cp->tx0 > cp->x0 || cp->ty0 > cp->y0)
      return false;
  }
  cp->numcomps = im->numcomps;
  cp->prec = im->comps[0].prec;
  cp->sgnd = im->comps[0].sgnd;
  for(uint16_t c = 0; c < im->numcomps; ++c)
  {
    const gpup_image_comp& k = im->comps[c];
    if(k.dx != 1 || k.dy != 1 || k.prec != cp->prec || (k.sgnd ? 1 : 0) != cp->sgnd || !k.data)
      return false;
    if(k.w != cp->x1 - cp->x0 || k.h != cp->y1 - cp->y0)
      return false;
  }
  cp->numres = p->numresolution;
  cp->cblkw_exp = (uint8_t)t2::floorlog2(p->cblockw_init ? p->cblockw_init : 64);
  cp->cblkh_exp = (uint8_t)t2::floorlog2(p->cblockh_init ? p->cblockh_init : 64);
  cp->irreversible = p->irreversible;
  cp->mct = p->mct ? 1 : 0;
  if(p->mct > 1)
    return false; /* custom (array) MCT */
  cp->numgbits = p->numgbits;
  for(int r = 0; r < 33; ++r)
  {
    cp->prcw_exp[r] = 15;
    cp->prch_exp[r] = 15;
  }
  if((p->csty & 1) && p->res_spec)
  { /* CodeStreamCompress.cpp L793-825: sizes are given finest resolution first; once the list runs out every
       coarser resolution takes the last given size halved again per level; a size below 1 means exponent 1 */
    const uint32_t spec = p->res_spec < 33 ? p->res_spec : 33;
    uint32_t k = 0;
    for(int rr = (int)p->numresolution - 1; rr >= 0; --rr, ++k)
    {
      uint32_t pw, ph;
      if(k < spec)
      {
        pw = p->prcw_init[k];
        ph = p->prch_init[k];
      }
      else
      {
        const uint32_t sh = k - (spec - 1);
        pw = sh < 32 ? p->prcw_init[spec - 1] >> sh : 0;
        ph = sh < 32 ? p->prch_init[spec - 1] >> sh : 0;
      }
      const int ew = pw < 1 ? 1 : t2::floorlog2(pw), eh = ph < 1 ? 1 : t2::floorlog2(ph);
      if(ew < 1 || eh < 1 || ew > 15 || eh > 15)
        return false; /* 1-sample precincts: b2k_coding reads exponent 0 as "default"; left to the host */
      if(rr < 33)
      {
        cp->prcw_exp[rr] = (uint8_t)ew;
        cp->prch_exp[rr] = (uint8_t)eh;
      }
    }
  }
  return unsupported_reason(*cp) == nullptr;
}

/* One calloc'ed slab per tree; gpup_tile_free releases it. */
extern "C" gpup_tile* b2k_result_to_gpup_tile(const b2k_coding* cp, const b2k_result* r, uint32_t tile)
{
  if(!cp || !r)
    return nullptr;
  /* count */
  const int ncomp = cp->numcomps, numres = cp->numres;
  std::vector<const b2k_block*> blks;
  for(uint64_t i = 0; i < r->num_blocks; ++i)
    if(r->blocks[i].tile == tile)
      blks.push_back(&r->blocks[i]);
  const TileGrid g = tile_grid(*cp);
  const Rect tr = tile_rect(*cp, g, tile);
  const std::vector<std::vector<BandQuant>> q = component_quant(*cp);

  gpup_tile* T = (gpup_tile*)calloc(1, sizeof(gpup_tile));
  T->decompress_flags = 0;
  T->numComponents = (size_t)ncomp;
  T->tileComponents = (gpup_tile_component**)calloc(ncomp, sizeof(void*));
  size_t cursor = 0;
  for(int c = 0; c < ncomp; ++c)
  {
    gpup_tile_component* tc = (gpup_tile_component*)calloc(1, sizeof(gpup_tile_component));
    T->tileComponents[c] = tc;
    tc->numResolutions = (size_t)numres;
    tc->resolutions = (gpup_resolution**)calloc(numres, sizeof(void*));
    for(int resno = 0; resno < numres; ++resno)
    {
      gpup_resolution* res = (gpup_resolution*)calloc(1, sizeof(gpup_resolution));
      tc->resolutions[resno] = res;
      res->level = (size_t)resno;
      res->numBands = resno == 0 ? 1 : 3;
      res->band = (gpup_band**)calloc(res->numBands, sizeof(void*));
      const PrecinctGrid pg = precinct_grid(*cp, tr, resno);
      const uint64_t nprec = (uint64_t)pg.gw * pg.gh;
      for(size_t b = 0; b < res->numBands; ++b)
      {
        gpup_band* band = (gpup_band*)calloc(1, sizeof(gpup_band));
        res->band[b] = band;
        band->orientation = (uint8_t)(resno == 0 ? 0 : b + 1);
        band->stepsize = q[c][band_quant_index(resno, band->orientation)].step_enc;
        band->numPrecincts = nprec;
        band->precincts = (gpup_precinct**)calloc(nprec ? nprec : 1, sizeof(void*));
        for(uint64_t p = 0; p < nprec; ++p)
          band->precincts[p] = (gpup_precinct*)calloc(1, sizeof(gpup_precinct));
        /* blocks of this band are contiguous in enumeration order */
        size_t first = cursor;
        while(cursor < blks.size() && blks[cursor]->comp == c && blks[cursor]->resno == resno &&
              blks[cursor]->band_index == b)
          ++cursor;
        for(size_t i = first; i < cursor;)
        {
          const uint32_t p = blks[i]->precno;
          size_t j = i;
          while(j < cursor && blks[j]->precno == p)
            ++j;
          gpup_precinct* prc = band->precincts[p];
          prc->numBlocks = j - i;
          prc->blocks = (gpup_code_block**)calloc(j - i, sizeof(void*));
          for(size_t k = i; k < j; ++k)
          {
            const b2k_block& s = *blks[k];
            gpup_code_block* cb = (gpup_code_block*)calloc(1, sizeof(gpup_code_block));
            prc->blocks[k - i] = cb;
            cb->x0 = s.x0; cb->y0 = s.y0; cb->x1 = s.x1; cb->y1 = s.y1;
            cb->numPix = (s.x1 - s.x0) * (s.y1 - s.y0);
            cb->compressedData = s.length ? r->bytes + s.offset : nullptr;
            cb->compressedDataLength = s.length;
            cb->numBitPlanes = s.numbps;
            cb->numPasses = s.numpasses;
            if(s.numpasses)
            { /* plugin_bridge.cpp L221-227: rate is the index of the last byte */
              cb->passes[0].rate = s.length ? s.length - 1 : 0;
              cb->passes[0].length = s.length;
              cb->passes[0].distortionDecrease = 0.0;
            }
            cb->sortedIndex = (unsigned int)(k - i);
          }
          i = j;
        }
      }
    }
  }
  return T;
}

void b2k_plugin_free_tree(gpup_tile* T);
static void free_tree(gpup_tile* T) { b2k_plugin_free_tree(T); }
void b2k_plugin_free_tree(gpup_tile* T)
{
  if(!T)
    return;
  for(size_t c = 0; c < T->numComponents; ++c)
  {
    gpup_tile_component* tc = T->tileComponents[c];
    for(size_t r = 0; r < tc->numResolutions; ++r)
    {
      gpup_resolution* res = tc->resolutions[r];
      for(size_t b = 0; b < res->numBands; ++b)
      {
        gpup_band* band = res->band[b];
        for(uint64_t p = 0; p < band->numPrecincts; ++p)
        {
          gpup_precinct* prc = band->precincts[p];
          for(uint64_t k = 0; k < prc->numBlocks; ++k)
            free(prc->blocks[k]);
          free(prc->blocks);
          free(prc);
        }
        free(band->precincts);
        free(band);
      }
      free(res->band);
      free(res);
    }
    free(tc->resolutions);
    free(tc);
  }
  free(T->tileComponents);
  free(T);
}

int32_t b2k_plugin_device(void) { return g_device; }
void b2k_gpup_tile_free_tree(gpup_tile* tile)
{
  if(tile)
    free_tree(tile);
}

/* the engine the stock entry points share (created by plugin_init, or lazily on first use) */
b2k_engine* b2k_plugin_engine(void)
{
  std::lock_guard<std::mutex> lock(g_mu);
  if(!g_engine && b2k_engine_create(g_device, &g_engine) != 0)
    return nullptr;
  return g_engine;
}

extern "C" int32_t gpup_encode_mem(gpup_compress_params* params, gpup_image* image, gpup_tile** out)
{
  if(!out)
    return -1;
  *out = nullptr;
  b2k_coding cp;
  if(!coding_from_gpup(params, image, &cp))
    return 1; /* not handled -> host CPU path */
  {
    std::lock_guard<std::mutex> lock(g_mu);
    if(!g_engine && b2k_engine_create(g_device, &g_engine) != 0)
      return -1;
  }
  const int32_t* planes[4];
  uint32_t strides[4];
  for(uint16_t c = 0; c < image->numcomps; ++c)
  {
    planes[c] = image->comps[c].data;
    strides[c] = image->comps[c].stride;
  }
  b2k_result* R = nullptr;
  const int32_t rc = b2k_encode(g_engine, &cp, planes, strides, 1, 0, &R);
  if(rc != 0)
    return rc;
  gpup_tile* T = b2k_result_to_gpup_tile(&cp, R, 0);
  if(!T)
  {
    b2k_result_free(R);
    return -1;
  }
  std::lock_guard<std::mutex> lock(g_mu);
  g_owned[T] = R;
  *out = T;
  return 0;
}

extern "C" void gpup_tile_free(gpup_tile* tile)
{
  if(!tile)
    return;
  b2k_result* R = nullptr;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_owned.find(tile);
    if(it != g_owned.end())
    {
      R = it->second;
      g_owned.erase(it);
    }
  }
  free_tree(tile);
  if(R)
    b2k_result_free(R);
}

/* exported for hosts and tests: the coding b2k_* calls would use for these stock parameters; 0 handled, 1 not */
extern "C" int32_t b2k_coding_from_gpup(const gpup_compress_params* params, const gpup_image* image, int32_t allow_tiles,
                                        b2k_coding* out)
{
  if(!out)
    return -1;
  return coding_from_gpup(params, image, out, allow_tiles != 0) ? 0 : 1;
}

/* ---- multi-tile images (host patch baseline/patches/0001-...): every tile of the image is compressed in ONE
 * call -- one upload, one pipeline over all tiles, which is where the device is efficient and where tiles would be
 * sharded over GPUs -- and the host gets one stock gpup_tile tree per tile index for its per-tile T2 tasks
 * (ITileProcessor::setCurrentPluginTile, ITileProcessor.h L270-276).  The trees share one result's byte arena. */
struct TileSet
{
  b2k_result* result;
  std::vector<gpup_tile*> tiles;
};
static std::unordered_map<gpup_tile**, TileSet*> g_tilesets;

extern "C" int32_t gpup_encode_mem_tiles(gpup_compress_params* params, gpup_image* image, gpup_tile*** out_tiles,
                                         uint32_t* out_num_tiles)
{
  if(!out_tiles || !out_num_tiles)
    return -1;
  *out_tiles = nullptr;
  *out_num_tiles = 0;
  b2k_coding cp;
  if(!coding_from_gpup(params, image, &cp, true))
    return 1;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    if(!g_engine && b2k_engine_create(g_device, &g_engine) != 0)
    {
      b2k_plugin_log(LOG_ERROR, "no engine: %s", b2k_last_error());
      return -1;
    }
  }
  const int32_t* planes[4];
  uint32_t strides[4];
  for(uint16_t c = 0; c < image->numcomps; ++c)
  {
    planes[c] = image->comps[c].data;
    strides[c] = image->comps[c].stride;
  }
  b2k_result* R = nullptr;
  const int32_t rc = b2k_encode(g_engine, &cp, planes, strides, 1, 0, &R);
  if(rc != 0)
  {
    if(rc < 0)
      b2k_plugin_log(LOG_ERROR, "b2k_encode failed: %s", b2k_last_error());
    return rc;
  }
  TileSet* S = new TileSet{R, {}};
  S->tiles.resize(R->num_tiles);
  for(uint32_t t = 0; t < R->num_tiles; ++t)
    S->tiles[t] = b2k_result_to_gpup_tile(&cp, R, t);
  std::lock_guard<std::mutex> lock(g_mu);
  g_tilesets[S->tiles.data()] = S;
  *out_tiles = S->tiles.data();
  *out_num_tiles = R->num_tiles;
  return 0;
}

extern "C" void gpup_tiles_free(gpup_tile** tiles, uint32_t)
{
  if(!tiles)
    return;
  TileSet* S = nullptr;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    auto it = g_tilesets.find(tiles);
    if(it == g_tilesets.end())
      return;
    S = it->second;
    g_tilesets.erase(it);
  }
  for(gpup_tile* t : S->tiles)
    free_tree(t);
  b2k_result_free(S->result);
  delete S;
}

/* ---- multi-tile code streams (decode side of the same patch): the host hands over the code stream it holds in
 * memory (raw, or inside a JP2 / JPH container) and an image whose int32 planes it has allocated; tile parts are
 * located, packet headers parsed and all tiles decoded here (b2k_codestream_parse + b2k_decode). */
extern "C" int32_t plugin_decompress_codestream(const uint8_t* file, uint64_t length, gpup_image* image)
{
  if(!file || !image || !image->comps)
    return -1;
  uint64_t off = 0, len = length;
  if(b2k_jph_codestream(file, length, &off, &len) != 0)
    return 1;
  b2k_coding cp;
  const int64_t n = b2k_codestream_parse(file + off, len, &cp, nullptr, 0);
  if(n == 1 || n == 0)
    return 1; /* something this path does not cover: the host decodes on the CPU */
  if(n < 0)
  {
    b2k_plugin_log(LOG_WARN, "code stream not parsed (%s); left to the host", b2k_last_error());
    return 1;
  }
  if(image->numcomps != cp.numcomps)
    return 1;
  int32_t* planes[4];
  uint32_t strides[4];
  for(uint16_t c = 0; c < image->numcomps; ++c)
  {
    const gpup_image_comp& k = image->comps[c];
    if(!k.data || k.w != cp.x1 - cp.x0 || k.h != cp.y1 - cp.y0 || k.dx != 1 || k.dy != 1)
      return 1;
    planes[c] = k.data;
    strides[c] = k.stride ? k.stride : k.w;
  }
  std::vector<b2k_block> blocks((size_t)n);
  if(b2k_codestream_parse(file + off, len, &cp, blocks.data(), (uint64_t)n) != n)
    return 1;
  {
    std::lock_guard<std::mutex> lock(g_mu);
    if(!g_engine && b2k_engine_create(g_device, &g_engine) != 0)
    {
      b2k_plugin_log(LOG_ERROR, "no engine: %s", b2k_last_error());
      return -1;
    }
  }
  const int32_t rc = b2k_decode(g_engine, &cp, blocks.data(), (uint64_t)n, file + off, len, planes, strides, 1, 0, nullptr);
  if(rc < 0)
    b2k_plugin_log(LOG_ERROR, "b2k_decode failed: %s", b2k_last_error());
  return rc;
}
