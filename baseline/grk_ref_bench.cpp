// grk_ref_bench -- the reference arm of bench.py: times the UNMODIFIED reference's own public API,
// grk_compress() into a memory stream and grk_decompress() from it (grok.h; the flow follows the
// reference's examples/core/core_compress.cpp and core_decompress.cpp), on caller-provided planes.
// Built by oracle/build_ref.sh against oracle/_ref/grok/bin/libgrokj2k.so; called from bench.py and the
// interop tests through ctypes.  Test / measurement infrastructure -- the product never links it.
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <algorithm>
#include <atomic>
#include <mutex>
#include <thread>
#include <vector>

#include "grok.h"

namespace {
double now() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
bool g_init = false;
uint32_t g_threads = 0;
}  // namespace

extern "C" {

struct grb_params {
  uint32_t w, h, ncomp, prec, sgnd;
  uint32_t tile_w, tile_h;        // 0 = one tile
  uint32_t numres;
  uint32_t cblk_w, cblk_h;        // 0 = 64
  uint32_t irreversible;          // 0: 5/3 + RCT, 1: 9/7 + ICT
  uint32_t mct;                   // 0/1
  uint32_t ht;                    // 1 = HTJ2K (cblk_sty HT_ONLY, numgbits 1 as grk_compress does for .jph)
  uint32_t tlm, plt;
  int32_t device_id;              // >= 0 with a plugin loaded: take the plugin route
  uint32_t numgbits;              // 0 = default for the mode
  uint32_t prc_w, prc_h;          // 0 = default precincts; else one (w,h) spec (res_spec = 1)
};

// plugin_path may be NULL (CPU only).  Returns 1 when a plugin was loaded and initialised, 0 otherwise.
int grb_init(uint32_t threads, const char* plugin_path, int32_t device_id) {
  bool plugin = false;
  if (g_init && threads == g_threads && !plugin_path) return 0;
  if (g_init) grk_deinitialize();
  grk_initialize(plugin_path, threads, plugin_path ? &plugin : nullptr);
  g_init = true;
  g_threads = threads;
  if (plugin) {
    grk_plugin_init_info info = {};
    info.device_id = device_id;
    info.verbose = false;
    plugin = grk_plugin_init(info);
  }
  return plugin ? 1 : 0;
}

// frames the plugin handled since it was loaded (grk_plugin_accelerated_frames, grok.cpp L1278-1281)
uint64_t grb_accelerated_frames() { return grk_plugin_accelerated_frames(); }
// switch an initialised plugin in or out of grk_compress() / grk_decompress() (grok.cpp L1274-1277)
void grb_plugin_set_enabled(int on) { grk_plugin_set_enabled(on != 0); }

void grb_deinit() {
  if (g_init) grk_deinitialize();
  g_init = false;
}

// Compress planes[c] (int32, row stride `stride` elements) into out[0..cap); *out_len = codestream bytes.
// Returns seconds spent inside grk_compress() alone (negative on failure).  codestream is raw J2K (.j2k/.jhc).
static void grb_fill_cparameters(const grb_params* p, grk_cparameters& cp);

double grb_compress(const grb_params* p, const int32_t* const* planes, uint32_t stride, uint8_t* out, uint64_t cap,
                    uint64_t* out_len) {
  grk_cparameters cp;
  grb_fill_cparameters(p, cp);

  auto comps = std::make_unique<grk_image_comp[]>(p->ncomp);
  memset(comps.get(), 0, sizeof(grk_image_comp) * p->ncomp);
  for (uint32_t c = 0; c < p->ncomp; ++c) {
    comps[c].w = p->w;
    comps[c].h = p->h;
    comps[c].dx = comps[c].dy = 1;
    comps[c].prec = (uint8_t)p->prec;
    comps[c].sgnd = p->sgnd != 0;
  }
  grk_image* img = grk_image_new((uint16_t)p->ncomp, comps.get(), p->ncomp >= 3 ? GRK_CLRSPC_SRGB : GRK_CLRSPC_GRAY, true);
  if (!img) return -1.0;
  for (uint32_t c = 0; c < p->ncomp; ++c) {
    auto comp = img->comps + c;
    auto dst = (int32_t*)comp->data;
    for (uint32_t y = 0; y < p->h; ++y) memcpy(dst + (size_t)y * comp->stride, planes[c] + (size_t)y * stride, (size_t)p->w * 4);
  }
  grk_stream_params sp = {};
  sp.buf = out;
  sp.buf_len = cap;
  grk_object* codec = grk_compress_init(&sp, &cp, img);
  if (!codec) {
    grk_object_unref(&img->obj);
    return -2.0;
  }
  double t0 = now();
  uint64_t len = grk_compress(codec, nullptr);
  double dt = now() - t0;
  *out_len = len;
  grk_object_unref(codec);
  grk_object_unref(&img->obj);
  return len ? dt : -3.0;
}

// Decompress cs[0..len) into planes[c] (int32, row stride `stride` elements).  Returns seconds from
// grk_decompress() to the composited image being available (header parsing reported in *header_s).
double grb_decompress(const uint8_t* cs, uint64_t len, int32_t* const* planes, uint32_t stride, uint32_t ncomp, uint32_t w,
                      uint32_t h, int32_t device_id, uint32_t reduce, double* header_s) {
  grk_decompress_parameters dp = {};
  dp.core.reduce = (uint8_t)reduce;
  dp.device_id = device_id;
  grk_stream_params sp = {};
  sp.buf = const_cast<uint8_t*>(cs);
  sp.buf_len = len;
  double th = now();
  grk_object* codec = grk_decompress_init(&sp, &dp);
  if (!codec) return -1.0;
  grk_header_info hi = {};
  if (!grk_decompress_read_header(codec, &hi)) {
    grk_object_unref(codec);
    return -2.0;
  }
  if (header_s) *header_s = now() - th;
  double t0 = now();
  bool ok = grk_decompress(codec, nullptr);
  grk_image* img = ok ? grk_decompress_get_image(codec) : nullptr;
  double dt = now() - t0;
  if (!img || img->numcomps < ncomp) {
    grk_object_unref(codec);
    return -3.0;
  }
  if (planes) {
    for (uint32_t c = 0; c < ncomp; ++c) {
      auto comp = img->comps + c;
      if (!comp->data || comp->w > w || comp->h > h) {
        grk_object_unref(codec);
        return -4.0;
      }
      // the decompressor may hand narrow samples back in a 16-bit (or 8-bit) container (grk_image_comp.data_type)
      for (uint32_t y = 0; y < comp->h; ++y) {
        int32_t* d = planes[c] + (size_t)y * stride;
        if (comp->data_type == GRK_INT_16) {
          auto s16 = (const int16_t*)comp->data + (size_t)y * comp->stride;
          for (uint32_t x = 0; x < comp->w; ++x) d[x] = s16[x];
        } else if (comp->data_type == GRK_INT_8) {
          auto s8 = (const int8_t*)comp->data + (size_t)y * comp->stride;
          for (uint32_t x = 0; x < comp->w; ++x) d[x] = s8[x];
        } else {
          memcpy(d, (const int32_t*)comp->data + (size_t)y * comp->stride, (size_t)comp->w * 4);
        }
      }
    }
  }
  grk_object_unref(codec);
  return dt;
}

static void grb_fill_cparameters(const grb_params* p, grk_cparameters& cp) {
  grk_compress_set_default_params(&cp);
  cp.cod_format = GRK_FMT_J2K;
  cp.numresolution = (uint8_t)p->numres;
  cp.irreversible = p->irreversible != 0;
  cp.mct = (uint8_t)p->mct;
  if (p->tile_w && p->tile_h) {
    cp.tile_size_on = true;
    cp.t_width = p->tile_w;
    cp.t_height = p->tile_h;
  }
  if (p->cblk_w) cp.cblockw_init = p->cblk_w;
  if (p->cblk_h) cp.cblockh_init = p->cblk_h;
  if (p->ht) {
    cp.cblk_sty = GRK_CBLKSTY_HT_ONLY;
    cp.numgbits = 1;
  }
  if (p->numgbits) cp.numgbits = (uint8_t)p->numgbits;
  cp.write_tlm = p->tlm != 0;
  cp.write_plt = p->plt != 0;
  if (p->prc_w && p->prc_h) {
    cp.csty |= 0x01;
    cp.res_spec = 1;
    cp.prcw_init[0] = p->prc_w;
    cp.prch_init[0] = p->prc_h;
  }
  cp.device_id = p->device_id;
  cp.num_threads = g_threads;

}

// ---- the host's in-memory batch interfaces (grok.h grk_plugin_batch_memory_*, grk_plugin_batch_decompress_memory_*) ----
namespace {
struct BatchOut {
  uint8_t* out;
  uint64_t cap_per_frame;
  uint64_t* lens;
  std::mutex mu;
};
void batch_frame_done(void* user, void* frame, const uint8_t* codestream, size_t length) {
  auto B = static_cast<BatchOut*>(user);
  size_t i = (size_t)(uintptr_t)frame - 1;
  if (length && length <= B->cap_per_frame) memcpy(B->out + i * B->cap_per_frame, codestream, length);
  B->lens[i] = length <= B->cap_per_frame ? length : 0;
}
}  // namespace

// nframes frames, frame f's component c at planes[f * ncomp + c] (int32 planar).  rgb48 != 0: the frames are handed over as
// GRK_SOURCE_RGB48LE (one interleaved 16-bit buffer each, packed here).  Code streams land at out + f * cap_per_frame.
// Returns the begin() code when it is not 0 (1 = the plugin declined), -2 on a submit failure, else 0; *seconds = submit..end.
int grb_batch_compress(const grb_params* p, const int32_t* const* planes, uint32_t stride, uint32_t nframes, int rgb48,
                       uint8_t* out, uint64_t cap_per_frame, uint64_t* out_lens, double* seconds) {
  grk_cparameters cp;
  grb_fill_cparameters(p, cp);
  BatchOut B{out, cap_per_frame, out_lens, {}};
  for (uint32_t f = 0; f < nframes; ++f) out_lens[f] = 0;
  grk_plugin_batch_memory_info info = {};
  info.compress_parameters = &cp;
  info.width = p->w;
  info.height = p->h;
  info.numcomps = (uint16_t)p->ncomp;
  info.prec = (uint8_t)p->prec;
  info.source_prec = (uint8_t)p->prec;
  info.callback = batch_frame_done;
  info.user = &B;
  info.source_format = rgb48 ? GRK_SOURCE_RGB48LE : GRK_SOURCE_PLANAR_RGB;
  int32_t rc = grk_plugin_batch_memory_begin(info);
  if (rc != 0) return rc;
  std::vector<grk_image_comp> comps(p->ncomp);
  std::vector<uint16_t> packed;
  double t0 = now();
  bool ok = true;
  for (uint32_t f = 0; f < nframes && ok; ++f) {
    memset(comps.data(), 0, sizeof(grk_image_comp) * p->ncomp);
    grk_image img = {};
    img.x1 = p->w;
    img.y1 = p->h;
    img.numcomps = (uint16_t)p->ncomp;
    img.comps = comps.data();
    for (uint32_t c = 0; c < p->ncomp; ++c) {
      comps[c].w = p->w;
      comps[c].h = p->h;
      comps[c].dx = comps[c].dy = 1;
      comps[c].prec = (uint8_t)p->prec;
      comps[c].stride = stride;
      comps[c].data = const_cast<int32_t*>(planes[(size_t)f * p->ncomp + c]);
      comps[c].data_type = GRK_INT_32;
    }
    if (rgb48) {
      packed.resize((size_t)p->w * p->h * p->ncomp);
      for (uint32_t c = 0; c < p->ncomp; ++c)
        for (uint32_t y = 0; y < p->h; ++y)
          for (uint32_t x = 0; x < p->w; ++x)
            packed[((size_t)y * p->w + x) * p->ncomp + c] = (uint16_t)planes[(size_t)f * p->ncomp + c][(size_t)y * stride + x];
      for (uint32_t c = 0; c < p->ncomp; ++c) {
        comps[c].data_type = GRK_INT_16;
        comps[c].data = c == 0 ? packed.data() : nullptr;
        comps[c].stride = c == 0 ? p->w * p->ncomp : 0;
      }
    }
    ok = grk_plugin_batch_memory_submit(&img, (void*)(uintptr_t)(f + 1));
  }
  bool drained = grk_plugin_batch_memory_end();
  if (seconds) *seconds = now() - t0;
  return ok && drained ? 0 : -2;
}

namespace {
struct BatchIn {
  const uint8_t* cs;
  const uint64_t* offs;  // nframes + 1
  uint32_t nframes, ncomp, w, h, stride;
  int32_t* const* planes;  // [nframes * ncomp]
  std::atomic<uint32_t> next{0};
  std::atomic<uint32_t> good{0};
  std::atomic<bool> ended{false};
};
bool batch_pull(void* user, const uint8_t** codestream, size_t* length, void** frame_user) {
  auto B = static_cast<BatchIn*>(user);
  if (B->ended) return false;
  uint32_t i = B->next.fetch_add(1);
  if (i >= B->nframes) {
    // nothing more: block the way a caller with an empty queue would, until end() flips the flag
    while (!B->ended) std::this_thread::sleep_for(std::chrono::milliseconds(1));
    return false;
  }
  *codestream = B->cs + B->offs[i];
  *length = (size_t)(B->offs[i + 1] - B->offs[i]);
  *frame_user = (void*)(uintptr_t)(i + 1);
  return true;
}
void batch_decoded(void* user, void* frame, const grk_image* image) {
  auto B = static_cast<BatchIn*>(user);
  size_t i = (size_t)(uintptr_t)frame - 1;
  if (!image || image->numcomps < B->ncomp) return;
  for (uint32_t c = 0; c < B->ncomp; ++c) {
    auto comp = image->comps + c;
    if (!comp->data || comp->w != B->w || comp->h != B->h) return;
    for (uint32_t y = 0; y < B->h; ++y)
      memcpy(B->planes[i * B->ncomp + c] + (size_t)y * B->stride, (const int32_t*)comp->data + (size_t)y * comp->stride,
             (size_t)B->w * 4);
  }
  B->good++;
}
}  // namespace

// nframes code streams (frame f = cs[offs[f] .. offs[f+1])) through grk_plugin_batch_decompress_memory_begin/_end; decoded
// int32 planes land in planes[f * ncomp + c].  Returns begin()'s code when not 0, else the number of frames that came back good.
int grb_batch_decompress(const uint8_t* cs, const uint64_t* offs, uint32_t nframes, int32_t* const* planes, uint32_t stride,
                         uint32_t ncomp, uint32_t w, uint32_t h, double* seconds) {
  BatchIn B;
  B.cs = cs; B.offs = offs; B.nframes = nframes; B.ncomp = ncomp; B.w = w; B.h = h; B.stride = stride; B.planes = planes;
  grk_plugin_batch_decompress_memory_info info = {};
  info.codestream = cs + offs[0];
  info.codestream_length = (size_t)(offs[1] - offs[0]);
  info.pull = batch_pull;
  info.callback = batch_decoded;
  info.user = &B;
  double t0 = now();
  int32_t rc = grk_plugin_batch_decompress_memory_begin(info);
  if (rc != 0) return rc > 0 ? -100 - rc : rc;
  // every frame handed out and reported back (good or not) -> the caller ends the batch
  while (B.next.load() < nframes) std::this_thread::sleep_for(std::chrono::milliseconds(1));
  B.ended = true;
  bool drained = grk_plugin_batch_decompress_memory_end();
  if (seconds) *seconds = now() - t0;
  return drained ? (int)B.good.load() : -3;
}

}  // extern "C"
