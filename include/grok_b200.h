/*
 * include/grok_b200.h -- C ABI of libgrokj2k_plugin.so, the CUDA (sm_90a, H100) JPEG 2000 tile engine.
 *
 * Two groups of entry points:
 *
 *  (1) The STOCK accelerator-plugin symbols Grok's host library resolves with dlsym()
 *      (reference: src/lib/core/grok.cpp L1177-1186, L1297-1300; typedefs
 *      src/lib/core/plugin/plugin_interface.h L50-133; structs
 *      src/lib/core/plugin/gpup/gpu_plugin_shared.h L215-530).  The struct layouts below are
 *      binary-compatible restatements of that contract: field order and types must not change.
 *
 *  (2) The tile-aware b2k_* engine API.  The stock contract is "whole image = one tile"
 *      (CodeStreamCompress.cpp L908-912, CodeStreamDecompress.cpp L199-205); multi-tile
 *      codestreams, multi-GPU sharding, device-resident buffers and per-stage parity hooks go
 *      through these.  INTEGRATION.md shows the ~30-line host patch that binds them.
 *
 * All functions are extern "C", plain pointers and sizes, no C++ or torch types.
 * Return convention (plugin_accelerate.h L32-36): 0 = handled, >0 = not handled (host falls
 * back to its CPU path), <0 = device failure.
 */
#ifndef GROK_B200_H
#define GROK_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2K_API __attribute__((visibility("default")))

/* ============================================================================================
 * (1) stock plugin contract -- gpu_plugin_shared.h
 * ========================================================================================== */
#define GPUP_PATH_LEN 4096
#define GPUP_MAX_LAYERS 256
#define GPUP_MAX_DECOMP_LVLS 32
#define GPUP_MAXRLVLS (GPUP_MAX_DECOMP_LVLS + 1)
#define GPUP_MAX_SUPPORTED_PREC 16
#define GPUP_BIBO_EXTRA_BITS 7
#define GPUP_MAX_PASSES (3 * (GPUP_MAX_SUPPORTED_PREC + GPUP_BIBO_EXTRA_BITS) - 2)
#define GPUP_BUFFER_ALIGNMENT 64

#define GPUP_DECODE_HEADER (1 << 0)
#define GPUP_DECODE_T2 (1 << 1)
#define GPUP_DECODE_T1 (1 << 2)
#define GPUP_DECODE_POST_T1 (1 << 3)
#define GPUP_DECODE_CLEAN (1 << 4)

#define GPUP_STATE_NO_DEBUG 0x0
#define GPUP_CBLKSTY_HT 0x040

/* enums of gpu_plugin_shared.h L63-146 are plain C enums (int sized) */
typedef int32_t gpup_prog_order;
typedef int32_t gpup_color_space;
typedef int32_t gpup_file_fmt;
typedef int32_t gpup_codec_fmt;
typedef int32_t gpup_rate_control;

typedef struct _gpup_image_comp /* L215-225 */
{
  uint32_t x0, y0;
  uint32_t w;
  uint32_t stride;
  uint32_t h;
  uint8_t dx, dy;
  uint8_t prec;
  bool sgnd;
  int32_t* data;
  bool owns_data;
} gpup_image_comp;

typedef struct _gpup_image /* L227-233 */
{
  uint32_t x0, y0, x1, y1;
  uint16_t numcomps;
  gpup_color_space color_space;
  gpup_image_comp* comps;
} gpup_image;

typedef struct _gpup_pass /* L240-245 */
{
  double distortionDecrease;
  size_t rate;
  size_t length;
} gpup_pass;

typedef struct _gpup_code_block /* L247-261 */
{
  uint32_t x0, y0, x1, y1;
  unsigned int* contextStream;
  uint32_t numPix;
  uint8_t* compressedData;
  uint32_t compressedDataLength;
  uint8_t numBitPlanes;
  size_t numPasses;
  gpup_pass passes[GPUP_MAX_PASSES];
  unsigned int sortedIndex;
} gpup_code_block;

typedef struct _gpup_precinct
{
  uint64_t numBlocks;
  gpup_code_block** blocks;
} gpup_precinct;

typedef struct _gpup_band
{
  uint8_t orientation;
  uint64_t numPrecincts;
  gpup_precinct** precincts;
  float stepsize;
} gpup_band;

typedef struct _gpup_resolution
{
  size_t level;
  size_t numBands;
  gpup_band** band;
} gpup_resolution;

typedef struct _gpup_tile_component
{
  size_t numResolutions;
  gpup_resolution** resolutions;
} gpup_tile_component;

typedef struct _gpup_tile /* L289-294 */
{
  uint32_t decompress_flags;
  size_t numComponents;
  gpup_tile_component** tileComponents;
} gpup_tile;

typedef struct _gpup_header_info /* L300-318 */
{
  uint32_t cblockw_init;
  uint32_t cblockh_init;
  bool irreversible;
  uint8_t mct;
  uint16_t rsiz;
  uint8_t numresolutions;
  gpup_prog_order prog_order;
  uint8_t csty;
  uint8_t cblk_sty;
  uint32_t prcw_init[GPUP_MAXRLVLS];
  uint32_t prch_init[GPUP_MAXRLVLS];
  uint32_t tx0, ty0;
  uint32_t t_width, t_height;
  uint16_t t_grid_width, t_grid_height;
  uint16_t max_layers_;
} gpup_header_info;

typedef struct _gpup_compress_params /* L324-374 */
{
  bool tile_size_on;
  uint32_t tx0, ty0, t_width, t_height;
  uint16_t numlayers;
  bool allocationByRateDistoration;
  double layer_rate[GPUP_MAX_LAYERS];
  bool allocationByQuality;
  double layer_distortion[GPUP_MAX_LAYERS];
  uint8_t csty;
  uint8_t numgbits;
  gpup_prog_order prog_order;
  uint32_t numpocs;
  uint8_t numresolution;
  uint32_t cblockw_init;
  uint32_t cblockh_init;
  uint8_t cblk_sty;
  bool irreversible;
  int32_t roi_compno;
  uint32_t roi_shift;
  uint32_t res_spec;
  uint32_t prcw_init[GPUP_MAXRLVLS];
  uint32_t prch_init[GPUP_MAXRLVLS];
  char infile[GPUP_PATH_LEN];
  char outfile[GPUP_PATH_LEN];
  uint32_t image_offset_x0;
  uint32_t image_offset_y0;
  uint8_t subsampling_dx;
  uint8_t subsampling_dy;
  gpup_file_fmt decod_format;
  gpup_file_fmt cod_format;
  bool enableTilePartGeneration;
  uint8_t newTilePartProgressionDivider;
  uint8_t mct;
  uint64_t max_cs_size;
  uint64_t max_comp_size;
  uint16_t rsiz;
  uint16_t framerate;
  gpup_rate_control rateControlAlgorithm;
  uint32_t numThreads;
  int32_t deviceId;
  uint32_t duration;
  uint32_t kernelBuildOptions;
  uint32_t repeats;
  bool verbose;
  bool sharedMemoryInterface;
  bool apply_xyz_transform;
} gpup_compress_params;

typedef struct _gpup_decompress_core_params
{
  uint8_t reduce;
  uint16_t layers_to_decompress_;
} gpup_decompress_core_params;

typedef struct _gpup_decompress_params /* L386-401 */
{
  gpup_decompress_core_params core;
  char infile[GPUP_PATH_LEN];
  char outfile[GPUP_PATH_LEN];
  gpup_codec_fmt decod_format;
  gpup_file_fmt cod_format;
  double dw_x0, dw_y0, dw_x1, dw_y1;
  uint16_t tileIndex;
  int32_t deviceId;
  uint32_t kernelBuildOptions;
  uint32_t repeats;
  uint32_t numThreads;
  bool verbose_;
  void* user_data;
} gpup_decompress_params;

typedef struct _gpup_init_info /* L403-409 */
{
  int32_t deviceId;
  bool verbose;
  const char* license;
  const char* server;
} gpup_init_info;

typedef int (*GPUP_INIT_DECOMPRESSORS)(gpup_header_info* header_info, gpup_image* image);

typedef struct _gpup_decompress_callback_info /* L503-524 */
{
  size_t deviceId;
  GPUP_INIT_DECOMPRESSORS init_decompressors_func;
  const char* input_file_name;
  const char* output_file_name;
  gpup_codec_fmt decod_format;
  gpup_file_fmt cod_format;
  void* codec;
  gpup_header_info header_info;
  gpup_decompress_params* decompressor_parameters;
  gpup_image* image;
  bool plugin_owns_image;
  gpup_tile* tile;
  unsigned int error_code;
  uint32_t decompress_flags;
  uint32_t full_image_x0;
  uint32_t full_image_y0;
  void* user_data;
  void* format_private;
} gpup_decompress_callback_info;

typedef int32_t (*GPUP_DECOMPRESS_USER_CALLBACK)(gpup_decompress_callback_info* info);

/* minpf loader handshake: minpf_plugin.h L98-111 */
typedef int32_t (*minpf_exit_func)(void);
typedef struct _minpf_platform_services minpf_platform_services; /* opaque here; see INTEGRATION.md */

/* --- symbols resolved by name by libgrokj2k (grok.cpp L1177-1186, L1297-1298) --- */
B2K_API minpf_exit_func minpf_post_load_plugin(const minpf_platform_services* services); /* minpf_plugin.h L109 */
B2K_API bool plugin_init(gpup_init_info info);                    /* plugin_interface.h L60 */
B2K_API uint32_t plugin_get_debug_state(void);                    /* plugin_interface.h L56 */
B2K_API int32_t gpup_encode_mem(gpup_compress_params* params, gpup_image* image,
                                gpup_tile** out);                 /* grok.cpp L1299-1300 */
B2K_API void gpup_tile_free(gpup_tile* tile);                     /* grok.cpp L1330 */
/* --- optional symbols the PATCHED host resolves (baseline/patches/0001-multi-tile-plugin-encode-decode.patch;
 * the stock contract is one tile per image, CodeStreamCompress.cpp L908-912 / CodeStreamDecompress.cpp L199-205) --- */
/* all tiles of a multi-tile image in one call; (*out_tiles)[t] is the stock tree of tile index t in the tile's
 * canvas coordinates; the array and the trees stay valid until gpup_tiles_free(*out_tiles, n) */
B2K_API int32_t gpup_encode_mem_tiles(gpup_compress_params* params, gpup_image* image, gpup_tile*** out_tiles,
                                      uint32_t* out_num_tiles);
B2K_API void gpup_tiles_free(gpup_tile** tiles, uint32_t num_tiles);
/* a whole (multi-tile) code stream the host holds in memory -> the int32 planes of `image` (allocated by the host) */
B2K_API int32_t plugin_decompress_codestream(const uint8_t* codestream, uint64_t length, gpup_image* image);

/* --- in-memory batch compress (grok.cpp L1538-1545, L1655-1857): frames of one shape, several in flight --- */
typedef struct _gpup_stream_params /* gpu_plugin_shared.h L415-421 */
{
  const char* file;
  uint8_t* buf;
  size_t buf_len;
  size_t buf_compressed_len;
} gpup_stream_params;
typedef struct _gpup_compress_callback_info /* L428-440 */
{
  const char* input_file_name;
  bool outputFileNameIsRelative;
  const char* output_file_name;
  gpup_compress_params* compressor_parameters;
  gpup_image* image;
  gpup_tile* tile;
  gpup_stream_params stream_params;
  unsigned int error_code;
  void* host_data;
} gpup_compress_callback_info;
typedef uint64_t (*GPUP_COMPRESS_USER_CALLBACK)(gpup_compress_callback_info* info); /* L442 */
typedef enum { GPUP_SOURCE_PLANAR_RGB = 0, GPUP_SOURCE_YUV420P = 1, GPUP_SOURCE_YUV422P = 2, GPUP_SOURCE_RGB48LE = 3 } gpup_source_format; /* L127-136 */
typedef enum { GPUP_YUV_BT601 = 0, GPUP_YUV_BT709 = 1, GPUP_YUV_BT2020 = 2 } gpup_yuv_matrix;                                             /* L139-144 */
typedef struct _gpup_batch_memory_info /* L454-473 */
{
  gpup_compress_params* compress_parameters;
  uint32_t width, height, numcomps;
  uint32_t source_prec; /* bits per sample the caller submits */
  uint32_t prec;        /* bits per sample the code stream carries */
  GPUP_COMPRESS_USER_CALLBACK callback;
  bool xyz_on_device;   /* written by begin */
  gpup_source_format source_format;
  gpup_yuv_matrix yuv_matrix;
  bool yuv_full_range;
} gpup_batch_memory_info;
B2K_API int32_t gpup_batch_memory_begin(gpup_batch_memory_info* info);
B2K_API bool gpup_batch_memory_submit(const uint8_t* packed, void* host_data);
B2K_API bool gpup_batch_memory_submit_planes(const uint8_t* const planes[3], const size_t stride_bytes[3], void* host_data);
B2K_API bool gpup_batch_memory_end(void);
/* --- in-memory batch decompress (grok.cpp L2023-2188): the plugin's workers pull code streams of one shape --- */
typedef bool (*GPUP_BATCH_DECOMPRESS_PULL)(void* user, const uint8_t** codestream, size_t* length, void** frame_user); /* L477-478 */
typedef struct _gpup_display_transform /* L481-487 */
{
  const float* transfer;
  const float* matrix;
} gpup_display_transform;
typedef struct _gpup_batch_decompress_memory_info /* L492-506 */
{
  gpup_decompress_params* decompress_parameters;
  gpup_header_info header_info;
  gpup_image* image;
  GPUP_BATCH_DECOMPRESS_PULL pull;
  void* pull_user;
  bool srgb8_output;
  const gpup_display_transform* display_transform;
  bool rgb8_on_device; /* written by begin: stays false here (frames come back as int32 planes) */
} gpup_batch_decompress_memory_info;
/* plugin_batch_decompress_memory_begin(info, PLUGIN_DECODE_USER_CALLBACK) takes the same C++ callback type as
 * plugin_decompress (below), so it is declared with it; its end has a plain C signature: */
B2K_API bool plugin_batch_decompress_memory_end(void);            /* plugin_interface.h L133 */
/* plugin_decompress (plugin_interface.h L117-120) takes a C++ struct with std::string members
 * (PluginDecodeCallbackInfo L78-115): it is declared in grok_b200/csrc/plugin_decode.cpp and
 * documented in INTEGRATION.md, not here, so that this header stays C. */

/* ============================================================================================
 * (2) tile-aware engine API
 * ========================================================================================== */
typedef struct b2k_engine b2k_engine;

/* coding parameters of one image; the subset of grk_cparameters / SIZ+COD+QCD the tile engine
 * depends on (CodeStreamCompress::init, CodeStreamCompress.cpp L229-855) */
typedef struct b2k_coding
{
  uint32_t x0, y0, x1, y1;         /* image area on the canvas (SIZ) */
  uint32_t tx0, ty0, tw, th;       /* tile grid origin and nominal tile size (tw==0: one tile) */
  uint16_t numcomps;               /* 1..4; all components dx=dy=1 and same precision */
  uint8_t prec;                    /* bits per sample */
  uint8_t sgnd;                    /* 1 = signed samples */
  uint8_t numres;                  /* resolutions = decomposition levels + 1 */
  uint8_t cblkw_exp, cblkh_exp;    /* log2 nominal code-block size (6,6 = 64x64) */
  uint8_t irreversible;            /* 0: 5/3 + RCT, 1: 9/7 + ICT */
  uint8_t mct;                     /* 1: colour transform on components 0..2 */
  uint8_t numgbits;                /* guard bits; Grok's HT CLI forces 1 (GrkCompress.cpp L849) */
  uint8_t prcw_exp[33], prch_exp[33]; /* precinct exponents per resolution, 1..15 (15 = maximal); 0 reads as 15.
                                         A true exponent 0 (1-sample precincts) is declined by every entry point */
  uint8_t cblk_sty;                /* code-block style bits (COD); only 0x08 = vertically stripe-causal matters,
                                      and only to the decoder's SigProp pass (CoderOJPH.cpp L248) */
  uint8_t qcd_explicit;            /* 0: band exponents / mantissas are the HT quantiser's (QuantizerOJPH.cpp L193-259),
                                      as Grok's encoder signals them.  1: take them from qcd_expn / qcd_mant below --
                                      what b2k_codestream_parse fills in for a foreign stream's QCD (band order of QCD:
                                      LL, then HL, LH, HH per resolution) */
  uint8_t qcd_expn[97];
  uint16_t qcd_mant[97];
  uint8_t qfactor;                 /* 0: off.  1..100: every component's band steps are those grk_compress --qfactor derives
                                      for this coding (a JPEG-style quality factor: 9/7 synthesis norms, visual weights
                                      per band and component, ICT column gains); component 0's go to QCD, the others'
                                      to QCC.  Needs irreversible = 1 and 1 or 3 components; overrides qcd_explicit and
                                      qcc_mask.  b2k_codestream_parse sets it when QCD / QCC hold exactly such tables */
  uint8_t qcc_mask;                /* bit c: component c takes its band exponents / mantissas from qcc_expn[c] /
                                      qcc_mant[c] (same band order as QCD) instead of from QCD's; the parser sets the
                                      bit of every component a main-header QCC names */
  uint8_t qcc_expn[4][97];
  uint16_t qcc_mant[4][97];
} b2k_coding;

/* One coded block as the host's T2 needs it (cf. compress_synch_with_plugin,
 * plugin_bridge.cpp L113-243), in Grok's enumeration order tile->comp->res->band->prec->cblk */
typedef struct b2k_block
{
  uint32_t tile;                   /* tile index, raster order */
  uint16_t comp;
  uint8_t resno, band_index, orient;
  uint8_t kmax;                    /* band->maxBitPlanes_ (TileProcessor.cpp L417-419) */
  uint8_t numbps;                  /* coded bit planes as T2 signals them: Kmax - zero bit planes.
                                      The encoder returns 1 (CoderOJPH.cpp L203-206) */
  uint8_t numpasses;               /* 0 not coded; 1 HT cleanup (all the encoder emits); decode also takes 2
                                      (+ SigProp) and 3 (+ SigProp + MagRef) from foreign streams */
  uint32_t precno, cblkno;
  uint32_t x0, y0, x1, y1;         /* block rect, band canvas coordinates */
  uint32_t buf_x, buf_y;           /* position inside the tile-component Mallat buffer */
  uint32_t length;                 /* bytes of the HT cleanup segment */
  uint64_t offset;                 /* byte offset into the result's byte arena */
  float stepsize;                  /* band step size (encoder convention) */
  uint32_t length2;                /* decode: bytes of the refinement segment (SigProp, MagRef) that follows
                                      the cleanup segment at offset + length; 0 from the encoder */
} b2k_block;

typedef struct b2k_result
{
  uint64_t num_blocks;
  b2k_block* blocks;               /* host memory, owned by the result */
  uint8_t* bytes;                  /* host memory (pinned), owned by the result */
  uint64_t num_bytes;
  uint32_t num_tiles;
  double ms_h2d, ms_dwt, ms_t1, ms_d2h, ms_total; /* device-event timings of the call */
} b2k_result;

B2K_API int32_t b2k_engine_create(int32_t device, b2k_engine** out);
B2K_API void b2k_engine_destroy(b2k_engine* e);
B2K_API const char* b2k_last_error(void);

/* the b2k_coding that gpup_encode_mem (allow_tiles = 0) / gpup_encode_mem_tiles (1) derive from the host's stock
 * parameters, precinct sizes as CodeStreamCompress.cpp L793-825 derives them (0 handled, 1 not handled) */
B2K_API int32_t b2k_coding_from_gpup(const gpup_compress_params* params, const gpup_image* image, int32_t allow_tiles,
                                     b2k_coding* out);

/* pinned host memory for image planes / codestream arenas (what Grok's allocator should hand
 * to grk_image when the plugin is loaded; see INTEGRATION.md) */
B2K_API void* b2k_host_alloc(size_t bytes);
B2K_API void b2k_host_free(void* p);
/* b2k_encode / b2k_decode can carry samples of <= 16 bits over PCIe in 16-bit containers: each
 * pipeline chunk is narrowed (widened) between the caller's int32 planes and a pinned staging
 * buffer by host threads while its neighbour is on the bus.  That halves the PCIe bytes and costs
 * host DRAM bandwidth, so whether it pays depends on the machine and on what else runs on it.
 *   n < 0 (default): min(cores the process may run on, 24) threads (env B2K_HOST_THREADS); each
 *          job times both ways on its first calls and keeps the faster one;
 *   n = 0: never (int32 planes are copied as they are and should be pinned);
 *   n > 0: always, with n threads (also the way to feed unpinned planes).
 * Returns the thread count in force.  b2k_host_pack_last(decode) tells which way the last
 * b2k_encode (0) / b2k_decode (1) went: 1 packed, 0 direct, -1 none yet. */
B2K_API int32_t b2k_set_host_threads(int32_t n);
B2K_API int32_t b2k_host_pack_last(int32_t decode);

/* Encode every tile of the image for which (tile_index % tile_mod) == tile_rem (tile_mod=1:
 * all tiles).  planes[c] = int32 samples, row stride strides[c] elements, origin (x0,y0). */
B2K_API int32_t b2k_encode(b2k_engine* e, const b2k_coding* cp, const int32_t* const* planes,
                           const uint32_t* strides, uint32_t tile_mod, uint32_t tile_rem,
                           b2k_result** out);
/* same, 16-bit unsigned/signed sample containers (cf. gpup_batch_memory_submit_planes) */
B2K_API int32_t b2k_encode16(b2k_engine* e, const b2k_coding* cp, const uint16_t* const* planes,
                             const uint32_t* strides, uint32_t tile_mod, uint32_t tile_rem,
                             b2k_result** out);
/* same, ONE pixel-interleaved buffer of 16-bit samples (component c of pixel x at pixels[y*stride + x*numcomps + c],
 * stride in samples >= numcomps * width): the layout of gpup_batch_memory_submit's packed frames and of
 * GPUP_SOURCE_RGB48LE (grok.cpp L1806-1836, grok.h "GRK_SOURCE_RGB48LE").  The rows cross PCIe as they are and are
 * split into planes on the device -- no host pass over the samples. */
B2K_API int32_t b2k_encode16_interleaved(b2k_engine* e, const b2k_coding* cp, const uint16_t* pixels, uint32_t stride,
                                         uint32_t tile_mod, uint32_t tile_rem, b2k_result** out);
B2K_API void b2k_result_free(b2k_result* r);

/* Decode: blocks[] (same enumeration, with length/offset filled by the host's T2 parse) and the
 * byte arena in; planes out (int32, clamped, DC shift restored). */
B2K_API int32_t b2k_decode(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks,
                           uint64_t num_blocks, const uint8_t* bytes, uint64_t num_bytes,
                           int32_t* const* planes, const uint32_t* strides, uint32_t tile_mod,
                           uint32_t tile_rem, double* ms_total);
/* b2k_decode / b2k_decode16 returning only `window` = (x0, y0, x1, y1), in cp's canvas coordinates, of the pixels:
 * planes[c] holds the window's rows (strides[c] samples apart), sample_bytes = 4 (int32) or 2 (16-bit containers).  The tiles
 * of cp are decoded as usual; only the window's pixels cross PCIe.  Made for the virtual coding of
 * b2k_codestream_parse_window (windowed / reduced decode, SURVEY 8f N3). */
B2K_API int32_t b2k_decode_window(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                                  const uint8_t* bytes, uint64_t num_bytes, void* const* planes, const uint32_t* strides,
                                  const uint32_t* window, uint32_t sample_bytes, double* ms_total);
/* same, pixels returned in 16-bit containers (reversible path) */
B2K_API int32_t b2k_decode16(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks,
                             uint64_t num_blocks, const uint8_t* bytes, uint64_t num_bytes,
                             uint16_t* const* planes, const uint32_t* strides, uint32_t tile_mod,
                             uint32_t tile_rem, double* ms_total);

/* ---- images in device memory: encode from / decode into a buffer the caller keeps on the engine's GPU ---------------
 * A renderer's frame, a video pipeline's surface or a CUDA tensor need not cross PCIe: only the coded bytes do.  The image
 * is described per component; component c of pixel (x, y) (counted from the image's, or the window's, first pixel) is at
 *   (char*)comp[c] + (y * row_pitch[c] + x * col_step[c]) * sample_bytes
 * so planar buffers (col_step 1), pixel-interleaved ones (col_step = numcomps, comp[c] = comp[0] + c samples) and views
 * such as the RGB of an RGBA buffer (col_step 4) all fit.  Samples are sample_bytes wide, signed when cp->sgnd. */
typedef struct b2k_device_planes
{
  void* comp[4];          /* device address of component c's first sample (canvas x0, y0 of the image, or of the window) */
  uint32_t row_pitch[4];  /* samples between the starts of two rows */
  uint32_t col_step[4];   /* samples between two pixels of a row: 1 planar, numcomps pixel-interleaved, 4 for RGB of RGBA */
  uint32_t sample_bytes;  /* 1, 2 or 4; signedness is cp->sgnd */
} b2k_device_planes;
/* b2k_encode_device gives exactly what b2k_encode gives for the same samples; b2k_decode_device writes exactly what
 * b2k_decode writes, cast to the container (the decoder clamps to cp->prec, so narrowing only truncates).  Only the
 * selected tiles (tile % tile_mod == tile_rem) are read or written.  window works as in b2k_decode_window: img then holds
 * the window, and tile_mod must be 1.  The coded data (`bytes`, the result's arena) stay in host memory: T2 is host code.
 * Samples are converted between the container and the engine's int32 planes on the device, chunk by chunk in place of the
 * host calls' PCIe copies (int32 planar images are copied device to device).
 * Stream order: the call first records an event on cuda_stream (NULL = the legacy default stream) and the engine's
 * streams wait for it, so work the caller queued before the call (the kernel that produced the frame) is finished before
 * the engine reads the buffer; before returning, it makes cuda_stream wait for the engine's last access to the buffer.
 * Like the host calls it returns once its work is done (the encode result is in host memory; decode reports HT decoder
 * errors as b2k_decode does, -2).
 * Returns 0 handled; 1 not handled (a container narrower than cp->prec, more than 4 components); -1 bad input (a comp[c]
 * that cudaPointerGetAttributes does not report as device or managed memory of the engine's device, one that is not a
 * multiple of sample_bytes, col_step 0, a window outside the image).  b2k_last_error says which.
 * These calls share the engine's cached job with b2k_encode / b2k_decode and leave the host-packing policy alone
 * (b2k_host_pack_last keeps reporting the last host call). */
B2K_API int32_t b2k_encode_device(b2k_engine* e, const b2k_coding* cp, const b2k_device_planes* img, uint32_t tile_mod,
                                  uint32_t tile_rem, void* cuda_stream, b2k_result** out);
B2K_API int32_t b2k_decode_device(b2k_engine* e, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                                  const uint8_t* bytes, uint64_t num_bytes, const b2k_device_planes* img, const uint32_t* window,
                                  uint32_t tile_mod, uint32_t tile_rem, void* cuda_stream, double* ms_total);
/* An image in device memory -> a complete HTJ2K code stream assembled in device memory, byte-identical to
 * b2k_encode_device + b2k_codestream_write(cp, result, flags) over the whole image; any flags b2k_codestream_write takes.
 * *cs = device address of the code stream, in a buffer the engine owns; valid until the next call of this function on e,
 * or b2k_engine_destroy.  Returns the length (> 1); 1 not handled (as b2k_encode_device); < 0 on error: -2 a block
 * overflowed the coder (as b2k_encode_device), -1 otherwise, in the cases and with the b2k_last_error text of
 * b2k_encode_device and b2k_codestream_write (a tile grid the writer declines, more than 65535 tiles, more than 255 tile
 * parts in a tile, a tile part of 4 GiB or more, ...).
 * Input ordering on cuda_stream as b2k_encode_device; returns once the code stream is written.  Packet headers, PLT, TLM
 * and the tile-part layout are computed by kernels and the block bytes go from the coder's scratch to the file without
 * leaving the GPU: no block table or arena crosses PCIe, only the final length does.  The plan of the code stream
 * (geometry and flags) is made once per coding and flags and kept with the engine's cached job. */
B2K_API int64_t b2k_encode_codestream_device(b2k_engine* e, const b2k_coding* cp, const b2k_device_planes* img,
                                             uint32_t flags, void* cuda_stream, const uint8_t** cs);
/* A batch: n images in device memory, all of coding cp -> n HTJ2K code streams in device memory, in one launch chain.
 * status[i] and b2k_encode_codestreams_error(e, i) are what b2k_encode_codestream_device(e, cp, &imgs[i], flags, ...)
 * returns for image i alone and its b2k_last_error text: 0 where it returns a length, else 1, -1 or -2, the checks in the
 * same order (imgs[i]'s descriptor, the coding, the writer's plan, blocks that overflowed the coder, the writer's limits).
 * A verdict that depends only on the coding or the flags is every image's, with the same text.  Status 0: the
 * length[i] bytes at *cs + offset[i] are byte-identical to that single call's code stream; any other status: length[i] = 0
 * and the image takes no bytes of the output.
 * The streams lie in image order in one device buffer the engine owns, each at a 256-byte boundary.  It is not the buffer
 * of b2k_encode_codestream_device, whose pointer a batch leaves valid; it stays valid until the next
 * b2k_encode_codestreams_device on e, or b2k_engine_destroy.
 * Stream order as b2k_encode_codestream_device: the images are read after the work queued on cuda_stream, which then
 * waits for the engine's last read of them; the call returns once the code streams are written.  Synchronisations: one
 * per call (statuses, offsets and lengths come home in one read), a second when the output buffer has to grow.  For a
 * fixed coding and flags the launch count does not depend on n once n x tiles reaches the pipeline's chunk count.
 * Returns < 0 for a failure of the whole call (NULL arrays, n == 0, imgs whose sample_bytes differ, a CUDA error, more
 * code blocks than one job indexes), b2k_last_error set; else the number of images whose status is not 0. */
B2K_API int32_t b2k_encode_codestreams_device(b2k_engine* e, const b2k_coding* cp, uint32_t n, const b2k_device_planes* imgs,
                                              uint32_t flags, void* cuda_stream, const uint8_t** cs, uint64_t* offset,
                                              uint64_t* length, int32_t* status, double* ms_total);
/* the b2k_last_error text of image i in the last b2k_encode_codestreams_device call on e ("" for status 0); valid until
   the next such call */
B2K_API const char* b2k_encode_codestreams_error(b2k_engine* e, uint32_t i);
/* A complete HTJ2K code stream in device memory (cs, len bytes, on the engine's GPU) -> the image in img.
 * Equal, for every input, to copying cs to the host and calling b2k_codestream_parse + b2k_decode_device:
 * the same return code, the same b2k_last_error text for 1 and -1, the same pixels for 0.  Only the main header (a
 * 64 KiB prefix, longer when the header is) and a small parse status cross PCIe; the tile parts and packet headers are
 * parsed by kernels.  cs is read after the work queued on cuda_stream, which then waits for the image writes. */
B2K_API int32_t b2k_decode_codestream_device(b2k_engine* e, const uint8_t* cs, uint64_t len, const b2k_device_planes* img,
                                             void* cuda_stream, b2k_coding* cp_out, double* ms_total);
/* A batch: n HTJ2K code streams in device memory, all with one coding -> n images in device memory, in one launch chain.
 * status[i] and b2k_decode_codestreams_error(e, i) are what b2k_decode_codestream_device(e, cs[i], len[i], &imgs[i], ...)
 * returns alone and its b2k_last_error text: 0, 1, -1 or -2, the checks in the same order (cs[i]'s memory, the main header,
 * the tile parts and packets, imgs[i], the HT decoder's verdict on stream i's blocks).  Status 0: imgs[i] holds exactly
 * the single call's pixels; any other status: imgs[i] is not written.
 * The batch's coding is that of the lowest-index stream whose main header parses (*cp_out receives it); another stream
 * whose header parses but whose b2k_coding, progression order, SOP or EPH differ gets status 1 with a text naming that
 * stream.  TLM, PLT, the tile-part layout and COM may differ from stream to stream.
 * imgs == NULL: headers only -- each stream is checked up to its main header and the coding match, and cp_out and the
 * statuses are filled from that.  Stream order as b2k_decode_codestream_device: every stream is read after the work queued
 * on cuda_stream, which then waits for the image writes.
 * Synchronisations: three per call (headers, parse statuses, end), one more for the streams whose main header runs past
 * the first few KiB, all together.  For a fixed coding the launch count does not depend on n once n x tiles reaches the
 * pipeline's chunk count.
 * Memory: the engine keeps the batch's job (n image-sized int32 plane sets for the transform, besides the arena) for the
 * next batch of the coding, beside the single-image job; a later batch of more streams, of fewer than a quarter as many,
 * or of another coding replaces it, and b2k_engine_destroy frees it.
 * Returns < 0 for a failure of the whole call (NULL arrays, n == 0, imgs whose sample_bytes differ, a CUDA error, more
 * code blocks than one job indexes), b2k_last_error set; else the number of streams whose status is not 0. */
B2K_API int32_t b2k_decode_codestreams_device(b2k_engine* e, uint32_t n, const uint8_t* const* cs, const uint64_t* len,
                                              const b2k_device_planes* imgs, void* cuda_stream, b2k_coding* cp_out,
                                              int32_t* status, double* ms_total);
/* the b2k_last_error text of stream i in the last b2k_decode_codestreams_device call on e ("" for status 0); valid until
   the next such call */
B2K_API const char* b2k_decode_codestreams_error(b2k_engine* e, uint32_t i);
/* Stage hook / size query: the block table b2k_codestream_parse would return for the same bytes (offsets into cs),
 * parsed by the device kernels.  blocks = NULL: read the main header only and return the block count (Python's
 * decode_codestream_device makes this call first when it needs the image's shape, so it reads the header twice). */
B2K_API int64_t b2k_codestream_parse_device(b2k_engine* e, const uint8_t* cs, uint64_t len, void* cuda_stream,
                                            b2k_coding* cp_out, b2k_block* blocks, uint64_t cap_blocks);
/* How the last device parse on this engine read its tiles: tiles whose packets were parsed one thread per packet from
 * their PLT packet starts, and tiles with data walked packet after packet (no PLT, a PLT that does not add up, or a packet
 * that did not end where PLT said).  The results do not depend on the split; the time does.  After a windowed device
 * parse, the counts are of the wanted tiles only. */
B2K_API int32_t b2k_codestream_parse_device_stats(b2k_engine* e, uint32_t* tiles_indexed, uint32_t* tiles_walked);

/* Windowed / reduced-resolution decode of a code stream in device memory: b2k_codestream_parse_window and
 * b2k_decode_window for a stream on the engine's GPU.  Equal, for every input, to copying cs to the host and calling
 * b2k_codestream_parse_window(cs, len, window, reduce, ...) + b2k_decode_device(virtual coding, blocks, ..., cs, ..., img,
 * rect): the same return code and b2k_last_error text, the same virtual coding, the same block table (offsets into cs),
 * the same pixels.  Every SOT of the stream is checked, but only the wanted tiles' tile-part headers and packets are read,
 * in place from cs, and only their packet data is copied, into the engine's arena: the cost follows the window, not the
 * stream.  A window that takes every tile at reduce 0 is the stream's own coding and takes b2k_decode_codestream_device's
 * path.  Ordering against cuda_stream, the check of cs and -2 for blocks the HT decoder rejects are as there.
 *
 * window = x0,y0,x1,y1 on the full-resolution canvas (NULL: whole image), reduce = highest resolutions to drop.
 * blocks == NULL: main header only, returns the block count and the virtual coding (as the host call does). */
B2K_API int64_t b2k_codestream_parse_window_device(b2k_engine* e, const uint8_t* cs, uint64_t len, const uint32_t* window,
                                                   uint32_t reduce, void* cuda_stream, b2k_coding* cp_out,
                                                   b2k_block* blocks, uint64_t cap_blocks);
/* img holds rect_out = the window's pixels at 1/2^reduce on cp_out's canvas: x0,y0,x1,y1 of the window divided by 2^reduce
 * (rounded up), clipped to the virtual image; the whole virtual image when window is NULL */
B2K_API int32_t b2k_decode_codestream_window_device(b2k_engine* e, const uint8_t* cs, uint64_t len, const uint32_t* window,
                                                   uint32_t reduce, const b2k_device_planes* img, void* cuda_stream,
                                                   b2k_coding* cp_out, uint32_t* rect_out, double* ms_total);
/* last windowed device parse: wanted tiles, and bytes of their tile parts copied into the job's arena (the packet data of
 * their tile parts; the whole stream when every tile was wanted at reduce 0) */
B2K_API int32_t b2k_codestream_window_device_stats(b2k_engine* e, uint32_t* tiles_wanted, uint64_t* arena_bytes);
/* A batch of windows: n HTJ2K code streams in device memory, each with its own window (windows[4 i .. 4 i + 3] = x0, y0,
 * x1, y1 on its full-resolution canvas; windows == NULL: every whole image) and one `reduce` -> n images in device memory,
 * in one launch chain.  status[i] and b2k_decode_codestreams_error(e, i) are what b2k_decode_codestream_window_device(e,
 * cs[i], len[i], &windows[4 i], reduce, &imgs[i], ...) returns alone and its b2k_last_error text, the checks in the same
 * order: cs[i]'s memory, the main header, the window (b2k_codestream_parse_window's window errors), the tile parts and
 * packets of the wanted tiles only (damage outside the window passes, as it does alone), imgs[i], the HT decoder's
 * verdict on stream i's blocks.  Status 0: imgs[i] holds exactly the single call's pixels and rects_out[4 i .. 4 i + 3]
 * is its rect_out; any other status (-2 included): imgs[i] is not written.
 * The batch's coding is the virtual coding of the lowest-index stream whose header and window pass (*cp_out receives it).
 * Another stream whose virtual coding, tile grid or wanted tiles differ, or whose progression order, SOP or EPH differ,
 * gets status 1 with a text naming that stream.  So any windows go together for single-tile streams (the box is always
 * the one tile); tiled streams go together when their windows touch the same tiles, e.g. one window for the whole batch.
 * Different tile boxes in one call are not supported.
 * imgs == NULL: headers only -- cp_out, rects_out and the statuses up to the coding match.  rects_out holds zeros for a
 * stream that fails before its window's coding.  Streams are read in place after the work queued on cuda_stream, which
 * then waits for the image writes; only the wanted tiles' packet data is copied, into the engine's arena.
 * Synchronisations: the header prefixes, the parse statuses, the end (as b2k_decode_codestreams_device).  For a fixed
 * virtual coding the launch count does not depend on n once n x tiles reaches the pipeline's chunk count.
 * Memory: the batch job of the virtual coding (n virtual-image-sized int32 plane sets), kept as b2k_decode_codestreams_device
 * keeps its own.  Returns < 0 for a failure of the whole call (NULL arrays, n == 0, imgs whose sample_bytes differ, a CUDA
 * error), b2k_last_error set; else the number of streams whose status is not 0.  b2k_codestream_window_device_stats then
 * reports the box's wanted tiles and the bytes gathered for all streams together. */
B2K_API int32_t b2k_decode_codestreams_window_device(b2k_engine* e, uint32_t n, const uint8_t* const* cs, const uint64_t* len,
                                                     const uint32_t* windows, uint32_t reduce, const b2k_device_planes* imgs,
                                                     void* cuda_stream, b2k_coding* cp_out, uint32_t* rects_out, int32_t* status,
                                                     double* ms_total);

/* Geometry only (host): enumerate the blocks of the selected tiles, lengths zero.  Returns the
 * count; fills at most cap entries. */
B2K_API int64_t b2k_enumerate(const b2k_coding* cp, uint32_t tile_mod, uint32_t tile_rem,
                              b2k_block* out, uint64_t cap);

/* Build / free the stock gpup_tile tree for ONE tile from a result (what gpup_encode_mem
 * returns; layout rules plugin_bridge.cpp L62-111). */
B2K_API gpup_tile* b2k_result_to_gpup_tile(const b2k_coding* cp, const b2k_result* r, uint32_t tile);

/* ---- device-resident path (inputs already in HBM; what bench.py's `value` times) ---------- */
typedef struct b2k_device_job b2k_device_job;
B2K_API int32_t b2k_job_create(b2k_engine* e, const b2k_coding* cp, uint32_t tile_mod,
                               uint32_t tile_rem, b2k_device_job** out);
B2K_API void b2k_job_destroy(b2k_device_job* j);
/* upload planes into the job's device image (untimed set-up for the device-resident bench) */
B2K_API int32_t b2k_job_upload(b2k_device_job* j, const int32_t* const* planes, const uint32_t* strides);
/* run stages on device-resident data; each returns 0 and the elapsed device ms via *ms */
B2K_API int32_t b2k_job_forward(b2k_device_job* j, float* ms);  /* DC shift+MCT+DWT, all levels */
B2K_API int32_t b2k_job_t1_encode(b2k_device_job* j, float* ms, uint64_t* total_bytes);
B2K_API int32_t b2k_job_t1_decode(b2k_device_job* j, float* ms);/* from the job's own coded blocks */
B2K_API int32_t b2k_job_inverse(b2k_device_job* j, float* ms);  /* inverse DWT+MCT into image */
/* all four stages enqueued back to back, one synchronisation; stage_ms[4] optional.  The first call after an upload
 * (or after b2k_job_inverse) sizes the byte arena for the job's image (one extra synchronising pass).  Returns 2 if the coded size outgrew the
 * arena (a 9/7 step codes the previous step's reconstruction): the arena has been resized, and the image planes hold
 * the reconstruction of a partial decode, so upload the image again before calling again.  The same holds for
 * b2k_job_roundtrip_n and b2k_job_roundtrip_pipelined_n. */
B2K_API int32_t b2k_job_roundtrip(b2k_device_job* j, float* ms_total, float* stage_ms, uint64_t* total_bytes);
/* `steps` round trips queued back to back with one synchronisation after the last (a benchmark loop without the
 * host in it); stage_ms[4] and level1_ms are sums over the steps, ms_total spans first start to last end. */
B2K_API int32_t b2k_job_roundtrip_n(b2k_device_job* j, uint32_t steps, float* ms_total, float* stage_ms, float* level1_ms,
                                    uint64_t* total_bytes);
/* the same round trips with the block-coder stage pipelined over `chunks` block ranges on `streams` side streams (0: the
 * defaults, 2 and 2): the transforms run alone, between them every range goes encode -> compact -> decode on its stream, so
 * the latency-bound kernels of one range run under the issue-bound kernels of its neighbours.  stage_ms[3] = forward, block
 * coder (encode + decode), inverse.  Results are those of b2k_job_roundtrip_n, byte for byte. */
B2K_API int32_t b2k_job_roundtrip_pipelined_n(b2k_device_job* j, uint32_t steps, uint32_t chunks, uint32_t streams, float* ms_total,
                                              float* stage_ms, float* level1_ms, uint64_t* total_bytes);
B2K_API int32_t b2k_job_download(b2k_device_job* j, int32_t* const* planes, const uint32_t* strides);
/* copy the coefficient planes (Mallat layout per tile, image-shaped, int32 or float bits) */
B2K_API int32_t b2k_job_download_coeffs(b2k_device_job* j, int32_t* const* planes, const uint32_t* strides);
B2K_API int32_t b2k_job_upload_coeffs(b2k_device_job* j, const int32_t* const* planes, const uint32_t* strides);
/* block-decode a caller-supplied block table + byte arena (as b2k_decode takes them) into the job's
 * coefficient planes; 1 = not handled (e.g. more than 3 HT passes), < 0 failure */
B2K_API int32_t b2k_job_t1_decode_blocks(b2k_device_job* j, const b2k_block* blocks, uint64_t num_blocks,
                                         const uint8_t* bytes, uint64_t num_bytes, float* ms);
/* fetch coded blocks of the last b2k_job_t1_encode as a host result */
B2K_API int32_t b2k_job_fetch_result(b2k_device_job* j, b2k_result** out);
B2K_API uint64_t b2k_job_num_blocks(const b2k_device_job* j);
/* Merge per-rank results (rank r coded the tiles t with t % nshards == r) into one result in full enumeration order,
 * for the writer rank after it has gathered the shards (block tables + byte arenas).  Free with b2k_result_free. */
B2K_API int32_t b2k_result_merge(const b2k_coding* cp, const b2k_result* const* shards, uint32_t nshards, b2k_result** out);

/* ---- codestream assembly / parsing on the host (SURVEY.md 8f N1: the T2 step) -------------------------
 * b2k_codestream_write: a complete HTJ2K codestream (SOC, SIZ, CAP, COD, QCD, [TLM], per tile SOT [PLT] SOD
 * + packets, EOC; one layer, any of the five progression orders, optionally a tile part per resolution) from an
 * encode result that holds every tile
 * (cf. CodeStreamCompress::compress / T2Compress::compressPacket).  Returns the size; copies it to `out` if
 * cap suffices (call with out = NULL to size the buffer).  < 0 on error.
 * b2k_codestream_parse: main header -> *cp, packet headers -> block table in enumeration order with
 * numbps / numpasses / length / length2 and offsets INTO `cs`, so that b2k_decode(engine, cp, blocks, n, cs,
 * len, ...) decodes the file in place.  Returns the number of blocks (call with blocks = NULL to size the
 * table), 1 if the codestream uses something this path does not cover (b2k_last_error says what), < 0 if it
 * is damaged. */
#define B2K_CS_TLM 1u
#define B2K_CS_PLT 2u
#define B2K_CS_SOP 16u                     /* SOP marker segment before every packet */
#define B2K_CS_EPH 32u                     /* EPH marker after every packet header */
#define B2K_CS_TPARTS_R 4u                 /* one tile part per resolution (LRCP / RLCP / RPCL only), cf. grk_compress -u R */
#define B2K_CS_PROG(n) (((n) & 7u) << 8)   /* progression order: 0 LRCP (default), 1 RLCP, 2 RPCL, 3 PCRL, 4 CPRL */
B2K_API int64_t b2k_codestream_write(const b2k_coding* cp, const b2k_result* r, uint32_t flags, uint8_t* out, uint64_t cap);
B2K_API int64_t b2k_codestream_parse(const uint8_t* cs, uint64_t len, b2k_coding* cp, b2k_block* blocks, uint64_t cap_blocks);
/* Per-rank writers (tiles sharded over ranks, SURVEY.md 8e): every rank turns ITS tiles (t % tile_mod == tile_rem, the result
 * b2k_encode gave it) into finished tile parts -- consecutive in tile order in `out`, tile_bytes[k] = length of the k-th of its
 * tiles -- and the writer rank only needs the lengths of all tiles for the header (+ TLM): code stream = header + tile parts in
 * tile-index order + 0xFFD9, byte-identical to b2k_codestream_write over the merged result.  One tile part per tile. */
B2K_API int64_t b2k_codestream_write_tiles(const b2k_coding* cp, const b2k_result* shard, uint32_t flags, uint32_t tile_mod,
                                           uint32_t tile_rem, uint8_t* out, uint64_t cap, uint64_t* tile_bytes);
B2K_API int64_t b2k_codestream_write_header(const b2k_coding* cp, uint32_t flags, const uint64_t* tile_bytes, uint32_t ntiles,
                                            uint8_t* out, uint64_t cap);
/* as b2k_codestream_write_tiles, the k-th of the shard's tiles written at out + tile_at[k] */
B2K_API int64_t b2k_codestream_write_tiles_at(const b2k_coding* cp, const b2k_result* shard, uint32_t flags, uint32_t tile_mod,
                                              uint32_t tile_rem, uint8_t* out, uint64_t cap, const uint64_t* tile_at);
/* Windowed / reduced-resolution decode (SURVEY.md 8f N3), tile-granular: `window` = x0,y0,x1,y1 on the full-resolution
 * canvas (NULL: whole image), `reduce` = highest resolutions to drop.  *cp becomes a VIRTUAL coding: the image made of the
 * tiles the window touches, at 1 / 2^reduce of the resolution -- decode it with b2k_decode(cp, blocks, ..., cs, ...) into
 * planes of (cp->x1 - cp->x0) x (cp->y1 - cp->y0) samples and crop: window column x (reduced resolution, x >=
 * ceil(wx0 / 2^reduce)) is plane column x - cp->x0.  Only the wanted tiles' packets are parsed and decoded.  Return as
 * b2k_codestream_parse (reduce > 0 needs a tile grid aligned to 2^reduce: 1 = not handled otherwise). */
B2K_API int64_t b2k_codestream_parse_window(const uint8_t* cs, uint64_t len, const uint32_t* window, uint32_t reduce, b2k_coding* cp,
                                            b2k_block* blocks, uint64_t cap_blocks);

/* JPH container (JP2 boxes, brand 'jph '): wrap a codestream / find the codestream inside a .jph / .jp2 file
 * (a raw codestream is accepted as it is). */
B2K_API int64_t b2k_jph_wrap(const b2k_coding* cp, const uint8_t* cs, uint64_t cs_len, uint8_t* out, uint64_t cap);
B2K_API int32_t b2k_jph_codestream(const uint8_t* file, uint64_t len, uint64_t* offset, uint64_t* length);

/* ---- streaming (SURVEY.md 8f N2): `depth` frames in flight on one GPU, so that frame k+1's host->device copies
 * overlap frame k's kernels and device->host copies.  Each of the `depth` workers is a host thread with its own engine;
 * a submit hands the frame to an idle worker (and blocks while all are busy); results come back through the callback on
 * that worker's thread, possibly out of submission order.  The caller's planes / code-stream bytes are NOT copied: they
 * must stay valid and unchanged until the frame's callback has run.
 *   on_encoded: `result` is valid during the call; return non-zero to keep it (then free it with b2k_result_free).
 * b2k_stream_end drains the stream, joins the workers, frees everything; returns the first device error (< 0) or 0. */
typedef struct b2k_stream b2k_stream;
typedef int32_t (*b2k_encoded_fn)(void* user, void* frame_user, b2k_result* result, int32_t status);
typedef void (*b2k_decoded_fn)(void* user, void* frame_user, int32_t status);
#define B2K_SAMPLES_U16_INTERLEAVED 0x102u /* sample_bytes of an encode stream fed b2k_encode16_interleaved frames: planes[0] = pixels */
B2K_API int32_t b2k_stream_encode_begin(int32_t device, const b2k_coding* cp, uint32_t depth, uint32_t sample_bytes /* 2, 4 or B2K_SAMPLES_U16_INTERLEAVED */,
                                        b2k_encoded_fn on_encoded, void* user, b2k_stream** out);
B2K_API int32_t b2k_stream_encode_submit(b2k_stream* s, const void* const* planes, const uint32_t* strides, void* frame_user);
B2K_API int32_t b2k_stream_decode_begin(int32_t device, uint32_t depth, uint32_t sample_bytes /* 2 or 4 */, b2k_decoded_fn on_decoded,
                                        void* user, b2k_stream** out);
B2K_API int32_t b2k_stream_decode_submit(b2k_stream* s, const b2k_coding* cp, const b2k_block* blocks, uint64_t num_blocks,
                                         const uint8_t* bytes, uint64_t num_bytes, void* const* planes, const uint32_t* strides,
                                         void* frame_user);
B2K_API int32_t b2k_stream_decode_submit_codestream(b2k_stream* s, const uint8_t* codestream, uint64_t length, uint32_t numcomps,
                                                    void* const* planes, const uint32_t* strides, void* frame_user);
B2K_API int32_t b2k_stream_end(b2k_stream* s);

/* launches issued by this library since engine creation (bench.py "gpu_launches") */
B2K_API uint64_t b2k_launch_count(void);
/* per-kernel timing of the last forward()/inverse(): ms of the level-1 kernel and algorithmic
 * bytes it moved (for the roofline line of bench.py) */
B2K_API int32_t b2k_job_last_kernel_stats(const b2k_device_job* j, int which, float* ms, uint64_t* alg_bytes);

#ifdef __cplusplus
}
#endif
#endif /* GROK_B200_H */
