/*
 * grok_b200/csrc/t2_decode.h -- the device code-stream parser (t2_decode.cu) as the engine drives it.
 */
#pragma once
#include <vector>
#include "b2k_internal.h"
#include "t2_plan.h"
#include "t2_parse.h"

struct T2Parse; /* a job's packet plan and device buffers for one progression order and SOP / EPH setting */

/* plan + device buffers for the coding whose block table (enumeration order) is `blocks` and whose coded blocks are
   blocks[coded_index[k]]; flags: the stream's progression order (B2K_CS_PROG) and SOP / EPH.  0, or -1 with
   b2k_last_error set. */
int b2k_t2_parse_create(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles,
                        const uint32_t* coded_index, uint64_t ncoded, T2Parse** out, uint32_t streams = 1);
void b2k_t2_parse_destroy(T2Parse* j);
uint32_t b2k_t2_parse_flags(const T2Parse* j);
/* once st has reached the end of b2k_t2_window_enqueue's work: 0, or b2k_codestream_parse's return code with its text;
   *refinement: a block has refinement passes to decode */
int b2k_t2_parse_result(const T2Parse* j, bool* refinement);
/* ---- streams of one coding (a single stream is a batch of one), a parse made with `streams` >= n --------------------
 * On st: the parse of the n code streams arena[at[s], at[s] + len[s]) whose first SOT is at sot[s] (sot[s] = 0: stream s
 * failed before its tile parts and is not parsed), in five launches whatever the tile count, then (d_dec != NULL)
 * descriptor s * ncoded + k of every stream's coded block k from d_enc's templates and d_quant's step sizes of the same
 * index, pointing into the arena.  A stream that fails, or is not parsed, gets length-0 descriptors (all-zero blocks).
 * The statuses to the host. */
int b2k_t2_batch_enqueue(T2Parse* j, const uint8_t* arena, uint32_t n, const uint64_t* at, const uint64_t* len, const uint64_t* sot,
                         const HtBlockDesc* d_enc, const float* d_quant, HtBlockDesc* d_dec, cudaStream_t st);
/* once the statuses have arrived: stream s's b2k_codestream_parse return code (its text set when not 0) */
int b2k_t2_batch_result(const T2Parse* j, uint32_t s, bool* refinement);
uint32_t b2k_t2_parse_streams(const T2Parse* j);
/* one entry of a gather: len bytes from device address src to out + dst */
struct CopyEntry
{
  const uint8_t* src;
  uint64_t len, dst;
};
/* on st, one launch: every entry of the device table d_tab[0, n) (none longer than max_len) */
int b2k_copy_table(const CopyEntry* d_tab, uint32_t n, uint64_t max_len, uint8_t* out, cudaStream_t st);

/* after the status has arrived (over the streams of the last enqueue): tiles parsed packet by packet from their PLT starts, and tiles walked */
void b2k_t2_parse_stats(const T2Parse* j, uint32_t* indexed, uint32_t* walked);
/* after a result of 0: the block table b2k_codestream_parse returns (offsets into cs) into out[0, nblocks) */
int b2k_t2_parse_blocks(const T2Parse* j, b2k_block* out, cudaStream_t st);

/* ---- windowed parse (b2k_codestream_parse_window on streams in device memory; a single stream is a batch of one) -------
 * The plan is the box coding's (wc.box: the wanted tiles at full resolution), so the same five launches parse exactly the
 * wanted tiles' packets of every stream; the virtual coding's blocks vblocks[0, nv) map onto box blocks, and its coded
 * blocks vblocks[coded_index[k]] get descriptors.  Keyed by the box coding, flags, reduce and the stream capacity.  0, or
 * -1 with b2k_last_error set. */
int b2k_t2_window_create(const b2k::t2::WindowCoding& wc, uint32_t flags, uint32_t reduce, const b2k_block* vblocks, uint64_t nv,
                         const uint32_t* coded_index, uint64_t ncoded, T2Parse** out, uint32_t streams = 1);
bool b2k_t2_window_matches(const T2Parse* j, const b2k_coding& box, uint32_t flags, uint32_t reduce, uint32_t streams);
/* on st: the parse of the n streams cs[s][0, len[s]) (read in place, each from its own buffer; sot[s] = 0: not parsed) for
   the tiles of `box` among each stream's ntiles, with need[s]'s rectangles (NULL or empty: no filter); with d_dec the
   arena layout (each stream's gathered packet data at a 256-byte boundary) and descriptor s * ncoded + k of every stream's
   coded block k, addressing the bytes where b2k_t2_window_gather puts them.  The statuses to the host. */
int b2k_t2_window_enqueue(T2Parse* j, uint32_t n, const uint8_t* const* cs, const uint64_t* len, const uint64_t* sot,
                          const std::vector<b2k::Rect>* const* need, const b2k::t2::TileBox& box, uint32_t ntiles,
                          const HtBlockDesc* d_enc, const float* d_quant, HtBlockDesc* d_dec, cudaStream_t st);
/* after the status: bytes of packet data in the wanted tiles' parts, over the streams that parsed */
uint64_t b2k_t2_window_bytes(const T2Parse* j);
/* after the status: the arena bytes the gather lays the streams' packet data out in (the decoder's slack not included) */
uint64_t b2k_t2_window_arena(const T2Parse* j);
/* on st, one launch: the packet data of the streams that parsed, from their buffers into out as the descriptors address it */
int b2k_t2_window_gather(const T2Parse* j, uint8_t* out, cudaStream_t st);
/* after a result of 0 (a batch of one): b2k_codestream_parse_window's block table (offsets into cs) of the virtual coding
   into out[0, nv) */
int b2k_t2_window_blocks(const T2Parse* j, const b2k_block* vblocks, uint64_t nv, const std::vector<b2k::Rect>& need, b2k_block* out,
                         cudaStream_t st);
