/*
 * grok_b200/csrc/t2_decode.h -- the device code-stream parser (t2_decode.cu) as the engine drives it.
 */
#pragma once
#include <vector>
#include "b2k_internal.h"
#include "t2_plan.h"

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

/* ---- windowed parse (b2k_codestream_parse_window on a stream in device memory) ----------------------------------------
 * The plan is the box coding's (wc.box: the wanted tiles at full resolution), so the same five launches parse exactly the
 * wanted tiles' packets; the virtual coding's blocks vblocks[0, nv) map onto box blocks, and its coded blocks
 * vblocks[coded_index[k]] get descriptors.  Keyed by the box coding, flags and reduce.  0, or -1 with b2k_last_error set. */
int b2k_t2_window_create(const b2k::t2::WindowCoding& wc, uint32_t flags, uint32_t reduce, const b2k_block* vblocks, uint64_t nv,
                         const uint32_t* coded_index, uint64_t ncoded, T2Parse** out);
bool b2k_t2_window_matches(const T2Parse* j, const b2k_coding& box, uint32_t flags, uint32_t reduce);
/* on st: the parse of cs[0, len) (read in place) for the wanted tiles of a stream of ntiles tiles, grid_nx wide, with
   wc's need rectangles; the descriptors address the packet data as b2k_t2_window_gather lays it out */
int b2k_t2_window_enqueue(T2Parse* j, const uint8_t* cs, uint64_t len, uint64_t sot, uint32_t grid_nx, uint32_t ntiles,
                          const b2k::t2::WindowCoding& wc, const HtBlockDesc* d_enc, const float* d_quant, HtBlockDesc* d_dec,
                          cudaStream_t st);
/* after the status: bytes of packet data in the wanted tiles' parts */
uint64_t b2k_t2_window_bytes(const T2Parse* j);
/* on st, one launch: those bytes from cs, end to end, into out (b2k_t2_window_bytes of them) */
int b2k_t2_window_gather(const T2Parse* j, const uint8_t* cs, uint8_t* out, cudaStream_t st);
/* after a result of 0: b2k_codestream_parse_window's block table (offsets into cs) of the virtual coding into out[0, nv) */
int b2k_t2_window_blocks(const T2Parse* j, const b2k_block* vblocks, uint64_t nv, const std::vector<b2k::Rect>& need, b2k_block* out,
                         cudaStream_t st);
