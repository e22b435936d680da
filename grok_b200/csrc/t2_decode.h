/*
 * grok_b200/csrc/t2_decode.h -- the device code-stream parser (t2_decode.cu) as the engine drives it.
 */
#pragma once
#include "b2k_internal.h"

struct T2Parse; /* a job's packet plan and device buffers for one progression order and SOP / EPH setting */

/* plan + device buffers for the coding whose block table (enumeration order) is `blocks` and whose coded blocks are
   blocks[coded_index[k]]; flags: the stream's progression order (B2K_CS_PROG) and SOP / EPH.  0, or -1 with
   b2k_last_error set. */
int b2k_t2_parse_create(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles,
                        const uint32_t* coded_index, uint64_t ncoded, T2Parse** out);
void b2k_t2_parse_destroy(T2Parse* j);
uint32_t b2k_t2_parse_flags(const T2Parse* j);
/* on st: the parse of the code stream cs[0, len) in device memory, whose first SOT is at sot, then (d_dec != NULL) the
   decoder's descriptors of the coded blocks from d_enc's templates and d_quant's step sizes; the status to the host.
   Five launches, whatever the tile count. */
int b2k_t2_parse_enqueue(T2Parse* j, const uint8_t* cs, uint64_t len, uint64_t sot, const HtBlockDesc* d_enc, const float* d_quant,
                         HtBlockDesc* d_dec, cudaStream_t st);
/* once st has reached the end of b2k_t2_parse_enqueue's work: 0, or b2k_codestream_parse's return code with its text;
   *refinement: a block has refinement passes to decode */
int b2k_t2_parse_result(const T2Parse* j, bool* refinement);
/* after the status has arrived: tiles parsed packet by packet from their PLT starts, and tiles walked */
void b2k_t2_parse_stats(const T2Parse* j, uint32_t* indexed, uint32_t* walked);
/* after a result of 0: the block table b2k_codestream_parse returns (offsets into cs) into out[0, nblocks) */
int b2k_t2_parse_blocks(const T2Parse* j, b2k_block* out, cudaStream_t st);
