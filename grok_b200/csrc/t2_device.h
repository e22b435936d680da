/*
 * grok_b200/csrc/t2_device.h -- the device code-stream writer (t2_device.cu) as the engine drives it.
 */
#pragma once
#include "b2k_internal.h"

struct T2Job; /* a job's plan and device buffers for one set of code-stream flags and up to `streams` code streams */

/* plan + device buffers for the job whose block table (enumeration order, one image's) is `blocks` and whose coded blocks
   are blocks[coded_index[k]]; streams: the code streams one enqueue may write, coded block k of stream s being the coder's
   output s * ncoded + k.  0; 1 when b2k_t2_plan declines, -1 for a CUDA failure, b2k_last_error set (for 1 as
   b2k_codestream_write sets it). */
int b2k_t2_create(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles,
                  const uint32_t* coded_index, uint64_t ncoded, T2Job** out, uint32_t streams = 1);
void b2k_t2_destroy(T2Job* j);
uint32_t b2k_t2_flags(const T2Job* j);
uint32_t b2k_t2_streams(const T2Job* j);
/* n <= streams code streams of the coder's output (d_out, scratch slots) into cs[0, cap) on st, then their statuses and
   placement to the host; a constant number of launches.  Stream s starts at a 256-byte boundary behind stream s - 1; a
   stream with a verdict takes no bytes.  Nothing is written beyond cap: when b2k_t2_used exceeds it, grow cs and enqueue
   again. */
int b2k_t2_enqueue(T2Job* j, const HtBlockDesc* d_enc, const HtBlockOut* d_out, const uint8_t* d_scratch, uint8_t* cs, uint64_t cap,
                   cudaStream_t st, uint32_t n = 1);
/* once st has reached the end of b2k_t2_enqueue's work: stream s's length, or -2 (blocks overflowed the coder) / -1 (the
   writer's limits) with b2k_last_error set as b2k_encode_device / b2k_codestream_write set it */
int64_t b2k_t2_result(const T2Job* j, uint32_t s = 0);
/* likewise: where stream s starts in cs, and the bytes from cs to the end of the last stream with a length */
uint64_t b2k_t2_offset(const T2Job* j, uint32_t s);
uint64_t b2k_t2_used(const T2Job* j);
