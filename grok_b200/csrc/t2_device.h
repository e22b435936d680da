/*
 * grok_b200/csrc/t2_device.h -- the device code-stream writer (t2_device.cu) as the engine drives it.
 */
#pragma once
#include "b2k_internal.h"

struct T2Job; /* a job's plan and device buffers for one set of code-stream flags */
struct T2Status
{
  uint64_t total;      /* code-stream length */
  uint32_t bad_blocks; /* blocks that overflowed the coder */
  uint32_t errors;
};

/* plan + device buffers for the job whose block table (enumeration order) is `blocks` and whose coded blocks are
   blocks[coded_index[k]].  0, or -1 with b2k_last_error set as b2k_codestream_write sets it. */
int b2k_t2_create(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles,
                  const uint32_t* coded_index, uint64_t ncoded, T2Job** out);
void b2k_t2_destroy(T2Job* j);
uint32_t b2k_t2_flags(const T2Job* j);
/* the code stream of the coder's output (d_out, scratch slots) into cs[0, cap) on st, then its status to the host; a
   constant number of launches.  Nothing is written beyond cap: when the length exceeds it, grow cs and enqueue again. */
int b2k_t2_enqueue(T2Job* j, const HtBlockDesc* d_enc, const HtBlockOut* d_out, const uint8_t* d_scratch, uint8_t* cs, uint64_t cap,
                   cudaStream_t st);
/* once st has reached the end of b2k_t2_enqueue's work: the code-stream length, or -2 (blocks overflowed the coder) /
   -1 (the writer's limits) with b2k_last_error set as b2k_encode_device / b2k_codestream_write set it */
int64_t b2k_t2_result(const T2Job* j);
