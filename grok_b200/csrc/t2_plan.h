/*
 * grok_b200/csrc/t2_plan.h -- what the code-stream writer (t2_write.h, on the device and on the host) needs to know about
 * an image's code stream before any block is coded: its packets in code-stream order, its tile parts and its main header.
 * Geometry and flags only, so one plan serves every frame of a job.  Built on the host (codestream.cpp) by b2k_t2_plan,
 * or for a shard's tiles by the per-rank writers; the device parser reads its packets too.
 */
#pragma once
#include <stdint.h>
#include <vector>
#include "t2_packet.h"
#include "geometry.h"
#include "../../include/grok_b200.h"

namespace b2k
{
namespace t2
{
struct DevPacket /* one packet, in code-stream order */
{
  BandGrid band[3];  /* band[b].first: index into the image's block enumeration */
  uint32_t nbands;
  uint32_t sop;      /* SOP counter: the packet's index in its tile, modulo 65536 */
  uint32_t hdr_cap;  /* header bytes reserved (packet_header_bound) */
  uint64_t hdr_at;   /* where they are reserved in the header scratch */
  uint64_t tag_at;   /* its tag-tree scratch, in nodes (packet_tag_nodes) */
};
struct DevPart /* one tile part, in code-stream order: packets [p0, p1) */
{
  uint64_t p0, p1;
  uint32_t tile, index, count; /* tile index, index of the part in its tile, tile parts of the tile */
};
struct Plan
{
  uint32_t flags = 0;
  std::vector<uint8_t> head; /* SOC .. QCD, then the TLM segments with their entries zero */
  uint64_t tlm_at = 0;       /* where the TLM segments start in head */
  std::vector<DevPacket> packets;
  std::vector<DevPart> parts;
  uint64_t hdr_bytes = 0, tag_nodes = 0;
};
struct MainHeader /* what a code stream's main header says (b2k_parse_main_header) */
{
  b2k_coding cp{};
  int progression = 0;
  bool sop = false, eph = false;
  uint64_t sot = 0;        /* where the first SOT starts */
  bool short_read = false; /* the failure came from reaching the end of the bytes given */
  /* the B2K_CS_* flags a plan of this stream's packets is made with */
  uint32_t flags() const { return B2K_CS_PROG(progression) | (sop ? B2K_CS_SOP : 0u) | (eph ? B2K_CS_EPH : 0u); }
};
/* what a window and a reduce make of a stream's coding (b2k_window_coding) */
struct WindowCoding
{
  bool whole = false;                 /* every tile at full resolution: the stream's own coding, nothing filtered */
  uint32_t ta_x = 0, ta_y = 0;        /* the wanted tiles: columns [ta_x, tb_x), rows [ta_y, tb_y) of the stream's grid */
  uint32_t tb_x = 0, tb_y = 0;
  b2k_coding vcp{};                   /* the coding to decode with (the virtual image) */
  b2k_coding box{};                   /* the box coding: the wanted tiles at full resolution with the stream's numres, whose
                                         tiles, precincts and packets are those of the stream's tiles */
  std::vector<Rect> need;             /* per resolution of vcp: the samples the window depends on; empty: no filter */
};
} // namespace t2
} // namespace b2k

/* the main header of cs[0, len), read by b2k_codestream_parse's own code: 0, or its return code with b2k_last_error set */
int b2k_parse_main_header(const uint8_t* cs, uint64_t len, b2k::t2::MainHeader& h);

/* a batch of code streams (b2k_decode_codestreams_device) takes the coding of stream ref_index, whose main header is ref:
   0 when stream `index` (main header h) may join it, else 1 with b2k_last_error naming both streams (another b2k_coding, or
   another progression order, SOP or EPH) */
int b2k_batch_coding_check(const b2k::t2::MainHeader& ref, uint32_t ref_index, const b2k::t2::MainHeader& h, uint32_t index);

/* a windowed batch (b2k_decode_codestreams_window_device) takes the window coding ref_wc of stream ref_index (main header
   ref): 0 when stream `index` (main header h, window coding wc) may join it -- the same virtual coding, box coding, tile
   grid and wanted tiles, progression order, SOP and EPH -- else 1 with b2k_last_error naming both streams */
int b2k_batch_window_check(const b2k::t2::MainHeader& ref, const b2k::t2::WindowCoding& ref_wc, uint32_t ref_index,
                           const b2k::t2::MainHeader& h, const b2k::t2::WindowCoding& wc, uint32_t index);

/* the wanted tiles, the virtual coding and the window's need rectangles of b2k_codestream_parse_window(window, reduce) on a
   stream of coding cp: 0, or its return code and text for the window errors, in its order */
int b2k_window_coding(const b2k_coding& cp, const uint32_t* window, uint32_t reduce, b2k::t2::WindowCoding& w);

/* the box coding's block enumeration, and for each of the virtual coding's blocks vblocks[0, nv) (enumeration order) the
   box block it is: the box tile's blocks of the resolutions vcp keeps, in order.  0, or -1 with the host parser's text when
   the two enumerations disagree. */
int b2k_window_blocks(const b2k::t2::WindowCoding& w, const b2k_block* vblocks, uint64_t nv, std::vector<b2k_block>& box_blocks,
                      std::vector<uint32_t>& vmap);

/* the plan of the code stream b2k_codestream_write(cp, r, flags) writes, for the block table `blocks` (every block of the
   tiles of r, enumeration order) and r->num_tiles = num_tiles.  0, or -1 with b2k_last_error set in the cases, and with the
   text, of b2k_codestream_write. */
int b2k_t2_plan(const b2k_coding& cp, uint32_t flags, const b2k_block* blocks, uint64_t nblocks, uint32_t num_tiles, b2k::t2::Plan& plan);
