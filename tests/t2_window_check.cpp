/*
 * tests/t2_window_check.cpp -- the windowed device parse (engine.cu b2k_codestream_parse_window_device, t2_decode.cu) run
 * on the host in the order of its steps: the window's coding (b2k_window_coding), the box coding's plan and block map
 * (b2k_t2_plan, b2k_window_blocks), the box-aware tile-part walk (locate_tile_parts_box), PLT packet starts, one packet
 * at a time from them, the walk for the tiles not indexed or marked, then the descriptor rule: the virtual block's box
 * block, the need filter and the offset into the gathered packet data.  Compared with b2k_codestream_parse_window on the
 * same bytes.  Built with g++ together with codestream.cpp and geometry.cpp (test_t2_window_host.py), under the address
 * and undefined-behaviour sanitizers, so that every byte read is checked against the stream's bounds.
 *
 *   t2_window_check LIST   LIST holds one case per line: "<file> <reduce> -" (no window) or "<file> <reduce> x0 y0 x1 y1".
 *                          Prints one line per case: "<file> <reduce> <window> <rc> <wanted tiles> <gathered bytes> same
 *                          <text>" or what differs; exit 1 on any difference
 */
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <fstream>
#include <functional>
#include <sstream>
#include <string>
#include <vector>

#include "geometry.h"
#include "t2_parse.h"
#include "t2_plan.h"

using namespace b2k;
using namespace b2k::t2;

static std::string g_err;
void b2k_set_error(const char* m) { g_err = m ? m : ""; }
extern "C" const char* b2k_last_error(void) { return g_err.c_str(); }
void b2k_host_parallel(size_t n, const std::function<void(size_t)>& fn)
{
  for(size_t i = 0; i < n; ++i)
    fn(i);
}
extern "C" int64_t b2k_codestream_parse_window(const uint8_t* cs, uint64_t len, const uint32_t* window, uint32_t reduce, b2k_coding* cp_out,
                                               b2k_block* blocks, uint64_t cap_blocks);

struct Stats
{
  uint32_t wanted = 0;
  uint64_t bytes = 0;
};

static int fail_with(uint32_t r)
{
  b2k_set_error(parse_reason_text(r));
  return parse_reason_rc(r);
}

/* the device's verdict and table for a window, computed as its steps compute them; out == NULL: the header-only call */
static int64_t device_order_window(const uint8_t* cs, uint64_t len, const uint32_t* window, uint32_t reduce, b2k_coding& vcp,
                                   std::vector<b2k_block>* out, Stats& st)
{
  MainHeader h;
  if(int rc = b2k_parse_main_header(cs, len, h))
    return rc;
  WindowCoding wc;
  if(int rc = b2k_window_coding(h.cp, window, reduce, wc))
    return rc;
  vcp = wc.vcp;
  const TileGrid vg = tile_grid(vcp);
  const uint32_t vnt = vg.nx * vg.ny;
  std::vector<b2k_block> vblocks;
  const std::vector<BandQuant> vq = band_quant(vcp);
  for(uint32_t t = 0; t < vnt; ++t)
    enumerate_tile_blocks(vcp, t, tile_rect(vcp, vg, t), vq, vblocks);
  if(!out)
    return (int64_t)vblocks.size();
  /* the plan: the box coding's packets, and the virtual blocks' box blocks */
  std::vector<b2k_block> blocks;
  std::vector<uint32_t> vmap;
  if(b2k_window_blocks(wc, vblocks.data(), vblocks.size(), blocks, vmap))
    return -1;
  const TileGrid bg = tile_grid(wc.box);
  const uint32_t bnt = bg.nx * bg.ny;
  if(bnt != vnt)
    return -101;
  st.wanted = bnt;
  Plan plan;
  if(b2k_t2_plan(wc.box, B2K_CS_PROG(h.progression), blocks.data(), blocks.size(), bnt, plan))
    return -1;
  /* kernel 1: every SOT, the wanted tiles' parts */
  const TileGrid g = tile_grid(h.cp);
  const uint32_t ntiles = g.nx * g.ny;
  const uint64_t cap = std::min<uint64_t>(len / 12 + 1, 256ull * bnt);
  std::vector<PartRange> parts(cap);
  std::vector<uint64_t> body_at(cap);
  std::vector<uint32_t> head(bnt), last(bnt), count(ntiles);
  uint32_t nparts = 0;
  if(uint32_t r = locate_tile_parts_box(cs, len, h.sot, ntiles, TileBox{g.nx, wc.ta_x, wc.ta_y, wc.tb_x, wc.tb_y}, parts.data(), cap,
                                        head.data(), last.data(), count.data(), &nparts, body_at.data(), &st.bytes))
    return fail_with(r);
  std::vector<uint8_t> kmax(blocks.size());
  for(size_t i = 0; i < blocks.size(); ++i)
    kmax[i] = blocks[i].kmax;
  std::vector<ParsedBlock> pb(blocks.size());
  std::vector<TagNode> tags(plan.tag_nodes + 1);
  const uint64_t np = plan.packets.size();
  std::vector<uint64_t> start(np), end(np), part_end(np);
  std::vector<uint8_t> indexed(bnt), marked(bnt);
  /* kernel 2: packet starts from PLT */
  for(uint32_t t = 0; t < bnt; ++t)
  {
    const DevPart& T = plan.parts[t];
    indexed[t] = plt_index(cs, parts.data(), head[t], T.p1 - T.p0, start.data() + T.p0, end.data() + T.p0, part_end.data() + T.p0);
  }
  /* kernel 3: one packet at a time from its PLT start */
  for(uint32_t t = 0; t < bnt; ++t)
    for(uint64_t k = plan.parts[t].p0; indexed[t] && k < plan.parts[t].p1; ++k)
    {
      uint64_t at = start[k];
      if(parse_packet(cs, plan.packets[k], &at, part_end[k], kmax.data(), pb.data(), tags.data() + plan.packets[k].tag_at, h.sop, h.eph) ||
         at != end[k])
        marked[t] = 1;
    }
  /* kernel 4: the walk; the lowest failing wanted tile decides */
  uint32_t first_err = PR_NONE;
  for(uint32_t t = 0; t < bnt; ++t)
  {
    const DevPart& T = plan.parts[t];
    if(T.p1 == T.p0 || (indexed[t] && !marked[t]))
      continue;
    for(uint64_t i = 0; i < blocks.size(); ++i)
      if(blocks[i].tile == t)
        pb[i] = ParsedBlock{};
    const uint32_t r = parse_tile(cs, parts.data(), head[t], plan.packets.data() + T.p0, T.p1 - T.p0, kmax.data(), pb.data(),
                                  tags.data() + plan.packets[T.p0].tag_at, h.sop, h.eph);
    if(r && !first_err)
      first_err = r;
  }
  if(first_err)
    return fail_with(first_err);
  /* the gather: the wanted parts' packet data end to end (k_t2_gather) */
  std::vector<uint8_t> arena(st.bytes);
  for(uint32_t p = 0; p < nparts; ++p)
    if(parts[p].end > parts[p].begin)
    {
      if(body_at[p] + (parts[p].end - parts[p].begin) > st.bytes)
        return -102;
      memcpy(arena.data() + body_at[p], cs + parts[p].begin, parts[p].end - parts[p].begin);
    }
  /* kernel 5: the virtual block's box block, the need filter, the offset into the gathered data */
  for(size_t i = 0; i < vblocks.size(); ++i)
  {
    b2k_block& v = vblocks[i];
    const ParsedBlock& b = pb[vmap[i]];
    bool wanted = true;
    if(!wc.need.empty())
    {
      const Rect& n = wc.need[v.resno ? v.resno - 1 : 0];
      const uint32_t r[4] = {n.x0, n.y0, n.x1, n.y1};
      wanted = window_needs(r, v.x0, v.y0, v.x1, v.y1);
    }
    if(!wanted)
      continue;
    if(b.length)
    { /* the decoder reads the block's segments where the gather put them */
      const uint64_t at = gathered_offset(parts.data(), head[v.tile], body_at.data(), b.offset);
      const uint64_t n = (uint64_t)b.length + b.length2;
      if(at + n > arena.size() || memcmp(arena.data() + at, cs + b.offset, n))
        return -103;
    }
    v.offset = b.offset;
    v.length = b.length;
    v.length2 = b.length2;
    v.numbps = b.numbps;
    v.numpasses = b.numpasses;
  }
  out->swap(vblocks);
  return (int64_t)out->size();
}

static std::vector<uint8_t> read_file(const std::string& path)
{
  std::ifstream f(path, std::ios::binary);
  return std::vector<uint8_t>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv)
{
  if(argc != 2)
  {
    printf("usage: t2_window_check LIST\n");
    return 2;
  }
  std::ifstream list(argv[1]);
  std::string line, path;
  std::vector<uint8_t> cs;
  int bad = 0;
  while(std::getline(list, line))
  {
    std::istringstream in(line);
    std::string file, w0;
    uint32_t reduce = 0;
    in >> file >> reduce >> w0;
    uint32_t win[4] = {0, 0, 0, 0};
    const bool has_window = w0 != "-";
    if(has_window)
    {
      win[0] = (uint32_t)std::stoul(w0);
      in >> win[1] >> win[2] >> win[3];
    }
    if(file != path)
    {
      cs = read_file(file);
      path = file;
    }
    /* an exact-size heap copy, so that the sanitizer sees any read past the stream */
    uint8_t* exact = new uint8_t[cs.size() ? cs.size() : 1];
    if(!cs.empty())
      memcpy(exact, cs.data(), cs.size());
    const uint32_t* wp = has_window ? win : nullptr;
    b2k_coding hcp{}, dcp{}, hcp0{}, dcp0{};
    /* the header-only calls (a count of 1 is a return of 1 too: its text stays empty) */
    g_err.clear();
    const int64_t hn0 = b2k_codestream_parse_window(exact, cs.size(), wp, reduce, &hcp0, nullptr, 0);
    const std::string herr0 = hn0 < 0 || hn0 == 1 ? g_err : "";
    Stats st;
    g_err.clear();
    const int64_t dn0 = device_order_window(exact, cs.size(), wp, reduce, dcp0, nullptr, st);
    const std::string derr0 = dn0 < 0 || dn0 == 1 ? g_err : "";
    /* the full calls */
    int64_t hn = hn0;
    std::vector<b2k_block> hb, db;
    std::string herr = herr0, derr;
    if(hn0 > 1)
    {
      hb.resize(hn0);
      g_err.clear();
      hn = b2k_codestream_parse_window(exact, cs.size(), wp, reduce, &hcp, hb.data(), hb.size());
      herr = hn <= 1 ? g_err : "";
    }
    g_err.clear();
    const int64_t dn = device_order_window(exact, cs.size(), wp, reduce, dcp, &db, st);
    derr = dn <= 1 ? g_err : "";
    delete[] exact;
    std::string why;
    if(hn0 != dn0)
      why = "header-only return " + std::to_string(hn0) + " vs " + std::to_string(dn0) + " (" + herr0 + " | " + derr0 + ")";
    else if(hn0 > 1 && memcmp(&hcp0, &dcp0, sizeof(hcp0)))
      why = "header-only coding differs";
    else if((hn0 < 0 || hn0 == 1) && herr0 != derr0)
      why = "header-only text '" + herr0 + "' vs '" + derr0 + "'";
    else if(hn0 > 1 && hn != dn)
      why = "return " + std::to_string(hn) + " vs " + std::to_string(dn) + " (" + herr + " | " + derr + ")";
    else if(hn0 > 1 && hn <= 1 && herr != derr)
      why = "text '" + herr + "' vs '" + derr + "'";
    else if(hn0 > 1 && hn > 1 && (memcmp(&hcp, &dcp, sizeof(hcp)) || memcmp(hb.data(), db.data(), hb.size() * sizeof(b2k_block))))
      why = "table differs";
    if(!why.empty())
      ++bad;
    const int64_t rc = hn0 > 1 ? hn : hn0;
    const std::string text = rc > 1 ? "" : (hn0 > 1 ? herr : herr0);
    std::string wtxt = has_window ? std::to_string(win[0]) + "," + std::to_string(win[1]) + "," + std::to_string(win[2]) + "," +
                                        std::to_string(win[3])
                                  : "-";
    printf("%s %u %s %lld %u %llu %s\n", file.c_str(), reduce, wtxt.c_str(), (long long)rc, st.wanted, (unsigned long long)st.bytes,
           why.empty() ? ("same " + text).c_str() : why.c_str());
  }
  return bad ? 1 : 0;
}
