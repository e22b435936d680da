/*
 * tests/t2_parse_check.cpp -- the device code-stream parser's functions (grok_b200/csrc/t2_parse.h) run on the host, in the
 * order of its kernels (t2_decode.cu: locate, PLT packet starts per tile, one packet at a time from them, the walk for the
 * tiles not indexed or marked, the descriptor rule), against b2k_codestream_parse on the same
 * bytes.  Built with g++ together with codestream.cpp and geometry.cpp (test_t2_parse_host.py), under the address and
 * undefined-behaviour sanitizers, so that every byte the parser reads is checked against the stream's bounds.
 *
 *   t2_parse_check FILE...   prints one line per file: "<file> <rc> <indexed tiles> <walked tiles> same <text>" or what
 *                            differs; exit 1 on any difference
 */
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <functional>
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
extern "C" int64_t b2k_codestream_parse(const uint8_t* cs, uint64_t len, b2k_coding* cp_out, b2k_block* blocks, uint64_t cap_blocks);

/* the device parser's verdict and table, computed as its kernels compute them */
static int64_t device_order_parse(const uint8_t* cs, uint64_t len, b2k_coding& cp, std::vector<b2k_block>& out, uint32_t* stats)
{
  MainHeader h;
  if(int rc = b2k_parse_main_header(cs, len, h))
    return rc;
  cp = h.cp;
  const TileGrid g = tile_grid(cp);
  const uint32_t ntiles = g.nx * g.ny;
  const std::vector<BandQuant> q = band_quant(cp);
  std::vector<b2k_block> blocks;
  for(uint32_t t = 0; t < ntiles; ++t)
    enumerate_tile_blocks(cp, t, tile_rect(cp, g, t), q, blocks);
  Plan plan;
  if(b2k_t2_plan(cp, B2K_CS_PROG(h.progression), blocks.data(), blocks.size(), ntiles, plan))
    return -1;
  /* kernel 1: the tile parts */
  const uint64_t cap = std::min<uint64_t>(len / 12 + 1, 256ull * ntiles);
  std::vector<PartRange> parts(cap);
  std::vector<uint32_t> head(ntiles), last(ntiles), count(ntiles);
  uint32_t nparts = 0;
  if(uint32_t r = locate_tile_parts(cs, len, h.sot, ntiles, parts.data(), cap, head.data(), last.data(), count.data(), &nparts))
  {
    b2k_set_error(parse_reason_text(r));
    return parse_reason_rc(r);
  }
  std::vector<uint8_t> kmax(blocks.size());
  for(size_t i = 0; i < blocks.size(); ++i)
    kmax[i] = blocks[i].kmax;
  std::vector<ParsedBlock> pb(blocks.size());
  std::vector<TagNode> tags(plan.tag_nodes + 1);
  const uint64_t np = plan.packets.size();
  std::vector<uint64_t> start(np), end(np), part_end(np);
  std::vector<uint8_t> indexed(ntiles), marked(ntiles);
  /* kernel 2: packet starts from PLT (the blocks are zero already) */
  for(uint32_t t = 0; t < ntiles; ++t)
  {
    const DevPart& T = plan.parts[t];
    indexed[t] = plt_index(cs, parts.data(), head[t], T.p1 - T.p0, start.data() + T.p0, end.data() + T.p0, part_end.data() + T.p0);
  }
  /* kernel 3: one packet at a time from its PLT start, each with its own tag-tree scratch */
  for(uint32_t t = 0; t < ntiles; ++t)
    for(uint64_t g = plan.parts[t].p0; indexed[t] && g < plan.parts[t].p1; ++g)
    {
      uint64_t at = start[g];
      if(parse_packet(cs, plan.packets[g], &at, part_end[g], kmax.data(), pb.data(), tags.data() + plan.packets[g].tag_at, h.sop, h.eph) ||
         at != end[g])
        marked[t] = 1;
    }
  /* kernel 4: the walk for every other tile; the lowest failing tile decides */
  uint32_t first_err = PR_NONE;
  for(uint32_t t = 0; t < ntiles; ++t)
  {
    const DevPart& T = plan.parts[t];
    if(T.p1 == T.p0 || (indexed[t] && !marked[t]))
      continue;
    if(head[t] != PART_NONE)
      ++stats[1];
    for(uint64_t i = 0; i < blocks.size(); ++i)
      if(blocks[i].tile == t)
        pb[i] = ParsedBlock{};
    const uint32_t r = parse_tile(cs, parts.data(), head[t], plan.packets.data() + T.p0, T.p1 - T.p0, kmax.data(), pb.data(),
                                  tags.data() + plan.packets[T.p0].tag_at, h.sop, h.eph);
    if(r && !first_err)
      first_err = r;
  }
  for(uint32_t t = 0; t < ntiles; ++t)
    stats[0] += indexed[t] && plan.parts[t].p1 > plan.parts[t].p0;
  if(first_err)
  {
    b2k_set_error(parse_reason_text(first_err));
    return parse_reason_rc(first_err);
  }
  /* kernel 5: the descriptor fields against prepare_decode's rule (engine.cu), restated */
  for(size_t i = 0; i < blocks.size(); ++i)
  {
    uint8_t mmsbs = 0, passes = 0;
    uint32_t length2 = 0;
    block_decode_fields(pb[i], blocks[i].kmax, &mmsbs, &passes, &length2);
    const int nb = pb[i].length ? pb[i].numbps : 0;
    const uint8_t want_mmsbs = (uint8_t)std::max(0, (int)blocks[i].kmax - nb);
    const uint8_t want_passes = (pb[i].length && pb[i].numpasses > 1 && pb[i].length2 > 0 && want_mmsbs < 29) ? pb[i].numpasses : 1;
    const uint32_t want_length2 = want_passes > 1 ? pb[i].length2 : 0;
    if(mmsbs != want_mmsbs || passes != want_passes || length2 != want_length2)
      return -100;
    blocks[i].offset = pb[i].offset;
    blocks[i].length = pb[i].length;
    blocks[i].length2 = pb[i].length2;
    blocks[i].numbps = pb[i].numbps;
    blocks[i].numpasses = pb[i].numpasses;
  }
  out.swap(blocks);
  return (int64_t)out.size();
}

int main(int argc, char** argv)
{
  int bad = 0;
  for(int a = 1; a < argc; ++a)
  {
    FILE* f = fopen(argv[a], "rb");
    if(!f)
    {
      printf("%s: cannot open\n", argv[a]);
      return 2;
    }
    std::vector<uint8_t> cs;
    uint8_t buf[65536];
    size_t n;
    while((n = fread(buf, 1, sizeof(buf), f)) > 0)
      cs.insert(cs.end(), buf, buf + n);
    fclose(f);
    /* an exact-size heap copy, so that the sanitizer sees any read past the stream */
    uint8_t* exact = new uint8_t[cs.size() ? cs.size() : 1];
    if(!cs.empty())
      memcpy(exact, cs.data(), cs.size());
    b2k_coding hcp{}, dcp{};
    int64_t hn = b2k_codestream_parse(exact, cs.size(), &hcp, nullptr, 0);
    std::vector<b2k_block> hb;
    if(hn > 1)
    {
      hb.resize(hn);
      hn = b2k_codestream_parse(exact, cs.size(), &hcp, hb.data(), hb.size());
    }
    const std::string herr = hn <= 1 ? g_err : "";
    std::vector<b2k_block> db;
    uint32_t stats[2] = {0, 0}; /* tiles indexed, tiles walked */
    const int64_t dn = device_order_parse(exact, cs.size(), dcp, db, stats);
    const std::string derr = dn <= 1 ? g_err : "";
    delete[] exact;
    std::string why;
    if(hn != dn)
      why = "return " + std::to_string(hn) + " vs " + std::to_string(dn) + " (" + herr + " | " + derr + ")";
    else if(hn <= 1 && herr != derr)
      why = "text '" + herr + "' vs '" + derr + "'";
    else if(hn > 1 && (memcmp(&hcp, &dcp, sizeof(hcp)) || memcmp(hb.data(), db.data(), hb.size() * sizeof(b2k_block))))
      why = "table differs";
    if(!why.empty())
      ++bad;
    printf("%s %lld %u %u %s\n", argv[a], (long long)hn, stats[0], stats[1], why.empty() ? ("same " + herr).c_str() : why.c_str());
  }
  return bad ? 1 : 0;
}
