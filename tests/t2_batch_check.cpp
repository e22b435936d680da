/*
 * tests/t2_batch_check.cpp -- the batched device parse (b2k_decode_codestreams_device up to the decoder's descriptors) run
 * on the host, in the order of its steps: the main headers from BATCH_HEADER_PREFIX-byte prefixes, doubled while a header
 * runs past its prefix; the batch's coding (b2k_batch_coding_check); the streams laid out in one arena at
 * batch_arena_next boundaries; then the five kernels' thread bodies (t2_parse.h batch_locate / batch_plt / batch_packet /
 * batch_walk / batch_block) over every (stream, item) of the batch, with the per-stream state sliced as the kernels slice
 * it.  Every stream is compared with b2k_codestream_parse of its bytes alone.  Built with g++ together with codestream.cpp
 * and geometry.cpp (test_t2_batch_host.py) under the address and undefined-behaviour sanitizers; the gaps between the
 * streams in the arena are poisoned, and while one stream's threads run every other stream's slices (arena bytes, part
 * table, per-stream arrays) are poisoned too, so a thread that strays outside its own stream's slice is reported.
 *
 *   t2_batch_check FILE... [-- FILE...]...   one batch per group.  Prints one line per stream:
 *     "<file> <rc> <ref> same <text>"     rc as b2k_codestream_parse of the file alone, text its b2k_last_error
 *     "<file> <rc> <ref> rule <text>"     status 1 by the batch rule (another coding, progression, SOP or EPH than stream ref)
 *     "<file> ... <what differs>"          and exit 1
 *   ref: the stream the batch takes its coding from (-1: none).  For every stream that parses, the harness also checks the
 *   block table and that every coded block's bytes are where its descriptor points in the arena; a stream that fails gets
 *   empty descriptors.
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

#if defined(__SANITIZE_ADDRESS__)
#include <sanitizer/asan_interface.h>
#define POISON(p, n) ASAN_POISON_MEMORY_REGION((p), (n))
#define UNPOISON(p, n) ASAN_UNPOISON_MEMORY_REGION((p), (n))
#else
#define POISON(p, n) ((void)(p), (void)(n))
#define UNPOISON(p, n) ((void)(p), (void)(n))
#endif

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

struct Stream
{
  std::string name;
  std::vector<uint8_t> bytes;
  /* b2k_codestream_parse alone */
  int64_t hn = 0;
  b2k_coding hcp{};
  std::vector<b2k_block> hb;
  std::string herr;
  /* the batch */
  int32_t status = 0;
  std::string text;
  bool rule = false;
  MainHeader h;
};

static void host_parse(Stream& S)
{
  const uint64_t len = S.bytes.size();
  uint8_t* exact = new uint8_t[len ? len : 1];
  if(len)
    memcpy(exact, S.bytes.data(), len);
  S.hn = b2k_codestream_parse(exact, len, &S.hcp, nullptr, 0);
  if(S.hn > 1)
  {
    S.hb.resize(S.hn);
    S.hn = b2k_codestream_parse(exact, len, &S.hcp, S.hb.data(), S.hb.size());
  }
  S.herr = S.hn <= 1 ? g_err : "";
  delete[] exact;
}

/* the main header as the batch reads it: an exact-size copy of the prefix, doubled while the header runs past it */
static int batch_header(Stream& S)
{
  const uint64_t len = S.bytes.size();
  if(!len)
  {
    b2k_set_error("no SOC marker"); /* the device-memory check of an empty stream */
    return -1;
  }
  uint64_t n = std::min<uint64_t>(len, BATCH_HEADER_PREFIX);
  for(;;)
  {
    uint8_t* exact = new uint8_t[n];
    memcpy(exact, S.bytes.data(), n);
    const int rc = b2k_parse_main_header(exact, n, S.h);
    delete[] exact;
    if(rc && S.h.short_read && n < len)
    {
      n = std::min<uint64_t>(len, 2 * n);
      continue;
    }
    return rc;
  }
}

/* one batch: returns the number of streams whose result differs */
static int run_batch(std::vector<Stream>& B)
{
  const uint32_t n = (uint32_t)B.size();
  for(Stream& S : B)
    host_parse(S);
  uint32_t ref = n;
  for(uint32_t i = 0; i < n; ++i)
  {
    if(int rc = batch_header(B[i]))
    {
      B[i].status = rc;
      B[i].text = g_err;
    }
    else if(ref == n)
      ref = i;
    else if(b2k_batch_coding_check(B[ref].h, ref, B[i].h, i))
    {
      B[i].status = 1;
      B[i].text = g_err;
      B[i].rule = true;
    }
  }
  std::vector<std::string> why(n);
  if(ref < n)
  {
    const MainHeader& H = B[ref].h;
    const b2k_coding& cp = H.cp;
    const TileGrid g = tile_grid(cp);
    const uint32_t ntiles = g.nx * g.ny;
    const std::vector<BandQuant> q = band_quant(cp);
    std::vector<b2k_block> blocks;
    for(uint32_t t = 0; t < ntiles; ++t)
      enumerate_tile_blocks(cp, t, tile_rect(cp, g, t), q, blocks);
    if(const char* unsupported = unsupported_reason(cp))
    { /* the engine declines the coding: every stream of it gets 1, as in the single call */
      for(Stream& S : B)
        if(!S.status)
        {
          S.status = 1;
          S.text = unsupported;
          S.rule = true;
        }
    }
    Plan plan;
    if(!unsupported_reason(cp) &&
       b2k_t2_plan(cp, H.flags() & ~(uint32_t)(B2K_CS_TPARTS_R | B2K_CS_TLM), blocks.data(), blocks.size(), ntiles, plan))
      return printf("batch: no plan (%s)\n", g_err.c_str()), (int)n;
    if(!unsupported_reason(cp))
    {
      const uint64_t nblocks = blocks.size(), np = plan.packets.size(), nt = plan.parts.size();
      std::vector<uint32_t> coded;
      for(uint32_t i = 0; i < nblocks; ++i)
        if(blocks[i].x1 > blocks[i].x0 && blocks[i].y1 > blocks[i].y0)
          coded.push_back(i);
      const uint64_t ncoded = coded.size();
      std::vector<uint8_t> kmax(nblocks);
      std::vector<uint64_t> tile_first(nt + 1, nblocks);
      for(uint64_t i = nblocks; i-- > 0;)
      {
        kmax[i] = blocks[i].kmax;
        tile_first[blocks[i].tile] = i;
      }
      for(uint64_t t = nt; t-- > 0;)
        tile_first[t] = std::min(tile_first[t], tile_first[t + 1]);
      std::vector<uint32_t> pkt_tile(np);
      for(uint32_t t = 0; t < nt; ++t)
        for(uint64_t k = plan.parts[t].p0; k < plan.parts[t].p1; ++k)
          pkt_tile[k] = t;
      /* the arena: the streams that reach their tile parts at batch_arena_next boundaries, each followed by a poisoned gap
         of at least 256 bytes */
      std::vector<StreamDesc> sd(n);
      uint64_t total = 0, parts = 0;
      for(uint32_t i = 0; i < n; ++i)
      {
        if(B[i].status)
        {
          sd[i] = StreamDesc{0, 0, 0, parts, 0};
          continue;
        }
        const uint64_t len = B[i].bytes.size();
        sd[i] = StreamDesc{total, len, B[i].h.sot, parts, part_capacity(len, (uint32_t)nt)};
        parts += sd[i].parts_cap;
        total = batch_arena_next(total, len + 256);
      }
      uint8_t* arena = new uint8_t[total + 64];
      POISON(arena, total + 64);
      for(uint32_t i = 0; i < n; ++i)
        if(!B[i].status && sd[i].len)
        {
          UNPOISON(arena + sd[i].at, sd[i].len);
          memcpy(arena + sd[i].at, B[i].bytes.data(), sd[i].len);
        }
      std::vector<ParseStatus> status(n);
      for(uint32_t i = 0; i < n; ++i)
        status[i] = ParseStatus{NO_TILE_ERROR, B[i].status ? (uint32_t)PR_SKIPPED : (uint32_t)PR_NONE, 0, 0, 0, 0, 0};
      std::vector<PartRange> part(std::max<uint64_t>(parts, 1));
      std::vector<uint32_t> head(n * nt), last(n * nt), count(n * (uint64_t)ntiles), indexed(n * nt), marked(n * nt);
      std::vector<ParsedBlock> blk(n * nblocks);
      std::vector<uint64_t> start(n * np), end(n * np), part_end(n * np);
      std::vector<TagNode> tags(n * plan.tag_nodes + 1);
      const TileBox box{ntiles, 0, 0, ntiles, 1};
      /* While stream s's threads run, only stream s's slices are addressable: every other stream's bytes in the arena,
         its part-table entries and its slice of every per-stream array are poisoned, so a thread that strays into another
         stream's slice is reported, not just one that leaves the arrays. */
      struct Region
      {
        uint8_t* p;
        uint64_t bytes;
        std::vector<std::pair<uint64_t, uint64_t>> slice; /* per stream: byte offset, bytes */
      };
      std::vector<Region> regions;
      auto uniform = [&](auto& v, uint64_t per) {
        Region r{reinterpret_cast<uint8_t*>(v.data()), v.size() * sizeof(v[0]), {}};
        for(uint32_t i = 0; i < n; ++i)
          r.slice.push_back({i * per * sizeof(v[0]), per * sizeof(v[0])});
        regions.push_back(r);
      };
      uniform(head, nt);
      uniform(last, nt);
      uniform(count, ntiles);
      uniform(indexed, nt);
      uniform(marked, nt);
      uniform(blk, nblocks);
      uniform(start, np);
      uniform(end, np);
      uniform(part_end, np);
      uniform(tags, plan.tag_nodes);
      uniform(status, 1);
      Region pr{reinterpret_cast<uint8_t*>(part.data()), part.size() * sizeof(PartRange), {}};
      Region ar{arena, total + 64, {}};
      for(uint32_t i = 0; i < n; ++i)
      {
        pr.slice.push_back({sd[i].parts0 * sizeof(PartRange), sd[i].parts_cap * sizeof(PartRange)});
        ar.slice.push_back({sd[i].at, sd[i].len});
      }
      regions.push_back(pr);
      regions.push_back(ar);
      auto only = [&](uint32_t s) {
        for(const Region& r : regions)
        {
          POISON(r.p, r.bytes);
          UNPOISON(r.p + r.slice[s].first, r.slice[s].second);
        }
      };
      /* the five kernels, one after another, every thread of each (in flattened order: stream by stream) */
      for(uint32_t s = 0; s < n; ++s)
      {
        only(s);
        batch_locate(arena, sd.data(), s, ntiles, box, part.data(), head.data(), last.data(), count.data(), nullptr, status.data());
      }
      for(uint32_t s = 0; s < n; ++s)
      {
        only(s);
        for(uint64_t t = s * nt; t < (s + 1) * nt; ++t)
          batch_plt(arena, sd.data(), t, part.data(), head.data(), plan.parts.data(), (uint32_t)nt, tile_first.data(), nblocks, np,
                    blk.data(), start.data(), end.data(), part_end.data(), indexed.data(), marked.data(), status.data());
      }
      for(uint32_t s = 0; s < n; ++s)
      {
        only(s);
        for(uint64_t k = s * np; k < (s + 1) * np; ++k)
          batch_packet(arena, sd.data(), k, plan.packets.data(), np, pkt_tile.data(), (uint32_t)nt, nblocks, plan.tag_nodes,
                       indexed.data(), start.data(), end.data(), part_end.data(), kmax.data(), blk.data(), tags.data(), marked.data(),
                       H.sop, H.eph, status.data());
      }
      for(uint32_t s = 0; s < n; ++s)
      {
        only(s);
        for(uint64_t t = s * nt; t < (s + 1) * nt; ++t)
          batch_walk(arena, sd.data(), t, part.data(), head.data(), plan.parts.data(), (uint32_t)nt, plan.packets.data(), kmax.data(),
                     tile_first.data(), nblocks, plan.tag_nodes, blk.data(), tags.data(), indexed.data(), marked.data(), H.sop, H.eph,
                     status.data());
      }
      for(uint32_t s = 0; s < n; ++s)
      { /* the descriptor step reads stream s's blocks and status */
        only(s);
        for(uint64_t d = s * ncoded; d < (s + 1) * ncoded; ++d)
        {
          uint32_t t = 0;
          (void)batch_block(blk.data(), nblocks, coded.data(), d, ncoded, status.data(), &t);
        }
      }
      for(const Region& r : regions)
        UNPOISON(r.p, r.bytes);
      for(uint32_t i = 0; i < n; ++i)
        if(!B[i].status)
          if(const uint32_t r = status_reason(status[i]))
          {
            B[i].status = parse_reason_rc(r);
            B[i].text = parse_reason_text(r);
          }
      /* the descriptors: a parsed stream's coded blocks point at their bytes in the arena; a failed stream's are empty */
      for(uint64_t d = 0; ncoded && d < n * ncoded; ++d)
      {
        uint32_t s = 0;
        const ParsedBlock b = batch_block(blk.data(), nblocks, coded.data(), d, ncoded, status.data(), &s);
        const b2k_block* want = B[s].status || B[s].hn <= 1 ? nullptr : &B[s].hb[coded[d % ncoded]];
        if(!want)
        {
          if(b.length && why[s].empty())
            why[s] = "a failed stream's descriptor has bytes";
          continue;
        }
        if(b.length != want->length || (b.length && b.length2 != want->length2))
        {
          if(why[s].empty())
            why[s] = "descriptor " + std::to_string(d) + ": length " + std::to_string(b.length) + " vs " + std::to_string(want->length);
          continue;
        }
        const uint64_t at = sd[s].at + b.offset, nb = (uint64_t)b.length + b.length2;
        if(b.length && (b.offset + nb > sd[s].len || memcmp(arena + at, B[s].bytes.data() + want->offset, nb)) && why[s].empty())
          why[s] = "descriptor " + std::to_string(d) + ": the bytes at its arena offset are not the block's";
      }
      /* the block tables of the streams that parse */
      for(uint32_t i = 0; i < n; ++i)
      {
        if(B[i].status || B[i].hn <= 1 || !why[i].empty())
          continue;
        std::vector<b2k_block> tb = blocks;
        for(uint64_t k = 0; k < nblocks; ++k)
        {
          const ParsedBlock& p = blk[i * nblocks + k];
          tb[k].offset = p.offset;
          tb[k].length = p.length;
          tb[k].length2 = p.length2;
          tb[k].numbps = p.numbps;
          tb[k].numpasses = p.numpasses;
        }
        if(tb.size() != B[i].hb.size() || memcmp(tb.data(), B[i].hb.data(), tb.size() * sizeof(b2k_block)) ||
           memcmp(&cp, &B[i].hcp, sizeof(cp)))
          why[i] = "table differs";
      }
      UNPOISON(arena, total + 64);
      delete[] arena;
    }
  }
  int bad = 0;
  for(uint32_t i = 0; i < n; ++i)
  {
    Stream& S = B[i];
    const int64_t want_rc = S.hn > 1 ? 0 : S.hn;
    if(why[i].empty() && !S.rule)
    {
      if(S.status != want_rc)
        why[i] = "return " + std::to_string(want_rc) + " vs " + std::to_string(S.status) + " (" + S.herr + " | " + S.text + ")";
      else if(S.status && S.text != S.herr)
        why[i] = "text '" + S.herr + "' vs '" + S.text + "'";
    }
    bad += !why[i].empty();
    printf("%s %lld %d %s %s\n", S.name.c_str(), (long long)(S.rule ? 1 : want_rc), ref < n ? (int)ref : -1,
           !why[i].empty() ? why[i].c_str() : S.rule ? "rule" : "same", why[i].empty() ? S.text.c_str() : "");
  }
  return bad;
}

int main(int argc, char** argv)
{
  int bad = 0;
  std::vector<Stream> batch;
  for(int a = 1; a <= argc; ++a)
  {
    if(a == argc || !strcmp(argv[a], "--"))
    {
      if(!batch.empty())
        bad += run_batch(batch);
      batch.clear();
      continue;
    }
    FILE* f = fopen(argv[a], "rb");
    if(!f)
    {
      printf("%s: cannot open\n", argv[a]);
      return 2;
    }
    Stream S;
    S.name = argv[a];
    uint8_t buf[65536];
    size_t k;
    while((k = fread(buf, 1, sizeof(buf), f)) > 0)
      S.bytes.insert(S.bytes.end(), buf, buf + k);
    fclose(f);
    batch.push_back(std::move(S));
  }
  return bad ? 1 : 0;
}
