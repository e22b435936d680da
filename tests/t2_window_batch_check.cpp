/*
 * tests/t2_window_batch_check.cpp -- the windowed batch parse (b2k_decode_codestreams_window_device up to the gather) run on
 * the host in the order of its steps: each stream's main header from BATCH_HEADER_PREFIX-byte prefixes (doubled while a
 * header runs past its prefix) and its window's coding (b2k_window_coding); the batch's coding (b2k_batch_window_check);
 * the box coding's plan and block map; then the kernels' thread bodies from t2_parse.h over every (stream, item):
 * batch_locate with the box, batch_plt, batch_packet, batch_walk, window_arena_at, window_block (the descriptors) and
 * window_gather_part (the gather).  Each stream is compared with b2k_codestream_parse_window of its bytes, window and
 * reduce alone: the same return code and text, the same virtual coding and block table (offsets into its own bytes); and
 * every coded block its descriptor keeps has its bytes where the descriptor points in the gathered arena.
 * Built with g++ together with codestream.cpp and geometry.cpp (test_t2_window_batch_host.py) under the address and
 * undefined-behaviour sanitizers.  Every stream lives in its own exact-size heap allocation, read in place as the device
 * reads the callers' buffers, and while one stream's threads run every other stream's bytes and slices (part table,
 * per-stream arrays, arena slice) are poisoned, so a thread that strays outside its own stream is reported.
 *
 *   t2_window_batch_check LIST   LIST: batches, each a line "batch <reduce>" followed by one line per stream, "<file> -"
 *                                (no window) or "<file> x0 y0 x1 y1".  Prints one line per stream:
 *     "<file> <rc> <ref> same <text>"   rc as b2k_codestream_parse_window alone (0 for a table), text its b2k_last_error
 *     "<file> 1 <ref> rule <text>"      status 1 by the batch rule (another virtual coding, tile box, progression, SOP or EPH)
 *     "<file> ... <what differs>"       and exit 1
 *   After each batch: "batch <wanted tiles> <gathered bytes>" (bytes: the parsed streams' wanted packet data together).
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
extern "C" int64_t b2k_codestream_parse_window(const uint8_t* cs, uint64_t len, const uint32_t* window, uint32_t reduce, b2k_coding* cp_out,
                                               b2k_block* blocks, uint64_t cap_blocks);

struct Stream
{
  std::string name;
  std::vector<uint8_t> bytes;
  bool has_window = false;
  uint32_t win[4] = {0, 0, 0, 0};
  uint8_t* exact = nullptr; /* its own allocation, exactly its bytes */
  /* b2k_codestream_parse_window alone */
  int64_t hn = 0;
  bool table = false; /* hn is a block count (a count of 1 reads like a return of 1: its text stays empty) */
  b2k_coding hcp{};
  std::vector<b2k_block> hb;
  std::string herr;
  /* the batch */
  int32_t status = 0;
  std::string text;
  bool rule = false;
  MainHeader h;
  WindowCoding wc;
};

static void host_parse(Stream& S, uint32_t reduce)
{
  const uint32_t* w = S.has_window ? S.win : nullptr;
  g_err.clear();
  S.hn = b2k_codestream_parse_window(S.exact, S.bytes.size(), w, reduce, &S.hcp, nullptr, 0);
  if(S.hn > 1 || (S.hn == 1 && g_err.empty()))
  {
    const int64_t count = S.hn;
    S.hb.resize(count);
    g_err.clear();
    S.hn = b2k_codestream_parse_window(S.exact, S.bytes.size(), w, reduce, &S.hcp, S.hb.data(), S.hb.size());
    S.table = S.hn == count && g_err.empty();
  }
  S.herr = S.table ? "" : g_err;
}

/* the main header as the batch reads it: an exact-size copy of the prefix, doubled while the header runs past it */
static int batch_header(Stream& S)
{
  const uint64_t len = S.bytes.size();
  if(!len)
  {
    b2k_set_error("no SOC marker");
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

/* a region of per-stream slices: only stream s's is addressable while its threads run */
struct Region
{
  uint8_t* p;
  uint64_t bytes;
  std::vector<std::pair<uint64_t, uint64_t>> slice; /* per stream: byte offset, bytes */
};

/* one batch: returns the number of streams whose result differs */
static int run_batch(std::vector<Stream>& B, uint32_t reduce)
{
  const uint32_t n = (uint32_t)B.size();
  for(Stream& S : B)
  {
    S.exact = new uint8_t[S.bytes.size() ? S.bytes.size() : 1];
    if(!S.bytes.empty())
      memcpy(S.exact, S.bytes.data(), S.bytes.size());
    host_parse(S, reduce);
  }
  uint32_t ref = n;
  for(uint32_t i = 0; i < n; ++i)
  {
    Stream& S = B[i];
    int rc = batch_header(S);
    if(!rc)
      rc = b2k_window_coding(S.h.cp, S.has_window ? S.win : nullptr, reduce, S.wc);
    if(rc)
    {
      S.status = rc;
      S.text = g_err;
    }
    else if(ref == n)
      ref = i;
    else if(b2k_batch_window_check(B[ref].h, B[ref].wc, ref, S.h, S.wc, i))
    {
      S.status = 1;
      S.text = g_err;
      S.rule = true;
    }
  }
  std::vector<std::string> why(n);
  uint32_t wanted = 0;
  uint64_t gathered = 0;
  if(ref < n && unsupported_reason(B[ref].wc.vcp))
  { /* the engine declines the virtual coding: every stream of it gets 1, as in the single call */
    for(Stream& S : B)
      if(!S.status)
      {
        S.status = 1;
        S.text = unsupported_reason(B[ref].wc.vcp);
        S.rule = true;
      }
  }
  else if(ref < n)
  {
    const MainHeader& H = B[ref].h;
    const WindowCoding& wc = B[ref].wc;
    const b2k_coding& vcp = wc.vcp;
    /* the virtual coding's blocks (the job's enumeration) and its coded ones */
    const TileGrid vg = tile_grid(vcp);
    const std::vector<std::vector<BandQuant>> vq = component_quant(vcp);
    std::vector<b2k_block> vblocks;
    for(uint32_t t = 0; t < vg.nx * vg.ny; ++t)
      enumerate_tile_blocks(vcp, t, tile_rect(vcp, vg, t), vq, vblocks);
    std::vector<uint32_t> coded;
    for(uint32_t i = 0; i < vblocks.size(); ++i)
      if(vblocks[i].x1 > vblocks[i].x0 && vblocks[i].y1 > vblocks[i].y0)
        coded.push_back(i);
    const uint64_t ncoded = coded.size();
    /* the box coding's plan, its blocks, and each coded block's WinBlock (b2k_t2_window_create) */
    std::vector<b2k_block> blocks;
    std::vector<uint32_t> vmap;
    if(b2k_window_blocks(wc, vblocks.data(), vblocks.size(), blocks, vmap))
      return printf("batch: no block map (%s)\n", g_err.c_str()), (int)n;
    const TileGrid bg = tile_grid(wc.box);
    const uint32_t nt = bg.nx * bg.ny;
    Plan plan;
    if(b2k_t2_plan(wc.box, H.flags() & ~(uint32_t)(B2K_CS_TPARTS_R | B2K_CS_TLM), blocks.data(), blocks.size(), nt, plan))
      return printf("batch: no plan (%s)\n", g_err.c_str()), (int)n;
    std::vector<uint32_t> coded_box(ncoded);
    std::vector<WinBlock> win(std::max<uint64_t>(ncoded, 1));
    for(uint64_t k = 0; k < ncoded; ++k)
    {
      const b2k_block& v = vblocks[coded[k]];
      coded_box[k] = vmap[coded[k]];
      win[k] = WinBlock{v.tile, v.resno ? v.resno - 1u : 0u, v.x0, v.y0, v.x1, v.y1};
    }
    const uint64_t nblocks = blocks.size(), np = plan.packets.size();
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
    const TileGrid g = tile_grid(H.cp);
    const uint32_t ntiles = g.nx * g.ny;
    const TileBox box{g.nx, wc.ta_x, wc.ta_y, wc.tb_x, wc.tb_y};
    const uint32_t bt = box.tiles();
    wanted = bt;
    /* the stream table (b2k_t2_window_enqueue): each stream read in place, its part table slice from its length */
    std::vector<StreamDesc> sd(n);
    std::vector<NeedRects> need(n);
    std::vector<ParseStatus> status(n);
    uint64_t parts = 0;
    for(uint32_t i = 0; i < n; ++i)
    {
      const Stream& S = B[i];
      const uint64_t len = S.bytes.size();
      const uint64_t sot = S.status ? 0 : S.h.sot;
      sd[i] = StreamDesc{0, len, sot, parts, sot ? part_capacity(len, nt) : 0, S.exact};
      parts += sd[i].parts_cap;
      need[i] = NeedRects{};
      if(!S.status)
      {
        need[i].n = (uint32_t)std::min<size_t>(S.wc.need.size(), WINDOW_MAX_RES);
        for(uint32_t r = 0; r < need[i].n; ++r)
        {
          const Rect& R = S.wc.need[r];
          need[i].r[r][0] = R.x0;
          need[i].r[r][1] = R.y0;
          need[i].r[r][2] = R.x1;
          need[i].r[r][3] = R.y1;
        }
      }
      status[i] = ParseStatus{NO_TILE_ERROR, sot ? (uint32_t)PR_NONE : (uint32_t)PR_SKIPPED, 0, 0, 0, 0, 0};
    }
    std::vector<PartRange> part(std::max<uint64_t>(parts, 1));
    std::vector<uint64_t> body_at(std::max<uint64_t>(parts, 1));
    std::vector<uint32_t> head(n * (uint64_t)bt), last(n * (uint64_t)bt), count(n * (uint64_t)ntiles), indexed(n * (uint64_t)nt),
        marked(n * (uint64_t)nt);
    std::vector<ParsedBlock> blk(n * nblocks);
    std::vector<uint64_t> start(n * np), end(n * np), part_end(n * np);
    std::vector<TagNode> tags(n * plan.tag_nodes + 1);
    std::vector<Region> regions;
    auto uniform = [&](auto& v, uint64_t per) {
      Region r{reinterpret_cast<uint8_t*>(v.data()), v.size() * sizeof(v[0]), {}};
      for(uint32_t i = 0; i < n; ++i)
        r.slice.push_back({i * per * sizeof(v[0]), per * sizeof(v[0])});
      regions.push_back(r);
    };
    uniform(head, bt);
    uniform(last, bt);
    uniform(count, ntiles);
    uniform(indexed, nt);
    uniform(marked, nt);
    uniform(blk, nblocks);
    uniform(start, np);
    uniform(end, np);
    uniform(part_end, np);
    uniform(tags, plan.tag_nodes);
    uniform(status, 1);
    uniform(need, 1);
    Region pr{reinterpret_cast<uint8_t*>(part.data()), part.size() * sizeof(PartRange), {}};
    Region br{reinterpret_cast<uint8_t*>(body_at.data()), body_at.size() * sizeof(uint64_t), {}};
    for(uint32_t i = 0; i < n; ++i)
    {
      pr.slice.push_back({sd[i].parts0 * sizeof(PartRange), sd[i].parts_cap * sizeof(PartRange)});
      br.slice.push_back({sd[i].parts0 * sizeof(uint64_t), sd[i].parts_cap * sizeof(uint64_t)});
    }
    regions.push_back(pr);
    regions.push_back(br);
    for(uint32_t i = 0; i < n; ++i)
    { /* the streams' own buffers */
      Region r{B[i].exact, B[i].bytes.size(), {}};
      for(uint32_t j = 0; j < n; ++j)
        r.slice.push_back({0, i == j ? B[i].bytes.size() : 0});
      regions.push_back(r);
    }
    auto only = [&](uint32_t s) {
      for(const Region& r : regions)
      {
        POISON(r.p, r.bytes);
        UNPOISON(r.p + r.slice[s].first, r.slice[s].second);
      }
    };
    auto all = [&] {
      for(const Region& r : regions)
        UNPOISON(r.p, r.bytes);
    };
    /* the parse kernels, every thread of each in flattened order (no arena: every stream is read in place) */
    for(uint32_t s = 0; s < n; ++s)
    {
      only(s);
      batch_locate(nullptr, sd.data(), s, ntiles, box, part.data(), head.data(), last.data(), count.data(), body_at.data(), status.data());
    }
    for(uint32_t s = 0; s < n; ++s)
    {
      only(s);
      for(uint64_t t = s * (uint64_t)nt; t < (s + 1) * (uint64_t)nt; ++t)
        batch_plt(nullptr, sd.data(), t, part.data(), head.data(), plan.parts.data(), nt, tile_first.data(), nblocks, np, blk.data(),
                  start.data(), end.data(), part_end.data(), indexed.data(), marked.data(), status.data());
    }
    for(uint32_t s = 0; s < n; ++s)
    {
      only(s);
      for(uint64_t k = s * np; k < (s + 1) * np; ++k)
        batch_packet(nullptr, sd.data(), k, plan.packets.data(), np, pkt_tile.data(), nt, nblocks, plan.tag_nodes, indexed.data(),
                     start.data(), end.data(), part_end.data(), kmax.data(), blk.data(), tags.data(), marked.data(), H.sop, H.eph,
                     status.data());
    }
    for(uint32_t s = 0; s < n; ++s)
    {
      only(s);
      for(uint64_t t = s * (uint64_t)nt; t < (s + 1) * (uint64_t)nt; ++t)
        batch_walk(nullptr, sd.data(), t, part.data(), head.data(), plan.parts.data(), nt, plan.packets.data(), kmax.data(),
                   tile_first.data(), nblocks, plan.tag_nodes, blk.data(), tags.data(), indexed.data(), marked.data(), H.sop, H.eph,
                   status.data());
    }
    all();
    /* the arena layout (k_t2_window_at: one scan over every stream's status) */
    const uint64_t total = window_arena_at(sd.data(), status.data(), 0, n, 0);
    /* the descriptors of stream s read its own slices and the plan's WinBlock table */
    std::vector<ParsedBlock> desc(n * ncoded);
    std::vector<uint64_t> slot_off(n * ncoded);
    for(uint32_t s = 0; s < n; ++s)
    {
      only(s);
      for(uint64_t d = s * ncoded; d < (s + 1) * ncoded; ++d)
      {
        uint32_t t = 0;
        desc[d] = window_block(blk.data(), nblocks, coded_box.data(), d, ncoded, status.data(), sd.data(), win.data(), need.data(),
                               part.data(), head.data(), bt, body_at.data(), &t, &slot_off[d]);
        if(t != s)
          why[s] = "descriptor " + std::to_string(d) + " is stream " + std::to_string(t) + "'s";
      }
    }
    all();
    /* the gather: stream s's items write only its arena slice */
    uint64_t per = 0;
    for(uint32_t s = 0; s < n; ++s)
      if(status_reason(status[s]) == PR_NONE)
      {
        per = std::max<uint64_t>(per, status[s].nparts);
        gathered += status[s].bytes;
      }
    uint8_t* arena = new uint8_t[total + 64];
    Region ar{arena, total + 64, {}};
    for(uint32_t i = 0; i < n; ++i)
      ar.slice.push_back({sd[i].at, window_gathered_bytes(status[i])});
    regions.push_back(ar);
    for(uint32_t s = 0; s < n; ++s)
    {
      only(s);
      for(uint64_t e = s * per; e < (s + 1) * per; ++e)
      {
        const uint8_t* src = nullptr;
        uint64_t dst = 0, len = 0;
        if(window_gather_part(sd.data(), part.data(), body_at.data(), status.data(), e, per, &src, &dst, &len))
          memcpy(arena + dst, src, len);
      }
    }
    all();
    for(uint32_t i = 0; i < n; ++i)
      if(!B[i].status)
        if(const uint32_t r = status_reason(status[i]))
        {
          B[i].status = parse_reason_rc(r);
          B[i].text = parse_reason_text(r);
        }
    /* the descriptors against each stream's own table: the same lengths, and the kept blocks' bytes in the arena */
    for(uint64_t d = 0; d < n * ncoded; ++d)
    {
      const uint32_t s = (uint32_t)(d / ncoded);
      const ParsedBlock& b = desc[d];
      if(!why[s].empty())
        continue;
      const b2k_block* want = B[s].status || !B[s].table ? nullptr : &B[s].hb[coded[d % ncoded]];
      if(!want)
      {
        if(b.length)
          why[s] = "a failed stream's descriptor has bytes";
        continue;
      }
      if(b.length != want->length || (b.length && b.length2 != want->length2))
      {
        why[s] = "descriptor " + std::to_string(d) + ": length " + std::to_string(b.length) + " vs " + std::to_string(want->length);
        continue;
      }
      const uint64_t nb = (uint64_t)b.length + b.length2;
      if(b.length && (slot_off[d] < sd[s].at || slot_off[d] + nb > sd[s].at + window_gathered_bytes(status[s]) ||
                      memcmp(arena + slot_off[d], B[s].bytes.data() + want->offset, nb)))
        why[s] = "descriptor " + std::to_string(d) + ": the bytes at its arena offset are not the block's";
    }
    /* the block tables (b2k_t2_window_blocks): the virtual blocks' box blocks, the need filter */
    for(uint32_t i = 0; i < n; ++i)
    {
      if(B[i].status || !B[i].table || !why[i].empty())
        continue;
      std::vector<b2k_block> tb = vblocks;
      for(uint64_t k = 0; k < tb.size(); ++k)
      {
        b2k_block& v = tb[k];
        const ParsedBlock& p = blk[i * nblocks + vmap[k]];
        if(need[i].n && !window_needs(need[i].r[v.resno ? v.resno - 1 : 0], v.x0, v.y0, v.x1, v.y1))
          continue;
        v.offset = p.offset;
        v.length = p.length;
        v.length2 = p.length2;
        v.numbps = p.numbps;
        v.numpasses = p.numpasses;
      }
      if(tb.size() != B[i].hb.size() || memcmp(tb.data(), B[i].hb.data(), tb.size() * sizeof(b2k_block)) ||
         memcmp(&vcp, &B[i].hcp, sizeof(vcp)))
        why[i] = "table differs";
    }
    delete[] arena;
  }
  int bad = 0;
  for(uint32_t i = 0; i < n; ++i)
  {
    Stream& S = B[i];
    const int64_t want_rc = S.table ? 0 : S.hn;
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
    delete[] S.exact;
  }
  printf("batch %u %llu\n", wanted, (unsigned long long)gathered);
  return bad;
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
    printf("usage: t2_window_batch_check LIST\n");
    return 2;
  }
  std::ifstream list(argv[1]);
  std::string line;
  std::vector<Stream> batch;
  uint32_t reduce = 0;
  int bad = 0;
  auto flush = [&] {
    if(!batch.empty())
      bad += run_batch(batch, reduce);
    batch.clear();
  };
  while(std::getline(list, line))
  {
    std::istringstream in(line);
    std::string file, w0;
    in >> file;
    if(file == "batch")
    {
      flush();
      in >> reduce;
      continue;
    }
    in >> w0;
    Stream S;
    S.name = file;
    S.bytes = read_file(file);
    S.has_window = w0 != "-";
    if(S.has_window)
    {
      S.win[0] = (uint32_t)std::stoul(w0);
      in >> S.win[1] >> S.win[2] >> S.win[3];
    }
    batch.push_back(std::move(S));
  }
  flush();
  return bad ? 1 : 0;
}
