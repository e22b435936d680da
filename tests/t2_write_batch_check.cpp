/*
 * tests/t2_write_batch_check.cpp -- the batched device code-stream writer (b2k_encode_codestreams_device after the block
 * coder) run on the host, in the order of its steps: the writer's thread bodies (t2_write.h write_header / write_part /
 * write_emit / write_packet, the scan as write_scan_host) over every (stream, item) of the batch, with the per-stream state
 * sliced as the kernels slice it, then the encoder's gather.  As in the engine, the first round runs against an empty
 * output buffer and the second against one of exactly the bytes the first asked for.  Built with g++ together with
 * codestream.cpp and geometry.cpp (test_t2_write_batch_host.py) under the address and undefined-behaviour sanitizers;
 * while one stream's threads run, every other stream's slices (coder output, header scratch, tag trees, per-packet and
 * per-part arrays, block destinations, output bytes) are poisoned, so a thread that strays outside its own stream is
 * reported.
 *
 *   t2_write_batch_check -- FLAGS CODING NAME TABLE DATA INJECT [NAME TABLE DATA INJECT]... [-- ...]...
 *     one batch per group: code-stream flags, a file holding the b2k_coding, then per stream a block table (b2k_block,
 *     every block of every tile, enumeration order) and its byte arena.  INJECT >= 0 marks that coded block of the
 *     stream as overflowed (total 0xFFFFFFFF), as the coder reports a block that did not fit its scratch slot.
 *   Prints one line per stream:
 *     "<name> <rc> <offset> <length> same <text>"   rc and text as the single call gives them; for rc 0 the bytes at
 *                                                   offset are those of b2k_codestream_write of the stream's table,
 *                                                   and are written to TABLE.cs
 *     "<name> plan <text>"                          b2k_t2_plan declined the coding and flags (every stream of the batch)
 *     "<name> ... <what differs>"                   and exit 1
 */
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <functional>
#include <string>
#include <vector>

#include "b2k_internal.h"
#include "geometry.h"
#include "t2_plan.h"
#include "t2_write.h"

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

static std::vector<uint8_t> read_file(const char* path)
{
  std::vector<uint8_t> v;
  if(FILE* f = fopen(path, "rb"))
  {
    uint8_t buf[65536];
    size_t k;
    while((k = fread(buf, 1, sizeof buf, f)) > 0)
      v.insert(v.end(), buf, buf + k);
    fclose(f);
  }
  return v;
}

struct Stream
{
  std::string name, table_path;
  std::vector<b2k_block> table; /* as the coder reports it: coded blocks one pass, one bit plane */
  std::vector<uint8_t> data;
  long inject = -1;
};

/* the per-stream slices of one array of T, `per` elements each */
template <class T>
struct Sliced
{
  std::vector<T> v;
  uint64_t per = 0;
  void init(uint32_t n, uint64_t p)
  {
    per = p;
    v.assign(std::max<uint64_t>(1, n * p), T{});
  }
  T* data() { return v.data(); }
  void poison_others(uint32_t n, uint32_t s, bool on)
  {
    for(uint32_t j = 0; j < n; ++j)
      if(j != s && per)
      {
        if(on)
          POISON(v.data() + j * per, per * sizeof(T));
        else
          UNPOISON(v.data() + j * per, per * sizeof(T));
      }
  }
};

/* one batch; returns the number of streams whose result differs */
static int run_batch(uint32_t flags, const b2k_coding& cp, std::vector<Stream>& B)
{
  const uint32_t n = (uint32_t)B.size();
  const TileGrid g = tile_grid(cp);
  const uint32_t ntiles = g.nx * g.ny;
  const std::vector<b2k_block>& blocks = B[0].table;
  const uint64_t nblocks = blocks.size();
  Plan P;
  if(b2k_t2_plan(cp, flags, blocks.data(), nblocks, ntiles, P))
  {
    for(const Stream& S : B)
      printf("%s plan %s\n", S.name.c_str(), g_err.c_str());
    return 0;
  }
  /* the coded blocks (blocks with area), as the engine's job numbers them */
  std::vector<int32_t> coded(nblocks, -1);
  std::vector<uint8_t> kmax(nblocks);
  std::vector<uint32_t> coded_index;
  for(uint64_t i = 0; i < nblocks; ++i)
  {
    kmax[i] = blocks[i].kmax;
    if(blocks[i].x1 > blocks[i].x0 && blocks[i].y1 > blocks[i].y0)
    {
      coded[i] = (int32_t)coded_index.size();
      coded_index.push_back((uint32_t)i);
    }
  }
  const uint64_t ncoded = coded_index.size(), np = P.packets.size(), nparts = P.parts.size();
  Sliced<HtBlockOut> outs;
  outs.init(n, ncoded);
  for(uint32_t s = 0; s < n; ++s)
    for(uint64_t k = 0; k < ncoded; ++k)
    {
      const b2k_block& b = B[s].table[coded_index[k]];
      outs.v[s * ncoded + k].total = (long)k == B[s].inject ? 0xFFFFFFFFu : (b.numpasses ? b.length : 0u);
    }
  Sliced<uint8_t> hdr;
  Sliced<TagNode> tags;
  Sliced<uint32_t> hdr_len;
  Sliced<uint64_t> body_len, pkt_at, part_plt, part_bytes, part_at, dst;
  std::vector<WriteStatus> status(n);
  WritePlace place{};
  std::vector<uint8_t> cs;
  const bool sop = (flags & B2K_CS_SOP) != 0, eph = (flags & B2K_CS_EPH) != 0;
  const bool plt = (flags & B2K_CS_PLT) != 0, tlm = (flags & B2K_CS_TLM) != 0;
  auto poison = [&](uint32_t s, bool on) {
    outs.poison_others(n, s, on);
    hdr.poison_others(n, s, on);
    tags.poison_others(n, s, on);
    hdr_len.poison_others(n, s, on);
    body_len.poison_others(n, s, on);
    pkt_at.poison_others(n, s, on);
    part_plt.poison_others(n, s, on);
    part_bytes.poison_others(n, s, on);
    part_at.poison_others(n, s, on);
    dst.poison_others(n, s, on);
  };
  /* the output bytes of every stream but s (once the streams are placed and fit) */
  auto poison_out = [&](uint32_t s, bool on, uint64_t cap) {
    if(place.used > cap)
      return;
    for(uint32_t j = 0; j < n; ++j)
      if(j != s && status[j].total)
      {
        if(on)
          POISON(cs.data() + status[j].at, status[j].total);
        else
          UNPOISON(cs.data() + status[j].at, status[j].total);
      }
  };
  auto round = [&](uint64_t cap) {
    cs.assign(cap + 1, 0);
    hdr.init(n, P.hdr_bytes);
    tags.init(n, P.tag_nodes);
    hdr_len.init(n, np);
    body_len.init(n, np);
    pkt_at.init(n, np);
    part_plt.init(n, nparts);
    part_bytes.init(n, nparts);
    part_at.init(n, nparts);
    dst.init(n, ncoded);
    std::fill(status.begin(), status.end(), WriteStatus{});
    place = WritePlace{};
    for(uint32_t s = 0; s < n; ++s)
    {
      poison(s, true);
      for(uint64_t p = 0; p < np; ++p)
        write_header(s * np + p, P.packets.data(), np, coded.data(), kmax.data(), ncoded, outs.data(), hdr.data(), P.hdr_bytes, tags.data(),
                     P.tag_nodes, hdr_len.data(), body_len.data(), dst.data(), status.data(), sop, eph);
      poison(s, false);
    }
    for(uint32_t s = 0; s < n; ++s)
    {
      poison(s, true);
      for(uint64_t t = 0; t < nparts; ++t)
        write_part(s * nparts + t, P.parts.data(), nparts, np, hdr_len.data(), body_len.data(), part_plt.data(), part_bytes.data(),
                   status.data(), plt);
      poison(s, false);
    }
    write_scan_host(n, part_bytes.data(), nparts, part_at.data(), P.head.size(), status.data(), &place);
    for(uint32_t s = 0; s < n; ++s)
    {
      poison(s, true);
      poison_out(s, true, cap);
      for(uint64_t t = 0; t < nparts; ++t)
        write_emit(s * nparts + t, P.parts.data(), nparts, np, part_at.data(), part_plt.data(), part_bytes.data(), hdr_len.data(),
                   body_len.data(), pkt_at.data(), cs.data(), cap, status.data(), &place, P.head.data(), P.head.size(), plt, tlm,
                   P.tlm_at);
      for(uint64_t p = 0; p < np; ++p)
        write_packet(s * np + p, 0, 1, P.packets.data(), np, coded.data(), ncoded, outs.data(), hdr.data(), P.hdr_bytes, hdr_len.data(),
                     pkt_at.data(), dst.data(), cs.data(), cap, status.data(), &place);
      /* the gather (ht_enc.cu k_ht_gather): a block's bytes to its place, unless it overflowed or is not placed */
      for(uint64_t k = 0; k < ncoded; ++k)
      {
        const HtBlockOut& o = outs.v[s * ncoded + k];
        const uint64_t at = dst.v[s * ncoded + k];
        if(o.total == 0xFFFFFFFFu || at + o.total > cap)
          continue;
        const b2k_block& b = B[s].table[coded_index[k]];
        memcpy(cs.data() + at, B[s].data.data() + b.offset, o.total);
      }
      poison_out(s, false, cap);
      poison(s, false);
    }
  };
  round(0);
  const uint64_t need = place.used;
  round(need);
  int bad = 0;
  uint64_t end = 0;
  for(uint32_t s = 0; s < n; ++s)
  {
    const Stream& S = B[s];
    std::string text, why;
    const int64_t r = write_verdict(status[s], &text);
    const uint64_t at = status[s].at, len = r > 0 ? (uint64_t)r : 0;
    if(place.used != need)
      why = "the second round asked for other bytes";
    if(r > 0)
    {
      b2k_result R{};
      R.num_blocks = S.table.size();
      R.blocks = const_cast<b2k_block*>(S.table.data());
      R.bytes = const_cast<uint8_t*>(S.data.data());
      R.num_bytes = S.data.size();
      R.num_tiles = ntiles;
      const int64_t hn = b2k_codestream_write(&cp, &R, flags, nullptr, 0);
      std::vector<uint8_t> want(hn > 0 ? hn : 0);
      if(hn <= 0 || b2k_codestream_write(&cp, &R, flags, want.data(), want.size()) != hn)
        why = "the host writer fails: " + g_err;
      else if((uint64_t)hn != len)
        why = "length " + std::to_string(len) + " against the host writer's " + std::to_string(hn);
      else if(memcmp(cs.data() + at, want.data(), len))
        why = "bytes differ from the host writer's";
      if(at % 256 || at < end || at + len > need)
        why = "misplaced at " + std::to_string(at);
      end = at + len;
      if(FILE* f = fopen((S.table_path + ".cs").c_str(), "wb"))
      {
        fwrite(cs.data() + at, 1, len, f);
        fclose(f);
      }
    }
    if(why.empty())
      printf("%s %lld %llu %llu same %s\n", S.name.c_str(), (long long)(r > 0 ? 0 : r), (unsigned long long)at, (unsigned long long)len,
             text.c_str());
    else
    {
      printf("%s %lld %llu %llu %s\n", S.name.c_str(), (long long)r, (unsigned long long)at, (unsigned long long)len, why.c_str());
      ++bad;
    }
  }
  return bad;
}

int main(int argc, char** argv)
{
  int bad = 0;
  for(int i = 1; i < argc;)
  {
    if(strcmp(argv[i], "--") || i + 2 >= argc)
    {
      fprintf(stderr, "usage: %s -- FLAGS CODING NAME TABLE DATA INJECT... [-- ...]\n", argv[0]);
      return 2;
    }
    const uint32_t flags = (uint32_t)strtoul(argv[i + 1], nullptr, 0);
    const std::vector<uint8_t> cpb = read_file(argv[i + 2]);
    b2k_coding cp{};
    if(cpb.size() != sizeof cp)
    {
      fprintf(stderr, "%s: not a b2k_coding\n", argv[i + 2]);
      return 2;
    }
    memcpy(&cp, cpb.data(), sizeof cp);
    i += 3;
    std::vector<Stream> B;
    while(i + 3 < argc && strcmp(argv[i], "--"))
    {
      Stream S;
      S.name = argv[i];
      S.table_path = argv[i + 1];
      const std::vector<uint8_t> t = read_file(argv[i + 1]);
      S.table.resize(t.size() / sizeof(b2k_block));
      if(!S.table.empty())
        memcpy(S.table.data(), t.data(), S.table.size() * sizeof(b2k_block));
      S.data = read_file(argv[i + 2]);
      S.inject = strtol(argv[i + 3], nullptr, 0);
      B.push_back(std::move(S));
      i += 4;
    }
    if(B.empty())
      return 2;
    bad += run_batch(flags, cp, B);
  }
  return bad ? 1 : 0;
}
