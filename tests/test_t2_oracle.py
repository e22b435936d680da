"""The code-stream writers' shared packet and marker code (csrc/t2_packet.h) checked against references that share nothing
with it: the plain-Python T2 of tests/oracle_t2.py (byte for byte), the marker validator of tests/t2_markers.py
(structure) and OpenJPEG (pixels).  CPU only: the blocks come from the oracle's coder (test_codestream.oracle_encode), the
stream from b2k_codestream_write.  tests/test_device_t2_oracle.py holds the device writer to the same references.

The block coder codes every block that has samples, an all-zero block included (a short cleanup segment), so a table
straight from the coder includes every block.  The inclusion cases of the packet header -- blocks left out, packets with
no block at all, inclusion tag trees whose leaves differ -- are reached with `sparse` tables: the same blocks, with those
whose coefficients are all zero left out (length 0), as an encoder that skips empty blocks, or a foreign stream's parsed
table, hands them to the writer."""
import numpy as np
import pytest

import grok_b200 as G
import oracle_pipeline as P
import oracle_t2 as T2
import t2_markers as M
from test_codestream import oracle_decode, oracle_encode, openjpeg_pillow
from test_device_codestream import FLAGS

# ---------------------------------------------------------------------------------------------------------------------
# the case list: geometries x contents, plus the edge shapes
# ---------------------------------------------------------------------------------------------------------------------
GEOMS = {
    # precincts of a different size per resolution, ragged tiles, odd image and tile-grid origins
    "prec-ragged": dict(width=290, height=203, numcomps=3, prec=8, numres=4, tile=(128, 96), origin=(5, 3), tile_origin=(2, 1),
                        precincts=[(16, 16), (32, 16), (32, 64), (64, 64)], cblk=(16, 16)),
    # a tile grid anchored before the image, tall blocks
    "grid-before-image": dict(width=130, height=70, numcomps=3, prec=8, numres=3, tile=(64, 64), origin=(64, 33),
                              tile_origin=(1, 1), cblk=(16, 64)),
    # small precincts at an odd origin: precincts cut by the tile edge, bands of one block
    "small-precincts": dict(width=133, height=117, numcomps=1, prec=8, numres=5, origin=(3, 5),
                            precincts=[(8, 8), (16, 16), (32, 32)], cblk=(8, 8)),
    # tiles 1 to 3 samples wide and tall at an odd origin, five wavelet levels and small precincts: resolutions without
    # samples, hence without precincts or packets, beside ones whose only precinct is cut by the tile edge
    "sliver-tiles": dict(width=67, height=37, numcomps=3, prec=8, numres=6, tile=(32, 32), origin=(31, 31), tile_origin=(1, 2),
                         precincts=[(4, 4), (8, 8), (16, 16)], cblk=(8, 8)),
    # 4x4 blocks: 16 x 16 blocks in the LL band's one precinct, a five-level tag tree
    "4x4-blocks": dict(width=256, height=192, numcomps=1, prec=8, numres=3, cblk=(4, 4)),
    # no wavelet level over ragged tiles
    "no-dwt-tiles": dict(width=100, height=60, numcomps=3, prec=8, numres=1, tile=(33, 25), origin=(7, 2), cblk=(8, 8)),
    # no wavelet level, 4x4 blocks: the band is the image, so `sparse` leaves out 3 of 4 ... 255 of 256 blocks by quadrant
    "sparse-band": dict(width=128, height=128, numcomps=1, prec=8, numres=1, cblk=(4, 4)),
    # 9/7
    "97": dict(width=160, height=96, numcomps=3, prec=8, numres=4, irreversible=True, tile=(96, 64), precincts=[(32, 32)]),
}
CONTENTS = ["zero", "flat", "sparse", "noise", "synthetic"]
# 16 bit, 7 guard bits and 2 more in every band exponent: Kmax 29, the deepest zero-bit-plane trees
KMAX29 = dict(width=96, height=80, numcomps=1, prec=16, numres=6, numgbits=7, qcd_raise=3)

EDGES = {
    # 1,025 tile parts of one tile each: the tile-part scan's second round holds one
    "1025-parts": (dict(width=164, height=100, numcomps=1, prec=8, numres=1, tile=(4, 4)), "synthetic", G.CS_TLM | G.CS_PLT),
    # 1,056 tiles x a tile part per resolution: 3,168 tile parts, three full rounds and a partial fourth
    "3168-parts": (dict(width=256, height=264, numcomps=1, prec=8, numres=3, tile=(8, 8)), "synthetic",
                   G.CS_TLM | G.CS_PLT | G.CS_TPARTS_R),
    # exactly one full TLM segment, and one entry more
    "10000-parts": (dict(width=400, height=400, numcomps=1, prec=8, numres=1, tile=(4, 4)), "noise", G.CS_TLM),
    "10001-parts": (dict(width=548, height=292, numcomps=1, prec=8, numres=1, tile=(4, 4)), "noise", G.CS_TLM | G.CS_PLT),
    # 65,792 packets in one tile part: Nsop wraps, and PLT splits; 16-bit noise gives 2-byte entries, the empty packets of
    # three mid-scale precincts 1-byte ones, so that a 2-byte entry meets the end of a segment
    "plt-split": (dict(width=2048, height=2056, numcomps=1, prec=16, numres=1, precincts=[(8, 8)]), "noise-corner",
                  G.CS_PLT | G.CS_SOP | G.CS_EPH),
    # lengths searched so that a packet header ends on 0xFF and flush appends a byte (the arena is zeros)
    "ff-ending-header": (dict(width=16, height=8, numcomps=1, prec=8, numres=1, cblk=(8, 8)), "ff-end", G.CS_PLT | G.CS_SOP),
    # one precinct band of 64 x 64 noise blocks
    "4096-block-band": (dict(width=256, height=256, numcomps=1, prec=8, numres=1, cblk=(4, 4)), "noise", G.CS_TLM | G.CS_PLT),
}


def coding(args):
    from test_dynamic_range import coding as dr_coding
    return dr_coding(args)


def image(args, kind, seed=7):
    w, h, n, prec = args["width"], args["height"], args["numcomps"], args["prec"]
    origin = args.get("origin", (0, 0))
    mid = 1 << (prec - 1)
    if kind == "synthetic":
        return P.synthetic_image(w, h, n, prec, seed=seed, origin=origin)
    if kind == "zero":              # mid-scale: every coefficient 0
        return [np.full((h, w), mid, np.int32) for _ in range(n)]
    if kind == "flat":              # off mid-scale: only the LL band has non-zero coefficients
        return [np.full((h, w), mid // 3 + 5 * c, np.int32) for c in range(n)]
    rng = np.random.default_rng(seed)
    if kind in ("noise", "noise-corner"):
        planes = [rng.integers(0, 1 << prec, (h, w)).astype(np.int32) for _ in range(n)]
        if kind == "noise-corner":
            for p in planes:
                p[:8, :24] = mid
        return planes
    assert kind == "sparse"
    # impulses on a grid of 4-sample cells whose period doubles from quadrant to quadrant: without a wavelet level and
    # with 4x4 blocks, one block in 4, 16, 64 and 256 of the band carries one; with levels they spread over each band
    planes = [np.full((h, w), mid, np.int32) for _ in range(n)]
    y, x = np.mgrid[0:h, 0:w]
    period = np.where(y < h // 2, np.where(x < w // 2, 8, 16), np.where(x < w // 2, 32, 64))
    hit = (x % period == 1) & (y % period == 2)
    for c, p in enumerate(planes):
        p[hit] = mid + (mid // 2 if c == 0 else -(mid // 3))
    return planes


def sparse_table(cp, table, data):
    """the coder's table with every block whose decoded coefficients are all zero left out (length 0)"""
    t = table.copy()
    blks = P.enumerate_all(cp)
    for i, (_, c, b) in enumerate(blks):
        n = int(t[i]["length"])
        if n and not np.any(P.decode_block(cp, data[int(t[i]["offset"]):int(t[i]["offset"]) + n], c, b)):
            t[i]["length"] = 0
    return t


_cache = {}


def encoded(args, kind):
    """(cp, planes, coder table, sparse table, arena), computed once per module run"""
    key = (repr(sorted(args.items())), kind)
    if key not in _cache and kind == "ff-end":
        _cache[key] = ff_ending_table(args)
    if key not in _cache:
        cp = coding(args)
        planes = image(args, kind)
        table, data, _ = oracle_encode(cp, planes)
        _cache[key] = (cp, planes, table, sparse_table(cp, table, data) if kind in ("zero", "flat", "sparse") else table, data)
    return _cache[key]


def ff_ending_table(args):
    """a table for `args` (one packet of single-block bands) whose lengths and bit-plane counts are the first, in a search,
    with which the packet header ends on 0xFF"""
    cp = coding(args)
    table = G.enumerate_blocks(cp)
    (first, blocks), = T2.tile_blocks(cp)
    (bands,) = T2.tile_packets(cp, P.tile_rects(cp)[0], blocks).values()
    for numbps in range(1, int(table["kmax"].min()) + 1):
        for L in range(1, 4096):
            table["length"], table["numbps"], table["numpasses"] = L, numbps, 1
            table["offset"] = np.arange(len(table)) * L
            bits = CountingBits()
            T2.packet_header(bits, bands, table)
            if bits.stuffed_end:
                return cp, None, table, table, np.zeros(L * len(table), np.uint8)
    raise AssertionError("no length makes the header end on 0xFF")


# ---------------------------------------------------------------------------------------------------------------------
# what the case list reaches
# ---------------------------------------------------------------------------------------------------------------------
class CountingBits(T2.Bits):
    """the oracle's bit writer, noting when flush appends a byte after a final 0xFF"""
    stuffed_end = False

    def flush(self):
        if self.room != self.cap:
            self._emit()
        self.stuffed_end = bool(self.out) and self.out[-1] == 0xFF
        if self.stuffed_end:
            self._emit()
        return bytes(self.out)


def _tag_levels(gw, gh, values):
    """the levels (leaves first) of a tag tree of minima over `values` (row-major gw x gh)"""
    lv = [np.asarray(values).reshape(gh, gw)]
    while lv[-1].shape != (1, 1):
        a = lv[-1]
        hh, ww = -(-a.shape[0] // 2), -(-a.shape[1] // 2)
        pad = np.full((2 * hh, 2 * ww), 10 ** 9)
        pad[:a.shape[0], :a.shape[1]] = a
        lv.append(pad.reshape(hh, 2, ww, 2).min(axis=(1, 3)))
    return lv


def cells(cp, table, flags):
    """the conditions one (coding, table, flags) reaches"""
    out = set()
    rows = table
    included = (table["numpasses"] > 0) & (table["length"] > 0)
    if included.any():
        kmax = int(table["kmax"][included].max())
        if kmax >= 27:
            out.add("Kmax >= 27")
        if int(table["length"][included].max()) >= 1024:
            out.add("Lblock increment >= 8")
    rects = P.tile_rects(cp)
    nparts, max_packets = 0, 0
    for t, (first, blocks) in enumerate(T2.tile_blocks(cp)):
        have = T2.tile_packets(cp, rects[t], blocks)
        max_packets = max(max_packets, len(have))
        res = {k[0] for k in have}
        nparts += len(res) if (flags & G.CS_TPARTS_R and (flags >> 8) & 7 <= 2 and res) else 1
        rt = rows[first:first + len(blocks)]
        for bands in have.values():
            if not any(included[first + i] for _, _, idx in bands for i in idx):
                out.add("packet without an included block")
            for gw, gh, idx in bands:
                if gw * gh >= 4096:
                    out.add("band of >= 4096 blocks")
                inc = [0 if included[first + i] else 1 for i in idx]
                if idx and 0 < sum(inc) < len(inc):
                    lv = _tag_levels(gw, gh, inc)
                    if any(l.min() == 0 and l.max() == 1 for l in lv[3:]):
                        out.add("mixed inclusion at tree depth >= 3")
            bits = CountingBits()
            hdr = T2.packet_header(bits, bands, rt)
            if 0xFF in hdr:
                out.add("header with 0xFF")
            if bits.stuffed_end:
                out.add("header ending on 0xFF")
    if nparts > 1024 and nparts % 1024:
        out.add("> 1024 tile parts, partial last round")
    if flags & G.CS_TLM and nparts in (10000, 10001):
        out.add("%d TLM entries" % nparts)
    if flags & G.CS_SOP and max_packets > 65536:
        out.add("Nsop wraps")
    return out


ALL_CELLS = {"packet without an included block", "mixed inclusion at tree depth >= 3", "header with 0xFF",
             "header ending on 0xFF", "Lblock increment >= 8", "Kmax >= 27", "> 1024 tile parts, partial last round",
             "10000 TLM entries", "10001 TLM entries", "PLT split before a multi-byte entry", "Nsop wraps",
             "band of >= 4096 blocks"}


def plt_cells(cs):
    """the PLT conditions a written stream reaches (from the validator's walk)"""
    out = set()
    for pt in M.validate(cs)["parts"]:
        segs = pt["plt"]
        for s, nxt in zip(segs[:-1], segs[1:]):
            first = M.plt_lengths(nxt)[:1]
            if len(s) < T2.IPLT_MAX and len(first) and first[0] >= 128:
                out.add("PLT split before a multi-byte entry")
    return out


def test_case_list_reaches_every_cell():
    reached = set()
    for name, args in GEOMS.items():
        for kind in CONTENTS:
            cp, _, table, sparse, _ = encoded(args, kind)
            for t in (table, sparse):
                reached |= cells(cp, t, G.CS_TLM | G.CS_SOP)
    cp, _, table, _, _ = encoded(KMAX29, "noise")
    reached |= cells(cp, table, 0)
    for name, (args, kind, flags) in EDGES.items():
        cp, _, table, _, data = encoded(args, kind)
        reached |= cells(cp, table, flags)
        if flags & G.CS_PLT:
            reached |= plt_cells(G.codestream_write(cp, table, data, flags))
    assert reached <= ALL_CELLS, sorted(reached - ALL_CELLS)
    assert reached == ALL_CELLS, "not reached: %s" % sorted(ALL_CELLS - reached)


# ---------------------------------------------------------------------------------------------------------------------
# the host writer against the oracle, the validator and OpenJPEG
# ---------------------------------------------------------------------------------------------------------------------
def check_stream(cp, table, data, flags):
    want = T2.write_flags(cp, table, data, flags)
    got = G.codestream_write(cp, table, data, flags)
    assert len(got) == len(want) and np.array_equal(got, want), "flags 0x%x: %d vs %d bytes, first difference at %s" % (
        flags, len(got), len(want), np.flatnonzero(got[:min(len(got), len(want))] != want[:min(len(got), len(want))])[:1])
    info = M.validate(got)
    assert info["sop"] == bool(flags & G.CS_SOP) and info["eph"] == bool(flags & G.CS_EPH)
    assert bool(info["tlm"]) == bool(flags & G.CS_TLM)
    assert all(bool(pt["plt"]) == bool(flags & G.CS_PLT) for pt in info["parts"])
    return got, info


def decoded_by_openjpeg(cp, cs, planes, table, data):
    got = openjpeg_pillow(cs).astype(np.int64)
    got = got[..., None] if got.ndim == 2 else got
    src = np.stack(planes, axis=-1).astype(np.int64)
    if cp.irreversible:          # within one code of the oracle's own decode of the same stream
        ours = np.stack(oracle_decode(cp, table, data), axis=-1).astype(np.int64)
        assert got.shape == ours.shape and np.abs(got - ours).max() <= 1
    else:
        assert got.shape == src.shape and np.array_equal(got, src)


@pytest.mark.parametrize("content", CONTENTS)
@pytest.mark.parametrize("geom", list(GEOMS))
def test_host_writer_matches_the_oracle_for_every_flag(geom, content):
    cp, planes, table, sparse, data = encoded(GEOMS[geom], content)
    tables = [table] if sparse is table else [table, sparse]
    for t in tables:
        for flags in FLAGS:
            cs, _ = check_stream(cp, t, data, flags)
            if t is tables[-1] or flags in (0, FLAGS[5]):
                decoded_by_openjpeg(cp, cs, planes, t, data)


def test_kmax_29_streams_match_the_oracle():
    cp, planes, table, _, data = encoded(KMAX29, "noise")
    from test_dynamic_range import band_kmaxes
    assert max(band_kmaxes(cp)) == 29 and int(table["kmax"].max()) == 29
    for flags in FLAGS:
        cs, _ = check_stream(cp, table, data, flags)
    decoded_by_openjpeg(cp, cs, planes, table, data)


def test_empty_contents_write_empty_packets():
    """the sparse tables do what they are for: `zero` leaves every block out, `flat` keeps the LL band's and few others
    (a band sample that is alone in its row of a tile keeps a non-zero high-pass value)"""
    for name, args in GEOMS.items():
        cp, _, table, sparse, data = encoded(args, "zero")
        assert (table["length"] > 0).all() and (sparse["length"] == 0).all(), name
        cs, info = check_stream(cp, sparse, data, G.CS_PLT | G.CS_SOP | G.CS_EPH)
        # every packet: SOP, the one header byte 0x00 (empty), EPH
        assert all(np.all(pt["packets"] == 9) for pt in info["parts"]), name
        cp, _, table, sparse, data = encoded(args, "flat")
        kept = sparse["length"] > 0
        if not cp.irreversible:
            hp = table["resno"] > 0
            assert kept[~hp].any() and (not hp.any() or kept[hp].mean() < 0.5), name


@pytest.mark.parametrize("edge", list(EDGES))
def test_edge_shapes_match_the_oracle(edge):
    args, kind, flags = EDGES[edge]
    cp, _, table, _, data = encoded(args, kind)
    cs, info = check_stream(cp, table, data, flags)
    parts = info["parts"]
    if edge.endswith("-parts"):
        assert len(parts) == int(edge.split("-")[0])
        if flags & G.CS_TLM:
            assert info["tlm"] == [10000] * (len(parts) // 10000) + ([len(parts) % 10000] if len(parts) % 10000 else [])
    if edge == "plt-split":
        assert len(parts) == 1 and len(parts[0]["plt"]) >= 2 and len(parts[0]["packets"]) > 65536


# ---------------------------------------------------------------------------------------------------------------------
# the validator rejects what it is there to catch
# ---------------------------------------------------------------------------------------------------------------------
def _mutations(cs):
    """(name, damaged stream) pairs, each breaking one rule the validator checks"""
    b = bytearray(bytes(cs))
    info = M.validate(cs)
    out = []
    p = info["parts"][0]["at"]
    for d in (1, -1):                                           # Psot +- 1
        m = bytearray(b)
        m[p + 6:p + 10] = (info["parts"][0]["psot"] + d).to_bytes(4, "big")
        out.append(("Psot %+d" % d, m))
    q = bytes(b).find(b"\xff\x58", p)                           # one PLT entry + 1 (a 1-byte entry below 0x7F)
    iplt = q + 5
    k = next(i for i in range(iplt, iplt + 64) if b[i] < 0x7F and (i == iplt or b[i - 1] < 0x80))
    m = bytearray(b)
    m[k] += 1
    out.append(("PLT entry + 1", m))
    t = bytes(b).find(b"\xff\x55")                              # two TLM entries swapped
    m = bytearray(b)
    e0, e1 = t + 6, t + 12
    m[e0:e0 + 6], m[e1:e1 + 6] = b[e1:e1 + 6], b[e0:e0 + 6]
    out.append(("TLM entries swapped", m))
    s = bytes(b).find(b"\xff\x91\x00\x04", p) + 4               # Nsop of the second packet off by one
    s = bytes(b).find(b"\xff\x91\x00\x04", s) + 4
    m = bytearray(b)
    m[s:s + 2] = ((((b[s] << 8) | b[s + 1]) + 1) & 0xFFFF).to_bytes(2, "big")
    out.append(("Nsop + 1", m))
    # a repeated Zplt: the second of two PLT segments numbered 0 again
    z = bytes(b).find(b"\xff\x58", q + 2)
    m = bytearray(b)
    m[z + 4] = m[q + 4]
    out.append(("Zplt repeated", m))
    return out


def test_the_validator_rejects_broken_streams():
    cp, _, table, _, data = encoded(GEOMS["prec-ragged"], "synthetic")
    # PLT segments of at most a handful of entries would need another writer; take a stream with two PLT segments in a
    # tile part from the edge case list instead for the repeated Zplt
    cs = G.codestream_write(cp, table, data, G.CS_TLM | G.CS_PLT | G.CS_SOP | G.CS_EPH)
    M.validate(cs)
    args, kind, flags = EDGES["plt-split"]
    cp2, _, t2, _, d2 = encoded(args, kind)
    big = G.codestream_write(cp2, t2, d2, flags | G.CS_TLM)
    M.validate(big)
    names = set()
    for name, m in _mutations(cs)[:-1] + _mutations(big)[-1:]:
        with pytest.raises(M.Invalid):
            M.validate(np.frombuffer(bytes(m), np.uint8))
        names.add(name)
    assert names == {"Psot +1", "Psot -1", "PLT entry + 1", "TLM entries swapped", "Nsop + 1", "Zplt repeated"}
