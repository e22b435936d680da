"""TEST INFRASTRUCTURE: a plain-Python restatement of Grok's T2 for the path this repo covers -- main header, tile parts
and packets of an HTJ2K codestream with one layer, in any of the five progression orders, with SOP / EPH, a tile part per
resolution and TLM / PLT split into several marker segments -- written independently of grok_b200/csrc/codestream.cpp
(and its shared bit writer, csrc/t2_packet.h) so that the two can be compared byte for byte.  It follows the reference's writer step by step:
  main header order     codestream/compress/CodeStreamCompress.cpp L1064-1098 (SOC, SIZ, CAP, COD, QCD, [TLM])
  CAP / MAGB            t2/quantizer/part15/QuantizerOJPH.cpp L259-330
  packet header / body  t2/T2Compress.cpp L261-489 (empty-packet bit always 1, inclusion + zero-bit-plane tag trees,
                        putnumpasses, comma-coded Lblock increment, lengths, flush; bodies in band / block order)
  tag tree              t2/TagTree.h (encode with threshold, value known once written)
  bit stuffing          t1_t2 BitIO: after a 0xFF byte the next one carries 7 bits; flush appends a byte after 0xFF
  packet order          T.800 B.12.1.1-B.12.1.5 as the literal nested loops: layer / resolution / component / precinct,
                        and for RPCL, PCRL, CPRL the walk over the tile's reference grid with the precinct-origin tests
  SOP / EPH             T.800 A.8.1 (FF91, Lsop = 4, Nsop = the packet's index in its tile mod 65536), A.8.2 (FF92)
  TLM / PLT             A.7.1 (at most 10,000 entries per segment, Ztlm = 0, 1, ...; Stlm = 0x60), A.7.3 (a segment is
                        closed before an entry would take Iplt past 65,532 bytes; entries are never split; Zplt = 0, 1, ...)
Pinning: whole codestreams written this way are byte-identical to grk_compress's (the real libgrokj2k built by
oracle/build_ref.sh; tests/test_interop.py, COM marker aside), and OpenJPEG decodes them (tests/test_codestream.py).
Pure Python loops: small cases only."""
import numpy as np

import oracle_lib as O
import oracle_pipeline as P


class Bits:
    def __init__(self):
        self.out = bytearray()
        self.acc, self.room, self.cap = 0, 8, 8

    def put(self, b):
        self.room -= 1
        self.acc |= (b & 1) << self.room
        if self.room == 0:
            self._emit()

    def put_n(self, v, n):
        for i in range(n - 1, -1, -1):
            self.put((v >> i) & 1)

    def _emit(self):
        self.out.append(self.acc)
        self.cap = self.room = 7 if self.acc == 0xFF else 8
        self.acc = 0

    def flush(self):
        if self.room != self.cap:
            self._emit()
        if self.out and self.out[-1] == 0xFF:
            self._emit()
        return bytes(self.out)


class TagTree:
    """T.800 B.10.2: quad tree of minima; encode(leaf, threshold) emits what is not known yet about 'value < threshold'."""

    def __init__(self, w, h):
        self.levels = []
        while True:
            self.levels.append((w, h))
            if w <= 1 and h <= 1:
                break
            w, h = (w + 1) // 2, (h + 1) // 2
        self.val = [[10 ** 9] * (a * b) for a, b in self.levels]
        self.low = [[0] * (a * b) for a, b in self.levels]
        self.known = [[False] * (a * b) for a, b in self.levels]

    def _path(self, leaf):
        x, y = leaf % self.levels[0][0], leaf // self.levels[0][0]
        path = []
        for lv, (w, _) in enumerate(self.levels):
            path.append((lv, y * w + x))
            x, y = x // 2, y // 2
        return path[::-1]

    def set(self, leaf, v):
        for lv, i in self._path(leaf):
            self.val[lv][i] = min(self.val[lv][i], v)

    def encode(self, bits, leaf, threshold):
        low = 0
        for lv, i in self._path(leaf):
            low = max(low, self.low[lv][i])
            while low < threshold:
                if low >= self.val[lv][i]:
                    if not self.known[lv][i]:
                        bits.put(1)
                        self.known[lv][i] = True
                    break
                bits.put(0)
                low += 1
            self.low[lv][i] = low


def _floorlog2(v):
    return v.bit_length() - 1


def _u16(v):
    return int(v).to_bytes(2, "big")


def _u32(v):
    return int(v).to_bytes(4, "big")


# flag bits of b2k_codestream_write (include/grok_b200.h), restated so that this module stays free of the product
TLM, PLT, TPARTS_R, SOP, EPH = 1, 2, 4, 16, 32
TLM_PER_SEGMENT = 10000
IPLT_MAX = 65535 - 3


def tile_blocks(cp):
    """[(first index into enumerate_all(cp), [(comp, block)])] per tile: the enumeration walked once"""
    out = []
    for i, (t, c, b) in enumerate(P.enumerate_all(cp)):
        while len(out) <= t:
            out.append((i, []))
        out[t][1].append((c, b))
    rects = P.tile_rects(cp)
    while len(out) < len(rects):
        out.append((0, []))
    return out


def _ceil_shift(v, s):
    return -(-v >> s)


def resolution_grid(cp, rect, r):
    """(nd, trx0, try0, PPx, PPy, precincts across, precincts down) of resolution r of the tile at rect; no precincts
    when the resolution is empty (T.800 B.5, B.6)"""
    x0, y0, x1, y1 = rect
    nd = cp.numres - 1 - r
    rx0, ry0, rx1, ry1 = (_ceil_shift(v, nd) for v in (x0, y0, x1, y1))
    pw, ph = cp.prcw_exp[r] or 15, cp.prch_exp[r] or 15
    if rx1 <= rx0 or ry1 <= ry0:
        return nd, rx0, ry0, pw, ph, 0, 0
    return nd, rx0, ry0, pw, ph, _ceil_shift(rx1, pw) - (rx0 >> pw), _ceil_shift(ry1, ph) - (ry0 >> ph)


def tile_packets(cp, rect, blocks):
    """{(resno, comp, precno): [(gw, gh, [block indices into `blocks`])] per band} of one tile; blocks = [(comp, block)]"""
    by = {}
    for i, (c, b) in enumerate(blocks):
        by.setdefault((b.resno, c, b.precno, b.band_index), []).append((b.cblkno, i, b))
    out = {}
    for r in range(cp.numres):
        _, _, _, pw, ph, gw, gh = resolution_grid(cp, rect, r)
        for c in range(cp.numcomps):
            for p in range(gw * gh):
                bands = []
                for bi in range(1 if r == 0 else 3):
                    lst = sorted(by.get((r, c, p, bi), []))
                    if not lst:
                        bands.append((0, 0, []))
                        continue
                    cbw = min(cp.cblkw_exp, pw - (1 if r else 0))
                    cbh = min(cp.cblkh_exp, ph - (1 if r else 0))
                    xs = sorted({b.x0 >> cbw for _, _, b in lst})
                    ys = sorted({b.y0 >> cbh for _, _, b in lst})
                    bands.append((len(xs), len(ys), [i for _, i, _ in lst]))
                out[(r, c, p)] = bands
    return out


def packet_order(cp, rect, prog):
    """[(resno, comp, precno)] of one tile in progression order `prog` (0 LRCP .. 4 CPRL), one layer, written as the
    nested loops of T.800 B.12.1.1-B.12.1.5.  For the position-driven orders x and y walk the tile's reference grid; a
    precinct is met where its origin lies (x divisible by 2^(PPx + NL - r)), or at the tile's edge when the resolution's
    first precinct column / row starts before the tile.  x steps to the next multiple of the smallest precinct step
    after the tile's x0 (as OpenJPEG's pi_next_rpcl does), so a tile origin off that step is visited too."""
    x0, y0, x1, y1 = rect
    nres, ncomp = cp.numres, cp.numcomps
    grids = [resolution_grid(cp, rect, r) for r in range(nres)]
    if prog in (0, 1):              # LRCP: l, r, c, p; RLCP: r, l, c, p -- the same walk with one layer
        return [(r, c, p) for r in range(nres) for c in range(ncomp) for p in range(grids[r][5] * grids[r][6])]
    live = [g for g in grids if g[5]]
    if not live:
        return []
    dx = min(1 << (g[3] + g[0]) for g in live)
    dy = min(1 << (g[4] + g[0]) for g in live)

    def steps(lo, hi, d):
        v = lo
        while v < hi:
            yield v
            v += d - v % d

    def precinct(r, x, y):
        nd, rx0, ry0, pw, ph, gw, gh = grids[r]
        if not gw:
            return None
        if not (x % (1 << (pw + nd)) == 0 or (x == x0 and (rx0 << nd) % (1 << (pw + nd)))):
            return None
        if not (y % (1 << (ph + nd)) == 0 or (y == y0 and (ry0 << nd) % (1 << (ph + nd)))):
            return None
        kx = (_ceil_shift(x, nd) >> pw) - (rx0 >> pw)
        ky = (_ceil_shift(y, nd) >> ph) - (ry0 >> ph)
        return ky * gw + kx

    out = []
    if prog == 2:                   # RPCL
        for r in range(nres):
            for y in steps(y0, y1, dy):
                for x in steps(x0, x1, dx):
                    for c in range(ncomp):
                        k = precinct(r, x, y)
                        if k is not None:
                            out.append((r, c, k))
    elif prog == 3:                 # PCRL
        for y in steps(y0, y1, dy):
            for x in steps(x0, x1, dx):
                for c in range(ncomp):
                    for r in range(nres):
                        k = precinct(r, x, y)
                        if k is not None:
                            out.append((r, c, k))
    else:                           # CPRL
        for c in range(ncomp):
            for y in steps(y0, y1, dy):
                for x in steps(x0, x1, dx):
                    for r in range(nres):
                        k = precinct(r, x, y)
                        if k is not None:
                            out.append((r, c, k))
    return out


def packet_header(bits, bands, rows):
    """the header bits of one packet (T.800 B.10, T.814 B.10.7): rows[i] is block i's table row"""
    bits.put(1)
    for gw, gh, idx in bands:
        if not idx:
            continue
        incl, imsb = TagTree(gw, gh), TagTree(gw, gh)
        for k, i in enumerate(idx):
            inc = rows[i]["numpasses"] and rows[i]["length"]
            incl.set(k, 0 if inc else 1)
            if inc:
                imsb.set(k, int(rows[i]["kmax"]) - int(rows[i]["numbps"]))
        for k, i in enumerate(idx):
            row = rows[i]
            incl.encode(bits, k, 1)
            if not (row["numpasses"] and row["length"]):
                continue
            imsb.encode(bits, k, 10 ** 8)
            npass = int(row["numpasses"])
            if npass == 1:
                bits.put(0)
            elif npass == 2:
                bits.put_n(2, 2)
            else:
                bits.put_n(12, 4)
            len1, len2 = int(row["length"]), int(row["length2"]) if npass > 1 else 0
            lblock, x2 = 3, (_floorlog2(npass - 1) if npass > 1 else 0)
            inc = max(0, _floorlog2(len1) + 1 - lblock)
            if npass > 1:
                inc = max(inc, _floorlog2(max(len2, 1)) + 1 - (lblock + x2))
            for _ in range(inc):
                bits.put(1)
            bits.put(0)
            lblock += inc
            bits.put_n(len1, lblock)
            if npass > 1:
                bits.put_n(len2, lblock + x2)
    return bits.flush()


def plt_segments(lens):
    """PLT marker segments (A.7.3) for packet lengths `lens`; one empty segment when there are none"""
    segs, cur = [], bytearray()
    for L in lens:
        g = []
        while True:
            g.append(L & 0x7F)
            L >>= 7
            if not L:
                break
        entry = bytes([(v | 0x80) if k else v for k, v in list(enumerate(g))[::-1]])
        if len(cur) + len(entry) > IPLT_MAX:
            segs.append(cur)
            cur = bytearray()
        cur += entry
    segs.append(cur)
    return b"".join(b"\xff\x58" + _u16(len(s) + 3) + bytes([z]) + s for z, s in enumerate(segs))


def tlm_segments(entries):
    """TLM marker segments (A.7.1): at most TLM_PER_SEGMENT (tile, length) entries each, Ttlm 16 bits, Ptlm 32 bits"""
    o = bytearray()
    for z, e0 in enumerate(range(0, len(entries), TLM_PER_SEGMENT)):
        part = entries[e0:e0 + TLM_PER_SEGMENT]
        o += b"\xff\x55" + _u16(4 + 6 * len(part)) + bytes([z, 0x60])
        for t, n in part:
            o += _u16(t) + _u32(n)
    return bytes(o)


def write_codestream(cp, table, data, tlm=False, plt=False, sop=False, eph=False, prog=0, tparts=False, places=None):
    """table: the FULL block table (enumeration order, all tiles), data: its byte arena.  tparts: a tile part per
    resolution, for the resolution-major orders (LRCP, RLCP, RPCL) only, as the writer does.  places: a dict that
    receives, per table row whose bytes the stream carries, where in the stream they start."""
    expn, mant = P.quant_tables(cp)
    rects = P.tile_rects(cp)
    o = bytearray(b"\xff\x4f\xff\x51")
    o += _u16(38 + 3 * cp.numcomps) + _u16(0x4000) + _u32(cp.x1) + _u32(cp.y1) + _u32(cp.x0) + _u32(cp.y0)
    tw, th = (cp.tw, cp.th) if cp.tw else (cp.x1 - cp.x0, cp.y1 - cp.y0)
    tx0, ty0 = (cp.tx0, cp.ty0) if cp.tw else (cp.x0, cp.y0)
    o += _u32(tw) + _u32(th) + _u32(tx0) + _u32(ty0) + _u16(cp.numcomps)
    for _ in range(cp.numcomps):
        o += bytes([(cp.prec - 1) | (0x80 if cp.sgnd else 0), 1, 1])
    B = 0
    for i in range(len(expn)):
        if not cp.irreversible:
            B = max(B, int(expn[i]) + cp.numgbits - 1)
        elif cp.qcd_explicit:
            nb = (cp.numres - 1) - ((i - 1) // 3 if i else 0)
            B = max(B, max(0, int(expn[i]) + cp.numgbits - nb))
        elif i < 3 * (cp.numres - 1) + 1:
            # QuantizerOJPH::get_MAGBp as it actually runs (Sqcd's style bits are never set, Quantizer.cpp L24): the
            # reversible branch over the first 3*ndecomp+1 BYTES of the little-endian 16-bit SPqcd array
            word = (int(expn[i // 2]) << 11) | int(mant[i // 2])
            byte = (word >> 8) & 0xFF if i & 1 else word & 0xFF
            B = max(B, (byte >> 3) + cp.numgbits - 1)
    Bp = 0 if B <= 8 else (B - 8 if B < 28 else (13 + (B >> 2) if B < 48 else 31))
    o += b"\xff\x50" + _u16(8) + _u32(0x00020000) + _u16((0x20 if cp.irreversible else 0) | Bp)
    user = any((cp.prcw_exp[r] or 15) != 15 or (cp.prch_exp[r] or 15) != 15 for r in range(cp.numres))
    o += b"\xff\x52" + _u16(12 + (cp.numres if user else 0))
    o += bytes([(1 if user else 0) | (2 if sop else 0) | (4 if eph else 0), prog]) + _u16(1)
    o += bytes([1 if cp.mct else 0, cp.numres - 1, cp.cblkw_exp - 2, cp.cblkh_exp - 2, 0x40 | (cp.cblk_sty & 8),
                0 if cp.irreversible else 1])
    if user:
        o += bytes([((cp.prch_exp[r] or 15) << 4) | (cp.prcw_exp[r] or 15) for r in range(cp.numres)])
    o += b"\xff\x5c" + _u16(3 + len(expn) * (2 if cp.irreversible else 1)) + bytes([(cp.numgbits << 5) | (2 if cp.irreversible else 0)])
    for e, m in zip(expn, mant):
        o += _u16((int(e) << 11) | int(m)) if cp.irreversible else bytes([int(e) << 3])
    parts = []                                  # (tile, bytes of the tile part)
    spots = []                                  # (part, packet of the part, offset in the packet, row)
    split = tparts and prog <= 2
    for t, (first, blocks) in enumerate(tile_blocks(cp)):
        rows = table[first:first + len(blocks)]
        have = tile_packets(cp, rects[t], blocks)
        order = packet_order(cp, rects[t], prog)
        assert sorted(order) == sorted(have), "the progression walk must meet every packet of the tile once"
        runs = []                               # [(resno, [packet bytes])]
        for k, key in enumerate(order):
            bands = have[key]
            pk = bytearray()
            if sop:
                pk += b"\xff\x91" + _u16(4) + _u16(k & 0xFFFF)
            pk += packet_header(Bits(), bands, rows)
            if eph:
                pk += b"\xff\x92"
            for gw, gh, idx in bands:
                for i in idx:
                    row = rows[i]
                    if row["numpasses"] and row["length"]:
                        n = int(row["length"]) + (int(row["length2"]) if row["numpasses"] > 1 else 0)
                        spots.append([len(pk), first + i])
                        pk += bytes(data[int(row["offset"]):int(row["offset"]) + n])
            if not runs or (split and runs[-1][0] != key[0]):
                runs.append((key[0], []))
            runs[-1][1].append(bytes(pk))
            for sp in spots:
                if len(sp) == 2:
                    sp[:0] = [len(parts) + len(runs) - 1, len(runs[-1][1]) - 1]
        if not runs:                            # a tile without packets still has one (empty) tile part
            runs.append((0, []))
        assert len(runs) <= 255
        for i, (_, pks) in enumerate(runs):
            pl = plt_segments([len(p) for p in pks]) if plt else b""
            body = b"".join(pks)
            psot = 12 + len(pl) + 2 + len(body)
            parts.append((t, b"\xff\x90" + _u16(10) + _u16(t) + _u32(psot) + bytes([i, len(runs)]) + pl + b"\xff\x93" + body,
                          14 + len(pl), np.cumsum([0] + [len(p) for p in pks])))
    if tlm:
        o += tlm_segments([(t, len(tp)) for t, tp, *_ in parts])
    part_at = len(o) + np.cumsum([0] + [len(tp) for _, tp, *_ in parts])
    for _, tp, *_ in parts:
        o += tp
    if places is not None:
        for part, k, off, row in spots:
            places[row] = int(part_at[part]) + parts[part][2] + int(parts[part][3][k]) + off
    o += b"\xff\xd9"
    return np.frombuffer(bytes(o), np.uint8)


def write_flags(cp, table, data, flags):
    """write_codestream driven by b2k_codestream_write's flag word"""
    return write_codestream(cp, table, data, tlm=bool(flags & TLM), plt=bool(flags & PLT), sop=bool(flags & SOP),
                            eph=bool(flags & EPH), prog=(flags >> 8) & 7, tparts=bool(flags & TPARTS_R))
