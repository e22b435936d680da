"""TEST INFRASTRUCTURE: a plain-Python restatement of Grok's T2 for the path this repo covers -- main header, tile parts
and packets of an HTJ2K codestream with one layer in LRCP order -- written independently of grok_b200/csrc/codestream.cpp
so that the two can be compared byte for byte.  It follows the reference's writer step by step:
  main header order     codestream/compress/CodeStreamCompress.cpp L1064-1098 (SOC, SIZ, CAP, COD, QCD, [TLM])
  CAP / MAGB            t2/quantizer/part15/QuantizerOJPH.cpp L259-330
  packet header / body  t2/T2Compress.cpp L261-489 (empty-packet bit always 1, inclusion + zero-bit-plane tag trees,
                        putnumpasses, comma-coded Lblock increment, lengths, flush; bodies in band / block order)
  tag tree              t2/TagTree.h (encode with threshold, value known once written)
  bit stuffing          t1_t2 BitIO: after a 0xFF byte the next one carries 7 bits; flush appends a byte after 0xFF
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


def packets_lrcp(cp, tile_index):
    """[(resno, comp, precno, [(gw, gh, [block indices into enumerate_all(cp, tiles=[tile])])] per band)] in LRCP order."""
    blks = P.enumerate_all(cp, tiles=[tile_index])
    by = {}
    for i, (t, c, b) in enumerate(blks):
        by.setdefault((b.resno, c, b.precno, b.band_index), []).append((b.cblkno, i, b))
    x0, y0, x1, y1 = P.tile_rects(cp)[tile_index]
    out = []
    for r in range(cp.numres):
        nd = cp.numres - 1 - r
        rx0, ry0 = -(-x0 // (1 << nd)), -(-y0 // (1 << nd))
        rx1, ry1 = -(-x1 // (1 << nd)), -(-y1 // (1 << nd))
        pw, ph = cp.prcw_exp[r] or 15, cp.prch_exp[r] or 15
        if rx1 <= rx0 or ry1 <= ry0:
            continue
        gw = -(-rx1 // (1 << pw)) - (rx0 >> pw)
        gh = -(-ry1 // (1 << ph)) - (ry0 >> ph)
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
                out.append((r, c, p, bands))
    return out, blks


def write_codestream(cp, table, data, tlm=False, plt=False):
    """table: the FULL block table (enumeration order, all tiles), data: its byte arena."""
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
    o += b"\xff\x52" + _u16(12 + (cp.numres if user else 0)) + bytes([1 if user else 0, 0]) + _u16(1)
    o += bytes([1 if cp.mct else 0, cp.numres - 1, cp.cblkw_exp - 2, cp.cblkh_exp - 2, 0x40 | (cp.cblk_sty & 8),
                0 if cp.irreversible else 1])
    if user:
        o += bytes([((cp.prch_exp[r] or 15) << 4) | (cp.prcw_exp[r] or 15) for r in range(cp.numres)])
    o += b"\xff\x5c" + _u16(3 + len(expn) * (2 if cp.irreversible else 1)) + bytes([(cp.numgbits << 5) | (2 if cp.irreversible else 0)])
    for e, m in zip(expn, mant):
        o += _u16((int(e) << 11) | int(m)) if cp.irreversible else bytes([int(e) << 3])
    parts = []
    first = 0
    for t in range(len(rects)):
        pk, blks = packets_lrcp(cp, t)
        rows = table[first:first + len(blks)]
        first += len(blks)
        body, lens = bytearray(), []
        for (r, c, p, bands) in pk:
            bits = Bits()
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
            start = len(body)
            body += bits.flush()
            for gw, gh, idx in bands:
                for i in idx:
                    row = rows[i]
                    if row["numpasses"] and row["length"]:
                        n = int(row["length"]) + (int(row["length2"]) if row["numpasses"] > 1 else 0)
                        body += bytes(data[int(row["offset"]):int(row["offset"]) + n])
            lens.append(len(body) - start)
        tp = bytearray()
        pl = bytearray()
        if plt:
            seg = bytearray()
            for L in lens:
                g = []
                while True:
                    g.append(L & 0x7F)
                    L >>= 7
                    if not L:
                        break
                seg += bytes([(v | 0x80) if k else v for k, v in list(enumerate(g))[::-1]])
            pl = b"\xff\x58" + _u16(len(seg) + 3) + b"\x00" + seg
        psot = 12 + len(pl) + 2 + len(body)
        tp += b"\xff\x90" + _u16(10) + _u16(t) + _u32(psot) + bytes([0, 1]) + pl + b"\xff\x93" + body
        parts.append(bytes(tp))
    if tlm:
        o += b"\xff\x55" + _u16(4 + 6 * len(parts)) + bytes([0, 0x60])
        for t, tp in enumerate(parts):
            o += _u16(t) + _u32(len(tp))
    for tp in parts:
        o += tp
    o += b"\xff\xd9"
    return np.frombuffer(bytes(o), np.uint8)
