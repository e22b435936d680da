"""Every parse, refill, store and refinement path of the HT block decoder (ht_dec.cu), and damaged blocks against the
reference's verdicts.

A decode launches k_ht_decode_vlc (phase A, a thread per block) as its WIDE instance when the launch's widest block is
over 64 samples, narrow blocks included; k_ht_decode_magsgn (phase B, a warp per block) as one of four instances
(IRREV x REFINE: REFINE when any block of the launch carries refinement passes), with `line_entries` exponent slots per
row; and k_ht_decode_refine when any block is refined.  `launch_plan` and `decode_fields` restate those rules and
t2::block_decode_fields' pass rules; the CPU tests pin them to hand-computed plans.

Most of the decoder's branches are decided by the coded bytes and by where they lie in the byte arena, so the model
parses each block in Python:
  - `parse_cleanup` restates phase A over the readers' 8-byte windows (vlcf_fill32's fast path, its byte path and the
    rotation inside it, the straddling and wholly-below windows, melf_bit's stuffing, forced nibble and reads past the
    segment, MEL k, every U-VLC mode and suffix length), from orc_ht_dec_table's CxtVLC rows.  Its per-quad rho is
    checked against the significance of orc_ht_decode's output on every case block.
  - `magsgn_cells` restates phase B's 256-byte refills (the lane ends, the 0xFF carried by ballot and by ms_prevff,
    the ring wrapping) and its U_q test, from the parse and the oracle's decode of the rows above.
  - `refine_cells` restates k_ht_decode_refine's stripes, bitmap words and both bit readers.
`test_cases_reach_every_cell` asserts that the geometry codings and the constructed blocks below reach every cell.

Damaged blocks (single seeded edits of valid blocks: a flipped byte in MagSgn, MEL or VLC, another Scup, Lcup, numbps,
refinement bytes or length, the pass rules) are pinned to the reference's verdicts and words by
tests/golden/ht_damaged.npz (tests/golden/make_golden_damaged.py); the oracle must give both, and the device must
reject exactly the blocks the reference rejects and decode the others to the reference's words.

GPU: the case tables through job.t1_decode_blocks at two placements in the arena (block k at residue k mod 8 with 0x00
gaps, and at (k + 4) mod 8 with 0xFF gaps and the last block ending at the arena's end); the constructed blocks alone
and 16 to a launch; the damaged corpus, one table per block shape, reversible and irreversible, at both placements; and
the same tables as 4-tile code streams (chunked launches, first_block > 0), through engine.decode and, clean and damaged
streams alternating, through decode_codestreams_device, each stream with its own rejection count.
"""
import functools
import os

import numpy as np
import pytest

import grok_b200 as G
import oracle_lib as O
import oracle_pipeline as P
import test_ht_coder_paths as CP
import test_ht_foreign as HF

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ht_damaged.npz")
WARPS_PER_CTA = 4               # B2K_WARPS_PER_CTA
RING_BITS = 256 * 32            # MS_RING_WORDS
KINDS = ("rev", "irrev")


# ---------------------------------------------------------------------------------------------------------------------
# the launch model (b2k_launch_ht_decode_vlc / _magsgn / _refine, prepare_decode, t2::block_decode_fields)
# ---------------------------------------------------------------------------------------------------------------------
def decode_fields(kmax, length, numbps, numpasses, length2):
    """(missing MSBs, passes, length2) the decoder is given for one table entry"""
    nb = numbps if length else 0
    mm = max(kmax - nb, 0)
    passes = numpasses if (length and numpasses > 1 and length2 > 0 and mm < 29) else 1
    return mm, passes, length2 if passes > 1 else 0


def launch_plan(blocks, irreversible):
    """blocks: [(w, h, passes)] of one launch"""
    n = len(blocks)
    max_w = max(w for w, _, _ in blocks)
    refine = any(p > 1 for _, _, p in blocks)
    return dict(vlc="wide" if max_w > 64 else "narrow", magsgn=(bool(irreversible), refine),
                line_entries=((max_w + 1) // 2 + 4 + 1) & ~1, vlc_ctas=-(-n // 32), vlc_tail=n % 32 != 0,
                ctas=-(-n // WARPS_PER_CTA), cta_tail=n % WARPS_PER_CTA != 0, refine=refine)


# ---------------------------------------------------------------------------------------------------------------------
# phase A: k_ht_decode_vlc restated over its 8-byte windows
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _dec_tables():
    L = O.lib()
    return tuple(np.ctypeslib.as_array(L.orc_ht_dec_table(t), (1024,)).astype(np.int64).tolist() for t in (0, 1))


MEL_EXP = (0, 0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 4, 5)          # mel_exp_d


def _uvlc_prefix(bits):
    for k in range(3):
        if bits >> k & 1:
            return k + 1, k + 1
    return 5, 3


def _uvlc_entry(mode, bits):
    """(plen, l0, l1, p0, p1) of uvlc_entry"""
    sl = lambda p: 1 if p == 3 else (5 if p == 5 else 0)      # noqa: E731
    plen = l0 = l1 = p0 = p1 = 0
    if mode < 4:
        if mode & 1:
            p0, n = _uvlc_prefix(bits)
            bits >>= n
            plen += n
            l0 = sl(p0)
        if mode & 2:
            p1, n = _uvlc_prefix(bits)
            plen += n
            l1 = sl(p1)
    else:
        p0, n = _uvlc_prefix(bits)
        bits >>= n
        plen += n
        if p0 > 2:
            p1 = 1 + (bits & 1)
            plen += 1
            l0 = sl(p0)
        else:
            p1, n = _uvlc_prefix(bits)
            plen += n
            l1 = sl(p1)
    return plen, l0, l1, p0, p1


class _Vlc:
    """VlcFast: pos / lo are segment positions, addresses are base + position (base: the block's offset mod 8)"""

    def __init__(self, data, lcup, scup, base, cells):
        self.d, self.base, self.cells = data, base, cells
        self.pos, self.lo = lcup - 3, lcup - scup
        b = int(data[lcup - 2])
        self.tmp = b >> 4
        self.bits = 4 - (1 if (self.tmp & 7) == 7 else 0)
        self.unstuff = (b | 0xF) > 0x8F
        self.A = (base + max(self.pos, 0)) & ~7
        for k in range(3):
            self._load(self.A - 8 * k)

    def _load(self, a):
        if a + 7 < self.base + self.lo:
            self.cells.add(("vlc", "window_below"))

    def _rotate(self):
        self.A -= 8
        self._load(self.A - 16)

    def _byte(self, i):
        if ((self.base + i) & ~7) < self.base + self.lo:
            self.cells.add(("vlc", "straddling_window_read"))
        return int(self.d[i])

    def fill32(self):
        if self.bits >= 32:
            return
        if self.pos - 3 >= self.lo:
            if self.base + self.pos < self.A:
                self._rotate()
            o = self.base + self.pos - self.A
            if o < 3:
                self.cells.add(("vlc", "straddle", o))
            w = 0
            for k in range(4):
                w |= self._byte(self.pos - k) << (8 * k)
            if (((w & 0x7F7F7F7F) + 0x01010101) & 0x80808080) == 0:
                self.cells.add(("vlc", "fast"))
                self.tmp |= w << self.bits
                self.bits += 32
                self.unstuff = (w >> 24) > 0x8F
                self.pos -= 4
                if self.base + self.pos < self.A:
                    self._rotate()
                return
            self.cells.add(("vlc", "bytewise", "7f"))
        else:
            self.cells.add(("vlc", "bytewise", "segment_start"))
        while self.bits < 32:
            b = 0
            if self.pos >= self.lo:
                if self.base + self.pos < self.A:
                    self.cells.add(("vlc", "bytewise_rotate"))
                    self._rotate()
                b = self._byte(self.pos)
            self.pos -= 1
            nb = 8 - (1 if (self.unstuff and (b & 0x7F) == 0x7F) else 0)
            self.tmp |= b << self.bits
            self.bits += nb
            self.unstuff = b > 0x8F


class _Mel:
    def __init__(self, data, start, size, cells):
        self.d, self.start, self.size, self.cells = data, start, size, cells
        self.pos = self.bits = self.unstuff = self.k = self.run = self.have = self.tmp = 0

    def bit(self):
        if self.bits == 0:
            v = 0xFF
            if self.pos < self.size:
                v = int(self.d[self.start + self.pos])
                if self.unstuff:
                    self.cells.add(("mel", "ff_then_7bit"))
                if self.pos == self.size - 1:
                    v |= 0xF
                    self.cells.add(("mel", "forced_nibble"))
                self.pos += 1
            else:
                self.cells.add(("mel", "past_end"))
            self.bits = 8 - self.unstuff
            self.tmp = v
            self.unstuff = int(v == 0xFF)
        self.bits -= 1
        return (self.tmp >> self.bits) & 1

    def symbol(self):
        if not self.have:
            ev = MEL_EXP[self.k]
            if self.bit():
                self.run, self.have = 1 << ev, 1
                self.k = min(12, self.k + 1)
                if self.k == 12:
                    self.cells.add(("mel", "k12"))
            else:
                r = 0
                for _ in range(ev):
                    r = (r << 1) | self.bit()
                self.run, self.have = r, 2
                self.k = max(0, self.k - 1)
        if self.run > 0:
            self.run -= 1
            if self.run == 0 and self.have == 1:
                self.have = 0
            return 0
        self.have = 0
        return 1


def parse_cleanup(data, lcup, w, h, wide, base=0):
    """k_ht_decode_vlc on one block: (status total, per quad row a list of (rho, u, e_k, e_1) per quad, cells).
    total: 0 decoded, 1 empty, 2 rejected before the parse"""
    cells = set()
    if lcup < 2:
        return (1 if lcup == 0 else 2), None, cells
    scup = (int(data[lcup - 1]) << 4) + (int(data[lcup - 2]) & 0xF)
    if scup < 2 or scup > lcup or scup > 4079:
        return 2, None, cells
    T0, T1 = _dec_tables()
    mel = _Mel(data, lcup - scup, scup - 1, cells)
    vlc = _Vlc(data, lcup, scup, base, cells)
    nq = (w + 1) >> 1
    nseg = 16 if wide else 1
    pbl, pbr = [0] * nseg, [0] * nseg
    rows = []
    for y in range(0, h, 2):
        tbl = T1 if y else T0
        rho_left, br_left = 0, 0
        row = []
        for s in range(((nq + 31) >> 5) if wide else 1):
            qs = 32 * s
            qe = min(nq, qs + 32) if wide else nq
            bl_next = pbl[s + 1] if wide and qe < nq else 0
            if y and bl_next & 1:
                cells.add(("seam", "bl_next"))
            if y and s and br_left >> 31:
                cells.add(("seam", "br_left"))
            A = pbl[s] | (bl_next << 32) | (pbr[s] << 1) | (br_left >> 31)
            br_left = pbr[s]
            cbl = cbr = 0
            for q0 in range(qs, qe, 2):
                vlc.fill32()
                has1 = q0 + 1 < nq
                j = q0 - qs
                tmp = vlc.tmp
                if y == 0:
                    cq0 = (rho_left >> 1) | (rho_left & 1)
                else:
                    cq0 = ((A >> j) & 1) | (2 if rho_left & 0xC else 0) | (((A >> (j + 1)) & 1) << 2)
                t0 = tbl[(cq0 << 7) | (tmp & 0x7F)]
                if cq0 == 0 and not mel.symbol():
                    t0 = 0
                tmp >>= t0 >> 13
                used = t0 >> 13
                rho0, t1, rho1 = t0 & 0xF, 0, 0
                if has1:
                    if y == 0:
                        cq1 = (rho0 >> 1) | (rho0 & 1)
                    else:
                        cq1 = ((A >> (j + 1)) & 1) | (2 if rho0 & 0xC else 0) | (((A >> (j + 2)) & 1) << 2)
                    t1 = tbl[(cq1 << 7) | (tmp & 0x7F)]
                    if cq1 == 0 and not mel.symbol():
                        t1 = 0
                    tmp >>= t1 >> 13
                    used += t1 >> 13
                    rho1 = t1 & 0xF
                rho_left = rho1 if has1 else rho0
                cbl |= (((rho0 >> 1) & 1) << j) | (((rho1 >> 1) & 1) << (j + 1))
                cbr |= (((rho0 >> 3) & 1) << j) | (((rho1 >> 3) & 1) << (j + 1))
                u0 = u1 = 0
                uo = ((t0 >> 12) & 1) | (((t1 >> 12) & 1) << 1)
                if uo:
                    mode, add = uo, 0
                    if y == 0 and uo == 3:
                        if mel.symbol():
                            add = 2
                            cells.add(("uvlc", "mel1"))
                        else:
                            mode = 4
                    plen, l0, l1, p0, p1 = _uvlc_entry(mode, tmp & 63)
                    cells.add(("uvlc", "mode", mode) if mode < 4 else ("uvlc", "mode4", "p0>2" if p0 > 2 else "p0<=2"))
                    for active, ln in ((mode == 4 or uo & 1, l0), (mode == 4 and p0 <= 2 or uo & 2, l1)):
                        if active:
                            cells.add(("uvlc", "suffix", ln))
                    if l0 == 5 and l1 == 5:
                        cells.add(("uvlc", "suffix5_both"))
                    tmp >>= plen
                    u0 = p0 + (tmp & ((1 << l0) - 1))
                    tmp >>= l0
                    u1 = p1 + (tmp & ((1 << l1) - 1))
                    tmp >>= l1
                    used += plen + l0 + l1
                    if uo & 1:
                        u0 += add
                    if uo & 2:
                        u1 += add
                vlc.tmp = tmp
                vlc.bits -= used
                row.append((rho0, u0, (t0 >> 4) & 0xF, (t0 >> 8) & 0xF))
                if has1:
                    row.append((rho1, u1, (t1 >> 4) & 0xF, (t1 >> 8) & 0xF))
            pbl[s], pbr[s] = cbl, cbr
        rows.append(row)
    return 0, rows, cells


def rho_matches_decode(rows, dec, w, h, upto=None):
    """the parse's rho against the significance of a decode, row pairs [0, upto)"""
    for r, row in enumerate(rows[:upto]):
        for q, (rho, *_) in enumerate(row):
            for i in range(4):
                x, y = 2 * q + (i >> 1), 2 * r + (i & 1)
                if x < w and y < h and bool(rho >> i & 1) != bool(dec[y, x]):
                    return False
    return True


# ---------------------------------------------------------------------------------------------------------------------
# phase B: k_ht_decode_magsgn's refills, rounds and U_q test
# ---------------------------------------------------------------------------------------------------------------------
def _exponent(word, p):
    """31 - clz(v_n | 2) of a decoded sample (0 when insignificant)"""
    if not word:
        return 0
    v_n = ((int(word) & 0x7FFFFFFF) >> (p - 1)) - 2
    return (v_n | 2).bit_length() - 1


def magsgn_cells(data, lcup, w, h, mm, rows, dec, vec_ok):
    """phase B of a block phase A parsed: (rejected, cells).  dec: orc_ht_decode's output (complete up to the row pair
    it rejects the block in)."""
    cells = {("vec_ok", bool(vec_ok))}
    if w % 2:
        cells.add(("ragged", "column"))
    if h % 2:
        cells.add(("ragged", "row"))
    scup = (int(data[lcup - 1]) << 4) + (int(data[lcup - 2]) & 0xF)
    ms = np.asarray(data[:lcup - scup], np.int64)
    size = len(ms)
    if size == 0:
        cells.add(("ms", "empty"))
    elif ms[-1] == 0xFF:
        cells.add(("ms", "ff_last"))
    nq = (w + 1) >> 1
    rounds = -(-nq // 32)
    cells.add(("rounds", "1" if rounds == 1 else ">1"))
    p = 30 - mm
    head = tail = pos = 0
    prevff = False
    nrefill = 0

    def refill():
        nonlocal tail, pos, prevff, nrefill
        chunk = np.full(256, 0xFF, np.int64)
        real = max(0, min(256, size - pos))
        chunk[:real] = ms[pos:pos + real]
        prev = np.concatenate([[0xFF if prevff else 0], chunk[:-1]])
        tail += int(np.sum(8 - (prev == 0xFF)))
        if tail > RING_BITS:
            cells.add(("ring", "wraps"))
        if nrefill and prevff and pos <= size:
            cells.add(("ff", "refill_carry"))
        for lane in range(32):
            at = pos + 8 * lane
            if at >= size:
                break
            left = size - at
            if left < 8:
                cells.add(("left", "1-3" if left < 4 else ("4" if left == 4 else "5-7")))
            elif left == 8:
                cells.add(("left", "8"))
            for k, name in ((3, "byte3"), (7, "ballot" if lane < 31 else "refill_carry")):
                if at + k + 1 < size and ms[at + k] == 0xFF:
                    if name != "refill_carry":
                        cells.add(("ff", name))
                    if ms[at + k + 1] >= 0x80:      # the top bit of the byte after it lands on the next byte's bit 0
                        cells.add(("ff_top_bit", name))
        if pos < size <= pos + 256 and size % 256 == 0:
            cells.add(("left", "refill_end"))
        prevff = bool(chunk[255] == 0xFF)
        pos += 256
        nrefill += 1

    labove = [0] * (nq + 3)
    for r, row in enumerate(rows):
        y = 2 * r
        lcur = [0] * (nq + 3)
        for qb in range(0, nq, 32):
            while tail - head < 4096:
                refill()
            bad = False
            for q in range(qb, min(nq, qb + 32)):
                rho, u, ek, _ = row[q]
                kappa = 1
                if y > 0 and rho & (rho - 1):
                    a, b, c = labove[q], labove[q + 1], labove[q + 2]
                    kappa = max(1, a >> 8, b & 0xFF, b >> 8, c & 0xFF)
                U = u + kappa
                if U > mm + 2:
                    bad = True
                    cells.add(("verdict", "uq", "first_pair" if y == 0 else ("later_round" if qb else "later_pair")))
                    continue
                x = 2 * q
                eff = rho if x + 1 < w else rho & 3
                head += sum(U - (ek >> i & 1) for i in range(4) if eff >> i & 1)
                eb = [0, 0]
                for i in (1, 3):
                    xx, yy = x + (i >> 1), y + 1
                    if eff >> i & 1 and yy < h:
                        eb[i >> 1] = _exponent(dec[yy, xx], p)
                lcur[q + 1] = eb[0] | (eb[1] << 8)
            if bad:
                return True, cells
        labove = lcur
    return False, cells


# ---------------------------------------------------------------------------------------------------------------------
# k_ht_decode_refine: stripes, bitmap words, the SigProp and MagRef readers
# ---------------------------------------------------------------------------------------------------------------------
def refine_cells(seg, w, h, passes, causal, sig):
    """cells of the refinement of a block whose cleanup significance is `sig` (h, w bool)"""
    cells = {("refine", "passes", passes, bool(causal)), ("refine", "h%4", h % 4)}
    nwords = -(-w // 32)
    cells.add(("refine", "nwords", "1" if nwords == 1 else ("32" if nwords == 32 else "2-31")))
    seg = np.asarray(seg, np.int64)
    size = len(seg)
    # SigProp: how many bits the scan reads, and how many the segment holds
    bits = _unstuffed_forward(bytes(seg.tolist()))
    need = 0
    s = np.zeros((h + 2, w + 2), bool)
    s[1:h + 1, 1:w + 1] = sig
    cup = s.copy()
    for y0 in range(0, h, 4):
        lim = y0 + 4 if causal else h
        for gx in range(0, w, 4):
            nnew = 0
            for x in range(gx, min(gx + 4, w)):
                for y in range(y0, min(y0 + 4, h)):
                    if cup[y + 1, x + 1]:
                        continue
                    nb = s[y:y + 3, x:x + 3].copy()
                    if y + 1 >= lim:
                        nb[2, :] = False
                    if not nb.any():
                        continue
                    k = need
                    need += 1
                    if k < len(bits) and bits[k]:
                        s[y + 1, x + 1] = True
                        nnew += 1
            need += nnew
    have = 0
    prev = 0
    for i in range(size):
        have += 7 if prev == 0xFF else 8
        prev = seg[i]
    if need > have:
        cells.add(("refine", "sigprop_exhausted"))
    if (seg[:min(size, -(-need // 7))] == 0xFF).any():
        cells.add(("refine", "sigprop_ff"))
    if passes > 2:
        nmr = int(sig.sum())
        unstuff, got = True, 0
        for i in range(size):
            if got >= nmr:
                break
            b = int(seg[size - 1 - i])
            stuffed = unstuff and (b & 0x7F) == 0x7F
            if stuffed:
                cells.add(("refine", "magref_stuffed"))
            got += 7 if stuffed else 8
            unstuff = b > 0x8F
    return cells


def _unstuffed_forward(seg_bytes):
    """SigProp's bits (LSB first, a byte after 0xFF carries 7, zeros after the end)"""
    out, prev = [], 0
    for b in seg_bytes:
        n = 7 if prev == 0xFF else 8
        out += [(b >> i) & 1 for i in range(n)]
        prev = b
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
# geometry codings: (name, make_coding arguments); each runs reversible and irreversible, cleanup-only and refined
GEOMETRIES = [
    ("64x64-odd-origin", dict(width=203, height=157, numres=3, origin=(3, 5))),
    ("128x32", dict(width=300, height=70, numres=2, cblk=(128, 32))),
    ("512x8", dict(width=1100, height=19, numres=1, cblk=(512, 8))),
    ("1024x4", dict(width=2100, height=13, numres=1, cblk=(1024, 4))),
    ("4x1024", dict(width=11, height=1100, numres=1, cblk=(4, 1024))),
]
# (npass, stripe-causal) per variant: cleanup only, then 3 and 2 passes, plain and causal between the two kinds
VARIANTS = {"rev": [(1, False), (3, False), (2, True)], "irrev": [(1, False), (3, True), (2, False)]}


@functools.lru_cache(maxsize=None)
def geometry_case(name, kind, variant):
    """(coding, block table, byte arena, the oracle's coefficient planes) of a geometry case"""
    args = dict(dict(GEOMETRIES)[name], numcomps=1, prec=12, irreversible=kind == "irrev")
    npass, causal = VARIANTS[kind][variant]
    cp = G.make_coding(**args)
    if causal:
        cp.cblk_sty = 0x08
    planes = P.synthetic_image(args["width"], args["height"], 1, 12, seed=5 + variant,
                               origin=args.get("origin", (0, 0)))
    table, data, want = HF._foreign_blocks(cp, P.forward(cp, planes), npass, 1 if npass > 1 else 0, seed=23 + variant)
    return cp, table, data, want


def _coded(table):
    return [i for i in range(len(table)) if table[i]["x1"] > table[i]["x0"] and table[i]["y1"] > table[i]["y0"]]


def table_blocks(cp, table, data):
    """the blocks of a table as the model takes them"""
    rects = P.tile_rects(cp)
    blks = P.enumerate_all(cp)
    out = []
    for i in _coded(table):
        t = table[i]
        w, h = int(t["x1"] - t["x0"]), int(t["y1"] - t["y0"])
        mm, passes, len2 = decode_fields(int(t["kmax"]), int(t["length"]), int(t["numbps"]), int(t["numpasses"]),
                                         int(t["length2"]))
        tt, _, b = blks[i]
        off, lcup = int(t["offset"]), int(t["length"])
        out.append(dict(data=np.asarray(data[off:off + lcup + int(t["length2"])], np.uint8), lcup=lcup, len2=len2,
                        w=w, h=h, mm=mm, passes=passes, causal=bool(cp.cblk_sty & 0x08), irrev=bool(cp.irreversible),
                        col=CP.plane_column(cp, rects[tt], b)))
    return out


def block_cells(b, wide, base=0):
    """every cell one block reaches, and whether the parse matched the oracle's significance"""
    kind = "irrev" if b["irrev"] else "rev"
    w, h, lcup = b["w"], b["h"], b["lcup"]
    data = b["data"]
    cells = set()
    nq = (w + 1) >> 1
    if wide:
        nseg = -(-nq // 32)
        cells.add(("segments", "1" if nseg == 1 else ("16" if nseg == 16 else "2-15")))
        if nq % 32:
            cells.add(("segments", "partial"))
        if nseg >= 2 and h > 2:
            cells.add(("segments", "seam_rows"))
    if w % 2:
        cells.add(("geometry", "odd_w"))
    if h % 2:
        cells.add(("geometry", "odd_h"))
    total, rows, pc = parse_cleanup(data, lcup, w, h, wide, base)
    cells |= pc
    ok = True
    if total == 1:
        cells.add(("verdict", "empty"))
        return cells, ok
    if total == 2:
        if lcup < 2:
            cells.add(("verdict", "lcup1"))
        else:
            scup = (int(data[lcup - 1]) << 4) + (int(data[lcup - 2]) & 0xF)
            cells.add(("verdict", "scup<2" if scup < 2 else ("scup>4079" if scup > 4079 else "scup>lcup")))
        return cells, ok
    rc, dec = O.ht_decode(data[:lcup], b["mm"], w, h)
    rejected, mc = magsgn_cells(data, lcup, w, h, b["mm"], rows, dec, b["col"] % 2 == 0)
    cells |= {c + (kind,) if c[0] in ("ring", "vec_ok") else c for c in mc}
    ok = (rc != 0) == rejected and rho_matches_decode(rows, dec, w, h, None if rc == 0 else 0)
    if b["passes"] > 1:
        if rejected:
            cells.add(("refine", "rejected_in_phase_b"))
        else:
            cells |= refine_cells(data[lcup:lcup + b["len2"]], w, h, b["passes"], b["causal"], dec != 0)
            cells.add(("refine", kind))
    return cells, ok


def _sm(coef, kmax):
    return O.to_sgnmag(np.asarray(coef, np.int64), kmax)


def _pad_magsgn(data, pad):
    """`data` with the bytes `pad` put after its MagSgn segment (Scup unchanged)"""
    lcup = len(data)
    scup = (int(data[-1]) << 4) + (int(data[-2]) & 0xF)
    return np.concatenate([data[:lcup - scup], np.asarray(pad, np.uint8), data[lcup - scup:]])


@functools.lru_cache(maxsize=None)
def constructed():
    """{label: (coefficients or None, cleanup bytes, missing MSBs)}: blocks for the cells content alone rarely reaches"""
    out = {}
    for label in ("chain-64x64-packed", "chain-1024x4", "chain-4x1024", "vlc-first-row-1024x2",
                  "vlc-first-row-1024x2-shifted", "vlc-first-row-300x2"):
        coef, _, kmax = CP.chain_case(label)
        out[label] = (coef, O.ht_encode(_sm(coef, kmax), kmax, cap=65536), kmax)
    # a long insignificant run (MEL k reaches 12, MEL bytes of 0xFF each followed by a 7-bit byte), and no MagSgn bytes
    z = np.zeros((64, 64), np.int64)
    out["mel-run-64x64"] = (z, O.ht_encode(_sm(z, 9), 9), 9)
    z = z.copy()
    z[63, 62] = -3
    out["mel-run-then-one-64x64"] = (z, O.ht_encode(_sm(z, 9), 9), 9)
    # U_q >= kappa + 5 on both quads of pairs (suffix length 5), in the first row and below
    rng = np.random.default_rng(3)
    top = rng.integers(1 << 15, 1 << 16, (64, 64)) * rng.choice([-1, 1], (64, 64))
    out["top-64x64"] = (top, O.ht_encode(_sm(top, 16), 16, cap=65536), 16)
    # MagSgn segments padded to 256 bytes (a segment that ends on a refill), the last padding byte 0xFF
    small = rng.integers(-200, 201, (16, 16)) * (rng.random((16, 16)) < 0.5)
    d = O.ht_encode(_sm(small, 9), 9)
    ms = len(d) - ((int(d[-1]) << 4) + (int(d[-2]) & 0xF))
    out["magsgn-256-16x16"] = (small, _pad_magsgn(d, rng.integers(0, 0x80, 256 - ms)), 9)
    out["magsgn-ff-last-16x16"] = (small, _pad_magsgn(d, [0x11, 0x22, 0xFF]), 9)
    out["empty-16x16"] = (np.zeros((16, 16), np.int64), np.zeros(0, np.uint8), 9)
    return out


def constructed_block(label):
    coef, data, mm = constructed()[label]
    h, w = coef.shape
    return dict(data=data, lcup=len(data), len2=0, w=w, h=h, mm=mm, passes=1, causal=False, irrev=False, col=0)


def damaged(g):
    """the blocks of tests/golden/ht_damaged.npz: (block as the model takes it, verdict, reference words or None)"""
    for i, row in enumerate(g["meta"]):
        w, h, mm, npass, lcup, len2, causal, rc, kind = (int(v) for v in row)
        data = g["data"][g["data_off"][i]:g["data_off"][i + 1]]
        dec = g["dec"][g["dec_off"][i]:g["dec_off"][i + 1]]
        _, passes, l2 = decode_fields(29, lcup, 29 - mm, npass, len2)
        b = dict(data=data, lcup=lcup, len2=l2, w=w, h=h, mm=mm, passes=passes, causal=bool(causal), irrev=False,
                 col=0, npass=npass, len2_table=len2, kind=kind)
        yield b, rc, (dec.reshape(h, w) if rc == 0 else None)


def _launch_cells(cp, table, blocks):
    kind = "irrev" if cp.irreversible else "rev"
    plan = launch_plan([(b["w"], b["h"], b["passes"]) for b in blocks], cp.irreversible)
    cells = {("vlc_instance", plan["vlc"]), ("magsgn_instance",) + plan["magsgn"]}
    if plan["vlc"] == "wide" and any(b["w"] <= 64 for b in blocks):
        cells.add(("narrow_under_wide", kind))
    if plan["vlc_tail"] and plan["cta_tail"]:
        cells.add(("launch_tail", kind))
    if plan["refine"]:
        cells.add(("refine_launch", kind))
    return cells


def case_cells(placements=(0,)):
    """(cells the cases reach, blocks whose parse disagreed with the oracle's significance)"""
    reached, bad = set(), []
    for name, _ in GEOMETRIES:
        for kind in KINDS:
            for v in range(3):
                cp, table, data, _ = geometry_case(name, kind, v)
                blocks = table_blocks(cp, table, data)
                reached |= _launch_cells(cp, table, blocks)
                wide = max(b["w"] for b in blocks) > 64
                for k, b in enumerate(blocks):
                    for base in placements:
                        c, ok = block_cells(b, wide, (k + base) % 8)
                        reached |= c
                        if not ok:
                            bad.append((name, kind, v, k))
    for label in constructed():
        b = constructed_block(label)
        for base in placements:
            c, ok = block_cells(b, b["w"] > 64, base)
            reached |= c
            if not ok:
                bad.append((label, base))
    if os.path.exists(GOLD):
        g = np.load(GOLD)
        index = {}
        for b, rc, _ in damaged(g):
            k = index[b["w"], b["h"]] = index.get((b["w"], b["h"]), -1) + 1     # its place in its shape's table
            for base in placements:
                c, _ = block_cells(b, b["w"] > 64, (k + base) % 8)
                reached |= c
            if b["npass"] > 1 and b["len2_table"] == 0:
                reached.add(("pass_rule", "no_refinement_bytes"))
            if b["npass"] > 1 and b["mm"] >= 29 and b["len2_table"]:
                reached.add(("pass_rule", "mmsbs_29"))
        # the code-stream test: damaged streams in batch slots 1 and 3, 4 tiles (chunks past block 0)
        if any(CS_BATCH[1:]) and CS_TILES > 1:
            reached.add(("codestream_batch", "reject_in_slot>=1_first_block>0"))
    return reached, bad


ALL_CELLS = (
    {("vlc_instance", v) for v in ("wide", "narrow")}
    | {("magsgn_instance", i, r) for i in (False, True) for r in (False, True)}
    | {(c, k) for c in ("narrow_under_wide", "launch_tail", "refine_launch") for k in KINDS}
    | {("segments", s) for s in ("1", "2-15", "16", "partial", "seam_rows")}
    | {("seam", s) for s in ("bl_next", "br_left")}
    | {("geometry", s) for s in ("odd_w", "odd_h")}
    | {("rounds", s) for s in ("1", ">1")}
    | {("ring", "wraps", k) for k in KINDS}
    | {("ms", s) for s in ("empty", "ff_last")}
    | {("left", s) for s in ("1-3", "4", "5-7", "8", "refill_end")}
    | {("ff", s) for s in ("byte3", "ballot", "refill_carry")}
    | {("ff_top_bit", s) for s in ("byte3", "ballot", "refill_carry")}
    | {("codestream_batch", "reject_in_slot>=1_first_block>0")}
    | {("vec_ok", v, k) for v in (False, True) for k in KINDS}
    | {("ragged", s) for s in ("column", "row")}
    | {("verdict", s) for s in ("empty", "lcup1", "scup<2", "scup>lcup", "scup>4079")}
    | {("verdict", "uq", s) for s in ("first_pair", "later_pair", "later_round")}
    | {("refine", "passes", n, c) for n in (2, 3) for c in (False, True)}
    | {("refine", "h%4", r) for r in range(4)}
    | {("refine", "nwords", s) for s in ("1", "2-31", "32")}
    | {("refine", s) for s in ("sigprop_exhausted", "sigprop_ff", "magref_stuffed", "rejected_in_phase_b") + KINDS}
    | {("pass_rule", s) for s in ("no_refinement_bytes", "mmsbs_29")}
    | {("vlc", s) for s in ("fast", "bytewise_rotate", "window_below", "straddling_window_read")}
    | {("vlc", "bytewise", s) for s in ("7f", "segment_start")}
    | {("vlc", "straddle", o) for o in range(3)}
    | {("mel", s) for s in ("ff_then_7bit", "forced_nibble", "past_end", "k12")}
    | {("uvlc", "mode", m) for m in (1, 2, 3)}
    | {("uvlc", "mode4", s) for s in ("p0>2", "p0<=2")}
    | {("uvlc", s) for s in ("mel1", "suffix5_both")}
    | {("uvlc", "suffix", n) for n in (0, 1, 5)})


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_model_reproduces_known_plans():
    # 64x64 blocks only: the narrow parse, 32 + 4 + 1 exponent slots rounded down to even, 13 CTAs of phase A for 400 blocks
    p = launch_plan([(64, 64, 1)] * 400, False)
    assert (p["vlc"], p["magsgn"], p["line_entries"], p["vlc_ctas"], p["ctas"], p["refine"]) == \
        ("narrow", (False, False), 36, 13, 100, False)
    # one 65-wide block makes every block of the launch parse under WIDE; 3 blocks leave tails in both grids
    p = launch_plan([(65, 8, 1), (64, 64, 3), (4, 4, 1)], True)
    assert (p["vlc"], p["magsgn"], p["line_entries"], p["vlc_tail"], p["cta_tail"], p["refine"]) == \
        ("wide", (True, True), 38, True, True, True)
    assert launch_plan([(1024, 4, 1)] * 32, False)["line_entries"] == 516
    # the pass rules: no refinement bytes, or 29 missing MSBs, leave the cleanup pass alone; an empty block has Kmax
    assert decode_fields(12, 100, 3, 3, 20) == (9, 3, 20)
    assert decode_fields(12, 100, 3, 3, 0) == (9, 1, 0)
    assert decode_fields(30, 100, 1, 3, 20) == (29, 1, 0)
    assert decode_fields(29, 100, 1, 2, 20) == (28, 2, 20)
    assert decode_fields(12, 0, 3, 3, 20) == (12, 1, 0)


def test_parse_matches_the_oracle_significance():
    """The phase-A restatement gives each quad the rho the oracle's decode says is significant, on every case block,
    and phase B's U_q test rejects exactly the blocks the oracle rejects."""
    _, bad = case_cells()
    assert not bad, bad[:10]


def test_cases_reach_every_cell():
    reached, _ = case_cells(placements=(0, 4))
    assert reached <= ALL_CELLS, sorted(reached - ALL_CELLS, key=str)
    assert reached == ALL_CELLS, "not reached: %s" % sorted(ALL_CELLS - reached, key=str)


def test_oracle_gives_the_reference_verdicts_on_damaged_blocks():
    """Every damaged block: the oracle's verdict and words are the reference's (and, where the reference is built,
    the reference still gives them)."""
    g = np.load(GOLD)
    Rf = O.ref()
    n = 0
    for b, rc, want in damaged(g):
        w, h = b["w"], b["h"]
        got_rc, dec = O.ht_decode_passes(b["data"], b["len2_table"], b["npass"], b["mm"], w, h, causal=b["causal"])
        assert (got_rc == 0) == (rc == 0), (n, b["kind"], got_rc, rc)
        if rc == 0:
            assert np.array_equal(dec, want), (n, b["kind"])
        if Rf is not None:
            r2, d2 = O.ref_ht_decode(b["data"], b["mm"], w, h, num_passes=b["npass"], len2=b["len2_table"],
                                     causal=b["causal"])
            assert (r2 == 0) == (rc == 0) and (rc != 0 or np.array_equal(d2, want)), n
        n += 1
    m = g["meta"]
    assert n == len(m) and 0 < int((m[:, 7] != 0).sum()) < n
    assert set(m[:, 8]) == set(range(13))


def _encoded_table(cp, seed):
    """the block table and arena of a synthetic image of `cp` coded by the oracle encoder, as this project's encoder
    writes it (one bit-plane signalled, cleanup pass only)"""
    planes = P.synthetic_image(cp.x1 - cp.x0, cp.y1 - cp.y0, cp.numcomps, cp.prec, seed=seed, origin=(cp.x0, cp.y0))
    coefs = P.forward(cp, planes)
    rects = P.tile_rects(cp)
    table = G.enumerate_blocks(cp)
    chunks, off = [], 0
    for i, (t, c, b) in enumerate(P.enumerate_all(cp)):
        if b.x1 > b.x0 and b.y1 > b.y0:
            d = P.encode_block(cp, coefs, rects[t], c, b)
            table[i]["length"], table[i]["offset"], table[i]["numbps"], table[i]["numpasses"] = len(d), off, 1, 1
            chunks.append(d)
            off += len(d)
    return table, np.concatenate(chunks)


def _other_suites():
    """(suite, coding, foreign-coding case or None) of suites that reach the decoder's paths by chance"""
    import test_device_io as DI
    import test_dynamic_range as DR
    import test_gpu as TG
    for a in TG.GEOMS[:2]:
        yield "test_gpu", G.make_coding(**a), None
    for a in DR.BLOCK_CASES[:2]:
        yield "test_dynamic_range", DR.coding(a), None
    for i in (0, 1):
        yield "test_device_batch_decode", G.make_coding(**DI._geoms()[i]), None
    for c in HF.FOREIGN_CODINGS[:3]:
        yield "test_ht_foreign", G.make_coding(**c["args"]), c


def test_gap_report_of_the_other_suites(capsys):
    """Which cells the codings of the suites that decode HT blocks reach (printed, not asserted: the cases above are
    what reach every cell).  test_gpu, test_dynamic_range and test_device_batch_decode decode what this project's encoder
    writes: their codings are parsed here as the oracle encoder codes a synthetic image of them."""
    reached = {}
    for suite, cp, case in _other_suites():
        if case is None:
            table, data = _encoded_table(cp, seed=1)
        else:
            args = case["args"]
            if case.get("causal"):
                cp.cblk_sty = 0x08
            planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=11,
                                       origin=args.get("origin", (0, 0)))
            table, data, _ = HF._foreign_blocks(cp, P.forward(cp, planes), case["npass"], case["dropped"], seed=17)
        blocks = table_blocks(cp, table, data)
        r = _launch_cells(cp, table, blocks)
        wide = max(b["w"] for b in blocks) > 64
        for b in blocks[:300]:
            r |= block_cells(b, wide)[0]
        reached.setdefault(suite, set()).update(r)
    with capsys.disabled():
        print()
        for suite, r in reached.items():
            print("%s misses %d of %d cells: %s" % (suite, len(ALL_CELLS - r), len(ALL_CELLS), sorted(ALL_CELLS - r, key=str)))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def placed(table, data, second):
    """the table's bytes laid out again: block k at residue k mod 8 after 0x00 gaps, or (second) at (k + 4) mod 8 after
    0xFF gaps with the last block ending at the arena's end"""
    t = table.copy()
    chunks, off = [], 0
    for k, i in enumerate(i for i in range(len(t)) if t[i]["length"] + t[i]["length2"] > 0):
        n = int(t[i]["length"] + t[i]["length2"])
        pad = ((k + (4 if second else 0)) - off) % 8
        chunks.append(np.full(pad, 0xFF if second else 0x00, np.uint8))
        chunks.append(np.asarray(data[int(table[i]["offset"]):int(table[i]["offset"]) + n], np.uint8))
        t[i]["offset"] = off + pad
        off += pad + n
    return t, (np.concatenate(chunks) if chunks else np.zeros(0, np.uint8))


def _decode_blocks(engine, cp, table, data, shape_planes, expect_rejected=0):
    job = engine.job(cp)
    try:
        job.upload([np.zeros_like(p) for p in shape_planes])
        got = [np.full_like(p, -1) for p in shape_planes]
        job.upload_coeffs(got)
        if expect_rejected:
            with pytest.raises(G.EngineError, match=r"-2: HT decoder rejected %d block\(s\)" % expect_rejected):
                job.t1_decode_blocks(table, data)
        else:
            job.t1_decode_blocks(table, data)
        job.download_coeffs(got)
    finally:
        job.close()
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("variant", range(3))
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", [g[0] for g in GEOMETRIES])
def test_geometry_case_at_both_placements(engine, name, kind, variant):
    cp, table, data, want = geometry_case(name, kind, variant)
    for second in (False, True):
        t, d = placed(table, data, second)
        got = _decode_blocks(engine, cp, t, d, want)
        for c, (g, r) in enumerate(zip(got, want)):
            assert np.array_equal(g, r), "placement %d, component %d: %d coefficients differ" % (
                second, c, int((g != r).sum()))


def _repeat_coding(w, h, mm, reps, tiles=1, irreversible=False):
    """a coding of `reps` blocks of w x h in one band with band Kmax 29 (a block's missing MSBs set by numbps), in
    `tiles` tiles side by side"""
    pw = lambda n: max(4, 1 << (int(n) - 1).bit_length())     # noqa: E731
    rw = reps if w == pw(w) or h != pw(h) else 1
    rh = reps // rw
    assert rw % tiles == 0
    cp = G.make_coding(w * rw, h * rh, 1, 16, numres=1, cblk=(pw(w), pw(h)), irreversible=irreversible,
                       tile=(w * rw // tiles, h * rh) if tiles > 1 else None)
    cp.qcd_explicit = 1
    cp.qcd_expn[0], cp.qcd_mant[0] = 29, 0
    table = G.enumerate_blocks(cp)
    assert len(table) == rw * rh and all((t["x1"] - t["x0"], t["y1"] - t["y0"]) == (w, h) for t in table)
    return cp, table, (h * rh, w * rw)


def _post_rev(words, kmax=29):
    h, w = words.shape
    out = np.zeros((h, w), np.int32)
    O.lib().orc_ht_post_rev(np.ascontiguousarray(words, np.uint32), w, w, h, kmax, out, w)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("label", list(constructed()))
def test_constructed_block_at_both_placements(engine, label):
    """Each constructed block alone, then 16 times in one launch (where it fills its code-block size across)."""
    coef, data, mm = constructed()[label]
    h, w = coef.shape
    rc, dec = O.ht_decode(data, mm, w, h) if len(data) else (0, np.zeros((h, w), np.uint32))
    assert rc == 0
    want_blk = _post_rev(dec)
    pw = lambda n: max(4, 1 << (int(n) - 1).bit_length())     # noqa: E731
    for reps in (1, 16) if pw(w) == w or pw(h) == h else (1,):
        cp, table, shape = _repeat_coding(w, h, mm, reps)
        chunks = []
        for k in range(len(table)):
            table[k]["length"], table[k]["length2"], table[k]["offset"] = len(data), 0, k * len(data)
            table[k]["numbps"], table[k]["numpasses"] = 29 - mm, 1
            chunks.append(data)
        arena = np.concatenate(chunks)
        want = np.tile(want_blk, (shape[0] // h, shape[1] // w))
        for second in (False, True):
            t, d = placed(table, arena, second)
            got = _decode_blocks(engine, cp, t, d, [want])
            assert np.array_equal(got[0], want), (label, reps, second, int((got[0] != want).sum()))


def _post(cp, words):
    """the oracle's dequantisation of a block's words in `cp`'s one band"""
    if not cp.irreversible:
        return _post_rev(words)
    h, w = words.shape
    kmax, _, step = P.band_params(cp, 0, 0)
    out = np.zeros((h, w), np.float32)
    O.lib().orc_ht_post_irrev(np.ascontiguousarray(words, np.uint32), w, w, h, kmax, step, out, w)
    return out.view(np.int32)


def _damaged_tables(g, tiles=1, irreversible=False, codestream=False):
    """per block shape: (shape, coding, table, arena, expected coefficient plane, rejected count, per-block verdicts).
    codestream: a block a code stream cannot carry (its parser refuses a cleanup segment of 1 byte) is left empty"""
    shapes = {}
    for b, rc, want in damaged(g):
        if codestream and b["lcup"] < 2:
            b, rc, want = dict(b, data=np.zeros(0, np.uint8), lcup=0, len2_table=0, npass=0), 0, np.zeros((b["h"], b["w"]), np.uint32)
        shapes.setdefault((b["w"], b["h"]), []).append((b, rc, want))
    for (w, h), items in shapes.items():
        cp, table, shape = _repeat_coding(w, h, 0, len(items), tiles, irreversible)
        assert P.band_params(cp, 0, 0)[0] == 29
        causal = {b["causal"] for b, _, _ in items}
        assert len(causal) == 1          # one coding style per table: the blocks of a shape share it
        if causal.pop():
            cp.cblk_sty = 0x08
        want = np.zeros(shape, np.int32)
        chunks, off = [], 0
        per_row = shape[1] // w
        for k, (b, rc, words) in enumerate(items):
            t = table[k]
            t["length"], t["length2"], t["offset"] = b["lcup"], b["len2_table"], off
            t["numbps"], t["numpasses"] = 29 - b["mm"], b["npass"]
            chunks.append(b["data"])
            off += len(b["data"])
            y0, x0 = (k // per_row) * h, (k % per_row) * w
            assert (t["x0"], t["y0"]) == (x0, y0)
            if rc == 0:
                want[y0:y0 + h, x0:x0 + w] = _post(cp, words)
        yield (w, h), cp, table, np.concatenate(chunks), want, sum(rc != 0 for _, rc, _ in items), \
            [rc for _, rc, _ in items]


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
def test_damaged_blocks_get_the_reference_verdicts(engine, kind):
    """One table per block shape: the blocks the reference accepts decode to its words (dequantised by the oracle), the
    ones it rejects to zeros, and the call reports as many rejected blocks as the reference rejects."""
    g = np.load(GOLD)
    for shape, cp, table, data, want, nrej, _ in _damaged_tables(g, irreversible=kind == "irrev"):
        for second in (False, True):
            t, d = placed(table, data, second)
            got = _decode_blocks(engine, cp, t, d, [want], expect_rejected=nrej)
            assert np.array_equal(got[0], want), (shape, second, int((got[0] != want).sum()))


CS_TILES = 4
CS_BATCH = (False, True, False, True)       # damaged stream per batch slot


@pytest.mark.gpu
def test_damaged_code_streams_carry_their_own_rejection_counts(engine):
    """Each shape's damaged table written as a 4-tile code stream, and a clean stream of the same coding (the blocks the
    reference rejects left out).  engine.decode gives the inverse of the expected coefficients and reports the
    reference's rejection count; decode_codestreams_device over clean, damaged, clean, damaged gives each stream its
    own (rc, text), and the clean streams' pixels."""
    torch = pytest.importorskip("torch")
    g = np.load(GOLD)
    for shape, cp, table, data, want, nrej, verdicts in _damaged_tables(g, tiles=CS_TILES, codestream=True):
        clean = table.copy()
        for k, rc in enumerate(verdicts):
            if rc != 0:
                clean[k]["length"] = clean[k]["length2"] = clean[k]["numpasses"] = clean[k]["numbps"] = 0
        ref = P.inverse(cp, [want])[0]
        for t, n in ((clean, 0), (table, nrej)):
            out = [np.full(want.shape, -7, np.int32)]
            if n:
                with pytest.raises(G.EngineError, match=r"-2: HT decoder rejected %d block\(s\)" % n):
                    engine.decode(cp, t, data, out)
            else:
                engine.decode(cp, t, data, out)
            assert np.array_equal(out[0], ref), (shape, n, int((out[0] != ref).sum()))
        streams = {False: G.codestream_write(cp, clean, data), True: G.codestream_write(cp, table, data)}
        dcs = [torch.from_numpy(np.array(streams[bad], np.uint8)).cuda() for bad in CS_BATCH]
        _, imgs, status = engine.decode_codestreams_device(dcs, dtype=torch.int32)
        torch.cuda.synchronize()
        assert status == [(-2, "HT decoder rejected %d block(s)" % nrej) if bad else (0, "") for bad in CS_BATCH], \
            (shape, status)
        imgs = imgs.cpu().numpy()
        for i, bad in enumerate(CS_BATCH):
            if not bad:
                assert np.array_equal(imgs[i, 0], ref), (shape, i)
