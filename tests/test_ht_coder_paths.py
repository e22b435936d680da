"""Every staging and launch path of the HT block encoder (ht_enc.cu), and its MagSgn and VLC drains at their longest
fix-up chains, bit for bit against the oracle.

A launch of k_ht_encode picks one of four instances (IRREV x PACK: PACK when every block's Kmax is at most 24), a warp
count per CTA (fewer for a launch of fewer than 132 x that many blocks, fewer when wide blocks need more shared memory
per warp) and a grid of at most one CTA per SM, so that a warp of a large launch codes several blocks.  Each block is
staged with 8-byte or 4-byte loads (its address, the plane pitch and an even width decide), R quad rows per round (32
units fill the warp), in one or two code trips per round (two for blocks wider than 512), with a partial last round
and odd rows or columns at the block's edge.  `launch_plan` and `block_staging` restate those rules from the block
table; the CPU tests pin them to hand-computed plans and check that the cases below reach every cell.

The MagSgn bytes leave the per-warp ring 128 at a time (ms_drain128, 4 bytes per lane) while 1024 raw bits are queued,
and 32 at a time at the end (ms_drain32<true>).  A byte after 0xFF carries 7 bits, so where a lane's window starts
depends on the stuffing in every lane below it: the drains speculate and fix that up on ballots, at most 34 times.
`ms_drains` restates both loops and counts their iterations.  `chain_block` builds a block whose raw MagSgn bits make
every lane's stuffing visible only after the lane below it is fixed: each 128-byte drain needs 33 iterations, each
final drain more than 30.  A drain loop cut below that leaves a lane's bytes unresolved, which the GPU tests see.

The VLC stream is drained the same way (vlc_drain128 while 1024 bits are queued, vlc_drain32 while 256 are, after each
1024-bit gather of a code trip): a byte after one above 0x8F whose low 7 bits are ones is 0x7F and carries 7 bits.
`raw_streams` restates T.814's VLC bits and `vlc_trips` the bits each code trip joins, both in Python, so that
`vlc_drains` knows where every drain falls; it reproduces the oracle's VLC bytes.  `vlc_first_row_block` builds first
quad rows whose VLC bits are all ones, so each lane's stuffing is known only after the lane below: 33 iterations in
vlc_drain128, 32 in vlc_drain32.

The end of a block: `Mel` restates the MEL coder, `vlc_serial` the VLC stream bit by bit and `terminate` the
reference's terminate_mel_vlc, driven by the MEL events `raw_streams` computes; `block_model` predicts the segment
lengths, Scup, the MEL bytes and how the block ends, and reproduces the oracle on ordinary content.  The termination
cells are the outcome (nothing pending, one fused byte, or two bytes because the bits conflict, because the fused byte
would be 0xFF or because no VLC byte was written yet), and for each outcome but the first the MEL bits left (rem 1..8,
and 7 after a 0xFF MEL byte: a byte that carries 7 bits and none of them yet), the VLC bits left (0..7) and whether
the last VLC byte was above 0x8F; then whether a MEL run is pending and how the MagSgn stream ends.  The reachable
set TERM_REACHABLE is what terminate gives from every state the two streams can be in (`terminate_states`, less the
states the context-0 codewords rule out); TERM_UNREACHABLE_WHY gives the reason for each other cell and a test checks
it.  TERM_SEEDS keeps `small_block`s (found by a search over 200,000 of them: 4..16 x 2..16, exponents 1..4, all-zero
blocks included) that reach all of TERM_REACHABLE.

The MEL segment cannot overflow: `mel_bound` runs the MEL coder as a finite machine over every event sequence, and a
block has at most one event per quad (1024).  `mel_longest_block` builds, per block shape, the block with the longest
segment (192 bytes for 4 x 1024: the limit, met and not passed).  `slot_block` builds the largest blocks for their
scratch slot (every MagSgn bit a one; the longest U-VLC codewords) at Kmax 24 and 29; they fit slot_capacity.

k_scan_lengths and k_ht_gather: `gather_cells` computes from a block's segment lengths and its destination offset the
residue of its first whole word, the short path, the tail bytes, where the MagSgn|MEL / VLC seam falls, the funnel
shift of each source piece and whether a lane takes a second pass; `scan_cells` the scan's round edges and base.
They are counted in three placements: the arena from 0 (the constructed blocks, alone and 16 in one launch), the arena
after an earlier range (the length sweeps through the pipelined round trip) and the code stream (the same sweeps through
the device writer, offsets from tests/oracle_t2.py).

GPU: per case, every block's bytes equal the oracle's, the block offsets are the exclusive scan of the oracle's
lengths, the device decode of the coded bytes equals the oracle's decode (and the source on the reversible path), and
the same bytes decode again through a caller's block table that puts each block at every residue mod 4.
tests/golden/ht_stuffing.npz pins the oracle's bytes and decodes of the constructed blocks to the reference
(tests/golden/make_golden_stuffing.py).
"""
import functools
import os

import numpy as np
import pytest

import grok_b200 as G
import oracle_lib as O
import oracle_pipeline as P

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ht_stuffing.npz")

# ---------------------------------------------------------------------------------------------------------------------
# the launch and staging model (b2k_launch_ht_encode, k_ht_encode, engine.cu alloc_planes / build_block_plan)
# ---------------------------------------------------------------------------------------------------------------------
SMS = 132                   # H100 SXM
ENC_WARPS = 20
UNIT_QUADS = 8
TABLE_BYTES = 2 * 2048 * 2 + 64 * 2
SMEM_MAX = 227 * 1024
FIXED_WARP_WORDS = 32 * 5 + 128 + 64 + 256 // 4 + 2 * 34     # VLC strings, both rings, MEL buffer, unit offsets
R_VALUES = (32, 16, 10, 8, 6, 5, 4, 3, 2, 1)                  # 32 // units per quad row, for 1..32+ units


def _cdiv(a, b):
    return -(-a // b)


def units_per_row(w):
    return _cdiv((w + 1) >> 1, UNIT_QUADS)


def rows_per_round(w):
    upr = units_per_row(w)
    return 1 if upr >= 32 else 32 // upr


def stage_words(w):
    c = w + 6
    pitch = (c + (c >> 5)) | 1
    return _cdiv(2 * rows_per_round(w) + 1, 6) * 6 * pitch


def launch_plan(blocks, irreversible):
    """blocks: [(w, h, kmax)] of one launch.  Returns its instance, warps per CTA (and what the shared memory alone
    would allow), grid and how many blocks the busiest warp codes."""
    n = len(blocks)
    kmax = max(k for _, _, k in blocks)
    ms_w = min(32, kmax + 2) | 1
    warp_words = max(stage_words(w) for w, _, _ in blocks) + 32 * ms_w + FIXED_WARP_WORDS
    cta_max = max(1, min(ENC_WARPS, (SMEM_MAX - TABLE_BYTES) // (4 * warp_words)))
    cta = cta_max if n >= SMS * cta_max else max(1, _cdiv(n, SMS))
    smem = TABLE_BYTES + 4 * cta * warp_words
    want = _cdiv(n, cta)
    if want > SMS:
        # a launch larger than one CTA per SM: the model takes the occupancy query's answer to be one, which holds
        # while a CTA needs more than half of an SM's shared memory
        assert 2 * (smem + 1024) > 228 * 1024, (smem, cta)
    grid = min(want, SMS)
    return dict(irrev=bool(irreversible), pack=kmax <= 24, cta=cta, cta_max=cta_max, grid=grid,
                per_warp=_cdiv(n, grid * cta), widths=len({stage_words(w) for w, _, _ in blocks}))


def plane_column(cp, rect, b):
    """column of the block's first sample in the engine's coefficient plane: planes start at canvas column
    x0 & ~31, their pitch is a multiple of 32 samples, and the allocation is aligned"""
    return rect[0] + b.buf_x - (cp.x0 & ~31)


def block_staging(w, h, col):
    R = rows_per_round(w)
    return dict(vec=(col % 2 == 0 and w % 2 == 0), R=R, trips=_cdiv(R * units_per_row(w), 32),
                partial=h % (2 * R) != 0 and h > 2 * R, odd_h=h % 2 == 1, odd_w=w % 2 == 1)


def coded_blocks(cp):
    """[(i, tile, comp, block, w, h, kmax, column)] of the blocks the engine codes, in its order"""
    rects = P.tile_rects(cp)
    out = []
    for i, (t, c, b) in enumerate(P.enumerate_all(cp)):
        w, h = b.x1 - b.x0, b.y1 - b.y0
        if w and h:
            out.append((i, t, c, b, w, h, P.band_params(cp, b.resno, b.orient)[0], plane_column(cp, rects[t], b)))
    return out


def cells(cp):
    """the cells one coding's launch reaches"""
    kind = "irrev" if cp.irreversible else "rev"
    blks = coded_blocks(cp)
    plan = launch_plan([(w, h, k) for *_, w, h, k, _ in blks], cp.irreversible)
    out = {("instance", plan["irrev"], plan["pack"])}
    if plan["cta"] < plan["cta_max"]:
        out.add(("launch", kind, "small"))
    elif plan["cta_max"] < ENC_WARPS:
        out.add(("launch", kind, "wide"))
    else:
        out.add(("launch", kind, "full"))
    if plan["per_warp"] > 1:
        out.add(("launch", kind, "persistent"))
    if plan["widths"] > 1:
        out.add(("mixed_widths", kind, plan["pack"]))
    for *_, w, h, _, col in blks:
        s = block_staging(w, h, col)
        out.add(("stage", kind, "vector" if s["vec"] else "scalar"))
        out.add(("R", kind, s["R"]))
        out.add(("trips", kind, s["trips"]))
        for k in ("partial", "odd_h", "odd_w"):
            if s[k]:
                out.add((k, kind))
    return out


KINDS = ("rev", "irrev")
ALL_CELLS = ({("instance", i, p) for i in (False, True) for p in (False, True)}
             | {("launch", k, s) for k in KINDS for s in ("small", "full", "wide", "persistent")}
             | {("mixed_widths", k, p) for k in KINDS for p in (False, True)}
             | {("stage", k, s) for k in KINDS for s in ("vector", "scalar")}
             | {("R", k, r) for k in KINDS for r in R_VALUES}
             | {("trips", k, t) for k in KINDS for t in (1, 2)}
             | {(c, k) for k in KINDS for c in ("partial", "odd_h", "odd_w")})

# ---------------------------------------------------------------------------------------------------------------------
# the geometry cases: each runs reversible (5/3) and irreversible (9/7)
# ---------------------------------------------------------------------------------------------------------------------
CASES = {
    # 64x64 blocks at an odd origin, two resolutions: R = 32, 16 and 8 at the band edges, odd rows and columns,
    # 4-byte staging for odd widths; a small launch
    "edges": dict(width=301, height=157, numcomps=1, prec=12, numres=3, origin=(3, 5)),
    # 256x16 blocks in 328-column tiles: band edges cut blocks 8 to 256 wide, R = 32, 16, 10, 8, 6, 5, 4, 3 and 2
    "tiles": dict(width=3418, height=37, numcomps=1, prec=10, numres=1, cblk=(256, 16), tile=(328, 37)),
    # 1024x4 blocks: two code trips per round, fewer warps per CTA for shared memory, a warp codes several blocks;
    # widths 1024 and 22 share the launch
    "1024x4": dict(width=2048 + 1046, height=1200, numcomps=1, prec=8, numres=1, cblk=(1024, 4)),
    # more than 132 x 20 64x64 blocks: full CTAs, persistent warps; Kmax 24 and 25 in one launch (unpacked)
    "full": dict(width=4160, height=2624, numcomps=1, prec=12, numres=2, kmax=(24, 25, 25, 25)),
    # the same grid of blocks with Kmax at most 24: packed, with two widths
    "full-packed": dict(width=4160, height=2624, numcomps=1, prec=12, numres=2, kmax=(23, 24, 24, 24)),
}
ORDER = list(CASES)


def coding(name, kind):
    args = dict(CASES[name])
    kmax = args.pop("kmax", None)
    cp = G.make_coding(irreversible=kind == "irrev", **args)
    if kmax:        # explicit band exponents: Kmax = exponent + guard bits - 1, one guard bit
        cp.qcd_explicit = 1
        for i, k in enumerate(kmax):
            cp.qcd_expn[i], cp.qcd_mant[i] = k, 0
    return cp


# ---------------------------------------------------------------------------------------------------------------------
# the MagSgn drain model (ms_drain128, ms_drain32<true>)
# ---------------------------------------------------------------------------------------------------------------------
DRAIN128_BOUND = 34
DRAIN32_BOUND = 34


class _Bits:
    """raw MagSgn bits (LSB first); bits at or beyond `tail` read as ones (the final drain's fill)"""

    def __init__(self, bits):
        b = np.concatenate([np.asarray(bits, np.uint8), np.ones(2048, np.uint8)])
        self.bytes = np.packbits(b, bitorder="little")

    def get(self, start, nbits):
        """nbits (<= 32) bits from each position of the integer array `start`"""
        start = np.asarray(start, np.int64)
        v = np.zeros(start.shape, np.uint64)
        for k in range(5):
            v |= self.bytes[(start >> 3) + k].astype(np.uint64) << np.uint64(8 * k)
        v >>= (start & 7).astype(np.uint64)
        return (v & np.uint64((1 << nbits) - 1)).astype(np.int64)


_LANE = np.arange(32)


def _popc_below(mask):
    """per lane: set bits of mask in lanes below it"""
    bits = (mask >> _LANE) & 1
    return np.concatenate([[0], np.cumsum(bits)[:-1]])


def _drain128(bits, head, last_ff):
    m1 = m2 = lf = 0
    for it in range(DRAIN128_BOUND):
        start = head + 32 * _LANE - _popc_below(m1) - _popc_below(m2)
        raw = bits.get(start, 32)
        f = np.where(_LANE == 0, int(last_ff), (lf >> np.maximum(_LANE - 1, 0)) & 1).astype(bool)
        sev = np.zeros(32, np.int64)
        word = np.zeros(32, np.int64)
        for j in range(4):
            b = np.where(f, raw & 0x7F, raw & 0xFF)
            raw = np.where(f, raw >> 7, raw >> 8)
            sev += f
            f = b == 0xFF
            word |= b << (8 * j)
        n1, n2, nf = (int(np.sum((c.astype(np.int64)) << _LANE)) for c in (sev >= 1, sev >= 2, f))
        if (n1, n2, nf) == (m1, m2, lf):
            out = word.astype("<u4").view(np.uint8)
            return it + 1, out, head + 1024 - bin(m1).count("1") - bin(m2).count("1"), bool((lf >> 31) & 1)
        m1, m2, lf = n1, n2, nf
    return None, None, None, None


def _drain32_final(bits, head, tail, last_ff):
    ffmask = 0
    for it in range(DRAIN32_BOUND):
        prevff = ((ffmask << 1) | int(last_ff)) & 0xFFFFFFFF
        seven = ((prevff >> _LANE) & 1).astype(bool)
        start = head + 8 * _LANE - _popc_below(prevff)
        byte = np.where(seven, bits.get(start, 8) & 0x7F, bits.get(start, 8))
        nf = int(np.sum((byte == 0xFF).astype(np.int64) << _LANE))
        if nf == ffmask:
            complete = start < tail
            nb = 32 if complete.all() else int(np.argmin(complete))
            if nb == 0:
                return it + 1, np.zeros(0, np.uint8), head, last_ff
            end = int(start[nb - 1]) + (7 if seven[nb - 1] else 8)
            return it + 1, byte[:nb].astype(np.uint8), end, bool(byte[nb - 1] == 0xFF)
        ffmask = nf
    return None, None, None, None


def ms_drains(raw):
    """The MagSgn drains of a block whose raw MagSgn bits are `raw`: (iterations of each 128-byte drain, of each final
    drain, the MagSgn bytes).  An iteration count of None is a drain the loop bound leaves unresolved."""
    bits = _Bits(raw)
    tail, head, last_ff = len(raw), 0, False
    it128, it32, out = [], [], []
    while tail - head >= 1024:
        it, o, head, last_ff = _drain128(bits, head, last_ff)
        it128.append(it)
        if it is None:
            return it128, it32, None
        out.append(o)
    while head < tail:
        it, o, head, last_ff = _drain32_final(bits, head, tail, last_ff)
        it32.append(it)
        if it is None:
            return it128, it32, None
        out.append(o)
    data = np.concatenate(out) if out else np.zeros(0, np.uint8)
    dropped = bool(len(data) and last_ff)
    if dropped:
        data = data[:-1]          # a final 0xFF is not written
    return it128, it32, data, dropped


# ---------------------------------------------------------------------------------------------------------------------
# the VLC drain model (vlc_drain128, vlc_drain32 and the join loop that calls them)
# ---------------------------------------------------------------------------------------------------------------------
VLC128_BOUND = 40
VLC32_BOUND = 34


def _masked(bits, start, n, tail):
    """n bits from each start; bits at or beyond tail read as zeros (ring_get15's fill for VLC)"""
    v = bits.get(start, n)
    avail = np.clip(tail - np.asarray(start, np.int64), 0, n)
    return v & ((1 << avail) - 1)


def _vlc_drain128(bits, head, prev):
    m1 = m2 = 0
    word = last = np.zeros(32, np.int64)
    for it in range(VLC128_BOUND):
        start = head + 32 * _LANE - _popc_below(m1) - _popc_below(m2)
        raw = bits.get(start, 32)
        pb = np.concatenate([[prev], last[:-1]])
        st = np.zeros(32, np.int64)
        nword = np.zeros(32, np.int64)
        for j in range(4):
            stuffed = (pb > 0x8F) & ((raw & 0x7F) == 0x7F)
            b = np.where(stuffed, 0x7F, raw & 0xFF)
            raw = np.where(stuffed, raw >> 7, raw >> 8)
            st += stuffed
            pb = b
            nword |= b << (8 * j)
        n1, n2 = (int(np.sum(c.astype(np.int64) << _LANE)) for c in (st >= 1, st >= 2))
        same = np.array_equal(nword, word) and (n1, n2) == (m1, m2)
        word, last, m1, m2 = nword, pb, n1, n2
        if same and it > 0:
            return it + 1, word.astype("<u4").view(np.uint8), head + 1024 - bin(m1).count("1") - bin(m2).count("1"), \
                int(last[31])
    return None, None, None, None


def _vlc_drain32(bits, head, tail, prev):
    smask = 0
    byte = np.zeros(32, np.int64)
    for it in range(VLC32_BOUND):
        start = head + 8 * _LANE - _popc_below(smask)
        raw = _masked(bits, start, 15, tail)
        pb = np.concatenate([[prev], byte[:-1]])
        stuffed = (pb > 0x8F) & ((raw & 0x7F) == 0x7F)
        nbyte = np.where(stuffed, 0x7F, raw & 0xFF)
        ns = int(np.sum(stuffed.astype(np.int64) << _LANE))
        same = np.array_equal(nbyte, byte) and ns == smask
        byte, smask = nbyte, ns
        if same and it > 0:
            nbits = np.where(stuffed, 7, 8)
            complete = start + nbits <= tail
            nb = 32 if complete.all() else int(np.argmin(complete))
            if nb == 0:
                return it + 1, np.zeros(0, np.uint8), head, prev
            return it + 1, byte[:nb].astype(np.uint8), int(start[nb - 1] + nbits[nb - 1]), int(byte[nb - 1])
    return None, None, None, None


def vlc_drains(vlc, trips):
    """The VLC drains of a block whose raw VLC bits are `vlc` and whose code trips join `trips` bits each: (iterations
    of each 128-byte drain, of each 32-byte drain, VLC bytes 1.. in stream order, the bits left for the last byte).
    The stream starts with four one bits after the virtual byte 0xFF; each trip's bits are gathered 1024 at a time and
    drained 128 bytes while 1024 bits are queued, then 32 while 256 are."""
    bits = _Bits(np.concatenate([np.ones(4, np.uint8), vlc]))
    head, tail, prev = 0, 4, 0xFF
    it128, it32, out = [], [], []
    for tb in trips:
        t0 = tail
        tail += tb
        wb = t0 >> 5
        while (wb << 5) < tail:
            have = min(tail, (wb + 32) << 5)
            while have - head >= 1024:
                it, o, head, prev = _vlc_drain128(bits, head, prev)
                it128.append(it)
                if it is None:
                    return it128, it32, None, None
                out.append(o)
            while have - head >= 256:
                it, o, head, prev = _vlc_drain32(bits, head, have, prev)
                it32.append(it)
                if it is None:
                    return it128, it32, None, None
                out.append(o)
            wb += 32
    while True:
        it, o, head, prev = _vlc_drain32(bits, head, tail, prev)
        it32.append(it)
        if it is None:
            return it128, it32, None, None
        out.append(o)
        if len(o) < 32:
            break
    return it128, it32, np.concatenate(out), tail - head


# ---------------------------------------------------------------------------------------------------------------------
# constructed content: raw MagSgn bits with the longest fix-up chains
# ---------------------------------------------------------------------------------------------------------------------
def _group_bits(first):
    """one lane's 4 bytes in the chain pattern: 0x54 (8 bits, only lane 0 of the first drain) or 0x2A (7 bits, after
    the 0xFF of the lane below), 0x54, 0x2A, 0xFF.  The bits next to each 0xFF are zeros and no other eight ones meet,
    so a window one bit off reads no 0xFF: each lane sees its stuffing only once the lane below is fixed."""
    out = []
    for v, n in ((0x54, 8) if first else (0x2A, 7), (0x54, 8), (0x2A, 8), (0xFF, 8)):
        out += [(v >> i) & 1 for i in range(n)]
    return out


def chain_raw(total):
    """`total` raw MagSgn bits: the chain pattern for every 128-byte drain, then ones (a final drain of ones stuffs
    every other byte, 0xFF then 0x7F, and each of those is seen only after the byte below it)"""
    raw, first = [], True
    head = 0
    while total - head >= 1024:
        for _ in range(32):
            raw += _group_bits(first)
            first = False
        head = len(raw)
    return np.array(raw + [1] * (total - len(raw)), np.uint8)


def _quad_order(w, h):
    """(y, x) of every sample in coding order: quad rows, quads, then (x,y) (x,y+1) (x+1,y) (x+1,y+1)"""
    order = []
    for y in range(0, h, 2):
        for x in range(0, w, 2):
            for dx, dy in ((0, 0), (0, 1), (1, 0), (1, 1)):
                order.append((y + dy, x + dx))
    return order


def chain_block(w, h, e):
    """(coefficients (h, w) int32, intended raw MagSgn bits) of a block whose samples all have exponent e (|c| in
    (2^(e-2), 2^(e-1)]).  Every quad is significant with U_q = e; a quad codes each sample's low m bits of
    2(|c| - 1) + sign, m = e - 1 where the CxtVLC row marks the sample in EMB (top bit implied), e otherwise (top bit
    1).  Interior quads are coded with e_k = 1111; the first quad of each row (context 0 or 5) with e_k = 1001, so
    two samples per quad row carry a forced one -- inside a byte of the pattern, where it changes no stuffing."""
    assert w % 2 == 0 and h % 2 == 0 and w >= 4
    emb_first = 0b1001
    fields = []
    for y, x in _quad_order(w, h):
        i = 2 * (x & 1) + (y & 1)
        full = x >= 2 or (emb_first >> i) & 1
        fields.append((y, x, e - 1 if full else e))
    total = sum(m for *_, m in fields)
    raw = chain_raw(total)
    coef = np.zeros((h, w), np.int64)
    pos = 0
    for y, x, m in fields:
        t = 0
        for k in range(e - 1):
            t |= int(raw[pos + k]) << k if k < m else 0
        if m == e:
            raw[pos + e - 1] = 1        # the forced top bit
        v = (1 << (e - 1)) + t          # 2(mu - 1) + sign
        mu, s = (v >> 1) + 1, v & 1
        coef[y, x] = -mu if s else mu
        pos += m
    return coef.astype(np.int32), raw


# the constructed blocks: (label, w, h, exponent, Kmax)
CHAIN_BLOCKS = [("chain-64x64-packed", 64, 64, 20, 20), ("chain-64x64-unpacked", 64, 64, 26, 27),
                ("chain-1024x4", 1024, 4, 16, 18), ("chain-4x1024", 4, 1024, 12, 12),
                ("chain-32x8-final", 32, 8, 9, 10)]




def vlc_first_row_block(w, shifts=()):
    """(2, w) coefficients whose one quad row writes nothing but one bits to the VLC stream: the first quad (context
    0) has only its sample (x, y+1) significant, then quads alternate between samples (x, y), (x+1, y) (context 1)
    and (x, y), (x, y+1) (context 3), one of exponent 2 and one of exponent 1 each, so u_q = 1 everywhere.  Those
    rows' CxtVLC codewords are 1111111 and the UVLC prefix of u = 1 is 1.  All-ones VLC bits stuff every other byte
    (0xFF, then 0x7F carrying 7 bits), and each byte learns whether it is stuffed only from the byte below it.
    The quads in `shifts` (odd) get exponent 3 instead of 2 (u = 2, prefix 01): each puts one zero into the stream,
    and two of them move the stuffed bytes from even to odd positions of a 4-byte word."""
    c = np.zeros((2, w), np.int32)
    for q in range(w // 2):
        x = 2 * q
        if q == 0:
            c[1, x] = 2
        elif q % 2:
            c[0, x], c[0, x + 1] = 3 if q in shifts else 2, -1
        else:
            c[0, x], c[1, x] = -1, 2
    return c


# VLC-heavy blocks: (label, w, Kmax); 1024 wide: two code trips per round, 128- and 32-byte drains
VLC_BLOCKS = [("vlc-first-row-1024x2", 1024, 4), ("vlc-first-row-1024x2-shifted", 1024, 4), ("vlc-first-row-300x2", 300, 4)]
VLC_SHIFTS = {"vlc-first-row-1024x2-shifted": (129, 301)}
# the termination blocks: small_block(seed) for the seeds that, between them, reach every reachable termination cell
# (a greedy cover of the first blocks the search found per cell; seed 9 is all zeros; SEAM_SEED puts the gather's seam
# among the head bytes)
TERM_SEEDS = (3, 5, 6, 7, 8, 9, 11, 13, 15, 16, 20, 23, 30, 49, 57, 66, 113, 115, 122, 129, 156, 172, 270, 329, 1063, 1157,
              2911, 3002, 4623, 5253, 17112, 18078, 25014, 28780, 55448, 56259, 58057, 66647, 81246, 152477)
TERM_OUTCOMES = ("none", "fused", "conflict", "ff", "novlc", "ff+novlc")
_REMS = tuple(range(1, 9)) + ("7 after 0xFF",)
TERM_CELLS = ({("outcome", o) for o in TERM_OUTCOMES} | {("mel_run", r) for r in ("pending", "none")}
              | {("ms_end", e) for e in ("empty", "dropped", "other")}
              | {(o, "rem", r) for o in TERM_OUTCOMES[1:] for r in _REMS}
              | {(o, "vlc_bits", u) for o in TERM_OUTCOMES[1:] for u in range(8)}
              | {(o, "last_vlc>0x8F", g) for o in TERM_OUTCOMES[1:] for g in (False, True)})
# Why the other cells cannot occur; test_termination_cells_left_out_are_unreachable checks both reasons.  rem counts the
# MEL bits still free in the last byte, so pending MEL bits occupy its top 8 - rem bits (none at rem 8, or at 7 after a
# 0xFF byte, whose top bit is a forced 0) and pending VLC bits its low `used` bits.
_NO_STATE = ("terminate_mel_vlc gives this from no state the two streams can be in (terminate_states): bits conflict only "
             "where both sides have bits (used > rem); a fused 0xFF needs every bit set by one side; before the first "
             "VLC byte vlc_init's four bits are pending and the byte before is its virtual 0xFF")
_FIRST_CODEWORD = ("needs 1 or 2 VLC bits before the first VLC byte: the first significant quad of a block is in context "
                   "0, whose CxtVLC codewords have 3 bits or more, so 4 or 7 bits are pending until a byte is written")
TERM_UNREACHABLE_WHY = dict(
    [(c, _NO_STATE) for c in [("conflict", "rem", r) for r in (7, 8, "7 after 0xFF")]
     + [("conflict", "vlc_bits", u) for u in (0, 1)] + [("ff", "rem", r) for r in (8, "7 after 0xFF")]
     + [("ff", "vlc_bits", 0), ("novlc", "last_vlc>0x8F", False), ("ff+novlc", "last_vlc>0x8F", False)]
     + [("novlc", "vlc_bits", u) for u in range(4)] + [("ff+novlc", "vlc_bits", u) for u in (0, 1, 2, 3, 7)]
     + [("ff+novlc", "rem", r) for r in (7, 8, "7 after 0xFF")]]
    + [(c, _FIRST_CODEWORD) for c in [("novlc", "vlc_bits", 5), ("novlc", "vlc_bits", 6), ("ff+novlc", "vlc_bits", 5),
                                      ("ff+novlc", "vlc_bits", 6), ("ff+novlc", "rem", 5), ("ff+novlc", "rem", 6)]])
TERM_REACHABLE = TERM_CELLS - set(TERM_UNREACHABLE_WHY)
# the longest MEL segment of each block shape
MEL_SHAPES = ((64, 64), (1024, 4), (4, 1024))
# the largest blocks for their scratch slot: (kind, Kmax) per shape; "ones" codes every sample's MagSgn bits as ones,
# "vlc" adds the longest VLC codewords
SLOT_KINDS = (("ones", 24), ("ones", 29), ("vlc", 29))
CONSTRUCTED = [c[0] for c in CHAIN_BLOCKS] + [c[0] for c in VLC_BLOCKS] + ["term-%d" % s for s in TERM_SEEDS] + \
    ["mel-longest-%dx%d" % s for s in MEL_SHAPES] + \
    ["slot-%s-k%d-%dx%d" % (k, km, w, h) for w, h in MEL_SHAPES for k, km in SLOT_KINDS]


@functools.lru_cache(maxsize=None)
def chain_case(label):
    """(coefficients, raw MagSgn bits, Kmax) of a constructed block"""
    if label.startswith("term-"):
        coef = small_block(int(label[5:]))
        return coef, raw_streams(coef, TERM_KMAX)[0], TERM_KMAX
    if label.startswith("mel-longest-"):
        coef = mel_longest_block(*(int(v) for v in label[12:].split("x")))[0]
        return coef, raw_streams(coef, TERM_KMAX)[0], TERM_KMAX
    if label.startswith("slot-"):
        _, kind, km, shape = label.split("-")
        coef = slot_block(*(int(v) for v in shape.split("x")), int(km[1:]), kind)
        return coef, raw_streams(coef, int(km[1:]))[0], int(km[1:])
    for lab, w, kmax in VLC_BLOCKS:
        if lab == label:
            coef = vlc_first_row_block(w, VLC_SHIFTS.get(label, ()))
            return coef, raw_streams(coef, kmax)[0], kmax
    _, w, h, e, kmax = next(c for c in CHAIN_BLOCKS if c[0] == label)
    coef, raw = chain_block(w, h, e)
    return coef, raw, kmax


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the models and the case lists
# ---------------------------------------------------------------------------------------------------------------------
def test_cases_reach_every_cell():
    reached = set()
    for name in CASES:
        for kind in KINDS:
            reached |= cells(coding(name, kind))
    assert reached <= ALL_CELLS, sorted(reached - ALL_CELLS, key=str)
    assert reached == ALL_CELLS, "not reached: %s" % sorted(ALL_CELLS - reached, key=str)


def test_model_reproduces_known_plans():
    # config 2 (8192x8192x3, 1024x1024 tiles, 64x64 blocks): 20 warps per CTA, 132 CTAs, a warp codes up to 19 of the 49728 blocks,
    # 18 staged rows of pitch 73 per warp (R = 8), 8-byte loads
    cp2 = G.make_coding(8192, 8192, 3, 12, numres=6, tile=(1024, 1024))
    blks = coded_blocks(cp2)
    plan = launch_plan([(w, h, k) for *_, w, h, k, _ in blks], False)
    assert (plan["cta"], plan["cta_max"], plan["grid"], plan["pack"]) == (20, 20, 132, True)
    assert plan["per_warp"] == _cdiv(len(blks), 132 * 20) == 19
    assert stage_words(64) == 18 * 73
    assert all(block_staging(w, h, col)["vec"] for *_, w, h, _, col in blks)
    # 1024x4 blocks: R = 1 in two code trips, 7 warps per CTA (shared memory), Kmax 10 packed
    p = launch_plan([(1024, 4, 10)] * 2000, False)
    assert (p["cta"], p["cta_max"], p["grid"], p["per_warp"]) == (7, 7, 132, 3)
    assert block_staging(1024, 4, 0) == dict(vec=True, R=1, trips=2, partial=False, odd_h=False, odd_w=False)
    # fewer than 132 x 20 blocks: ceil(n / 132) warps per CTA, one block per warp
    p = launch_plan([(64, 64, 12)] * 1000, True)
    assert (p["cta"], p["grid"], p["per_warp"], p["irrev"]) == (8, 125, 1, True)
    # R for each count of units per quad row; a block at an odd plane column stages with 4-byte loads
    assert [rows_per_round(w) for w in (16, 32, 48, 64, 80, 96, 128, 160, 256, 512)] == list(R_VALUES)
    assert not block_staging(64, 64, 3)["vec"] and not block_staging(63, 64, 0)["vec"]


def test_magsgn_drain_model_reproduces_the_oracle():
    """The drain model, fed the raw MagSgn bits of ordinary content, writes the oracle's MagSgn bytes."""
    rng = np.random.default_rng(1)
    for w, h, kmax in ((64, 64, 12), (33, 17, 20), (1024, 4, 9), (4, 1024, 27)):
        e = rng.integers(2, kmax, (h, w))
        coef = np.where(rng.random((h, w)) < 0.7, rng.integers(0, 1 << 30, (h, w)) % (1 << (e - 1)) + 1, 0)
        coef = coef * rng.choice([-1, 1], (h, w))
        data = O.ht_encode(O.to_sgnmag(coef, kmax), kmax, cap=65536)
        raw = _oracle_magsgn_bits(coef, kmax)
        _, _, ms, _ = ms_drains(raw)
        assert np.array_equal(data[:len(ms)], ms), (w, h, kmax)


def _uvlc(u):
    """UVLC prefix and suffix of u as (bits, length) pairs (uvlc_tbl)"""
    if u == 0:
        return (0, 0), (0, 0)
    if u <= 2:
        return (1 if u == 1 else 2, u), (0, 0)
    if u <= 4:
        return (4, 3), (u - 3, 1)
    return (0, 3), (u - 5, 5)


def raw_streams(coef, kmax):
    """The raw (unstuffed) MagSgn and VLC bits of a block, straight from T.814's rules (ht_encode_core's ms_put and
    vlc_put calls), the VLC bits of each unit (UNIT_QUADS quads of a quad row) as [quad row][unit], and the MEL events in
    coding order: a quad in context 0 codes whether it is significant, and a first-row quad pair whose u_q are both
    non-zero whether both exceed 2 (quad 2p, quad 2p+1, then the pair)."""
    L = O.lib()
    T = [np.ctypeslib.as_array(L.orc_ht_enc_table(t), (2048,)) for t in (0, 1)]
    c = np.asarray(coef, np.int64)
    h, w = c.shape
    mu = np.abs(c)
    e = np.where(mu > 0, np.floor(np.log2(np.maximum(2 * mu - 1, 1))).astype(np.int64) + 1, 0)
    pad = np.zeros((h + 2, w + 4), np.int64)
    pad[:h, :w] = e
    bits, vlc, unit_bits, events = [], [], [], []
    put = lambda v, n: vlc.extend((v >> k) & 1 for k in range(n))      # noqa: E731
    eab = np.zeros(w + 4, np.int64)
    nq = (w + 1) // 2
    for y in range(0, h, 2):
        enew = np.zeros(w + 4, np.int64)
        rho_left = 0
        row_units = []
        for q0 in range(0, nq, 2):
            if q0 % UNIT_QUADS == 0:
                row_units.append(len(vlc))
            u = [0, 0]
            for j, x in enumerate(range(2 * q0, min(2 * q0 + 4, 2 * nq), 2)):
                smp = [(x, y), (x, y + 1), (x + 1, y), (x + 1, y + 1)]
                es = [int(pad[yy, xx]) if xx < w and yy < h else 0 for xx, yy in smp]
                rho = sum(1 << i for i in range(4) if es[i])
                emax = max(es)
                if y == 0:
                    cq, kappa = (rho_left >> 1) | (rho_left & 1), 1
                else:
                    E = eab[x:x + 4]          # columns x-1 .. x+2
                    cq = (1 if E[0] | E[1] else 0) | (2 if rho_left & 0xC else 0) | (4 if E[2] | E[3] else 0)
                    kappa = max(1, int(E.max()) - 1) if rho & (rho - 1) else 1
                U = max(emax, kappa)
                u[j] = U - kappa
                eps = sum(1 << i for i in range(4) if es[i] == U) if u[j] > 0 else 0
                tup = int(T[1 if y else 0][(cq << 8) + (rho << 4) + eps])
                put(tup >> 8, (tup >> 4) & 7)
                for i, (xx, yy) in enumerate(smp):
                    if es[i]:
                        m = U - ((tup >> i) & 1)
                        v = 2 * (int(mu[yy, xx]) - 1) + (1 if c[yy, xx] < 0 else 0)
                        bits += [(v >> k) & 1 for k in range(m)]
                enew[x + 1] = es[1]
                enew[x + 2] = es[3]
                rho_left = rho
                if cq == 0:
                    events.append(1 if rho else 0)
            if y == 0 and u[0] > 0 and u[1] > 0:
                events.append(1 if min(u) > 2 else 0)
            if y == 0 and u[0] > 2 and u[1] > 2:
                (p0, s0), (p1, s1) = _uvlc(u[0] - 2), _uvlc(u[1] - 2)
                for v in (p0, p1, s0, s1):
                    put(*v)
            elif y == 0 and u[0] > 2 and u[1] > 0:
                p0, s0 = _uvlc(u[0])
                put(*p0)
                put(u[1] - 1, 1)
                put(*s0)
            else:
                (p0, s0), (p1, s1) = _uvlc(u[0]), _uvlc(u[1])
                for v in (p0, p1, s0, s1):
                    put(*v)
        row_units.append(len(vlc))
        unit_bits.append(list(np.diff(row_units)))
        eab = enew
    return np.array(bits, np.uint8), np.array(vlc, np.uint8), unit_bits, events


def _oracle_magsgn_bits(coef, kmax):
    return raw_streams(coef, kmax)[0]


def vlc_trips(w, unit_bits):
    """the VLC bits each code trip of k_ht_encode joins: R quad rows per round, 32 units per trip"""
    upr, R = units_per_row(w), rows_per_round(w)
    trips = []
    for r0 in range(0, len(unit_bits), R):
        units = [b for row in unit_bits[r0:r0 + R] for b in row]
        trips += [sum(units[k:k + 32]) for k in range(0, R * upr, 32)]
    return trips


# ---------------------------------------------------------------------------------------------------------------------
# the MEL coder and the end of a block (mel_emit / mel_zeros / mel_one and terminate_mel_vlc of k_ht_encode)
# ---------------------------------------------------------------------------------------------------------------------
MEL_EXP = (0, 0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 4, 5)
MEL_LIMIT = 192         # the reference's MEL buffer: a longer segment is its "mel encoder's buffer is full"


class Mel:
    """mel_struct, mel_emit_bit and mel_encode of the reference (L273-347): the MEL bytes of a list of events"""

    def __init__(self, events=()):
        self.buf, self.rem, self.tmp, self.run, self.k, self.width = [], 8, 0, 0, 0, 8
        for e in events:
            self.encode(e)

    def bit(self, v):
        self.tmp = (self.tmp << 1) + v
        self.rem -= 1
        if self.rem == 0:
            self.buf.append(self.tmp)
            self.rem = self.width = 7 if self.tmp == 0xFF else 8
            self.tmp = 0

    def encode(self, e):
        if not e:
            self.run += 1
            if self.run >= 1 << MEL_EXP[self.k]:
                self.bit(1)
                self.run, self.k = 0, min(12, self.k + 1)
        else:
            self.bit(0)
            for t in range(MEL_EXP[self.k] - 1, -1, -1):
                self.bit((self.run >> t) & 1)
            self.run, self.k = 0, max(0, self.k - 1)


def vlc_serial(vlc):
    """vlc_encode bit by bit after vlc_init's virtual 0xFF and four one bits: (VLC bytes 1.. in stream order, the
    bits left for the last byte, their value)"""
    out, used, tmp, gt8f = [], 4, 0xF, True
    for b in vlc:
        tmp |= int(b) << used
        used += 1
        if used + gt8f == 8:
            if gt8f and tmp != 0x7F:
                gt8f = False            # a byte after one above 0x8F carries 7 bits only when they are 0x7F
                continue
            out.append(tmp)
            gt8f, tmp, used = tmp > 0x8F, 0, 0
    return out, used, tmp


def terminate(mel, vlc_bytes, used, vtmp):
    """terminate_mel_vlc on the MEL coder `mel` and the VLC stream's state: (outcome, the MEL state it saw as (rem,
    whether the last MEL byte was 0xFF), whether a MEL run was pending).  Appends the last MEL byte (fused or not)
    to mel.buf; returns the VLC byte it appends (None: none).  Outcomes: "none" (nothing pending on either side),
    "fused" (one byte carries both), and the three reasons for two bytes: "conflict" (a bit of one side's pending
    bits differs from the other's fill), "ff" (the fused byte would be 0xFF) and "novlc" (no VLC byte written yet).
    A block that meets both of the last two is "ff+novlc"."""
    pending = mel.run > 0
    if pending:
        mel.bit(1)
    state = (mel.rem, mel.width == mel.rem == 7)
    mtmp = mel.tmp << mel.rem
    mel_mask = (0xFF << mel.rem) & 0xFF
    vlc_mask = 0xFF >> (8 - used) if used else 0
    if not (mel_mask | vlc_mask):
        return "none", state, pending, None
    fuse = mtmp | vtmp
    conflict = ((fuse ^ mtmp) & mel_mask) | ((fuse ^ vtmp) & vlc_mask)
    wrote = len(vlc_bytes) > 0
    if not conflict and fuse != 0xFF and wrote:
        mel.buf.append(fuse)
        return "fused", state, pending, None
    outcome = "conflict" if conflict else ("ff" if wrote else "ff+novlc") if fuse == 0xFF else "novlc"
    mel.buf.append(mtmp)
    return outcome, state, pending, vtmp


def end_cells(outcome, rem, after_ff, used, last_gt8f):
    """the cells of an outcome other than "none": the MEL bits left, the VLC bits left, the last VLC byte"""
    if outcome == "none":
        return set()
    return {(outcome, "rem", "7 after 0xFF" if after_ff else rem), (outcome, "vlc_bits", used),
            (outcome, "last_vlc>0x8F", last_gt8f)}


def terminate_states():
    """Every state terminate_mel_vlc can start from, as far as the two streams' own rules go: MEL rem 1..8 (1..7 in
    the byte after a 0xFF) with any pending bits; VLC with `used` bits pending and the last byte above 0x8F or not --
    but before the first VLC byte, vlc_init's four one bits plus fewer than four more (the virtual 0xFF before them),
    and after a byte above 0x8F, never 0x7F in seven bits (that byte is complete).  Yields (Mel, wrote, used, vtmp,
    last byte above 0x8F)."""
    for width in (8, 7):
        for rem in range(1, width + 1):
            for tmp in range(1 << (width - rem)):
                for wrote in (False, True):
                    for used in range(8) if wrote else range(4, 8):
                        for vtmp in range(1 << used) if wrote else (0xF | x << 4 for x in range(1 << (used - 4))):
                            for gt in (False, True) if wrote else (True,):
                                if gt and used == 7 and vtmp == 0x7F:
                                    continue
                                mel = Mel()
                                mel.width, mel.rem, mel.tmp = width, rem, tmp
                                yield mel, wrote, used, vtmp, gt


def block_model(coef, kmax):
    """The coded block as the models predict it: its segments' lengths, Scup, the MEL and VLC bytes, how the block
    ends and the termination cells it reaches."""
    ms, vlc, _, events = raw_streams(coef, kmax)
    _, _, ms_bytes, dropped = ms_drains(ms)
    mel = Mel(events)
    vb, used, vtmp = vlc_serial(vlc)
    last_vlc = vb[-1] if vb else 0xFF           # the virtual byte before the first
    outcome, (rem, after_ff), pending, vlast = terminate(mel, vb, used, vtmp)
    if vlast is not None:
        vb = vb + [vlast]
    vlc_len = 1 + len(vb)                       # + the Scup byte
    ms_end = "empty" if len(ms_bytes) == 0 else "dropped" if dropped else "other"
    cells = {("outcome", outcome), ("mel_run", "pending" if pending else "none"), ("ms_end", ms_end)}
    cells |= end_cells(outcome, rem, after_ff, used, last_vlc > 0x8F)
    return dict(ms_len=len(ms_bytes), mel_len=len(mel.buf), vlc_len=vlc_len, scup=len(mel.buf) + vlc_len,
                mel=np.array(mel.buf, np.uint8), vlc=np.array(vb, np.uint8), outcome=outcome, cells=cells,
                events=len(events))


TERM_KMAX = 5


def small_block(seed):
    """the search's block `seed`: 4, 8 or 16 wide (a whole code block's width, so that one launch can repeat it), 2 to 16
    high, a density of significant samples and exponents 1..4 drawn per block"""
    rng = np.random.default_rng(seed)
    w, h = 4 << int(rng.integers(0, 3)), int(rng.integers(2, 17))
    e = rng.integers(1, 5, (h, w))
    lo = np.where(e > 1, (1 << np.maximum(e - 2, 0)) + 1, 1)
    mag = lo + rng.integers(0, 1 << 20, (h, w)) % ((1 << (e - 1)) - lo + 1)
    on = rng.random((h, w)) < rng.choice([0.03, 0.1, 0.3, 0.6, 1.0])
    return (mag * on * rng.choice([-1, 1], (h, w))).astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------------
# the longest MEL segment: an exact search over the MEL coder's states
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def _mel_machine():
    """The MEL coder as a finite machine: its states (k, run, byte width, bits pending, their value), per event value
    the next state and the bytes it completes, and per state the bytes the end of the block adds: the pending run's
    bit, then terminate_mel_vlc's MEL-side byte (the fused byte or the MEL bits), which it writes whenever either
    stream has bits pending.  Any block may end with VLC bits pending, so `most` counts that byte always; `least`
    only where MEL bits are pending (or the byte after a 0xFF has none yet)."""
    states = [(k, run, wd, n, t) for k in range(13) for run in range(1 << MEL_EXP[k]) for wd in (8, 7)
              for n in range(wd) for t in range(1 << n)]
    index = {s: i for i, s in enumerate(states)}

    def emit(st, v):
        k, run, wd, n, t, pos = st
        t, n = (t << 1) | v, n + 1
        return (k, run, 7 if t == 0xFF else 8, 0, 0, pos + 1) if n == wd else (k, run, wd, n, t, pos)

    nxt, add, most, least = np.zeros((2, len(states)), np.int64), np.zeros((2, len(states)), np.int64), [], []
    for i, s in enumerate(states):
        k, run = s[:2]
        for e in (0, 1):
            st = s + (0,)
            if not e and run + 1 < 1 << MEL_EXP[k]:
                st = (k, run + 1) + st[2:]
            elif not e:
                st = (min(12, k + 1), 0) + emit(st, 1)[2:]
            else:
                st = emit(st, 0)
                for t in range(MEL_EXP[k] - 1, -1, -1):
                    st = emit(st, (run >> t) & 1)
                st = (max(0, k - 1), 0) + st[2:]
            nxt[e, i], add[e, i] = index[st[:5]], st[5]
        st = emit(s + (0,), 1) if run else s + (0,)
        most.append(st[5] + 1)
        least.append(st[5] + (1 if st[3] or st[2] == 7 else 0))
    return nxt, add, np.array(most), np.array(least), index[(0, 0, 8, 0, 0)]


def mel_bound(n):
    """the most MEL bytes any n events (or fewer) code to, termination included"""
    nxt, add, V, _, start = _mel_machine()
    best = V[start]
    for _ in range(n):
        V = np.maximum(add[0] + V[nxt[0]], add[1] + V[nxt[1]])
        best = max(best, V[start])
    return int(best)


# the first quad row, pair by pair: the quads' significance (and, for two significant quads with u_q > 0, whether both
# u_q exceed 2), the events the pair codes after a significant (True) or insignificant left neighbour, and whether its
# second quad is significant
_FIRST_ROW = {"00": (lambda p: ([] if p else [0]) + [0], False), "0S": (lambda p: ([] if p else [0]) + [1], True),
              "S0": (lambda p: [] if p else [1], False), "SS": (lambda p: [] if p else [1], True),
              "SS-u1": (lambda p: ([] if p else [1]) + [0], True), "SS-u3": (lambda p: ([] if p else [1]) + [1], True)}
_FIRST_ROW_COEF = {"00": (0, 0), "0S": (0, 1), "S0": (1, 0), "SS": (1, 1), "SS-u1": (2, 2), "SS-u3": (8, 8)}


@functools.lru_cache(maxsize=None)
def mel_longest_block(w, h):
    """(coefficients, the least MEL bytes it can code to) of the w x h block (w, h even) with the longest MEL segment
    the first-row and free events allow, counting the end of the block without VLC bits pending.  Below the first quad row
    a quad whose only significant sample is its top-left one leaves every neighbour's context at 0, so each of those
    quads is a free event; the first row's events depend on the left neighbour and pair events need u_q > 0 on both
    quads.  A backward pass over the MEL machine's states finds the best events, pair choices included."""
    nxt, add, _, V, start = _mel_machine()
    free = (h // 2 - 1) * (w // 2)
    Vs = [V]
    for _ in range(free):
        Vs.append(np.maximum(add[0] + Vs[-1][nxt[0]], add[1] + Vs[-1][nxt[1]]))
    Vs.reverse()

    def take(evs, V):
        for e in reversed(evs):
            V = add[e] + V[nxt[e]]
        return V

    rows, Vrow = [], {False: Vs[0], True: Vs[0]}
    for _ in range(w // 4):
        cand = {p: {o: take(f(p), Vrow[sig]) for o, (f, sig) in _FIRST_ROW.items()} for p in (False, True)}
        rows.append(cand)
        Vrow = {p: np.max(np.stack(list(cand[p].values())), axis=0) for p in (False, True)}
    coef = np.zeros((h, w), np.int32)
    s, prev = start, False
    for q, cand in enumerate(reversed(rows)):
        o = max(cand[prev], key=lambda o: cand[prev][o][s])
        for e in _FIRST_ROW[o][0](prev):
            s = nxt[e, s]
        prev = _FIRST_ROW[o][1]
        coef[0, 4 * q], coef[0, 4 * q + 2] = _FIRST_ROW_COEF[o]
    for i in range(free):
        e = int(add[1, s] + Vs[i + 1][nxt[1, s]] > add[0, s] + Vs[i + 1][nxt[0, s]])
        s = nxt[e, s]
        y, x = 2 + 2 * (i // (w // 2)), 2 * (i % (w // 2))
        coef[y, x] = e
    return coef, int(Vrow[False][start])


# ---------------------------------------------------------------------------------------------------------------------
# the scratch slot (engine.cu slot_capacity) and the largest blocks for it
# ---------------------------------------------------------------------------------------------------------------------
def slot_capacity(w, h, kmax):
    samples, quads = w * h, ((w + 1) // 2) * ((h + 1) // 2)
    ms = (samples * (kmax + 2) + 6) // 7 + 16
    vlc = (quads * 15 + 6) // 7 + 16
    return (ms + vlc + 256 + 15) & ~15


def slot_block(w, h, kmax, kind):
    """"ones": every sample -2^(kmax-1), whose MagSgn bits are all ones (a byte after 0xFF carries 7 bits, so every
    other byte is stuffed).  "vlc": the same on the top row of each quad and -1 below it: the row below sees exponent
    1 above, so kappa = 1 and u_q = kmax - 1 in every quad (the longest U-VLC codewords), while every sample still
    codes U_q MagSgn bits."""
    c = np.full((h, w), -(1 << (kmax - 1)), np.int64)
    if kind == "vlc":
        c[1::2] = -1
    return c.astype(np.int32)


# ---------------------------------------------------------------------------------------------------------------------
# the length scan (k_scan_lengths) and the compaction (k_ht_gather)
# ---------------------------------------------------------------------------------------------------------------------
SCAN_ROUND = 1024 * 8           # 1024 threads x SCAN_ITEMS blocks per round
PLACEMENTS = ("arena", "arena after a range", "code stream")
GATHER_CELLS = ({("head", r) for r in range(4)} | {("tail", r) for r in range(4)} | {("short",), ("words > 128",)}
                | {("seam", s) for s in ("head bytes", "word boundary", 1, 2, 3, "tail bytes")}
                | {("shift", p, r) for p in ("front", "vlc") for r in range(4)})
ALL_GATHER_CELLS = {(p,) + c for p in PLACEMENTS for c in GATHER_CELLS}
SCAN_CELLS = {"n = 1", "n < 32", "n = 8192", "n = 8192k + 1", "3+ rounds, partial last", "non-zero base"}


def gather_cells(fronts, totals, dst):
    """The cells k_ht_gather reaches for blocks whose MagSgn|MEL bytes number `fronts`, whose lengths are `totals` and
    whose bytes go to byte offsets `dst` of a word-aligned buffer.  The slots are 16-aligned, so source byte j of the
    front piece is at residue j mod 4 and of the VLC piece (at the slot's end) at residue (j - total) mod 4."""
    out = set()
    for front, total, d in zip(fronts, totals, dst):
        if not total:
            continue
        head = -int(d) & 3
        out.add(("head", head))
        if total < head + 4:
            out.add(("short",))
            continue
        words = (total - head) >> 2
        tail0 = head + 4 * words
        out.add(("tail", total - tail0))
        if words > 128:
            out.add(("words > 128",))
        out.add(("seam", "head bytes" if front < head else "tail bytes" if front >= tail0 else
                  (front - head) % 4 or "word boundary"))
        if head + 4 <= front:
            out.add(("shift", "front", head))
        if tail0 - 4 >= front:
            out.add(("shift", "vlc", (head - total) % 4))
    return out


def scan_cells(n, base):
    out = set()
    if n == 1:
        out.add("n = 1")
    if n < 32:
        out.add("n < 32")
    if n == SCAN_ROUND:
        out.add("n = 8192")
    if n > SCAN_ROUND and n % SCAN_ROUND == 1:
        out.add("n = 8192k + 1")
    if -(-n // SCAN_ROUND) >= 3 and n % SCAN_ROUND:
        out.add("3+ rounds, partial last")
    if base:
        out.add("non-zero base")
    return out


# the length sweeps: point-transform codings (coefficient = pixel - 16, Kmax 5), run whole through the pipelined round
# trip in 128-block ranges and through the device code-stream writer.  "sweep": 400 32x32 blocks, each the search's
# small_block(k) in its corner or, every tenth, dense noise (more than 128 words).  "seam": 160 8x4 blocks, each
# small_block(SEAM_SEED), whose 2 MagSgn|MEL bytes and 7 bytes in all put the seam among the head bytes of the copies
# that start at residue 1 of a word (consecutive copies step through the residues)
SEAM_SEED = 172
SWEEPS = {"sweep": dict(width=640, height=640, numcomps=1, prec=5, numres=1, cblk=(32, 32), numgbits=1),
          "seam": dict(width=320, height=16, numcomps=1, prec=5, numres=1, cblk=(8, 4), numgbits=1)}
SWEEP_SHAPE = (64, 8)           # (chunks, streams) of b2k_job_roundtrip_pipelined_n: 128-block ranges
SWEEP_FLAGS = (0, G.CS_TLM | G.CS_PLT, G.CS_SOP | G.CS_EPH)
# exactly one and one more than one round of the length scan
SCAN_CODINGS = {"8192": dict(width=256, height=512, numcomps=1, prec=8, numres=1, cblk=(4, 4)),
                "8193": dict(width=10924, height=12, numcomps=1, prec=8, numres=1, cblk=(4, 4))}


def coding_of(a):
    return G.make_coding(**a)


def _sweep_grid(name):
    a = SWEEPS[name]
    (bw, bh), nx = a["cblk"], a["width"] // a["cblk"][0]
    return bw, bh, [(bh * (k // nx), bw * (k % nx)) for k in range(nx * (a["height"] // bh))]


@functools.lru_cache(maxsize=None)
def sweep_coefs(name):
    rng = np.random.default_rng(5)
    a = SWEEPS[name]
    bw, bh, at = _sweep_grid(name)
    c = np.zeros((a["height"], a["width"]), np.int32)
    for k, (y, x) in enumerate(at):
        if name == "sweep" and k % 10 == 9:
            c[y:y + bh, x:x + bw] = rng.integers(-15, 16, (bh, bw))
        else:
            b = small_block(SEAM_SEED if name == "seam" else k)
            c[y:y + b.shape[0], x:x + b.shape[1]] = b
    return c


def sweep_planes(name):
    return [sweep_coefs(name) + 16]


@functools.lru_cache(maxsize=None)
def sweep_lengths(name):
    """(MagSgn|MEL bytes, total bytes) of a sweep's blocks in coded order"""
    c = sweep_coefs(name)
    bw, bh, at = _sweep_grid(name)
    fronts, totals = [], []
    for y, x in at:
        m = block_model(c[y:y + bh, x:x + bw], TERM_KMAX)
        fronts.append(m["ms_len"] + m["mel_len"])
        totals.append(fronts[-1] + m["vlc_len"])
    return np.array(fronts), np.array(totals)


def sweep_ranges(name):
    import test_device_roundtrip as RT
    return RT.ranges(len(_sweep_grid(name)[2]), *SWEEP_SHAPE)[0]


@functools.lru_cache(maxsize=None)
def sweep_encoded(name):
    from test_codestream import oracle_encode
    cp = coding_of(SWEEPS[name])
    table, data, _ = oracle_encode(cp, sweep_planes(name))
    return cp, table, data


def sweep_places(name, flags):
    """where each of a sweep's blocks starts in the code stream written with `flags`"""
    import oracle_t2 as T2
    cp, table, data = sweep_encoded(name)
    places = {}
    T2.write_codestream(cp, table, data, tlm=bool(flags & G.CS_TLM), plt=bool(flags & G.CS_PLT),
                        sop=bool(flags & G.CS_SOP), eph=bool(flags & G.CS_EPH), places=places)
    return np.array([places[i] for i in range(len(table))])


def _repeats(coef):
    """how many copies of a constructed block test_constructed_stuffing_matches_oracle codes in one launch"""
    h, w = coef.shape
    return 16 if w >= 4 and w & (w - 1) == 0 else 0


@pytest.mark.parametrize("label", [c[0] for c in CHAIN_BLOCKS])
def test_constructed_magsgn_reaches_the_longest_chains(label):
    """The constructed blocks carry the intended raw MagSgn bits (the oracle's bytes, un-stuffed, are them), and
    their drains need 33 iterations per 128-byte drain (all but a few) and more than 30 in a final drain."""
    coef, raw, kmax = chain_case(label)
    assert np.array_equal(_oracle_magsgn_bits(coef, kmax), raw), label
    data = O.ht_encode(O.to_sgnmag(coef, kmax), kmax, cap=65536)
    it128, it32, ms, dropped = ms_drains(raw)
    assert ms is not None and np.array_equal(data[:len(ms)], ms), label
    assert None not in it128 and None not in it32
    if len(it128):
        assert max(it128) == 33 and sum(i >= 32 for i in it128) >= 0.9 * len(it128), (label, it128)
    assert max(it32) >= 31, (label, it32)
    # the bytes: 0xFF at the end of every lane's word in the 128-byte drains, and a stream that ends in 0xFF (dropped)
    if len(it128):
        words = ms[:128 * len(it128)].reshape(-1, 4)
        assert (words[:, 3] == 0xFF).mean() > 0.95
    # a final 0xFF of the MagSgn stream is left out: pinned for the blocks whose stream ends in one
    assert dropped == (label in ("chain-4x1024", "chain-32x8-final")), label


def _vlc_check(coef, kmax):
    """the VLC drain model on a block: (its 128- and 32-byte drain iterations, its VLC bytes), after checking the
    bytes against the oracle's (stored backwards from the end of the block; byte 1 shares its low nibble with Scup)"""
    w = coef.shape[1]
    _, vlc, unit_bits, _ = raw_streams(coef, kmax)
    it128, it32, vb, _ = vlc_drains(vlc, vlc_trips(w, unit_bits))
    assert vb is not None and None not in it128 + it32
    data = O.ht_encode(O.to_sgnmag(coef, kmax), kmax, cap=65536)
    got = data[::-1][1:1 + len(vb)]
    assert np.array_equal(got[1:], vb[1:]) and (got[0] & 0xF0) == (vb[0] & 0xF0)
    return it128, it32, vb


def test_vlc_drain_model_reproduces_the_oracle():
    """The VLC model, fed the raw VLC bits and code-trip totals of ordinary content (both computed in Python from
    T.814's rules, not taken from the encoder), writes the oracle's VLC bytes."""
    rng = np.random.default_rng(2)
    for w, h, kmax in ((64, 64, 12), (33, 17, 20), (1024, 4, 9), (4, 1024, 27), (600, 6, 5)):
        e = rng.integers(2, kmax, (h, w))
        coef = np.where(rng.random((h, w)) < 0.7, rng.integers(0, 1 << 30, (h, w)) % (1 << (e - 1)) + 1, 0)
        _vlc_check(coef * rng.choice([-1, 1], (h, w)), kmax)


def test_constructed_vlc_reaches_the_longest_chains():
    """The all-ones first-row blocks' VLC drains need 33 of vlc_drain128's 40 iterations and 32 of vlc_drain32's 34
    (one byte per iteration over the 32 lanes, plus the pass that finds nothing moved).  With two zeros in the stream,
    stuffed 0x7F bytes sit at all four byte positions of the 128-byte drains' words, and the chains are still longer
    than 16 in the first three 128-byte drains."""
    it128, it32, _ = _vlc_check(*chain_case("vlc-first-row-1024x2")[::2])
    assert it128 == [33] * 4 and max(it32) == 32, (it128, it32)
    it128, it32, _ = _vlc_check(*chain_case("vlc-first-row-300x2")[::2])
    assert it128 == [33] and max(it32) == 32, (it128, it32)
    it128, it32, vb = _vlc_check(*chain_case("vlc-first-row-1024x2-shifted")[::2])
    assert it128 == [33, 32, 18, 2] and max(it32) == 33, (it128, it32)
    words = vb[:128 * len(it128)].reshape(-1, 4)
    assert all((words[:, k] == 0x7F).any() for k in range(4))


def test_mel_and_termination_model_reproduces_the_oracle():
    """The MEL coder and terminate_mel_vlc, fed the MEL events and VLC bits of ordinary content (computed in Python
    from T.814's rules), predict the oracle's segment lengths, Scup, MEL bytes and last VLC byte."""
    rng = np.random.default_rng(3)
    for w, h, kmax in ((64, 64, 12), (33, 17, 20), (1024, 4, 9), (4, 1024, 27), (600, 6, 5), (5, 3, 4), (2, 2, 3)):
        for density in (0.7, 0.05, 0.002):
            e = rng.integers(2, kmax, (h, w))
            coef = np.where(rng.random((h, w)) < density, rng.integers(0, 1 << 30, (h, w)) % (1 << (e - 1)) + 1, 0)
            coef = coef * rng.choice([-1, 1], (h, w))
            if coef.any():
                _model_check(coef, kmax)


def _model_check(coef, kmax):
    data = O.ht_encode(O.to_sgnmag(coef, kmax), kmax, cap=65536)
    m = block_model(coef, kmax)
    assert m["ms_len"] + m["mel_len"] + m["vlc_len"] == len(data), (m["ms_len"], m["mel_len"], m["vlc_len"], len(data))
    assert (int(data[-1]) << 4) | (int(data[-2]) & 0xF) == m["scup"]
    assert np.array_equal(data[m["ms_len"]:m["ms_len"] + m["mel_len"]], m["mel"])
    vlc = data[::-1][1:m["vlc_len"]]
    assert np.array_equal(vlc[1:], m["vlc"][1:]) and (vlc[0] & 0xF0) == (m["vlc"][0] & 0xF0)
    return m, data


def test_constructed_blocks_reach_every_termination_cell():
    """Each termination block codes as the model predicts, and together they reach every reachable cell."""
    reached = set()
    for s in TERM_SEEDS:
        m, _ = _model_check(small_block(s), TERM_KMAX)
        reached |= m["cells"]
    assert reached <= TERM_CELLS, sorted(reached - TERM_CELLS, key=str)
    assert reached == TERM_REACHABLE, "not reached: %s" % sorted(TERM_REACHABLE - reached, key=str)


def test_termination_cells_left_out_are_unreachable():
    """Every cell TERM_UNREACHABLE_WHY leaves out is shown unreachable, for the reason it gives, and every other cell of
    the ending is reachable from some state of the streams (so the constructed blocks must reach it).  The first
    reason: terminate_mel_vlc, run from every state terminate_states yields, never gives the cell.  The second: every
    context-0 CxtVLC codeword of both tables (first quad row and the rest) has 3 bits or more, so no state with 5 or 6
    bits pending before the first VLC byte occurs; terminate gives those cells only from such states.  A bounded re-run
    of the search then finds nothing outside TERM_REACHABLE."""
    L = O.lib()
    idx = np.arange(2048)
    for t in (0, 1):
        table = np.ctypeslib.as_array(L.orc_ht_enc_table(t), (2048,)).astype(np.int64)
        ctx0 = (idx >> 8 == 0) & ((idx >> 4) & 15 != 0) & ((idx & 15) & ~((idx >> 4) & 15) == 0)
        assert ((table[ctx0] >> 4) & 7).min() == 3, t
    by_state, by_codeword = set(), set()
    for mel, wrote, used, vtmp, gt8f in terminate_states():
        outcome, (rem, after_ff), _, _ = terminate(mel, [0] if wrote else [], used, vtmp)
        got = {("outcome", outcome)} | end_cells(outcome, rem, after_ff, used, gt8f)
        (by_state if wrote or used not in (5, 6) else by_codeword).update(got)
    rest = {c for c in TERM_CELLS if c[0] in ("mel_run", "ms_end")}
    for cell, why in TERM_UNREACHABLE_WHY.items():
        assert cell not in by_state, cell
        assert (cell in by_codeword) == (why == _FIRST_CODEWORD), cell
    assert by_state | rest == TERM_REACHABLE, sorted((by_state | rest) ^ TERM_REACHABLE, key=str)
    for seed in range(1500):
        assert block_model(small_block(seed), TERM_KMAX)["cells"] <= TERM_REACHABLE, seed


def test_mel_segment_never_overflows():
    """No block can write more than the reference's 192 MEL bytes: a block has at most one MEL event per quad (a quad
    in context 0; in the first row, a quad pair whose first quad is significant leaves its second out of context 0, so
    a pair event never adds to two quad events) and at most 1024 quads, and no 1024 events code to more than 192 bytes
    even when every block is taken to end with VLC bits pending (one more MEL-side byte).  The longest segments built
    for the three block shapes are 191, 161 and 192 bytes: the 4 x 1024 block meets the limit and the overflow verdict
    (mel.pos > 192) cannot be reached."""
    assert mel_bound(1024) == MEL_LIMIT
    want = {(64, 64): 191, (1024, 4): 161, (4, 1024): 192}
    for w, h in MEL_SHAPES:
        coef, least = mel_longest_block(w, h)
        m, _ = _model_check(coef, TERM_KMAX)
        assert m["events"] <= (w // 2) * (h // 2)
        assert least <= m["mel_len"] == want[(w, h)] <= MEL_LIMIT, (w, h, m["mel_len"], least)


def test_largest_blocks_fit_their_slot():
    """The encoder writes a block into its scratch slot before it compares the total with slot_cap, so the slot must
    hold the longest block.  The largest blocks of each shape fit with room to spare."""
    for w, h in MEL_SHAPES:
        for kind, kmax in SLOT_KINDS:
            coef = slot_block(w, h, kmax, kind)
            m, data = _model_check(coef, kmax)
            assert len(data) <= slot_capacity(w, h, kmax), (w, h, kind, kmax, len(data), slot_capacity(w, h, kmax))
            assert len(data) > 0.75 * (slot_capacity(w, h, kmax) - 256 - 32), (w, h, kind, kmax)


def test_case_lists_reach_every_scan_and_gather_cell():
    reached = set()
    for label in CONSTRUCTED:
        coef, _, kmax = chain_case(label)
        m = block_model(coef, kmax)
        total = m["ms_len"] + m["mel_len"] + m["vlc_len"]
        front = m["ms_len"] + m["mel_len"]
        reps = _repeats(coef)
        for n in (1, reps):
            if n:
                reached |= {("arena",) + c for c in gather_cells([front] * n, [total] * n, total * np.arange(n))}
    scans = []
    for name in SWEEPS:
        fronts, totals = sweep_lengths(name)
        assert np.array_equal(totals, sweep_encoded(name)[1]["length"])     # the model's lengths are the oracle's
        dst = np.concatenate([[0], np.cumsum(totals)[:-1]])
        rngs = sweep_ranges(name)
        scans += [(b1 - b0, b0) for b0, b1 in rngs]
        for b0, b1 in rngs[1:]:
            reached |= {("arena after a range",) + c for c in gather_cells(fronts[b0:b1], totals[b0:b1], dst[b0:b1])}
        for flags in SWEEP_FLAGS:
            reached |= {("code stream",) + c for c in gather_cells(fronts, totals, sweep_places(name, flags))}
    assert reached == ALL_GATHER_CELLS, "not reached: %s" % sorted(ALL_GATHER_CELLS - reached, key=str)
    import test_device_roundtrip as RT
    scans += [(1, 0), (16, 0)] + [(len(coded_blocks(coding_of(a))), 0) for a in SCAN_CODINGS.values()]
    scans += [(len(RT.coded_blocks(RT.coding(RT.CASES["4x4-blocks"]))), 0)]     # test_device_roundtrip runs it
    got = set().union(*(scan_cells(n, base) for n, base in scans))
    assert got == SCAN_CELLS, "not reached: %s" % sorted(SCAN_CELLS - got)
    assert [len(coded_blocks(coding_of(a))) for a in SCAN_CODINGS.values()] == [SCAN_ROUND, SCAN_ROUND + 1]


def test_oracle_matches_the_golden_stuffing_file():
    g = np.load(GOLD)
    for label in CONSTRUCTED:
        coef, _, kmax = chain_case(label)
        h, w = coef.shape
        assert np.array_equal(g[label + "/coef"], coef), label
        data = O.ht_encode(O.to_sgnmag(coef, kmax), kmax, cap=65536)
        assert np.array_equal(g[label + "/data"], data), label
        rc, dec = O.ht_decode(data, kmax, w, h)
        assert rc == 0 and np.array_equal(g[label + "/dec"], dec), label


def _other_suites():
    """(suite, coding) of the image-shaped cases of the suites that reach the encoder by chance"""
    import test_device_roundtrip as RT
    import test_dynamic_range as DR
    import test_gpu as TG
    import test_ht_foreign as HF
    for a in TG.GEOMS:
        for irr in (False, True):
            yield "test_gpu", G.make_coding(irreversible=irr, **a)
    for a in DR.BLOCK_CASES + DR.SWEEP:
        yield "test_dynamic_range", DR.coding(a)
    for a in RT.CASES.values():
        yield "test_device_roundtrip", G.make_coding(**a)
    for c in HF.FOREIGN_CODINGS:
        yield "test_ht_foreign", G.make_coding(**c["args"])


def test_gap_report_of_the_other_suites(capsys):
    """Which staging and launch cells the case lists of the other suites reach, and the longest MagSgn and VLC fix-up
    chains of the synthetic images test_gpu.py codes (printed, not asserted: the cases above are what reach every
    cell and chain)."""
    reached, scans = {}, set()
    for suite, cp in _other_suites():
        reached.setdefault(suite, set()).update(cells(cp))
        scans |= scan_cells(len(coded_blocks(cp)), 0)
    term = set()
    longest128 = longest32 = vlc128 = vlc32 = 0
    for a in __import__("test_gpu").GEOMS[:3]:
        cp = G.make_coding(**a)
        coefs = P.forward(cp, P.synthetic_image(a["width"], a["height"], a["numcomps"], a["prec"], seed=1))
        rects = P.tile_rects(cp)
        for i, t, c, b, w, h, kmax, _ in coded_blocks(cp)[:150]:
            x0, y0 = rects[t][0] - cp.x0 + b.buf_x, rects[t][1] - cp.y0 + b.buf_y
            ms, vlc, unit_bits, _ = raw_streams(coefs[c][y0:y0 + h, x0:x0 + w], kmax)
            it128, it32, _, _ = ms_drains(ms)
            longest128, longest32 = max([longest128] + it128), max([longest32] + it32)
            it128, it32, _, _ = vlc_drains(vlc, vlc_trips(w, unit_bits))
            vlc128, vlc32 = max([vlc128] + it128), max([vlc32] + it32)
            term |= block_model(coefs[c][y0:y0 + h, x0:x0 + w], kmax)["cells"]
    with capsys.disabled():
        print()
        for suite, r in reached.items():
            print("%s misses %d of %d cells: %s" % (suite, len(ALL_CELLS - r), len(ALL_CELLS), sorted(ALL_CELLS - r, key=str)))
        together = set().union(*reached.values())
        print("all four together miss: %s" % sorted(ALL_CELLS - together, key=str))
        print("longest MagSgn drain chains of test_gpu.py's first three images: %d iterations in a 128-byte drain, %d "
              "in a final drain (a final drain's lanes past the stream read ones, which stuff every other byte)"
              % (longest128, longest32))
        print("longest VLC drain chains of the same images: %d iterations in a 128-byte drain, %d in a 32-byte drain"
              % (vlc128, vlc32))
        print("termination cells the same blocks miss: %s" % sorted(TERM_REACHABLE - term, key=str))
        print("length-scan cells the four suites' single-launch codings miss: %s" % sorted(SCAN_CELLS - scans))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _content(cp, seed):
    """coefficient planes: per block, by turns, sparse small values, dense values at the band's top planes, noise
    over a few planes and a few isolated samples (long runs of insignificant quads: MEL bytes of 0xFF, each followed by
    a 7-bit byte) -- int32, or float bits for 9/7 whose quantised indices stay below 2^Kmax"""
    rng = np.random.default_rng(seed)
    w, h = cp.x1 - cp.x0, cp.y1 - cp.y0
    out = [np.zeros((h, w), np.int32) for _ in range(cp.numcomps)]
    rects = P.tile_rects(cp)
    for i, t, c, b, bw, bh, kmax, _ in coded_blocks(cp):
        top = (1 << min(kmax, 20)) - 1
        kind = i % 4
        if kind == 0:
            idx = rng.integers(-15, 16, (bh, bw)) * (rng.random((bh, bw)) < 0.2)
        elif kind == 1:
            idx = rng.integers(top // 2, top + 1, (bh, bw)) * rng.choice([-1, 1], (bh, bw))
        elif kind == 2:
            idx = rng.integers(-255, 256, (bh, bw))
        else:
            idx = rng.integers(-255, 256, (bh, bw)) * (rng.random((bh, bw)) < 0.002)
        x0, y0 = rects[t][0] - cp.x0 + b.buf_x, rects[t][1] - cp.y0 + b.buf_y
        if cp.irreversible:
            step = float(P.band_params(cp, b.resno, b.orient)[1])
            idx = np.clip(idx, -(top - (1 << max(0, kmax - 21))), top - (1 << max(0, kmax - 21)))
            out[c][y0:y0 + bh, x0:x0 + bw] = (np.sign(idx) * (np.abs(idx) + 0.5) * step).astype(np.float32).view(np.int32)
        else:
            out[c][y0:y0 + bh, x0:x0 + bw] = idx
    return out


def _run(engine, cp, coefs, want_blocks=None):
    """encode on the device, compare bytes / offsets / decodes with the oracle; returns nothing, asserts"""
    blks = coded_blocks(cp)
    rects = P.tile_rects(cp)
    job = engine.job(cp)
    try:
        job.upload([np.zeros_like(p) for p in coefs])
        job.upload_coeffs(coefs)
        job.t1_encode()
        res = job.fetch_result()
        lengths, wants = [], []
        for i, t, c, b, w, h, kmax, _ in blks:
            want = P.encode_block(cp, coefs, rects[t], c, b) if want_blocks is None else want_blocks[i]
            got = res.block_bytes(i)
            assert np.array_equal(want, got), "block %d (%dx%d, Kmax %d): %s bytes, want %d" % (
                i, w, h, kmax, len(got), len(want))
            lengths.append(len(want))
            wants.append(want)
        offs = np.array([int(res.blocks[i]["offset"]) for i, *_ in blks])
        assert np.array_equal(offs, np.concatenate([[0], np.cumsum(lengths)[:-1]])), "offsets are not the scan"
        table = res.blocks.copy()
        res.free()
        want_dec = [np.zeros_like(p) for p in coefs]
        for (i, t, c, b, w, h, _, _), data in zip(blks, wants):
            x0, y0 = rects[t][0] - cp.x0 + b.buf_x, rects[t][1] - cp.y0 + b.buf_y
            want_dec[c][y0:y0 + h, x0:x0 + w] = P.decode_block(cp, data, c, b)
        got = [np.full_like(p, -1) for p in coefs]
        job.upload_coeffs(got)
        job.t1_decode()
        job.download_coeffs(got)
        for c, (g, r) in enumerate(zip(got, want_dec)):
            assert np.array_equal(g, r), "component %d: %d coefficients differ from the oracle's decode" % (
                c, int((g != r).sum()))
            if not cp.irreversible:
                assert np.array_equal(g, coefs[c])
        # the same bytes from a caller's table: block k starts at residue k mod 4 of a word
        chunks, off = [], 0
        for k, ((i, *_), data) in enumerate(zip(blks, wants)):
            pad = (k - off) % 4
            chunks.append(np.full(pad, 0xA5, np.uint8))
            off += pad
            table[i]["offset"] = off
            chunks.append(data)
            off += len(data)
        got = [np.full_like(p, -1) for p in coefs]
        job.upload_coeffs(got)
        job.t1_decode_blocks(table, np.concatenate(chunks))
        job.download_coeffs(got)
        for c, (g, r) in enumerate(zip(got, want_dec)):
            assert np.array_equal(g, r), "caller's table, component %d: %d coefficients differ" % (c, int((g != r).sum()))
    finally:
        job.close()


@pytest.mark.gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("name", ORDER)
def test_geometry_case_matches_oracle(engine, name, kind):
    cp = coding(name, kind)
    _run(engine, cp, _content(cp, seed=len(name)))


def _one_block_coding(w, h, kmax):
    pw = lambda n: max(4, 1 << (int(n) - 1).bit_length())     # noqa: E731
    cp = G.make_coding(w, h, 1, 16, numres=1, cblk=(pw(w), pw(h)))
    cp.qcd_explicit = 1
    cp.qcd_expn[0], cp.qcd_mant[0] = kmax, 0                   # Kmax = exponent + guard bits - 1, one guard bit
    return cp


@pytest.mark.gpu
@pytest.mark.parametrize("label", CONSTRUCTED)
def test_constructed_stuffing_matches_oracle(engine, label):
    """The constructed blocks, alone and repeated 16 times over one launch (so that warps meet them at several
    positions; blocks narrower or lower than the code-block size are not repeated along that side), against the
    golden bytes."""
    g = np.load(GOLD)
    coef = g[label + "/coef"]
    h, w = coef.shape
    kmax = chain_case(label)[2]
    cp = _one_block_coding(w, h, kmax)
    assert P.band_params(cp, 0, 0)[0] == kmax
    _run(engine, cp, [coef.astype(np.int32)], want_blocks=[g[label + "/data"]])
    full_w, full_h = w == 1 << cp.cblkw_exp, h == 1 << cp.cblkh_exp
    if not full_w:
        return
    reps = (4, 4) if full_h else (1, 16)
    cp16 = _one_block_coding(reps[1] * w, reps[0] * h, kmax)
    cp16.cblkw_exp, cp16.cblkh_exp = cp.cblkw_exp, cp.cblkh_exp
    tiled = np.tile(coef, reps).astype(np.int32)
    assert all((b.x1 - b.x0, b.y1 - b.y0) == (w, h) for _, _, b in P.enumerate_all(cp16))
    _run(engine, cp16, [tiled], want_blocks=[g[label + "/data"]] * 16)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SWEEPS))
def test_length_sweep_after_a_range_and_in_the_code_stream(engine, name):
    """The sweep's blocks through the pipelined round trip in 128-block ranges (each range's scan starts from the
    previous range's end, its gather writes after it) and through the device code-stream writer (each block's bytes
    at the place the packets give them), against the oracle and the T2 oracle."""
    import oracle_t2 as T2
    import test_device_roundtrip as RT
    torch = pytest.importorskip("torch")
    cp, table, data = sweep_encoded(name)
    planes = sweep_planes(name)
    job = engine.job(cp)
    try:
        nbytes = RT.run(job, planes, ("pipelined", SWEEP_SHAPE), steps=1)
        RT.check_job(job, cp, RT.oracle_step(cp, planes), nbytes, name + ", pipelined")
    finally:
        job.close()
    img = torch.from_numpy(np.stack(planes).astype(np.uint8)).cuda()
    for flags in SWEEP_FLAGS:
        want = T2.write_flags(cp, table, data, flags)
        got = engine.encode_codestream_device(cp, img, flags, device_output=True).cpu().numpy()
        diff = np.flatnonzero(got[:len(want)] != want[:len(got)])
        assert len(got) == len(want) and not len(diff), "%s, flags 0x%x: %d vs %d bytes, first difference at %s" % (
            name, flags, len(got), len(want), diff[:1])


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SCAN_CODINGS))
def test_length_scan_round_edges(engine, name):
    """8192 blocks fill exactly one round of the length scan; 8193 leave one block for a second round."""
    cp = coding_of(SCAN_CODINGS[name])
    _run(engine, cp, _content(cp, seed=8))
