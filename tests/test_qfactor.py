"""Lossy HT coding at a JPEG-style quality factor (b2k_coding.qfactor) and per-component quantisation (QCC).

Pinned to the reference: tests/golden/qfactor.npz holds what grk_compress -I --qfactor Q writes (make_golden_qfactor.py),
and a restatement of the quality model here, from the published sources (T.800 Annex F 9/7 synthesis filters, Zeng, Daly
and Lei's visual weights, the ICT column norms of T.800 Annex G), agrees with both."""
import copy
import ctypes as C
import hashlib
import math
import os

import numpy as np
import pytest

import grok_b200 as G
import oracle_pipeline as P

HERE = os.path.dirname(os.path.abspath(__file__))
REC = np.load(os.path.join(HERE, "golden", "qfactor.npz"))
PROG = {"LRCP": 0, "RPCL": 2}

# ---- the quality model, restated ------------------------------------------------------------------------------------
LO = [-0.091271763114250, -0.057543526228500, 0.591271763114250, 1.115087052457000, 0.591271763114250,
      -0.057543526228500, -0.091271763114250]
HI = [0.053497514821622, 0.033728236885750, -0.156446533057980, -0.533728236885750, 1.205898036472720,
      -0.533728236885750, -0.156446533057980, 0.033728236885750, 0.053497514821622]
VIS = [[0.0901, 0.2758, 0.2758, 0.7018, 0.8378, 0.8378] + [1.0] * 9,
       [0.0263, 0.0863, 0.0863, 0.1362, 0.2564, 0.2564, 0.3346, 0.4691, 0.4691, 0.5444, 0.6523, 0.6523, 0.7078, 0.7797, 0.7797],
       [0.0773, 0.1835, 0.1835, 0.2598, 0.4130, 0.4130, 0.5040, 0.6464, 0.6464, 0.7220, 0.8254, 0.8254, 0.8769, 0.9424, 0.9424]]
ICT = [1.7321, 1.8051, 1.5734]


def _energies(levels):
    lo, hi, out = list(LO), list(HI), []
    for _ in range(levels):
        out.append((sum(t * t for t in lo), sum(t * t for t in hi)))
        nl, nh = [0.0] * (7 + 2 * len(lo) - 1), [0.0] * (7 + 2 * len(hi) - 1)
        for i in range(7):
            for j, t in enumerate(lo):
                nl[i + 2 * j] += LO[i] * t
            for j, t in enumerate(hi):
                nh[i + 2 * j] += LO[i] * t
        lo, hi = nl, nh
    return out


ENERGY = _energies(7)


def qfactor_table(q, prec, numres, comp):
    """[(exponent, mantissa)] in QCD band order"""
    D = numres - 1
    m = 50.0 / q if q < 50 else 2.0 * (1.0 - q / 100.0)
    knee, top = 2.0 * (1.0 - 65 / 100.0), 2.0 * (1.0 - 97 / 100.0)
    alpha, wpow = 0.04, 1.0
    if q >= 97:
        alpha, wpow = 0.10, 0.0
    elif q > 65:
        wpow = (math.log(top) - math.log(m)) / (math.log(top) - math.log(knee))
        alpha = 0.10 * math.pow(0.04 / 0.10, wpow)
    ref = (alpha * m + math.sqrt(0.5) * math.ldexp(1.0, -prec)) * ICT[0]
    norm2 = []
    for lo, hi in ENERGY[:D]:
        norm2 += [hi * hi, lo * hi, hi * lo]
    norm2.append(ENERGY[D - 1][0] ** 2 if D else 1.0)
    out = []
    for k, n2 in enumerate(norm2):
        w = 1.0 if (k == len(norm2) - 1 or k >= 15) else math.pow(VIS[comp][k], wpow)
        step = ref / (math.sqrt(n2) * w * ICT[comp])
        e = 0
        while step < 1.0:
            step *= 2.0
            e += 1
        mu = int(math.floor((step - 1.0) * 2048.0 + 0.5))
        if mu > 2047:
            mu, e = 0, e - 1
        if e > 31:                       # the exponent field is five bits; a step above 2 is written as the largest
            e, mu = 31, 0
        if e < 0:
            e, mu = 0, 2047
        out.append((e, mu))
    return out[::-1]


# ---- reading headers ------------------------------------------------------------------------------------------------
def segments(cs):
    """[(marker, payload)] of a main header up to the first SOT"""
    cs, p, out = bytes(cs), 2, []
    while cs[p:p + 2] != b"\xff\x90" and p < len(cs):
        m, n = int.from_bytes(cs[p:p + 2], "big"), int.from_bytes(cs[p + 2:p + 4], "big")
        out.append((m, cs[p + 4:p + 2 + n]))
        p += 2 + n
    return out


def quant_of(cs, ncomp):
    """per component [(exponent, mantissa)] from QCD / QCC (irreversible)"""
    qcd, qcc = None, {}
    for m, b in segments(cs):
        if m == 0xFF5C:
            qcd = b[1:]
        elif m == 0xFF5D:
            qcc[b[0]] = b[2:]
    words = lambda b: [(int.from_bytes(b[i:i + 2], "big") >> 11, int.from_bytes(b[i:i + 2], "big") & 0x7FF)
                       for i in range(0, len(b), 2)]
    return [words(qcc.get(c, qcd)) for c in range(ncomp)]


def quant_bytes(cs):
    """CAP .. the last QCC, as the record holds them"""
    return b"".join(m.to_bytes(2, "big") + (len(b) + 2).to_bytes(2, "big") + b for m, b in segments(cs)
                    if m in (0xFF50, 0xFF52, 0xFF5C, 0xFF5D))


def table_coding(q, prec, numres, ncomp, numgbits=4):
    size = 1 << max(3, numres)
    return G.make_coding(size, size, ncomp, prec, numres=numres, irreversible=True, numgbits=numgbits, qfactor=q)


# ---- 1. tables ------------------------------------------------------------------------------------------------------
def test_tables_equal_grk_compress_and_the_restatement():
    ends = np.concatenate([[0], np.cumsum(REC["seg_len"])])
    raw = REC["seg_bytes"].tobytes()
    assert len(REC["cases"]) == 100 * 4 * 4 * 2
    for k, (q, prec, numres, ncomp) in enumerate(REC["cases"].tolist()):
        theirs = raw[ends[k]:ends[k + 1]]
        head = G.codestream_write_header(table_coding(q, prec, numres, ncomp), 0, [0])
        assert quant_bytes(head) == theirs, (q, prec, numres, ncomp)
        got = quant_of(head, ncomp)
        for c in range(ncomp):
            assert got[c] == qfactor_table(q, prec, numres, c), (q, prec, numres, ncomp, c)


def test_qcc_only_for_components_that_differ_and_only_in_the_main_header():
    head = G.codestream_write_header(table_coding(75, 8, 6, 3), 0, [0])
    assert [b[0] for m, b in segments(head) if m == 0xFF5D] == [1, 2]
    order = [m for m, _ in segments(head)]
    assert order.index(0xFF5C) < order.index(0xFF5D)
    grey = G.codestream_write_header(table_coding(75, 8, 6, 1), 0, [0])
    assert 0xFF5D not in [m for m, _ in segments(grey)]


# ---- 2. code streams ------------------------------------------------------------------------------------------------
def component_coding(cp, table):
    """cp with one component's table as its QCD (what the CPU oracle's per-band parameters read)"""
    cc = copy.deepcopy(cp)
    cc.qfactor, cc.qcd_explicit = 0, 1
    for i, (e, m) in enumerate(table):
        cc.qcd_expn[i], cc.qcd_mant[i] = e, m
    return cc


def oracle_encode(cp, planes):
    """the CPU oracle's blocks, each component quantised with its own table"""
    tables = quant_of(G.codestream_write_header(cp, 0, [0]), cp.numcomps)
    comp_cp = [component_coding(cp, t) for t in tables]
    coefs = P.forward(cp, planes)
    table = G.enumerate_blocks(cp)
    blks = P.enumerate_all(cp)
    rects = P.tile_rects(cp)
    assert len(table) == len(blks)
    chunks, off = [np.zeros(0, np.uint8)], 0
    for i, (t, c, b) in enumerate(blks):
        kmax, step, _ = P.band_params(comp_cp[c], b.resno, b.orient)
        assert table[i]["kmax"] == kmax and np.float32(table[i]["stepsize"]) == np.float32(step)
        if b.x1 == b.x0 or b.y1 == b.y0:
            continue
        data = P.encode_block(comp_cp[c], coefs, rects[t], c, b)
        table[i]["length"], table[i]["offset"], table[i]["numbps"], table[i]["numpasses"] = len(data), off, 1, 1
        chunks.append(data)
        off += len(data)
    return table, np.concatenate(chunks), comp_cp


STREAMS = {
    # name: (width, height, ncomp, prec, numres, qfactor, guard bits, tile, origin, TLM + PLT, progression, seed)
    "q50": (200, 136, 3, 8, 6, 50, 1, None, (0, 0), False, "LRCP", 1),
    "q60_tiled": (256, 192, 3, 10, 6, 60, 1, (128, 128), (0, 0), True, "LRCP", 2),
    "q75_rpcl": (160, 160, 3, 12, 5, 75, 1, (96, 64), (0, 0), True, "RPCL", 3),
    "q90_origin": (150, 130, 3, 8, 4, 90, 1, (64, 64), (17, 9), True, "LRCP", 4),
    "q97_grey": (128, 96, 1, 16, 6, 97, 1, None, (0, 0), False, "LRCP", 5),
    "q100": (96, 80, 3, 12, 3, 100, 1, None, (0, 0), True, "RPCL", 6),
    "q30_N2": (128, 128, 3, 8, 6, 30, 2, (64, 64), (0, 0), True, "LRCP", 7),
    "q10_N4": (120, 100, 1, 12, 6, 10, 4, None, (3, 5), False, "LRCP", 8),
    "q80_signed": (128, 96, 3, 8, 5, 80, 1, None, (0, 0), True, "LRCP", 9),
}
SIGNED = {"q80_signed"}
DECODED = ("q50", "q90_origin", "q80_signed")       # the record holds grk_decompress's pixels of these


def stream_case(name):
    w, h, nc, prec, numres, q, gb, tile, origin, tlm, prog, seed = STREAMS[name]
    cp = G.make_coding(w, h, nc, prec, sgnd=name in SIGNED, numres=numres, irreversible=True, numgbits=gb, tile=tile,
                       origin=origin, qfactor=q, tile_origin=(0, 0))
    if not tile and origin != (0, 0):       # grk_compress's single tile at an offset: anchored at 0, reaching the far corner
        cp.tx0, cp.ty0, cp.tw, cp.th = 0, 0, cp.x1, cp.y1
    planes = P.synthetic_image(w, h, nc, prec, seed=seed, origin=origin)
    if name in SIGNED:
        planes = [p - (1 << (prec - 1)) for p in planes]
    flags = (G.CS_TLM | G.CS_PLT if tlm else 0) | G.CS_PROG(PROG[prog])
    return cp, planes, flags


@pytest.mark.parametrize("name", sorted(STREAMS))
def test_codestream_equals_grk_compress(name):
    cp, planes, flags = stream_case(name)
    table, data, _ = oracle_encode(cp, planes)
    cs = G.codestream_write(cp, table, data, flags)
    k = list(REC["stream_names"]).index(name)
    assert len(cs) == REC["stream_len"][k]
    assert hashlib.sha256(bytes(cs)).hexdigest() == REC["stream_sha"][k], "differs from grk_compress --qfactor"
    cp2, blocks = G.codestream_parse(cs)
    assert cp2.qfactor == cp.qfactor and cp2.qcd_explicit == 0 and cp2.qcc_mask == 0       # parse(write(cp)) == cp
    assert bytes(cp2) == bytes(_with_explicit_grid(cp, cp2))
    assert np.array_equal(blocks["length"], table["length"])


def _with_explicit_grid(cp, cp2):
    """cp as the parser returns it: an untiled coding comes back as one explicit tile"""
    c = copy.deepcopy(cp)
    c.tx0, c.ty0, c.tw, c.th = cp2.tx0, cp2.ty0, cp2.tw, cp2.th
    return c


# ---- 3. decode of our streams -----------------------------------------------------------------------------------------
def oracle_decode(cp, comp_cp, blocks, cs):
    blks = P.enumerate_all(cp)
    rects = P.tile_rects(cp)
    w, h = cp.x1 - cp.x0, cp.y1 - cp.y0
    coefs = [np.zeros((h, w), np.int32) for _ in range(cp.numcomps)]
    for i, (t, c, b) in enumerate(blks):
        bw, bh = b.x1 - b.x0, b.y1 - b.y0
        if bw == 0 or bh == 0 or blocks[i]["length"] == 0:
            continue
        o, n = int(blocks[i]["offset"]), int(blocks[i]["length"])
        win = P.decode_block(comp_cp[c], cs[o:o + n], c, b, numbps=int(blocks[i]["numbps"]))
        x0, y0 = rects[t][0] - cp.x0, rects[t][1] - cp.y0
        coefs[c][y0 + b.buf_y:y0 + b.buf_y + bh, x0 + b.buf_x:x0 + b.buf_x + bw] = win
    return P.inverse(cp, coefs)


def psnr(a, b, prec):
    mse = np.mean((np.stack(a).astype(np.float64) - np.stack(b)) ** 2)
    return 10 * math.log10(((1 << prec) - 1) ** 2 / max(mse, 1e-12))


def test_openjpeg_decodes_a_qfactor_stream_as_the_oracle_does():
    cv2 = pytest.importorskip("cv2")
    cp, planes, flags = stream_case("q50")
    table, data, comp_cp = oracle_encode(cp, planes)
    cs = G.codestream_write(cp, table, data, flags)
    ours = oracle_decode(cp, comp_cp, G.codestream_parse(cs)[1], cs)
    img = cv2.imdecode(np.frombuffer(bytes(G.jph_wrap(cp, cs)), np.uint8), cv2.IMREAD_UNCHANGED)
    assert img is not None
    theirs = [img[..., 2 - c].astype(np.int32) for c in range(3)]                # OpenCV's BGR
    assert max(int(np.abs(a - b).max()) for a, b in zip(ours, theirs)) <= 1
    assert 25 < psnr(ours, planes, 8) < 60


@pytest.mark.parametrize("name", DECODED)
def test_oracle_decode_of_our_stream_matches_grk_decompress(name):
    """our streams are grk_compress's byte for byte, so grk_decompress's pixels of its own stream are its decode of ours;
    the oracle's float 9/7 agrees with Grok's fixed-point one within the reference's 2-code bar (test_interop.py)"""
    cp, planes, flags = stream_case(name)
    table, data, comp_cp = oracle_encode(cp, planes)
    cs = G.codestream_write(cp, table, data, flags)
    ours = np.stack(oracle_decode(cp, comp_cp, G.codestream_parse(cs)[1], cs))
    theirs = REC["decoded_" + name].astype(np.int64)
    assert ours.shape == theirs.shape
    assert int(np.abs(ours - theirs).max()) <= 2
    assert psnr(list(ours), planes, cp.prec) > 25


# ---- 4. foreign QCC ---------------------------------------------------------------------------------------------------
def with_segment(cs, marker, payload, after=0xFF5C):
    """cs with one more main-header segment behind the first `after` segment"""
    cs, p = bytes(cs), 2
    while True:
        m, n = int.from_bytes(cs[p:p + 2], "big"), int.from_bytes(cs[p + 2:p + 4], "big")
        p += 2 + n
        if m == after:
            break
    return np.frombuffer(cs[:p] + marker.to_bytes(2, "big") + (len(payload) + 2).to_bytes(2, "big") + payload + cs[p:], np.uint8)


def qcc_payload(comp, table, numgbits=1, irreversible=True):
    """T.800 A.6.5: Cqcc (8 bits), Sqcc, SPqcc"""
    body = bytes([comp, (numgbits << 5) | (2 if irreversible else 0)])
    for e, m in table:
        body += ((e << 11) | m).to_bytes(2, "big") if irreversible else bytes([e << 3])
    return body


def foreign(cp, planes, tables, flags=0):
    """a stream whose components c in `tables` carry those exponents / mantissas through a QCC we insert, with blocks
    coded to match: -> (stream, per-component codings for the oracle)"""
    base = quant_of(G.codestream_write_header(cp, 0, [0]), cp.numcomps)
    per = [tables.get(c, base[c]) for c in range(cp.numcomps)]
    comp_cp = [component_coding(cp, t) for t in per] if cp.irreversible else [cp] * cp.numcomps
    coefs = P.forward(cp, planes)
    table = G.enumerate_blocks(cp)
    blks = P.enumerate_all(cp)
    rects = P.tile_rects(cp)
    chunks, off = [np.zeros(0, np.uint8)], 0
    if not cp.irreversible:
        for c in tables:
            comp_cp[c] = copy.deepcopy(cp)
            comp_cp[c].qcd_explicit = 1
            for k, (e, _) in enumerate(tables[c]):
                comp_cp[c].qcd_expn[k] = e
    for i, (t, c, b) in enumerate(blks):
        cc = comp_cp[c]
        table[i]["kmax"] = P.band_params(cc, b.resno, b.orient)[0]
        if b.x1 == b.x0 or b.y1 == b.y0:
            continue
        data = P.encode_block(cc, coefs, rects[t], c, b)
        table[i]["length"], table[i]["offset"], table[i]["numbps"], table[i]["numpasses"] = len(data), off, 1, 1
        chunks.append(data)
        off += len(data)
    cs = G.codestream_write(cp, table, np.concatenate(chunks), flags)
    for c in sorted(tables, reverse=True):
        cs = with_segment(cs, 0xFF5D, qcc_payload(c, tables[c], cp.numgbits, cp.irreversible))
    return cs, table, comp_cp


def foreign_case(case):
    """(coding, planes, QCC tables by component) of the foreign-QCC cases"""
    nc = 4 if case == "one_of_four" else 3
    cp = G.make_coding(96, 80, nc, 8, numres=4, irreversible=case != "reversible", mct=nc == 3, tile=(64, 64))
    planes = P.synthetic_image(96, 80, nc, 8, seed=11)
    base = quant_of(G.codestream_write_header(cp, 0, [0]), nc) if cp.irreversible else None
    if case == "comp0":
        tables = {0: shifted(base[0], 1)}
    elif case == "equal_to_qcd":
        tables = {1: base[0], 2: base[0]}
    elif case == "reversible":
        head = [b for m, b in segments(G.codestream_write_header(cp, 0, [0])) if m == 0xFF5C][0]
        tables = {2: [((v >> 3) + 1, 0) for v in head[1:]]}
    else:
        tables = {3: shifted(base[3], -1)}
    return cp, planes, tables


def shifted(table, d):
    return [(e + d, (m + 97 * i) % 2048) for i, (e, m) in enumerate(table)]


@pytest.mark.parametrize("case", ["comp0", "equal_to_qcd", "reversible", "one_of_four"])
def test_foreign_qcc_parses_and_decodes_to_the_oracle(case):
    cp, planes, tables = foreign_case(case)
    nc = cp.numcomps
    cs, table, comp_cp = foreign(cp, planes, tables)
    cp2, blocks = G.codestream_parse(cs)
    assert np.array_equal(blocks["kmax"], table["kmax"])
    assert np.array_equal(blocks["length"], table["length"])
    if case == "equal_to_qcd":
        assert cp2.qcc_mask == 0                        # the HT quantiser's tables throughout: nothing to spell out
    else:
        assert cp2.qcc_mask == sum(1 << c for c in tables)
        for c, t in tables.items():
            n = len(t)
            assert list(cp2.qcc_expn[c])[:n] == [e for e, _ in t]
            assert list(cp2.qcc_mant[c])[:n] == [m if cp.irreversible else 0 for _, m in t]
    # the oracle decodes the parsed blocks with each component's own table: the source back (5/3), or close to it (9/7)
    pix = oracle_decode(cp2, comp_cp, blocks, cs)
    if cp.irreversible:
        assert psnr(pix, planes, 8) > 30
    else:
        assert all(np.array_equal(a, b) for a, b in zip(pix, planes))


def test_damaged_qcc_is_an_error_and_tile_part_qcc_and_coc_are_declined():
    cp = G.make_coding(64, 64, 3, 8, numres=3, irreversible=True, qfactor=80)
    cs = G.codestream_write(cp, *oracle_encode(cp, P.synthetic_image(64, 64, 3, 8, seed=3))[:2], 0)
    L = G.lib()
    probe = lambda s: L.b2k_codestream_parse(np.ascontiguousarray(s).ctypes.data, len(s), C.byref(G.Coding()), None, 0)
    table = quant_of(cs, 3)[1]
    assert probe(with_segment(cs, 0xFF5D, qcc_payload(3, table))) == -1                  # Cqcc >= Csiz
    assert probe(with_segment(cs, 0xFF5D, qcc_payload(1, table)[:-3])) == -1              # fewer values than bands
    assert probe(with_segment(cs, 0xFF5D, bytes([1]))) == -1                              # no Sqcc
    assert probe(with_segment(cs, 0xFF53, bytes([1, 0, 2, 4, 4, 0x40, 0]))) == 1          # COC
    # QCC in the first tile-part header
    sot = bytes(cs).index(b"\xff\x90")
    n = 2 + 10
    seg = b"\xff\x5d" + (len(qcc_payload(1, table)) + 2).to_bytes(2, "big") + qcc_payload(1, table)
    raw = bytearray(bytes(cs)[:sot + n] + seg + bytes(cs)[sot + n:])
    psot = int.from_bytes(raw[sot + 6:sot + 10], "big")
    raw[sot + 6:sot + 10] = (psot + len(seg)).to_bytes(4, "big")
    with pytest.raises(G.NotHandled, match="tile-part"):
        G.codestream_parse(np.frombuffer(bytes(raw), np.uint8))


# ---- 5. declines ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw, text", [
    (dict(irreversible=False, qfactor=50), "irreversible"),
    (dict(ncomp=2, qfactor=50, mct=False), "one or three components"),
    (dict(ncomp=4, qfactor=50), "one or three components"),
    (dict(qfactor=101), "quality factor 1..100"),
    (dict(qfactor=25), "quality factor 25 with 1 guard bit"),
])
def test_declined_codings(kw, text):
    kw = dict(kw)
    nc = kw.pop("ncomp", 3)
    cp = G.make_coding(64, 64, nc, 8, numres=6, **{"irreversible": True, **kw})
    n = G.lib().b2k_enumerate(C.byref(cp), 1, 0, None, 0)
    assert n == -1 and text in G.lib().b2k_last_error().decode()


def test_kmax0_declines_match_grk_compress():
    """at one guard bit (8-bit, 6 resolutions) the engine declines exactly the quality factors grk_compress refuses:
    the record holds its verdict for 20..50, across the boundary (36 refused, 37 written)"""
    verdict = dict(zip(REC["verdict_q"].tolist(), REC["verdict"].tolist()))
    assert verdict[36] == 0 and verdict[37] == 1
    for q, ok in verdict.items():
        cp = G.make_coding(64, 64, 3, 8, numres=6, irreversible=True, qfactor=q)
        assert (G.lib().b2k_enumerate(C.byref(cp), 1, 0, None, 0) > 0) == bool(ok), q
