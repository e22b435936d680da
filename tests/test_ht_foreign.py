"""HT cleanup segments written with the choices T.814 leaves to the encoder -- any legal CxtVLC row, a raised exponent
bound U_q, MEL / VLC terminated without the shared byte, padding after MagSgn and between MEL and VLC -- as other HTJ2K
encoders write them and this project's coders never do.

CPU: the oracle's foreign-choice encoder (orc_ht_encode_foreign) and decoders against tests/golden/ht_foreign.npz, which
holds what the reference's own decoders make of the same bytes (tests/golden/make_golden_foreign.py), plus a boundary
set edited from known streams: Scup = 2, Scup = 4079 and 4080, Lcup = Scup, U_q at the decoder's limit and one above,
missing MSBs 29, 30 and 31.
GPU: the device decoder (k_ht_decode_vlc + k_ht_decode_magsgn, and k_ht_decode_refine on top) on such streams for every
block of real codings, through the block-table, host and code-stream entry points, and on the boundary set."""
import os

import numpy as np
import pytest

import grok_b200 as G
import oracle_lib as O
import oracle_pipeline as P

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ht_foreign.npz")
CHOICE_BITS = (O.FOREIGN_ROWS, O.FOREIGN_RAISE_U, O.FOREIGN_NO_FUSE, O.FOREIGN_PAD_MAGSGN, O.FOREIGN_PAD_SCUP)


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def _bin_centre(sm, mm):
    mu = ((sm & 0x7FFFFFFF) >> (30 - mm)).astype(np.uint64)
    return np.where(mu > 0, (sm & 0x80000000) | ((2 * mu + 1) << np.uint64(29 - mm)), 0).astype(np.uint32)


def _group(g, prefix):
    """the blocks of one group of the golden file (tests/golden/make_golden_foreign.py, pack()): (meta row as ints,
    source words (h, w) or None, stream bytes, the reference's decode (h, w))"""
    meta = g[prefix + "meta"]
    arr = {k: (g[prefix + k], g[prefix + k + "_off"]) for k in ("src", "data", "dec_x")}
    for i, row in enumerate(meta):
        row = [int(v) for v in row]
        w, h = row[0], row[1]
        src, data, dec_x = (a[o[i]:o[i + 1]] for a, o in arr.values())
        src = src.reshape(h, w) if src.size else None
        dec = dec_x.reshape(h, w) ^ (src if src is not None else 0)
        yield row, src, data, dec.astype(np.uint32)


def _boundary(g):
    for label, ((w, h, mm, rc), src, data, dec) in zip(g["blabel"], _group(g, "b")):
        yield dict(label=str(label), w=w, h=h, mm=mm, rc=rc, data=data, dec=dec, src=src)


# ---------------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------------
def test_foreign_encoder_reproduces_the_golden_streams(gold):
    for (w, h, kmax, choices, seed), sm, data, _ in _group(gold, ""):
        assert np.array_equal(O.ht_encode_foreign(sm, kmax, choices, seed, cap=65536), data), (w, h, kmax, choices)
        assert np.array_equal(O.ht_encode_foreign(sm, kmax, 0, seed, cap=65536), O.ht_encode(sm, kmax, cap=65536))
    for (w, h, M, npass, len2, causal, kmax, choices, seed), sm, data, _ in _group(gold, "r"):
        assert np.array_equal(O.ht_encode_foreign(sm, M, choices, seed, cap=65536), data[:len(data) - len2]), (w, h, M)
        assert np.array_equal(O.ht_encode_refine(sm, M, npass, bool(causal)), data[len(data) - len2:]), (w, h, M)


def test_oracle_decodes_foreign_streams_as_the_reference_does(gold):
    Rf = O.ref()
    for (w, h, kmax, choices, seed), sm, data, want in _group(gold, ""):
        rc, dec = O.ht_decode(data, kmax, w, h)
        assert rc == 0 and np.array_equal(dec, want), (w, h, kmax, choices)
        assert np.array_equal(want, _bin_centre(sm, kmax)), (w, h, kmax, choices)
        if Rf is not None:
            rc2, d2 = O.ref_ht_decode(data, kmax, w, h)
            assert rc2 == 0 and np.array_equal(d2, want), (w, h, kmax, choices)
    for (w, h, M, npass, len2, causal, kmax, choices, seed), sm, data, want in _group(gold, "r"):
        rc, dec = O.ht_decode_passes(data, len2, npass, M, w, h, causal=bool(causal))
        assert rc == 0 and np.array_equal(dec, want), (w, h, M, npass, causal, choices)
        if Rf is not None:
            rc2, d2 = O.ref_ht_decode(data, M, w, h, num_passes=npass, len2=len2, causal=bool(causal))
            assert rc2 == 0 and np.array_equal(d2, want), (w, h, M, npass, causal, choices)


def test_oracle_boundary_verdicts_match_the_reference(gold):
    Rf = O.ref()
    for b in _boundary(gold):
        rc, dec = O.ht_decode(b["data"], b["mm"], b["w"], b["h"])
        assert rc == b["rc"], (b["label"], rc, b["rc"])
        if rc == 0:
            assert np.array_equal(dec, b["dec"]), b["label"]
            if b["src"] is not None:
                assert np.array_equal(dec, _bin_centre(b["src"], b["mm"])), b["label"]
        if Rf is not None:
            rc2, d2 = O.ref_ht_decode(b["data"], b["mm"], b["w"], b["h"])
            assert (rc2 == 0) == (b["rc"] == 0), b["label"]
            if rc2 == 0:
                assert np.array_equal(d2, b["dec"]), b["label"]


def _scup(d):
    return (int(d[-1]) << 4) | (int(d[-2]) & 0xF)


def test_golden_set_covers_every_choice_and_boundary(gold):
    """Each choice changes the bytes of some golden block; some quad codes U_q at the limit, some u_off = 1 quad an e_k
    the max-popcount rule would not pick; widths above 64, Kmax 2..29, 2- and 3-pass, plain and stripe-causal; and every
    boundary with the verdict it is there for."""
    g = gold
    differs, at_limit, other_rows, kmaxes, shapes = set(), 0, 0, set(), set()
    for (w, h, kmax, choices, seed), sm, _, _ in _group(g, ""):
        kmaxes.add(kmax)
        shapes.add((w, h))
        plain = O.ht_encode(sm, kmax, cap=65536)
        for bit in CHOICE_BITS:
            if choices & bit and not np.array_equal(O.ht_encode_foreign(sm, kmax, bit, seed, cap=65536), plain):
                differs.add(bit)
        _, st = O.ht_encode_foreign(sm, kmax, choices, seed, cap=65536, stats=True)
        at_limit += st[0] if choices & O.FOREIGN_RAISE_U else 0
        other_rows += st[1]
    assert differs == set(CHOICE_BITS)
    assert at_limit > 0 and other_rows > 0
    assert kmaxes == set(range(2, 30)) and any(64 < w < 1024 for w, _ in shapes)
    assert {(1, 1), (1024, 4), (4, 1024)} <= shapes
    refined = {(row[3], row[5]) for row, *_ in _group(g, "r")}
    assert refined == {(2, 0), (2, 1), (3, 0), (3, 1)}
    seen = {}
    for b in _boundary(g):
        seen.setdefault(b["label"], set()).add(b["rc"])
        lcup, scup = len(b["data"]), _scup(b["data"])
        if b["label"].startswith("scup_2"):
            assert scup == 2
        elif b["label"] in ("scup_4079", "scup_4080"):
            assert scup == int(b["label"][5:])
        elif b["label"] == "lcup_eq_scup":
            assert scup == lcup
    assert seen == {"lcup_eq_scup": {0}, "scup_2": {0}, "scup_2_nibble": {0}, "scup_4079": {0}, "scup_4080": {-1},
                    "u_at_limit": {0}, "u_above_limit": {-1}, "mmsbs_29": {0}, "mmsbs_30": {-1}, "mmsbs_31": {-1}}
    assert any(np.count_nonzero(b["dec"]) for b in _boundary(g) if b["label"] == "scup_2_nibble")


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def _foreign_blocks(cp, coefs, npass, dropped, seed):
    """Every block of `cp` coded by the oracle's foreign-choice encoder (a seeded choice set per block, all five choices
    among them), `dropped` bit-planes above the LSB with SigProp (+ MagRef) for the next plane when npass > 1; returns
    the block table, the byte arena and the oracle's decode of it (dequantised coefficient planes)."""
    L = O.lib()
    blks = P.enumerate_all(cp)
    rects = P.tile_rects(cp)
    table = G.enumerate_blocks(cp)
    assert len(table) == len(blks)
    chunks, off = [], 0
    want = [np.zeros_like(c) for c in coefs]
    causal = bool(cp.cblk_sty & 0x08)
    rng = np.random.default_rng(seed)
    used = 0
    for i, (t, c, b) in enumerate(blks):
        w, h = b.x1 - b.x0, b.y1 - b.y0
        if w == 0 or h == 0:
            continue
        x0, y0 = rects[t][0] - cp.x0, rects[t][1] - cp.y0
        kmax, step_enc, step_dec = P.band_params(cp, b.resno, b.orient)
        win = np.ascontiguousarray(coefs[c][y0 + b.buf_y:y0 + b.buf_y + h, x0 + b.buf_x:x0 + b.buf_x + w])
        sm = np.zeros(w * h, np.uint32)
        if cp.irreversible:
            L.orc_ht_pre_irrev(win.view(np.float32), w, w, h, kmax, np.float32(1.0) / np.float32(step_enc), sm)
        else:
            L.orc_ht_pre_rev(win, w, w, h, kmax, sm)
        W = (((sm & 0x7FFFFFFF) << 1) | (sm & 0x80000000)).astype(np.uint32).reshape(h, w)
        s = dropped if kmax - 1 - dropped >= 0 else 0
        mm = kmax - 1 - s
        np_blk = npass if (s > 0 and mm <= 28 and rng.random() < 0.85) else 1
        choices = int(rng.integers(1, 32))
        used |= choices
        cup = O.ht_encode_foreign(W, mm, choices, int(rng.integers(1, 1 << 30)), cap=65536)
        seg = O.ht_encode_refine(W, mm, np_blk, causal) if np_blk > 1 else np.zeros(0, np.uint8)
        data = np.concatenate([cup, seg])
        rc, dec = O.ht_decode_passes(data, len(seg), np_blk, mm, w, h, causal=causal)
        assert rc == 0
        if cp.irreversible:
            out = np.zeros((h, w), np.float32)
            L.orc_ht_post_irrev(dec, w, w, h, kmax, step_dec, out, w)
            out = out.view(np.int32)
        else:
            out = np.zeros((h, w), np.int32)
            L.orc_ht_post_rev(dec, w, w, h, kmax, out, w)
        want[c][y0 + b.buf_y:y0 + b.buf_y + h, x0 + b.buf_x:x0 + b.buf_x + w] = out
        table[i]["length"], table[i]["length2"], table[i]["offset"] = len(cup), len(seg), off
        table[i]["numbps"], table[i]["numpasses"] = 1 + s, np_blk
        chunks.append(data)
        off += len(data)
    assert used == O.FOREIGN_ALL
    return table, np.concatenate(chunks), want


FOREIGN_CODINGS = [
    dict(args=dict(width=333, height=217, numcomps=3, prec=12, numres=4, origin=(3, 5)), npass=1, dropped=0, cs=True),
    dict(args=dict(width=333, height=217, numcomps=3, prec=12, numres=4, origin=(3, 5)), npass=3, dropped=1),
    dict(args=dict(width=320, height=200, numcomps=3, prec=12, numres=5, irreversible=True), npass=1, dropped=0),
    dict(args=dict(width=320, height=200, numcomps=3, prec=12, numres=5, irreversible=True), npass=3, dropped=2),
    dict(args=dict(width=2100, height=40, numcomps=1, prec=10, numres=2, cblk=(1024, 4)), npass=1, dropped=1),
    dict(args=dict(width=256, height=96, numcomps=1, prec=16, numres=3, numgbits=5, cblk=(1024, 4)), npass=2, dropped=1),
    dict(args=dict(width=200, height=160, numcomps=3, prec=12, numres=4), npass=3, dropped=1, causal=True),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", FOREIGN_CODINGS)
def test_device_decodes_foreign_streams(engine, case):
    """Block tables of foreign-choice streams decode on the device to exactly the oracle's coefficients (the oracle being
    pinned to the reference decoder by ht_foreign.npz), b2k_decode returns their inverse, and a code stream written from
    such a table decodes through the single and the batch device code-stream calls to the same pixels."""
    args = case["args"]
    cp = G.make_coding(**args)
    if case.get("causal"):
        cp.cblk_sty = 0x08
    planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=11,
                               origin=args.get("origin", (0, 0)))
    coefs = P.forward(cp, planes)
    table, data, want = _foreign_blocks(cp, coefs, case["npass"], case["dropped"], seed=17)
    job = engine.job(cp)
    job.upload(planes)                                    # sizes the planes; content is overwritten below
    got = [np.full_like(p, -1) for p in planes]
    job.upload_coeffs(got)
    job.t1_decode_blocks(table, data)
    job.download_coeffs(got)
    job.close()
    for c, (g, r) in enumerate(zip(got, want)):
        assert np.array_equal(g, r), "component %d: %d coefficients differ" % (c, int((g != r).sum()))
    out = [np.zeros_like(p) for p in planes]
    engine.decode(cp, table, data, out)
    ref = P.inverse(cp, want)
    for g, r in zip(out, ref):
        assert np.array_equal(g, r)
    if not case.get("cs"):
        return
    import torch
    cs = G.codestream_write(cp, table, data)
    dcs = torch.from_numpy(np.array(cs, np.uint8)).cuda()
    _, img = engine.decode_codestream_device(dcs, dtype=torch.int32)
    torch.cuda.synchronize()
    img = img.cpu().numpy()
    for c in range(cp.numcomps):
        assert np.array_equal(img[c], out[c]), "single device code-stream decode, component %d" % c
    _, imgs, status = engine.decode_codestreams_device([dcs, dcs.clone(), dcs.clone()], dtype=torch.int32)
    torch.cuda.synchronize()
    assert [s[0] for s in status] == [0, 0, 0], status
    imgs = imgs.cpu().numpy()
    for i in range(3):
        for c in range(cp.numcomps):
            assert np.array_equal(imgs[i, c], out[c]), "batch slot %d, component %d" % (i, c)


def _one_block_coding(w, h, kmax):
    """a coding whose only code block is w x h (one component, no wavelet level), with band Kmax `kmax` (explicit QCD)"""
    pw = lambda n: max(4, 1 << (int(n) - 1).bit_length())     # noqa: E731
    cp = G.make_coding(w, h, 1, 16, numres=1, cblk=(pw(w), pw(h)))
    cp.qcd_explicit = 1
    cp.qcd_expn[0], cp.qcd_mant[0] = kmax, 0                   # Kmax = exponent + guard bits - 1, one guard bit
    return cp


@pytest.mark.gpu
def test_device_boundary_streams_match_the_reference_verdict(engine, gold):
    """Each boundary block alone in a coding: where the reference decodes it, the device gives its output (Scup = 2 and
    4079, Lcup = Scup, U_q at the limit, 29 missing MSBs); where the reference refuses it (Scup = 4080, U_q one above
    the limit), the engine reports the block rejected (-2) and decodes it as zero, as b2k_decode leaves a rejected
    block.  30 and 31 missing MSBs are checked on the CPU only: the engine refuses a band Kmax above 29, so no block
    table reaches them."""
    L = O.lib()
    tried = 0
    for b in _boundary(gold):
        w, h, mm = b["w"], b["h"], b["mm"]
        if mm > 29:
            continue
        kmax = 29
        cp = _one_block_coding(w, h, kmax)
        assert P.band_params(cp, 0, 0)[0] == kmax
        table = G.enumerate_blocks(cp)
        assert len(table) == 1 and (table[0]["x1"] - table[0]["x0"], table[0]["y1"] - table[0]["y0"]) == (w, h)
        data = np.asarray(b["data"], np.uint8)
        table[0]["length"], table[0]["length2"], table[0]["offset"] = len(data), 0, 0
        table[0]["numbps"], table[0]["numpasses"] = kmax - mm, 1
        want = np.zeros((h, w), np.int32)
        L.orc_ht_post_rev(np.ascontiguousarray(b["dec"]), w, w, h, kmax, want, w)
        job = engine.job(cp)
        job.upload([np.zeros((h, w), np.int32)])
        got = [np.full((h, w), -1, np.int32)]
        job.upload_coeffs(got)
        if b["rc"] == 0:
            job.t1_decode_blocks(table, data)
        else:
            with pytest.raises(G.EngineError, match=r"-2: HT decoder rejected 1 block"):
                job.t1_decode_blocks(table, data)
        job.download_coeffs(got)
        job.close()
        assert np.array_equal(got[0], want), (b["label"], w, h, mm, int((got[0] != want).sum()))
        out = [np.full((h, w), -7, np.int32)]
        if b["rc"] == 0:
            engine.decode(cp, table, data, out)
        else:
            with pytest.raises(G.EngineError, match=r"-2: HT decoder rejected 1 block"):
                engine.decode(cp, table, data, out)
        assert np.array_equal(out[0], P.inverse(cp, [want])[0]), b["label"]
        tried += 1
    assert tried == sum(1 for b in _boundary(gold) if b["mm"] <= 29)


def test_engine_refuses_a_band_kmax_above_29():
    """Why the device boundary test stops at 29 missing MSBs: a band with Kmax 30 is refused before any block decodes."""
    with pytest.raises(G.EngineError):
        G.enumerate_blocks(_one_block_coding(8, 8, 30))
