#!/usr/bin/env python3
"""Regenerates tests/golden/ht_foreign.npz from the REFERENCE's own HT decoders (oracle/_ref/libgrok_ref.so, built by
`make -C oracle ref`): HT cleanup segments written with the choices T.814 leaves to an encoder, as other HTJ2K encoders
make them and this project's coders never do.  Run in the build container only; the fixture is committed so that a
machine without the reference tree checks against it.

Layout: see pack().

  foreign blocks  : sign-magnitude blocks 1x1 .. 1024x4 / 4x1024 (widths above 64 included), Kmax 2..29, coded by the
                    oracle's orc_ht_encode_foreign with each choice alone and all of them together, + what
                    ojph_decode_codeblock32 and its SIMD variants (all agree; asserted here) return for those bytes.
  refined blocks  : a foreign cleanup segment 1 or 2 planes above the LSB + SigProp (+ MagRef) from the oracle's
                    refinement encoder, plain and stripe-causal, with the reference decoders' output.
  boundary blocks : streams edited byte by byte from known ones -- Scup = 2, Scup = 4079 and one more, Lcup = Scup,
                    U_q at the decoder's limit and one above it, missing MSBs at 29 (the largest the reference decodes)
                    and beyond -- with the reference's verdict and, where it accepts, its output.

Every choice the encoder offers is in the lists below: the reference decoders accept each of them and return the
source's bin-centre values (asserted here).  Padding bytes are kept below 0x80, so that no byte pair in a segment reads
as a marker code.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as O  # noqa: E402

CHOICES = [O.FOREIGN_ROWS, O.FOREIGN_RAISE_U, O.FOREIGN_NO_FUSE, O.FOREIGN_PAD_MAGSGN, O.FOREIGN_PAD_SCUP, O.FOREIGN_ALL]
SMALL = [(1, 1), (2, 1), (1, 3), (3, 2), (4, 4), (5, 7), (17, 9), (33, 17), (16, 16)]
LARGE = [(64, 64), (65, 8), (100, 4), (128, 32), (1024, 4), (4, 1024)]
KINDS = ("sparse", "noise", "smooth", "top")


def block(kind, kmax, w, h, rng):
    lim = (1 << kmax) - 1
    if kind == "noise":
        mag = rng.integers(0, lim + 1, (h, w))
    elif kind == "sparse":
        mag = rng.integers(0, lim + 1, (h, w)) * (rng.random((h, w)) < (0.15 if w * h <= 1024 else 0.04))
    elif kind == "smooth":         # a ramp: neighbours of similar size, exponents that predict each other
        mag = (np.add.outer(np.arange(h) * 3, np.arange(w)) * max(1, lim // (3 * h + w))) & lim
    else:                          # every sample in the top plane
        mag = rng.integers(1 << (kmax - 1), lim + 1, (h, w))
    return (mag * rng.choice([-1, 1], (h, w))).astype(np.int64)


def bin_centre(sm, mm):
    """what a decoder returns for words coded with `mm` missing MSBs: sign | (2 mu + 1) << (29 - mm)"""
    mu = ((sm & 0x7FFFFFFF) >> (30 - mm)).astype(np.uint64)
    return np.where(mu > 0, (sm & 0x80000000) | ((2 * mu + 1) << np.uint64(29 - mm)), 0).astype(np.uint32)


def ref_decode(data, mm, w, h, npass=1, len2=0, causal=False):
    """the reference's verdict and output; every SIMD variant built must agree with the generic decoder"""
    outs = [O.ref_ht_decode(data, mm, w, h, variant=v, num_passes=npass, len2=len2, causal=causal) for v in (0, 1, 2)]
    outs = [o for o in outs if o[0] != -2]
    assert all(o[0] == outs[0][0] for o in outs), "reference decoder variants disagree on the verdict"
    if outs[0][0] == 0:
        assert all(np.array_equal(outs[0][1], o[1]) for o in outs), "reference decoder variants disagree"
        return 0, outs[0][1]
    return -1, np.zeros((h, w), np.uint32)


def with_scup(data, scup_old, mel_len, extra, rng):
    """`data` with `extra` bytes below 0x80 put between its MEL and VLC bytes, and Scup rewritten"""
    lcup = len(data)
    at = lcup - scup_old + mel_len
    pad = rng.integers(0, 0x80, extra).astype(np.uint8)
    d = np.concatenate([data[:at], pad, data[at:]])
    scup = scup_old + extra
    d[-1] = scup >> 4
    d[-2] = (d[-2] & 0xF0) | (scup & 0xF)
    return d


def pack(out, prefix, recs):
    """a group of blocks as few arrays: <prefix>meta (one row per block) and, per named array, <prefix><name> (every
    block's array, flattened and concatenated) with <prefix><name>_off (block i's is [off[i], off[i + 1])).  A decode is
    kept as dec_x = decode ^ source words (the decode itself where a block has no source): the same words, which
    compress to almost nothing where the decode is the source's bin centre"""
    out[prefix + "meta"] = np.array([r[0] for r in recs], np.int64)
    for name in recs[0][1]:
        parts = [np.ravel(r[1][name]) for r in recs]
        out[prefix + name] = np.concatenate(parts)
        out[prefix + name + "_off"] = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)


def scup_of(data):
    return (int(data[-1]) << 4) | (int(data[-2]) & 0xF)


def main():
    assert O.ref() is not None, "build oracle/_ref first (make -C oracle ref)"
    rng = np.random.default_rng(20261017)
    out = {}

    # ---- foreign cleanup blocks ----
    cases = []
    for i, (w, h) in enumerate(SMALL):
        for kmax in (range(2, 30) if w * h <= 64 else (2, 5, 8, 11, 14, 17, 20, 23, 26, 29)):
            cases.append(((w, h), kmax, KINDS[(i + kmax) % 4], CHOICES[(i + kmax) % len(CHOICES)]))
    for i, (w, h) in enumerate(LARGE):          # two choice sets per Kmax: every set reaches every large shape
        for j, kmax in enumerate((3, 11, 20, 29)):
            for c in (CHOICES[(i + j) % 6], CHOICES[(i + j + 3) % 6]):
                kind = ("sparse", "smooth")[(i + j) % 2] if kmax > 3 else KINDS[(i + j + c) % 4]
                cases.append(((w, h), kmax, kind, c))
    recs = []
    for n, ((w, h), kmax, kind, choices) in enumerate(cases):
        sm = O.to_sgnmag(block(kind, kmax, w, h, rng), kmax)
        seed = 1000 + n
        data = O.ht_encode_foreign(sm, kmax, choices, seed, cap=65536)
        rc, dec = ref_decode(data, kmax, w, h)
        assert rc == 0 and np.array_equal(dec, bin_centre(sm, kmax)), (w, h, kmax, choices)
        recs.append(([w, h, kmax, choices, seed], dict(src=sm, data=data, dec_x=dec ^ sm)))
    pack(out, "", recs)

    # ---- refinement passes on a foreign cleanup segment ----
    m = 0
    recs = []
    for (w, h), kmaxes in [((4, 4), (7, 18, 27)), ((5, 3), (7, 18, 27)), ((33, 17), (7, 18, 27)), ((64, 64), (7, 18)),
                           ((1024, 4), (7, 27)), ((4, 1024), (7, 18))]:
        for kmax in kmaxes:
            for dropped in (1, 2):
                M = kmax - 1 - dropped                  # missing MSBs of the cleanup pass (decoder-aligned words)
                lim = (1 << kmax) - 1
                dense = (0.3, 1.0)[dropped - 1] if w * h <= 1024 else (0.05, 0.2)[dropped - 1]
                mag = rng.integers(0, lim + 1, (h, w)).astype(np.uint64) * (rng.random((h, w)) < dense)
                mag[0, 0] = lim
                v = (mag << np.uint64(31 - kmax)).astype(np.uint32)
                sm = np.where(v != 0, v | (rng.integers(0, 2, (h, w)).astype(np.uint32) << 31), 0).astype(np.uint32)
                for causal in (False, True):
                    choices = CHOICES[m % len(CHOICES)]
                    seed = 5000 + m
                    cup = O.ht_encode_foreign(sm, M, choices, seed, cap=65536)
                    npass = 3 if (kmax + dropped + int(causal)) % 2 else 2
                    seg = O.ht_encode_refine(sm, M, npass, causal)
                    data = np.concatenate([cup, seg])
                    rc, dec = ref_decode(data, M, w, h, npass, len(seg), causal)
                    assert rc == 0
                    recs.append(([w, h, M, npass, len(seg), int(causal), kmax, choices, seed], dict(src=sm, data=data, dec_x=dec ^ sm)))
                    m += 1
    pack(out, "r", recs)

    # ---- boundary blocks, each made by editing the bytes (or the missing-MSB count) of a known stream ----
    bnd = []   # (label, data, w, h, mm, source words or None)

    def add(label, data, w, h, mm, src=None):
        bnd.append((label, np.asarray(data, np.uint8), w, h, mm, src))

    # Lcup = Scup: an all-zero block has no MagSgn bytes
    for (w, h) in [(1, 1), (4, 4), (64, 64), (1024, 4), (4, 1024)]:
        z = np.zeros((h, w), np.uint32)
        d = O.ht_encode(z, 9)
        assert scup_of(d) == len(d)
        add("lcup_eq_scup", d, w, h, 9, z)
        d, st = O.ht_encode_foreign(z, 9, O.FOREIGN_NO_FUSE, 1, stats=True)
        add("lcup_eq_scup", with_scup(d, scup_of(d), st[3], 5, rng), w, h, 9, z)
    # Scup = 2: the two Scup bytes are all the MEL and VLC there is; the high nibble of the first is read by both
    for (w, h) in [(1, 1), (8, 8), (64, 64), (1024, 4)]:
        z = np.zeros((h, w), np.uint32)
        add("scup_2", [0xF2, 0x00], w, h, 9, z)
        add("scup_2", [0x35, 0x11, 0xF2, 0x00], w, h, 9, z)
    sm = O.to_sgnmag(np.array([[5, -3], [0, 7]]), 6)
    plain = O.ht_encode(sm, 6)
    for nib in range(16):                            # a MagSgn segment of a known 2x2 block, then every 2-byte MEL + VLC
        add("scup_2_nibble", np.concatenate([plain[:len(plain) - scup_of(plain)], [(nib << 4) | 2, 0]]), 2, 2, 6)
    # Scup = 4079 (the largest) and 4080: padding put between the MEL and the VLC bytes of known streams
    for (w, h), kmax, kind in [((64, 64), 12, "noise"), ((1024, 4), 20, "sparse"), ((4, 4), 5, "noise"), ((3, 2), 29, "top")]:
        sm = O.to_sgnmag(block(kind, kmax, w, h, rng), kmax)
        d, st = O.ht_encode_foreign(sm, kmax, O.FOREIGN_NO_FUSE, 7, stats=True)
        s0 = scup_of(d)
        add("scup_4079", with_scup(d, s0, st[3], 4079 - s0, rng), w, h, kmax, sm)
        add("scup_4080", with_scup(d, s0, st[3], 4080 - s0, rng), w, h, kmax, sm)
    # U_q at the decoder's limit (missing MSBs + 2), and the same bytes read with one missing MSB less: one above it
    for (w, h), kmax in [((32, 8), 4), ((16, 16), 9), ((64, 64), 17), ((100, 4), 24), ((32, 32), 29)]:
        src = O.to_sgnmag(block("sparse", kmax, w, h, rng), kmax)
        for seed in range(1, 400):
            d, st = O.ht_encode_foreign(src, kmax, O.FOREIGN_RAISE_U, seed, stats=True, cap=65536)
            if st[0] > 0:
                break
        assert st[0] > 0, "no quad reached the limit"
        add("u_at_limit", d, w, h, kmax, src)
        add("u_above_limit", d, w, h, kmax - 1)
    # missing MSBs: 29 is the most the reference decodes (p = 1); 30 and 31 are refused
    src = O.to_sgnmag(block("noise", 29, 6, 5, rng), 29)
    d = O.ht_encode(src, 29)
    add("mmsbs_29", d, 6, 5, 29, src)
    add("mmsbs_30", d, 6, 5, 30)
    add("mmsbs_31", d, 6, 5, 31)

    recs = []
    for label, data, w, h, mm, src in bnd:
        rc, dec = ref_decode(data, mm, w, h)
        if src is not None and rc == 0:
            assert np.array_equal(dec, bin_centre(src, mm)), label
        recs.append(([w, h, mm, rc], dict(src=src if src is not None else np.zeros(0, np.uint32), data=data,
                                          dec_x=dec ^ src if src is not None else dec)))
    pack(out, "b", recs)
    out["blabel"] = np.array([b[0] for b in bnd])
    np.savez_compressed(os.path.join(HERE, "ht_foreign.npz"), **out)
    print("wrote", len(cases), "foreign cleanup blocks,", m, "refined blocks and", len(bnd), "boundary blocks")


if __name__ == "__main__":
    main()
