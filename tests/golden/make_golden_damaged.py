#!/usr/bin/env python3
"""Regenerates tests/golden/ht_damaged.npz from the REFERENCE's own HT decoders (oracle/_ref/libgrok_ref.so, built by
`make -C oracle ref`): single seeded edits of valid HT code blocks, and what the reference makes of each.  Run in the
build container only; the fixture is committed so that a machine without the reference tree checks against it.

Per block shape (64x64, 128x32, 512x8, 1024x4, 4x1024) two valid blocks are coded by the oracle's foreign-choice
encoder: one cleanup-only, one with SigProp (+ MagRef) passes.  Each edit changes one thing (EDITS below): a byte of the
MagSgn, MEL or VLC range, Scup (in range or out of it), Lcup (shorter, down to 1, or longer), the missing-MSB count,
the refinement bytes or their length, more than one pass with no refinement bytes, or 29 missing MSBs with 3 passes.
Two more valid blocks (test_ht_coder_paths.chain_block at 64x64 and 1024x4, whose MagSgn bytes are 0xFF at byte 3 of
every 4) get the top bit of a byte after 0xFF set, where a valid encoder always leaves it 0: after byte 3 of a lane, after
byte 7 (the next lane's first byte) and after byte 255 of a 256-byte refill.  Decoders that OR whole bytes into their
bit buffer put that bit on the next byte's lowest bit.

Layout: meta row [w, h, missing MSBs, passes, Lcup, length2, stripe-causal, verdict, edit] per block, `data` / `data_off`
the bytes (Lcup + length2), `dec` / `dec_off` the reference's words where it accepts the block (empty where it rejects
it).  A block on which the reference's generic and SIMD decoders disagree is left out (the count is printed).
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import oracle_lib as O  # noqa: E402

SHAPES = [(64, 64), (128, 32), (512, 8), (1024, 4), (4, 1024)]
EDITS = ("flip_magsgn", "flip_mel", "flip_vlc", "scup_in_range", "scup_out_of_range", "lcup_shorter", "lcup_longer",
         "numbps", "refine_bytes", "length2", "passes_without_length2", "mmsbs_29_three_passes", "stuffed_top_bit")
PER_BASE = 30


def ref_verdict(data, mm, w, h, npass, len2, causal):
    """(verdict, words) of the reference, or None where its decoders disagree"""
    outs = [O.ref_ht_decode(data, mm, w, h, variant=v, num_passes=npass, len2=len2, causal=causal) for v in (0, 1, 2)]
    outs = [o for o in outs if o[0] != -2]
    if any(o[0] != outs[0][0] for o in outs):
        return None
    if outs[0][0] == 0 and not all(np.array_equal(outs[0][1], o[1]) for o in outs):
        return None
    return outs[0]


def base_blocks(w, h, rng):
    """(cleanup-only block, refined block): dicts of data, lcup, len2, mm, npass, causal, ms_len, mel_len"""
    out = []
    for refined in (False, True):
        kmax = 12
        lim = (1 << kmax) - 1
        dense = 0.6 if (w, h, refined) == (64, 64, False) else 0.15   # one block long enough for Scup above 4079
        mag = rng.integers(0, lim + 1, (h, w)).astype(np.uint64) * (rng.random((h, w)) < dense)
        v = (mag << np.uint64(31 - kmax)).astype(np.uint32)
        sm = np.where(v != 0, v | (rng.integers(0, 2, (h, w)).astype(np.uint32) << 31), 0).astype(np.uint32)
        mm = kmax - 1 - (1 if refined else 0)
        choices = int(rng.integers(1, 16))            # no padding between MEL and VLC: the ranges below stay exact
        cup, st = O.ht_encode_foreign(sm, mm, choices, int(rng.integers(1, 1 << 30)), cap=65536, stats=True)
        npass = 3 if (w + h) % 3 else 2
        causal = bool((w // 4) % 2)
        seg = O.ht_encode_refine(sm, mm, npass, causal) if refined else np.zeros(0, np.uint8)
        scup = (int(cup[-1]) << 4) | (int(cup[-2]) & 0xF)
        out.append(dict(data=np.concatenate([cup, seg]), lcup=len(cup), len2=len(seg), mm=mm,
                        npass=npass if refined else 1, causal=causal, ms_len=len(cup) - scup, mel_len=st[3]))
    return out


def edit(b, kind, rng):
    """one edit of base block b: (data, lcup, len2, mm, npass), or None where the edit does not apply"""
    d = b["data"].copy()
    lcup, len2, mm, npass = b["lcup"], b["len2"], b["mm"], b["npass"]
    ms, mel = b["ms_len"], b["mel_len"]
    ranges = {"flip_magsgn": (0, ms), "flip_mel": (ms, ms + mel), "flip_vlc": (ms + mel, lcup - 2)}
    if kind in ranges:
        lo, hi = ranges[kind]
        if hi <= lo:
            return None
        i = int(rng.integers(lo, hi))
        d[i] ^= np.uint8(rng.integers(1, 256))
    elif kind in ("scup_in_range", "scup_out_of_range"):
        if kind == "scup_in_range":
            s = int(rng.integers(2, min(lcup, 4079) + 1))
        else:
            opts = [0, 1] + ([int(rng.integers(lcup + 1, 4096))] if lcup < 4095 else []) + \
                   ([int(rng.integers(4080, min(lcup, 4095) + 1))] if lcup >= 4080 else [])
            s = opts[int(rng.integers(0, len(opts)))]
        d[lcup - 1] = s >> 4
        d[lcup - 2] = (int(d[lcup - 2]) & 0xF0) | (s & 0xF)
    elif kind == "lcup_shorter":
        k = lcup - 1 if rng.random() < 0.15 else int(rng.integers(1, min(lcup - 1, 24) + 1))
        lcup -= k
        d = np.concatenate([d[:lcup], d[lcup + k:]])
    elif kind == "lcup_longer":
        k = int(rng.integers(1, 24))
        d = np.concatenate([d[:lcup], rng.integers(0, 256, k).astype(np.uint8), d[lcup:]])
        lcup += k
    elif kind == "numbps":
        m = mm + int(rng.choice([-3, -2, -1, 1, 2, 3]))
        if not 0 <= m <= 29:
            return None
        mm = m
    elif kind == "refine_bytes":
        if not len2:
            return None
        d[lcup:] = rng.integers(0, 256, len2).astype(np.uint8)
    elif kind == "length2":
        if not len2:
            return None
        k = int(rng.integers(1, len2 + 8))
        if rng.random() < 0.5 and k < len2:
            len2 -= k
            d = d[:lcup + len2]
        else:
            d = np.concatenate([d, rng.integers(0, 256, k).astype(np.uint8)])
            len2 += k
    elif kind == "passes_without_length2":
        d, len2, npass = d[:lcup], 0, int(rng.integers(2, 4))
    elif kind == "mmsbs_29_three_passes":
        if not len2:
            return None
        mm, npass = 29, 3
    return d, lcup, len2, mm, npass


def stuffed_top_bit_blocks(rng):
    """(w, h, mm, data) of chain blocks with the top bit set in bytes that follow 0xFF in the MagSgn segment: one edit
    per position class (byte 4 of a lane, a lane's first byte, a refill's first byte), then one with all three"""
    import test_ht_coder_paths as CP
    out = []
    for label in ("chain-64x64-packed", "chain-1024x4"):
        coef, _, kmax = CP.chain_case(label)
        h, w = coef.shape
        d = O.ht_encode(O.to_sgnmag(coef, kmax), kmax, cap=65536)
        ms = len(d) - ((int(d[-1]) << 4) | (int(d[-2]) & 0xF))
        picks = []
        for cls in (lambda i: i % 8 == 4, lambda i: i % 8 == 0 and i % 256, lambda i: i % 256 == 0):
            cand = [i for i in range(1, min(ms, 2048)) if cls(i) and d[i - 1] == 0xFF and d[i] < 0x80]
            picks.append(cand[int(rng.integers(0, len(cand)))])
        for sel in [[p] for p in picks] + [picks]:
            e = d.copy()
            for i in sel:
                e[i] |= 0x80
            out.append((w, h, kmax, e))
    return out


def main():
    assert O.ref() is not None, "build oracle/_ref first (make -C oracle ref)"
    rng = np.random.default_rng(20261018)
    meta, datas, decs = [], [], []
    left_out = 0
    for w, h in SHAPES:
        for b in base_blocks(w, h, rng):
            made = 0
            while made < PER_BASE:
                edits = EDITS[:-1]                      # the last applies to the chain blocks only
                kind = edits[made % len(edits)] if made < len(edits) else edits[int(rng.integers(0, len(edits)))]
                e = edit(b, kind, rng)
                if e is None:
                    e = edit(b, "flip_magsgn" if made % 2 else "flip_vlc", rng)
                    kind = None
                d, lcup, len2, mm, npass = e
                kind = EDITS.index(kind) if kind else (0 if made % 2 else 2)
                made += 1
                r = ref_verdict(d, mm, w, h, npass, len2, b["causal"])
                if r is None:
                    left_out += 1
                    continue
                rc, dec = r
                meta.append([w, h, mm, npass, lcup, len2, int(b["causal"]), 0 if rc == 0 else -1, kind])
                datas.append(d)
                decs.append(dec.ravel() if rc == 0 else np.zeros(0, np.uint32))
    for w, h, mm, d in stuffed_top_bit_blocks(rng):
        r = ref_verdict(d, mm, w, h, 1, 0, False)
        if r is None:
            left_out += 1
            continue
        rc, dec = r
        meta.append([w, h, mm, 1, len(d), 0, 0, 0 if rc == 0 else -1, EDITS.index("stuffed_top_bit")])
        datas.append(d)
        decs.append(dec.ravel() if rc == 0 else np.zeros(0, np.uint32))
    out = {"meta": np.array(meta, np.int64)}
    for name, parts in (("data", datas), ("dec", decs)):
        out[name] = np.concatenate(parts)
        out[name + "_off"] = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.int64)
    np.savez_compressed(os.path.join(HERE, "ht_damaged.npz"), **out)
    m = out["meta"]
    print("wrote %d damaged blocks (%d rejected by the reference); left out %d on which its decoders disagree"
          % (len(m), int((m[:, 7] != 0).sum()), left_out))


if __name__ == "__main__":
    main()
