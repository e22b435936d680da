#!/usr/bin/env python3
"""Regenerates tests/golden/ht_blocks_wide.npz from the REFERENCE's own HT kernels (oracle/_ref/libgrok_ref.so, built by
`make -C oracle ref`): the bit-plane range above the one ht_blocks.npz covers, Kmax 19..29, where the 32-bit HT coder's
MagSgn words are widest.  Run in the build container only; the fixture is committed so that a machine without the
reference tree checks against it.

  cleanup blocks : sign-magnitude code blocks (random, full-scale checkerboards +-(2^Kmax - 1), a single isolated
                   maximum, all zero) + the bytes ojph_encode_codeblock{32,_avx2,_avx512} produce for them (all variants
                   agree; asserted here) + what ojph_decode_codeblock32 returns for those bytes.
  refined blocks : Kmax 25..29, cleanup pass 1 or 2 planes above the LSB plus SigProp (+ MagRef) from the oracle's
                   test-only refinement encoder (the reference encoder writes no refinement passes), plain and
                   stripe-causal, with what the reference decoders (all variants agree) make of them.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import oracle_lib as O  # noqa: E402

SMALL = [(4, 4), (33, 17), (5, 3), (1, 1), (2, 9), (16, 16)]
LARGE = [(64, 64), (1024, 4), (4, 1024)]
# the few large random blocks: (shape, Kmax, kind); the large shapes otherwise see the kinds that compress well
LARGE_RANDOM = [((64, 64), 29, "noise"), ((1024, 4), 25, "noise"), ((64, 64), 25, "top"), ((4, 1024), 29, "top")]


def block(kind, kmax, w, h, rng):
    lim = (1 << kmax) - 1
    if kind == "noise":
        return rng.integers(-lim, lim + 1, (h, w))
    if kind == "checker":
        return np.where((np.add.outer(np.arange(h), np.arange(w)) & 1) == 0, lim, -lim)
    if kind == "top":          # every sample in the top plane, signs random
        return rng.integers(1 << (kmax - 1), lim + 1, (h, w)) * rng.choice([-1, 1], (h, w))
    if kind == "impulse":
        c = np.zeros((h, w), np.int64)
        c[int(rng.integers(0, h)), int(rng.integers(0, w))] = lim * int(rng.choice([-1, 1]))
        return c
    return np.zeros((h, w), np.int64)


def main():
    assert O.ref() is not None, "build oracle/_ref first (make -C oracle ref)"
    rng = np.random.default_rng(20261015)
    out = {}
    n = 0
    cases = [((w, h), kmax, ("noise", "checker", "top", "impulse", "zero")[(i + kmax) % 5])
             for i, (w, h) in enumerate(SMALL) for kmax in range(19, 30)]
    cases += [(shape, kmax, kind) for shape in LARGE for kmax in (19, 24, 25, 29) for kind in ("checker", "impulse", "zero")]
    cases += LARGE_RANDOM
    for (w, h), kmax, kind in cases:
        sm = O.to_sgnmag(block(kind, kmax, w, h, rng), kmax)
        outs = [o for o in (O.ref_ht_encode(sm, kmax, v) for v in (0, 1, 2)) if o is not None]
        assert all(np.array_equal(outs[0], o) for o in outs), "reference encoder variants disagree"
        rc, dec = O.ref_ht_decode(outs[0], kmax, w, h, 0)
        assert rc == 0
        out["in%03d" % n], out["kmax%03d" % n], out["out%03d" % n], out["dec%03d" % n] = sm, np.int32(kmax), outs[0], dec
        n += 1
    out["count"] = np.int32(n)
    m = 0
    for (w, h) in SMALL[:4] + LARGE[:2]:
        for kmax in (range(25, 30) if (w, h) in SMALL else (29,)):
            for dropped in (1, 2):
                M = kmax - 1 - dropped                  # missing MSBs of the cleanup pass (decoder-aligned words)
                lim = (1 << kmax) - 1
                mag = rng.integers(0, lim + 1, (h, w)).astype(np.uint64) * (rng.random((h, w)) < (0.3, 1.0)[dropped - 1])
                mag[0, 0] = lim
                v = (mag << np.uint64(31 - kmax)).astype(np.uint32)
                sm = np.where(v != 0, v | (rng.integers(0, 2, (h, w)).astype(np.uint32) << 31), 0).astype(np.uint32)
                cup = O.ref_ht_encode(sm, M, 0)
                for causal in (False, True):
                    npass = 3 if (kmax + dropped) % 2 else 2
                    seg = O.ht_encode_refine(sm, M, npass, causal)
                    data = np.concatenate([cup, seg])
                    decs = [O.ref_ht_decode(data, M, w, h, variant=vv, num_passes=npass, len2=len(seg), causal=causal)
                            for vv in (0, 1, 2)]
                    decs = [d for d in decs if d[0] != -2]
                    assert all(rc == 0 for rc, _ in decs)
                    assert all(np.array_equal(decs[0][1], d) for _, d in decs), "reference decoder variants disagree"
                    out["rdata%03d" % m] = data
                    out["rmeta%03d" % m] = np.array([w, h, M, npass, len(seg), int(causal), kmax], np.int32)
                    out["rsrc%03d" % m] = sm
                    out["rdec%03d" % m] = decs[0][1]
                    m += 1
    out["rcount"] = np.int32(m)
    np.savez_compressed(os.path.join(HERE, "ht_blocks_wide.npz"), **out)
    print("wrote", n, "cleanup blocks and", m, "refined blocks at Kmax 19..29")


if __name__ == "__main__":
    main()
