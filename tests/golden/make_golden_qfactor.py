#!/usr/bin/env python3
"""Regenerates tests/golden/qfactor.npz from the REFERENCE's grk_compress (oracle/_ref/grok/bin, built by build()):
what `grk_compress -I --qfactor Q` writes for an HTJ2K (.jph) output.  Run where the reference was built; the record is
committed so that a machine without it checks against it.

  tables  : for qfactor 1..100 x precision {8, 10, 12, 16} x resolutions {1, 2, 6, 8} x {1, 3} components (-N 4, so that
            no band is left without bit planes), the main header from CAP to the last QCC -- CAP, COD, QCD and the QCCs.
  streams : whole code streams (COM removed) of seeded images (oracle_pipeline.synthetic_image) for the cases in
            STREAMS: their SHA-256 and length.
  verdict : for qfactor 20..50 at one guard bit (8-bit, 6 resolutions), whether grk_compress writes a stream (1) or
            refuses it (0: a band with Kmax 0, "exceeding band maximum").
  decoded : grk_decompress's pixels of its own streams for DECODED (which ours equal byte for byte).
"""
import hashlib
import os
import sys
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import grok_ref as R  # noqa: E402
import oracle_pipeline as P  # noqa: E402

QFACTORS = list(range(1, 101))
PRECS = (8, 10, 12, 16)
NUMRES = (1, 2, 6, 8)
NCOMPS = (1, 3)
# (name, width, height, ncomp, prec, numres, qfactor, guard bits, tile, origin, tlm+plt, progression, seed)
STREAMS = [
    ("q50", 200, 136, 3, 8, 6, 50, 0, None, (0, 0), False, "LRCP", 1),
    ("q60_tiled", 256, 192, 3, 10, 6, 60, 0, (128, 128), (0, 0), True, "LRCP", 2),
    ("q75_rpcl", 160, 160, 3, 12, 5, 75, 0, (96, 64), (0, 0), True, "RPCL", 3),
    ("q90_origin", 150, 130, 3, 8, 4, 90, 0, (64, 64), (17, 9), True, "LRCP", 4),
    ("q97_grey", 128, 96, 1, 16, 6, 97, 0, None, (0, 0), False, "LRCP", 5),
    ("q100", 96, 80, 3, 12, 3, 100, 0, None, (0, 0), True, "RPCL", 6),
    ("q30_N2", 128, 128, 3, 8, 6, 30, 2, (64, 64), (0, 0), True, "LRCP", 7),
    ("q10_N4", 120, 100, 1, 12, 6, 10, 4, None, (3, 5), False, "LRCP", 8),
    ("q80_signed", 128, 96, 3, 8, 5, 80, 0, None, (0, 0), True, "LRCP", 9),
]
SIGNED = {"q80_signed"}
DECODED = ("q50", "q90_origin", "q80_signed")
VERDICT_Q = list(range(20, 51))


def signed(planes, prec):
    return [p - (1 << (prec - 1)) for p in planes]


def write_pnm(path, planes, prec):
    h, w = planes[0].shape
    img = np.stack(planes, axis=-1) if len(planes) == 3 else planes[0]
    maxval = (1 << prec) - 1
    data = img.astype(">u2" if prec > 8 else "u1").tobytes()
    with open(path, "wb") as f:
        f.write(b"%s\n%d %d\n%d\n" % (b"P6" if len(planes) == 3 else b"P5", w, h, maxval) + data)


def compress(planes, prec, qfactor, numres, guard=0, tile=None, origin=(0, 0), tlm=False, prog="LRCP", sgnd=False):
    """grk_compress's code stream (bytes), or None when it refuses.  Signed samples (8-bit only) go in as raw"""
    with tempfile.TemporaryDirectory() as d:
        src, dst = os.path.join(d, "in.raw" if sgnd else "in.pnm"), os.path.join(d, "out.jph")
        args = ["-i", src, "-o", dst, "-I", "--qfactor", str(qfactor), "-n", str(numres), "-p", prog]
        if sgnd:
            assert prec == 8
            h, w = planes[0].shape
            np.stack(planes).astype(np.int8).tofile(src)
            args += ["-F", "%d,%d,%d,%d,s" % (w, h, len(planes), prec)]
        else:
            write_pnm(src, planes, prec)
        if guard:
            args += ["-N", str(guard)]
        if tile:
            args += ["-t", "%d,%d" % tile]
        if origin != (0, 0):
            args += ["-d", "%d,%d" % origin]
        if tlm:
            args += ["-X", "-L"]
        r = R.run_cli("grk_compress", args, timeout=120)
        if r.returncode != 0 or not os.path.exists(dst):
            return None
        with open(dst, "rb") as f:
            jph = f.read()
    return jph[jph.index(b"\xff\x4f\xff\x51"):]


def strip_com(cs):
    i = cs.find(b"\xff\x64")
    while i >= 0 and i < cs.find(b"\xff\x90"):
        n = int.from_bytes(cs[i + 2:i + 4], "big")
        cs = cs[:i] + cs[i + 2 + n:]
        i = cs.find(b"\xff\x64")
    return cs


def quant_segments(cs):
    """CAP .. the last QCC of a main header"""
    a = cs.index(b"\xff\x50")
    p = a
    while True:
        m = cs[p:p + 2]
        if m not in (b"\xff\x50", b"\xff\x52", b"\xff\x5c", b"\xff\x5d"):
            return cs[a:p]
        p += 2 + int.from_bytes(cs[p + 2:p + 4], "big")


def table_case(args):
    q, prec, numres, ncomp = args
    size = 1 << max(3, numres)
    planes = P.synthetic_image(size, size, ncomp, prec, seed=q)
    cs = compress(planes, prec, q, numres, guard=4)
    assert cs is not None, args
    return quant_segments(cs)


def main():
    assert R.available(), "build the reference first (build())"
    cases = [(q, p, n, c) for q in QFACTORS for p in PRECS for n in NUMRES for c in NCOMPS]
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        segs = list(ex.map(table_case, cases))
    streams, decoded = [], {}
    for name, w, h, nc, prec, numres, q, guard, tile, origin, tlm, prog, seed in STREAMS:
        planes = P.synthetic_image(w, h, nc, prec, seed=seed, origin=origin)
        if name in SIGNED:
            planes = signed(planes, prec)
        cs = compress(planes, prec, q, numres, guard, tile, origin, tlm, prog, sgnd=name in SIGNED)
        assert cs is not None, name
        cs = strip_com(cs)
        streams.append((name, hashlib.sha256(cs).hexdigest(), len(cs)))
        print(name, len(cs))
        if name in DECODED:
            with tempfile.TemporaryDirectory() as d:
                src, dst = os.path.join(d, "in.j2k"), os.path.join(d, "out.raw")
                with open(src, "wb") as f:
                    f.write(cs)
                r = R.run_cli("grk_decompress", ["-i", src, "-o", dst], timeout=120)
                assert r.returncode == 0, r.stdout
                decoded["decoded_" + name] = np.fromfile(dst, np.int8 if name in SIGNED else (">u2" if prec > 8 else np.uint8)).reshape(nc, h, w)
    planes = P.synthetic_image(64, 64, 3, 8, seed=0)
    verdict = [int(compress(planes, 8, q, 6, 1) is not None) for q in VERDICT_Q]
    print("accepted at one guard bit:", [q for q, v in zip(VERDICT_Q, verdict) if v])
    lens = np.array([len(s) for s in segs], np.int64)
    np.savez_compressed(os.path.join(HERE, "qfactor.npz"), cases=np.array(cases, np.int32),
                        seg_len=lens, seg_bytes=np.frombuffer(b"".join(segs), np.uint8),
                        stream_names=np.array([s[0] for s in streams]), stream_sha=np.array([s[1] for s in streams]),
                        stream_len=np.array([s[2] for s in streams], np.int64),
                        verdict_q=np.array(VERDICT_Q, np.int32), verdict=np.array(verdict, np.int32), **decoded)


if __name__ == "__main__":
    main()
