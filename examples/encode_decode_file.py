#!/usr/bin/env python3
"""Encode an image to an HTJ2K file on the GPU and read it back (needs an H100; uses only the public API).

  python examples/encode_decode_file.py in.ppm out.jph [--lossy] [--tile 1024]      # PGM / PPM (8 or 16 bit) in, .jph or .j2c out
  python examples/encode_decode_file.py --decode in.jph out.ppm

The same calls from C: b2k_encode + b2k_codestream_write (+ b2k_jph_wrap), b2k_jph_codestream + b2k_codestream_parse +
b2k_decode (include/grok_b200.h, INTEGRATION.md section 3)."""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import grok_b200 as G  # noqa: E402


def read_pnm(path):
    with open(path, "rb") as f:
        data = f.read()
    tok, pos = [], 0
    while len(tok) < 4:                                   # magic, width, height, maxval (comments allowed)
        while data[pos:pos + 1].isspace():
            pos += 1
        if data[pos:pos + 1] == b"#":
            pos = data.index(b"\n", pos) + 1
            continue
        end = pos
        while not data[end:end + 1].isspace():
            end += 1
        tok.append(data[pos:end])
        pos = end
    pos += 1
    magic, w, h, maxval = tok[0], int(tok[1]), int(tok[2]), int(tok[3])
    nc = {b"P5": 1, b"P6": 3}[magic]
    dt = np.dtype(">u2") if maxval > 255 else np.uint8
    a = np.frombuffer(data, dt, w * h * nc, pos).reshape(h, w, nc).astype(np.int32)
    return [np.ascontiguousarray(a[:, :, c]) for c in range(nc)], maxval.bit_length()


def write_pnm(path, planes, prec):
    a = np.stack(planes, axis=-1)
    with open(path, "wb") as f:
        f.write(b"%s\n%d %d\n%d\n" % (b"P5" if len(planes) == 1 else b"P6", a.shape[1], a.shape[0], (1 << prec) - 1))
        f.write(a.astype(">u2" if prec > 8 else np.uint8).tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("src")
    ap.add_argument("dst")
    ap.add_argument("--decode", action="store_true")
    ap.add_argument("--lossy", action="store_true", help="9/7 + ICT with the HT quantiser's step sizes instead of lossless 5/3 + RCT")
    ap.add_argument("--qfactor", type=int, default=0,
                    help="1..100: lossy 9/7 + ICT at a JPEG-style quality factor (grk_compress --qfactor's step sizes)")
    ap.add_argument("--tile", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args()
    eng = G.Engine(a.device)
    if a.decode:
        cs = G.jph_codestream(np.fromfile(a.src, np.uint8))
        cp, planes = eng.decode_codestream(cs)
        write_pnm(a.dst, planes, cp.prec)
        print("decoded %dx%dx%d, %d bit" % (cp.x1 - cp.x0, cp.y1 - cp.y0, cp.numcomps, cp.prec))
        return
    planes, prec = read_pnm(a.src)
    h, w = planes[0].shape
    cp = G.make_coding(w, h, len(planes), prec, numres=6 if min(w, h) >= 64 else 2, irreversible=a.lossy or a.qfactor > 0,
                       tile=(a.tile, a.tile) if a.tile else None, qfactor=a.qfactor or None)
    cs = eng.encode_codestream(cp, planes)
    out = G.jph_wrap(cp, cs) if a.dst.endswith(".jph") else cs
    out.tofile(a.dst)
    _, back = eng.decode_codestream(cs)
    err = max(int(np.abs(x - y).max()) for x, y in zip(back, planes))
    print("%s: %d bytes, %.3f bpp; round trip max error %d" % (a.dst, len(out), 8.0 * len(out) / (w * h), err))


if __name__ == "__main__":
    main()
