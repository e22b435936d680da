"""Runs in a SUBPROCESS of tests/test_codestream.py (a crash must not take pytest down): mutated code streams and JPH files
through b2k_codestream_parse_window / b2k_jph_codestream.  Every call has to come back -- an error (< 0), "not handled" (1)
or a block table whose byte ranges lie inside the buffer -- and a block count has to stay in proportion to the input.

usage: python fuzz_parser_driver.py SEED ROUNDS [path of an alternative (sanitised) library]"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), HERE]
import grok_b200 as G           # noqa: E402
import oracle_pipeline as P     # noqa: E402
from test_interop import oracle_encode   # noqa: E402


def main():
    seed, rounds = int(sys.argv[1]), int(sys.argv[2])
    if len(sys.argv) > 3:
        G.LIB_PATH = sys.argv[3]
    L = G.lib()
    rng = np.random.default_rng(seed)

    def parse(buf, win, reduce):
        raw = (C.c_uint8 * max(1, len(buf))).from_buffer_copy(buf.tobytes() if len(buf) else b"\0")   # exact-size copy
        cp = G.Coding()
        w = (C.c_uint32 * 4)(*win) if win else None
        n = L.b2k_codestream_parse_window(raw, len(buf), w, reduce, C.byref(cp), None, 0)
        if n <= 1:
            return
        assert n <= 64 * len(buf) + 4096, "block count out of proportion: %d for %d bytes" % (n, len(buf))
        blocks = np.zeros(n, G.BLOCK_DTYPE)
        m = L.b2k_codestream_parse_window(raw, len(buf), w, reduce, C.byref(cp), blocks.ctypes.data, n)
        if m > 1:
            end = blocks["offset"].astype(np.uint64) + blocks["length"] + blocks["length2"]
            assert (end <= len(buf)).all(), "a block's bytes lie outside the buffer"

    total = 0
    for args, flags in ((dict(width=200, height=150, numcomps=3, prec=8, numres=4, tile=(64, 64)), G.CS_TLM | G.CS_PLT),
                        (dict(width=130, height=90, numcomps=1, prec=12, numres=3, irreversible=True), 0)):
        cp = G.make_coding(**args)
        planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=5)
        table, data, _ = oracle_encode(cp, planes)
        cs = np.array(G.codestream_write(cp, table, data, flags))
        hdr_end = int(np.flatnonzero((cs[:-1] == 0xFF) & (cs[1:] == 0x90))[0])
        sots = np.flatnonzero((cs[:-1] == 0xFF) & (cs[1:] == 0x90))
        for _ in range(rounds):
            b = cs.copy()
            kind = rng.integers(0, 5)
            if kind == 0:      # the main header
                for _ in range(rng.integers(1, 4)):
                    b[rng.integers(2, hdr_end)] = rng.integers(0, 256)
            elif kind == 1:    # anywhere
                for _ in range(rng.integers(1, 6)):
                    b[rng.integers(0, len(b))] = rng.integers(0, 256)
            elif kind == 2:    # cut short
                b = b[:rng.integers(1, len(b))].copy()
            elif kind == 3:    # tile-part and packet headers
                p = int(sots[rng.integers(0, len(sots))]) + int(rng.integers(0, 40))
                if p < len(b):
                    b[p] = rng.integers(0, 256)
            else:              # a run of garbage
                p = rng.integers(0, len(b) - 8)
                b[p:p + 8] = rng.integers(0, 256, 8)
            win = None if rng.integers(0, 2) else (int(rng.integers(0, 100)), int(rng.integers(0, 80)), int(rng.integers(100, 200)),
                                                   int(rng.integers(80, 150)))
            parse(b, win, int(rng.integers(0, 3)))
            total += 1
        # the file format wrapper around it
        n = G.lib().b2k_jph_wrap(C.byref(cp), cs.ctypes.data, len(cs), None, 0)
        f = np.zeros(n, np.uint8)
        G.lib().b2k_jph_wrap(C.byref(cp), cs.ctypes.data, len(cs), f.ctypes.data, n)
        for _ in range(rounds):
            b = f.copy()
            k = rng.integers(0, 3)
            if k == 0:
                for _ in range(rng.integers(1, 5)):
                    b[rng.integers(0, min(len(b), 120))] = rng.integers(0, 256)
            elif k == 1:
                b = b[:rng.integers(0, len(b))].copy()
            else:
                p = rng.integers(0, 100)
                b[p:p + 4] = rng.integers(0, 256, 4)
            raw = (C.c_uint8 * max(1, len(b))).from_buffer_copy(b.tobytes() if len(b) else b"\0")
            off, ln = C.c_uint64(), C.c_uint64()
            if L.b2k_jph_codestream(raw, len(b), C.byref(off), C.byref(ln)) == 0:
                assert off.value + ln.value <= len(b)
            total += 1
    print("FUZZ ok %d" % total)


if __name__ == "__main__":
    main()
