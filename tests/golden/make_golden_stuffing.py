#!/usr/bin/env python3
"""Regenerates tests/golden/ht_stuffing.npz from the REFERENCE's own HT block coder (oracle/_ref/libgrok_ref.so, built by
`make -C oracle ref`): the blocks tests/test_ht_coder_paths.py constructs so that the MagSgn and VLC byte stuffing reach
the encoder's longest fix-up chains, the end of a block reaches every termination cell and the segments reach their
longest.  Run in the build container only; the fixture is committed so that a machine without
the reference tree checks the oracle against it.

Per block <label> (CONSTRUCTED: the MagSgn chain blocks, the VLC-heavy first-row blocks, the termination blocks term-<seed>,
the longest MEL segment per block shape mel-longest-<w>x<h> and the largest blocks for their scratch slot
slot-<kind>-k<Kmax>-<w>x<h>):
  <label>/coef : the block's coefficients (h, w), int32 (reversible: the quantisation indices themselves)
  <label>/data : the reference encoder's bytes; every SIMD variant built here writes the same (asserted)
  <label>/dec  : what the reference decoders (all variants agree; asserted) return for them, sign-magnitude words
"""
import io
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.dirname(os.path.dirname(HERE))]
import oracle_lib as O  # noqa: E402
import test_ht_coder_paths as T  # noqa: E402


def main():
    assert O.ref() is not None, "build the reference kernels first: make -C oracle ref"
    out = {}
    for label in T.CONSTRUCTED:
        coef, _, kmax = T.chain_case(label)
        h, w = coef.shape
        sm = O.to_sgnmag(coef, kmax)
        encs = [O.ref_ht_encode(sm, kmax, variant=v, cap=65536) for v in (0, 1, 2)]
        encs = [e for e in encs if e is not None]
        assert all(np.array_equal(encs[0], e) for e in encs), label + ": reference encoder variants disagree"
        decs = [O.ref_ht_decode(encs[0], kmax, w, h, variant=v) for v in (0, 1, 2)]
        decs = [d for d in decs if d[0] != -2]
        assert all(d[0] == 0 and np.array_equal(decs[0][1], d[1]) for d in decs), label + ": reference decoders disagree"
        out[label + "/coef"] = coef.astype(np.int32)
        out[label + "/data"] = encs[0]
        out[label + "/dec"] = decs[0][1]
    buf = io.BytesIO()
    np.savez_compressed(buf, **out)
    path = os.path.join(HERE, "ht_stuffing.npz")
    # np.savez_compressed stamps the zip entries with the current time: rewrite them with a fixed one
    import zipfile
    src = zipfile.ZipFile(io.BytesIO(buf.getvalue()))
    with zipfile.ZipFile(path, "w", zipfile.ZIP_DEFLATED) as dst:
        for name in sorted(src.namelist()):
            info = zipfile.ZipInfo(name, date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            dst.writestr(info, src.read(name))
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
