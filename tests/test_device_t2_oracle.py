"""The device code-stream writer (b2k_encode_codestream_device, csrc/t2_device.cu) against references that share nothing
with its packet and marker code: the plain-Python T2 of tests/oracle_t2.py and the marker validator of tests/t2_markers.py.
The device block coder's bytes are bit-identical to the oracle coder's (test_device_roundtrip.py, test_dwt_paths.py), so the
oracle's stream over the oracle coder's table is the exact expected output.  The case lists are test_t2_oracle.py's."""
import numpy as np
import pytest

import grok_b200 as G
import oracle_t2 as T2
import t2_markers as M
from test_codestream import openjpeg_pillow
from test_device_codestream import FLAGS
from test_t2_oracle import CONTENTS, EDGES, GEOMS, KMAX29, encoded


def _image(planes, prec):
    torch = pytest.importorskip("torch")
    return torch.from_numpy(np.stack(planes).astype(np.uint8 if prec <= 8 else np.uint16)).cuda()


def _device(engine, cp, img, flags):
    out = engine.encode_codestream_device(cp, img, flags, device_output=True)
    assert str(out.dtype) == "torch.uint8" and out.is_cuda
    return out.cpu().numpy()


def _same(got, want, what):
    n = min(len(got), len(want))
    diff = np.flatnonzero(got[:n] != want[:n])
    assert len(got) == len(want) and not len(diff), "%s: %d vs %d bytes, first difference at %s" % (what, len(got), len(want), diff[:1])


@pytest.mark.gpu
@pytest.mark.parametrize("geom", list(GEOMS) + ["kmax29"])
def test_device_writer_matches_the_oracle(engine, geom):
    args = KMAX29 if geom == "kmax29" else GEOMS[geom]
    for content in (["noise", "synthetic"] if geom == "kmax29" else CONTENTS):
        cp, planes, table, _, data = encoded(args, content)
        img = _image(planes, args["prec"])
        for flags in FLAGS:
            want = T2.write_flags(cp, table, data, flags)
            got = _device(engine, cp, img, flags)
            _same(got, want, "%s %s flags 0x%x" % (geom, content, flags))
            M.validate(got)
            # OpenJPEG: one stream per progression order, and the zero and sparse streams
            if (content == "synthetic" and flags & 0x700 and not flags & G.CS_TPARTS_R) or \
                    (content in ("zero", "sparse") and flags == FLAGS[5]):
                dec = openjpeg_pillow(got).astype(np.int64)
                dec = dec[..., None] if dec.ndim == 2 else dec
                src = np.stack(planes, axis=-1).astype(np.int64)
                if cp.irreversible:
                    assert dec.shape == src.shape and np.abs(dec - src).max() <= 16
                else:
                    assert np.array_equal(dec, src), (geom, content, flags)


@pytest.mark.gpu
@pytest.mark.parametrize("edge", [e for e in EDGES if EDGES[e][1] != "ff-end"])
def test_device_writer_edge_shapes(engine, edge):
    args, kind, flags = EDGES[edge]
    cp, planes, table, _, data = encoded(args, kind)
    img = _image(planes, args["prec"])
    got = _device(engine, cp, img, flags)
    _same(got, engine.encode_codestream_device(cp, img, flags), edge + ", host T2")
    _same(got, T2.write_flags(cp, table, data, flags), edge + ", oracle")
    info = M.validate(got)
    if edge == "plt-split":
        (pt,) = info["parts"]
        assert len(pt["plt"]) >= 2 and len(pt["packets"]) > 65536


@pytest.mark.gpu
def test_plt_split_with_2_and_3_byte_entries(engine):
    """a tile part of 65,540 packets: the LL band's 512 x 512 precincts code to more than 16 KiB each (3-byte PLT entries),
    the 8 x 8 precincts above it to 2-byte entries; SOP and EPH on, so Nsop wraps.  Too large for the pure-Python
    oracle: device against host T2 and the validator."""
    import oracle_pipeline as P
    rng = np.random.default_rng(3)
    cp = G.make_coding(2048, 2048, 1, 16, numres=2, cblk=(64, 64), precincts=[(512, 512), (8, 8)])
    img = _image([rng.integers(0, 1 << 16, (2048, 2048))], 16)
    flags = G.CS_TLM | G.CS_PLT | G.CS_SOP | G.CS_EPH
    got = _device(engine, cp, img, flags)
    _same(got, engine.encode_codestream_device(cp, img, flags), "host T2")
    (pt,) = M.validate(got)["parts"]
    sizes = np.where(pt["packets"] < 128, 1, np.where(pt["packets"] < 1 << 14, 2, 3))
    assert len(pt["packets"]) > 65536 and len(pt["plt"]) >= 2 and {2, 3} <= set(np.unique(sizes).tolist())
    assert P.tile_rects(cp) == [(0, 0, 2048, 2048)]


@pytest.mark.gpu
def test_state_under_one_engine():
    """One engine, so that its cached job, T2 plan and output buffer carry over: contents zero -> noise -> zero -> noise on
    one coding (the buffer grows under the cached plan, then the stream fits again); flags A -> B -> A (the plan is rebuilt
    and rebuilt back); a tile-sharded encode_device between two device code streams (the job is replaced)."""
    args = GEOMS["prec-ragged"]
    eng = G.Engine(0)
    try:
        sizes = []
        for content in ("zero", "noise", "zero", "noise"):
            cp, planes, table, _, data = encoded(args, content)
            got = _device(eng, cp, _image(planes, 8), G.CS_TLM | G.CS_PLT)
            _same(got, T2.write_flags(cp, table, data, G.CS_TLM | G.CS_PLT), content + " after %s" % sizes)
            sizes.append(len(got))
        assert sizes[0] == sizes[2] < sizes[1] == sizes[3]
        cp, planes, table, _, data = encoded(args, "synthetic")
        img = _image(planes, 8)
        for flags in (FLAGS[5], G.CS_PROG(G.PCRL) | G.CS_PLT, FLAGS[5]):
            _same(_device(eng, cp, img, flags), T2.write_flags(cp, table, data, flags), "flags 0x%x" % flags)
        res = eng.encode_device(cp, img, tile_mod=2, tile_rem=1)
        res.free()
        _same(_device(eng, cp, img, FLAGS[5]), T2.write_flags(cp, table, data, FLAGS[5]), "after a sharded encode")
    finally:
        eng.close()
