"""Batches of code streams decoded from device memory (b2k_decode_codestreams_device, Engine.decode_codestreams_device).

Every stream of a batch must get what b2k_decode_codestream_device gives it alone: the same return code and text, and,
where that is 0, the same pixels; a stream that fails leaves its image alone.  The batch rules on top: the coding is that
of the first stream whose main header parses, and a stream of another coding or progression / SOP / EPH gets 1."""
import ctypes as C

import numpy as np
import pytest

import grok_b200 as G
import test_device_io as D

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A


def _dev(torch, cs):
    return torch.from_numpy(np.array(cs, np.uint8)).cuda()


def _single(engine, torch, dcs, layout="CHW", dtype=None):
    """(rc, text, CHW image or None) of b2k_decode_codestream_device on one stream, called directly"""
    L = G.lib()
    hdr = G.Coding()
    try:
        hdr, _ = engine.codestream_parse_device(dcs)
    except (G.EngineError, AttributeError):   # a failing header, or a stream in host memory
        pass
    h, w, nc = max(hdr.y1 - hdr.y0, 1), max(hdr.x1 - hdr.x0, 1), max(hdr.numcomps, 1)
    shape = (nc, h, w) if layout == "CHW" else (h, w, nc)
    out = torch.full(shape, SENTINEL, dtype=dtype or torch.uint16, device="cuda")
    img = G.device_planes(out, nc, h, w, layout, writable=True)
    ptr, n = (dcs.data_ptr(), dcs.numel()) if hasattr(dcs, "data_ptr") else (int(dcs.ctypes.data), len(dcs))
    cp, ms = G.Coding(), C.c_double()
    rc = L.b2k_decode_codestream_device(engine._h, ptr, n, C.byref(img), None, C.byref(cp), C.byref(ms))
    torch.cuda.synchronize()
    text = (L.b2k_last_error() or b"").decode() if rc else ""
    return rc, text, (D._to_chw(out, layout) if rc == 0 else None)


def _batch(engine, torch, streams, cp_shape, layout="CHW", dtype=None, n=None):
    """decode_codestreams_device into a sentinel-filled output; returns (Coding, output as n CHW arrays, status)"""
    n = len(streams)
    nc, h, w = cp_shape
    shape = (n, nc, h, w) if layout == "CHW" else (n, h, w, nc)
    out = torch.full(shape, SENTINEL, dtype=dtype or torch.uint16, device="cuda")
    cp, out, status = engine.decode_codestreams_device(streams, out=out, layout=layout)
    torch.cuda.synchronize()
    return cp, [D._to_chw(out[i], layout) for i in range(n)], status


def _check_batch(engine, torch, streams, layout="CHW", dtype=None, rules=None):
    """each stream's status and pixels against its single call; rules: {index: (rc, text)} the batch rules decide"""
    rules = rules or {}
    singles = [_single(engine, torch, s, layout, dtype) for s in streams]
    ref = next((i for i, s in enumerate(singles) if s[0] == 0), None)
    if ref is None:   # no stream decodes alone: the batch has no coding and raises with stream 0's text
        with pytest.raises((G.NotHandled, G.EngineError)) as err:
            engine.decode_codestreams_device(streams, layout=layout)
        assert str(err.value).endswith(singles[0][1]) and (singles[0][0] == 1) == (err.type is G.NotHandled)
        return None, [s[:2] for s in singles]
    shape = tuple(singles[ref][2].shape)
    cp, got, status = _batch(engine, torch, streams, shape, layout, dtype)
    for i, ((rc, text, img), (brc, btext)) in enumerate(zip(singles, status)):
        if i in rules:
            assert (brc, btext) == rules[i], (i, brc, btext)
        else:
            assert (brc, btext) == (rc, text), (i, (brc, btext), (rc, text))
        if brc == 0:
            assert np.array_equal(got[i], img), "stream %d: pixels differ" % i
        else:
            assert (got[i] == SENTINEL).all(), "stream %d failed (%d) but its image was written" % (i, brc)
    return cp, status


def _seeded_streams(engine, case, count=5):
    """count code streams of one coding (case of test_device_io) from seeded images, TLM / PLT mixed"""
    import oracle_pipeline as P
    i, irr = case
    cp, _ = D._case(i, irr)
    args = dict(D._geoms()[i], irreversible=irr)
    flags = [G.CS_TLM | G.CS_PLT, 0, G.CS_PLT, G.CS_TLM, G.CS_TLM | G.CS_PLT]
    out = []
    for k in range(count):
        planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=1000 + 17 * k + i,
                                   origin=args.get("origin", (0, 0)))
        if args.get("sgnd"):
            planes = [p - (1 << (args["prec"] - 1)) for p in planes]
        res = engine.encode(cp, planes)
        out.append(np.array(G.codestream_write(cp, res.blocks, res.bytes, flags[k % len(flags)])))
        res.free()
    return cp, out


@pytest.mark.parametrize("case", D.CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in D.CASES])
def test_geometries(engine, case):
    torch = pytest.importorskip("torch")
    cp, streams = _seeded_streams(engine, case)
    dstreams = [_dev(torch, s) for s in streams]
    for dt in D._containers(cp):
        tdt = getattr(torch, np.dtype(dt).name)
        for layout in (("CHW", "HWC") if case[0] % 4 == 0 else ("CHW",)):
            cp_b, status = _check_batch(engine, torch, dstreams, layout, tdt)
            assert cp_b is None or all(rc == 0 for rc, _ in status), status


def _base(engine):
    import test_device_codestream_decode as E
    return E._base_stream(engine), E._edits(engine)


def test_mixed_batch(engine):
    """good streams interleaved with damaged ones, another coding, another progression, no bytes, host memory"""
    torch = pytest.importorskip("torch")
    good, edits = _base(engine)
    cp = G.codestream_parse(good)[0]
    streams, rules = [], {}
    for k, (name, cs) in enumerate(edits.items()):
        streams.append(_dev(torch, good))
        streams.append(_dev(torch, cs))
    other = D._host_result(engine, 9, False)                       # another coding
    streams.append(_dev(torch, G.codestream_write(other[0], other[2], other[3], G.CS_TLM | G.CS_PLT)))
    rules[len(streams) - 1] = (1, "code stream %d: its coding differs from that of code stream 0, which the batch takes "
                                  "its coding from" % (len(streams) - 1))
    res = G.codestream_parse(good)
    streams.append(_dev(torch, G.codestream_write(cp, res[1], good, G.CS_PROG(2))))   # another progression
    rules[len(streams) - 1] = (1, "code stream %d: its progression order, SOP or EPH differ from those of code stream 0, "
                                  "which the batch takes its coding from" % (len(streams) - 1))
    streams.append(torch.zeros(0, dtype=torch.uint8, device="cuda"))   # no bytes
    streams.append(_dev(torch, good))
    _check_batch(engine, torch, streams, rules=rules)
    # a stream in host memory: refused as the single call refuses it (the Python wrapper only passes CUDA arrays on)
    L = G.lib()
    host = np.array(good)
    n = 3
    ptrs = (C.c_void_p * n)(streams[0].data_ptr(), host.ctypes.data, streams[0].data_ptr())
    lens = (C.c_uint64 * n)(len(good), len(good), len(good))
    outs = [torch.full((cp.numcomps, cp.y1 - cp.y0, cp.x1 - cp.x0), SENTINEL, dtype=torch.uint16, device="cuda") for _ in range(n)]
    imgs = (G.DevicePlanes * n)(*[G.device_planes(o, cp.numcomps, cp.y1 - cp.y0, cp.x1 - cp.x0) for o in outs])
    bad = torch.zeros(1, dtype=torch.uint16, device="cuda")
    imgs[2].comp[1] = bad.data_ptr() + 1                           # an invalid image descriptor: not a multiple of sample_bytes
    st, ms, bcp = (C.c_int32 * n)(), C.c_double(), G.Coding()
    assert L.b2k_decode_codestreams_device(engine._h, n, ptrs, lens, imgs, None, C.byref(bcp), st, C.byref(ms)) == 2
    torch.cuda.synchronize()
    want0 = _single(engine, torch, _dev(torch, good))
    assert st[0] == 0 and torch.equal(outs[0].cpu(), torch.from_numpy(want0[2].astype(np.uint16)))
    host_rc = _single(engine, torch, host)
    assert (st[1], L.b2k_decode_codestreams_error(engine._h, 1).decode()) == host_rc[:2]
    assert st[2] == -1 and L.b2k_decode_codestreams_error(engine._h, 2).decode() == \
        "device image component 1: address not a multiple of sample_bytes"
    assert (outs[1] == SENTINEL).all() and (outs[2][0] == SENTINEL).all()


def _ht_reject(engine, torch, good):
    """a seeded edit of packet-body bytes the single call rejects with -2"""
    import test_device_codestream_decode as E
    rng = np.random.default_rng(7)
    sots = E._sots(good)
    for _ in range(400):
        b = good.copy()
        s = sots[int(rng.integers(len(sots)))]
        sod = int(np.flatnonzero((good[s:-1] == 0xFF) & (good[s + 1:] == 0x93))[0]) + s
        psot = int.from_bytes(bytes(good[s + 6:s + 10]), "big")
        lo, hi = sod + 40, s + psot - 4
        if hi <= lo:
            continue
        at = int(rng.integers(lo, hi))
        b[at:at + 3] = rng.integers(0, 255, 3)
        rc, text, _ = _single(engine, torch, _dev(torch, b))
        if rc == -2:
            return b, text
    pytest.fail("no seeded edit made the HT decoder reject a block")


def test_ht_decoder_rejection_is_per_stream(engine):
    torch = pytest.importorskip("torch")
    good, _ = _base(engine)
    bad, text = _ht_reject(engine, torch, good)
    _, status = _check_batch(engine, torch, [_dev(torch, good), _dev(torch, bad), _dev(torch, good)])
    assert [s[0] for s in status] == [0, -2, 0] and status[1][1] == text


def test_first_stream_damaged(engine):
    """stream 0's main header is damaged: the batch takes its coding from stream 1"""
    torch = pytest.importorskip("torch")
    good, _ = _base(engine)
    bad = good.copy()
    bad[0:2] = 0
    cp, status = _check_batch(engine, torch, [_dev(torch, bad), _dev(torch, good), _dev(torch, good)])
    assert status[0][0] != 0 and status[1][0] == 0
    want = G.codestream_parse(good)[0]
    assert bytes(cp) == bytes(want)


def test_refinement_passes(engine):
    torch = pytest.importorskip("torch")
    import test_t2_parse_host as H
    for name, (cp, table, data) in H.refinement_stream().items():
        cut = table.copy()                                          # the same table cut to cleanup passes
        cut["numpasses"] = np.minimum(cut["numpasses"], 1)
        cut["length2"] = 0
        a = G.codestream_write(cp, table, data, G.CS_PLT)
        b = G.codestream_write(cp, cut, data, G.CS_PLT)
        _, status = _check_batch(engine, torch, [_dev(torch, a), _dev(torch, b)], dtype=torch.int32)
        assert [s[0] for s in status] == [0, 0], (name, status)


def test_one_stream_equals_the_single_call(engine):
    torch = pytest.importorskip("torch")
    good, _ = _base(engine)
    _check_batch(engine, torch, [_dev(torch, good)])


def _small_batch(engine, torch, n, size=64, seed=0):
    cp = G.make_coding(size, size, 3, 8, numres=3, cblk=(32, 32))
    g = torch.Generator(device="cuda").manual_seed(seed)
    imgs = torch.randint(0, 256, (n, 3, size, size), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8)
    streams = [engine.encode_codestream_device(cp, imgs[i], G.CS_PLT if i % 2 else G.CS_TLM, device_output=True) for i in range(n)]
    return cp, imgs, streams


def test_hundreds_of_small_images(engine):
    torch = pytest.importorskip("torch")
    cp, imgs, streams = _small_batch(engine, torch, 300)
    _, out, status = engine.decode_codestreams_device(streams, dtype=torch.uint8)
    assert all(rc == 0 for rc, _ in status)
    assert torch.equal(out, imgs)


def test_launches_do_not_grow_with_the_batch(engine):
    torch = pytest.importorskip("torch")
    counts = []
    for n in (64, 160):
        cp, imgs, streams = _small_batch(engine, torch, n, seed=n)
        out = torch.empty_like(imgs)
        engine.decode_codestreams_device(streams, out=out)           # plan / grow once
        L = G.lib()
        before = L.b2k_launch_count()
        engine.decode_codestreams_device(streams, out=out)
        counts.append(L.b2k_launch_count() - before)
        assert torch.equal(out, imgs)
    assert counts[0] == counts[1], counts


def test_every_stream_failing(engine):
    torch = pytest.importorskip("torch")
    good, _ = _base(engine)
    bad = good.copy()
    bad[0:2] = 0
    streams = [_dev(torch, bad)] * 4
    L = G.lib()
    n = len(streams)
    ptrs = (C.c_void_p * n)(*[s.data_ptr() for s in streams])
    lens = (C.c_uint64 * n)(*[s.numel() for s in streams])
    out = torch.full((n, 3, 8, 8), SENTINEL, dtype=torch.uint16, device="cuda")
    imgs = (G.DevicePlanes * n)(*[G.device_planes(out[i], 3, 8, 8) for i in range(n)])
    st, ms, cp = (C.c_int32 * n)(), C.c_double(), G.Coding()
    assert L.b2k_decode_codestreams_device(engine._h, n, ptrs, lens, imgs, None, C.byref(cp), st, C.byref(ms)) == n
    assert (out == SENTINEL).all()
    with pytest.raises(G.EngineError):
        engine.decode_codestreams_device(streams)
    with pytest.raises(ValueError):
        engine.decode_codestreams_device([])


def test_streams_filled_late_on_a_side_stream(engine):
    torch = pytest.importorskip("torch")
    cp, imgs, streams = _small_batch(engine, torch, 6)
    side = torch.cuda.Stream()
    late = [torch.zeros_like(s) for s in streams]
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        for d, s in zip(late, streams):
            d.copy_(s)                                           # the bytes arrive late, on the side stream
        _, out, status = engine.decode_codestreams_device(late, stream=side, dtype=torch.uint8)
        after = out.clone()                                      # queued after the call: must see the pixels
    side.synchronize()
    assert all(rc == 0 for rc, _ in status)
    assert torch.equal(after, imgs)


def test_one_engine_alternates(engine):
    """batch, single decode, window decode, device encode, and a batch of another size and coding: results unchanged"""
    torch = pytest.importorskip("torch")
    good, _ = _base(engine)
    dgood = _dev(torch, good)
    cp_a, imgs_a, streams_a = _small_batch(engine, torch, 12, seed=1)
    cp_b, imgs_b, streams_b = _small_batch(engine, torch, 5, size=96, seed=2)
    single = _single(engine, torch, dgood)[2]
    window = engine.decode_window_device(dgood, window=(0, 0, 40, 40))[1].cpu()
    for _ in range(2):
        _, out, _ = engine.decode_codestreams_device(streams_a, dtype=torch.uint8)
        assert torch.equal(out, imgs_a)
        assert np.array_equal(_single(engine, torch, dgood)[2], single)
        assert torch.equal(engine.decode_window_device(dgood, window=(0, 0, 40, 40))[1].cpu(), window)
        again = engine.encode_codestream_device(cp_a, imgs_a[3], G.CS_PLT, device_output=True)
        assert torch.equal(again, streams_a[3])
        _, out, _ = engine.decode_codestreams_device(streams_b, dtype=torch.uint8)
        assert torch.equal(out, imgs_b)
        _, out, _ = engine.decode_codestreams_device(streams_a[:7], dtype=torch.uint8)   # fewer than the job's slots
        assert torch.equal(out, imgs_a[:7])
    ix, wk = engine.codestream_parse_device_stats()
    assert ix + wk == 7                                          # totals over the last batch
