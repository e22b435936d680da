"""Code streams written on the GPU (b2k_encode_codestream_device, Engine.encode_codestream_device(device_output=True)).

The device writer shares its packet-header, PLT, TLM and SOT code with the host writer (csrc/t2_packet.h), which the CPU
suites pin to Grok and OpenJPEG.  Here, on the GPU, every geometry of test_device_io and every code-stream flag must give
the bytes of the host-T2 path (b2k_encode_device + b2k_codestream_write), decline where it declines with the same
message, split PLT and TLM segments where it splits them, and keep working as the engine's buffers grow."""
import numpy as np
import pytest

import grok_b200 as G
import test_device_io as D

FLAGS = [0, G.CS_TLM, G.CS_PLT, G.CS_TLM | G.CS_PLT, G.CS_SOP | G.CS_EPH, G.CS_SOP | G.CS_EPH | G.CS_TLM | G.CS_PLT] + \
        [G.CS_PROG(p) | t for p in range(5) for t in (0, G.CS_TPARTS_R)]


def _device(engine, cp, img, flags=G.CS_TLM | G.CS_PLT, **kw):
    out = engine.encode_codestream_device(cp, img, flags, device_output=True, **kw)
    assert str(out.dtype) == "torch.uint8" and out.is_cuda
    return out.cpu().numpy()


def _reason(err):
    """the b2k_last_error text of a wrapper's exception ('<call>[ -> rc]: <text>')"""
    return str(err).split(": ", 1)[1]


def _image(torch, planes, dt):
    return torch.from_numpy(np.stack(planes).astype(dt)).cuda()


def _markers(cs):
    """(TLM segments in the main header, PLT segments in each tile part's header, tile parts)"""
    cs = bytes(cs)
    p, tlm = 2, 0
    while cs[p:p + 2] != b"\xff\x90":
        tlm += cs[p:p + 2] == b"\xff\x55"
        p += 2 + int.from_bytes(cs[p + 2:p + 4], "big")
    plt = []
    while cs[p:p + 2] == b"\xff\x90":
        psot = int.from_bytes(cs[p + 6:p + 10], "big")
        q, n = p + 12, 0
        while cs[q:q + 2] != b"\xff\x93":
            n += cs[q:q + 2] == b"\xff\x58"
            q += 2 + int.from_bytes(cs[q + 2:q + 4], "big")
        plt.append(n)
        p += psot
    assert cs[p:] == b"\xff\xd9"
    return tlm, plt


@pytest.mark.gpu
@pytest.mark.parametrize("case", D.CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in D.CASES])
def test_device_codestream_matches_host_t2(engine, case):
    torch = pytest.importorskip("torch")
    cp, planes, _, _, _ = D._host_result(engine, *case)
    img = _image(torch, planes, D._containers(cp)[0])
    for flags in FLAGS:
        try:
            want = engine.encode_codestream_device(cp, img, flags)
        except G.EngineError as e:      # a tile grid the writer declines: so must the device writer, with the same text
            with pytest.raises(type(e)) as got:
                _device(engine, cp, img, flags)
            assert _reason(got.value) == _reason(e), flags
            continue
        got = _device(engine, cp, img, flags)
        assert np.array_equal(got, want), "flags 0x%x: %d vs %d bytes" % (flags, len(got), len(want))


@pytest.mark.gpu
def test_plt_splits_into_several_segments(engine):
    torch = pytest.importorskip("torch")
    import oracle_pipeline as P
    # 81,920 packets of 8x8 precincts in the one tile part: more than 65,532 bytes of packet lengths
    cp = G.make_coding(2048, 2048, 1, 8, numres=2, cblk=(4, 4), precincts=[(8, 8)])
    img = _image(torch, P.synthetic_image(2048, 2048, 1, 8, seed=7), np.uint8)
    want = engine.encode_codestream_device(cp, img, G.CS_PLT)
    got = _device(engine, cp, img, G.CS_PLT)
    assert np.array_equal(got, want)
    tlm, plt = _markers(got)
    assert tlm == 0 and len(plt) == 1 and plt[0] >= 2, plt


@pytest.mark.gpu
def test_tlm_splits_into_several_segments(engine):
    torch = pytest.importorskip("torch")
    import oracle_pipeline as P
    # 4096 tiles of 4x4, a tile part per resolution: 12,288 TLM entries, more than the 10,000 of one segment
    cp = G.make_coding(256, 256, 1, 8, numres=3, tile=(4, 4))
    img = _image(torch, P.synthetic_image(256, 256, 1, 8, seed=8), np.uint8)
    flags = G.CS_TLM | G.CS_PLT | G.CS_TPARTS_R
    want = engine.encode_codestream_device(cp, img, flags)
    got = _device(engine, cp, img, flags)
    assert np.array_equal(got, want)
    tlm, plt = _markers(got)
    assert tlm == 2 and len(plt) == 3 * 4096 and all(n == 1 for n in plt)


@pytest.mark.gpu
def test_narrow_container_is_declined_as_on_the_host(engine):
    torch = pytest.importorskip("torch")
    cp, planes, _, _, _ = D._host_result(engine, 1, False)               # prec 12
    img = _image(torch, planes, np.uint8)
    with pytest.raises(G.NotHandled) as host:
        engine.encode_codestream_device(cp, img)
    with pytest.raises(G.NotHandled) as dev:
        _device(engine, cp, img)
    assert _reason(dev.value) == _reason(host.value) and "8-bit containers" in _reason(dev.value)


@pytest.mark.gpu
def test_engine_reuse_small_large_small():
    torch = pytest.importorskip("torch")
    eng = G.Engine(0)
    try:
        for i, irr in [(0, False), (1, True), (0, False), (1, True)]:
            cp, planes = D._case(i, irr)
            img = _image(torch, planes, np.uint16)
            want = eng.encode_codestream_device(cp, img)
            assert np.array_equal(_device(eng, cp, img), want), (i, irr)
    finally:
        eng.close()


@pytest.mark.gpu
def test_image_written_on_a_side_stream_is_the_one_coded(engine):
    torch = pytest.importorskip("torch")
    cp, planes, _, _, _ = D._host_result(engine, 8, False)
    frame = _image(torch, planes, np.uint16)
    want = engine.encode_codestream_device(cp, frame)
    dst = torch.zeros_like(frame)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        dst.copy_(frame)
    out = engine.encode_codestream_device(cp, dst, stream=s, device_output=True)
    s.synchronize()
    assert np.array_equal(out.cpu().numpy(), want)


@pytest.mark.gpu
def test_device_codestream_round_trip(engine):
    torch = pytest.importorskip("torch")
    cp, planes, _, _, _ = D._host_result(engine, 2, False)
    cs = _device(engine, cp, _image(torch, planes, np.uint16), G.CS_TLM | G.CS_PLT | G.CS_SOP | G.CS_EPH)
    _, got = engine.decode_codestream_device(cs)
    assert np.array_equal(got.cpu().numpy(), np.stack(planes).astype(np.uint16))


@pytest.mark.gpu
def test_config2_once(engine):
    torch = pytest.importorskip("torch")
    import bench
    cp = G.make_coding(bench.W, bench.H, bench.NCOMP, bench.PREC, numres=bench.NUMRES, tile=(bench.TILE, bench.TILE))
    img = _image(torch, bench.make_image(), np.uint16)
    want = engine.encode_codestream_device(cp, img)
    got = _device(engine, cp, img)
    assert len(got) == 151_685_678 and np.array_equal(got, want)
