"""Encode from and decode into device memory (b2k_encode_device / b2k_decode_device, Engine.encode_device & co).

The CPU tests check how the Python layer turns __cuda_array_interface__ descriptions into b2k_device_planes (pointers,
row pitches, column steps) and what it refuses, with fake arrays.  The GPU tests (-m gpu) use torch CUDA tensors and
compare with the host entry points, which the other suites pin to the oracle and to Grok: the same code blocks and bytes
on encode, the same samples (cast to the container) on decode."""
import ctypes as C

import numpy as np
import pytest

import grok_b200 as G


class FakeCudaArray:
    """Just enough of a CUDA array for the layout derivation: the interface and nothing else."""

    def __init__(self, shape, typestr="<u2", strides=None, ptr=0x7f0000000000, readonly=False):
        self.__cuda_array_interface__ = dict(shape=tuple(shape), typestr=typestr, strides=strides, data=(ptr, readonly),
                                             version=2)


BASE = 0x7f0000000000
H, W = 37, 53


def _fields(img, n):
    return ([img.comp[c] for c in range(n)], [img.row_pitch[c] for c in range(n)], [img.col_step[c] for c in range(n)],
            img.sample_bytes)


def test_chw_contiguous():
    img = G.device_planes(FakeCudaArray((3, H, W)), 3, H, W, "CHW")
    assert _fields(img, 3) == ([BASE + c * H * W * 2 for c in range(3)], [W] * 3, [1] * 3, 2)


def test_hwc_contiguous():
    img = G.device_planes(FakeCudaArray((H, W, 3), "|u1"), 3, H, W, "HWC")
    assert _fields(img, 3) == ([BASE + c for c in range(3)], [3 * W] * 3, [3] * 3, 1)


def test_row_padded_view_of_a_larger_array():
    # t[:, 2:2+H, 5:5+W] of a (3, H+4, W+11) int32 array
    Hp, Wp = H + 4, W + 11
    ptr = BASE + (2 * Wp + 5) * 4
    img = G.device_planes(FakeCudaArray((3, H, W), "<i4", strides=(Hp * Wp * 4, Wp * 4, 4), ptr=ptr), 3, H, W)
    assert _fields(img, 3) == ([ptr + c * Hp * Wp * 4 for c in range(3)], [Wp] * 3, [1] * 3, 4)


def test_rgb_view_of_rgba():
    # t[..., :3] of an (H, W, 4) uint16 tensor: same base, pixel step 4
    img = G.device_planes(FakeCudaArray((H, W, 3), "<u2", strides=(W * 4 * 2, 4 * 2, 2)), 3, H, W, "HWC")
    assert _fields(img, 3) == ([BASE + 2 * c for c in range(3)], [4 * W] * 3, [4] * 3, 2)


def test_one_component_and_component_lists():
    img = G.device_planes(FakeCudaArray((H, W), "|i1"), 1, H, W)
    assert _fields(img, 1) == ([BASE], [W], [1], 1)
    arrays = [FakeCudaArray((H, W), "<u4", strides=(256 * 4, 4), ptr=BASE + 4096 * k) for k in range(4)]
    img = G.device_planes(arrays, 4, H, W)
    assert _fields(img, 4) == ([BASE + 4096 * k for k in range(4)], [256] * 4, [1] * 4, 4)


@pytest.mark.parametrize("shape,layout,n", [((3, H, W + 1), "CHW", 3), ((H, W, 3), "CHW", 3), ((3, H, W), "HWC", 3),
                                            ((H, W), "CHW", 3), ((4, H, W), "CHW", 3)])
def test_wrong_shape_is_rejected(shape, layout, n):
    with pytest.raises(ValueError, match="shape"):
        G.device_planes(FakeCudaArray(shape), n, H, W, layout)
    with pytest.raises(ValueError, match="shape"):
        G.device_planes([FakeCudaArray((H, W))] * (n - 1), n, H, W)


@pytest.mark.parametrize("typestr", ["<f4", "<i8", "<f2", "|b1", ">u2"])
def test_wrong_dtype_is_rejected(typestr):
    with pytest.raises(ValueError, match="dtype"):
        G.device_planes(FakeCudaArray((3, H, W), typestr), 3, H, W)


def test_negative_strides_are_rejected():
    with pytest.raises(ValueError, match="negative"):
        G.device_planes(FakeCudaArray((H, W), "<u2", strides=(-W * 2, 2)), 1, H, W)


@pytest.mark.parametrize("strides", [(W * 2 + 1, 2), (W * 2, 3), (W * 4, 5)])
def test_strides_that_are_not_whole_samples_are_rejected(strides):
    with pytest.raises(ValueError, match="whole"):
        G.device_planes(FakeCudaArray((H, W), "<u2", strides=strides), 1, H, W)


def test_other_rejections():
    with pytest.raises(TypeError):
        G.device_planes(np.zeros((H, W), np.uint16), 1, H, W)        # host memory has no CUDA array interface
    with pytest.raises(ValueError, match="layout"):
        G.device_planes(FakeCudaArray((3, H, W)), 3, H, W, "WHC")
    with pytest.raises(ValueError, match="read-only"):
        G.device_planes(FakeCudaArray((H, W), readonly=True), 1, H, W, writable=True)


def test_stream_handles():
    class S:
        cuda_stream = 0x1234
    assert G._stream_handle(None, FakeCudaArray((H, W))) is None       # legacy default stream
    assert G._stream_handle(0x55, FakeCudaArray((H, W))) == 0x55
    assert G._stream_handle(S(), [FakeCudaArray((H, W))]) == 0x1234


# ------------------------------------------------------------------------------------------------
# GPU: parity with the host entry points
# ------------------------------------------------------------------------------------------------
def _geoms():
    import test_gpu
    return test_gpu.GEOMS + [dict(width=150, height=97, numcomps=3, prec=8, sgnd=True, numres=1, tile=(64, 40))]  # signed, no level, ragged


IRREVERSIBLE = [1, 2, 3, 9, 15, 17]
CASES = [(i, False) for i in range(18)] + [(i, True) for i in IRREVERSIBLE]


def _case(i, irreversible):
    args = dict(_geoms()[i], irreversible=irreversible)
    import oracle_pipeline as P
    planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=42 + i,
                               origin=args.get("origin", (0, 0)))
    if args.get("sgnd"):
        planes = [p - (1 << (args["prec"] - 1)) for p in planes]
    return G.make_coding(**args), planes


def _containers(cp):
    signed = bool(cp.sgnd)
    out = [np.int8 if signed else np.uint8] if cp.prec <= 8 else []
    return out + [np.int16 if signed else np.uint16, np.int32]


def _images(torch, planes, dt):
    """(name, device image, layout) of the samples in container dt: CHW, HWC, a row-padded CHW slice of a larger tensor,
    a CHW slice that starts at an odd column (no 128-bit path), and for 3 components the RGB view of an RGBA tensor."""
    chw = np.stack(planes).astype(dt)
    n, h, w = chw.shape
    out = [("CHW", torch.from_numpy(chw).cuda(), "CHW"),
           ("HWC", torch.from_numpy(np.ascontiguousarray(chw.transpose(1, 2, 0))).cuda(), "HWC")]
    big = np.zeros((n, h, (w + 63) // 64 * 64 + 64), dt)
    big[:, :, :w] = chw
    out.append(("row_padded", torch.from_numpy(big).cuda()[:, :, :w], "CHW"))
    big = np.zeros((n, h + 3, w + 7), dt)
    big[:, 2:h + 2, 5:w + 5] = chw
    out.append(("odd_offset", torch.from_numpy(big).cuda()[:, 2:h + 2, 5:w + 5], "CHW"))
    if n == 3:
        rgba = np.full((h, w, 4), 7, dt)
        rgba[..., :3] = chw.transpose(1, 2, 0)
        out.append(("rgb_of_rgba", torch.from_numpy(rgba).cuda()[..., :3], "HWC"))
    return out


def _to_chw(t, layout):
    a = t.cpu().numpy()
    return a.transpose(2, 0, 1) if layout == "HWC" else a


_host = {}


def _host_result(engine, i, irreversible):
    """(cp, planes, host block table, host bytes, host-decoded planes), once per case."""
    key = (i, irreversible)
    if key not in _host:
        cp, planes = _case(i, irreversible)
        res = engine.encode(cp, planes)
        blocks, data = res.blocks.copy(), res.bytes.copy()
        res.free()
        rec = [np.zeros_like(p) for p in planes]
        engine.decode(cp, blocks, data, rec)
        _host[key] = (cp, planes, blocks, data, rec)
    return _host[key]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in CASES])
def test_encode_device_matches_encode(engine, case):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, _ = _host_result(engine, *case)
    for dt in _containers(cp):
        for name, img, layout in _images(torch, planes, dt):
            res = engine.encode_device(cp, img, layout=layout)
            try:
                assert res.blocks.tobytes() == blocks.tobytes(), "block table differs: %s %s" % (np.dtype(dt).name, name)
                assert np.array_equal(res.bytes, data), "coded bytes differ: %s %s" % (np.dtype(dt).name, name)
            finally:
                res.free()
    img = _images(torch, planes, _containers(cp)[0])[0][1]
    try:
        want = engine.encode_codestream(cp, planes)
    except G.EngineError:        # a tile grid the writer declines (tiles outside the image): so must the device call
        with pytest.raises(G.EngineError):
            engine.encode_codestream_device(cp, img)
        return
    assert np.array_equal(engine.encode_codestream_device(cp, img), want)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in CASES])
def test_decode_device_matches_decode(engine, case):
    torch = pytest.importorskip("torch")
    cp, _, blocks, data, rec = _host_result(engine, *case)
    for dt in _containers(cp):
        want = np.stack(rec).astype(dt)
        for name, img, layout in _images(torch, [np.zeros_like(p) for p in rec], dt):
            engine.decode_device(cp, blocks, data, img, layout=layout)
            assert np.array_equal(_to_chw(img, layout), want), "decoded samples differ: %s %s" % (np.dtype(dt).name, name)


@pytest.mark.gpu
def test_decode_into_rgba_leaves_alpha_alone(engine):
    torch = pytest.importorskip("torch")
    cp, _, blocks, data, rec = _host_result(engine, 2, False)
    h, w = rec[0].shape
    rgba = torch.from_numpy(np.full((h, w, 4), 0x5A5A, np.uint16)).cuda()
    engine.decode_device(cp, blocks, data, rgba[..., :3], layout="HWC")
    got = rgba.cpu().numpy()
    assert np.array_equal(got[..., :3].transpose(2, 0, 1), np.stack(rec).astype(np.uint16))
    assert (got[..., 3] == 0x5A5A).all()


@pytest.mark.gpu
def test_codestream_windows_and_reductions(engine):
    torch = pytest.importorskip("torch")
    import oracle_pipeline as P
    cp = G.make_coding(1000, 700, 3, 12, numres=5, tile=(256, 256))
    planes = P.synthetic_image(1000, 700, 3, 12, seed=11)
    cs = engine.encode_codestream(cp, planes)
    vcp, full = engine.decode_codestream_device(cs)
    assert full.dtype == torch.uint16 and tuple(full.shape) == (3, 700, 1000)
    assert np.array_equal(full.cpu().numpy(), np.stack(planes).astype(np.uint16))
    rng = np.random.default_rng(5)
    for k in range(12):
        reduce = k % 3
        x0, y0 = int(rng.integers(0, 900)), int(rng.integers(0, 600))
        window = (x0, y0, x0 + int(rng.integers(1, 1000 - x0)), y0 + int(rng.integers(1, 700 - y0)))
        _, want = engine.decode_window(cs, window, reduce)
        want = np.stack([p.copy() for p in want])
        layout = "HWC" if k % 4 == 1 else "CHW"
        _, got = engine.decode_codestream_device(cs, window=window, reduce=reduce, layout=layout,
                                                  dtype=torch.int32 if k % 4 == 3 else None)
        assert np.array_equal(_to_chw(got, layout).astype(np.int32), want), (window, reduce, layout)


@pytest.mark.gpu
def test_tile_selection_writes_only_the_selected_tiles(engine):
    torch = pytest.importorskip("torch")
    import oracle_pipeline as P
    cp = G.make_coding(600, 300, 3, 12, numres=4, tile=(256, 128), origin=(8, 0))
    planes = P.synthetic_image(600, 300, 3, 12, seed=3, origin=(8, 0))
    res = engine.encode(cp, planes, tile_mod=2, tile_rem=1)
    blocks, data = res.blocks.copy(), res.bytes.copy()
    res.free()
    sentinel = 0xBEEF
    out = torch.from_numpy(np.full((3, 300, 600), sentinel, np.uint16)).cuda()
    engine.decode_device(cp, blocks, data, out, tile_mod=2, tile_rem=1)
    got = out.cpu().numpy()
    want = np.full((3, 300, 600), sentinel, np.uint16)
    for t, (x0, y0, x1, y1) in enumerate(P.tile_rects(cp)):
        if t % 2 == 1:
            want[:, y0:y1, x0 - 8:x1 - 8] = np.stack(planes)[:, y0:y1, x0 - 8:x1 - 8]
    assert np.array_equal(got, want)
    # and an encode of the same tiles from the device equals the host's
    dres = engine.encode_device(cp, torch.from_numpy(np.stack(planes).astype(np.uint16)).cuda(), tile_mod=2, tile_rem=1)
    assert dres.blocks.tobytes() == blocks.tobytes() and np.array_equal(dres.bytes, data)
    dres.free()


@pytest.mark.gpu
def test_calls_are_ordered_on_the_callers_stream(engine):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, rec = _host_result(engine, 8, False)
    frame = torch.from_numpy(np.stack(planes).astype(np.uint16)).cuda()
    n, h, w = frame.shape
    s = torch.cuda.Stream()
    # encode: the frame is written on s behind a long sleep; the engine must read what the copy writes
    dst = torch.from_numpy(np.zeros((n, h, w), np.uint16)).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        dst.copy_(frame)
    res = engine.encode_device(cp, dst, stream=s)
    assert res.blocks.tobytes() == blocks.tobytes() and np.array_equal(res.bytes, data)
    res.free()
    # decode: a late write of s must land before the engine's, and a read queued on s after the call sees the pixels
    out = torch.from_numpy(np.zeros((n, h, w), np.uint16)).cuda()
    junk = torch.from_numpy(np.full((n, h, w), 0xFFFF, np.uint16)).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        out.copy_(junk)
    engine.decode_device(cp, blocks, data, out, stream=s)
    with torch.cuda.stream(s):
        seen = out.clone()
    s.synchronize()
    assert np.array_equal(seen.cpu().numpy(), np.stack(rec).astype(np.uint16))


@pytest.mark.gpu
def test_host_memory_is_refused(engine):
    cp, planes, _, _, _ = _host_result(engine, 0, False)
    pinned = G.pinned_empty(planes[0].shape, np.uint16)
    img = G.DevicePlanes()
    img.comp[0], img.row_pitch[0], img.col_step[0], img.sample_bytes = pinned.ctypes.data, pinned.shape[1], 1, 2
    out = C.POINTER(G.Result)()
    rc = G.lib().b2k_encode_device(engine._h, C.byref(cp), C.byref(img), 1, 0, None, C.byref(out))
    assert rc == -1
    assert b"not device or managed memory" in G.lib().b2k_last_error()
    ms = C.c_double()
    rc = G.lib().b2k_decode_device(engine._h, C.byref(cp), None, 0, None, 0, C.byref(img), None, 1, 0, None, C.byref(ms))
    assert rc == -1


@pytest.mark.gpu
def test_narrow_containers_are_not_handled(engine):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, _ = _host_result(engine, 1, False)               # prec 12
    img = torch.from_numpy(np.stack(planes).astype(np.uint8)).cuda()
    with pytest.raises(G.NotHandled, match="8-bit containers"):
        engine.encode_device(cp, img)
    with pytest.raises(G.NotHandled):
        engine.decode_device(cp, blocks, data, img)


@pytest.mark.gpu
def test_device_calls_leave_host_calls_alone(engine):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, _ = _host_result(engine, 1, False)
    before = engine.encode(cp, planes)
    want = (before.blocks.tobytes(), before.bytes.copy())
    before.free()
    packing = G.host_pack_last()
    d = engine.encode_device(cp, torch.from_numpy(np.stack(planes).astype(np.uint16)).cuda())
    d.free()
    engine.decode_device(cp, blocks, data, torch.from_numpy(np.zeros((3,) + planes[0].shape, np.uint16)).cuda())
    assert G.host_pack_last() == packing
    after = engine.encode(cp, planes)
    assert after.blocks.tobytes() == want[0] and np.array_equal(after.bytes, want[1])
    after.free()
