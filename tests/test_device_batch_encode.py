"""Batches of images encoded into code streams in device memory (b2k_encode_codestreams_device,
Engine.encode_codestreams_device).

Every image of a batch must get what b2k_encode_codestream_device gives it alone: the same return code and text, and,
where that is 0, the same bytes.  An image that fails takes no bytes of the output and leaves every other stream as it
would be without it; the streams lie in image order at 256-byte boundaries."""
import ctypes as C

import numpy as np
import pytest

import grok_b200 as G
import test_device_codestream as DC
import test_device_io as D

pytestmark = pytest.mark.gpu


def _bytes(torch, ptr, n):
    return torch.as_tensor(G._DeviceBytes(ptr, n), device="cuda").cpu().numpy().copy()


def _single(engine, torch, cp, img, flags):
    """(rc, text, bytes or None) of b2k_encode_codestream_device on one image descriptor, called directly"""
    L = G.lib()
    ptr = C.c_void_p()
    n = L.b2k_encode_codestream_device(engine._h, C.byref(cp), C.byref(img), flags, None, C.byref(ptr))
    torch.cuda.synchronize()
    if n <= 1:
        return int(n), (L.b2k_last_error() or b"").decode(), None
    return 0, "", _bytes(torch, ptr.value, n)


def _raw_batch(engine, torch, cp, imgs, flags):
    """(return value, [(rc, text)], [bytes or None], offsets) of b2k_encode_codestreams_device, called directly"""
    L = G.lib()
    n = len(imgs)
    arr = (G.DevicePlanes * n)(*imgs)
    ptr, off, lens, st, ms = C.c_void_p(), (C.c_uint64 * n)(), (C.c_uint64 * n)(), (C.c_int32 * n)(), C.c_double()
    rc = L.b2k_encode_codestreams_device(engine._h, C.byref(cp), n, arr, flags, None, C.byref(ptr), off, lens, st, C.byref(ms))
    torch.cuda.synchronize()
    if rc < 0:
        return rc, None, None, None
    status = [(int(st[i]), (L.b2k_encode_codestreams_error(engine._h, i) or b"").decode()) for i in range(n)]
    out = [_bytes(torch, ptr.value + off[i], lens[i]) if st[i] == 0 else None for i in range(n)]
    for i in range(n):
        assert st[i] == 0 or lens[i] == 0, i
    return rc, status, out, [int(o) for o in off]


def _check_layout(status, offsets, lengths):
    """streams in image order, each at a 256-byte boundary, none overlapping"""
    end = 0
    for (rc, _), o, n in zip(status, offsets, lengths):
        if rc:
            continue
        assert o % 256 == 0 and o >= end, (o, end)
        end = o + n


def _check(engine, torch, cp, images, flags, layout="CHW", via_api=True):
    """every image's status and bytes in a batch against its single call; images: a list of CUDA arrays in layout, or an
    (n, ...) array.  Checks both the C entry point and the Python wrapper.  Returns the statuses."""
    n = len(images)
    h, w, nc = cp.y1 - cp.y0, cp.x1 - cp.x0, cp.numcomps
    descs = [G.device_planes(images[i], nc, h, w, layout) for i in range(n)]
    singles = [_single(engine, torch, cp, d, flags) for d in descs]
    rc, status, got, offsets = _raw_batch(engine, torch, cp, descs, flags)
    assert rc == sum(s[0] != 0 for s in singles), (rc, singles)
    for i, ((src, stext, sbytes), (brc, btext), b) in enumerate(zip(singles, status, got)):
        assert (brc, btext) == (src, stext), (i, (brc, btext), (src, stext))
        if src == 0:
            assert np.array_equal(b, sbytes), "image %d: %d vs %d bytes" % (i, len(b), len(sbytes))
    _check_layout(status, offsets, [0 if g is None else len(g) for g in got])
    if via_api:
        streams, api_status = engine.encode_codestreams_device(cp, images, flags, layout=layout)
        torch.cuda.synchronize()
        assert api_status == status
        for i, s in enumerate(streams):
            if status[i][0]:
                assert s is None
            else:
                assert str(s.dtype) == "torch.uint8" and s.is_cuda and np.array_equal(s.cpu().numpy(), singles[i][2]), i
    return status


def _seeded(case, count, dt, seed=0):
    """count distinct images of case (test_device_io) in container dt, as CHW numpy arrays"""
    import oracle_pipeline as P
    i, irr = case
    args = dict(D._geoms()[i], irreversible=irr)
    out = []
    for k in range(count):
        planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=500 + 31 * k + i + seed,
                                   origin=args.get("origin", (0, 0)))
        if args.get("sgnd"):
            planes = [p - (1 << (args["prec"] - 1)) for p in planes]
        out.append(np.stack(planes).astype(dt))
    return out


@pytest.mark.parametrize("case", D.CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in D.CASES])
def test_geometries(engine, case):
    torch = pytest.importorskip("torch")
    cp, _ = D._case(*case)
    flag_sets = [DC.FLAGS[(case[0] + 5 * k + (7 if case[1] else 0)) % len(DC.FLAGS)] for k in range(3)]
    for j, dt in enumerate(D._containers(cp)):
        chw = _seeded(case, 3, dt, seed=j)
        stacked = torch.from_numpy(np.stack(chw)).cuda()
        for flags in flag_sets:
            _check(engine, torch, cp, stacked, flags)                                       # one (n, C, H, W) tensor
        _check(engine, torch, cp, [torch.from_numpy(a).cuda() for a in chw], flag_sets[0])  # separate tensors
        if case[0] % 4 == 0:
            hwc = torch.from_numpy(np.ascontiguousarray(np.stack(chw).transpose(0, 2, 3, 1))).cuda()
            _check(engine, torch, cp, hwc, flag_sets[1], layout="HWC")
        if cp.numcomps == 3:
            rgba = []
            for a in chw:
                t = np.full(a.shape[1:] + (4,), 7, dt)
                t[..., :3] = a.transpose(1, 2, 0)
                rgba.append(torch.from_numpy(t).cuda()[..., :3])
            _check(engine, torch, cp, rgba, flag_sets[2], layout="HWC")


@pytest.mark.parametrize("case", [(0, False), (4, False), (8, False), (17, False)])
def test_round_trip(engine, case):
    """the batch's streams decode, through decode_codestreams_device, to the sources"""
    torch = pytest.importorskip("torch")
    cp, _ = D._case(*case)
    chw = np.stack(_seeded(case, 4, np.int32 if cp.sgnd else np.uint16))
    streams, status = engine.encode_codestreams_device(cp, torch.from_numpy(chw).cuda(), G.CS_TLM | G.CS_PLT)
    assert all(rc == 0 for rc, _ in status)
    _, out, dstatus = engine.decode_codestreams_device(streams, dtype=torch.int32)
    assert all(rc == 0 for rc, _ in dstatus)
    assert np.array_equal(out.cpu().numpy(), chw.astype(np.int32))


def test_mixed_batch(engine):
    """host-memory and misaligned images between good ones get the single call's code and text; the good streams are
    those of their single calls"""
    torch = pytest.importorskip("torch")
    case = (2, False)
    cp, _ = D._case(*case)
    chw = _seeded(case, 5, np.uint16)
    good = [torch.from_numpy(a).cuda() for a in chw]
    h, w, nc = cp.y1 - cp.y0, cp.x1 - cp.x0, cp.numcomps
    descs = [G.device_planes(t, nc, h, w) for t in good]
    host = chw[1].copy()
    descs[1] = G.device_planes(good[1], nc, h, w)
    for c in range(nc):                                            # the same image in host memory
        descs[1].comp[c] = host.ctypes.data + c * host.strides[0]
    bad = torch.zeros(h * w * nc + 8, dtype=torch.uint16, device="cuda")
    descs[3] = G.device_planes(good[3], nc, h, w)
    descs[3].comp[1] = bad.data_ptr() + 1                          # not a multiple of sample_bytes
    singles = [_single(engine, torch, cp, d, G.CS_TLM | G.CS_PLT) for d in descs]
    assert [s[0] for s in singles] == [0, -1, 0, -1, 0]
    rc, status, got, offsets = _raw_batch(engine, torch, cp, descs, G.CS_TLM | G.CS_PLT)
    assert rc == 2
    for i in range(5):
        assert status[i] == singles[i][:2], (i, status[i], singles[i][:2])
        if singles[i][0] == 0:
            assert np.array_equal(got[i], singles[i][2]), i
    assert status[3][1] == "device image component 1: address not a multiple of sample_bytes"
    # the good streams alone, as a batch of three: the same bytes, packed closer
    rc, alone, got3, _ = _raw_batch(engine, torch, cp, [descs[0], descs[2], descs[4]], G.CS_TLM | G.CS_PLT)
    assert rc == 0 and all(np.array_equal(a, b) for a, b in zip(got3, [got[0], got[2], got[4]]))


def test_verdicts_of_the_coding_and_flags(engine):
    """an 8-bit container under a 12-bit coding, flags whose progression order the writer does not know, and a tile grid
    the writer declines: every image gets the single call's verdict and text, and the call returns n"""
    torch = pytest.importorskip("torch")
    cp, _ = D._case(1, False)                                      # prec 12
    imgs = [torch.from_numpy(a).cuda() for a in _seeded((1, False), 3, np.uint8)]
    status = _check(engine, torch, cp, imgs, G.CS_TLM | G.CS_PLT, via_api=False)
    assert all(rc == 1 and "8-bit containers" in text for rc, text in status)
    _, api = engine.encode_codestreams_device(cp, imgs)
    assert api == status
    # the writer's plan declines: progression order 5, and 264 x 256 tiles of one sample (more than 65535)
    grid = G.make_coding(264, 256, 1, 8, numres=1, tile=(1, 1))
    for cp, flags in ((D._case(0, False)[0], G.CS_PROG(5) | G.CS_PLT), (grid, G.CS_TLM)):
        h, w = cp.y1 - cp.y0, cp.x1 - cp.x0
        g = torch.Generator(device="cuda").manual_seed(5)
        imgs = torch.randint(0, 256, (3, 1, h, w), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8)
        descs = [G.device_planes(imgs[i], 1, h, w) for i in range(3)]
        single = _single(engine, torch, cp, descs[0], flags)
        assert single[0] == -1 and single[1], single
        rc, status, got, _ = _raw_batch(engine, torch, cp, descs, flags)
        assert rc == 3 and status == [single[:2]] * 3 and got == [None] * 3, (rc, status)
        streams, api = engine.encode_codestreams_device(cp, imgs, flags)
        assert api == status and streams == [None] * 3


def test_whole_call_failures(engine):
    torch = pytest.importorskip("torch")
    cp, _ = D._case(0, False)
    h, w, nc = cp.y1 - cp.y0, cp.x1 - cp.x0, cp.numcomps
    a = torch.zeros((nc, h, w), dtype=torch.uint8, device="cuda")
    b = torch.zeros((nc, h, w), dtype=torch.uint16, device="cuda")
    rc, *_ = _raw_batch(engine, torch, cp, [G.device_planes(a, nc, h, w), G.device_planes(b, nc, h, w)], 0)
    assert rc < 0 and G.lib().b2k_last_error().decode() == "b2k_encode_codestreams_device: the images' sample_bytes differ"
    with pytest.raises(G.EngineError):
        engine.encode_codestreams_device(cp, [a, b])
    with pytest.raises(ValueError):
        engine.encode_codestreams_device(cp, [])
    L = G.lib()
    st = (C.c_int32 * 1)()
    assert L.b2k_encode_codestreams_device(engine._h, C.byref(cp), 0, None, 0, None, None, None, None, st, None) < 0


def _small(torch, n, size=64, seed=0):
    cp = G.make_coding(size, size, 3, 8, numres=3, cblk=(32, 32))
    g = torch.Generator(device="cuda").manual_seed(seed)
    imgs = torch.randint(0, 256, (n, 3, size, size), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8)
    return cp, imgs


def test_hundreds_of_small_images(engine):
    torch = pytest.importorskip("torch")
    cp, imgs = _small(torch, 300)
    streams, status = engine.encode_codestreams_device(cp, imgs, G.CS_PLT)
    assert all(rc == 0 for rc, _ in status)
    for i in range(0, 300, 7):
        want = engine.encode_codestream_device(cp, imgs[i], G.CS_PLT, device_output=True)
        assert torch.equal(streams[i], want), i
    _, out, dstatus = engine.decode_codestreams_device(streams, dtype=torch.uint8)
    assert all(rc == 0 for rc, _ in dstatus) and torch.equal(out, imgs)


def test_launches_do_not_grow_with_the_batch(engine):
    torch = pytest.importorskip("torch")
    L = G.lib()
    counts = []
    for n in (64, 160):
        cp, imgs = _small(torch, n, seed=n)
        engine.encode_codestreams_device(cp, imgs, G.CS_TLM)            # plan / grow once
        before = L.b2k_launch_count()
        streams, status = engine.encode_codestreams_device(cp, imgs, G.CS_TLM)
        counts.append(L.b2k_launch_count() - before)
        assert all(rc == 0 for rc, _ in status)
    assert counts[0] == counts[1], counts


def test_images_written_late_on_a_side_stream(engine):
    torch = pytest.importorskip("torch")
    cp, imgs = _small(torch, 6, seed=3)
    want, _ = engine.encode_codestreams_device(cp, imgs)
    want = [s.clone() for s in want]
    late = torch.zeros_like(imgs)
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        late.copy_(imgs)                                         # the samples arrive late, on the side stream
        streams, status = engine.encode_codestreams_device(cp, late, stream=side)
        late.zero_()                                             # queued after the call: must not reach the coder
    side.synchronize()
    assert all(rc == 0 for rc, _ in status)
    assert all(torch.equal(a, b) for a, b in zip(streams, want))


def test_one_engine_alternates():
    """batch encode, single device encode, batch decode of the batch's output, single device decode, a larger batch (the
    output buffer grows) and a batch of another coding, on one engine; a pointer the single call returned keeps its bytes"""
    torch = pytest.importorskip("torch")
    eng = G.Engine(0)
    try:
        L = G.lib()
        cp_a, imgs_a = _small(torch, 12, seed=1)
        cp_b, imgs_b = _small(torch, 5, size=96, seed=2)
        ref_a = [eng.encode_codestream_device(cp_a, imgs_a[i], G.CS_TLM | G.CS_PLT, device_output=True) for i in range(12)]
        ref_b = [eng.encode_codestream_device(cp_b, imgs_b[i], G.CS_TLM | G.CS_PLT, device_output=True) for i in range(5)]
        img = G.device_planes(imgs_a[0], 3, 64, 64)
        ptr = C.c_void_p()
        n = L.b2k_encode_codestream_device(eng._h, C.byref(cp_a), C.byref(img), G.CS_TLM | G.CS_PLT, None, C.byref(ptr))
        torch.cuda.synchronize()
        held = _bytes(torch, ptr.value, n)
        for _ in range(2):
            streams, status = eng.encode_codestreams_device(cp_a, imgs_a[:7])
            assert all(rc == 0 for rc, _ in status) and all(torch.equal(s, r) for s, r in zip(streams, ref_a))
            assert np.array_equal(_bytes(torch, ptr.value, n), held)            # the single call's buffer is untouched
            assert torch.equal(eng.encode_codestream_device(cp_a, imgs_a[3], G.CS_TLM | G.CS_PLT, device_output=True), ref_a[3])
            _, out, dstatus = eng.decode_codestreams_device(streams, dtype=torch.uint8)
            assert all(rc == 0 for rc, _ in dstatus) and torch.equal(out, imgs_a[:7])
            _, one = eng.decode_codestream_device(streams[2], dtype=torch.uint8)
            assert torch.equal(one, imgs_a[2])
            streams, _ = eng.encode_codestreams_device(cp_a, imgs_a)                # more streams: the buffer grows
            assert all(torch.equal(s, r) for s, r in zip(streams, ref_a))
            streams, _ = eng.encode_codestreams_device(cp_b, imgs_b)                # another coding
            assert all(torch.equal(s, r) for s, r in zip(streams, ref_b))
            n = L.b2k_encode_codestream_device(eng._h, C.byref(cp_a), C.byref(img), G.CS_TLM | G.CS_PLT, None, C.byref(ptr))
            torch.cuda.synchronize()
            held = _bytes(torch, ptr.value, n)
    finally:
        eng.close()


def test_one_image_equals_the_single_call(engine):
    torch = pytest.importorskip("torch")
    cp, imgs = _small(torch, 1, seed=9)
    for flags in DC.FLAGS:
        _check(engine, torch, cp, imgs, flags)


def test_large_batch(engine):
    """64 x 1024^2 x 3, 12 bit, TLM + PLT"""
    torch = pytest.importorskip("torch")
    cp = G.make_coding(1024, 1024, 3, 12, numres=6)
    g = torch.Generator(device="cuda").manual_seed(64)
    base = torch.randint(0, 4096, (3, 1024, 1024), dtype=torch.int32, device="cuda", generator=g)
    ramp = torch.arange(1024, device="cuda", dtype=torch.int32)
    imgs = torch.stack([((base >> (k % 5)) + ramp * k + ramp[:, None]) % 4096 for k in range(64)]).to(torch.int16)
    streams, status = engine.encode_codestreams_device(cp, imgs, G.CS_TLM | G.CS_PLT)
    assert all(rc == 0 for rc, _ in status)
    for i in (0, 1, 31, 63):
        want = engine.encode_codestream_device(cp, imgs[i], G.CS_TLM | G.CS_PLT, device_output=True)
        assert torch.equal(streams[i], want), i
    _, out, dstatus = engine.decode_codestreams_device(streams, dtype=torch.int16)
    assert all(rc == 0 for rc, _ in dstatus) and torch.equal(out, imgs)
