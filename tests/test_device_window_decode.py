"""Windows and reduced resolutions of code streams in device memory (b2k_codestream_parse_window_device /
b2k_decode_codestream_window_device, Engine.codestream_parse_window_device / Engine.decode_window_device).

For every input the device path must give what copying the stream to the host and calling b2k_codestream_parse_window +
b2k_decode_device gives: the same return code and b2k_last_error text, the same virtual coding and block table, the same
pixels.  The CPU suite (test_t2_window_host.py) runs the same steps under the sanitizers on random damage; here the
device-I/O suite's geometries and flag sets, seeded windows, fixed damage cases, ordering, reuse and a large image run
once on the GPU."""
import ctypes as C

import numpy as np
import pytest

import grok_b200 as G
import test_device_io as D
from test_device_codestream import FLAGS
from test_device_codestream_decode import _dev, _same_coding, _base_stream, _sots

pytestmark = pytest.mark.gpu


def _win(window):
    return (C.c_uint32 * 4)(*window) if window is not None else None


def _host_parse(cs, window, reduce):
    """b2k_codestream_parse_window on host bytes: (rc, text, Coding, table)"""
    L = G.lib()
    cs = np.ascontiguousarray(cs, np.uint8)
    cp = G.Coding()
    n = L.b2k_codestream_parse_window(cs.ctypes.data, len(cs), _win(window), reduce, C.byref(cp), None, 0)
    if n <= 1:
        return n, L.b2k_last_error().decode(), cp, None
    blocks = np.zeros(n, G.BLOCK_DTYPE)
    m = L.b2k_codestream_parse_window(cs.ctypes.data, len(cs), _win(window), reduce, C.byref(cp), blocks.ctypes.data, n)
    return m, L.b2k_last_error().decode() if m <= 1 else "", cp, blocks


def _dev_parse(engine, dcs, window, reduce, cap=None):
    """b2k_codestream_parse_window_device on a CUDA tensor: (rc, text, Coding, table)"""
    L = G.lib()
    cp = G.Coding()
    n = L.b2k_codestream_parse_window_device(engine._h, dcs.data_ptr(), dcs.numel(), _win(window), reduce, None, C.byref(cp), None, 0)
    if n <= 1:
        return n, L.b2k_last_error().decode(), cp, None
    blocks = np.zeros(n, G.BLOCK_DTYPE)
    m = L.b2k_codestream_parse_window_device(engine._h, dcs.data_ptr(), dcs.numel(), _win(window), reduce, None, C.byref(cp),
                                             blocks.ctypes.data, n if cap is None else cap)
    return m, L.b2k_last_error().decode() if m <= 1 else "", cp, blocks


def _check_parse(engine, cs, dcs, window, reduce):
    h, d = _host_parse(cs, window, reduce), _dev_parse(engine, dcs, window, reduce)
    assert h[0] == d[0], (window, reduce, h[:2], d[:2])
    if h[0] <= 1:
        assert h[1] == d[1], (window, reduce)
        return h[0]
    _same_coding(h[2], d[2])
    assert h[3].tobytes() == d[3].tobytes(), (window, reduce)
    return h[0]


def _outcome(fn):
    try:
        return "ok", fn()
    except G.NotHandled as e:
        return "NotHandled", str(e).split(": ", 1)[1]
    except G.EngineError as e:
        return "EngineError", str(e).split(": ", 1)[1]


def _check_pixels(engine, torch, cs, dcs, window, reduce, dtypes, layouts=("CHW",)):
    """decode_window_device against today's path from host bytes, for each container and layout"""
    for dt in dtypes:
        tdt = getattr(torch, np.dtype(dt).name)
        for layout in layouts:
            want = _outcome(lambda: engine.decode_codestream_device(cs, dtype=tdt, layout=layout, window=window, reduce=reduce))
            got = _outcome(lambda: engine.decode_window_device(dcs, window=window, reduce=reduce, dtype=tdt, layout=layout))
            assert (want[0] == "ok") == (got[0] == "ok"), (window, reduce, want, got)
            if want[0] != "ok":   # the host wrapper raises EngineError("<rc> <text>") for every failed parse
                assert want[1].endswith(got[1]), (want, got)
                continue
            _same_coding(want[1][0], got[1][0])
            a, b = D._to_chw(want[1][1], layout), D._to_chw(got[1][1], layout)
            assert np.array_equal(a, b), "pixels differ: %s %s %s %d" % (np.dtype(dt).name, layout, window, reduce)


def _windows(cp, rng):
    """a one-tile corner, a window across the first tile corner, a seeded one"""
    x0, y0, x1, y1 = cp.x0, cp.y0, cp.x1, cp.y1
    cx = min(x1 - 1, cp.tx0 + cp.tw) if cp.tw and cp.tx0 + cp.tw < x1 else (x0 + x1) // 2
    cy = min(y1 - 1, cp.ty0 + cp.th) if cp.th and cp.ty0 + cp.th < y1 else (y0 + y1) // 2
    a, b = sorted(int(v) for v in rng.integers(x0, x1 + 1, 2))
    c, d = sorted(int(v) for v in rng.integers(y0, y1 + 1, 2))
    return [(x0, y0, x0 + 2, y0 + 2), (max(x0, cx - 5), max(y0, cy - 5), min(x1, cx + 5), min(y1, cy + 5)),
            (a, c, max(b, a + 1), max(d, c + 1))]


def _parts(cs):
    """(tile, packet-data bytes) of every tile part, from the SOTs"""
    cs = bytes(cs)
    out = []
    for p in _sots(np.frombuffer(cs, np.uint8)):
        psot = int.from_bytes(cs[p + 6:p + 10], "big")
        q = p + 12
        while cs[q:q + 2] != b"\xff\x93":
            q += 2 + int.from_bytes(cs[q + 2:q + 4], "big")
        out.append((int.from_bytes(cs[p + 4:p + 6], "big"), p + psot - (q + 2)))
    return out


def _wanted_tiles(cp, window, reduce):
    """the stream's tiles a window touches (every tile without one)"""
    tw, th = cp.tw or cp.x1 - cp.tx0, cp.th or cp.y1 - cp.ty0
    nx = -(-(cp.x1 - cp.tx0) // tw)
    ny = -(-(cp.y1 - cp.ty0) // th)
    if window is None:
        return {t for t in range(nx * ny)}
    wx0, wy0, wx1, wy1 = max(window[0], cp.x0), max(window[1], cp.y0), min(window[2], cp.x1), min(window[3], cp.y1)
    xs = range((wx0 - cp.tx0) // tw, -(-(wx1 - cp.tx0) // tw))
    ys = range((wy0 - cp.ty0) // th, -(-(wy1 - cp.ty0) // th))
    return {y * nx + x for y in ys for x in xs}


@pytest.mark.parametrize("case", D.CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in D.CASES])
def test_host_written_streams(engine, case):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, _ = D._host_result(engine, *case)
    rng = np.random.default_rng(1000 + case[0] * 2 + case[1])
    ws = _windows(cp, rng)
    every = _wanted_tiles(cp, None, 0)
    for fi, flags in enumerate(FLAGS):
        try:
            cs = np.array(G.codestream_write(cp, blocks, data, flags))
        except G.EngineError:
            continue
        dcs = _dev(torch, cs)
        for wi, w in enumerate(ws):
            for r in range(3):
                rc = _check_parse(engine, cs, dcs, w, r)
                if rc <= 1:
                    continue
                ntiles, nbytes = engine.codestream_window_device_stats()
                want = _wanted_tiles(cp, w, r)
                assert ntiles == len(want)
                if want == every and r == 0:   # the stream's own coding: the whole stream is copied
                    assert nbytes == len(cs)
                else:                          # only the wanted tiles' packet data
                    assert nbytes == sum(n for t, n in _parts(cs) if t in want), (w, r)
                if (fi + wi + r) % 4 == 0:
                    _check_pixels(engine, torch, cs, dcs, w, r, [D._containers(cp)[0]])
        if fi == 0:
            for w in ws[:2]:
                _check_pixels(engine, torch, cs, dcs, w, 1, D._containers(cp), ("CHW", "HWC"))
                _check_pixels(engine, torch, cs, dcs, w, 0, D._containers(cp)[-1:], ("CHW", "HWC"))
            _check_pixels(engine, torch, cs, dcs, None, 1, D._containers(cp)[:1])
            _check_pixels(engine, torch, cs, dcs, (cp.x0, cp.y0, cp.x1, cp.y1), 0, D._containers(cp)[:1])


def test_errors_and_their_order(engine):
    torch = pytest.importorskip("torch")
    cs = _base_stream(engine)                                  # 12 tiles of 64 x 64
    dcs = _dev(torch, cs)
    cp = G.codestream_parse(cs)[0]
    for w, r in [((cp.x1 + 1, 0, cp.x1 + 5, 5), 0), ((0, 0, 8, 8), cp.numres), ((0, 0, 100, 100), 7), (None, cp.numres + 3),
                 ((0, 0, 8, 8), 0)]:
        _check_parse(engine, cs, dcs, w, r)
    # the caller's table is checked before any tile part is read
    b = cs.copy()
    b[_sots(cs)[0] + 2] = 0xAA                                 # a bad SOT in tile 0
    db = _dev(torch, b)
    assert _host_parse(b, (0, 0, 8, 8), 0)[:2] == _dev_parse(engine, db, (0, 0, 8, 8), 0)[:2]
    rc, text, _, _ = _dev_parse(engine, db, (0, 0, 8, 8), 0, cap=1)
    assert rc == -1 and text == "block table too small"


def test_damage_inside_and_outside_the_window(engine):
    """damage in a tile outside the window passes unless it is in an SOT; inside the window it fails as on the host"""
    torch = pytest.importorskip("torch")
    cs = _base_stream(engine)                                  # 333 x 217 from (3, 5) in 100 x 90 tiles, one resolution
    cp = G.codestream_parse(cs)[0]
    last = _sots(cs)[-1]                                       # tile 11, the bottom-right one
    sod = int(np.flatnonzero((cs[last:-1] == 0xFF) & (cs[last + 1:] == 0x93))[0]) + last
    edits = {}
    b = cs.copy()
    b[sod + 2:sod + 10] = 0xFF
    edits["packet"] = b
    b = cs.copy()
    b[last + 14:last + 16] = 0xFF                              # the PLT segment's length
    edits["tp_header"] = b
    b = cs.copy()
    b[last + 2:last + 4] = [0, 11]
    edits["sot"] = b
    outside, inside = (0, 0, 8, 8), (cp.x1 - 8, cp.y1 - 8, cp.x1, cp.y1)
    for name, b in edits.items():
        db = _dev(torch, b)
        for w in (outside, inside):
            rc = _check_parse(engine, b, db, w, 0)
            if w == outside:
                assert (rc > 1) == (name != "sot"), (name, rc)
            else:
                assert rc <= 1, name
            _check_pixels(engine, torch, b, db, w, 0, [np.int32])


def test_stream_ordering(engine):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, _ = D._host_result(engine, 1, False)     # 2048 x 1024 in 1024^2 tiles
    cs = np.array(G.codestream_write(cp, blocks, data, G.CS_TLM | G.CS_PLT))
    w = (900, 500, 1200, 700)                                              # both tiles
    _, want = engine.decode_codestream_device(cs, dtype=torch.int32, window=w, reduce=1)
    side = torch.cuda.Stream()
    dcs = torch.zeros(len(cs), dtype=torch.uint8, device="cuda")
    src = torch.from_numpy(cs).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        dcs.copy_(src)                                         # the bytes arrive late, on the side stream
        _, got = engine.decode_window_device(dcs, window=w, reduce=1, dtype=torch.int32, stream=side)
        after = got.clone()                                    # queued after the call: must see the pixels
    side.synchronize()
    assert torch.equal(after, want)


def test_one_engine_reused(engine):
    """full device decode, windowed decode and device encode alternate on one engine"""
    torch = pytest.importorskip("torch")
    small = D._host_result(engine, 9, False)
    big = D._host_result(engine, 1, False)
    streams = {"small": np.array(G.codestream_write(small[0], small[2], small[3], G.CS_TLM | G.CS_PLT)),
               "big": np.array(G.codestream_write(big[0], big[2], big[3], G.CS_SOP | G.CS_EPH | G.CS_PROG(2)))}
    ws = [((0, 0, 40, 40), 0), ((30, 20, 180, 120), 1), (None, 2)]
    want = {}
    for name, cs in streams.items():
        want[name] = engine.decode_codestream_device(cs, dtype=torch.int32)[1].cpu()
        for w, r in ws:
            want[name, w, r] = engine.decode_codestream_device(cs, dtype=torch.int32, window=w, reduce=r)[1].cpu()
    for step in range(2):
        for name, cs in streams.items():
            dcs = _dev(torch, cs)
            for w, r in ws:
                _, got = engine.decode_window_device(dcs, window=w, reduce=r, dtype=torch.int32)
                assert torch.equal(got.cpu(), want[name, w, r]), (name, w, r)
                _, got = engine.decode_codestream_device(dcs, dtype=torch.int32)
                assert torch.equal(got.cpu(), want[name]), name
            cp, planes = (small if name == "small" else big)[:2]
            img = torch.from_numpy(np.stack(planes).astype(D._containers(cp)[0])).cuda()
            engine.encode_codestream_device(cp, img, device_output=True)
            _, got = engine.decode_window_device(dcs, window=ws[1][0], reduce=ws[1][1], dtype=torch.int32)
            assert torch.equal(got.cpu(), want[name, ws[1][0], ws[1][1]]), name
    assert engine.codestream_window_device_stats()[0] >= 1


def test_large_image_window_against_the_generator(engine):
    """16384^2 x 3, 12 bit, 1024^2 tiles, TLM + PLT, in device memory: a window over 3 x 3 tiles equals the generator's
    pixels, and only those tiles' packet data are copied"""
    torch = pytest.importorskip("torch")
    n, tile = 16384, 1024
    cp = G.make_coding(n, n, 3, 12, numres=6, tile=(tile, tile))
    g = torch.Generator(device="cuda").manual_seed(5)
    img = torch.randint(0, 1 << 12, (3, n, n), dtype=torch.int32, device="cuda", generator=g).to(torch.uint16)
    cs = engine.encode_codestream_device(cp, img, G.CS_TLM | G.CS_PLT, device_output=True)
    w = (5 * tile - 700, 7 * tile - 300, 7 * tile - 100, 9 * tile - 5)     # tile columns 4-6, rows 6-8
    vcp, out = engine.decode_window_device(cs, window=w)
    assert torch.equal(out, img[:, w[1]:w[3], w[0]:w[2]])
    ntiles, nbytes = engine.codestream_window_device_stats()
    assert ntiles == 9 and nbytes < cs.numel() // 20        # 9 of the 256 tiles
    host = cs.cpu().numpy()
    assert nbytes == sum(b for t, b in _parts(host) if t in _wanted_tiles(cp, w, 0))
    _, red = engine.decode_window_device(cs, window=w, reduce=2)
    _, ref = engine.decode_codestream_device(host, window=w, reduce=2)
    assert torch.equal(red, ref)
