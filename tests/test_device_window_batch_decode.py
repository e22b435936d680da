"""Batches of windows of code streams in device memory (b2k_decode_codestreams_window_device,
Engine.decode_windows_device).

Every stream of a batch must get what b2k_decode_codestream_window_device gives it alone with its window and the batch's
reduce: the same return code and text, the same rect and, where that is 0, the same pixels; a stream that fails leaves its
image alone, and nothing outside a rect is written.  The batch rules on top: the coding is the virtual coding of the first
stream whose header and window pass, and a stream of another virtual coding, tile box or progression / SOP / EPH gets 1.
The CPU suite (test_t2_window_batch_host.py) runs the parse steps under the sanitizers on random damage."""
import ctypes as C

import numpy as np
import pytest

import grok_b200 as G
import test_device_io as D
from test_device_batch_decode import SENTINEL, _dev, _base, _ht_reject, _seeded_streams, _small_batch

pytestmark = pytest.mark.gpu

RULE_BOX = ("code stream %d: its window's coding (tile grid, wanted tiles or virtual coding) differs from that of code "
            "stream %d, which the batch takes its coding from")


def _win(window):
    return (C.c_uint32 * 4)(*window) if window is not None else None


def _ptr(dcs):
    return (dcs.data_ptr(), dcs.numel()) if hasattr(dcs, "data_ptr") else (int(dcs.ctypes.data), len(dcs))


def _shape(engine, dcs, window, reduce):
    """(numcomps, h, w) of the window's rect from the header-only device parse, or None when it fails"""
    L = G.lib()
    cp = G.Coding()
    ptr, n = _ptr(dcs)
    rc = L.b2k_codestream_parse_window_device(engine._h, ptr, n, _win(window), reduce, None, C.byref(cp), None, 0)
    if rc < 1 or (rc == 1 and L.b2k_last_error()):
        return None
    x0, y0, x1, y1 = G.window_rect(cp, window, reduce)
    return cp.numcomps, y1 - y0, x1 - x0


def _single(engine, torch, dcs, window, reduce, layout="CHW", dtype=None):
    """(rc, text, rect, CHW image or None) of b2k_decode_codestream_window_device on one stream, called directly"""
    L = G.lib()
    nc, h, w = _shape(engine, dcs, window, reduce) or (1, 1, 1)
    out = torch.full((nc, h, w) if layout == "CHW" else (h, w, nc), SENTINEL, dtype=dtype or torch.uint16, device="cuda")
    img = G.device_planes(out, nc, h, w, layout, writable=True)
    ptr, n = _ptr(dcs)
    cp, rect, ms = G.Coding(), (C.c_uint32 * 4)(), C.c_double()
    rc = L.b2k_decode_codestream_window_device(engine._h, ptr, n, _win(window), reduce, C.byref(img), None, C.byref(cp), rect,
                                               C.byref(ms))
    torch.cuda.synchronize()
    text = (L.b2k_last_error() or b"").decode() if rc else ""
    return rc, text, tuple(rect) if rc == 0 else None, (D._to_chw(out, layout) if rc == 0 else None)


def _check(engine, torch, streams, windows, reduce, layout="CHW", dtype=None, rules=None):
    """each stream's status, rect and pixels against its single call, into sentinel-filled outputs one size larger than
    its rect (so that a write outside the rect shows); rules: {index: (rc, text)} the batch rules decide"""
    rules = rules or {}
    n = len(streams)
    ws = [None] * n if windows is None else [windows] * n if len(windows) == 4 and np.isscalar(windows[0]) else list(windows)
    singles = [_single(engine, torch, s, w, reduce, layout, dtype) for s, w in zip(streams, ws)]
    if all(_shape(engine, s, w, reduce) is None for s, w in zip(streams, ws)):
        # no stream has a header and window that pass: the batch has no coding and raises with stream 0's text
        with pytest.raises((G.NotHandled, G.EngineError)) as err:
            engine.decode_windows_device(streams, windows, reduce, layout=layout)
        assert str(err.value).endswith(singles[0][1])
        return None, [s[:2] for s in singles]
    big, outs = [], []
    for s, w in zip(streams, ws):
        nc, h, wd = _shape(engine, s, w, reduce) or (1, 1, 1)
        t = torch.full((nc, h + 1, wd + 1) if layout == "CHW" else (h + 1, wd + 1, nc), SENTINEL, dtype=dtype or torch.uint16,
                       device="cuda")
        big.append(t)
        outs.append(t[:, :h, :wd] if layout == "CHW" else t[:h, :wd, :])
    cp, _, rects, status = engine.decode_windows_device(streams, windows, reduce, out=outs, layout=layout)
    torch.cuda.synchronize()
    for i, ((rc, text, rect, img), (brc, btext)) in enumerate(zip(singles, status)):
        assert (brc, btext) == rules.get(i, (rc, text)), (i, (brc, btext), rules.get(i, (rc, text)))
        full = D._to_chw(big[i], layout)
        if brc == 0:
            assert rects[i] == rect, (i, rects[i], rect)
            assert np.array_equal(full[:, :-1, :-1], img), "stream %d: pixels differ" % i
            assert (full[:, -1, :] == SENTINEL).all() and (full[:, :, -1] == SENTINEL).all(), "stream %d: written past its rect" % i
        else:
            assert (full == SENTINEL).all(), "stream %d failed (%d) but its image was written" % (i, brc)
    return cp, status


def _seeded_windows(cp, rng, n):
    out = []
    for _ in range(n):
        a, b = sorted(int(v) for v in rng.integers(cp.x0, cp.x1 + 1, 2))
        c, d = sorted(int(v) for v in rng.integers(cp.y0, cp.y1 + 1, 2))
        out.append((a, c, max(b, a + 1), max(d, c + 1)))
    return out


@pytest.mark.parametrize("case", D.CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in D.CASES])
def test_geometries(engine, case):
    """per-stream seeded windows (tiled streams whose windows touch another box take the rule) and one shared window,
    reduce 0-2, every container; HWC too on every fourth geometry"""
    torch = pytest.importorskip("torch")
    cp, streams = _seeded_streams(engine, case)
    dstreams = [_dev(torch, s) for s in streams]
    rng = np.random.default_rng(3000 + case[0] * 2 + case[1])
    for r in range(3):
        per = _seeded_windows(cp, rng, len(dstreams))
        shared = _seeded_windows(cp, rng, 1)[0]
        for k, dt in enumerate(D._containers(cp)):
            tdt = getattr(torch, np.dtype(dt).name)
            for layout in (("CHW", "HWC") if case[0] % 4 == 0 else ("CHW",)):
                _, status = _check(engine, torch, dstreams, per if (k + r) % 2 == 0 else shared, r, layout, tdt,
                                   rules=_box_rules(engine, dstreams, per if (k + r) % 2 == 0 else [shared] * len(dstreams), r))
                assert status[0][0] in (0, 1, -1)


def _box_rules(engine, streams, windows, reduce):
    """the batch rule's verdicts for streams whose window's coding differs from the reference stream's"""
    L = G.lib()
    codings = []
    for s, w in zip(streams, windows):
        cp = G.Coding()
        ptr, n = _ptr(s)
        rc = L.b2k_codestream_parse_window_device(engine._h, ptr, n, _win(w), reduce, None, C.byref(cp), None, 0)
        codings.append(bytes(cp) if rc > 1 or (rc == 1 and not L.b2k_last_error()) else None)
    ref = next((i for i, c in enumerate(codings) if c is not None), None)
    if ref is None:
        return {}
    return {i: (1, RULE_BOX % (i, ref)) for i, c in enumerate(codings) if i > ref and c is not None and c != codings[ref]}


def test_thumbnails_and_the_whole_case(engine):
    """windows=None at reduce 0-2 (thumbnails), and single-tile streams at reduce 0 with per-stream crops (the virtual
    coding is the streams' own: the whole-stream parse)"""
    torch = pytest.importorskip("torch")
    cp, streams = _seeded_streams(engine, (9, False), count=6)
    dstreams = [_dev(torch, s) for s in streams]
    for r in range(3):
        _, status = _check(engine, torch, dstreams, None, r)
        assert all(rc == 0 for rc, _ in status)
    rng = np.random.default_rng(11)
    one = G.make_coding(96, 80, 3, 8, numres=4, cblk=(32, 32))
    g = torch.Generator(device="cuda").manual_seed(3)
    imgs = torch.randint(0, 256, (6, 3, 80, 96), dtype=torch.int32, device="cuda", generator=g).to(torch.uint8)
    single_tile = [engine.encode_codestream_device(one, imgs[i], G.CS_PLT, device_output=True) for i in range(6)]
    crops = _seeded_windows(one, rng, 6)
    _, status = _check(engine, torch, single_tile, crops, 0, dtype=torch.uint8)
    assert all(rc == 0 for rc, _ in status)
    tiles, nbytes = engine.codestream_window_device_stats()
    assert tiles == 1 and nbytes == sum(s.numel() for s in single_tile)   # whole streams, as each single call copies
    _, out, rects, _ = engine.decode_windows_device(single_tile, crops, dtype=torch.uint8)
    for i, (x0, y0, x1, y1) in enumerate(rects):
        assert torch.equal(out[i], imgs[i][:, y0:y1, x0:x1])


def test_mixed_batch(engine):
    """good streams interleaved with the single call's damage cases, another coding, another box, no bytes, host memory
    and a bad image descriptor"""
    torch = pytest.importorskip("torch")
    good, edits = _base(engine)                                  # 12 tiles; a window on tile 0
    w = (2, 2, 30, 30)
    streams, ws, rules = [], [], {}
    for name, cs in edits.items():
        streams += [_dev(torch, good), _dev(torch, cs)]
        ws += [w, w]
    other = D._host_result(engine, 9, False)
    streams.append(_dev(torch, G.codestream_write(other[0], other[2], other[3], G.CS_TLM | G.CS_PLT)))
    ws.append(w)
    rules[len(streams) - 1] = (1, RULE_BOX % (len(streams) - 1, 0))
    streams.append(_dev(torch, good))                            # another tile box
    ws.append((200, 150, 260, 200))
    rules[len(streams) - 1] = (1, RULE_BOX % (len(streams) - 1, 0))
    streams.append(torch.zeros(0, dtype=torch.uint8, device="cuda"))
    ws.append(w)
    streams.append(_dev(torch, good))
    ws.append((1, 1, 9, 9))
    _check(engine, torch, streams, ws, 0, rules=rules)
    # the stream has one resolution: at reduce 1 every window of it fails on its own, and the other coding is the batch's
    _, status = _check(engine, torch, streams, ws, 1)
    assert status[-4][0] == 0 and status[0][0] == -1
    # host memory and a bad image descriptor, through the C ABI
    L = G.lib()
    host = np.array(good)
    d0 = _dev(torch, good)
    n = 3
    ptrs = (C.c_void_p * n)(d0.data_ptr(), host.ctypes.data, d0.data_ptr())
    lens = (C.c_uint64 * n)(len(good), len(good), len(good))
    win = (C.c_uint32 * 12)(*(list(w) * 3))
    nc, h, wd = _shape(engine, d0, w, 0)
    outs = [torch.full((nc, h, wd), SENTINEL, dtype=torch.uint16, device="cuda") for _ in range(n)]
    imgs = (G.DevicePlanes * n)(*[G.device_planes(o, nc, h, wd) for o in outs])
    bad = torch.zeros(1, dtype=torch.uint16, device="cuda")
    imgs[2].comp[1] = bad.data_ptr() + 1
    st, ms, bcp, rects = (C.c_int32 * n)(), C.c_double(), G.Coding(), (C.c_uint32 * 12)()
    assert L.b2k_decode_codestreams_window_device(engine._h, n, ptrs, lens, win, 0, imgs, None, C.byref(bcp), rects, st, C.byref(ms)) == 2
    torch.cuda.synchronize()
    want0 = _single(engine, torch, d0, w, 0)
    assert st[0] == 0 and np.array_equal(D._to_chw(outs[0], "CHW"), want0[3])
    host_rc = _single(engine, torch, host, w, 0)
    assert (st[1], L.b2k_decode_codestreams_error(engine._h, 1).decode()) == host_rc[:2]
    assert st[2] == -1 and L.b2k_decode_codestreams_error(engine._h, 2).decode() == \
        "device image component 1: address not a multiple of sample_bytes"
    assert (outs[1] == SENTINEL).all() and (outs[2][0] == SENTINEL).all()


def test_ht_decoder_rejection_is_per_stream(engine):
    torch = pytest.importorskip("torch")
    good, _ = _base(engine)
    bad, text = _ht_reject(engine, torch, good)
    streams = [_dev(torch, good), _dev(torch, bad), _dev(torch, good)]
    _, status = _check(engine, torch, streams, None, 0)
    assert [s[0] for s in status] == [0, -2, 0] and status[1][1] == text
    _, status = _check(engine, torch, streams, (0, 0, 40, 40), 0)    # a window: the rejected block may lie outside it
    assert status[0][0] == 0 and status[2][0] == 0


def test_headers_only_and_window_statistics(engine):
    torch = pytest.importorskip("torch")
    good, _ = _base(engine)
    L = G.lib()
    bad = good.copy()
    bad[0:2] = 0
    streams = [_dev(torch, bad), _dev(torch, good), _dev(torch, good), _dev(torch, good)]
    x0, y0 = G.codestream_parse(good)[0].x0, G.codestream_parse(good)[0].y0
    # all in the first tile; the stream has one resolution
    ws = [(x0, y0, x0 + 8, y0 + 8), (x0 + 3, y0 + 3, x0 + 40, y0 + 40), (x0 + 10, y0 + 10, x0 + 20, y0 + 20), (x0, y0, x0 + 1, y0 + 1)]
    n = len(streams)
    ptrs = (C.c_void_p * n)(*[s.data_ptr() for s in streams])
    lens = (C.c_uint64 * n)(*[s.numel() for s in streams])
    win = (C.c_uint32 * (4 * n))(*[v for w in ws for v in w])
    st, ms, cp, rects = (C.c_int32 * n)(), C.c_double(), G.Coding(), (C.c_uint32 * (4 * n))()
    assert L.b2k_decode_codestreams_window_device(engine._h, n, ptrs, lens, win, 0, None, None, C.byref(cp), rects, st, C.byref(ms)) == 1
    assert st[0] == -1 and list(st)[1:] == [0, 0, 0] and tuple(rects[0:4]) == (0, 0, 0, 0)
    want = G.codestream_parse_window(good, ws[1], 0)[0]
    assert bytes(cp) == bytes(want)
    for i in (1, 2, 3):
        assert tuple(rects[4 * i:4 * i + 4]) == G.window_rect(want, ws[i], 0)
    total = 0
    for s, w in zip(streams[1:], ws[1:]):
        engine.decode_window_device(s, window=w, reduce=0)
        total += engine.codestream_window_device_stats()[1]
    engine.decode_windows_device(streams, ws, 0)
    assert engine.codestream_window_device_stats() == (1, total)


def test_launches_do_not_grow_with_the_batch(engine):
    torch = pytest.importorskip("torch")
    counts = []
    for n in (64, 160):
        cp, imgs, streams = _small_batch(engine, torch, n, seed=n)
        engine.decode_windows_device(streams, (5, 7, 50, 41), 1, dtype=torch.uint8)   # plan / grow once
        L = G.lib()
        before = L.b2k_launch_count()
        _, out, _, status = engine.decode_windows_device(streams, (5, 7, 50, 41), 1, dtype=torch.uint8)
        counts.append(L.b2k_launch_count() - before)
        assert all(rc == 0 for rc, _ in status)
    assert counts[0] == counts[1], counts


def test_streams_filled_late_on_a_side_stream(engine):
    torch = pytest.importorskip("torch")
    cp, imgs, streams = _small_batch(engine, torch, 6)
    w = (10, 4, 60, 50)
    want = [engine.decode_window_device(s, window=w, reduce=1, dtype=torch.uint8)[1] for s in streams]
    side = torch.cuda.Stream()
    late = [torch.zeros_like(s) for s in streams]
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        for d, s in zip(late, streams):
            d.copy_(s)
        _, out, _, status = engine.decode_windows_device(late, w, 1, stream=side, dtype=torch.uint8)
        after = out.clone()
    side.synchronize()
    assert all(rc == 0 for rc, _ in status)
    assert torch.equal(after, torch.stack(want))


def test_one_engine_alternates(engine):
    """windowed batch, batch, single window and batch encode on one engine: results unchanged"""
    torch = pytest.importorskip("torch")
    cp, imgs, streams = _small_batch(engine, torch, 12, seed=4)
    w = (3, 9, 41, 60)
    want = torch.stack([engine.decode_window_device(s, window=w, reduce=1, dtype=torch.uint8)[1] for s in streams])
    for _ in range(2):
        _, out, _, _ = engine.decode_windows_device(streams, w, 1, dtype=torch.uint8)
        assert torch.equal(out, want)
        _, full, _ = engine.decode_codestreams_device(streams, dtype=torch.uint8)
        assert torch.equal(full, imgs)
        assert torch.equal(engine.decode_window_device(streams[2], window=w, reduce=1, dtype=torch.uint8)[1], want[2])
        again, status = engine.encode_codestreams_device(cp, imgs[:4], G.CS_PLT)
        assert all(rc == 0 for rc, _ in status)
        _, out, _, _ = engine.decode_windows_device(streams[:5], w, 1, dtype=torch.uint8)
        assert torch.equal(out, want[:5])


def test_hundreds_of_small_streams(engine):
    torch = pytest.importorskip("torch")
    cp, imgs, streams = _small_batch(engine, torch, 300)
    rng = np.random.default_rng(300)
    ws = _seeded_windows(cp, rng, 300)
    _, out, rects, status = engine.decode_windows_device(streams, ws, 0, dtype=torch.uint8)
    assert all(rc == 0 for rc, _ in status)
    for i, (x0, y0, x1, y1) in enumerate(rects):
        assert torch.equal(out[i], imgs[i][:, y0:y1, x0:x1])
    _, out, _, status = engine.decode_windows_device(streams, None, 1, dtype=torch.uint8)
    want = torch.stack([engine.decode_window_device(s, reduce=1, dtype=torch.uint8)[1] for s in streams[:20]])
    assert torch.equal(out[:20], want)
