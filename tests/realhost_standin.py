"""The checks of tests/test_realhost.py where Grok's host library is not built (it comes from the reference sources,
oracle/build_ref.sh).  The host is replaced by what it does with the plugin loaded: plugin_init, the coding the stock
entry points derive from the host's parameters, the plugin's code blocks written as a code stream, the code stream
decoded through plugin_decompress_codestream.  What the host's own CPU path gives -- its code streams and its decodes --
comes from the record in tests/golden/ (tests/grok_golden.py), so "the code stream through the plugin equals the
host's own" and "the pixels equal the host's" are checked against the real host's outputs."""
import ctypes as C

import numpy as np

import grok_b200 as G
import grok_golden as GG
import grok_ref as R
import oracle_pipeline as P
from gpup_ctypes import GpupImage, GpupImageComp
from grok_golden import grok


class InitInfo(C.Structure):
    _fields_ = [("deviceId", C.c_int32), ("verbose", C.c_bool), ("license", C.c_char_p), ("server", C.c_char_p)]


def plugin_init(device=0):
    """the host's grk_plugin_init: the plugin's plugin_init(gpup_init_info), True when a device engine is up"""
    lib = G.lib()
    for s in ("minpf_post_load_plugin", "plugin_init", "plugin_get_debug_state", "gpup_encode_mem", "gpup_tile_free",
              "plugin_decompress", "gpup_batch_memory_begin", "plugin_batch_decompress_memory_begin"):
        assert hasattr(lib, s), s
    lib.plugin_init.argtypes = [InitInfo]
    lib.plugin_init.restype = C.c_bool
    return bool(lib.plugin_init(InitInfo(device, False, None, None)))


def plugin_decompress(cs, w, h, n):
    """plugin_decompress_codestream into host-allocated int32 planes -> (rc, planes)"""
    lib = G.lib()
    out = [np.zeros((h, w), np.int32) for _ in range(n)]
    comps = (GpupImageComp * n)(*[GpupImageComp(0, 0, w, w, h, 1, 1, 0, False, o.ctypes.data_as(C.POINTER(C.c_int32)), False)
                                  for o in out])
    img = GpupImage(0, 0, w, h, n, 0, C.cast(comps, C.POINTER(GpupImageComp)))
    lib.plugin_decompress_codestream.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(GpupImage)]
    cs = np.ascontiguousarray(cs, dtype=np.uint8)
    return lib.plugin_decompress_codestream(cs.ctypes.data, cs.size, C.byref(img)), out


def coding(case):
    """the coding the stock entry points derive from the host's parameters (precinct sizes halved per coarser level)"""
    numres = case.get("numres", 6)
    prc = case.get("precinct")
    kw = dict(precincts=[(max(prc[0] >> k, 2), max(prc[1] >> k, 2)) for k in range(numres)][::-1]) if prc else {}
    return G.make_coding(case["width"], case["height"], case["numcomps"], case["prec"], numres=numres,
                         tile=tuple(case["tile"]) if case.get("tile") else None, irreversible=case.get("irreversible", False), **kw)


def _host_decode_matches(k, got, cs, case, tol):
    w, h, n = case["width"], case["height"], case["numcomps"]
    live = grok(lambda: R.decompress(cs, w, h, n)[0])
    if tol:
        GG.close(k, got, live, tol=tol)
    else:
        GG.same(k, got, live)


def check_case(case, engine):
    """tests/test_realhost.py's single image: encode and decode through the plugin, both equal to the host's CPU path"""
    w, h, n, prec = case["width"], case["height"], case["numcomps"], case["prec"]
    planes = P.synthetic_image(w, h, n, prec, seed=case.get("seed", 7))
    kw = dict(tile=tuple(case["tile"]) if case.get("tile") else None, numres=case.get("numres", 6),
              irreversible=case.get("irreversible", False), tlm=True, plt=True,
              precinct=tuple(case["precinct"]) if case.get("precinct") else None)
    assert plugin_init(0), "plugin_init failed: %s" % G.lib().b2k_last_error()
    ours = engine.encode_codestream(coding(case), planes, flags=G.CS_TLM | G.CS_PLT)
    cs_cpu = GG.grok_stream(GG.key("host stream", case), ours, grok(lambda: R.compress(planes, prec, **kw)[0]))
    if not case.get("irreversible"):      # the host's own round trip is lossless
        GG.same(GG.key("host decode", case), planes, grok(lambda: R.decompress(cs_cpu, w, h, n)[0]))
    rc, dec = plugin_decompress(cs_cpu, w, h, n)
    assert rc == 0, G.lib().b2k_last_error()
    _host_decode_matches(GG.key("host decode", case), dec, cs_cpu, case, 1 if case.get("irreversible") else 0)


def check_batch(case, engine):
    """tests/test_realhost.py's batch: planar and RGB48LE frames in, code streams equal to the host's own out; the host's
    code streams in, its frames out; a frame of another shape fails alone"""
    w, h, n, prec, nframes = case["width"], case["height"], case["numcomps"], case["prec"], case["frames"]
    frames = [P.synthetic_image(w, h, n, prec, seed=case.get("seed", 7) + f) for f in range(nframes)]
    kw = dict(numres=case.get("numres", 6), irreversible=case.get("irreversible", False))
    assert plugin_init(0), "plugin_init failed: %s" % G.lib().b2k_last_error()
    cp = coding(case)
    tol = 1 if case.get("irreversible") else 0
    for f, planes in enumerate(frames):
        k = GG.key("host batch stream %d" % f, case)
        ours = engine.encode_codestream(cp, planes, flags=0)
        cs_cpu = GG.grok_stream(k, ours, grok(lambda: R.compress(planes, prec, **kw)[0]))
        r = engine.encode_interleaved(cp, np.ascontiguousarray(np.stack(planes, axis=-1).astype(np.uint16)))
        rgb48 = G.codestream_write(cp, r.blocks, r.bytes, 0)
        r.free()
        assert bytes(rgb48) == bytes(ours), "frame %d: RGB48LE code stream differs from the planar one" % f
        rc, dec = plugin_decompress(cs_cpu, w, h, n)
        assert rc == 0, G.lib().b2k_last_error()
        _host_decode_matches(GG.key("host batch decode %d" % f, case), dec, cs_cpu, case, tol)
    if case.get("odd_one"):
        other = engine.encode_codestream(G.make_coding(w // 2, h, n, prec, numres=kw["numres"]),
                                         P.synthetic_image(w // 2, h, n, prec, seed=3), flags=0)
        assert plugin_decompress(other, w, h, n)[0] == 1      # declined: the host decodes that one itself
