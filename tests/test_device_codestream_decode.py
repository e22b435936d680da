"""Code streams decoded from device memory (b2k_decode_codestream_device / b2k_codestream_parse_device,
Engine.decode_codestream_device(cuda tensor), Engine.codestream_parse_device).

The device parser must give, for every input, what copying the stream to the host and calling b2k_codestream_parse +
b2k_decode_device gives: the same block table, the same return code and b2k_last_error text, the same pixels.  The CPU
suite (test_t2_parse_host.py) runs the parser's functions under the sanitizers on random damage; here every geometry and
flag set of the device-I/O suite, the T2 oracle's streams, the edge shapes and fixed damage cases run once on the GPU."""
import numpy as np
import pytest

import grok_b200 as G
import test_device_io as D
from test_device_codestream import FLAGS, _reason

pytestmark = pytest.mark.gpu


def _dev(torch, cs):
    return torch.from_numpy(np.array(cs, np.uint8)).cuda()


def _same_coding(a, b):
    for name, _ in G.Coding._fields_:
        va, vb = getattr(a, name), getattr(b, name)
        if hasattr(va, "__len__"):
            va, vb = list(va), list(vb)
        assert va == vb, name


def _outcome(fn):
    """(rc class, text) of a call that may raise: ('ok', result) / ('NotHandled' | 'EngineError', reason)"""
    try:
        return "ok", fn()
    except G.NotHandled as e:
        return "NotHandled", _reason(e)
    except G.EngineError as e:
        return "EngineError", _reason(e)


def _check_parse(engine, torch, cs):
    host = _outcome(lambda: G.codestream_parse(cs))
    dev = _outcome(lambda: engine.codestream_parse_device(_dev(torch, cs)))
    assert host[0] == dev[0], (host, dev)
    if host[0] != "ok":
        assert host[1] == dev[1]
        return None
    (hcp, hb), (dcp, db) = host[1], dev[1]
    _same_coding(hcp, dcp)
    assert hb.tobytes() == db.tobytes()
    return hcp, hb


def _check_decode(engine, torch, cs, dtypes=None, layouts=("CHW",)):
    """device decode of cs against today's path (host bytes); returns the decoded CHW array of the first container"""
    dcs = _dev(torch, cs)
    first = None
    host = _outcome(lambda: G.codestream_parse(cs))
    if host[0] != "ok":
        dev = _outcome(lambda: engine.decode_codestream_device(dcs))
        assert (host[0], host[1]) == dev, (host, dev)
        return None
    cp = host[1][0]
    for dt in dtypes or D._containers(cp):
        tdt = getattr(torch, np.dtype(dt).name)
        for layout in layouts:
            want = _outcome(lambda: engine.decode_codestream_device(cs, dtype=tdt, layout=layout))
            got = _outcome(lambda: engine.decode_codestream_device(dcs, dtype=tdt, layout=layout))
            assert want[0] == got[0], (want, got)
            if want[0] != "ok":
                assert want[1] == got[1]
                continue
            _same_coding(want[1][0], got[1][0])
            a, b = D._to_chw(want[1][1], layout), D._to_chw(got[1][1], layout)
            assert np.array_equal(a, b), "pixels differ: %s %s" % (np.dtype(dt).name, layout)
            if first is None:
                first = b
    return first


@pytest.mark.parametrize("case", D.CASES, ids=["%d%s" % (i, "_97" if irr else "") for i, irr in D.CASES])
def test_host_written_streams(engine, case):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, _ = D._host_result(engine, *case)
    for flags in FLAGS:
        try:
            cs = G.codestream_write(cp, blocks, data, flags)
        except G.EngineError:
            continue
        _check_parse(engine, torch, cs)
        _check_decode(engine, torch, cs, dtypes=None if flags == FLAGS[0] else D._containers(cp)[:1],
                      layouts=("CHW", "HWC") if flags == FLAGS[0] else ("CHW",))


@pytest.mark.parametrize("content", ["zero", "flat", "sparse", "noise", "synthetic"])
def test_oracle_written_streams(engine, content):
    torch = pytest.importorskip("torch")
    import oracle_t2 as T2
    import test_t2_oracle as O
    for geom, args in list(O.GEOMS.items()) + [("kmax29", O.KMAX29)]:
        cp, planes, _, table, data = O.encoded(args, content)
        for flags in (0, G.CS_SOP | G.CS_EPH | G.CS_PLT | G.CS_TLM):
            cs = np.frombuffer(T2.write_flags(cp, table, data, flags), np.uint8)
            _, db = engine.codestream_parse_device(_dev(torch, cs))
            for f in ("numbps", "numpasses", "length", "length2"):
                got, want = db[f].copy(), table[f].copy()
                coded = table["length"] > 0
                assert np.array_equal(got[coded], want[coded]), (geom, content, f)
                assert not got[~coded].any() or f == "numbps", (geom, content, f)
            for i in np.flatnonzero(table["length"]):
                o, n = int(db[i]["offset"]), int(table[i]["length"])
                assert np.array_equal(cs[o:o + n], data[int(table[i]["offset"]):int(table[i]["offset"]) + n]), (geom, i)
            rec = _check_decode(engine, torch, cs, dtypes=[np.int32])
            if not cp.irreversible:   # the blocks a sparse table leaves out decode to zero coefficients, as coded
                assert np.array_equal(rec, np.stack(planes).astype(np.int32)), (geom, content)


@pytest.mark.parametrize("edge", ["plt-split", "4096-block-band", "ff-ending-header", "3168-parts"])
def test_edge_shapes(engine, edge):
    torch = pytest.importorskip("torch")
    import test_t2_oracle as O
    args, kind, flags = O.EDGES[edge]
    cp, _, _, table, data = O.encoded(args, kind)
    cs = G.codestream_write(cp, table, data, flags)
    _check_parse(engine, torch, cs)
    _check_decode(engine, torch, cs, dtypes=[np.int32])


def _tlm_split_image(torch):
    cp = G.make_coding(2048, 1536, 1, 8, numres=2, tile=(16, 16), cblk=(16, 16))
    img = torch.randint(0, 256, (1, 1536, 2048), dtype=torch.uint8, device="cuda")
    return cp, img


def test_tlm_split_stream(engine):
    """12,288 tile parts: TLM splits over two segments; every tile parsed by its own thread"""
    torch = pytest.importorskip("torch")
    cp, img = _tlm_split_image(torch)
    cs = engine.encode_codestream_device(cp, img, G.CS_TLM | G.CS_PLT | G.CS_TPARTS_R)
    _check_parse(engine, torch, cs)
    _check_decode(engine, torch, cs, dtypes=[np.uint8])


def _refinement_streams():
    import test_t2_parse_host as H
    return H.refinement_stream()


def test_refinement_streams(engine):
    torch = pytest.importorskip("torch")
    for name, (cp, table, data) in _refinement_streams().items():
        for flags in (0, G.CS_SOP | G.CS_EPH | G.CS_PLT):
            cs = G.codestream_write(cp, table, data, flags)
            _, blocks = _check_parse(engine, torch, cs)
            assert (blocks["numpasses"] == 3).any() and (blocks["numpasses"] == 2).any()
            _check_decode(engine, torch, cs, dtypes=[np.int32])


# ---- PLT that cannot be trusted, and damage --------------------------------------------------------------------------
def _base_stream(engine, flags=G.CS_TLM | G.CS_PLT):
    cp, planes, blocks, data, _ = D._host_result(engine, 15, False)   # 12 tiles
    return np.array(G.codestream_write(cp, blocks, data, flags))


def _sots(cs):
    out, p = [], 2
    while bytes(cs[p:p + 2]) != b"\xff\x90":
        p += 2 + int.from_bytes(bytes(cs[p + 2:p + 4]), "big")
    while p + 12 <= len(cs) and bytes(cs[p:p + 2]) == b"\xff\x90":
        out.append(p)
        psot = int.from_bytes(bytes(cs[p + 6:p + 10]), "big")
        if not psot:
            break
        p += psot
    return out


def _edits(engine):
    cs = _base_stream(engine)
    sots = _sots(cs)
    assert len(sots) >= 3
    e = {}
    b = cs.copy()                                    # one Iplt entry changed: the tile's PLT no longer adds up
    b[sots[0] + 12 + 5] ^= 0x01
    e["iplt_changed"] = b
    from test_t2_parse_host import _plt_entries      # two entries moved by one: PLT adds up, the boundaries are wrong
    ent = _plt_entries(cs)
    # neighbours in one segment whose last bytes take +1 / -1 without a carry (so no entry changes width or becomes 0)
    k = next(k for k in range(len(ent) - 1) if ent[k][0] + ent[k][1] == ent[k + 1][0] and (cs[ent[k + 1][0] - 1] & 0x7F) < 127 and
             (cs[ent[k + 1][0] + ent[k + 1][1] - 1] & 0x7F) > (1 if ent[k + 1][1] == 1 else 0))
    b = cs.copy()
    b[ent[k][0] + ent[k][1] - 1] += 1
    b[ent[k + 1][0] + ent[k + 1][1] - 1] -= 1
    e["iplt_moved"] = b
    s = sots[1]                                      # PLT removed from one tile part of several
    L = 2 + int.from_bytes(bytes(cs[s + 14:s + 16]), "big")
    assert bytes(cs[s + 12:s + 14]) == b"\xff\x58"
    b = np.concatenate([cs[:s + 12], cs[s + 12 + L:]])
    psot = int.from_bytes(bytes(cs[s + 6:s + 10]), "big") - L
    b[s + 6:s + 10] = np.frombuffer(psot.to_bytes(4, "big"), np.uint8)
    e["plt_removed"] = b                             # (TLM now disagrees: the parser reads Psot, as the host does)
    e["tlm_only"] = _base_stream(engine, G.CS_TLM)
    last = sots[-1]
    e["cut_in_last_part"] = cs[:last + (len(cs) - last) // 2].copy()
    b = e["cut_in_last_part"].copy()                 # the same with Psot = 0: a packet body runs past the data
    b[last + 6:last + 10] = 0
    e["cut_psot0"] = b
    mine = [v for at, _, v in _plt_entries(cs) if at > last]   # cut after half the last part's packets, Psot = 0:
    sod = int(np.flatnonzero((cs[last:-1] == 0xFF) & (cs[last + 1:] == 0x93))[0]) + last   # the data ends early and
    b = cs[:sod + 2 + sum(mine[:len(mine) // 2])].copy()                                     # the later packets stay
    b[last + 6:last + 10] = 0                                                                # uncoded, as on the host
    e["cut_at_a_packet"] = b
    e["missing_eoc"] = cs[:-2].copy()
    b = cs.copy()
    b[last + 6:last + 10] = 0
    e["psot0_last"] = b
    b = cs.copy()
    b[last + 6:last + 10] = np.frombuffer((len(cs)).to_bytes(4, "big"), np.uint8)
    e["psot_past_end"] = b
    b = cs.copy()
    b[last + 4:last + 6] = 0xFF
    e["tile_out_of_range"] = b
    b = cs.copy()                                    # a packet-header byte: the second byte after the first SOD
    sod = int(np.flatnonzero((cs[sots[0]:-1] == 0xFF) & (cs[sots[0] + 1:] == 0x93))[0]) + sots[0]
    b[sod + 3] ^= 0x5A
    e["packet_header_byte"] = b
    b = cs.copy()                                    # layers = 2 in COD
    cod = int(np.flatnonzero((cs[:-1] == 0xFF) & (cs[1:] == 0x52))[0])
    b[cod + 6:cod + 8] = [0, 2]
    e["layers2"] = b
    cod_seg = cs[cod:cod + 2 + int.from_bytes(bytes(cs[cod + 2:cod + 4]), "big")]
    s = sots[0]                                      # COD in the first tile-part header
    b = np.concatenate([cs[:s + 12], cod_seg, cs[s + 12:]])
    psot = int.from_bytes(bytes(cs[s + 6:s + 10]), "big") + len(cod_seg)
    b[s + 6:s + 10] = np.frombuffer(psot.to_bytes(4, "big"), np.uint8)
    e["cod_in_tile_part"] = b
    return e


def test_untrusted_plt_and_damage(engine):
    """every edit gives the host's table, text and pixels; the PLT edits send their tiles to the walk (12 tiles)"""
    torch = pytest.importorskip("torch")
    seen = set()
    walked = {}
    for name, cs in _edits(engine).items():
        host = _outcome(lambda: G.codestream_parse(cs))
        seen.add(host[0])
        _check_parse(engine, torch, cs)
        if host[0] == "ok":
            walked[name] = engine.codestream_parse_device_stats()
        _check_decode(engine, torch, cs, dtypes=[np.int32])
    assert seen == {"ok", "NotHandled", "EngineError"}, seen
    engine.codestream_parse_device(_dev(torch, _base_stream(engine)))
    assert engine.codestream_parse_device_stats() == (12, 0)     # a whole PLT: every tile packet by packet
    assert walked["tlm_only"] == (0, 12)                         # no PLT: every tile walked
    assert walked["iplt_changed"] == (11, 1)                     # does not add up: not indexed
    assert walked["iplt_moved"] == (12, 1)                       # adds up: indexed, marked by its packets, walked
    assert walked["plt_removed"] == (11, 1)                      # a tile part without PLT: not indexed
    assert walked["cut_at_a_packet"] == (11, 1)                  # PLT runs past the data: the walk stops where it ends


def test_ht_decoder_rejection_writes_the_image(engine):
    """a stream the HT decoder rejects: -2 with the host path's text, and the image written all the same, with the pixels
    b2k_codestream_parse + b2k_decode_device of its bytes write (a batch leaves such an image alone)"""
    torch = pytest.importorskip("torch")
    import test_device_batch_decode as B
    bad, text = B._ht_reject(engine, torch, _base_stream(engine))
    cp, blocks = G.codestream_parse(bad)
    shape = (cp.numcomps, cp.y1 - cp.y0, cp.x1 - cp.x0)
    want = torch.full(shape, B.SENTINEL, dtype=torch.uint16, device="cuda")
    with pytest.raises(G.EngineError) as host:
        engine.decode_device(cp, blocks, bad, want)
    got = torch.full(shape, B.SENTINEL, dtype=torch.uint16, device="cuda")
    with pytest.raises(G.EngineError) as dev:
        engine.decode_codestream_device(_dev(torch, bad), out=got)
    torch.cuda.synchronize()
    assert " -> -2: " in str(host.value) and " -> -2: " in str(dev.value)
    assert _reason(dev.value) == _reason(host.value) == text
    assert not (want == B.SENTINEL).all()
    assert torch.equal(got, want)


# ---- ordering, reuse, size ------------------------------------------------------------------------------------------------
def test_stream_ordering(engine):
    torch = pytest.importorskip("torch")
    cp, planes, blocks, data, _ = D._host_result(engine, 9, False)
    cs = np.array(G.codestream_write(cp, blocks, data, G.CS_TLM | G.CS_PLT))
    _, want = engine.decode_codestream_device(cs, dtype=torch.int32)
    side = torch.cuda.Stream()
    dcs = torch.zeros(len(cs), dtype=torch.uint8, device="cuda")
    src = torch.from_numpy(cs).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        dcs.copy_(src)                              # the bytes arrive late, on the side stream
        _, got = engine.decode_codestream_device(dcs, dtype=torch.int32, stream=side)
        after = got.clone()                          # queued after the call: must see the pixels
    side.synchronize()
    assert torch.equal(after, want)


def test_one_engine_reused(engine):
    torch = pytest.importorskip("torch")
    small = D._host_result(engine, 9, False)
    big = D._host_result(engine, 15, False)
    cs_small = np.array(G.codestream_write(small[0], small[2], small[3], G.CS_TLM | G.CS_PLT))
    cs_big = np.array(G.codestream_write(big[0], big[2], big[3], G.CS_SOP | G.CS_EPH | G.CS_PROG(2)))
    want = {}
    for name, cs in (("small", cs_small), ("big", cs_big)):
        want[name] = engine.decode_codestream_device(cs, dtype=torch.int32)[1].cpu()
    for name, cs in (("small", cs_small), ("big", cs_big), ("small", cs_small), ("big", cs_big)):
        _, got = engine.decode_codestream_device(_dev(torch, cs), dtype=torch.int32)
        assert torch.equal(got.cpu(), want[name]), name
        cp, planes = (small if name == "small" else big)[:2]
        img = torch.from_numpy(np.stack(planes).astype(D._containers(cp)[0])).cuda()
        engine.encode_codestream_device(cp, img, device_output=True)
        _, got = engine.decode_codestream_device(cs, dtype=torch.int32)
        assert torch.equal(got.cpu(), want[name]), name


def test_window_and_reduce_are_not_handled(engine):
    torch = pytest.importorskip("torch")
    cs = _base_stream(engine)
    with pytest.raises(G.NotHandled):
        engine.decode_codestream_device(_dev(torch, cs), window=(0, 0, 8, 8))
    with pytest.raises(G.NotHandled):
        engine.decode_codestream_device(_dev(torch, cs), reduce=1)


def test_config2_round_trip_on_the_device(engine):
    """config 2 (8192 x 8192 x 3, 12 bit, 1024^2 tiles): image -> code stream -> image without the samples crossing PCIe"""
    torch = pytest.importorskip("torch")
    import bench
    cp = G.make_coding(8192, 8192, 3, bench.PREC, numres=bench.NUMRES, tile=(bench.TILE, bench.TILE))
    g = torch.Generator(device="cuda").manual_seed(3)
    img = torch.randint(0, 1 << bench.PREC, (3, 8192, 8192), dtype=torch.int32, device="cuda", generator=g).to(torch.uint16)
    cs = engine.encode_codestream_device(cp, img, device_output=True)
    _, out = engine.decode_codestream_device(cs)
    assert torch.equal(out, img)
