"""Quality-factor codings and foreign per-component quantisation (QCC) through every device entry point: the bytes of the
host path and of tests/golden/qfactor.npz (grk_compress --qfactor), and the pixels and return codes of the host parse +
decode."""
import hashlib

import numpy as np
import pytest

import grok_b200 as G
import oracle_pipeline as P
import test_qfactor as Q

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def eng():
    e = G.Engine(0)
    yield e
    e.close()


def dev(planes):
    return torch.as_tensor(np.stack(planes).astype(np.int32)).cuda()


def record_sha(name):
    return Q.REC["stream_sha"][list(Q.REC["stream_names"]).index(name)]


@pytest.mark.parametrize("name", ["q50", "q60_tiled", "q75_rpcl", "q90_origin", "q97_grey", "q30_N2"])
def test_every_encode_entry_point_writes_grk_compress_bytes(eng, name):
    cp, planes, flags = Q.stream_case(name)
    want = record_sha(name)
    host = eng.encode_codestream(cp, planes, flags)
    assert hashlib.sha256(bytes(host)).hexdigest() == want
    if cp.prec <= 16:
        assert np.array_equal(eng.encode_codestream(cp, [p.astype(np.uint16) for p in planes], flags), host)   # encode16
    img = dev(planes)
    assert np.array_equal(eng.encode_codestream_device(cp, img, flags), host)                                  # encode_device
    on_dev = eng.encode_codestream_device(cp, img, flags, device_output=True)
    assert np.array_equal(on_dev.cpu().numpy(), host)
    other = dev(P.synthetic_image(cp.x1 - cp.x0, cp.y1 - cp.y0, cp.numcomps, cp.prec, seed=99, origin=(cp.x0, cp.y0)))
    streams, status = eng.encode_codestreams_device(cp, [img, other, img], flags)
    assert [s for s, _ in status] == [0, 0, 0]
    assert np.array_equal(streams[0].cpu().numpy(), host) and np.array_equal(streams[2].cpu().numpy(), host)
    assert not np.array_equal(streams[1].cpu().numpy(), host)
    got = {}
    enc = G.EncodeStream(cp, depth=2, on_encoded=lambda tag, res, st: got.__setitem__(tag, (res, st)))   # encode stream
    enc.submit(planes, "a")
    enc.submit(planes, "b")
    assert enc.end() == 0
    for tag in ("a", "b"):
        res, st = got[tag]
        assert st == 0
        try:
            assert np.array_equal(G.codestream_write(cp, res.blocks, res.bytes, flags, num_tiles=res.num_tiles), host)
        finally:
            res.free()


@pytest.mark.parametrize("name", Q.DECODED)
def test_device_decode_of_our_stream_matches_grk_decompress(eng, name):
    """grk_decompress's pixels of its own stream, which ours equals byte for byte: within the reference's 2-code bar"""
    cp, planes, flags = Q.stream_case(name)
    cs = eng.encode_codestream(cp, planes, flags)
    _, img = eng.decode_codestream_device(torch.from_numpy(np.array(cs)).cuda(), dtype=torch.int32)
    assert int(np.abs(img.cpu().numpy().astype(np.int64) - Q.REC["decoded_" + name]).max()) <= 2


def host_decode(eng, cs):
    cp, planes = eng.decode_codestream(cs)
    return cp, planes


@pytest.mark.parametrize("name", ["q50", "q60_tiled", "q75_rpcl", "q90_origin"])
def test_every_decode_entry_point_gives_the_host_pixels(eng, name):
    cp, planes, flags = Q.stream_case(name)
    cs = eng.encode_codestream(cp, planes, flags)
    cp_h, want = host_decode(eng, cs)
    assert cp_h.qfactor == cp.qfactor
    assert Q.psnr(want, planes, cp.prec) > 25
    cp2, blocks = G.codestream_parse(cs)
    out = torch.zeros((cp.numcomps, cp.y1 - cp.y0, cp.x1 - cp.x0), dtype=torch.int32, device="cuda")
    eng.decode_device(cp2, blocks, cs, out)
    assert np.array_equal(out.cpu().numpy(), np.stack(want))
    dcs = torch.from_numpy(np.array(cs)).cuda()
    _, img = eng.decode_codestream_device(dcs, dtype=torch.int32)
    assert np.array_equal(img.cpu().numpy(), np.stack(want))
    pcp, pblocks = eng.codestream_parse_device(dcs)
    assert bytes(pcp) == bytes(cp2) and np.array_equal(pblocks, blocks)
    for reduce in range(3):
        win = (cp.x0 + 7, cp.y0 + 5, cp.x1 - 3, cp.y1 - 9)
        _, hw = eng.decode_window(cs, win, reduce)
        _, dw = eng.decode_window_device(dcs, win, reduce, dtype=torch.int32)
        assert np.array_equal(dw.cpu().numpy(), np.stack(hw)), reduce
        if reduce == 0:
            x0, y0 = win[0] - cp.x0, win[1] - cp.y0
            assert np.array_equal(np.stack(hw), np.stack(want)[:, y0:y0 + win[3] - win[1], x0:x0 + win[2] - win[0]])


def test_batch_decode_with_a_different_qfactor_is_a_coding_mismatch(eng):
    cp, planes, flags = Q.stream_case("q50")
    cs = eng.encode_codestream(cp, planes, flags)
    cp75 = G.make_coding(cp.x1, cp.y1, 3, 8, numres=6, irreversible=True, qfactor=75)
    cs75 = eng.encode_codestream(cp75, planes, flags)
    _, want = host_decode(eng, cs)
    streams = [torch.from_numpy(np.array(s)).cuda() for s in (cs, cs75, cs)]
    _, out, status = eng.decode_codestreams_device(streams, dtype=torch.int32)
    assert status[0][0] == 0 and status[2][0] == 0 and status[1][0] == 1
    assert np.array_equal(out[0].cpu().numpy(), np.stack(want)) and np.array_equal(out[2].cpu().numpy(), np.stack(want))


@pytest.mark.parametrize("case", ["comp0", "one_of_four", "reversible"])
def test_foreign_qcc_streams_decode_on_the_device_to_the_oracle(eng, case):
    cp, planes, tables = Q.foreign_case(case)
    cs, _, comp_cp = Q.foreign(cp, planes, tables)
    cp_h, want = host_decode(eng, cs)
    oracle = np.stack(Q.oracle_decode(cp, comp_cp, G.codestream_parse(cs)[1], cs))
    if case == "reversible":
        assert np.array_equal(np.stack(want), oracle) and np.array_equal(oracle, np.stack(planes))   # lossless
    else:
        assert int(np.abs(np.stack(want).astype(np.int64) - oracle).max()) <= 1       # float 9/7 on both sides
    dcs = torch.from_numpy(np.array(cs)).cuda()
    _, img = eng.decode_codestream_device(dcs, dtype=torch.int32)
    assert np.array_equal(img.cpu().numpy(), np.stack(want))
    _, win = eng.decode_window_device(dcs, (10, 10, 90, 70), 1, dtype=torch.int32)
    _, hwin = eng.decode_window(cs, (10, 10, 90, 70), 1)
    assert np.array_equal(win.cpu().numpy(), np.stack(hwin))
