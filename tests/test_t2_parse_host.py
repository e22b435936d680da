"""The device code-stream parser's functions (grok_b200/csrc/t2_parse.h), run on the host in the order of its kernels by
tests/t2_parse_check.cpp under the address and undefined-behaviour sanitizers, against b2k_codestream_parse on the same
bytes: the same return code, the same b2k_last_error text, the same block table.  CPU only.  This is where random damage
is exercised; the GPU suite runs fixed damage cases once each."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import grok_b200 as G
import test_t2_oracle as O
from test_device_codestream import FLAGS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "grok_b200", "csrc")
ALL_FLAGS = FLAGS + [G.CS_SOP, G.CS_EPH, G.CS_PLT | G.CS_EPH, G.CS_TLM | G.CS_SOP]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("t2pc") / "t2_parse_check")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                    "-I", CSRC, "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "t2_parse_check.cpp"),
                    os.path.join(CSRC, "codestream.cpp"), os.path.join(CSRC, "geometry.cpp"), "-o", exe], check=True)
    return exe


def check(harness, tmp_path, streams):
    """run the harness over {name: bytes}; every stream must give the host parser's verdict and table"""
    paths = []
    for name, cs in streams.items():
        p = tmp_path / (name + ".j2c")
        p.write_bytes(bytes(cs))
        paths.append(str(p))
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([harness] + paths, capture_output=True, text=True, env=env)
    bad = [ln for ln in r.stdout.splitlines() if " same" not in ln]
    assert r.returncode == 0 and not bad, (r.returncode, bad[:10], r.stderr[-3000:])
    return r.stdout.splitlines()


@pytest.mark.parametrize("content", O.CONTENTS)
@pytest.mark.parametrize("geom", list(O.GEOMS))
def test_parse_matches_host_for_every_flag(harness, tmp_path, geom, content):
    cp, _, _, table, data = O.encoded(O.GEOMS[geom], content)
    streams = {}
    for f in ALL_FLAGS:
        try:
            streams["f%d" % f] = G.codestream_write(cp, table, data, f)
        except G.EngineError:
            continue
    assert streams
    check(harness, tmp_path, streams)


def test_parse_matches_host_kmax29(harness, tmp_path):
    cp, _, _, table, data = O.encoded(O.KMAX29, "noise")
    check(harness, tmp_path, {"f%d" % f: G.codestream_write(cp, table, data, f) for f in (0, G.CS_SOP | G.CS_EPH | G.CS_PLT)})


@pytest.mark.parametrize("edge", list(O.EDGES))
def test_parse_matches_host_on_edge_shapes(harness, tmp_path, edge):
    args, kind, flags = O.EDGES[edge]
    cp, _, _, table, data = O.encoded(args, kind)
    check(harness, tmp_path, {edge: G.codestream_write(cp, table, data, flags)})


def refinement_stream():
    """the 2/3-pass stream of test_codestream.test_refinement_passes_survive_the_packet_headers, stripe-causal or not"""
    import oracle_lib as OL
    import oracle_pipeline as P
    out = {}
    for sty in (0, 8):
        w, h = 96, 80
        cp = G.make_coding(w, h, 1, 8, numres=3, cblk=(32, 32))
        cp.cblk_sty = sty
        planes = P.synthetic_image(w, h, 1, 8, seed=23)
        coefs = P.forward(cp, planes)
        table = G.enumerate_blocks(cp)
        chunks, off = [], 0
        L = OL.lib()
        for i, (t, c, b) in enumerate(P.enumerate_all(cp)):
            bw, bh = b.x1 - b.x0, b.y1 - b.y0
            kmax, _, _ = P.band_params(cp, b.resno, b.orient)
            win = np.ascontiguousarray(coefs[c][b.buf_y:b.buf_y + bh, b.buf_x:b.buf_x + bw])
            sm = np.zeros(bw * bh, np.uint32)
            L.orc_ht_pre_rev(win, bw, bw, bh, kmax, sm)
            W = (((sm & 0x7FFFFFFF) << 1) | (sm & 0x80000000)).astype(np.uint32).reshape(bh, bw)
            npass = 1 + i % 3
            s = 1 if (npass > 1 and kmax >= 3) else 0
            npass = npass if s else 1
            mm = kmax - 1 - s
            cup = OL.ht_encode(W, mm)
            seg = OL.ht_encode_refine(W, mm, npass) if npass > 1 else np.zeros(0, np.uint8)
            table[i]["length"], table[i]["length2"], table[i]["offset"] = len(cup), len(seg), off
            table[i]["numbps"], table[i]["numpasses"] = 1 + s, npass
            chunks += [cup, seg]
            off += len(cup) + len(seg)
        out["refine_sty%d" % sty] = (cp, table, np.concatenate(chunks))
    return out


def test_parse_matches_host_on_refinement_streams(harness, tmp_path):
    streams = {}
    for name, (cp, table, data) in refinement_stream().items():
        for f in (0, G.CS_SOP | G.CS_EPH | G.CS_PLT):
            streams["%s_%d" % (name, f)] = G.codestream_write(cp, table, data, f)
    check(harness, tmp_path, streams)


def mutations(cs, rng, rounds):
    """seeded damage of the kinds tests/fuzz_parser_driver.py makes"""
    cs = np.asarray(cs)
    sots = np.flatnonzero((cs[:-1] == 0xFF) & (cs[1:] == 0x90))
    hdr_end = int(sots[0])
    for _ in range(rounds):
        b = cs.copy()
        kind = rng.integers(0, 5)
        if kind == 0:      # the main header
            for _ in range(rng.integers(1, 4)):
                b[rng.integers(2, hdr_end)] = rng.integers(0, 256)
        elif kind == 1:    # anywhere
            for _ in range(rng.integers(1, 6)):
                b[rng.integers(0, len(b))] = rng.integers(0, 256)
        elif kind == 2:    # cut short
            b = b[:rng.integers(1, len(b))].copy()
        elif kind == 3:    # tile-part and packet headers
            p = int(sots[rng.integers(0, len(sots))]) + int(rng.integers(0, 40))
            if p < len(b):
                b[p] = rng.integers(0, 256)
        else:              # a run of garbage
            p = rng.integers(0, len(b) - 8)
            b[p:p + 8] = rng.integers(0, 256, 8)
        yield b


@pytest.mark.parametrize("seed", [1, 2])
def test_parse_matches_host_on_damaged_streams(harness, tmp_path, seed):
    import oracle_pipeline as P
    from test_interop import oracle_encode
    rng = np.random.default_rng(seed)
    streams = {}
    for j, (args, flags) in enumerate(((dict(width=200, height=150, numcomps=3, prec=8, numres=4, tile=(64, 64)), G.CS_TLM | G.CS_PLT),
                                       (dict(width=130, height=90, numcomps=1, prec=12, numres=3, irreversible=True),
                                        G.CS_SOP | G.CS_EPH | G.CS_TPARTS_R))):
        cp = G.make_coding(**args)
        planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=5)
        table, data, _ = oracle_encode(cp, planes)
        cs = G.codestream_write(cp, table, data, flags)
        for i, b in enumerate(mutations(cs, rng, 300)):
            streams["m%d_%d" % (j, i)] = b
    lines = check(harness, tmp_path, streams)
    codes = {ln.split()[1] for ln in lines}
    assert {"-1"} <= codes and len(codes) >= 2, codes   # damage reaches the error paths, and some streams still parse


def _stats(lines):
    """[(rc, tiles indexed from PLT, tiles walked)] of the harness's lines"""
    return [tuple(int(v) for v in ln.split()[1:4]) for ln in lines]


def _plt_entries(cs):
    """(position, bytes, value) of every Iplt entry in the tile-part headers of cs"""
    cs = bytes(cs)
    p, out = 2, []
    while cs[p:p + 2] != b"\xff\x90":
        p += 2 + int.from_bytes(cs[p + 2:p + 4], "big")
    while cs[p:p + 2] == b"\xff\x90":
        psot = int.from_bytes(cs[p + 6:p + 10], "big")
        q = p + 12
        while cs[q:q + 2] != b"\xff\x93":
            L = int.from_bytes(cs[q + 2:q + 4], "big")
            if cs[q:q + 2] == b"\xff\x58":
                i, v, at = q + 5, 0, q + 5
                while i < q + 2 + L:
                    v = (v << 7) | (cs[i] & 0x7F)
                    i += 1
                    if not cs[i - 1] & 0x80:
                        out.append((at, i - at, v))
                        v, at = 0, i
            q += 2 + L
        p += psot
    return out


def _tiled_stream(flags):
    import oracle_pipeline as P
    from test_interop import oracle_encode
    args = dict(width=200, height=150, numcomps=3, prec=8, numres=4, tile=(64, 64))
    cp = G.make_coding(**args)
    planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=5)
    table, data, _ = oracle_encode(cp, planes)
    return np.array(G.codestream_write(cp, table, data, flags))


def test_plt_indexes_every_tile_and_an_untrusted_plt_falls_back_to_the_walk(harness, tmp_path):
    """With PLT every tile is parsed packet by packet; without it every tile is walked.  A PLT whose entries still add up
    but put packet boundaries in the wrong places is indexed, then marked by the packets that do not end where it says,
    and walked; a PLT that does not add up is not indexed.  Each gives the host parser's table."""
    cs = _tiled_stream(G.CS_TLM | G.CS_PLT)
    ent = _plt_entries(cs)
    one = [k for k in range(len(ent) - 1) if ent[k][1] == 1 and ent[k + 1][1] == 1 and 2 < ent[k][2] < 126 and 2 < ent[k + 1][2] < 126
           and ent[k][0] + 1 == ent[k + 1][0]]   # neighbours in one PLT segment
    assert one
    k = one[0]
    moved = cs.copy()
    moved[ent[k][0]] += 1
    moved[ent[k + 1][0]] -= 1
    changed = cs.copy()
    changed[ent[k][0]] += 1
    lines = check(harness, tmp_path, {"plt": cs, "tlm_only": _tiled_stream(G.CS_TLM), "moved": moved, "changed": changed})
    (rc0, ix0, wk0), (rc1, ix1, wk1), (rc2, ix2, wk2), (rc3, ix3, wk3) = _stats(lines)
    assert rc0 > 1 and ix0 == 12 and wk0 == 0
    assert rc1 > 1 and ix1 == 0 and wk1 == 12
    assert ix2 == 12 and wk2 == 1          # indexed, marked, walked
    assert ix3 == 11 and wk3 == 1          # not indexed, walked


def test_placeholder_passes_are_declined_like_the_host(harness, tmp_path):
    """a packet header whose pass count reads 4 (placeholder passes, "1100" + "01"): the host declines the stream with
    'not handled', and so must the device's functions, with and without PLT"""
    cp = G.make_coding(16, 8, 1, 8, numres=1, cblk=(8, 8))   # two blocks: a block count of 1 would read as "not handled"
    table = G.enumerate_blocks(cp)
    assert len(table) == 2
    table["length"], table["numbps"], table["numpasses"], table["offset"] = 4, table["kmax"], 1, np.arange(2) * 4
    streams = {}
    for flags in (0, G.CS_PLT):
        cs = np.array(G.codestream_write(cp, table, np.full(8, 0x11, np.uint8), flags))
        sod = int(np.flatnonzero((cs[:-1] == 0xFF) & (cs[1:] == 0x93))[-1])
        # non-empty 1; block 0 included (root 1, leaf 1), no zero bit plane (root 1, leaf 1); passes "11" "01" (= 4)
        cs[sod + 2], cs[sod + 3] = 0b11111110, 0b10000000
        streams["placeholder_%d" % flags] = cs
    lines = check(harness, tmp_path, streams)
    assert all(ln.split()[1] == "1" and "placeholder passes" in ln for ln in lines), lines
