"""The windowed device parse (b2k_codestream_parse_window_device), run on the host in the order of its steps by
tests/t2_window_check.cpp under the address and undefined-behaviour sanitizers, against b2k_codestream_parse_window on the
same bytes, window and reduce: the same return code, the same b2k_last_error text, the same virtual coding and block
table, for the header-only call and the full one.  The harness also checks that every parsed block's bytes are where the
descriptors address them once the wanted tile parts' packet data are gathered.  CPU only; the GPU suite
(test_device_window_decode.py) runs fixed cases once each."""
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import grok_b200 as G
import test_t2_oracle as O
from test_t2_parse_host import ALL_FLAGS, mutations, _tiled_stream

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "grok_b200", "csrc")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("t2wc") / "t2_window_check")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                    "-I", CSRC, "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "t2_window_check.cpp"),
                    os.path.join(CSRC, "codestream.cpp"), os.path.join(CSRC, "geometry.cpp"), "-o", exe], check=True)
    return exe


def run(harness, tmp_path, cases):
    """cases: [(name, bytes, reduce, window or None)]; every case must give the host parser's verdict and table.
    Returns [(rc, wanted tiles, gathered bytes, text)] in order."""
    files, lines = {}, []
    for name, cs, reduce, window in cases:
        if name not in files:
            p = tmp_path / (name + ".j2c")
            p.write_bytes(bytes(cs))
            files[name] = str(p)
        lines.append("%s %d %s" % (files[name], reduce, "-" if window is None else " ".join(str(int(v)) for v in window)))
    spec = tmp_path / "cases.txt"
    spec.write_text("\n".join(lines) + "\n")
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([harness, str(spec)], capture_output=True, text=True, env=env)
    out = r.stdout.splitlines()
    bad = [ln for ln in out if " same" not in ln]
    assert r.returncode == 0 and not bad and len(out) == len(cases), (r.returncode, bad[:10], len(out), len(cases), r.stderr[-3000:])
    res = []
    for ln in out:
        f = ln.split(" ", 7)
        res.append((int(f[3]), int(f[4]), int(f[5]), f[7] if len(f) > 7 else ""))
    return res


def windows(cp, rng, n_random=3):
    """None, the whole image, one tile's corner, a window across a tile corner, seeded random ones and one beside the image"""
    x0, y0, x1, y1 = cp.x0, cp.y0, cp.x1, cp.y1
    tw = cp.tw or (x1 - x0)
    th = cp.th or (y1 - y0)
    out = [None, (x0, y0, x1, y1), (x0, y0, x0 + 1, y0 + 1)]
    cx = min(x1 - 1, cp.tx0 + tw) if cp.tw else (x0 + x1) // 2
    cy = min(y1 - 1, cp.ty0 + th) if cp.th else (y0 + y1) // 2
    out.append((max(x0, cx - 3), max(y0, cy - 3), min(x1, cx + 3), min(y1, cy + 3)))   # up to four tiles
    for _ in range(n_random):
        a, b = sorted(rng.integers(x0, x1 + 1, 2))
        c, d = sorted(rng.integers(y0, y1 + 1, 2))
        out.append((int(a), int(c), int(max(b, a + 1)), int(max(d, c + 1))))
    out.append((x1 + 1, y1 + 1, x1 + 9, y1 + 9))                                       # no intersection
    out.append((0, 0, 1 << 31, 1 << 31))                                               # larger than the canvas
    return out


@pytest.mark.parametrize("content", O.CONTENTS)
@pytest.mark.parametrize("geom", list(O.GEOMS))
def test_window_parse_matches_host_for_every_flag(harness, tmp_path, geom, content):
    cp, _, _, table, data = O.encoded(O.GEOMS[geom], content)
    rng = np.random.default_rng(zlib.crc32(("%s/%s" % (geom, content)).encode()))
    cases = []
    for f in ALL_FLAGS:
        try:
            cs = G.codestream_write(cp, table, data, f)
        except G.EngineError:
            continue
        for w in windows(cp, rng):
            for r in range(cp.numres + 1):                                              # reduce = numres is refused
                cases.append(("f%d" % f, cs, r, w))
    res = run(harness, tmp_path, cases)
    codes = {rc for rc, _, _, _ in res}
    assert any(rc > 1 for rc in codes) and -1 in codes, codes


def test_window_parse_matches_host_kmax29(harness, tmp_path):
    cp, _, _, table, data = O.encoded(O.KMAX29, "noise")
    rng = np.random.default_rng(29)
    cases = [("f%d" % f, G.codestream_write(cp, table, data, f), r, w)
             for f in (0, G.CS_SOP | G.CS_EPH | G.CS_PLT) for w in windows(cp, rng) for r in (0, 1, 3, 5)]
    run(harness, tmp_path, cases)


@pytest.mark.parametrize("edge", list(O.EDGES))
def test_window_parse_matches_host_on_edge_shapes(harness, tmp_path, edge):
    args, kind, flags = O.EDGES[edge]
    cp, _, _, table, data = O.encoded(args, kind)
    cs = G.codestream_write(cp, table, data, flags)
    rng = np.random.default_rng(7)
    ws = windows(cp, rng, 1)
    cases = [(edge, cs, r, w) for w in ws for r in sorted({0, 1, cp.numres - 1, cp.numres})]
    res = run(harness, tmp_path, cases)
    if edge == "3168-parts":   # a tile part per resolution: a one-tile window takes 3 of the 3,168 parts
        one = [res[i] for i, c in enumerate(cases) if c[3] == (cp.x0, cp.y0, cp.x0 + 1, cp.y0 + 1) and c[2] == 0]
        assert one and one[0][0] > 1 and one[0][1] == 1, one


def test_tile_counts_and_grid_alignment(harness, tmp_path):
    """200 x 150 in 64 x 64 tiles (4 x 3): a window in one tile, across four, over all; reduce 1..3 keeps the grid aligned,
    while a 48 x 48 grid is unaligned at reduce 5 once a window spans tiles"""
    cs = _tiled_stream(G.CS_TLM | G.CS_PLT)
    cases = [("t", cs, r, w) for r in (0, 1, 2, 3) for w in [(3, 3, 10, 10), (60, 60, 70, 70), (0, 0, 200, 150), None]]
    res = run(harness, tmp_path, cases)
    wanted = {(c[2], c[3]): res[i][1] for i, c in enumerate(cases)}
    assert wanted[(0, (3, 3, 10, 10))] == 1 and wanted[(0, (60, 60, 70, 70))] == 4 and wanted[(2, None)] == 12
    assert all(res[i][0] > 1 for i in range(len(cases)))
    cp = G.make_coding(200, 150, 1, 8, numres=6, tile=(48, 48))
    import oracle_pipeline as P
    from test_interop import oracle_encode
    table, data, _ = oracle_encode(cp, P.synthetic_image(200, 150, 1, 8, seed=3))
    cs = G.codestream_write(cp, table, data, G.CS_PLT)
    res = run(harness, tmp_path, [("u", cs, 5, (40, 40, 60, 60)), ("u", cs, 4, (40, 40, 60, 60)), ("u", cs, 5, (1, 1, 9, 9)),
                                  ("u", cs, 6, (1, 1, 9, 9)), ("u", cs, 0, (300, 0, 400, 10))])
    assert res[0][0] == 1 and "aligned" in res[0][3]       # 48 = 16 x 3: not a multiple of 32
    assert res[1][0] > 1                                   # aligned at 16
    assert res[2][0] == 1 and res[2][3] == ""              # one tile needs no alignment: its one code block left
    assert res[3][0] == -1 and "reduce exceeds" in res[3][3]
    assert res[4][0] == -1 and "does not intersect" in res[4][3]


def _parts(cs):
    """(SOT position, tile, SOD position, end) of every tile part"""
    cs = bytes(cs)
    p, out = 2, []
    while cs[p:p + 2] != b"\xff\x90":
        p += 2 + int.from_bytes(cs[p + 2:p + 4], "big")
    while cs[p:p + 2] == b"\xff\x90":
        tile, psot = int.from_bytes(cs[p + 4:p + 6], "big"), int.from_bytes(cs[p + 6:p + 10], "big")
        q = p + 12
        while cs[q:q + 2] != b"\xff\x93":
            q += 2 + int.from_bytes(cs[q + 2:q + 4], "big")
        out.append((p, tile, q, p + psot))
        p += psot
    return out


def test_damage_outside_the_window(harness, tmp_path):
    """in a tile outside the window, damage to its packets or its tile-part header fails nothing; damage to its SOT
    fails with the host's text.  The same damage inside the window fails."""
    cs = _tiled_stream(G.CS_TLM | G.CS_PLT)
    parts = _parts(cs)
    sot, tile, sod, end = parts[-1]                       # tile 11, outside a window on tile 0
    assert tile == 11
    e = {}
    b = cs.copy()
    b[sod + 2:sod + 10] = 0xFF                            # its first packet header
    e["packet"] = b
    b = cs.copy()
    assert bytes(cs[sot + 12:sot + 14]) == b"\xff\x58"
    b[sot + 14:sot + 16] = 0xFF                           # its PLT's length runs past the tile part
    e["tp_header"] = b
    b = cs.copy()
    b[sot + 2:sot + 4] = [0, 11]                          # Lsot 11
    e["sot"] = b
    b = cs.copy()
    b[sot + 8:sot + 10] = [0xFF, 0xFF]                    # Psot past the end of the stream
    b[sot + 6:sot + 8] = [0xFF, 0xFF]
    e["psot"] = b
    cases = []
    for name, bb in e.items():
        cases += [(name, bb, 0, (0, 0, 8, 8)), (name, bb, 1, (0, 0, 8, 8)), (name, bb, 0, (190, 140, 200, 150))]
    res = dict(zip([(c[0], c[2], c[3]) for c in cases], run(harness, tmp_path, cases)))
    outside, inside = (0, (0, 0, 8, 8)), (0, (190, 140, 200, 150))
    assert res[("packet",) + outside][0] > 1 and res[("packet", 1, (0, 0, 8, 8))][0] > 1
    assert res[("packet",) + inside][0] <= 1
    assert res[("tp_header",) + outside][0] > 1
    assert res[("tp_header",) + inside][0] == -1 and res[("tp_header",) + inside][3] == "bad tile-part marker segment"
    assert res[("sot",) + outside][0] == -1 and res[("sot",) + outside][3] == "bad SOT"
    assert res[("psot",) + outside][0] == -1 and res[("psot",) + outside][3] == "Psot exceeds the codestream"


def _gathered_bytes(cs, wanted_tiles):
    return sum(end - (sod + 2) for _, t, sod, end in _parts(cs) if t in wanted_tiles)


def test_gathered_bytes_are_the_wanted_tiles_packet_data(harness, tmp_path):
    cs = _tiled_stream(G.CS_TLM | G.CS_PLT | G.CS_TPARTS_R)
    ws = [(3, 3, 10, 10), (60, 60, 70, 70), (130, 0, 200, 70)]
    res = run(harness, tmp_path, [("g", cs, 0, w) for w in ws])
    assert res[0][2] == _gathered_bytes(cs, {0})
    assert res[1][2] == _gathered_bytes(cs, {0, 1, 4, 5})
    assert res[2][2] == _gathered_bytes(cs, {2, 3, 6, 7})


@pytest.mark.parametrize("seed", [1, 2])
def test_window_parse_matches_host_on_damaged_streams(harness, tmp_path, seed):
    """over 1,000 seeded mutations in all, each with a seeded window and reduce"""
    rng = np.random.default_rng(100 + seed)
    cases = []
    for j, flags in enumerate((G.CS_TLM | G.CS_PLT, G.CS_SOP | G.CS_EPH | G.CS_TPARTS_R)):
        cs = _tiled_stream(flags)
        for i, b in enumerate(mutations(cs, rng, 280)):
            x0, y0 = int(rng.integers(0, 200)), int(rng.integers(0, 150))
            w = None if i % 7 == 0 else (x0, y0, x0 + int(rng.integers(1, 120)), y0 + int(rng.integers(1, 90)))
            cases.append(("m%d_%d" % (j, i), b, int(rng.integers(0, 5)), w))
    res = run(harness, tmp_path, cases)
    codes = {rc for rc, _, _, _ in res}
    assert -1 in codes and any(rc > 1 for rc in codes), codes
