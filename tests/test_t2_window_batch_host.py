"""The windowed batch parse (b2k_decode_codestreams_window_device up to the gather), run on the host by
tests/t2_window_batch_check.cpp in the order of its steps, with the kernels' own thread bodies and per-stream slicing, each
stream read in place from its own allocation, under the address and undefined-behaviour sanitizers.  Every stream must get
what b2k_codestream_parse_window gives its bytes, window and reduce alone (code, text, virtual coding, block table), every
kept block's bytes must be where its descriptor points in the gathered arena, and the batch rule must hold: the first
stream whose header and window pass sets the coding, and another virtual coding or tile box gives 1 to that stream only.
CPU only; the GPU suite (test_device_window_batch_decode.py) decodes fixed cases once each."""
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import grok_b200 as G
import test_t2_oracle as O
from test_t2_parse_host import ALL_FLAGS, mutations, _tiled_stream
from test_t2_window_host import windows, _parts, _gathered_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "grok_b200", "csrc")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("t2wbc") / "t2_window_batch_check")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                    "-I", CSRC, "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "t2_window_batch_check.cpp"),
                    os.path.join(CSRC, "codestream.cpp"), os.path.join(CSRC, "geometry.cpp"), "-o", exe], check=True)
    return exe


def run(harness, tmp_path, batches):
    """batches: [(reduce, [(name, bytes, window or None)])]; every stream is checked.  Returns per batch
    (rows, wanted tiles, gathered bytes), rows[i] = (status, ref, 'same' | 'rule', text)."""
    lines, files = [], {}
    for reduce, streams in batches:
        lines.append("batch %d" % reduce)
        for name, cs, w in streams:
            if name not in files:
                p = tmp_path / ("%s.j2c" % name)
                p.write_bytes(bytes(np.asarray(cs, np.uint8)))
                files[name] = str(p)
            lines.append("%s %s" % (files[name], "-" if w is None else " ".join(str(int(v)) for v in w)))
    spec = tmp_path / "batches.txt"
    spec.write_text("\n".join(lines) + "\n")
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([harness, str(spec)], capture_output=True, text=True, env=env)
    out = r.stdout.splitlines()
    rows_out = [ln for ln in out if not ln.startswith("batch ")]
    bad = [ln for ln in rows_out if ln.split(" ", 4)[3:4] not in (["same"], ["rule"])]
    assert r.returncode == 0 and not bad and len(rows_out) == sum(len(s) for _, s in batches), (r.returncode, bad[:10], r.stderr[-3000:])
    res, k = [], 0
    for _, streams in batches:
        rows = []
        for _ in streams:
            f = out[k].split(" ", 4)
            rows.append((int(f[1]), int(f[2]), f[3], f[4] if len(f) > 4 else ""))
            k += 1
        b = out[k].split()
        k += 1
        res.append((rows, int(b[1]), int(b[2])))
    return res


def _random_window(cp, rng):
    a, b = sorted(rng.integers(cp.x0, cp.x1 + 1, 2))
    c, d = sorted(rng.integers(cp.y0, cp.y1 + 1, 2))
    return (int(a), int(c), int(max(b, a + 1)), int(max(d, c + 1)))


@pytest.mark.parametrize("content", O.CONTENTS)
@pytest.mark.parametrize("geom", list(O.GEOMS))
def test_window_batches_match_host_for_every_flag(harness, tmp_path, geom, content):
    """per flag set and reduce: one batch of the windows test_t2_window_host uses (per-stream windows; for tiled streams the
    ones on another tile box take the rule), and one batch of three streams under one seeded window"""
    cp, _, _, table, data = O.encoded(O.GEOMS[geom], content)
    rng = np.random.default_rng(zlib.crc32(("wb/%s/%s" % (geom, content)).encode()))
    batches = []
    for f in ALL_FLAGS:
        try:
            cs = G.codestream_write(cp, table, data, f)
        except G.EngineError:
            continue
        for r in range(cp.numres + 1):                              # reduce = numres is every stream's own error
            batches.append((r, [("f%d" % f, cs, w) for w in windows(cp, rng)]))
            w = _random_window(cp, rng)
            batches.append((r, [("f%d" % f, cs, w)] * 3))
    res = run(harness, tmp_path, batches)
    assert any(rows[0][0] == 0 for rows, _, _ in res)
    assert any(kind == "same" and rc == 0 for rows, _, _ in res for rc, ref, kind, _ in rows[1:])


def test_kmax29_and_edge_shapes(harness, tmp_path):
    batches = []
    cp, _, _, table, data = O.encoded(O.KMAX29, "noise")
    rng = np.random.default_rng(29)
    for f in (0, G.CS_SOP | G.CS_EPH | G.CS_PLT):
        cs = G.codestream_write(cp, table, data, f)
        for r in (0, 1, 3, 5):
            batches.append((r, [("k%d" % f, cs, w) for w in windows(cp, rng)]))
    for edge, (args, kind, flags) in O.EDGES.items():
        cp, _, _, table, data = O.encoded(args, kind)
        cs = G.codestream_write(cp, table, data, flags)
        for r in sorted({0, 1, cp.numres - 1}):
            batches.append((r, [(edge, cs, w) for w in windows(cp, rng, 1)]))
    run(harness, tmp_path, batches)


@pytest.mark.parametrize("seed", [1, 2])
def test_good_streams_mixed_with_mutations(harness, tmp_path, seed):
    """batches of 8: good streams of one seeded window interleaved with seeded mutations of the same stream under their own
    windows; every stream's verdict is its own"""
    rng = np.random.default_rng(200 + seed)
    batches = []
    for j, flags in enumerate((G.CS_TLM | G.CS_PLT, G.CS_SOP | G.CS_EPH | G.CS_TPARTS_R)):
        cs = _tiled_stream(flags)
        muts = list(mutations(cs, rng, 240))
        for b in range(0, len(muts), 4):
            x0, y0 = int(rng.integers(0, 200)), int(rng.integers(0, 150))
            w = (x0, y0, x0 + int(rng.integers(1, 120)), y0 + int(rng.integers(1, 90)))
            streams = []
            for i, m in enumerate(muts[b:b + 4]):
                streams.append(("g%d" % j, cs, w))
                streams.append(("m%d_%d" % (j, b + i), m, w if i % 2 else None))
            batches.append((int(rng.integers(0, 4)), streams))
    res = run(harness, tmp_path, batches)
    codes = {rc for rows, _, _ in res for rc, _, kind, _ in rows if kind == "same"}
    assert -1 in codes and 0 in codes, codes


def test_window_errors_and_unaligned_grids_are_per_stream(harness, tmp_path):
    """a window outside the image, one stream's reduce past its levels (the batch's reduce is shared, so a second coding
    with fewer levels), and a 48 x 48 grid unaligned for reduce 5: each stream's own verdict, the others decode"""
    import oracle_pipeline as P
    from test_interop import oracle_encode
    cs = _tiled_stream(G.CS_TLM | G.CS_PLT)
    res = run(harness, tmp_path, [(0, [("t", cs, (300, 0, 400, 10)), ("t", cs, (3, 3, 10, 10)), ("t", cs, (210, 160, 220, 170)),
                                       ("t", cs, (1, 1, 9, 9))])])
    rows = res[0][0]
    assert rows[0][0] == -1 and "does not intersect" in rows[0][3] and rows[0][2] == "same"
    assert rows[1][:3] == (0, 1, "same") and rows[3][:3] == (0, 1, "same")
    assert rows[2][0] == -1 and "does not intersect" in rows[2][3]
    cp = G.make_coding(200, 150, 1, 8, numres=6, tile=(48, 48))
    table, data, _ = oracle_encode(cp, P.synthetic_image(200, 150, 1, 8, seed=3))
    u = G.codestream_write(cp, table, data, G.CS_PLT)
    res = run(harness, tmp_path, [(5, [("u", u, (40, 40, 60, 60)), ("u", u, (1, 1, 9, 9)), ("u", u, (2, 2, 8, 8))]),
                                  (6, [("u", u, (1, 1, 9, 9)), ("t", cs, None)])])
    rows = res[0][0]
    assert rows[0][0] == 1 and "aligned" in rows[0][3] and rows[0][2] == "same"
    assert rows[1][:3] == (0, 1, "same") and rows[2][:3] == (0, 1, "same")
    rows = res[1][0]
    assert rows[0][0] == -1 and "reduce exceeds" in rows[0][3]
    assert rows[1][0] == -1 and "reduce exceeds" in rows[1][3]


def test_another_tile_box_takes_the_rule(harness, tmp_path):
    cs = _tiled_stream(G.CS_TLM | G.CS_PLT)
    res = run(harness, tmp_path, [(1, [("t", cs, (3, 3, 10, 10)), ("t", cs, (60, 60, 70, 70)), ("t", cs, (5, 5, 60, 60)),
                                       ("t", cs, None)])])
    rows, wanted, gathered = res[0]
    assert rows[0][:3] == (0, 0, "same") and rows[2][:3] == (0, 0, "same")
    for i in (1, 3):
        assert rows[i][:3] == (1, 0, "rule"), rows[i]
        assert rows[i][3] == ("code stream %d: its window's coding (tile grid, wanted tiles or virtual coding) differs from that "
                              "of code stream 0, which the batch takes its coding from" % i)
    assert wanted == 1 and gathered == 2 * _gathered_bytes(cs, {0})


def test_damage_outside_a_window_passes_and_sot_damage_fails(harness, tmp_path):
    """in tile 11, outside windows on tile 0: damage to its packets passes; to its SOT or Psot fails with the host's text,
    for that stream only"""
    cs = _tiled_stream(G.CS_TLM | G.CS_PLT)
    sot, tile, sod, end = _parts(cs)[-1]
    assert tile == 11
    pk = cs.copy()
    pk[sod + 2:sod + 10] = 0xFF
    bad_sot = cs.copy()
    bad_sot[sot + 2:sot + 4] = [0, 11]
    psot = cs.copy()
    psot[sot + 6:sot + 10] = 0xFF
    for r in (0, 1):
        res = run(harness, tmp_path, [(r, [("c", cs, (0, 0, 8, 8)), ("pk", pk, (1, 1, 30, 30)), ("sot", bad_sot, (0, 0, 8, 8)),
                                           ("psot", psot, (2, 2, 9, 9)), ("c", cs, (4, 4, 40, 40))])])
        rows, wanted, gathered = res[0]
        assert [row[0] for row in rows] == [0, 0, -1, -1, 0], rows
        assert rows[2][3] == "bad SOT" and rows[3][3] == "Psot exceeds the codestream"
        assert gathered == 3 * _gathered_bytes(cs, {0})
    res = run(harness, tmp_path, [(0, [("c", cs, (190, 140, 200, 150)), ("pk", pk, (190, 140, 200, 150))])])
    rows = res[0][0]
    assert rows[0][0] == 0 and rows[1][0] != 0 and rows[1][2] == "same"
