"""The batched device parse (b2k_decode_codestreams_device up to the decoder's descriptors), run on the host by
tests/t2_batch_check.cpp in the order of its steps, with the kernels' own thread bodies and per-stream slicing, under the
address and undefined-behaviour sanitizers.  Each batch mixes good and damaged streams, streams with and without TLM / PLT;
every stream must get what b2k_codestream_parse gives it alone (code, text, block table), every coded block's bytes must be
where its descriptor points in the batch's arena, and the batch rules must hold: the first stream whose main header parses
sets the coding, and another coding or another progression / SOP / EPH gives 1 to that stream only.  CPU only; the GPU
suite (test_device_batch_decode.py) runs fixed cases once each."""
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
PLAN_FLAGS = G.CS_PROG(7) | G.CS_SOP | G.CS_EPH   # what the packet plan depends on


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("t2bc") / "t2_batch_check")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                    "-I", CSRC, "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "t2_batch_check.cpp"),
                    os.path.join(CSRC, "codestream.cpp"), os.path.join(CSRC, "geometry.cpp"), "-o", exe], check=True)
    return exe


def run(harness, tmp_path, batches):
    """batches: [[(name, bytes)]]; returns [[(status, ref, 'same' | 'rule', text)]] per batch, every stream checked"""
    args, names = [], []
    for b, batch in enumerate(batches):
        if b:
            args.append("--")
        for name, cs in batch:
            p = tmp_path / ("b%d_%s.j2c" % (b, name))
            p.write_bytes(bytes(np.asarray(cs, np.uint8)))
            args.append(str(p))
            names.append(str(p))
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([harness] + args, capture_output=True, text=True, env=env)
    lines = r.stdout.splitlines()
    bad = [ln for ln in lines if ln.split(" ", 4)[3:4] not in (["same"], ["rule"])]
    assert r.returncode == 0 and not bad and len(lines) == len(names), (r.returncode, bad[:10], r.stderr[-3000:])
    out, k = [], 0
    for batch in batches:
        rows = []
        for _ in batch:
            f = lines[k].split(" ", 4)
            rows.append((int(f[1]), int(f[2]), f[3], f[4] if len(f) > 4 else ""))
            k += 1
        out.append(rows)
    return out


def _check_rules(rows, flags, damaged):
    """'rule' exactly for the intact streams whose plan flags differ from the reference stream's; a damaged stream whose
    main header still parses may also read as another coding"""
    for i, (rc, ref, kind, text) in enumerate(rows):
        if ref < 0 or i <= ref:
            assert kind == "same", (i, rows[i])
            continue
        differs = (flags[i] & PLAN_FLAGS) != (flags[ref] & PLAN_FLAGS)
        prog = "code stream %d: its progression order, SOP or EPH differ from those of code stream %d" % (i, ref)
        coding = "code stream %d: its coding differs from that of code stream %d" % (i, ref)
        if damaged[i]:
            assert kind == "same" or (rc == 1 and (text.startswith(prog) or text.startswith(coding))), (i, rows[i])
        else:
            assert (kind == "rule") == differs, (i, rows[i], flags[i], flags[ref])
            assert kind == "same" or (rc == 1 and text.startswith(prog)), (i, rows[i])


@pytest.mark.parametrize("content", O.CONTENTS)
@pytest.mark.parametrize("geom", list(O.GEOMS))
def test_oracle_streams_mixed_with_damage(harness, tmp_path, geom, content):
    """every flag set of one coding in one batch (progressions other than the first's fall to the rule), each followed by
    a damaged copy of itself"""
    cp, _, _, table, data = O.encoded(O.GEOMS[geom], content)
    rng = np.random.default_rng(zlib.crc32((geom + content).encode()))
    batch, flags, damaged = [], [], []
    for f in ALL_FLAGS:
        try:
            cs = G.codestream_write(cp, table, data, f)
        except G.EngineError:
            continue
        batch += [("f%d" % f, cs), ("f%d_damaged" % f, next(mutations(cs, rng, 1)))]
        flags += [f, f]
        damaged += [False, True]
    _check_rules(run(harness, tmp_path, [batch])[0], flags, damaged)


def test_kmax29_and_edge_shapes(harness, tmp_path):
    batches = []
    cp, _, _, table, data = O.encoded(O.KMAX29, "noise")
    batches.append([("kmax29_%d" % f, G.codestream_write(cp, table, data, f)) for f in (0, G.CS_PLT)])
    for edge, (args, kind, flags) in O.EDGES.items():
        cp, _, _, table, data = O.encoded(args, kind)
        cs = np.array(G.codestream_write(cp, table, data, flags))
        batches.append([(edge, cs), (edge + "_cut", cs[:len(cs) * 2 // 3].copy()), (edge + "_again", cs)])
    for rows in run(harness, tmp_path, batches):
        assert all(kind == "same" for _, _, kind, _ in rows), rows


def test_seeded_mutations_in_batches(harness, tmp_path):
    """damaged streams in batches of 8 between good ones, TLM + PLT and SOP + EPH + tile parts"""
    rng = np.random.default_rng(11)
    batches = []
    for j, flags in enumerate((G.CS_TLM | G.CS_PLT, G.CS_SOP | G.CS_EPH | G.CS_TPARTS_R)):
        good = _tiled_stream(flags)
        muts = list(mutations(good, rng, 160))
        for b in range(0, len(muts), 8):
            batch = [("good%d" % j, good)]
            for i, m in enumerate(muts[b:b + 8]):
                batch += [("m%d_%d" % (j, b + i), m), ("good%d_%d" % (j, b + i), good)]
            batches.append(batch)
    results = run(harness, tmp_path, batches)
    codes = {rc for rows in results for rc, _, _, _ in rows}
    assert {0, -1} <= codes, codes
    for rows in results:   # the good streams between damaged ones parse whatever their neighbours do
        assert all(rc == 0 for k, (rc, _, kind, _) in enumerate(rows) if k % 2 == 0 and kind == "same"), rows


def test_batch_rules(harness, tmp_path):
    """a damaged first stream: the batch takes its coding from the next; another coding gives 1 to that stream only; a
    stream without TLM / PLT keeps its place"""
    a = _tiled_stream(G.CS_TLM | G.CS_PLT)
    bad = a.copy()
    bad[0:2] = 0
    cp, _, _, table, data = O.encoded(O.GEOMS[next(iter(O.GEOMS))], "noise")
    other = G.codestream_write(cp, table, data, G.CS_TLM | G.CS_PLT)
    rows = run(harness, tmp_path, [[("bad", bad), ("a", a), ("other", other), ("plain", _tiled_stream(0)),
                                    ("prog", _tiled_stream(G.CS_PROG(2)))]])[0]
    assert rows[0][0] == -1 and rows[0][1] == 1 and rows[0][2] == "same"
    assert [r[2] for r in rows[1:]] == ["same", "rule", "same", "rule"], rows
    assert rows[2][3] == "code stream 2: its coding differs from that of code stream 1, which the batch takes its coding from"
    assert rows[4][3].startswith("code stream 4: its progression order, SOP or EPH differ from those of code stream 1")
    assert rows[1][0] == 0 and rows[3][0] == 0
