"""The batched device code-stream writer (b2k_encode_codestreams_device after the block coder), run on the host by
tests/t2_write_batch_check.cpp in the order of its steps, with the kernels' own thread bodies (t2_write.h) and per-stream
slicing, under the address and undefined-behaviour sanitizers.  Each batch holds several streams of one coding and one
flag set; every stream's bytes must be those of the plain-Python T2 writer (tests/oracle_t2.py) and of
b2k_codestream_write of its block table alone, the streams must lie in order at 256-byte boundaries, and a stream with an
overflowed block must get the single call's -2 and text and take no bytes, leaving every other stream as it is.  CPU only;
the GPU suite (test_device_batch_encode.py) compares the device batch with the single device call."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import grok_b200 as G
import oracle_t2 as T2
import test_device_codestream as DC
import test_t2_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "grok_b200", "csrc")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("no g++")
    exe = str(tmp_path_factory.mktemp("t2wb") / "t2_write_batch_check")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
                    "-I", CSRC, "-I", "/usr/local/cuda/include", os.path.join(ROOT, "tests", "t2_write_batch_check.cpp"),
                    os.path.join(CSRC, "codestream.cpp"), os.path.join(CSRC, "geometry.cpp"), "-o", exe], check=True)
    return exe


def coder_table(table):
    """the table as the block coder reports it, the only form the device writer sees: every block with area one cleanup
    pass of one bit plane, its length the coder's total"""
    t = np.array(table, dtype=G.BLOCK_DTYPE)
    area = (t["x1"] > t["x0"]) & (t["y1"] > t["y0"])
    t["numpasses"] = np.where(area, 1, 0)
    t["numbps"] = np.where(area, 1, 0)
    t["length"] = np.where(area, t["length"], 0)
    t["length2"] = 0
    return t


def run(harness, tmp_path, batches):
    """batches: [(flags, cp, [(name, table, data, inject)])]; returns [[(rc, offset, length, text)]] per batch, or
    [[('plan', text)]] for a batch the writer's plan declines; every stream checked by the harness, and every stream
    written compared with the oracle's stream of its table"""
    args, count, files = [], 0, []
    for b, (flags, cp, streams) in enumerate(batches):
        cpf = tmp_path / ("b%d_cp.bin" % b)
        cpf.write_bytes(bytes(cp))
        args += ["--", str(flags), str(cpf)]
        for name, table, data, inject in streams:
            tf, df = tmp_path / ("b%d_%s.tab" % (b, name)), tmp_path / ("b%d_%s.dat" % (b, name))
            tf.write_bytes(coder_table(table).tobytes())
            df.write_bytes(np.asarray(data, np.uint8).tobytes())
            args += [name, str(tf), str(df), str(inject)]
            files.append(tf)
            count += 1
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([harness] + args, capture_output=True, text=True, env=env)
    lines = r.stdout.splitlines()
    bad = [ln for ln in lines if ln.split(" ", 5)[1] != "plan" and ln.split(" ", 5)[4:5] != ["same"]]
    assert r.returncode == 0 and not bad and len(lines) == count, (r.returncode, bad[:10], r.stderr[-3000:])
    out, k, oracle = [], 0, {}
    for flags, cp, streams in batches:
        rows = []
        for name, table, data, _ in streams:
            f = lines[k].split(" ", 5)
            if f[1] == "plan":
                rows.append(("plan", lines[k].split(" ", 2)[2]))
            else:
                rows.append((int(f[1]), int(f[2]), int(f[3]), f[5] if len(f) > 5 else ""))
            if rows[-1][0] == 0:
                key = (id(table), id(data), flags)
                if key not in oracle:
                    oracle[key] = T2.write_flags(cp, coder_table(table), data, flags)
                got = np.fromfile(str(files[k]) + ".cs", np.uint8)
                assert np.array_equal(got, oracle[key]), (name, flags, len(got), len(oracle[key]))
            k += 1
        out.append(rows)
    return out


def _check_declined(cp, streams, flags, rows):
    """a batch the plan declines: every stream says so, with b2k_codestream_write's text"""
    with pytest.raises(G.EngineError) as e:
        G.codestream_write(cp, coder_table(streams[0][1]), streams[0][2], flags)
    assert all(r == ("plan", str(e.value).split(": ", 1)[1]) for r in rows), rows


@pytest.mark.parametrize("geom", list(O.GEOMS))
def test_geometries_contents_and_flags(harness, tmp_path, geom):
    """every content of one geometry in one batch (the first again at the end), under each of the 16 flag sets"""
    streams = []
    for content in O.CONTENTS:
        cp, _, _, table, data = O.encoded(O.GEOMS[geom], content)
        streams.append((content, table, data, -1))
    streams.append(("again", streams[0][1], streams[0][2], -1))
    batches = [(f, cp, streams) for f in DC.FLAGS]
    for (flags, _, _), rows in zip(batches, run(harness, tmp_path, batches)):
        if rows[0][0] == "plan":
            _check_declined(cp, streams, flags, rows)
            continue
        assert all(r[0] == 0 and r[3] == "" for r in rows), (flags, rows)
        assert rows[0][1] == 0 and rows[-1][2] == rows[0][2]


def test_kmax29_and_edge_shapes(harness, tmp_path):
    batches = []
    cp, _, _, table, data = O.encoded(O.KMAX29, "noise")
    for f in (0, G.CS_PLT, G.CS_TLM | G.CS_PLT | G.CS_SOP | G.CS_EPH):
        batches.append((f, cp, [("kmax29_a", table, data, -1), ("kmax29_b", table, data, -1)]))
    for edge, (args, kind, flags) in O.EDGES.items():
        cp, _, _, table, data = O.encoded(args, kind)
        batches.append((flags, cp, [(edge, table, data, -1), (edge + "_again", table, data, -1)]))
    for (flags, cp, streams), rows in zip(batches, run(harness, tmp_path, batches)):
        if rows[0][0] == "plan":
            _check_declined(cp, streams, flags, rows)
            continue
        assert all(r[0] == 0 for r in rows), (streams[0][0], rows)


def test_plan_declines_every_stream(harness, tmp_path):
    """a progression order the writer does not know, and more than 65535 tiles: every stream of the batch gets
    b2k_codestream_write's text"""
    geom = next(iter(O.GEOMS))
    cp, _, _, table, data = O.encoded(O.GEOMS[geom], "noise")
    streams = [("a", table, data, -1), ("b", table, data, 0), ("c", table, data, -1)]
    grid = G.make_coding(264, 256, 1, 8, numres=1, tile=(1, 1))
    gtable = G.enumerate_blocks(grid)
    gtable["length"] = 1
    gtable["offset"] = np.arange(len(gtable))
    gstreams = [("g%d" % i, gtable, np.full(len(gtable), 0x11 * (i + 1), np.uint8), -1) for i in range(2)]
    batches = [(G.CS_PROG(5) | G.CS_PLT, cp, streams), (G.CS_TLM, grid, gstreams)]
    for (flags, bcp, bstreams), rows in zip(batches, run(harness, tmp_path, batches)):
        assert rows[0][0] == "plan", rows
        _check_declined(bcp, bstreams, flags, rows)


def test_overflowed_block_fails_its_stream_only(harness, tmp_path):
    """an overflowed block in streams 1 and 3: -2 with the single call's text, no bytes; the others keep their bytes and
    are packed behind each other"""
    geom = next(iter(O.GEOMS))
    contents = [O.encoded(O.GEOMS[geom], c) for c in ("noise", "synthetic", "sparse", "noise", "flat")]
    cp = contents[0][0]
    t = contents[0][3]
    ncoded = int(((t["x1"] > t["x0"]) & (t["y1"] > t["y0"])).sum())
    text = "1 code block(s) overflowed the coder's buffers"
    for flags in (G.CS_TLM | G.CS_PLT, G.CS_SOP | G.CS_EPH | G.CS_TPARTS_R):
        inject = [-1, 0, -1, ncoded // 2, -1]
        streams = [("s%d" % i, c[3], c[4], inject[i]) for i, c in enumerate(contents)]
        alone = [(flags, cp, [s]) for s in streams]
        rows, *single = run(harness, tmp_path, [(flags, cp, streams)] + alone)
        for i, r in enumerate(rows):
            assert r[:1] + r[2:] == single[i][0][:1] + single[i][0][2:], (i, r, single[i])
            if inject[i] >= 0:
                assert r[0] == -2 and r[2] == 0 and r[3] == text, r
            else:
                assert r[0] == 0
        assert rows[0][1] == 0 and rows[2][1] == -(-rows[0][2] // 256) * 256 and rows[4][1] == rows[2][1] + -(-rows[2][2] // 256) * 256
