"""The device-resident round trips (b2k_job_roundtrip, b2k_job_roundtrip_n, b2k_job_roundtrip_pipelined_n) against the
oracle.  They queue forward -> HT encode -> scan -> gather -> decode -> inverse without a synchronisation between the
stages, so the paths that exist only there are checked here: the byte arena sized once per uploaded image, the decode
descriptors built on the device (k_build_dec_desc), 9/7 steps that code the previous step's reconstruction, the byte
offsets chained from one block range to the next in the pipelined call, and images whose coded size outgrows the arena
of an earlier image.  The host encode's own "arena estimate too small" branch is reached on purpose as well.

The oracle restates one step with tests/oracle_pipeline.py's stages (forward, HT encode and decode per code block,
inverse); the device's transforms are bit-exact against those (tests/test_dwt_paths.py), so every comparison is exact."""
import numpy as np
import pytest

import grok_b200 as G
import oracle_pipeline as P

CASES = {
    # many 512x512 tiles: the pipelined call's ranges start inside tiles
    "tiles-53": dict(width=2048, height=1536, numcomps=3, prec=12, numres=6, tile=(512, 512)),
    # one tile, odd origin, 9/7: three steps, each coding the previous step's reconstruction
    "one-tile-97": dict(width=333, height=217, numcomps=3, prec=12, numres=5, origin=(3, 5), irreversible=True),
    # 16,900 coded 4x4 blocks: the length scan takes three rounds of 8,192, the last one partial
    "4x4-blocks": dict(width=520, height=514, numcomps=1, prec=8, numres=2, cblk=(4, 4)),
    # 1024x4 blocks: the wide-block VLC parse
    "1024x4-blocks": dict(width=1500, height=24, numcomps=1, prec=10, numres=2, cblk=(1024, 4)),
    # no wavelet level (point transform) over ragged tiles
    "no-dwt-ragged-tiles": dict(width=333, height=217, numcomps=3, prec=12, numres=1, origin=(3, 5), tile=(100, 90)),
    # fewer coded blocks than one 128-block range
    "under-one-range": dict(width=333, height=217, numcomps=1, prec=8, numres=4),
    # 16 bit with 5 guard bits: Kmax 25, the encoder instances that stage samples unpacked
    "16bit-5-guard-bits": dict(width=160, height=120, numcomps=3, prec=16, numres=6, numgbits=5),
}
# images whose content changes inside one job: several tiles, so that the host encode runs several chunks and the
# pipelined round trip several block ranges
CHANGE_CASE = dict(width=512, height=384, numcomps=3, prec=12, numres=5, tile=(256, 256), irreversible=False)

STEPS = 3
SHAPES = [(0, 0), (1, 1), (3, 2), (64, 8)]   # (chunks, streams) of b2k_job_roundtrip_pipelined_n
CALLS = [("roundtrip", None), ("roundtrip_n", None)] + [("pipelined", s) for s in SHAPES]
PACKED_KMAX = 24        # b2k_launch_ht_encode stages samples packed with their exponent up to this Kmax
SCAN_ROUND = 1024 * 8   # k_scan_lengths: 1024 threads x SCAN_ITEMS blocks per round


def coding(a):
    return G.make_coding(**a)


def image(a, content, seed=11):
    w, h, nc, prec = a["width"], a["height"], a["numcomps"], a["prec"]
    if content == "synthetic":
        return P.synthetic_image(w, h, nc, prec, seed=seed, origin=a.get("origin", (0, 0)))
    if content == "flat":   # not mid-scale, so the LL band carries a few coded bytes
        return [np.full((h, w), (1 << prec) // 5 + 7 * c, np.int32) for c in range(nc)]
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 1 << prec, (h, w)).astype(np.int32) for _ in range(nc)]


def oracle_step(cp, planes):
    """One round-trip step: forward, HT encode of every coded block, decode of those bytes into the coefficient planes
    (each window at its tile rectangle + (buf_x, buf_y)), inverse."""
    coefs = P.forward(cp, planes)
    rects = P.tile_rects(cp)
    dec = [np.zeros_like(c) for c in coefs]
    coded, lengths, data = [], [], []
    for t, c, b in P.enumerate_all(cp):
        has_area = b.x1 > b.x0 and b.y1 > b.y0
        coded.append(has_area)
        if not has_area:
            lengths.append(0)
            continue
        d = P.encode_block(cp, coefs, rects[t], c, b)
        win = P.decode_block(cp, d, c, b)
        x0, y0 = rects[t][0] - cp.x0 + b.buf_x, rects[t][1] - cp.y0 + b.buf_y
        dec[c][y0:y0 + win.shape[0], x0:x0 + win.shape[1]] = win
        lengths.append(len(d))
        data.append(d)
    return dict(coded=np.array(coded), lengths=np.array(lengths, np.uint32),
                bytes=np.concatenate(data) if data else np.zeros(0, np.uint8), coefs=dec, pixels=P.inverse(cp, dec))


@pytest.fixture(scope="module")
def oracle():
    """oracle(a, content, k) -> the oracle's step k (1-based) of case `a` on `content`, step k coding step k-1's pixels;
    steps are computed once per module."""
    cache = {}

    def get(a, content, k=1):
        key = (repr(sorted(a.items())), content)
        steps = cache.setdefault(key, [])
        cp = coding(a)
        while len(steps) < k:
            src = steps[-1]["pixels"] if steps else image(a, content)
            steps.append(oracle_step(cp, src))
        return steps[k - 1]

    return get


def arena_after_sizing(total):
    """bytes_cap after a job's first sizing pass over an image that codes to `total` bytes (finish_t1_encode)"""
    return total + total // 8 + 4096


# ---------------------------------------------------------------------------------------------------------------------
# CPU: what the cases and call shapes reach
# ---------------------------------------------------------------------------------------------------------------------
def ranges(n, chunks, streams):
    """b2k_job_roundtrip_pipelined_n's cut of n coded blocks -> ([(b0, b1)], streams, per_chunk)"""
    chunks = max(1, min(chunks or 2, 64))
    streams = max(1, min(streams or 2, 8))
    per = max(128, -(-(-(-n // chunks)) // 128) * 128)
    return [(b0, min(n, b0 + per)) for b0 in range(0, n, per)], streams, per


def coded_blocks(cp):
    """(tile, block) of every coded block, in coded order"""
    return [(t, b) for t, c, b in P.enumerate_all(cp) if b.x1 > b.x0 and b.y1 > b.y0]


def cells(a):
    cp = coding(a)
    blocks = coded_blocks(cp)
    tiles = np.array([t for t, _ in blocks])
    n = len(blocks)
    out = set()
    for shape in SHAPES:
        rng, streams, per = ranges(n, *shape)
        if len(rng) == 1:
            out.add("one range")
        if len(rng) > streams:
            out.add("more ranges than streams")
        if any(tiles[b0 - 1] == tiles[b0] for b0, _ in rng[1:]):
            out.add("range boundary inside a tile")
        if len(rng) > 1 and rng[-1][1] - rng[-1][0] < per:
            out.add("short last range")
        if max(1, min(shape[0] or 2, 64)) == 64 and max(1, min(shape[1] or 2, 8)) == 8:
            out.add("clamped shape (64, 8)")
    if n < 128:
        out.add("fewer blocks than one range")
    if -(-n // SCAN_ROUND) >= 3 and n % 8:
        out.add("3+ scan rounds, partial last")
    if max(b.x1 - b.x0 for _, b in blocks) > 64:
        out.add("blocks wider than 64")
    if a.get("irreversible") and STEPS >= 3:
        out.add("9/7 over 3 steps")
    if a.get("numres") == 1 and cp.tw and ((cp.x1 - cp.tx0) % cp.tw or (cp.y1 - cp.ty0) % cp.th):
        out.add("point transform, ragged tiles")
    if max(P.band_params(cp, b.resno, b.orient)[0] for _, b in blocks) > PACKED_KMAX:
        out.add("Kmax above the packed staging")
    return out


ALL_CELLS = {"one range", "more ranges than streams", "range boundary inside a tile", "short last range",
             "clamped shape (64, 8)", "fewer blocks than one range", "3+ scan rounds, partial last", "blocks wider than 64",
             "9/7 over 3 steps", "point transform, ragged tiles", "Kmax above the packed staging"}


def test_cases_reach_every_cell():
    reached = set()
    for a in CASES.values():
        reached |= cells(a)
    assert reached <= ALL_CELLS, sorted(reached - ALL_CELLS)
    assert reached == ALL_CELLS, "not reached: %s" % sorted(ALL_CELLS - reached)


def test_range_model_reproduces_known_cuts():
    # 2,520 coded blocks (tiles-53): the default shape cuts two ranges of 1,280 and 1,240 blocks; (64, 8) cuts 20 ranges
    # of 128 blocks on 8 streams; (3, 2) three ranges of 896, the last one short
    n = len(coded_blocks(coding(CASES["tiles-53"])))
    assert n == 2520
    assert ranges(n, 0, 0)[0] == [(0, 1280), (1280, 2520)]
    assert ranges(n, 64, 8)[0][:2] == [(0, 128), (128, 256)] and len(ranges(n, 64, 8)[0]) == 20
    assert ranges(n, 100, 20)[1:] == ranges(n, 64, 8)[1:]
    assert [b1 - b0 for b0, b1 in ranges(n, 3, 2)[0]] == [896, 896, 728]


@pytest.mark.parametrize("irreversible", [False, True])
def test_content_changes_outgrow_the_arena(oracle, irreversible):
    """Full-range noise codes to more than the arena a flat image's sizing pass leaves (and than the arena
    t1_decode_blocks leaves for a flat image's stream), so the content-change tests below do reach the case where an
    arena taken from the earlier image is too small.  Steps 2 and 3 of each image fit the arena its own first step sizes,
    so no call here is expected to take the overflow branch."""
    a = dict(CHANGE_CASE, irreversible=irreversible)
    flat, noisy = (oracle(a, c)["bytes"].size for c in ("flat", "noise"))
    assert noisy > arena_after_sizing(flat)
    assert noisy > flat + 4096          # b2k_job_t1_decode_blocks: an arena of the caller's bytes + 4096
    for content in ("flat", "noise"):
        first = oracle(a, content, 1)["bytes"].size
        assert all(oracle(a, content, k)["bytes"].size + 64 <= arena_after_sizing(first) for k in range(2, STEPS + 1))
    assert len(P.tile_rects(coding(a))) > 1   # the host encode pipelines several chunks


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
def run(job, planes, call, steps=STEPS):
    """Upload `planes`, make one round-trip call; returns the coded byte count it reports."""
    job.upload(planes)
    kind, shape = call
    if kind == "roundtrip":
        return job.roundtrip()[2]
    if kind == "roundtrip_n":
        return job.roundtrip_n(steps)[3]
    return job.roundtrip_pipelined_n(steps, *shape)[3]


def call_steps(call):
    return 1 if call[0] == "roundtrip" else STEPS


def check_job(job, cp, want, nbytes, what):
    assert nbytes == want["bytes"].size, "%s: %d coded bytes, want %d" % (what, nbytes, want["bytes"].size)
    res = job.fetch_result()
    try:
        blocks, coded = res.blocks, want["coded"]
        bad = np.flatnonzero(blocks["length"] != want["lengths"])
        assert not len(bad), "%s: %d block lengths differ, first block %d (%d, want %d)" % (
            what, len(bad), bad[0], blocks["length"][bad[0]], want["lengths"][bad[0]])
        lengths = want["lengths"][coded].astype(np.uint64)
        assert np.array_equal(blocks["offset"][coded], np.cumsum(lengths) - lengths), what + ": offsets"
        assert (blocks["numbps"][coded] == 1).all() and (blocks["numpasses"][coded] == 1).all(), what
        assert res.num_bytes == want["bytes"].size
        diff = np.flatnonzero(res.bytes != want["bytes"])
        assert not len(diff), "%s: %d coded bytes differ, first at %d" % (what, len(diff), diff[0])
    finally:
        res.free()
    got = [np.zeros_like(p) for p in want["coefs"]]
    job.download_coeffs(got)
    for c, (g, w) in enumerate(zip(got, want["coefs"])):
        assert np.array_equal(g, w), "%s: %d decoded coefficients of component %d differ" % (what, int((g != w).sum()), c)
    job.download(got)
    for c, (g, w) in enumerate(zip(got, want["pixels"])):
        assert np.array_equal(g, w), "%s: %d pixels of component %d differ from the oracle's inverse" % (what, int((g != w).sum()), c)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_every_entry_point_matches_the_oracle(engine, oracle, name):
    a = CASES[name]
    cp = coding(a)
    planes = image(a, "synthetic")
    job = engine.job(cp)
    try:
        for call in CALLS:
            k = call_steps(call) if a.get("irreversible") else 1
            px = check_job(job, cp, oracle(a, "synthetic", k), run(job, planes, call), "%s %s" % (name, call))
            if not a.get("irreversible"):
                for g, p in zip(px, planes):
                    assert np.array_equal(g, p), "%s %s: 5/3 round trip is not lossless" % (name, call)
    finally:
        job.close()


@pytest.mark.gpu
@pytest.mark.parametrize("irreversible", [False, True], ids=["53", "97"])
@pytest.mark.parametrize("call", [CALLS[0], CALLS[1], ("pipelined", (3, 2))], ids=["roundtrip", "roundtrip_n", "pipelined"])
def test_the_image_changes_inside_one_job(engine, oracle, call, irreversible):
    """flat, full-range noise, flat again through one job: each call codes the image just uploaded, although the noise
    outgrows the arena the flat image left, and coming back to flat gives flat's bytes again."""
    a = dict(CHANGE_CASE, irreversible=irreversible)
    cp = coding(a)
    k = call_steps(call) if irreversible else 1
    job = engine.job(cp)
    try:
        sizes = []
        for content in ("flat", "noise", "flat"):
            nbytes = run(job, image(a, content), call)
            check_job(job, cp, oracle(a, content, k), nbytes, "%s after %s" % (content, sizes))
            sizes.append(nbytes)
        assert sizes[2] == sizes[0] < sizes[1]
    finally:
        job.close()


@pytest.mark.gpu
def test_round_trip_after_a_callers_arena(engine, oracle):
    """b2k_job_t1_decode_blocks leaves an arena the size of the caller's stream; a round trip after it sizes its own."""
    a = CHANGE_CASE
    cp = coding(a)
    flat = oracle(a, "flat")
    blocks = G.enumerate_blocks(cp)
    blocks["length"] = flat["lengths"]
    lengths = flat["lengths"].astype(np.uint64)
    blocks["offset"] = np.cumsum(lengths) - lengths
    blocks["numbps"][flat["coded"]] = 1
    blocks["numpasses"][flat["coded"]] = 1
    noise = image(a, "noise")
    job = engine.job(cp)
    try:
        job.t1_decode_blocks(blocks, flat["bytes"])       # a fresh job: the arena is the flat stream's
        got = [np.zeros_like(p) for p in noise]
        job.download_coeffs(got)
        assert all(np.array_equal(g, w) for g, w in zip(got, flat["coefs"]))
        check_job(job, cp, oracle(a, "noise"), run(job, noise, CALLS[0]), "noise after a caller's arena")
    finally:
        job.close()


@pytest.mark.gpu
def test_round_trip_after_an_image_made_from_coefficients(engine, oracle):
    """b2k_job_inverse of uploaded coefficients gives the job a new image without an upload: the next round trip sizes
    the arena for it, not for the flat image coded before."""
    a = CHANGE_CASE
    cp = coding(a)
    noise = image(a, "noise")
    job = engine.job(cp)
    try:
        check_job(job, cp, oracle(a, "flat"), run(job, image(a, "flat"), CALLS[0]), "flat")
        job.upload_coeffs(oracle(a, "noise")["coefs"])
        job.inverse()
        got = [np.zeros_like(p) for p in noise]
        job.download(got)
        assert all(np.array_equal(g, p) for g, p in zip(got, noise))
        check_job(job, cp, oracle(a, "noise"), job.roundtrip()[2], "noise made from coefficients")
    finally:
        job.close()


@pytest.mark.gpu
@pytest.mark.parametrize("api", ["encode", "encode_device"])
def test_host_encode_regathers_an_arena_that_was_too_small(oracle, api):
    """b2k_encode / b2k_encode_device stream every chunk's bytes home against the previous call's arena size; noise after
    flat outgrows it, and the bytes are gathered again from the coder's slots.  A fresh engine, so that its cached job
    holds the flat image's arena."""
    a = CHANGE_CASE
    cp = coding(a)
    eng = G.Engine(0)
    try:
        for content in ("flat", "noise", "flat"):
            planes = image(a, content)
            if api == "encode":
                res = eng.encode(cp, planes)
            else:
                import torch
                t = torch.from_numpy(np.stack(planes)).cuda()
                res = eng.encode_device(cp, t)
                torch.cuda.synchronize()
            want = oracle(a, content)
            try:
                assert np.array_equal(res.blocks["length"], want["lengths"]), content
                lengths = want["lengths"][want["coded"]].astype(np.uint64)
                assert np.array_equal(res.blocks["offset"][want["coded"]], np.cumsum(lengths) - lengths), content
                assert np.array_equal(res.bytes, want["bytes"]), content
                out = [np.zeros_like(p) for p in planes]
                eng.decode(cp, res.blocks.copy(), res.bytes.copy(), out)
                assert all(np.array_equal(o, p) for o, p in zip(out, planes)), content
            finally:
                res.free()
    finally:
        eng.close()
