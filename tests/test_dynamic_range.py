"""Value range: every sample precision the engine accepts (1..16), signed and unsigned samples on both paths, guard bits
0..7 and band bit-plane counts (Kmax) up to the 32-bit HT coder's limit of 29.

* The oracle's HT coder is pinned to the reference's own kernels at Kmax 19..29 (tests/golden/ht_blocks_wide.npz, made by
  tests/golden/make_golden_wide.py), so that the device tests above Kmax 24 compare with something trusted.
* The device block coder is run on coefficient planes written directly, with magnitudes that fill each band's top bit
  plane, at Kmax 24..29: a launch whose Kmax exceeds 24 takes the encoder instances that stage samples unpacked.
* The whole pipeline runs at precisions 1..16, signed and unsigned, 5/3 and 9/7, with synthetic and full-scale content.
* Streams with more guard bits and signed 9/7 streams are pinned to Grok (live where it is built, else its record).

Reversible results are bit-exact.  For 9/7 the forward coefficients and coded bytes are bit-exact, and the device's
reconstruction is within one code of the oracle's (the bar of test_gpu.py), inside [lo, hi], and exactly lo / hi
wherever the oracle's unclamped reconstruction lies a whole code or more outside the range."""
import os

import numpy as np
import pytest

import grok_b200 as G
import grok_golden as GG
import grok_ref as R
import oracle_lib as O
import oracle_pipeline as P
from grok_golden import grok
from test_codestream import oracle_decode, oracle_encode
from test_interop import strip_com

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PACKED_KMAX = 24        # b2k_launch_ht_encode: launches whose Kmax is at most this stage samples with their exponent


@pytest.fixture(scope="module", autouse=True)
def _grok():
    if R.available():
        R.init(4)
    yield


def sample_range(prec, sgnd):
    return (-(1 << (prec - 1)), (1 << (prec - 1)) - 1) if sgnd else (0, (1 << prec) - 1)


def band_kmaxes(cp):
    return [P.band_params(cp, r, o)[0] for r in range(cp.numres) for o in ((0,) if r == 0 else (1, 2, 3))]


def coding(args):
    """make_coding(**args); `qcd_raise` adds that many to every band exponent of the HT quantiser (explicit QCD)"""
    a = dict(args)
    raise_by = a.pop("qcd_raise", 0)
    cp = G.make_coding(**a)
    if raise_by:
        e, m = P.quant_tables(cp)
        cp.qcd_explicit = 1
        for i in range(len(e)):
            cp.qcd_expn[i] = int(e[i]) + raise_by
            cp.qcd_mant[i] = int(m[i])
    return cp


# ---------------------------------------------------------------------------------------------------------------------
# the case lists
# ---------------------------------------------------------------------------------------------------------------------
# block coder at full magnitude (coefficients written directly)
BLOCK_CASES = [
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=4),                                   # 5/3 top 24: packed
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=5, cblk=(32, 32)),                    # 5/3 23..25: mixed
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=7, tile=(61, 40), origin=(3, 5)),     # 5/3 25..27
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=7, qcd_raise=2),                      # 5/3 up to 29
    dict(width=1100, height=12, numcomps=1, prec=16, numres=2, numgbits=6, cblk=(1024, 4)),                  # widest blocks
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=3, irreversible=True),                # 9/7 top 24: packed
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=4, irreversible=True),                # 9/7 21..25: mixed
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=7, irreversible=True, cblk=(16, 64)),  # 9/7 24..28
    dict(width=128, height=96, numcomps=3, prec=16, numres=6, numgbits=7, irreversible=True, qcd_raise=1),   # 9/7 up to 29
    dict(width=96, height=80, numcomps=1, prec=16, sgnd=True, numres=4, numgbits=7, irreversible=True, qcd_raise=1, cblk=(4, 4)),
]

# the whole pipeline: precision x sign x path, geometry taken in turn
SWEEP_PRECS = list(range(1, 17))
SWEEP_GEOMS = [
    dict(width=128, height=96, numcomps=1, numres=1),
    dict(width=128, height=96, numcomps=3, numres=3, origin=(3, 5)),                    # MCT, odd origin
    dict(width=125, height=93, numcomps=4, numres=6, tile=(61, 40), origin=(5, 2)),     # MCT + a 4th component, ragged tiles
]
SWEEP = [dict(prec=p, sgnd=s, irreversible=irr, **SWEEP_GEOMS[(i + int(s) + 2 * int(irr)) % len(SWEEP_GEOMS)])
         for i, p in enumerate(SWEEP_PRECS) for s in (False, True) for irr in (False, True)]

CONTENT_GEOM = dict(width=128, height=96, numcomps=3, numres=5, tile=(96, 64), origin=(1, 3))
CONTENTS = ["const_min", "const_max", "checkerboard", "impulse_grid", "noise"]

# guard bits on the host entry points (int32 and 16-bit containers)
GUARD = [dict(width=160, height=120, numcomps=3, prec=p, sgnd=(p == 12), numres=5, tile=(128, 64), numgbits=g, irreversible=irr)
         for p in (12, 16) for irr in (False, True) for g in range(8)]

# code streams pinned to Grok
GROK_CASES = [
    dict(width=160, height=120, numcomps=3, prec=12, sgnd=True, numres=5, irreversible=True),
    dict(width=160, height=120, numcomps=3, prec=16, sgnd=True, numres=5, irreversible=True),
    dict(width=160, height=120, numcomps=3, prec=3, numres=5),
    dict(width=160, height=120, numcomps=3, prec=16, numres=6, numgbits=5),                      # Kmax 25
    dict(width=160, height=120, numcomps=3, prec=16, numres=6, numgbits=6, irreversible=True),   # Kmax 27
]


def test_case_lists_cover_the_range():
    """The matrices above keep their point: every precision, both signs on both paths, Kmax above the packed staging's
    limit on both paths (the unpacked encoder instances), mixed launches, and Kmax 29."""
    precs = {a["prec"] for a in SWEEP + GUARD + GROK_CASES + BLOCK_CASES} | {8, 16}       # 8 and 16: the content sweep
    assert precs == set(range(1, 17))
    assert {(a["sgnd"], a["irreversible"]) for a in SWEEP} == {(s, i) for s in (False, True) for i in (False, True)}
    for irr in (False, True):
        tops = [max(band_kmaxes(coding(a))) for a in BLOCK_CASES if bool(a.get("irreversible")) == irr]
        assert PACKED_KMAX in tops and max(tops) == 29
        assert any(min(band_kmaxes(coding(a))) <= PACKED_KMAX < max(band_kmaxes(coding(a)))
                   for a in BLOCK_CASES if bool(a.get("irreversible")) == irr)
    assert {g["numgbits"] for g in GUARD} == set(range(8))
    assert max(band_kmaxes(coding(GROK_CASES[3]))) == 25 and max(band_kmaxes(coding(GROK_CASES[4]))) == 27


# ---------------------------------------------------------------------------------------------------------------------
# 1. the oracle's HT coder against the reference's, Kmax 19..29 (CPU)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def wide_gold():
    return np.load(os.path.join(GOLD, "ht_blocks_wide.npz"))


def test_ht_coder_matches_reference_at_kmax_19_to_29(wide_gold):
    g = wide_gold
    Rf = O.ref()
    seen = set()
    for i in range(int(g["count"])):
        sm, kmax, want = g["in%03d" % i], int(g["kmax%03d" % i]), g["out%03d" % i]
        h, w = sm.shape
        seen.add(kmax)
        enc = O.ht_encode(sm, kmax)
        assert np.array_equal(enc, want), (i, kmax, w, h)
        rc, dec = O.ht_decode(want, kmax, w, h)
        assert rc == 0 and np.array_equal(dec, g["dec%03d" % i]), (i, kmax, w, h)
        mu = ((sm & 0x7FFFFFFF) >> (30 - kmax)).astype(np.uint64)
        bc = np.where(mu > 0, (sm & 0x80000000) | ((2 * mu + 1) << np.uint64(29 - kmax)), 0).astype(np.uint32)
        assert np.array_equal(dec, bc), (i, kmax)                 # sign | (2 mu + 1) << (p - 1): lossless at every Kmax
        if Rf is not None:
            theirs = [t for t in (O.ref_ht_encode(sm, kmax, v) for v in (0, 1, 2)) if t is not None]
            assert all(np.array_equal(want, t) for t in theirs), (i, kmax)
            rc2, d2 = O.ref_ht_decode(want, kmax, w, h, 0)
            assert rc2 == 0 and np.array_equal(d2, g["dec%03d" % i]), (i, kmax)
    assert seen == set(range(19, 30))


def test_ht_refinement_passes_match_reference_at_kmax_25_to_29(wide_gold):
    g = wide_gold
    Rf = O.ref()
    seen = set()
    for i in range(int(g["rcount"])):
        w, h, M, npass, len2, causal, kmax = (int(v) for v in g["rmeta%03d" % i])
        data, sm = g["rdata%03d" % i], g["rsrc%03d" % i]
        seen.add((kmax, npass, causal))
        assert np.array_equal(np.concatenate([O.ht_encode(sm, M), O.ht_encode_refine(sm, M, npass, bool(causal))]), data), i
        rc, dec = O.ht_decode_passes(data, len2, npass, M, w, h, causal=bool(causal))
        assert rc == 0 and np.array_equal(dec, g["rdec%03d" % i]), (i, kmax, M, npass, causal)
        if Rf is not None:
            rc2, d2 = O.ref_ht_decode(data, M, w, h, variant=-1, num_passes=npass, len2=len2, causal=bool(causal))
            assert rc2 == 0 and np.array_equal(d2, g["rdec%03d" % i]), i
    assert {k for k, _, _ in seen} == set(range(25, 30)) and {(n, c) for _, n, c in seen} == {(2, 0), (2, 1), (3, 0), (3, 1)}


# ---------------------------------------------------------------------------------------------------------------------
# 2. the device block coder at full magnitude
# ---------------------------------------------------------------------------------------------------------------------
def _rev_block(kind, kmax, h, w, rng):
    lim = (1 << kmax) - 1
    if kind == 0:
        return np.where((np.add.outer(np.arange(h), np.arange(w)) & 1) == 0, lim, -lim)
    if kind == 1:
        c = np.zeros((h, w), np.int64)
        c[int(rng.integers(0, h)), int(rng.integers(0, w))] = lim * int(rng.choice([-1, 1]))
        return c
    if kind == 2:
        return np.zeros((h, w), np.int64)
    return rng.integers(-lim, lim + 1, (h, w))


def full_scale_coefficients(cp, seed):
    """Coefficient planes (int32, or float bits for 9/7) whose code blocks, by turns, are full-scale checkerboards
    +-(2^Kmax - 1), one isolated maximum, all zero and random over the band's whole range.  For 9/7 the values are
    chosen so that the quantised indices fill the band's planes; the premise -- every index below 2^Kmax, the top
    plane reached -- is asserted on the oracle's quantiser."""
    rng = np.random.default_rng(seed)
    w, h = cp.x1 - cp.x0, cp.y1 - cp.y0
    out = [np.zeros((h, w), np.int32) for _ in range(cp.numcomps)]
    rects = P.tile_rects(cp)
    for i, (t, c, b) in enumerate(P.enumerate_all(cp)):
        bw, bh = b.x1 - b.x0, b.y1 - b.y0
        if bw == 0 or bh == 0:
            continue
        kmax, step_enc, _ = P.band_params(cp, b.resno, b.orient)
        idx = _rev_block(i % 4, kmax, bh, bw, rng)
        x0, y0 = rects[t][0] - cp.x0 + b.buf_x, rects[t][1] - cp.y0 + b.buf_y
        if not cp.irreversible:
            out[c][y0:y0 + bh, x0:x0 + bw] = idx
            continue
        # a float32 holds 24 bits: keep the targets far enough below 2^Kmax that rounding cannot reach it
        top = (1 << kmax) - 1 - (1 << max(0, kmax - 21))
        idx = np.clip(idx, -top, top)
        f = (np.sign(idx) * (np.abs(idx) + 0.5) * float(step_enc)).astype(np.float32)
        shift = 30 - kmax
        t32 = (f * (np.float32(1.0) / np.float32(step_enc))) * np.float32(1 << shift)   # orc_ht_pre_irrev's product, float32
        q = np.abs(np.trunc(t32.astype(np.float64)).astype(np.int64)) >> shift
        assert q.max() < (1 << kmax), (kmax, int(q.max()))
        if i % 4 in (0, 1):
            assert q.max() >= (1 << (kmax - 1)), (kmax, int(q.max()))
        out[c][y0:y0 + bh, x0:x0 + bw] = f.view(np.int32)
    return out


def compare_blocks(cp, res, coefs):
    blks = P.enumerate_all(cp)
    rects = P.tile_rects(cp)
    assert len(blks) == res.num_blocks
    for i, (t, c, b) in enumerate(blks):
        if b.x1 == b.x0 or b.y1 == b.y0:
            assert res.blocks[i]["length"] == 0
            continue
        want = P.encode_block(cp, coefs, rects[t], c, b)
        assert np.array_equal(want, res.block_bytes(i)), "code block %d (res %d orient %d kmax %d)" % (
            i, b.resno, b.orient, P.band_params(cp, b.resno, b.orient)[0])


def oracle_block_decode(cp, res):
    """the oracle's decode of the device's coded blocks, as coefficient planes"""
    w, h = cp.x1 - cp.x0, cp.y1 - cp.y0
    out = [np.zeros((h, w), np.int32) for _ in range(cp.numcomps)]
    rects = P.tile_rects(cp)
    for i, (t, c, b) in enumerate(P.enumerate_all(cp)):
        bw, bh = b.x1 - b.x0, b.y1 - b.y0
        if bw == 0 or bh == 0:
            continue
        x0, y0 = rects[t][0] - cp.x0 + b.buf_x, rects[t][1] - cp.y0 + b.buf_y
        out[c][y0:y0 + bh, x0:x0 + bw] = P.decode_block(cp, res.block_bytes(i), c, b)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("args", BLOCK_CASES)
def test_block_coder_at_full_magnitude(engine, args):
    cp = coding(args)
    coefs = full_scale_coefficients(cp, seed=len(args) + args["numgbits"])
    job = engine.job(cp)
    try:
        _block_coder_job(job, cp, coefs, args)
    finally:
        job.close()


def _block_coder_job(job, cp, coefs, args):
    job.upload([np.zeros_like(p) for p in coefs])          # sizes the planes; the coefficients are written below
    job.upload_coeffs(coefs)
    job.t1_encode()
    res = job.fetch_result()
    assert int(res.blocks["kmax"].max()) == max(band_kmaxes(cp))
    compare_blocks(cp, res, coefs)
    got = [np.full_like(p, -1) for p in coefs]
    job.upload_coeffs(got)
    job.t1_decode()
    job.download_coeffs(got)
    want = oracle_block_decode(cp, res)
    for c, (g, r) in enumerate(zip(got, want)):
        assert np.array_equal(g, r), "component %d: %d coefficients differ from the oracle's decode" % (c, int((g != r).sum()))
        if not cp.irreversible:
            assert np.array_equal(g, coefs[c])
    res.free()
    if max(band_kmaxes(cp)) >= 25 and args.get("qcd_raise"):
        # foreign streams: cleanup pass one or two planes above the LSB, SigProp (+ MagRef) below it
        from test_gpu import _refined_blocks
        table, data, want = _refined_blocks(cp, coefs, 3, 1 + (args["numgbits"] & 1), seed=5)
        assert (table["numpasses"] > 1).sum() > 0
        got = [np.full_like(p, -1) for p in coefs]
        job.upload_coeffs(got)
        job.t1_decode_blocks(table, data)
        job.download_coeffs(got)
        for c, (g, r) in enumerate(zip(got, want)):
            assert np.array_equal(g, r), "refined, component %d: %d coefficients differ" % (c, int((g != r).sum()))


# ---------------------------------------------------------------------------------------------------------------------
# 3. the whole pipeline at every precision, signed and unsigned, both paths
# ---------------------------------------------------------------------------------------------------------------------
def content(kind, args, seed=3):
    w, h, n, prec, sgnd = args["width"], args["height"], args["numcomps"], args["prec"], args.get("sgnd", False)
    lo, hi = sample_range(prec, sgnd)
    origin = args.get("origin", (0, 0))
    y, x = np.mgrid[origin[1]:origin[1] + h, origin[0]:origin[0] + w]
    if kind == "synthetic":
        planes = P.synthetic_image(w, h, n, prec, seed=seed, origin=origin)
        return [p + lo for p in planes]
    if kind == "const_min":
        return [np.full((h, w), lo, np.int32) for _ in range(n)]
    if kind == "const_max":
        return [np.full((h, w), hi, np.int32) for _ in range(n)]
    if kind == "checkerboard":      # G opposite to R and B: both colour transforms reach their extremes
        return [np.where((x + y + c + (c >> 1)) & 1, hi, lo).astype(np.int32) for c in range(n)]
    if kind == "impulse_grid":
        return [np.where(((x + 2 * c) % 7 == 0) & ((y + c) % 5 == 0), hi, lo).astype(np.int32) for c in range(n)]
    rng = np.random.default_rng(seed)
    return [rng.integers(lo, hi + 1, (h, w)).astype(np.int32) for _ in range(n)]


def inverse97_unclamped(cp, coefs):
    """P.inverse for 9/7 without the final clamp (int64 planes)"""
    L = O.lib()
    H, W = coefs[0].shape
    out = [np.zeros((H, W), np.int64) for _ in coefs]
    sh = -P.dc_shift(cp)
    wide = np.array([-(1 << 30)] * 3, np.int32), np.array([1 << 30] * 3, np.int32)
    for (x0, y0, x1, y1) in P.tile_rects(cp):
        w, h = x1 - x0, y1 - y0
        sl = (slice(y0 - cp.y0, y1 - cp.y0), slice(x0 - cp.x0, x1 - cp.x0))
        fl = []
        for c in range(len(coefs)):
            buf = np.ascontiguousarray(coefs[c][sl]).view(np.float32).copy()
            L.orc_dwt97_inv_2d(buf, w, x0, y0, x1, y1, cp.numres)
            fl.append(buf)
        if cp.mct:
            r, g, b = (np.zeros(w * h, np.int32) for _ in range(3))
            L.orc_ict_inv(fl[0].ravel(), fl[1].ravel(), fl[2].ravel(), r, g, b, w * h, np.array([sh] * 3, np.int32), *wide)
            out[0][sl], out[1][sl], out[2][sl] = r.reshape(h, w), g.reshape(h, w), b.reshape(h, w)
        for c in range(3 if cp.mct else 0, len(coefs)):
            out[c][sl] = np.rint(fl[c]).astype(np.int64) + sh
    return out


def run_pipeline(engine, cp, planes):
    """forward -> block encode -> block decode -> inverse on the device, each stage against the oracle.  Returns the
    number of 9/7 samples whose clamp was checked exactly."""
    lo, hi = sample_range(cp.prec, cp.sgnd)
    for p in planes:
        assert p.min() >= lo and p.max() <= hi
    ref = P.forward(cp, planes)
    job = engine.job(cp)
    try:
        return _run_pipeline_job(job, cp, planes, ref, lo, hi)
    finally:
        job.close()


def _run_pipeline_job(job, cp, planes, ref, lo, hi):
    job.upload(planes)
    job.forward()
    got = [np.zeros_like(p) for p in planes]
    job.download_coeffs(got)
    for c, (g, r) in enumerate(zip(got, ref)):
        assert np.array_equal(g, r), "forward, component %d: %d coefficients differ" % (c, int((g != r).sum()))
    job.t1_encode()
    res = job.fetch_result()
    compare_blocks(cp, res, ref)
    for p in got:
        p[:] = -1
    job.upload_coeffs(got)
    job.t1_decode()
    job.download_coeffs(got)
    dec = oracle_block_decode(cp, res)
    for c, (g, r) in enumerate(zip(got, dec)):
        assert np.array_equal(g, r), "block decode, component %d: %d coefficients differ" % (c, int((g != r).sum()))
    res.free()
    job.inverse()
    rec = [np.zeros_like(p) for p in planes]
    job.download(rec)
    if not cp.irreversible:
        for c, (g, s) in enumerate(zip(rec, planes)):
            assert np.array_equal(g, s), "component %d: %d samples differ from the source" % (c, int((g != s).sum()))
        return 0
    oracle_rec = P.inverse(cp, dec)
    wide = inverse97_unclamped(cp, dec)
    checked = 0
    for c, (g, r, u, s) in enumerate(zip(rec, oracle_rec, wide, planes)):
        assert np.array_equal(g, r), "component %d: %d samples differ from the oracle's inverse" % (c, int((g != r).sum()))
        assert g.min() >= lo and g.max() <= hi, "component %d outside [%d, %d]" % (c, lo, hi)
        over, under = u >= hi + 1, u <= lo - 1
        assert np.all(g[over] == hi) and np.all(g[under] == lo), "component %d: the clamp is off" % c
        checked += int(over.sum() + under.sum())
        assert np.abs(g.astype(np.int64) - s).max() <= np.abs(r.astype(np.int64) - s).max() + 1
    return checked


@pytest.mark.gpu
@pytest.mark.parametrize("args", SWEEP, ids=lambda a: "p%d-%s-%s-%dc" % (a["prec"], "s" if a["sgnd"] else "u",
                                                                         "97" if a["irreversible"] else "53", a["numcomps"]))
def test_precision_sign_path_sweep(engine, args):
    cp = coding(args)
    for kind in ("synthetic", "checkerboard"):
        run_pipeline(engine, cp, content(kind, args, seed=args["prec"]))


@pytest.mark.gpu
@pytest.mark.parametrize("prec", [8, 16])
@pytest.mark.parametrize("sgnd", [False, True])
@pytest.mark.parametrize("irreversible", [False, True])
def test_content_sweep(engine, prec, sgnd, irreversible):
    args = dict(CONTENT_GEOM, prec=prec, sgnd=sgnd, irreversible=irreversible)
    cp = coding(args)
    checked = sum(run_pipeline(engine, cp, content(kind, args)) for kind in CONTENTS)
    if irreversible:
        assert checked > 0          # full-scale content drives the 9/7 reconstruction past both ends of the range


# ---------------------------------------------------------------------------------------------------------------------
# 4. guard bits 0..7 through the host entry points, int32 and 16-bit containers
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("args", GUARD, ids=lambda a: "p%d-%s-g%d" % (a["prec"], "97" if a["irreversible"] else "53", a["numgbits"]))
def test_guard_bits_on_the_host_entry_points(engine, args):
    cp = coding(args)
    planes = content("synthetic", args, seed=args["numgbits"])
    coefs = P.forward(cp, planes)
    res = engine.encode(cp, planes)
    compare_blocks(cp, res, coefs)
    blocks, data = res.blocks.copy(), res.bytes.copy()
    res.free()
    p16 = [p.astype(np.int16 if cp.sgnd else np.uint16) for p in planes]
    r16 = engine.encode(cp, p16)
    assert np.array_equal(r16.blocks["length"], blocks["length"]) and np.array_equal(r16.bytes, data)
    r16.free()
    out = [np.zeros_like(p) for p in planes]
    engine.decode(cp, blocks, data, out)
    out16 = [np.zeros_like(p) for p in p16]
    engine.decode(cp, blocks, data, out16)
    for a, b in zip(out16, out):
        assert np.array_equal(a.astype(np.int32), b)
    if cp.irreversible:
        for a, r in zip(out, oracle_decode(cp, blocks, data)):
            assert np.abs(a - r).max() <= 1
    else:
        for a, s in zip(out, planes):
            assert np.array_equal(a, s)


# ---------------------------------------------------------------------------------------------------------------------
# 5. code streams: headers, and Grok's streams
# ---------------------------------------------------------------------------------------------------------------------
HEADER_CASES = GROK_CASES + [BLOCK_CASES[3], BLOCK_CASES[8], BLOCK_CASES[9]] + [a for a in SWEEP if a["prec"] in (1, 7, 13)] + \
    [g for g in GUARD if g["numgbits"] in (0, 7)]


@pytest.mark.parametrize("args", HEADER_CASES)
def test_codestream_header_keeps_precision_sign_guard_bits_and_exponents(args):
    cp = coding(args)
    planes = content("synthetic", args, seed=1)
    table, data, _ = oracle_encode(cp, planes)
    cs = G.codestream_write(cp, table, data, G.CS_TLM | G.CS_PLT)
    cp2, blocks = G.codestream_parse(cs)
    assert (cp2.prec, cp2.sgnd, cp2.numgbits, cp2.irreversible) == (cp.prec, cp.sgnd, cp.numgbits, cp.irreversible)
    e1, m1 = P.quant_tables(cp)
    e2, m2 = P.quant_tables(cp2)
    assert np.array_equal(e1, e2) and np.array_equal(m1, m2)
    assert band_kmaxes(cp2) == band_kmaxes(cp)
    assert np.array_equal(blocks["length"], table["length"])


def _grok_compress(args, planes):
    cs, _ = R.compress(planes, args["prec"], sgnd=args.get("sgnd", False), numres=args.get("numres", 6),
                       irreversible=args.get("irreversible", False), tlm=True, plt=True, numgbits=args.get("numgbits", 1))
    return np.frombuffer(bytes(cs), np.uint8)


def _grok_decode(cs, args):
    return grok(lambda: R.decompress(cs, args["width"], args["height"], args["numcomps"])[0])


GROK_SEED = 17


@pytest.mark.parametrize("args", GROK_CASES)
def test_oracle_streams_equal_grok(args):
    cp = coding(args)
    planes = content("synthetic", args, seed=GROK_SEED)
    table, data, _ = oracle_encode(cp, planes)
    ours = G.codestream_write(cp, table, data, G.CS_TLM | G.CS_PLT)
    theirs = GG.grok_stream(GG.key("stream", args, GROK_SEED), ours, grok(lambda: _grok_compress(args, planes)))
    assert bytes(ours) == strip_com(theirs)
    cp2, blocks = G.codestream_parse(theirs)
    assert (cp2.prec, cp2.sgnd, cp2.numgbits) == (cp.prec, cp.sgnd, cp.numgbits)
    od = oracle_decode(cp2, blocks, theirs)
    k = GG.key("grok decode", args, GROK_SEED)
    if args.get("irreversible"):
        GG.close(k, od, _grok_decode(theirs, args), tol=0)
    else:
        for a, b in zip(od, planes):
            assert np.array_equal(a, b)
        GG.same(k, planes, _grok_decode(theirs, args))


@pytest.mark.gpu
@pytest.mark.parametrize("args", GROK_CASES)
def test_device_streams_equal_grok_and_decode_it(engine, args):
    cp = coding(args)
    planes = content("synthetic", args, seed=GROK_SEED)
    ours = engine.encode_codestream(cp, planes, flags=G.CS_TLM | G.CS_PLT)
    theirs = GG.grok_stream(GG.key("stream", args, GROK_SEED), ours, grok(lambda: _grok_compress(args, planes)))
    assert bytes(ours) == strip_com(theirs), "the device's code stream differs from grk_compress's"
    _, rec = engine.decode_codestream(theirs)
    k = GG.key("grok decode", args, GROK_SEED)
    if args.get("irreversible"):
        GG.close(k, rec, _grok_decode(theirs, args), tol=1)
    else:
        for a, s in zip(rec, planes):
            assert np.array_equal(a, s)
        GG.same(k, rec, _grok_decode(theirs, args))


# ---------------------------------------------------------------------------------------------------------------------
# 6. the edge of the range
# ---------------------------------------------------------------------------------------------------------------------
KMAX30 = [dict(width=64, height=64, numcomps=3, prec=16, numres=6, numgbits=7, qcd_raise=3),
          dict(width=64, height=64, numcomps=3, prec=16, numres=6, numgbits=7, irreversible=True, qcd_raise=2)]


@pytest.mark.parametrize("args", KMAX30)
def test_kmax_30_is_refused(args):
    cp = coding(args)
    assert max(band_kmaxes(cp)) == 30
    with pytest.raises(G.EngineError, match="band bit planes outside"):
        G.enumerate_blocks(cp)
    a = dict(args, qcd_raise=args["qcd_raise"] - 1)      # one plane less is accepted
    assert len(G.enumerate_blocks(coding(a))) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("args", KMAX30)
def test_kmax_30_is_not_handled_on_the_device(engine, args):
    with pytest.raises(G.EngineError, match=r"b2k_job_create -> 1: band bit planes outside"):
        engine.job(coding(args))
