"""Every staging path of the four lifting kernels (dwt.cu), both directions, bit for bit against the oracle.

A warp job of k_dwt53_fwd / k_dwt97_fwd / k_dwt53_inv / k_dwt97_inv (each built for NC = 1 and NC = 3 components)
brings its rows into shared memory one of three ways: the unpipelined degenerate job (a line one sample wide or
high), per-lane cp.async copies with mirrored edge lanes, or bulk (TMA) copies issued by lane 0 when all 32 lanes
are interior and 16-byte aligned.  Which one it takes follows from the tile and resolution geometry, the canvas
origin against the plane layout and the job count of the whole launch, which also sets the row-segment length
(32, 16 or 8 pairs).  `job_paths` restates those rules; the CPU tests check them on known plans and that the
cases below reach every cell of them, and the GPU tests compare the device with the oracle on every case:
  - forward: the coefficients bit for bit (int32, float bits for 9/7);
  - inverse: the oracle's forward coefficients with a seeded perturbation in every band (so that matched forward
    and inverse errors cannot cancel), reconstructed exactly -- 9/7 included: the device does the oracle's float
    operations in the oracle's order, so anything but equality is a kernel error.
"""
import functools

import numpy as np
import pytest

import grok_b200 as G
import oracle_pipeline as P

# ---------------------------------------------------------------------------------------------------------------------
# the path model
# ---------------------------------------------------------------------------------------------------------------------
RESIDENT_JOBS = 3552        # build_dwt_plan: segments are halved until a launch has this many warp jobs (or 8 pairs)
FILTERS = ("53", "97")


def _cdiv(a, b):
    return -(-a // b)


def _res_rect(tc, numres, resno):
    n = numres - 1 - resno
    return tuple(_cdiv(v, 1 << n) for v in tc)


def _strips(rect, pairs):
    """fill_strips: (number of strips, strip width, number of row segments) of a descriptor"""
    u0, v0, u1, v1 = rect
    span = u1 - (u0 & ~7)
    ns = max(1, (span + 239) // 240)
    sw = (_cdiv(span, ns) + 7) & ~7
    npairs = ((v1 - 1) >> 1) - (v0 >> 1) + 1
    return ns, sw, _cdiv(npairs, pairs)


def dwt_plan(cp):
    """build_dwt_plan: per level (finest first) the level-1 MCT-group launch (NC = 3) and the single-component launch
    (NC = 1), each with its segment length in pairs and its descriptors.  The inverse runs the same launches."""
    L = cp.numres - 1
    X0 = cp.x0 & ~31                     # alloc_planes: canvas column at column 0 of the image / coefficient planes
    out = []
    for lvl in range(1, L + 1):
        groups = {3: [], 1: []}
        for tc in P.tile_rects(cp):
            r = _res_rect(tc, cp.numres, cp.numres - lvl)
            if r[2] <= r[0] or r[3] <= r[1]:
                continue
            c = 0
            while c < cp.numcomps:
                nc = 3 if (lvl == 1 and cp.mct and c == 0) else 1
                groups[nc].append(dict(rect=r, cbase=tc[0] - X0, coarsest=lvl == L))
                c += nc
        for nc in (3, 1):
            descs = groups[nc]
            if not descs:
                continue
            pairs = 32
            while pairs > 8 and sum(_strips(d["rect"], pairs)[0] * _strips(d["rect"], pairs)[2] for d in descs) < RESIDENT_JOBS:
                pairs >>= 1
            out.append(dict(level=lvl, nc=nc, pairs=pairs, descs=descs))
    return out


def _strip_paths(d, pairs):
    """(forward path, inverse path, inverse refused for alignment alone) of each strip of descriptor d.
    Forward (RowStage::lane_fast): bulk when every lane's 8 columns lie inside the line.  Their 16-byte alignment always
    holds: the planes start at canvas columns that are multiples of 32 (alloc_planes) and a lane's columns at multiples
    of 8.  Inverse (BandStage::setup, all_fast): bulk when every lane's LL, HL, LH and HH quads lie inside the line and
    are 16-byte aligned in their planes: the coefficient plane, whose column 0 is canvas column X0 of the tile's
    image, and for LL above the coarsest level the LL scratch plane, whose column 0 is band column 0."""
    u0, v0, u1, v1 = d["rect"]
    wn, hn = u1 - u0, v1 - v0
    ns, sw, _ = _strips(d["rect"], pairs)
    if wn == 1 or hn == 1:
        return [("degenerate", "degenerate", False)] * ns
    x0l, x0h = (u0 + 1) >> 1, u0 >> 1
    snx = ((u1 + 1) >> 1) - x0l
    cbase = d["cbase"]
    llbase = cbase if d["coarsest"] else x0l
    out = []
    for s in range(ns):
        fwd = interior = aligned = True
        for lane in range(32):                 # decode_job
            ulane = (u0 & ~7) + s * sw + (lane - 1) * 8
            need = lane <= (sw >> 3) + 1 and ulane < u1 + 8
            rel = ulane - u0
            fwd = fwd and need and rel >= 0 and rel + 8 <= wn
            k0 = ulane >> 1
            interior = interior and need and 2 * k0 >= u0 and 2 * k0 + 7 < u1
            aligned = aligned and (llbase + k0 - x0l) % 4 == 0 and (cbase + snx + k0 - x0h) % 4 == 0 \
                and (cbase + k0 - x0l) % 4 == 0
        out.append(("bulk" if fwd else "async", "bulk" if interior and aligned else "async", interior and not aligned))
    return out


def job_paths(cp):
    """For each level launch of a coding: its level, NC, segment length in pairs, and how many of its warp jobs take
    each path, forward ("fwd") and inverse ("inv")."""
    out = []
    for launch in dwt_plan(cp):
        counts = {"fwd": {}, "inv": {}}
        for d in launch["descs"]:
            nseg = _strips(d["rect"], launch["pairs"])[2]
            for fwd, inv, _ in _strip_paths(d, launch["pairs"]):
                counts["fwd"][fwd] = counts["fwd"].get(fwd, 0) + nseg
                counts["inv"][inv] = counts["inv"].get(inv, 0) + nseg
        out.append(dict(level=launch["level"], nc=launch["nc"], pairs=launch["pairs"], **counts))
    return out


def _reflects_twice(lo, hi, n):
    """an index range [lo, hi] used on a line of n samples needs more than one reflection (mirror_rel_slow)"""
    return lo < -(n - 1) or hi > 2 * (n - 1)


# rows a warp job reads below and above its pairs [jbeg, jend): forward 5/3 rows 2(jbeg-1) .. 2 jend, 9/7
# 2(jbeg-2) .. 2 jend+2; inverse 5/3 the band rows of pairs jbeg-1 .. jend, 9/7 of pairs jbeg-2 .. jend+1
_ROW_HALO = {("fwd", "53"): (2, 0), ("fwd", "97"): (4, 2), ("inv", "53"): (2, 1), ("inv", "97"): (4, 3)}


def cells(cp, filt):
    """The cells a coding reaches with filter `filt`: (direction, filter, NC, path), ("seg", filter, NC, pairs) and
    (direction, filter, boundary condition) for the conditions of non-degenerate descriptors."""
    out = set()
    for launch in job_paths(cp):
        out.add(("seg", filt, launch["nc"], launch["pairs"]))
        for dirn in ("fwd", "inv"):
            out |= {(dirn, filt, launch["nc"], path) for path in launch[dirn]}
    for launch in dwt_plan(cp):
        pairs = launch["pairs"]
        for d in launch["descs"]:
            u0, v0, u1, v1 = d["rect"]
            wn, hn = u1 - u0, v1 - v0
            ns, sw, nseg = _strips(d["rect"], pairs)
            paths = _strip_paths(d, pairs)
            if paths[0][0] == "degenerate":
                continue
            if any(refused for _, _, refused in paths):
                out.add(("inv", filt, "unaligned_origin"))
            jlo, jhi = v0 >> 1, (v1 - 1) >> 1
            # columns the needed lanes use: from lane 0 of the first strip to the last needed lane of the last one
            last = (u0 & ~7) + (ns - 1) * sw
            cmax = max(last + (lane - 1) * 8 for lane in range((sw >> 3) + 2) if last + (lane - 1) * 8 < u1 + 8) + 7
            for dirn in ("fwd", "inv"):
                below, above = _ROW_HALO[(dirn, filt)]
                if _reflects_twice(2 * jlo - below - v0, 2 * (jhi + 1) + above - v0, hn) or \
                        _reflects_twice((u0 & ~7) - 8 - u0, cmax - u0, wn):
                    out.add((dirn, filt, "short_line"))
                if u0 & 1:
                    out.add((dirn, filt, "odd_u0"))
                if v0 & 1:
                    out.add((dirn, filt, "odd_v0"))
                if nseg > 1 and (jhi - jlo + 1) % pairs == 1:
                    out.add((dirn, filt, "one_pair_segment"))
                if ns > 1 and (u0 & ~7) + ns * sw > u1:
                    out.add((dirn, filt, "ragged_strip"))
    return out


BOUNDARIES = ("short_line", "odd_u0", "odd_v0", "one_pair_segment", "ragged_strip")
ALL_CELLS = ({(dirn, f, nc, p) for dirn in ("fwd", "inv") for f in FILTERS for nc in (1, 3)
              for p in ("bulk", "async", "degenerate")}
             | {("seg", f, nc, p) for f in FILTERS for nc in (1, 3) for p in (8, 16, 32)}
             | {(dirn, f, b) for dirn in ("fwd", "inv") for f in FILTERS for b in BOUNDARIES}
             | {("inv", f, "unaligned_origin") for f in FILTERS})

# ---------------------------------------------------------------------------------------------------------------------
# the cases: every one runs with both filters
# ---------------------------------------------------------------------------------------------------------------------
CASES = {
    # three 240-column strips, the middle one interior: bulk on both sides, NC = 3 (components 0-2) and NC = 1 (3)
    "bulk": dict(width=720, height=200, numcomps=4, prec=12, numres=2),
    # the same strip width at origin x = 4: the forward takes bulk, the inverse's band quads are not 16-byte aligned
    "bulk-unaligned": dict(width=712, height=70, numcomps=4, prec=12, numres=3, origin=(4, 3)),
    # odd origin on every level, ragged last strips
    "odd-origin": dict(width=501, height=183, numcomps=4, prec=16, numres=6, origin=(3, 5)),
    # tiles one column wide and one row high: degenerate jobs, NC = 3 and 1
    "one-column-tiles": dict(width=23, height=37, numcomps=4, prec=12, numres=3, tile=(1, 37)),
    "one-row-tiles": dict(width=45, height=9, numcomps=4, prec=12, numres=2, tile=(45, 1), origin=(0, 4)),
    # 800 tiles of 16x130: level 1 has 2400 jobs of 32 pairs, so it runs in 16-pair segments, the last of one pair
    "seg16": dict(width=640, height=2600, numcomps=4, prec=16, numres=2, tile=(16, 130)),
    # 1200 such tiles: 32-pair segments on every level, the last of one pair at level 1; level 3 lines are 4 columns
    # wide, shorter than the lifting halo
    "seg32": dict(width=640, height=3900, numcomps=4, prec=16, numres=4, tile=(16, 130)),
}
ORDER = list(CASES)     # cheapest first


def coding(name, filt):
    return G.make_coding(irreversible=filt == "97", **CASES[name])


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the model and the case list
# ---------------------------------------------------------------------------------------------------------------------
def test_cases_reach_every_cell():
    reached = set()
    for name in CASES:
        for filt in FILTERS:
            reached |= cells(coding(name, filt), filt)
    assert reached <= ALL_CELLS, sorted(reached - ALL_CELLS, key=str)
    assert reached == ALL_CELLS, "not reached: %s" % sorted(ALL_CELLS - reached, key=str)


def test_model_reproduces_known_plans():
    # config 2 (8192x8192x3, 1024x1024 tiles): 208-column strips at level 1, and no bulk copy on any level
    cp2 = G.make_coding(8192, 8192, 3, 12, numres=6, tile=(1024, 1024))
    lvl1 = dwt_plan(cp2)[0]
    assert (lvl1["level"], lvl1["nc"]) == (1, 3)
    assert {_strips(d["rect"], lvl1["pairs"])[:2] for d in lvl1["descs"]} == {(5, 208)}
    assert all("bulk" not in launch[dirn] for launch in job_paths(cp2) for dirn in ("fwd", "inv"))
    # config 3 (8192x8192x3, one tile, 9/7): level 1 cuts 35 strips of 240 columns into 128 segments of 32 pairs, and
    # the 33 interior strips take bulk copies both ways
    cp3 = G.make_coding(8192, 8192, 3, 12, numres=6, irreversible=True)
    l1 = job_paths(cp3)[0]
    assert (l1["level"], l1["nc"], l1["pairs"]) == (1, 3, 32)
    assert l1["fwd"] == l1["inv"] == {"async": 2 * 128, "bulk": 33 * 128}
    # 720x64x3 5/3 with two resolutions reaches the inverse bulk path for NC = 3; at origin (1, 0) it does not
    assert ("inv", "53", 3, "bulk") in cells(G.make_coding(720, 64, 3, 12, numres=2), "53")
    assert ("inv", "53", 3, "bulk") not in cells(G.make_coding(720, 64, 3, 12, numres=2, origin=(1, 0)), "53")


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=2)
def _source(name, filt):
    a = CASES[name]
    cp = coding(name, filt)
    planes = P.synthetic_image(a["width"], a["height"], a["numcomps"], a["prec"], seed=len(name),
                               origin=a.get("origin", (0, 0)))
    if name in ("one-column-tiles", "one-row-tiles"):
        # the 9/7 inverse returns a lone sample at an odd coordinate doubled (the reference does not halve it,
        # WaveletReverse97.cpp L839): content within 1/16 of the range around mid-scale keeps it inside the sample range
        planes = [(p >> 3) + (7 << (a["prec"] - 4)) for p in planes]
    return cp, planes, P.forward(cp, planes)


def _first_difference(got, want):
    for c, (g, w) in enumerate(zip(got, want)):
        bad = np.argwhere(g != w)
        if len(bad):
            y, x = bad[0]
            return "component %d: %d values differ, first at row %d column %d (%d, want %d)" % (
                c, len(bad), y, x, g[y, x], w[y, x])
    return ""


@pytest.mark.gpu
@pytest.mark.parametrize("filt", FILTERS)
@pytest.mark.parametrize("name", ORDER)
def test_forward_matches_oracle(engine, name, filt):
    cp, planes, ref = _source(name, filt)
    job = engine.job(cp)
    try:
        job.upload(planes)
        job.forward()
        got = [np.zeros_like(p) for p in planes]
        job.download_coeffs(got)
    finally:
        job.close()
    msg = _first_difference(got, ref)
    assert not msg, msg


def _perturbed(cp, coefs, seed):
    """the coefficients with a seeded offset on every one: integers in [-3, 3] for 5/3, floats in (-0.5, 0.5) for 9/7"""
    rng = np.random.default_rng(seed)
    out = []
    for c in coefs:
        if cp.irreversible:
            f = c.view(np.float32) + rng.uniform(-0.5, 0.5, c.shape).astype(np.float32)
            out.append(np.ascontiguousarray(f).view(np.int32))
        else:
            out.append(c + rng.integers(-3, 4, c.shape).astype(np.int32))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("filt", FILTERS)
@pytest.mark.parametrize("name", ORDER)
def test_inverse_matches_oracle_exactly(engine, name, filt):
    cp, planes, ref = _source(name, filt)
    coefs = _perturbed(cp, ref, seed=7)
    want = P.inverse(cp, coefs)
    lo, hi = (-(1 << (cp.prec - 1)), (1 << (cp.prec - 1)) - 1) if cp.sgnd else (0, (1 << cp.prec) - 1)
    inside = sum(int(((w > lo) & (w < hi)).sum()) for w in want)
    assert inside >= 0.95 * sum(w.size for w in want), "the clamp would decide too many samples"
    job = engine.job(cp)
    try:
        job.upload(planes)                  # sizes the planes; the coefficients below replace what a forward would give
        job.upload_coeffs(coefs)
        job.inverse()
        got = [np.full_like(p, -1) for p in planes]
        job.download(got)
    finally:
        job.close()
    msg = _first_difference(got, want)
    assert not msg, msg
