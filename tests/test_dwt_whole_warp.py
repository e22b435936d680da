"""The reversible (5/3) lifting kernels on whole-warp strips, both directions, bit for bit against the oracle.

k_dwt53_fwd / k_dwt53_inv (NC = 1 and NC = 3 components) cut every level's span into strips of 256 columns, one per warp
job: each of the 32 lanes owns 8 columns, and the neighbours outside the warp arrive as ghost columns, loaded from
mirrored addresses like the body (forward: the vertically lifted columns x0-2, x0-1 and x0+256 of the strip that starts
at x0; inverse: the high-band samples at x0-1 and x0+257 and the low-band sample at x0+256 of each band row).  Only the
last strip of a span may be narrower.  A strip whose body lies inside the line (and, inverse, whose band quads are
16-byte aligned) is staged by bulk (TMA) copies, any other by per-lane cp.async with mirrored edge columns; lines one
sample wide or high take the unpipelined degenerate job.  `job_paths` restates the planner and those rules; the CPU
tests check them on config 2 and that the cases below reach every cell of them, and the GPU tests compare the device
with the oracle on every case:
  - forward: the coefficients bit for bit;
  - inverse: the oracle's forward coefficients with a seeded perturbation in every band, reconstructed exactly.
"""
import functools

import numpy as np
import pytest

import grok_b200 as G
import oracle_pipeline as P

STRIP = 256                 # columns of a whole-warp strip: 32 lanes x 8
RESIDENT_JOBS = 3552        # build_dwt_plan: segments are halved until a launch has this many warp jobs (or 8 pairs)


def _cdiv(a, b):
    return -(-a // b)


def _res_rect(tc, numres, resno):
    n = numres - 1 - resno
    return tuple(_cdiv(v, 1 << n) for v in tc)


def strips(rect, pairs):
    """fill_strips for 5/3: (number of strips, number of row segments) of a descriptor"""
    u0, v0, u1, v1 = rect
    span = u1 - (u0 & ~7)
    npairs = ((v1 - 1) >> 1) - (v0 >> 1) + 1
    return max(1, _cdiv(span, STRIP)), _cdiv(npairs, pairs)


def dwt_plan(cp):
    """build_dwt_plan for a reversible coding: per level (finest first) the level-1 MCT-group launch (NC = 3) and the
    single-component launch (NC = 1), each with its segment length in pairs and its descriptors."""
    assert not cp.irreversible
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
            while pairs > 8 and sum(strips(d["rect"], pairs)[0] * strips(d["rect"], pairs)[1] for d in descs) < RESIDENT_JOBS:
                pairs >>= 1
            out.append(dict(level=lvl, nc=nc, pairs=pairs, descs=descs))
    return out


def strip_jobs(d, pairs):
    """Per strip of descriptor d: its first column x0, its owner lanes, and the forward and inverse staging path.
    decode_job<true>: lane L starts at column x0 + 8L and owns when that is left of u1; it is needed when it owns or is
    the right neighbour of the line's last owner.  Forward (RowStage::lane_fast): bulk when every lane's 8 columns lie
    inside the line (their 16-byte alignment holds: planes start at canvas columns that are multiples of 32).  Inverse
    (BandStage::setup, all_fast): bulk when every lane's LL, HL, LH and HH quads lie inside the line and are 16-byte
    aligned in their planes (the coefficient plane, whose column 0 is canvas column X0 of the tile's image, and for LL
    above the coarsest level the LL scratch plane, whose column 0 is band column 0)."""
    u0, v0, u1, v1 = d["rect"]
    wn, hn = u1 - u0, v1 - v0
    ns, _ = strips(d["rect"], pairs)
    x0l, x0h = (u0 + 1) >> 1, u0 >> 1
    snx = ((u1 + 1) >> 1) - x0l
    cbase = d["cbase"]
    llbase = cbase if d["coarsest"] else x0l
    out = []
    for s in range(ns):
        x0 = (u0 & ~7) + s * STRIP
        owners = sum(1 for lane in range(32) if x0 + 8 * lane < u1)
        if wn == 1 or hn == 1:
            out.append(dict(x0=x0, owners=owners, fwd="degenerate", inv="degenerate"))
            continue
        fwd = inv = True
        for lane in range(32):
            ulane = x0 + 8 * lane
            need = ulane < u1 + 8
            rel = ulane - u0
            fwd = fwd and need and rel >= 0 and rel + 8 <= wn
            k0 = ulane >> 1
            inv = inv and need and 2 * k0 >= u0 and 2 * k0 + 7 < u1 \
                and (llbase + k0 - x0l) % 4 == 0 and (cbase + snx + k0 - x0h) % 4 == 0 and (cbase + k0 - x0l) % 4 == 0
        out.append(dict(x0=x0, owners=owners, fwd="bulk" if fwd else "async", inv="bulk" if inv else "async"))
    return out


def job_paths(cp):
    """For each level launch of a coding: its level, NC, segment length in pairs, and how many of its warp jobs take
    each path, forward ("fwd") and inverse ("inv")."""
    out = []
    for launch in dwt_plan(cp):
        counts = {"fwd": {}, "inv": {}}
        for d in launch["descs"]:
            nseg = strips(d["rect"], launch["pairs"])[1]
            for job in strip_jobs(d, launch["pairs"]):
                for dirn in ("fwd", "inv"):
                    counts[dirn][job[dirn]] = counts[dirn].get(job[dirn], 0) + nseg
        out.append(dict(level=launch["level"], nc=launch["nc"], pairs=launch["pairs"], **counts))
    return out


# ghost columns used by lane 0 (left) and lane 31 (right) of a strip starting at x0, per direction
_GHOSTS = {"fwd": ((-2, -1), (STRIP,)), "inv": ((-1,), (STRIP, STRIP + 1))}
# rows a warp job reads below and above its pairs [jbeg, jend): forward rows 2(jbeg-1) .. 2 jend, inverse the band rows
# of pairs jbeg-1 .. jend
_ROW_HALO = {"fwd": (2, 0), "inv": (2, 1)}


def _reflects_twice(lo, hi, n):
    """an index range [lo, hi] used on a line of n samples needs more than one reflection (mirror_rel_slow)"""
    return lo < -(n - 1) or hi > 2 * (n - 1)


def cells(cp):
    """The cells a reversible coding reaches: (direction, NC, path), ("seg", NC, pairs) and (direction, condition)
    for the conditions of non-degenerate descriptors: where the left and right ghosts come from ("mirrored" at the
    line's end or "inside" the line; the right ghosts only of strips whose lane 31 owns), a last strip narrower than
    8 lanes, a line shorter than the ghost support, odd u0 / v0."""
    out = set()
    for launch in job_paths(cp):
        out.add(("seg", launch["nc"], launch["pairs"]))
        for dirn in ("fwd", "inv"):
            out |= {(dirn, launch["nc"], path) for path in launch[dirn]}
    for launch in dwt_plan(cp):
        for d in launch["descs"]:
            u0, v0, u1, v1 = d["rect"]
            wn, hn = u1 - u0, v1 - v0
            jobs = strip_jobs(d, launch["pairs"])
            if jobs[0]["fwd"] == "degenerate":
                continue
            jlo, jhi = v0 >> 1, (v1 - 1) >> 1
            for dirn in ("fwd", "inv"):
                left, right = _GHOSTS[dirn]
                below, above = _ROW_HALO[dirn]
                cols = []
                for job in jobs:
                    x0 = job["x0"]
                    out.add((dirn, "left_ghost", "mirrored" if x0 + min(left) < u0 else "inside"))
                    if job["owners"] == 32:
                        out.add((dirn, "right_ghost", "mirrored" if x0 + max(right) >= u1 else "inside"))
                    cols += [x0 + min(left), x0 + max(right), x0 + 8 * job["owners"] + 7]
                if jobs[-1]["owners"] < 8 and len(jobs) > 1:
                    out.add((dirn, "ragged_narrow"))
                if _reflects_twice(2 * jlo - below - v0, 2 * (jhi + 1) + above - v0, hn) or \
                        _reflects_twice(min(cols) - u0, max(cols) - u0, wn):
                    out.add((dirn, "short_line"))
                if u0 & 1:
                    out.add((dirn, "odd_u0"))
                if v0 & 1:
                    out.add((dirn, "odd_v0"))
    return out


ALL_CELLS = ({(dirn, nc, p) for dirn in ("fwd", "inv") for nc in (1, 3) for p in ("bulk", "async", "degenerate")}
             | {("seg", nc, p) for nc in (1, 3) for p in (8, 16, 32)}
             | {(dirn, side, src) for dirn in ("fwd", "inv") for side in ("left_ghost", "right_ghost")
                for src in ("mirrored", "inside")}
             | {(dirn, b) for dirn in ("fwd", "inv") for b in ("ragged_narrow", "short_line", "odd_u0", "odd_v0")})

# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
CASES = {
    # three whole strips at level 1 (bulk both ways, ghosts mirrored at both tile edges and read from the neighbour
    # strips), two at level 2, NC = 3 (components 0-2) and NC = 1 (component 3)
    "whole": dict(width=768, height=72, numcomps=4, prec=12, numres=3),
    # several tiles in a row: strips end at the tile edges, the last strip of each 600-wide tile is ragged
    "tiled": dict(width=1200, height=50, numcomps=3, prec=16, numres=4, tile=(600, 50)),
    # odd origin on every level: the first strip starts left of the line (cp.async, mirrored lane 0), ragged last strips
    "odd-origin": dict(width=541, height=183, numcomps=4, prec=16, numres=6, origin=(3, 5)),
    # tiles one column wide and one row high (degenerate jobs, NC = 3 and 1); the rows span three strips, whose ghost
    # columns the degenerate job lifts as well
    "one-column-tiles": dict(width=23, height=37, numcomps=4, prec=12, numres=3, tile=(1, 37)),
    "one-row-tiles": dict(width=600, height=3, numcomps=4, prec=12, numres=2, tile=(600, 1), origin=(0, 4)),
    # 800 tiles of 16x130: 16-pair segments at level 1, strips of 2 lanes
    "seg16": dict(width=640, height=2600, numcomps=4, prec=16, numres=2, tile=(16, 130)),
    # 1200 such tiles: 32-pair segments; level 3 lines are 4 columns wide, shorter than the ghost support
    "seg32": dict(width=640, height=3900, numcomps=4, prec=16, numres=4, tile=(16, 130)),
}
ORDER = list(CASES)     # cheapest first


def coding(name):
    return G.make_coding(**CASES[name])


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the model and the case list
# ---------------------------------------------------------------------------------------------------------------------
def test_cases_reach_every_cell():
    reached = set()
    for name in CASES:
        reached |= cells(coding(name))
    assert reached <= ALL_CELLS, sorted(reached - ALL_CELLS, key=str)
    assert reached == ALL_CELLS, "not reached: %s" % sorted(ALL_CELLS - reached, key=str)


def test_config2_takes_bulk_copies():
    # config 2 (8192x8192x3, 1024x1024 tiles): every strip of levels 1-3 is a whole 256-column strip inside its tile,
    # staged by bulk copies both ways; levels 4 and 5 (128 and 64 columns) are ragged strips on cp.async
    cp2 = G.make_coding(8192, 8192, 3, 12, numres=6, tile=(1024, 1024))
    plan = dwt_plan(cp2)
    assert [(lp["level"], lp["nc"], lp["pairs"]) for lp in plan] == [(1, 3, 32), (2, 1, 16), (3, 1, 8), (4, 1, 8), (5, 1, 8)]
    assert {strips(d["rect"], plan[0]["pairs"]) for d in plan[0]["descs"]} == {(4, 16)}
    for launch in job_paths(cp2):
        for dirn in ("fwd", "inv"):
            if launch["level"] <= 3:
                assert set(launch[dirn]) == {"bulk"}, (launch["level"], dirn, launch[dirn])
            else:
                assert set(launch[dirn]) == {"async"}, (launch["level"], dirn, launch[dirn])


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=2)
def _source(name):
    a = CASES[name]
    cp = coding(name)
    planes = P.synthetic_image(a["width"], a["height"], a["numcomps"], a["prec"], seed=3 * len(name) + 1,
                               origin=a.get("origin", (0, 0)))
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
@pytest.mark.parametrize("name", ORDER)
def test_forward_matches_oracle(engine, name):
    cp, planes, ref = _source(name)
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


@pytest.mark.gpu
@pytest.mark.parametrize("name", ORDER)
def test_inverse_matches_oracle_exactly(engine, name):
    cp, planes, ref = _source(name)
    rng = np.random.default_rng(11)
    coefs = [c + rng.integers(-3, 4, c.shape).astype(np.int32) for c in ref]
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
