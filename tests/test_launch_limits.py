"""Launch grids that grow with the data, at and past the limits of a CUDA grid.

A grid holds at most 65,535 CTAs in y and in z.  Every launch whose y or z dimension counts something the caller
decides -- DWT descriptors, rows, images, copy entries, tile parts, streams -- either caps that dimension and loops
(a stride over gridDim, or one launch per piece of 65,535), or it fails with an invalid configuration once the count
passes the limit.  This file restates each such launcher's grid in Python:
  - dwt_enqueues / dwt_pieces:    b2k_launch_dwt_fwd / _inv (dwt.cu) over the level launches of build_dwt_plan
                                  (engine.cu), for the whole job (Job API) or per B2K_CHUNKS chunk;
  - point_transform_grid:         b2k_launch_point_transform (numres = 1);
  - convert_grid / batch_grid / batch_pieces / conversion_paths:
                                  the container <-> plane conversions of one image and of a batch;
  - batch_chunk_images:           which images a batch call converts in each chunk of its (slot, tile) range;
  - copy_table_grid / copy_entry_paths:
                                  gather_streams / b2k_copy_table (engine.cu, t2_decode.cu);
  - t2_gather_grid:               b2k_t2_window_gather;
  - t2_scan_plan:                 k_t2_scan (t2_device.cu): the batch writer's part scans and stream placement;
  - header_reads:                 read_batch_headers (engine.cu): a prefix, then twice the prefix until the main
                                  header fits.
The CPU tests pin each function to hand-computed plans and check that the GPU cases reach every cell.  The GPU tests
run each case against an exact reference: the oracle's transforms bit for bit, the oracle's block coder, the host entry
points (which the other suites pin to the oracle), and the input itself for every lossless round trip."""
import functools

import numpy as np
import pytest

import grok_b200 as G
import oracle_pipeline as P
from test_dwt_paths import dwt_plan, _perturbed, _first_difference

GRID_LIMIT = 65535          # the most CTAs of a grid's y or z dimension
DEFAULT_CHUNKS = 8          # build_job's chunk count without B2K_CHUNKS
HEADER_PREFIX = 4096        # t2::BATCH_HEADER_PREFIX: the first read of a batch's main headers
SINGLE_PREFIX = 64 << 10    # read_main_header: the first read of one stream's main header
SCAN_THREADS = 1024         # t2_device.cu: the threads of k_t2_scan's CTA, the values one round of cta_scan takes


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------------------------
# the launch model
# ---------------------------------------------------------------------------------------------------------------------
def dwt_pieces(ndesc):
    """b2k_launch_dwt_fwd / _inv: the descriptor counts of the launches one enqueue of ndesc descriptors makes (the
    descriptor is blockIdx.y, so one launch per 65,535 of them)"""
    return [min(GRID_LIMIT, ndesc - d0) for d0 in range(0, ndesc, GRID_LIMIT)]


def chunk_tiles(ntiles, chunks):
    """build_job: the tile boundaries of the chunks a chunked host or device call enqueues one by one"""
    n = max(1, min(chunks, ntiles))
    return [k * ntiles // n for k in range(n + 1)]


def dwt_enqueues(cp, chunks=None):
    """Per level launch of build_dwt_plan (finest first): (level, NC, [descriptors of each enqueue]).  chunks=None: the
    Job API's forward / inverse, which enqueue every tile at once; else one enqueue per chunk.  Every tile of the codings
    here has the same number of descriptors in a launch."""
    ntiles = len(P.tile_rects(cp))
    out = []
    for launch in dwt_plan(cp):
        n = len(launch["descs"])
        assert n % ntiles == 0, "a tile without descriptors in this launch"
        per_tile = n // ntiles
        bounds = [0, ntiles] if chunks is None else chunk_tiles(ntiles, chunks)
        out.append((launch["level"], launch["nc"], [(b - a) * per_tile for a, b in zip(bounds, bounds[1:])]))
    return out


def point_descs(cp):
    """build_dwt_plan for numres = 1: one point-transform descriptor per tile and component group (RCT / ICT on the
    first three components together)"""
    groups = 1 + (cp.numcomps - 3) if cp.mct else cp.numcomps
    return len(P.tile_rects(cp)) * groups


def point_transform_grid(ndesc, max_w, max_h):
    """b2k_launch_point_transform: (x, y, z); rows past grid.y and descriptors past grid.z are strided"""
    return (_cdiv(max_w, 128), min(max_h, GRID_LIMIT), min(ndesc, GRID_LIMIT))


def convert_grid(w, h):
    """b2k_launch_container_to_planes / _planes_to_container: 8 pixels per thread, 128 threads, rows strided by grid.y"""
    return (_cdiv(w, 8 * 128), min(h, GRID_LIMIT))


def batch_grid(n, w, h):
    """the batch conversions' (x, y): grid.y shrinks with the batch, to 8 rows at the least (or h)"""
    gx, gy = convert_grid(w, h)
    gy = min(gy, max(1, 16384 // max(1, n)))
    gy = min(max(gy, 8), max(1, h))
    return gx, gy


def batch_pieces(n):
    """launch_planes_to_containers / launch_containers_to_planes: images per launch (image = blockIdx.z)"""
    return [min(GRID_LIMIT, n - i0) for i0 in range(0, n, GRID_LIMIT)]


def conversion_paths(S, NC, w, h, step, pitch, base):
    """The container-side paths a conversion of a w x h rectangle takes: a thread moves its 8 pixels as one group of
    8 * NC * S bytes ("group128" when that is a multiple of 16, else "group64") when they are whole, step == NC and the
    address is aligned to the access; otherwise sample by sample, because of the row's tail, a step wider than NC or an
    unaligned address.  pitch and step in samples, base: the byte address of pixel (0, 0) modulo 16."""
    V = 16 if (8 * NC * S) % 16 == 0 else 8
    out = set()
    for y in range(min(h, 64)):             # row alignment repeats with a period of at most 16 rows
        for x8 in range(0, w, 8):
            addr = base + (y * pitch + x8 * step) * S
            if x8 + 8 > w:
                out.add("tail")
            elif step != NC:
                out.add("step>NC")
            elif addr % V:
                out.add("unaligned")
            else:
                out.add("group%d" % (8 * V))
    return out


def batch_chunk_images(n, tiles, chunks=DEFAULT_CHUNKS):
    """The batch calls' chunks over the n * tiles (slot, tile) pairs: per chunk, the images the encoder converts there
    (those whose first tile is in it: ceil) and the images the decoder writes there (those whose last tile is in it:
    floor), each as a range [s0, s1)"""
    used = n * tiles
    nch = min(chunks, used)
    out = []
    for k in range(nch):
        t0, t1 = k * used // nch, (k + 1) * used // nch
        if t1 > t0:
            out.append(((_cdiv(t0, tiles), _cdiv(t1, tiles)), (t0 // tiles, t1 // tiles)))
    return out


def copy_table_grid(n, longest):
    """gather_streams: None for one entry (a plain device-to-device copy), else k_copy_table's (x, y) -- entries
    strided by grid.y, the longest entry's bytes by a strip of grid.x CTAs"""
    if n == 1:
        return None
    return (min(256, longest // (256 * 16 * 4) + 1), min(n, GRID_LIMIT))


def copy_entry_paths(src, dst, length):
    """k_copy_table on one entry: 16 bytes per step when source and destination are both 16-byte aligned, then the
    length's tail byte by byte; otherwise every byte one by one"""
    if (src | dst) % 16:
        return {"bytes"}
    return {"16-byte", "tail"} if length % 16 else {"16-byte"}


def t2_gather_grid(nparts, nbytes):
    """b2k_t2_window_gather: k_t2_gather's (x, y) -- parts strided by grid.y, x sized by the mean part"""
    return (min(256, (nbytes // nparts) // (256 * 16) + 1), min(nparts, GRID_LIMIT))


def t2_scan_plan(n, nparts):
    """k_t2_scan for a batch of n streams of nparts tile parts: (CTAs, streams of the busiest CTA, rounds of each
    stream's part scan, rounds of the placement scan the last CTA runs over the n streams)"""
    ctas = min(n, GRID_LIMIT)
    return ctas, _cdiv(n, ctas), _cdiv(nparts, SCAN_THREADS), _cdiv(n, SCAN_THREADS)


def header_reads(length, header, prefix=HEADER_PREFIX):
    """read_batch_headers for one stream of `length` bytes whose main header needs its first `header` bytes: the
    sizes of the reads, and whether the header is cut (the stream ends inside it)"""
    reads = [min(length, prefix)]
    while reads[-1] < header:
        if reads[-1] >= length:
            return reads, True
        reads.append(min(length, 2 * reads[-1]))
    return reads, False


def placement(lengths):
    """the batch encoder's layout: stream i at the sum of the 256-byte-rounded lengths before it"""
    out, at = [], 0
    for n in lengths:
        out.append(at)
        at += (n + 255) & ~255
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the cases
# ---------------------------------------------------------------------------------------------------------------------
# DWT descriptors: exactly the limit, one past it at level 1, past it at level 2 only
DWT_CASES = {
    "65535": dict(width=85 * 8, height=257 * 8, numcomps=3, prec=8, numres=2, tile=(8, 8), mct=False),
    "65536": dict(width=128 * 8, height=128 * 8, numcomps=4, prec=8, numres=2, tile=(8, 8), mct=False),
    "level2": dict(width=66 * 8, height=331 * 8, numcomps=3, prec=8, numres=3, tile=(8, 8)),
}
# the same codings with no wavelet level: the point transform, one descriptor per tile and group
POINT_CASES = {name: dict(a, numres=1) for name, a in DWT_CASES.items()}
FILTERS = ("53", "97")

# an image taller than a grid: the conversions' and the point transform's rows loop
TALL = dict(width=8, height=65600, prec=8)
TALL_NC = (1, 3)
TALL_NUMRES = (1, 3)
DTYPES = ("uint8", "uint16", "int32")    # the 8-bit, 16-bit and 32-bit containers the device entry points take

# every sample width x component count in a small image: contiguous HWC, the first NC channels of a 4-channel buffer
# (5 channels for NC = 4), and the same one sample off a 16-byte boundary
CONV_W, CONV_H = 21, 13
CONV_VARIANTS = ("contiguous", "wider_pixel", "one_sample_off")

# more streams than a grid: every batch launch that counts streams or copy entries strides or loops
MANY = 65537
MANY_NUMRES = (1, 2)
CHUNK_SETTINGS = (None, 1)
PLACEMENT_BATCHES = (1024, 1025, 2049)

# tile parts: 200 x 150 tiles of 16 x 16, three resolutions, one tile part per resolution
PARTS = dict(width=200 * 16, height=150 * 16, numcomps=1, prec=8, numres=3, tile=(16, 16))
PARTS_FLAGS = G.CS_TLM | G.CS_PLT | G.CS_TPARTS_R
PARTS_TILES = (PARTS["width"] // 16) * (PARTS["height"] // 16)
# a main header between one and two batch prefixes: 32 x 32 tiles of 16 x 16 with TLM
ONE_REREAD = dict(width=32 * 16, height=32 * 16, numcomps=1, prec=8, numres=3, tile=(16, 16))

# large copies: 256 x 256 16-bit noise, one tile part of about 140 KB, in views at these offsets from a 16-byte boundary
LARGE = dict(width=256, height=256, numcomps=1, prec=16, numres=3)
LARGE_SKEWS = (0, 1, 3)


def main_header_length(args, flags, ntiles):
    """the main header b2k_codestream_write_header writes for a coding (one tile part per tile: without CS_TPARTS_R)"""
    assert not flags & G.CS_TPARTS_R
    return len(G.codestream_write_header(G.make_coding(**args), flags, np.full(ntiles, 1000)))


def _wider(NC):
    """the channels of the buffer whose first NC channels the "wider_pixel" views take"""
    return max(4, NC + 1)


def _coding(args, filt="53"):
    return G.make_coding(irreversible=filt == "97", **args)


def case_cells():
    """the cells the GPU cases below reach, by the model"""
    cells = set()
    # DWT level launches: one enqueue of the Job API, and one per chunk with B2K_CHUNKS=1 and by default
    for args in DWT_CASES.values():
        cp = _coding(args)
        for api, chunks in (("job", None), ("chunked", 1), ("chunked", DEFAULT_CHUNKS)):
            for _, nc, enq in dwt_enqueues(cp, chunks):
                for n in enq:
                    cells.add(("dwt", api, nc, "<" if n < GRID_LIMIT else "=" if n == GRID_LIMIT else ">"))
    # the point transform
    for args in POINT_CASES.values():
        cp = _coding(args)
        if point_transform_grid(point_descs(cp), 8, 8)[2] < point_descs(cp):
            cells.add(("point", "z loop"))
    for numres in TALL_NUMRES:
        if numres == 1 and point_transform_grid(1, TALL["width"], TALL["height"])[1] < TALL["height"]:
            cells.add(("point", "y loop"))
    # conversions of one image
    if convert_grid(TALL["width"], TALL["height"])[1] < TALL["height"]:
        cells.add(("convert", "rows loop"))
    for S in (1, 2, 4):
        for NC in (1, 2, 3, 4):
            for v in CONV_VARIANTS:
                step = _wider(NC) if v == "wider_pixel" else NC
                base = S if v == "one_sample_off" else 0
                for path in conversion_paths(S, NC, CONV_W, CONV_H, step, CONV_W * step, base):
                    cells.add(("convert", S, NC, path))
    # batch conversions: the tall pair, and the many small images
    if batch_grid(2, TALL["width"], TALL["height"])[1] < TALL["height"]:
        cells.add(("batch", "rows loop"))
    if batch_grid(2, TALL["width"], TALL["height"])[1] < convert_grid(TALL["width"], TALL["height"])[1]:
        cells.add(("batch", "y clamp"))
    if len(batch_pieces(MANY)) > 1:
        cells.add(("batch", "images in pieces"))
    # chunks without an image: a batch of two PARTS images in eight chunks, encoded and decoded
    for (e0, e1), (d0, d1) in batch_chunk_images(2, PARTS_TILES):
        if e1 == e0:
            cells.add(("batch", "encode chunk without image"))
        if d1 == d0:
            cells.add(("batch", "decode chunk without image"))
    # copy tables: the many streams' headers and bodies, and the large copies
    for n, longest in ((MANY, 100), (3, 140000), (1, 140000)):
        g = copy_table_grid(n, longest)
        if g is None:
            cells.add(("copy", "plain"))
        else:
            if g[1] < n:
                cells.add(("copy", "y stride"))
            if g[0] > 1:
                cells.add(("copy", "gx > 1"))
    # the large copies: views at 16-byte boundaries into the arena's 256-byte ones, and off them (the GPU test asserts
    # that a length is not a multiple of 16)
    for skew in LARGE_SKEWS:
        cells |= {("copy", p) for p in copy_entry_paths(skew, 0, 16 * 8000 + 5)}
    # the tile parts' gather: 90,000 parts of about 40 bytes, and the large copies' one part of about 140 KB
    nparts = PARTS_TILES * PARTS["numres"]
    for n, nbytes in ((nparts, nparts * 40), (1, 140000)):
        gx, gy = t2_gather_grid(n, nbytes)
        if gy < n:
            cells.add(("gather", "y stride"))
        if gx > 1:
            cells.add(("gather", "gx > 1"))
    # the batch writer's scans: two PARTS streams, the placement batches and the many small streams
    for n, parts in [(2, nparts)] + [(k, 1) for k in PLACEMENT_BATCHES] + [(MANY, 1)]:
        ctas, per_cta, part_rounds, place_rounds = t2_scan_plan(n, parts)
        cells.add(("scan", "parts", "1 round" if part_rounds == 1 else "rounds"))
        cells.add(("scan", "placement", min(place_rounds, 3)))
        if per_cta > 1:
            cells.add(("scan", "streams loop"))
    # main headers in the batches: PARTS without TLM, with one tile part per tile (about 180 KB), the ONE_REREAD stream;
    # one part per resolution (about 540 KB, asserted on the GPU) and a copy of it cut inside its main header
    for args, flags, ntiles in ((PARTS, G.CS_PLT, PARTS_TILES), (PARTS, G.CS_TLM | G.CS_PLT, PARTS_TILES),
                                (ONE_REREAD, G.CS_TLM | G.CS_PLT, 1024)):
        reads, cut = header_reads(10 ** 7, main_header_length(args, flags, ntiles))
        cells.add(("headers", min(len(reads) - 1, 3)))
    if header_reads(5000, 540000)[1]:
        cells.add(("headers", "cut"))
    # one stream's header from a 64 KiB prefix: the PARTS stream alone
    if len(header_reads(10 ** 7, main_header_length(PARTS, G.CS_TLM | G.CS_PLT, PARTS_TILES), SINGLE_PREFIX)[0]) > 1:
        cells.add(("headers", "single-stream re-read"))
    return cells


ALL_CELLS = ({("dwt", "job", 1, rel) for rel in "=>"} | {("dwt", "chunked", 1, rel) for rel in "<=>"}
             | {("dwt", api, 3, "<") for api in ("job", "chunked")}
             | {("point", "z loop"), ("point", "y loop"), ("convert", "rows loop")}
             | {("convert", S, NC, p) for S in (1, 2, 4) for NC in (1, 2, 3, 4) for p in ("tail", "step>NC", "unaligned")}
             | {("convert", S, NC, "group%d" % (64 if S == 1 and NC % 2 else 128)) for S in (1, 2, 4) for NC in (1, 2, 3, 4)}
             | {("batch", "rows loop"), ("batch", "y clamp"), ("batch", "images in pieces"),
                ("batch", "encode chunk without image"), ("batch", "decode chunk without image")}
             | {("copy", "plain"), ("copy", "y stride"), ("copy", "gx > 1"), ("copy", "16-byte"), ("copy", "tail"), ("copy", "bytes")}
             | {("gather", "y stride"), ("gather", "gx > 1")}
             | {("scan", "parts", "1 round"), ("scan", "parts", "rounds"), ("scan", "streams loop")}
             | {("scan", "placement", k) for k in (1, 2, 3)}
             | {("headers", k) for k in (0, 1, 3, "cut", "single-stream re-read")})


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the model against hand-computed plans, and the cases against the cells
# ---------------------------------------------------------------------------------------------------------------------
def test_model_reproduces_known_plans():
    # 1024 x 1024, 4 components without MCT, 8 x 8 tiles: 16,384 tiles x 4 components at level 1
    cp = _coding(DWT_CASES["65536"])
    assert dwt_enqueues(cp) == [(1, 1, [65536])]
    assert dwt_enqueues(cp, 1) == [(1, 1, [65536])]
    assert dwt_enqueues(cp, DEFAULT_CHUNKS) == [(1, 1, [8192] * 8)]
    assert dwt_pieces(65536) == [65535, 1] and dwt_pieces(65535) == [65535] and dwt_pieces(3) == [3]
    # 21,845 tiles x 3 components: exactly the limit
    assert dwt_enqueues(_coding(DWT_CASES["65535"])) == [(1, 1, [65535])]
    # with MCT, 21,846 tiles: one NC = 3 descriptor per tile at level 1, three NC = 1 at level 2
    assert dwt_enqueues(_coding(DWT_CASES["level2"])) == [(1, 3, [21846]), (2, 1, [65538])]
    assert chunk_tiles(21846, 8) == [0, 2730, 5461, 8192, 10923, 13653, 16384, 19115, 21846]
    assert chunk_tiles(3, 8) == [0, 1, 2, 3]
    # config 2 (8192 x 8192 x 3, 1024 x 1024 tiles): 64 descriptors per level, 8 per chunk
    cp2 = G.make_coding(8192, 8192, 3, 12, numres=6, tile=(1024, 1024))
    assert dwt_enqueues(cp2, DEFAULT_CHUNKS) == [(1, 3, [8] * 8)] + [(lvl, 1, [24] * 8) for lvl in range(2, 6)]
    # the point transform
    assert point_descs(_coding(POINT_CASES["65536"])) == 65536
    assert point_descs(_coding(POINT_CASES["level2"])) == 21846
    assert point_transform_grid(65536, 8, 8) == (1, 8, 65535)
    assert point_transform_grid(1, 8, 65600) == (1, 65535, 1)
    assert point_transform_grid(64, 1024, 1024) == (8, 1024, 64)
    # conversions
    assert convert_grid(8, 65600) == (1, 65535) and convert_grid(8192, 8192) == (8, 8192) and convert_grid(1025, 3) == (2, 3)
    assert batch_grid(2, 8, 65600) == (1, 8192)
    assert batch_grid(65537, 8, 8) == (1, 8) and batch_grid(1000, 8, 3) == (1, 3) and batch_grid(1, 64, 64) == (1, 64)
    assert batch_pieces(65537) == [65535, 2] and batch_pieces(65535) == [65535] and batch_pieces(5) == [5]
    assert conversion_paths(1, 3, 21, 1, 3, 63, 0) == {"group64", "tail"}
    assert conversion_paths(2, 4, 16, 1, 5, 80, 0) == {"step>NC"}
    assert conversion_paths(4, 4, 16, 2, 4, 64, 4) == {"unaligned"}
    assert conversion_paths(2, 2, 16, 2, 2, 32, 0) == {"group128"}
    # copies: 16 KiB of the longest entry per CTA along x, at most 256
    assert copy_table_grid(1, 10 ** 6) is None
    assert copy_table_grid(65537, 100) == (1, 65535)
    assert copy_table_grid(3, 16383) == (1, 3) and copy_table_grid(3, 16384) == (2, 3) and copy_table_grid(2, 1 << 30) == (256, 2)
    assert t2_gather_grid(90000, 90000 * 40) == (1, 65535) and t2_gather_grid(4, 4 * 4096) == (2, 4)
    # main headers: 4 KiB, then doubling; a stream that ends inside its header is cut
    assert header_reads(10 ** 6, 3000) == ([4096], False)
    assert header_reads(10 ** 6, 6000) == ([4096, 8192], False)
    assert header_reads(10 ** 6, 20000) == ([4096, 8192, 16384, 32768], False)
    assert header_reads(5000, 540000) == ([4096, 5000], True)
    assert header_reads(10 ** 6, 540000, SINGLE_PREFIX) == ([65536, 131072, 262144, 524288, 1000000], False)
    assert placement([10, 256, 257, 1]) == [0, 256, 512, 1024]
    # batch chunks: two images of 30,000 tiles in 8 chunks of 7,500; the encoder converts image 1 in chunk 4 (tiles
    # 30,000 - 37,500), the decoder writes image 0 in chunk 3 (22,500 - 30,000)
    chunks = batch_chunk_images(2, 30000)
    assert [e for e, _ in chunks] == [(0, 1), (1, 1), (1, 1), (1, 1), (1, 2), (2, 2), (2, 2), (2, 2)]
    assert [d for _, d in chunks] == [(0, 0), (0, 0), (0, 0), (0, 1), (1, 1), (1, 1), (1, 1), (1, 2)]
    assert batch_chunk_images(3, 1) == [((0, 1), (0, 1)), ((1, 2), (1, 2)), ((2, 3), (2, 3))]
    assert copy_entry_paths(0, 256, 4096) == {"16-byte"} and copy_entry_paths(16, 0, 17) == {"16-byte", "tail"}
    assert copy_entry_paths(1, 0, 4096) == {"bytes"} and copy_entry_paths(0, 8, 4096) == {"bytes"}
    # the writer's scans: 1,024 values per round; a CTA per stream up to 65,535 of them
    assert t2_scan_plan(2, 90000) == (2, 1, 88, 1)
    assert t2_scan_plan(1024, 1) == (1024, 1, 1, 1) and t2_scan_plan(1025, 3) == (1025, 1, 1, 2)
    assert t2_scan_plan(2049, 1024) == (2049, 1, 1, 3) and t2_scan_plan(65537, 1) == (65535, 2, 1, 65)
    # main headers: 6 bytes of TLM per tile part
    assert main_header_length(ONE_REREAD, G.CS_TLM | G.CS_PLT, 1024) == 6231
    assert main_header_length(PARTS, G.CS_TLM | G.CS_PLT, PARTS_TILES) == 180099
    assert main_header_length(PARTS, G.CS_PLT, PARTS_TILES) == 81


def test_cases_reach_every_cell():
    reached = case_cells()
    assert reached <= ALL_CELLS, sorted(reached - ALL_CELLS, key=str)
    assert reached == ALL_CELLS, "not reached: %s" % sorted(ALL_CELLS - reached, key=str)


OTHER_SUITES = ("test_device_io", "test_device_batch_encode", "test_device_batch_decode", "test_device_codestream",
                "test_device_codestream_decode", "test_device_window_decode")
# the helpers those suites make batches with, and the position of their count argument
_BATCH_HELPERS = {"_small": 1, "_small_batch": 2, "_seeded": 1, "_seeded_streams": 2}


def _other_suites_cases():
    """(codings, batch sizes) the other device suites spell out: test_device_io's geometries (the batch suites reuse
    them), every make_coding call with literal arguments, and the literal counts given to the batch helpers"""
    import ast
    import os
    import test_device_io as D
    here = os.path.dirname(os.path.abspath(__file__))
    codings = [G.make_coding(**g) for g in D._geoms()]
    batches = []
    for name in OTHER_SUITES:
        with open(os.path.join(here, name + ".py")) as f:
            tree = ast.parse(f.read())
        for node in ast.walk(tree):
            if not isinstance(node, ast.Call):
                continue
            fn = node.func.attr if isinstance(node.func, ast.Attribute) else getattr(node.func, "id", "")
            try:
                if fn == "make_coding":
                    codings.append(G.make_coding(*[ast.literal_eval(a) for a in node.args],
                                                 **{k.arg: ast.literal_eval(k.value) for k in node.keywords}))
                elif fn in _BATCH_HELPERS:
                    at = _BATCH_HELPERS[fn]
                    count = [k.value for k in node.keywords if k.arg in ("n", "count")] or node.args[at:at + 1]
                    if count:
                        batches.append(ast.literal_eval(count[0]))
            except ValueError:          # arguments that are not literals
                pass
    return codings, batches


def test_report_what_the_other_suites_reach(capsys):
    """Which limit cells the device I/O, batch, code-stream and window suites reach, from the codings and batch sizes
    they spell out (printed, not asserted)"""
    codings, batches = _other_suites_cases()
    reached = set()
    descs = rows = tiles = 0
    for cp in codings:
        rows = max(rows, cp.y1 - cp.y0)
        tiles = max(tiles, len(P.tile_rects(cp)))
        for launch in dwt_plan(cp):             # a chunk holds at most the whole launch
            n = len(launch["descs"])
            descs = max(descs, n)
            reached.add(("dwt", "chunked", launch["nc"], "<" if n < GRID_LIMIT else "=" if n == GRID_LIMIT else ">"))
        if convert_grid(cp.x1 - cp.x0, cp.y1 - cp.y0)[1] < cp.y1 - cp.y0:
            reached.add(("convert", "rows loop"))
    most = max(batches or [1])
    if len(batch_pieces(most)) > 1:
        reached.add(("batch", "images in pieces"))
    if copy_table_grid(most, 1) and copy_table_grid(most, 1)[1] < most:
        reached.add(("copy", "y stride"))
    if t2_scan_plan(most, 1)[3] > 1:
        reached.add(("scan", "placement", min(t2_scan_plan(most, 1)[3], 3)))
    limits = {c for c in ALL_CELLS if c[0] != "convert" or c[1] == "rows loop"}   # the conversions' paths left out
    lines = ["%s: %d codings, at most %d rows, %d tiles, %d DWT descriptors in one level launch; largest literal batch %d"
             % (", ".join(OTHER_SUITES), len(codings), rows, tiles, descs, most),
             "cells reached: %s" % sorted(reached & limits, key=str),
             "cells not reached: %s" % sorted(limits - reached, key=str)]
    with capsys.disabled():
        print("\n" + "\n".join(lines))


# ---------------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture
def make_engine(monkeypatch):
    """a fresh Engine whose jobs are built with B2K_CHUNKS set to `chunks` (None: the default), closed at the end"""
    made = []

    def make(chunks=None):
        if chunks is None:
            monkeypatch.delenv("B2K_CHUNKS", raising=False)
        else:
            monkeypatch.setenv("B2K_CHUNKS", str(chunks))
        eng = G.Engine(0)
        made.append(eng)
        return eng

    yield make
    for eng in made:
        eng.close()


@functools.lru_cache(maxsize=1)
def _dwt_source(name, filt, point=False):
    args = (POINT_CASES if point else DWT_CASES)[name]
    cp = _coding(args, filt)
    planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=len(name) + 11 * point)
    return cp, planes, P.forward(cp, planes)


def _encode_matches(cp, coefs, res, ref, sample=257):
    """res (one engine) has ref's (another's) block table and bytes, and every `sample`th code block, the last ones
    included, the oracle's bytes"""
    assert res.num_blocks == ref.num_blocks
    assert np.array_equal(res.blocks, ref.blocks), "block tables differ"
    assert np.array_equal(res.bytes, ref.bytes), "coded bytes differ"
    rects = P.tile_rects(cp)
    blks = P.enumerate_all(cp)
    assert len(blks) == res.num_blocks
    for i in list(range(0, len(blks), sample)) + list(range(len(blks) - 16, len(blks))):
        t, c, b = blks[i]
        if b.x1 == b.x0 or b.y1 == b.y0:
            continue
        assert np.array_equal(P.encode_block(cp, coefs, rects[t], c, b), res.block_bytes(i)), "block %d differs from the oracle" % i


def _dwt_case(engine, make_engine, cp, planes, ref):
    # the Job API: every tile in one enqueue per level
    job = engine.job(cp)
    try:
        job.upload(planes)
        job.forward()
        got = [np.zeros_like(p) for p in planes]
        job.download_coeffs(got)
        msg = _first_difference(got, ref)
        assert not msg, "forward: " + msg
        coefs = _perturbed(cp, ref, seed=5)
        want = P.inverse(cp, coefs)
        job.upload_coeffs(coefs)
        job.inverse()
        got = [np.full_like(p, -1) for p in planes]
        job.download(got)
        msg = _first_difference(got, want)
        assert not msg, "inverse: " + msg
    finally:
        job.close()
    # the chunked host calls by default (8 chunks, each far below the limit) on an engine made and used while B2K_CHUNKS
    # is unset -- a job reads it when it is built -- and then with one chunk on another engine
    L = G.lib()
    default = make_engine(None)
    n0 = L.b2k_launch_count()
    res8 = default.encode(cp, planes)
    launches8 = L.b2k_launch_count() - n0
    try:
        if cp.irreversible:
            want = [np.full_like(p, -1) for p in planes]
            default.decode(cp, res8.blocks.copy(), res8.bytes.copy(), want)
        else:
            want = planes
        cs = G.codestream_write(cp, res8.blocks, res8.bytes, num_tiles=res8.num_tiles).copy()
        one = make_engine(1)
        n0 = L.b2k_launch_count()
        res1 = one.encode(cp, planes)
        launches1 = L.b2k_launch_count() - n0
        try:
            assert launches1 < launches8, "one chunk made %d launches, the default chunks %d" % (launches1, launches8)
            _encode_matches(cp, ref, res1, res8)
            out = [np.full_like(p, -1) for p in planes]
            one.decode(cp, res1.blocks.copy(), res1.bytes.copy(), out)
            msg = _first_difference(out, want)
            assert not msg, "decode: " + msg
        finally:
            res1.free()
    finally:
        res8.free()
    # the single-stream device code-stream calls with one chunk
    import torch
    img = torch.from_numpy(np.stack(planes).astype(np.uint8)).cuda()
    dcs = one.encode_codestream_device(cp, img, device_output=True)
    torch.cuda.synchronize()
    assert np.array_equal(dcs.cpu().numpy(), cs), "device code stream differs from the host writer's"
    _, dec = one.decode_codestream_device(dcs, dtype=torch.int32)
    torch.cuda.synchronize()
    got = list(dec.cpu().numpy())
    if not cp.irreversible:
        msg = _first_difference(got, planes)
        assert not msg, "device code stream round trip: " + msg


@pytest.mark.gpu
@pytest.mark.parametrize("filt", FILTERS)
@pytest.mark.parametrize("name", list(DWT_CASES))
def test_dwt_descriptors_past_the_grid(engine, make_engine, name, filt):
    cp, planes, ref = _dwt_source(name, filt)
    _dwt_case(engine, make_engine, cp, planes, ref)


@pytest.mark.gpu
@pytest.mark.parametrize("filt", FILTERS)
@pytest.mark.parametrize("name", list(POINT_CASES))
def test_point_transform_descriptors_past_the_grid(engine, make_engine, name, filt):
    cp, planes, ref = _dwt_source(name, filt, point=True)
    _dwt_case(engine, make_engine, cp, planes, ref)


# ---- rows past the grid -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("numres", TALL_NUMRES)
@pytest.mark.parametrize("nc", TALL_NC)
def test_image_taller_than_the_grid(engine, nc, numres):
    import torch
    cp = G.make_coding(TALL["width"], TALL["height"], nc, TALL["prec"], numres=numres)
    planes = P.synthetic_image(TALL["width"], TALL["height"], nc, TALL["prec"], seed=40 + nc + numres)
    ref = engine.encode(cp, planes)
    try:
        for dt in DTYPES:
            chw = np.stack(planes).astype(dt)
            for layout in ("CHW", "HWC"):
                host = chw if layout == "CHW" else np.ascontiguousarray(chw.transpose(1, 2, 0))
                img = torch.from_numpy(host).cuda()
                res = engine.encode_device(cp, img, layout=layout)
                try:
                    assert np.array_equal(res.blocks, ref.blocks) and np.array_equal(res.bytes, ref.bytes), (dt, layout)
                finally:
                    res.free()
                out = torch.from_numpy(np.full_like(host, np.iinfo(dt).max)).cuda()
                engine.decode_device(cp, ref.blocks, ref.bytes, out, layout=layout)
                torch.cuda.synchronize()
                got = out.cpu().numpy()
                got = (got if layout == "CHW" else got.transpose(2, 0, 1)).astype(np.int32)
                msg = _first_difference(list(got), planes)
                assert not msg, "%s %s: %s" % (dt, layout, msg)
        cs = G.codestream_write(cp, ref.blocks, ref.bytes, num_tiles=ref.num_tiles).copy()
    finally:
        ref.free()
    # a batch of two: the batch conversions loop over the rows with a clamped grid.y
    pair = torch.from_numpy(np.stack([np.stack(planes), np.stack(planes)[:, ::-1].copy()])).to(torch.int16).cuda()
    streams, status = engine.encode_codestreams_device(cp, pair)
    torch.cuda.synchronize()
    assert status == [(0, "")] * 2
    assert np.array_equal(streams[0].cpu().numpy(), cs)
    single = engine.encode_codestream_device(cp, pair[1], device_output=True)
    torch.cuda.synchronize()
    assert np.array_equal(streams[1].cpu().numpy(), single.cpu().numpy())
    _, out, status = engine.decode_codestreams_device(streams, dtype=torch.int16, layout="HWC")
    torch.cuda.synchronize()
    assert status == [(0, "")] * 2
    assert torch.equal(out.permute(0, 3, 1, 2), pair)


# ---- every sample width and component count, HWC ------------------------------------------------------------------------
def _conv_view(torch, base, S, NC, variant):
    """a (CONV_H, CONV_W, NC) view of `base` (CONV_H, CONV_W, NC) in the variant's layout, holding base's samples"""
    dt = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[S]
    n = CONV_H * CONV_W * NC
    if variant == "contiguous":
        buf = base.to(dt).contiguous()
        return buf, buf
    if variant == "wider_pixel":
        buf = torch.zeros((CONV_H, CONV_W, _wider(NC)), dtype=dt, device="cuda")
        buf[..., :NC] = base.to(dt)
        return buf[..., :NC], buf
    flat = torch.zeros(n + 16, dtype=dt, device="cuda")
    view = flat[1:1 + n].view(CONV_H, CONV_W, NC)
    view.copy_(base.to(dt))
    return view, flat


@pytest.mark.gpu
@pytest.mark.parametrize("S", (1, 2, 4))
def test_interleaved_conversions(engine, S):
    import torch
    for NC in (1, 2, 3, 4):
        prec = 8 if S == 1 else 12
        cp = G.make_coding(CONV_W, CONV_H, NC, prec, numres=2, mct=False)
        planes = P.synthetic_image(CONV_W, CONV_H, NC, prec, seed=S * 10 + NC)
        ref = engine.encode(cp, planes)
        base = torch.from_numpy(np.stack(planes)).permute(1, 2, 0).contiguous().cuda()
        try:
            for variant in CONV_VARIANTS:
                view, buf = _conv_view(torch, base, S, NC, variant)
                res = engine.encode_device(cp, view, layout="HWC")
                try:
                    assert np.array_equal(res.blocks, ref.blocks) and np.array_equal(res.bytes, ref.bytes), (NC, variant)
                finally:
                    res.free()
                before = buf.clone()
                view.fill_(0)
                engine.decode_device(cp, ref.blocks, ref.bytes, view, layout="HWC")
                torch.cuda.synchronize()
                assert torch.equal(view.to(torch.int32), base.to(torch.int32)), (NC, variant)
                assert torch.equal(buf, before), (NC, variant, "bytes outside the view were written")
        finally:
            ref.free()


# ---- more streams than the grid -------------------------------------------------------------------------------------------
def _many_images(torch, n, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    ramp = torch.arange(64, dtype=torch.int32).view(1, 1, 8, 8)
    noise = torch.randint(0, 16, (n, 1, 8, 8), generator=g, dtype=torch.int32)
    return ((ramp * 3 + noise + torch.arange(n).view(n, 1, 1, 1)) & 255).to(torch.uint8).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("chunks", CHUNK_SETTINGS)
@pytest.mark.parametrize("numres", MANY_NUMRES)
def test_more_streams_than_the_grid(make_engine, numres, chunks):
    import torch
    eng = make_engine(chunks)
    cp = G.make_coding(8, 8, 1, 8, numres=numres)
    imgs = _many_images(torch, MANY, seed=numres)
    streams, status = eng.encode_codestreams_device(cp, imgs)
    torch.cuda.synchronize()
    failed = [(i, s) for i, s in enumerate(status) if s != (0, "")]
    assert not failed, "%d streams failed, first %s" % (len(failed), failed[:3])
    lengths = [int(s.numel()) for s in streams]
    assert [int(s.storage_offset()) for s in streams] == placement(lengths)
    for i in (0, 1023, 1024, MANY - 3, MANY - 2, MANY - 1):
        single = eng.encode_codestream_device(cp, imgs[i], device_output=True)
        torch.cuda.synchronize()
        assert torch.equal(streams[i], single), i
    # decode from views of one buffer: at 16-byte boundaries, then at odd offsets
    host = streams[0].untyped_storage()
    arena = torch.empty(0, dtype=torch.uint8, device="cuda").set_(host).cpu().numpy()
    for align, skew in ((16, 0), (16, 1)):
        at, pos = 0, []
        for n in lengths:
            at = (at + align - 1) // align * align + skew
            pos.append(at)
            at += n
        buf = np.zeros(at + 16, np.uint8)
        offs = placement(lengths)
        for p, o, n in zip(pos, offs, lengths):
            buf[p:p + n] = arena[o:o + n]
        dbuf = torch.from_numpy(buf).cuda()
        views = [dbuf[p:p + n] for p, n in zip(pos, lengths)]
        assert skew == 0 or all(p % 2 for p in pos)
        _, out, dstatus = eng.decode_codestreams_device(views, dtype=torch.uint8)
        torch.cuda.synchronize()
        failed = [(i, s) for i, s in enumerate(dstatus) if s != (0, "")]
        assert not failed, "skew %d: %d streams failed, first %s" % (skew, len(failed), failed[:3])
        bad = (out != imgs).flatten(1).any(1).nonzero().flatten().tolist()
        assert not bad, "images %s differ (of %d)" % (bad[:8], len(bad))
    eng.close()


@pytest.mark.gpu
def test_placement_scan_rounds(engine):
    import torch
    cp = G.make_coding(8, 8, 1, 8, numres=2)
    imgs = _many_images(torch, max(PLACEMENT_BATCHES), seed=9)
    singles = [engine.encode_codestream_device(cp, imgs[i], device_output=True) for i in range(len(imgs))]
    torch.cuda.synchronize()
    for n in PLACEMENT_BATCHES:
        streams, status = engine.encode_codestreams_device(cp, imgs[:n])
        torch.cuda.synchronize()
        assert all(s == (0, "") for s in status)
        assert [int(s.storage_offset()) for s in streams] == placement([int(s.numel()) for s in streams])
        bad = [i for i in range(n) if not torch.equal(streams[i], singles[i])]
        assert not bad, (n, bad[:8])


# ---- tile parts past the grid, long main headers ----------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def _parts_streams():
    """the 90,000-part stream and its variants, encoded by the host path: (coding, image, {name: bytes})"""
    eng = G.Engine(0)
    try:
        cp = G.make_coding(**PARTS)
        planes = P.synthetic_image(PARTS["width"], PARTS["height"], 1, 8, seed=77)
        res = eng.encode(cp, planes)
        try:
            out = {name: G.codestream_write(cp, res.blocks, res.bytes, flags, num_tiles=res.num_tiles).copy()
                   for name, flags in (("parts", PARTS_FLAGS), ("tiles", G.CS_TLM | G.CS_PLT), ("no_tlm", G.CS_PLT))}
        finally:
            res.free()
    finally:
        eng.close()
    return cp, planes, out


def _main_header_end(cs):
    """the offset of the first SOT marker: where the main header ends"""
    b = np.asarray(cs)
    at = np.flatnonzero((b[:-1] == 0xFF) & (b[1:] == 0x90))
    return int(at[0])


@pytest.mark.gpu
def test_tile_parts_past_the_grid(engine):
    import torch
    import test_device_batch_decode as BD
    cp, planes, cs = _parts_streams()
    full = cs["parts"]
    assert _main_header_end(full) > 500000
    assert _main_header_end(cs["tiles"]) == main_header_length(PARTS, G.CS_TLM | G.CS_PLT, PARTS_TILES)
    assert _main_header_end(cs["no_tlm"]) == main_header_length(PARTS, G.CS_PLT, PARTS_TILES)
    dcs = torch.from_numpy(full).cuda()
    # every tile in the window, at half resolution: the device parse and gather against the host-bytes path, and
    # sampled tiles -- the first ones, and ones whose parts lie past the 65,535th -- against the oracle's decoder
    win = (cp.x0, cp.y0, cp.x1, cp.y1)
    vcp, got = engine.decode_window_device(dcs, window=win, reduce=1, dtype=torch.int32)
    _, want = engine.decode_codestream_device(full, window=win, reduce=1, dtype=torch.int32)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert engine.codestream_window_device_stats()[0] == PARTS_TILES
    vcp, vblocks, _ = G.codestream_parse_window(full, win, 1)
    got = got.cpu().numpy()[0]
    for t, rec in _oracle_tiles(vcp, vblocks, full, (0, 1, 200, 21845, 22000, PARTS_TILES - 1)).items():
        x0, y0, x1, y1 = P.tile_rects(vcp)[t]
        assert np.array_equal(got[y0 - vcp.y0:y1 - vcp.y0, x0 - vcp.x0:x1 - vcp.x0], rec), "tile %d differs from the oracle" % t
    # two such images through the batch writer: each stream's part scan takes 88 rounds, the encoder converts no image
    # in some chunks; every stream as its single call writes it
    pair = torch.from_numpy(np.stack([planes[0], planes[0][::-1]])[:, None].astype(np.uint8)).cuda()
    streams, status = engine.encode_codestreams_device(cp, pair, PARTS_FLAGS)
    torch.cuda.synchronize()
    assert status == [(0, "")] * 2
    assert [int(x.storage_offset()) for x in streams] == placement([int(x.numel()) for x in streams])
    assert np.array_equal(streams[0].cpu().numpy(), full)
    single = engine.encode_codestream_device(cp, pair[1], PARTS_FLAGS, device_output=True)
    torch.cuda.synchronize()
    assert torch.equal(streams[1], single)
    # the whole image, alone and as a batch of two
    _, img = engine.decode_codestream_device(dcs, dtype=torch.int32)
    torch.cuda.synchronize()
    assert np.array_equal(img.cpu().numpy()[0], planes[0])
    _, out, status = engine.decode_codestreams_device([dcs, dcs.clone()], dtype=torch.int32)
    torch.cuda.synchronize()
    assert status == [(0, "")] * 2
    assert all(np.array_equal(out[i, 0].cpu().numpy(), planes[0]) for i in range(2))
    # headers of 540 KB, 180 KB and a few hundred bytes, and one cut inside its main header, in one batch: each
    # stream's status, text and pixels as its single call gives them
    reads = {k: len(header_reads(len(v), _main_header_end(v))[0]) - 1 for k, v in cs.items()}
    assert reads["parts"] >= 3 and reads["tiles"] >= 3 and reads["no_tlm"] == 0, reads
    cut = full[:5000].copy()
    assert header_reads(len(cut), _main_header_end(full))[1]
    batch = [BD._dev(torch, s) for s in (cs["no_tlm"], full, cut, cs["tiles"])]
    BD._check_batch(engine, torch, batch, dtype=torch.int32)


def _oracle_tiles(cp, blocks, cs, tiles):
    """{tile: its pixels} decoded by the oracle from a parsed block table (the tiles of a coding whose tiles all have
    the same blocks)"""
    rects = P.tile_rects(cp)
    per = len(blocks) // len(rects)
    out = {}
    for t in tiles:
        x0, y0, x1, y1 = rects[t]
        coefs = [np.zeros((cp.y1 - cp.y0, cp.x1 - cp.x0), np.int32) for _ in range(cp.numcomps)]
        for j, (_, c, b) in enumerate(P.enumerate_all(cp, tiles={t})):
            blk = blocks[t * per + j]
            assert (int(blk["tile"]), int(blk["comp"]), int(blk["x0"]), int(blk["y0"])) == (t, c, b.x0, b.y0)
            bw, bh = b.x1 - b.x0, b.y1 - b.y0
            if bw == 0 or bh == 0 or blk["length"] == 0:
                continue
            o, n = int(blk["offset"]), int(blk["length"])
            win = P.decode_block(cp, cs[o:o + n], c, b, numbps=int(blk["numbps"]))
            coefs[c][y0 - cp.y0 + b.buf_y:y0 - cp.y0 + b.buf_y + bh, x0 - cp.x0 + b.buf_x:x0 - cp.x0 + b.buf_x + bw] = win
        rec = P.inverse(cp, coefs, tiles={t})
        out[t] = rec[0][y0 - cp.y0:y1 - cp.y0, x0 - cp.x0:x1 - cp.x0]
    return out


@pytest.mark.gpu
def test_main_header_one_prefix_longer(engine):
    """a main header between 4 and 8 KiB: read again once with twice the prefix, in a batch with a stream read once"""
    import torch
    import test_device_batch_decode as BD
    cp = G.make_coding(**ONE_REREAD)
    planes = P.synthetic_image(ONE_REREAD["width"], ONE_REREAD["height"], 1, 8, seed=5)
    res = engine.encode(cp, planes)
    try:
        tlm = G.codestream_write(cp, res.blocks, res.bytes, G.CS_TLM | G.CS_PLT, num_tiles=res.num_tiles).copy()
        plain = G.codestream_write(cp, res.blocks, res.bytes, G.CS_PLT, num_tiles=res.num_tiles).copy()
    finally:
        res.free()
    assert _main_header_end(tlm) == main_header_length(ONE_REREAD, G.CS_TLM | G.CS_PLT, 1024)
    assert header_reads(len(tlm), _main_header_end(tlm))[0] == [HEADER_PREFIX, 2 * HEADER_PREFIX]
    BD._check_batch(engine, torch, [BD._dev(torch, s) for s in (tlm, plain, tlm)], dtype=torch.int32)
    _, out, status = engine.decode_codestreams_device([BD._dev(torch, tlm), BD._dev(torch, plain)], dtype=torch.int32)
    torch.cuda.synchronize()
    assert status == [(0, "")] * 2
    assert all(np.array_equal(out[i, 0].cpu().numpy(), planes[0]) for i in range(2))


# ---- large copies --------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_large_stream_copies(engine):
    import torch
    import test_device_batch_decode as BD
    cp = G.make_coding(**LARGE)
    rng = np.random.default_rng(3)
    raw = []
    for k in range(3):
        plane = rng.integers(0, 1 << 16, (256, 256)).astype(np.int32)
        res = engine.encode(cp, [plane])
        try:
            raw.append((plane, G.codestream_write(cp, res.blocks, res.bytes, num_tiles=res.num_tiles).copy()))
        finally:
            res.free()
    longest = max(len(s) for _, s in raw)
    assert copy_table_grid(3, longest)[0] > 1, longest
    assert any(len(s) % 16 for _, s in raw), "every length a multiple of 16: no tail"
    reached = set()
    for skew in LARGE_SKEWS:
        at, pos = 0, []
        for _, s in raw:
            at = (at + 15) // 16 * 16 + skew
            pos.append(at)
            at += len(s)
        buf = np.zeros(at + 16, np.uint8)
        for p, (_, s) in zip(pos, raw):
            buf[p:p + len(s)] = s
        dbuf = torch.from_numpy(buf).cuda()
        assert dbuf.data_ptr() % 256 == 0
        views = [dbuf[p:p + len(s)] for p, (_, s) in zip(pos, raw)]
        for p, (_, s) in zip(pos, raw):      # into the arena at 256-byte boundaries
            reached |= copy_entry_paths(p % 16, 0, len(s))
        _, out, status = engine.decode_codestreams_device(views, dtype=torch.int32)
        torch.cuda.synchronize()
        assert status == [(0, "")] * 3
        for i, (plane, _) in enumerate(raw):
            assert np.array_equal(out[i, 0].cpu().numpy(), plane), (skew, i)
    assert reached == {"16-byte", "tail", "bytes"}, reached
    # one stream's window: its one tile part of more than 4 KiB gathered by a strip of CTAs
    plane, cs = raw[0]
    dcs = torch.from_numpy(cs).cuda()
    win = (0, 0, LARGE["width"], LARGE["height"])
    _, got = engine.decode_window_device(dcs, window=win, dtype=torch.int32)
    _, want = engine.decode_codestream_device(cs, window=win, dtype=torch.int32)
    torch.cuda.synchronize()
    assert t2_gather_grid(1, engine.codestream_window_device_stats()[1])[0] > 1
    assert torch.equal(got, want) and np.array_equal(got.cpu().numpy()[0], plane)
    # one stream whose header parses among streams that do not: its bytes go by a plain copy
    good = BD._dev(torch, raw[0][1])
    bad = [BD._dev(torch, np.zeros(64, np.uint8)), BD._dev(torch, raw[1][1][:40])]
    BD._check_batch(engine, torch, [bad[0], good, bad[1]], dtype=torch.int32)
