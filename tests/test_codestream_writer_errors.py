"""Return codes and error texts of the host code-stream writers (b2k_codestream_write, _write_tiles, _write_tiles_at,
_write_header) on crafted block tables: each fault alone, two faults in one tile and in different tiles (which one a
writer reports), the size query, a buffer too small, tile parts placed outside the buffer, and refinement (2/3-pass)
tables.  The faults that need more than 4 GiB of block bytes claim a large arena (num_bytes) over a small buffer: a
writer that finds a fault reads no block byte.  CPU only."""
import ctypes as C

import numpy as np
import pytest

import grok_b200 as G

RANGE = "code block outside the writer's range (bit planes / passes)"
ARENA = "block offsets exceed the byte arena"
PACKET = "packet longer than 4 GiB"
PART = "tile part longer than 4 GiB"
ENUM = "block table does not match the tile's enumeration"
BIG = 0xC0000000  # a block length of which two make more than 4 GiB
HUGE_ARENA = 1 << 40


@pytest.fixture(scope="module")
def L():
    return G.lib()


def coding():
    """2 x 2 tiles, 2 components, 2 resolutions: 4 packets per tile (r0c0 r0c1 r1c0 r1c1 in LRCP)"""
    return G.make_coding(128, 128, 2, 8, numres=2, tile=(64, 64), cblk=(32, 32))


def table(cp, tile_mod=1, tile_rem=0, length=10):
    t = G.enumerate_blocks(cp, tile_mod, tile_rem)
    t["numpasses"], t["numbps"], t["length"], t["length2"] = 1, 1, length, 0
    t["offset"] = np.arange(len(t)) * length
    return t


def where(t, tile, comp, resno, k=0):
    """index of the k-th block of (tile, comp, resno) in table t"""
    return int(np.flatnonzero((t["tile"] == tile) & (t["comp"] == comp) & (t["resno"] == resno))[k])


def fault(t, kind, tile, comp=0, resno=0, k=0):
    """t with one fault in block k of (tile, comp, resno); returns the arena size the table claims"""
    i = where(t, tile, comp, resno, k)
    if kind == "range":
        t["numbps"][i] = t["kmax"][i] + 1
    elif kind == "passes":
        t["numpasses"][i] = 4
    elif kind == "arena":
        t["offset"][i] = HUGE_ARENA << 1
    elif kind == "packet":  # two blocks of one packet of resolution 1
        i, j = where(t, tile, comp, 1, k), where(t, tile, comp, 1, k + 1)
        t["length"][i] = t["length"][j] = BIG
        return HUGE_ARENA
    elif kind == "part":  # one block in each of two packets of one tile part
        j = where(t, tile, comp, 1 - resno, 0)
        t["length"][i] = t["length"][j] = BIG
        return HUGE_ARENA
    else:
        raise ValueError(kind)
    return None


def drop(t, tile, comp=0, resno=1):
    """t without one block of (tile, comp, resno): the tile no longer matches its enumeration"""
    return np.delete(t, where(t, tile, comp, resno))


class Call:
    def __init__(self, L, cp, t, num_bytes=None):
        self.L, self.cp, self.t = L, cp, np.ascontiguousarray(t)
        end = int(np.minimum(t["offset"] + t["length"] + t["length2"], 1 << 20).max()) if num_bytes is None else 1 << 12
        self.data = np.arange(max(1, end), dtype=np.uint64).astype(np.uint8)
        self.r = G.result_from_tables(self.t, self.data, 4)
        if num_bytes is not None:
            self.r.num_bytes = num_bytes

    def _rc(self, rc):
        return (rc, self.L.b2k_last_error().decode() if rc < 0 else "")

    def write(self, flags, out=None, cap=0):
        return self._rc(self.L.b2k_codestream_write(C.byref(self.cp), C.byref(self.r), flags,
                                                    None if out is None else out.ctypes.data, cap))

    def tiles(self, flags, mod=1, rem=0, out=None, cap=0, tile_bytes=None):
        return self._rc(self.L.b2k_codestream_write_tiles(C.byref(self.cp), C.byref(self.r), flags, mod, rem,
                                                          None if out is None else out.ctypes.data, cap,
                                                          None if tile_bytes is None else tile_bytes.ctypes.data))

    def tiles_at(self, flags, tile_at, mod=1, rem=0, out=None, cap=0):
        ta = np.ascontiguousarray(tile_at, dtype=np.uint64)
        return self._rc(self.L.b2k_codestream_write_tiles_at(C.byref(self.cp), C.byref(self.r), flags, mod, rem,
                                                             None if out is None else out.ctypes.data, cap, ta.ctypes.data))


def all_writers(L, cp, t, flags, num_bytes=None):
    """(whole image, per-rank, per-rank at) of the full table t"""
    c = Call(L, cp, t, num_bytes)
    out = np.zeros(1 << 16, np.uint8)
    return c.write(flags), c.tiles(flags), c.tiles_at(flags, np.arange(4) * 4096, out=out, cap=out.size)


SINGLE = [("range", RANGE), ("passes", RANGE), ("arena", ARENA), ("packet", PACKET), ("part", PART)]


@pytest.mark.parametrize("kind,text", SINGLE)
@pytest.mark.parametrize("tile", [0, 3])
def test_single_fault(L, kind, text, tile):
    cp = coding()
    t = table(cp)
    nb = fault(t, kind, tile, comp=1, resno=0)
    for rc in all_writers(L, cp, t, G.CS_TLM | G.CS_PLT, nb):
        assert rc == (-1, text)


def test_single_enumeration_mismatch(L):
    cp = coding()
    for tile in (0, 2):
        for rc in all_writers(L, cp, drop(table(cp), tile), G.CS_PLT):
            assert rc == (-1, ENUM)


def test_part_fault_gone_with_a_tile_part_per_resolution(L):
    """the two big blocks lie in different tile parts when each resolution has its own"""
    cp = coding()
    t = table(cp)
    nb = fault(t, "part", 1, comp=0, resno=0)
    c = Call(L, cp, t, nb)
    assert c.write(G.CS_TPARTS_R | G.CS_TLM)[0] > 2 * BIG  # the size query alone: no block byte is read
    assert c.write(G.CS_TLM) == (-1, PART)


# (fault a, fault b, LRCP's text, CPRL's text): a = (kind, comp, resno), both in tile 1
SAME_TILE = [
    (("range", 0, 1), ("arena", 1, 0), ARENA, RANGE),    # code-stream order of their packets decides
    (("arena", 0, 1), ("range", 1, 0), RANGE, ARENA),
    (("packet", 0, 1), ("arena", 1, 0), ARENA, PACKET),
    (("part", 0, 0), ("range", 1, 0), RANGE, RANGE),     # packet faults before the tile part's
    (("part", 1, 0), ("arena", 0, 1), ARENA, ARENA),
    (("range", 1, 1), ("arena", 1, 1), RANGE, RANGE),   # one packet: the writer's range before the arena
    (("arena", 1, 1), ("packet", 1, 1), ARENA, ARENA),  # one packet: the arena before its length
]


@pytest.mark.parametrize("a,b,lrcp,cprl", SAME_TILE)
def test_two_faults_in_one_tile(L, a, b, lrcp, cprl):
    cp = coding()
    for prog, text in ((G.LRCP, lrcp), (G.CPRL, cprl)):
        t = table(cp)
        nb = fault(t, a[0], 1, a[1], a[2])
        nb = fault(t, b[0], 1, b[1], b[2]) or nb
        for rc in all_writers(L, cp, t, G.CS_PROG(prog) | G.CS_PLT, nb):
            assert rc == (-1, text), (a, b, prog)


@pytest.mark.parametrize("first,second", [("range", "arena"), ("part", "range"), ("arena", "packet"), ("packet", "part"),
                                          ("arena", "enum"), ("part", "enum")])
def test_the_first_failing_tile_decides(L, first, second):
    cp = coding()
    text = dict(SINGLE)[first]
    for tiles in ((0, 1), (1, 3)):
        t = table(cp)
        nb = fault(t, first, tiles[0], comp=1, resno=1 if first != "part" else 0)
        if second == "enum":
            t = drop(t, tiles[1])
        else:
            nb = fault(t, second, tiles[1]) or nb
        for rc in all_writers(L, cp, t, G.CS_TLM, nb):
            assert rc == (-1, text), (first, second, tiles)
    t = drop(table(cp), 0)
    fault(t, "arena", 1)
    for rc in all_writers(L, cp, t, 0):
        assert rc == (-1, ENUM)


def test_enumeration_mismatch_before_the_tiles_packet_faults(L):
    cp = coding()
    t = table(cp)
    fault(t, "range", 2, comp=0, resno=0)
    for rc in all_writers(L, cp, drop(t, 2, comp=1, resno=1), 0):
        assert rc == (-1, ENUM)


def test_whole_image_entry_checks(L):
    cp = coding()
    t = table(cp)
    c = Call(L, cp, t)
    assert c.write(G.CS_PROG(5)) == (-1, "unknown progression order")
    c.r.num_tiles = 3
    assert c.write(0) == (-1, "the result does not hold every tile of the image (gather the shards first)")
    c = Call(L, cp, t[np.argsort(-t["tile"].astype(np.int64), kind="stable")])
    assert c.write(0) == (-1, "block table is not in tile order")
    grid = G.make_coding(264, 256, 1, 8, numres=1, tile=(1, 1))
    g = table(grid, length=1)
    c = Call(L, grid, g)
    c.r.num_tiles = 264 * 256
    assert c.write(G.CS_TLM) == (-1, "more than 65535 tiles")
    assert c.tiles(0) == (-1, "unknown progression order / too many tiles")


def test_per_rank_entry_checks(L):
    cp = coding()
    t = table(cp)
    c = Call(L, cp, t)
    out = np.zeros(1 << 16, np.uint8)
    assert c.tiles(G.CS_TPARTS_R) == (-1, "per-rank writers emit one tile part per tile")
    assert c.tiles_at(G.CS_TPARTS_R, np.zeros(4), out=out, cap=out.size) == (-1, "per-rank writers emit one tile part per tile")
    assert c.tiles(G.CS_PROG(6)) == (-1, "unknown progression order / too many tiles")
    assert c.tiles_at(G.CS_PROG(5), np.zeros(4), out=out, cap=out.size) == (-1, "unknown progression order / too many tiles")
    assert c.tiles(0, mod=2, rem=0)[1] == "the block table is not the shard's tiles in tile order"
    assert c.tiles(0, mod=0)[0] == -1 and c.tiles(0, mod=2, rem=2)[0] == -1
    s = Call(L, cp, table(cp, 2, 1))
    assert s.tiles(0, mod=2, rem=0) == (-1, "the block table is not the shard's tiles in tile order")
    assert s.tiles(0, mod=2, rem=1)[0] > 0
    assert L.b2k_codestream_write_tiles_at(C.byref(cp), C.byref(s.r), 0, 2, 1, out.ctypes.data, out.size, None) == -1


@pytest.mark.parametrize("flags", [0, G.CS_TLM | G.CS_PLT, G.CS_SOP | G.CS_EPH | G.CS_PROG(G.RPCL)])
def test_size_query_and_small_buffers(L, flags):
    cp = coding()
    t = table(cp)
    c = Call(L, cp, t)
    n, _ = c.write(flags)
    assert n > 0
    small = np.full(n - 1, 0xAB, np.uint8)
    assert c.write(flags, small, small.size) == (n, "")
    assert (small == 0xAB).all()
    full = np.zeros(n, np.uint8)
    assert c.write(flags, full, 0) == (n, "") and not full.any()
    assert c.write(flags, full, n) == (n, "")
    # the shards: sizes, then the tile parts behind each other or at given places
    tb = np.zeros(4, np.uint64)
    m, _ = c.tiles(flags, tile_bytes=tb)
    assert m == int(tb.sum())
    assert c.tiles(flags, out=small[:m - 1], cap=m - 1) == (m, "") and (small == 0xAB).all()
    parts = np.zeros(m, np.uint8)
    assert c.tiles(flags, out=parts, cap=m) == (m, "")
    header = np.zeros(n, np.uint8)
    hl = L.b2k_codestream_write_header(C.byref(cp), flags, tb.ctypes.data, 4, None, 0)
    assert hl == n - m - 2
    assert L.b2k_codestream_write_header(C.byref(cp), flags, tb.ctypes.data, 4, header.ctypes.data, hl - 1) == hl and not header.any()
    assert L.b2k_codestream_write_header(C.byref(cp), flags, tb.ctypes.data, 4, header.ctypes.data, hl) == hl
    assert np.array_equal(np.concatenate([header[:hl], parts, [0xFF, 0xD9]]), full)
    # at given places: reversed order, a gap between them; then one tile a byte past the end of the buffer
    at = np.zeros(4, np.uint64)
    pos = 0
    for k in (3, 2, 1, 0):
        at[k] = pos
        pos += int(tb[k]) + 7
    spread = np.zeros(pos, np.uint8)
    assert c.tiles_at(flags, at, out=spread, cap=pos) == (m, "")
    starts = np.concatenate([[0], np.cumsum(tb)[:-1]]).astype(np.int64)
    for k in range(4):
        assert np.array_equal(spread[at[k]:at[k] + tb[k]], parts[starts[k]:starts[k] + int(tb[k])])
    assert c.tiles_at(flags, at, out=None) == (m, "")
    bad = at.copy()
    bad[2] = pos - int(tb[2]) + 1
    assert c.tiles_at(flags, bad, out=spread, cap=pos) == (-1, "a tile part would land outside the buffer")
    assert c.tiles_at(flags, at, out=spread, cap=pos - 8) == (-1, "a tile part would land outside the buffer")
    # shard 1 of 2 on its own table
    s = Call(L, cp, table(cp, 2, 1))
    tb2 = np.zeros(2, np.uint64)
    assert s.tiles(flags, mod=2, rem=1, tile_bytes=tb2) == (int(tb2.sum()), "")
    assert list(tb2) == [tb[1], tb[3]]


def test_header_writer_checks(L):
    cp = coding()
    tb = np.full(4, 100, np.uint64)
    text = "TLM needs the length of every tile's tile part"
    h = L.b2k_codestream_write_header
    assert h(C.byref(cp), G.CS_TLM, None, 4, None, 0) == -1 and L.b2k_last_error().decode() == text
    assert h(C.byref(cp), G.CS_TLM, tb.ctypes.data, 3, None, 0) == -1 and L.b2k_last_error().decode() == text
    assert h(C.byref(cp), G.CS_PROG(5), tb.ctypes.data, 4, None, 0) == -1 and L.b2k_last_error().decode() == text
    assert h(C.byref(cp), 0, None, 0, None, 0) > 0
    assert h(C.byref(cp), G.CS_TLM, tb.ctypes.data, 4, None, 0) == h(C.byref(cp), 0, None, 0, None, 0) + 6 + 6 * 4


def test_refinement_tables(L):
    """2- and 3-pass blocks: the body is length + length2; a block without cleanup bytes is left out"""
    cp = coding()
    t = table(cp)
    t["numpasses"][::3], t["numpasses"][1::3] = 2, 3
    t["length2"] = np.where(t["numpasses"] > 1, 4, 0)
    t["offset"] = np.concatenate([[0], np.cumsum(t["length"] + t["length2"])[:-1]])
    c = Call(L, cp, t)
    n, _ = c.write(G.CS_TLM | G.CS_PLT)
    assert n > 0
    out = np.zeros(n, np.uint8)
    assert c.write(G.CS_TLM | G.CS_PLT, out, n) == (n, "")
    # the last block's refinement bytes end past the arena
    c.r.num_bytes -= 1
    assert c.write(0) == (-1, ARENA)
    assert c.tiles(0)[1] == ARENA
    # numpasses > 1 and no cleanup bytes: not included, so its refinement bytes need not lie in the arena
    u = t.copy()
    i = where(u, 2, 1, 1)
    u["numpasses"][i], u["length"][i], u["length2"][i], u["offset"][i] = 2, 0, 9, 1 << 36
    c = Call(L, cp, u)
    assert c.write(0)[0] > 0 and c.tiles(0)[0] > 0
    u["numpasses"][i] = 4
    assert c.write(0)[0] > 0
    u["length"][i] = 1
    assert c.write(0) == (-1, RANGE) and c.tiles(0) == (-1, RANGE)
