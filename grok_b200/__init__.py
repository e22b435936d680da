"""grok_b200 -- host-side Python mirror of the JPEG 2000 tile engine's C ABI.

The product is ``libgrokj2k_plugin.so`` (hand-written sm_90a CUDA behind the C ABI of
``include/grok_b200.h``); this module is only the ctypes doorway tests, ``bench.py`` and Python
hosts use.  It mirrors the reference's plugin surface (``src/lib/core/plugin/plugin_interface.h``,
``gpup/gpu_plugin_shared.h``): same entry-point names, argument meaning and return convention
(0 handled, >0 not handled -> host CPU path, <0 device failure).

There is NO CPU fallback here: if the shared library is missing or no CUDA device is present the
calls raise.  (The CPU oracle lives under ``oracle/`` and is test infrastructure only.)
"""
import ctypes as C
import os
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2K_LIB") or os.path.join(_HERE, "libgrokj2k_plugin.so")   # B2K_LIB: an experimental build (tools/build_variant.py)

GPUP_MAX_PASSES = 3 * (16 + 7) - 2


def _by_value(array_type, doc):
    """a ctypes array type whose instances (and rows) compare by value, as the scalar fields of two codings do"""
    return type(array_type.__name__, (array_type,), {"__doc__": doc, "__hash__": None,
                                                      "__eq__": lambda a, b: type(a) is type(b) and bytes(a) == bytes(b)})


_QccExpnRow = _by_value(C.c_uint8 * 97, "one component's b2k_coding.qcc_expn")
_QccMantRow = _by_value(C.c_uint16 * 97, "one component's b2k_coding.qcc_mant")
_QccExpn = _by_value(_QccExpnRow * 4, "b2k_coding.qcc_expn")
_QccMant = _by_value(_QccMantRow * 4, "b2k_coding.qcc_mant")


class Coding(C.Structure):
    """b2k_coding (include/grok_b200.h)."""
    _fields_ = [("x0", C.c_uint32), ("y0", C.c_uint32), ("x1", C.c_uint32), ("y1", C.c_uint32),
                ("tx0", C.c_uint32), ("ty0", C.c_uint32), ("tw", C.c_uint32), ("th", C.c_uint32),
                ("numcomps", C.c_uint16), ("prec", C.c_uint8), ("sgnd", C.c_uint8),
                ("numres", C.c_uint8), ("cblkw_exp", C.c_uint8), ("cblkh_exp", C.c_uint8),
                ("irreversible", C.c_uint8), ("mct", C.c_uint8), ("numgbits", C.c_uint8),
                ("prcw_exp", C.c_uint8 * 33), ("prch_exp", C.c_uint8 * 33), ("cblk_sty", C.c_uint8),
                ("qcd_explicit", C.c_uint8), ("qcd_expn", C.c_uint8 * 97), ("qcd_mant", C.c_uint16 * 97),
                ("qfactor", C.c_uint8), ("qcc_mask", C.c_uint8), ("qcc_expn", _QccExpn), ("qcc_mant", _QccMant)]


class Block(C.Structure):
    """b2k_block."""
    _fields_ = [("tile", C.c_uint32), ("comp", C.c_uint16), ("resno", C.c_uint8), ("band_index", C.c_uint8),
                ("orient", C.c_uint8), ("kmax", C.c_uint8), ("numbps", C.c_uint8), ("numpasses", C.c_uint8),
                ("precno", C.c_uint32), ("cblkno", C.c_uint32),
                ("x0", C.c_uint32), ("y0", C.c_uint32), ("x1", C.c_uint32), ("y1", C.c_uint32),
                ("buf_x", C.c_uint32), ("buf_y", C.c_uint32), ("length", C.c_uint32),
                ("offset", C.c_uint64), ("stepsize", C.c_float), ("length2", C.c_uint32)]


class Result(C.Structure):
    """b2k_result."""
    _fields_ = [("num_blocks", C.c_uint64), ("blocks", C.POINTER(Block)), ("bytes", C.POINTER(C.c_uint8)),
                ("num_bytes", C.c_uint64), ("num_tiles", C.c_uint32),
                ("ms_h2d", C.c_double), ("ms_dwt", C.c_double), ("ms_t1", C.c_double), ("ms_d2h", C.c_double),
                ("ms_total", C.c_double)]


class DevicePlanes(C.Structure):
    """b2k_device_planes: an image in the engine GPU's memory (component c of pixel (x, y) at
    comp[c] + (y * row_pitch[c] + x * col_step[c]) * sample_bytes)."""
    _fields_ = [("comp", C.c_void_p * 4), ("row_pitch", C.c_uint32 * 4), ("col_step", C.c_uint32 * 4), ("sample_bytes", C.c_uint32)]


BLOCK_DTYPE = np.dtype([("tile", "<u4"), ("comp", "<u2"), ("resno", "u1"), ("band_index", "u1"), ("orient", "u1"),
                        ("kmax", "u1"), ("numbps", "u1"), ("numpasses", "u1"), ("precno", "<u4"), ("cblkno", "<u4"),
                        ("x0", "<u4"), ("y0", "<u4"), ("x1", "<u4"), ("y1", "<u4"), ("buf_x", "<u4"), ("buf_y", "<u4"),
                        ("length", "<u4"), ("offset", "<u8"), ("stepsize", "<f4"), ("length2", "<u4")])
assert BLOCK_DTYPE.itemsize == C.sizeof(Block), (BLOCK_DTYPE.itemsize, C.sizeof(Block))

# the streaming callbacks (b2k_encoded_fn, b2k_decoded_fn)
_ENCODED_FN = C.CFUNCTYPE(C.c_int32, C.c_void_p, C.c_void_p, C.POINTER(Result), C.c_int32)
_DECODED_FN = C.CFUNCTYPE(None, C.c_void_p, C.c_void_p, C.c_int32)


def _signatures():
    """name -> (restype, argtypes) of every b2k_* function include/grok_b200.h declares (tests/test_host.py checks them
    against the header), and of gpup_tile_free.  Block tables, byte buffers and device addresses pass as c_void_p."""
    vp, pp, i32, u32, i64, u64 = C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_uint32, C.c_int64, C.c_uint64
    cp, res, img = C.POINTER(Coding), C.POINTER(Result), C.POINTER(DevicePlanes)
    pres, pi32, pu32, pu64 = C.POINTER(res), C.POINTER(i32), C.POINTER(u32), C.POINTER(u64)
    pf, pd = C.POINTER(C.c_float), C.POINTER(C.c_double)
    return {
        "b2k_engine_create": (i32, [i32, pp]),
        "b2k_engine_destroy": (None, [vp]),
        "b2k_last_error": (C.c_char_p, []),
        "b2k_coding_from_gpup": (i32, [vp, vp, i32, cp]),
        "b2k_host_alloc": (vp, [C.c_size_t]),
        "b2k_host_free": (None, [vp]),
        "b2k_set_host_threads": (i32, [i32]),
        "b2k_host_pack_last": (i32, [i32]),
        "b2k_encode": (i32, [vp, cp, pp, pu32, u32, u32, pres]),
        "b2k_encode16": (i32, [vp, cp, pp, pu32, u32, u32, pres]),
        "b2k_encode16_interleaved": (i32, [vp, cp, vp, u32, u32, u32, pres]),
        "b2k_result_free": (None, [res]),
        "b2k_decode": (i32, [vp, cp, vp, u64, vp, u64, pp, pu32, u32, u32, pd]),
        "b2k_decode_window": (i32, [vp, cp, vp, u64, vp, u64, pp, pu32, pu32, u32, pd]),
        "b2k_decode16": (i32, [vp, cp, vp, u64, vp, u64, pp, pu32, u32, u32, pd]),
        "b2k_encode_device": (i32, [vp, cp, img, u32, u32, vp, pres]),
        "b2k_decode_device": (i32, [vp, cp, vp, u64, vp, u64, img, pu32, u32, u32, vp, pd]),
        "b2k_encode_codestream_device": (i64, [vp, cp, img, u32, vp, pp]),
        "b2k_encode_codestreams_device": (i32, [vp, cp, u32, img, u32, vp, pp, pu64, pu64, pi32, pd]),
        "b2k_encode_codestreams_error": (C.c_char_p, [vp, u32]),
        "b2k_decode_codestream_device": (i32, [vp, vp, u64, img, vp, cp, pd]),
        "b2k_decode_codestreams_device": (i32, [vp, u32, pp, pu64, img, vp, cp, pi32, pd]),
        "b2k_decode_codestreams_error": (C.c_char_p, [vp, u32]),
        "b2k_codestream_parse_device": (i64, [vp, vp, u64, vp, cp, vp, u64]),
        "b2k_codestream_parse_device_stats": (i32, [vp, pu32, pu32]),
        "b2k_codestream_parse_window_device": (i64, [vp, vp, u64, pu32, u32, vp, cp, vp, u64]),
        "b2k_decode_codestream_window_device": (i32, [vp, vp, u64, pu32, u32, img, vp, cp, pu32, pd]),
        "b2k_codestream_window_device_stats": (i32, [vp, pu32, pu64]),
        "b2k_decode_codestreams_window_device": (i32, [vp, u32, pp, pu64, pu32, u32, img, vp, cp, pu32, pi32, pd]),
        "b2k_enumerate": (i64, [cp, u32, u32, vp, u64]),
        "b2k_result_to_gpup_tile": (vp, [cp, res, u32]),
        "gpup_tile_free": (None, [vp]),
        "b2k_job_create": (i32, [vp, cp, u32, u32, pp]),
        "b2k_job_destroy": (None, [vp]),
        "b2k_job_upload": (i32, [vp, pp, pu32]),
        "b2k_job_forward": (i32, [vp, pf]),
        "b2k_job_t1_encode": (i32, [vp, pf, pu64]),
        "b2k_job_t1_decode": (i32, [vp, pf]),
        "b2k_job_inverse": (i32, [vp, pf]),
        "b2k_job_roundtrip": (i32, [vp, pf, pf, pu64]),
        "b2k_job_roundtrip_n": (i32, [vp, u32, pf, pf, pf, pu64]),
        "b2k_job_roundtrip_pipelined_n": (i32, [vp, u32, u32, u32, pf, pf, pf, pu64]),
        "b2k_job_download": (i32, [vp, pp, pu32]),
        "b2k_job_download_coeffs": (i32, [vp, pp, pu32]),
        "b2k_job_upload_coeffs": (i32, [vp, pp, pu32]),
        "b2k_job_t1_decode_blocks": (i32, [vp, vp, u64, vp, u64, pf]),
        "b2k_job_fetch_result": (i32, [vp, pres]),
        "b2k_job_num_blocks": (u64, [vp]),
        "b2k_result_merge": (i32, [cp, pres, u32, pres]),
        "b2k_codestream_write": (i64, [cp, res, u32, vp, u64]),
        "b2k_codestream_parse": (i64, [vp, u64, cp, vp, u64]),
        "b2k_codestream_write_tiles": (i64, [cp, res, u32, u32, u32, vp, u64, vp]),
        "b2k_codestream_write_header": (i64, [cp, u32, vp, u32, vp, u64]),
        "b2k_codestream_write_tiles_at": (i64, [cp, res, u32, u32, u32, vp, u64, vp]),
        "b2k_codestream_parse_window": (i64, [vp, u64, pu32, u32, cp, vp, u64]),
        "b2k_jph_wrap": (i64, [cp, vp, u64, vp, u64]),
        "b2k_jph_codestream": (i32, [vp, u64, pu64, pu64]),
        "b2k_stream_encode_begin": (i32, [i32, cp, u32, u32, _ENCODED_FN, vp, pp]),
        "b2k_stream_encode_submit": (i32, [vp, pp, pu32, vp]),
        "b2k_stream_decode_begin": (i32, [i32, u32, u32, _DECODED_FN, vp, pp]),
        "b2k_stream_decode_submit": (i32, [vp, cp, vp, u64, vp, u64, pp, pu32, vp]),
        "b2k_stream_decode_submit_codestream": (i32, [vp, vp, u64, u32, pp, pu32, vp]),
        "b2k_stream_end": (i32, [vp]),
        "b2k_launch_count": (u64, []),
        "b2k_job_last_kernel_stats": (i32, [vp, C.c_int, pf, pu64]),
    }


_SIGNATURES = _signatures()

# every symbol include/grok_b200.h declares
# plugin_decompress (C++-ABI callback struct) is declared in csrc/plugin_decode_abi.h, not in the C header
EXPORTS = [n for n in _SIGNATURES if n.startswith("b2k_")] + [
    "minpf_post_load_plugin", "plugin_init", "plugin_get_debug_state", "gpup_encode_mem", "gpup_tile_free",
    "gpup_encode_mem_tiles", "gpup_tiles_free", "plugin_decompress_codestream",
    "gpup_batch_memory_begin", "gpup_batch_memory_submit", "gpup_batch_memory_submit_planes", "gpup_batch_memory_end",
    "plugin_decompress", "plugin_batch_decompress_memory_begin", "plugin_batch_decompress_memory_end"]

_lib = None


def lib():
    """Load libgrokj2k_plugin.so (built in-tree by __graft_entry__.build / grok_b200/build.py), its functions declared."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(there is no CPU fallback for the engine)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in _SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
    _lib = L
    return L


class EngineError(RuntimeError):
    pass


class NotHandled(EngineError):
    pass


# message layouts: _RC for the calls that return 0 on success; _TEXT for those that return a size or a count, and for
# b2k_jph_codestream
_RC, _TEXT = "{what} -> {rc}: {text}", "{what}: {text}"


def _raise_for(rc, what, not_handled=False, msg=_RC, text=None):
    """Raise unless rc, what the b2k_* call `what` returned, is 0: NotHandled if rc is 1 and the call returns 1 for input
    it declines (not_handled), else EngineError.  The message is msg filled in with what, rc and text (by default
    b2k_last_error()'s)."""
    if rc != 0:
        text = (lib().b2k_last_error() or b"").decode() if text is None else text
        raise (NotHandled if not_handled and rc == 1 else EngineError)(msg.format(what=what, rc=rc, text=text))


def _size(call, what, not_handled=False):
    """call(None, 0): the size a b2k_* call(buffer, capacity) needs, in items (< 0 on failure; 1 for input it declines
    when not_handled)"""
    n = call(None, 0)
    if n < 0 or (not_handled and n == 1):
        _raise_for(n, what, not_handled, _TEXT)
    return n


def _size_then_fill(call, what, dtype=np.uint8, not_handled=False):
    """A new array of the size call(None, 0) asks for, filled by call(array, size)"""
    n = _size(call, what, not_handled)
    out = np.zeros(n, dtype)
    m = call(out.ctypes.data, n)
    if m != n:      # a failure, or 0 when the input changed between the calls
        _raise_for(m or -1, what, not_handled, _TEXT)
    return out


def make_coding(width, height, numcomps=1, prec=8, sgnd=False, numres=6, tile=None, cblk=(64, 64), irreversible=False,
                mct=None, numgbits=1, origin=(0, 0), tile_origin=None, precincts=None, qfactor=None):
    """Convenience constructor; defaults follow grk_compress for an HT (.jph) output:
    6 resolutions (CodeStream.h L43), 64x64 blocks (L40), one guard bit (GrkCompress.cpp L849).
    qfactor: 1..100, the band steps grk_compress --qfactor derives (needs irreversible=True)."""
    cp = Coding()
    cp.x0, cp.y0 = origin
    cp.x1, cp.y1 = origin[0] + width, origin[1] + height
    if tile:
        cp.tw, cp.th = tile
        cp.tx0, cp.ty0 = tile_origin if tile_origin else origin
    cp.numcomps, cp.prec, cp.sgnd, cp.numres = numcomps, prec, int(sgnd), numres
    cp.cblkw_exp, cp.cblkh_exp = int(np.log2(cblk[0])), int(np.log2(cblk[1]))
    cp.irreversible = int(irreversible)
    cp.mct = int(numcomps >= 3) if mct is None else int(mct)
    cp.numgbits = numgbits
    for r in range(33):
        cp.prcw_exp[r] = 15
        cp.prch_exp[r] = 15
    if precincts:  # [(w, h)] per resolution, coarsest first; the last entry repeats
        for r in range(numres):
            pw, ph = precincts[min(r, len(precincts) - 1)]
            cp.prcw_exp[r], cp.prch_exp[r] = int(np.log2(pw)), int(np.log2(ph))
    if qfactor is not None:
        cp.qfactor = qfactor
    return cp


def _plane_ptrs(planes):
    n = len(planes)
    arr = (C.c_void_p * n)(*[p.ctypes.data for p in planes])
    strides = (C.c_uint32 * n)(*[p.strides[0] // p.itemsize for p in planes])
    return arr, strides


# ------------------------------------------------------------------------------------------------
# images in device memory: anything with __cuda_array_interface__ (torch CUDA tensors, CuPy, ...)
# ------------------------------------------------------------------------------------------------
DEVICE_DTYPES = ("u1", "i1", "u2", "i2", "i4", "u4")


def _cuda_array(a):
    try:
        iface = a.__cuda_array_interface__
    except AttributeError:
        raise TypeError("%s has no __cuda_array_interface__: a CUDA array is needed (e.g. a torch tensor on a GPU)"
                        % type(a).__name__) from None
    t = iface["typestr"]
    if t[1:] not in DEVICE_DTYPES or (t[0] == ">" and t[2:] != "1"):
        raise ValueError("dtype %r is not one of the sample containers %s (little-endian)" % (t, ", ".join(DEVICE_DTYPES)))
    size = int(t[2:])
    shape = tuple(int(n) for n in iface["shape"])
    strides = iface.get("strides")
    if strides is None:  # C-contiguous
        strides, acc = [], size
        for n in reversed(shape):
            strides.insert(0, acc)
            acc *= n
    for s in strides:
        if s < 0:
            raise ValueError("negative strides %s are not supported" % (tuple(strides),))
        if s % size:
            raise ValueError("strides %s (bytes) are not whole %d-byte samples" % (tuple(strides), size))
    ptr, readonly = iface["data"]
    return dict(ptr=int(ptr or 0), shape=shape, steps=[s // size for s in strides], size=size, typestr=t[1:], readonly=bool(readonly))


def device_planes(image, numcomps, height, width, layout="CHW", writable=False):
    """b2k_device_planes for `image`: one array of shape (C, H, W) (layout "CHW") or (H, W, C) ("HWC"), an (H, W) array
    for one component, or a list of C arrays of shape (H, W).  Pointers, row pitches and column steps come from the
    arrays' __cuda_array_interface__ strides, so padded rows, slices of larger tensors and views such as t[..., :3] of
    an RGBA tensor need no copy.  Raises on a shape that is not (numcomps, height, width), a dtype that is not a
    sample container, or strides that are negative or not whole samples.  Returns the DevicePlanes."""
    if layout not in ("CHW", "HWC"):
        raise ValueError("layout must be 'CHW' or 'HWC', not %r" % (layout,))
    arrays = list(image) if isinstance(image, (list, tuple)) else [image]
    descs = [_cuda_array(a) for a in arrays]
    if len({d["typestr"] for d in descs}) != 1:
        raise ValueError("the components have different dtypes: %s" % [d["typestr"] for d in descs])
    if writable and any(d["readonly"] for d in descs):
        raise ValueError("the image is read-only")
    if numcomps > 4:
        raise ValueError("a device image holds at most 4 components, not %d" % numcomps)
    img = DevicePlanes()
    img.sample_bytes = descs[0]["size"]
    comps = []  # (address, row pitch, column step) per component, in samples
    if isinstance(image, (list, tuple)) or len(descs[0]["shape"]) == 2:
        want = [(height, width)] * numcomps
        got = [d["shape"] for d in descs]
        if got != want:
            raise ValueError("shape %s does not match the image: %d component(s) of %s"
                             % (got if len(got) > 1 else got[0], numcomps, (height, width)))
        comps = [(d["ptr"], d["steps"][0], d["steps"][1]) for d in descs]
    else:
        d = descs[0]
        want = (numcomps, height, width) if layout == "CHW" else (height, width, numcomps)
        if d["shape"] != want:
            raise ValueError("shape %s does not match the image: %s for layout %s" % (d["shape"], want, layout))
        cstep, rstep, xstep = (d["steps"][0], d["steps"][1], d["steps"][2]) if layout == "CHW" else \
            (d["steps"][2], d["steps"][0], d["steps"][1])
        comps = [(d["ptr"] + c * cstep * d["size"], rstep, xstep) for c in range(numcomps)]
    for c, (ptr, pitch, step) in enumerate(comps):
        if pitch >= 1 << 32 or step >= 1 << 32:
            raise ValueError("component %d: row pitch %d / column step %d samples do not fit 32 bits" % (c, pitch, step))
        img.comp[c], img.row_pitch[c], img.col_step[c] = ptr, pitch, step
    return img


class _DeviceBytes:
    """A CUDA array interface over n bytes of device memory the engine owns (torch.as_tensor makes a view of it)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="|u1", strides=None, data=(ptr, False), version=2)


def _stream_handle(stream, image):
    """cudaStream_t for `stream`: None = torch's current stream of a torch tensor's device, else the legacy default stream
    (as the CUDA Array Interface assumes); an int handle; or anything with .cuda_stream (torch / CuPy streams)."""
    if stream is None:
        torch = sys.modules.get("torch")
        first = image[0] if isinstance(image, (list, tuple)) else image
        if torch is not None and isinstance(first, torch.Tensor) and first.is_cuda:
            return torch.cuda.current_stream(first.device).cuda_stream or None
        return None
    if isinstance(stream, int):
        return stream or None
    return int(stream.cuda_stream) or None


def set_host_threads(n):
    """Host threads that narrow/widen int32 planes to 16-bit PCIe containers (0 = off, <0 = default)."""
    return int(lib().b2k_set_host_threads(int(n)))


def host_pack_last():
    """(encode, decode): 1 if the last int32 call went through 16-bit host packing, 0 direct, -1 none yet."""
    return int(lib().b2k_host_pack_last(0)), int(lib().b2k_host_pack_last(1))


CS_TLM, CS_PLT, CS_TPARTS_R, CS_SOP, CS_EPH = 1, 2, 4, 16, 32
LRCP, RLCP, RPCL, PCRL, CPRL = range(5)


def CS_PROG(n):
    return (n & 7) << 8


def codestream_write(cp, blocks, data, flags=CS_TLM | CS_PLT, num_tiles=None, out=None):
    """HTJ2K codestream (bytes, numpy uint8) from a coding, a full block table (BLOCK_DTYPE) and its byte arena
    -- an EncodeResult's .blocks / .bytes, or tables built elsewhere (tests build them with the oracle).
    out: optional uint8 buffer to write into (e.g. pinned); a view of the written part is returned."""
    blocks = np.ascontiguousarray(blocks, dtype=BLOCK_DTYPE)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    r = result_from_tables(blocks, data, int(blocks["tile"].max()) + 1 if num_tiles is None else num_tiles)

    def write(buf, cap):
        return lib().b2k_codestream_write(C.byref(cp), C.byref(r), flags, buf, cap)
    if out is not None:
        n = write(out.ctypes.data, out.size)
        if 0 <= n <= out.size:
            return out[:n]
    return _size_then_fill(write, "b2k_codestream_write")


def window_rect(cp, window, reduce):
    """(x0, y0, x1, y1): the pixels of `window` (x0, y0, x1, y1 on the full-resolution canvas; None for the whole image)
    at 1 / 2**reduce resolution on the canvas of cp, the virtual coding codestream_parse_window gives for them"""
    if window is None:
        return (cp.x0, cp.y0, cp.x1, cp.y1)
    sh = (1 << reduce) - 1
    x0, y0, x1, y1 = [(v + sh) >> reduce for v in window]
    return (max(x0, cp.x0), max(y0, cp.y0), min(x1, cp.x1), min(y1, cp.y1))


def codestream_parse_window(cs, window=None, reduce=0):
    """b2k_codestream_parse_window -> (virtual Coding, block table, rect): rect = (x0, y0, x1, y1) of the window's pixels
    at 1 / 2**reduce resolution on the virtual coding's canvas (the whole virtual image when window is None)."""
    cs = np.ascontiguousarray(cs, dtype=np.uint8)
    win = (C.c_uint32 * 4)(*window) if window is not None else None
    cp = Coding()

    def parse(blocks, cap):
        n = lib().b2k_codestream_parse_window(cs.ctypes.data, len(cs), win, reduce, C.byref(cp), blocks, cap)
        if n <= 1:
            _raise_for(n, "b2k_codestream_parse_window", msg="{what}: {rc} {text}")
        return n
    blocks = _size_then_fill(parse, "b2k_codestream_parse_window", BLOCK_DTYPE)
    return cp, blocks, window_rect(cp, window, reduce)


def codestream_parse(cs):
    """-> (Coding, block table with offsets into cs).  Raises NotHandled for codestreams outside the path's scope."""
    cs = np.ascontiguousarray(cs, dtype=np.uint8)
    cp = Coding()
    blocks = _size_then_fill(lambda blocks, cap: lib().b2k_codestream_parse(cs.ctypes.data, len(cs), C.byref(cp), blocks, cap),
                             "b2k_codestream_parse", BLOCK_DTYPE, not_handled=True)
    return cp, blocks


def result_from_tables(blocks, data, num_tiles):
    """A ctypes Result viewing a numpy block table + byte arena (keep both alive while it is in use)."""
    r = Result()
    r.num_blocks = len(blocks)
    r.blocks = C.cast(blocks.ctypes.data, C.POINTER(Block))
    r.bytes = C.cast(data.ctypes.data, C.POINTER(C.c_uint8))
    r.num_bytes = len(data)
    r.num_tiles = num_tiles
    return r


def codestream_write_tiles(cp, blocks, data, flags=CS_TLM | CS_PLT, tile_mod=1, tile_rem=0, out=None, tile_at=None, sizes_only=False):
    """A shard's tiles as finished tile parts (b2k_codestream_write_tiles) -> (bytes, per-tile lengths of the shard's tiles).
    sizes_only: just the lengths.  tile_at (uint64 offsets, one per tile of the shard): write each tile part at out[tile_at[k]:]
    (b2k_codestream_write_tiles_at) and return (out, None)."""
    blocks = np.ascontiguousarray(blocks, dtype=BLOCK_DTYPE)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    r = result_from_tables(blocks, data, 0)
    L = lib()
    g_nx = -(-(cp.x1 - cp.tx0) // cp.tw) if cp.tw else 1
    g_ny = -(-(cp.y1 - cp.ty0) // cp.th) if cp.th else 1
    nmine = len(range(tile_rem, g_nx * g_ny, tile_mod))
    lens = np.zeros(nmine, np.uint64)
    if tile_at is not None:
        ta = np.ascontiguousarray(tile_at, dtype=np.uint64)
        n = L.b2k_codestream_write_tiles_at(C.byref(cp), C.byref(r), flags, tile_mod, tile_rem, out.ctypes.data, out.size, ta.ctypes.data)
        if n < 0:
            _raise_for(n, "b2k_codestream_write_tiles_at", msg=_TEXT)
        return out, None

    def write(buf, cap):
        return L.b2k_codestream_write_tiles(C.byref(cp), C.byref(r), flags, tile_mod, tile_rem, buf, cap, lens.ctypes.data)
    n = _size(write, "b2k_codestream_write_tiles")
    if sizes_only:
        return None, lens
    if out is None or out.size < n:
        out = np.zeros(max(n, 1), np.uint8)
    assert write(out.ctypes.data, out.size) == n
    return out[:n], lens


def codestream_write_header(cp, flags, tile_bytes_all):
    """Main header (+ TLM) from the tile-part length of every tile (b2k_codestream_write_header)."""
    tb = np.ascontiguousarray(tile_bytes_all, dtype=np.uint64)
    return _size_then_fill(lambda buf, cap: lib().b2k_codestream_write_header(C.byref(cp), flags, tb.ctypes.data, len(tb), buf, cap),
                           "b2k_codestream_write_header")


def merge_shards(cp, shards):
    """shards: [(block table, byte arena)] of ranks 0..n-1 (rank r coded the tiles t % n == r) -> EncodeResult holding
    every tile in enumeration order (b2k_result_merge)."""
    keep = [(np.ascontiguousarray(b, dtype=BLOCK_DTYPE), np.ascontiguousarray(d, dtype=np.uint8)) for b, d in shards]
    rs = [result_from_tables(b, d, 0) for b, d in keep]
    arr = (C.POINTER(Result) * len(rs))(*[C.pointer(r) for r in rs])
    out = C.POINTER(Result)()
    _raise_for(lib().b2k_result_merge(C.byref(cp), arr, len(rs), C.byref(out)), "b2k_result_merge")
    return EncodeResult(out)


def jph_wrap(cp, cs):
    """codestream -> .jph file bytes (JP2 boxes, brand 'jph ')."""
    cs = np.ascontiguousarray(cs, dtype=np.uint8)
    return _size_then_fill(lambda buf, cap: lib().b2k_jph_wrap(C.byref(cp), cs.ctypes.data, len(cs), buf, cap), "b2k_jph_wrap")


def jph_codestream(data):
    """.jph / .jp2 file bytes (or a raw codestream) -> view of the contiguous codestream."""
    data = np.ascontiguousarray(data, dtype=np.uint8)
    off, n = C.c_uint64(), C.c_uint64()
    _raise_for(lib().b2k_jph_codestream(data.ctypes.data, len(data), C.byref(off), C.byref(n)), "b2k_jph_codestream", msg=_TEXT)
    return data[off.value:off.value + n.value]


def pinned_empty(shape, dtype):
    """numpy array in cudaHostAlloc'ed (pinned) memory; keep the returned array alive, free with
    ``lib().b2k_host_free(arr.ctypes.data)`` (or let the process end)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    p = lib().b2k_host_alloc(n)
    if not p:
        raise EngineError("b2k_host_alloc(%d) failed" % n)
    buf = (C.c_uint8 * n).from_address(p)
    return np.frombuffer(buf, dtype=dtype).reshape(shape)


class EncodeResult:
    """Owns a b2k_result; exposes numpy views of the block table and the byte arena."""

    def __init__(self, ptr):
        self._ptr = ptr
        r = ptr.contents
        self.num_blocks = int(r.num_blocks)
        self.num_bytes = int(r.num_bytes)
        self.num_tiles = int(r.num_tiles)
        self.timings = dict(h2d=r.ms_h2d, dwt=r.ms_dwt, t1=r.ms_t1, d2h=r.ms_d2h, total=r.ms_total)
        self.blocks = np.frombuffer((C.c_uint8 * (self.num_blocks * C.sizeof(Block))).from_address(
            C.addressof(r.blocks.contents)), dtype=BLOCK_DTYPE) if self.num_blocks else np.zeros(0, BLOCK_DTYPE)
        self.bytes = np.frombuffer((C.c_uint8 * max(1, self.num_bytes)).from_address(
            C.addressof(r.bytes.contents)), dtype=np.uint8)[:self.num_bytes]

    def block_bytes(self, i):
        b = self.blocks[i]
        return self.bytes[int(b["offset"]):int(b["offset"]) + int(b["length"])]

    def free(self):
        if self._ptr is not None:
            lib().b2k_result_free(self._ptr)
            self._ptr = None
            self.blocks = self.bytes = None

    def __del__(self):
        self.free()


class Engine:
    """b2k_engine: one per process per GPU (one process per GPU is the deployment model)."""

    def __init__(self, device=0):
        self._h = C.c_void_p()
        self.device = device
        _raise_for(lib().b2k_engine_create(device, C.byref(self._h)), "b2k_engine_create")

    def close(self):
        if self._h:
            lib().b2k_engine_destroy(self._h)
            self._h = C.c_void_p()

    def encode(self, cp, planes, tile_mod=1, tile_rem=0):
        """planes: list of 2-D int32 arrays (row stride may exceed width), or uint16 / int16 arrays
        (16-bit containers, b2k_encode16)."""
        ptrs, strides = _plane_ptrs(planes)
        out = C.POINTER(Result)()
        fn = "b2k_encode16" if planes[0].itemsize == 2 else "b2k_encode"
        _raise_for(getattr(lib(), fn)(self._h, C.byref(cp), ptrs, strides, tile_mod, tile_rem, C.byref(out)), fn)
        return EncodeResult(out)

    def encode_interleaved(self, cp, pixels, tile_mod=1, tile_rem=0):
        """pixels: one (H, W, numcomps) uint16 / int16 array (RGB48LE rows; the row stride may exceed W * numcomps
        samples): b2k_encode16_interleaved -- the rows cross PCIe as they are, planes are made on the device."""
        assert pixels.ndim == 3 and pixels.itemsize == 2 and pixels.strides[2] == 2 and pixels.strides[1] == 2 * pixels.shape[2]
        out = C.POINTER(Result)()
        _raise_for(lib().b2k_encode16_interleaved(self._h, C.byref(cp), pixels.ctypes.data, pixels.strides[0] // 2, tile_mod,
                                                  tile_rem, C.byref(out)), "b2k_encode16_interleaved")
        return EncodeResult(out)

    def encode_codestream(self, cp, planes, flags=CS_TLM | CS_PLT, out=None):
        """planes -> a complete HTJ2K codestream (numpy uint8): b2k_encode + b2k_codestream_write."""
        res = self.encode(cp, planes)
        try:
            return codestream_write(cp, res.blocks, res.bytes, flags, num_tiles=res.num_tiles, out=out)
        finally:
            res.free()

    def decode_codestream(self, cs, dtype=np.int32, out=None):
        """HTJ2K codestream -> (Coding, list of planes): b2k_codestream_parse + b2k_decode, block bytes read in place."""
        cs = np.ascontiguousarray(cs, dtype=np.uint8)
        cp, blocks = codestream_parse(cs)
        if out is None:
            out = [np.zeros((cp.y1 - cp.y0, cp.x1 - cp.x0), dtype) for _ in range(cp.numcomps)]
        self.decode(cp, blocks, cs, out)
        return cp, out

    def decode_window(self, cs, window=None, reduce=0, dtype=np.int32):
        """Tile-granular windowed / reduced-resolution decode of an HTJ2K codestream (b2k_codestream_parse_window +
        b2k_decode_window: the touched tiles are decoded, the window's pixels alone are copied back).  window = (x0, y0, x1, y1) on the full-resolution canvas or None; returns (virtual Coding,
        planes of the window at 1 / 2**reduce resolution).  The planes are views of pinned buffers the engine keeps and
        reuses for later windows of the same tile-box shape: copy them to keep them."""
        cs = np.ascontiguousarray(cs, dtype=np.uint8)
        cp, blocks, rect = codestream_parse_window(cs, window, reduce)
        # pinned landing planes of the WINDOW's size, kept per shape: only the window's pixels come back over PCIe
        cache = self.__dict__.setdefault("_win_planes", {})
        key = (rect[3] - rect[1], rect[2] - rect[0], cp.numcomps, np.dtype(dtype).str)
        out = cache.get(key)
        if out is None:
            if len(cache) >= 8:
                cache.pop(next(iter(cache)))
            out = cache[key] = [pinned_empty((key[0], key[1]), dtype) for _ in range(cp.numcomps)]
        ptrs, strides = _plane_ptrs(out)
        ms = C.c_double()
        _raise_for(lib().b2k_decode_window(self._h, C.byref(cp), blocks.ctypes.data, len(blocks), cs.ctypes.data, len(cs), ptrs,
                                           strides, (C.c_uint32 * 4)(*rect), np.dtype(dtype).itemsize, C.byref(ms)), "b2k_decode_window")
        return cp, out

    def decode(self, cp, blocks, data, out_planes, tile_mod=1, tile_rem=0):
        ptrs, strides = _plane_ptrs(out_planes)
        blocks = np.ascontiguousarray(blocks, dtype=BLOCK_DTYPE)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        ms = C.c_double()
        fn = "b2k_decode16" if out_planes[0].itemsize == 2 else "b2k_decode"
        _raise_for(getattr(lib(), fn)(self._h, C.byref(cp), blocks.ctypes.data, len(blocks), data.ctypes.data, len(data),
                                      ptrs, strides, tile_mod, tile_rem, C.byref(ms)), fn)
        return ms.value

    # ---- images in device memory (b2k_encode_device / b2k_decode_device) ----
    def encode_device(self, cp, image, layout="CHW", stream=None, tile_mod=1, tile_rem=0):
        """Encode an image that is already on the engine's GPU: any object (or list of per-component objects) with
        __cuda_array_interface__ -- see device_planes() for the shapes.  Samples are read where they are, ordered after
        the work queued on `stream` (None: torch's current stream for a torch tensor, else the legacy default stream);
        the result equals encode() of the same samples."""
        img = device_planes(image, cp.numcomps, cp.y1 - cp.y0, cp.x1 - cp.x0, layout)
        out = C.POINTER(Result)()
        _raise_for(lib().b2k_encode_device(self._h, C.byref(cp), C.byref(img), tile_mod, tile_rem, _stream_handle(stream, image),
                                           C.byref(out)), "b2k_encode_device", not_handled=True)
        return EncodeResult(out)

    def decode_device(self, cp, blocks, data, out, layout="CHW", window=None, stream=None, tile_mod=1, tile_rem=0):
        """Decode into `out` on the engine's GPU (shapes as for encode_device; a window (x0, y0, x1, y1) in cp's canvas
        coordinates makes `out` the window's pixels).  The block table and coded bytes stay in host memory.  Work queued
        on `stream` after the call sees the pixels.  Returns the device ms of the call."""
        if window is None:
            h, w = cp.y1 - cp.y0, cp.x1 - cp.x0
        else:
            h, w = window[3] - window[1], window[2] - window[0]
        img = device_planes(out, cp.numcomps, h, w, layout, writable=True)
        blocks = np.ascontiguousarray(blocks, dtype=BLOCK_DTYPE)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        win = (C.c_uint32 * 4)(*window) if window is not None else None
        ms = C.c_double()
        _raise_for(lib().b2k_decode_device(self._h, C.byref(cp), blocks.ctypes.data, len(blocks), data.ctypes.data, len(data),
                                           C.byref(img), win, tile_mod, tile_rem, _stream_handle(stream, out), C.byref(ms)),
                   "b2k_decode_device", not_handled=True)
        return ms.value

    def encode_codestream_device(self, cp, image, flags=CS_TLM | CS_PLT, layout="CHW", stream=None, device_output=False):
        """An image on the GPU -> a complete HTJ2K codestream (numpy uint8): b2k_encode_device + b2k_codestream_write.
        device_output=True: the code stream is written on the GPU (b2k_encode_codestream_device, the same bytes) and
        returned as a new torch.uint8 CUDA tensor, copied out of the engine's buffer on `stream`."""
        if device_output:
            return self._encode_codestream_on_device(cp, image, flags, layout, stream)
        res = self.encode_device(cp, image, layout=layout, stream=stream)
        try:
            return codestream_write(cp, res.blocks, res.bytes, flags, num_tiles=res.num_tiles)
        finally:
            res.free()

    def _encode_codestream_on_device(self, cp, image, flags, layout, stream):
        import torch
        img = device_planes(image, cp.numcomps, cp.y1 - cp.y0, cp.x1 - cp.x0, layout)
        handle = _stream_handle(stream, image)
        ptr = C.c_void_p()
        n = lib().b2k_encode_codestream_device(self._h, C.byref(cp), C.byref(img), flags, handle, C.byref(ptr))
        if n <= 1:
            _raise_for(n, "b2k_encode_codestream_device", not_handled=True)
        view = torch.as_tensor(_DeviceBytes(ptr.value, n), device="cuda:%d" % self.device)
        s = torch.cuda.ExternalStream(handle, device=self.device) if handle else torch.cuda.default_stream(self.device)
        with torch.cuda.stream(s):
            out = torch.empty(n, dtype=torch.uint8, device="cuda:%d" % self.device)
            out.copy_(view)
        return out

    def encode_codestreams_device(self, cp, images, flags=CS_TLM | CS_PLT, layout="CHW", stream=None):
        """A batch of images on the engine's GPU, all of coding cp -> (streams, status) in one launch chain
        (b2k_encode_codestreams_device).  images: one CUDA array (n, C, H, W) / (n, H, W, C) in `layout`, or a sequence of
        n CUDA arrays each as encode_device takes it (device_planes: views such as RGB of RGBA need no copy).  The streams
        are copied once, on `stream`, into one new torch.uint8 CUDA tensor: streams[i] is a view of it holding exactly
        the bytes encode_codestream_device(cp, images[i], flags, device_output=True) returns, or None where status[i] is
        not 0.  status[i] = (rc, text): what that single call returns (0, or the code it would raise with).  Raises only
        when the call fails as a whole."""
        import torch
        n = len(images)
        if n == 0:
            raise ValueError("encode_codestreams_device: no images")
        h, w, nc = cp.y1 - cp.y0, cp.x1 - cp.x0, cp.numcomps
        imgs = (DevicePlanes * n)(*[device_planes(images[i], nc, h, w, layout) for i in range(n)])
        handle = _stream_handle(stream, images)
        L = lib()
        ptr = C.c_void_p()
        off = (C.c_uint64 * n)()
        lens = (C.c_uint64 * n)()
        st = (C.c_int32 * n)()
        ms = C.c_double()
        rc = L.b2k_encode_codestreams_device(self._h, C.byref(cp), n, imgs, flags, handle, C.byref(ptr), off, lens, st, C.byref(ms))
        if rc < 0:
            _raise_for(rc, "b2k_encode_codestreams_device", msg=_TEXT)
        status = [(int(st[i]), (L.b2k_encode_codestreams_error(self._h, i) or b"").decode()) for i in range(n)]
        span = max([int(off[i]) + int(lens[i]) for i in range(n) if st[i] == 0] or [0])
        dev = "cuda:%d" % self.device
        s = torch.cuda.ExternalStream(handle, device=self.device) if handle else torch.cuda.default_stream(self.device)
        with torch.cuda.stream(s):
            out = torch.empty(span, dtype=torch.uint8, device=dev)
            if span:
                out.copy_(torch.as_tensor(_DeviceBytes(ptr.value, span), device=dev))
        streams = [out[int(off[i]):int(off[i]) + int(lens[i])] if st[i] == 0 else None for i in range(n)]
        return streams, status

    def decode_codestream_device(self, cs, out=None, dtype=None, layout="CHW", window=None, reduce=0, stream=None):
        """HTJ2K codestream -> (Coding, image on the GPU).  window (x0, y0, x1, y1 on the full-resolution canvas) and
        reduce work as in decode_window (the Coding is then the virtual one).  out: a CUDA array of the (window's) shape
        in `layout`, or None for a new torch tensor of `dtype` (default torch.uint16) on the engine's GPU.
        cs may itself be on the engine's GPU (a 1-D contiguous uint8 CUDA array): it is then parsed there
        (b2k_decode_codestream_device) and never crosses PCIe; window / reduce are not available on that path: a window
        of a code stream in device memory is decode_window_device."""
        if hasattr(cs, "__cuda_array_interface__"):
            if window is not None or reduce:
                raise NotHandled("decode_codestream_device: window / reduce of a code stream in device memory are "
                                 "decode_window_device's")
            return self._decode_device_codestream(cs, out, dtype, layout, stream)
        cs = np.ascontiguousarray(cs, dtype=np.uint8)
        if window is not None or reduce:
            cp, blocks, rect = codestream_parse_window(cs, window, reduce)
        else:
            (cp, blocks), rect = codestream_parse(cs), None
        x0, y0, x1, y1 = rect if rect is not None else (cp.x0, cp.y0, cp.x1, cp.y1)
        if out is None:
            import torch
            shape = (cp.numcomps, y1 - y0, x1 - x0) if layout == "CHW" else (y1 - y0, x1 - x0, cp.numcomps)
            out = torch.empty(shape, dtype=torch.uint16 if dtype is None else dtype, device="cuda:%d" % self.device)
        self.decode_device(cp, blocks, cs, out, layout=layout, window=rect, stream=stream)
        return cp, out

    def _device_codestream_bytes(self, cs):
        iface = cs.__cuda_array_interface__
        shape = tuple(int(n) for n in iface["shape"])
        if iface["typestr"][1:] != "u1" or len(shape) != 1:
            raise ValueError("a device code stream is a 1-D uint8 CUDA array, not %s of shape %s" % (iface["typestr"], shape))
        strides = iface.get("strides")
        if strides is not None and shape[0] > 1 and int(strides[0]) != 1:
            raise ValueError("a device code stream must be contiguous (strides %s)" % (tuple(strides),))
        return int(iface["data"][0] or 0), shape[0]

    def _parse_call(self, ptr, n, handle, cp):
        """b2k_codestream_parse_device of the n bytes at device address ptr into cp, as a call(blocks, capacity)"""
        return lambda blocks, cap: lib().b2k_codestream_parse_device(self._h, ptr, n, handle, C.byref(cp), blocks, cap)

    def codestream_parse_device(self, cs, stream=None):
        """b2k_codestream_parse_device: (Coding, block table) of a code stream on the engine's GPU, parsed there; the
        same as codestream_parse of its bytes."""
        ptr, n = self._device_codestream_bytes(cs)
        cp = Coding()
        blocks = _size_then_fill(self._parse_call(ptr, n, _stream_handle(stream, cs), cp), "b2k_codestream_parse_device",
                                 BLOCK_DTYPE, not_handled=True)
        return cp, blocks

    def codestream_parse_device_stats(self):
        """(tiles parsed packet by packet from PLT, tiles walked) of the last device parse on this engine"""
        ix, wk = C.c_uint32(), C.c_uint32()
        _raise_for(lib().b2k_codestream_parse_device_stats(self._h, C.byref(ix), C.byref(wk)), "b2k_codestream_parse_device_stats")
        return ix.value, wk.value

    def _window_parse_call(self, ptr, n, win, reduce, handle, cp):
        """b2k_codestream_parse_window_device of the n bytes at device address ptr into cp, as a call(blocks, capacity)"""
        return lambda blocks, cap: lib().b2k_codestream_parse_window_device(self._h, ptr, n, win, reduce, handle, C.byref(cp),
                                                                            blocks, cap)

    def codestream_parse_window_device(self, cs, window=None, reduce=0, stream=None):
        """b2k_codestream_parse_window_device -> (virtual Coding, block table, rect), as codestream_parse_window of the
        stream's bytes gives them, for a code stream on the engine's GPU (a 1-D uint8 CUDA array) parsed there.  Only the
        wanted tiles' tile-part headers and packets are read."""
        ptr, n = self._device_codestream_bytes(cs)
        win = (C.c_uint32 * 4)(*window) if window is not None else None
        cp = Coding()
        blocks = _size_then_fill(self._window_parse_call(ptr, n, win, reduce, _stream_handle(stream, cs), cp),
                                 "b2k_codestream_parse_window_device", BLOCK_DTYPE, not_handled=True)
        return cp, blocks, window_rect(cp, window, reduce)

    def decode_window_device(self, cs, window=None, reduce=0, out=None, dtype=None, layout="CHW", stream=None):
        """Windowed / reduced-resolution decode of a code stream on the engine's GPU (a 1-D uint8 CUDA array), into an
        image on the GPU: decode_codestream_device(host bytes, window=, reduce=) without the stream leaving the device.
        Only the tiles the window touches are parsed, copied and decoded.  out: a CUDA array of the window's shape at
        1 / 2**reduce in `layout`, or None for a new torch tensor of `dtype` (default torch.uint16).  Returns
        (virtual Coding, out)."""
        ptr, n = self._device_codestream_bytes(cs)
        handle = _stream_handle(stream, cs)
        win = (C.c_uint32 * 4)(*window) if window is not None else None
        cp = Coding()
        _size(self._window_parse_call(ptr, n, win, reduce, handle, cp), "b2k_codestream_parse_window_device",
              not_handled=True)   # the main header: the window's shape
        x0, y0, x1, y1 = window_rect(cp, window, reduce)
        h, w = y1 - y0, x1 - x0
        if out is None:
            import torch
            shape = (cp.numcomps, h, w) if layout == "CHW" else (h, w, cp.numcomps)
            out = torch.empty(shape, dtype=torch.uint16 if dtype is None else dtype, device="cuda:%d" % self.device)
        img = device_planes(out, cp.numcomps, h, w, layout, writable=True)
        rect = (C.c_uint32 * 4)()
        ms = C.c_double()
        _raise_for(lib().b2k_decode_codestream_window_device(self._h, ptr, n, win, reduce, C.byref(img), handle, C.byref(cp),
                                                             rect, C.byref(ms)), "b2k_decode_codestream_window_device",
                   not_handled=True)
        assert tuple(rect) == (x0, y0, x1, y1), (tuple(rect), (x0, y0, x1, y1))
        return cp, out

    def codestream_window_device_stats(self):
        """(wanted tiles, bytes copied into the engine's arena) of the last windowed device parse on this engine"""
        t, b = C.c_uint32(), C.c_uint64()
        _raise_for(lib().b2k_codestream_window_device_stats(self._h, C.byref(t), C.byref(b)), "b2k_codestream_window_device_stats")
        return t.value, b.value

    def _decode_device_codestream(self, cs, out, dtype, layout, stream):
        ptr, n = self._device_codestream_bytes(cs)
        handle = _stream_handle(stream, cs)
        cp = Coding()
        _size(self._parse_call(ptr, n, handle, cp), "b2k_codestream_parse_device", not_handled=True)   # the main header: the image's shape
        h, w = cp.y1 - cp.y0, cp.x1 - cp.x0
        if out is None:
            import torch
            shape = (cp.numcomps, h, w) if layout == "CHW" else (h, w, cp.numcomps)
            out = torch.empty(shape, dtype=torch.uint16 if dtype is None else dtype, device="cuda:%d" % self.device)
        img = device_planes(out, cp.numcomps, h, w, layout, writable=True)
        ms = C.c_double()
        _raise_for(lib().b2k_decode_codestream_device(self._h, ptr, n, C.byref(img), handle, C.byref(cp), C.byref(ms)),
                   "b2k_decode_codestream_device", not_handled=True)
        return cp, out

    def decode_codestreams_device(self, streams, out=None, dtype=None, layout="CHW", stream=None):
        """A batch of HTJ2K code streams on the engine's GPU (1-D contiguous uint8 CUDA arrays), all with one coding ->
        (Coding, out, status) in one launch chain (b2k_decode_codestreams_device).  out: None for a new torch tensor
        (n, C, H, W) or (n, H, W, C) of `dtype` (default torch.uint16), or a CUDA array of that shape.  status[i] =
        (rc, text) is what decode_codestream_device of stream i alone returns (0, or the code it would raise with);
        out[i] is written only where rc is 0.  Raises only when the call fails as a whole, or when no stream has a
        coding (with stream 0's error)."""
        n = len(streams)
        if n == 0:
            raise ValueError("decode_codestreams_device: no code streams")
        ptrs = (C.c_void_p * n)()
        lens = (C.c_uint64 * n)()
        for i, cs in enumerate(streams):
            if not hasattr(cs, "__cuda_array_interface__"):
                raise ValueError("decode_codestreams_device: stream %d is not a CUDA array" % i)
            ptrs[i], lens[i] = self._device_codestream_bytes(cs)
        L = lib()
        handle = _stream_handle(stream, out if out is not None else streams[0])
        cp = Coding()
        st = (C.c_int32 * n)()
        ms = C.c_double()

        def status():
            return [(int(st[i]), (L.b2k_decode_codestreams_error(self._h, i) or b"").decode()) for i in range(n)]

        # headers only: the batch's coding, which sizes the output -- and, when `out` is given, is checked against it before
        # anything is written: a b2k_device_planes has no extent, so an `out` of the wrong shape would otherwise be written
        # past its end
        rc = L.b2k_decode_codestreams_device(self._h, n, ptrs, lens, None, handle, C.byref(cp), st, C.byref(ms))
        if rc < 0:
            _raise_for(rc, "b2k_decode_codestreams_device", msg=_TEXT)
        if rc == n:
            code, text = status()[0]
            _raise_for(code, "b2k_decode_codestreams_device: stream 0", not_handled=True, msg=_TEXT, text=text)
        h, w, nc = cp.y1 - cp.y0, cp.x1 - cp.x0, cp.numcomps
        shape = (n, nc, h, w) if layout == "CHW" else (n, h, w, nc)
        if out is None:
            import torch
            out = torch.empty(shape, dtype=torch.uint16 if dtype is None else dtype, device="cuda:%d" % self.device)
        iface = out.__cuda_array_interface__
        if tuple(int(v) for v in iface["shape"]) != shape:
            raise ValueError("decode_codestreams_device: out has shape %s, the batch needs %s" % (tuple(iface["shape"]), shape))
        imgs = (DevicePlanes * n)(*[device_planes(out[i], nc, h, w, layout, writable=True) for i in range(n)])
        rc = L.b2k_decode_codestreams_device(self._h, n, ptrs, lens, imgs, handle, C.byref(cp), st, C.byref(ms))
        if rc < 0:
            _raise_for(rc, "b2k_decode_codestreams_device", msg=_TEXT)
        return cp, out, status()

    def decode_windows_device(self, streams, windows=None, reduce=0, out=None, dtype=None, layout="CHW", stream=None):
        """A batch of windows: HTJ2K code streams on the engine's GPU (1-D contiguous uint8 CUDA arrays), each with its
        window at 1 / 2**reduce -> (virtual Coding, out, rects, status) in one launch chain
        (b2k_decode_codestreams_window_device).  windows: None (every whole image), one (x0, y0, x1, y1) on the
        full-resolution canvas for every stream, or one per stream.  rects[i] is the window's pixels on the virtual
        canvas, as decode_window_device gives them.  out: None for new torch tensors of `dtype` (default torch.uint16) --
        one (n, C, h, w) / (n, h, w, C) tensor when the rects of the streams that pass their headers share one size, else a
        list of n tensors each of its rect's size -- or a CUDA array or list of n CUDA arrays of those shapes, checked
        before anything is written.  status[i] = (rc, text) is what decode_window_device of stream i alone returns (0,
        or the code it would raise with); out[i] is written only where rc is 0.  Raises only when the call fails as a
        whole, or when no stream has a coding (with stream 0's error)."""
        n = len(streams)
        if n == 0:
            raise ValueError("decode_windows_device: no code streams")
        ptrs = (C.c_void_p * n)()
        lens = (C.c_uint64 * n)()
        for i, cs in enumerate(streams):
            if not hasattr(cs, "__cuda_array_interface__"):
                raise ValueError("decode_windows_device: stream %d is not a CUDA array" % i)
            ptrs[i], lens[i] = self._device_codestream_bytes(cs)
        win = None
        if windows is not None:
            ws = [tuple(windows)] * n if len(windows) == 4 and all(np.isscalar(v) for v in windows) else [tuple(w) for w in windows]
            if len(ws) != n or any(len(w) != 4 for w in ws):
                raise ValueError("decode_windows_device: windows must be one (x0, y0, x1, y1) or one per stream")
            win = (C.c_uint32 * (4 * n))(*[int(v) for w in ws for v in w])
        L = lib()
        first_out = out[0] if isinstance(out, (list, tuple)) and out else out
        handle = _stream_handle(stream, first_out if first_out is not None else streams[0])
        cp = Coding()
        rects = (C.c_uint32 * (4 * n))()
        st = (C.c_int32 * n)()
        ms = C.c_double()

        def status():
            return [(int(st[i]), (L.b2k_decode_codestreams_error(self._h, i) or b"").decode()) for i in range(n)]

        # headers only: the virtual coding and every stream's rect, which size the outputs and check a given `out`
        rc = L.b2k_decode_codestreams_window_device(self._h, n, ptrs, lens, win, reduce, None, handle, C.byref(cp), rects, st,
                                                    C.byref(ms))
        if rc < 0:
            _raise_for(rc, "b2k_decode_codestreams_window_device", msg=_TEXT)
        if rc == n:
            code, text = status()[0]
            _raise_for(code, "b2k_decode_codestreams_window_device: stream 0", not_handled=True, msg=_TEXT, text=text)
        nc = cp.numcomps
        rect = [tuple(int(v) for v in rects[4 * i:4 * i + 4]) for i in range(n)]
        size = [(r[3] - r[1], r[2] - r[0]) for r in rect]
        sizes = {size[i] for i in range(n) if st[i] == 0}

        def shape(hw):
            return (nc,) + hw if layout == "CHW" else hw + (nc,)

        if out is None:
            import torch
            dev, dt = "cuda:%d" % self.device, torch.uint16 if dtype is None else dtype
            if len(sizes) == 1:
                out = torch.empty((n,) + shape(sizes.pop()), dtype=dt, device=dev)
            else:
                out = [torch.empty(shape(size[i]), dtype=dt, device=dev) for i in range(n)]
        if isinstance(out, (list, tuple)):
            if len(out) != n:
                raise ValueError("decode_windows_device: out holds %d images, the batch has %d" % (len(out), n))
            images = list(out)
            want = [shape(size[i]) for i in range(n)]
        else:
            if len(sizes) > 1:
                raise ValueError("decode_windows_device: the rects differ in size (%s): out must be a list" % sorted(sizes))
            full = tuple(int(v) for v in out.__cuda_array_interface__["shape"])
            if len(full) != 4 or full[0] != n or (sizes and full[1:] != shape(next(iter(sizes)))):
                raise ValueError("decode_windows_device: out has shape %s, the batch needs %s"
                                 % (full, (n,) + shape(next(iter(sizes))) if sizes else n))
            images = [out[i] for i in range(n)]
            want = [full[1:]] * n
        imgs = (DevicePlanes * n)()
        for i in range(n):
            got = tuple(int(v) for v in images[i].__cuda_array_interface__["shape"])
            if st[i] == 0:
                if got != want[i]:
                    raise ValueError("decode_windows_device: out[%d] has shape %s, its rect needs %s" % (i, got, want[i]))
                imgs[i] = device_planes(images[i], nc, size[i][0], size[i][1], layout, writable=True)
        sb = {imgs[i].sample_bytes for i in range(n) if st[i] == 0}
        for i in range(n):   # a stream that failed its headers is not written: its descriptor only carries the sample size
            if st[i] != 0:
                imgs[i].sample_bytes = min(sb) if sb else 2
        rc = L.b2k_decode_codestreams_window_device(self._h, n, ptrs, lens, win, reduce, imgs, handle, C.byref(cp), rects, st,
                                                    C.byref(ms))
        if rc < 0:
            _raise_for(rc, "b2k_decode_codestreams_window_device", msg=_TEXT)
        return cp, out, [tuple(int(v) for v in rects[4 * i:4 * i + 4]) for i in range(n)], status()

    def job(self, cp, tile_mod=1, tile_rem=0):
        return Job(self, cp, tile_mod, tile_rem)


class Job:
    """b2k_device_job: device-resident buffers + per-stage entry points (parity tests, bench `value`)."""

    def __init__(self, eng, cp, tile_mod=1, tile_rem=0):
        self._h = C.c_void_p()
        self.cp = cp
        _raise_for(lib().b2k_job_create(eng._h, C.byref(cp), tile_mod, tile_rem, C.byref(self._h)), "b2k_job_create")

    def close(self):
        if self._h:
            lib().b2k_job_destroy(self._h)
            self._h = C.c_void_p()

    def _planes(self, fn, planes):
        ptrs, strides = _plane_ptrs(planes)
        _raise_for(getattr(lib(), fn)(self._h, ptrs, strides), fn)

    def upload(self, planes):
        self._planes("b2k_job_upload", planes)

    def download(self, planes):
        self._planes("b2k_job_download", planes)

    def download_coeffs(self, planes):
        self._planes("b2k_job_download_coeffs", planes)

    def upload_coeffs(self, planes):
        self._planes("b2k_job_upload_coeffs", planes)

    def forward(self):
        ms = C.c_float()
        _raise_for(lib().b2k_job_forward(self._h, C.byref(ms)), "b2k_job_forward")
        return ms.value

    def inverse(self):
        ms = C.c_float()
        _raise_for(lib().b2k_job_inverse(self._h, C.byref(ms)), "b2k_job_inverse")
        return ms.value

    def t1_encode(self):
        ms, total = C.c_float(), C.c_uint64()
        _raise_for(lib().b2k_job_t1_encode(self._h, C.byref(ms), C.byref(total)), "b2k_job_t1_encode")
        return ms.value, total.value

    def t1_decode(self):
        ms = C.c_float()
        _raise_for(lib().b2k_job_t1_decode(self._h, C.byref(ms)), "b2k_job_t1_decode")
        return ms.value

    def t1_decode_blocks(self, blocks, data):
        """Block-decode a caller-supplied block table (BLOCK_DTYPE) + byte arena into the coefficient planes."""
        blocks = np.ascontiguousarray(blocks, dtype=BLOCK_DTYPE)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        ms = C.c_float()
        _raise_for(lib().b2k_job_t1_decode_blocks(self._h, blocks.ctypes.data, len(blocks), data.ctypes.data, len(data), C.byref(ms)),
                   "b2k_job_t1_decode_blocks")
        return ms.value

    # The round trips raise EngineError on return code 2 (the coded size of a 9/7 step outgrew the byte arena): the arena
    # has been grown, but the image planes then hold a partial decode's reconstruction, so upload() again before a retry.
    def roundtrip_n(self, steps):
        """`steps` round trips queued back to back, one synchronisation.  Returns (total ms, [fwd, enc, dec, inv] ms
        summed over the steps, level-1 DWT kernel ms summed, coded bytes)."""
        ms, st, l1, nb = C.c_float(), (C.c_float * 4)(), C.c_float(), C.c_uint64()
        _raise_for(lib().b2k_job_roundtrip_n(self._h, steps, C.byref(ms), st, C.byref(l1), C.byref(nb)), "b2k_job_roundtrip_n")
        return ms.value, [float(v) for v in st], l1.value, int(nb.value)

    def roundtrip_pipelined_n(self, steps, chunks=0, streams=0):
        """`steps` round trips with the block-coder stage pipelined over block ranges on side streams
        (b2k_job_roundtrip_pipelined_n).  Returns (total ms, [fwd, block coder, inv] ms summed, level-1 kernel ms summed, bytes)."""
        ms, st, l1, nb = C.c_float(), (C.c_float * 3)(), C.c_float(), C.c_uint64()
        _raise_for(lib().b2k_job_roundtrip_pipelined_n(self._h, steps, chunks, streams, C.byref(ms), st, C.byref(l1), C.byref(nb)),
                   "b2k_job_roundtrip_pipelined_n")
        return ms.value, [float(v) for v in st], l1.value, int(nb.value)

    def roundtrip(self):
        """forward -> block encode -> block decode -> inverse, device-resident, one synchronisation.
        Returns (total ms, [fwd, enc, dec, inv] ms, coded bytes)."""
        ms, st, nb = C.c_float(), (C.c_float * 4)(), C.c_uint64()
        _raise_for(lib().b2k_job_roundtrip(self._h, C.byref(ms), st, C.byref(nb)), "b2k_job_roundtrip")
        return ms.value, list(st), nb.value

    def fetch_result(self):
        out = C.POINTER(Result)()
        _raise_for(lib().b2k_job_fetch_result(self._h, C.byref(out)), "b2k_job_fetch_result")
        return EncodeResult(out)

    def num_blocks(self):
        return int(lib().b2k_job_num_blocks(self._h))

    def kernel_stats(self, which=0):
        ms, nb = C.c_float(), C.c_uint64()
        lib().b2k_job_last_kernel_stats(self._h, which, C.byref(ms), C.byref(nb))
        return ms.value, nb.value


def enumerate_blocks(cp, tile_mod=1, tile_rem=0):
    return _size_then_fill(lambda out, cap: lib().b2k_enumerate(C.byref(cp), tile_mod, tile_rem, out, cap), "b2k_enumerate",
                           BLOCK_DTYPE)


# ------------------------------------------------------------------------------------------------
# streaming (include/grok_b200.h "streaming", csrc/stream.cpp): `depth` frames in flight on one GPU
# ------------------------------------------------------------------------------------------------
class _Stream:
    """What EncodeStream and DecodeStream share: the frames in flight, each under a key (its frame_user) with its tag and
    what has to stay alive until its callback has run, and end()."""

    def __init__(self, on_done):
        self._tags = {}
        self._next = 1
        self._user_cb = on_done
        self._h = C.c_void_p()

    def _key(self, tag, *keep):
        key = self._next
        self._next += 1
        self._tags[key] = (tag,) + keep
        return C.c_void_p(key)

    def _tag(self, frame_user):
        return self._tags.pop(int(frame_user or 0), (None,))[0]

    def end(self):
        if self._h:
            rc = lib().b2k_stream_end(self._h)
            self._h = C.c_void_p()
            return rc
        return 0


class EncodeStream(_Stream):
    """b2k_stream_encode_*: submit(planes, tag) hands a frame to an idle worker (blocks while `depth` frames are in
    flight); on_encoded(tag, EncodeResult or None, status) runs on a worker thread -- the EncodeResult is the caller's
    (free it).  The planes must stay alive and unchanged until the callback for their frame has run."""

    def __init__(self, cp, depth=3, sample_bytes=4, on_encoded=None, device=0):
        super().__init__(on_encoded)
        self._cp = cp

        def cb(_user, frame_user, result, status):
            tag = self._tag(frame_user)
            res = EncodeResult(result) if (status == 0 and result) else None
            if self._user_cb:
                self._user_cb(tag, res, status)
            elif res is not None:
                res.free()
            return 1 if res is not None else 0      # the EncodeResult owns the b2k_result now

        self._cb = _ENCODED_FN(cb)
        _raise_for(lib().b2k_stream_encode_begin(device, C.byref(cp), depth, sample_bytes, self._cb, None, C.byref(self._h)),
                   "b2k_stream_encode_begin")

    def submit(self, planes, tag=None):
        ptrs, strides = _plane_ptrs(planes)
        key = self._key(tag, planes)                 # keeps the planes alive until the callback
        _raise_for(lib().b2k_stream_encode_submit(self._h, ptrs, strides, key), "b2k_stream_encode_submit")


class DecodeStream(_Stream):
    """b2k_stream_decode_*: submit(cp, blocks, data, out_planes, tag) / submit_codestream(cs, out_planes, tag);
    on_decoded(tag, status) runs on a worker thread once out_planes hold the pixels."""

    def __init__(self, depth=3, sample_bytes=4, on_decoded=None, device=0):
        super().__init__(on_decoded)

        def cb(_user, frame_user, status):
            tag = self._tag(frame_user)
            if self._user_cb:
                self._user_cb(tag, status)

        self._cb = _DECODED_FN(cb)
        _raise_for(lib().b2k_stream_decode_begin(device, depth, sample_bytes, self._cb, None, C.byref(self._h)),
                   "b2k_stream_decode_begin")

    def submit(self, cp, blocks, data, out_planes, tag=None):
        ptrs, strides = _plane_ptrs(out_planes)
        blocks = np.ascontiguousarray(blocks, dtype=BLOCK_DTYPE)
        data = np.ascontiguousarray(data, dtype=np.uint8)
        key = self._key(tag, blocks, data, out_planes, cp)
        _raise_for(lib().b2k_stream_decode_submit(self._h, C.byref(cp), blocks.ctypes.data, len(blocks), data.ctypes.data, len(data),
                                                  ptrs, strides, key), "b2k_stream_decode_submit")

    def submit_codestream(self, cs, out_planes, tag=None):
        ptrs, strides = _plane_ptrs(out_planes)
        cs = np.ascontiguousarray(cs, dtype=np.uint8)
        key = self._key(tag, cs, out_planes)
        _raise_for(lib().b2k_stream_decode_submit_codestream(self._h, cs.ctypes.data, len(cs), len(out_planes), ptrs, strides, key),
                   "b2k_stream_decode_submit_codestream")
