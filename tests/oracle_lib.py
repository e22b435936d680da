"""ctypes bindings for oracle/libj2k_oracle.so (the C restatement) and, when present,
oracle/_ref/libgrok_ref.so (the reference's own kernels).  TEST INFRASTRUCTURE ONLY:
imported by tests/, __graft_entry__.smoke() and bench.py's CPU legs, never by grok_b200/."""
import ctypes as C
import os
import subprocess
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C")
_u32p = np.ctypeslib.ndpointer(np.uint32, flags="C")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C")
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C")


def build_oracle():
    subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "libj2k_oracle.so"])
    if os.path.isdir("/root/reference/src/lib/core"):
        subprocess.check_call(["make", "-s", "-C", ORACLE_DIR, "ref"])


class Block(C.Structure):
    _fields_ = [("resno", C.c_uint8), ("orient", C.c_uint8), ("band_index", C.c_uint8),
                ("precno", C.c_uint32), ("cblkno", C.c_uint32),
                ("x0", C.c_uint32), ("y0", C.c_uint32), ("x1", C.c_uint32), ("y1", C.c_uint32),
                ("buf_x", C.c_uint32), ("buf_y", C.c_uint32)]


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        path = os.path.join(ORACLE_DIR, "libj2k_oracle.so")
        if not os.path.exists(path):
            build_oracle()
        L = C.CDLL(path)
        L.orc_rct_fwd.argtypes = [_i32p, _i32p, _i32p, C.c_size_t, _i32p]
        L.orc_rct_inv.argtypes = [_i32p, _i32p, _i32p, C.c_size_t, _i32p, _i32p, _i32p]
        L.orc_ict_fwd.argtypes = [_i32p, _i32p, _i32p, _f32p, _f32p, _f32p, C.c_size_t, _i32p]
        L.orc_ict_inv.argtypes = [_f32p, _f32p, _f32p, _i32p, _i32p, _i32p, C.c_size_t, _i32p, _i32p, _i32p]
        for n, t in (("dwt53", _i32p), ("dwt97", _f32p)):
            for d in ("fwd", "inv"):
                getattr(L, "orc_%s_%s_2d" % (n, d)).argtypes = [t, C.c_uint32] + [C.c_uint32] * 4 + [C.c_int]
        L.orc_fwd53_line.argtypes = [_i32p, C.c_int, C.c_int]
        L.orc_inv53_line.argtypes = [_i32p, C.c_int, C.c_int]
        L.orc_fwd97_line.argtypes = [_f32p, C.c_int, C.c_int]
        L.orc_inv97_line.argtypes = [_f32p, C.c_int, C.c_int]
        L.orc_ht_stepsizes.argtypes = [C.c_int] * 5 + [_u8p, np.ctypeslib.ndpointer(np.uint16, flags="C")]
        L.orc_band_stepsize.argtypes = [C.c_int] * 6
        L.orc_band_stepsize.restype = C.c_float
        L.orc_band_kmax.argtypes = [C.c_int] * 3
        L.orc_enumerate_blocks.argtypes = [C.c_uint32] * 4 + [C.c_int] * 3 + [C.c_void_p, C.c_void_p,
                                                                              C.POINTER(Block), C.c_int]
        L.orc_ht_pre_rev.argtypes = [_i32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _u32p]
        L.orc_ht_pre_irrev.argtypes = [_f32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float, _u32p]
        L.orc_ht_post_rev.argtypes = [_u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _i32p, C.c_uint32]
        L.orc_ht_post_irrev.argtypes = [_u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_float,
                                        _f32p, C.c_uint32]
        L.orc_ht_encode.argtypes = [_u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _u8p, C.c_uint32]
        L.orc_ht_decode.argtypes = [_u8p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _u32p]
        L.orc_ht_enc_table.restype = C.POINTER(C.c_uint16)
        L.orc_ht_dec_table.restype = C.POINTER(C.c_uint16)
        _lib = L
    return _lib


def ref():
    """The reference's own kernels, or None when oracle/_ref was not (pre)built."""
    global _ref
    if _ref is None:
        path = os.path.join(ORACLE_DIR, "_ref", "libgrok_ref.so")
        if not os.path.exists(path):
            return None
        R = C.CDLL(path)
        R.ref_ht_encode.argtypes = [C.c_int, _u32p, C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, _u8p, C.c_uint32]
        R.ref_ht_decode.argtypes = [C.c_int, C.c_void_p, _u32p] + [C.c_uint32] * 7
        R.ref_dwt53_fwd_2d.argtypes = [_i32p, C.c_uint32] + [C.c_uint32] * 4 + [C.c_int, C.c_int32]
        R.ref_dwt97_fwd_2d.argtypes = [_f32p, C.c_uint32] + [C.c_uint32] * 4 + [C.c_int, C.c_float, C.c_int]
        _ref = R
    return _ref


# ---- convenience wrappers -------------------------------------------------------------------
def ht_encode(sgnmag, missing_msbs, cap=24576):
    """sgnmag: (h, w) uint32 sign-magnitude words.  Returns the coded bytes."""
    a = np.ascontiguousarray(sgnmag, dtype=np.uint32)
    h, w = a.shape
    out = np.zeros(cap, np.uint8)
    n = lib().orc_ht_encode(a, missing_msbs, w, h, w, out, cap)
    assert n >= 0, "oracle encoder overflow"
    return out[:n].copy()


# the encoder choices of orc_ht_encode_foreign (ORC_FOREIGN_* in oracle/j2k_oracle.c)
FOREIGN_ROWS, FOREIGN_RAISE_U, FOREIGN_NO_FUSE, FOREIGN_PAD_MAGSGN, FOREIGN_PAD_SCUP = 1, 2, 4, 8, 16
FOREIGN_ALL = 31


def ht_encode_foreign(sgnmag, missing_msbs, choices, seed, cap=24576, stats=False):
    """The cleanup pass as another encoder may write it: the choices set in `choices`, picked by an LCG seeded with
    `seed` (choices = 0: ht_encode's bytes).  stats=True also returns the encoder's counts of the choices made:
    (quads with U_q at the decoder's limit, u_off = 1 quads whose e_k the max-popcount rule would not pick, raises
    dropped for want of a row, MEL bytes)."""
    a = np.ascontiguousarray(sgnmag, dtype=np.uint32)
    h, w = a.shape
    out = np.zeros(cap, np.uint8)
    L = lib()
    L.orc_ht_encode_foreign.argtypes = [_u32p] + [C.c_uint32] * 5 + [C.c_uint64, _u8p, C.c_uint32]
    n = L.orc_ht_encode_foreign(a, missing_msbs, w, h, w, choices, seed, out, cap)
    assert n >= 0, "oracle encoder overflow"
    if not stats:
        return out[:n].copy()
    s = np.zeros(4, np.int32)
    L.orc_ht_encode_foreign_stats.argtypes = [_i32p]
    L.orc_ht_encode_foreign_stats(s)
    return out[:n].copy(), tuple(int(v) for v in s)


def ht_decode(data, missing_msbs, w, h):
    d = np.concatenate([np.asarray(data, np.uint8), np.zeros(8, np.uint8)])
    out = np.zeros((h, w), np.uint32)
    rc = lib().orc_ht_decode(d, len(data), missing_msbs, w, h, w, out)
    return rc, out


def ht_encode_refine(sgnmag, missing_msbs, num_passes, causal=False, cap=8192):
    """SigProp (+ MagRef) segment for a block whose cleanup pass was coded with the same missing_msbs."""
    a = np.ascontiguousarray(sgnmag, dtype=np.uint32)
    h, w = a.shape
    out = np.zeros(cap, np.uint8)
    L = lib()
    L.orc_ht_encode_refine.argtypes = [_u32p] + [C.c_uint32] * 5 + [C.c_int, _u8p, C.c_uint32]
    n = L.orc_ht_encode_refine(a, missing_msbs, num_passes, w, h, w, int(causal), out, cap)
    assert n >= 0, "oracle refinement encoder overflow"
    return out[:n].copy()


def ht_decode_passes(data, len2, num_passes, missing_msbs, w, h, causal=False):
    """cleanup + refinement segments (len2 = bytes of the latter) -> sign-magnitude words."""
    d = np.concatenate([np.asarray(data, np.uint8), np.zeros(8, np.uint8)])
    out = np.zeros((h, w), np.uint32)
    L = lib()
    L.orc_ht_decode_passes.argtypes = [_u8p] + [C.c_uint32] * 7 + [C.c_int, _u32p]
    rc = L.orc_ht_decode_passes(d, len(data) - len2, len2, num_passes, missing_msbs, w, h, w, int(causal), out)
    return rc, out


def ref_ht_encode(sgnmag, missing_msbs, variant=-1, cap=24576):
    a = np.ascontiguousarray(sgnmag, dtype=np.uint32)
    h, w = a.shape
    # the SIMD encoders read whole vectors: give them slack after the block
    pad = np.zeros(a.size + 64, np.uint32)
    pad[:a.size] = a.ravel()
    out = np.zeros(cap, np.uint8)
    n = ref().ref_ht_encode(variant, pad, missing_msbs, w, h, w, out, cap)
    if n == -2:
        return None
    assert n >= 0
    return out[:n].copy()


def ref_ht_decode(data, missing_msbs, w, h, variant=-1, num_passes=1, len2=0, causal=False):
    stride = (w + 7) & ~7
    buf = np.zeros(len(data) + 64, np.uint8)
    buf[16:16 + len(data)] = data
    out = np.zeros((h + 2, stride), np.uint32)
    R = ref()
    R.ref_ht_decode_vsc.argtypes = [C.c_int, C.c_void_p, _u32p] + [C.c_uint32] * 7 + [C.c_int]
    rc = R.ref_ht_decode_vsc(variant, buf.ctypes.data + 16, out, missing_msbs, num_passes,
                             len(data) - len2, len2, w, h, stride, int(causal))
    return rc, out[:h, :w].copy()


def to_sgnmag(coef, kmax):
    """CoderOJPH.cpp L121-185 (reversible): int32 coefficient -> sign | mag << (30-kmax)."""
    c = np.asarray(coef, np.int64)
    mag = np.abs(c).astype(np.uint64) << np.uint64(30 - kmax)
    return ((c < 0).astype(np.uint64) << np.uint64(31) | mag).astype(np.uint32)


def enumerate_blocks(tc, numres, cbw_exp=6, cbh_exp=6, prcw_exp=None, prch_exp=None):
    pw = (C.c_uint8 * 33)(*prcw_exp) if prcw_exp is not None else None
    ph = (C.c_uint8 * 33)(*prch_exp) if prch_exp is not None else None
    cap = 256                          # orc_enumerate_blocks returns the whole count: grow and enumerate again
    while True:
        arr = (Block * cap)()
        n = lib().orc_enumerate_blocks(tc[0], tc[1], tc[2], tc[3], numres, cbw_exp, cbh_exp, pw, ph, arr, cap)
        if n <= cap:
            return [arr[i] for i in range(n)]
        cap = n


def aligned_zeros(shape, dtype, align=64):
    """numpy array whose data pointer is `align`-byte aligned (the reference's SIMD kernels use
    aligned vector loads on tile buffers, which Grok allocates with grk_aligned_malloc)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) * dtype.itemsize
    raw = np.zeros(n + align, np.uint8)
    off = (-raw.ctypes.data) % align
    return raw[off:off + n].view(dtype).reshape(shape)
