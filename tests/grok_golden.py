"""What the reference gives for the cases the interop and oracle tests compare with it, kept in tests/golden/:
grok_outputs.json holds SHA-256 digests of its outputs (and, per code stream, the COM marker segment Grok writes),
grok_samples.npz holds seeded samples of the outputs a test compares with a tolerance.

Every comparison takes the reference's output as a callable, or None where the reference is not built
(oracle/build_ref.sh, `make -C oracle ref`).  With it, the test compares with the reference live and checks the
record against it; without it, the test compares with the record.  B2K_RECORD_GOLDEN=<dir> writes the record of
the cases a run visits to <dir>/grok_outputs.json and <dir>/grok_samples.npz instead of checking it."""
import atexit
import hashlib
import json
import os
import zlib

import numpy as np

import grok_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
RECORD = os.environ.get("B2K_RECORD_GOLDEN")
SAMPLES = 2048      # per array, for comparisons with a tolerance

_json = os.path.join(GOLD, "grok_outputs.json")
_npz = os.path.join(GOLD, "grok_samples.npz")
_outputs = json.load(open(_json)) if os.path.exists(_json) else {}
_samples = dict(np.load(_npz)) if os.path.exists(_npz) else {}
_rec_outputs, _rec_samples = {}, {}


def _write_record():
    os.makedirs(RECORD, exist_ok=True)
    with open(os.path.join(RECORD, "grok_outputs.json"), "w") as f:
        json.dump(_rec_outputs, f, indent=0, sort_keys=True)
    np.savez_compressed(os.path.join(RECORD, "grok_samples.npz"), **_rec_samples)


if RECORD:
    atexit.register(_write_record)


def grok(fn):
    """fn where the reference library is built, else None"""
    return fn if R.available() else None


def key(name, args, seed=None):
    return "%s %s seed=%s" % (name, json.dumps(args, sort_keys=True), seed)


def digest(arrays):
    """SHA-256 of the values and shapes of integer arrays (independent of their dtype)"""
    h = hashlib.sha256()
    for a in arrays:
        a = np.asarray(a)
        h.update(repr(a.shape).encode())
        h.update(np.ascontiguousarray(a, dtype=np.int64).tobytes())
    return h.hexdigest()


def _stored(k, live_value):
    """The record for k, checked against (or recorded from) live_value when there is one."""
    if RECORD:
        assert live_value is not None, "recording needs the reference"
        _rec_outputs[k] = live_value
        return live_value
    assert k in _outputs, "no record of the reference's output for %r" % k
    if live_value is not None:
        assert live_value == _outputs[k], "the stored record of %r differs from the reference" % k
    return _outputs[k]


def _com_segment(cs):
    """(offset, bytes) of the one COM (0xFF64) marker segment in the main header of cs"""
    cs = bytes(cs)
    i, found = 2, []
    while i + 4 <= len(cs):
        m = (cs[i] << 8) | cs[i + 1]
        if m == 0xFF90:
            break
        ln = (cs[i + 2] << 8) | cs[i + 3]
        if m == 0xFF64:
            found.append((i, bytes(cs[i:i + 2 + ln])))
        i += 2 + ln
    assert len(found) == 1, found
    return found[0]


def grok_stream(k, ours, compress):
    """Grok's code stream for case k as np.uint8.  Live, `compress()` makes it.  From the record, it is `ours` with
    Grok's COM segment put back, which holds only when ours is Grok's stream byte for byte apart from that segment."""
    if compress is not None:
        theirs = np.frombuffer(bytes(compress()), np.uint8)
        at, com = _com_segment(theirs)
        if ours is not None:
            assert bytes(ours) == theirs[:at].tobytes() + theirs[at + len(com):].tobytes(), "%s: code stream differs from Grok's (COM aside)" % k
        _stored(k, {"sha256": hashlib.sha256(theirs.tobytes()).hexdigest(), "com_at": at, "com": com.hex()})
        return theirs
    rec = _stored(k, None)
    ours = bytes(ours)
    at = rec["com_at"]
    theirs = np.frombuffer(ours[:at] + bytes.fromhex(rec["com"]) + ours[at:], np.uint8)
    assert hashlib.sha256(theirs.tobytes()).hexdigest() == rec["sha256"], "%s: code stream differs from Grok's (COM aside)" % k
    return theirs


def same(k, ours, theirs_fn):
    """ours (a list of integer arrays) equals what the reference gives, element for element"""
    theirs = theirs_fn() if theirs_fn is not None else None
    if theirs is not None:
        assert len(ours) == len(theirs)
        for i, (a, b) in enumerate(zip(ours, theirs)):
            assert np.shape(a) == np.shape(b) and np.array_equal(a, b), "%s: array %d differs from the reference" % (k, i)
    want = _stored(k, digest(theirs) if theirs is not None else None)
    assert digest(ours) == want, "%s: differs from the reference" % k


def close(k, ours, theirs_fn, tol):
    """ours (a list of integer arrays) is within tol of what the reference gives: everywhere when it is live, at a seeded
    sample of positions against the record"""
    theirs = theirs_fn() if theirs_fn is not None else None
    for i, a in enumerate(ours):
        a = np.asarray(a)
        rng = np.random.default_rng(zlib.crc32(("%s/%d" % (k, i)).encode()))
        idx = rng.integers(0, a.size, min(SAMPLES, a.size))
        name = "%08x_%d" % (zlib.crc32(k.encode()), i)
        if theirs is not None:
            b = np.asarray(theirs[i])
            assert a.shape == b.shape and np.abs(a.astype(np.int64) - b).max() <= tol, "%s: array %d" % (k, i)
            live = b.reshape(-1)[idx].astype(np.int32)
            if RECORD:
                _rec_samples[name] = live
                continue
            assert np.array_equal(live, _samples[name]), "the stored sample of %r differs from the reference" % k
        else:
            assert name in _samples, "no record of the reference's output for %r" % k
        assert np.abs(a.reshape(-1)[idx].astype(np.int64) - _samples[name]).max() <= tol, "%s: array %d" % (k, i)
