"""TEST INFRASTRUCTURE: a structural validator for the HTJ2K code streams this repo writes, independent of the writers
and of tests/oracle_t2.py.  validate(cs) walks the stream marker by marker and raises Invalid at the first rule broken:

  main header  SOC, SIZ, CAP, COD, QCD in that order (Lsiz = 38 + 3 Csiz), then any TLM segments, then the first SOT
  TLM          Ztlm = 0, 1, ...; Ltlm holds a whole number of entries; the entries are the (Isot, Psot) of the tile parts
               in stream order (T.800 A.7.1)
  SOT          Lsot = 10; Psot lands on the next SOT or on EOC; TPsot counts 0 .. TNsot - 1 within each tile, and every
               tile has TNsot parts (A.4.2)
  PLT          Zplt = 0, 1, ... within each tile part; Lplt agrees with its bytes; no entry runs over the end of its
               segment; the decoded lengths add up to the bytes after SOD (A.7.3)
  SOP          FF91 0004 Nsop at every packet start the PLT lengths predict, Nsop = the packet's index in its tile mod 65536
               (A.8.1); without PLT the SOP markers themselves mark the packets
  EPH          exactly one FF92 in every packet (A.8.2)
  in-body      no other two-byte value above 0xFF8F after SOD: packet headers stuff a 0 bit after 0xFF, and code-block
               bytes never form one (T.800 A.1, T.814 Annex B)
  EOC          last, and nothing after it

Everything per packet is done with numpy, so streams of 10^5 packets take well under a second."""
import numpy as np


class Invalid(ValueError):
    pass


def _check(cond, msg, *args):
    if not cond:
        raise Invalid(msg % args if args else msg)


def _u16(b, p):
    return (b[p] << 8) | b[p + 1]


def _u32(b, p):
    return (b[p] << 24) | (b[p + 1] << 16) | (b[p + 2] << 8) | b[p + 3]


def plt_lengths(iplt):
    """the packet lengths of one PLT segment's Iplt bytes (7 bits per byte, MSB = more to come)"""
    a = np.frombuffer(bytes(iplt), np.uint8)
    if not len(a):
        return np.zeros(0, np.int64)
    _check(a[-1] < 0x80, "PLT: the last entry runs over the end of its segment")
    ends = np.flatnonzero(a < 0x80)
    entry = np.concatenate([[0], np.cumsum(a < 0x80)[:-1]])
    shift = 7 * (ends[entry] - np.arange(len(a)))
    _check(shift.max() < 63, "PLT: an entry longer than 9 bytes")
    return np.add.reduceat((a.astype(np.int64) & 0x7F) << shift, np.concatenate([[0], ends[:-1] + 1]))


def validate(cs):
    """-> dict(sop, eph, tlm=[entries per TLM segment], parts=[dict(tile, index, count, psot, plt=[Iplt bytes per
    segment], packets=[lengths] or None, first_packet)]); raises Invalid"""
    b = bytes(cs)
    n = len(b)
    _check(b[:2] == b"\xff\x4f", "no SOC")
    p = 2
    seen = []
    for m in (0x51, 0x50, 0x52, 0x5C):
        _check(p + 4 <= n and b[p] == 0xFF and b[p + 1] == m, "main header: FF%02X expected at %d after %s", m, p, seen)
        L = _u16(b, p + 2)
        if m == 0x51:
            _check(L == 38 + 3 * _u16(b, p + 38), "SIZ: Lsiz %d for %d components", L, _u16(b, p + 38))
        if m == 0x52:
            scod = b[p + 4]
        seen.append("FF%02X" % m)
        p += 2 + L
    sop, eph = bool(scod & 2), bool(scod & 4)
    tlm = []                                       # [(tile or None, length)] per segment
    while p + 2 <= n and b[p:p + 2] == b"\xff\x55":
        L = _u16(b, p + 2)
        z, s = b[p + 4], b[p + 5]
        _check(z == len(tlm), "TLM: Ztlm %d where %d was due", z, len(tlm))
        st, sp = (s >> 4) & 3, (s >> 6) & 1
        _check(st != 3, "TLM: ST = 3")
        es = st + (4 if sp else 2)
        _check(L >= 4 and (L - 4) % es == 0, "TLM %d: Ltlm %d is not 4 + a whole number of %d-byte entries", z, L, es)
        ent = []
        for q in range(p + 6, p + 2 + L, es):
            t = (_u16(b, q) if st == 2 else b[q]) if st else None
            ent.append((t, _u32(b, q + st) if sp else _u16(b, q + st)))
        tlm.append(ent)
        p += 2 + L
    _check(b[p:p + 2] == b"\xff\x90", "main header: FF%02X%02X where SOT (or TLM) was due at %d", b[p], b[p + 1], p)
    parts, next_part, count, next_packet = [], {}, {}, {}
    arr = np.frombuffer(b, np.uint8)
    while p + 2 <= n and b[p:p + 2] == b"\xff\x90":
        _check(_u16(b, p + 2) == 10, "SOT at %d: Lsot %d", p, _u16(b, p + 2))
        tile, psot, tp, tn = _u16(b, p + 4), _u32(b, p + 6), b[p + 10], b[p + 11]
        end = p + psot
        _check(psot >= 14 and end + 2 <= n and b[end:end + 2] in (b"\xff\x90", b"\xff\xd9"),
               "SOT at %d: Psot %d does not land on SOT or EOC", p, psot)
        _check(tp == next_part.get(tile, 0), "tile %d: TPsot %d where %d was due", tile, tp, next_part.get(tile, 0))
        _check(count.setdefault(tile, tn) == tn and tp < tn, "tile %d: TNsot %d (part %d)", tile, tn, tp)
        next_part[tile] = tp + 1
        q, plt, lens = p + 12, [], []
        while b[q:q + 2] != b"\xff\x93":
            _check(q + 4 <= end, "tile part at %d: no SOD", p)
            _check(b[q:q + 2] == b"\xff\x58", "tile part at %d: FF%02X%02X in its header", p, b[q], b[q + 1])
            L = _u16(b, q + 2)
            _check(L >= 3 and q + 2 + L <= end, "PLT at %d: Lplt %d", q, L)
            _check(b[q + 4] == len(plt), "tile part at %d: Zplt %d where %d was due", p, b[q + 4], len(plt))
            plt.append(b[q + 5:q + 2 + L])
            lens.append(plt_lengths(plt[-1]))
            q += 2 + L
        body0 = q + 2
        body = arr[body0:end]
        k0 = next_packet.get(tile, 0)
        # every two-byte value above 0xFF8F in the body: SOP and EPH, nothing else (Nsop itself is a parameter: its bytes
        # may be 0xFF and followed by anything)
        hi = np.flatnonzero((body[:-1] == 0xFF) & (body[1:] > 0x8F)) if len(body) > 1 else np.zeros(0, np.int64)
        packets, starts = None, None
        if plt:
            packets = np.concatenate(lens)
            _check(int(packets.sum()) == len(body), "tile part at %d: PLT lengths add up to %d, the body has %d bytes",
                   p, int(packets.sum()), len(body))
            _check(np.all(packets > 0), "tile part at %d: a zero packet length", p)
            starts = np.concatenate([[0], np.cumsum(packets)[:-1]]).astype(np.int64)
        if sop:
            if starts is None:          # the SOP markers mark the packets: FF91 0004, each 6 bytes past the last one
                cand = hi[(body[hi + 1] == 0x91)]
                cand = cand[(cand + 3 < len(body))]
                cand = cand[(body[cand + 2] == 0) & (body[cand + 3] == 4)]
                keep, last = [], -6
                for s in cand.tolist():
                    if s >= last + 6:
                        keep.append(s)
                        last = s
                sops = np.array(keep, np.int64)
                _check(len(body) == 0 or (len(sops) and sops[0] == 0), "tile part at %d: the body does not start with SOP", p)
            else:
                sops = starts
                _check(np.all(starts + 6 <= len(body)) and np.all(body[starts] == 0xFF) and np.all(body[starts + 1] == 0x91),
                       "tile part at %d: SOP markers are not at the packet starts", p)
            _check(np.all(body[sops + 2] == 0) and np.all(body[sops + 3] == 4), "tile part at %d: Lsop", p)
            got = (body[sops + 4].astype(np.int64) << 8) | body[sops + 5]
            nsop = (k0 + np.arange(len(sops))) & 0xFFFF
            bad = np.flatnonzero(got != nsop)
            _check(not len(bad), "tile part at %d: packet %d has Nsop %d, not %d", p, k0 + int(bad[0]) if len(bad) else 0,
                   int(got[bad[0]]) if len(bad) else 0, int(nsop[bad[0]]) if len(bad) else 0)
            hi = hi[~np.isin(hi, np.concatenate([sops + 4, sops + 5]))]
            kinds = body[hi + 1]
            _check(np.array_equal(hi[kinds == 0x91], sops), "tile part at %d: an SOP marker off a packet start", p)
        else:
            sops = None
            kinds = body[hi + 1]
        ephs = hi[kinds == 0x92]
        _check(np.all((kinds == 0x92) | ((kinds == 0x91) if sop else False)) and (eph or not len(ephs)),
               "tile part at %d: a marker-range byte pair in the body that is neither SOP nor EPH", p)
        marks = starts if starts is not None else sops
        if eph and marks is not None and len(marks):
            per = np.bincount(np.searchsorted(marks, ephs, "right") - 1, minlength=len(marks))
            _check(np.all(per == 1), "tile part at %d: a packet with %d EPH markers", p, int(per[per != 1][0]) if np.any(per != 1) else 1)
        npk = len(marks) if marks is not None else None
        if npk is not None:
            next_packet[tile] = k0 + npk
        parts.append(dict(tile=tile, index=tp, count=tn, psot=psot, plt=plt, packets=packets, first_packet=k0, at=p))
        p = end
    _check(b[p:] == b"\xff\xd9", "EOC is not last (%d bytes from %d)", n - p, p)
    for t, c in count.items():
        _check(next_part[t] == c, "tile %d: %d tile parts of TNsot %d", t, next_part[t], c)
    if tlm:
        ent = [e for s in tlm for e in s]
        _check(len(ent) == len(parts), "TLM: %d entries for %d tile parts", len(ent), len(parts))
        for i, ((t, L), pt) in enumerate(zip(ent, parts)):
            _check((t is None or t == pt["tile"]) and L == pt["psot"], "TLM entry %d: (%s, %d), the tile part is (%d, %d)",
                   i, t, L, pt["tile"], pt["psot"])
    return dict(sop=sop, eph=eph, tlm=[len(s) for s in tlm], parts=parts)
