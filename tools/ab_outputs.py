"""Byte-for-byte A/B check of two library builds on seeded inputs.

    B2K_LIB=<build A> python tools/ab_outputs.py OUT_A
    B2K_LIB=<build B> python tools/ab_outputs.py OUT_B
    python tools/ab_outputs.py --compare OUT_A OUT_B

Each run writes, per case, the forward coefficients, the coded bytes and block lengths and the planes that inverse()
rebuilds from them, as .npy files under OUT.  Cases: tests/test_gpu.py's GEOMS, reversible and irreversible (shapes whose
coding the engine refuses are skipped), the 9/7 degenerate-geometry shapes, a 2048^2 single-tile 9/7 image, and the
sample transports of the one-call entry points: a b2k_encode16 / b2k_decode16 round trip, b2k_encode16_interleaved,
b2k_encode / b2k_decode with host packing forced on, 16-bit windowed decodes (b2k_decode_window), and, where torch has
CUDA, b2k_encode_device / b2k_decode_device with uint16 tensors and the entry points whose code streams live in device
memory (device_codestreams: single and batch encodes and decodes, the parse, windows and failures).  Every one-call entry
point except the host windowed decode also stores the launches it made (b2k_launch_count() after the call minus before),
so that a change in one leg's count does not show in the legs after it.  Last come the device-resident round trips
(b2k_job_roundtrip, _roundtrip_n, _roundtrip_pipelined_n (2, 2)): on config 2 the launches of each and its coded size, on a tiled 9/7
image the same and the planes left after four steps.  --compare exits 1 when any array differs; tolerances would
hide a drift of one rounding step in the 9/7 inverse, so there are none."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]


def cases():
    import test_gpu
    degenerate = next(m.args[1] for m in test_gpu.test_irreversible_degenerate_geometry.pytestmark if m.name == "parametrize")
    out = [("geom%02d_%s" % (i, "irrev" if irr else "rev"), dict(g, irreversible=irr))
           for irr in (False, True) for i, g in enumerate(test_gpu.GEOMS)]
    out += [("degen97_%d" % i, dict(g, irreversible=True)) for i, g in enumerate(degenerate)]
    out.append(("single_tile_97_2048", dict(width=2048, height=2048, numcomps=3, prec=12, irreversible=True)))
    return out


def one_case(G, P, eng, args):
    planes = P.synthetic_image(args["width"], args["height"], args["numcomps"], args["prec"], seed=42,
                               origin=args.get("origin", (0, 0)))
    if args.get("sgnd"):
        planes = [p - (1 << (args["prec"] - 1)) for p in planes]
    job = eng.job(G.make_coding(**args))
    try:
        job.upload(planes)
        job.forward()
        coef = [np.zeros_like(p) for p in planes]
        job.download_coeffs(coef)
        arrs = {"coef%d" % c: a for c, a in enumerate(coef)}
        job.t1_encode()
        res = job.fetch_result()
        arrs["bytes"], arrs["lengths"] = res.bytes.copy(), res.blocks["length"].copy()
        res.free()
        job.t1_decode()
        job.inverse()
        rec = [np.zeros_like(p) for p in planes]
        job.download(rec)
        arrs.update(("rec%d" % c, a) for c, a in enumerate(rec))
        return arrs
    finally:
        job.close()


def device_codestreams(G, P, eng, torch, counted, arrs):
    """The code-stream entry points whose streams live in device memory, on a 9-tile 12-bit image (tensors of uint16 and
    int32, CHW and HWC): the single and batch encodes (bytes, offsets, statuses), the single decode, the parse (coding,
    block table, stats), windows at reduce 0 and 2 (one window takes every tile, one does not), and the batch decode
    (pixels, statuses).  Failures record the return code, the text and the Coding left in cp_out (pre-filled with 0xA5):
    a damaged SOT, a damaged main header, a block table too small, a bad image descriptor, a stream the HT decoder
    rejects (with the pixels the single call writes), an 8-bit container under a 12-bit coding and flags the writer
    declines."""
    import ctypes as C
    import test_device_batch_decode as BD
    import test_device_batch_encode as BE
    import test_device_codestream_decode as E
    L = G.lib()

    def text(rc):
        return np.frombuffer((L.b2k_last_error() or b"").decode().encode() if rc else b"", np.uint8)

    def sentinel_coding():
        got = G.Coding()
        C.memset(C.addressof(got), 0xA5, C.sizeof(got))
        return got

    def dev(a):
        return torch.from_numpy(np.array(a, np.uint8)).cuda()

    cp = G.make_coding(700, 500, 3, 12, numres=5, tile=(256, 192), origin=(5, 11), tile_origin=(0, 0))
    h, w = cp.y1 - cp.y0, cp.x1 - cp.x0
    chw = [torch.from_numpy(np.stack(P.synthetic_image(w, h, 3, 12, seed=s, origin=(5, 11))).astype(np.uint16)).cuda()
           for s in (31, 32, 33)]
    flags = G.CS_TLM | G.CS_PLT
    # encodes: one image; a batch of three with a misaligned descriptor between them
    cs = counted("dcs_enc", lambda: eng.encode_codestream_device(cp, chw[0], flags, device_output=True))
    arrs["dcs_enc_bytes"] = cs.cpu().numpy()
    descs = [G.device_planes(t, 3, h, w) for t in chw]
    bad = torch.zeros(16, dtype=torch.uint16, device="cuda")
    descs.insert(1, G.device_planes(chw[1], 3, h, w))
    descs[1].comp[1] = bad.data_ptr() + 1
    rc, status, got, offsets = counted("dcs_enc_batch", lambda: BE._raw_batch(eng, torch, cp, descs, flags))
    arrs["dcs_enc_batch_rc"] = np.array([rc])
    arrs["dcs_enc_batch_status"] = np.array([s[0] for s in status])
    arrs["dcs_enc_batch_text"] = np.frombuffer("\n".join(s[1] for s in status).encode(), np.uint8)
    arrs["dcs_enc_batch_offsets"] = np.array(offsets, np.uint64)
    arrs["dcs_enc_batch_bytes"] = np.concatenate([g for g in got if g is not None])
    # single decodes of that stream, its parse
    for tag, dtype, layout in (("u16", torch.uint16, "CHW"), ("u16_hwc", torch.uint16, "HWC"), ("i32", torch.int32, "CHW")):
        _, out = counted("dcs_dec_" + tag, lambda: eng.decode_codestream_device(cs, dtype=dtype, layout=layout))
        torch.cuda.synchronize()
        arrs["dcs_dec_%s_rec" % tag] = out.cpu().numpy()
    pcp, blocks = counted("dcs_parse", lambda: eng.codestream_parse_device(cs))
    arrs["dcs_parse_coding"], arrs["dcs_parse_blocks"] = np.frombuffer(bytes(pcp), np.uint8), blocks
    arrs["dcs_parse_stats"] = np.array(eng.codestream_parse_device_stats())
    # windows
    for i, win in enumerate([(5, 11, 705, 511), (37, 200, 650, 333)]):
        for reduce in (0, 2):
            tag = "dcs_win%d_r%d" % (i, reduce)
            vcp, out = counted(tag, lambda: eng.decode_window_device(cs, win, reduce))
            torch.cuda.synchronize()
            arrs[tag + "_rec"], arrs[tag + "_coding"] = out.cpu().numpy(), np.frombuffer(bytes(vcp), np.uint8)
            arrs[tag + "_rect"] = np.array(G.window_rect(vcp, win, reduce))
            arrs[tag + "_stats"] = np.array(eng.codestream_window_device_stats(), np.uint64)
            arrs[tag + "_parse_stats"] = np.array(eng.codestream_parse_device_stats())
    # damaged streams
    host = cs.cpu().numpy()
    last = E._sots(host)[-1]
    sot = host.copy()
    sot[last + 4:last + 6] = 0xFF                                   # a tile index out of range
    hdr = host.copy()
    hdr[0:2] = 0                                                    # no SOC
    good = E._base_stream(eng)                                      # the stream the batch tests find an HT rejection in
    ht, _ = BD._ht_reject(eng, torch, good)
    hcp = G.codestream_parse(good)[0]

    def raw_decode(tag, stream, coding, misaligned=False):
        nc, hh, ww = coding.numcomps, coding.y1 - coding.y0, coding.x1 - coding.x0
        out = torch.full((nc, hh, ww), 0x5A, dtype=torch.uint16, device="cuda")
        img = G.device_planes(out, nc, hh, ww, writable=True)
        if misaligned:
            img.comp[1] = bad.data_ptr() + 1
        d, got, ms = dev(stream), sentinel_coding(), C.c_double()
        rc = counted(tag, lambda: L.b2k_decode_codestream_device(eng._h, d.data_ptr(), d.numel(), C.byref(img), None, C.byref(got),
                                                                 C.byref(ms)))
        torch.cuda.synchronize()
        arrs[tag + "_rc"], arrs[tag + "_text"], arrs[tag + "_cp"] = np.array([rc]), text(rc), np.frombuffer(bytes(got), np.uint8)
        arrs[tag + "_rec"] = out.cpu().numpy()

    def raw_parse(tag, stream, cap):
        d, got = dev(stream), sentinel_coding()
        blocks = np.zeros(max(cap, 1), G.BLOCK_DTYPE)
        rc = counted(tag, lambda: L.b2k_codestream_parse_device(eng._h, d.data_ptr(), d.numel(), None, C.byref(got), blocks.ctypes.data,
                                                                cap))
        arrs[tag + "_rc"], arrs[tag + "_cp"] = np.array([rc]), np.frombuffer(bytes(got), np.uint8)
        arrs[tag + "_text"] = text(rc < 0 or rc == 1)
        arrs[tag + "_blocks"] = blocks

    nb = len(blocks)
    for tag, stream in (("sot", sot), ("header", hdr)):
        raw_decode("dcs_fail_%s_dec" % tag, stream, cp)
        raw_parse("dcs_fail_%s_parse" % tag, stream, nb)
    raw_parse("dcs_fail_table_parse", host, nb - 1)
    raw_decode("dcs_fail_image_dec", host, cp, misaligned=True)
    raw_decode("dcs_fail_ht_dec", ht, hcp)
    # a batch of good and failing streams: statuses, and the pixels of the streams that decode
    batch = [cs, dev(sot), eng.encode_codestream_device(cp, chw[1], flags, device_output=True), dev(hdr),
             eng.encode_codestream_device(cp, chw[2], flags, device_output=True)]
    _, out, status = counted("dcs_dec_batch", lambda: eng.decode_codestreams_device(batch))
    torch.cuda.synchronize()
    arrs["dcs_dec_batch_rec"] = out.cpu().numpy()
    arrs["dcs_dec_batch_status"] = np.array([s[0] for s in status])
    arrs["dcs_dec_batch_text"] = np.frombuffer("\n".join(s[1] for s in status).encode(), np.uint8)
    arrs["dcs_dec_batch_stats"] = np.array(eng.codestream_parse_device_stats())
    hbatch = [dev(good), dev(ht), dev(good)]
    _, out, status = counted("dcs_dec_batch_ht", lambda: eng.decode_codestreams_device(hbatch))
    torch.cuda.synchronize()
    arrs["dcs_dec_batch_ht_rec"] = out.cpu().numpy()
    arrs["dcs_dec_batch_ht_status"] = np.array([s[0] for s in status])
    # encode verdicts: an 8-bit container under a 12-bit coding, and progression order 5, which the writer declines
    u8_image = chw[0].to(torch.uint8)
    u8 = G.device_planes(u8_image, 3, h, w)
    for tag, img, f in (("u8", u8, flags), ("prog5", descs[0], G.CS_PROG(5) | G.CS_PLT)):
        rc, txt, data = counted("dcs_fail_enc_" + tag, lambda: BE._single(eng, torch, cp, img, f))
        arrs["dcs_fail_enc_%s_rc" % tag] = np.array([rc])
        arrs["dcs_fail_enc_%s_text" % tag] = np.frombuffer(txt.encode(), np.uint8)
        rc, status, _, _ = counted("dcs_fail_enc_batch_" + tag, lambda: BE._raw_batch(eng, torch, cp, [img, img], f))
        arrs["dcs_fail_enc_batch_%s_rc" % tag] = np.array([rc])
        arrs["dcs_fail_enc_batch_%s_status" % tag] = np.frombuffer(repr(status).encode(), np.uint8)
    for k in sorted(arrs):
        if k.startswith("dcs_") and k.endswith("_launches"):
            print("%s: %d launches" % (k[:-len("_launches")], arrs[k][0]))


def run(outdir):
    import grok_b200 as G
    import oracle_pipeline as P
    os.makedirs(outdir, exist_ok=True)
    eng = G.Engine()
    for name, args in cases():
        try:
            arrs = one_case(G, P, eng, args)
        except G.EngineError as e:
            print("skip %s: %s" % (name, e))
            continue
        for k, a in arrs.items():
            np.save(os.path.join(outdir, "%s.%s.npy" % (name, k)), a)
    arrs = {}

    def counted(name, fn):
        before = int(G.lib().b2k_launch_count())
        r = fn()
        arrs[name + "_launches"] = np.array([int(G.lib().b2k_launch_count()) - before], np.uint64)
        return r

    def keep(name, res):
        arrs[name + "_bytes"], arrs[name + "_lengths"] = res.bytes.copy(), res.blocks["length"].copy()
        res.free()

    # 16-bit containers: b2k_encode16 / b2k_decode16, and the same pixels interleaved (b2k_encode16_interleaved)
    cp = G.make_coding(600, 300, 3, 12, numres=5, tile=(256, 128), origin=(8, 0))
    p16 = [p.astype(np.uint16) for p in P.synthetic_image(600, 300, 3, 12, seed=77)]
    res = counted("u16_enc", lambda: eng.encode(cp, p16))
    blocks, data = res.blocks.copy(), res.bytes.copy()
    keep("u16", res)
    rec = [np.zeros_like(p) for p in p16]
    counted("u16_dec", lambda: eng.decode(cp, blocks, data, rec))
    arrs.update(("u16_rec%d" % c, a) for c, a in enumerate(rec))
    keep("u16_interleaved", counted("u16_interleaved", lambda: eng.encode_interleaved(cp, np.ascontiguousarray(np.stack(p16, -1)))))
    # int32 planes through the host-packing ring: large enough (>= 4 Msamples, several chunks) to be packed
    w, h = 2501, 1803
    cp = G.make_coding(w, h, 3, 12, numres=5, tile=(700, 500), origin=(3, 5))
    planes = P.synthetic_image(w, h, 3, 12, seed=11, origin=(3, 5))
    G.set_host_threads(3)
    try:
        res = counted("packed_enc", lambda: eng.encode(cp, planes))
        blocks, data = res.blocks.copy(), res.bytes.copy()
        keep("packed", res)
        rec = [np.zeros_like(p) for p in planes]
        counted("packed_dec", lambda: eng.decode(cp, blocks, data, rec))
        arrs["packed_used"] = np.array(G.host_pack_last())
        arrs.update(("packed_rec%d" % c, a) for c, a in enumerate(rec))
    finally:
        G.set_host_threads(-1)
    # b2k_encode_device / b2k_decode_device from and into uint16 tensors, planar and pixel-interleaved
    try:
        import torch
        cuda = torch.cuda.is_available()
    except ImportError:
        cuda = False
    if cuda:
        cp = G.make_coding(600, 300, 3, 12, numres=5, tile=(256, 128), origin=(8, 0))
        chw = torch.from_numpy(np.stack(p16)).cuda()
        for layout, img in (("CHW", chw), ("HWC", chw.permute(1, 2, 0).contiguous())):
            res = counted("dev_%s_enc" % layout, lambda: eng.encode_device(cp, img, layout=layout))
            blocks, data = res.blocks.copy(), res.bytes.copy()
            keep("dev_%s" % layout, res)
            out = torch.zeros_like(img)
            counted("dev_%s_dec" % layout, lambda: eng.decode_device(cp, blocks, data, out, layout=layout))
            torch.cuda.synchronize()
            arrs["dev_%s_rec" % layout] = out.cpu().numpy()
        device_codestreams(G, P, eng, torch, counted, arrs)
    # 16-bit windowed decodes of a tiled image with an odd origin, at full and half resolution
    cp = G.make_coding(700, 500, 3, 12, numres=5, tile=(256, 192), origin=(5, 11), tile_origin=(0, 0), irreversible=True)
    cs = eng.encode_codestream(cp, P.synthetic_image(700, 500, 3, 12, seed=23, origin=(5, 11)))
    for i, win in enumerate([(5, 11, 705, 511), (37, 200, 650, 333), (261, 11, 517, 203)]):
        for reduce in (0, 1):
            _, got = eng.decode_window(cs, win, reduce, dtype=np.uint16)
            arrs.update(("win%d_r%d_rec%d" % (i, reduce, c), g.copy()) for c, g in enumerate(got))
    # the device-resident round trips: config 2 (the first call's sizing pass included) and four 9/7 steps of a tiled image
    for tag, cp, img in (("rt_config2", G.make_coding(8192, 8192, 3, 12, numres=6, tile=(1024, 1024)),
                          P.synthetic_image(8192, 8192, 3, 12, seed=20260924)),
                         ("rt_97", G.make_coding(700, 500, 3, 12, numres=5, tile=(256, 192), irreversible=True),
                          P.synthetic_image(700, 500, 3, 12, seed=23))):
        job = eng.job(cp)
        try:
            job.upload(img)
            for name, fn in (("one", job.roundtrip), ("n", lambda: job.roundtrip_n(8 if tag == "rt_config2" else 1)),
                             ("pipelined", lambda: job.roundtrip_pipelined_n(8 if tag == "rt_config2" else 2, 2, 2))):
                arrs["%s_%s_coded" % (tag, name)] = np.array([counted("%s_%s" % (tag, name), fn)[-1]], np.uint64)
                print("%s %s: %d launches" % (tag, name, arrs["%s_%s_launches" % (tag, name)][0]))
            rec = [np.zeros_like(p) for p in img]
            job.download(rec)
            if tag == "rt_97":
                arrs.update(("rt_97_rec%d" % c, a) for c, a in enumerate(rec))
            else:
                arrs["rt_config2_lossless"] = np.array([all(np.array_equal(a, b) for a, b in zip(rec, img))])
        finally:
            job.close()
    for k, a in arrs.items():
        np.save(os.path.join(outdir, "transport.%s.npy" % k), a)
    eng.close()
    print("wrote %d arrays to %s" % (len(os.listdir(outdir)), outdir))


def compare(a, b):
    fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
    bad = sorted(set(fa) ^ set(fb))
    for f in sorted(set(fa) & set(fb)):
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        if x.dtype != y.dtype or x.shape != y.shape or x.tobytes() != y.tobytes():
            bad.append(f)
    for f in bad:
        print("DIFFERS:", f)
    print("%d arrays compared, %d differ" % (len(set(fa) | set(fb)), len(bad)))
    return 1 if bad else 0


if __name__ == "__main__":
    if sys.argv[1] == "--compare":
        sys.exit(compare(sys.argv[2], sys.argv[3]))
    run(sys.argv[1])
