"""Encode from and decode into device memory on config 2 (8192x8192x3, 12 bit, 1024^2 tiles), in one GPU job.

    python tools/device_io_bench.py [--steps K] [--warmup W] [--out DIR]

Three legs, alternated step by step so that all of them see the same machine:
  dev_chw  Engine.encode_device + Engine.decode_device from / into a torch uint16 (3, H, W) tensor on the GPU
  dev_hwc  the same with a pixel-interleaved (H, W, 3) tensor
  host     b2k_encode + b2k_decode from / into pinned int32 planes (bench.py's `e2e` leg)
Each step is timed with the host clock around calls that return with their work done; the first --warmup steps of
every leg are not timed.  Then, in a run of its own under torch.profiler, the conversion kernels of the two device legs
are timed and their algorithmic bytes (2 B read + 4 B written per sample on encode, the reverse on decode) are turned
into bytes/s, next to the H100 SXM data sheet's 3.35 TB/s.  Prints one JSON line with the GPU's name and power limit;
--out DIR also writes it, and the profiler's kernel table, there."""
import argparse
import json
import os
import re
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HBM_DATASHEET_BPS = 3.35e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import bench
    import grok_b200 as G

    W, H, NC = bench.W, bench.H, bench.NCOMP
    cp = G.make_coding(W, H, NC, bench.PREC, numres=bench.NUMRES, tile=(bench.TILE, bench.TILE))
    img = bench.make_image()
    planes = [G.pinned_empty((H, W), np.int32) for _ in range(NC)]
    out = [G.pinned_empty((H, W), np.int32) for _ in range(NC)]
    for p, q in zip(planes, img):
        p[:] = q
    chw = torch.from_numpy(np.stack(img).astype(np.uint16)).cuda()
    hwc = chw.permute(1, 2, 0).contiguous()
    dec_chw, dec_hwc = torch.empty_like(chw), torch.empty_like(hwc)
    eng = G.Engine(0)
    G.set_host_threads(-1)   # the host leg as bench.py runs it: the engine picks packed or direct PCIe transfers

    def dev_step(frame, dec, layout):
        res = eng.encode_device(cp, frame, layout=layout)
        eng.decode_device(cp, res.blocks, res.bytes, dec, layout=layout)
        n = res.num_bytes
        res.free()
        return n

    def host_step():
        res = eng.encode(cp, planes)
        eng.decode(cp, res.blocks, res.bytes, out)
        n = res.num_bytes
        res.free()
        return n

    legs = {"dev_chw": lambda: dev_step(chw, dec_chw, "CHW"), "dev_hwc": lambda: dev_step(hwc, dec_hwc, "HWC"), "host": host_step}
    times = {k: [] for k in legs}
    coded = {}
    for i in range(args.warmup + args.steps):
        for name, step in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            coded[name] = step()
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[name].append((time.perf_counter() - t0) * 1e3)
    assert coded["dev_chw"] == coded["dev_hwc"] == coded["host"], coded
    want = np.stack(img).astype(np.uint16)
    assert np.array_equal(dec_chw.cpu().numpy(), want), "device CHW round trip is not lossless"
    assert np.array_equal(dec_hwc.permute(2, 0, 1).cpu().numpy(), want), "device HWC round trip is not lossless"
    assert all(np.array_equal(a, b) for a, b in zip(out, planes)), "host round trip is not lossless"

    # conversion kernels, in a run of their own under the profiler
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.profile_steps):
            legs["dev_chw"]()
            legs["dev_hwc"]()
        torch.cuda.synchronize()
    samples = NC * W * H
    alg_bytes = samples * (2 + 4)   # per direction, per step, u16 container <-> int32 planes
    kernels = {}
    for ev in prof.key_averages():
        if "k_container_to_planes" not in ev.key and "k_planes_to_container" not in ev.key:
            continue
        us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        # <2, 1>: 16-bit planar (the CHW leg, one launch per component); <2, 3>: 16-bit pixel-interleaved (the HWC leg)
        name = re.search(r"k_(?:container_to_planes|planes_to_container)<[^>]*>", ev.key).group(0)
        k = kernels.setdefault(name, {"launches": 0, "us": 0.0})
        k["launches"] += ev.count
        k["us"] += us
    for k in kernels.values():
        us = k.pop("us")
        k.update(ms_per_step=us / 1e3 / args.profile_steps, alg_bytes_per_step=alg_bytes,
                 bytes_per_s=alg_bytes * args.profile_steps / (us * 1e-6) if us else None)
        k["share_of_datasheet_hbm"] = k["bytes_per_s"] / HBM_DATASHEET_BPS if us else None
    line = {"tool": "device_io_bench", "gpu": bench.gpu_info(0),
            "workload": "config 2: 8192x8192x3 12-bit, 5/3 + RCT, 1024x1024 tiles, 6 resolutions; torch uint16 tensors",
            "steps": args.steps, "warmup": args.warmup, "coded_bytes": coded["host"],
            "ms_per_step": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                            for k, v in times.items()},
            "conversion_kernels": kernels,
            "hbm_reference": "H100 SXM data sheet, 3.35 TB/s (not measured here)"}
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_io_bench.json"), "w") as f:
            f.write(text + "\n")
        with open(os.path.join(args.out, "device_io_kernels.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=40))
    eng.close()


if __name__ == "__main__":
    main()
