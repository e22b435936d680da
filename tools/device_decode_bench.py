"""Code streams decoded from device memory (Engine.decode_codestream_device of a CUDA tensor) against the path through the
host, on config 2 (8192x8192x3, 12 bit, 1024^2 tiles), from a torch uint8 CUDA tensor into a uint16 CHW tensor, in one
GPU job.

    python tools/device_decode_bench.py [--steps K] [--warmup W] [--out DIR]

Legs, alternated step by step so that all of them see the same machine:
  via_host            cs.cpu().numpy(), then decode_codestream_device of the host bytes (host parse, bytes up over PCIe)
  device              the TLM + PLT stream parsed on the device: every tile packet by packet from its PLT starts
  device_no_plt       a TLM-only stream of the same image: every tile walked by one thread
  single_tile_no_plt  8192x8192x3 as one tile, no PLT: one thread walks every packet (the walk's worst case)
Each step is timed with the host clock around calls that return with their work done; the first --warmup steps of every
leg are not timed.  All legs must give the source image; the JSON line reports, per device leg, how many tiles went packet
by packet and how many were walked.  Then, in a run of its own under torch.profiler, the parse
kernels of the device leg and the arena copy (device to device, 2 x code-stream bytes of HBM traffic) are timed.  Prints
one JSON line with the GPU's name and power limit; --out DIR also writes it, and the profiler's kernel table, there."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HBM_DATASHEET_BPS = 3.35e12
PARSE_KERNELS = ("k_t2_locate", "k_t2_plt", "k_t2_packets", "k_t2_walk", "k_t2_desc", "Memcpy DtoD")


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
    one = G.make_coding(W, H, NC, bench.PREC, numres=bench.NUMRES)
    chw = torch.from_numpy(np.stack(bench.make_image()).astype(np.uint16)).cuda()
    eng = G.Engine(0)
    streams = {"device": eng.encode_codestream_device(cp, chw, G.CS_TLM | G.CS_PLT, device_output=True),
               "device_no_plt": eng.encode_codestream_device(cp, chw, G.CS_TLM, device_output=True),
               "single_tile_no_plt": eng.encode_codestream_device(one, chw, G.CS_TLM, device_output=True)}
    legs = {"via_host": lambda: eng.decode_codestream_device(streams["device"].cpu().numpy())[1],
            "device": lambda: eng.decode_codestream_device(streams["device"])[1],
            "device_no_plt": lambda: eng.decode_codestream_device(streams["device_no_plt"])[1],
            "single_tile_no_plt": lambda: eng.decode_codestream_device(streams["single_tile_no_plt"])[1]}
    times = {k: [] for k in legs}
    last = {}
    for i in range(args.warmup + args.steps):
        for name, step in legs.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            last[name] = step()
            torch.cuda.synchronize()
            if i >= args.warmup:
                times[name].append((time.perf_counter() - t0) * 1e3)
    for name, out in last.items():
        assert torch.equal(out, chw), "%s: decoded pixels differ from the source" % name
    split = {}   # (tiles parsed packet by packet from PLT, tiles walked) per device leg
    for name in streams:
        legs[name]()
        split[name] = eng.codestream_parse_device_stats()

    from torch.profiler import ProfilerActivity, profile
    launches0 = G.lib().b2k_launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.profile_steps):
            legs["device"]()
        torch.cuda.synchronize()
    launches = (G.lib().b2k_launch_count() - launches0) / args.profile_steps
    kernels = {}
    for ev in prof.key_averages():
        name = next((k for k in PARSE_KERNELS if k in ev.key), None)
        if name is None:
            continue
        us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        k = kernels.setdefault(name, {"count": 0, "us": 0.0})
        k["count"] += ev.count
        k["us"] += us
    for k in kernels.values():
        k["ms_per_step"] = k.pop("us") / 1e3 / args.profile_steps
    n = int(streams["device"].numel())
    copy = kernels.get("Memcpy DtoD")
    if copy and copy["ms_per_step"]:
        copy["alg_bytes_per_step"] = 2 * n   # the stream read once and written once into the arena
        copy["bytes_per_s"] = 2 * n / (copy["ms_per_step"] * 1e-3)
        copy["share_of_datasheet_hbm"] = copy["bytes_per_s"] / HBM_DATASHEET_BPS
    line = {"tool": "device_decode_bench", "gpu": bench.gpu_info(0),
            "workload": "config 2: 8192x8192x3 12-bit, 5/3 + RCT, 1024x1024 tiles, 6 resolutions; uint8 CUDA tensor -> uint16 CHW",
            "steps": args.steps, "warmup": args.warmup,
            "codestream_bytes": {k: int(v.numel()) for k, v in streams.items()},
            "ms_per_step": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                            for k, v in times.items()},
            "tiles_indexed_walked": split, "parse_kernels_device_leg": kernels, "engine_launches_per_call": launches,
            "hbm_reference": "H100 SXM data sheet, 3.35 TB/s (not measured here)"}
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_decode_bench.json"), "w") as f:
            f.write(text + "\n")
        with open(os.path.join(args.out, "device_decode_kernels.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=40))
    eng.close()


if __name__ == "__main__":
    main()
