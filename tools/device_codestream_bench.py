"""Code streams written on the GPU (b2k_encode_codestream_device) against host T2, on config 2 (8192x8192x3, 12 bit,
1024^2 tiles) from a torch uint16 CHW tensor, in one GPU job.

    python tools/device_codestream_bench.py [--steps K] [--warmup W] [--out DIR]

Three legs, alternated step by step so that all of them see the same machine:
  host_t2     Engine.encode_codestream_device(cp, img): the result comes home, b2k_codestream_write plans and copies on the
              host, a numpy array
  device      the same with device_output=True: T2 on the device, a torch uint8 CUDA tensor
  device_cpu  device followed by .cpu(): the bytes in host memory, as host_t2 leaves them
Each step is timed with the host clock around calls that return with their work done; the first --warmup steps of every
leg are not timed.  All three must give the same bytes.  Then, in a run of its own under torch.profiler, the T2 kernels
of the device leg are timed; the body copy (the encoder's gather kernel, run by T2) reads and writes each coded byte
once, so its bytes/s are 2 x coded bytes over its time.  Prints one JSON line with the GPU's name and power limit;
--out DIR also writes it, and the profiler's kernel table, there."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HBM_DATASHEET_BPS = 3.35e12
T2_KERNELS = ("k_t2_headers", "k_t2_parts", "k_t2_scan", "k_t2_emit", "k_t2_packets", "k_ht_gather")


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
    chw = torch.from_numpy(np.stack(bench.make_image()).astype(np.uint16)).cuda()
    eng = G.Engine(0)
    flags = G.CS_TLM | G.CS_PLT

    legs = {"host_t2": lambda: eng.encode_codestream_device(cp, chw, flags),
            "device": lambda: eng.encode_codestream_device(cp, chw, flags, device_output=True),
            "device_cpu": lambda: eng.encode_codestream_device(cp, chw, flags, device_output=True).cpu()}
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
    want = last["host_t2"]
    assert np.array_equal(last["device"].cpu().numpy(), want), "device code stream differs from host T2"
    assert np.array_equal(last["device_cpu"].numpy(), want), "device code stream (.cpu()) differs from host T2"

    # T2 kernels, in a run of their own under the profiler
    from torch.profiler import ProfilerActivity, profile
    launches0 = G.lib().b2k_launch_count()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.profile_steps):
            legs["device"]()
        torch.cuda.synchronize()
    launches = (G.lib().b2k_launch_count() - launches0) / args.profile_steps
    kernels = {}
    for ev in prof.key_averages():
        name = next((k for k in T2_KERNELS if k in ev.key), None)
        if name is None:
            continue
        us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
        k = kernels.setdefault(name, {"launches": 0, "us": 0.0})
        k["launches"] += ev.count
        k["us"] += us
    t2_us = sum(k["us"] for k in kernels.values())
    for k in kernels.values():
        k["ms_per_step"] = k.pop("us") / 1e3 / args.profile_steps
    body = kernels.get("k_ht_gather")
    body_bytes = 2 * int(want.size)   # every coded byte read once and written once (headers and markers are a rounding error)
    if body:
        body["alg_bytes_per_step"] = body_bytes
        body["bytes_per_s"] = body_bytes / (body["ms_per_step"] * 1e-3) if body["ms_per_step"] else None
        body["share_of_datasheet_hbm"] = body["bytes_per_s"] / HBM_DATASHEET_BPS if body["bytes_per_s"] else None
    line = {"tool": "device_codestream_bench", "gpu": bench.gpu_info(0),
            "workload": "config 2: 8192x8192x3 12-bit, 5/3 + RCT, 1024x1024 tiles, 6 resolutions, TLM + PLT; torch uint16 CHW tensor",
            "steps": args.steps, "warmup": args.warmup, "codestream_bytes": int(want.size),
            "ms_per_step": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                            for k, v in times.items()},
            "t2_kernels": kernels, "t2_ms_per_step": t2_us / 1e3 / args.profile_steps,
            "engine_launches_per_call": launches,
            "hbm_reference": "H100 SXM data sheet, 3.35 TB/s (not measured here)"}
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_codestream_bench.json"), "w") as f:
            f.write(text + "\n")
        with open(os.path.join(args.out, "device_codestream_kernels.txt"), "w") as f:
            f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=40))
    eng.close()


if __name__ == "__main__":
    main()
