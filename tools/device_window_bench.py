"""Windows of a large code stream held in device memory (Engine.decode_window_device) against today's ways of getting
them from HBM, on config 5's stream: SIZE x SIZE x 3, 12 bit, 1024^2 tiles, TLM + PLT, generator pixels (per-tile offsets
of one synthetic tile, as tools/config5_roi_bench.py makes them), encoded on the GPU into a uint8 CUDA tensor.

    python tools/device_window_bench.py [--size 32768] [--roi 2048] [--steps K] [--warmup W] [--out DIR]

Seeded ROI x ROI windows at reduce 0 and 2.  Legs, alternated step by step so that all of them see the same machine:
  via_host       cs.cpu() + decode_codestream_device(host bytes, window, reduce): today's path from HBM
  host_resident  the host bytes already resident: the host parser's floor
  device         decode_window_device(cs, window, reduce): only the touched tiles' parts are parsed and copied
Each step is timed with the host clock around calls that return with their work done; the first --warmup steps of every
leg are not timed.  Every window's pixels are checked: against the generator at reduce 0, against host_resident at reduce 2.
Then, in a run of its own under torch.profiler, the device leg's kernels are timed: k_t2_locate (the serial walk over every
SOT of the stream), the other parse kernels, the gather, and the decode chain.  Prints one JSON line with the GPU's name and
power limit; --out DIR also writes it, and the profiler's kernel table, there."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

TILE = 1024
PARSE = ("k_t2_plt", "k_t2_packets", "k_t2_walk", "k_t2_desc")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=32768)
    ap.add_argument("--roi", type=int, default=2048)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import bench
    import grok_b200 as G
    import oracle_pipeline as P

    S, T = args.size, TILE
    reps = S // T
    base = torch.from_numpy(np.stack(P.synthetic_image(T, T, 3, 12, seed=20260927)).astype(np.int32)).cuda()

    def tile_pixels(t):
        return ((base + 37 * t) & 0xFFF).to(torch.uint16)

    cp = G.make_coding(S, S, 3, 12, numres=6, tile=(T, T))
    img = torch.empty((3, S, S), dtype=torch.uint16, device="cuda")
    for t in range(reps * reps):
        ty, tx = divmod(t, reps)
        img[:, ty * T:(ty + 1) * T, tx * T:(tx + 1) * T] = tile_pixels(t)
    enc = G.Engine(0)
    cs = enc.encode_codestream_device(cp, img, G.CS_TLM | G.CS_PLT, device_output=True)
    enc.close()
    del img
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    host_cs = cs.cpu().numpy()

    def expected(x0, y0):
        out = torch.empty((3, args.roi, args.roi), dtype=torch.uint16, device="cuda")
        for ty in range(y0 // T, (y0 + args.roi - 1) // T + 1):
            for tx in range(x0 // T, (x0 + args.roi - 1) // T + 1):
                ya, yb, xa, xb = max(y0, ty * T), min(y0 + args.roi, (ty + 1) * T), max(x0, tx * T), min(x0 + args.roi, (tx + 1) * T)
                out[:, ya - y0:yb - y0, xa - x0:xb - x0] = tile_pixels(ty * reps + tx)[:, ya - ty * T:yb - ty * T, xa - tx * T:xb - tx * T]
        return out

    eng = G.Engine(0)
    rng = np.random.default_rng(20260927)
    n_win = args.warmup + args.steps
    wins = [(int(rng.integers(0, S - args.roi)), int(rng.integers(0, S - args.roi))) for _ in range(n_win)]
    legs = {"via_host": lambda w, r: eng.decode_codestream_device(cs.cpu().numpy(), window=w, reduce=r)[1],
            "host_resident": lambda w, r: eng.decode_codestream_device(host_cs, window=w, reduce=r)[1],
            "device": lambda w, r: eng.decode_window_device(cs, window=w, reduce=r)[1]}
    result = {}
    ok = True
    stats = {}
    for reduce in (0, 2):
        times = {k: [] for k in legs}
        for i, (x0, y0) in enumerate(wins):
            w = (x0, y0, x0 + args.roi, y0 + args.roi)
            got = {}
            for name, step in legs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                got[name] = step(w, reduce)
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[name].append((time.perf_counter() - t0) * 1e3)
                if name == "device":
                    stats[reduce] = eng.codestream_window_device_stats()
            want = expected(x0, y0) if reduce == 0 else got["host_resident"]
            ok &= all(torch.equal(v, want) for v in got.values())
        result["reduce_%d" % reduce] = {
            "ms_per_window": {k: {"median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))} for k, v in times.items()},
            "tiles_wanted_arena_bytes_last_window": list(stats[reduce])}

    from torch.profiler import ProfilerActivity, profile
    prof_out = {}
    for reduce in (0, 2):
        launches0 = G.lib().b2k_launch_count()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for (x0, y0) in wins[:args.profile_steps]:
                eng.decode_window_device(cs, window=(x0, y0, x0 + args.roi, y0 + args.roi), reduce=reduce)
            torch.cuda.synchronize()
        launches = (G.lib().b2k_launch_count() - launches0) / args.profile_steps
        groups = {"k_t2_locate": 0.0, "parse_other": 0.0, "k_t2_gather": 0.0, "decode_chain": 0.0}
        for ev in prof.key_averages():
            us = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0.0)
            if not us:
                continue
            if "k_t2_locate" in ev.key:
                groups["k_t2_locate"] += us
            elif any(k in ev.key for k in PARSE):
                groups["parse_other"] += us
            elif "k_t2_gather" in ev.key:
                groups["k_t2_gather"] += us
            else:
                groups["decode_chain"] += us
        total = sum(groups.values())
        prof_out["reduce_%d" % reduce] = {"ms_per_window": {k: v / 1e3 / args.profile_steps for k, v in groups.items()},
                                          "locate_share_of_device_time": groups["k_t2_locate"] / total if total else None,
                                          "engine_launches_per_call": launches}
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "device_window_kernels_r%d.txt" % reduce), "w") as f:
                f.write(prof.key_averages().table(sort_by="device_time_total", row_limit=40))
    line = {"tool": "device_window_bench", "gpu": bench.gpu_info(0),
            "workload": "config 5: %dx%dx3 12-bit, 5/3 + RCT, %d tiles of 1024^2, TLM + PLT, %d-byte stream in a uint8 CUDA tensor; "
                        "%dx%d windows -> uint16 CHW" % (S, S, reps * reps, int(cs.numel()), args.roi, args.roi),
            "steps": args.steps, "warmup": args.warmup, "pixels_match": bool(ok), **result, "device_kernels": prof_out}
    text = json.dumps(line)
    print(text)
    if args.out:
        with open(os.path.join(args.out, "device_window_bench.json"), "w") as f:
            f.write(text + "\n")
    eng.close()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
