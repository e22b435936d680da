"""Windows of batches of code streams held in device memory: one Engine.decode_windows_device call against a loop of
decode_window_device, one call per stream.

    python tools/device_window_batch_bench.py [--steps K] [--warmup W] [--out DIR]

Workloads (streams from encode_codestream_device of seeded images, as CUDA tensors):
  256 x 512^2 x 3, 8 bit, one tile, PLT: seeded random 224^2 crops at reduce 0 (the virtual coding is the streams' own:
      the whole-stream parse), and thumbnails (no window) at reduce 1
  64 x 4096^2 x 3, 12 bit, 1024^2 tiles, TLM + PLT: thumbnails at reduce 2, and one shared 1024^2 window at reduce 0
Legs, alternated step by step: `loop` (decode_window_device per stream into its own output) and `batch` (one
decode_windows_device).  Each step is timed with the host clock around calls that return with their work done; the first
--warmup steps are not timed, the median of the rest is reported.  Both legs' pixels must be equal.  Reports ms per
call, images/s and the engine's launches per call, then, in a run of its own under torch.profiler, the batch leg's
parse, gather, HT decode, inverse and conversion per call.  Prints one JSON line with the GPU's name and power limit;
--out DIR also writes it, and the profiler's tables, there."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")]

from device_batch_bench import timed_legs, summary, profiled, gpu_info   # noqa: E402

WORKLOADS = [dict(name="256x512sq_rgb8_crop224", n=256, size=512, comps=3, prec=8, tile=None, flags="PLT", window="crop", reduce=0),
             dict(name="256x512sq_rgb8_thumb_r1", n=256, size=512, comps=3, prec=8, tile=None, flags="PLT", window=None, reduce=1),
             dict(name="64x4096sq_rgb12_thumb_r2", n=64, size=4096, comps=3, prec=12, tile=1024, flags="TLM|PLT", window=None,
                  reduce=2),
             dict(name="64x4096sq_rgb12_win1024", n=64, size=4096, comps=3, prec=12, tile=1024, flags="TLM|PLT",
                  window=(1500, 900, 2524, 1924), reduce=0)]
GROUPS = {"parse": ("k_t2_locate", "k_t2_plt", "k_t2_packets", "k_t2_walk", "k_t2_window_at", "k_t2_desc"),
          "gather": ("k_t2_gather", "k_copy_table"), "ht_decode": ("k_ht_decode",), "inverse": ("k_dwt", "k_point_transform"),
          "conversion": ("k_planes_to_container",)}


def make(torch, G, w, cache):
    key = (w["n"], w["size"], w["comps"], w["prec"], w["tile"], w["flags"])
    if key in cache:
        return cache[key]
    flags = 0
    for f in w["flags"].split("|"):
        flags |= getattr(G, "CS_" + f)
    tile = (w["tile"], w["tile"]) if w["tile"] else None
    cp = G.make_coding(w["size"], w["size"], w["comps"], w["prec"], numres=6, tile=tile)
    g = torch.Generator(device="cuda").manual_seed(2026)
    eng = G.Engine(0)
    streams = []
    for i in range(w["n"]):   # one image at a time: 64 x 4096^2 x 3 samples need not be resident together
        img = torch.randint(0, 1 << w["prec"], (w["comps"], w["size"], w["size"]), dtype=torch.int32, device="cuda", generator=g)
        img = img.to(torch.uint8) if w["prec"] <= 8 else img.to(torch.uint16)
        streams.append(eng.encode_codestream_device(cp, img, flags, device_output=True))
    eng.close()
    cache.clear()
    cache[key] = (cp, streams)
    return cp, streams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    import grok_b200 as G
    L = G.lib()
    name, power = gpu_info()
    result = dict(gpu=name, power_limit=power, steps=args.steps, warmup=args.warmup, workloads={})
    tables = []
    cache = {}
    for w in WORKLOADS:
        cp, streams = make(torch, G, w, cache)
        n, r = w["n"], w["reduce"]
        if w["window"] == "crop":
            rng = np.random.default_rng(224)
            xs, ys = rng.integers(0, w["size"] - 224 + 1, n), rng.integers(0, w["size"] - 224 + 1, n)
            windows = [(int(x), int(y), int(x) + 224, int(y) + 224) for x, y in zip(xs, ys)]
        else:
            windows = [w["window"]] * n
        eng = G.Engine(0)
        dt = torch.uint8 if w["prec"] <= 8 else torch.uint16
        out_loop = [eng.decode_window_device(s, window=win, reduce=r, dtype=dt)[1] for s, win in zip(streams, windows)]
        out_batch = {}

        def loop():
            for s, win, o in zip(streams, windows, out_loop):
                eng.decode_window_device(s, window=win, reduce=r, out=o)

        def batch():
            _, out_batch["out"], _, status = eng.decode_windows_device(streams, windows if w["window"] else None, r, dtype=dt)
            assert all(rc == 0 for rc, _ in status)

        times, launches = timed_legs(L, (("loop", loop), ("batch", batch)), args.steps, args.warmup, torch)
        got = out_batch["out"]
        assert all(torch.equal(got[i], out_loop[i]) for i in range(n)), w["name"]
        px = sum(o.numel() // w["comps"] for o in out_loop)
        row = summary(times, launches, n, px)
        row["kernels_ms_per_call"], kernels, table = profiled(batch, args.profile_steps, GROUPS, torch)
        row["all_kernels_ms_per_call"] = kernels
        tables.append("== %s ==\n%s" % (w["name"], table))
        result["workloads"][w["name"]] = row
        eng.close()
        del out_loop, out_batch, got
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_window_batch_bench.json"), "w") as f:
            f.write(line + "\n")
        with open(os.path.join(args.out, "device_window_batch_bench_profile.txt"), "w") as f:
            f.write("\n\n".join(tables) + "\n")


if __name__ == "__main__":
    main()
