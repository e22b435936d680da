"""Batches of small code streams held in device memory: one Engine.decode_codestreams_device call against a loop of
decode_codestream_device, one call per stream.

    python tools/device_batch_bench.py [--steps K] [--warmup W] [--out DIR]

Workloads (streams from encode_codestream_device of seeded images, as CUDA tensors):
  256 x 512^2 x 3, 8 bit, 5/3, one tile, PLT
  64 x 1024^2 x 3, 12 bit
  1024 x 256^2 x 1, 16 bit
Legs, alternated step by step: `loop` (decode_codestream_device per stream into out[i]) and `batch` (one
decode_codestreams_device).  Each step is timed with the host clock around calls that return with their work done; the
first --warmup steps are not timed.  Both legs' pixels are checked against the source images.  Reports ms per batch,
images/s, Mpixel/s and the engine's launches per call, then, in a run of its own under torch.profiler, the batch leg's
parse kernels, arena gather, HT decode, inverse and conversion per batch.  Prints one JSON line with the GPU's name and
power limit; --out DIR also writes it, and the profiler's tables, there."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

WORKLOADS = [dict(name="256x512sq_rgb8", n=256, size=512, comps=3, prec=8, flags="PLT"),
             dict(name="64x1024sq_rgb12", n=64, size=1024, comps=3, prec=12, flags="TLM|PLT"),
             dict(name="1024x256sq_gray16", n=1024, size=256, comps=1, prec=16, flags="TLM|PLT")]
GROUPS = {"parse": ("k_t2_locate", "k_t2_plt", "k_t2_packets", "k_t2_walk", "k_t2_desc"), "gather": ("k_copy_table",),
          "ht_decode": ("k_ht_decode",), "inverse": ("k_dwt", "k_point_transform"), "conversion": ("k_planes_to_container",)}


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in out.split(",")]
        return name, power
    except Exception as e:  # the numbers still stand; say why the label is missing
        return "unknown (%s)" % e, "unknown"


def make(torch, G, w):
    flags = 0
    for f in w["flags"].split("|"):
        flags |= getattr(G, "CS_" + f)
    cp = G.make_coding(w["size"], w["size"], w["comps"], w["prec"], numres=6)
    g = torch.Generator(device="cuda").manual_seed(2026)
    dt = torch.uint8 if w["prec"] <= 8 else torch.int16 if w["prec"] < 16 else torch.int32
    imgs = torch.randint(0, 1 << w["prec"], (w["n"], w["comps"], w["size"], w["size"]), dtype=torch.int32, device="cuda",
                         generator=g)
    imgs = imgs.to(torch.uint8) if w["prec"] <= 8 else imgs.to(torch.uint16) if w["prec"] <= 16 else imgs
    eng = G.Engine(0)
    streams = [eng.encode_codestream_device(cp, imgs[i], flags, device_output=True) for i in range(w["n"])]
    eng.close()
    return cp, imgs, streams


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--profile-steps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    import grok_b200 as G
    L = G.lib()
    L.b2k_launch_count.restype = C.c_uint64
    name, power = gpu_info()
    result = dict(gpu=name, power_limit=power, steps=args.steps, warmup=args.warmup, workloads={})
    tables = []
    for w in WORKLOADS:
        cp, imgs, streams = make(torch, G, w)
        eng = G.Engine(0)
        out_loop, out_batch = torch.empty_like(imgs), torch.empty_like(imgs)

        def loop():
            for i, s in enumerate(streams):
                eng.decode_codestream_device(s, out=out_loop[i])

        def batch():
            _, _, status = eng.decode_codestreams_device(streams, out=out_batch)
            assert all(rc == 0 for rc, _ in status)

        times = {"loop": [], "batch": []}
        launches = {}
        for step in range(args.warmup + args.steps):
            for leg, fn in (("loop", loop), ("batch", batch)):
                torch.cuda.synchronize()
                l0 = L.b2k_launch_count()
                t0 = time.perf_counter()
                fn()
                t1 = time.perf_counter()
                launches[leg] = int(L.b2k_launch_count() - l0)
                if step >= args.warmup:
                    times[leg].append((t1 - t0) * 1e3)
        assert torch.equal(out_loop, imgs) and torch.equal(out_batch, imgs), w["name"]
        px = w["n"] * w["size"] * w["size"]
        row = {}
        for leg in ("loop", "batch"):
            ms = sorted(times[leg])[len(times[leg]) // 2]
            row[leg] = dict(ms=round(ms, 3), images_per_s=round(w["n"] / ms * 1e3, 1), mpixel_per_s=round(px / ms / 1e3, 1),
                            launches=launches[leg], ms_all=[round(t, 3) for t in times[leg]])
        row["speedup"] = round(row["loop"]["ms"] / row["batch"]["ms"], 2)
        # the batch leg's kernels under the profiler, a run of its own
        from torch.profiler import profile, ProfilerActivity
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(args.profile_steps):
                batch()
            torch.cuda.synchronize()
        per = {k: 0.0 for k in GROUPS}
        for ev in prof.key_averages():
            for k, pats in GROUPS.items():
                if any(p in ev.key for p in pats):
                    per[k] += ev.device_time_total / 1e3 / args.profile_steps
        row["kernels_ms_per_batch"] = {k: round(v, 3) for k, v in per.items()}
        tables.append("== %s ==\n%s" % (w["name"], prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)))
        result["workloads"][w["name"]] = row
        eng.close()
        del imgs, streams, out_loop, out_batch
        torch.cuda.empty_cache()
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "device_batch_bench.json"), "w") as f:
            f.write(line + "\n")
        with open(os.path.join(args.out, "device_batch_bench_profile.txt"), "w") as f:
            f.write("\n\n".join(tables) + "\n")


if __name__ == "__main__":
    main()
