"""Batches of small images and code streams held in device memory: one Engine.decode_codestreams_device call against a
loop of decode_codestream_device, and one Engine.encode_codestreams_device call against a loop of
encode_codestream_device(device_output=True), one call per image.

    python tools/device_batch_bench.py [--steps K] [--warmup W] [--out DIR]

Workloads (streams from encode_codestream_device of seeded images, as CUDA tensors):
  256 x 512^2 x 3, 8 bit, 5/3, one tile, PLT
  64 x 1024^2 x 3, 12 bit
  1024 x 256^2 x 1, 16 bit
Legs, alternated step by step: `loop` (decode_codestream_device per stream into out[i]) and `batch` (one
decode_codestreams_device).  Each step is timed with the host clock around calls that return with their work done; the
first --warmup steps are not timed.  Both legs' pixels are checked against the source images.  Reports ms per batch,
images/s, Mpixel/s and the engine's launches per call, then, in a run of its own under torch.profiler, the batch leg's
parse kernels, arena gather, HT decode, inverse and conversion per batch.
Encode legs over the same images, alternated step by step: `loop` (encode_codestream_device(device_output=True) per
image) and `batch` (one encode_codestreams_device).  Both legs' streams must be byte-identical, and the batch's streams
must decode, through decode_codestreams_device, to the source images.  The same figures, then, under torch.profiler,
the batch leg's conversion, forward DWT, HT encode, T2 kernels and gather per batch, and the share of the batch's time
the kernels leave to the host.  Prints one JSON line with the GPU's name and power limit; --out DIR also writes it, and
the profiler's tables, there."""
import argparse
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
ENC_GROUPS = {"conversion": ("k_containers_to_planes",), "forward": ("k_dwt", "k_point_transform"), "ht_encode": ("k_ht_encode",),
              "t2": ("k_t2_",), "gather": ("k_ht_gather",)}


def timed_legs(L, legs, steps, warmup, torch):
    """legs: [(name, fn)] run alternately; returns (per-leg host-clock ms after the warmup steps, launches of the last call)"""
    times = {name: [] for name, _ in legs}
    launches = {}
    for step in range(warmup + steps):
        for leg, fn in legs:
            torch.cuda.synchronize()
            l0 = L.b2k_launch_count()
            t0 = time.perf_counter()
            fn()
            t1 = time.perf_counter()
            launches[leg] = int(L.b2k_launch_count() - l0)
            if step >= warmup:
                times[leg].append((t1 - t0) * 1e3)
    return times, launches


def summary(times, launches, n, px):
    row = {}
    for leg in times:
        ms = sorted(times[leg])[len(times[leg]) // 2]
        row[leg] = dict(ms=round(ms, 3), images_per_s=round(n / ms * 1e3, 1), mpixel_per_s=round(px / ms / 1e3, 1),
                        launches=launches[leg], ms_all=[round(t, 3) for t in times[leg]])
    row["speedup"] = round(row["loop"]["ms"] / row["batch"]["ms"], 2)
    return row


def profiled(fn, steps, groups, torch):
    """fn's kernels under torch.profiler, a run of its own: ms per call per group, all kernels' ms per call, the table"""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    per = {k: 0.0 for k in groups}
    total = 0.0
    for ev in prof.key_averages():
        if ev.device_time_total <= 0:
            continue
        total += ev.device_time_total / 1e3 / steps
        for k, pats in groups.items():
            if any(p in ev.key for p in pats):
                per[k] += ev.device_time_total / 1e3 / steps
    return {k: round(v, 3) for k, v in per.items()}, round(total, 3), prof.key_averages().table(sort_by="cuda_time_total", row_limit=25)


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

        times, launches = timed_legs(L, (("loop", loop), ("batch", batch)), args.steps, args.warmup, torch)
        assert torch.equal(out_loop, imgs) and torch.equal(out_batch, imgs), w["name"]
        px = w["n"] * w["size"] * w["size"]
        row = summary(times, launches, w["n"], px)
        # the batch leg's kernels under the profiler, a run of its own
        row["kernels_ms_per_batch"], _, table = profiled(batch, args.profile_steps, GROUPS, torch)
        tables.append("== %s ==\n%s" % (w["name"], table))
        result["workloads"][w["name"]] = row
        # encode: the same images into code streams, a loop of single calls against one batch call
        flags = 0
        for f in w["flags"].split("|"):
            flags |= getattr(G, "CS_" + f)
        got = {}

        def enc_loop():
            got["loop"] = [eng.encode_codestream_device(cp, imgs[i], flags, device_output=True) for i in range(w["n"])]

        def enc_batch():
            got["batch"], status = eng.encode_codestreams_device(cp, imgs, flags)
            assert all(rc == 0 for rc, _ in status)

        times, launches = timed_legs(L, (("loop", enc_loop), ("batch", enc_batch)), args.steps, args.warmup, torch)
        assert all(torch.equal(a, b) for a, b in zip(got["loop"], got["batch"])), w["name"]
        _, back, dstatus = eng.decode_codestreams_device(got["batch"], out=out_batch)
        assert all(rc == 0 for rc, _ in dstatus) and torch.equal(back, imgs), w["name"]
        enc = summary(times, launches, w["n"], px)
        enc["kernels_ms_per_batch"], kernels, table = profiled(enc_batch, args.profile_steps, ENC_GROUPS, torch)
        enc["all_kernels_ms_per_batch"] = kernels
        enc["host_share"] = round(max(0.0, 1 - kernels / enc["batch"]["ms"]), 3)
        tables.append("== %s encode ==\n%s" % (w["name"], table))
        row["encode"] = enc
        del got
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
