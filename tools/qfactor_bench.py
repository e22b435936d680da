#!/usr/bin/env python3
"""Quality-factor operating points on one GPU: an 8192 x 8192 x 3 12-bit image (9/7 + ICT, 1024 x 1024 tiles, 64 x 64
blocks, 6 resolutions) encoded at --qfactor 50 / 75 / 90 / 100 with encode_codestream_device(device_output=True) and
decoded back with decode_codestream_device.  Prints one JSON line per quality factor: median device-event times over
--iters warmed calls, code-stream bytes, bits per sample and PSNR against the source, with the card's name and power limit
read in the same run.

    python tools/qfactor_bench.py [--size 8192] [--iters 5] [--qfactors 50,75,90,100]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import grok_b200 as G  # noqa: E402


def card():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True)
        name, limit = [s.strip() for s in out.splitlines()[0].split(",")]
        return name, limit
    except (OSError, subprocess.CalledProcessError, ValueError):
        import torch
        return torch.cuda.get_device_name(0), "not measured"


def timed(torch, fn, iters):
    ms = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        r = fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=8192)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--qfactors", default="50,75,90,100")
    a = ap.parse_args()
    import torch
    name, limit = card()
    n, prec = a.size, 12
    g = torch.Generator(device="cuda").manual_seed(20261018)
    y, x = torch.meshgrid(torch.arange(n, device="cuda"), torch.arange(n, device="cuda"), indexing="ij")
    img = torch.stack([((x * (3 + c) + y * (5 - c)) // 16 + (64 * torch.sin((x + 2 * y) / (97.0 + 13 * c))).long()
                        + torch.randint(0, 32, (n, n), device="cuda", generator=g)) % (1 << prec) for c in range(3)])
    img = img.to(torch.int32).contiguous()
    eng = G.Engine(0)
    for q in [int(v) for v in a.qfactors.split(",")]:
        cp = G.make_coding(n, n, 3, prec, numres=6, tile=(1024, 1024), irreversible=True, qfactor=q)
        enc = lambda: eng.encode_codestream_device(cp, img, device_output=True)
        cs = enc()                                                              # warm-up
        enc_ms, cs = timed(torch, enc, a.iters)
        out = torch.empty_like(img)
        dec = lambda: eng.decode_codestream_device(cs, out=out)
        dec()
        dec_ms, _ = timed(torch, dec, a.iters)
        mse = torch.mean((out.double() - img.double()) ** 2).item()
        psnr = 10 * np.log10(((1 << prec) - 1) ** 2 / max(mse, 1e-12))
        print(json.dumps({"qfactor": q, "size": [n, n, 3], "prec": prec, "encode_ms": round(enc_ms, 2), "decode_ms": round(dec_ms, 2),
                          "bytes": int(cs.numel()), "bits_per_sample": round(8.0 * cs.numel() / (3 * n * n), 4),
                          "psnr_db": round(psnr, 2), "gpu": name, "power_limit": limit}), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
