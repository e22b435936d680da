"""Per-level wavelet kernel times of config 2 under torch.profiler, for the library in B2K_LIB (or the product):
python tools/dwt_level_times.py [steps]  -- prints one JSON line: the GPU, its power limit, and per direction and level the
mean kernel time in ms.  A step launches the forward levels finest first and the inverse levels coarsest first, one launch
per level (config 2 has one launch group per level), so the launch order within a step names the level."""
import json, os, subprocess, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch
from torch.profiler import ProfilerActivity, profile
import grok_b200 as G
import oracle_pipeline as P

steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
W = H = 8192
L = 5
cp = G.make_coding(W, H, 3, 12, numres=L + 1, tile=(1024, 1024))
eng = G.Engine(0)
job = eng.job(cp)
job.upload(P.synthetic_image(W, H, 3, 12, 20260924))
for _ in range(3):
    job.roundtrip()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    job.roundtrip_n(steps)
kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "k_dwt" in e.name),
              key=lambda e: e.time_range.start)
out = {}
for dirn, tag, order in (("fwd", "_fwd", range(1, L + 1)), ("inv", "_inv", range(L, 0, -1))):
    ev = [e for e in kern if tag in e.name]
    assert len(ev) == steps * L, (dirn, len(ev))
    ms = np.array([(e.time_range.end - e.time_range.start) / 1e3 for e in ev]).reshape(steps, L).mean(0)
    out[dirn] = {"level%d" % lvl: round(float(t), 4) for lvl, t in zip(order, ms)}
    out[dirn]["sum"] = round(float(ms.sum()), 4)
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
print(json.dumps({"lib": os.environ.get("B2K_LIB", "product"), "gpu": gpu, "steps": steps, "dwt_ms": out}))
job.close()
eng.close()
