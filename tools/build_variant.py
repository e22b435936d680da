"""Build an experimental variant of the library next to the product: python tools/build_variant.py NAME -DFOO -DBAR=2 ...
-> grok_b200/variants/NAME/libgrokj2k_plugin.so; run anything against it with B2K_LIB=<that path>.  For A/B runs of kernel
options in ONE GPU call (several variants, one bench each)."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from grok_b200 import build as B
name, defs = sys.argv[1], sys.argv[2:]
out = os.path.join(ROOT, "grok_b200", "variants", name)
os.makedirs(os.path.join(out, "obj"), exist_ok=True)
objs, procs = [], []
for src in B.SOURCES:
    obj = os.path.join(out, "obj", src + ".o")
    cmd = [B.NVCC] + B.FLAGS + defs + (["-x", "cu"] if src.endswith(".cu") else []) + ["-c", os.path.join(B.CSRC, src), "-o", obj]
    procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    objs.append(obj)
for src, p in procs:
    o, _ = p.communicate()
    if p.returncode:
        sys.stderr.write(o.decode()); raise SystemExit("nvcc failed on " + src)
lib = os.path.join(out, "libgrokj2k_plugin.so")
subprocess.check_call([B.NVCC, "-shared", "-o", lib] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-lpthread"])
print(lib)
