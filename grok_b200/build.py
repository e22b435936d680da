"""Build libgrokj2k_plugin.so (CUDA kernels + C ABI) in-tree with nvcc for sm_90a (H100)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libgrokj2k_plugin.so")
SOURCES = ["engine.cu", "dwt.cu", "ht_enc.cu", "ht_dec.cu", "geometry.cpp", "plugin.cpp", "plugin_decode.cpp", "host_pack.cpp", "codestream.cpp", "stream.cpp", "plugin_batch.cpp", "t2_device.cu", "t2_decode.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# host code: no contraction into FMAs, so that the quality-factor step tables (geometry.cpp) are the same on every target
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
         "-Xcompiler", "-fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function,-ffp-contract=off", "--use_fast_math=false"]
FLAGS = [f for f in FLAGS if not f.startswith("--use_fast_math")]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "grok_b200.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(HERE, "build", src + ".o")
        cmd = [NVCC] + FLAGS + (["-x", "cu"] if src.endswith(".cu") else []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError("nvcc failed on " + src)
        if verbose and out:
            print(out.decode())
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-lpthread"]
    subprocess.check_call(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
