"""Where k_ht_encode's cycles go, per phase, on config 2: python tools/enc_phases.py [NAME [-DFOO ...]]

Builds the variant NAME (default `phases`) with -DENC_PHASE_CLOCKS plus the given options through tools/build_variant.py,
unless grok_b200/variants/NAME/ already holds it, then runs config 2's block encoder (forward transform once, then encode
only, 20 calls) against it and prints, per phase, the clock64() cycles one warp spends on one code block, and the SM clock
while the kernel ran (warp cycles over %globaltimer nanoseconds).  A warp's cycles include the time it waits for its
scheduler, so the phases' sum is the latency of a block with all the kernel's warps resident, not the SM's cost of it."""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["setup", "staging", "in-lane coding", "MEL join", "scan", "MagSgn gather/drain", "VLC gather/drain", "termination"]
SLOTS = len(PHASES) + 3  # + blocks, warp cycles, warp nanoseconds (the PH_ enum of ht_enc.cu)


def run(steps=20):
    import numpy as np
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import grok_b200 as G
    import oracle_pipeline as P
    L = G.lib()
    L.b2k_enc_phase_clocks.argtypes = [C.POINTER(C.c_uint64), C.c_int32]
    L.b2k_enc_phase_clocks.restype = C.c_int32
    cp = G.make_coding(8192, 8192, 3, 12, numres=6, tile=(1024, 1024))
    img = P.synthetic_image(8192, 8192, 3, 12, 20260924)
    eng = G.Engine(0)
    job = eng.job(cp)
    job.upload(img)
    job.forward()
    for _ in range(3):
        job.t1_encode()
    buf = (C.c_uint64 * SLOTS)()
    if L.b2k_enc_phase_clocks(buf, SLOTS) != SLOTS:
        raise SystemExit("b2k_enc_phase_clocks failed (a library built without -DENC_PHASE_CLOCKS?)")
    ms = [job.t1_encode()[0] for _ in range(steps)]
    L.b2k_enc_phase_clocks(buf, SLOTS)
    v = [int(x) for x in buf]
    blocks, cyc, ns = v[len(PHASES)], v[len(PHASES) + 1], v[len(PHASES) + 2]
    print("library %s, %d encode calls, %d code blocks each" % (os.environ.get("B2K_LIB"), steps, blocks // steps))
    print("encode call (kernel + scan + compaction): median %.3f ms" % float(np.median(ms)))
    print("SM clock while k_ht_encode ran: %.0f MHz" % (1e3 * cyc / ns))
    print("%-22s %12s %7s" % ("phase", "cycles/block", "share"))
    tot = sum(v[:len(PHASES)])
    for name, c in zip(PHASES, v):
        print("%-22s %12.0f %6.1f%%" % (name, c / blocks, 100.0 * c / tot))
    print("%-22s %12.0f   (warp start to exit: %.0f)" % ("sum", tot / blocks, cyc / blocks))
    eng.close()


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "--run":
        return run()
    name = sys.argv[1] if len(sys.argv) > 1 else "phases"
    lib = os.path.join(ROOT, "grok_b200", "variants", name, "libgrokj2k_plugin.so")
    if not os.path.exists(lib):
        subprocess.check_call([sys.executable, os.path.join(ROOT, "tools", "build_variant.py"), name, "-DENC_PHASE_CLOCKS"]
                              + sys.argv[2:])
    subprocess.check_call([sys.executable, os.path.abspath(__file__), "--run"], env=dict(os.environ, B2K_LIB=lib))


if __name__ == "__main__":
    main()
