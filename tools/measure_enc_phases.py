#!/usr/bin/env python3
"""Where the fused Hap Q encoder that writes the frames spends its clocks (hapq_fused.cuh, HAPB200_ENC_PHASE_CLOCKS) on
bench.py's headline batch: 444 frames of 3840x2160 RGBA8 to Hap Q, 8 chunks, Snappy.  Builds the library with
-DHAPB200_ENC_PHASE_CLOCKS=1 (plus --flags, e.g. -DHAPB200_FUSED_WS=0 for hapq_fused_place_kernel) into a temporary
directory, encodes the batch --repeats times in a process of its own, and prints the clocks per fragment of every phase.
Thread 0 of the compressor takes the compressor's clocks (in hapq_fused_place_kernel it fits too); in hapq_ws_place_kernel
thread 0 of the fit group takes the fit group's.  A phase that ends at a barrier is its warp group's time; the fit in
hapq_fused_place_kernel ends at none, so there it is thread 0's own fit and the barrier behind it holds the wait for the
slowest thread.  The clocks of a measurement build are not those of the product (its extra stores and spills cost a little);
the split is what it is for.  Reports the card's name, power limit and SM clocks.  Needs a CUDA device.
    python tools/measure_enc_phases.py [--repeats 3] [--flags -DHAPB200_FUSED_WS=0] [--lib PATH]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# snappy_encode.cuh, kEp*
COMPRESSOR = ("fit", "fit_wait", "hash", "candidates", "propagation", "run_scan", "size_scan", "write", "look_back", "store", "other")
FIT_GROUP = ("group_fit", "group_empty_wait", "group_ticket")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else None


def child(repeats):
    import torch

    import bench
    import hap_b200
    from hap_b200.lib import HapB200Codec_HapY
    lib = hap_b200.load()
    read = lib.lib.HapB200EncodePhaseClocks
    read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    read.restype = C.c_int
    dev = torch.device("cuda", 0)
    A = bench.Roundtrip(lib, dev, bench.W, bench.H, HapB200Codec_HapY, bench.CHUNKS, 444)
    stream = torch.cuda.Stream(device=dev)
    sp = stream.cuda_stream
    A.encode(sp)
    torch.cuda.synchronize()
    slots = (C.c_ulonglong * 32)()
    read(slots, 32)                       # (warm-up encode dropped)
    with torch.cuda.stream(stream):
        for _ in range(repeats):
            A.encode(sp)
    n = read(slots, 32)
    A.decode(sp)
    A.check()
    names = COMPRESSOR + FIT_GROUP
    assert n == len(names) + 1, n
    clocks = dict(zip(names, (int(slots[i]) for i in range(len(names)))))
    frags = int(slots[len(names)])
    comp_total = sum(clocks[p] for p in COMPRESSOR)
    fit_total = sum(clocks[p] for p in FIT_GROUP)
    out = {"library": os.environ.get("HAPB200_LIBRARY"), "frames": A.F, "repeats": repeats, "card": card(),
           "fragments_per_batch": frags / repeats,
           "compressor_clocks_per_fragment": {p: round(clocks[p] / max(frags, 1)) for p in COMPRESSOR},
           "compressor_share": {p: round(clocks[p] / max(comp_total, 1), 4) for p in COMPRESSOR}}
    if fit_total:
        out["fit_group_clocks_per_fragment"] = {p: round(clocks[p] / max(frags, 1)) for p in FIT_GROUP}
        out["fit_group_share"] = {p: round(clocks[p] / fit_total, 4) for p in FIT_GROUP}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--flags", nargs="*", default=[], help="more nvcc flags of the measured build")
    ap.add_argument("--lib", help="a prebuilt -DHAPB200_ENC_PHASE_CLOCKS=1 library (default: built into a temporary directory)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.repeats)
        return
    from hap_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        lib = args.lib or build.build(extra_flags=["-DHAPB200_ENC_PHASE_CLOCKS=1"] + args.flags, out=os.path.join(tmp, "libhap_b200_phases.so"))
        env = dict(os.environ, HAPB200_LIBRARY=lib)
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--repeats", str(args.repeats)], env=env,
                           capture_output=True, text=True, cwd=ROOT)
        if p.returncode != 0:
            sys.exit(p.stdout[-2000:] + p.stderr[-4000:])
        r = json.loads(p.stdout.strip().splitlines()[-1])
    r["flags"] = args.flags
    print(json.dumps(r))


if __name__ == "__main__":
    main()
