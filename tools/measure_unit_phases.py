#!/usr/bin/env python3
"""Where the unit path of the Snappy decoder spends its clocks (snappy_decode.cuh, HAPB200_EX_PHASE_CLOCKS) on bench.py's
headline batch: 444 frames of 3840x2160 Hap Q, 8 chunks, encoded on the device with the fragment index.  Builds the library
with -DHAPB200_EX_PHASE_CLOCKS=1 (plus --flags, e.g. -DHAPB200_EX_UNIT_KERNEL=0) into a temporary directory, decodes the
batch --repeats times in a process of its own, and prints each phase's share of the summed CTA clocks, the clocks per unit
window and the pointer-jumping rounds per window.  Thread 0 of each CTA takes the clocks; a phase that ends without a
barrier (the walk) is thread 0's own time.  Reports the card's name, power limit and SM clocks.  Needs a CUDA device.
    python tools/measure_unit_phases.py [--repeats 5] [--flags -DHAPB200_EX_UNIT_KERNEL=0] [--lib PATH]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PHASES = ("ticket_and_stage_wait", "walk", "scans_and_checks", "records", "map", "jumping_rounds", "write", "other_windows")


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
    read = lib.lib.HapB200UnitPhaseClocks
    read.argtypes = [C.POINTER(C.c_ulonglong), C.c_int]
    read.restype = C.c_int
    dev = torch.device("cuda", 0)
    lib.set_option(lib.OPTION_WRITE_INDEX, 1)
    lib.set_option(lib.OPTION_USE_INDEX, 1)
    A = bench.Roundtrip(lib, dev, bench.W, bench.H, HapB200Codec_HapY, bench.CHUNKS, 444)
    stream = torch.cuda.Stream(device=dev)
    sp = stream.cuda_stream
    A.encode(sp)
    A.decode(sp)
    torch.cuda.synchronize()
    slots = (C.c_ulonglong * 16)()
    n = read(slots, 16)                   # (warm-up decode dropped)
    with torch.cuda.stream(stream):
        for _ in range(repeats):
            A.decode(sp)
    n = read(slots, 16)
    A.check()
    assert n == len(PHASES) + 2, n
    clocks = [int(slots[i]) for i in range(len(PHASES))]
    windows, rounds = int(slots[len(PHASES)]), int(slots[len(PHASES) + 1])
    total = sum(clocks)
    unit = sum(clocks[:7])
    out = {"library": os.environ.get("HAPB200_LIBRARY"), "frames": A.F, "repeats": repeats, "card": card(),
           "unit_windows_per_batch": windows / repeats, "rounds_per_unit_window": rounds / max(windows, 1),
           "share": {p: round(c / total, 4) for p, c in zip(PHASES, clocks)},
           "cta_clocks_per_unit_window": {p: round(c / max(windows, 1)) for p, c in zip(PHASES[:7], clocks[:7])},
           "unit_cta_clocks_per_window": round(unit / max(windows, 1))}
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--flags", nargs="*", default=[], help="more nvcc flags of the measured build")
    ap.add_argument("--lib", help="a prebuilt -DHAPB200_EX_PHASE_CLOCKS=1 library (default: built into a temporary directory)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.repeats)
        return
    from hap_b200 import build
    with tempfile.TemporaryDirectory() as tmp:
        lib = args.lib or build.build(extra_flags=["-DHAPB200_EX_PHASE_CLOCKS=1"] + args.flags, out=os.path.join(tmp, "libhap_b200_phases.so"))
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
