#!/usr/bin/env python3
"""A/B of the fused Hap Q encoder with its fit and compressor in warp groups of their own (hapq_fused.cuh,
hapq_ws_place_kernel, HAPB200_FUSED_WS) on bench.py's headline batch: 444 frames of 3840x2160 RGBA8 to Hap Q, 8 chunks,
Snappy.  Times HapB200EncodeRGBABatch and reports the per-stage share (CUDA events), for the product library and for a
build with -DHAPB200_FUSED_WS=0 (hapq_fused_place_kernel: every thread fits, then compresses).  Each variant runs in its
own process (HAPB200_LIBRARY), the two alternate for `--rounds` rounds, and the encoded frames are fingerprinted so that
the variants can be seen to agree.  Reports the card's name, power limit and SM clocks.  Needs a CUDA device.
    python tools/measure_fused_ws.py [--rounds 3] [--repeats 10] [--ws-lib PATH] [--fused-lib PATH]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from measure_fused_encode import card, child  # noqa: E402  (same child: time, fingerprint, stage events)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--ws-lib", help="a prebuilt product library (default: hap_b200.build.build())")
    ap.add_argument("--fused-lib", help="a prebuilt -DHAPB200_FUSED_WS=0 library (default: built into a temporary directory)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.repeats)
        return
    from hap_b200 import build
    product = args.ws_lib or build.build()
    with tempfile.TemporaryDirectory() as tmp:
        fused = args.fused_lib or build.build(extra_flags=["-DHAPB200_FUSED_WS=0"], out=os.path.join(tmp, "libhap_b200_fused.so"))
        variants = {"warp_groups": product, "fused_place": fused}
        runs = {k: [] for k in variants}
        for _ in range(args.rounds):
            for name, path in variants.items():
                env = dict(os.environ, HAPB200_LIBRARY=path)
                p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--repeats", str(args.repeats)], env=env,
                                   capture_output=True, text=True, cwd=ROOT)
                if p.returncode != 0:
                    sys.exit(p.stdout[-2000:] + p.stderr[-4000:])
                runs[name].append(json.loads(p.stdout.strip().splitlines()[-1]))
    summary = {"card_before": card(), "rounds": args.rounds, "repeats": args.repeats}
    for name, rs in runs.items():
        summary[name] = {"encode_ms_per_batch": [round(r["encode_ms_per_batch"], 3) for r in rs],
                         "stage_ms_per_batch": [{k: round(v, 3) for k, v in r["stage_ms_per_batch"].items()} for r in rs],
                         "fingerprints_agree": all(r["fingerprint"] == runs["warp_groups"][0]["fingerprint"] for r in rs),
                         "cards": sorted({r["card"] for r in rs if r["card"]})}
    summary["detail"] = runs
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
