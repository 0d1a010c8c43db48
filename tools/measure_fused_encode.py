#!/usr/bin/env python3
"""A/B of the fused Hap Q encoder (hapq_fused.cuh, HAPB200_FUSED_HAPQ) on bench.py's headline batch: 444 frames of
3840x2160 RGBA8 to Hap Q, 8 chunks, Snappy.  Times HapB200EncodeRGBABatch and reports the per-stage share (CUDA events),
for the product library and for a build with -DHAPB200_FUSED_HAPQ=0 (the block encoder, then the fragment compressor).
Each variant runs in its own process (HAPB200_LIBRARY), the two alternate for `--rounds` rounds, and the encoded frames
are fingerprinted so that the variants can be seen to agree.  Reports the card's name, power limit and SM clocks.
Needs a CUDA device.
    python tools/measure_fused_encode.py [--rounds 3] [--repeats 10] [--fused-lib PATH] [--two-kernel-lib PATH]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


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
    dev = torch.device("cuda", 0)
    A = bench.Roundtrip(lib, dev, bench.W, bench.H, HapB200Codec_HapY, bench.CHUNKS, 444)
    stream = torch.cuda.Stream(device=dev)
    sp = stream.cuda_stream
    A.frames.zero_()   # the slack behind each frame enters the fingerprint
    torch.cuda.synchronize(dev)
    ms = bench.time_on_stream(torch, stream, lambda: A.encode(sp), repeats)
    A.decode(sp)
    A.check()
    used = A.used.cpu()
    f = A.frames.view(torch.int64)
    fp = [int(used.sum()), int(f.sum()), int(f[::7].sum())]   # fingerprint of the frames (wrapping sums)
    lib.set_stage_timing(True)
    lib.stage_times()
    with torch.cuda.stream(stream):
        for _ in range(3):
            A.encode(sp)
    st = lib.stage_times()
    lib.set_stage_timing(False)
    print(json.dumps({"library": os.environ.get("HAPB200_LIBRARY"), "frames": A.F, "mean_frame_bytes": A.mean_frame_bytes(),
                      "encode_ms_per_batch": ms, "stage_ms_per_batch": {k: v[0] / 3 for k, v in st.items() if v[0] > 0},
                      "fingerprint": fp, "card": card()}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--fused-lib", help="a prebuilt product library (default: hap_b200.build.build())")
    ap.add_argument("--two-kernel-lib", help="a prebuilt -DHAPB200_FUSED_HAPQ=0 library (default: built into a temporary directory)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.repeats)
        return
    from hap_b200 import build
    product = args.fused_lib or build.build()
    with tempfile.TemporaryDirectory() as tmp:
        two = args.two_kernel_lib or build.build(extra_flags=["-DHAPB200_FUSED_HAPQ=0"], out=os.path.join(tmp, "libhap_b200_two_kernel.so"))
        variants = {"fused": product, "two_kernel": two}
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
                         "fingerprints_agree": all(r["fingerprint"] == runs["fused"][0]["fingerprint"] for r in rs),
                         "cards": sorted({r["card"] for r in rs if r["card"]})}
    summary["detail"] = runs
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
