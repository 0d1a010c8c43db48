#!/usr/bin/env python3
"""A/B of the Snappy execute kernel's unit path (snappy_decode.cuh, HAPB200_EX_UNIT_PATH) on bench.py's headline batch:
444 frames of 3840x2160 Hap Q, 8 chunks, encoded on the device with the fragment index.  Times HapB200DecodeBatch with
the index and with it ignored (on-the-fly index), and the execute kernel's own share (per-stage CUDA events), for the
product library and for a build with -DHAPB200_EX_UNIT_PATH=0.  Each variant runs in its own process (HAPB200_LIBRARY),
the two alternate for `--rounds` rounds, and the decoded textures are fingerprinted so that the variants can be seen to
agree.  Reports the card's name, power limit and SM clocks.  Needs a CUDA device.
    python tools/measure_decode_paths.py [--rounds 3] [--repeats 10] [--unit-lib PATH] [--general-lib PATH]"""
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
    lib.set_option(lib.OPTION_WRITE_INDEX, 1)
    lib.set_option(lib.OPTION_USE_INDEX, 1)
    A = bench.Roundtrip(lib, dev, bench.W, bench.H, HapB200Codec_HapY, bench.CHUNKS, 444)
    stream = torch.cuda.Stream(device=dev)
    sp = stream.cuda_stream
    A.encode(sp)
    torch.cuda.synchronize()
    out = {"library": os.environ.get("HAPB200_LIBRARY"), "frames": A.F, "mean_frame_bytes": A.mean_frame_bytes()}

    def leg(use_index):
        lib.set_option(lib.OPTION_USE_INDEX, use_index)
        ms = bench.time_on_stream(torch, stream, lambda: A.decode(sp), repeats)
        A.check()
        t = A.tex[0].view(torch.int64)
        fp = [int(t.sum()), int(t[::7].sum())]   # fingerprint of the decoded textures (wrapping sums)
        lib.set_stage_timing(True)
        lib.stage_times()
        with torch.cuda.stream(stream):
            for _ in range(3):
                A.decode(sp)
        st = lib.stage_times()
        lib.set_stage_timing(False)
        lib.set_option(lib.OPTION_USE_INDEX, 1)
        return {"ms_per_batch": ms, "stage_ms_per_batch": {k: v[0] / 3 for k, v in st.items() if v[0] > 0}, "fingerprint": fp}

    out["with_index"] = leg(1)
    out["without_index"] = leg(0)
    out["card"] = card()
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--unit-lib", help="a prebuilt product library (default: hap_b200.build.build())")
    ap.add_argument("--general-lib", help="a prebuilt -DHAPB200_EX_UNIT_PATH=0 library (default: built into a temporary directory)")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        child(args.repeats)
        return
    from hap_b200 import build
    product = args.unit_lib or build.build()
    with tempfile.TemporaryDirectory() as tmp:
        general = args.general_lib or build.build(extra_flags=["-DHAPB200_EX_UNIT_PATH=0"], out=os.path.join(tmp, "libhap_b200_general.so"))
        variants = {"unit_path": product, "general_path": general}
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
        summary[name] = {leg: {"ms_per_batch": [round(r[leg]["ms_per_batch"], 3) for r in rs],
                               "snappy_decode_stage_ms": [round(r[leg]["stage_ms_per_batch"].get("snappy_decode", 0.0), 3) for r in rs],
                               "fingerprints_agree": all(r[leg]["fingerprint"] == runs["unit_path"][0][leg]["fingerprint"] for r in rs)}
                         for leg in ("with_index", "without_index")}
        summary[name]["cards"] = sorted({r["card"] for r in rs if r["card"]})
    summary["detail"] = runs
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
