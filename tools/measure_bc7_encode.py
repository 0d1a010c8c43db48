#!/usr/bin/env python3
"""Hap R (BC7) encoding on 3840x2160 frames, timed with CUDA events around the library's calls:
  * HapB200BlockEncodeBC7Batch on opaque synth "video" content and on the same class with alpha="ramp";
  * HapB200EncodeRGBABC7Batch end to end (Snappy, 4 chunks), opaque video;
  * HapB200BlockEncodeBatch with Hap5 (DXT5) on the same geometry, in the same run, for context.
Reports the median ms per frame, GB/s of RGBA8 input, blocks per second, and the card's name and power limit.  Needs a
CUDA device.
    python tools/measure_bc7_encode.py [frames] [repeats]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import hap_b200  # noqa: E402
import hap_b200.lib as L  # noqa: E402
from hap_b200 import synth  # noqa: E402
from hap_b200.abi import HapCompressorSnappy  # noqa: E402

W, H = 3840, 2160
NB = (W // 4) * (H // 4)
RGBA = 4 * W * H


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() if q.returncode == 0 else None}


def timed(fn, stream, repeats):
    """median ms of fn() over `repeats` calls, CUDA events on `stream` (one untimed call first)"""
    fn()
    ms = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    if not torch.cuda.is_available():
        sys.exit("measure_bc7_encode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def rate(ms):
        return {"ms_per_frame": round(ms / F, 3), "input_GBps": round(F * RGBA / (ms * 1e-3) / 1e9, 3),
                "blocks_per_s": round(F * NB / (ms * 1e-3) / 1e6, 3) * 1e6}

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H),
           "block_encode_bc7": {}, "encode_rgba_bc7_batch": {}, "block_encode_rgba8": {}}
    blocks = torch.empty(F * NB * 16, dtype=torch.uint8, device=dev)
    for alpha in ("opaque", "ramp"):
        src = torch.from_numpy(np.stack([synth.frame(W, H, i, kind="video", alpha=alpha).numpy() for i in range(F)]).reshape(-1)).to(dev)
        fn = lambda: check(lib.block_encode_bc7_batch(src.data_ptr(), F, RGBA, W, H, blocks.data_ptr(), NB * 16, stream=sh))
        res["block_encode_bc7"]["video_" + alpha] = rate(timed(fn, stream, repeats))
        if alpha == "opaque":
            ostride = (lib.max_encoded_length_rgba(W, H, L.HapB200Codec_Hap7, 4) + 15) // 16 * 16
            out = torch.empty(F * ostride, dtype=torch.uint8, device=dev)
            used = torch.zeros(F, dtype=torch.int64, device=dev)
            fn = lambda: check(lib.encode_rgba_bc7_batch(src.data_ptr(), F, RGBA, W, H, HapCompressorSnappy, 4, out.data_ptr(), ostride,
                                                         used.data_ptr(), stream=sh))
            ms = timed(fn, stream, repeats)
            res["encode_rgba_bc7_batch"]["video_opaque_snappy_4_chunks"] = dict(rate(ms), mean_frame_bytes=int(used.float().mean().item()))
            fn = lambda: check(lib.block_encode_batch(src.data_ptr(), F, RGBA, W, H, L.HapB200Codec_Hap5, blocks.data_ptr(), NB * 16,
                                                      stream=sh))
            res["block_encode_rgba8"]["Hap5_DXT5_video_opaque"] = rate(timed(fn, stream, repeats))
        del src
    print(json.dumps(res))


if __name__ == "__main__":
    main()
