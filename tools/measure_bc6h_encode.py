#!/usr/bin/env python3
"""Hap HDR (BC6H) encoding on 3840x2160 frames, timed with CUDA events around the library's calls:
  * HapB200BlockEncodeHalfBatch, UF16 and SF16, on HDR content (the synth.frame video class made linear at peak 64; for
    SF16 centred on zero: tests/bc6h_encode_util.hdr_content);
  * HapB200EncodeRGBAHalfBatch end to end (Snappy, 4 chunks);
  * HapB200BlockEncodeBatch with Hap5 (DXT5) on the same geometry, in the same run, for context.
Reports the median ms per frame, GB/s of half input (8 bytes per pixel; RGBA8 input for DXT5: 4), blocks per second,
and the card's name and power limit.  Needs a CUDA device.
    python tools/measure_bc6h_encode.py [frames] [repeats]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bc6h_encode_util as E  # noqa: E402
import hap_b200  # noqa: E402
import hap_b200.lib as L  # noqa: E402
from hap_b200 import synth  # noqa: E402
from hap_b200.abi import (HapCompressorSnappy, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT,  # noqa: E402
                          HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT)

W, H = 3840, 2160
NB = (W // 4) * (H // 4)
HALF, RGBA = 8 * W * H, 4 * W * H
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT


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
        sys.exit("measure_bc6h_encode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def rate(ms, in_bytes):
        return {"ms_per_frame": round(ms / F, 3), "input_GBps": round(F * in_bytes / (ms * 1e-3) / 1e9, 2),
                "blocks_per_s": round(F * NB / (ms * 1e-3) / 1e6, 2) * 1e6}

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H), "content": "video, peak 64",
           "block_encode_half": {}, "encode_rgba_half_batch": {}, "block_encode_rgba8": {}}
    blocks = torch.empty(F * NB * 16, dtype=torch.uint8, device=dev)
    for fmt, tag in ((UF16, "UF16"), (SF16, "SF16")):
        pics = [E.hdr_content("video", W, H, 64.0, fmt == SF16, i) for i in range(F)]
        src = torch.from_numpy(np.stack(pics).view(np.uint8).reshape(-1)).to(dev)
        fn = lambda: check(lib.block_encode_half_batch(src.data_ptr(), F, HALF, W, H, fmt, blocks.data_ptr(), NB * 16, stream=sh))
        res["block_encode_half"][tag] = rate(timed(fn, stream, repeats), HALF)
        ostride = (lib.max_encoded_length_half(W, H, fmt, 4) + 15) // 16 * 16
        out = torch.empty(F * ostride, dtype=torch.uint8, device=dev)
        used = torch.zeros(F, dtype=torch.int64, device=dev)
        fn = lambda: check(lib.encode_rgba_half_batch(src.data_ptr(), F, HALF, W, H, fmt, HapCompressorSnappy, 4, out.data_ptr(), ostride,
                                                      used.data_ptr(), stream=sh))
        ms = timed(fn, stream, repeats)
        res["encode_rgba_half_batch"][tag + "_snappy_4_chunks"] = dict(rate(ms, HALF), mean_frame_bytes=int(used.float().mean().item()))
        del src
    rgba = torch.from_numpy(np.stack([synth.frame(W, H, i, kind="video").numpy() for i in range(F)]).reshape(-1)).to(dev)
    fn = lambda: check(lib.block_encode_batch(rgba.data_ptr(), F, RGBA, W, H, L.HapB200Codec_Hap5, blocks.data_ptr(), NB * 16, stream=sh))
    res["block_encode_rgba8"]["Hap5_DXT5"] = rate(timed(fn, stream, repeats), RGBA)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
