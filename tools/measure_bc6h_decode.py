#!/usr/bin/env python3
"""Hap HDR (BC6H) decoding on 3840x2160 frames, timed with CUDA events around the library's calls:
  * HapB200BlockDecodeHalfBatch, UF16 and SF16, on random all-mode batches (each block a random one of the 14 modes: the
    worst case for a per-mode branch) and picture-like batches (mode 11, tests/bc6h_util.pack_picture);
  * HapB200BlockDecodeBatch for Hap7 (BC7) and Hap5 (DXT5) on the same geometry, in the same run;
  * HapB200DecodeRGBAHalfBatch end to end (Snappy frames from HapEncode, 4 chunks).
Reports the median ms per frame and GB/s of pixels written (RGBA16F: 8 bytes per pixel; RGBA8: 4), with the card's name
and power limit.  Needs a CUDA device.
    python tools/measure_bc6h_decode.py [frames] [repeats]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bc6h_util as U  # noqa: E402
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
    """median ms of fn() over `repeats` calls, CUDA events on `stream` (two untimed calls first)"""
    for _ in range(2):
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
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 10
    if not torch.cuda.is_available():
        sys.exit("measure_bc6h_decode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream
    rng = np.random.default_rng(7)
    out = torch.empty((F, HALF), dtype=torch.uint8, device=dev)

    def rate(ms, frame_bytes):
        return {"ms_per_frame": round(ms / F, 4), "written_GBps": round(F * frame_bytes / (ms * 1e-3) / 1e9, 1)}

    def check(r):
        assert r == 0, r

    modes = rng.integers(0, U.NMODES, F * NB)
    mixed = rng.integers(0, 256, (F * NB, 16), dtype=np.uint8)
    for m in range(U.NMODES):
        sel = modes == m
        mixed[sel] = U.random_blocks(rng, int(sel.sum()), m)
    inputs = {"all_modes_random": {UF16: mixed, SF16: mixed}}
    pics = {s: [np.frombuffer(U.pack_picture(synth.frame(W, H, i, kind="video").numpy(), s == SF16), np.uint8).reshape(NB, 16)
                for i in range(min(F, 4))] for s in (UF16, SF16)}
    inputs["picture_mode11"] = {s: np.concatenate([pics[s][i % len(pics[s])] for i in range(F)]) for s in (UF16, SF16)}

    other = torch.from_numpy(rng.integers(0, 256, F * NB * 16, dtype=np.uint8)).to(dev)
    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H),
           "half_bytes_per_frame": HALF, "rgba8_bytes_per_frame": RGBA, "block_bytes_per_frame": 16 * NB,
           "block_decode": {}, "decode_rgba_half_batch": {}}
    for codec, name in ((L.HapB200Codec_Hap7, "Hap7"), (L.HapB200Codec_Hap5, "Hap5")):
        fn = lambda: check(lib.block_decode_batch(other.data_ptr(), F, 16 * NB, W, H, codec, out.data_ptr(), HALF, stream=sh))
        res["block_decode"][name + "_rgba8_random_blocks"] = rate(timed(fn, stream, repeats), RGBA)
    for name, per in inputs.items():
        for fmt, tag in ((UF16, "UF16"), (SF16, "SF16")):
            blocks = torch.from_numpy(per[fmt].reshape(-1)).to(dev)
            fn = lambda: check(lib.block_decode_half_batch(blocks.data_ptr(), F, 16 * NB, W, H, fmt, out.data_ptr(), HALF, stream=sh))
            res["block_decode"]["%s_%s" % (tag, name)] = rate(timed(fn, stream, repeats), HALF)

    # end to end: Snappy frames of each input
    max_len = lib.max_encoded_length([16 * NB], [UF16], [4])
    stride = (max_len + 15) // 16 * 16
    for name, per in inputs.items():
        for fmt, tag in ((UF16, "UF16"), (SF16, "SF16")):
            src = per[fmt].reshape(F, NB * 16)
            frames = []
            for f in range(F):
                r, fr = lib.encode([src[f].tobytes()], [fmt], [HapCompressorSnappy], [4])
                assert r == 0, r
                frames.append(fr)
            buf = np.zeros(F * stride, np.uint8)
            for f, fr in enumerate(frames):
                buf[f * stride: f * stride + len(fr)] = np.frombuffer(fr, np.uint8)
            d = torch.from_numpy(buf).to(dev)
            nbytes = torch.tensor([len(fr) for fr in frames], dtype=torch.int64, device=dev)
            results = torch.zeros(F, dtype=torch.int32, device=dev)
            torch.cuda.synchronize()
            fn = lambda: check(lib.decode_rgba_half_batch(d.data_ptr(), F, stride, nbytes.data_ptr(), 4, W, H, out.data_ptr(), HALF,
                                                          results.data_ptr(), stream=sh))
            ms = timed(fn, stream, repeats)
            assert (results.cpu() == 0).all()
            res["decode_rgba_half_batch"]["%s_%s" % (tag, name)] = dict(rate(ms, HALF),
                                                                        mean_frame_bytes=int(np.mean([len(fr) for fr in frames])))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
