#!/usr/bin/env python3
"""Hap R (BC7) decoding on 3840x2160 frames, timed with CUDA events around the library's calls:
  * HapB200BlockDecodeBatch for Hap7 next to Hap5 (DXT5, the same 16-byte blocks) on the same geometry, in the same run;
  * HapB200DecodeRGBABatch end to end (Snappy frames from HapEncode, 4 chunks).
Three inputs: one-mode batches (every block of the batch in one mode), random all-mode batches (each block a random mode:
the worst case for a per-mode branch) and picture-like batches (mode 6, tests/bc7_util.pack_picture).  Reports ms per frame
and GB/s of RGBA written, with the card's name and power limit.  Needs a CUDA device.
    python tools/measure_bc7_decode.py [frames] [repeats]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import bc7_util as U  # noqa: E402
import hap_b200  # noqa: E402
import hap_b200.lib as L  # noqa: E402
from hap_b200 import synth  # noqa: E402
from hap_b200.abi import HapCompressorSnappy, HapTextureFormat_RGBA_BPTC_UNORM  # noqa: E402

W, H = 3840, 2160
NB = (W // 4) * (H // 4)
RGBA = 4 * W * H


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
        sys.exit("measure_bc7_decode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream
    rng = np.random.default_rng(7)
    rgba = torch.empty((F, H, W, 4), dtype=torch.uint8, device=dev)

    def rate(ms):
        return {"ms_per_frame": round(ms / F, 4), "rgba_GBps": round(F * RGBA / (ms * 1e-3) / 1e9, 1)}

    def block_decode(codec, blocks):
        return lambda: lib.block_decode_batch(blocks.data_ptr(), F, 16 * NB, W, H, codec, rgba.data_ptr(), RGBA, stream=sh)

    def check(r):
        assert r == 0, r

    inputs = {}
    for m in range(8):
        inputs["mode%d" % m] = np.concatenate([U.random_blocks(rng, NB, m) for _ in range(F)])
    modes = rng.integers(0, 8, F * NB)
    mixed = rng.integers(0, 256, (F * NB, 16), dtype=np.uint8)
    for m in range(8):
        sel = modes == m
        mixed[sel] = U.random_blocks(rng, int(sel.sum()), m)
    inputs["all_modes_random"] = mixed
    pics = [np.frombuffer(U.pack_picture(synth.frame(W, H, i, kind="video", alpha="ramp").numpy()), np.uint8).reshape(NB, 16)
            for i in range(min(F, 4))]
    inputs["picture_mode6"] = np.concatenate([pics[i % len(pics)] for i in range(F)])

    dxt5 = torch.from_numpy(rng.integers(0, 256, F * NB * 16, dtype=np.uint8)).to(dev)
    out = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H),
           "rgba_bytes_per_frame": RGBA, "block_bytes_per_frame": 16 * NB, "block_decode": {}, "decode_rgba_batch": {}}
    for name, blocks_np in inputs.items():
        blocks = torch.from_numpy(blocks_np.reshape(-1)).to(dev)
        f7, f5 = block_decode(L.HapB200Codec_Hap7, blocks), block_decode(L.HapB200Codec_Hap5, dxt5)
        # Hap7 and Hap5 alternate, twice, in the same run
        t7 = [timed(lambda: check(f7()), stream, repeats) for _ in range(2)]
        t5 = [timed(lambda: check(f5()), stream, repeats) for _ in range(2)]
        out["block_decode"][name] = {"Hap7": rate(min(t7)), "Hap5_same_geometry": rate(min(t5)),
                                     "Hap7_over_Hap5": round(min(t7) / min(t5), 3)}

    # end to end: Snappy frames of each input's first frames
    max_len = lib.max_encoded_length_rgba(W, H, L.HapB200Codec_Hap7, 4)
    stride = (max_len + 15) // 16 * 16
    for name in ("mode6", "all_modes_random", "picture_mode6"):
        src = inputs[name].reshape(F, NB * 16)
        frames = []
        for f in range(F):
            r, fr = lib.encode([src[f].tobytes()], [HapTextureFormat_RGBA_BPTC_UNORM], [HapCompressorSnappy], [4])
            assert r == 0, r
            frames.append(fr)
        buf = np.zeros(F * stride, np.uint8)
        for f, fr in enumerate(frames):
            buf[f * stride: f * stride + len(fr)] = np.frombuffer(fr, np.uint8)
        d = torch.from_numpy(buf).to(dev)
        nbytes = torch.tensor([len(fr) for fr in frames], dtype=torch.int64, device=dev)
        res = torch.zeros(F, dtype=torch.int32, device=dev)
        torch.cuda.synchronize()
        fn = lambda: check(lib.decode_rgba_batch(d.data_ptr(), F, stride, nbytes.data_ptr(), 4, L.HapB200Codec_Hap7, W, H,
                                                 rgba.data_ptr(), RGBA, res.data_ptr(), stream=sh))
        ms = timed(fn, stream, repeats)
        assert (res.cpu() == 0).all()
        out["decode_rgba_batch"][name] = dict(rate(ms), mean_frame_bytes=int(np.mean([len(fr) for fr in frames])))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
