#!/usr/bin/env python3
"""Block encoding from planar Y'CbCr on 3840x2160 frames, timed with CUDA events around the library's calls, all in one run:
  * HapB200BlockEncodePlanarBatch from 4:2:0 8-bit (yuv420p), 4:2:2 10-bit (yuv422p10le) and 4:4:4 12-bit with alpha
    (yuva444p12le);
  * HapB200BlockEncodeYUVBatch from NV12 and P010 (the semi-planar 4:2:0 sources);
  * HapB200BlockEncodeBatch from RGBA8 (the block encode alone);
for Hap1, Hap5, HapY and HapM, on synth "video" content (BT.709, limited range; alpha a ramp with detail).  The calls are
alternated so that clocks and neighbours weigh on each alike.  Reports median ms per frame and the card's name and power
limit.  Needs a CUDA device.
    python tools/measure_planar_encode.py [frames] [repeats] [rounds]"""
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

W, H = 3840, 2160
CS = L.HapB200YUV_BT709_Limited
KR, KB = 0.2126, 0.0722
CODECS = (("Hap1", L.HapB200Codec_Hap1), ("Hap5", L.HapB200Codec_Hap5), ("HapY", L.HapB200Codec_HapY), ("HapM", L.HapB200Codec_HapM))


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


def to_planes(rgba, n, fy, fx):
    """(F, H, W, 4) uint8 -> luma (F, H, W), Cb and Cr (F, H/fy, W/fx), alpha (F, H, W) at depth n: uint8, or int16 words"""
    s = 1 << (n - 8)
    top = (1 << n) - 1
    rgb = rgba[..., :3].float() / 255.0
    ey = KR * rgb[..., 0] + (1 - KR - KB) * rgb[..., 1] + KB * rgb[..., 2]
    pb = (rgb[..., 2] - ey) / (2 * (1 - KB))
    pr = (rgb[..., 0] - ey) / (2 * (1 - KR))
    foot = lambda p: p.reshape(p.shape[0], H // fy, fy, W // fx, fx).mean(dim=(2, 4))
    q = lambda v: torch.round(v).clamp(0, top).to(torch.int32)
    planes = [q(16 * s + 219 * s * ey), q((1 << (n - 1)) + 224 * s * foot(pb)), q((1 << (n - 1)) + 224 * s * foot(pr)),
              q(rgba[..., 3].float() * top / 255.0)]
    return [p.to(torch.uint8) if n == 8 else p.to(torch.int16) for p in planes]


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 9
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 3
    if not torch.cuda.is_available():
        sys.exit("measure_planar_encode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "rounds": rounds, "geometry": "%dx%d" % (W, H),
           "color_space": "BT.709 limited"}
    rgba = torch.from_numpy(np.stack([synth.frame(W, H, i, kind="video").numpy() for i in range(F)])).to(dev)
    ramp = (torch.arange(W, device=dev).view(1, 1, W) * 255 // (W - 1) + torch.arange(H, device=dev).view(1, H, 1) % 7)
    rgba[..., 3] = ramp.clamp(max=255).to(torch.uint8)
    blocks = torch.empty(F * (W // 4) * (H // 4) * 24, dtype=torch.uint8, device=dev)

    # the sources: name -> callable(codec, texture bytes) that encodes all F frames on `stream`
    sources = {"rgba8": lambda c, t: check(lib.block_encode_batch(rgba.data_ptr(), F, 4 * W * H, W, H, c, blocks.data_ptr(), t, stream=sh))}
    keep = []
    for name, n in (("nv12", 8), ("p010", 10)):
        y, cb, cr, _ = to_planes(rgba, n, 2, 2)
        if n == 10:
            y, cb, cr = [(p.to(torch.int32) << 6).to(torch.int16) for p in (y, cb, cr)]   # P010: the sample in the high bits
        sb = 1 if n == 8 else 2
        pitch, fstride = W * sb, W * sb * H * 3 // 2
        buf = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
        v = buf.view(F, fstride)
        v[:, : pitch * H] = y.reshape(F, -1).view(torch.uint8)
        v[:, pitch * H:] = torch.stack([cb, cr], -1).reshape(F, -1).view(torch.uint8)
        keep.append(buf)
        layout = L.HapB200YUV_NV12 if n == 8 else L.HapB200YUV_P010
        lp, cp = buf.data_ptr(), buf.data_ptr() + pitch * H
        sources[name] = (lambda lp, cp, pitch, fstride, layout: lambda c, t: check(
            lib.block_encode_yuv_batch(lp, cp, F, fstride, W, H, pitch, layout, CS, c, blocks.data_ptr(), t, stream=sh)))(
            lp, cp, pitch, fstride, layout)
    for name, sub, n, fy, fx, alpha in (("yuv420p", L.HapB200Chroma_420, 8, 2, 2, False), ("yuv422p10le", L.HapB200Chroma_422, 10, 1, 2, False),
                                        ("yuva444p12le", L.HapB200Chroma_444, 12, 1, 1, True)):
        planes = to_planes(rgba, n, fy, fx)
        sb = 1 if n == 8 else 2
        # one frame after another in each plane; the planes in buffers of their own (frame stride: the luma plane's size)
        fstride = W * sb * H
        bufs = []
        for p in planes:
            b = torch.zeros(F * fstride, dtype=torch.uint8, device=dev)
            flat = p.reshape(F, -1).view(torch.uint8)
            b.view(F, fstride)[:, : flat.shape[1]] = flat
            bufs.append(b)
        keep += bufs
        ptrs = [b.data_ptr() for b in bufs]
        if not alpha:
            ptrs[3] = 0
        lpitch, cpitch = W * sb, (W // fx) * sb
        sources[name] = (lambda ptrs, fstride, lpitch, cpitch, sub, n: lambda c, t: check(
            lib.block_encode_planar_batch(*ptrs, F, fstride, W, H, lpitch, cpitch, sub, n, CS, c, blocks.data_ptr(), t, stream=sh)))(
            ptrs, fstride, lpitch, cpitch, sub, n)
    torch.cuda.synchronize()
    for cname, codec in CODECS:
        t = lib.texture_bytes(W, H, codec, 0) + lib.texture_bytes(W, H, codec, 1)   # per frame (HapM: + the RGTC1 plane)
        row = {}
        for _ in range(rounds):
            for sname, fn in sources.items():
                row.setdefault(sname, []).append(timed(lambda: fn(codec, t), stream, repeats) / F)
        res["%s_ms_per_frame" % cname] = {k: {"median": round(float(np.median(v)), 4), "min": round(min(v), 4), "max": round(max(v), 4)}
                                          for k, v in row.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
