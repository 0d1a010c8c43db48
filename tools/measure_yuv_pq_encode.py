#!/usr/bin/env python3
"""Hap HDR block encoding from HDR10 P010 (BT.2020, PQ) on 3840x2160 frames, timed with CUDA events around the library's
calls, all in one run:
  * HapB200BlockEncodeYUVPQBatch (the conversion fused into the BC6H encoder's load);
  * the two-pass path a caller would otherwise write: a torch P010 -> RGBA16F conversion (the same definition: integer
    matrix to 12 bits, then the PQ table) into an RGBA16F batch, then HapB200BlockEncodeHalfBatch.
UF16 and SF16, synth "video" content made linear and scaled to 0.005-4000 cd/m2, BT.2020 limited range, unitNits 203.  The
fused and the two-pass textures are compared byte for byte.  Reports median ms per frame and the card's name and power
limit, read in the same run.  Needs a CUDA device.
    python tools/measure_yuv_pq_encode.py [frames] [repeats]"""
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
from hap_b200.abi import HapTextureFormat_RGB_BPTC_SIGNED_FLOAT, HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT  # noqa: E402

W, H = 3840, 2160
NB = (W // 4) * (H // 4)
CS, UNIT = L.HapB200YUV_BT2020_Limited, 203
KR, KB = 0.2627, 0.0593
# HAPB200_YUV_PQ_COEFFICIENTS row of BT.2020 limited: {cy, crR, cbG, crG, cbB, yOff, cOff}
K = (306358, 55209, -6161, -21391, 70440, 64, 512)
M1, M2, C1, C2, C3 = 2610 / 16384, 2523 / 32, 3424 / 4096, 2413 / 128, 2392 / 128


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


def pq_table(unit):
    """T of include/hap_b200.h in float64, rounded once to binary16 by numpy"""
    e = (np.arange(4096) / 4095.0) ** (1 / M2)
    return (10000 * (np.maximum(e - C1, 0) / (C2 - C3 * e)) ** (1 / M1) / unit).astype(np.float16)


def to_p010(src):
    """(F, H, W, 4) uint8 synth frames -> tight P010 planes (luma (F, H, W), chroma (F, H/2, W) int16 words): linear light
    0.005-4000 cd/m2, PQ, BT.2020 limited range, 2 x 2 chroma means"""
    lin = (src[..., :3].double() / 255.0) ** 2.2
    y = ((0.005 + (4000 - 0.005) * lin) / 10000).clamp(0, 1) ** M1
    sig = ((C1 + C2 * y) / (1 + C3 * y)) ** M2
    ey = KR * sig[..., 0] + (1 - KR - KB) * sig[..., 1] + KB * sig[..., 2]
    pb = (sig[..., 2] - ey) / (2 * (1 - KB))
    pr = (sig[..., 0] - ey) / (2 * (1 - KR))
    quad = lambda p: p.reshape(p.shape[0], H // 2, 2, W // 2, 2).mean(dim=(2, 4))
    yl = torch.round(64 + 876 * ey).clamp(0, 1023).to(torch.int32)
    c = torch.stack([quad(pb), quad(pr)], -1).reshape(-1, H // 2, W)
    c = torch.round(512 + 896 * c).clamp(0, 1023).to(torch.int32)
    return (yl << 6).to(torch.int16), (c << 6).to(torch.int16)


def torch_p010_to_rgba_half(luma, chroma, table, out):
    """the conversion of include/hap_b200.h in eager torch ops, into out (F, H, W, 4) float16"""
    yv = (luma.to(torch.int32) & 0xFFFF) >> 6
    c = ((chroma.to(torch.int32) & 0xFFFF) >> 6).reshape(-1, H // 2, W // 2, 2)
    j = torch.arange(H, device=luma.device) // 2
    rn = torch.where(torch.arange(H, device=luma.device) % 2 == 1, j + 1, j - 1).clamp(0, H // 2 - 1)
    v = 3 * c[:, j] + c[:, rn]
    i = torch.arange(W, device=luma.device) // 2
    cn = (i + 1).clamp(max=W // 2 - 1)
    odd = (torch.arange(W, device=luma.device) % 2 == 1).view(1, 1, W, 1)
    c8 = torch.where(odd, v[:, :, i] + v[:, :, cn], 2 * v[:, :, i]) - 8 * K[6]
    yd = K[0] * (yv - K[5])
    cb, cr = c8[..., 0], c8[..., 1]
    out[..., 0] = table[((yd + K[1] * cr + 32768) >> 16).clamp(0, 4095)]
    out[..., 1] = table[((yd + K[2] * cb + K[3] * cr + 32768) >> 16).clamp(0, 4095)]
    out[..., 2] = table[((yd + K[4] * cb + 32768) >> 16).clamp(0, 4095)]
    out[..., 3] = 1.0


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    if not torch.cuda.is_available():
        sys.exit("measure_yuv_pq_encode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H), "color_space": "BT.2020 limited",
           "unit_nits": UNIT}
    src = torch.from_numpy(np.stack([synth.frame(W, H, i, kind="video").numpy() for i in range(F)])).to(dev)
    luma, chroma = to_p010(src)
    del src
    pitch, fstride = 2 * W, 2 * W * H * 3 // 2
    planes = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
    pv = planes.view(F, fstride)
    pv[:, : pitch * H] = luma.reshape(F, -1).view(torch.uint8)
    pv[:, pitch * H:] = chroma.reshape(F, -1).view(torch.uint8)
    lp, cp = planes.data_ptr(), planes.data_ptr() + pitch * H
    table = torch.from_numpy(pq_table(UNIT)).to(dev)
    rgba = torch.empty((F, H, W, 4), dtype=torch.float16, device=dev)
    blocks = torch.empty(F * NB * 16, dtype=torch.uint8, device=dev)
    ref = torch.empty(F * NB * 16, dtype=torch.uint8, device=dev)
    for fname, fmt in (("UF16", HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT), ("SF16", HapTextureFormat_RGB_BPTC_SIGNED_FLOAT)):
        fused = lambda: check(lib.block_encode_yuv_pq_batch(lp, cp, F, fstride, W, H, pitch, CS, UNIT, fmt, blocks.data_ptr(), NB * 16,
                                                            stream=sh))
        half_only = lambda: check(lib.block_encode_half_batch(rgba.data_ptr(), F, 8 * W * H, W, H, fmt, ref.data_ptr(), NB * 16, stream=sh))

        def conversion():
            with torch.cuda.stream(stream):
                torch_p010_to_rgba_half(luma, chroma, table, rgba)

        def two_pass():
            conversion()
            half_only()
        row = {}
        for _ in range(2):   # alternate, so that clocks weigh on both alike
            for name, fn in (("fused_yuv_pq_block_encode", fused), ("two_pass_torch_then_half", two_pass),
                             ("torch_conversion_alone", conversion)):
                row.setdefault(name, []).append(timed(fn, stream, repeats) / F)
        row = {k: round(min(v), 4) for k, v in row.items()}
        fused()
        two_pass()
        stream.synchronize()
        row["fused_equals_two_pass"] = bool(torch.equal(blocks, ref))
        res["%s_ms_per_frame" % fname] = row
    # what the two-pass path moves beyond the fused one, at the least: the RGBA16F picture written and read back
    res["extra_bytes_per_frame_two_pass"] = 16 * W * H
    print(json.dumps(res))


if __name__ == "__main__":
    main()
