#!/usr/bin/env python3
"""Block encoding from NV12 / P010 on 3840x2160 frames, timed with CUDA events around the library's calls, all in one run:
  * HapB200BlockEncodeYUVBatch (the conversion fused into the block encoder's load);
  * HapB200BlockEncodeBatch on the RGBA8 picture that conversion makes (the block encode alone);
  * the two-pass path a caller would otherwise write: a torch YUV -> RGBA8 conversion (the same integer definition, eager
    torch ops) into an RGBA8 batch, then HapB200BlockEncodeBatch.
for Hap1, Hap5 and HapY, on synth "video" content converted to NV12 and P010 (BT.709, limited range).  The fused and the
two-pass textures are compared byte for byte.  Reports median ms per frame and the card's name and power limit.  Needs a
CUDA device.
    python tools/measure_yuv_encode.py [frames] [repeats]"""
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
NB = (W // 4) * (H // 4)
CS = L.HapB200YUV_BT709_Limited
KR, KB = 0.2126, 0.0722
# HAPB200_YUV_COEFFICIENTS rows of BT.709 limited: {cy, crR, cbG, crG, cbB, yOff, cOff}
COEFFS = {L.HapB200YUV_NV12: (76308, 14688, -1748, -4364, 17304, 16, 128), L.HapB200YUV_P010: (19077, 3672, -437, -1091, 4326, 64, 512)}


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


def to_yuv(rgba, layout):
    """(F, H, W, 4) uint8 on the device -> tight planes: luma (F, H, W), chroma (F, H/2, W) as uint8 or P010 words"""
    n = 10 if layout == L.HapB200YUV_P010 else 8
    s = 1 << (n - 8)
    rgb = rgba[..., :3].float() / 255.0
    ey = KR * rgb[..., 0] + (1 - KR - KB) * rgb[..., 1] + KB * rgb[..., 2]
    pb = (rgb[..., 2] - ey) / (2 * (1 - KB))
    pr = (rgb[..., 0] - ey) / (2 * (1 - KR))
    quad = lambda p: p.reshape(p.shape[0], H // 2, 2, W // 2, 2).mean(dim=(2, 4))
    y = torch.round(16 * s + 219 * s * ey).clamp(0, (1 << n) - 1).to(torch.int32)
    c = torch.stack([quad(pb), quad(pr)], -1).reshape(-1, H // 2, W)
    c = torch.round((1 << (n - 1)) + 224 * s * c).clamp(0, (1 << n) - 1).to(torch.int32)
    if n == 10:
        return (y << 6).to(torch.int16), (c << 6).to(torch.int16)
    return y.to(torch.uint8), c.to(torch.uint8)


def torch_yuv_to_rgba(luma, chroma, layout, out):
    """the conversion of include/hap_b200.h in eager torch integer ops, into out (F, H, W, 4) uint8"""
    k = COEFFS[layout]
    if layout == L.HapB200YUV_P010:
        yv = (luma.to(torch.int32) & 0xFFFF) >> 6
        c = ((chroma.to(torch.int32) & 0xFFFF) >> 6).reshape(-1, H // 2, W // 2, 2)
    else:
        yv = luma.to(torch.int32)
        c = chroma.to(torch.int32).reshape(-1, H // 2, W // 2, 2)
    j = torch.arange(H, device=luma.device) // 2
    rn = torch.where(torch.arange(H, device=luma.device) % 2 == 1, j + 1, j - 1).clamp(0, H // 2 - 1)
    v = 3 * c[:, j] + c[:, rn]                                              # (F, H, W/2, 2)
    i = torch.arange(W, device=luma.device) // 2
    cn = (i + 1).clamp(max=W // 2 - 1)
    odd = (torch.arange(W, device=luma.device) % 2 == 1).view(1, 1, W, 1)
    c8 = torch.where(odd, v[:, :, i] + v[:, :, cn], 2 * v[:, :, i]) - 8 * k[6]
    yd = k[0] * (yv - k[5])
    cb, cr = c8[..., 0], c8[..., 1]
    out[..., 0] = ((yd + k[1] * cr + 32768) >> 16).clamp(0, 255)
    out[..., 1] = ((yd + k[2] * cb + k[3] * cr + 32768) >> 16).clamp(0, 255)
    out[..., 2] = ((yd + k[4] * cb + 32768) >> 16).clamp(0, 255)
    out[..., 3] = 255


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 9
    if not torch.cuda.is_available():
        sys.exit("measure_yuv_encode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H), "color_space": "BT.709 limited"}
    src = torch.from_numpy(np.stack([synth.frame(W, H, i, kind="video").numpy() for i in range(F)])).to(dev)
    rgba = torch.empty((F, H, W, 4), dtype=torch.uint8, device=dev)
    blocks = torch.empty(F * NB * 16, dtype=torch.uint8, device=dev)
    ref = torch.empty(F * NB * 16, dtype=torch.uint8, device=dev)
    for layout, lname in ((L.HapB200YUV_NV12, "NV12"), (L.HapB200YUV_P010, "P010")):
        sb = 2 if layout == L.HapB200YUV_P010 else 1
        luma, chroma = to_yuv(src, layout)
        # one buffer per frame: luma then chroma, rows W*sb bytes apart (a multiple of 16)
        pitch = W * sb
        fstride = pitch * H * 3 // 2
        planes = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
        pv = planes.view(F, fstride)
        pv[:, : pitch * H] = luma.reshape(F, -1).view(torch.uint8)
        pv[:, pitch * H:] = chroma.reshape(F, -1).view(torch.uint8)
        lp, cp = planes.data_ptr(), planes.data_ptr() + pitch * H
        with torch.cuda.stream(stream):
            torch_yuv_to_rgba(luma, chroma, layout, rgba)
        stream.synchronize()
        for cname, codec in (("Hap1", L.HapB200Codec_Hap1), ("Hap5", L.HapB200Codec_Hap5), ("HapY", L.HapB200Codec_HapY)):
            t = lib.texture_bytes(W, H, codec, 0)
            fused = lambda: check(lib.block_encode_yuv_batch(lp, cp, F, fstride, W, H, pitch, layout, CS, codec, blocks.data_ptr(), t, stream=sh))
            rgba_only = lambda: check(lib.block_encode_batch(rgba.data_ptr(), F, 4 * W * H, W, H, codec, ref.data_ptr(), t, stream=sh))

            def two_pass():
                with torch.cuda.stream(stream):
                    torch_yuv_to_rgba(luma, chroma, layout, rgba)
                rgba_only()
            row = {}
            # alternate the three so that clocks and neighbours weigh on each alike
            for _ in range(2):
                for name, fn in (("fused_yuv_block_encode", fused), ("rgba_block_encode", rgba_only), ("two_pass_torch_then_rgba", two_pass)):
                    row.setdefault(name, []).append(timed(fn, stream, repeats) / F)
            row = {k: round(min(v), 4) for k, v in row.items()}
            fused()
            two_pass()
            stream.synchronize()
            row["fused_equals_two_pass"] = bool(torch.equal(blocks[: F * t], ref[: F * t]))
            res["%s_%s_ms_per_frame" % (lname, cname)] = row
        del planes, luma, chroma
    # what the two-pass path moves beyond the fused one, at the least: the RGBA picture written and read back
    res["extra_bytes_per_frame_two_pass"] = 8 * W * H
    print(json.dumps(res))


if __name__ == "__main__":
    main()
