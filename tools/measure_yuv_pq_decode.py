#!/usr/bin/env python3
"""Decoding Hap HDR to HDR10 P010 (BT.2020, PQ) on 3840x2160 frames, timed with CUDA events around the library's calls, all in
one run:
  * HapB200BlockDecodeYUVPQBatch (the conversion fused into the BC6H block decoder, K8);
  * HapB200BlockDecodeHalfBatch to RGBA16F (K8 alone);
  * the two-pass path a caller would otherwise write: HapB200BlockDecodeHalfBatch, then a torch RGBA16F -> P010 conversion
    (the same definition: the table P, then the integer matrix and 4:2:0 filter, eager torch ops) into the planes;
  * HapB200DecodeYUVPQBatch end to end (Snappy frames -> planes) against HapB200DecodeRGBAHalfBatch (Snappy frames -> RGBA16F).
Two contents: picture-like (synth "video" frames made HDR10 as tools/measure_yuv_pq_encode.py does, then encoded by
HapB200BlockEncodeYUVPQBatch) and random blocks (uniformly random bytes: every BC6H mode, the reserved ones included, side by
side).  UF16 and SF16, BT.2020 limited range, unitNits 203.  The variants are alternated so that clocks and neighbours weigh
on each alike.  The fused and the two-pass planes are compared byte for byte.  Reports the best of two median ms per frame,
and the card's name, power limit and SM clocks read in the same run.  Needs a CUDA device.
    python tools/measure_yuv_pq_decode.py [frames] [repeats]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import hap_b200  # noqa: E402
import hap_b200.lib as L  # noqa: E402
from hap_b200 import synth  # noqa: E402
from hap_b200.abi import HapCompressorSnappy, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT, HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT  # noqa: E402
from measure_yuv_pq_encode import to_p010  # noqa: E402

W, H = 3840, 2160
NB = (W // 4) * (H // 4)
CS, UNIT = L.HapB200YUV_BT2020_Limited, 203
CHUNKS = 16
M1, M2, C1, C2, C3 = 2610 / 16384, 2523 / 32, 3424 / 4096, 2413 / 128, 2392 / 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
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


def coefficients():
    """the HAPB200_YUV_PQ_OUT_COEFFICIENTS row of BT.2020 limited, read from the header"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_PQ_OUT_COEFFICIENTS"):]
    line = body.split("\n")[2]
    return [int(v) for v in line[line.index("{") + 1: line.index("}")].split(",")]


def pq_out_table(unit):
    """P of include/hap_b200.h in float64 (the library builds it the same way, in C++)"""
    h = np.arange(0x7C00, dtype=np.uint16).view(np.float16).astype(np.float64)
    y = np.minimum(h * unit / 10000, 1.0) ** M1
    return np.floor(4095 * ((C1 + C2 * y) / (1 + C3 * y)) ** M2 + 0.5).astype(np.int32)


def torch_half_to_p010(rgba, table, luma, chroma):
    """the conversion of include/hap_b200.h in eager torch ops: rgba (F, H, W, 4) int16 binary16 bits -> luma (F, H, W) and
    chroma (F, H/2, W) int16 P010 words, views of the plane buffer"""
    k = coefficients()
    v = rgba[..., :3].to(torch.int32) & 0xFFFF
    p = torch.where(v >= 0x8000, torch.zeros_like(v), table[v.clamp(max=0x7BFF)])
    y = (((k[0] * p[..., 0] + k[1] * p[..., 1] + k[2] * p[..., 2] + 32768) >> 16) + k[9]).clamp(0, 1023)
    left = (2 * torch.arange(W // 2, device=rgba.device) - 1).clamp(min=0)
    hs = p[:, :, left] + 2 * p[:, :, 0::2] + p[:, :, 1::2]
    s = hs[:, 0::2] + hs[:, 1::2]
    cb = ((k[3] * s[..., 0] + k[4] * s[..., 1] + k[5] * s[..., 2] + (1 << 18)) >> 19) + k[10]
    cr = ((k[6] * s[..., 0] + k[7] * s[..., 1] + k[8] * s[..., 2] + (1 << 18)) >> 19) + k[10]
    c = torch.stack([cb, cr], -1).reshape(-1, H // 2, W).clamp(0, 1023)
    luma.copy_((y << 6).to(torch.int16))
    chroma.copy_((c << 6).to(torch.int16))


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 9
    if not torch.cuda.is_available():
        sys.exit("measure_yuv_pq_decode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H), "color_space": "BT.2020 limited",
           "unit_nits": UNIT, "frames": "Snappy, %d chunks" % CHUNKS}
    table = torch.from_numpy(pq_out_table(UNIT)).to(dev)
    pic = torch.empty((F, H * 3 // 2, W), dtype=torch.int16, device=dev)
    for i in range(F):
        pic[i, :H], pic[i, H:] = to_p010(synth.frame(W, H, i, kind="video")[None].to(dev))
    t0 = 16 * NB
    pitch, fstride = 2 * W, 2 * W * H * 3 // 2                       # one buffer per frame: luma, then chroma
    rgba = torch.empty((F, H, W, 4), dtype=torch.int16, device=dev)
    planes = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
    ref = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
    lp, cp = planes.data_ptr(), planes.data_ptr() + pitch * H
    rv = ref.view(F, fstride)
    ref_l, ref_c = rv[:, : pitch * H].view(torch.int16).view(F, H, W), rv[:, pitch * H:].view(torch.int16).view(F, H // 2, W)
    results = torch.zeros(F, dtype=torch.int32, device=dev)
    for fname, fmt in (("UF16", HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT), ("SF16", HapTextureFormat_RGB_BPTC_SIGNED_FLOAT)):
        for content in ("picture", "random"):
            blocks = torch.empty(F * t0, dtype=torch.uint8, device=dev)
            if content == "picture":
                check(lib.block_encode_yuv_pq_batch(pic.data_ptr(), pic.data_ptr() + pitch * H, F, fstride, W, H, pitch, CS, UNIT, fmt,
                                                    blocks.data_ptr(), t0, stream=sh))
            else:
                with torch.cuda.stream(stream):
                    blocks.random_(0, 256, generator=torch.Generator(dev).manual_seed(F))
            ostride = (lib.max_encoded_length_half(W, H, fmt, CHUNKS) + 15) // 16 * 16
            frames = torch.empty(F * ostride, dtype=torch.uint8, device=dev)
            used = torch.zeros(F, dtype=torch.int64, device=dev)
            check(lib.encode_batch([blocks.data_ptr()], [t0], [t0], [fmt], [HapCompressorSnappy], [CHUNKS], F, frames.data_ptr(), ostride,
                                   used.data_ptr(), stream=sh))
            stream.synchronize()
            fused = lambda: check(lib.block_decode_yuv_pq_batch(blocks.data_ptr(), F, t0, W, H, fmt, lp, cp, fstride, pitch, CS, UNIT,
                                                                stream=sh))
            half_only = lambda: check(lib.block_decode_half_batch(blocks.data_ptr(), F, t0, W, H, fmt, rgba.data_ptr(), 8 * W * H, stream=sh))

            def two_pass():
                half_only()
                with torch.cuda.stream(stream):
                    torch_half_to_p010(rgba, table, ref_l, ref_c)
            e2e_yuv = lambda: check(lib.decode_yuv_pq_batch(frames.data_ptr(), F, ostride, used.data_ptr(), CHUNKS + 1, W, H, lp, cp, fstride,
                                                            pitch, CS, UNIT, results.data_ptr(), stream=sh))
            e2e_half = lambda: check(lib.decode_rgba_half_batch(frames.data_ptr(), F, ostride, used.data_ptr(), CHUNKS + 1, W, H,
                                                                rgba.data_ptr(), 8 * W * H, results.data_ptr(), stream=sh))
            row = {}
            for _ in range(2):
                for name, fn in (("fused_block_decode_yuv_pq", fused), ("block_decode_half", half_only), ("two_pass_half_then_torch", two_pass),
                                 ("decode_yuv_pq_batch", e2e_yuv), ("decode_rgba_half_batch", e2e_half)):
                    row.setdefault(name, []).append(timed(fn, stream, repeats) / F)
            row = {k: round(min(v), 4) for k, v in row.items()}
            fused()
            two_pass()
            stream.synchronize()
            row["fused_equals_two_pass"] = bool(torch.equal(planes, ref))
            e2e_yuv()
            stream.synchronize()
            row["decode_yuv_pq_batch_equals_fused"] = bool((results == 0).all()) and bool(torch.equal(planes, ref))
            res["%s_%s_ms_per_frame" % (fname, content)] = row
            del blocks, frames
    res["card_after"] = card()
    # bytes each path writes per frame: the P010 planes, against the RGBA16F picture the two-pass path writes and reads back
    res["p010_bytes_per_frame"] = pitch * H * 3 // 2
    res["rgba16f_bytes_per_frame"] = 8 * W * H
    print(json.dumps(res))


if __name__ == "__main__":
    main()
