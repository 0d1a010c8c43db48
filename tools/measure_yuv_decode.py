#!/usr/bin/env python3
"""Decoding to NV12 / P010 on 3840x2160 frames, timed with CUDA events around the library's calls, all in one run:
  * HapB200BlockDecodeYUVBatch (the conversion fused into the block decoder, K8);
  * HapB200BlockDecodeBatch to RGBA8 (K8 alone);
  * the two-pass path a caller would otherwise write: HapB200BlockDecodeBatch, then a torch RGBA8 -> Y'CbCr 4:2:0 conversion
    (the same integer definition, eager torch ops) into the planes;
  * HapB200DecodeYUVBatch end to end (Snappy frames -> planes) against HapB200DecodeRGBABatch (Snappy frames -> RGBA8).
for Hap1, Hap5, HapY, HapM and Hap7, on synth "video" content, NV12 and P010, BT.709 limited range.  The variants are
alternated so that clocks and neighbours weigh on each alike.  The fused and the two-pass planes are compared byte for byte.
Reports the best of two median ms per frame and the card's name and power limit.  Needs a CUDA device.
    python tools/measure_yuv_decode.py [frames] [repeats]"""
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
CS = L.HapB200YUV_BT709_Limited
CODECS = (("Hap1", L.HapB200Codec_Hap1, (0x83F0,)), ("Hap5", L.HapB200Codec_Hap5, (0x83F3,)), ("HapY", L.HapB200Codec_HapY, (0x01,)),
          ("HapM", L.HapB200Codec_HapM, (0x01, 0x8DBB)), ("Hap7", L.HapB200Codec_Hap7, (0x8E8C,)))
CHUNKS = 16


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


def coefficients(layout):
    """the HAPB200_YUV_OUT_COEFFICIENTS row of BT.709 limited, read from the header"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_OUT_COEFFICIENTS"):]
    rows = [[int(v) for v in line[line.index("{") + 1: line.index("}")].split(",")] for line in body.split("\n")[2:10]]
    return rows[layout * 4 + CS]


def torch_rgba_to_yuv(rgba, layout, luma, chroma):
    """the conversion of include/hap_b200.h in eager torch integer ops: rgba (F, H, W, 4) uint8 -> luma (F, H, W) and chroma
    (F, H/2, W) views of the plane buffer (uint8, or int16 P010 words)"""
    k = coefficients(layout)
    top = 1023 if layout == L.HapB200YUV_P010 else 255
    p = rgba[..., :3].to(torch.int32)
    y = ((k[0] * p[..., 0] + k[1] * p[..., 1] + k[2] * p[..., 2] + 32768) >> 16) + k[9]
    left = (2 * torch.arange(W // 2, device=rgba.device) - 1).clamp(min=0)
    hs = p[:, :, left] + 2 * p[:, :, 0::2] + p[:, :, 1::2]
    s = hs[:, 0::2] + hs[:, 1::2]
    cb = ((k[3] * s[..., 0] + k[4] * s[..., 1] + k[5] * s[..., 2] + (1 << 18)) >> 19) + k[10]
    cr = ((k[6] * s[..., 0] + k[7] * s[..., 1] + k[8] * s[..., 2] + (1 << 18)) >> 19) + k[10]
    c = torch.stack([cb, cr], -1).reshape(-1, H // 2, W).clamp(0, top)
    y = y.clamp(0, top)
    if layout == L.HapB200YUV_P010:
        luma.copy_((y << 6).to(torch.int16))
        chroma.copy_((c << 6).to(torch.int16))
    else:
        luma.copy_(y.to(torch.uint8))
        chroma.copy_(c.to(torch.uint8))


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 9
    if not torch.cuda.is_available():
        sys.exit("measure_yuv_decode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H), "color_space": "BT.709 limited",
           "frames": "Snappy, %d chunks" % CHUNKS}
    src = torch.from_numpy(np.stack([synth.frame(W, H, i, kind="video").numpy() for i in range(F)])).to(dev)
    rgba = torch.empty((F, H, W, 4), dtype=torch.uint8, device=dev)
    results = torch.zeros(F, dtype=torch.int32, device=dev)
    for cname, codec, fmts in CODECS:
        t = [lib.texture_bytes(W, H, codec, i) for i in range(2)]
        bstride = t[0] + t[1]
        blocks = torch.empty(F * bstride, dtype=torch.uint8, device=dev)
        if codec == L.HapB200Codec_Hap7:
            check(lib.block_encode_bc7_batch(src.data_ptr(), F, 4 * W * H, W, H, blocks.data_ptr(), bstride, stream=sh))
        else:
            check(lib.block_encode_batch(src.data_ptr(), F, 4 * W * H, W, H, codec, blocks.data_ptr(), bstride, stream=sh))
        ostride = (lib.max_encoded_length_rgba(W, H, codec, CHUNKS) + 15) // 16 * 16
        frames = torch.empty(F * ostride, dtype=torch.uint8, device=dev)
        used = torch.zeros(F, dtype=torch.int64, device=dev)
        n = len(fmts)
        check(lib.encode_batch([blocks.data_ptr() + (t[0] if i else 0) for i in range(n)], [bstride] * n, t[:n], list(fmts),
                               [HapCompressorSnappy] * n, [CHUNKS] * n, F, frames.data_ptr(), ostride, used.data_ptr(), stream=sh))
        stream.synchronize()
        for layout, lname in ((L.HapB200YUV_NV12, "NV12"), (L.HapB200YUV_P010, "P010")):
            sb = 2 if layout == L.HapB200YUV_P010 else 1
            pitch = W * sb
            fstride = pitch * H * 3 // 2                               # one buffer per frame: luma, then chroma
            planes = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
            ref = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
            lp, cp = planes.data_ptr(), planes.data_ptr() + pitch * H
            rv = ref.view(F, fstride)
            dt = torch.int16 if sb == 2 else torch.uint8
            ref_l, ref_c = rv[:, : pitch * H].view(dt).view(F, H, W), rv[:, pitch * H:].view(dt).view(F, H // 2, W)
            fused = lambda: check(lib.block_decode_yuv_batch(blocks.data_ptr(), F, bstride, W, H, codec, lp, cp, fstride, pitch, layout, CS,
                                                             stream=sh))
            rgba_only = lambda: check(lib.block_decode_batch(blocks.data_ptr(), F, bstride, W, H, codec, rgba.data_ptr(), 4 * W * H, stream=sh))

            def two_pass():
                rgba_only()
                with torch.cuda.stream(stream):
                    torch_rgba_to_yuv(rgba, layout, ref_l, ref_c)
            e2e_yuv = lambda: check(lib.decode_yuv_batch(frames.data_ptr(), F, ostride, used.data_ptr(), CHUNKS + 1, codec, W, H, lp, cp,
                                                         fstride, pitch, layout, CS, results.data_ptr(), stream=sh))
            e2e_rgba = lambda: check(lib.decode_rgba_batch(frames.data_ptr(), F, ostride, used.data_ptr(), CHUNKS + 1, codec, W, H,
                                                           rgba.data_ptr(), 4 * W * H, results.data_ptr(), stream=sh))
            row = {}
            for _ in range(2):
                for name, fn in (("fused_block_decode_yuv", fused), ("block_decode_rgba", rgba_only), ("two_pass_rgba_then_torch", two_pass),
                                 ("decode_yuv_batch", e2e_yuv), ("decode_rgba_batch", e2e_rgba)):
                    row.setdefault(name, []).append(timed(fn, stream, repeats) / F)
            row = {k: round(min(v), 4) for k, v in row.items()}
            fused()
            two_pass()
            stream.synchronize()
            row["fused_equals_two_pass"] = bool(torch.equal(planes, ref))
            e2e_yuv()
            stream.synchronize()
            row["decode_yuv_batch_equals_fused"] = bool((results == 0).all()) and bool(torch.equal(planes, ref))
            res["%s_%s_ms_per_frame" % (cname, lname)] = row
            del planes, ref
        del blocks, frames
    # what the two-pass path moves beyond the fused one, at the least: the RGBA picture written and read back
    res["extra_bytes_per_frame_two_pass"] = 8 * W * H
    print(json.dumps(res))


if __name__ == "__main__":
    main()
