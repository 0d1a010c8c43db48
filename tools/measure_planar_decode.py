#!/usr/bin/env python3
"""Decoding to planar Y'CbCr (+ alpha) on 3840x2160 frames, timed with CUDA events around the library's calls, all in one run:
  * HapB200BlockDecodePlanarBatch (the conversion fused into the block decoder, K8 with the planar sink);
  * HapB200BlockDecodeBatch to RGBA8 (K8 alone);
  * the two-pass path a caller would otherwise write: HapB200BlockDecodeBatch, then a torch RGBA8 -> planar conversion (the
    same integer definition, eager torch ops) into the planes;
  * for 4:2:0 at 8 and 10 bits without alpha, HapB200BlockDecodeYUVBatch (the NV12 / P010 sink: the same samples, interleaved).
for Hap Q (HapY) and Hap Q Alpha (HapM), on synth "video" content with a ramp alpha, every subsampling and depth, with and
without the alpha plane, BT.709 limited range.  The variants are alternated so that clocks and neighbours weigh on each alike.
The fused and the two-pass planes are compared byte for byte.  Reports the best of two median ms per frame, the fused sink's
algorithmic bytes per frame (texture read + planes written) and rate, and the card's name and power limit.  Needs a CUDA device.
    python tools/measure_planar_decode.py [frames] [repeats]"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hap_b200  # noqa: E402
import hap_b200.lib as L  # noqa: E402
import planar_out_util as Q  # noqa: E402
from hap_b200 import synth  # noqa: E402

W, H = 3840, 2160
CS = L.HapB200YUV_BT709_Limited
CODECS = (("HapY", L.HapB200Codec_HapY), ("HapM", L.HapB200Codec_HapM))
HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


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


def torch_rgba_to_planar(rgba, sub, n, planes):
    """the conversion of include/hap_b200.h in eager torch integer ops: rgba (F, H, W, 4) uint8 -> planes (luma, cb, cr, alpha
    or None: views of the plane buffer, uint8 or int16 words)"""
    k = Q.row(n, CS)
    top = (1 << n) - 1
    p = rgba[..., :3].to(torch.int32)
    y = ((k[0] * p[..., 0] + k[1] * p[..., 1] + k[2] * p[..., 2] + 32768) >> 16) + k[9]
    if sub == Q.S444:
        s = 8 * p
    else:
        left = (2 * torch.arange(W // 2, device=rgba.device) - 1).clamp(min=0)
        hs = p[:, :, left] + 2 * p[:, :, 0::2] + p[:, :, 1::2]
        s = hs[:, 0::2] + hs[:, 1::2] if sub == Q.S420 else 2 * hs
    cb = ((k[3] * s[..., 0] + k[4] * s[..., 1] + k[5] * s[..., 2] + (1 << 18)) >> 19) + k[10]
    cr = ((k[6] * s[..., 0] + k[7] * s[..., 1] + k[8] * s[..., 2] + (1 << 18)) >> 19) + k[10]
    dt = torch.uint8 if n == 8 else torch.int16
    for dst, v in zip(planes, (y, cb, cr)):
        dst.copy_(v.clamp(0, top).to(dt))
    if planes[3] is not None:
        planes[3].copy_(((2 * top * rgba[..., 3].to(torch.int32) + 255) // 510).to(dt))


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 9
    if not torch.cuda.is_available():
        sys.exit("measure_planar_decode.py needs a CUDA device")
    lib = hap_b200.load()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.Stream(dev)
    sh = stream.cuda_stream

    def check(r):
        assert r == 0, r

    res = {"card": card(), "frames_per_call": F, "repeats": repeats, "geometry": "%dx%d" % (W, H), "color_space": "BT.709 limited"}
    src = torch.from_numpy(np.stack([synth.frame(W, H, i, kind="video", alpha="ramp").numpy() for i in range(F)])).to(dev)
    rgba = torch.empty((F, H, W, 4), dtype=torch.uint8, device=dev)
    for cname, codec in CODECS:
        t = [lib.texture_bytes(W, H, codec, i) for i in range(2)]
        bstride = t[0] + t[1]
        blocks = torch.empty(F * bstride, dtype=torch.uint8, device=dev)
        check(lib.block_encode_batch(src.data_ptr(), F, 4 * W * H, W, H, codec, blocks.data_ptr(), bstride, stream=sh))
        rgba_only = lambda: check(lib.block_decode_batch(blocks.data_ptr(), F, bstride, W, H, codec, rgba.data_ptr(), 4 * W * H, stream=sh))
        for sub in Q.SUBSAMPLINGS:
            for n in Q.DEPTHS:
                sb = 1 if n == 8 else 2
                ch, cw = (H // 2 if sub == Q.S420 else H), (W if sub == Q.S444 else W // 2)
                lp, cp = sb * W, sb * cw
                sizes = [lp * H, cp * ch, cp * ch, lp * H]
                offs = np.cumsum([0] + sizes).tolist()
                fstride = offs[4]                                        # one buffer per frame: luma, Cb, Cr, alpha
                buf = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
                ref = torch.empty(F * fstride, dtype=torch.uint8, device=dev)
                dt = torch.int16 if sb == 2 else torch.uint8
                shapes = [(H, W), (ch, cw), (ch, cw), (H, W)]
                ref_planes = [ref.view(F, fstride)[:, offs[i]: offs[i + 1]].view(dt).view(F, *shapes[i]) for i in range(4)]
                for alpha in (False, True):
                    ptrs = [buf.data_ptr() + offs[i] for i in range(3)] + [buf.data_ptr() + offs[3] if alpha else 0]
                    fused = lambda: check(lib.block_decode_planar_batch(blocks.data_ptr(), F, bstride, W, H, codec, *ptrs, fstride, lp, cp, sub,
                                                                        n, CS, stream=sh))

                    def two_pass():
                        rgba_only()
                        with torch.cuda.stream(stream):
                            torch_rgba_to_planar(rgba, sub, n, ref_planes[:3] + [ref_planes[3] if alpha else None])
                    variants = [("fused_block_decode_planar", fused), ("block_decode_rgba", rgba_only), ("two_pass_rgba_then_torch", two_pass)]
                    if sub == Q.S420 and n < 12 and not alpha:
                        layout = L.HapB200YUV_P010 if n == 10 else L.HapB200YUV_NV12
                        nv = torch.empty(F * lp * H * 3 // 2, dtype=torch.uint8, device=dev)
                        variants.append(("nv12_p010_sink", lambda: check(lib.block_decode_yuv_batch(
                            blocks.data_ptr(), F, bstride, W, H, codec, nv.data_ptr(), nv.data_ptr() + lp * H, lp * H * 3 // 2, lp, layout, CS,
                            stream=sh))))
                    row = {}
                    for _ in range(2):
                        for name, fn in variants:
                            row.setdefault(name, []).append(timed(fn, stream, repeats) / F)
                    row = {k: round(min(v), 4) for k, v in row.items()}
                    buf.fill_(0)
                    ref.fill_(0)
                    fused()
                    two_pass()
                    stream.synchronize()
                    row["fused_equals_two_pass"] = bool(torch.equal(buf, ref))
                    moved = sum(t[: 2 if codec == L.HapB200Codec_HapM and alpha else 1]) + sum(sizes[:3]) + (sizes[3] if alpha else 0)
                    row["fused_bytes_per_frame"] = moved
                    row["fused_GB_per_s"] = round(moved / (row["fused_block_decode_planar"] * 1e-3) / 1e9, 1)
                    row["fused_share_of_hbm_peak"] = round(moved / (row["fused_block_decode_planar"] * 1e-3) / HBM_BYTES_PER_S, 3)
                    res["%s_%s_%d_%s_ms_per_frame" % (cname, ("420", "422", "444")[sub], n, "alpha" if alpha else "no_alpha")] = row
                    print(json.dumps({"progress": [cname, sub, n, alpha, row]}), flush=True)
                del buf, ref
        del blocks
    print(json.dumps(res))


if __name__ == "__main__":
    main()
