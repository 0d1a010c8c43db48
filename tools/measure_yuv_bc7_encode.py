#!/usr/bin/env python3
"""Hap R (BC7) block encoding from Y'CbCr pictures on 3840x2160 frames, timed with CUDA events around the library's calls,
all in one run:
  * HapB200BlockEncodeYUVBC7Batch from NV12 and P010;
  * HapB200BlockEncodePlanarBC7Batch from 4:2:0 8-bit (yuv420p), 4:2:2 10-bit (yuv422p10le) and 4:4:4 12-bit with alpha
    (yuva444p12le);
  * HapB200BlockEncodeBC7Batch from the synth RGBA8 picture, opaque and with its alpha ramp, and from the RGBA8 picture each
    Y'CbCr source converts to (the definitions of tests/yuv_util.py and tests/planar_util.py, in numpy);
on synth "video" content (BT.709, limited range; alpha a ramp with detail), built as tools/measure_planar_encode.py builds
it.  The Y'CbCr calls convert into an RGBA8 scratch picture and then run the same BC7 kernel, so each should take the time
of the RGBA8 call on its converted picture plus the conversion pass.  The BC7 search's time depends on the content (alpha,
and the requantised, subsampled chroma of a Y'CbCr picture), so only that RGBA8 call is a like-for-like baseline.  The calls
are alternated so that clocks and neighbours weigh on each alike.  Reports median ms per frame (and the difference from the
converted picture's call) with the card's name and power limit.  After the timed calls, one call per source runs under
torch.profiler, apart from them, for the conversion kernel's own time per frame.  Needs a CUDA device.
    python tools/measure_yuv_bc7_encode.py [frames] [repeats] [rounds]"""
import json
import os
import sys

import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import hap_b200  # noqa: E402
import hap_b200.lib as L  # noqa: E402
from hap_b200 import synth  # noqa: E402
import planar_util  # noqa: E402
import yuv_util  # noqa: E402
from measure_planar_encode import CS, H, W, card, timed, to_planes  # noqa: E402

NB = (W // 4) * (H // 4)


def main():
    F = int(sys.argv[1]) if len(sys.argv) > 1 else 2
    repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 2
    if not torch.cuda.is_available():
        sys.exit("measure_yuv_bc7_encode.py needs a CUDA device")
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
    blocks = torch.empty(F * NB * 16, dtype=torch.uint8, device=dev)
    t = NB * 16

    # the sources: name -> callable that encodes all F frames on `stream`
    opaque = rgba.clone()
    opaque[..., 3] = 255
    sources = {"rgba8_opaque": lambda: check(lib.block_encode_bc7_batch(opaque.data_ptr(), F, 4 * W * H, W, H, blocks.data_ptr(), t, stream=sh)),
               "rgba8_alpha": lambda: check(lib.block_encode_bc7_batch(rgba.data_ptr(), F, 4 * W * H, W, H, blocks.data_ptr(), t, stream=sh))}
    keep = []

    def add_converted(name, pictures):
        """BC7 on the RGBA8 pictures (F numpy (H, W, 4)) a source converts to"""
        pic = torch.from_numpy(np.stack(pictures)).to(dev)
        keep.append(pic)
        sources["rgba8_of_" + name] = lambda: check(lib.block_encode_bc7_batch(pic.data_ptr(), F, 4 * W * H, W, H, blocks.data_ptr(), t,
                                                                               stream=sh))
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
        host = lambda p: p.cpu().numpy().view(np.uint8 if n == 8 else np.uint16)
        chroma = torch.stack([cb, cr], -1).reshape(F, H // 2, W)
        add_converted(name, [yuv_util.yuv_to_rgba(host(y[f]), host(chroma[f]), layout, CS) for f in range(F)])
        sources[name] = (lambda lp, cp, pitch, fstride, layout: lambda: check(
            lib.block_encode_yuv_bc7_batch(lp, cp, F, fstride, W, H, pitch, layout, CS, blocks.data_ptr(), t, stream=sh)))(
            lp, cp, pitch, fstride, layout)
    for name, sub, n, fy, fx, alpha in (("yuv420p", L.HapB200Chroma_420, 8, 2, 2, False), ("yuv422p10le", L.HapB200Chroma_422, 10, 1, 2, False),
                                        ("yuva444p12le", L.HapB200Chroma_444, 12, 1, 1, True)):
        planes = to_planes(rgba, n, fy, fx)
        sb = 1 if n == 8 else 2
        fstride = W * sb * H   # each plane in a buffer of its own, frames one luma plane apart
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
        host = [p.cpu().numpy().view(np.uint8 if n == 8 else np.uint16) for p in planes]
        add_converted(name, [planar_util.planar_to_rgba(host[0][f], host[1][f], host[2][f], host[3][f] if alpha else None, sub, n, CS)
                             for f in range(F)])
        sources[name] = (lambda ptrs, fstride, lpitch, cpitch, sub, n: lambda: check(
            lib.block_encode_planar_bc7_batch(*ptrs, F, fstride, W, H, lpitch, cpitch, sub, n, CS, blocks.data_ptr(), t, stream=sh)))(
            ptrs, fstride, lpitch, cpitch, sub, n)
    torch.cuda.synchronize()
    row = {}
    for _ in range(rounds):
        for sname, fn in sources.items():
            row.setdefault(sname, []).append(timed(fn, stream, repeats) / F)
    med = {k: float(np.median(v)) for k, v in row.items()}
    res["bc7_ms_per_frame"] = {k: dict({"median": round(med[k], 3), "min": round(min(v), 3), "max": round(max(v), 3)},
                                       **({"over_its_converted_rgba8": round(med[k] - med["rgba8_of_" + k], 4)} if "rgba8_of_" + k in med else {}))
                               for k, v in row.items()}
    # one profiled call per source in one session; each source has its own instantiation (BcSource, yuv_source.cuh)
    src_id = {"nv12": 1, "p010": 2, "yuv420p": 5, "yuv422p10le": 8, "yuva444p12le": 10}
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for sname in src_id:
            sources[sname]()
        torch.cuda.synchronize()
    avg = prof.key_averages()
    res["conversion_pass_ms_per_frame_profiled"] = {
        sname: round(sum(e.device_time_total for e in avg if "bc_source_to_rgba8_kernel<%d>" % i in e.key) / 1000 / F, 4)
        for sname, i in src_id.items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
