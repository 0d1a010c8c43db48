#!/usr/bin/env python3
"""TEST INFRASTRUCTURE (it lives under tests/ because it drives the reference build, which only tests may touch).
How fast do the decode kernels take frames made by the REFERENCE encoder (unmodified hap.c + Google Snappy)?
bench.py times streams from our own encoder; players mostly meet files written by others.  Run on a GPU:

    python tests/measure_ref_decode.py [--frames 16] > ref_decode.json

Uses oracle/_ref only to PRODUCE the input frames (on the host, outside every timed region)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))  # oracles.py


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--chunks", type=int, default=8)
    args = ap.parse_args()
    import numpy as np
    import torch

    import hap_b200
    import oracles
    from hap_b200 import synth
    from hap_b200.lib import HapB200Codec_HapY

    W, H = 3840, 2160
    lib = hap_b200.load()
    ref = oracles.ref_abi() or oracles.oracle_abi()
    n = lib.texture_bytes(W, H, HapB200Codec_HapY)
    F, K = args.frames, args.chunks
    cap = (lib.max_encoded_length([n], [1], [K]) + 15) // 16 * 16
    frames = torch.zeros(F * cap, dtype=torch.uint8)
    used = torch.zeros(F, dtype=torch.int64)
    stats = None
    for f in range(F):
        img = synth.frame(W, H, f, device="cuda")
        tex = torch.zeros(n, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_batch(img.data_ptr(), 1, img.numel(), W, H, HapB200Codec_HapY, tex.data_ptr(), n) == 0
        host = tex.cpu().numpy().tobytes()
        r, fr = ref.encode([host], [1], [1], [K])
        assert r == 0
        frames[f * cap: f * cap + len(fr)] = torch.frombuffer(bytearray(fr), dtype=torch.uint8)
        used[f] = len(fr)
        if f == 0:
            # element statistics of chunk 3 (picture content)
            _, st = oracles.snappy_scan(fr[4 + 4 + 5 * K + 8 + sum(int.from_bytes(fr[8 + K + 4 + 4 * c: 12 + K + 4 + 4 * c], "little") for c in range(3)):][: int.from_bytes(fr[8 + K + 4 + 12: 8 + K + 4 + 16], "little")])
            stats = {"literals": st.literals, "copies": st.copy1 + st.copy2 + st.copy4,
                     "elements_per_KiB_out": 1024.0 * (st.literals + st.copy1 + st.copy2 + st.copy4) / max(st.literal_bytes + st.copy_bytes, 1)}
    d_frames, d_used = frames.cuda(), used.cuda()
    out = torch.zeros(F * n, dtype=torch.uint8, device="cuda")
    o_used = torch.zeros(F, dtype=torch.int64, device="cuda")
    fmts = torch.zeros(F, dtype=torch.int32, device="cuda")
    res = torch.zeros(F, dtype=torch.int32, device="cuda")
    st = torch.cuda.Stream()

    def run():
        r = lib.decode_batch(d_frames.data_ptr(), F, cap, d_used.data_ptr(), 0, K, out.data_ptr(), n, o_used.data_ptr(),
                             fmts.data_ptr(), res.data_ptr(), stream=st.cuda_stream)
        assert r == 0

    with torch.cuda.stream(st):
        for _ in range(3):
            run()
        torch.cuda.synchronize()
        assert res.tolist() == [0] * F and o_used.tolist() == [n] * F
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        iters = 5
        for _ in range(iters):
            run()
        e1.record(st)
        torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    lib.set_stage_timing(True)
    lib.stage_times()
    with torch.cuda.stream(st):
        for _ in range(3):
            run()
    stages = {k: v[0] / 3 for k, v in lib.stage_times().items() if v[0] > 0}
    lib.set_stage_timing(False)
    print(json.dumps({"what": "decode of reference-encoded 4K Hap Q frames (Google Snappy), device-resident batch",
                      "frames": F, "chunks": K, "ms_per_batch": ms, "ratio": float(used.double().mean()) / n,
                      "texture_GBps": F * n / ms / 1e6, "rgba_equiv_GBps": F * 4 * W * H / ms / 1e6, "stage_ms_per_batch": stages,
                      "stream_elements_of_one_chunk": stats}))


if __name__ == "__main__":
    main()
