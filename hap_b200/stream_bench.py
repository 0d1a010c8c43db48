"""bench.py --workload 16k_stream: BASELINE.json configs[4] -- a 16384 x 16384 RGBA stream, Hap Q (scaled YCoCg DXT5,
64 chunks, Snappy), frames sharded round-robin over the GPUs of one box, the ENCODED frames delivered to rank 0 (where a
muxer would sit) inside the timed region.

One process per GPU (torchrun).  Two ways to deliver, both timed; `value` is the faster one at the N at hand (`delivery` names it):

  ring: rank 0 owns a delivery ring (HapB200RingCreate, CUDA IPC).  Every rank passes an
      address INSIDE that ring as the output of HapB200EncodeRGBABatch: the kernel that lays a frame out stores it over
      NVLink / NVSwitch straight into rank 0's memory, the frame lengths go to the slot's header the same way, and a
      release store publishes the slot (HapB200RingPublish).  Rank 0's consumer stream waits on the flags
      (HapB200RingWait).  No staging copy, no collective, no host synchronisation inside a step.
  nccl (`nccl_gatherv_baseline`): encode into local memory, all-gather the lengths, grouped
      ncclSend/ncclRecv of exactly the encoded bytes (sharding.gatherv_frames_to_root), the delivery of batch i
      overlapping the encode of batch i+1.

Timing: CUDA events on the streams around K steps, barrier + synchronize on both sides, max over ranks (rank 0: the later
of its producer and its consumer stream).  `value` = RGBA bytes of all frames encoded and delivered per second; fps next to
it.  Outside the timed region rank 0 decodes one frame that came from another rank and compares it with a checksum of that
rank's own texture.  Two slots per rank alternate; the consumer here only waits for the frames (a real one would hand
slots back through the same kind of flag in the other direction).
"""
from __future__ import annotations

import os
import time

HEADER = 4096          # per slot: flag (u32) at 0, frame lengths (u64 each) at 64


class _DeviceBytes:
    """torch view of device memory the library allocated (the ring)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def run(args, rank, local_rank, world, emit, ClockSampler, measured_peak_hbm):
    import torch
    import torch.distributed as dist

    import hap_b200
    from hap_b200 import sharding, synth
    from hap_b200.lib import HapB200Codec_HapY

    W = H = int(os.environ.get("HAPB200_STREAM_SIZE", "16384"))
    CH = 64
    B = int(os.environ.get("HAPB200_STREAM_BATCH", "2"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    lib = hap_b200.load()
    lib.set_option(lib.OPTION_WRITE_INDEX, 0 if args.no_index else 1)
    codec = HapB200Codec_HapY
    rgba_bytes = 4 * W * H
    tex_bytes = lib.texture_bytes(W, H, codec)
    cap = (lib.max_encoded_length_rgba(W, H, codec, CH) + 255) // 256 * 256
    peak, peak_src = measured_peak_hbm()

    # B distinct frames per rank, built tile by tile (a 16K frame of int64 intermediates would not fit otherwise)
    rgba = torch.empty((B, H, W, 4), dtype=torch.uint8, device=dev)
    th = min(2048, H)
    for b in range(B):
        for ty in range(0, H, th):
            for tx in range(0, W, 2 * th):
                tw = min(2 * th, W - tx)
                rgba[b, ty:ty + th, tx:tx + tw] = synth.frame(tw, th, (rank * B + b) * 64 + (ty // th) * 8 + tx // (2 * th), device=dev)
    stream = torch.cuda.Stream(device=dev)
    stream2 = torch.cuda.Stream(device=dev)      # peer delivery: batches alternate between two producer streams, so the NVLink-bound
    producers = [stream, stream2]                # frame-layout stage of batch i overlaps the block encode of batch i+1
    consumer = torch.cuda.Stream(device=dev)
    sp = stream.cuda_stream

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize(dev)

    # ---- the delivery ring on rank 0: [slot k][rank r] = header + B frames -----------------------------------------
    slot_bytes = HEADER + B * cap
    ring_bytes = 2 * world * slot_bytes
    handle = torch.zeros(lib.RING_HANDLE_BYTES, dtype=torch.uint8, device=dev)
    ring = 0
    if rank == 0:
        r, ring, h = lib.ring_create(local_rank, ring_bytes)
        assert r == 0, f"HapB200RingCreate: {r}"
        handle.copy_(torch.frombuffer(bytearray(h), dtype=torch.uint8))
    if world > 1:
        dist.broadcast(handle, 0)
        if rank != 0:
            r, ring = lib.ring_open(local_rank, bytes(handle.cpu().numpy().tobytes()))
            assert r == 0, f"HapB200RingOpen: {r}"

    def slot(k, r):
        return ring + (k * world + r) * slot_bytes

    state = {"n": 0, "works": [[], []]}

    def step_peer():
        k = state["n"] & 1
        state["n"] += 1
        s = slot(k, rank)
        ps = producers[k].cuda_stream
        r = lib.encode_rgba_batch(rgba.data_ptr(), B, rgba_bytes, W, H, codec, 1, CH, s + HEADER, cap, s + 64, stream=ps)
        assert r == 0, r
        assert lib.ring_publish(local_rank, s, state["n"], stream=ps) == 0
        if rank == 0:
            for q in range(world):
                assert lib.ring_wait(local_rank, slot(k, q), state["n"], 0, stream=consumer.cuda_stream) == 0

    # ---- the NCCL baseline: two sets of local buffers, the delivery of batch i overlaps the encode of batch i+1 ---------
    frames2 = [torch.empty((B, cap), dtype=torch.uint8, device=dev) for _ in range(2)] if world > 1 else None
    used2 = [torch.zeros(B, dtype=torch.int64, device=dev) for _ in range(2)] if world > 1 else None
    gather2 = [torch.empty((world, B, cap), dtype=torch.uint8, device=dev) for _ in range(2)] if (rank == 0 and world > 1) else [None, None]
    moved = {"bytes": 0}

    def finish(k):
        for w in state["works"][k]:
            w.wait()
        state["works"][k] = []

    def step_nccl():
        k = state["n"] & 1
        state["n"] += 1
        finish(k)                       # the transfers that read / wrote buffer set k two batches ago
        r = lib.encode_rgba_batch(rgba.data_ptr(), B, rgba_bytes, W, H, codec, 1, CH, frames2[k].data_ptr(), cap, used2[k].data_ptr(), stream=sp)
        assert r == 0, r
        _, lengths, works = sharding.gatherv_frames_to_root(frames2[k], used2[k], 0, gather2[k], wait=False)
        state["works"][k] = works
        moved["bytes"] = int(lengths.sum() - lengths[0].sum())

    def timed(step, steps, drain=None):
        """K steps between events on the producer stream (and, on rank 0, the consumer stream); max over ranks, ms"""
        with torch.cuda.stream(stream):
            barrier()
            e0, e1, f1 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            c0, c1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            stream2.wait_event(e0)                 # the second producer stream starts inside the timed region too
            c0.record(consumer)
            for _ in range(steps):
                step()
            if drain:
                drain()
            e1.record(stream)
            f1.record(stream2)
            c1.record(consumer)
            barrier()
            t = max(e0.elapsed_time(e1), e0.elapsed_time(f1), c0.elapsed_time(c1), e0.elapsed_time(c1))
            ms = torch.tensor([t], dtype=torch.float64, device=dev)
            if world > 1:
                dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        return float(ms.item())

    sampler = ClockSampler(local_rank)
    with torch.cuda.stream(stream):
        for _ in range(max(args.warmup, 4)):
            step_peer()
    barrier()
    if rank == 0:
        sampler.start()
    launches0 = lib.launches()
    wall0 = time.time()
    ms_total = timed(step_peer, args.steps)
    wall1 = time.time()
    launches = lib.launches() - launches0
    clocks = sampler.stop(wall0, wall1) if rank == 0 else None
    last_k = (state["n"] - 1) & 1

    # encode alone into local memory (no delivery), for the share of the step the delivery costs
    local = torch.empty((B, cap), dtype=torch.uint8, device=dev)
    lused = torch.zeros(B, dtype=torch.int64, device=dev)

    def step_local():
        assert lib.encode_rgba_batch(rgba.data_ptr(), B, rgba_bytes, W, H, codec, 1, CH, local.data_ptr(), cap, lused.data_ptr(), stream=sp) == 0
    with torch.cuda.stream(stream):
        step_local()
    ms_enc = timed(step_local, args.steps)

    # ---- verification (outside the timed region): a frame the LAST rank wrote into the ring decodes on rank 0 to that rank's texture
    tex = torch.empty(tex_bytes, dtype=torch.uint8, device=dev)
    assert lib.block_encode_batch(rgba.data_ptr(), 1, rgba_bytes, W, H, codec, tex.data_ptr(), tex_bytes) == 0
    mine = torch.stack([tex.view(torch.int32).sum(dtype=torch.int64), tex[::4099].to(torch.int64).sum()])
    sums = torch.zeros((world, 2), dtype=torch.int64, device=dev)
    if world > 1:
        dist.all_gather_into_tensor(sums.view(-1), mine)
    else:
        sums[0] = mine
    verified, lengths, nvlink_bytes = None, None, 0
    if rank == 0:
        ring_t = torch.as_tensor(_DeviceBytes(ring, ring_bytes), device=dev)
        lengths = torch.zeros((world, B), dtype=torch.int64)
        for q in range(world):
            o = (last_k * world + q) * slot_bytes
            lengths[q] = ring_t[o + 64: o + 64 + 8 * B].view(torch.int64).cpu()
            assert int(ring_t[o: o + 4].view(torch.int32).item()) == state["n"], "a slot was not published"
        nvlink_bytes = int(lengths.sum() - lengths[0].sum())
        src_rank = world - 1
        n = int(lengths[src_rank, 0])
        back = torch.empty(tex_bytes, dtype=torch.uint8, device=dev)
        bu, bf, br = torch.zeros(1, dtype=torch.int64, device=dev), torch.zeros(1, dtype=torch.int32, device=dev), torch.full((1,), 9, dtype=torch.int32, device=dev)
        ln = torch.tensor([n], dtype=torch.int64, device=dev)
        src = slot(last_k, src_rank) + HEADER
        assert lib.decode_batch(src, 1, cap, ln.data_ptr(), 0, CH, back.data_ptr(), tex_bytes, bu.data_ptr(), bf.data_ptr(), br.data_ptr()) == 0
        got = torch.stack([back.view(torch.int32).sum(dtype=torch.int64), back[::4099].to(torch.int64).sum()])
        verified = bool(br.tolist() == [0] and bu.tolist() == [tex_bytes] and torch.equal(got, sums[src_rank]))
        assert verified, "a frame delivered to rank 0 does not decode to its sender's texture"
        del ring_t

    # ---- the NCCL gatherv baseline, same frames, same steps ------------------------------------------------------------
    ms_nccl = None
    if world > 1:
        state["n"] = 0
        with torch.cuda.stream(stream):
            for _ in range(3):
                step_nccl()
            finish(0)
            finish(1)
        ms_nccl = timed(step_nccl, args.steps, drain=lambda: (finish(0), finish(1)))

    barrier()
    if rank != 0:
        if world > 1:
            assert lib.ring_close(local_rank, ring) == 0
            dist.barrier()
            dist.destroy_process_group()
        return
    ms_step = ms_total / args.steps
    ms_enc_step = ms_enc / args.steps
    frames_per_step = world * B
    fps = frames_per_step / (ms_step * 1e-3)
    mean_frame = float(lengths.double().mean())
    line = {
        "metric": "hapq_16k_stream_encode_deliver_rgba_GBps", "value": frames_per_step * rgba_bytes / (ms_step * 1e-3) / 1e9, "unit": "GB/s",
        "n_gpus": world, "steps": args.steps, "warmup": max(args.warmup, 4), "ms_per_step": ms_step, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "u8", "data": "synthetic",
        "config": {"workload": f"hap_q_16k_stream({W}x{H},YCoCg-DXT5,snappy,{CH}chunks), frames round-robin over {world} gpu(s), encoded frames "
                               "delivered to rank 0 inside the timed region", "frames_per_gpu_per_step": B,
                   "l2": f"inputs larger than L2 ({B * rgba_bytes / 1e9:.2f} GB RGBA per step per GPU)",
                   "parallelism": f"dp{world}: every rank's frame-layout kernel stores its frames (and their lengths) straight into a delivery ring "
                                  "in rank 0's memory over NVLink (CUDA IPC peer mapping, HapB200Ring*), release-store flags, no collective; "
                                  "batches alternate between two producer streams per rank"},
        "fps": fps, "fps_target_of_config": 60,
        "encode_only_ms_per_step": ms_enc_step, "delivery_share_of_step": max(0.0, 1.0 - ms_enc_step / ms_step),
        "nvlink_bytes_per_step": nvlink_bytes, "nvlink_GBps_into_rank0": nvlink_bytes / (ms_step * 1e-3) / 1e9,
        "compression_ratio": mean_frame / tex_bytes, "delivered_frame_verified": verified,
        "roofline": {"bound": "hbm", "kernel": "encode pipeline (RGBA read)", "achieved": B * rgba_bytes / (ms_enc_step * 1e-3) / 1e9, "peak": peak,
                     "unit": "GB/s", "frac": B * rgba_bytes / (ms_enc_step * 1e-3) / 1e9 / peak, "traffic": None, "peak_source": peak_src},
        "clocks": clocks, "gpu_launches": launches,
    }
    line["delivery"] = "ring"
    if ms_nccl is not None:
        ms_n = ms_nccl / args.steps
        line["nccl_gatherv_baseline"] = {
            "what": "the same frames encoded into local memory, all-gather of the lengths + grouped ncclSend/ncclRecv to rank 0, the delivery of "
                    "batch i overlapping the encode of batch i+1", "ms_per_step": ms_n, "fps": frames_per_step / (ms_n * 1e-3),
            "value": frames_per_step * rgba_bytes / (ms_n * 1e-3) / 1e9, "nvlink_bytes_per_step": moved["bytes"],
            "nvlink_GBps_into_rank0": moved["bytes"] / (ms_n * 1e-3) / 1e9}
        if ms_n < ms_step:
            # Once rank 0's NVLink ingress is the bound (2.9 GB per step at N=8), a layout kernel that stores remotely holds its
            # SMs while the link is busy, whereas NCCL's copies run beside the next batch's encode, so which delivery is faster
            # depends on N.  The headline is the faster delivery at this N; both are in the line.
            b = line["nccl_gatherv_baseline"]
            line["ring_delivery"] = {"ms_per_step": ms_step, "fps": fps, "value": line["value"], "nvlink_GBps_into_rank0": line["nvlink_GBps_into_rank0"],
                                     "delivery_share_of_step": line["delivery_share_of_step"]}
            line.update({"delivery": "nccl_gatherv", "value": b["value"], "fps": b["fps"], "ms_per_step": b["ms_per_step"],
                         "nvlink_bytes_per_step": b["nvlink_bytes_per_step"], "nvlink_GBps_into_rank0": b["nvlink_GBps_into_rank0"],
                         "delivery_share_of_step": max(0.0, 1.0 - ms_enc_step / b["ms_per_step"])})
            line["config"]["parallelism"] = (f"dp{world}: frames encoded into local memory, all-gather of the lengths + grouped ncclSend/ncclRecv to rank 0 overlapping "
                                             "the next batch's encode (faster than the delivery ring at this N: `ring_delivery`)")
    emit(line)
    assert lib.ring_destroy(local_rank, ring) == 0
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
