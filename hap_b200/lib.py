"""Loader + ctypes signatures for libhap_b200.so (include/hap.h and include/hap_b200.h)."""
from __future__ import annotations

import ctypes as C
import functools
import os

from .abi import HapABI

HERE = os.path.dirname(os.path.abspath(__file__))

HapB200Codec_Hap1, HapB200Codec_Hap5, HapB200Codec_HapY, HapB200Codec_HapM, HapB200Codec_HapA = range(5)


def library_path() -> str:
    # HAPB200_LIBRARY: another build of the same library (A/B measurements of kernel variants)
    return os.environ.get("HAPB200_LIBRARY") or os.path.join(HERE, "libhap_b200.so")


class HapB200(HapABI):
    """The six hap.h entry points (inherited) plus the extensions of include/hap_b200.h.
    Batch calls take raw device addresses (ints, e.g. torch.Tensor.data_ptr())."""

    def __init__(self, path: str):
        super().__init__(path)
        L = self.lib
        vp, u, ul, ull_p, u_p = C.c_void_p, C.c_uint, C.c_ulong, C.POINTER(C.c_ulonglong), C.POINTER(C.c_uint)
        L.HapB200Version.restype = C.c_char_p
        L.HapB200KernelLaunchCount.restype = C.c_ulonglong
        L.HapB200SetDevice.restype = C.c_int
        L.HapB200SetDevice.argtypes = [C.c_int]
        L.HapB200GetDevice.restype = C.c_int
        L.HapB200SetOption.restype = C.c_int
        L.HapB200SetOption.argtypes = [C.c_int, C.c_int]
        L.HapB200SetStageTiming.restype = None
        L.HapB200SetStageTiming.argtypes = [C.c_int]
        L.HapB200StageTimes.restype = C.c_int
        L.HapB200StageTimes.argtypes = [C.POINTER(C.c_double), C.POINTER(C.c_ulonglong), C.c_int]
        L.HapB200MaxEncodedLengthRGBA.restype = ul
        L.HapB200MaxEncodedLengthRGBA.argtypes = [u, u, u, u]
        L.HapB200TextureBytes.restype = ul
        L.HapB200TextureBytes.argtypes = [u, u, u, u]
        L.HapB200EncodeRGBA.restype = u
        L.HapB200EncodeRGBA.argtypes = [vp, u, u, ul, u, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200DecodeRGBA.restype = u
        L.HapB200DecodeRGBA.argtypes = [vp, ul, u, u, vp, ul]
        L.HapB200EncodeRGBABatch.restype = u
        L.HapB200EncodeRGBABatch.argtypes = [vp, u, ul, u, u, ul, u, u, u, vp, ul, vp, vp]
        L.HapB200EncodeBatch.restype = u
        L.HapB200EncodeBatch.argtypes = [u, C.POINTER(vp), C.POINTER(ul), C.POINTER(ul), u_p, u_p, u_p, u, vp, ul, vp, vp]
        L.HapB200DecodeBatch.restype = u
        L.HapB200DecodeBatch.argtypes = [vp, u, ul, vp, u, u, vp, ul, vp, vp, vp, vp]
        L.HapB200DecodeRGBABatch.restype = u
        L.HapB200DecodeRGBABatch.argtypes = [vp, u, ul, vp, u, u, u, u, vp, ul, ul, vp, vp]
        L.HapB200BlockEncodeBatch.restype = u
        L.HapB200BlockEncodeBatch.argtypes = [vp, u, ul, u, u, ul, u, vp, ul, vp]
        L.HapB200BlockDecodeBatch.restype = u
        L.HapB200BlockDecodeBatch.argtypes = [vp, u, ul, u, u, u, vp, ul, ul, vp]
        for name, args in (("RingCreate", [C.c_int, ul, C.POINTER(vp), vp]), ("RingDestroy", [C.c_int, vp]),
                           ("RingOpen", [C.c_int, vp, C.POINTER(vp)]), ("RingClose", [C.c_int, vp]),
                           ("RingAttach", [C.c_int, C.c_int]), ("RingPublish", [C.c_int, vp, u, vp]), ("RingWait", [C.c_int, vp, u, u, vp])):
            f = getattr(L, "HapB200" + name)
            f.restype = u
            f.argtypes = args

    def version(self) -> str:
        return self.lib.HapB200Version().decode()

    def launches(self) -> int:
        return int(self.lib.HapB200KernelLaunchCount())

    OPTION_USE_INDEX, OPTION_WRITE_INDEX, OPTION_WRITE_OFFSET_TABLE, OPTION_CHROMA_REFINE = 1, 2, 3, 4

    def set_option(self, option: int, value: int) -> int:
        """OPTION_USE_INDEX: the decoder uses a frame's embedded fragment index (default on).  OPTION_WRITE_INDEX: the
        encoder adds the private fragment index section to Complex texture sections (default off: frames are laid out
        exactly as the reference lays them out)."""
        return int(self.lib.HapB200SetOption(option, value))

    STAGES = ("bc_encode", "snappy_encode", "plan", "place", "parse", "snappy_decode", "collect", "bc_decode", "snappy_index", "windows")

    def set_stage_timing(self, on: bool):
        self.lib.HapB200SetStageTiming(1 if on else 0)

    def stage_times(self):
        """{stage: (total ms, launches)} since the last call; synchronises the device."""
        ms = (C.c_double * 10)()
        n = (C.c_ulonglong * 10)()
        self.lib.HapB200StageTimes(ms, n, 10)
        return {s: (float(ms[i]), int(n[i])) for i, s in enumerate(self.STAGES)}

    @staticmethod
    def stage_algorithmic_bytes(frames, rgba_bytes, texture_bytes, mean_frame_bytes):
        """Algorithmic bytes one launch of each stage moves for a batch of `frames` frames (DESIGN.md section 4)."""
        F = frames
        return {
            "bc_encode": F * (rgba_bytes + texture_bytes),                 # RGBA read once + DXT written once
            "snappy_encode": F * texture_bytes + F * mean_frame_bytes,     # DXT read + element streams written
            "plan": F * 4096.0,
            "place": 2 * F * mean_frame_bytes,                             # element streams read + frame written
            "parse": F * 256.0,
            "snappy_decode": F * mean_frame_bytes + F * texture_bytes,     # execute kernel: frame read + texture written
            "snappy_index": F * mean_frame_bytes * (1.0 + 1.0 / 64),       # index kernel: frame read + one entry per 64 bytes written
            "windows": F * 4096.0,
            "collect": F * 64.0,
            "bc_decode": F * (texture_bytes + rgba_bytes),
        }

    def max_encoded_length_rgba(self, w, h, codec, chunks) -> int:
        return int(self.lib.HapB200MaxEncodedLengthRGBA(w, h, codec, chunks))

    def texture_bytes(self, w, h, codec, index=0) -> int:
        return int(self.lib.HapB200TextureBytes(w, h, codec, index))

    # -- single frame, host or device pointers ------------------------------------------------------
    def encode_rgba(self, rgba, w, h, codec, compressor=1, chunks=1, row_bytes=None, out=None, out_capacity=None):
        """rgba: buffer object or (addr, nbytes).  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        addr, _ = _as_ptr(rgba)
        cap = self.max_encoded_length_rgba(w, h, codec, chunks) if out_capacity is None else out_capacity
        own = out is None
        if own:
            out = bytearray(max(cap, 1))
        oaddr, _ = _as_ptr(out)
        used = C.c_ulong(0)
        r = self.lib.HapB200EncodeRGBA(addr, w, h, row_bytes or 4 * w, codec, compressor, chunks, oaddr, cap, C.byref(used))
        if r != 0:
            return int(r), None
        return 0, (bytes(memoryview(out)[: used.value]) if own else used.value)

    def decode_rgba(self, frame, w, h, out=None, row_bytes=None, frame_bytes=None):
        from .abi import _as_ptr
        faddr, fn = _as_ptr(frame)
        if frame_bytes is not None:
            fn = frame_bytes
        own = out is None
        if own:
            out = bytearray(4 * w * h)
        oaddr, _ = _as_ptr(out)
        r = self.lib.HapB200DecodeRGBA(faddr, fn, w, h, oaddr, row_bytes or 4 * w)
        return int(r), (bytes(out) if own and r == 0 else None)

    # -- device-resident batches (addresses are ints) ---------------------------------------------
    def encode_rgba_batch(self, rgba, frames, frame_stride, w, h, codec, compressor, chunks, out, out_stride, used,
                          row_bytes=None, stream=None):
        return int(self.lib.HapB200EncodeRGBABatch(rgba, frames, frame_stride, w, h, row_bytes or 4 * w, codec, compressor,
                                                   chunks, out, out_stride, used, stream))

    def encode_batch(self, textures, strides, nbytes, formats, compressors, chunks, frames, out, out_stride, used, stream=None):
        n = len(textures)
        return int(self.lib.HapB200EncodeBatch(n, (C.c_void_p * n)(*textures), (C.c_ulong * n)(*strides),
                                               (C.c_ulong * n)(*nbytes), (C.c_uint * n)(*formats),
                                               (C.c_uint * n)(*compressors), (C.c_uint * n)(*chunks), frames, out,
                                               out_stride, used, stream))

    def decode_batch(self, frames_ptr, frames, in_stride, in_bytes, index, max_chunks, out, out_stride, used, formats,
                     results, stream=None):
        return int(self.lib.HapB200DecodeBatch(frames_ptr, frames, in_stride, in_bytes, index, max_chunks, out, out_stride,
                                               used, formats, results, stream))

    def decode_rgba_batch(self, frames_ptr, frames, in_stride, in_bytes, max_chunks, codec, w, h, rgba, frame_stride,
                          results, row_bytes=None, stream=None):
        return int(self.lib.HapB200DecodeRGBABatch(frames_ptr, frames, in_stride, in_bytes, max_chunks, codec, w, h, rgba,
                                                   frame_stride, row_bytes or 4 * w, results, stream))

    def block_encode_batch(self, rgba, frames, frame_stride, w, h, codec, blocks, blocks_stride, row_bytes=None, stream=None):
        return int(self.lib.HapB200BlockEncodeBatch(rgba, frames, frame_stride, w, h, row_bytes or 4 * w, codec, blocks,
                                                    blocks_stride, stream))

    def block_decode_batch(self, blocks, frames, blocks_stride, w, h, codec, rgba, frame_stride, row_bytes=None, stream=None):
        return int(self.lib.HapB200BlockDecodeBatch(blocks, frames, blocks_stride, w, h, codec, rgba, frame_stride,
                                                    row_bytes or 4 * w, stream))


    # -- delivery rings (include/hap_b200.h): frames written straight into another GPU's memory -----------------
    RING_HANDLE_BYTES = 64

    def ring_create(self, device: int, nbytes: int):
        """(result, ring address, 64-byte handle for the producers)"""
        ring = C.c_void_p(0)
        handle = (C.c_ubyte * self.RING_HANDLE_BYTES)()
        r = self.lib.HapB200RingCreate(device, nbytes, C.byref(ring), handle)
        return int(r), int(ring.value or 0), bytes(handle)

    def ring_destroy(self, device: int, ring: int) -> int:
        return int(self.lib.HapB200RingDestroy(device, ring))

    def ring_open(self, device: int, handle: bytes):
        ring = C.c_void_p(0)
        buf = (C.c_ubyte * self.RING_HANDLE_BYTES).from_buffer_copy(handle)
        r = self.lib.HapB200RingOpen(device, buf, C.byref(ring))
        return int(r), int(ring.value or 0)

    def ring_close(self, device: int, ring: int) -> int:
        return int(self.lib.HapB200RingClose(device, ring))

    def ring_attach(self, device: int, ring_device: int) -> int:
        return int(self.lib.HapB200RingAttach(device, ring_device))

    def ring_publish(self, device: int, flag: int, value: int, stream=None) -> int:
        return int(self.lib.HapB200RingPublish(device, flag, value, stream))

    def ring_wait(self, device: int, flag: int, value: int, timeout_ms: int = 0, stream=None) -> int:
        return int(self.lib.HapB200RingWait(device, flag, value, timeout_ms, stream))


@functools.lru_cache(None)
def load() -> HapB200:
    path = library_path()
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} is missing: build it with `python -m hap_b200.build` (nvcc, sm_90a). "
            "hap_b200 has no CPU implementation to fall back to.")
    return HapB200(path)
