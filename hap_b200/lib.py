"""Loader + ctypes signatures for libhap_b200.so (include/hap.h and include/hap_b200.h)."""
from __future__ import annotations

import ctypes as C
import functools
import os

from .abi import HapABI

HERE = os.path.dirname(os.path.abspath(__file__))

HapB200Codec_Hap1, HapB200Codec_Hap5, HapB200Codec_HapY, HapB200Codec_HapM, HapB200Codec_HapA, HapB200Codec_Hap7 = range(6)
# HapB200Codec_Hap7 ("Hap R", BC7): the codec-taking RGBA encode entry points refuse it with HapResult_Bad_Arguments; the
# BC7 encoders (encode_rgba_bc7, encode_rgba_bc7_batch, block_encode_bc7_batch; from NV12 / P010 and planar pictures
# encode_yuv_bc7, encode_planar_bc7 and their batch forms) ask for it by name
HapB200YUV_NV12, HapB200YUV_P010 = range(2)
HapB200YUV_BT601_Limited, HapB200YUV_BT601_Full, HapB200YUV_BT709_Limited, HapB200YUV_BT709_Full = range(4)
# BT.2020: taken only by the HDR10 encoders (encode_yuv_pq, encode_yuv_pq_batch, block_encode_yuv_pq_batch) and decoders
# (decode_yuv_pq, decode_yuv_pq_batch, block_decode_yuv_pq_batch)
HapB200YUV_BT2020_Limited, HapB200YUV_BT2020_Full = 4, 5
HapB200Chroma_420, HapB200Chroma_422, HapB200Chroma_444 = range(3)


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
        L.HapB200DecodeRGBAHalf.restype = u
        L.HapB200DecodeRGBAHalf.argtypes = [vp, ul, u, u, vp, ul]
        L.HapB200DecodeRGBAHalfBatch.restype = u
        L.HapB200DecodeRGBAHalfBatch.argtypes = [vp, u, ul, vp, u, u, u, vp, ul, ul, vp, vp]
        L.HapB200BlockDecodeHalfBatch.restype = u
        L.HapB200BlockDecodeHalfBatch.argtypes = [vp, u, ul, u, u, u, vp, ul, ul, vp]
        L.HapB200EncodeRGBAHalf.restype = u
        L.HapB200EncodeRGBAHalf.argtypes = [vp, u, u, ul, u, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200EncodeRGBAHalfBatch.restype = u
        L.HapB200EncodeRGBAHalfBatch.argtypes = [vp, u, ul, u, u, ul, u, u, u, vp, ul, vp, vp]
        L.HapB200BlockEncodeHalfBatch.restype = u
        L.HapB200EncodeRGBABC7.restype = u
        L.HapB200EncodeRGBABC7.argtypes = [vp, u, u, ul, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200EncodeRGBABC7Batch.restype = u
        L.HapB200EncodeRGBABC7Batch.argtypes = [vp, u, ul, u, u, ul, u, u, vp, ul, vp, vp]
        L.HapB200BlockEncodeBC7Batch.restype = u
        L.HapB200BlockEncodeBC7Batch.argtypes = [vp, u, ul, u, u, ul, vp, ul, vp]
        L.HapB200BlockEncodeHalfBatch.argtypes = [vp, u, ul, u, u, ul, u, vp, ul, vp]
        L.HapB200EncodeYUV.restype = u
        L.HapB200EncodeYUV.argtypes = [vp, vp, u, u, ul, u, u, u, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200EncodeYUVBatch.restype = u
        L.HapB200EncodeYUVBatch.argtypes = [vp, vp, u, ul, u, u, ul, u, u, u, u, u, vp, ul, vp, vp]
        L.HapB200BlockEncodeYUVBatch.restype = u
        L.HapB200BlockEncodeYUVBatch.argtypes = [vp, vp, u, ul, u, u, ul, u, u, u, vp, ul, vp]
        L.HapB200EncodeYUVBC7.restype = u
        L.HapB200EncodeYUVBC7.argtypes = [vp, vp, u, u, ul, u, u, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200EncodeYUVBC7Batch.restype = u
        L.HapB200EncodeYUVBC7Batch.argtypes = [vp, vp, u, ul, u, u, ul, u, u, u, u, vp, ul, vp, vp]
        L.HapB200BlockEncodeYUVBC7Batch.restype = u
        L.HapB200BlockEncodeYUVBC7Batch.argtypes = [vp, vp, u, ul, u, u, ul, u, u, vp, ul, vp]
        L.HapB200EncodePlanarBC7.restype = u
        L.HapB200EncodePlanarBC7.argtypes = [vp, vp, vp, vp, u, u, ul, ul, u, u, u, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200EncodePlanarBC7Batch.restype = u
        L.HapB200EncodePlanarBC7Batch.argtypes = [vp, vp, vp, vp, u, ul, u, u, ul, ul, u, u, u, u, u, vp, ul, vp, vp]
        L.HapB200BlockEncodePlanarBC7Batch.restype = u
        L.HapB200BlockEncodePlanarBC7Batch.argtypes = [vp, vp, vp, vp, u, ul, u, u, ul, ul, u, u, u, vp, ul, vp]
        L.HapB200EncodePlanar.restype = u
        L.HapB200EncodePlanar.argtypes = [vp, vp, vp, vp, u, u, ul, ul, u, u, u, u, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200EncodePlanarBatch.restype = u
        L.HapB200EncodePlanarBatch.argtypes = [vp, vp, vp, vp, u, ul, u, u, ul, ul, u, u, u, u, u, u, vp, ul, vp, vp]
        L.HapB200BlockEncodePlanarBatch.restype = u
        L.HapB200BlockEncodePlanarBatch.argtypes = [vp, vp, vp, vp, u, ul, u, u, ul, ul, u, u, u, u, vp, ul, vp]
        L.HapB200DecodeYUV.restype = u
        L.HapB200DecodeYUV.argtypes = [vp, ul, u, u, vp, vp, ul, u, u]
        L.HapB200DecodeYUVBatch.restype = u
        L.HapB200DecodeYUVBatch.argtypes = [vp, u, ul, vp, u, u, u, u, vp, vp, ul, ul, u, u, vp, vp]
        L.HapB200BlockDecodeYUVBatch.restype = u
        L.HapB200BlockDecodeYUVBatch.argtypes = [vp, u, ul, u, u, u, vp, vp, ul, ul, u, u, vp]
        L.HapB200DecodePlanar.restype = u
        L.HapB200DecodePlanar.argtypes = [vp, ul, u, u, vp, vp, vp, vp, ul, ul, u, u, u]
        L.HapB200DecodePlanarBatch.restype = u
        L.HapB200DecodePlanarBatch.argtypes = [vp, u, ul, vp, u, u, u, u, vp, vp, vp, vp, ul, ul, ul, u, u, u, vp, vp]
        L.HapB200BlockDecodePlanarBatch.restype = u
        L.HapB200BlockDecodePlanarBatch.argtypes = [vp, u, ul, u, u, u, vp, vp, vp, vp, ul, ul, ul, u, u, u, vp]
        L.HapB200EncodeYUVPQ.restype = u
        L.HapB200EncodeYUVPQ.argtypes = [vp, vp, u, u, ul, u, u, u, u, u, vp, ul, C.POINTER(ul)]
        L.HapB200EncodeYUVPQBatch.restype = u
        L.HapB200EncodeYUVPQBatch.argtypes = [vp, vp, u, ul, u, u, ul, u, u, u, u, u, vp, ul, vp, vp]
        L.HapB200BlockEncodeYUVPQBatch.restype = u
        L.HapB200BlockEncodeYUVPQBatch.argtypes = [vp, vp, u, ul, u, u, ul, u, u, u, vp, ul, vp]
        L.HapB200DecodeYUVPQ.restype = u
        L.HapB200DecodeYUVPQ.argtypes = [vp, ul, u, u, vp, vp, ul, u, u]
        L.HapB200DecodeYUVPQBatch.restype = u
        L.HapB200DecodeYUVPQBatch.argtypes = [vp, u, ul, vp, u, u, u, vp, vp, ul, ul, u, u, vp, vp]
        L.HapB200BlockDecodeYUVPQBatch.restype = u
        L.HapB200BlockDecodeYUVPQBatch.argtypes = [vp, u, ul, u, u, u, vp, vp, ul, ul, u, u, vp]
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
    @staticmethod
    def _encode_frame(cap, out, encode):
        """The single-frame encoders' tail: encode(out address, cap, pointer to the bytes used) writes the frame into `out`, or
        into a new buffer of cap bytes when `out` is None.  Returns (result, frame bytes | used), (result, None) on failure."""
        from .abi import _as_ptr
        own = out is None
        if own:
            out = bytearray(max(cap, 1))
        oaddr, _ = _as_ptr(out)
        used = C.c_ulong(0)
        r = encode(oaddr, cap, C.byref(used))
        if r != 0:
            return int(r), None
        return 0, (bytes(memoryview(out)[: used.value]) if own else used.value)

    @staticmethod
    def _decode_frame(frame, frame_bytes, planes, sizes, decode):
        """The single-frame decoders' tail: decode(frame address, frame bytes, plane addresses...) writes the picture's planes
        (buffer objects or (addr, nbytes)); when none is given they are allocated here, sizes[i] bytes each.  Returns (result,
        the planes' bytes when allocated here and the call succeeded -- one plane: its bytes, else a tuple -- else None)."""
        from .abi import _as_ptr
        faddr, fn = _as_ptr(frame)
        if frame_bytes is not None:
            fn = frame_bytes
        own = all(p is None for p in planes)
        if own:
            planes = [bytearray(n) for n in sizes]
        r = decode(faddr, fn, *[_as_ptr(p)[0] for p in planes])
        if not (own and r == 0):
            return int(r), None
        return int(r), (bytes(planes[0]) if len(planes) == 1 else tuple(bytes(p) for p in planes))

    def encode_rgba(self, rgba, w, h, codec, compressor=1, chunks=1, row_bytes=None, out=None, out_capacity=None):
        """rgba: buffer object or (addr, nbytes).  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        addr, _ = _as_ptr(rgba)
        cap = self.max_encoded_length_rgba(w, h, codec, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodeRGBA(addr, w, h, row_bytes or 4 * w, codec, compressor,
                                                                                         chunks, o, n, used))

    def decode_rgba(self, frame, w, h, out=None, row_bytes=None, frame_bytes=None):
        return self._decode_frame(frame, frame_bytes, [out], [4 * w * h],
                                  lambda f, n, o: self.lib.HapB200DecodeRGBA(f, n, w, h, o, row_bytes or 4 * w))

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

    # -- Hap HDR (BC6H) -> RGBA16F: 8 bytes per pixel, binary16 R, G, B, A (A = 1.0) ---------------------------------------
    def decode_rgba_half(self, frame, w, h, out=None, row_bytes=None, frame_bytes=None):
        """One Hap HDR frame (buffer object or (addr, nbytes)) -> (result, RGBA16F bytes when `out` is not given)"""
        return self._decode_frame(frame, frame_bytes, [out], [8 * w * h],
                                  lambda f, n, o: self.lib.HapB200DecodeRGBAHalf(f, n, w, h, o, row_bytes or 8 * w))

    def decode_rgba_half_batch(self, frames_ptr, frames, in_stride, in_bytes, max_chunks, w, h, rgba, frame_stride, results,
                               row_bytes=None, stream=None):
        return int(self.lib.HapB200DecodeRGBAHalfBatch(frames_ptr, frames, in_stride, in_bytes, max_chunks, w, h, rgba,
                                                       frame_stride, row_bytes or 8 * w, results, stream))

    def block_decode_half_batch(self, blocks, frames, blocks_stride, w, h, texture_format, rgba, frame_stride, row_bytes=None,
                                stream=None):
        return int(self.lib.HapB200BlockDecodeHalfBatch(blocks, frames, blocks_stride, w, h, texture_format, rgba, frame_stride,
                                                        row_bytes or 8 * w, stream))

    # -- RGBA16F -> Hap HDR (BC6H): texture_format UF16 or SF16; A is ignored --------------------------------------------------
    def max_encoded_length_half(self, w, h, texture_format, chunks) -> int:
        """the output a frame of encode_rgba_half / encode_rgba_half_batch needs (HapMaxEncodedLength of its one texture)"""
        return self.max_encoded_length([(w // 4) * (h // 4) * 16], [texture_format], [chunks])

    def encode_rgba_half(self, rgba, w, h, texture_format, compressor=1, chunks=1, row_bytes=None, out=None, out_capacity=None):
        """rgba: buffer object or (addr, nbytes), 8 bytes per pixel.  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        addr, _ = _as_ptr(rgba)
        cap = self.max_encoded_length_half(w, h, texture_format, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodeRGBAHalf(addr, w, h, row_bytes or 8 * w, texture_format,
                                                                                             compressor, chunks, o, n, used))

    def encode_rgba_half_batch(self, rgba, frames, frame_stride, w, h, texture_format, compressor, chunks, out, out_stride, used,
                               row_bytes=None, stream=None):
        return int(self.lib.HapB200EncodeRGBAHalfBatch(rgba, frames, frame_stride, w, h, row_bytes or 8 * w, texture_format,
                                                       compressor, chunks, out, out_stride, used, stream))

    def block_encode_half_batch(self, rgba, frames, frame_stride, w, h, texture_format, blocks, blocks_stride, row_bytes=None,
                                stream=None):
        return int(self.lib.HapB200BlockEncodeHalfBatch(rgba, frames, frame_stride, w, h, row_bytes or 8 * w, texture_format,
                                                        blocks, blocks_stride, stream))

    # -- RGBA8 -> Hap R (BC7): frames need max_encoded_length_rgba(w, h, HapB200Codec_Hap7, chunks) --------------------------
    def encode_rgba_bc7(self, rgba, w, h, compressor=1, chunks=1, row_bytes=None, out=None, out_capacity=None):
        """rgba: buffer object or (addr, nbytes), 4 bytes per pixel.  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        addr, _ = _as_ptr(rgba)
        cap = self.max_encoded_length_rgba(w, h, HapB200Codec_Hap7, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodeRGBABC7(addr, w, h, row_bytes or 4 * w, compressor, chunks,
                                                                                            o, n, used))

    def encode_rgba_bc7_batch(self, rgba, frames, frame_stride, w, h, compressor, chunks, out, out_stride, used, row_bytes=None,
                              stream=None):
        return int(self.lib.HapB200EncodeRGBABC7Batch(rgba, frames, frame_stride, w, h, row_bytes or 4 * w, compressor, chunks, out,
                                                      out_stride, used, stream))

    def block_encode_bc7_batch(self, rgba, frames, frame_stride, w, h, blocks, blocks_stride, row_bytes=None, stream=None):
        return int(self.lib.HapB200BlockEncodeBC7Batch(rgba, frames, frame_stride, w, h, row_bytes or 4 * w, blocks, blocks_stride,
                                                       stream))

    # -- NV12 / P010 -> Hap, Hap Alpha, Hap Q, Hap Q Alpha: layout HapB200YUV_*, color_space HapB200YUV_BT*; both planes
    #    have the row pitch `pitch` (default: width bytes per sample); frames need max_encoded_length_rgba(w, h, codec, chunks)
    def encode_yuv(self, luma, chroma, w, h, layout, color_space, codec, compressor=1, chunks=1, pitch=None, out=None,
                   out_capacity=None):
        """luma, chroma: buffer objects or (addr, nbytes).  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        laddr, _ = _as_ptr(luma)
        caddr, _ = _as_ptr(chroma)
        cap = self.max_encoded_length_rgba(w, h, codec, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodeYUV(
            laddr, caddr, w, h, pitch or (2 if layout == HapB200YUV_P010 else 1) * w, layout, color_space, codec, compressor, chunks, o, n,
            used))

    def encode_yuv_batch(self, luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, codec, compressor, chunks, out,
                         out_stride, used, stream=None):
        return int(self.lib.HapB200EncodeYUVBatch(luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, codec,
                                                  compressor, chunks, out, out_stride, used, stream))

    def block_encode_yuv_batch(self, luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, codec, blocks,
                               blocks_stride, stream=None):
        return int(self.lib.HapB200BlockEncodeYUVBatch(luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, codec,
                                                       blocks, blocks_stride, stream))

    # -- planar Y'CbCr (+ alpha) -> Hap, Hap Alpha, Hap Q, Hap Q Alpha, Hap Alpha-Only: subsampling HapB200Chroma_*, bit_depth
    #    8 / 10 / 12 (10 and 12: little-endian 16-bit words, sample in the low bits), color_space BT.601 / BT.709; luma and alpha
    #    rows luma_pitch apart (default: width samples), Cb and Cr rows chroma_pitch apart (default: their width in samples);
    #    alpha None: A = 255; HapA reads alpha alone (luma, cb, cr may be None).  Frames need max_encoded_length_rgba(w, h, codec,
    #    chunks)
    @staticmethod
    def _planar_pitches(w, subsampling, bit_depth, luma_pitch, chroma_pitch):
        sb = 1 if bit_depth == 8 else 2
        cw = w if subsampling == HapB200Chroma_444 else w // 2
        return luma_pitch or sb * w, chroma_pitch or sb * cw

    def encode_planar(self, luma, cb, cr, alpha, w, h, subsampling, bit_depth, color_space, codec, compressor=1, chunks=1,
                      luma_pitch=None, chroma_pitch=None, out=None, out_capacity=None):
        """luma, cb, cr, alpha: buffer objects, (addr, nbytes) or None.  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        addrs = [0 if b is None else _as_ptr(b)[0] for b in (luma, cb, cr, alpha)]
        lp, cp = self._planar_pitches(w, subsampling, bit_depth, luma_pitch, chroma_pitch)
        cap = self.max_encoded_length_rgba(w, h, codec, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodePlanar(
            *addrs, w, h, lp, cp, subsampling, bit_depth, color_space, codec, compressor, chunks, o, n, used))

    def encode_planar_batch(self, luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch, subsampling, bit_depth,
                            color_space, codec, compressor, chunks, out, out_stride, used, stream=None):
        return int(self.lib.HapB200EncodePlanarBatch(luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch,
                                                     subsampling, bit_depth, color_space, codec, compressor, chunks, out, out_stride,
                                                     used, stream))

    def block_encode_planar_batch(self, luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch, subsampling,
                                  bit_depth, color_space, codec, blocks, blocks_stride, stream=None):
        return int(self.lib.HapB200BlockEncodePlanarBatch(luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch,
                                                          subsampling, bit_depth, color_space, codec, blocks, blocks_stride, stream))

    # -- NV12 / P010 and planar Y'CbCr (+ alpha) -> Hap R (BC7): the arguments of encode_yuv* / encode_planar* without the
    #    codec; exactly the bytes of the RGBA8 BC7 encoders on the converted picture; a planar alpha None means A = 255.
    #    Frames need max_encoded_length_rgba(w, h, HapB200Codec_Hap7, chunks)
    def encode_yuv_bc7(self, luma, chroma, w, h, layout, color_space, compressor=1, chunks=1, pitch=None, out=None, out_capacity=None):
        """luma, chroma: buffer objects or (addr, nbytes).  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        laddr, _ = _as_ptr(luma)
        caddr, _ = _as_ptr(chroma)
        cap = self.max_encoded_length_rgba(w, h, HapB200Codec_Hap7, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodeYUVBC7(
            laddr, caddr, w, h, pitch or (2 if layout == HapB200YUV_P010 else 1) * w, layout, color_space, compressor, chunks, o, n, used))

    def encode_yuv_bc7_batch(self, luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, compressor, chunks, out,
                             out_stride, used, stream=None):
        return int(self.lib.HapB200EncodeYUVBC7Batch(luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, compressor,
                                                     chunks, out, out_stride, used, stream))

    def block_encode_yuv_bc7_batch(self, luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, blocks, blocks_stride,
                                   stream=None):
        return int(self.lib.HapB200BlockEncodeYUVBC7Batch(luma, chroma, frames, frame_stride, w, h, pitch, layout, color_space, blocks,
                                                          blocks_stride, stream))

    def encode_planar_bc7(self, luma, cb, cr, alpha, w, h, subsampling, bit_depth, color_space, compressor=1, chunks=1,
                          luma_pitch=None, chroma_pitch=None, out=None, out_capacity=None):
        """luma, cb, cr, alpha: buffer objects, (addr, nbytes) or None.  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        addrs = [0 if b is None else _as_ptr(b)[0] for b in (luma, cb, cr, alpha)]
        lp, cp = self._planar_pitches(w, subsampling, bit_depth, luma_pitch, chroma_pitch)
        cap = self.max_encoded_length_rgba(w, h, HapB200Codec_Hap7, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodePlanarBC7(
            *addrs, w, h, lp, cp, subsampling, bit_depth, color_space, compressor, chunks, o, n, used))

    def encode_planar_bc7_batch(self, luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch, subsampling,
                                bit_depth, color_space, compressor, chunks, out, out_stride, used, stream=None):
        return int(self.lib.HapB200EncodePlanarBC7Batch(luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch,
                                                        subsampling, bit_depth, color_space, compressor, chunks, out, out_stride, used,
                                                        stream))

    def block_encode_planar_bc7_batch(self, luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch, subsampling,
                                      bit_depth, color_space, blocks, blocks_stride, stream=None):
        return int(self.lib.HapB200BlockEncodePlanarBC7Batch(luma, cb, cr, alpha, frames, frame_stride, w, h, luma_pitch, chroma_pitch,
                                                             subsampling, bit_depth, color_space, blocks, blocks_stride, stream))

    # -- Hap (every codec but Hap HDR) -> NV12 / P010: layout HapB200YUV_*, color_space BT.601 / BT.709 (no BT.2020); both
    #    planes have the row pitch `pitch` (default: width bytes per sample)
    def decode_yuv(self, frame, w, h, layout, color_space, pitch=None, luma=None, chroma=None, frame_bytes=None):
        """frame, luma, chroma: buffer objects or (addr, nbytes).  Returns (result, (luma bytes, chroma bytes)) when it
        allocates the planes (luma and chroma not given), else (result, None)."""
        pitch = pitch or (2 if layout == HapB200YUV_P010 else 1) * w
        return self._decode_frame(frame, frame_bytes, [luma, chroma], [pitch * h, pitch * (h // 2)],
                                  lambda f, n, lu, ch: self.lib.HapB200DecodeYUV(f, n, w, h, lu, ch, pitch, layout, color_space))

    def decode_yuv_batch(self, frames_ptr, frames, in_stride, in_bytes, max_chunks, codec, w, h, luma, chroma, frame_stride, pitch, layout,
                         color_space, results, stream=None):
        return int(self.lib.HapB200DecodeYUVBatch(frames_ptr, frames, in_stride, in_bytes, max_chunks, codec, w, h, luma, chroma, frame_stride,
                                                  pitch, layout, color_space, results, stream))

    def block_decode_yuv_batch(self, blocks, frames, blocks_stride, w, h, codec, luma, chroma, frame_stride, pitch, layout, color_space,
                               stream=None):
        return int(self.lib.HapB200BlockDecodeYUVBatch(blocks, frames, blocks_stride, w, h, codec, luma, chroma, frame_stride, pitch, layout,
                                                       color_space, stream))

    # -- Hap (every codec but Hap HDR) -> planar Y'CbCr (+ alpha): subsampling HapB200Chroma_*, bit_depth 8 / 10 / 12 (10 and 12:
    #    little-endian 16-bit words, sample in the low bits), color_space BT.601 / BT.709 (no BT.2020); pitches as for
    #    encode_planar; alpha None: no alpha is written; HapA writes alpha alone (luma, cb, cr may be None)
    def decode_planar(self, frame, w, h, subsampling, bit_depth, color_space, *, with_alpha=True, luma=None, cb=None, cr=None, alpha=None,
                      luma_pitch=None, chroma_pitch=None, frame_bytes=None):
        """frame and the planes: buffer objects, (addr, nbytes) or None.  When no plane is given they are allocated here, the
        alpha plane only when with_alpha.  Returns (result, (luma, cb, cr, alpha or None) bytes) when it allocated the planes and
        the call succeeded, else (result, None)."""
        from .abi import _as_ptr
        lp, cp = self._planar_pitches(w, subsampling, bit_depth, luma_pitch, chroma_pitch)
        rows = h // 2 if subsampling == HapB200Chroma_420 else h
        planes = [luma, cb, cr, alpha]
        own = all(p is None for p in planes)
        if own:
            planes = [bytearray(lp * h), bytearray(cp * rows), bytearray(cp * rows), bytearray(lp * h) if with_alpha else None]
        faddr, fn = _as_ptr(frame)
        r = int(self.lib.HapB200DecodePlanar(faddr, fn if frame_bytes is None else frame_bytes, w, h,
                                             *[0 if p is None else _as_ptr(p)[0] for p in planes], lp, cp, subsampling, bit_depth,
                                             color_space))
        if not (own and r == 0):
            return r, None
        return r, tuple(None if p is None else bytes(p) for p in planes)

    def decode_planar_batch(self, frames_ptr, frames, in_stride, in_bytes, max_chunks, codec, w, h, luma, cb, cr, alpha, frame_stride,
                            luma_pitch, chroma_pitch, subsampling, bit_depth, color_space, results, stream=None):
        return int(self.lib.HapB200DecodePlanarBatch(frames_ptr, frames, in_stride, in_bytes, max_chunks, codec, w, h, luma, cb, cr, alpha,
                                                     frame_stride, luma_pitch, chroma_pitch, subsampling, bit_depth, color_space, results,
                                                     stream))

    def block_decode_planar_batch(self, blocks, frames, blocks_stride, w, h, codec, luma, cb, cr, alpha, frame_stride, luma_pitch,
                                  chroma_pitch, subsampling, bit_depth, color_space, stream=None):
        return int(self.lib.HapB200BlockDecodePlanarBatch(blocks, frames, blocks_stride, w, h, codec, luma, cb, cr, alpha, frame_stride,
                                                          luma_pitch, chroma_pitch, subsampling, bit_depth, color_space, stream))

    # -- HDR10 P010 (BT.2020, PQ) -> Hap HDR (BC6H): color_space HapB200YUV_BT2020_*, unit_nits the cd/m2 of 1.0 (1-10000),
    #    texture_format UF16 or SF16; planes as for encode_yuv with HapB200YUV_P010 (pitch default 2 * width); frames need
    #    max_encoded_length_half(w, h, texture_format, chunks)
    def encode_yuv_pq(self, luma, chroma, w, h, color_space, unit_nits, texture_format, compressor=1, chunks=1, pitch=None, out=None,
                      out_capacity=None):
        """luma, chroma: buffer objects or (addr, nbytes).  Returns (result, frame bytes | used)."""
        from .abi import _as_ptr
        laddr, _ = _as_ptr(luma)
        caddr, _ = _as_ptr(chroma)
        cap = self.max_encoded_length_half(w, h, texture_format, chunks) if out_capacity is None else out_capacity
        return self._encode_frame(cap, out, lambda o, n, used: self.lib.HapB200EncodeYUVPQ(
            laddr, caddr, w, h, pitch or 2 * w, color_space, unit_nits, texture_format, compressor, chunks, o, n, used))

    def encode_yuv_pq_batch(self, luma, chroma, frames, frame_stride, w, h, pitch, color_space, unit_nits, texture_format, compressor,
                            chunks, out, out_stride, used, stream=None):
        return int(self.lib.HapB200EncodeYUVPQBatch(luma, chroma, frames, frame_stride, w, h, pitch, color_space, unit_nits,
                                                    texture_format, compressor, chunks, out, out_stride, used, stream))

    def block_encode_yuv_pq_batch(self, luma, chroma, frames, frame_stride, w, h, pitch, color_space, unit_nits, texture_format, blocks,
                                  blocks_stride, stream=None):
        return int(self.lib.HapB200BlockEncodeYUVPQBatch(luma, chroma, frames, frame_stride, w, h, pitch, color_space, unit_nits,
                                                         texture_format, blocks, blocks_stride, stream))

    # -- Hap HDR (BC6H) -> HDR10 P010 (BT.2020, PQ): color_space HapB200YUV_BT2020_*, unit_nits the cd/m2 of 1.0 (1-10000);
    #    planes as for decode_yuv with HapB200YUV_P010 (pitch default 2 * width)
    def decode_yuv_pq(self, frame, w, h, color_space, unit_nits, pitch=None, luma=None, chroma=None, frame_bytes=None):
        """frame, luma, chroma: buffer objects or (addr, nbytes).  Returns (result, (luma bytes, chroma bytes)) when it
        allocates the planes (luma and chroma not given), else (result, None)."""
        pitch = pitch or 2 * w
        return self._decode_frame(frame, frame_bytes, [luma, chroma], [pitch * h, pitch * (h // 2)],
                                  lambda f, n, lu, ch: self.lib.HapB200DecodeYUVPQ(f, n, w, h, lu, ch, pitch, color_space, unit_nits))

    def decode_yuv_pq_batch(self, frames_ptr, frames, in_stride, in_bytes, max_chunks, w, h, luma, chroma, frame_stride, pitch, color_space,
                            unit_nits, results, stream=None):
        return int(self.lib.HapB200DecodeYUVPQBatch(frames_ptr, frames, in_stride, in_bytes, max_chunks, w, h, luma, chroma, frame_stride,
                                                    pitch, color_space, unit_nits, results, stream))

    def block_decode_yuv_pq_batch(self, blocks, frames, blocks_stride, w, h, texture_format, luma, chroma, frame_stride, pitch,
                                  color_space, unit_nits, stream=None):
        return int(self.lib.HapB200BlockDecodeYUVPQBatch(blocks, frames, blocks_stride, w, h, texture_format, luma, chroma, frame_stride,
                                                         pitch, color_space, unit_nits, stream))

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
