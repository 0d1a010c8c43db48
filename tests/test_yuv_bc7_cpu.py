"""The argument rules of the Hap R (BC7) encoders from NV12 / P010 and planar Y'CbCr pictures (HapB200EncodeYUVBC7*,
HapB200EncodePlanarBC7*), without a GPU: every refusal comes before anything touches the GPU, and valid arguments fail
loudly (HapResult_Internal_Error) where there is no CUDA device."""
import numpy as np
import pytest

import hap_b200
import planar_util as P
import yuv_util as Y
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy
from hap_b200.lib import HapB200Codec_Hap7

BAD_ARGUMENTS, BUFFER_TOO_SMALL, INTERNAL_ERROR = 1, 2, 4
W, H = 64, 32


@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def arena():
    """a 16-byte aligned host arena that holds every plane of two frames: its base, and the buffer that keeps it alive"""
    buf = np.zeros(64 * W * H + 64, np.uint8)
    return (buf.ctypes.data + 15) // 16 * 16, buf


@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_yuv_bc7_entry_points_refuse_bad_arguments(lib, layout):
    sb = Y.sample_bytes(layout)
    base, keep = arena()
    lum, chr_ = base, base + sb * W * H
    fb = 2 * sb * W * H
    used = np.zeros(4, np.uint64)
    cap = lib.max_encoded_length_rgba(W, H, HapB200Codec_Hap7, 1)
    ostride = (cap + 15) // 16 * 16
    luma, chroma = np.zeros(sb * W * H, np.uint8), np.zeros(sb * W * H // 2, np.uint8)

    def block(l=lum, c=chr_, frames=1, fstride=fb, gw=W, gh=H, pitch=sb * W, lay=layout, cs=0, blocks=base, bstride=4096):
        return lib.block_encode_yuv_bc7_batch(l, c, frames, fstride, gw, gh, pitch, lay, cs, blocks, bstride)

    def batch(l=lum, c=chr_, frames=1, fstride=fb, gw=W, gh=H, pitch=sb * W, lay=layout, cs=0, comp=HapCompressorSnappy, chunks=1,
              out=base, out_stride=ostride, used_p=used.ctypes.data):
        return lib.encode_yuv_bc7_batch(l, c, frames, fstride, gw, gh, pitch, lay, cs, comp, chunks, out, out_stride, used_p)

    def single(l=luma, c=chroma, gw=W, gh=H, pitch=sb * W, lay=layout, cs=0, comp=HapCompressorSnappy, chunks=1, cap_=None):
        k = cap_ if cap_ is not None else 1 << 20
        return lib.encode_yuv_bc7(l, c, gw, gh, lay, cs, comp, chunks, pitch=pitch, out=bytearray(max(k, 1 << 20)), out_capacity=k)[0]

    for f in (block, batch, single):
        # layouts and colour spaces out of range (BT.2020 among them)
        for lay in (2, 3, 0xFFFFFFFF):
            assert f(lay=lay) == BAD_ARGUMENTS, (f.__name__, lay)
        for cs in (4, 5, 6, 0xFFFFFFFF):
            assert f(cs=cs) == BAD_ARGUMENTS, (f.__name__, cs)
        # geometry: sizes not multiples of 4, empty, the pitch below the row or at 2^32
        for gw, gh in ((6, 4), (4, 6), (0, 4), (4, 0), (W + 2, H), (W, H + 2)):
            assert f(gw=gw, gh=gh) == BAD_ARGUMENTS, (f.__name__, gw, gh)
        for pitch in (sb * W - 16, sb * W - 1, 1 << 32):
            assert f(pitch=pitch) == BAD_ARGUMENTS, (f.__name__, pitch)
        # the RGBA8 picture's row, 4 * width bytes, must fit HAPB200_MAX_ROW_BYTES although the luma row does
        assert f(gw=1 << 30, gh=4, pitch=sb << 30) == BAD_ARGUMENTS, f.__name__
    # null planes
    assert block(l=0) == BAD_ARGUMENTS and block(c=0) == BAD_ARGUMENTS and block(blocks=0) == BAD_ARGUMENTS
    assert batch(l=0) == BAD_ARGUMENTS and batch(c=0) == BAD_ARGUMENTS
    assert lib.encode_yuv_bc7((0, 0), chroma, W, H, layout, 0)[0] == BAD_ARGUMENTS
    assert lib.encode_yuv_bc7(luma, (0, 0), W, H, layout, 0)[0] == BAD_ARGUMENTS
    assert lib.encode_yuv_bc7(luma, chroma, W, H, layout, 0, out=(0, cap), out_capacity=cap)[0] == BAD_ARGUMENTS
    # no frames, no output, chunk count 0, unknown compressor
    assert block(frames=0) == BAD_ARGUMENTS and batch(frames=0) == BAD_ARGUMENTS
    assert batch(out=0) == BAD_ARGUMENTS and batch(used_p=0) == BAD_ARGUMENTS
    assert batch(chunks=0) == BAD_ARGUMENTS and batch(comp=0xC1) == BAD_ARGUMENTS
    assert single(chunks=0) == BAD_ARGUMENTS and single(comp=0xC1) == BAD_ARGUMENTS
    # the batch rules: 16-byte aligned planes, pitch, frame stride, blocks and block stride
    for kw in ({"l": lum + 8}, {"c": chr_ + 8}, {"fstride": fb + 8}, {"pitch": sb * W + 8}, {"blocks": base + 8}, {"bstride": 4096 + 8}):
        assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
    for kw in ({"l": lum + 8}, {"c": chr_ + 8}, {"fstride": fb + 8}, {"pitch": sb * W + 8}):
        assert batch(frames=2, **kw) == BAD_ARGUMENTS, kw
    # below the HapB200MaxEncodedLengthRGBA bound of Hap7
    for k in (1, 3, 8):
        need = lib.max_encoded_length_rgba(W, H, HapB200Codec_Hap7, k)
        assert batch(chunks=k, out_stride=(need - 1) // 16 * 16) == BUFFER_TOO_SMALL, k
        assert single(chunks=k, cap_=need - 1) == BUFFER_TOO_SMALL, k
    del keep


@pytest.mark.parametrize("n", P.DEPTHS)
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_planar_bc7_entry_points_refuse_bad_arguments(lib, sub, n):
    sb = P.sample_bytes(n)
    ch, cw = P.chroma_shape(W, H, sub)
    lp, cp = sb * W, sb * cw
    base, keep = arena()
    fb = 4 * sb * W * H
    lum, cbp, crp, alp = base, base + sb * W * H, base + 2 * sb * W * H, base + 3 * sb * W * H
    used = np.zeros(4, np.uint64)
    cap = lib.max_encoded_length_rgba(W, H, HapB200Codec_Hap7, 1)
    ostride = (cap + 15) // 16 * 16
    luma, cb, cr, alpha = (np.zeros(sb * W * H, np.uint8), np.zeros(sb * cw * ch, np.uint8), np.zeros(sb * cw * ch, np.uint8),
                           np.zeros(sb * W * H, np.uint8))

    def block(l=lum, b=cbp, r=crp, a=alp, frames=1, fstride=fb, gw=W, gh=H, lpitch=lp, cpitch=cp, s=sub, d=n, cs=0, blocks=base,
              bstride=4096):
        return lib.block_encode_planar_bc7_batch(l, b, r, a, frames, fstride, gw, gh, lpitch, cpitch, s, d, cs, blocks, bstride)

    def batch(l=lum, b=cbp, r=crp, a=alp, frames=1, fstride=fb, gw=W, gh=H, lpitch=lp, cpitch=cp, s=sub, d=n, cs=0,
              comp=HapCompressorSnappy, chunks=1, out=base, out_stride=ostride, used_p=used.ctypes.data):
        return lib.encode_planar_bc7_batch(l, b, r, a, frames, fstride, gw, gh, lpitch, cpitch, s, d, cs, comp, chunks, out, out_stride,
                                           used_p)

    def single(l=luma, b=cb, r=cr, a=alpha, gw=W, gh=H, lpitch=lp, cpitch=cp, s=sub, d=n, cs=0, comp=HapCompressorSnappy, chunks=1,
               cap_=None):
        k = cap_ if cap_ is not None else 1 << 20
        return lib.encode_planar_bc7(l, b, r, a, gw, gh, s, d, cs, comp, chunks, luma_pitch=lpitch, chroma_pitch=cpitch,
                                     out=bytearray(max(k, 1 << 20)), out_capacity=k)[0]

    for f in (block, batch, single):
        # depths, subsamplings and colour spaces out of range (BT.2020 among them)
        for d in (0, 1, 9, 11, 14, 16, 0xFFFFFFFF):
            assert f(d=d) == BAD_ARGUMENTS, (f.__name__, d)
        assert f(s=3) == BAD_ARGUMENTS and f(s=0xFFFFFFFF) == BAD_ARGUMENTS
        for cs in (4, 5, 6, 0xFFFFFFFF):
            assert f(cs=cs) == BAD_ARGUMENTS, (f.__name__, cs)
        # geometry: sizes not multiples of 4, empty, each pitch below its row or at 2^32
        for gw, gh in ((6, 4), (4, 6), (0, 4), (4, 0), (W + 2, H), (W, H + 2)):
            assert f(gw=gw, gh=gh) == BAD_ARGUMENTS, (f.__name__, gw, gh)
        for kw in ({"lpitch": lp - 16}, {"lpitch": lp - 1}, {"lpitch": 1 << 32}, {"cpitch": cp - 16}, {"cpitch": cp - 1},
                   {"cpitch": 1 << 32}):
            assert f(**kw) == BAD_ARGUMENTS, (f.__name__, kw)
        # the RGBA8 picture's row, 4 * width bytes, must fit HAPB200_MAX_ROW_BYTES although the luma and chroma rows do
        wide_cw = (1 << 30) if sub == P.S444 else (1 << 29)
        assert f(gw=1 << 30, gh=4, lpitch=sb << 30, cpitch=sb * wide_cw) == BAD_ARGUMENTS, f.__name__
    # null planes: luma, Cb and Cr are always read (there is no alpha-only form); alpha may be NULL
    for kw in ({"l": 0}, {"b": 0}, {"r": 0}):
        assert block(**kw) == BAD_ARGUMENTS and batch(**kw) == BAD_ARGUMENTS, kw
    for kw in ({"l": None}, {"b": None}, {"r": None}):
        assert single(**kw) == BAD_ARGUMENTS, kw
        assert single(a=None, **kw) == BAD_ARGUMENTS, kw
    assert block(blocks=0) == BAD_ARGUMENTS
    assert lib.encode_planar_bc7(luma, cb, cr, alpha, W, H, sub, n, 0, out=(0, cap), out_capacity=cap)[0] == BAD_ARGUMENTS
    # no frames, no output, chunk count 0, unknown compressor
    assert block(frames=0) == BAD_ARGUMENTS and batch(frames=0) == BAD_ARGUMENTS
    assert batch(out=0) == BAD_ARGUMENTS and batch(used_p=0) == BAD_ARGUMENTS
    assert batch(chunks=0) == BAD_ARGUMENTS and batch(comp=0xC1) == BAD_ARGUMENTS
    assert single(chunks=0) == BAD_ARGUMENTS and single(comp=0xC1) == BAD_ARGUMENTS
    # the batch rules: 16-byte aligned planes, pitches, frame stride, blocks and block stride
    for kw in ({"l": lum + 8}, {"b": cbp + 8}, {"r": crp + 8}, {"a": alp + 8}, {"fstride": fb + 8}, {"lpitch": lp + 8},
               {"cpitch": cp + 8}, {"blocks": base + 8}, {"bstride": 4096 + 8}):
        assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
    for kw in ({"l": lum + 8}, {"b": cbp + 8}, {"r": crp + 8}, {"a": alp + 8}, {"fstride": fb + 8}, {"lpitch": lp + 8},
               {"cpitch": cp + 8}):
        assert batch(frames=2, **kw) == BAD_ARGUMENTS, kw
    # below the HapB200MaxEncodedLengthRGBA bound of Hap7
    for k in (1, 3, 8):
        need = lib.max_encoded_length_rgba(W, H, HapB200Codec_Hap7, k)
        assert batch(chunks=k, out_stride=(need - 1) // 16 * 16) == BUFFER_TOO_SMALL, k
        assert single(chunks=k, cap_=need - 1) == BUFFER_TOO_SMALL, k
    del keep


def test_codec_taking_yuv_and_planar_encoders_still_refuse_hap7(lib):
    base, keep = arena()
    assert lib.block_encode_yuv_batch(base, base, 1, 4096, 16, 8, 16, Y.NV12, 0, HapB200Codec_Hap7, base, 4096) == BAD_ARGUMENTS
    assert lib.block_encode_planar_batch(base, base, base, 0, 1, 4096, 16, 8, 16, 16, P.S444, 8, 0, HapB200Codec_Hap7, base,
                                         4096) == BAD_ARGUMENTS
    del keep


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_yuv_and_planar_bc7_valid_arguments_fail_loudly_without_a_gpu(lib):
    w, h = 16, 8
    rng = np.random.default_rng(0)
    for layout in Y.LAYOUTS:
        luma, chroma = Y.random_planes(rng, w, h, layout)
        for cs in Y.COLOR_SPACES:
            for comp in (HapCompressorNone, HapCompressorSnappy):
                assert lib.encode_yuv_bc7(luma, chroma, w, h, layout, cs, comp, 3)[0] == INTERNAL_ERROR, (layout, cs, comp)
    for sub in P.SUBSAMPLINGS:
        for n in P.DEPTHS:
            for with_alpha in (True, False):
                planes = P.random_planes(rng, w, h, sub, n, alpha=with_alpha)
                assert lib.encode_planar_bc7(*planes, w, h, sub, n, Y.BT709_LIMITED)[0] == INTERNAL_ERROR, (sub, n, with_alpha)
    # a picture whose RGBA8 row is exactly HAPB200_MAX_ROW_BYTES - 3 bytes passes the width rule (nothing is read without a GPU)
    base, keep = arena()
    used = np.zeros(1, np.uint64)
    wide = (1 << 30) - 4
    assert lib.block_encode_yuv_bc7_batch(base, base, 1, 1 << 34, wide, 4, 2 * (1 << 30), Y.P010, 0, base, 1 << 34) == INTERNAL_ERROR
    assert lib.encode_planar_bc7_batch(base, base, base, 0, 1, 1 << 34, wide, 4, 1 << 30, 1 << 30, P.S444, 8, 0, HapCompressorNone,
                                       1, base, 1 << 36, used.ctypes.data) == INTERNAL_ERROR
    del keep
