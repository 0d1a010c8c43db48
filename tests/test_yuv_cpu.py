"""The NV12 / P010 -> RGBA8 conversion of include/hap_b200.h and the argument rules of the YUV encoders, without a GPU.
yuv_util.yuv_to_rgba (the definition restated in numpy integers) is held to the real matrix in float64, to the colour bars
BT.601 and BT.709 publish, to OpenCV's NV12 conversion, and to the C++ pixel-by-pixel conversion the emulated kernel test
uses (tests/emu/yuv_twin.cc)."""
import numpy as np
import pytest

import hap_b200
import yuv_util as Y
from hap_b200.abi import HapCompressorSnappy
from hap_b200.lib import (HapB200Codec_Hap1, HapB200Codec_Hap5, HapB200Codec_Hap7, HapB200Codec_HapA, HapB200Codec_HapM,
                          HapB200Codec_HapY)

BAD_ARGUMENTS, BUFFER_TOO_SMALL, INTERNAL_ERROR = 1, 2, 4
CASES = [(layout, cs) for layout in Y.LAYOUTS for cs in Y.COLOR_SPACES]


@pytest.mark.parametrize("layout,cs", CASES)
def test_integer_conversion_is_within_one_of_the_real_matrix(layout, cs):
    rng = np.random.default_rng(1000 + 10 * layout + cs)
    w, h = 500, 200                                   # 10^5 pixels, every sample value of the layout's range
    luma, chroma = Y.random_planes(rng, w, h, layout)
    got = Y.yuv_to_rgba(luma, chroma, layout, cs)
    want = Y.yuv_to_rgb_float(luma, chroma, layout, cs)
    err = np.abs(got[..., :3].astype(np.float64) - want)
    assert err.max() <= 1.0, err.max()
    assert (got[..., 3] == 255).all()
    # the coefficients' own rounding adds under 0.1 to the 0.5 of rounding the result
    assert err.max() < 0.6, err.max()


def test_coefficients_are_the_rounded_matrix():
    for layout, cs in CASES:
        yoff, ys, csc, coff = Y.scales(layout, cs)
        kr, kb = Y.KRKB[cs]
        kg = 1 - kr - kb
        f = 65536 * 255
        want = [f / ys, f * 2 * (1 - kr) / csc / 8, -f * 2 * kb * (1 - kb) / kg / csc / 8, -f * 2 * kr * (1 - kr) / kg / csc / 8,
                f * 2 * (1 - kb) / csc / 8]
        row = Y.coefficients()[layout * 4 + cs]
        if layout == Y.NV12 and not Y.is_full(cs):      # 4 times the P010 row: P010 of 4 x NV12 samples converts as NV12
            want = [4 * np.floor(v / 4 + 0.5) for v in want]
        assert list(row[:5]) == [int(np.floor(v + 0.5)) for v in want]
        assert list(row[5:]) == [yoff, coff]


# 75 % colour bars (white at 100 %), limited range 8-bit: Y'CbCr as ITU-R BT.801 (BT.601) and SMPTE RP 219 (BT.709) list them
BARS = {
    Y.BT601_LIMITED: {"white": (235, 128, 128, (255, 255, 255)), "black": (16, 128, 128, (0, 0, 0)),
                      "grey75": (180, 128, 128, (191, 191, 191)), "yellow": (162, 44, 142, (191, 191, 0)),
                      "cyan": (131, 156, 44, (0, 191, 191)), "green": (112, 72, 58, (0, 191, 0)),
                      "magenta": (84, 184, 198, (191, 0, 191)), "red": (65, 100, 212, (191, 0, 0)), "blue": (35, 212, 114, (0, 0, 191))},
    Y.BT709_LIMITED: {"white": (235, 128, 128, (255, 255, 255)), "black": (16, 128, 128, (0, 0, 0)),
                      "grey75": (180, 128, 128, (191, 191, 191)), "yellow": (168, 44, 136, (191, 191, 0)),
                      "cyan": (145, 147, 44, (0, 191, 191)), "green": (133, 63, 52, (0, 191, 0)),
                      "magenta": (63, 193, 204, (191, 0, 191)), "red": (51, 109, 212, (191, 0, 0)), "blue": (28, 212, 120, (0, 0, 191))},
}


@pytest.mark.parametrize("layout", Y.LAYOUTS)
@pytest.mark.parametrize("cs", sorted(BARS))
def test_colour_bars(layout, cs):
    for name, (yv, cb, cr, rgb) in BARS[cs].items():
        s = 4 if layout == Y.P010 else 1                 # the 10-bit code of an 8-bit value is 4 times it
        luma = np.full((4, 4), yv * s, np.int64)
        chroma = np.tile(np.array([cb * s, cr * s], np.int64), (2, 2))
        if layout == Y.P010:
            luma, chroma = (luma << 6).astype(np.uint16), (chroma << 6).astype(np.uint16)
        else:
            luma, chroma = luma.astype(np.uint8), chroma.astype(np.uint8)
        got = Y.yuv_to_rgba(luma, chroma, layout, cs)
        assert (np.abs(got[..., :3].astype(int) - np.array(rgb)) <= 1).all(), (name, got[0, 0], rgb)


def test_matches_opencv_nv12_bt601_limited():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(7)
    w, h = 64, 32
    for _ in range(200):
        # chroma constant over the picture, so that OpenCV's upsampling and the bilinear one agree; samples in range
        luma = rng.integers(16, 236, (h, w), dtype=np.int64).astype(np.uint8)
        cb, cr = rng.integers(16, 241, 2)
        chroma = np.tile(np.array([cb, cr], np.uint8), (h // 2, w // 2))
        ocv = cv2.cvtColorTwoPlane(luma, chroma.reshape(h // 2, w // 2, 2), cv2.COLOR_YUV2RGB_NV12)
        got = Y.yuv_to_rgba(luma, chroma, Y.NV12, Y.BT601_LIMITED)
        assert np.abs(got[..., :3].astype(int) - ocv.astype(int)).max() <= 1


@pytest.mark.parametrize("cs", [Y.BT601_LIMITED, Y.BT709_LIMITED])
def test_p010_of_four_times_nv12_gives_the_nv12_picture(cs):
    rng = np.random.default_rng(11 + cs)
    w, h = 96, 64
    luma, chroma = Y.random_planes(rng, w, h, Y.NV12)
    lp = ((luma.astype(np.int64) << 8) | rng.integers(0, 64, luma.shape)).astype(np.uint16)       # 4x in 10 bits, junk below
    cp = ((chroma.astype(np.int64) << 8) | rng.integers(0, 64, chroma.shape)).astype(np.uint16)
    np.testing.assert_array_equal(Y.yuv_to_rgba(lp, cp, Y.P010, cs), Y.yuv_to_rgba(luma, chroma, Y.NV12, cs))


@pytest.mark.parametrize("layout,cs", CASES)
def test_cpp_conversion_equals_the_numpy_definition(layout, cs):
    """tests/emu/yuv_twin.cc, on which the emulated kernel test rests, is the conversion of the header"""
    rng = np.random.default_rng(300 + 10 * layout + cs)
    for w, h, pad in ((4, 4, 0), (12, 8, 16), (36, 20, 48), (132, 12, 0)):
        luma, chroma = Y.random_planes(rng, w, h, layout)
        want = Y.yuv_to_rgba(luma, chroma, layout, cs)
        got = Y.twin_to_rgba(luma, chroma, layout, cs, pitch=w * Y.sample_bytes(layout) + pad)
        np.testing.assert_array_equal(got, want)


# ---- argument rules of the entry points -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def test_yuv_entry_points_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(16 * w * h + 64, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    c = p + 4 * w * h                                      # a 16-byte aligned chroma plane
    used = np.zeros(4, np.uint64)
    u = used.ctypes.data
    cap = lib.max_encoded_length_rgba(w, h, HapB200Codec_HapY, 1)
    ostride = (cap + 15) // 16 * 16
    fb = 4 * w * h
    for layout in Y.LAYOUTS:
        sb = Y.sample_bytes(layout)
        luma, chroma = np.zeros(sb * w * h, np.uint8), np.zeros(sb * w * h // 2, np.uint8)

        def block(lp=p, cp=c, frames=1, fstride=fb, gw=w, gh=h, pitch=sb * w, lay=layout, cs=0, codec=HapB200Codec_HapY, blocks=p,
                  bstride=2048):
            return lib.block_encode_yuv_batch(lp, cp, frames, fstride, gw, gh, pitch, lay, cs, codec, blocks, bstride)

        def batch(lp=p, cp=c, frames=1, fstride=fb, gw=w, gh=h, pitch=sb * w, lay=layout, cs=0, codec=HapB200Codec_HapY,
                  comp=HapCompressorSnappy, chunks=1, out=p, out_stride=ostride, used_p=u):
            return lib.encode_yuv_batch(lp, cp, frames, fstride, gw, gh, pitch, lay, cs, codec, comp, chunks, out, out_stride, used_p)

        def single(lb=luma, cb=chroma, gw=w, gh=h, pitch=None, lay=layout, cs=0, codec=HapB200Codec_HapY, comp=HapCompressorSnappy,
                   chunks=1, cap_=None):
            n = cap_ if cap_ is not None else 1 << 20
            return lib.encode_yuv(lb, cb, gw, gh, lay, cs, codec, comp, chunks, pitch=pitch, out=bytearray(max(n, 1 << 20)),
                                  out_capacity=n)[0]

        for f in (block, batch, single):
            # codecs: Hap Alpha-Only (no alpha to encode), Hap R, unknown; layouts and colour spaces out of range
            for codec in (HapB200Codec_HapA, HapB200Codec_Hap7, 6, 0xFFFFFFFF):
                assert f(codec=codec) == BAD_ARGUMENTS, (f.__name__, codec)
            assert f(lay=2) == BAD_ARGUMENTS and f(lay=0xFFFFFFFF) == BAD_ARGUMENTS
            assert f(cs=4) == BAD_ARGUMENTS and f(cs=0xFFFFFFFF) == BAD_ARGUMENTS
            # geometry: sizes not multiples of 4, empty, pitch below the row, pitch >= 2^32
            for gw, gh, pitch in ((6, 4, 16), (4, 6, 16), (0, 4, 16), (4, 0, 16), (w, h, sb * w - 16), (w, h, 1 << 32)):
                assert f(gw=gw, gh=gh, pitch=pitch) == BAD_ARGUMENTS, (f.__name__, gw, gh, pitch)
        # null planes
        assert block(lp=0) == BAD_ARGUMENTS and block(cp=0) == BAD_ARGUMENTS and block(blocks=0) == BAD_ARGUMENTS
        assert batch(lp=0) == BAD_ARGUMENTS and batch(cp=0) == BAD_ARGUMENTS
        assert single(lb=(0, 16)) == BAD_ARGUMENTS and single(cb=(0, 16)) == BAD_ARGUMENTS
        assert lib.encode_yuv(luma, chroma, w, h, layout, 0, HapB200Codec_HapY, out=(0, cap), out_capacity=cap)[0] == BAD_ARGUMENTS
        # no frames, no output, chunk count 0, unknown compressor
        assert block(frames=0) == BAD_ARGUMENTS and batch(frames=0) == BAD_ARGUMENTS
        assert batch(out=0) == BAD_ARGUMENTS and batch(used_p=0) == BAD_ARGUMENTS
        assert batch(chunks=0) == BAD_ARGUMENTS and batch(comp=0xC1) == BAD_ARGUMENTS
        assert single(chunks=0) == BAD_ARGUMENTS and single(comp=0xC1) == BAD_ARGUMENTS
        # the batch rules: 16-byte aligned planes, pitch, frame stride, blocks and block stride
        for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": sb * w + 8}, {"blocks": p + 8}, {"bstride": 2048 + 8}):
            assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
        for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": sb * w + 8}):
            assert batch(frames=2, **kw) == BAD_ARGUMENTS, kw
        # below the HapB200MaxEncodedLengthRGBA bound
        for codec in (HapB200Codec_Hap1, HapB200Codec_Hap5, HapB200Codec_HapY, HapB200Codec_HapM):
            for k in (1, 3, 8):
                need = lib.max_encoded_length_rgba(w, h, codec, k)
                assert batch(codec=codec, chunks=k, out_stride=need - 1) == BUFFER_TOO_SMALL
                assert single(codec=codec, chunks=k, cap_=need - 1) == BUFFER_TOO_SMALL


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_yuv_valid_arguments_fail_loudly_without_a_gpu(lib):
    w, h = 16, 8
    for layout in Y.LAYOUTS:
        luma, chroma = Y.random_planes(np.random.default_rng(0), w, h, layout)
        assert lib.encode_yuv(luma, chroma, w, h, layout, Y.BT709_LIMITED, HapB200Codec_HapY)[0] == INTERNAL_ERROR
