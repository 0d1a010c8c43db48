"""The RGBA8 -> NV12 / P010 conversion of include/hap_b200.h (HapB200DecodeYUV) and the argument rules of the YUV decoders,
without a GPU.  yuv_out_util.rgba_to_yuv_out (the definition restated in numpy integers) is held to its coefficient rule, to
the real matrix in float64, to neutral greys and nominal black and white, to the colour bars BT.601 and BT.709 publish, to
OpenCV's I420 conversion, to an exact round trip through the YUV encoders' conversion (yuv_util.yuv_to_rgba), and to the C++
sample-by-sample conversion the emulated kernel test uses (tests/emu/yuv_out_twin.cc)."""
import numpy as np
import pytest

import hap_b200
import test_yuv_cpu as T
import yuv_out_util as O
import yuv_util as Y
from golden_util import b64, golden
from hap_b200.lib import HapB200Codec_Hap1, HapB200Codec_Hap7, HapB200Codec_HapA, HapB200Codec_HapM, HapB200Codec_HapY

BAD_ARGUMENTS, INTERNAL_ERROR = 1, 4
CASES = [(layout, cs) for layout in Y.LAYOUTS for cs in Y.COLOR_SPACES]


def test_coefficients_follow_the_rule():
    for layout, cs in CASES:
        assert list(O.coefficients()[layout * 4 + cs]) == O.rule_coefficients(layout, cs), (layout, cs)


@pytest.mark.parametrize("layout,cs", CASES)
def test_integer_conversion_is_within_half_a_code_of_the_real_matrix(layout, cs):
    rng = np.random.default_rng(2000 + 10 * layout + cs)
    rgba = rng.integers(0, 256, (200, 500, 4), dtype=np.uint8)
    luma, chroma = O.samples(rgba, layout, cs)
    fl, fc = O.rgba_to_yuv_out_float(rgba, layout, cs)
    err = max(np.abs(luma - fl).max(), np.abs(chroma - fc).max())
    assert err <= 0.51, err


@pytest.mark.parametrize("layout,cs", CASES)
def test_greys_are_neutral_and_black_and_white_nominal(layout, cs):
    v = np.arange(256, dtype=np.uint8)
    rgba = np.zeros((2, 2 * 256, 4), np.uint8)
    rgba[..., :3] = np.repeat(v, 2)[None, :, None]                   # each grey over a 2 x 2 quad: one chroma sample of its own
    luma, chroma = O.samples(rgba, layout, cs)
    yoff, ys, _, coff = Y.scales(layout, cs)
    assert (chroma == coff).all()
    assert luma[0, 0] == yoff and luma[0, -1] == yoff + ys
    assert (np.diff(luma[0, ::2]) >= 0).all()
    if not Y.is_full(cs):
        assert (luma[0, 0], luma[0, -1]) == ((16, 235) if layout == Y.NV12 else (64, 940))


@pytest.mark.parametrize("cs", sorted(T.BARS))
def test_colour_bars(cs):
    off = 0
    for name, (yv, cb, cr, rgb) in T.BARS[cs].items():
        rgba = np.zeros((2, 2, 4), np.uint8)
        rgba[..., :3] = rgb
        luma, chroma = O.samples(rgba, Y.NV12, cs)
        got = (int(luma[0, 0]), int(chroma[0, 0]), int(chroma[0, 1]))
        assert all(abs(g - w) <= 1 for g, w in zip(got, (yv, cb, cr))), (name, got)
        off += got != (yv, cb, cr)
    assert off <= 1                                                    # BT.601 yellow: Y 161 for the published 162


def test_luma_matches_opencv_i420():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(17)
    h, w = 64, 96
    for _ in range(50):
        rgb = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ocv = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
        rgba = np.concatenate([rgb, np.full((h, w, 1), 255, np.uint8)], -1)
        luma, _ = O.samples(rgba, Y.NV12, Y.BT601_LIMITED)
        assert np.abs(luma - ocv[:h].astype(int)).max() <= 1


def test_chroma_matches_opencv_i420_where_the_decimations_agree():
    """pictures constant across columns and within each row pair: every chroma filter gives the row pair's colour"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(18)
    h, w = 64, 96
    for _ in range(50):
        rows = rng.integers(0, 256, (h // 2, 1, 3), dtype=np.uint8)
        rgb = np.ascontiguousarray(np.repeat(np.repeat(rows, 2, axis=0), w, axis=1))
        ocv = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
        u = ocv[h: h + h // 4].reshape(h // 2, w // 2).astype(int)
        v = ocv[h + h // 4:].reshape(h // 2, w // 2).astype(int)
        rgba = np.concatenate([rgb, np.full((h, w, 1), 255, np.uint8)], -1)
        _, chroma = O.samples(rgba, Y.NV12, Y.BT601_LIMITED)
        assert np.abs(chroma[:, 0::2] - u).max() <= 1 and np.abs(chroma[:, 1::2] - v).max() <= 1


@pytest.mark.parametrize("layout,cs", CASES)
def test_flat_colours_return_through_the_encoders_conversion(layout, cs):
    """all 2^24 flat colours -> Y'CbCr here -> RGBA by yuv_util.yuv_to_rgba: P010 exactly, NV12 within 2 (limited) or 1 (full)"""
    k = O.coefficients()[layout * 4 + cs]
    top = (1 << Y.bits(layout)) - 1
    worst = 0
    n = 1 << 20
    for start in range(0, 1 << 24, n):
        c = np.arange(start, start + n, dtype=np.int64)
        r, g, b = c & 255, (c >> 8) & 255, c >> 16
        yv = np.clip(((k[0] * r + k[1] * g + k[2] * b + 32768) >> 16) + k[9], 0, top)   # a flat colour's filtered sums are 8 x it
        cb = np.clip(((k[3] * 8 * r + k[4] * 8 * g + k[5] * 8 * b + (1 << 18)) >> 19) + k[10], 0, top)
        cr = np.clip(((k[6] * 8 * r + k[7] * 8 * g + k[8] * 8 * b + (1 << 18)) >> 19) + k[10], 0, top)
        # a 2 x 2n picture whose even columns hold the colours: there the upsampler reads only their own chroma sample
        luma = np.repeat(yv, 2)[None].repeat(2, 0)
        chroma = np.stack([cb, cr], -1).reshape(1, 2 * n)
        back = Y.yuv_to_rgba(O.store(luma, layout), O.store(chroma, layout), layout, cs)[0, 0::2, :3].astype(np.int64)
        worst = max(worst, int(np.abs(back - np.stack([r, g, b], -1)).max()))
    assert worst <= (0 if layout == Y.P010 else 1 if Y.is_full(cs) else 2), worst


@pytest.mark.parametrize("layout,cs", CASES)
def test_cpp_conversion_equals_the_numpy_definition(layout, cs):
    """tests/emu/yuv_out_twin.cc, on which the emulated kernel test rests, is the conversion of the header"""
    rng = np.random.default_rng(400 + 10 * layout + cs)
    for w, h, pad in ((4, 4, 0), (12, 8, 16), (36, 20, 48), (132, 12, 0), (124, 8, 32), (260, 4, 16)):
        rgba = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        want = O.rgba_to_yuv_out(rgba, layout, cs)
        got = O.twin_to_yuv(rgba, layout, cs, pitch=w * Y.sample_bytes(layout) + pad)
        np.testing.assert_array_equal(got[0], want[0])
        np.testing.assert_array_equal(got[1], want[1])


# ---- argument rules of the entry points -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def a_frame():
    """a Hap frame the reference wrote (DXT1, 4096 blocks: 256 x 256)"""
    return b64(golden()["ref_frames"]["dxt1"]["frame_b64"])


def test_yuv_decoders_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(16 * w * h + 64, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    c = p + 4 * w * h                                      # a 16-byte aligned chroma plane
    res = np.zeros(4, np.uint32)
    nb = np.full(4, 64, np.uint64)
    frame = a_frame()
    fb = 4 * w * h
    for layout in Y.LAYOUTS:
        sb = Y.sample_bytes(layout)

        def block(blocks=p, frames=1, bstride=2048, gw=w, gh=h, codec=HapB200Codec_HapY, lp=p, cp=c, fstride=fb, pitch=sb * w, lay=layout,
                  cs=0):
            return lib.block_decode_yuv_batch(blocks, frames, bstride, gw, gh, codec, lp, cp, fstride, pitch, lay, cs)

        def batch(src=p, frames=1, istride=2048, in_bytes=nb.ctypes.data, chunks=4, codec=HapB200Codec_HapY, gw=w, gh=h, lp=p, cp=c,
                  fstride=fb, pitch=sb * w, lay=layout, cs=0, results=res.ctypes.data):
            return lib.decode_yuv_batch(src, frames, istride, in_bytes, chunks, codec, gw, gh, lp, cp, fstride, pitch, lay, cs, results)

        def single(fr=frame, gw=256, gh=256, pitch=None, lay=layout, cs=0, lp=None, cp=None):
            pitch = pitch if pitch is not None else sb * gw
            lp = lp if lp is not None else bytearray(64)              # (every call here is refused before the planes are touched)
            cp = cp if cp is not None else bytearray(64)
            return lib.decode_yuv(fr, gw, gh, lay, cs, pitch=pitch, luma=lp, chroma=cp)[0]

        for f in (block, batch, single):
            # layouts and colour spaces out of range; BT.2020
            assert f(lay=2) == BAD_ARGUMENTS and f(lay=0xFFFFFFFF) == BAD_ARGUMENTS, f.__name__
            for cs in (Y.BT709_FULL + 1, Y.BT709_FULL + 2, 6, 0xFFFFFFFF):
                assert f(cs=cs) == BAD_ARGUMENTS, (f.__name__, cs)
            # geometry: sizes not multiples of 4, empty, pitch below the row, pitch >= 2^32
            for gw, gh, pitch in ((6, 4, 16), (4, 6, 16), (0, 4, 16), (4, 0, 16), (64, 32, sb * 64 - 16), (64, 32, 1 << 32)):
                assert f(gw=gw, gh=gh, pitch=pitch) == BAD_ARGUMENTS, (f.__name__, gw, gh, pitch)
        # unknown codecs (every HapB200Codec is taken)
        for codec in (6, 0xFFFFFFFF):
            assert block(codec=codec) == BAD_ARGUMENTS and batch(codec=codec) == BAD_ARGUMENTS
        # null pointers, no frames, no chunks
        assert block(blocks=0) == BAD_ARGUMENTS and block(lp=0) == BAD_ARGUMENTS and block(cp=0) == BAD_ARGUMENTS
        assert batch(src=0) == BAD_ARGUMENTS and batch(in_bytes=0) == BAD_ARGUMENTS and batch(results=0) == BAD_ARGUMENTS
        assert batch(lp=0) == BAD_ARGUMENTS and batch(cp=0) == BAD_ARGUMENTS
        assert single(lp=(0, 16)) == BAD_ARGUMENTS and single(cp=(0, 16)) == BAD_ARGUMENTS and single(fr=(0, 16)) == BAD_ARGUMENTS
        assert block(frames=0) == BAD_ARGUMENTS and batch(frames=0) == BAD_ARGUMENTS and batch(chunks=0) == BAD_ARGUMENTS
        # the batch rules: 16-byte aligned planes, pitch, frame stride, blocks and block stride
        for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": sb * w + 8}, {"blocks": p + 8}, {"bstride": 2048 + 8}):
            assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
        for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": sb * w + 8}):
            assert batch(frames=2, **kw) == BAD_ARGUMENTS, kw


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_yuv_decoders_fail_loudly_without_a_gpu(lib):
    w, h = 256, 256
    frame = a_frame()
    for layout in Y.LAYOUTS:
        assert lib.decode_yuv(frame, w, h, layout, Y.BT709_LIMITED)[0] == INTERNAL_ERROR
        sb = Y.sample_bytes(layout)
        buf = np.zeros(4 * sb * w * h + 64, np.uint8)
        p = (buf.ctypes.data + 15) // 16 * 16
        res = np.zeros(1, np.uint32)
        nb = np.array([len(frame)], np.uint64)
        for codec in (HapB200Codec_Hap1, HapB200Codec_HapM, HapB200Codec_HapA, HapB200Codec_Hap7):
            assert lib.block_decode_yuv_batch(p, 1, 16, 8, 8, codec, p, p + 1024, 0, 16 * sb, layout, Y.BT601_FULL) == INTERNAL_ERROR
            assert lib.decode_yuv_batch(p, 1, 4096, nb.ctypes.data, 4, codec, 8, 8, p, p + 1024, 0, 16 * sb, layout, Y.BT601_FULL,
                                        res.ctypes.data) == INTERNAL_ERROR
