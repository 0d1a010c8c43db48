"""The RGBA8 -> planar Y'CbCr (+ alpha) conversion of include/hap_b200.h (HapB200DecodePlanar) and the argument rules of the
planar decoders, without a GPU.  planar_out_util.rgba_to_planar_out (the definition restated in numpy integers) is held to the
rule of its rows, to the real matrix in float64, to neutral greys and nominal black and white, to the NV12 / P010 decoders'
conversion at 4:2:0, to exact round trips through the planar encoders' conversion (planar_util.planar_to_rgba), to OpenCV's
YCrCb conversion, and to the C++ sample-by-sample conversion the emulated kernel test uses (tests/emu/planar_out_twin.cc)."""
import numpy as np
import pytest

import hap_b200
import planar_out_util as Q
import planar_util as P
import yuv_out_util as O
import yuv_util as Y
from golden_util import b64, golden
from hap_b200.lib import HapB200Codec_Hap1, HapB200Codec_Hap7, HapB200Codec_HapA, HapB200Codec_HapM, HapB200Codec_HapY

BAD_ARGUMENTS, INTERNAL_ERROR = 1, 4
ROWS = [(n, cs) for n in Q.DEPTHS for cs in Q.COLOR_SPACES]
CASES = [(sub, n, cs) for sub in Q.SUBSAMPLINGS for n in Q.DEPTHS for cs in Q.COLOR_SPACES]


@pytest.mark.parametrize("n,cs", ROWS)
def test_rows_follow_the_rule(n, cs):
    assert Q.row(n, cs) == Q.rule_row(n, cs)
    if n < 12:   # the 8- and 10-bit rows are the NV12 and P010 ones
        assert Q.rule_row(n, cs) == O.rule_coefficients(Y.P010 if n == 10 else Y.NV12, cs)


def test_largest_intermediate_fits_int32():
    worst = 0
    for n, cs in ROWS:
        k = np.abs(np.array(Q.row(n, cs), np.int64))
        worst = max(worst, int(k[:3].sum()) * 255 + 32768, int(max(k[3:6].sum(), k[6:9].sum())) * 8 * 255 + (1 << 18))
    assert worst < 2 ** 31, worst


@pytest.mark.parametrize("sub,n,cs", CASES)
def test_integer_conversion_is_within_half_a_code_of_the_real_matrix(sub, n, cs):
    rng = np.random.default_rng(3000 + 100 * sub + 10 * n + cs)
    rgba = rng.integers(0, 256, (64, 200, 4), dtype=np.uint8)
    luma, cb, cr, _ = Q.samples(rgba, sub, n, cs)
    fl, fcb, fcr = Q.rgba_to_planar_out_float(rgba, sub, n, cs)
    err = max(np.abs(luma - fl).max(), np.abs(cb - fcb).max(), np.abs(cr - fcr).max())
    assert err <= 0.51, err


@pytest.mark.parametrize("n,cs", ROWS)
def test_greys_are_neutral_and_black_and_white_nominal(n, cs):
    v = np.arange(256, dtype=np.uint8)
    rgba = np.zeros((2, 4 * 256, 4), np.uint8)
    rgba[..., :3] = np.repeat(v, 4)[None, :, None]                 # each grey over 4 columns: every filter sees it alone
    yoff, ys, _, coff = P.scales(n, cs)
    for sub in Q.SUBSAMPLINGS:
        luma, cb, cr, _ = Q.samples(rgba, sub, n, cs)
        assert (cb == coff).all() and (cr == coff).all(), sub
        assert luma[0, 0] == yoff and luma[0, -1] == yoff + ys
        assert (np.diff(luma[0, ::4]) >= 0).all()
    if n == 12 and not Y.is_full(cs):
        assert (yoff, yoff + ys) == (256, 3760)


@pytest.mark.parametrize("n", (8, 10))
@pytest.mark.parametrize("cs", Q.COLOR_SPACES)
def test_420_is_the_nv12_and_p010_conversion(n, cs):
    rng = np.random.default_rng(50 + n + cs)
    rgba = rng.integers(0, 256, (36, 132, 4), dtype=np.uint8)
    layout = Y.P010 if n == 10 else Y.NV12
    luma, chroma = O.rgba_to_yuv_out(rgba, layout, cs)
    shift = 6 if n == 10 else 0
    got = Q.rgba_to_planar_out(rgba, Q.S420, n, cs, alpha=False)
    np.testing.assert_array_equal(got[0], luma >> shift)
    np.testing.assert_array_equal(got[1], chroma[:, 0::2] >> shift)
    np.testing.assert_array_equal(got[2], chroma[:, 1::2] >> shift)
    assert got[3] is None


@pytest.mark.parametrize("n", (10, 12))
@pytest.mark.parametrize("cs", Q.COLOR_SPACES)
def test_flat_colours_return_exactly_through_the_encoders_conversion(n, cs):
    """all 2^24 colours, each a 4:4:4 pixel (a flat colour: every filter sees it alone) -> Y'CbCr here -> RGBA by
    planar_util.planar_to_rgba"""
    step = 1 << 21
    for start in range(0, 1 << 24, step):
        c = np.arange(start, start + step, dtype=np.int64)
        rgba = np.stack([c & 255, (c >> 8) & 255, c >> 16, np.full_like(c, 255)], -1).astype(np.uint8)[None]
        luma, cb, cr, _ = Q.rgba_to_planar_out(rgba, Q.S444, n, cs, alpha=False)
        back = P.planar_to_rgba(luma, cb, cr, None, Q.S444, n, cs)
        np.testing.assert_array_equal(back, rgba)


@pytest.mark.parametrize("n", (10, 12))
@pytest.mark.parametrize("cs", Q.COLOR_SPACES)
def test_444_with_alpha_returns_any_picture_exactly(n, cs):
    """yuva444p10le / yuva444p12le are lossless against the RGBA8 decoders"""
    rng = np.random.default_rng(70 + n + cs)
    rgba = rng.integers(0, 256, (48, 96, 4), dtype=np.uint8)
    planes = Q.rgba_to_planar_out(rgba, Q.S444, n, cs)
    np.testing.assert_array_equal(P.planar_to_rgba(*planes, Q.S444, n, cs), rgba)


@pytest.mark.parametrize("n", Q.DEPTHS)
def test_alpha_is_inverted_exactly_by_the_encoders_alpha_rule(n):
    a = np.arange(256)
    out = Q.alpha_out(a, n)
    assert out[0] == 0 and out[255] == (1 << n) - 1 and (np.diff(out) > 0).all()
    np.testing.assert_array_equal(P.alpha8(out, n), a)
    # rounded to nearest, and no tie: 2 (2^n - 1) A + 255 is never a multiple of 510 plus 255 away from one
    exact = a * ((1 << n) - 1) / 255.0
    assert np.abs(out - exact).max() <= 0.5 and (np.abs(out - exact) != 0.5).all()


def test_bt601_full_444_matches_opencv_ycrcb():
    """an independent implementation of the full-range BT.601 matrix (JPEG's), at 8 bits and 4:4:4"""
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(19)
    for _ in range(20):
        rgb = rng.integers(0, 256, (64, 96, 3), dtype=np.uint8)
        ocv = cv2.cvtColor(rgb, cv2.COLOR_RGB2YCrCb).astype(int)
        rgba = np.concatenate([rgb, np.full((64, 96, 1), 255, np.uint8)], -1)
        luma, cb, cr, _ = Q.samples(rgba, Q.S444, 8, Y.BT601_FULL, alpha=False)
        assert np.abs(luma - ocv[..., 0]).max() <= 1
        assert np.abs(cr - ocv[..., 1]).max() <= 1 and np.abs(cb - ocv[..., 2]).max() <= 1


@pytest.mark.parametrize("sub,n,cs", CASES)
def test_cpp_conversion_equals_the_numpy_definition(sub, n, cs):
    """tests/emu/planar_out_twin.cc, on which the emulated kernel test rests, is the conversion of the header"""
    rng = np.random.default_rng(500 + 100 * sub + 10 * n + cs)
    for w, h, lpad, cpad, alpha in ((4, 4, 0, 0, True), (12, 8, 16, 0, False), (36, 20, 48, 32, True), (132, 12, 0, 16, True)):
        rgba = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        want = Q.rgba_to_planar_out(rgba, sub, n, cs, alpha)
        got = Q.twin_to_planar(rgba, sub, n, cs, alpha, luma_pad=lpad, chroma_pad=cpad)
        for g, wnt in zip(got, want):
            if wnt is None:
                assert g is None
            else:
                np.testing.assert_array_equal(g, wnt)


# ---- argument rules of the entry points -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def ref_frame(kind="dxt1"):
    """a 256 x 256 Hap frame the reference wrote"""
    return b64(golden()["ref_frames"][kind]["frame_b64"])


def test_planar_decoders_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(64 * w * h + 64, np.uint8)
    base = (buf.ctypes.data + 15) // 16 * 16
    res = np.zeros(4, np.uint32)
    nb = np.full(4, 64, np.uint64)
    fb = 8 * w * h
    lu, cbp, crp, al = base, base + fb * 2, base + fb * 4, base + fb * 6   # 16-byte aligned planes, two frames of room each
    frame = ref_frame()
    for sub in Q.SUBSAMPLINGS:
        for n in Q.DEPTHS:
            sb = P.sample_bytes(n)
            cw = w if sub == Q.S444 else w // 2

            def block(blocks=base, frames=1, bstride=2048, gw=w, gh=h, codec=HapB200Codec_HapY, l=lu, b=cbp, r=crp, a=al, fstride=fb,
                      lp=sb * w, cp=sb * cw, s=sub, d=n, cs=0):
                return lib.block_decode_planar_batch(blocks, frames, bstride, gw, gh, codec, l, b, r, a, fstride, lp, cp, s, d, cs)

            def batch(src=base, frames=1, istride=2048, in_bytes=nb.ctypes.data, chunks=4, codec=HapB200Codec_HapY, gw=w, gh=h, l=lu,
                      b=cbp, r=crp, a=al, fstride=fb, lp=sb * w, cp=sb * cw, s=sub, d=n, cs=0, results=res.ctypes.data):
                return lib.decode_planar_batch(src, frames, istride, in_bytes, chunks, codec, gw, gh, l, b, r, a, fstride, lp, cp, s, d, cs,
                                               results)

            def single(fr=frame, gw=256, gh=256, lp=None, cp=None, s=sub, d=n, cs=0, l=True, b=True, r=True, a=True):
                # (every call here is refused before the planes are touched)
                room = lambda on: bytearray(64) if on is True else on
                lp = lp if lp is not None else sb * gw
                cp = cp if cp is not None else sb * (gw if s == Q.S444 else gw // 2)
                return lib.decode_planar(fr, gw, gh, s, d, cs, luma=room(l), cb=room(b), cr=room(r), alpha=room(a), luma_pitch=lp,
                                         chroma_pitch=cp)[0]

            for f in (block, batch, single):
                # subsamplings, depths and colour spaces out of range; BT.2020
                for kw in ({"s": 3}, {"s": 0xFFFFFFFF}, {"d": 0}, {"d": 9}, {"d": 11}, {"d": 16}, {"cs": 4}, {"cs": 5}, {"cs": 6},
                           {"cs": 0xFFFFFFFF}):
                    assert f(**kw) == BAD_ARGUMENTS, (f.__name__, kw)
                # geometry: sizes not multiples of 4, empty, pitches below their rows or at 2^32
                for gw, gh in ((6, 4), (4, 6), (0, 4), (4, 0)):
                    assert f(gw=gw, gh=gh, lp=16 * sb, cp=16 * sb) == BAD_ARGUMENTS, (f.__name__, gw, gh)
                gw = 256 if f is single else w
                gcw = gw if sub == Q.S444 else gw // 2
                for lp, cp in ((sb * gw - 16, sb * gcw), (1 << 32, sb * gcw), (sb * gw, sb * gcw - 16), (sb * gw, 1 << 32)):
                    assert f(lp=lp, cp=cp) == BAD_ARGUMENTS, (f.__name__, lp, cp)
            # unknown codecs (every HapB200Codec is taken)
            for codec in (6, 0xFFFFFFFF):
                assert block(codec=codec) == BAD_ARGUMENTS and batch(codec=codec) == BAD_ARGUMENTS
            # null pointers, no frames, no chunks; Hap Alpha-Only needs the alpha plane, the others luma, Cb and Cr
            for kw in ({"l": 0}, {"b": 0}, {"r": 0}, {"codec": HapB200Codec_HapA, "a": 0}):
                assert block(**kw) == BAD_ARGUMENTS and batch(**kw) == BAD_ARGUMENTS, kw
            assert block(blocks=0) == BAD_ARGUMENTS and block(frames=0) == BAD_ARGUMENTS
            assert batch(src=0) == BAD_ARGUMENTS and batch(in_bytes=0) == BAD_ARGUMENTS and batch(results=0) == BAD_ARGUMENTS
            assert batch(frames=0) == BAD_ARGUMENTS and batch(chunks=0) == BAD_ARGUMENTS
            assert single(fr=(0, 16)) == BAD_ARGUMENTS
            for kw in ({"l": (0, 16)}, {"b": (0, 16)}, {"r": (0, 16)}, {"l": (0, 16), "b": (0, 16), "r": (0, 16)}):
                assert single(**kw) == BAD_ARGUMENTS, kw                 # a Hap frame: luma, Cb and Cr are required
            assert single(l=(0, 16), b=(0, 16), r=(0, 16), a=(0, 16)) == BAD_ARGUMENTS
            # a Hap Alpha-Only frame: without alpha refused after its headers are read, before anything touches the GPU
            assert single(fr=ref_frame("rgtc1"), a=(0, 16)) == BAD_ARGUMENTS
            # the batch rules: 16-byte aligned planes, pitches, frame stride, blocks and block stride
            for kw in ({"l": lu + 8}, {"b": cbp + 8}, {"r": crp + 8}, {"a": al + 8}, {"fstride": fb + 8}, {"lp": sb * w + 8},
                       {"cp": sb * cw + 8}):
                assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
                assert batch(frames=2, **kw) == BAD_ARGUMENTS, kw
            for kw in ({"blocks": base + 8}, {"bstride": 2048 + 8}):
                assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
            # Hap Alpha-Only checks its alpha plane alone
            assert block(codec=HapB200Codec_HapA, l=0, b=0, r=0, a=al + 8, frames=2) == BAD_ARGUMENTS


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_planar_decoders_fail_loudly_without_a_gpu(lib):
    w, h = 256, 256
    frame = ref_frame()
    for sub in Q.SUBSAMPLINGS:
        for n in Q.DEPTHS:
            assert lib.decode_planar(frame, w, h, sub, n, Y.BT709_LIMITED)[0] == INTERNAL_ERROR
            # Hap Alpha-Only from its alpha plane alone passes the arguments, then finds no device
            assert lib.decode_planar(ref_frame("rgtc1"), w, h, sub, n, Y.BT709_LIMITED, alpha=bytearray(2 * w * h))[0] == INTERNAL_ERROR
            sb = P.sample_bytes(n)
            buf = np.zeros(16 * sb * 64 + 64, np.uint8)
            p = (buf.ctypes.data + 15) // 16 * 16
            res = np.zeros(1, np.uint32)
            nb = np.array([len(frame)], np.uint64)
            for codec in (HapB200Codec_Hap1, HapB200Codec_HapM, HapB200Codec_Hap7):
                assert lib.block_decode_planar_batch(p, 1, 16, 8, 8, codec, p, p + 256, p + 512, p + 768, 0, 16 * sb, 16 * sb, sub, n,
                                                     Y.BT601_FULL) == INTERNAL_ERROR
                assert lib.decode_planar_batch(p, 1, 4096, nb.ctypes.data, 4, codec, 8, 8, p, p + 256, p + 512, 0, 0, 16 * sb, 16 * sb, sub,
                                               n, Y.BT601_FULL, res.ctypes.data) == INTERNAL_ERROR
            assert lib.block_decode_planar_batch(p, 1, 16, 8, 8, HapB200Codec_HapA, 0, 0, 0, p, 0, 16 * sb, 16 * sb, sub, n,
                                                 Y.BT601_FULL) == INTERNAL_ERROR
