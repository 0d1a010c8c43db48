"""The HDR10 P010 -> RGBA16F conversion of include/hap_b200.h (HapB200EncodeYUVPQ*) and its argument rules, without a GPU.
The coefficient rows are the rule recomputed from Kr and Kb; the library's transfer table (built on the host in double
precision) equals an mpmath evaluation at 50 digits rounded once to binary16; the integer matrix is within 0.6 of a code
of the real one; the C++ pixel-by-pixel conversion the emulated kernel test uses (tests/emu/yuv_pq_twin.cc) equals the
numpy restatement (tests/yuv_pq_util.py); and the ST 2084 anchor luminances land where the formula puts them."""
import numpy as np
import pytest

import hap_b200
import yuv_pq_util as P
import yuv_util as Y
from hap_b200.abi import (HapCompressorSnappy, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT, HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT,
                          HapTextureFormat_RGBA_DXT5)
from hap_b200.lib import HapB200Codec_HapY

BAD_ARGUMENTS, BUFFER_TOO_SMALL, INTERNAL_ERROR = 1, 2, 4
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT


def test_coefficients_are_the_rounded_bt2020_matrix():
    kg = 1 - P.KR - P.KB
    f = 65536 * 4095
    for cs in P.COLOR_SPACES:
        yoff, ys, csc, coff = P.scales(cs)
        want = [f / ys, f * 2 * (1 - P.KR) / csc / 8, -f * 2 * P.KB * (1 - P.KB) / kg / csc / 8,
                -f * 2 * P.KR * (1 - P.KR) / kg / csc / 8, f * 2 * (1 - P.KB) / csc / 8]
        row = P.coefficients()[cs - P.BT2020_LIMITED]
        assert list(row[:5]) == [int(np.floor(v + 0.5)) for v in want]
        assert list(row[5:]) == [yoff, coff]
    assert P.coefficients().tolist() == [[306358, 55209, -6161, -21391, 70440, 64, 512], [262336, 48355, -5396, -18736, 61695, 0, 512]]


def test_the_8bit_rule_with_255_reproduces_the_p010_bt709_row():
    """the rule the PQ rows follow is the existing one with 4095 for 255"""
    kr, kb = Y.KRKB[Y.BT709_LIMITED]
    kg = 1 - kr - kb
    f = 65536 * 255
    want = [f / 876, f * 2 * (1 - kr) / 896 / 8, -f * 2 * kb * (1 - kb) / kg / 896 / 8, -f * 2 * kr * (1 - kr) / kg / 896 / 8,
            f * 2 * (1 - kb) / 896 / 8]
    assert list(Y.coefficients()[4 + Y.BT709_LIMITED][:5]) == [int(np.floor(v + 0.5)) for v in want]


def test_intermediates_stay_below_2_to_the_30():
    for row in P.coefficients():
        cy, crr, cbg, crg, cbb, yoff, coff = (int(v) for v in row)
        yd = max(abs(0 - yoff), 1023 - yoff)
        c8 = 8 * max(coff, 1023 - coff)
        for terms in ((cy * yd, abs(crr) * c8), (cy * yd, abs(cbg) * c8, abs(crg) * c8), (cy * yd, abs(cbb) * c8)):
            assert sum(terms) + 32768 < 1 << 30


@pytest.mark.parametrize("unit", P.UNITS)
def test_library_table_equals_mpmath_rounded_to_half(unit):
    """every entry of the table the library builds in double precision is the 50-digit value rounded once to binary16"""
    np.testing.assert_array_equal(P.twin_table(unit), P.pq_table(unit))


@pytest.mark.parametrize("unit", P.UNITS)
def test_table_ends_and_monotonic(unit):
    t = P.twin_table(unit)
    assert t[0] == 0
    assert t[4095] == np.float16(10000 / unit).view(np.uint16)
    assert (np.diff(t.astype(np.int64)) >= 0).all()
    v = t.view(np.float16).astype(np.float64)
    assert np.isfinite(v).all() and (v >= 0).all()


def test_table_step_above_one_nit():
    """the table's relative step is at most 0.48 % above 1 cd/m2 (float64, before rounding to half)"""
    import mpmath
    nits = np.array([float(v) for v in P._eotf_nits()])
    above = nits[:-1] >= 1.0
    step = (nits[1:] - nits[:-1])[above] / nits[:-1][above]
    assert step.max() < 0.0048, step.max()


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
def test_r12_is_within_0_6_of_the_real_matrix(cs):
    rng = np.random.default_rng(40 + cs)
    w, h = 500, 200
    luma, chroma = P.random_planes(rng, w, h)
    got = P.r12(luma, chroma, cs).astype(np.float64)
    want = P.r12_float(luma, chroma, cs)
    inside = (want >= 0) & (want <= 4095)
    assert inside.mean() > 0.2
    err = np.abs(got - want)[inside]
    assert err.max() < 0.6, err.max()
    # out of range: clamped
    assert (got[want < 0] == 0).all() and (got[want > 4095] == 4095).all()


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
@pytest.mark.parametrize("unit", (80, 203, 10000))
def test_cpp_conversion_equals_the_numpy_definition(cs, unit):
    """tests/emu/yuv_pq_twin.cc, on which the emulated kernel test rests, is the conversion of the header"""
    rng = np.random.default_rng(500 + cs + unit)
    for w, h, pad in ((4, 4, 0), (12, 8, 16), (36, 20, 48), (132, 12, 0), (20, 4, 8)):
        luma, chroma = P.random_planes(rng, w, h)
        want = P.yuv_pq_to_rgba_half(luma, chroma, cs, unit)
        got = P.twin_to_rgba_half(luma, chroma, cs, unit, pitch=2 * w + pad)
        np.testing.assert_array_equal(got, want, err_msg=str((w, h, pad)))
    luma, chroma = P.hdr10_planes("video", 68, 36, cs)
    np.testing.assert_array_equal(P.twin_to_rgba_half(luma, chroma, cs, unit), P.yuv_pq_to_rgba_half(luma, chroma, cs, unit))


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
def test_anchor_luminances(cs):
    """100, 203 and 1000 cd/m2 (grey) sit at the PQ codes ST 2084 gives (51 %, 58 %, 75 % of full scale; BT.2408 puts
    203 cd/m2 at 58 %), and a flat grey P010 picture at those codes converts back to within the table's step"""
    for nits, pct in ((100, 0.508), (203, 0.581), (1000, 0.752)):
        e = float(P.pq_inverse(nits))
        assert abs(e - pct) < 0.001, (nits, e)
        yoff, ys, _, coff = P.scales(cs)
        code = int(np.rint(yoff + ys * e))
        luma = np.full((4, 4), code << 6, np.uint16)
        chroma = np.full((2, 4), coff << 6, np.uint16)
        for unit in (1, 100, 203):
            got = P.yuv_pq_to_rgba_half(luma, chroma, cs, unit)[..., :3].view(np.float16).astype(np.float64) * unit
            # one 10-bit code is about 4 table steps of at most 0.48 % each: within 1 % of the anchor
            assert np.allclose(got, nits, rtol=0.01), (nits, unit, got[0, 0])


def test_content_maker_round_trips_flat_colours():
    """planes_from_rgb_signal (under hdr10_planes): flat BT.2020 colours through PQ and the matrix come back from the
    conversion within the 10-bit quantisation (a few per cent for saturated colours, whose chroma is quantised coarsely)"""
    rng = np.random.default_rng(3)
    for cs in P.COLOR_SPACES:
        for _ in range(200):
            nits = 10.0 ** rng.uniform(-1, 3.6, 3)
            luma, chroma = P.planes_from_rgb_signal(np.broadcast_to(P.pq_inverse(nits), (4, 4, 3)), cs, rng)
            got = P.yuv_pq_to_rgba_half(luma, chroma, cs, 1)[0, 0, :3].view(np.float16).astype(np.float64)
            k = np.array([P.KR, 1 - P.KR - P.KB, P.KB])
            assert abs(got @ k / (nits @ k) - 1) < 0.05, (nits, got)


# ---- argument rules of the entry points -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def test_yuv_pq_entry_points_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(16 * w * h + 64, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    c = p + 4 * w * h
    used = np.zeros(4, np.uint64)
    u = used.ctypes.data
    ostride = (lib.max_encoded_length_half(w, h, UF16, 1) + 15) // 16 * 16
    fb = 4 * w * h
    luma, chroma = np.zeros(2 * w * h, np.uint8), np.zeros(w * h, np.uint8)

    def block(lp=p, cp=c, frames=1, fstride=fb, gw=w, gh=h, pitch=2 * w, cs=P.BT2020_LIMITED, unit=203, fmt=UF16, blocks=p, bstride=2048):
        return lib.block_encode_yuv_pq_batch(lp, cp, frames, fstride, gw, gh, pitch, cs, unit, fmt, blocks, bstride)

    def batch(lp=p, cp=c, frames=1, fstride=fb, gw=w, gh=h, pitch=2 * w, cs=P.BT2020_LIMITED, unit=203, fmt=UF16, comp=HapCompressorSnappy,
              chunks=1, out=p, out_stride=ostride, used_p=u):
        return lib.encode_yuv_pq_batch(lp, cp, frames, fstride, gw, gh, pitch, cs, unit, fmt, comp, chunks, out, out_stride, used_p)

    def single(lb=luma, cb=chroma, gw=w, gh=h, pitch=None, cs=P.BT2020_LIMITED, unit=203, fmt=UF16, comp=HapCompressorSnappy, chunks=1,
               cap_=None):
        n = cap_ if cap_ is not None else 1 << 20
        return lib.encode_yuv_pq(lb, cb, gw, gh, cs, unit, fmt, comp, chunks, pitch=pitch, out=bytearray(max(n, 1 << 20)), out_capacity=n)[0]

    for f in (block, batch, single):
        for cs in (0, 1, 2, 3, 6, 0xFFFFFFFF):
            assert f(cs=cs) == BAD_ARGUMENTS, (f.__name__, cs)
        for unit in (0, 10001, 0xFFFFFFFF):
            assert f(unit=unit) == BAD_ARGUMENTS, (f.__name__, unit)
        for fmt in (0, HapTextureFormat_RGBA_DXT5, 0xA3, 0xFFFFFFFF):
            assert f(fmt=fmt) == BAD_ARGUMENTS, (f.__name__, fmt)
        for gw, gh, pitch in ((6, 4, 16), (4, 6, 16), (0, 4, 16), (4, 0, 16), (w, h, 2 * w - 16), (w, h, 1 << 32)):
            assert f(gw=gw, gh=gh, pitch=pitch) == BAD_ARGUMENTS, (f.__name__, gw, gh, pitch)
    assert block(lp=0) == BAD_ARGUMENTS and block(cp=0) == BAD_ARGUMENTS and block(blocks=0) == BAD_ARGUMENTS
    assert batch(lp=0) == BAD_ARGUMENTS and batch(cp=0) == BAD_ARGUMENTS
    assert single(lb=(0, 16)) == BAD_ARGUMENTS and single(cb=(0, 16)) == BAD_ARGUMENTS
    assert block(frames=0) == BAD_ARGUMENTS and batch(frames=0) == BAD_ARGUMENTS
    assert batch(out=0) == BAD_ARGUMENTS and batch(used_p=0) == BAD_ARGUMENTS
    assert batch(chunks=0) == BAD_ARGUMENTS and batch(comp=0xC1) == BAD_ARGUMENTS
    assert single(chunks=0) == BAD_ARGUMENTS and single(comp=0xC1) == BAD_ARGUMENTS
    for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": 2 * w + 8}, {"blocks": p + 8}, {"bstride": 2048 + 8}):
        assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
    for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": 2 * w + 8}, {"out": p + 8}, {"out_stride": ostride + 8}):
        assert batch(frames=2, **kw) == BAD_ARGUMENTS, kw
    for fmt in (UF16, SF16):
        for k in (1, 3, 8):
            need = lib.max_encoded_length_half(w, h, fmt, k)
            assert batch(fmt=fmt, chunks=k, out_stride=(need - 1) // 16 * 16) == BUFFER_TOO_SMALL
            assert single(fmt=fmt, chunks=k, cap_=need - 1) == BUFFER_TOO_SMALL


def test_8bit_yuv_encoders_still_refuse_bt2020(lib):
    w, h = 16, 8
    luma, chroma = np.zeros(2 * w * h, np.uint8), np.zeros(w * h, np.uint8)
    for cs in (P.BT2020_LIMITED, P.BT2020_FULL):
        assert lib.encode_yuv(luma, chroma, w, h, Y.P010, cs, HapB200Codec_HapY)[0] == BAD_ARGUMENTS


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_yuv_pq_valid_arguments_fail_loudly_without_a_gpu(lib):
    w, h = 16, 8
    luma, chroma = P.random_planes(np.random.default_rng(0), w, h)
    assert lib.encode_yuv_pq(luma, chroma, w, h, P.BT2020_LIMITED, 203, UF16)[0] == INTERNAL_ERROR
