"""The RGBA16F -> HDR10 P010 conversion of include/hap_b200.h (HapB200DecodeYUVPQ*) and the argument rules of the HDR10
decoders, without a GPU.  The coefficient rows are their rule recomputed from Kr and Kb and sit within 0.6 of a code of the
real BT.2020 matrix; greys are neutral and codes 0 / 4095 land on nominal black and white; the library's transfer table P
(built on the host in double precision) equals an mpmath evaluation at 50 digits; flat colours return exactly through the
HDR10 encoders' matrix; the transfer round trip P[T[c]] = c holds where the header says it does; and the C++ sample-by-sample
conversion the emulated kernel test uses (tests/emu/yuv_pq_out_twin.cc) equals the numpy restatement
(tests/yuv_pq_out_util.py)."""
import numpy as np
import pytest

import hap_b200
import yuv_pq_out_util as Q
import yuv_pq_util as P
import yuv_util as Y
from golden_util import b64, golden
from hap_b200.abi import HapTextureFormat_RGB_BPTC_SIGNED_FLOAT, HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGBA_DXT5

BAD_ARGUMENTS, INTERNAL_ERROR = 1, 4
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT


def test_coefficients_follow_the_rule():
    for cs in P.COLOR_SPACES:
        assert Q.row(cs) == Q.rule_coefficients(cs), cs


def test_intermediates_stay_below_2_to_the_29():
    for cs in P.COLOR_SPACES:
        k = Q.row(cs)
        assert sum(abs(v) for v in k[0:3]) * 4095 + 32768 < 1 << 29
        assert sum(abs(v) for v in k[3:6]) * 8 * 4095 + (1 << 18) < 1 << 29
        assert sum(abs(v) for v in k[6:9]) * 8 * 4095 + (1 << 18) < 1 << 29


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
def test_integer_matrix_is_within_0_6_of_the_real_one(cs):
    rng = np.random.default_rng(3000 + cs)
    c = rng.integers(0, 4096, (200, 500, 3), dtype=np.int64)
    luma, chroma = Q.samples_of_codes(c, cs)
    fl, fc = Q.samples_of_codes_float(c, cs)
    err = max(np.abs(luma - fl).max(), np.abs(chroma - fc).max())
    assert err <= 0.6, err


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
def test_greys_are_neutral_and_black_and_white_nominal(cs):
    v = np.arange(4096, dtype=np.int64)
    c = np.repeat(np.repeat(v, 2)[None, :, None], 3, -1).repeat(2, 0)     # each grey over a 2 x 2 quad
    luma, chroma = Q.samples_of_codes(c, cs)
    yoff, ys, _, coff = P.scales(cs)
    assert (chroma == coff).all()
    assert (np.diff(luma[0, ::2]) >= 0).all()
    assert (luma[0, 0], luma[0, -1]) == ((64, 940) if cs == P.BT2020_LIMITED else (0, 1023))
    assert Q.black(cs) == (yoff, 512)


@pytest.mark.parametrize("unit", P.UNITS)
def test_library_table_equals_mpmath(unit):
    """every entry of the table the library builds in double precision is the 50-digit value"""
    np.testing.assert_array_equal(Q.twin_table(unit), Q.pq_out_table(unit))


@pytest.mark.parametrize("unit", P.UNITS)
def test_table_ends_and_monotonic(unit):
    t = Q.twin_table(unit)
    assert t.shape == (0x7C00,) and t[0] == 0
    assert (np.diff(t) >= 0).all()
    h = np.arange(0x7C00)
    v = h.astype(np.uint16).view(np.float16).astype(np.float64)
    assert (t[v >= 10000 / unit] == 4095).all()
    assert t.max() == 4095 and t.min() == 0


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
def test_flat_colours_return_through_the_encoders_matrix(cs):
    """a flat P010 triple -> 12-bit R'G'B' by HAPB200_YUV_PQ_COEFFICIENTS -> back by the rows here: exact wherever R'G'B' is
    not clamped.  Every luma value of the nominal range with Cb and Cr on a grid of step 5 (the whole range, at a seventh of
    the work of an exhaustive sweep of it)."""
    cy, crr, cbg, crg, cbb, yoff_in, coff_in = (int(v) for v in P.coefficients()[cs - P.BT2020_LIMITED])
    k = Q.row(cs)
    lo, hi_y, hi_c = (64, 940, 960) if cs == P.BT2020_LIMITED else (0, 1023, 1023)
    ys = np.arange(lo, hi_y + 1, dtype=np.int64)
    checked = 0
    for cb in range(lo, hi_c + 1, 5):
        cr = np.arange(lo, hi_c + 1, 5, dtype=np.int64)
        yv, crv = np.meshgrid(ys, cr, indexing="ij")
        yd, cb8, cr8 = cy * (yv - yoff_in), 8 * (cb - coff_in), 8 * (crv - coff_in)
        rgb = np.stack([(yd + crr * cr8 + 32768) >> 16, (yd + cbg * cb8 + crg * cr8 + 32768) >> 16, (yd + cbb * cb8 + 32768) >> 16], -1)
        keep = ((rgb >= 0) & (rgb <= 4095)).all(-1)
        r, g, b = (rgb[..., i][keep] for i in range(3))
        y2 = np.clip(((k[0] * r + k[1] * g + k[2] * b + 32768) >> 16) + k[9], 0, 1023)
        cb2 = np.clip(((k[3] * 8 * r + k[4] * 8 * g + k[5] * 8 * b + (1 << 18)) >> 19) + k[10], 0, 1023)
        cr2 = np.clip(((k[6] * 8 * r + k[7] * 8 * g + k[8] * 8 * b + (1 << 18)) >> 19) + k[10], 0, 1023)
        assert (y2 == yv[keep]).all() and (cb2 == cb).all() and (cr2 == crv[keep]).all(), cb
        checked += int(keep.sum())
    assert checked > 1_000_000, checked


@pytest.mark.parametrize("unit,failing", [(1, []), (80, []), (100, []), (123, []), (124, [1]), (203, [1]), (1000, 16), (10000, 180)])
def test_transfer_round_trip_floors(unit, failing):
    """P[T[c]] == c at 50 digits (T of the HDR10 encoders, P of the decoders): every code up to unitNits 123; above, only the
    lowest codes miss (a list: exactly those; a number: every code from it on returns, and the one below it does not)"""
    t = P.pq_table(unit).astype(np.int64)
    back = np.array([Q.pq_out_code(int(h), unit) for h in t])
    bad = np.flatnonzero(back != np.arange(4096))
    if isinstance(failing, list):
        assert bad.tolist() == failing
    else:
        assert bad.max() == failing - 1
    # the library's double-precision tables agree
    assert (Q.twin_table(unit)[P.twin_table(unit).astype(np.int64)] == back).all()


def test_transfer_round_trip_holds_at_every_unit_up_to_123():
    """the library's tables (both equal to their 50-digit definitions at the units above) for every unitNits 1 .. 123"""
    for unit in range(1, 124):
        assert (Q.twin_table(unit)[P.twin_table(unit).astype(np.int64)] == np.arange(4096)).all(), unit


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
@pytest.mark.parametrize("unit", (80, 203, 10000))
def test_cpp_conversion_equals_the_numpy_definition(cs, unit):
    """tests/emu/yuv_pq_out_twin.cc, on which the emulated kernel test rests, is the conversion of the header"""
    rng = np.random.default_rng(600 + cs + unit)
    for w, h, pad in ((4, 4, 0), (12, 8, 16), (36, 20, 48), (132, 12, 0), (124, 8, 32), (260, 4, 16)):
        rgba = Q.random_halves(rng, h, w)
        want = Q.rgba_half_to_yuv_pq(rgba, cs, unit, table=Q.pq_out_table(unit))
        got = Q.twin_to_yuv(rgba, cs, unit, pitch=2 * w + pad)
        np.testing.assert_array_equal(got[0], want[0], err_msg=str((w, h, pad)))
        np.testing.assert_array_equal(got[1], want[1], err_msg=str((w, h, pad)))


def test_failed_frame_is_black():
    for cs in P.COLOR_SPACES:
        luma, chroma = Q.rgba_half_to_yuv_pq(np.zeros((4, 8, 4), np.uint16), cs, 203)
        yb, cb = Q.black(cs)
        assert (luma == yb << 6).all() and (chroma == cb << 6).all()


# ---- argument rules of the entry points -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def test_yuv_pq_decoders_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(16 * w * h + 64, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    c = p + 4 * w * h                                      # a 16-byte aligned chroma plane
    res = np.zeros(4, np.uint32)
    nb = np.full(4, 64, np.uint64)
    fb = 4 * w * h
    frame = bytes(64)

    def block(blocks=p, frames=1, bstride=2048, gw=w, gh=h, fmt=UF16, lp=p, cp=c, fstride=fb, pitch=2 * w, cs=P.BT2020_LIMITED, unit=203):
        return lib.block_decode_yuv_pq_batch(blocks, frames, bstride, gw, gh, fmt, lp, cp, fstride, pitch, cs, unit)

    def batch(src=p, frames=1, istride=2048, in_bytes=nb.ctypes.data, chunks=4, gw=w, gh=h, lp=p, cp=c, fstride=fb, pitch=2 * w,
              cs=P.BT2020_LIMITED, unit=203, results=res.ctypes.data):
        return lib.decode_yuv_pq_batch(src, frames, istride, in_bytes, chunks, gw, gh, lp, cp, fstride, pitch, cs, unit, results)

    def single(fr=frame, gw=w, gh=h, pitch=None, cs=P.BT2020_LIMITED, unit=203, lp=None, cp=None):
        pitch = pitch if pitch is not None else 2 * gw
        lp = lp if lp is not None else bytearray(64)              # (every call here is refused before the planes are touched)
        cp = cp if cp is not None else bytearray(64)
        return lib.decode_yuv_pq(fr, gw, gh, cs, unit, pitch=pitch, luma=lp, chroma=cp)[0]

    for f in (block, batch, single):
        # colour spaces other than BT.2020; unitNits outside 1 .. 10000
        for cs in (0, 1, 2, 3, 6, 0xFFFFFFFF):
            assert f(cs=cs) == BAD_ARGUMENTS, (f.__name__, cs)
        for unit in (0, 10001, 0xFFFFFFFF):
            assert f(unit=unit) == BAD_ARGUMENTS, (f.__name__, unit)
        # geometry: sizes not multiples of 4, empty, pitch below the row, pitch >= 2^32
        for gw, gh, pitch in ((6, 4, 16), (4, 6, 16), (0, 4, 16), (4, 0, 16), (64, 32, 2 * 64 - 16), (64, 32, 1 << 32)):
            assert f(gw=gw, gh=gh, pitch=pitch) == BAD_ARGUMENTS, (f.__name__, gw, gh, pitch)
    # texture formats other than BC6H
    for fmt in (0, HapTextureFormat_RGBA_DXT5, 0xA3, 0xFFFFFFFF):
        assert block(fmt=fmt) == BAD_ARGUMENTS, fmt
    # null pointers, no frames, no chunks
    assert block(blocks=0) == BAD_ARGUMENTS and block(lp=0) == BAD_ARGUMENTS and block(cp=0) == BAD_ARGUMENTS
    assert batch(src=0) == BAD_ARGUMENTS and batch(in_bytes=0) == BAD_ARGUMENTS and batch(results=0) == BAD_ARGUMENTS
    assert batch(lp=0) == BAD_ARGUMENTS and batch(cp=0) == BAD_ARGUMENTS
    assert single(lp=(0, 16)) == BAD_ARGUMENTS and single(cp=(0, 16)) == BAD_ARGUMENTS and single(fr=(0, 16)) == BAD_ARGUMENTS
    assert block(frames=0) == BAD_ARGUMENTS and batch(frames=0) == BAD_ARGUMENTS and batch(chunks=0) == BAD_ARGUMENTS
    # the batch rules: 16-byte aligned planes, pitch, frame stride, blocks and block stride
    for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": 2 * w + 8}, {"blocks": p + 8}, {"bstride": 2048 + 8}):
        assert block(frames=2, **kw) == BAD_ARGUMENTS, kw
    for kw in ({"lp": p + 8}, {"cp": c + 8}, {"fstride": fb + 8}, {"pitch": 2 * w + 8}):
        assert batch(frames=2, **kw) == BAD_ARGUMENTS, kw


def test_8bit_yuv_decoders_still_refuse_bt2020(lib):
    frame = b64(golden()["ref_frames"]["dxt1"]["frame_b64"])
    for cs in P.COLOR_SPACES:
        assert lib.decode_yuv(frame, 256, 256, Y.P010, cs, luma=bytearray(64), chroma=bytearray(64))[0] == BAD_ARGUMENTS


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_yuv_pq_decoders_fail_loudly_without_a_gpu(lib):
    w, h = 8, 8
    buf = np.zeros(4096, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    res = np.zeros(1, np.uint32)
    nb = np.array([64], np.uint64)
    for fmt in (UF16, SF16):
        assert lib.block_decode_yuv_pq_batch(p, 1, 64, w, h, fmt, p + 1024, p + 2048, 0, 16, P.BT2020_FULL, 100) == INTERNAL_ERROR
    assert lib.decode_yuv_pq_batch(p, 1, 1024, nb.ctypes.data, 4, w, h, p + 1024, p + 2048, 0, 16, P.BT2020_LIMITED, 203,
                                   res.ctypes.data) == INTERNAL_ERROR
    # a one-texture UF16 frame, uncompressed (section type 0xA2: no compressor, RGB BPTC unsigned float), 4 zero blocks
    tex = bytes(4 * 16)
    frame = bytes([len(tex), 0, 0, 0xA2]) + tex
    assert lib.decode_yuv_pq(frame, w, h, P.BT2020_LIMITED, 203)[0] == INTERNAL_ERROR
