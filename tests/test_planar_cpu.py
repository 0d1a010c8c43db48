"""The planar Y'CbCr -> RGBA8 conversion of include/hap_b200.h (HapB200EncodePlanar) and the argument rules of the planar
encoders, without a GPU.  planar_util.planar_to_rgba (the definition restated in numpy integers) is held to the real
matrix in float64, to the rounding rule of the 12-bit table, to the identities the definition implies, to the published
colour bars, and to the C++ pixel-by-pixel conversion the emulated kernel test uses (tests/emu/planar_twin.cc)."""
import numpy as np
import pytest

import hap_b200
import planar_util as P
import yuv_util as Y
from hap_b200.abi import HapCompressorSnappy
from hap_b200.lib import (HapB200Codec_Hap1, HapB200Codec_Hap5, HapB200Codec_Hap7, HapB200Codec_HapA, HapB200Codec_HapM,
                          HapB200Codec_HapY)

BAD_ARGUMENTS, BUFFER_TOO_SMALL, INTERNAL_ERROR = 1, 2, 4
CODECS = (HapB200Codec_Hap1, HapB200Codec_Hap5, HapB200Codec_HapY, HapB200Codec_HapM, HapB200Codec_HapA)


@pytest.mark.parametrize("n", P.DEPTHS)
@pytest.mark.parametrize("cs", P.COLOR_SPACES)
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_integer_conversion_is_within_0_6_of_the_real_matrix(sub, n, cs):
    rng = np.random.default_rng(2000 + 100 * sub + 10 * n + cs)
    w, h = 640, 320                                  # 204 800 pixels: every sample value of the depth, in every plane
    luma, cb, cr, _ = P.random_planes(rng, w, h, sub, n, alpha=False)
    for plane in (luma, cb, cr):
        assert len(np.unique(P.samples(plane, n))) == 1 << n
    got = P.planar_to_rgba(luma, cb, cr, None, sub, n, cs)
    want = P.planar_to_rgb_float(luma, cb, cr, sub, n, cs)
    err = np.abs(got[..., :3].astype(np.float64) - want)
    assert err.max() < 0.6, err.max()
    assert (got[..., 3] == 255).all()


def test_12bit_coefficients_are_the_rounded_matrix():
    for cs in P.COLOR_SPACES:
        yoff, ys, csc, coff = P.scales(12, cs)
        kr, kb = Y.KRKB[cs]
        kg = 1 - kr - kb
        f = (1 << 18) * 255
        want = [f / ys, f * 2 * (1 - kr) / csc / 8, -f * 2 * kb * (1 - kb) / kg / csc / 8, -f * 2 * kr * (1 - kr) / kg / csc / 8,
                f * 2 * (1 - kb) / csc / 8]
        row = P.coefficients12()[cs]
        assert list(row[:5]) == [int(np.floor(v + 0.5)) for v in want]
        assert list(row[5:]) == [yoff, coff] == [256 if not Y.is_full(cs) else 0, 2048]
        if not Y.is_full(cs):                        # the 12-bit limited scales are 4 x the 10-bit ones
            assert list(row[:5]) == list(Y.coefficients()[4 + cs][:5])


def test_12bit_intermediates_stay_below_2_31():
    for cs in P.COLOR_SPACES:
        cy, crr, cbg, crg, cbb, yoff, coff = (int(v) for v in P.coefficients12()[cs])
        yd = max(abs(0 - yoff), 4095 - yoff) * cy
        cd = 8 * max(coff, 4095 - coff)
        worst = yd + max(abs(crr), abs(cbb), abs(cbg) + abs(crg)) * cd + (1 << 17)
        assert worst < 1 << 31


# ---- identities of the definition ---------------------------------------------------------------------------------------

@pytest.mark.parametrize("cs", P.COLOR_SPACES)
def test_420_8bit_is_nv12(cs):
    rng = np.random.default_rng(40 + cs)
    w, h = 96, 64
    luma, cb, cr, _ = P.random_planes(rng, w, h, P.S420, 8, alpha=False)
    nv12 = np.stack([cb, cr], -1).reshape(h // 2, w)
    np.testing.assert_array_equal(P.planar_to_rgba(luma, cb, cr, None, P.S420, 8, cs), Y.yuv_to_rgba(luma, nv12, Y.NV12, cs))


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
def test_420_10bit_is_p010(cs):
    rng = np.random.default_rng(50 + cs)
    w, h = 96, 64
    luma, cb, cr, _ = P.random_planes(rng, w, h, P.S420, 10, alpha=False)
    word = lambda p: ((P.samples(p, 10) << 6) | rng.integers(0, 64, p.shape)).astype(np.uint16)
    p010 = np.stack([word(cb), word(cr)], -1).reshape(h // 2, w)
    np.testing.assert_array_equal(P.planar_to_rgba(luma, cb, cr, None, P.S420, 10, cs), Y.yuv_to_rgba(word(luma), p010, Y.P010, cs))


@pytest.mark.parametrize("cs", [Y.BT601_LIMITED, Y.BT709_LIMITED])
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_12bit_of_four_times_10bit_gives_the_10bit_picture(sub, cs):
    rng = np.random.default_rng(60 + 10 * sub + cs)
    w, h = 96, 64
    planes = P.random_planes(rng, w, h, sub, 10, alpha=False, junk_high_bits=False)[:3]
    four = [(P.samples(p, 10) << 2).astype(np.uint16) for p in planes]
    np.testing.assert_array_equal(P.planar_to_rgba(*four, None, sub, 12, cs), P.planar_to_rgba(*planes, None, sub, 10, cs))


@pytest.mark.parametrize("n", P.DEPTHS)
def test_422_equals_420_when_chroma_rows_repeat(n):
    rng = np.random.default_rng(70 + n)
    w, h = 64, 32
    luma, cb, cr, _ = P.random_planes(rng, w, h, P.S420, n, alpha=False)
    cb = np.repeat(cb[:1], h // 2, axis=0)           # every 4:2:0 chroma row the same ...
    cr = np.repeat(cr[:1], h // 2, axis=0)
    cb2, cr2 = np.repeat(cb[:1], h, axis=0), np.repeat(cr[:1], h, axis=0)   # ... and the 4:2:2 plane repeats it
    for cs in P.COLOR_SPACES:
        np.testing.assert_array_equal(P.planar_to_rgba(luma, cb, cr, None, P.S420, n, cs), P.planar_to_rgba(luma, cb2, cr2, None, P.S422, n, cs))


@pytest.mark.parametrize("n", P.DEPTHS)
def test_subsamplings_agree_on_flat_chroma(n):
    rng = np.random.default_rng(80 + n)
    w, h = 32, 16
    luma = P.random_planes(rng, w, h, P.S444, n, alpha=False)[0]
    for cs in P.COLOR_SPACES:
        for _ in range(20):
            b, r = rng.integers(0, 1 << n, 2)
            pics = []
            for sub in P.SUBSAMPLINGS:
                ch, cw = P.chroma_shape(w, h, sub)
                flat = lambda v: P.as_plane(np.full((ch, cw), v, np.int64), n)
                pics.append(P.planar_to_rgba(luma, flat(b), flat(r), None, sub, n, cs))
            np.testing.assert_array_equal(pics[0], pics[1])
            np.testing.assert_array_equal(pics[0], pics[2])


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


@pytest.mark.parametrize("n", P.DEPTHS)
@pytest.mark.parametrize("cs", sorted(BARS))
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_colour_bars(sub, cs, n):
    s = 1 << (n - 8)                                  # the n-bit code of an 8-bit value is 2^(n-8) times it
    ch, cw = P.chroma_shape(4, 4, sub)
    for name, (yv, cb, cr, rgb) in BARS[cs].items():
        flat = lambda v, shape: P.as_plane(np.full(shape, v * s, np.int64), n)
        got = P.planar_to_rgba(flat(yv, (4, 4)), flat(cb, (ch, cw)), flat(cr, (ch, cw)), None, sub, n, cs)
        assert (np.abs(got[..., :3].astype(int) - np.array(rgb)) <= 1).all(), (name, got[0, 0], rgb)


@pytest.mark.parametrize("n", P.DEPTHS)
def test_alpha_mapping_over_every_value(n):
    a = np.arange(1 << n, dtype=np.int64)
    m = (1 << n) - 1
    got = P.alpha8(a, n)
    # 255 a / (2^n - 1) rounded half up, in exact integers: floor((2 * 255 a + m) / (2 m))
    want = np.array([(2 * 255 * int(v) + m) // (2 * m) for v in a])
    np.testing.assert_array_equal(got, want)
    frac = 255 * a / m
    assert np.all(np.abs(got - frac) <= 0.5)
    assert got[0] == 0 and got[-1] == 255 and np.all(np.diff(got) >= 0)
    if n == 8:
        np.testing.assert_array_equal(got, a)
    else:                                             # the kernel's multiply-and-shift (planar_alpha16) gives the same
        assert [P.kernel_alpha(int(v), n) for v in a] == list(got)
    # through the whole conversion
    w = 1 << (n // 2)
    h = (1 << n) // w
    alpha = P.as_plane(a.reshape(h, w), n)
    luma, cb, cr, _ = P.random_planes(np.random.default_rng(n), w, h, P.S444, n, alpha=False)
    np.testing.assert_array_equal(P.planar_to_rgba(luma, cb, cr, alpha, P.S444, n, Y.BT709_FULL)[..., 3], got.reshape(h, w))


@pytest.mark.parametrize("n", (10, 12))
def test_junk_high_bits_are_ignored(n):
    rng = np.random.default_rng(90 + n)
    w, h = 64, 32
    for sub in P.SUBSAMPLINGS:
        clean = P.random_planes(rng, w, h, sub, n, junk_high_bits=False)
        dirty = [(p.astype(np.int64) | (rng.integers(0, 1 << (16 - n), p.shape) << n)).astype(np.uint16) for p in clean]
        for cs in P.COLOR_SPACES:
            np.testing.assert_array_equal(P.planar_to_rgba(*clean, sub, n, cs), P.planar_to_rgba(*dirty, sub, n, cs))
            np.testing.assert_array_equal(P.twin_to_rgba(*dirty, sub, n, cs), P.planar_to_rgba(*clean, sub, n, cs))


@pytest.mark.parametrize("n", P.DEPTHS)
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_cpp_conversion_equals_the_numpy_definition(sub, n):
    """tests/emu/planar_twin.cc, on which the emulated kernel test rests, is the conversion of the header"""
    rng = np.random.default_rng(300 + 10 * sub + n)
    for cs in P.COLOR_SPACES:
        for w, h, lpad, cpad, alpha in ((4, 4, 0, 0, True), (12, 8, 16, 48, False), (36, 20, 48, 0, True), (132, 12, 0, 16, True)):
            planes = P.random_planes(rng, w, h, sub, n, alpha=alpha)
            want = P.planar_to_rgba(*planes, sub, n, cs)
            np.testing.assert_array_equal(P.twin_to_rgba(*planes, sub, n, cs, lpad, cpad), want)


# ---- argument rules of the entry points -------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


@pytest.mark.parametrize("n", P.DEPTHS)
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_planar_entry_points_refuse_bad_arguments(lib, sub, n):
    w, h = 64, 32
    sb = P.sample_bytes(n)
    ch, cw = P.chroma_shape(w, h, sub)
    lp, cp = sb * w, sb * cw
    buf = np.zeros(64 * w * h + 64, np.uint8)
    base = (buf.ctypes.data + 15) // 16 * 16
    fb = 4 * sb * w * h                                  # a 16-byte multiple that holds every plane of a frame
    lum, cbp, crp, alp = base, base + sb * w * h, base + 2 * sb * w * h, base + 3 * sb * w * h
    used = np.zeros(4, np.uint64)
    u = used.ctypes.data
    cap = lib.max_encoded_length_rgba(w, h, HapB200Codec_HapM, 1)
    ostride = (cap + 15) // 16 * 16
    luma, cb, cr, alpha = (np.zeros(sb * w * h, np.uint8), np.zeros(sb * cw * ch, np.uint8), np.zeros(sb * cw * ch, np.uint8),
                           np.zeros(sb * w * h, np.uint8))

    def block(l=lum, b=cbp, r=crp, a=alp, frames=1, fstride=fb, gw=w, gh=h, lpitch=lp, cpitch=cp, s=sub, d=n, cs=0,
              codec=HapB200Codec_HapY, blocks=base, bstride=4096):
        return lib.block_encode_planar_batch(l, b, r, a, frames, fstride, gw, gh, lpitch, cpitch, s, d, cs, codec, blocks, bstride)

    def batch(l=lum, b=cbp, r=crp, a=alp, frames=1, fstride=fb, gw=w, gh=h, lpitch=lp, cpitch=cp, s=sub, d=n, cs=0,
              codec=HapB200Codec_HapY, comp=HapCompressorSnappy, chunks=1, out=base, out_stride=ostride, used_p=u):
        return lib.encode_planar_batch(l, b, r, a, frames, fstride, gw, gh, lpitch, cpitch, s, d, cs, codec, comp, chunks, out,
                                       out_stride, used_p)

    def single(l=luma, b=cb, r=cr, a=alpha, gw=w, gh=h, lpitch=lp, cpitch=cp, s=sub, d=n, cs=0, codec=HapB200Codec_HapY,
               comp=HapCompressorSnappy, chunks=1, cap_=None):
        k = cap_ if cap_ is not None else 1 << 20
        return lib.encode_planar(l, b, r, a, gw, gh, s, d, cs, codec, comp, chunks, luma_pitch=lpitch, chroma_pitch=cpitch,
                                 out=bytearray(max(k, 1 << 20)), out_capacity=k)[0]

    for f in (block, batch, single):
        # codecs: Hap R, unknown; Hap Alpha-Only without alpha
        for codec in (HapB200Codec_Hap7, 6, 0xFFFFFFFF):
            assert f(codec=codec) == BAD_ARGUMENTS, (f.__name__, codec)
        assert f(codec=HapB200Codec_HapA, a=None if f is single else 0) == BAD_ARGUMENTS
        # depths, subsamplings and colour spaces out of range (BT.2020 among them)
        for d in (0, 1, 9, 11, 14, 16, 0xFFFFFFFF):
            assert f(d=d) == BAD_ARGUMENTS, (f.__name__, d)
        assert f(s=3) == BAD_ARGUMENTS and f(s=0xFFFFFFFF) == BAD_ARGUMENTS
        for cs in (4, 5, 6, 0xFFFFFFFF):
            assert f(cs=cs) == BAD_ARGUMENTS, (f.__name__, cs)
        # geometry: sizes not multiples of 4, empty, each pitch below its row or at 2^32
        for gw, gh in ((6, 4), (4, 6), (0, 4), (4, 0), (w + 2, h), (w, h + 2)):
            assert f(gw=gw, gh=gh) == BAD_ARGUMENTS, (f.__name__, gw, gh)
        for kw in ({"lpitch": lp - 16}, {"lpitch": lp - 1}, {"lpitch": 1 << 32}, {"cpitch": cp - 16}, {"cpitch": cp - 1},
                   {"cpitch": 1 << 32}):
            assert f(**kw) == BAD_ARGUMENTS, (f.__name__, kw)
        # Hap Alpha-Only checks the alpha plane's geometry
        assert f(codec=HapB200Codec_HapA, lpitch=lp - 16) == BAD_ARGUMENTS
    # null planes: luma, Cb and Cr are required by every codec but HapA, which reads alpha alone
    for codec in (HapB200Codec_Hap1, HapB200Codec_Hap5, HapB200Codec_HapY, HapB200Codec_HapM):
        for kw in ({"l": 0}, {"b": 0}, {"r": 0}):
            assert block(codec=codec, **kw) == BAD_ARGUMENTS and batch(codec=codec, **kw) == BAD_ARGUMENTS, (codec, kw)
        for kw in ({"l": None}, {"b": None}, {"r": None}):
            assert single(codec=codec, **kw) == BAD_ARGUMENTS, (codec, kw)
    assert block(blocks=0) == BAD_ARGUMENTS
    assert lib.encode_planar(luma, cb, cr, alpha, w, h, sub, n, 0, HapB200Codec_HapY, out=(0, cap), out_capacity=cap)[0] == BAD_ARGUMENTS
    # no frames, no output, chunk count 0, unknown compressor
    assert block(frames=0) == BAD_ARGUMENTS and batch(frames=0) == BAD_ARGUMENTS
    assert batch(out=0) == BAD_ARGUMENTS and batch(used_p=0) == BAD_ARGUMENTS
    assert batch(chunks=0) == BAD_ARGUMENTS and batch(comp=0xC1) == BAD_ARGUMENTS
    assert single(chunks=0) == BAD_ARGUMENTS and single(comp=0xC1) == BAD_ARGUMENTS
    # the batch rules: 16-byte aligned planes, pitches, frame stride, blocks and block stride
    for kw in ({"l": lum + 8}, {"b": cbp + 8}, {"r": crp + 8}, {"a": alp + 8}, {"fstride": fb + 8}, {"lpitch": lp + 8},
               {"cpitch": cp + 8}, {"blocks": base + 8}, {"bstride": 4096 + 8}):
        assert block(frames=2, codec=HapB200Codec_HapM, **kw) == BAD_ARGUMENTS, kw
    for kw in ({"l": lum + 8}, {"b": cbp + 8}, {"r": crp + 8}, {"a": alp + 8}, {"fstride": fb + 8}, {"lpitch": lp + 8},
               {"cpitch": cp + 8}):
        assert batch(frames=2, codec=HapB200Codec_HapM, **kw) == BAD_ARGUMENTS, kw
    assert block(frames=2, codec=HapB200Codec_HapA, a=alp + 8) == BAD_ARGUMENTS
    # below the HapB200MaxEncodedLengthRGBA bound
    for codec in CODECS:
        for k in (1, 3, 8):
            need = lib.max_encoded_length_rgba(w, h, codec, k)
            assert batch(codec=codec, chunks=k, out_stride=need - 1) == BUFFER_TOO_SMALL, (codec, k)
            assert single(codec=codec, chunks=k, cap_=need - 1) == BUFFER_TOO_SMALL, (codec, k)


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_planar_valid_arguments_fail_loudly_without_a_gpu(lib):
    w, h = 16, 8
    for sub in P.SUBSAMPLINGS:
        for n in P.DEPTHS:
            planes = P.random_planes(np.random.default_rng(0), w, h, sub, n)
            for codec in CODECS:
                assert lib.encode_planar(*planes, w, h, sub, n, Y.BT709_LIMITED, codec)[0] == INTERNAL_ERROR, (sub, n, codec)
            # Hap Alpha-Only reads alpha alone
            assert lib.encode_planar(None, None, None, planes[3], w, h, sub, n, 0, HapB200Codec_HapA)[0] == INTERNAL_ERROR
