"""Hap HDR (BC6H) decoding without a GPU.  The oracle (tests/bc6h_oracle.c) against Pillow's independent "bcn" decoder on
random blocks of every mode and signedness, on blocks whose values stay inside [0, 1], on every partition and on the
reserved modes; hand-computed blocks for the points of the BPTC specification a decoder can get wrong; the oracle's
partition table against the BC7 tables probed from Pillow; the host build of the kernel's block math
(tests/emu/bc6h_twin.cc) against the oracle, bit for bit; and the library's argument checks for the RGBA16F entry points.

Pillow differs from the specification in two places, and the comparisons account for both:
  * it truncates the interpolation, (a (64 - w) + b w) >> 6, where the specification adds 32 before the shift: the oracle
    is compared with Pillow at rounding 0, and used at the specification's 32 everywhere else;
  * in SF16 it takes the endpoints of the transformed modes as non-negative after the delta is added and wrapped, where the
    specification sign-extends them: the random SF16 blocks of those modes are drawn with wrapped endpoints whose sign
    bit is clear, and test_pillow_does_not_sign_extend_wrapped_sf16_endpoints pins the difference.
Pillow returns only uint8(clamp(value, 0, 1) * 255) of each half (bc6h_util.project8)."""
import numpy as np
import pytest

import bc6h_util as U
import bc7_util
import hap_b200
from hap_b200.abi import (HapCompressorNone, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT, HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT,
                          HapTextureFormat_RGBA_BPTC_UNORM, HapTextureFormat_RGBA_DXT5)

pytest.importorskip("PIL")
BAD_ARGUMENTS, BAD_FRAME = 1, 3
W = 4 * 128    # pictures of test blocks are W pixels wide
N = 1 << 14
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT
W3 = [0, 9, 18, 27, 37, 46, 55, 64]                                      # the specification's weight tables
W4 = [0, 4, 9, 13, 17, 21, 26, 30, 34, 38, 43, 47, 51, 55, 60, 64]


def picture(blocks: np.ndarray):
    n = len(blocks)
    assert n % (W // 4) == 0
    return blocks.tobytes(), W, 4 * n // (W // 4)


def texels(img: np.ndarray) -> np.ndarray:
    """(h, w, C) picture -> (blocks, 16, C), blocks row-major, texels row-major inside a block"""
    h, w = img.shape[:2]
    return img.reshape(h // 4, 4, w // 4, 4, -1).transpose(0, 2, 1, 3, 4).reshape(-1, 16, img.shape[-1])


def sext(v, n):
    v = np.asarray(v, np.int64) & ((1 << n) - 1)
    return np.where(v >> (n - 1), v - (1 << n), v)


def sf16_random_blocks(rng, n: int, m: int) -> np.ndarray:
    """n blocks of transformed mode m whose every field is random, except that each channel's base and deltas are redrawn
    until every base + delta, wrapped to the base's precision, has its sign bit clear"""
    md = U.mode(m)
    ep = np.zeros((n, 12), np.int64)
    ne, d = 2 * md.regions, md.delta
    for c in range(3):
        bad = np.ones(n, bool)
        while bad.any():
            k = int(bad.sum())
            ep[bad, c] = rng.integers(0, 1 << md.prec, k)
            for e in range(1, ne):
                ep[bad, 3 * e + c] = rng.integers(0, 1 << d[c], k)
            wrapped = [(sext(ep[:, 3 * e + c], d[c]) + ep[:, c]) & ((1 << md.prec) - 1) for e in range(1, ne)]
            bad = np.any([(x >> (md.prec - 1)) & 1 == 1 for x in wrapped], axis=0)
    partition = rng.integers(0, 32, n)
    idx = rng.integers(0, 1 << md.index_bits, (n, 16))
    idx[:, 0] >>= 1
    if md.regions == 2:
        idx[np.arange(n), U.tables()[1][partition]] >>= 1
    return U.pack_blocks(m, ep, partition, idx)


def check_oracle_against_pillow(blocks, signed):
    data, w, h = picture(blocks)
    ours = U.oracle_decode(data, w, h, signed, round=0)
    assert np.array_equal(U.project8(ours[..., :3]), U.pil_decode(data, w, h, signed))
    assert (ours[..., 3] == U.ONE).all()
    return ours


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
@pytest.mark.parametrize("mode", range(U.NMODES + len(U.RESERVED)))
def test_oracle_matches_pillow_on_random_blocks(mode, signed):
    """2^14 random blocks per mode and signedness (modes 14-17 here: the four reserved mode values), byte for byte"""
    rng = np.random.default_rng(1000 + 2 * mode + signed)
    transformed = mode < U.NMODES and U.mode(mode).transformed
    blocks = sf16_random_blocks(rng, N, mode) if signed and transformed else U.random_blocks(rng, N, mode)
    ours = check_oracle_against_pillow(blocks, signed)
    if mode >= U.NMODES:
        assert (ours[..., :3] == 0).all()


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
def test_oracle_matches_pillow_inside_the_unit_range(signed):
    """blocks of every mode whose values all lie in [0, 1], where Pillow's 8-bit projection clamps nothing"""
    rng = np.random.default_rng(7 + signed)
    for m in range(U.NMODES):
        blocks = U.unit_blocks(rng, 4096, m, signed)
        ours = check_oracle_against_pillow(blocks, signed)
        assert (ours[..., :3] <= U.ONE).all(), m


def test_oracle_matches_pillow_on_every_partition():
    rng = np.random.default_rng(11)
    for m in range(U.NMODES):
        md = U.mode(m)
        if md.regions != 2:
            continue
        b = U.random_blocks(rng, 32 * 64, m)
        part = np.repeat(np.arange(32), 64)
        hi = b.view("<u8")[:, 1]
        shift = np.uint64(md.header - 5 - 64)
        hi &= ~(np.uint64(31) << shift)
        hi |= part.astype(np.uint64) << shift
        check_oracle_against_pillow(b, False)


def test_pillow_does_not_sign_extend_wrapped_sf16_endpoints():
    """Mode 1, SF16: base 511 plus delta +1 wraps to 512 (10 bits), which the specification sign-extends to -512 (unquantised
    -0x7FFF, written as -65504 = 0xFBFF); Pillow takes it as +512 and writes 255.  Base 0 plus delta -1 wraps to 1023 = -1
    (-96 unquantised, 0x805D) where Pillow again saturates."""
    ep = np.zeros((2, 12), np.int64)
    ep[0, [0, 1, 2]], ep[0, [3, 4, 5]] = 511, 1             # r0 g0 b0 = 511, deltas +1
    ep[1, [3, 4, 5]] = 31                                  # deltas -1 (5 bits)
    idx = np.full((2, 16), 7)
    idx[:, 0], idx[:, 15] = 3, 3                           # texel 0 and partition 0's anchor store 2 bits
    blocks = U.pack_blocks(0, ep, np.zeros(2, np.int64), idx)
    ours = U.oracle_decode(np.concatenate([blocks, np.zeros((2, 16), np.uint8)]).tobytes(), 16, 4, True)
    t = texels(ours)
    assert (t[0, 1, :3] == 0xFBFF).all() and (t[1, 1, :3] == 0x805D).all()
    pil = texels(U.pil_decode(np.concatenate([blocks, np.zeros((2, 16), np.uint8)]).tobytes(), 16, 4, True))
    assert (pil[0, 1] == 255).all() and (pil[1, 1] == 255).all()


# ---- hand-computed blocks --------------------------------------------------------------------------------------------------

def decode_both(blocks: np.ndarray, signed: bool, round: int = 32):
    """blocks (k, 16), k <= 128 -> per-block texels (k, 16, 4) of the oracle, also checked against the twin"""
    k = len(blocks)
    pad = np.zeros((W // 4 - k, 16), np.uint8)
    data, w, h = picture(np.concatenate([blocks, pad]))
    ours = U.oracle_decode(data, w, h, signed, round)
    if round == 32:
        assert np.array_equal(ours, U.twin_decode(data, w, h, signed))
    return texels(ours)[:k]


def test_interpolation_rounds_with_plus_32():
    """Mode 11 (UF16): endpoints 0 and 2 (unquantised 0 and 160), weight 9 (index 2): (160 * 9 + 32) >> 6 = 23 -> 23 * 31 >> 6
    = 11; truncating gives 22 -> 10"""
    ep = np.zeros((1, 12), np.int64)
    ep[0, 3:6] = 2
    b = U.pack_blocks(10, ep, np.zeros(1, np.int64), np.full((1, 16), 2))
    assert (decode_both(b, False)[0, :, :3] == 11).all()
    assert (decode_both(b, False, round=0)[0, :, :3] == 10).all()


def test_weight_tables_3_and_4_bit():
    """Mode 11 (4-bit indices, one region) and mode 10 (3-bit, two regions): every index of the table between a zero and a
    large endpoint, checked against the specification's weights"""
    unq = lambda v, p: ((v << 16) + 0x8000) >> p
    ep = np.zeros((1, 12), np.int64)
    ep[0, 3:6] = 1022
    idx = np.arange(16)[None, :].copy()
    idx[0, 0] = 0
    got = decode_both(U.pack_blocks(10, ep, np.zeros(1, np.int64), idx), False)[0, :, 0]
    assert list(got) == [((unq(1022, 10) * W4[i] + 32) >> 6) * 31 >> 6 for i in idx[0]]
    ep = np.zeros((1, 12), np.int64)
    ep[0, 3:6], ep[0, 6:9], ep[0, 9:12] = 62, 61, 0        # region 0: 0 .. 62, region 1: 61 .. 0 (partition 0)
    idx = (np.arange(16) % 8)[None, :].copy()
    idx[0, 0], idx[0, 15] = 0, 3
    got = decode_both(U.pack_blocks(9, ep, np.zeros(1, np.int64), idx), False)[0, :, 0]
    part = U.tables()[0][0]
    for t in range(16):
        a, b = (0, unq(62, 6)) if part[t] == 0 else (unq(61, 6), 0)
        w = W3[idx[0, t]]
        assert got[t] == ((a * (64 - w) + b * w + 32) >> 6) * 31 >> 6, t


def test_unquantisation_at_zero_and_the_largest_values():
    """Every mode, the base endpoint at 0 and at its extremes: UF16 0 -> 0, 2^p - 1 -> 0x7BFF; SF16 0 -> 0, 2^(p-1) - 1 ->
    0x7BFF, -(2^(p-1) - 1) and -2^(p-1) -> 0xFBFF (no -Inf)"""
    for m in range(U.NMODES):
        md = U.mode(m)
        p = md.prec
        for signed, values, want in ((False, [0, (1 << p) - 1], [0, 0x7BFF]),
                                     (True, [0, (1 << (p - 1)) - 1, -((1 << (p - 1)) - 1), -(1 << (p - 1))], [0, 0x7BFF, 0xFBFF, 0xFBFF])):
            ep = np.zeros((len(values), 12), np.int64)
            for c in range(3):
                ep[:, c] = np.array(values) & ((1 << p) - 1)
                if not md.transformed:
                    ep[:, 3 * 1 + c] = ep[:, c]
            got = decode_both(U.pack_blocks(m, ep, np.zeros(len(values), np.int64), np.zeros((len(values), 16), np.int64)), signed)
            for k, wv in enumerate(want):
                assert (got[k, 0, :3] == wv).all(), (m + 1, signed, values[k], got[k, 0])


def test_transformed_endpoints_wrap():
    """Mode 1 (UF16): base 1023 + delta 1 wraps to 0; base 0 + delta -1 wraps to 1023 (-> 0x7BFF); base 5 + 3 = 8 ->
    (8 << 16 | 0x8000) >> 10 = 544 -> 544 * 31 >> 6 = 263.  SF16: base 511 + 1 wraps to -512 -> 0xFBFF."""
    ep = np.zeros((2, 12), np.int64)
    ep[0, 0:3] = [1023, 0, 5]
    ep[0, 3:6] = [1, 31, 3]
    ep[1, 0:3], ep[1, 3:6] = 511, 1
    idx = np.full((2, 16), 7)
    idx[:, 0], idx[:, 15] = 3, 3
    b = U.pack_blocks(0, ep, np.zeros(2, np.int64), idx)
    assert list(decode_both(b[:1], False)[0, 1, :3]) == [0, 0x7BFF, 263]
    assert list(decode_both(b[1:], True)[0, 1, :3]) == [0xFBFF] * 3


def test_negative_values_that_scale_to_zero_are_plus_zero():
    """Mode 14, SF16, both endpoints -1 (16 bits, unquantised as they are): (-1 * 64 + 32) >> 6 = -1, magnitude 1 * 31 >> 5 = 0:
    written +0 (0x0000), never -0; -2 gives -1 in the half's bits (0x8001)"""
    ep = np.zeros((2, 12), np.int64)
    ep[0, 0:3], ep[1, 0:3] = 0xFFFF, 0xFFFE                 # deltas 0: both endpoints equal the base
    got = decode_both(U.pack_blocks(13, ep, np.zeros(2, np.int64), np.zeros((2, 16), np.int64)), True)
    assert (got[0, :, :3] == 0).all() and (got[1, :, :3] == 0x8001).all()


def test_reserved_modes_decode_to_black_with_alpha_one():
    rng = np.random.default_rng(5)
    for k in range(len(U.RESERVED)):
        got = decode_both(U.random_blocks(rng, 64, U.NMODES + k), bool(k & 1))
        assert (got[..., :3] == 0).all() and (got[..., 3] == U.ONE).all()


def test_no_output_is_inf_or_nan():
    rng = np.random.default_rng(6)
    b = rng.integers(0, 256, (N, 16), dtype=np.uint8)
    for signed in (False, True):
        data, w, h = picture(b)
        out = U.oracle_decode(data, w, h, signed)
        assert ((out & 0x7C00) != 0x7C00).all()


# ---- the kernel's tables and block math ------------------------------------------------------------------------------------

def test_partition_tables_equal_the_first_32_bc7_partitions_probed_from_pillow():
    masks, maps = bc7_util.probe_partitions()
    two, _ = bc7_util.probe_anchors(masks, maps)
    part, anchor = U.tables()
    assert [sum(int(part[p, t]) << t for t in range(16)) for p in range(32)] == masks[:32]
    assert list(anchor) == two[:32]
    kpart, kanchor = U.twin_tables()
    assert kpart == [sum(((m >> t) & 1) << (2 * t) for t in range(16)) for m in masks[:32]]
    assert kanchor == [1 | (1 << a) for a in two[:32]]


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
def test_kernel_block_decoder_source_is_bit_exact_against_oracle(signed):
    """The block math the kernel compiles (bc6h_decode.cuh), built for the host, on full-range random blocks of every mode
    and the reserved ones, uniform random bytes, blocks inside [0, 1] and picture-like blocks: every 16-bit output equal"""
    from hap_b200 import synth
    rng = np.random.default_rng(20 + signed)
    sets = [U.random_blocks(rng, N, m) for m in range(U.NMODES + len(U.RESERVED))]
    sets.append(rng.integers(0, 256, (N, 16), dtype=np.uint8))
    sets += [U.unit_blocks(rng, 1024, m, signed) for m in range(U.NMODES)]
    pic = synth.frame(W, 64, 0, kind="video").numpy()
    sets.append(np.frombuffer(U.pack_picture(pic, signed), np.uint8).reshape(-1, 16))
    for blocks in sets:
        data, w, h = picture(blocks)
        assert np.array_equal(U.twin_decode(data, w, h, signed), U.oracle_decode(data, w, h, signed))


def test_picture_packer_follows_its_picture():
    from hap_b200 import synth
    pic = synth.frame(256, 128, 1, kind="video").numpy()
    for signed in (False, True):
        dec = U.oracle_decode(U.pack_picture(pic, signed), 256, 128, signed)[..., :3].view(np.float16).astype(np.float64)
        want = (pic[..., :3] / 255.0) ** 2.2 * 4.0
        assert np.corrcoef(dec.ravel(), want.ravel())[0, 1] > 0.95 and dec.max() > 1.0


# ---- the library without a GPU ------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def test_half_entry_points_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(16 * w * h + 64, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    res = np.zeros(4, np.uint32)
    nbytes = np.zeros(4, np.uint64)
    frame = lib.encode([bytes((w // 4) * (h // 4) * 16)], [UF16], [HapCompressorNone], [1])[1]
    for fmt in (UF16, SF16):
        for gw, gh, row in ((6, 4, 48), (4, 6, 32), (0, 4, 32), (w, h, 4 * w), (w, h, 8 * w - 16), (w, h, 1 << 32)):
            assert lib.block_decode_half_batch(p, 1, 16 * 16 * 8, gw, gh, fmt, p, 8 * w * h, row_bytes=row) == BAD_ARGUMENTS
            assert lib.decode_rgba_half_batch(p, 1, 1024, nbytes.ctypes.data, 1, gw, gh, p, 8 * w * h, res.ctypes.data,
                                              row_bytes=row) == BAD_ARGUMENTS
            if gw and row < (1 << 32):
                assert lib.decode_rgba_half(frame, gw, gh, out=buf, row_bytes=row)[0] == BAD_ARGUMENTS
        # the batch rules: 16-byte aligned rows, pictures and strides, a frame at all
        for args in ((p, 1, 16, p + 8, 8 * w * h, 8 * w), (p, 1, 16, p, 8 * w * h + 8, 8 * w), (p, 1, 16, p, 8 * w * h, 8 * w + 8),
                     (p + 8, 1, 16, p, 8 * w * h, 8 * w), (p, 1, 24, p, 8 * w * h, 8 * w), (p, 0, 16, p, 8 * w * h, 8 * w)):
            blocks, frames, bstride, out, fstride, row = args
            assert lib.block_decode_half_batch(blocks, frames, bstride, w, h, fmt, out, fstride, row_bytes=row) == BAD_ARGUMENTS
    for fmt in (0, HapTextureFormat_RGBA_BPTC_UNORM, HapTextureFormat_RGBA_DXT5, UF16 + 1, SF16 - 1):
        assert lib.block_decode_half_batch(p, 1, 16, w, h, fmt, p, 8 * w * h) == BAD_ARGUMENTS
    assert lib.decode_rgba_half_batch(p, 1, 1024, nbytes.ctypes.data, 0, w, h, p, 8 * w * h, res.ctypes.data) == BAD_ARGUMENTS
    assert lib.decode_rgba_half_batch(p, 1, 1024, nbytes.ctypes.data, 1, w, h, p, 8 * w * h, 0) == BAD_ARGUMENTS


def test_half_decoder_refuses_frames_of_other_flavours_from_their_headers(lib):
    """HapB200DecodeRGBAHalf answers Bad_Frame for a frame that is not one BC6H texture before it touches a GPU"""
    w, h = 16, 8
    n = (w // 4) * (h // 4) * 16
    for fmt in (HapTextureFormat_RGBA_DXT5, HapTextureFormat_RGBA_BPTC_UNORM):
        r, frame = lib.encode([bytes(n)], [fmt], [HapCompressorNone], [1])
        assert r == 0
        assert lib.decode_rgba_half(frame, w, h)[0] == BAD_FRAME
