"""Hap HDR (BC6H) encoding without a GPU.  The oracle encoder (tests/bc6h_oracle_encode.c: exhaustive over the 14 modes and 32
partitions, least-squares endpoints and +-1 nudges) against Pillow's independent decoder; the host build of the kernel's
block encoder (tests/emu/bc6h_encode_twin.cc) on constant blocks, the input rules, its reported errors, its modes and the
quality bars against the oracle and a mode-11 baseline; and the library's argument checks for the three encode entry
points.

PSNR16 is 10 log10(0x7BFF^2 / MSE), the MSE over R, G and B of the sign-magnitude integers of the decoded and the clamped
source halves (bc6h_encode_util.psnr16).  Content: the synth.frame classes made linear, (v / 255)^2.2 x peak with peak 1 and 64,
for SF16 centred on zero, and an exposure ramp from 2^-12 to 2^15 (bc6h_encode_util.hdr_content, exposure_ramp)."""
import numpy as np
import pytest

import bc6h_encode_util as E
import bc6h_util as U
import hap_b200
from hap_b200.abi import (HapCompressorNone, HapCompressorSnappy, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT,
                          HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGBA_BPTC_UNORM, HapTextureFormat_RGBA_DXT5)

BAD_ARGUMENTS, BUFFER_TOO_SMALL, INTERNAL_ERROR = 1, 2, 4
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT
CONTENT = [(k, p) for k in E.CLASSES for p in (1.0, 64.0)] + [("ramp", 0.0)]


def content(kind, peak, w, h, signed, index=0):
    return E.exposure_ramp(w, h, signed) if kind == "ramp" else E.hdr_content(kind, w, h, peak, signed, index)


PER_ROW = 256   # blocks per block row of the constant pictures


def constant_picture(values: np.ndarray) -> np.ndarray:
    """one constant 4x4 block per value (n, 3) binary16 bits, PER_ROW blocks per block row (the last value repeated to fill
    the last row) -> (4 rows, 4 PER_ROW, 4)"""
    v = np.asarray(values, np.uint16)
    rows = -(-len(v) // PER_ROW)
    v = np.concatenate([v, np.repeat(v[-1:], rows * PER_ROW - len(v), axis=0)]).reshape(rows, PER_ROW, 3)
    img = np.empty((4 * rows, 4 * PER_ROW, 4), np.uint16)
    img[..., :3] = np.repeat(np.repeat(v, 4, axis=0), 4, axis=1)
    img[..., 3] = U.ONE
    return img


def block_texels(img: np.ndarray) -> np.ndarray:
    """(h, w, C) -> (blocks, 16, C), blocks row-major"""
    h, w = img.shape[:2]
    return img.reshape(h // 4, 4, w // 4, 4, -1).transpose(0, 2, 1, 3, 4).reshape(-1, 16, img.shape[-1])


def assert_constant_blocks(blocks, img, values, signed, decode):
    got = block_texels(decode(blocks, img.shape[1], img.shape[0], signed)[..., :3])[: len(values)]
    assert np.array_equal(got, np.repeat(rule_bits(values, signed)[:, None, :], 16, axis=1))


def rule_bits(values: np.ndarray, signed: bool) -> np.ndarray:
    """the binary16 bits each value must decode to after the input rules"""
    x = E.source_values(values[None], signed)[0]
    return np.where(x < 0, 0x8000 | -x, x).astype(np.uint16)


def specials(signed: bool) -> np.ndarray:
    sub = [0x0001, 0x0002, 0x01FF, 0x03FF, 0x8001, 0x83FF]
    vals = [0x0000, 0x8000, 0x7BFF, 0xFBFF, 0x7C00, 0xFC00, 0x7C01, 0x7E00, 0xFFFF, 0x3C00, 0xBC00, 0x0400] + sub
    v = np.array(vals, np.uint16)
    return np.stack([v, np.roll(v, 1), np.roll(v, 2)], 1)


# ---- the oracle encoder -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", E.CLASSES)
def test_oracle_encoder_blocks_decode_in_pillow_as_in_the_oracle(kind):
    """UF16 content inside [0, 1]: Pillow's 8-bit decoding of the oracle's blocks equals the oracle's decoding at rounding 0"""
    pytest.importorskip("PIL")
    w, h = 64, 32
    img = E.hdr_content(kind, w, h, 1.0)
    blocks, _ = E.in_blocks(E.oracle_encode, img, False)
    ours = U.oracle_decode(blocks, w, h, False, round=0)
    assert np.array_equal(U.project8(ours[..., :3]), U.pil_decode(blocks, w, h, False))
    assert set(E.block_modes(blocks).tolist()) - set(range(U.NMODES)) == set()


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
def test_oracle_encoder_constant_blocks_and_input_rules(signed):
    rng = np.random.default_rng(11 + signed)
    n = 3000
    v = rng.integers(0, 0x7C00, (n, 3)) | (rng.integers(0, 2, (n, 3)) << 15)
    v = np.concatenate([v.astype(np.uint16), specials(signed)])
    img = constant_picture(v)
    blocks, errs = E.in_blocks(E.oracle_encode, img, signed, rows=4)
    assert_constant_blocks(blocks, img, v, signed, U.oracle_decode)
    assert (errs == 0).all()


# ---- the kernel's block encoder on the host ---------------------------------------------------------------------------

@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
def test_twin_constant_blocks_decode_bit_exactly(signed):
    """10^5 random finite halves, then +-0, subnormals, +-65504, NaN and +-Inf: each constant block decodes to its colour
    after the input rules, with a chosen error of 0"""
    rng = np.random.default_rng(5 + signed)
    n = 100000
    mag = rng.integers(0, 0x7C00, (n, 3))
    v = (mag | (rng.integers(0, 2, (n, 3)) << 15)).astype(np.uint16)
    v = np.concatenate([v, specials(signed)])
    img = constant_picture(v)
    blocks, errs = E.in_blocks(E.twin_encode, img, signed, rows=4)
    assert_constant_blocks(blocks, img, v, signed, U.oracle_decode)
    assert_constant_blocks(blocks, img, v, signed, U.twin_decode)
    assert (errs == 0).all()
    assert (E.block_modes(blocks) >= 0).all()


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
def test_twin_reports_the_error_of_the_block_it_emits(signed):
    """the error the twin chose each block by equals the error of the oracle's decoding of the emitted block (delta ranges,
    wraps and packing); no reserved mode; the kernel's own decoder agrees with the oracle on the blocks"""
    w, h = 64, 64
    for i, (kind, peak) in enumerate(CONTENT):
        img = content(kind, peak, w, h, signed, i)
        blocks, errs = E.in_blocks(E.twin_encode, img, signed)
        dec = U.oracle_decode(blocks, w, h, signed)
        assert np.array_equal(E.block_errors(dec, img, signed), errs), kind
        assert (E.block_modes(blocks) >= 0).all(), kind
        assert np.array_equal(U.twin_decode(blocks, w, h, signed), dec), kind


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
def test_twin_random_halves_and_specials(signed):
    """random bit patterns (NaN, Inf, negatives, subnormals among them): the reported error is the decoded one against
    the input rules, and no reserved mode"""
    rng = np.random.default_rng(77 + signed)
    img = rng.integers(0, 1 << 16, (32, 64, 4)).astype(np.uint16)
    blocks, errs = E.twin_encode(img, signed)
    dec = U.oracle_decode(blocks, 64, 32, signed)
    assert np.array_equal(E.block_errors(dec, img, signed), errs)
    assert (E.block_modes(blocks) >= 0).all()


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
def test_the_search_is_live(signed):
    """edges get two-region modes on some blocks; the smooth regions of video content get the transformed one-region modes
    (12-14)"""
    w, h = 128, 64
    edges, _ = E.in_blocks(E.twin_encode, E.hdr_content("edges", w, h, 64.0, signed), signed)
    assert (E.block_modes(edges) < 10).any()
    smooth, _ = E.in_blocks(E.twin_encode, E.hdr_content("video", w, h, 1.0, signed), signed)
    assert np.isin(E.block_modes(smooth), [11, 12, 13]).any()


QUALITY = {}


@pytest.mark.parametrize("signed", [False, True], ids=["UF16", "SF16"])
@pytest.mark.parametrize("kind,peak", CONTENT, ids=["%s-%g" % c for c in CONTENT])
def test_quality_against_the_oracle_and_the_baseline(kind, peak, signed):
    """256x256 crops: twin PSNR16 >= oracle PSNR16 - 0.5 dB, and >= the mode-11 min / max baseline"""
    w = h = 256
    img = content(kind, peak, w, h, signed)
    tb, _ = E.in_blocks(E.twin_encode, img, signed)
    ob, _ = E.in_blocks(E.oracle_encode, img, signed)
    twin = E.psnr16(U.oracle_decode(tb, w, h, signed), img, signed)
    oracle = E.psnr16(U.oracle_decode(ob, w, h, signed), img, signed)
    base = E.psnr16(U.oracle_decode(E.baseline_encode(img, signed), w, h, signed), img, signed)
    QUALITY[(kind, peak, signed)] = (twin, oracle, base)
    assert twin >= oracle - 0.5, (twin, oracle)
    assert twin >= base, (twin, base)


# ---- the library's argument checks ----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def test_encode_half_entry_points_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(8 * w * h * 4 + 64, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    used = np.zeros(4, np.uint64)
    u = used.ctypes.data
    cap = lib.max_encoded_length_half(w, h, UF16, 1)
    ostride = (cap + 15) // 16 * 16
    src = np.zeros(8 * w * h, np.uint8)
    for fmt in (0, HapTextureFormat_RGBA_BPTC_UNORM, HapTextureFormat_RGBA_DXT5, UF16 + 1, SF16 - 1):
        assert lib.block_encode_half_batch(p, 1, 8 * w * h, w, h, fmt, p, 16 * 16 * 8) == BAD_ARGUMENTS
        assert lib.encode_rgba_half_batch(p, 1, 8 * w * h, w, h, fmt, HapCompressorSnappy, 1, p, ostride, u) == BAD_ARGUMENTS
        assert lib.encode_rgba_half(src, w, h, fmt, out_capacity=1 << 20, out=bytearray(1 << 20))[0] == BAD_ARGUMENTS
    for fmt in (UF16, SF16):
        # geometry: sizes not multiples of 4, empty, rowBytes < 8 * width, rowBytes >= 2^32
        for gw, gh, row in ((6, 4, 48), (4, 6, 32), (0, 4, 32), (w, h, 4 * w), (w, h, 8 * w - 16), (w, h, 1 << 32)):
            assert lib.block_encode_half_batch(p, 1, 8 * w * h, gw, gh, fmt, p, 16 * 16 * 8, row_bytes=row) == BAD_ARGUMENTS
            assert lib.encode_rgba_half_batch(p, 1, 8 * w * h, gw, gh, fmt, HapCompressorSnappy, 1, p, ostride, u,
                                              row_bytes=row) == BAD_ARGUMENTS
            if gw and row < (1 << 32):
                assert lib.encode_rgba_half(src, gw, gh, fmt, row_bytes=row, out=bytearray(1 << 20),
                                            out_capacity=1 << 20)[0] == BAD_ARGUMENTS
        # null pointers, no frames, chunk count 0, unknown compressor
        assert lib.block_encode_half_batch(0, 1, 8 * w * h, w, h, fmt, p, 4096) == BAD_ARGUMENTS
        assert lib.block_encode_half_batch(p, 1, 8 * w * h, w, h, fmt, 0, 4096) == BAD_ARGUMENTS
        assert lib.block_encode_half_batch(p, 0, 8 * w * h, w, h, fmt, p, 4096) == BAD_ARGUMENTS
        assert lib.encode_rgba_half_batch(0, 1, 8 * w * h, w, h, fmt, HapCompressorSnappy, 1, p, ostride, u) == BAD_ARGUMENTS
        assert lib.encode_rgba_half_batch(p, 1, 8 * w * h, w, h, fmt, HapCompressorSnappy, 1, 0, ostride, u) == BAD_ARGUMENTS
        assert lib.encode_rgba_half_batch(p, 1, 8 * w * h, w, h, fmt, HapCompressorSnappy, 1, p, ostride, 0) == BAD_ARGUMENTS
        assert lib.encode_rgba_half_batch(p, 0, 8 * w * h, w, h, fmt, HapCompressorSnappy, 1, p, ostride, u) == BAD_ARGUMENTS
        assert lib.encode_rgba_half_batch(p, 1, 8 * w * h, w, h, fmt, HapCompressorSnappy, 0, p, ostride, u) == BAD_ARGUMENTS
        assert lib.encode_rgba_half_batch(p, 1, 8 * w * h, w, h, fmt, 0xC1, 1, p, ostride, u) == BAD_ARGUMENTS
        assert lib.encode_rgba_half((0, 8 * w * h), w, h, fmt, out=bytearray(cap), out_capacity=cap)[0] == BAD_ARGUMENTS
        assert lib.encode_rgba_half(src, w, h, fmt, out=(0, cap), out_capacity=cap)[0] == BAD_ARGUMENTS
        assert lib.encode_rgba_half(src, w, h, fmt, chunks=0, out=bytearray(cap), out_capacity=cap)[0] == BAD_ARGUMENTS
        assert lib.encode_rgba_half(src, w, h, fmt, compressor=0xC1, out=bytearray(cap), out_capacity=cap)[0] == BAD_ARGUMENTS
        # the batch rules: 16-byte aligned rows, pictures, strides, blocks and output
        for args in ((p + 8, 8 * w * h, 8 * w, p, 4096), (p, 8 * w * h + 8, 8 * w, p, 4096), (p, 8 * w * h, 8 * w + 8, p, 4096),
                     (p, 8 * w * h, 8 * w, p + 8, 4096), (p, 8 * w * h, 8 * w, p, 4096 + 8)):
            src_p, fstride, row, blocks, bstride = args
            assert lib.block_encode_half_batch(src_p, 2, fstride, w, h, fmt, blocks, bstride, row_bytes=row) == BAD_ARGUMENTS
        for args in ((p + 8, 8 * w * h, 8 * w, p, ostride), (p, 8 * w * h + 8, 8 * w, p, ostride), (p, 8 * w * h, 8 * w + 8, p, ostride),
                     (p, 8 * w * h, 8 * w, p + 8, ostride), (p, 8 * w * h, 8 * w, p, ostride + 8)):
            src_p, fstride, row, out, os_ = args
            assert lib.encode_rgba_half_batch(src_p, 2, fstride, w, h, fmt, HapCompressorSnappy, 1, out, os_, u,
                                              row_bytes=row) == BAD_ARGUMENTS
        # below the HapMaxEncodedLength bound
        for k in (1, 3, 8):
            need = lib.max_encoded_length([(w // 4) * (h // 4) * 16], [fmt], [k])
            assert need == lib.max_encoded_length_half(w, h, fmt, k) and need > (w // 4) * (h // 4) * 16
            short = (need - 1) // 16 * 16
            assert lib.encode_rgba_half_batch(p, 1, 8 * w * h, w, h, fmt, HapCompressorSnappy, k, p, short, u) == BUFFER_TOO_SMALL
            assert lib.encode_rgba_half(src, w, h, fmt, chunks=k, out=bytearray(need), out_capacity=need - 1)[0] == BUFFER_TOO_SMALL


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_encode_half_valid_arguments_fail_loudly_without_a_gpu(lib):
    w, h = 16, 8
    src = np.zeros(8 * w * h, np.uint8)
    for fmt in (UF16, SF16):
        for comp in (HapCompressorNone, HapCompressorSnappy):
            assert lib.encode_rgba_half(src, w, h, fmt, compressor=comp)[0] == INTERNAL_ERROR
