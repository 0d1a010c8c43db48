"""Hap R (BC7) encoding without a GPU.  The oracle encoder (tests/bc7_oracle_encode.c: exhaustive over the 8 modes, every
partition, rotation, index selection and p-bit choice, least-squares endpoints and +-1 nudges) against Pillow's independent
decoder; the host build of the kernel's block encoder (tests/emu/bc7_encode_twin.cc) on constant and opaque blocks, its
reported errors, its modes and the quality bars against the oracle, a mode-6 baseline and this library's DXT5 encoder; and
the library's argument checks for the three BC7 encode entry points.

PSNR is 10 log10(255^2 / MSE), the MSE over R, G, B and A (bc7_encode_util.psnr).  Content: the synth.frame classes video,
gradient, texture and edges, opaque and with alpha="ramp", and noise opaque and with random alpha."""
import numpy as np
import pytest

import bc7_encode_util as E
import bc7_util as U
import hap_b200
import twin
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy
from hap_b200.lib import HapB200Codec_Hap7

BAD_ARGUMENTS, BUFFER_TOO_SMALL, INTERNAL_ERROR = 1, 2, 4
IDS = ["%s-%s" % c for c in E.CONTENT]
PER_ROW = 256   # blocks per block row of the constant pictures


def constant_picture(values: np.ndarray) -> np.ndarray:
    """one constant 4x4 block per RGBA value (n, 4), PER_ROW blocks per block row (the last value repeated to fill the last
    row) -> (4 rows, 4 PER_ROW, 4) uint8"""
    v = np.asarray(values, np.uint8)
    rows = -(-len(v) // PER_ROW)
    v = np.concatenate([v, np.repeat(v[-1:], rows * PER_ROW - len(v), axis=0)]).reshape(rows, PER_ROW, 4)
    return np.ascontiguousarray(np.repeat(np.repeat(v, 4, axis=0), 4, axis=1))


def corner_colours() -> np.ndarray:
    vals = [0, 1, 2, 127, 128, 129, 254, 255]
    return np.array([(r, g, b, a) for r in vals for g in vals for b in vals for a in (0, 255)], np.uint8)


# ---- the oracle encoder -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,alpha", E.CONTENT, ids=IDS)
def test_oracle_encoder_blocks_decode_in_pillow_as_in_the_oracle(kind, alpha):
    """Pillow's decoding of the oracle's blocks equals bc7_oracle_decode; no reserved block; the oracle's errors are its
    decoding's"""
    pytest.importorskip("PIL")
    w, h = 64, 32
    img = E.content(kind, alpha, w, h)
    blocks, errs = E.in_blocks(E.oracle_encode, img, rows=4)
    ours = U.oracle_decode(blocks, w, h)
    assert np.array_equal(U.pil_decode(blocks, w, h), ours)
    assert (E.block_modes(blocks) < 8).all()
    assert np.array_equal(E.block_errors(ours, img), errs)


def test_oracle_encoder_constant_and_opaque_blocks():
    rng = np.random.default_rng(3)
    v = np.concatenate([rng.integers(0, 256, (2000, 4)).astype(np.uint8), corner_colours()])
    img = constant_picture(v)
    blocks, errs = E.in_blocks(E.oracle_encode, img, rows=4)
    assert np.array_equal(U.oracle_decode(blocks, img.shape[1], img.shape[0]), img)
    assert (errs == 0).all()
    rnd = rng.integers(0, 256, (16, 64, 4)).astype(np.uint8)
    rnd[..., 3] = 255
    blocks, _ = E.in_blocks(E.oracle_encode, rnd, rows=4)
    assert (U.oracle_decode(blocks, 64, 16)[..., 3] == 255).all()


# ---- the kernel's block encoder on the host ---------------------------------------------------------------------------

def test_twin_constant_blocks_decode_bit_exactly():
    """10^5 random RGBA colours and the corner values (0, 1, 2, 127-129, 254, 255 per channel, A 0 and 255): each constant
    block decodes to its colour in the oracle decoder, the kernel decoder's twin and Pillow, with a chosen error of 0"""
    rng = np.random.default_rng(5)
    v = np.concatenate([rng.integers(0, 256, (100000, 4)).astype(np.uint8), corner_colours()])
    img = constant_picture(v)
    h, w = img.shape[:2]
    blocks, errs = E.in_blocks(E.twin_encode, img, rows=4)
    assert np.array_equal(U.oracle_decode(blocks, w, h), img)
    assert np.array_equal(U.twin_decode(blocks, w, h), img)
    assert (errs == 0).all()
    assert (E.block_modes(blocks) == 5).all()
    pytest.importorskip("PIL")
    assert np.array_equal(U.pil_decode(blocks, w, h), img)


@pytest.mark.parametrize("kind", [k for k, a in E.CONTENT if a == "opaque"])
def test_twin_opaque_content_decodes_opaque(kind):
    w, h = 128, 64
    img = E.content(kind, "opaque", w, h, 2)
    blocks, _ = E.in_blocks(E.twin_encode, img)
    assert (U.oracle_decode(blocks, w, h)[..., 3] == 255).all(), kind


def test_twin_random_opaque_blocks_decode_opaque():
    """random RGB with A = 255, and blocks with few colours or a single varying channel (which the rotations of modes 4 and 5
    and the p-bits of modes 6 and 7 would serve best without the rule)"""
    rng = np.random.default_rng(9)
    img = rng.integers(0, 256, (64, 256, 4)).astype(np.uint8)
    img[32:48] = img[32:48, :, :1]                          # grey: R = G = B = A before the alpha is set
    img[48:, :, :3] = rng.integers(0, 2, (16, 256, 3)).astype(np.uint8) * 255
    img[16:32, :, 1:3] = 77
    img[..., 3] = 255
    blocks, errs = E.in_blocks(E.twin_encode, img, rows=4)
    dec = U.oracle_decode(blocks, 256, 64)
    assert (dec[..., 3] == 255).all()
    assert np.array_equal(E.block_errors(dec, img), errs)


@pytest.mark.parametrize("kind,alpha", E.CONTENT, ids=IDS)
def test_twin_reports_the_error_of_the_block_it_emits(kind, alpha):
    """the error the twin chose each block by equals the error of the oracle's decoding of the emitted block; no reserved
    block; the kernel's own decoder agrees with the oracle on the blocks"""
    w, h = 64, 64
    img = E.content(kind, alpha, w, h, 1)
    blocks, errs = E.in_blocks(E.twin_encode, img)
    dec = U.oracle_decode(blocks, w, h)
    assert np.array_equal(E.block_errors(dec, img), errs)
    assert (E.block_modes(blocks) < 8).all()
    assert np.array_equal(U.twin_decode(blocks, w, h), dec)


def test_twin_random_bytes():
    rng = np.random.default_rng(77)
    img = rng.integers(0, 256, (32, 128, 4)).astype(np.uint8)
    blocks, errs = E.in_blocks(E.twin_encode, img, rows=4)
    dec = U.oracle_decode(blocks, 128, 32)
    assert np.array_equal(E.block_errors(dec, img), errs)
    assert (E.block_modes(blocks) < 8).all()


def test_the_search_is_live():
    """opaque edges get two- and three-subset blocks; alpha-ramp content gets blocks in modes 4-7"""
    w, h = 128, 64
    edges, _ = E.in_blocks(E.twin_encode, E.content("edges", "opaque", w, h))
    m = E.block_modes(edges)
    assert np.isin(m, [1, 3, 7]).any() and np.isin(m, [0, 2]).any()
    ramp, _ = E.in_blocks(E.twin_encode, E.content("video", "ramp", w, h))
    assert (E.block_modes(ramp) >= 4).any()


QUALITY = {}


@pytest.mark.parametrize("kind,alpha", E.CONTENT, ids=IDS)
def test_quality_against_the_oracle_the_baseline_and_dxt5(kind, alpha):
    """256x256 crops: twin PSNR >= oracle PSNR - 0.5 dB, >= the mode-6 baseline and >= this library's DXT5 (Hap Alpha)"""
    w = h = 256
    img = E.content(kind, alpha, w, h)
    tb, _ = E.in_blocks(E.twin_encode, img)
    ob, _ = E.in_blocks(E.oracle_encode, img)
    t = E.psnr(U.oracle_decode(tb, w, h), img)
    o = E.psnr(U.oracle_decode(ob, w, h), img)
    base = E.psnr(U.oracle_decode(E.baseline_encode(img), w, h), img)
    dxt5 = E.psnr(twin.decode("bc3", twin.encode("bc3", img), w, h), img)
    QUALITY[(kind, alpha)] = (t, o, base, dxt5)
    assert t >= o - 0.5, (t, o)
    assert t >= base, (t, base)
    assert t >= dxt5, (t, dxt5)


# ---- the library's argument checks ----------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def have_gpu():
    import torch
    return torch.cuda.is_available()


def test_encode_bc7_entry_points_refuse_bad_arguments(lib):
    w, h = 64, 32
    buf = np.zeros(4 * w * h * 4 + 64, np.uint8)
    p = (buf.ctypes.data + 15) // 16 * 16
    used = np.zeros(4, np.uint64)
    u = used.ctypes.data
    cap = lib.max_encoded_length_rgba(w, h, HapB200Codec_Hap7, 1)
    ostride = (cap + 15) // 16 * 16
    src = np.zeros(4 * w * h, np.uint8)
    fb = 4 * w * h
    # geometry: sizes not multiples of 4, empty, rowBytes < 4 * width, rowBytes >= 2^32
    for gw, gh, row in ((6, 4, 32), (4, 6, 16), (0, 4, 16), (4, 0, 16), (w, h, 4 * w - 16), (w, h, 1 << 32)):
        assert lib.block_encode_bc7_batch(p, 1, fb, gw, gh, p, 16 * 16 * 8, row_bytes=row) == BAD_ARGUMENTS
        assert lib.encode_rgba_bc7_batch(p, 1, fb, gw, gh, HapCompressorSnappy, 1, p, ostride, u, row_bytes=row) == BAD_ARGUMENTS
        if gw and gh and row < (1 << 32):
            assert lib.encode_rgba_bc7(src, gw, gh, row_bytes=row, out=bytearray(1 << 20), out_capacity=1 << 20)[0] == BAD_ARGUMENTS
    # null pointers, no frames, chunk count 0, unknown compressor
    assert lib.block_encode_bc7_batch(0, 1, fb, w, h, p, 2048) == BAD_ARGUMENTS
    assert lib.block_encode_bc7_batch(p, 1, fb, w, h, 0, 2048) == BAD_ARGUMENTS
    assert lib.block_encode_bc7_batch(p, 0, fb, w, h, p, 2048) == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7_batch(0, 1, fb, w, h, HapCompressorSnappy, 1, p, ostride, u) == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7_batch(p, 1, fb, w, h, HapCompressorSnappy, 1, 0, ostride, u) == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7_batch(p, 1, fb, w, h, HapCompressorSnappy, 1, p, ostride, 0) == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7_batch(p, 0, fb, w, h, HapCompressorSnappy, 1, p, ostride, u) == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7_batch(p, 1, fb, w, h, HapCompressorSnappy, 0, p, ostride, u) == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7_batch(p, 1, fb, w, h, 0xC1, 1, p, ostride, u) == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7((0, fb), w, h, out=bytearray(cap), out_capacity=cap)[0] == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7(src, w, h, out=(0, cap), out_capacity=cap)[0] == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7(src, w, h, chunks=0, out=bytearray(cap), out_capacity=cap)[0] == BAD_ARGUMENTS
    assert lib.encode_rgba_bc7(src, w, h, compressor=0xC1, out=bytearray(cap), out_capacity=cap)[0] == BAD_ARGUMENTS
    # the batch rules: 16-byte aligned rows, pictures, strides and blocks
    for args in ((p + 8, fb, 4 * w, p, 2048), (p, fb + 8, 4 * w, p, 2048), (p, fb, 4 * w + 8, p, 2048),
                 (p, fb, 4 * w, p + 8, 2048), (p, fb, 4 * w, p, 2048 + 8)):
        src_p, fstride, row, blocks, bstride = args
        assert lib.block_encode_bc7_batch(src_p, 2, fstride, w, h, blocks, bstride, row_bytes=row) == BAD_ARGUMENTS
    for args in ((p + 8, fb, 4 * w), (p, fb + 8, 4 * w), (p, fb, 4 * w + 8)):
        src_p, fstride, row = args
        assert lib.encode_rgba_bc7_batch(src_p, 2, fstride, w, h, HapCompressorSnappy, 1, p, ostride, u, row_bytes=row) == BAD_ARGUMENTS
    # below the HapB200MaxEncodedLengthRGBA(.., Hap7, ..) bound
    for k in (1, 3, 8):
        need = lib.max_encoded_length_rgba(w, h, HapB200Codec_Hap7, k)
        assert need > (w // 4) * (h // 4) * 16
        assert lib.encode_rgba_bc7_batch(p, 1, fb, w, h, HapCompressorSnappy, k, p, need - 1, u) == BUFFER_TOO_SMALL
        assert lib.encode_rgba_bc7(src, w, h, chunks=k, out=bytearray(need), out_capacity=need - 1)[0] == BUFFER_TOO_SMALL


@pytest.mark.skipif(have_gpu(), reason="only meaningful where there is no CUDA device")
def test_encode_bc7_valid_arguments_fail_loudly_without_a_gpu(lib):
    w, h = 16, 8
    src = np.zeros(4 * w * h, np.uint8)
    for comp in (HapCompressorNone, HapCompressorSnappy):
        assert lib.encode_rgba_bc7(src, w, h, compressor=comp)[0] == INTERNAL_ERROR
