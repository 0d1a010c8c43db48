"""Hap R (BC7) decoding without a GPU: the oracle's BC7 decoder against Pillow's independent "bcn" decoder on random
blocks of every mode, every partition, rotation and index selection; the partition and anchor tables the kernel compiles
against the ones Pillow reveals by probing; the host build of the kernel's block decoder against the oracle; and the
library's sizes and refusals for the Hap7 codec.  (The oracle is tests/bc7_oracle.c, the host build tests/emu/bc7_twin.cc.)"""
import numpy as np
import pytest

import bc7_util as U
import hap_b200
import hap_b200.lib as L
import oracles
from hap_b200.abi import (HapCompressorNone, HapCompressorSnappy, HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT,
                          HapTextureFormat_RGBA_BPTC_UNORM)

pytest.importorskip("PIL")
BAD_ARGUMENTS, BAD_FRAME = 1, 3
W = 4 * 128    # pictures of test blocks are W pixels wide


def set_field(blocks: np.ndarray, pos: int, n: int, value) -> np.ndarray:
    """blocks (k, 16) with bits pos .. pos+n-1 (inside the first 64) set to value (scalar or per block)"""
    b = np.ascontiguousarray(blocks).copy()
    lo = b.view("<u8")[:, 0]
    mask = np.uint64(((1 << n) - 1) << pos)
    lo &= ~mask
    lo |= (np.asarray(value, np.uint64) << np.uint64(pos)) & mask
    return b


def picture(blocks: np.ndarray):
    """(k, 16) blocks, k a multiple of W/4 -> (bytes, w, h)"""
    n = len(blocks)
    assert n % (W // 4) == 0
    return blocks.tobytes(), W, 4 * n // (W // 4)


def per_mode_blocks(seed=1, n=1 << 14):
    rng = np.random.default_rng(seed)
    return {m: U.random_blocks(rng, n, m) for m in range(9)}


def partition_blocks(seed=2, per=64):
    """every partition of modes 0, 1, 2, 3, 7 (per blocks each, the rest of the block random)"""
    rng = np.random.default_rng(seed)
    out = {}
    for mode in (0, 1, 2, 3, 7):
        pb = U.MODES[mode][1]
        b = U.random_blocks(rng, per << pb, mode)
        out[mode] = set_field(b, mode + 1, pb, np.repeat(np.arange(1 << pb), per))
    return out


def rotation_blocks(seed=3, per=2048):
    """every rotation of modes 4 and 5, with both index selections of mode 4"""
    rng = np.random.default_rng(seed)
    out = {}
    for mode in (4, 5):
        sels = (0, 1) if mode == 4 else (0,)
        for rot in range(4):
            for sel in sels:
                b = set_field(U.random_blocks(rng, per, mode), mode + 1, 2, rot)
                if mode == 4:
                    b = set_field(b, mode + 3, 1, sel)
                out[(mode, rot, sel)] = b
    return out


def check_oracle_against_pillow(blocks):
    data, w, h = picture(blocks)
    ours = U.oracle_decode(data, w, h)
    theirs = U.pil_decode(data, w, h)
    reserved = np.repeat(U.mode_of(blocks) == 8, 16).reshape(h // 4, w // 4, 4, 4).transpose(0, 2, 1, 3).reshape(h, w)
    assert np.array_equal(ours[~reserved], theirs[~reserved])
    assert (ours[reserved] == 0).all()
    return ours


@pytest.mark.parametrize("mode", range(9))
def test_oracle_matches_pillow_on_random_blocks_of_each_mode(mode):
    """2^14 random blocks per mode, byte-exact; reserved blocks (mode 8 here) are (0, 0, 0, 0) where Pillow gives A = 255"""
    blocks = per_mode_blocks()[mode]
    ours = check_oracle_against_pillow(blocks)
    if mode == 8:
        data, w, h = picture(blocks)
        assert (U.pil_decode(data, w, h)[..., :3] == 0).all() and (ours == 0).all()


def test_oracle_matches_pillow_on_every_partition():
    for mode, blocks in partition_blocks().items():
        check_oracle_against_pillow(blocks)


def test_oracle_matches_pillow_on_every_rotation_and_index_selection():
    for key, blocks in rotation_blocks().items():
        check_oracle_against_pillow(blocks)


def test_probed_partition_and_anchor_tables_equal_the_kernels_tables():
    masks, maps = U.probe_partitions()
    assert masks[:4] == [0xCCCC, 0x8888, 0xEEEE, 0xECC8]
    two, three = U.probe_anchors(masks, maps)
    part2, part3, anch2, anch3 = U.twin_tables()
    assert part2 == [sum(((m >> t) & 1) << (2 * t) for t in range(16)) for m in masks]
    assert part3 == [sum(s << (2 * t) for t, s in enumerate(mp)) for mp in maps]
    assert anch2 == [1 | (1 << a) for a in two]
    assert anch3 == [1 | (1 << a) | (1 << b) for a, b in three]


def test_kernel_block_decoder_source_is_bit_exact_against_oracle():
    """The BC7 block math the kernel compiles (bc7_decode.cuh), built for the host, on every block set above, on mode-6
    picture-like blocks and on uniform random bytes (all modes mixed, reserved blocks included)."""
    from hap_b200 import synth
    sets = list(per_mode_blocks().values()) + list(partition_blocks().values()) + list(rotation_blocks().values())
    sets.append(np.random.default_rng(4).integers(0, 256, (1 << 14, 16), dtype=np.uint8))
    pic = synth.frame(W, 64, 0, kind="video", alpha="ramp").numpy()
    sets.append(np.frombuffer(U.pack_picture(pic), np.uint8).reshape(-1, 16))
    for blocks in sets:
        data, w, h = picture(blocks)
        assert np.array_equal(U.twin_decode(data, w, h), U.oracle_decode(data, w, h))


def test_picture_packer_is_close_to_its_picture():
    from hap_b200 import synth
    pic = synth.frame(256, 128, 1, kind="video", alpha="ramp").numpy()
    dec = U.oracle_decode(U.pack_picture(pic), 256, 128)
    assert oracles.psnr(pic, dec, channels=(0, 1, 2, 3)) > 25.0


# ---- the library without a GPU ------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def test_hap7_sizes(lib):
    assert L.HapB200Codec_Hap7 == 5
    for w, h in ((4, 4), (1920, 1080), (3840, 2160), (1924, 1084)):
        n = (w // 4) * (h // 4) * 16
        assert lib.texture_bytes(w, h, L.HapB200Codec_Hap7, 0) == n
        assert lib.texture_bytes(w, h, L.HapB200Codec_Hap7, 1) == 0
        for chunks in (1, 4, 8):
            want = lib.max_encoded_length([n], [HapTextureFormat_RGBA_BPTC_UNORM], [chunks])
            assert want > n and lib.max_encoded_length_rgba(w, h, L.HapB200Codec_Hap7, chunks) == want
            assert want == lib.max_encoded_length_rgba(w, h, L.HapB200Codec_Hap5, chunks)
    assert lib.texture_bytes(6, 4, L.HapB200Codec_Hap7, 0) == 0
    assert lib.max_encoded_length_rgba(4, 4, 6, 1) == 0


def test_hap7_encode_entry_points_refuse(lib):
    w, h = 64, 32
    rgba = np.zeros(4 * w * h, np.uint8)
    out = np.zeros(lib.max_encoded_length_rgba(w, h, L.HapB200Codec_Hap7, 1) + 64, np.uint8)
    used = np.zeros(2, np.uint64)
    for comp in (HapCompressorNone, HapCompressorSnappy):
        assert lib.encode_rgba(rgba, w, h, L.HapB200Codec_Hap7, comp, 1)[0] == BAD_ARGUMENTS
        assert lib.encode_rgba_batch(rgba.ctypes.data, 1, rgba.nbytes, w, h, L.HapB200Codec_Hap7, comp, 1, out.ctypes.data,
                                     out.nbytes, used.ctypes.data) == BAD_ARGUMENTS
    assert lib.block_encode_batch(rgba.ctypes.data, 1, rgba.nbytes, w, h, L.HapB200Codec_Hap7, out.ctypes.data,
                                  out.nbytes) == BAD_ARGUMENTS


def test_bc6h_frames_are_refused_by_the_rgba_decoder(lib):
    """Hap HDR (BC6H) has no RGBA decoder: HapB200DecodeRGBA answers Bad_Frame from the frame's headers alone"""
    w, h = 16, 8
    tex = bytes(range(256))[: (w // 4) * (h // 4) * 16]
    r, frame = lib.encode([tex], [HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT], [HapCompressorNone], [1])
    assert r == 0
    assert lib.decode_rgba(frame, w, h)[0] == BAD_FRAME
