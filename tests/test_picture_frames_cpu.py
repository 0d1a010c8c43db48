"""The single-frame picture decoders pick a frame's flavour from its headers before they touch a GPU: Hap HDR (BC6H) frames
decode to RGBA16F and HDR10 P010 only, every other flavour to RGBA8, NV12 and P010 only; the others answer Bad_Frame."""
import pytest

import hap_b200
import hap_b200.lib as L
from hap_b200.abi import (HapCompressorNone, HapTextureFormat_A_RGTC1, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT,
                          HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGBA_BPTC_UNORM, HapTextureFormat_RGBA_DXT5,
                          HapTextureFormat_YCoCg_DXT5)

BAD_FRAME = 3
W, H = 16, 8
N = (W // 4) * (H // 4) * 16


@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def verbatim(lib, texs, fmts):
    """an uncompressed frame of these textures, laid out on the host (no GPU)"""
    r, frame = lib.encode(texs, fmts, [HapCompressorNone] * len(texs), [1] * len(texs))
    assert r == 0
    return frame


def test_rgba_and_yuv_decoders_refuse_hap_hdr_frames_from_their_headers(lib):
    for fmt in (HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT):
        frame = verbatim(lib, [bytes(N)], [fmt])
        assert lib.decode_rgba(frame, W, H)[0] == BAD_FRAME, fmt
        for layout in (L.HapB200YUV_NV12, L.HapB200YUV_P010):
            assert lib.decode_yuv(frame, W, H, layout, L.HapB200YUV_BT709_Limited)[0] == BAD_FRAME, (fmt, layout)


def test_hdr10_decoder_refuses_frames_of_other_flavours_from_their_headers(lib):
    cases = [([bytes(N)], [HapTextureFormat_RGBA_DXT5]), ([bytes(N)], [HapTextureFormat_RGBA_BPTC_UNORM]),
             ([bytes(N), bytes(N // 2)], [HapTextureFormat_YCoCg_DXT5, HapTextureFormat_A_RGTC1])]
    for texs, fmts in cases:
        frame = verbatim(lib, texs, fmts)
        assert lib.decode_yuv_pq(frame, W, H, L.HapB200YUV_BT2020_Limited, 203)[0] == BAD_FRAME, fmts
