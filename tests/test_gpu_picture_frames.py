"""The single-frame picture decoders on a well-formed frame whose texture is larger than the picture: the RGBA8 and NV12 /
P010 decoders answer what HapDecode answers when offered the picture's texture size; the Hap HDR decoders (RGBA16F, HDR10
P010) answer Bad_Frame, the frame's texture not being the picture's."""
import numpy as np
import pytest

import hap_b200
import hap_b200.lib as L
from hap_b200 import synth
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy, HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT

pytestmark = pytest.mark.gpu
BAD_FRAME = 3
CODECS = {"Hap1": L.HapB200Codec_Hap1, "Hap5": L.HapB200Codec_Hap5, "HapY": L.HapB200Codec_HapY, "HapM": L.HapB200Codec_HapM,
          "HapA": L.HapB200Codec_HapA, "Hap7": L.HapB200Codec_Hap7}


@pytest.fixture(scope="module")
def lib():
    return hap_b200.load()


def test_rgba_and_yuv_decoders_answer_as_hapdecode_for_a_texture_larger_than_the_picture(lib):
    w, h = 16, 12
    img = synth.frame(w, h, 0).numpy()
    for name, c in CODECS.items():
        for comp in (HapCompressorNone, HapCompressorSnappy):
            if c == L.HapB200Codec_Hap7:
                r, frame = lib.encode_rgba_bc7(img, w, h, comp)
            else:
                r, frame = lib.encode_rgba(img, w, h, c, comp)
            assert r == 0, name
            want = lib.decode(frame, 0, lib.texture_bytes(w, h - 4, c, 0))[0]
            assert want not in (0, BAD_FRAME), (name, want)
            assert lib.decode_rgba(frame, w, h - 4)[0] == want, name
            for layout in (L.HapB200YUV_NV12, L.HapB200YUV_P010):
                assert lib.decode_yuv(frame, w, h - 4, layout, L.HapB200YUV_BT709_Limited)[0] == want, (name, layout)


def test_hdr_decoders_refuse_a_texture_larger_than_the_picture(lib):
    w, h = 132, 20
    tex = np.random.default_rng(91).integers(0, 256, (w // 4) * (h // 4) * 16, dtype=np.uint8).tobytes()
    for comp in (HapCompressorNone, HapCompressorSnappy):
        r, frame = lib.encode([tex], [HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT], [comp], [1])
        assert r == 0
        assert lib.decode_rgba_half(frame, w, h - 4)[0] == BAD_FRAME
        assert lib.decode_yuv_pq(frame, w, h - 4, L.HapB200YUV_BT2020_Limited, 203)[0] == BAD_FRAME
        assert lib.decode_rgba_half(frame, w, h)[0] == 0
        assert lib.decode_yuv_pq(frame, w, h, L.HapB200YUV_BT2020_Limited, 203)[0] == 0
