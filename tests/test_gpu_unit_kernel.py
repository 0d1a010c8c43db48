"""snappy_execute_units_kernel on the device: the Snappy decoder's kernel for the 8-byte granular fragments of an embedded
index, launched ahead of the execute kernel, which takes every other window.  Batches that mix indexed, non-indexed,
verbatim and damaged-index frames decode in one call to the reference's bytes at ordinary and odd geometries; a decode
on one stream beside an encode on another (the benchmark's pattern) gives the same bytes as the decode alone."""
import numpy as np
import pytest
import torch

import hap_b200
from hap_b200 import synth
from hap_b200.lib import HapB200Codec_Hap1, HapB200Codec_HapY

from test_gpu_decode_units import decode_batch, frame_proper_bytes, reference

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    lib = hap_b200.load()
    yield lib
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_USE_INDEX, 1)


def encode_frame(lib, w, h, codec, k, seed, index, compressor=1):
    lib.set_option(lib.OPTION_WRITE_INDEX, index)
    try:
        img = synth.frame(w, h, seed, device="cuda")
        cap = (lib.max_encoded_length_rgba(w, h, codec, k) + 15) // 16 * 16
        out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        used = torch.zeros(1, dtype=torch.int64, device="cuda")
        assert lib.encode_rgba_batch(img.data_ptr(), 1, img.numel(), w, h, codec, compressor, k, out.data_ptr(), cap, used.data_ptr()) == 0
        return out.cpu().numpy()[: int(used[0])].tobytes()
    finally:
        lib.set_option(lib.OPTION_WRITE_INDEX, 0)


def damage_index(frame, seed):
    proper = frame_proper_bytes(frame)
    assert frame[proper + 3] == 0xFB   # the index section follows the frame
    damaged = bytearray(frame)
    rng = np.random.default_rng(seed)
    lo = proper + min(40, (len(frame) - proper) // 2)   # past the section header and the index's own header on all but tiny frames
    for _ in range(8):
        damaged[lo + int(rng.integers(0, len(frame) - lo))] ^= 1 << int(rng.integers(0, 8))
    return bytes(damaged)


@pytest.mark.parametrize("w,h,codec_name,k", [(3840, 2160, "HapY", 8), (1920, 1080, "Hap1", 4), (1004, 564, "HapY", 3), (4100, 36, "Hap1", 7),
                                              (36, 20, "HapY", 1)])
def test_mixed_batch_matches_the_reference(lib, w, h, codec_name, k):
    codec = {"HapY": HapB200Codec_HapY, "Hap1": HapB200Codec_Hap1}[codec_name]
    indexed = [encode_frame(lib, w, h, codec, k, s, 1) for s in (1, 2)]
    frames = [indexed[0], encode_frame(lib, w, h, codec, k, 3, 0), encode_frame(lib, w, h, codec, k, 4, 1, compressor=0),
              damage_index(indexed[1], 5), indexed[1], encode_frame(lib, w, h, codec, k, 6, 0, compressor=0), indexed[0]]
    n = lib.texture_bytes(w, h, codec, 0)
    ref = reference()
    want = []
    for fr in frames:
        r, tex, _, _ = ref.decode(fr, 0, n)
        assert r == 0 and len(tex) == n
        want.append(tex)
    res, got = decode_batch(lib, frames, 0, n, k)
    assert res == [0] * len(frames)
    assert got == want
    # and with the index ignored (every window through the execute kernel)
    lib.set_option(lib.OPTION_USE_INDEX, 0)
    try:
        res, got = decode_batch(lib, frames, 0, n, k)
    finally:
        lib.set_option(lib.OPTION_USE_INDEX, 1)
    assert res == [0] * len(frames) and got == want


def test_decode_beside_an_encode_on_another_stream(lib):
    w, h, k, F = 3840, 2160, 8, 24
    codec = HapB200Codec_HapY
    rgba = torch.empty((F, h, w, 4), dtype=torch.uint8, device="cuda")
    for i in range(F):
        rgba[i] = synth.frame(w, h, 40 + i, device="cuda")
    cap = (lib.max_encoded_length_rgba(w, h, codec, k) + 15) // 16 * 16
    n = lib.texture_bytes(w, h, codec, 0)
    stride = (n + 15) // 16 * 16
    bufs = [torch.zeros(F * cap, dtype=torch.uint8, device="cuda") for _ in range(2)]
    used = [torch.zeros(F, dtype=torch.int64, device="cuda") for _ in range(2)]
    tex = torch.zeros(F * stride, dtype=torch.uint8, device="cuda")
    tex_used = torch.zeros(F, dtype=torch.int64, device="cuda")
    fmts = torch.zeros(F, dtype=torch.int32, device="cuda")
    res = torch.full((F,), 9, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    s_enc, s_dec = torch.cuda.Stream(), torch.cuda.Stream()
    lib.set_option(lib.OPTION_WRITE_INDEX, 1)
    try:
        assert lib.encode_rgba_batch(rgba.data_ptr(), F, 4 * w * h, w, h, codec, 1, k, bufs[0].data_ptr(), cap, used[0].data_ptr(),
                                     stream=s_enc.cuda_stream) == 0
        s_enc.synchronize()

        def decode(st):
            assert lib.decode_batch(bufs[0].data_ptr(), F, cap, used[0].data_ptr(), 0, k, tex.data_ptr(), stride, tex_used.data_ptr(),
                                    fmts.data_ptr(), res.data_ptr(), stream=st) == 0

        decode(s_dec.cuda_stream)
        s_dec.synchronize()
        alone = tex.clone()
        assert res.tolist() == [0] * F
        for _ in range(3):
            tex.zero_()
            torch.cuda.synchronize()
            assert lib.encode_rgba_batch(rgba.data_ptr(), F, 4 * w * h, w, h, codec, 1, k, bufs[1].data_ptr(), cap, used[1].data_ptr(),
                                         stream=s_enc.cuda_stream) == 0
            decode(s_dec.cuda_stream)
            torch.cuda.synchronize()
            assert res.tolist() == [0] * F and torch.equal(tex, alone)
    finally:
        lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    # the encodes beside the decodes made the same frames
    assert torch.equal(used[0], used[1])
    ref = reference()
    host = bufs[0].cpu().numpy()
    for f in (0, F - 1):
        frame = host[f * cap: f * cap + int(used[0][f])].tobytes()
        r, want, _, _ = ref.decode(frame, 0, n)
        assert r == 0 and want == alone[f * stride: f * stride + n].cpu().numpy().tobytes()
