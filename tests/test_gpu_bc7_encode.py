"""Hap R (BC7) encoding from RGBA8 on the GPU.  HapB200BlockEncodeBC7Batch must give the host twin's blocks
(tests/emu/bc7_encode_twin.cc) byte for byte on every content class, pitched and strided, from 4x4 to 1924x1084 and on a
65537-frame batch.  HapB200EncodeRGBABC7Batch frames (chunk counts 1-8, compressor None and Snappy, fragment index and
offset table on and off) must report one RGBA_BPTC_UNORM texture, unwrap -- in this library, in the CPU oracle and in the
reference build when present -- to exactly those blocks, and decode through HapB200DecodeRGBABatch(Hap7) to the oracle
decoder's decoding of them.  HapB200EncodeRGBABC7 must equal frame 0 of the batch from host, pitched host and device
buffers.  Then the constant and opaque rules on the GPU and a Hap7 movie round trip."""
import numpy as np
import pytest
import torch

import bc7_encode_util as E
import bc7_util as U
import hap_b200
import oracles
from hap_b200 import mov
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy, HapTextureFormat_RGBA_BPTC_UNORM
from hap_b200.lib import HapB200Codec_Hap7

pytestmark = pytest.mark.gpu
BUFFER_TOO_SMALL = 2
PAD = 0xEE
FMT = HapTextureFormat_RGBA_BPTC_UNORM


@pytest.fixture(scope="module")
def lib():
    return hap_b200.load()


def align16(n):
    return (n + 15) // 16 * 16


def dev(a) -> torch.Tensor:
    if isinstance(a, (bytes, bytearray)):
        a = np.frombuffer(a, np.uint8)
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy()


def pictures_buffer(pics, pitch, fstride):
    """pictures (h, w, 4) uint8 -> one byte buffer, rows `pitch` bytes apart, pictures `fstride` apart, padding PAD"""
    h, w = pics[0].shape[:2]
    buf = np.full((len(pics) - 1) * fstride + (h - 1) * pitch + 4 * w, PAD, np.uint8)
    for f, p in enumerate(pics):
        for y in range(h):
            o = f * fstride + y * pitch
            buf[o: o + 4 * w] = p[y].reshape(-1)
    return buf


def block_encode(lib, pics, pitch=None, fstride=None, bstride=None):
    """HapB200BlockEncodeBC7Batch -> (list of textures, padding untouched)"""
    F, (h, w) = len(pics), pics[0].shape[:2]
    pitch = pitch or 4 * w
    fstride = fstride or h * pitch
    t0 = (w // 4) * (h // 4) * 16
    bstride = bstride or align16(t0)
    src = dev(pictures_buffer(pics, pitch, fstride))
    out = torch.full(((F - 1) * bstride + t0,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_bc7_batch(src.data_ptr(), F, fstride, w, h, out.data_ptr(), bstride, row_bytes=pitch) == 0
    o = host(out)
    texs = [o[f * bstride: f * bstride + t0].tobytes() for f in range(F)]
    clean = all((o[f * bstride + t0: (f + 1) * bstride] == PAD).all() for f in range(F - 1))
    return texs, clean


def test_device_blocks_equal_the_twin_on_every_content_class(lib):
    w, h = 256, 128
    for i, (kind, alpha) in enumerate(E.CONTENT):
        img = E.content(kind, alpha, w, h, i)
        texs, _ = block_encode(lib, [img])
        assert texs[0] == E.in_blocks(E.twin_encode, img)[0], (kind, alpha)


def test_block_encode_bc7_batch_pitched_strided_and_sizes(lib):
    for i, (w, h) in enumerate([(4, 4), (12, 8), (36, 20), (516, 20), (1924, 1084)]):
        F = 2 if w > 1000 else 3
        pics = [E.content(*E.CONTENT[(i + f) % len(E.CONTENT)], w, h, f) for f in range(F)]
        pitch = 4 * w + 16 * (1 + i % 3)
        fstride = h * pitch + 32
        bstride = align16((w // 4) * (h // 4) * 16) + 48
        texs, clean = block_encode(lib, pics, pitch, fstride, bstride)
        assert clean, (w, h)
        for f in range(F):
            assert texs[f] == E.in_blocks(E.twin_encode, pics[f], rows=64)[0], (w, h, f)


def test_block_encode_bc7_batch_of_65537_frames(lib):
    F = 65537
    rng = np.random.default_rng(65537)
    pics = rng.integers(0, 256, (F * 4, 4, 4)).astype(np.uint8)
    pics[::3, :, 3] = 255
    pics[4 * 5::4 * 11] = pics[4 * 5::4 * 11, :1, :1]            # some constant frames
    src = dev(pics)
    out = torch.full((F * 16,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_bc7_batch(src.data_ptr(), F, 64, 4, 4, out.data_ptr(), 16) == 0
    want, _ = E.in_blocks(E.twin_encode, pics, rows=4096)
    assert host(out).tobytes() == want


@pytest.fixture(params=[(0, 0), (1, 0), (0, 1), (1, 1)], ids=["plain", "index", "offsets", "index+offsets"])
def layout(lib, request):
    lib.set_option(lib.OPTION_WRITE_INDEX, request.param[0])
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, request.param[1])
    yield request.param
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def encode_batch(lib, pics, compressor, k, pitch, fstride):
    """HapB200EncodeRGBABC7Batch -> list of frames"""
    F, (h, w) = len(pics), pics[0].shape[:2]
    src = dev(pictures_buffer(pics, pitch, fstride))
    ostride = align16(lib.max_encoded_length_rgba(w, h, HapB200Codec_Hap7, k))
    out = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    assert lib.encode_rgba_bc7_batch(src.data_ptr(), F, fstride, w, h, compressor, k, out.data_ptr(), ostride, used.data_ptr(),
                                     row_bytes=pitch) == 0
    o, n = host(out), host(used)
    return [o[f * ostride: f * ostride + int(n[f])].tobytes() for f in range(F)]


def decode_rgba_batch(lib, frames, w, h, k):
    F = len(frames)
    stride = align16(max(len(f) for f in frames))
    buf = np.zeros(F * stride, np.uint8)
    for i, f in enumerate(frames):
        buf[i * stride: i * stride + len(f)] = np.frombuffer(f, np.uint8)
    d = dev(buf)
    nb = torch.tensor([len(f) for f in frames], dtype=torch.int64, device="cuda")
    out = torch.zeros(F * 4 * w * h, dtype=torch.uint8, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_batch(d.data_ptr(), F, stride, nb.data_ptr(), k, HapB200Codec_Hap7, w, h, out.data_ptr(), 4 * w * h,
                                 res.data_ptr()) == 0
    return res.tolist(), host(out).reshape(F, h, w, 4)


def test_encode_rgba_bc7_batch_frames(lib, layout):
    ref = oracles.ref_abi()
    orc = oracles.oracle_abi()
    for i, (w, h) in enumerate([(12, 8), (132, 68)]):
        pics = [E.content(*E.CONTENT[(3 * i + f) % len(E.CONTENT)], w, h, f) for f in range(2)]
        pitch, fstride = 4 * w + 16, h * (4 * w + 16) + 48
        texs, _ = block_encode(lib, pics)
        want = [U.oracle_decode(t, w, h) for t in texs]
        for comp in (HapCompressorNone, HapCompressorSnappy):
            for k in range(1, 9):
                frames = encode_batch(lib, pics, comp, k, pitch, fstride)
                for f, fr in enumerate(frames):
                    assert lib.texture_count(fr) == (0, 1) and lib.texture_format(fr, 0) == (0, FMT), (w, k, f)
                    for who in (lib, orc) + ((ref,) if ref is not None else ()):
                        r, tex, tf, _ = who.decode(fr, 0, out_capacity=len(texs[f]))
                        assert r == 0 and tex == texs[f] and tf == FMT, (w, h, comp, k, f)
                res, pix = decode_rgba_batch(lib, frames, w, h, k)
                assert res == [0, 0], (w, h, comp, k, res)
                for f in range(2):
                    assert np.array_equal(pix[f], want[f]), (w, h, comp, k, f)


def test_single_frame_host_and_device_buffers(lib):
    for i, (w, h) in enumerate([(4, 4), (36, 20), (516, 68)]):
        pic = E.content(*E.CONTENT[2 * i + 1], w, h, i)
        k = 1 + i
        batch = encode_batch(lib, [pic, pic], HapCompressorSnappy, k, 4 * w, 4 * w * h)[0]
        r, f = lib.encode_rgba_bc7(pic, w, h, HapCompressorSnappy, k)
        assert r == 0 and f == batch, (w, h)
        pitch = 4 * w + 24
        rows = np.zeros((h, pitch), np.uint8)
        rows[:, : 4 * w] = pic.reshape(h, 4 * w)
        r, f = lib.encode_rgba_bc7(rows, w, h, HapCompressorSnappy, k, row_bytes=pitch)
        assert r == 0 and f == batch, (w, h)
        cap = lib.max_encoded_length_rgba(w, h, HapB200Codec_Hap7, k)
        dsrc = dev(rows)
        dout = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        r, n = lib.encode_rgba_bc7((dsrc.data_ptr(), dsrc.numel()), w, h, HapCompressorSnappy, k, row_bytes=pitch,
                                   out=(dout.data_ptr(), cap), out_capacity=cap)
        assert r == 0 and host(dout)[:n].tobytes() == batch, (w, h)
        assert lib.encode_rgba_bc7(pic, w, h, HapCompressorSnappy, k, out=bytearray(cap), out_capacity=cap - 1)[0] == BUFFER_TOO_SMALL


def test_constant_and_opaque_rules_on_the_gpu(lib):
    rng = np.random.default_rng(17)
    n = 4096
    v = rng.integers(0, 256, (n, 4)).astype(np.uint8)
    v[:8] = [[0, 0, 0, 0], [255, 255, 255, 255], [0, 0, 0, 255], [255, 255, 255, 0], [1, 128, 254, 0], [127, 129, 2, 255],
             [255, 0, 255, 0], [0, 255, 0, 255]]
    img = np.ascontiguousarray(np.repeat(np.repeat(v.reshape(16, 256, 4), 4, axis=0), 4, axis=1))
    texs, _ = block_encode(lib, [img])
    assert np.array_equal(U.oracle_decode(texs[0], 1024, 64), img)
    opaque = rng.integers(0, 256, (64, 512, 4)).astype(np.uint8)
    opaque[..., 3] = 255
    opaque[32:] = E.content("edges", "opaque", 512, 32)
    texs, _ = block_encode(lib, [opaque])
    assert (U.oracle_decode(texs[0], 512, 64)[..., 3] == 255).all()
    assert texs[0] == E.in_blocks(E.twin_encode, opaque)[0]


def test_hap7_movie_round_trip(lib, tmp_path):
    w, h, n = 132, 68, 4
    pics = [E.content(*E.CONTENT[2 * i + 1], w, h, i) for i in range(n)]
    frames = encode_batch(lib, pics, HapCompressorSnappy, 4, 4 * w, 4 * w * h)
    texs, _ = block_encode(lib, pics)
    path = str(tmp_path / "hap7.mov")
    with mov.MovWriter(path, "Hap7", w, h, 600) as wr:
        for f in frames:
            assert mov.fourcc_for_frame(f) == (0, "Hap7")
            assert wr.write(f, 20) == 0
    with mov.MovReader(path) as rd:
        assert (rd.fourcc, rd.width, rd.height, rd.frames) == ("Hap7", w, h, n)
        for i in range(n):
            r, f, _ = rd.read(i)
            assert r == 0 and f == frames[i]
            r, got = lib.decode_rgba(f, w, h)
            assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, w, 4), U.oracle_decode(texs[i], w, h)), i
