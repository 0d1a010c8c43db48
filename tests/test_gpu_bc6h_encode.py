"""Hap HDR (BC6H) encoding from RGBA16F on the GPU.  HapB200BlockEncodeHalfBatch must give the host twin's blocks
(tests/emu/bc6h_encode_twin.cc) byte for byte on every content class and both formats, pitched and strided, at 4x4 and
1924x1084 and on a 65537-frame batch.  HapB200EncodeRGBAHalfBatch frames (chunk counts 1-8, compressor None and Snappy,
fragment index and offset table on and off) must unwrap -- in this library, in the CPU oracle and in the reference build
when present -- to exactly those blocks, say their texture format, and decode to the oracle's decoding of them.
HapB200EncodeRGBAHalf must equal frame 0 of the batch from host and device buffers.  Then the input rules on the GPU and
a HapH movie round trip."""
import numpy as np
import pytest
import torch

import bc6h_encode_util as E
import bc6h_util as U
import hap_b200
import oracles
from hap_b200 import mov
from hap_b200.abi import (HapCompressorNone, HapCompressorSnappy, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT,
                          HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT)

pytestmark = pytest.mark.gpu
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT
FORMATS = [(UF16, False), (SF16, True)]
IDS = ["UF16", "SF16"]
BUFFER_TOO_SMALL = 2
PAD = 0xEE
CONTENT = [(k, p) for k in E.CLASSES for p in (1.0, 64.0)] + [("ramp", 0.0)]


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


def content(kind, peak, w, h, signed, index=0):
    return E.exposure_ramp(w, h, signed) if kind == "ramp" else E.hdr_content(kind, w, h, peak, signed, index)


def pictures_buffer(pics, pitch, fstride):
    """pictures (h, w, 4) uint16 -> one byte buffer, rows `pitch` bytes apart, pictures `fstride` apart, padding PAD"""
    h, w = pics[0].shape[:2]
    buf = np.full((len(pics) - 1) * fstride + (h - 1) * pitch + 8 * w, PAD, np.uint8)
    for f, p in enumerate(pics):
        for y in range(h):
            o = f * fstride + y * pitch
            buf[o: o + 8 * w] = p[y].view(np.uint8).reshape(-1)
    return buf


def block_encode(lib, pics, fmt, pitch=None, fstride=None, bstride=None):
    """HapB200BlockEncodeHalfBatch -> (list of textures, padding untouched)"""
    F, (h, w) = len(pics), pics[0].shape[:2]
    pitch = pitch or 8 * w
    fstride = fstride or h * pitch
    t0 = (w // 4) * (h // 4) * 16
    bstride = bstride or align16(t0)
    src = dev(pictures_buffer(pics, pitch, fstride))
    out = torch.full(((F - 1) * bstride + t0,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_half_batch(src.data_ptr(), F, fstride, w, h, fmt, out.data_ptr(), bstride, row_bytes=pitch) == 0
    o = host(out)
    texs = [o[f * bstride: f * bstride + t0].tobytes() for f in range(F)]
    clean = all((o[f * bstride + t0: (f + 1) * bstride] == PAD).all() for f in range(F - 1))
    return texs, clean


@pytest.mark.parametrize("fmt,signed", FORMATS, ids=IDS)
def test_device_blocks_equal_the_twin_on_every_content_class(lib, fmt, signed):
    w, h = 256, 128
    for i, (kind, peak) in enumerate(CONTENT):
        img = content(kind, peak, w, h, signed, i)
        texs, _ = block_encode(lib, [img], fmt)
        assert texs[0] == E.in_blocks(E.twin_encode, img, signed)[0], kind


@pytest.mark.parametrize("fmt,signed", FORMATS, ids=IDS)
def test_block_encode_half_batch_pitched_strided_and_sizes(lib, fmt, signed):
    for i, (w, h) in enumerate([(4, 4), (12, 8), (36, 20), (516, 20), (1924, 1084)]):
        F = 2 if w > 1000 else 3
        pics = [content(E.CLASSES[(i + f) % 5], 64.0, w, h, signed, f) for f in range(F)]
        pitch = 8 * w + 16 * (1 + i % 3)
        fstride = h * pitch + 32
        bstride = align16((w // 4) * (h // 4) * 16) + 48
        texs, clean = block_encode(lib, pics, fmt, pitch, fstride, bstride)
        assert clean, (w, h)
        for f in range(F):
            assert texs[f] == E.in_blocks(E.twin_encode, pics[f], signed)[0], (w, h, f)


def test_block_encode_half_batch_of_65537_frames(lib):
    F = 65537
    rng = np.random.default_rng(65537)
    pics = rng.integers(0, 1 << 16, (F * 4, 4, 4)).astype(np.uint16)
    pics[::3, :, 3] = U.ONE
    src = dev(pics)
    for fmt, signed in FORMATS:
        out = torch.full((F * 16,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_half_batch(src.data_ptr(), F, 128, 4, 4, fmt, out.data_ptr(), 16) == 0
        want, _ = E.in_blocks(E.twin_encode, pics, signed, rows=4096)
        assert host(out).tobytes() == want


@pytest.fixture(params=[(0, 0), (1, 0), (0, 1), (1, 1)], ids=["plain", "index", "offsets", "index+offsets"])
def layout(lib, request):
    lib.set_option(lib.OPTION_WRITE_INDEX, request.param[0])
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, request.param[1])
    yield request.param
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def encode_batch(lib, pics, fmt, compressor, k, pitch, fstride):
    """HapB200EncodeRGBAHalfBatch -> list of frames"""
    F, (h, w) = len(pics), pics[0].shape[:2]
    src = dev(pictures_buffer(pics, pitch, fstride))
    ostride = align16(lib.max_encoded_length_half(w, h, fmt, k))
    out = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    assert lib.encode_rgba_half_batch(src.data_ptr(), F, fstride, w, h, fmt, compressor, k, out.data_ptr(), ostride, used.data_ptr(),
                                      row_bytes=pitch) == 0
    o, n = host(out), host(used)
    return [o[f * ostride: f * ostride + int(n[f])].tobytes() for f in range(F)]


def decode_half_batch(lib, frames, w, h, k):
    F = len(frames)
    stride = align16(max(len(f) for f in frames))
    buf = np.zeros(F * stride, np.uint8)
    for i, f in enumerate(frames):
        buf[i * stride: i * stride + len(f)] = np.frombuffer(f, np.uint8)
    d = dev(buf)
    nb = torch.tensor([len(f) for f in frames], dtype=torch.int64, device="cuda")
    out = torch.zeros(F * 8 * w * h, dtype=torch.uint8, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_half_batch(d.data_ptr(), F, stride, nb.data_ptr(), k, w, h, out.data_ptr(), 8 * w * h, res.data_ptr()) == 0
    return res.tolist(), host(out).reshape(F, h, 8 * w)


@pytest.mark.parametrize("fmt,signed", FORMATS, ids=IDS)
def test_encode_rgba_half_batch_frames(lib, layout, fmt, signed):
    ref = oracles.ref_abi()
    orc = oracles.oracle_abi()
    for i, (w, h) in enumerate([(12, 8), (132, 68)]):
        pics = [content(E.CLASSES[(i + f) % 5], 1.0 + 63.0 * f, w, h, signed, f) for f in range(2)]
        pitch, fstride = 8 * w + 16, h * (8 * w + 16) + 48
        texs, _ = block_encode(lib, pics, fmt)
        want = [U.oracle_decode(t, w, h, signed).view(np.uint8).reshape(h, 8 * w) for t in texs]
        for comp in (HapCompressorNone, HapCompressorSnappy):
            for k in range(1, 9):
                frames = encode_batch(lib, pics, fmt, comp, k, pitch, fstride)
                for f, fr in enumerate(frames):
                    assert lib.texture_count(fr) == (0, 1) and lib.texture_format(fr, 0) == (0, fmt), (w, k, f)
                    for who in (lib, orc) + ((ref,) if ref is not None else ()):
                        r, tex, tf, _ = who.decode(fr, 0, out_capacity=len(texs[f]))
                        assert r == 0 and tex == texs[f] and tf == fmt, (w, h, comp, k, f)
                res, pix = decode_half_batch(lib, frames, w, h, k)
                assert res == [0, 0], (w, h, comp, k, res)
                for f in range(2):
                    assert np.array_equal(pix[f], want[f]), (w, h, comp, k, f)


@pytest.mark.parametrize("fmt,signed", FORMATS, ids=IDS)
def test_single_frame_host_and_device_buffers(lib, fmt, signed):
    for i, (w, h) in enumerate([(4, 4), (36, 20), (516, 68)]):
        pic = content(E.CLASSES[i], 64.0, w, h, signed, i)
        k = 1 + i
        batch = encode_batch(lib, [pic, pic], fmt, HapCompressorSnappy, k, 8 * w, 8 * w * h)[0]
        r, f = lib.encode_rgba_half(pic, w, h, fmt, HapCompressorSnappy, k)
        assert r == 0 and f == batch, (w, h)
        pitch = 8 * w + 24
        rows = np.zeros((h, pitch), np.uint8)
        rows[:, : 8 * w] = pic.view(np.uint8).reshape(h, 8 * w)
        r, f = lib.encode_rgba_half(rows, w, h, fmt, HapCompressorSnappy, k, row_bytes=pitch)
        assert r == 0 and f == batch, (w, h)
        cap = lib.max_encoded_length_half(w, h, fmt, k)
        dsrc = dev(rows)
        dout = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        r, n = lib.encode_rgba_half((dsrc.data_ptr(), dsrc.numel()), w, h, fmt, HapCompressorSnappy, k, row_bytes=pitch,
                                    out=(dout.data_ptr(), cap), out_capacity=cap)
        assert r == 0 and host(dout)[:n].tobytes() == batch, (w, h)
        assert lib.encode_rgba_half(pic, w, h, fmt, HapCompressorSnappy, k, out=bytearray(cap), out_capacity=cap - 1)[0] == BUFFER_TOO_SMALL


@pytest.mark.parametrize("fmt,signed", FORMATS, ids=IDS)
def test_input_rules_on_the_gpu(lib, fmt, signed):
    """constant blocks of NaN, +-Inf, negatives, -0 and ordinary values decode as the input rules say"""
    vals = np.array([0x7E00, 0xFE00, 0x7C01, 0x7C00, 0xFC00, 0x8000, 0x0000, 0xBC00, 0xC500, 0x3C00, 0x7BFF, 0xFBFF, 0x8001, 0x0001],
                    np.uint16)
    n = len(vals)
    img = np.empty((4, 4 * n, 4), np.uint16)
    for c in range(3):
        img[..., c] = np.repeat(np.roll(vals, c), 4)[None]
    img[..., 3] = 0xFFFF        # A is ignored
    texs, _ = block_encode(lib, [img], fmt)
    got = U.oracle_decode(texs[0], 4 * n, 4, signed)[..., :3]
    x = E.source_values(img, signed)
    assert np.array_equal(got, np.where(x < 0, 0x8000 | -x, x).astype(np.uint16))
    assert texs[0] == E.twin_encode(img, signed)[0]


def test_hapH_movie_round_trip(lib, tmp_path):
    w, h, n = 132, 68, 4
    for fmt, signed in FORMATS:
        pics = [content(E.CLASSES[i], 64.0, w, h, signed, i) for i in range(n)]
        frames = encode_batch(lib, pics, fmt, HapCompressorSnappy, 4, 8 * w, 8 * w * h)
        texs, _ = block_encode(lib, pics, fmt)
        path = str(tmp_path / ("hapH_%d.mov" % signed))
        with mov.MovWriter(path, "HapH", w, h, 600) as wr:
            for f in frames:
                assert mov.fourcc_for_frame(f) == (0, "HapH")
                assert wr.write(f, 20) == 0
        with mov.MovReader(path) as rd:
            assert (rd.fourcc, rd.width, rd.height, rd.frames) == ("HapH", w, h, n)
            for i in range(n):
                r, f, _ = rd.read(i)
                assert r == 0 and f == frames[i]
                r, got = lib.decode_rgba_half(f, w, h)
                want = U.oracle_decode(texs[i], w, h, signed).view(np.uint8).reshape(-1)
                assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8), want), i
