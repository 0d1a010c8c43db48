"""Hap HDR encoding straight from HDR10 P010 (BT.2020, PQ) on the GPU.  HapB200BlockEncodeYUVPQBatch must give, byte for
byte, the blocks HapB200BlockEncodeHalfBatch gives for the RGBA16F picture the numpy restatement of the conversion
(tests/yuv_pq_util.py) makes of the planes; HapB200EncodeYUVPQBatch the frames of HapB200EncodeRGBAHalfBatch; and
HapB200EncodeYUVPQ frame 0 of the batch from host memory at any alignment and from device memory.  UF16 and SF16, both
ranges, several unitNits, Snappy with several chunks, the index and offset-table options, odd block widths, wide pitches,
frame-stride slack and an NVDEC-style chroma plane.  Sentinels around every texture and frame must survive and the planes
must be left as they were.  Then the refusals on the GPU and a decode round trip."""
import numpy as np
import pytest
import torch

import bc6h_encode_util as E
import hap_b200
import yuv_pq_util as P
import yuv_util as Y
from hap_b200.abi import (HapCompressorNone, HapCompressorSnappy, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT,
                          HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGBA_DXT5)
from hap_b200.lib import HapB200Codec_HapY

pytestmark = pytest.mark.gpu
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT
FORMATS = [UF16, SF16]
BAD_ARGUMENTS, BUFFER_TOO_SMALL = 1, 2
PAD = 0xEE


@pytest.fixture(scope="module")
def lib():
    return hap_b200.load()


def align16(n):
    return (n + 15) // 16 * 16


def dev(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy()


def planes_buffer(pics, pitch, fstride, surface_rows=None):
    """[(luma, chroma)] P010 planes -> one device byte buffer, frame f at f*fstride; chroma at pitch * surface_rows past
    luma (NVDEC) or, when None, in a second buffer.  Returns (buffer, luma offset 0, chroma buffer, chroma offset)."""
    F = len(pics)
    h, w = pics[0][0].shape
    if surface_rows is not None:
        at = pitch * surface_rows
        buf = np.full((F - 1) * fstride + at + (h // 2 - 1) * pitch + 2 * w, PAD, np.uint8)
        cbuf, cat = buf, at
    else:
        buf = np.full((F - 1) * fstride + (h - 1) * pitch + 2 * w, PAD, np.uint8)
        cbuf, cat = np.full((F - 1) * fstride + (h // 2 - 1) * pitch + 2 * w, PAD, np.uint8), 0
    for f, (luma, chroma) in enumerate(pics):
        for y in range(h):
            buf[f * fstride + y * pitch: f * fstride + y * pitch + 2 * w] = luma[y].view(np.uint8)
        for y in range(h // 2):
            o = f * fstride + cat + y * pitch
            cbuf[o: o + 2 * w] = chroma[y].view(np.uint8)
    d = dev(buf)
    return d, (d if cbuf is buf else dev(cbuf)), cat


def half_buffer(pics):
    return dev(np.concatenate([p.reshape(-1) for p in pics]))


def content(i, w, h, cs):
    if i % 3 == 2:
        return P.random_planes(np.random.default_rng(900 + i), w, h)
    return P.hdr10_planes(E.CLASSES[i % 5], w, h, cs, index=i)


def half_blocks(lib, halves, fmt):
    """HapB200BlockEncodeHalfBatch on tight RGBA16F pictures -> list of textures"""
    F, (h, w) = len(halves), halves[0].shape[:2]
    t0 = (w // 4) * (h // 4) * 16
    src = half_buffer(halves)
    out = torch.zeros(F * align16(t0), dtype=torch.uint8, device="cuda")
    assert lib.block_encode_half_batch(src.data_ptr(), F, 8 * w * h, w, h, fmt, out.data_ptr(), align16(t0)) == 0
    o = host(out)
    return [o[f * align16(t0): f * align16(t0) + t0].tobytes() for f in range(F)]


CASES = [(P.BT2020_LIMITED, 203, UF16), (P.BT2020_FULL, 100, SF16), (P.BT2020_LIMITED, 80, SF16), (P.BT2020_FULL, 10000, UF16),
         (P.BT2020_LIMITED, 1, UF16)]


@pytest.mark.parametrize("cs,unit,fmt", CASES)
def test_block_encode_equals_the_half_encoder_on_the_conversion(lib, cs, unit, fmt):
    for i, (w, h) in enumerate([(4, 4), (12, 8), (36, 20), (260, 68), (516, 36)]):
        F = 3
        pics = [content(i + f, w, h, cs) for f in range(F)]
        pitch = align16(2 * w) + 16 * (i % 3)
        nvdec = i % 2 == 1
        surface = h + 16 if nvdec else None
        fstride = align16(((surface + h // 2) if nvdec else h) * pitch) + 32
        luma, chroma, cat = planes_buffer(pics, pitch, fstride, surface)
        before = (host(luma).copy(), host(chroma).copy())
        t0 = (w // 4) * (h // 4) * 16
        bstride = align16(t0) + 48
        out = torch.full(((F - 1) * bstride + t0,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_yuv_pq_batch(luma.data_ptr(), chroma.data_ptr() + cat, F, fstride, w, h, pitch, cs, unit, fmt,
                                             out.data_ptr(), bstride) == 0
        o = host(out)
        want = half_blocks(lib, [P.yuv_pq_to_rgba_half(l, c, cs, unit) for l, c in pics], fmt)
        for f in range(F):
            assert o[f * bstride: f * bstride + t0].tobytes() == want[f], (w, h, f)
            if f + 1 < F:
                assert (o[f * bstride + t0: (f + 1) * bstride] == PAD).all(), (w, h, f)
        assert np.array_equal(host(luma), before[0]) and np.array_equal(host(chroma), before[1])


@pytest.fixture(params=[(0, 0), (1, 0), (0, 1), (1, 1)], ids=["plain", "index", "offsets", "index+offsets"])
def layout(lib, request):
    lib.set_option(lib.OPTION_WRITE_INDEX, request.param[0])
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, request.param[1])
    yield request.param
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def half_frames(lib, halves, fmt, comp, k):
    F, (h, w) = len(halves), halves[0].shape[:2]
    src = half_buffer(halves)
    ostride = align16(lib.max_encoded_length_half(w, h, fmt, k))
    out = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    assert lib.encode_rgba_half_batch(src.data_ptr(), F, 8 * w * h, w, h, fmt, comp, k, out.data_ptr(), ostride, used.data_ptr()) == 0
    o, n = host(out), host(used)
    return [o[f * ostride: f * ostride + int(n[f])].tobytes() for f in range(F)]


@pytest.mark.parametrize("fmt", FORMATS, ids=["UF16", "SF16"])
def test_batch_frames_equal_the_half_encoder(lib, layout, fmt):
    w, h, F = 132, 68, 2
    for cs, unit in ((P.BT2020_LIMITED, 203), (P.BT2020_FULL, 80)):
        pics = [content(f, w, h, cs) for f in range(F)]
        pitch = 2 * w + 24
        fstride = align16((h + 8 + h // 2) * pitch) + 16
        luma, chroma, cat = planes_buffer(pics, pitch, fstride, h + 8)
        halves = [P.yuv_pq_to_rgba_half(l, c, cs, unit) for l, c in pics]
        for comp in (HapCompressorNone, HapCompressorSnappy):
            for k in (1, 3, 8):
                ostride = align16(lib.max_encoded_length_half(w, h, fmt, k)) + 32
                out = torch.full((F * ostride,), PAD, dtype=torch.uint8, device="cuda")
                used = torch.zeros(F, dtype=torch.int64, device="cuda")
                assert lib.encode_yuv_pq_batch(luma.data_ptr(), chroma.data_ptr() + cat, F, fstride, w, h, pitch, cs, unit, fmt, comp, k,
                                               out.data_ptr(), ostride, used.data_ptr()) == 0
                o, n = host(out), host(used)
                want = half_frames(lib, halves, fmt, comp, k)
                for f in range(F):
                    assert o[f * ostride: f * ostride + int(n[f])].tobytes() == want[f], (cs, comp, k, f)
                    assert (o[f * ostride + int(n[f]): (f + 1) * ostride] == PAD).all(), (cs, comp, k, f)


@pytest.mark.parametrize("fmt", FORMATS, ids=["UF16", "SF16"])
def test_single_frame_from_host_and_device(lib, fmt):
    for i, (w, h) in enumerate([(4, 4), (36, 20), (260, 36)]):
        cs, unit, k = P.COLOR_SPACES[i % 2], (203, 100, 1000)[i], 1 + i
        luma, chroma = content(i, w, h, cs)
        batch = half_frames(lib, [P.yuv_pq_to_rgba_half(luma, chroma, cs, unit)], fmt, HapCompressorSnappy, k)[0]
        r, f = lib.encode_yuv_pq(luma, chroma, w, h, cs, unit, fmt, HapCompressorSnappy, k)
        assert r == 0 and f == batch, (w, h)
        # unaligned host planes with a pitch wider than the row
        pitch = 2 * w + 6
        lb = np.full(h * pitch + 3, PAD, np.uint8)
        cb = np.full((h // 2) * pitch + 5, PAD, np.uint8)
        lv, cv = lb[3:].reshape(h, pitch), cb[5:].reshape(h // 2, pitch)
        lv[:, : 2 * w] = luma.view(np.uint8).reshape(h, 2 * w)
        cv[:, : 2 * w] = chroma.view(np.uint8).reshape(h // 2, 2 * w)
        r, f = lib.encode_yuv_pq((lb.ctypes.data + 3, lv.size), (cb.ctypes.data + 5, cv.size), w, h, cs, unit, fmt, HapCompressorSnappy, k,
                                 pitch=pitch)
        assert r == 0 and f == batch, (w, h)
        # device planes and output
        cap = lib.max_encoded_length_half(w, h, fmt, k)
        dl, dc = dev(lv), dev(cv)
        dout = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        r, n = lib.encode_yuv_pq((dl.data_ptr(), dl.numel()), (dc.data_ptr(), dc.numel()), w, h, cs, unit, fmt, HapCompressorSnappy, k,
                                 pitch=pitch, out=(dout.data_ptr(), cap), out_capacity=cap)
        assert r == 0 and host(dout)[:n].tobytes() == batch, (w, h)
        assert lib.encode_yuv_pq(luma, chroma, w, h, cs, unit, fmt, HapCompressorSnappy, k, out=bytearray(cap),
                                 out_capacity=cap - 1)[0] == BUFFER_TOO_SMALL


def test_refusals_on_the_gpu(lib):
    w, h = 64, 32
    rng = np.random.default_rng(1)
    luma, chroma, _ = planes_buffer([P.random_planes(rng, w, h) for _ in range(2)], 2 * w, 2 * w * h)
    lp, cp = luma.data_ptr(), chroma.data_ptr()
    out = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    used = torch.zeros(4, dtype=torch.int64, device="cuda")
    o, u = out.data_ptr(), used.data_ptr()

    def block(cs=P.BT2020_LIMITED, unit=203, fmt=UF16, lp=lp, cp=cp, pitch=2 * w, bstride=8192):
        return lib.block_encode_yuv_pq_batch(lp, cp, 1, 2 * w * h, w, h, pitch, cs, unit, fmt, o, bstride)

    def batch(cs=P.BT2020_LIMITED, unit=203, fmt=UF16, lp=lp, cp=cp, pitch=2 * w, ostride=None):
        ostride = ostride if ostride is not None else align16(lib.max_encoded_length_half(w, h, UF16, 2))
        return lib.encode_yuv_pq_batch(lp, cp, 2, 2 * w * h, w, h, pitch, cs, unit, fmt, HapCompressorSnappy, 2, o, ostride, u)

    for f in (block, batch):
        for cs in (0, 1, 2, 3, 6):
            assert f(cs=cs) == BAD_ARGUMENTS, (f.__name__, cs)
        for unit in (0, 10001):
            assert f(unit=unit) == BAD_ARGUMENTS, (f.__name__, unit)
        for fmt in (HapTextureFormat_RGBA_DXT5, 0):
            assert f(fmt=fmt) == BAD_ARGUMENTS, (f.__name__, fmt)
        for kw in ({"lp": lp + 8}, {"cp": cp + 8}, {"pitch": 2 * w + 8}):
            assert f(**kw) == BAD_ARGUMENTS, (f.__name__, kw)
    assert batch(ostride=(lib.max_encoded_length_half(w, h, UF16, 2) - 1) // 16 * 16) == BUFFER_TOO_SMALL
    assert block(fmt=UF16) == 0 and batch() == 0
    # the 8-bit YUV encoders keep refusing BT.2020
    for cs in (P.BT2020_LIMITED, P.BT2020_FULL):
        assert lib.block_encode_yuv_batch(lp, cp, 1, 2 * w * h, w, h, 2 * w, Y.P010, cs, HapB200Codec_HapY, o, 8192) == BAD_ARGUMENTS


@pytest.mark.parametrize("fmt", FORMATS, ids=["UF16", "SF16"])
def test_round_trip_quality(lib, fmt):
    """HapB200DecodeRGBAHalf of a frame reproduces the conversion's picture, with PSNR16 at or above the RGBA16F encoder's
    figure for that content (the same bytes, so the same figure)"""
    w, h = 260, 132
    signed = fmt == SF16
    for cs, unit in ((P.BT2020_LIMITED, 203), (P.BT2020_FULL, 100)):
        luma, chroma = P.hdr10_planes("video", w, h, cs)
        pic = P.yuv_pq_to_rgba_half(luma, chroma, cs, unit)
        r, frame = lib.encode_yuv_pq(luma, chroma, w, h, cs, unit, fmt, HapCompressorSnappy, 2)
        assert r == 0
        r, half_frame = lib.encode_rgba_half(pic, w, h, fmt, HapCompressorSnappy, 2)
        assert r == 0 and frame == half_frame
        r, got = lib.decode_rgba_half(frame, w, h)
        assert r == 0
        psnr = E.psnr16(np.frombuffer(got, np.uint16).reshape(h, w, 4), pic, signed)
        r, ref = lib.decode_rgba_half(half_frame, w, h)
        assert r == 0
        assert psnr >= E.psnr16(np.frombuffer(ref, np.uint16).reshape(h, w, 4), pic, signed) and psnr > 30.0, psnr
