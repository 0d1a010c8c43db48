"""NV12 / P010 encoders on the GPU (HapB200BlockEncodeYUVBatch, HapB200EncodeYUVBatch, HapB200EncodeYUV): every texture and
frame must equal, byte for byte, what the RGBA8 encoders give for the picture yuv_util.yuv_to_rgba (the definition of
include/hap_b200.h) makes of the same planes -- for every codec, layout and colour space, with chroma refinement, Snappy
chunking and the index and offset-table options, at odd block widths, pitches wider than the row, frame-stride slack, an
NVDEC-style chroma plane, unaligned single-frame planes and a batch of more than 65535 frames.  Sentinels around every
texture and frame must survive, and the planes must be left as they were."""
import numpy as np
import pytest
import torch

import hap_b200
import hap_b200.lib as L
import yuv_util as Y
from hap_b200 import synth
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy

pytestmark = pytest.mark.gpu
PAD = 0xEE
CODECS = {"Hap1": L.HapB200Codec_Hap1, "Hap5": L.HapB200Codec_Hap5, "HapY": L.HapB200Codec_HapY, "HapM": L.HapB200Codec_HapM}
CASES = [(c, layout, cs, 0) for c in CODECS for layout in Y.LAYOUTS for cs in Y.COLOR_SPACES] + \
        [(c, layout, cs, 1) for c in ("HapY", "HapM") for layout in Y.LAYOUTS for cs in Y.COLOR_SPACES]
SHAPES = [(w, h) for w in (4, 8, 12, 20, 36, 132, 516) for h in (4, 8, 12, 20)] + [(1924, 1084)]


@pytest.fixture(scope="module")
def lib():
    return hap_b200.load()


@pytest.fixture
def refine(lib, request):
    lib.set_option(lib.OPTION_CHROMA_REFINE, request.param)
    yield request.param
    lib.set_option(lib.OPTION_CHROMA_REFINE, 0)


def align16(n):
    return (n + 15) // 16 * 16


def dev(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).copy()).cuda()


def pictures(w, h, layout, cs, n=3, seed=0):
    """n (luma, chroma) pairs: video content converted, random samples (P010: junk in the low bits), a steep gradient"""
    rng = np.random.default_rng(seed + 7919 * w + h)
    out = []
    for i in range(n):
        if i % 3 == 1:
            out.append(Y.random_planes(rng, w, h, layout))
        else:
            out.append(Y.rgba_to_yuv(synth.frame(w, h, i, kind="video" if i % 3 == 0 else "gradient").numpy(), layout, cs))
    return out


class Planes:
    """frames of (luma, chroma) in one byte buffer: frame f's luma at f*fstride, its chroma at chroma_at + f*fstride, rows
    `pitch` apart; the buffer ends with the last chroma sample and every other byte is PAD"""

    def __init__(self, pics, layout, pitch, fstride, chroma_at):
        h, w = pics[0][0].shape
        sb = Y.sample_bytes(layout)
        self.n = chroma_at + (len(pics) - 1) * fstride + (h // 2 - 1) * pitch + sb * w
        self.buf = np.full(self.n, PAD, np.uint8)
        for f, (lu, ch) in enumerate(pics):
            for off, plane in ((f * fstride, lu), (chroma_at + f * fstride, ch)):
                rows = np.ascontiguousarray(plane).view(np.uint8).reshape(plane.shape[0], -1)
                view = np.lib.stride_tricks.as_strided(self.buf[off:], shape=rows.shape, strides=(pitch, 1))
                view[...] = rows
        self.d = dev(self.buf)
        self.luma, self.chroma = self.d.data_ptr(), self.d.data_ptr() + chroma_at

    def unchanged(self) -> bool:
        return (self.d.cpu().numpy() == self.buf).all()


def rgba_batch(pics, layout, cs):
    """the RGBA8 pictures of the definition, tight, one after another on the device"""
    rgba = np.stack([Y.yuv_to_rgba(lu, ch, layout, cs) for lu, ch in pics])
    return rgba, dev(rgba)


@pytest.mark.parametrize("codec,layout,cs,refine", CASES, indirect=["refine"])
def test_block_encode_yuv_batch_equals_rgba(lib, codec, layout, cs, refine):
    c = CODECS[codec]
    w, h, F = 260, 132, 3
    sb = Y.sample_bytes(layout)
    pitch = align16(sb * w) + 32
    chroma_at = pitch * (h + 4)                                            # NVDEC: chroma after the surface's height
    fstride = align16(chroma_at + pitch * h // 2) + 64
    pics = pictures(w, h, layout, cs, F, seed=cs)
    src = Planes(pics, layout, pitch, fstride, chroma_at)
    t = lib.texture_bytes(w, h, c, 0) + lib.texture_bytes(w, h, c, 1)
    bstride = align16(t) + 48
    got = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_yuv_batch(src.luma, src.chroma, F, fstride, w, h, pitch, layout, cs, c, got.data_ptr(), bstride) == 0
    _, rgba = rgba_batch(pics, layout, cs)
    want = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_batch(rgba.data_ptr(), F, 4 * w * h, w, h, c, want.data_ptr(), bstride) == 0
    g, wn = got.cpu().numpy().reshape(F, bstride), want.cpu().numpy().reshape(F, bstride)
    assert (g[:, :t] == wn[:, :t]).all()
    assert (g[:, t:] == PAD).all()
    assert src.unchanged()


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_encode_yuv_batch_frames_equal_rgba(lib, codec, layout):
    c = CODECS[codec]
    w, h, F = 516, 260, 3
    sb = Y.sample_bytes(layout)
    pitch = align16(sb * w) + 16
    chroma_at = pitch * (h + 8)
    fstride = align16(chroma_at + pitch * h // 2) + 16
    try:
        for k, (comp, chunks, index, offsets) in enumerate([(HapCompressorSnappy, 1, 0, 0), (HapCompressorSnappy, 8, 0, 0),
                                                            (HapCompressorSnappy, 8, 1, 0), (HapCompressorSnappy, 8, 0, 1),
                                                            (HapCompressorNone, 1, 0, 0)]):
            lib.set_option(lib.OPTION_WRITE_INDEX, index)
            lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, offsets)
            cs = k % 4
            pics = pictures(w, h, layout, cs, F, seed=k)
            src = Planes(pics, layout, pitch, fstride, chroma_at)
            ostride = align16(lib.max_encoded_length_rgba(w, h, c, chunks)) + 32
            got = torch.full((F * ostride,), PAD, dtype=torch.uint8, device="cuda")
            gused = torch.zeros(F, dtype=torch.int64, device="cuda")
            assert lib.encode_yuv_batch(src.luma, src.chroma, F, fstride, w, h, pitch, layout, cs, c, comp, chunks, got.data_ptr(), ostride,
                                        gused.data_ptr()) == 0
            _, rgba = rgba_batch(pics, layout, cs)
            want = torch.full((F * ostride,), PAD, dtype=torch.uint8, device="cuda")
            wused = torch.zeros(F, dtype=torch.int64, device="cuda")
            assert lib.encode_rgba_batch(rgba.data_ptr(), F, 4 * w * h, w, h, c, comp, chunks, want.data_ptr(), ostride,
                                         wused.data_ptr()) == 0
            gu, wu = gused.cpu().numpy(), wused.cpu().numpy()
            assert (gu == wu).all(), (comp, chunks, index, offsets)
            g, wn = got.cpu().numpy().reshape(F, ostride), want.cpu().numpy().reshape(F, ostride)
            assert (g == wn).all(), (comp, chunks, index, offsets)          # the frames, and the bytes after them
            assert src.unchanged()
    finally:
        lib.set_option(lib.OPTION_WRITE_INDEX, 0)
        lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_encode_yuv_single_frame_host_and_device_unaligned(lib, codec, layout):
    c = CODECS[codec]
    w, h = 132, 68
    sb = Y.sample_bytes(layout)
    pitch = sb * w + 6                                                     # not a multiple of 16: the single-frame call copies
    for cs in Y.COLOR_SPACES:
        (lu, ch), = pictures(w, h, layout, cs, 1, seed=40 + cs)
        want_rgba = Y.yuv_to_rgba(lu, ch, layout, cs)
        r, want = lib.encode_rgba(want_rgba, w, h, c, HapCompressorSnappy, 4)
        assert r == 0
        lb, cb = Y.pitched(lu, pitch), Y.pitched(ch, pitch)
        # host planes at odd addresses
        hl = np.zeros(lb.size + 1, np.uint8)[1:]
        hc = np.zeros(cb.size + 3, np.uint8)[3:]
        hl[:], hc[:] = lb.ravel(), cb.ravel()
        r, got = lib.encode_yuv(hl, hc, w, h, layout, cs, c, HapCompressorSnappy, 4, pitch=pitch)
        assert r == 0 and got == want, cs
        # device planes at odd addresses
        dl, dc = dev(np.concatenate([[0], lb.ravel()]).astype(np.uint8)), dev(np.concatenate([[0, 0, 0], cb.ravel()]).astype(np.uint8))
        r, got = lib.encode_yuv((dl.data_ptr() + 1, lb.size), (dc.data_ptr() + 3, cb.size), w, h, layout, cs, c, HapCompressorSnappy, 4,
                                pitch=pitch)
        assert r == 0 and got == want, cs
        # a tight default pitch
        r, got = lib.encode_yuv(np.ascontiguousarray(lu), np.ascontiguousarray(ch), w, h, layout, cs, c, HapCompressorSnappy, 4)
        assert r == 0 and got == want, cs


@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_block_encode_yuv_geometry(lib, layout):
    """the shapes of test_gpu_geometry.py, with pitches wider than the row, frame-stride slack and the chroma plane at an
    NVDEC-style offset"""
    sb = Y.sample_bytes(layout)
    for i, (w, h) in enumerate(SHAPES):
        for codec in ("Hap1", "HapM"):
            c = CODECS[codec]
            F = 3
            cs = i % 4
            pitch = align16(sb * w) + 16 * (i % 3)
            chroma_at = pitch * (h + 16 * (i % 2))
            fstride = align16(chroma_at + pitch * h // 2) + 16 * (1 + i % 2)
            pics = pictures(w, h, layout, cs, F, seed=i)
            src = Planes(pics, layout, pitch, fstride, chroma_at)
            t = lib.texture_bytes(w, h, c, 0) + lib.texture_bytes(w, h, c, 1)
            bstride = align16(t) + 48
            got = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_yuv_batch(src.luma, src.chroma, F, fstride, w, h, pitch, layout, cs, c, got.data_ptr(), bstride) == 0
            _, rgba = rgba_batch(pics, layout, cs)
            want = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_batch(rgba.data_ptr(), F, 4 * w * h, w, h, c, want.data_ptr(), bstride) == 0
            g, wn = got.cpu().numpy().reshape(F, bstride), want.cpu().numpy().reshape(F, bstride)
            assert (g[:, :t] == wn[:, :t]).all(), (w, h, codec)
            assert (g[:, t:] == PAD).all(), (w, h, codec)
            assert src.unchanged(), (w, h, codec)


def test_yuv_batch_of_65537_frames(lib):
    """4x4 pictures, 65537 of them: two launches (65535 + 2 frames); seven distinct pictures repeat"""
    w, h, F = 4, 4, 65537
    for layout in Y.LAYOUTS:
        sb = Y.sample_bytes(layout)
        pitch = 16
        chroma_at, fstride = 4 * pitch, 6 * pitch
        distinct = pictures(w, h, layout, Y.BT709_LIMITED, 7, seed=layout)
        base = Planes(distinct, layout, pitch, fstride, chroma_at).buf
        n = chroma_at + (F - 1) * fstride + (h // 2 - 1) * pitch + sb * w
        buf = np.full(n, PAD, np.uint8)
        idx = np.arange(F) % 7
        full = np.full(7 * fstride, PAD, np.uint8)
        full[: base.size] = base
        tiles = full.reshape(7, fstride)
        buf[: (F - 1) * fstride] = tiles[idx[:-1]].ravel()
        buf[(F - 1) * fstride:] = tiles[idx[-1], : n - (F - 1) * fstride]
        d = dev(buf)
        rgba7, _ = rgba_batch(distinct, layout, Y.BT709_LIMITED)
        rgba = dev(rgba7[idx])
        for codec in ("Hap1", "HapY"):
            c = CODECS[codec]
            t = lib.texture_bytes(w, h, c, 0)
            got = torch.full((F * 16,), PAD, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_yuv_batch(d.data_ptr(), d.data_ptr() + chroma_at, F, fstride, w, h, pitch, layout, Y.BT709_LIMITED, c,
                                              got.data_ptr(), 16) == 0
            want = torch.full((F * 16,), PAD, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_batch(rgba.data_ptr(), F, 64, w, h, c, want.data_ptr(), 16) == 0
            assert torch.equal(got, want), codec
            assert (got.view(F, 16)[:, t:] == PAD).all()
        # whole frames, Hap Q
        c = CODECS["HapY"]
        ostride = align16(lib.max_encoded_length_rgba(w, h, c, 1))
        got = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
        gused = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_yuv_batch(d.data_ptr(), d.data_ptr() + chroma_at, F, fstride, w, h, pitch, layout, Y.BT709_LIMITED, c,
                                    HapCompressorSnappy, 1, got.data_ptr(), ostride, gused.data_ptr()) == 0
        want = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
        wused = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_rgba_batch(rgba.data_ptr(), F, 64, w, h, c, HapCompressorSnappy, 1, want.data_ptr(), ostride, wused.data_ptr()) == 0
        assert torch.equal(gused, wused) and torch.equal(got, want)
