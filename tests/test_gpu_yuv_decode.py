"""NV12 / P010 decoders on the GPU (HapB200BlockDecodeYUVBatch, HapB200DecodeYUVBatch, HapB200DecodeYUV): every plane must
equal, byte for byte, yuv_out_util.rgba_to_yuv_out (the definition of include/hap_b200.h) of what the RGBA8 decoders give for
the same input, and the batch results must equal theirs -- for every codec, layout and colour space; on Snappy-chunked frames
(with the index and offset-table options), uncompressed frames, the reference's own frames, the geometry shapes of the YUV
encoders' tests, a batch of more than 65535 frames and a batch mixing good, truncated and wrong-codec frames.  Sentinels
around every plane must survive and the inputs must be left as they were."""
import numpy as np
import pytest
import torch

import hap_b200
import hap_b200.lib as L
import yuv_out_util as O
import yuv_util as Y
from golden_util import b64, golden
from hap_b200 import synth
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy

pytestmark = pytest.mark.gpu
PAD = 0xEE
CODECS = {"Hap1": L.HapB200Codec_Hap1, "Hap5": L.HapB200Codec_Hap5, "HapY": L.HapB200Codec_HapY, "HapM": L.HapB200Codec_HapM,
          "HapA": L.HapB200Codec_HapA, "Hap7": L.HapB200Codec_Hap7}
CASES = [(c, layout, cs) for c in CODECS for layout in Y.LAYOUTS for cs in Y.COLOR_SPACES]
SHAPES = [(w, h) for w in (4, 8, 12, 20, 36, 132, 516) for h in (4, 8, 12, 20)] + [(1924, 1084)]
MAX_CHUNKS = 64
BAD_FRAME = 3


@pytest.fixture(scope="module")
def lib():
    return hap_b200.load()


def align16(n):
    return (n + 15) // 16 * 16


def dev(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a).copy()).cuda()


def textures(lib, w, h, c, F, seed):
    """F random textures of codec c, texture 1 (Hap Q Alpha) at texture_bytes(.., 0): every byte pattern is a valid block
    of these formats (BC7's reserved blocks decode to zeros)"""
    t = lib.texture_bytes(w, h, c, 0) + lib.texture_bytes(w, h, c, 1)
    return np.random.default_rng(seed).integers(0, 256, (F, t), dtype=np.uint8)


class Out:
    """F pictures' planes in one device buffer of PAD bytes: frame f's luma at f*fstride, its chroma at chroma_at + f*fstride,
    rows `pitch` apart; the buffer ends with the last chroma sample"""

    def __init__(self, F, w, h, layout, pitch, fstride, chroma_at):
        self.F, self.w, self.h, self.layout, self.pitch, self.fstride, self.chroma_at = F, w, h, layout, pitch, fstride, chroma_at
        self.sb = Y.sample_bytes(layout)
        self.n = chroma_at + (F - 1) * fstride + (h // 2 - 1) * pitch + self.sb * w
        self.d = torch.full((self.n,), PAD, dtype=torch.uint8, device="cuda")
        self.luma, self.chroma = self.d.data_ptr(), self.d.data_ptr() + chroma_at

    def want_buffer(self, planes):
        """the whole buffer as it must be: planes[f] = (luma, chroma) as stored, at their places; PAD elsewhere"""
        buf = np.full(self.n, PAD, np.uint8)
        for f, (lu, ch) in enumerate(planes):
            for off, plane in ((f * self.fstride, lu), (self.chroma_at + f * self.fstride, ch)):
                rows = np.ascontiguousarray(plane).view(np.uint8).reshape(plane.shape[0], -1)
                np.lib.stride_tricks.as_strided(buf[off:], shape=rows.shape, strides=(self.pitch, 1))[...] = rows
        return buf

    def check(self, rgba, cs, what=""):
        """the buffer equals the conversion of rgba[f] at every plane byte and PAD everywhere else"""
        want = self.want_buffer([O.rgba_to_yuv_out(p, self.layout, cs) for p in rgba])
        got = self.d.cpu().numpy()
        bad = np.flatnonzero(got != want)
        assert bad.size == 0, (what, bad.size, bad[:8])


def geometry(w, h, layout, i=1):
    """a pitch wider than the row, the chroma plane at an NVDEC-style offset, frame-stride slack"""
    sb = Y.sample_bytes(layout)
    pitch = align16(sb * w) + 16 * (1 + i % 3)
    chroma_at = pitch * (h + 16 * (i % 2))
    fstride = align16(chroma_at + pitch * h // 2) + 16 * (1 + i % 2)
    return pitch, fstride, chroma_at


def rgba_of_blocks(lib, blk, F, bstride, w, h, c):
    rgba = torch.zeros(F * 4 * w * h, dtype=torch.uint8, device="cuda")
    assert lib.block_decode_batch(blk.data_ptr(), F, bstride, w, h, c, rgba.data_ptr(), 4 * w * h) == 0
    return rgba.cpu().numpy().reshape(F, h, w, 4)


@pytest.mark.parametrize("codec,layout,cs", CASES)
def test_block_decode_yuv_batch_equals_rgba(lib, codec, layout, cs):
    c = CODECS[codec]
    w, h, F = 260, 132, 3                                                 # 65 block columns: three warp spans per row
    t = textures(lib, w, h, c, F, seed=10 * c + cs)
    bstride = align16(t.shape[1]) + 48
    blk_np = np.zeros((F, bstride), np.uint8)
    blk_np[:, : t.shape[1]] = t
    blk = dev(blk_np.ravel())
    pitch, fstride, chroma_at = geometry(w, h, layout, cs)
    out = Out(F, w, h, layout, pitch, fstride, chroma_at)
    assert lib.block_decode_yuv_batch(blk.data_ptr(), F, bstride, w, h, c, out.luma, out.chroma, fstride, pitch, layout, cs) == 0
    out.check(rgba_of_blocks(lib, blk, F, bstride, w, h, c), cs, (codec, layout, cs))
    assert (blk.cpu().numpy() == blk_np.ravel()).all()


@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_block_decode_yuv_geometry(lib, layout):
    for i, (w, h) in enumerate(SHAPES):
        for codec in ("Hap1", "HapM", "Hap7"):
            c = CODECS[codec]
            F, cs = 3, i % 4
            t = textures(lib, w, h, c, F, seed=i)
            bstride = align16(t.shape[1]) + 16 * (i % 3)
            blk_np = np.zeros((F, bstride), np.uint8)
            blk_np[:, : t.shape[1]] = t
            blk = dev(blk_np.ravel())
            pitch, fstride, chroma_at = geometry(w, h, layout, i)
            out = Out(F, w, h, layout, pitch, fstride, chroma_at)
            assert lib.block_decode_yuv_batch(blk.data_ptr(), F, bstride, w, h, c, out.luma, out.chroma, fstride, pitch, layout, cs) == 0
            out.check(rgba_of_blocks(lib, blk, F, bstride, w, h, c), cs, (w, h, codec))


def encode_frames(lib, pics, c, comp, chunks):
    """pictures (F, h, w, 4) uint8 -> (device frames at a common stride, stride, device lengths)"""
    F, h, w = pics.shape[:3]
    cap = lib.max_encoded_length_rgba(w, h, c, chunks)
    ostride = align16(cap)
    out = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    src = dev(pics)
    if c == L.HapB200Codec_Hap7:
        r = lib.encode_rgba_bc7_batch(src.data_ptr(), F, 4 * w * h, w, h, comp, chunks, out.data_ptr(), ostride, used.data_ptr())
    else:
        r = lib.encode_rgba_batch(src.data_ptr(), F, 4 * w * h, w, h, c, comp, chunks, out.data_ptr(), ostride, used.data_ptr())
    assert r == 0
    return out, ostride, used


def decode_both(lib, frames, F, istride, used, c, w, h, layout, cs, i=1):
    """HapB200DecodeRGBABatch and HapB200DecodeYUVBatch on the same frames: (RGBA pictures, RGBA results, Out, YUV results)"""
    rgba = torch.zeros(F * 4 * w * h, dtype=torch.uint8, device="cuda")
    rres = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_batch(frames.data_ptr(), F, istride, used.data_ptr(), MAX_CHUNKS, c, w, h, rgba.data_ptr(), 4 * w * h,
                                 rres.data_ptr()) == 0
    pitch, fstride, chroma_at = geometry(w, h, layout, i)
    out = Out(F, w, h, layout, pitch, fstride, chroma_at)
    yres = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_yuv_batch(frames.data_ptr(), F, istride, used.data_ptr(), MAX_CHUNKS, c, w, h, out.luma, out.chroma, fstride, pitch,
                                layout, cs, yres.data_ptr()) == 0
    return rgba.cpu().numpy().reshape(F, h, w, 4), rres.cpu().numpy(), out, yres.cpu().numpy()


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_decode_yuv_batch_equals_rgba(lib, codec, layout):
    c = CODECS[codec]
    w, h, F = 260, 132, 3
    pics = np.stack([synth.frame(w, h, i, kind="video" if i % 2 == 0 else "gradient", alpha="ramp").numpy() for i in range(F)])
    try:
        for k, (comp, chunks, index, offsets) in enumerate([(HapCompressorSnappy, 1, 0, 0), (HapCompressorSnappy, 8, 0, 0),
                                                            (HapCompressorSnappy, 8, 1, 0), (HapCompressorSnappy, 8, 0, 1),
                                                            (HapCompressorNone, 1, 0, 0)]):
            lib.set_option(lib.OPTION_WRITE_INDEX, index)
            lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, offsets)
            frames, istride, used = encode_frames(lib, pics, c, comp, chunks)
            before = frames.cpu().numpy()
            cs = k % 4
            rgba, rres, out, yres = decode_both(lib, frames, F, istride, used, c, w, h, layout, cs, k)
            assert (rres == 0).all() and (yres == rres).all(), (comp, chunks, index, offsets, rres, yres)
            out.check(rgba, cs, (comp, chunks, index, offsets))
            assert (frames.cpu().numpy() == before).all()
    finally:
        lib.set_option(lib.OPTION_WRITE_INDEX, 0)
        lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def test_decode_yuv_batch_of_the_reference_frames(lib):
    """frames the reference's encoder wrote: 4096 blocks each, decoded as 256 x 256 pictures"""
    names = {"dxt1": "Hap1", "dxt5": "Hap5", "ycocg": "HapY", "rgtc1": "HapA", "hapm": "HapM"}
    w = h = 256
    for name, e in golden()["ref_frames"].items():
        c = CODECS[names[name]]
        fr = np.frombuffer(b64(e["frame_b64"]), np.uint8)
        frames = dev(fr)
        used = torch.tensor([fr.size], dtype=torch.int64, device="cuda")
        for layout in Y.LAYOUTS:
            for cs in Y.COLOR_SPACES:
                rgba, rres, out, yres = decode_both(lib, frames, 1, fr.size, used, c, w, h, layout, cs, cs)
                assert rres[0] == 0 and yres[0] == 0, (name, rres, yres)
                out.check(rgba, cs, (name, layout, cs))
                # the single-frame call, host frame, tight planes
                r, planes = lib.decode_yuv(fr.tobytes(), w, h, layout, cs)
                lu, ch = O.rgba_to_yuv_out(rgba[0], layout, cs)
                assert r == 0 and planes == (lu.tobytes(), ch.tobytes()), (name, layout, cs)


def test_decode_yuv_batch_mixed_good_truncated_and_wrong_codec(lib):
    w, h = 132, 68
    c = L.HapB200Codec_HapY
    pics = np.stack([synth.frame(w, h, i).numpy() for i in range(4)])
    good, gstride, gused = encode_frames(lib, pics, c, HapCompressorSnappy, 4)
    other, ostride_, oused = encode_frames(lib, pics[:1], L.HapB200Codec_Hap1, HapCompressorSnappy, 4)
    istride = max(gstride, ostride_)
    F = 6
    buf = torch.zeros(F * istride, dtype=torch.uint8, device="cuda")
    lens = []
    # frames: good, truncated, good, wrong codec (Hap1 in a Hap Q stream), truncated to a header, good
    plan = [("good", 0), ("trunc", 1), ("good", 2), ("wrong", 0), ("head", 3), ("good", 3)]
    for f, (kind, src) in enumerate(plan):
        if kind == "wrong":
            n = int(oused[0])
            buf[f * istride: f * istride + n] = other[:n]
        else:
            n = int(gused[src])
            buf[f * istride: f * istride + n] = good[src * gstride: src * gstride + n]
            n = n // 2 if kind == "trunc" else 8 if kind == "head" else n
        lens.append(n)
    used = torch.tensor(lens, dtype=torch.int64, device="cuda")
    for layout in Y.LAYOUTS:
        for cs in Y.COLOR_SPACES:
            rgba, rres, out, yres = decode_both(lib, buf, F, istride, used, c, w, h, layout, cs, cs)
            assert (yres == rres).all(), (rres, yres)
            ok = np.array([k == "good" for k, _ in plan])
            assert (rres[ok] == 0).all() and (rres[~ok] != 0).all(), rres
            assert (rgba[~ok] == 0).all()
            out.check(rgba, cs, (layout, cs))
            # failed frames are black: Y = yOff, Cb = Cr = cOff
            yb, cb = O.black(layout, cs)
            got = out.d.cpu().numpy()
            for f in np.flatnonzero(~ok):
                lum = np.lib.stride_tricks.as_strided(got[f * out.fstride:], shape=(h, out.sb * w), strides=(out.pitch, 1))
                chm = np.lib.stride_tricks.as_strided(got[out.chroma_at + f * out.fstride:], shape=(h // 2, out.sb * w), strides=(out.pitch, 1))
                dt = np.uint16 if layout == Y.P010 else np.uint8
                s = 6 if layout == Y.P010 else 0
                assert (np.ascontiguousarray(lum).view(dt) == yb << s).all() and (np.ascontiguousarray(chm).view(dt) == cb << s).all()


def test_yuv_decode_batch_of_65537_frames(lib):
    """4x4 pictures, 65537 of them: two launches (65535 + 2 frames)"""
    w, h, F = 4, 4, 65537
    for layout in Y.LAYOUTS:
        sb = Y.sample_bytes(layout)
        pitch, fstride, chroma_at = 16, 96, 64
        for codec in ("Hap1", "Hap7"):
            c = CODECS[codec]
            t = textures(lib, w, h, c, F, seed=layout)
            blk = dev(np.pad(t, ((0, 0), (0, 16 - t.shape[1]))).ravel())
            out = Out(F, w, h, layout, pitch, fstride, chroma_at)
            assert lib.block_decode_yuv_batch(blk.data_ptr(), F, 16, w, h, c, out.luma, out.chroma, fstride, pitch, layout, Y.BT709_LIMITED) == 0
            out.check(rgba_of_blocks(lib, blk, F, 16, w, h, c), Y.BT709_LIMITED, codec)
        # whole frames, Hap Q: seven distinct pictures repeat
        c = CODECS["HapY"]
        pics = np.stack([synth.frame(w, h, i).numpy() for i in range(7)])
        frames7, istride, used7 = encode_frames(lib, pics, c, HapCompressorSnappy, 1)
        idx = torch.arange(F, device="cuda") % 7
        frames = frames7.view(7, istride)[idx].reshape(-1)
        used = used7[idx]
        rgba, rres, out, yres = decode_both(lib, frames, F, istride, used, c, w, h, layout, Y.BT601_FULL, 0)
        assert (rres == 0).all() and (yres == 0).all()
        out.check(rgba, Y.BT601_FULL, "HapY frames")
        del out, frames


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_decode_yuv_single_frame_host_and_device_unaligned(lib, codec, layout):
    c = CODECS[codec]
    w, h = 132, 68
    sb = Y.sample_bytes(layout)
    pitch = sb * w + 7                                                     # odd: the single-frame call copies
    pics = synth.frame(w, h, 3, alpha="ramp").numpy()[None]
    frames, _, used = encode_frames(lib, pics, c, HapCompressorSnappy, 4)
    fr = frames[: int(used[0])].cpu().numpy()
    r, rgba = lib.decode_rgba(fr.tobytes(), w, h)
    assert r == 0
    rgba = np.frombuffer(rgba, np.uint8).reshape(h, w, 4)
    for cs in Y.COLOR_SPACES:
        lu, ch = O.rgba_to_yuv_out(rgba, layout, cs)
        want_l, want_c = Y.pitched(lu, pitch, PAD), Y.pitched(ch, pitch, PAD)
        # host frame and planes at odd addresses
        hf = np.zeros(fr.size + 1, np.uint8)[1:]
        hf[:] = fr
        hl = np.full(want_l.size + 1, PAD, np.uint8)[1:]
        hc = np.full(want_c.size + 3, PAD, np.uint8)[3:]
        r, _ = lib.decode_yuv(hf, w, h, layout, cs, pitch=pitch, luma=hl, chroma=hc)
        assert r == 0 and (hl == want_l.ravel()).all() and (hc == want_c.ravel()).all(), cs
        # device frame and planes at odd addresses
        df = dev(np.concatenate([[0, 0, 0, 0, 0], fr]).astype(np.uint8))
        dl = torch.full((want_l.size + 1,), PAD, dtype=torch.uint8, device="cuda")
        dc = torch.full((want_c.size + 3,), PAD, dtype=torch.uint8, device="cuda")
        r, _ = lib.decode_yuv((df.data_ptr() + 5, fr.size), w, h, layout, cs, pitch=pitch, luma=(dl.data_ptr() + 1, want_l.size),
                              chroma=(dc.data_ptr() + 3, want_c.size))
        assert r == 0 and (dl.cpu().numpy()[1:] == want_l.ravel()).all() and (dc.cpu().numpy()[3:] == want_c.ravel()).all(), cs
        assert (df.cpu().numpy()[5:] == fr).all()
        # tight default pitch, planes allocated by the wrapper
        r, planes = lib.decode_yuv(fr.tobytes(), w, h, layout, cs)
        assert r == 0 and planes == (lu.tobytes(), ch.tobytes()), cs


def test_decode_yuv_answers_as_decode_rgba_for_hap_hdr_and_bad_frames(lib):
    w, h = 16, 8
    half = np.zeros((h, w, 4), np.float16)
    half[..., :3] = 0.5
    r, hdr = lib.encode_rgba_half(half.view(np.uint8), w, h, 0x8E8F)     # HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT
    assert r == 0
    for frame in (hdr, b"\x00\x00\x00\xbb", b"\x01"):
        want, _ = lib.decode_rgba(frame, w, h)
        for layout in Y.LAYOUTS:
            r, _ = lib.decode_yuv(frame, w, h, layout, Y.BT709_LIMITED)
            assert r == want != 0, (frame[:8], r, want)
    assert lib.decode_rgba(hdr, w, h)[0] == BAD_FRAME
