"""Hap R (BC7) from NV12 / P010 and planar Y'CbCr pictures on the GPU (HapB200EncodeYUVBC7*, HapB200EncodePlanarBC7*).
The textures must equal, byte for byte, those HapB200BlockEncodeBC7Batch gives for the RGBA8 picture the numpy definitions
(tests/yuv_util.py, tests/planar_util.py) make of the same picture: NV12 / P010 in every colour space, and every planar
subsampling and depth with and without alpha, from pitched and strided planes, with the padding of the output untouched.
Frames (chunks 1-8, None / Snappy, index and offset table on and off) report one RGBA_BPTC_UNORM texture that unwraps to
those blocks here, in the CPU oracle and in the reference build when present.  The single-frame calls equal frame 0 of the
batch from host, pitched host and unaligned device memory; a batch that spans more than one slice of the RGBA8 scratch
equals frame-by-frame calls; a NULL alpha decodes with A = 255; and flat pictures made by HapB200DecodePlanar return byte
for byte through HapB200EncodePlanarBC7.  Small pictures throughout: the BC7 search is slow."""
import numpy as np
import pytest
import torch

import hap_b200
import oracles
import planar_util as P
import yuv_util as Y
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
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda()


def host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy()


def plane_buffer(planes, pitch, fstride):
    """frames of one plane ((rows, n) uint8 or uint16) -> device bytes, rows `pitch` apart, frames `fstride` apart, padding PAD"""
    rows = planes[0].shape[0]
    row_bytes = planes[0].view(np.uint8).reshape(rows, -1).shape[1]
    buf = np.full((len(planes) - 1) * fstride + (rows - 1) * pitch + row_bytes, PAD, np.uint8)
    for f, p in enumerate(planes):
        b = np.ascontiguousarray(p).view(np.uint8).reshape(rows, -1)
        for y in range(rows):
            buf[f * fstride + y * pitch: f * fstride + y * pitch + row_bytes] = b[y]
    return dev(buf)


def rgba_blocks(lib, pics):
    """HapB200BlockEncodeBC7Batch on tight RGBA8 pictures -> list of textures"""
    F, (h, w) = len(pics), pics[0].shape[:2]
    t0 = (w // 4) * (h // 4) * 16
    src = dev(np.stack(pics))
    out = torch.zeros(F * align16(t0), dtype=torch.uint8, device="cuda")
    assert lib.block_encode_bc7_batch(src.data_ptr(), F, 4 * w * h, w, h, out.data_ptr(), align16(t0)) == 0
    o = host(out)
    return [o[f * align16(t0): f * align16(t0) + t0].tobytes() for f in range(F)]


def blocks_out(F, w, h, extra=48):
    t0 = (w // 4) * (h // 4) * 16
    bstride = align16(t0) + extra
    return t0, bstride, torch.full(((F - 1) * bstride + t0,), PAD, dtype=torch.uint8, device="cuda")


def split_blocks(out, F, t0, bstride):
    o = host(out)
    clean = all((o[f * bstride + t0: (f + 1) * bstride] == PAD).all() for f in range(F - 1))
    return [o[f * bstride: f * bstride + t0].tobytes() for f in range(F)], clean


# ---- the pictures: frames of planes, their device buffers and their RGBA8 pictures -----------------------------------------

class YuvPictures:
    def __init__(self, rng, F, w, h, layout, cs, pad=16):
        self.w, self.h, self.layout, self.cs, self.F = w, h, layout, cs, F
        self.frames = [Y.random_planes(rng, w, h, layout) for _ in range(F)]
        self.pitch = align16(Y.sample_bytes(layout) * w) + pad   # the batch calls take 16-byte aligned pitches
        self.fstride = align16(h * self.pitch) + 32
        self.luma = plane_buffer([f[0] for f in self.frames], self.pitch, self.fstride)
        self.chroma = plane_buffer([f[1] for f in self.frames], self.pitch, self.fstride)
        self.bufs = [self.luma, self.chroma]

    def rgba(self):
        return [Y.yuv_to_rgba(l, c, self.layout, self.cs) for l, c in self.frames]

    def block_encode(self, lib, blocks, bstride, frames=None):
        return lib.block_encode_yuv_bc7_batch(self.luma.data_ptr(), self.chroma.data_ptr(), frames or self.F, self.fstride, self.w, self.h,
                                              self.pitch, self.layout, self.cs, blocks, bstride)

    def encode_batch(self, lib, comp, k, out, ostride, used):
        return lib.encode_yuv_bc7_batch(self.luma.data_ptr(), self.chroma.data_ptr(), self.F, self.fstride, self.w, self.h, self.pitch,
                                        self.layout, self.cs, comp, k, out, ostride, used)

    def single(self, lib, comp, k, f=0, **kw):
        l, c = self.frames[f]
        return lib.encode_yuv_bc7(l, c, self.w, self.h, self.layout, self.cs, comp, k, **kw)

    def single_pitched(self, lib, comp, k, where):
        """frame 0 with rows pitch + 24 bytes apart, from host memory or from device memory at an odd address"""
        pitch = self.pitch + 24
        bufs = [Y.pitched(p, pitch) for p in self.frames[0]]
        if where == "host":
            return lib.encode_yuv_bc7(bufs[0], bufs[1], self.w, self.h, self.layout, self.cs, comp, k, pitch=pitch)
        d = [dev(np.concatenate([np.zeros(3, np.uint8), b.reshape(-1)])) for b in bufs]
        cap = lib.max_encoded_length_rgba(self.w, self.h, HapB200Codec_Hap7, k)
        out = torch.zeros(cap + 5, dtype=torch.uint8, device="cuda")
        r, n = lib.encode_yuv_bc7((d[0].data_ptr() + 3, d[0].numel() - 3), (d[1].data_ptr() + 3, d[1].numel() - 3), self.w, self.h,
                                  self.layout, self.cs, comp, k, pitch=pitch, out=(out.data_ptr() + 5, cap), out_capacity=cap)
        return r, (host(out)[5: 5 + n].tobytes() if r == 0 else None)


class PlanarPictures:
    def __init__(self, rng, F, w, h, sub, n, cs, alpha, lpad=16, cpad=48):
        self.w, self.h, self.sub, self.n, self.cs, self.F, self.alpha = w, h, sub, n, cs, F, alpha
        self.frames = [P.random_planes(rng, w, h, sub, n, alpha=alpha) for _ in range(F)]
        ch, cw = P.chroma_shape(w, h, sub)
        sb = P.sample_bytes(n)
        self.lp, self.cp = align16(sb * w) + lpad, align16(sb * cw) + cpad
        self.fstride = align16(h * max(self.lp, self.cp)) + 32
        self.bufs = [plane_buffer([f[i] for f in self.frames], self.lp if i in (0, 3) else self.cp, self.fstride) for i in range(3)]
        self.bufs.append(plane_buffer([f[3] for f in self.frames], self.lp, self.fstride) if alpha else None)

    def ptrs(self):
        return [0 if b is None else b.data_ptr() for b in self.bufs]

    def rgba(self):
        return [P.planar_to_rgba(*f, self.sub, self.n, self.cs) for f in self.frames]

    def block_encode(self, lib, blocks, bstride, frames=None):
        return lib.block_encode_planar_bc7_batch(*self.ptrs(), frames or self.F, self.fstride, self.w, self.h, self.lp, self.cp, self.sub,
                                                 self.n, self.cs, blocks, bstride)

    def encode_batch(self, lib, comp, k, out, ostride, used):
        return lib.encode_planar_bc7_batch(*self.ptrs(), self.F, self.fstride, self.w, self.h, self.lp, self.cp, self.sub, self.n, self.cs,
                                           comp, k, out, ostride, used)

    def single(self, lib, comp, k, f=0, **kw):
        return lib.encode_planar_bc7(*self.frames[f], self.w, self.h, self.sub, self.n, self.cs, comp, k, **kw)

    def single_pitched(self, lib, comp, k, where):
        lp, cp = self.lp + 24, self.cp + 8
        bufs = [None if p is None else Y.pitched(p, lp if i in (0, 3) else cp) for i, p in enumerate(self.frames[0])]
        if where == "host":
            return lib.encode_planar_bc7(*bufs, self.w, self.h, self.sub, self.n, self.cs, comp, k, luma_pitch=lp, chroma_pitch=cp)
        d = [None if b is None else dev(np.concatenate([np.zeros(3, np.uint8), b.reshape(-1)])) for b in bufs]
        cap = lib.max_encoded_length_rgba(self.w, self.h, HapB200Codec_Hap7, k)
        out = torch.zeros(cap + 5, dtype=torch.uint8, device="cuda")
        r, n = lib.encode_planar_bc7(*[None if t is None else (t.data_ptr() + 3, t.numel() - 3) for t in d], self.w, self.h, self.sub,
                                     self.n, self.cs, comp, k, luma_pitch=lp, chroma_pitch=cp, out=(out.data_ptr() + 5, cap),
                                     out_capacity=cap)
        return r, (host(out)[5: 5 + n].tobytes() if r == 0 else None)


def check_blocks(lib, pics, what):
    t0, bstride, out = blocks_out(pics.F, pics.w, pics.h)
    assert pics.block_encode(lib, out.data_ptr(), bstride) == 0, what
    texs, clean = split_blocks(out, pics.F, t0, bstride)
    assert clean, what
    want = rgba_blocks(lib, pics.rgba())
    for f in range(pics.F):
        assert texs[f] == want[f], (what, f)
    return texs


# ---- the blocks -------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("cs", Y.COLOR_SPACES)
@pytest.mark.parametrize("layout", Y.LAYOUTS)
def test_yuv_bc7_blocks_equal_the_rgba8_encoder_on_the_converted_picture(lib, layout, cs):
    rng = np.random.default_rng(10 * layout + cs)
    for w, h in ((4, 4), (36, 20), (132, 68)):
        check_blocks(lib, YuvPictures(rng, 3, w, h, layout, cs, pad=16 * (1 + cs % 3)), (layout, cs, w, h))


@pytest.mark.parametrize("alpha", [True, False], ids=["alpha", "no-alpha"])
@pytest.mark.parametrize("n", P.DEPTHS)
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_planar_bc7_blocks_equal_the_rgba8_encoder_on_the_converted_picture(lib, sub, n, alpha):
    rng = np.random.default_rng(100 * sub + n + alpha)
    for i, (w, h) in enumerate(((4, 4), (36, 20), (132, 68))):
        check_blocks(lib, PlanarPictures(rng, 3, w, h, sub, n, (sub + n + i) % 4, alpha), (sub, n, alpha, w, h))


# ---- frames -----------------------------------------------------------------------------------------------------------------

@pytest.fixture(params=[(0, 0), (1, 0), (0, 1), (1, 1)], ids=["plain", "index", "offsets", "index+offsets"])
def layout_opts(lib, request):
    lib.set_option(lib.OPTION_WRITE_INDEX, request.param[0])
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, request.param[1])
    yield request.param
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def encode_frames(lib, pics, comp, k):
    ostride = align16(lib.max_encoded_length_rgba(pics.w, pics.h, HapB200Codec_Hap7, k))
    out = torch.zeros(pics.F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(pics.F, dtype=torch.int64, device="cuda")
    assert pics.encode_batch(lib, comp, k, out.data_ptr(), ostride, used.data_ptr()) == 0
    o, nb = host(out), host(used)
    return [o[f * ostride: f * ostride + int(nb[f])].tobytes() for f in range(pics.F)]


def picture_sets(rng):
    return [YuvPictures(rng, 2, 132, 68, Y.NV12, Y.BT709_LIMITED), YuvPictures(rng, 2, 36, 20, Y.P010, Y.BT601_FULL),
            PlanarPictures(rng, 2, 132, 68, P.S444, 12, Y.BT709_FULL, True), PlanarPictures(rng, 2, 36, 20, P.S422, 10, Y.BT601_LIMITED, False)]


def test_batch_frames_unwrap_to_the_blocks(lib, layout_opts):
    ref = oracles.ref_abi()
    orc = oracles.oracle_abi()
    for pics in picture_sets(np.random.default_rng(7)):
        texs = rgba_blocks(lib, pics.rgba())
        for comp in (HapCompressorNone, HapCompressorSnappy):
            for k in range(1, 9):
                frames = encode_frames(lib, pics, comp, k)
                for f, fr in enumerate(frames):
                    assert lib.texture_count(fr) == (0, 1) and lib.texture_format(fr, 0) == (0, FMT), (pics.w, comp, k, f)
                    for who in (lib, orc) + ((ref,) if ref is not None else ()):
                        r, tex, tf, _ = who.decode(fr, 0, out_capacity=len(texs[f]))
                        assert r == 0 and tex == texs[f] and tf == FMT, (pics.w, comp, k, f)


def test_single_frame_calls_equal_frame_0_of_the_batch(lib):
    for i, pics in enumerate(picture_sets(np.random.default_rng(8))):
        k = 1 + 2 * i
        comp = HapCompressorSnappy if i % 2 == 0 else HapCompressorNone
        batch = encode_frames(lib, pics, comp, k)[0]
        r, fr = pics.single(lib, comp, k)
        assert r == 0 and fr == batch, i
        for where in ("host", "device"):
            r, fr = pics.single_pitched(lib, comp, k, where)
            assert r == 0 and fr == batch, (i, where)
        cap = lib.max_encoded_length_rgba(pics.w, pics.h, HapB200Codec_Hap7, k)
        assert pics.single(lib, comp, k, out=bytearray(cap), out_capacity=cap - 1)[0] == BUFFER_TOO_SMALL


def test_batch_over_several_scratch_slices_equals_frame_by_frame_calls(lib):
    # 64 x 64 frames: 16 KiB of RGBA8 each, so the 256 MiB scratch holds 16384 of them and this batch takes two slices.  The
    # frames cycle through 41 distinct pictures, so a slice that read or wrote another slice's frames would show.
    w, h, distinct, F = 64, 64, 41, 16384 + 123
    rng = np.random.default_rng(64)
    for pics in (YuvPictures(rng, distinct, w, h, Y.NV12, Y.BT709_LIMITED, pad=0),
                 PlanarPictures(rng, distinct, w, h, P.S444, 12, Y.BT601_FULL, True, lpad=0, cpad=0)):
        t0 = (w // 4) * (h // 4) * 16
        singles = []
        for f in range(distinct):
            out = torch.full((t0,), PAD, dtype=torch.uint8, device="cuda")
            # frame f alone: the planes from frame f on, a batch of one
            if isinstance(pics, YuvPictures):
                r = lib.block_encode_yuv_bc7_batch(pics.luma.data_ptr() + f * pics.fstride, pics.chroma.data_ptr() + f * pics.fstride, 1,
                                                   pics.fstride, w, h, pics.pitch, pics.layout, pics.cs, out.data_ptr(), t0)
            else:
                p = [q and q + f * pics.fstride for q in pics.ptrs()]
                r = lib.block_encode_planar_bc7_batch(*p, 1, pics.fstride, w, h, pics.lp, pics.cp, pics.sub, pics.n, pics.cs, out.data_ptr(),
                                                      t0)
            assert r == 0, f
            singles.append(host(out).tobytes())
        assert singles == rgba_blocks(lib, pics.rgba())
        # the big batch: every plane repeats its 41 frames
        idx = torch.arange(F, device="cuda") % distinct
        big = []
        for b in pics.bufs:
            if b is None:
                big.append(None)
                continue
            padded = torch.full((distinct * pics.fstride,), PAD, dtype=torch.uint8, device="cuda")
            padded[: b.numel()] = b
            big.append(padded.view(distinct, pics.fstride)[idx].reshape(-1))
        out = torch.full((F * t0,), PAD, dtype=torch.uint8, device="cuda")
        if isinstance(pics, YuvPictures):
            r = lib.block_encode_yuv_bc7_batch(big[0].data_ptr(), big[1].data_ptr(), F, pics.fstride, w, h, pics.pitch, pics.layout, pics.cs,
                                               out.data_ptr(), t0)
        else:
            r = lib.block_encode_planar_bc7_batch(*[0 if b is None else b.data_ptr() for b in big], F, pics.fstride, w, h, pics.lp, pics.cp,
                                                  pics.sub, pics.n, pics.cs, out.data_ptr(), t0)
        assert r == 0
        got = host(out).reshape(F, t0)
        for f in range(F):
            if got[f].tobytes() != singles[f % distinct]:
                pytest.fail(f"{type(pics).__name__}: frame {f} of {F} differs from the frame-by-frame call")
        del big, out


def test_null_alpha_decodes_opaque(lib):
    rng = np.random.default_rng(9)
    w, h = 132, 68
    for sub in P.SUBSAMPLINGS:
        for n in P.DEPTHS:
            luma, cb, cr, alpha = P.random_planes(rng, w, h, sub, n)
            r, fr = lib.encode_planar_bc7(luma, cb, cr, None, w, h, sub, n, Y.BT709_LIMITED, HapCompressorSnappy, 2)
            assert r == 0, (sub, n)
            r, pix = lib.decode_rgba(fr, w, h)
            assert r == 0 and (np.frombuffer(pix, np.uint8).reshape(h, w, 4)[..., 3] == 255).all(), (sub, n)
            # with the alpha plane, the same picture keeps its alpha (random alpha is not all 255)
            r, fr = lib.encode_planar_bc7(luma, cb, cr, alpha, w, h, sub, n, Y.BT709_LIMITED, HapCompressorSnappy, 2)
            r2, pix = lib.decode_rgba(fr, w, h)
            assert r == 0 and r2 == 0 and (np.frombuffer(pix, np.uint8).reshape(h, w, 4)[..., 3] != 255).any(), (sub, n)


@pytest.mark.parametrize("fmt", ["yuva444p12le", "yuv420p10le"])
def test_flat_pictures_from_the_planar_decoder_return_byte_for_byte(lib, fmt):
    sub, n, with_alpha = (P.S444, 12, True) if fmt == "yuva444p12le" else (P.S420, 10, False)
    w, h = 36, 20
    rng = np.random.default_rng(11)
    colours = [(0, 0, 0, 255), (255, 255, 255, 255), (255, 0, 0, 255), (12, 200, 77, 255)] + \
              [tuple(int(v) for v in rng.integers(0, 256, 4)) for _ in range(8)]
    for cs in Y.COLOR_SPACES:
        for c in colours:
            c = c if with_alpha else c[:3] + (255,)
            img = np.empty((h, w, 4), np.uint8)
            img[:] = c
            r, frame = lib.encode_rgba_bc7(img, w, h, HapCompressorSnappy, 1)
            assert r == 0
            r, planes = lib.decode_planar(frame, w, h, sub, n, cs, with_alpha=with_alpha)
            assert r == 0, (cs, c)
            r, frame2 = lib.encode_planar_bc7(*[None if p is None else bytearray(p) for p in planes], w, h, sub, n, cs, HapCompressorSnappy, 1)
            assert r == 0, (cs, c)
            r, planes2 = lib.decode_planar(frame2, w, h, sub, n, cs, with_alpha=with_alpha)
            assert r == 0 and planes2 == planes, (fmt, cs, c)
