"""Planar Y'CbCr encoders on the GPU (HapB200BlockEncodePlanarBatch, HapB200EncodePlanarBatch, HapB200EncodePlanar): every
texture and frame must equal, byte for byte, what the RGBA8 encoders give for the picture planar_util.planar_to_rgba (the
definition of include/hap_b200.h) makes of the same planes -- for every codec, subsampling, depth and colour space, with
and without alpha, with chroma refinement, Snappy chunking, the index and offset-table options and uncompressed frames, at
odd block widths, pitches wider than the row, frame-stride slack, chroma planes away from luma, unaligned single-frame
planes and a batch of more than 65535 frames.  Sentinels around every texture and frame must survive, and the planes must
be left as they were."""
import numpy as np
import pytest
import torch

import hap_b200
import hap_b200.lib as L
import planar_util as P
import yuv_util as Y
from hap_b200 import synth
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy

pytestmark = pytest.mark.gpu
PAD = 0xEE
CODECS = {"Hap1": L.HapB200Codec_Hap1, "Hap5": L.HapB200Codec_Hap5, "HapY": L.HapB200Codec_HapY, "HapM": L.HapB200Codec_HapM,
          "HapA": L.HapB200Codec_HapA}
CASES = [(c, sub, n, cs, alpha, 0) for c in CODECS for sub in P.SUBSAMPLINGS for n in P.DEPTHS for cs in P.COLOR_SPACES
         for alpha in (False, True)] + \
        [(c, sub, n, cs, alpha, 1) for c in ("HapY", "HapM") for sub in P.SUBSAMPLINGS for n in P.DEPTHS for cs in P.COLOR_SPACES
         for alpha in (False, True)]
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


def pictures(w, h, sub, n, cs, count=3, seed=0, alpha=True):
    """count (luma, cb, cr, alpha or None) pictures: video content converted, random samples (16-bit words: junk above the
    sample), a steep gradient"""
    rng = np.random.default_rng(seed + 7919 * w + h)
    out = []
    for i in range(count):
        if i % 3 == 1:
            out.append(P.random_planes(rng, w, h, sub, n, alpha=alpha))
        else:
            rgba = synth.frame(w, h, i, kind="video" if i % 3 == 0 else "gradient").numpy().copy()
            rgba[..., 3] = rng.integers(0, 256, (h, w))                          # an alpha with detail
            out.append(P.rgba_to_planar(rgba, sub, n, cs, alpha=alpha))
    return out


class Planes:
    """frames of the four planes, each plane in a device buffer of its own (so chroma lies away from luma): frame f's plane
    at its pointer + f*fstride, luma and alpha rows lpitch apart, Cb and Cr rows cpitch apart; each buffer ends with its
    last sample and every other byte is PAD"""

    def __init__(self, pics, lpitch, cpitch, fstride):
        self.bufs, self.d, self.ptr = [], [], []
        for k in range(4):
            if pics[0][k] is None:
                self.bufs.append(None), self.d.append(None), self.ptr.append(0)
                continue
            pitch = lpitch if k in (0, 3) else cpitch
            rows = [np.ascontiguousarray(p[k]).view(np.uint8).reshape(p[k].shape[0], -1) for p in pics]
            n = (len(pics) - 1) * fstride + (rows[0].shape[0] - 1) * pitch + rows[0].shape[1]
            buf = np.full(n, PAD, np.uint8)
            for f, r in enumerate(rows):
                view = np.lib.stride_tricks.as_strided(buf[f * fstride:], shape=r.shape, strides=(pitch, 1))
                view[...] = r
            self.bufs.append(buf)
            self.d.append(dev(buf))
            self.ptr.append(self.d[-1].data_ptr())

    def unchanged(self) -> bool:
        return all(b is None or (d.cpu().numpy() == b).all() for b, d in zip(self.bufs, self.d))


def rgba_batch(pics, sub, n, cs):
    """the RGBA8 pictures of the definition, tight, one after another on the device"""
    rgba = np.stack([P.planar_to_rgba(*p, sub, n, cs) for p in pics])
    return rgba, dev(rgba)


def geometry(w, h, sub, n, lslack=32, cslack=16, fslack=64):
    sb = P.sample_bytes(n)
    ch, cw = P.chroma_shape(w, h, sub)
    lpitch, cpitch = align16(sb * w) + lslack, align16(sb * cw) + cslack
    return lpitch, cpitch, align16(max(lpitch * h, cpitch * ch)) + fslack


def block_encode_both(lib, pics, w, h, sub, n, cs, c, lpitch, cpitch, fstride, F):
    """(got, want, texture bytes, block stride, source planes): the planar block encode and the RGBA8 one of the definition"""
    src = Planes(pics, lpitch, cpitch, fstride)
    t = lib.texture_bytes(w, h, c, 0) + lib.texture_bytes(w, h, c, 1)
    bstride = align16(t) + 48
    got = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_planar_batch(*src.ptr, F, fstride, w, h, lpitch, cpitch, sub, n, cs, c, got.data_ptr(), bstride) == 0
    _, rgba = rgba_batch(pics, sub, n, cs)
    want = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_batch(rgba.data_ptr(), F, 4 * w * h, w, h, c, want.data_ptr(), bstride) == 0
    return got.cpu().numpy().reshape(F, bstride), want.cpu().numpy().reshape(F, bstride), t, src


@pytest.mark.parametrize("codec,sub,n,cs,alpha,refine", CASES, indirect=["refine"])
def test_block_encode_planar_batch_equals_rgba(lib, codec, sub, n, cs, alpha, refine):
    c = CODECS[codec]
    w, h, F = 260, 132, 3
    lpitch, cpitch, fstride = geometry(w, h, sub, n)
    pics = pictures(w, h, sub, n, cs, F, seed=cs + 10 * n, alpha=alpha)
    if codec == "HapA" and not alpha:                     # Hap Alpha-Only needs the alpha plane
        src = Planes(pics, lpitch, cpitch, fstride)
        assert lib.block_encode_planar_batch(*src.ptr, F, fstride, w, h, lpitch, cpitch, sub, n, cs, c, src.ptr[0], 4096) == 1
        return
    if codec == "HapA":                                   # ... and reads it alone: the other planes may be absent
        pics = [(None, None, None, p[3]) for p in pics]
        src = Planes(pics, lpitch, cpitch, fstride)
        t = lib.texture_bytes(w, h, c, 0)
        bstride = align16(t) + 48
        got = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_planar_batch(*src.ptr, F, fstride, w, h, lpitch, 0, sub, n, cs, c, got.data_ptr(), bstride) == 0
        rgba = np.zeros((F, h, w, 4), np.uint8)
        rgba[..., 3] = np.stack([P.alpha8(P.samples(p[3], n), n) for p in pics])
        want = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_batch(dev(rgba).data_ptr(), F, 4 * w * h, w, h, c, want.data_ptr(), bstride) == 0
        g, wn = got.cpu().numpy().reshape(F, bstride), want.cpu().numpy().reshape(F, bstride)
    else:
        g, wn, t, src = block_encode_both(lib, pics, w, h, sub, n, cs, c, lpitch, cpitch, fstride, F)
    assert (g[:, :t] == wn[:, :t]).all()
    assert (g[:, t:] == PAD).all()
    assert src.unchanged()


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_encode_planar_batch_frames_equal_rgba(lib, codec, sub):
    c = CODECS[codec]
    w, h, F = 516, 260, 3
    try:
        for k, (comp, chunks, index, offsets) in enumerate([(HapCompressorSnappy, 1, 0, 0), (HapCompressorSnappy, 8, 0, 0),
                                                            (HapCompressorSnappy, 8, 1, 0), (HapCompressorSnappy, 8, 0, 1),
                                                            (HapCompressorNone, 1, 0, 0)]):
            lib.set_option(lib.OPTION_WRITE_INDEX, index)
            lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, offsets)
            cs, n = k % 4, P.DEPTHS[k % 3]
            alpha = codec == "HapA" or k % 2 == 0
            lpitch, cpitch, fstride = geometry(w, h, sub, n, 16, 48, 16)
            pics = pictures(w, h, sub, n, cs, F, seed=k, alpha=alpha)
            src = Planes(pics, lpitch, cpitch, fstride)
            ostride = align16(lib.max_encoded_length_rgba(w, h, c, chunks)) + 32
            got = torch.full((F * ostride,), PAD, dtype=torch.uint8, device="cuda")
            gused = torch.zeros(F, dtype=torch.int64, device="cuda")
            assert lib.encode_planar_batch(*src.ptr, F, fstride, w, h, lpitch, cpitch, sub, n, cs, c, comp, chunks, got.data_ptr(),
                                           ostride, gused.data_ptr()) == 0
            _, rgba = rgba_batch(pics, sub, n, cs)
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
@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_encode_planar_single_frame_host_and_device_unaligned(lib, codec, sub):
    c = CODECS[codec]
    w, h = 132, 68
    for n in P.DEPTHS:
        sb = P.sample_bytes(n)
        ch, cw = P.chroma_shape(w, h, sub)
        lpitch, cpitch = sb * w + 6, sb * cw + 10             # not multiples of 16: the single-frame call copies
        cs = (n + sub) % 4
        planes, = pictures(w, h, sub, n, cs, 1, seed=40 + n)
        r, want = lib.encode_rgba(P.planar_to_rgba(*planes, sub, n, cs), w, h, c, HapCompressorSnappy, 4)
        assert r == 0
        pitched = [Y.pitched(p, lpitch if k in (0, 3) else cpitch) for k, p in enumerate(planes)]
        # host planes at odd addresses
        host = []
        for k, b in enumerate(pitched):
            a = np.zeros(b.size + 1 + 2 * k, np.uint8)[1 + 2 * k:]
            a[:] = b.ravel()
            host.append(a)
        r, got = lib.encode_planar(*host, w, h, sub, n, cs, c, HapCompressorSnappy, 4, luma_pitch=lpitch, chroma_pitch=cpitch)
        assert r == 0 and got == want, (n, cs)
        # device planes at odd addresses
        devs = [dev(np.concatenate([np.zeros(1 + 2 * k, np.uint8), b.ravel()])) for k, b in enumerate(pitched)]
        ptrs = [(d.data_ptr() + 1 + 2 * k, b.size) for k, (d, b) in enumerate(zip(devs, pitched))]
        r, got = lib.encode_planar(*ptrs, w, h, sub, n, cs, c, HapCompressorSnappy, 4, luma_pitch=lpitch, chroma_pitch=cpitch)
        assert r == 0 and got == want, (n, cs)
        # tight default pitches
        r, got = lib.encode_planar(*[np.ascontiguousarray(p) for p in planes], w, h, sub, n, cs, c, HapCompressorSnappy, 4)
        assert r == 0 and got == want, (n, cs)
        if codec == "HapA":                                   # alpha alone
            r, got = lib.encode_planar(None, None, None, host[3], w, h, sub, n, cs, c, HapCompressorSnappy, 4, luma_pitch=lpitch)
            assert r == 0 and got == want, (n, cs)


@pytest.mark.parametrize("sub", P.SUBSAMPLINGS)
def test_block_encode_planar_geometry(lib, sub):
    """the shapes of test_gpu_geometry.py, with pitches wider than the row, frame-stride slack and each plane in a buffer of
    its own"""
    for i, (w, h) in enumerate(SHAPES):
        n = P.DEPTHS[i % 3]
        for codec in ("Hap1", "HapM"):
            c = CODECS[codec]
            F, cs = 3, i % 4
            lpitch, cpitch, fstride = geometry(w, h, sub, n, 16 * (i % 3), 16 * ((i + 1) % 3), 16 * (1 + i % 2))
            pics = pictures(w, h, sub, n, cs, F, seed=i, alpha=i % 2 == 0)
            g, wn, t, src = block_encode_both(lib, pics, w, h, sub, n, cs, c, lpitch, cpitch, fstride, F)
            assert (g[:, :t] == wn[:, :t]).all(), (w, h, codec)
            assert (g[:, t:] == PAD).all(), (w, h, codec)
            assert src.unchanged(), (w, h, codec)


def test_planar_batch_of_65537_frames(lib):
    """4x4 pictures, 65537 of them: two launches (65535 + 2 frames); seven distinct pictures repeat"""
    w, h, F = 4, 4, 65537
    pitch, fstride = 16, 64
    for sub, n in ((P.S420, 8), (P.S422, 10), (P.S444, 12)):
        distinct = pictures(w, h, sub, n, Y.BT709_LIMITED, 7, seed=sub)
        one = Planes(distinct, pitch, pitch, fstride)
        idx = np.arange(F) % 7
        ptrs, keep = [], []
        for b in one.bufs:
            full = np.full(7 * fstride, PAD, np.uint8)
            full[: b.size] = b
            tiles = full.reshape(7, fstride)
            last = b.size - 6 * fstride
            buf = np.concatenate([tiles[idx[:-1]].ravel(), tiles[idx[-1], :last]])
            keep.append(dev(buf))
            ptrs.append(keep[-1].data_ptr())
        rgba7, _ = rgba_batch(distinct, sub, n, Y.BT709_LIMITED)
        rgba = dev(rgba7[idx])
        for codec in ("Hap1", "HapM", "HapA"):
            c = CODECS[codec]
            t = lib.texture_bytes(w, h, c, 0) + lib.texture_bytes(w, h, c, 1)
            got = torch.full((F * 32,), PAD, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_planar_batch(*ptrs, F, fstride, w, h, pitch, pitch, sub, n, Y.BT709_LIMITED, c, got.data_ptr(), 32) == 0
            want = torch.full((F * 32,), PAD, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_batch(rgba.data_ptr(), F, 64, w, h, c, want.data_ptr(), 32) == 0
            assert torch.equal(got, want), codec
            assert (got.view(F, 32)[:, t:] == PAD).all()
        # whole frames, Hap Q Alpha
        c = CODECS["HapM"]
        ostride = align16(lib.max_encoded_length_rgba(w, h, c, 1))
        got = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
        gused = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_planar_batch(*ptrs, F, fstride, w, h, pitch, pitch, sub, n, Y.BT709_LIMITED, c, HapCompressorSnappy, 1,
                                       got.data_ptr(), ostride, gused.data_ptr()) == 0
        want = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
        wused = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_rgba_batch(rgba.data_ptr(), F, 64, w, h, c, HapCompressorSnappy, 1, want.data_ptr(), ostride, wused.data_ptr()) == 0
        assert torch.equal(gused, wused) and torch.equal(got, want)


@pytest.mark.parametrize("n", (8, 10))
def test_yuv420p_equals_the_semi_planar_encoder(lib, n):
    """HapY from yuv420p (yuv420p10le) equals HapB200EncodeYUV from the NV12 (P010) of the same samples"""
    w, h, F = 516, 260, 2
    layout = Y.NV12 if n == 8 else Y.P010
    sb = P.sample_bytes(n)
    for codec in ("HapY", "Hap1", "HapM"):
        c = CODECS[codec]
        for cs in P.COLOR_SPACES:
            pics = pictures(w, h, P.S420, n, cs, F, seed=cs, alpha=False)
            lpitch, cpitch, fstride = geometry(w, h, P.S420, n, 0, 0, 0)
            src = Planes(pics, lpitch, cpitch, fstride)
            # the NV12 / P010 planes: interleaved chroma, samples << 6 for P010, one pitch
            word = (lambda p: (P.samples(p, 10) << 6).astype(np.uint16)) if n == 10 else (lambda p: p)
            semi = [(word(l), np.stack([word(b), word(r)], -1).reshape(h // 2, w)) for l, b, r, _ in pics]
            pitch = align16(sb * w)
            sfs = align16(pitch * h * 3 // 2)
            buf = np.zeros(F * sfs, np.uint8)
            for f, (lu, chp) in enumerate(semi):
                buf[f * sfs: f * sfs + pitch * h] = Y.pitched(lu, pitch).ravel()
                buf[f * sfs + pitch * h: f * sfs + pitch * h * 3 // 2] = Y.pitched(chp, pitch).ravel()
            d = dev(buf)
            t = lib.texture_bytes(w, h, c, 0) + lib.texture_bytes(w, h, c, 1)
            bstride = align16(t)
            got = torch.zeros(F * bstride, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_planar_batch(*src.ptr, F, fstride, w, h, lpitch, cpitch, P.S420, n, cs, c, got.data_ptr(), bstride) == 0
            want = torch.zeros(F * bstride, dtype=torch.uint8, device="cuda")
            assert lib.block_encode_yuv_batch(d.data_ptr(), d.data_ptr() + pitch * h, F, sfs, w, h, pitch, layout, cs, c, want.data_ptr(),
                                              bstride) == 0
            assert torch.equal(got, want), (codec, cs)
            # and the whole frame, through the single-frame calls
            r1, f1 = lib.encode_planar(*pics[0], w, h, P.S420, n, cs, c, HapCompressorSnappy, 4)
            r2, f2 = lib.encode_yuv(semi[0][0], semi[0][1], w, h, layout, cs, c, HapCompressorSnappy, 4)
            assert r1 == r2 == 0 and f1 == f2, (codec, cs)


@pytest.mark.parametrize("n", P.DEPTHS)
def test_flat_hapm_round_trip_gives_back_alpha(lib, n):
    w, h = 64, 32
    rng = np.random.default_rng(n)
    for sub in P.SUBSAMPLINGS:
        ch, cw = P.chroma_shape(w, h, sub)
        for a in list(rng.integers(0, 1 << n, 8)) + [0, (1 << n) - 1]:
            flat = lambda v, shape: P.as_plane(np.full(shape, int(v), np.int64), n)
            y, b, r = rng.integers(0, 1 << n, 3)
            planes = (flat(y, (h, w)), flat(b, (ch, cw)), flat(r, (ch, cw)), flat(a, (h, w)))
            res, frame = lib.encode_planar(*planes, w, h, sub, n, Y.BT709_FULL, CODECS["HapM"], HapCompressorSnappy, 1)
            assert res == 0
            res, out = lib.decode_rgba(frame, w, h)
            assert res == 0
            got = np.frombuffer(out, np.uint8).reshape(h, w, 4)[..., 3]
            assert (got == P.alpha8(a, n)).all(), (sub, a)
