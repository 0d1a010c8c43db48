"""The geometry the batch and RGBA entry points accept, on the GPU: odd block widths, row pitches wider than the picture,
strided and repeated frames, block strides wider than the texture, unaligned single-frame pictures, batches of more than
65535 frames, refused geometry, two-texture batch encodes with texture 1 below texture 0, and batch decodes that mix
formats, chunk counts, section kinds, encoders and failing frames.  Every picture, block and frame is compared with the
host build of the block code (twin), the oracle's block decoder, a single-frame call, or the reference; every padding byte
around them must keep its sentinel."""
import numpy as np
import pytest
import torch

import hap_b200
import hap_b200.lib as L
import oracles
import twin
from hap_b200 import synth
from hap_b200.abi import (HapCompressorNone, HapCompressorSnappy, HapTextureFormat_A_RGTC1, HapTextureFormat_RGB_DXT1,
                          HapTextureFormat_RGBA_BPTC_UNORM, HapTextureFormat_RGBA_DXT5, HapTextureFormat_YCoCg_DXT5)

pytestmark = pytest.mark.gpu
DXT1, DXT5, YCOCG, RGTC1, BC7 = (HapTextureFormat_RGB_DXT1, HapTextureFormat_RGBA_DXT5, HapTextureFormat_YCoCg_DXT5,
                                 HapTextureFormat_A_RGTC1, HapTextureFormat_RGBA_BPTC_UNORM)
BAD_ARGUMENTS = 1
PAD = 0xEE
# codec -> (HapB200Codec, block kind of texture 0, block kind of texture 1 or None)
CODECS = {"Hap1": (L.HapB200Codec_Hap1, "bc1", None), "Hap5": (L.HapB200Codec_Hap5, "bc3", None),
          "HapY": (L.HapB200Codec_HapY, "ycocg", None), "HapM": (L.HapB200Codec_HapM, "ycocg", "bc4"),
          "HapA": (L.HapB200Codec_HapA, "bc4", None)}
# odd block widths: warps straddle block rows and inv_blocks_x is not exact
SHAPES = [(w, h) for w in (4, 8, 12, 20, 36, 132, 516) for h in (4, 8, 12, 20)] + [(1924, 1084)]


@pytest.fixture(scope="module")
def lib():
    return hap_b200.load()


def align16(n):
    return (n + 15) // 16 * 16


def dev(a) -> torch.Tensor:
    if isinstance(a, (bytes, bytearray)):
        a = np.frombuffer(a, np.uint8)
    return torch.from_numpy(np.ascontiguousarray(a).copy()).cuda()


def host(t: torch.Tensor) -> np.ndarray:
    return t.cpu().numpy()


def strided(buf, frames, h, w, pitch, fstride):
    """(frames, h, 4w) view of the pictures inside a pitched buffer"""
    return np.lib.stride_tricks.as_strided(buf, shape=(frames, h, 4 * w), strides=(fstride, pitch, 1))


def pitched(pics, pitch, fstride):
    """pictures (F, h, w, 4) -> (buffer exactly as long as the last picture needs, padding = PAD; mask of picture bytes)"""
    F, h, w, _ = pics.shape
    n = (F - 1) * fstride + (h - 1) * pitch + 4 * w
    buf = np.full(n, PAD, np.uint8)
    mask = np.zeros(n, bool)
    strided(buf, F, h, w, pitch, fstride)[...] = pics.reshape(F, h, 4 * w)
    strided(mask, F, h, w, pitch, fstride)[...] = True
    return buf, mask


def pictures(w, h, n=3, seed=0):
    """n distinct pictures: video with an alpha ramp, noise in every channel, steep gradients"""
    rng = np.random.default_rng(seed + w * 7919 + h)
    out = []
    for i in range(n):
        if i % 3 == 1:
            out.append(rng.integers(0, 256, (h, w, 4), dtype=np.uint8))
        else:
            out.append(synth.frame(w, h, i, kind="video" if i % 3 == 0 else "gradient", alpha="ramp").numpy())
    return np.stack(out)


def twin_blocks(codec, pic, refine=False):
    """the blocks the host build of bc_block.cuh gives for one tight picture, planes one after the other"""
    _, k0, k1 = CODECS[codec]
    b = twin.encode("ycocg_refine" if refine and k0 == "ycocg" else k0, pic)
    return b + (twin.encode(k1, pic) if k1 else b"")


def oracle_rgba(codec, t0, t1, w, h):
    """the oracle's block decoder on the texture(s) of one frame -> (h, w, 4), as HapB200DecodeRGBA composes them"""
    _, k0, k1 = CODECS[codec]
    want = oracles.bc_decode(k0, t0, w, h)
    if k0 == "bc4":
        want = np.stack([want, want, want, np.full_like(want, 255)], -1)
    if k1:
        want = want.copy()
        want[..., 3] = oracles.bc_decode("bc4", t1, w, h)
    return want


@pytest.fixture
def refine(lib, request):
    lib.set_option(lib.OPTION_CHROMA_REFINE, request.param)
    yield request.param
    lib.set_option(lib.OPTION_CHROMA_REFINE, 0)


# ---- block codecs, batched ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("codec,refine", [(c, 0) for c in CODECS] + [("HapY", 1), ("HapM", 1)], indirect=["refine"])
def test_block_encode_and_decode_batch_pitched_strided(lib, codec, refine):
    """HapB200BlockEncodeBatch: frame f equals the host build's blocks of tight picture f, the padding of the block slots
    keeps its sentinel, frameStride 0 repeats frame 0.  HapB200BlockDecodeBatch of those blocks, and of random blocks, into
    pitched strided pictures equals the oracle's block decoder and leaves row and frame padding alone."""
    c = CODECS[codec][0]
    rng = np.random.default_rng(17)
    for i, (w, h) in enumerate(SHAPES):
        F = 3
        pitch, fstride = 4 * w + 16 * (i % 3), h * (4 * w + 16 * (i % 3)) + 16 * (1 + i % 2)
        t0, t1 = lib.texture_bytes(w, h, c, 0), lib.texture_bytes(w, h, c, 1)
        bstride = align16(t0 + t1) + 48                                    # wider than the frame's blocks
        pics = pictures(w, h, F, seed=i)
        buf, _ = pitched(pics, pitch, fstride)
        src = dev(buf)
        blocks = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_batch(src.data_ptr(), F, fstride, w, h, c, blocks.data_ptr(), bstride, row_bytes=pitch) == 0, (w, h)
        got = host(blocks).reshape(F, bstride)
        for f in range(F):
            assert got[f, : t0 + t1].tobytes() == twin_blocks(codec, pics[f], refine), (w, h, f)
        assert (got[:, t0 + t1:] == PAD).all(), (w, h)
        # frameStride 0: every frame is picture 0
        rep = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_batch(src.data_ptr(), F, 0, w, h, c, rep.data_ptr(), bstride, row_bytes=pitch) == 0
        rep = host(rep).reshape(F, bstride)
        assert (rep == got[0]).all(), (w, h)

        # decode: the blocks above, then random blocks, into pitched strided pictures
        for source in ("encoded", "random"):
            if source == "random":
                blk = got.copy()
                blk[:, : t0 + t1] = rng.integers(0, 256, (F, t0 + t1), dtype=np.uint8)
            else:
                blk = got
            out = torch.full((len(buf),), PAD, dtype=torch.uint8, device="cuda")
            assert lib.block_decode_batch(dev(blk.reshape(-1)).data_ptr(), F, bstride, w, h, c, out.data_ptr(), fstride,
                                          row_bytes=pitch) == 0
            o = host(out)
            _, mask = pitched(pics, pitch, fstride)
            pix = strided(o, F, h, w, pitch, fstride)
            for f in range(F):
                want = oracle_rgba(codec, blk[f, :t0].tobytes(), blk[f, t0: t0 + t1].tobytes(), w, h)
                assert np.array_equal(pix[f].reshape(h, w, 4), want), (w, h, f, source)
            assert (o[~mask] == PAD).all(), (w, h, source)


# ---- RGBA batches --------------------------------------------------------------------------------------------------------

def encode_batch_pitched(lib, codec, pics, pitch, fstride, comp, k):
    """HapB200EncodeRGBABatch of pictures laid out pitched and strided -> list of frames"""
    F, h, w, _ = pics.shape
    c = CODECS[codec][0]
    buf, _ = pitched(pics, pitch, fstride)
    src = dev(buf)
    ostride = align16(lib.max_encoded_length_rgba(w, h, c, k)) + 32
    out = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    assert lib.encode_rgba_batch(src.data_ptr(), F, fstride, w, h, c, comp, k, out.data_ptr(), ostride, used.data_ptr(), row_bytes=pitch) == 0
    o = host(out)
    return [o[f * ostride: f * ostride + int(used[f])].tobytes() for f in range(F)]


def slots(frames, pad=PAD, extra=16):
    """frames -> (device buffer of one slot per frame, slot stride, device inBytes); bytes behind each frame are `pad`"""
    stride = align16(max(len(f) for f in frames) + extra)
    buf = np.full(len(frames) * stride, pad, np.uint8)
    for i, f in enumerate(frames):
        buf[i * stride: i * stride + len(f)] = np.frombuffer(f, np.uint8)
    return dev(buf), stride, torch.tensor([len(f) for f in frames], dtype=torch.int64, device="cuda")


def decode_rgba_batch_pitched(lib, codec, frames, w, h, pitch, fstride, k, in_bytes=None):
    """HapB200DecodeRGBABatch -> (results, pictures (F, h, w, 4), padding untouched)"""
    F = len(frames)
    d, stride, nb = slots(frames)
    if in_bytes is not None:
        nb = torch.tensor(in_bytes, dtype=torch.int64, device="cuda")
    n = (F - 1) * fstride + (h - 1) * pitch + 4 * w
    out = torch.full((n,), PAD, dtype=torch.uint8, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_batch(d.data_ptr(), F, stride, nb.data_ptr(), k, CODECS[codec][0], w, h, out.data_ptr(), fstride, res.data_ptr(),
                                 row_bytes=pitch) == 0
    o = host(out)
    mask = np.zeros(n, bool)
    strided(mask, F, h, w, pitch, fstride)[...] = True
    pix = strided(o, F, h, w, pitch, fstride).reshape(F, h, w, 4).copy()
    return res.tolist(), pix, bool((o[~mask] == PAD).all())


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("comp", [HapCompressorNone, HapCompressorSnappy])
def test_rgba_batches_pitched_strided(lib, codec, comp):
    """HapB200EncodeRGBABatch over pitched strided pictures gives, frame by frame, the bytes HapB200EncodeRGBA gives for the
    tight picture; HapB200DecodeRGBABatch into pitched strided pictures gives the oracle's block decoding of the
    reference-decoded textures and writes nothing else."""
    c = CODECS[codec][0]
    ref = oracles.ref_abi() or oracles.oracle_abi()
    shapes = [(36, 4), (132, 20), (516, 12)] + ([(1924, 1084)] if comp == HapCompressorSnappy else [])
    for i, (w, h) in enumerate(shapes):
        k = 1 + i % 3
        pitch, fstride = 4 * w + 16 * (1 + i % 3), h * (4 * w + 16 * (1 + i % 3)) + 32
        pics = pictures(w, h, 3, seed=100 + i)
        frames = encode_batch_pitched(lib, codec, pics, pitch, fstride, comp, k)
        for f, fr in enumerate(frames):
            r, want = lib.encode_rgba(pics[f], w, h, c, comp, k)
            assert r == 0 and fr == want, (w, h, f)
        res, pix, clean = decode_rgba_batch_pitched(lib, codec, frames, w, h, pitch, fstride, k)
        assert res == [0] * len(frames) and clean, (w, h, res)
        for f, fr in enumerate(frames):
            t = [ref.decode(fr, j, lib.texture_bytes(w, h, c, j)) for j in range(2 if CODECS[codec][2] else 1)]
            assert all(x[0] == 0 for x in t)
            want = oracle_rgba(codec, t[0][1], t[1][1] if len(t) > 1 else None, w, h)
            assert np.array_equal(pix[f], want), (w, h, f)


def test_rgba_batch_decode_reports_failing_frames_alone(lib):
    """A Hap Q Alpha batch holding a Hap Q frame, a Hap frame and a truncated frame: each of those reports what it reports
    when decoded alone, its picture is zeros, and the frames around it decode as they do alone."""
    w, h, k = 132, 20, 3
    pitch, fstride = 4 * w + 48, h * (4 * w + 48) + 16
    pics = pictures(w, h, 6, seed=7)
    good = encode_batch_pitched(lib, "HapM", pics, pitch, fstride, HapCompressorSnappy, k)
    other_y = lib.encode_rgba(pics[1], w, h, CODECS["HapY"][0], HapCompressorSnappy, k)[1]
    other_1 = lib.encode_rgba(pics[3], w, h, CODECS["Hap1"][0], HapCompressorSnappy, k)[1]
    frames = [good[0], other_y, good[2], good[3], other_1, good[5]]
    lens = [len(f) for f in frames]
    lens[3] -= 9                                                      # truncated
    res, pix, clean = decode_rgba_batch_pitched(lib, "HapM", frames, w, h, pitch, fstride, k, in_bytes=lens)
    assert clean
    for f in range(len(frames)):
        r1, p1, c1 = decode_rgba_batch_pitched(lib, "HapM", [frames[f][: lens[f]]], w, h, pitch, fstride, k)
        assert c1 and res[f] == r1[0], (f, res, r1)
        assert np.array_equal(pix[f], p1[0]), f
    assert [r != 0 for r in res] == [False, True, False, True, True, False], res
    for f in (1, 3, 4):
        assert int(pix[f].max()) == 0, f


@pytest.mark.parametrize("codec", list(CODECS))
def test_single_frame_rgba_unaligned_pitched(lib, codec):
    """HapB200EncodeRGBA / HapB200DecodeRGBA with pictures at addresses that are not 16-byte aligned and a pitch of 4w + 4:
    host pointers, then device pointers.  The frame equals the tight picture's frame; the decode writes the tight decode's
    pixels and nothing else."""
    c = CODECS[codec][0]
    w, h, k = 132, 20, 3
    pitch = 4 * w + 4
    pic = pictures(w, h, 2, seed=3)[1]
    r, want = lib.encode_rgba(pic, w, h, c, HapCompressorSnappy, k)
    assert r == 0
    r, tight = lib.decode_rgba(want, w, h)
    assert r == 0
    buf, mask = pitched(pic[None], pitch, 0)
    buf = np.concatenate([np.full(4, PAD, np.uint8), buf])             # the picture starts at offset 4
    mask = np.concatenate([np.zeros(4, bool), mask])
    view = buf[4:]
    assert view.ctypes.data % 16 != 0
    r, got = lib.encode_rgba(view, w, h, c, HapCompressorSnappy, k, row_bytes=pitch)
    assert r == 0 and got == want
    d = dev(buf)
    r, got = lib.encode_rgba((d.data_ptr() + 4, len(buf) - 4), w, h, c, HapCompressorSnappy, k, row_bytes=pitch)
    assert r == 0 and got == want
    tight = np.frombuffer(tight, np.uint8).reshape(h, 4 * w)
    out = np.full(len(buf), PAD, np.uint8)
    r, _ = lib.decode_rgba(want, w, h, out=out[4:], row_bytes=pitch)
    assert r == 0
    assert np.array_equal(strided(out[4:], 1, h, w, pitch, 0)[0], tight) and (out[~mask] == PAD).all()
    dout = torch.full((len(buf),), PAD, dtype=torch.uint8, device="cuda")
    r, _ = lib.decode_rgba(want, w, h, out=(dout.data_ptr() + 4, len(buf) - 4), row_bytes=pitch)
    assert r == 0
    o = host(dout)
    assert np.array_equal(strided(o[4:], 1, h, w, pitch, 0)[0], tight) and (o[~mask] == PAD).all()


# ---- more frames than gridDim.y holds ------------------------------------------------------------------------------------

def test_batches_of_65537_frames(lib):
    """The block kernels put the frame on gridDim.y (at most 65535): 65537 distinct 4x4 pictures through the four batch
    entry points that run them.  With one block per picture the blocks of the batch are the blocks of the pictures stacked
    into one 4 x (4*65537) column."""
    F = 65537
    rng = np.random.default_rng(65537)
    pics = rng.integers(0, 256, (F, 4, 4, 4), dtype=np.uint8)
    column = pics.reshape(F * 4, 4, 4)
    src = dev(pics.reshape(-1))
    for codec in ("HapM", "Hap1"):
        c, k0, k1 = CODECS[codec]
        t0, t1 = lib.texture_bytes(4, 4, c, 0), lib.texture_bytes(4, 4, c, 1)
        bstride = align16(t0 + t1)
        blocks = torch.full((F * bstride,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_batch(src.data_ptr(), F, 64, 4, 4, c, blocks.data_ptr(), bstride) == 0
        b = host(blocks).reshape(F, bstride)
        assert b[:, :t0].tobytes() == twin.encode(k0, column), codec
        if k1:
            assert b[:, t0: t0 + t1].tobytes() == twin.encode(k1, column)
        assert (b[:, t0 + t1:] == PAD).all()
        out = torch.full((F * 64,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_decode_batch(blocks.data_ptr(), F, bstride, 4, 4, c, out.data_ptr(), 64) == 0
        want = oracle_rgba(codec, b[:, :t0].tobytes(), b[:, t0: t0 + t1].tobytes(), 4, 4 * F)
        assert np.array_equal(host(out).reshape(F * 4, 4, 4), want), codec
    # RGBA batches, Hap Q without Snappy (with it, the fragment compressor's scratch would be ~2 GB)
    c = CODECS["HapY"][0]
    cap = align16(lib.max_encoded_length_rgba(4, 4, c, 1))
    out = torch.zeros(F * cap, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    assert lib.encode_rgba_batch(src.data_ptr(), F, 64, 4, 4, c, HapCompressorNone, 1, out.data_ptr(), cap, used.data_ptr()) == 0
    frames = host(out).reshape(F, cap)
    u = int(used[0])
    assert (host(used) == u).all()
    tex = np.frombuffer(twin.encode("ycocg", column), np.uint8).reshape(F, 16)
    assert np.array_equal(frames[:, u - 16: u], tex)                  # every frame's texture
    head = frames[0, : u - 16]
    assert (frames[:, : u - 16] == head).all()                         # and the same headers
    for f in (0, 65535, 65536):
        assert frames[f, :u].tobytes() == lib.encode_rgba(pics[f], 4, 4, c, HapCompressorNone, 1)[1], f
    rgba = torch.full((F * 64,), PAD, dtype=torch.uint8, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_batch(out.data_ptr(), F, cap, used.data_ptr(), 1, c, 4, 4, rgba.data_ptr(), 64, res.data_ptr()) == 0
    assert (host(res) == 0).all()
    assert np.array_equal(host(rgba).reshape(F * 4, 4, 4), oracles.bc_decode("ycocg", tex.tobytes(), 4, 4 * F))


# ---- refused geometry ----------------------------------------------------------------------------------------------------

def test_geometry_the_kernels_cannot_address_is_refused(lib):
    """rowBytes above 2^32 - 1 and pictures of 2^32 blocks are Bad_Arguments (include/hap_b200.h), not a silent encode or
    decode of the wrong rows or of a prefix.  (A 64-byte buffer: a library that truncated the pitch to 16 bytes would stay
    inside it.)"""
    c = CODECS["HapY"][0]
    big = 2 ** 32 + 16
    buf = torch.zeros(64, dtype=torch.uint8, device="cuda")
    blk = torch.zeros(64, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_batch(buf.data_ptr(), 1, 64, 4, 4, c, blk.data_ptr(), 16, row_bytes=big) == BAD_ARGUMENTS
    assert lib.block_decode_batch(blk.data_ptr(), 1, 16, 4, 4, c, buf.data_ptr(), 64, row_bytes=big) == BAD_ARGUMENTS
    cap = align16(lib.max_encoded_length_rgba(4, 4, c, 1))
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.encode_rgba_batch(buf.data_ptr(), 1, 64, 4, 4, c, HapCompressorNone, 1, out.data_ptr(), cap, used.data_ptr(),
                                 row_bytes=big) == BAD_ARGUMENTS
    r, frame = lib.encode_rgba(np.zeros((4, 4, 4), np.uint8), 4, 4, c, HapCompressorNone, 1)
    assert r == 0
    d, stride, nb = slots([frame])
    res = torch.full((1,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_batch(d.data_ptr(), 1, stride, nb.data_ptr(), 1, c, 4, 4, buf.data_ptr(), 64, res.data_ptr(),
                                 row_bytes=big) == BAD_ARGUMENTS
    side = 262144                                                      # (side/4)^2 = 2^32 blocks
    assert lib.block_encode_batch(buf.data_ptr(), 1, 64, side, side, c, blk.data_ptr(), 16) == BAD_ARGUMENTS
    assert lib.block_decode_batch(blk.data_ptr(), 1, 16, side, side, c, buf.data_ptr(), 64) == BAD_ARGUMENTS


# ---- two-texture batch encode --------------------------------------------------------------------------------------------

@pytest.fixture(params=[0, 1], ids=["plain", "index+offsets"])
def layout_options(lib, request):
    lib.set_option(lib.OPTION_WRITE_INDEX, request.param)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, request.param)
    yield request.param
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def test_encode_batch_two_textures_texture1_below_texture0(lib, layout_options):
    """HapB200EncodeBatch with a YCoCg and an RGTC1 texture in one allocation, texture 1 at the LOWER address (the 64-bit
    offset wraps), different strides, the compressor chosen per texture, and content that takes every storage path:
    noise (whole-texture fallback), half noise (per-chunk fallback), flat, picture.  Frame f is byte-identical to HapEncode
    of its two textures, and the reference decodes it to them; textureStrides 0 repeats frame 0."""
    w, h = 256, 64
    n0, n1 = (w // 4) * (h // 4) * 16, (w // 4) * (h // 4) * 8
    rng = np.random.default_rng(31)
    pic = pictures(w, h, 1, seed=5)[0]
    half = lambda n: np.concatenate([rng.integers(0, 256, n // 2, dtype=np.uint8), np.tile(np.arange(64, dtype=np.uint8), n // 128)])
    tex0 = [rng.integers(0, 256, n0, dtype=np.uint8), half(n0), np.full(n0, 0x5A, np.uint8),
            np.frombuffer(twin.encode("ycocg", pic), np.uint8)]
    tex1 = [rng.integers(0, 256, n1, dtype=np.uint8), half(n1), np.full(n1, 0x11, np.uint8),
            np.frombuffer(twin.encode("bc4", pic), np.uint8)]
    F = len(tex0)
    s0, s1 = align16(n0) + 48, align16(n1) + 80
    buf = np.full(F * s1 + F * s0, PAD, np.uint8)
    for f in range(F):
        buf[f * s1: f * s1 + n1] = tex1[f]                             # texture 1 first: below texture 0
        buf[F * s1 + f * s0: F * s1 + f * s0 + n0] = tex0[f]
    d = dev(buf)
    p0, p1 = d.data_ptr() + F * s1, d.data_ptr()
    ks = [4, 3]
    ref = oracles.ref_abi() or oracles.oracle_abi()
    for comps in ((HapCompressorSnappy, HapCompressorSnappy), (HapCompressorNone, HapCompressorSnappy),
                  (HapCompressorSnappy, HapCompressorNone), (HapCompressorNone, HapCompressorNone)):
        ostride = align16(lib.max_encoded_length([n0, n1], [YCOCG, RGTC1], ks)) + 4096
        out = torch.full((F * ostride + 256,), PAD, dtype=torch.uint8, device="cuda")
        used = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_batch([p0, p1], [s0, s1], [n0, n1], [YCOCG, RGTC1], list(comps), ks, F, out.data_ptr(), ostride,
                                used.data_ptr()) == 0
        o = host(out)
        assert (o[F * ostride:] == PAD).all(), comps                  # nothing behind the last slot
        for f in range(F):
            fr = o[f * ostride: f * ostride + int(used[f])].tobytes()
            r, want = lib.encode([tex0[f].tobytes(), tex1[f].tobytes()], [YCOCG, RGTC1], list(comps), ks)
            assert r == 0 and fr == want, (comps, f)
            assert ref.decode(fr, 0, n0)[:3] == (0, tex0[f].tobytes(), YCOCG), (comps, f)
            assert ref.decode(fr, 1, n1)[:3] == (0, tex1[f].tobytes(), RGTC1), (comps, f)
        rep = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
        assert lib.encode_batch([p0, p1], [0, 0], [n0, n1], [YCOCG, RGTC1], list(comps), ks, F, rep.data_ptr(), ostride, used.data_ptr()) == 0
        rep = host(rep).reshape(F, ostride)
        u = int(used[0])
        assert (host(used) == u).all() and (rep[:, :u] == rep[0, :u]).all(), comps
        assert rep[0, :u].tobytes() == lib.encode([tex0[0].tobytes(), tex1[0].tobytes()], [YCOCG, RGTC1], list(comps), ks)[1]


# ---- mixed batch decode --------------------------------------------------------------------------------------------------

MAX_CHUNKS = 8


def dxt_like(rng, blocks, bs):
    """block-structured bytes that Snappy compresses partly"""
    base = rng.integers(0, 256, size=bs * 8, dtype=np.uint8)
    p = np.tile(base, blocks // 8 + 1)[: blocks * bs].copy()
    p[:: int(rng.integers(5, 60))] = rng.integers(0, 256)
    return p.tobytes()


def mixed_frames(lib):
    """[(name, frame, damaged)]: about a dozen unrelated frames of every format, chunk count, section kind and encoder"""
    rng = np.random.default_rng(77)
    orc, ref = oracles.oracle_abi(), oracles.ref_abi()
    out = []

    def gpu(name, texs, fmts, comps, ks, index=0, offsets=0):
        lib.set_option(lib.OPTION_WRITE_INDEX, index)
        lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, offsets)
        try:
            r, f = lib.encode(texs, fmts, comps, ks)
        finally:
            lib.set_option(lib.OPTION_WRITE_INDEX, 0)
            lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)
        assert r == 0, name
        return f

    p1 = dxt_like(rng, 3000, 8)
    out.append(("gpu dxt1 k1", gpu("a", [p1], [DXT1], [1], [1]), False))
    py = dxt_like(rng, 9000, 16)
    out.append(("gpu ycocg k5 index", gpu("b", [py], [YCOCG], [1], [5], index=1), False))
    p5 = dxt_like(rng, 7000, 16)
    out.append(("gpu dxt5 k3 offsets", gpu("c", [p5], [DXT5], [1], [3], offsets=1), False))
    m0, m1 = dxt_like(rng, 4096, 16), dxt_like(rng, 4096, 8)
    out.append(("gpu hapm k4+2", gpu("d", [m0, m1], [YCOCG, RGTC1], [1, 1], [4, 2]), False))
    out.append(("gpu hapm k8+8 index offsets", gpu("e", [m1 + m1, m0], [RGTC1, YCOCG], [1, 0], [8, 8], index=1, offsets=1), False))
    pa = dxt_like(rng, 5000, 8)
    out.append(("oracle rgtc1 k2", orc.encode([pa], [RGTC1], [1], [2])[1], False))
    p7 = dxt_like(rng, 6000, 16)
    out.append(("oracle bc7 k6", orc.encode([p7], [BC7], [1], [6])[1], False))
    out.append(("oracle hapm k1+7", orc.encode([m0, m1], [YCOCG, RGTC1], [1, 1], [1, 7])[1], False))
    if ref is not None:
        pr = dxt_like(rng, 8000, 16)
        out.append(("reference ycocg k8", ref.encode([pr], [YCOCG], [1], [8])[1], False))
    out.append(("raw dxt1", gpu("f", [p1[:4096]], [DXT1], [0], [1]), False))
    s = oracles.snappy_compress(p5[:8192])
    out.append(("whole snappy dxt5", len(s).to_bytes(3, "little") + b"\xbe" + s, False))
    t = gpu("g", [py], [YCOCG], [1], [6])
    out.append(("truncated", t[: len(t) - 11], True))
    x = bytearray(gpu("h", [p5], [DXT5], [1], [2]))
    x[len(x) * 2 // 3] ^= 0x24
    out.append(("flipped byte", bytes(x), True))
    out.append(("over max chunks", gpu("i", [py], [YCOCG], [1], [12]), False))
    return out


@pytest.mark.parametrize("index", [0, 1])
@pytest.mark.parametrize("order", ["forward", "reverse"])
def test_decode_batch_of_unrelated_frames(lib, index, order):
    """HapB200DecodeBatch of one call holding frames of every format, chunk counts 1..maxChunks, Complex / whole-texture Snappy /
    raw sections, with and without fragment index and offset table, written by this encoder, the oracle and the reference,
    plus a truncated frame, a damaged frame and one with more chunks than maxChunks.  Every frame gives what HapDecode gives
    for it alone (the frame over maxChunks: Bad_Arguments), the reference's bytes where the reference decodes it, and writes
    nothing past its texture."""
    frames = mixed_frames(lib)
    if order == "reverse":
        frames = frames[::-1]
    raw = [f for _, f, _ in frames]
    d, stride, nb = slots(raw, pad=0xEE, extra=48)                     # inBytes < inStride, 0xEE behind every frame
    F = len(raw)
    ostride = align16(max(len(f) for f in raw) * 2 + 200000)
    out = torch.full((F * ostride,), PAD, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    fmts = torch.zeros(F, dtype=torch.int32, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_batch(d.data_ptr(), F, stride, nb.data_ptr(), index, MAX_CHUNKS, out.data_ptr(), ostride, used.data_ptr(),
                            fmts.data_ptr(), res.data_ptr()) == 0
    o, res, fmts, used = host(out).reshape(F, ostride), res.tolist(), fmts.tolist(), used.tolist()
    ref = oracles.ref_abi() or oracles.oracle_abi()
    for f, (name, fr, damaged) in enumerate(frames):
        r, data, fmt, _ = lib.decode(fr, index, ostride)
        if name == "over max chunks":                                  # (a one-texture frame: texture 1 is missing)
            assert res[f] == BAD_ARGUMENTS and (r == 0) == (index == 0), (name, res[f], r)
            continue
        assert (res[f], fmts[f]) == (r, fmt), (name, res[f], fmts[f], r, fmt)
        if r != 0:
            continue
        assert used[f] == len(data) and o[f, : used[f]].tobytes() == data, name
        assert (o[f, used[f]:] == PAD).all(), name
        if not damaged:
            rr = ref.decode(fr, index, ostride)
            if rr[0] == 0:
                assert rr[1] == data, name
    ok = [n for (n, _, _), r in zip(frames, res) if r == 0]
    assert len(ok) >= (3 if index else 8), (res, [n for n, _, _ in frames])
