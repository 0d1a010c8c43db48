"""Hap HDR (BC6H) frames and textures to RGBA16F on the GPU.  Content: random blocks of every mode (the reserved mode values
included) and picture-like mode-11 textures (tests/bc6h_util.pack_picture), UF16 and SF16.  Textures are wrapped into
frames by this library's HapEncode (Snappy, chunk counts 1..8, fragment index and offset table on and off), by the
oracle's encoder and, when it is built, by the reference's.  HapB200BlockDecodeHalfBatch, HapB200DecodeRGBAHalfBatch and
HapB200DecodeRGBAHalf must give the oracle's decoding bit for bit on every half value, at 4x4, odd sizes up to 1924x1084,
pitched rows and strided frames, and a 65537-frame block batch; padding around every picture keeps its sentinel."""
import numpy as np
import pytest
import torch

import bc6h_util as U
import hap_b200
import oracles
from hap_b200 import mov, synth
from hap_b200.abi import (HapCompressorNone, HapCompressorSnappy, HapTextureFormat_A_RGTC1, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT,
                          HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGBA_BPTC_UNORM)

pytestmark = pytest.mark.gpu
UF16, SF16 = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT, HapTextureFormat_RGB_BPTC_SIGNED_FLOAT
BAD_FRAME = 3
PAD = 0xEE
SHAPES = [(4, 4), (8, 4), (12, 8), (20, 12), (36, 20), (132, 4), (516, 20), (1924, 1084)]


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
    return np.lib.stride_tricks.as_strided(buf, shape=(frames, h, 8 * w), strides=(fstride, pitch, 1))


def textures(w, h, n, seed, signed=False):
    """n BC6H textures of a w x h picture: even ones picture-like (mode 11), odd ones random blocks, every mode and the
    reserved mode values side by side"""
    rng = np.random.default_rng(seed + 131 * w + h)
    nb = (w // 4) * (h // 4)
    out = []
    for i in range(n):
        if i % 2 == 0:
            out.append(U.pack_picture(synth.frame(w, h, i, kind="video").numpy(), signed))
        else:
            b = rng.integers(0, 256, (nb, 16), dtype=np.uint8)
            modes = (np.arange(nb) + i) % 18
            for m in range(18):
                sel = modes == m
                b[sel] = U.random_blocks(rng, int(sel.sum()), m)
            out.append(b.tobytes())
    return out


def want(tex, w, h, signed) -> np.ndarray:
    """the oracle's RGBA16F picture as (h, 8 w) bytes"""
    return U.oracle_decode(tex, w, h, signed).view(np.uint8).reshape(h, 8 * w)


def decode_half_batch(lib, frames, w, h, pitch, fstride, k, in_bytes=None):
    """HapB200DecodeRGBAHalfBatch -> (results, pictures (F, h, 8 w) bytes, padding untouched)"""
    F = len(frames)
    stride = align16(max(len(f) for f in frames) + 16)
    buf = np.full(F * stride, PAD, np.uint8)
    for i, f in enumerate(frames):
        buf[i * stride: i * stride + len(f)] = np.frombuffer(f, np.uint8)
    d = dev(buf)
    nb = torch.tensor(in_bytes if in_bytes is not None else [len(f) for f in frames], dtype=torch.int64, device="cuda")
    n = (F - 1) * fstride + (h - 1) * pitch + 8 * w
    out = torch.full((n,), PAD, dtype=torch.uint8, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_half_batch(d.data_ptr(), F, stride, nb.data_ptr(), k, w, h, out.data_ptr(), fstride, res.data_ptr(),
                                      row_bytes=pitch) == 0
    o = host(out)
    mask = np.zeros(n, bool)
    strided(mask, F, h, w, pitch, fstride)[...] = True
    return res.tolist(), strided(o, F, h, w, pitch, fstride).copy(), bool((o[~mask] == PAD).all())


def frames_of(lib, texs, fmt, k, encoder):
    out = []
    for t in texs:
        r, f = encoder.encode([t], [fmt], [HapCompressorSnappy], [k])
        assert r == 0
        assert lib.texture_format(f, 0) == (0, fmt)
        out.append(f)
    return out


@pytest.fixture(params=[(0, 0), (1, 0), (0, 1), (1, 1)], ids=["plain", "index", "offsets", "index+offsets"])
def layout(lib, request):
    lib.set_option(lib.OPTION_WRITE_INDEX, request.param[0])
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, request.param[1])
    yield request.param
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


# ---- block batches -------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", [UF16, SF16], ids=["UF16", "SF16"])
def test_block_decode_half_batch_pitched_strided(lib, fmt):
    for i, (w, h) in enumerate(SHAPES):
        F = 3
        pitch = 8 * w + 16 * (i % 3)
        fstride = h * pitch + 16 * (1 + i % 2)
        t0 = (w // 4) * (h // 4) * 16
        bstride = align16(t0) + 48
        texs = textures(w, h, F, seed=i, signed=fmt == SF16)
        blk = np.full(F * bstride, PAD, np.uint8)
        for f in range(F):
            blk[f * bstride: f * bstride + t0] = np.frombuffer(texs[f], np.uint8)
        n = (F - 1) * fstride + (h - 1) * pitch + 8 * w
        out = torch.full((n,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_decode_half_batch(dev(blk).data_ptr(), F, bstride, w, h, fmt, out.data_ptr(), fstride, row_bytes=pitch) == 0
        o = host(out)
        mask = np.zeros(n, bool)
        strided(mask, F, h, w, pitch, fstride)[...] = True
        pix = strided(o, F, h, w, pitch, fstride)
        for f in range(F):
            assert np.array_equal(pix[f], want(texs[f], w, h, fmt == SF16)), (w, h, f)
        assert (o[~mask] == PAD).all(), (w, h)


def test_block_decode_half_batch_of_65537_frames(lib):
    F = 65537
    rng = np.random.default_rng(65537)
    blocks = rng.integers(0, 256, (F, 16), dtype=np.uint8)
    for m in range(18):
        blocks[m::18] = U.random_blocks(rng, len(blocks[m::18]), m)
    d = dev(blocks.reshape(-1))
    for fmt in (UF16, SF16):
        out = torch.full((F * 128,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_decode_half_batch(d.data_ptr(), F, 16, 4, 4, fmt, out.data_ptr(), 128) == 0
        assert np.array_equal(host(out).reshape(F * 4, 32), want(blocks.tobytes(), 4, 4 * F, fmt == SF16))


# ---- frames ---------------------------------------------------------------------------------------------------------------

def test_half_batch_this_encoder_every_chunk_count(lib, layout):
    for i, (w, h) in enumerate([(4, 4), (36, 20), (516, 12), (1924, 1084)]):
        pitch = 8 * w + 16 * (1 + i % 3)
        fstride = h * pitch + 32
        for fmt in (UF16, SF16):
            texs = textures(w, h, 2, seed=40 + i, signed=fmt == SF16)
            for k in range(1, 9):
                frames = frames_of(lib, texs, fmt, k, lib)
                res, pix, clean = decode_half_batch(lib, frames, w, h, pitch, fstride, k)
                assert res == [0] * len(frames) and clean, (w, h, k, res)
                for f in range(len(frames)):
                    assert np.array_equal(pix[f], want(texs[f], w, h, fmt == SF16)), (w, h, k, f)


@pytest.mark.parametrize("who", ["oracle", "reference"])
def test_half_batch_other_encoders(lib, who):
    enc = oracles.oracle_abi() if who == "oracle" else oracles.ref_abi()
    if enc is None:
        pytest.skip("the reference build is not present")
    for i, (w, h) in enumerate([(12, 8), (132, 20), (1924, 1084)]):
        pitch, fstride = 8 * w + 48, h * (8 * w + 48) + 16
        for fmt in (UF16, SF16):
            texs = textures(w, h, 2, seed=60 + i, signed=fmt == SF16)
            for k in (1, 3, 8):
                frames = frames_of(lib, texs, fmt, k, enc)
                res, pix, clean = decode_half_batch(lib, frames, w, h, pitch, fstride, k)
                assert res == [0] * len(frames) and clean, (who, w, h, k, res)
                for f in range(len(frames)):
                    assert np.array_equal(pix[f], want(texs[f], w, h, fmt == SF16)), (who, w, h, k, f)


def test_half_batch_mixes_uf16_sf16_and_reports_other_flavours_and_truncated_frames(lib):
    """One batch: UF16 and SF16 frames, a Hap R frame and a truncated frame.  Each good frame decodes as its own section
    says and as it does alone; the Hap R frame reports Bad_Frame, the truncated one what it reports alone; both pictures
    are zero bytes"""
    w, h, k = 132, 20, 3
    pitch, fstride = 8 * w + 48, h * (8 * w + 48) + 16
    tu = textures(w, h, 2, seed=7)
    ts = textures(w, h, 2, seed=8, signed=True)
    fu, fs = frames_of(lib, tu, UF16, k, lib), frames_of(lib, ts, SF16, k, lib)
    hapr = lib.encode([tu[1]], [HapTextureFormat_RGBA_BPTC_UNORM], [HapCompressorSnappy], [k])[1]
    frames = [fu[0], fs[0], hapr, fu[1], fs[1], fu[0]]
    texs = [(tu[0], False), (ts[0], True), None, (tu[1], False), (ts[1], True), (tu[0], False)]
    lens = [len(f) for f in frames]
    lens[5] -= 9
    res, pix, clean = decode_half_batch(lib, frames, w, h, pitch, fstride, k, in_bytes=lens)
    assert clean
    assert [r != 0 for r in res] == [False, False, True, False, False, True], res
    assert res[2] == BAD_FRAME
    for f in range(len(frames)):
        r1, p1, c1 = decode_half_batch(lib, [frames[f][: lens[f]]], w, h, pitch, fstride, k)
        assert c1 and res[f] == r1[0], (f, res, r1)
        if res[f] == 0:
            assert np.array_equal(pix[f], want(texs[f][0], w, h, texs[f][1])) and np.array_equal(pix[f], p1[0]), f
            r2, got = lib.decode_rgba_half(frames[f], w, h)
            assert r2 == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, 8 * w), pix[f]), f
        else:
            assert int(pix[f].max()) == 0, f


def test_half_batch_reports_frames_that_are_not_one_bc6h_texture_of_the_picture(lib):
    """Frames whose texture is 4 rows larger or smaller than the picture's, and a frame of two textures (BC6H of the right
    size + RGTC1, which HapEncode accepts), among good UF16 and SF16 frames: each bad one reports Bad_Frame in the batch and
    from HapB200DecodeRGBAHalf, and its picture is zero bytes; the good ones decode as alone"""
    w, h, k = 132, 20, 3
    pitch, fstride = 8 * w + 48, h * (8 * w + 48) + 16
    good_u, good_s = textures(w, h, 1, seed=30)[0], textures(w, h, 1, seed=31, signed=True)[0]
    big, small = textures(w, h + 4, 1, seed=32)[0], textures(w, h - 4, 1, seed=33, signed=True)[0]
    alpha = bytes(np.random.default_rng(34).integers(0, 256, (w // 4) * (h // 4) * 8, dtype=np.uint8))
    r, two = lib.encode([good_u, alpha], [UF16, HapTextureFormat_A_RGTC1], [HapCompressorSnappy] * 2, [k, k])
    assert r == 0 and lib.texture_count(two) == (0, 2)
    frames = [frames_of(lib, [good_u], UF16, k, lib)[0], frames_of(lib, [big], UF16, k, lib)[0],
              frames_of(lib, [good_s], SF16, k, lib)[0], frames_of(lib, [small], SF16, k, lib)[0], two]
    res, pix, clean = decode_half_batch(lib, frames, w, h, pitch, fstride, k)
    assert clean and res == [0, BAD_FRAME, 0, BAD_FRAME, BAD_FRAME], res
    for f, (tex, signed) in ((0, (good_u, False)), (2, (good_s, True))):
        assert np.array_equal(pix[f], want(tex, w, h, signed)), f
    for f in (1, 3, 4):
        assert int(pix[f].max()) == 0, f
        assert lib.decode_rgba_half(frames[f], w, h)[0] == BAD_FRAME, f
        r1, _, c1 = decode_half_batch(lib, [frames[f]], w, h, pitch, fstride, k)
        assert c1 and r1 == [BAD_FRAME], (f, r1)


def test_single_frame_host_and_device_buffers(lib):
    for i, (w, h) in enumerate([(4, 4), (36, 20), (1924, 1084)]):
        for fmt in (UF16, SF16):
            texs = textures(w, h, 2, seed=80 + i, signed=fmt == SF16)
            for t, f in zip(texs, frames_of(lib, texs, fmt, 1 + i, lib)):
                wnt = want(t, w, h, fmt == SF16)
                r, got = lib.decode_rgba_half(f, w, h)
                assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, 8 * w), wnt), (w, h)
                pitch = 8 * w + 8
                n = 4 + (h - 1) * pitch + 8 * w
                mask = np.zeros(n, bool)
                strided(mask[4:], 1, h, w, pitch, 0)[...] = True
                out = np.full(n, PAD, np.uint8)
                assert lib.decode_rgba_half(f, w, h, out=out[4:], row_bytes=pitch)[0] == 0
                assert np.array_equal(strided(out[4:], 1, h, w, pitch, 0)[0], wnt) and (out[~mask] == PAD).all()
                df = dev(f)
                dout = torch.full((n,), PAD, dtype=torch.uint8, device="cuda")
                assert lib.decode_rgba_half((df.data_ptr(), len(f)), w, h, out=(dout.data_ptr() + 4, n - 4), row_bytes=pitch)[0] == 0
                o = host(dout)
                assert np.array_equal(strided(o[4:], 1, h, w, pitch, 0)[0], wnt) and (o[~mask] == PAD).all()


def test_single_frame_refuses_wrong_size_and_verbatim_frames_decode(lib):
    w, h = 132, 20
    t = textures(w, h, 1, seed=90)[0]
    r, f = lib.encode([t], [UF16], [HapCompressorNone], [1])
    assert r == 0
    r, got = lib.decode_rgba_half(f, w, h)
    assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, 8 * w), want(t, w, h, False))
    assert lib.decode_rgba_half(f, w, h - 4)[0] == BAD_FRAME          # a texture larger than the picture
    res, pix, clean = decode_half_batch(lib, [f], w, h, 8 * w, 8 * w * h, 1)
    assert res == [0] and clean and np.array_equal(pix[0], want(t, w, h, False))


def test_hapH_movie_round_trip(lib, tmp_path):
    w, h, n = 516, 20, 4
    texs = textures(w, h, n, seed=99, signed=True)
    frames = frames_of(lib, texs, SF16, 4, lib)
    path = str(tmp_path / "hapH.mov")
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
            assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, 8 * w), want(texs[i], w, h, True)), i
