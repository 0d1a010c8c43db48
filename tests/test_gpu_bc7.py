"""Hap R (BC7) frames and textures to RGBA on the GPU.  Content: random blocks of every mode (reserved blocks included) and
picture-like mode-6 textures (tests/bc7_util.pack_picture).  Textures are wrapped into frames by this library's HapEncode
(Snappy, chunk counts 1..8, fragment index and offset table on and off), by the oracle's encoder and, when it is built, by
the reference's.  HapB200BlockDecodeBatch, HapB200DecodeRGBABatch and HapB200DecodeRGBA must give the oracle's BC7 decoding
byte for byte, at 4x4, odd sizes up to 1924x1084, pitched rows and strided frames, and a 65537-frame block batch; padding
around every picture keeps its sentinel."""
import numpy as np
import pytest
import torch

import bc7_util as U
import hap_b200
import hap_b200.lib as L
import oracles
from hap_b200 import mov, synth
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy, HapTextureFormat_RGBA_BPTC_UNORM

pytestmark = pytest.mark.gpu
BC7, HAP7 = HapTextureFormat_RGBA_BPTC_UNORM, L.HapB200Codec_Hap7
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
    return np.lib.stride_tricks.as_strided(buf, shape=(frames, h, 4 * w), strides=(fstride, pitch, 1))


def textures(w, h, n, seed):
    """n BC7 textures of a w x h picture: even ones picture-like (mode 6), odd ones random blocks, every mode and the
    reserved block side by side"""
    rng = np.random.default_rng(seed + 131 * w + h)
    nb = (w // 4) * (h // 4)
    out = []
    for i in range(n):
        if i % 2 == 0:
            out.append(U.pack_picture(synth.frame(w, h, i, kind="video", alpha="ramp").numpy()))
        else:
            b = rng.integers(0, 256, (nb, 16), dtype=np.uint8)
            modes = (np.arange(nb) + i) % 9
            for m in range(9):
                sel = modes == m
                b[sel] = U.random_blocks(rng, int(sel.sum()), m)
            out.append(b.tobytes())
    return out


def want_rgba(tex, w, h):
    return U.oracle_decode(tex, w, h)


def decode_rgba_batch(lib, frames, w, h, pitch, fstride, k, in_bytes=None, codec=HAP7):
    """HapB200DecodeRGBABatch -> (results, pictures (F, h, w, 4), padding untouched)"""
    F = len(frames)
    stride = align16(max(len(f) for f in frames) + 16)
    buf = np.full(F * stride, PAD, np.uint8)
    for i, f in enumerate(frames):
        buf[i * stride: i * stride + len(f)] = np.frombuffer(f, np.uint8)
    d = dev(buf)
    nb = torch.tensor(in_bytes if in_bytes is not None else [len(f) for f in frames], dtype=torch.int64, device="cuda")
    n = (F - 1) * fstride + (h - 1) * pitch + 4 * w
    out = torch.full((n,), PAD, dtype=torch.uint8, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_batch(d.data_ptr(), F, stride, nb.data_ptr(), k, codec, w, h, out.data_ptr(), fstride, res.data_ptr(),
                                 row_bytes=pitch) == 0
    o = host(out)
    mask = np.zeros(n, bool)
    strided(mask, F, h, w, pitch, fstride)[...] = True
    return res.tolist(), strided(o, F, h, w, pitch, fstride).reshape(F, h, w, 4).copy(), bool((o[~mask] == PAD).all())


@pytest.fixture(params=[(0, 0), (1, 0), (0, 1), (1, 1)], ids=["plain", "index", "offsets", "index+offsets"])
def layout(lib, request):
    lib.set_option(lib.OPTION_WRITE_INDEX, request.param[0])
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, request.param[1])
    yield request.param
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


# ---- block batches -------------------------------------------------------------------------------------------------------

def test_block_decode_batch_pitched_strided(lib):
    """HapB200BlockDecodeBatch of BC7 blocks into pitched strided pictures, a block stride wider than the texture: the
    oracle's decoding, and nothing written outside the pictures"""
    for i, (w, h) in enumerate(SHAPES):
        F = 3
        pitch = 4 * w + 16 * (i % 3)
        fstride = h * pitch + 16 * (1 + i % 2)
        t0 = lib.texture_bytes(w, h, HAP7, 0)
        bstride = align16(t0) + 48
        texs = textures(w, h, F, seed=i)
        blk = np.full(F * bstride, PAD, np.uint8)
        for f in range(F):
            blk[f * bstride: f * bstride + t0] = np.frombuffer(texs[f], np.uint8)
        n = (F - 1) * fstride + (h - 1) * pitch + 4 * w
        out = torch.full((n,), PAD, dtype=torch.uint8, device="cuda")
        assert lib.block_decode_batch(dev(blk).data_ptr(), F, bstride, w, h, HAP7, out.data_ptr(), fstride, row_bytes=pitch) == 0
        o = host(out)
        mask = np.zeros(n, bool)
        strided(mask, F, h, w, pitch, fstride)[...] = True
        pix = strided(o, F, h, w, pitch, fstride)
        for f in range(F):
            assert np.array_equal(pix[f].reshape(h, w, 4), want_rgba(texs[f], w, h)), (w, h, f)
        assert (o[~mask] == PAD).all(), (w, h)


def test_block_decode_batch_of_65537_frames(lib):
    """One 4x4 block per frame, 65537 frames (more than gridDim.y holds): the launches are sliced, and frame f's picture
    is block f decoded"""
    F = 65537
    rng = np.random.default_rng(65537)
    blocks = rng.integers(0, 256, (F, 16), dtype=np.uint8)
    for m in range(9):
        blocks[m::9] = U.random_blocks(rng, len(blocks[m::9]), m)
    out = torch.full((F * 64,), PAD, dtype=torch.uint8, device="cuda")
    assert lib.block_decode_batch(dev(blocks.reshape(-1)).data_ptr(), F, 16, 4, 4, HAP7, out.data_ptr(), 64) == 0
    assert np.array_equal(host(out).reshape(F * 4, 4, 4), want_rgba(blocks.tobytes(), 4, 4 * F))


# ---- frames ---------------------------------------------------------------------------------------------------------------

def frames_of(lib, texs, k, encoder):
    """texs wrapped into Hap R frames by `encoder` (lib = this library's HapEncode, Snappy), k chunks requested"""
    out = []
    for t in texs:
        r, f = encoder.encode([t], [BC7], [HapCompressorSnappy], [k])
        assert r == 0
        assert lib.texture_format(f, 0) == (0, BC7)
        out.append(f)
    return out


def test_rgba_batch_this_encoder_every_chunk_count(lib, layout):
    """HapB200DecodeRGBABatch of frames from this library's HapEncode, chunk counts 1..8, into pitched strided pictures"""
    for i, (w, h) in enumerate([(4, 4), (36, 20), (132, 20), (516, 12), (1924, 1084)]):
        pitch, fstride = 4 * w + 16 * (1 + i % 3), h * (4 * w + 16 * (1 + i % 3)) + 32
        texs = textures(w, h, 4, seed=40 + i)
        for k in range(1, 9):
            frames = frames_of(lib, texs, k, lib)
            res, pix, clean = decode_rgba_batch(lib, frames, w, h, pitch, fstride, k)
            assert res == [0] * len(frames) and clean, (w, h, k, res)
            for f in range(len(frames)):
                assert np.array_equal(pix[f], want_rgba(texs[f], w, h)), (w, h, k, f)


@pytest.mark.parametrize("who", ["oracle", "reference"])
def test_rgba_batch_other_encoders(lib, who):
    enc = oracles.oracle_abi() if who == "oracle" else oracles.ref_abi()
    if enc is None:
        pytest.skip("the reference build is not present")
    for i, (w, h) in enumerate([(12, 8), (132, 20), (1924, 1084)]):
        pitch, fstride = 4 * w + 48, h * (4 * w + 48) + 16
        texs = textures(w, h, 3, seed=60 + i)
        for k in (1, 3, 8):
            frames = frames_of(lib, texs, k, enc)
            res, pix, clean = decode_rgba_batch(lib, frames, w, h, pitch, fstride, k)
            assert res == [0] * len(frames) and clean, (who, w, h, k, res)
            for f in range(len(frames)):
                assert np.array_equal(pix[f], want_rgba(texs[f], w, h)), (who, w, h, k, f)


def test_rgba_batch_reports_frames_of_another_flavour_and_truncated_frames(lib):
    """A Hap R batch holding Hap Q frames and a truncated frame: those report Bad_Frame (the truncated one what it reports
    alone) and get a zero picture; every other frame decodes as it does alone"""
    w, h, k = 132, 20, 3
    pitch, fstride = 4 * w + 48, h * (4 * w + 48) + 16
    texs = textures(w, h, 6, seed=7)
    good = frames_of(lib, texs, k, lib)
    pic = synth.frame(w, h, 1).numpy()
    hapq = lib.encode_rgba(pic, w, h, L.HapB200Codec_HapY, HapCompressorSnappy, k)[1]
    frames = [good[0], hapq, good[2], good[3], hapq, good[5]]
    lens = [len(f) for f in frames]
    lens[3] -= 9
    res, pix, clean = decode_rgba_batch(lib, frames, w, h, pitch, fstride, k, in_bytes=lens)
    assert clean
    assert [r != 0 for r in res] == [False, True, False, True, True, False], res
    assert res[1] == res[4] == BAD_FRAME
    for f in range(len(frames)):
        r1, p1, c1 = decode_rgba_batch(lib, [frames[f][: lens[f]]], w, h, pitch, fstride, k)
        assert c1 and res[f] == r1[0], (f, res, r1)
        if res[f] == 0:
            assert np.array_equal(pix[f], want_rgba(texs[f], w, h)), f
        else:
            assert int(pix[f].max()) == 0, f


def test_single_frame_host_and_device_buffers(lib):
    """HapB200DecodeRGBA of Hap R frames: host frame and picture, device frame and picture, pitched and unaligned"""
    for i, (w, h) in enumerate([(4, 4), (36, 20), (1924, 1084)]):
        texs = textures(w, h, 2, seed=80 + i)
        for t, f in zip(texs, frames_of(lib, texs, 1 + i, lib)):
            want = want_rgba(t, w, h)
            r, got = lib.decode_rgba(f, w, h)
            assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, w, 4), want), (w, h)
            pitch = 4 * w + 4
            n = 4 + (h - 1) * pitch + 4 * w
            mask = np.zeros(n, bool)
            strided(mask[4:], 1, h, w, pitch, 0)[...] = True
            out = np.full(n, PAD, np.uint8)
            assert lib.decode_rgba(f, w, h, out=out[4:], row_bytes=pitch)[0] == 0
            assert np.array_equal(strided(out[4:], 1, h, w, pitch, 0)[0].reshape(h, w, 4), want) and (out[~mask] == PAD).all()
            df = dev(f)
            dout = torch.full((n,), PAD, dtype=torch.uint8, device="cuda")
            assert lib.decode_rgba((df.data_ptr(), len(f)), w, h, out=(dout.data_ptr() + 4, n - 4), row_bytes=pitch)[0] == 0
            o = host(dout)
            assert np.array_equal(strided(o[4:], 1, h, w, pitch, 0)[0].reshape(h, w, 4), want) and (o[~mask] == PAD).all()


def test_verbatim_frames(lib):
    """Frames whose BC7 texture is stored without Snappy decode the same way"""
    w, h = 132, 20
    texs = textures(w, h, 2, seed=90)
    for t in texs:
        r, f = lib.encode([t], [BC7], [HapCompressorNone], [1])
        assert r == 0
        r, got = lib.decode_rgba(f, w, h)
        assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, w, 4), want_rgba(t, w, h))
        res, pix, clean = decode_rgba_batch(lib, [f], w, h, 4 * w, 4 * w * h, 1)
        assert res == [0] and clean and np.array_equal(pix[0], want_rgba(t, w, h))


def test_hap7_movie_round_trip(lib, tmp_path):
    """Hap R frames written into a QuickTime file (hap_mov.h) and read back decode to the same pixels"""
    w, h, n = 516, 20, 4
    texs = textures(w, h, n, seed=99)
    frames = frames_of(lib, texs, 4, lib)
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
            assert r == 0 and np.array_equal(np.frombuffer(got, np.uint8).reshape(h, w, 4), want_rgba(texs[i], w, h)), i
