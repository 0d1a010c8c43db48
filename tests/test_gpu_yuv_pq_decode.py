"""HDR10 decoders on the GPU (HapB200BlockDecodeYUVPQBatch, HapB200DecodeYUVPQBatch, HapB200DecodeYUVPQ): every plane must
equal, byte for byte, yuv_pq_out_util.rgba_half_to_yuv_pq (the definition of include/hap_b200.h) of what the RGBA16F
decoders give for the same input, and the batch results must equal theirs -- for both ranges, UF16 and SF16 and several
unitNits; on random blocks of every BC6H mode (the reserved mode values and SF16 negatives included), picture-like HDR
content, Snappy-chunked frames (with the index and offset-table options), uncompressed frames, a batch of more than 65535
frames and a batch mixing good, truncated, non-BC6H, wrong-size and two-texture frames, whose failed frames must be black.
Sentinels around every plane must survive and the inputs must be left as they were.  Flat HDR10 pictures must come back
byte for byte through HapB200EncodeYUVPQBatch and HapB200DecodeYUVPQBatch wherever the header says they do."""
import numpy as np
import pytest
import torch

import bc6h_util as U
import hap_b200
import test_gpu_bc6h as B
import test_gpu_yuv_decode as D
import yuv_pq_out_util as Q
import yuv_pq_util as P
import yuv_util as Y
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy, HapTextureFormat_A_RGTC1, HapTextureFormat_YCoCg_DXT5

pytestmark = pytest.mark.gpu
UF16, SF16 = B.UF16, B.SF16
PAD = D.PAD
MAX_CHUNKS = 64
BAD_FRAME = 3


@pytest.fixture(scope="module")
def lib():
    return hap_b200.load()


def out_of(F, w, h, i=1):
    pitch, fstride, chroma_at = D.geometry(w, h, Y.P010, i)
    return D.Out(F, w, h, Y.P010, pitch, fstride, chroma_at)


def check(out, halves, cs, unit, what=""):
    """out's buffer equals the conversion of halves[f] ((h, w, 4) uint16) at every plane byte and PAD everywhere else"""
    want = out.want_buffer([Q.rgba_half_to_yuv_pq(p, cs, unit) for p in halves])
    got = out.d.cpu().numpy()
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, (what, bad.size, bad[:8])


def halves_of_blocks(lib, blk, F, bstride, w, h, fmt):
    rgba = torch.zeros(F * 8 * w * h, dtype=torch.uint8, device="cuda")
    assert lib.block_decode_half_batch(blk.data_ptr(), F, bstride, w, h, fmt, rgba.data_ptr(), 8 * w * h) == 0
    return rgba.cpu().numpy().view(np.uint16).reshape(F, h, w, 4)


def random_textures(w, h, F, seed):
    """F textures of random blocks, every mode and the reserved mode values side by side"""
    rng = np.random.default_rng(seed)
    nb = (w // 4) * (h // 4)
    out = np.zeros((F, nb * 16), np.uint8)
    for f in range(F):
        b = rng.integers(0, 256, (nb, 16), dtype=np.uint8)
        modes = (np.arange(nb) + f) % 18
        for m in range(18):
            sel = modes == m
            b[sel] = U.random_blocks(rng, int(sel.sum()), m)
        out[f] = b.reshape(-1)
    return out


@pytest.mark.parametrize("cs", P.COLOR_SPACES)
@pytest.mark.parametrize("unit", (1, 203, 10000))
@pytest.mark.parametrize("fmt", [UF16, SF16], ids=["UF16", "SF16"])
def test_block_decode_equals_the_half_decoder(lib, cs, unit, fmt):
    w, h, F = 260, 132, 3                                                 # 65 block columns: three warp spans per row
    t = random_textures(w, h, F, seed=cs + unit + fmt)
    bstride = D.align16(t.shape[1]) + 48
    blk_np = np.zeros((F, bstride), np.uint8)
    blk_np[:, : t.shape[1]] = t
    blk = D.dev(blk_np.ravel())
    out = out_of(F, w, h, cs + unit)
    assert lib.block_decode_yuv_pq_batch(blk.data_ptr(), F, bstride, w, h, fmt, out.luma, out.chroma, out.fstride, out.pitch, cs, unit) == 0
    halves = halves_of_blocks(lib, blk, F, bstride, w, h, fmt)
    if fmt == SF16:
        assert (halves[..., :3] >= 0x8000).any()                          # negatives are there
    check(out, halves, cs, unit, (cs, unit, fmt))
    assert (blk.cpu().numpy() == blk_np.ravel()).all()


def test_block_decode_geometry(lib):
    for i, (w, h) in enumerate(D.SHAPES):
        F, cs, unit, fmt = 3, P.COLOR_SPACES[i % 2], (80, 100, 1000)[i % 3], (UF16, SF16)[i % 2]
        t = random_textures(w, h, F, seed=i)
        bstride = D.align16(t.shape[1]) + 16 * (i % 3)
        blk_np = np.zeros((F, bstride), np.uint8)
        blk_np[:, : t.shape[1]] = t
        blk = D.dev(blk_np.ravel())
        out = out_of(F, w, h, i)
        assert lib.block_decode_yuv_pq_batch(blk.data_ptr(), F, bstride, w, h, fmt, out.luma, out.chroma, out.fstride, out.pitch, cs, unit) == 0
        check(out, halves_of_blocks(lib, blk, F, bstride, w, h, fmt), cs, unit, (w, h))


def decode_both(lib, frames, F, istride, used, w, h, cs, unit, i=1):
    """HapB200DecodeRGBAHalfBatch and HapB200DecodeYUVPQBatch on the same device frames: (halves, half results, Out, YUV results)"""
    rgba = torch.zeros(F * 8 * w * h, dtype=torch.uint8, device="cuda")
    rres = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_half_batch(frames.data_ptr(), F, istride, used.data_ptr(), MAX_CHUNKS, w, h, rgba.data_ptr(), 8 * w * h,
                                      rres.data_ptr()) == 0
    out = out_of(F, w, h, i)
    yres = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_yuv_pq_batch(frames.data_ptr(), F, istride, used.data_ptr(), MAX_CHUNKS, w, h, out.luma, out.chroma, out.fstride,
                                   out.pitch, cs, unit, yres.data_ptr()) == 0
    return rgba.cpu().numpy().view(np.uint16).reshape(F, h, w, 4), rres.cpu().numpy(), out, yres.cpu().numpy()


def hdr_pictures(w, h, F, cs, signed):
    """picture-like HDR content as RGBA16F: HDR10 test pictures through the encoders' conversion, SF16 with some negatives"""
    pics = []
    for i in range(F):
        luma, chroma = P.hdr10_planes("video" if i % 2 == 0 else "gradient", w, h, cs, index=i)
        p = P.yuv_pq_to_rgba_half(luma, chroma, cs, 100)
        if signed:
            p[::3, ::5, 0] |= 0x8000
        pics.append(p)
    return np.stack(pics)


def encode_half_frames(lib, pics, fmt, comp, chunks):
    F, h, w = pics.shape[:3]
    ostride = D.align16(lib.max_encoded_length_half(w, h, fmt, chunks))
    out = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    src = D.dev(pics.view(np.uint8))
    assert lib.encode_rgba_half_batch(src.data_ptr(), F, 8 * w * h, w, h, fmt, comp, chunks, out.data_ptr(), ostride, used.data_ptr()) == 0
    return out, ostride, used


@pytest.mark.parametrize("fmt", [UF16, SF16], ids=["UF16", "SF16"])
def test_decode_batch_equals_the_half_decoder(lib, fmt):
    w, h, F = 260, 132, 3
    try:
        for k, (comp, chunks, index, offsets) in enumerate([(HapCompressorSnappy, 1, 0, 0), (HapCompressorSnappy, 8, 0, 0),
                                                            (HapCompressorSnappy, 8, 1, 0), (HapCompressorSnappy, 8, 0, 1),
                                                            (HapCompressorNone, 1, 0, 0)]):
            cs, unit = P.COLOR_SPACES[k % 2], (100, 203, 1000, 80, 10000)[k]
            lib.set_option(lib.OPTION_WRITE_INDEX, index)
            lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, offsets)
            frames, istride, used = encode_half_frames(lib, hdr_pictures(w, h, F, cs, fmt == SF16), fmt, comp, chunks)
            before = frames.cpu().numpy()
            halves, rres, out, yres = decode_both(lib, frames, F, istride, used, w, h, cs, unit, k)
            assert (rres == 0).all() and (yres == rres).all(), (comp, chunks, index, offsets, rres, yres)
            check(out, halves, cs, unit, (comp, chunks, index, offsets))
            assert (frames.cpu().numpy() == before).all()
    finally:
        lib.set_option(lib.OPTION_WRITE_INDEX, 0)
        lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def test_mixed_batch_results_equal_the_half_decoder_and_failed_frames_are_black(lib):
    """UF16 and SF16 frames, a truncated one, a Hap Q frame, frames 4 rows too large and too small, a frame of two textures"""
    w, h, k = 132, 20, 3
    tu, ts = B.textures(w, h, 2, seed=7), B.textures(w, h, 2, seed=8, signed=True)
    fu, fs = B.frames_of(lib, tu, UF16, k, lib), B.frames_of(lib, ts, SF16, k, lib)
    big, small = B.textures(w, h + 4, 1, seed=32)[0], B.textures(w, h - 4, 1, seed=33, signed=True)[0]
    alpha = bytes(np.random.default_rng(34).integers(0, 256, (w // 4) * (h // 4) * 8, dtype=np.uint8))
    r, two = lib.encode([tu[0], alpha], [UF16, HapTextureFormat_A_RGTC1], [HapCompressorSnappy] * 2, [k, k])
    assert r == 0
    r, hapq = lib.encode([bytes((w // 4) * (h // 4) * 16)], [HapTextureFormat_YCoCg_DXT5], [HapCompressorSnappy], [k])
    assert r == 0
    frames = [fu[0], fs[0], fu[1], hapq, B.frames_of(lib, [big], UF16, k, lib)[0], fs[1], B.frames_of(lib, [small], SF16, k, lib)[0], two]
    lens = [len(f) for f in frames]
    lens[2] -= 9                                                         # truncated
    istride = D.align16(max(lens) + 16)
    buf = np.zeros(len(frames) * istride, np.uint8)
    for i, f in enumerate(frames):
        buf[i * istride: i * istride + len(f)] = np.frombuffer(f, np.uint8)
    d = D.dev(buf)
    used = torch.tensor(lens, dtype=torch.int64, device="cuda")
    for cs in P.COLOR_SPACES:
        halves, rres, out, yres = decode_both(lib, d, len(frames), istride, used, w, h, cs, 203, cs)
        assert (yres == rres).all(), (rres, yres)
        assert [x != 0 for x in rres] == [False, False, True, True, True, False, True, True], rres
        check(out, halves, cs, 203, cs)
        yb, cb = Q.black(cs)
        got = out.d.cpu().numpy()
        for f in np.flatnonzero(rres != 0):
            lum = np.lib.stride_tricks.as_strided(got[f * out.fstride:], shape=(h, 2 * w), strides=(out.pitch, 1))
            chm = np.lib.stride_tricks.as_strided(got[out.chroma_at + f * out.fstride:], shape=(h // 2, 2 * w), strides=(out.pitch, 1))
            assert (np.ascontiguousarray(lum).view(np.uint16) == yb << 6).all() and (np.ascontiguousarray(chm).view(np.uint16) == cb << 6).all()
        # the single-frame call answers as HapB200DecodeRGBAHalf does
        for f, fr in enumerate(frames):
            fr = fr[: lens[f]]
            want = lib.decode_rgba_half(fr, w, h)[0]
            assert lib.decode_yuv_pq(fr, w, h, cs, 203)[0] == want, f
    assert (d.cpu().numpy() == buf).all()


def test_batch_of_65537_frames(lib):
    """4x4 pictures, 65537 of them: two launches (65535 + 2 frames)"""
    w, h, F = 4, 4, 65537
    pitch, fstride, chroma_at = 16, 96, 64
    rng = np.random.default_rng(65537)
    blocks = rng.integers(0, 256, (F, 16), dtype=np.uint8)
    for m in range(18):
        blocks[m::18] = U.random_blocks(rng, len(blocks[m::18]), m)
    blk = D.dev(blocks.ravel())
    for fmt in (UF16, SF16):
        out = D.Out(F, w, h, Y.P010, pitch, fstride, chroma_at)
        assert lib.block_decode_yuv_pq_batch(blk.data_ptr(), F, 16, w, h, fmt, out.luma, out.chroma, fstride, pitch, P.BT2020_LIMITED, 203) == 0
        check(out, halves_of_blocks(lib, blk, F, 16, w, h, fmt), P.BT2020_LIMITED, 203, fmt)
        del out
    # whole frames: seven distinct pictures repeat
    pics = hdr_pictures(w, h, 7, P.BT2020_FULL, False)
    frames7, istride, used7 = encode_half_frames(lib, pics, UF16, HapCompressorSnappy, 1)
    idx = torch.arange(F, device="cuda") % 7
    frames = frames7.view(7, istride)[idx].reshape(-1)
    halves, rres, out, yres = decode_both(lib, frames, F, istride, used7[idx], w, h, P.BT2020_FULL, 1000, 0)
    assert (rres == 0).all() and (yres == 0).all()
    check(out, halves, P.BT2020_FULL, 1000, "frames")


@pytest.mark.parametrize("fmt", [UF16, SF16], ids=["UF16", "SF16"])
def test_single_frame_host_and_device_unaligned(lib, fmt):
    w, h = 132, 68
    pitch = 2 * w + 7                                                      # odd: the single-frame call copies
    frames, _, used = encode_half_frames(lib, hdr_pictures(w, h, 1, P.BT2020_LIMITED, fmt == SF16), fmt, HapCompressorSnappy, 4)
    fr = frames[: int(used[0])].cpu().numpy()
    r, half = lib.decode_rgba_half(fr.tobytes(), w, h)
    assert r == 0
    half = np.frombuffer(half, np.uint16).reshape(h, w, 4)
    for cs in P.COLOR_SPACES:
        for unit in (100, 10000):
            lu, ch = Q.rgba_half_to_yuv_pq(half, cs, unit)
            want_l, want_c = Y.pitched(lu, pitch, PAD), Y.pitched(ch, pitch, PAD)
            hf = np.zeros(fr.size + 1, np.uint8)[1:]
            hf[:] = fr
            hl = np.full(want_l.size + 1, PAD, np.uint8)[1:]
            hc = np.full(want_c.size + 3, PAD, np.uint8)[3:]
            r, _ = lib.decode_yuv_pq(hf, w, h, cs, unit, pitch=pitch, luma=hl, chroma=hc)
            assert r == 0 and (hl == want_l.ravel()).all() and (hc == want_c.ravel()).all(), (cs, unit)
            df = D.dev(np.concatenate([[0, 0, 0, 0, 0], fr]).astype(np.uint8))
            dl = torch.full((want_l.size + 1,), PAD, dtype=torch.uint8, device="cuda")
            dc = torch.full((want_c.size + 3,), PAD, dtype=torch.uint8, device="cuda")
            r, _ = lib.decode_yuv_pq((df.data_ptr() + 5, fr.size), w, h, cs, unit, pitch=pitch, luma=(dl.data_ptr() + 1, want_l.size),
                                     chroma=(dc.data_ptr() + 3, want_c.size))
            assert r == 0 and (dl.cpu().numpy()[1:] == want_l.ravel()).all() and (dc.cpu().numpy()[3:] == want_c.ravel()).all(), (cs, unit)
            assert (df.cpu().numpy()[5:] == fr).all()
            r, planes = lib.decode_yuv_pq(fr.tobytes(), w, h, cs, unit)
            assert r == 0 and planes == (lu.tobytes(), ch.tobytes()), (cs, unit)


def flat_triples(cs, unit, n, seed):
    """n random nominal-range P010 triples whose 12-bit R'G'B' (HAPB200_YUV_PQ_COEFFICIENTS) is not clamped and whose codes
    all sit at or above the round-trip floor of unit (the lowest code from which P[T[c]] = c holds)"""
    floor = {1: 0, 100: 0, 123: 0, 203: 2, 1000: 16, 10000: 180}[unit]
    cy, crr, cbg, crg, cbb, yoff, coff = (int(v) for v in P.coefficients()[cs - P.BT2020_LIMITED])
    lo, hi_y, hi_c = (64, 940, 960) if cs == P.BT2020_LIMITED else (0, 1023, 1023)
    rng = np.random.default_rng(seed)
    y = rng.integers(lo, hi_y + 1, 8 * n)
    cb, cr = rng.integers(lo, hi_c + 1, 8 * n), rng.integers(lo, hi_c + 1, 8 * n)
    yd, cb8, cr8 = cy * (y - yoff), 8 * (cb - coff), 8 * (cr - coff)
    rgb = np.stack([(yd + crr * cr8 + 32768) >> 16, (yd + cbg * cb8 + crg * cr8 + 32768) >> 16, (yd + cbb * cb8 + 32768) >> 16], -1)
    keep = ((rgb >= floor) & (rgb <= 4095)).all(-1)
    assert keep.sum() >= n
    return y[keep][:n], cb[keep][:n], cr[keep][:n]


@pytest.mark.parametrize("fmt", [UF16, SF16], ids=["UF16", "SF16"])
def test_flat_pictures_round_trip_through_the_hdr10_encoder(lib, fmt):
    w, h, F = 8, 8, 512
    pitch, fstride = 2 * w, 2 * w * h + 2 * w * h // 2
    for i, (cs, unit) in enumerate([(P.BT2020_LIMITED, 1), (P.BT2020_FULL, 100), (P.BT2020_LIMITED, 123), (P.BT2020_FULL, 203),
                                    (P.BT2020_LIMITED, 1000), (P.BT2020_FULL, 10000)]):
        y, cb, cr = flat_triples(cs, unit, F, seed=i)
        pic = np.zeros((F, fstride // 2), np.uint16)
        pic[:, : w * h] = (y << 6)[:, None]
        pic[:, w * h:] = np.tile(np.stack([cb, cr], -1)[:, None, :], (1, w * h // 4, 1)).reshape(F, -1) << 6
        src = D.dev(pic.view(np.uint8).ravel())
        ostride = D.align16(lib.max_encoded_length_half(w, h, fmt, 1))
        frames = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
        used = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_yuv_pq_batch(src.data_ptr(), src.data_ptr() + 2 * w * h, F, fstride, w, h, pitch, cs, unit, fmt, HapCompressorSnappy,
                                       1, frames.data_ptr(), ostride, used.data_ptr()) == 0
        back = torch.full((F * fstride,), PAD, dtype=torch.uint8, device="cuda")
        res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
        assert lib.decode_yuv_pq_batch(frames.data_ptr(), F, ostride, used.data_ptr(), 1, w, h, back.data_ptr(), back.data_ptr() + 2 * w * h,
                                       fstride, pitch, cs, unit, res.data_ptr()) == 0
        assert (res.cpu().numpy() == 0).all()
        got = back.cpu().numpy().view(np.uint16).reshape(F, -1)
        bad = np.flatnonzero((got != pic).any(-1))
        assert bad.size == 0, (cs, unit, bad.size, y[bad[:3]], cb[bad[:3]], cr[bad[:3]])
