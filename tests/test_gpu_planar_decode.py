"""Planar decoders on the GPU (HapB200BlockDecodePlanarBatch, HapB200DecodePlanarBatch, HapB200DecodePlanar): every plane must
equal, byte for byte, planar_out_util.rgba_to_planar_out (the definition of include/hap_b200.h) of what the RGBA8 decoders give
for the same input, and the batch results must equal theirs -- for every codec, subsampling, depth and colour space, with and
without the alpha plane; on random textures at small shapes, Snappy-chunked frames (with the index and offset-table options),
uncompressed frames, the reference's own frames, a batch of more than 65535 frames and a batch mixing good, truncated,
wrong-codec and Hap HDR frames; single frames from host and device memory at odd addresses and pitches.  Hap Alpha-Only writes
its matte to the alpha plane alone.  Sentinels around every plane must survive and the inputs must be left as they were.  End
to end, Hap Q and Hap Q Alpha batches decoded to yuva444p12le and encoded again by the planar encoder give the frames the RGBA8
encoder gives from the RGBA8 decode."""
import numpy as np
import pytest
import torch

import hap_b200
import hap_b200.lib as L
import planar_out_util as Q
import planar_util as P
from golden_util import b64, golden
from hap_b200 import synth
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy

pytestmark = pytest.mark.gpu
PAD = 0xEE
CODECS = {"Hap1": L.HapB200Codec_Hap1, "Hap5": L.HapB200Codec_Hap5, "HapY": L.HapB200Codec_HapY, "HapM": L.HapB200Codec_HapM,
          "HapA": L.HapB200Codec_HapA, "Hap7": L.HapB200Codec_Hap7}
CASES = [(c, sub, n, cs, alpha) for c in CODECS for sub in Q.SUBSAMPLINGS for n in Q.DEPTHS for cs in Q.COLOR_SPACES
         for alpha in (True, False) if c != "HapA" or alpha]
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
    """F random textures of codec c, texture 1 (Hap Q Alpha) at texture_bytes(.., 0)"""
    t = lib.texture_bytes(w, h, c, 0) + lib.texture_bytes(w, h, c, 1)
    return np.random.default_rng(seed).integers(0, 256, (F, t), dtype=np.uint8)


def want_planes(rgba, codec, sub, n, cs, alpha):
    """the four planes (as stored, None where nothing is written) of RGBA8 pictures (h, w, 4) or (F, h, w, 4) decoded from frames
    of `codec`.  Pictures stacked vertically convert as one: no filter reaches across a picture's top or bottom edge."""
    rgba = np.asarray(rgba)
    if rgba.ndim == 4:
        F, h = rgba.shape[:2]
        planes = want_planes(rgba.reshape(F * h, *rgba.shape[2:]), codec, sub, n, cs, alpha)
        return tuple(None if p is None else p.reshape(F, p.shape[0] // F, p.shape[1]) for p in planes)
    if codec == "HapA":   # the matte v is R (= G = B) of the RGBA8 picture
        return None, None, None, Q.store(Q.alpha_out(rgba[..., 0], n), n)
    return Q.rgba_to_planar_out(rgba, sub, n, cs, alpha)


class Out:
    """F pictures' four planes, each in a device buffer of its own filled with PAD that ends with its last frame's last sample:
    frame f's plane at its pointer + f*fstride, luma and alpha rows lpitch apart, Cb and Cr rows cpitch apart"""

    def __init__(self, F, w, h, sub, n, lpitch, cpitch, fstride):
        self.F, self.w, self.h, self.sub, self.n = F, w, h, sub, n
        self.lpitch, self.cpitch, self.fstride = lpitch, cpitch, fstride
        sb = P.sample_bytes(n)
        ch, cw = P.chroma_shape(w, h, sub)
        self.shape = [(h, sb * w, lpitch), (ch, sb * cw, cpitch), (ch, sb * cw, cpitch), (h, sb * w, lpitch)]
        self.d = [torch.full(((F - 1) * fstride + (r - 1) * p + b,), PAD, dtype=torch.uint8, device="cuda") for r, b, p in self.shape]

    def ptrs(self, alpha=True, colour=True):
        return [t.data_ptr() if (k == 3 and alpha) or (k < 3 and colour) else 0 for k, t in enumerate(self.d)]

    def check(self, planes, what=""):
        """planes[k]: plane k of every frame as stored, (F, rows, samples) (None: that plane must be untouched); every other
        byte PAD"""
        for k in range(4):
            rows, nbytes, pitch = self.shape[k]
            want = np.full(self.d[k].numel(), PAD, np.uint8)
            if planes[k] is not None:
                r = np.ascontiguousarray(planes[k]).view(np.uint8).reshape(self.F, rows, nbytes)
                np.lib.stride_tricks.as_strided(want, shape=r.shape, strides=(self.fstride, pitch, 1))[...] = r
            got = self.d[k].cpu().numpy()
            bad = np.flatnonzero(got != want)
            assert bad.size == 0, (what, "plane", k, bad.size, bad[:8])

    def check_rgba(self, rgba, codec, cs, alpha, what=""):
        self.check(want_planes(rgba, codec, self.sub, self.n, cs, alpha), what)


def geometry(w, h, sub, n, i=1):
    """pitches wider than the rows and unequal, frame-stride slack"""
    sb = P.sample_bytes(n)
    ch, cw = P.chroma_shape(w, h, sub)
    lpitch, cpitch = align16(sb * w) + 16 * (1 + i % 3), align16(sb * cw) + 16 * (1 + (i + 1) % 3)
    return lpitch, cpitch, align16(max(lpitch * h, cpitch * ch)) + 16 * (1 + i % 2)


def rgba_of_blocks(lib, blk, F, bstride, w, h, c):
    rgba = torch.zeros(F * 4 * w * h, dtype=torch.uint8, device="cuda")
    assert lib.block_decode_batch(blk.data_ptr(), F, bstride, w, h, c, rgba.data_ptr(), 4 * w * h) == 0
    return rgba.cpu().numpy().reshape(F, h, w, 4)


def padded_blocks(t, extra):
    bstride = align16(t.shape[1]) + extra
    blk_np = np.zeros((t.shape[0], bstride), np.uint8)
    blk_np[:, : t.shape[1]] = t
    return blk_np, bstride


@pytest.mark.parametrize("codec,sub,n,cs,alpha", CASES)
def test_block_decode_planar_batch_equals_rgba(lib, codec, sub, n, cs, alpha):
    c = CODECS[codec]
    w, h, F = 132, 20, 3                                                  # 33 block columns: two warp spans per row
    blk_np, bstride = padded_blocks(textures(lib, w, h, c, F, seed=100 * c + 10 * n + cs), 48)
    blk = dev(blk_np.ravel())
    lpitch, cpitch, fstride = geometry(w, h, sub, n, cs)
    out = Out(F, w, h, sub, n, lpitch, cpitch, fstride)
    assert lib.block_decode_planar_batch(blk.data_ptr(), F, bstride, w, h, c, *out.ptrs(alpha, codec != "HapA"), fstride, lpitch, cpitch,
                                         sub, n, cs) == 0
    out.check_rgba(rgba_of_blocks(lib, blk, F, bstride, w, h, c), codec, cs, alpha, (codec, sub, n, cs, alpha))
    assert (blk.cpu().numpy() == blk_np.ravel()).all()
    if codec == "HapA":   # luma, Cb and Cr given: still untouched
        out2 = Out(F, w, h, sub, n, lpitch, cpitch, fstride)
        assert lib.block_decode_planar_batch(blk.data_ptr(), F, bstride, w, h, c, *out2.ptrs(), fstride, lpitch, cpitch, sub, n, cs) == 0
        out2.check_rgba(rgba_of_blocks(lib, blk, F, bstride, w, h, c), codec, cs, alpha, "HapA with every plane")


@pytest.mark.parametrize("sub", Q.SUBSAMPLINGS)
def test_block_decode_planar_geometry(lib, sub):
    shapes = [(w, h) for w in (4, 8, 12, 20, 36, 124, 128, 132, 516) for h in (4, 8, 12, 20)] + [(1924, 1084)]
    for i, (w, h) in enumerate(shapes):
        for codec in ("Hap1", "HapM", "Hap7", "HapA"):
            c = CODECS[codec]
            F, cs, n, alpha = 3, i % 4, Q.DEPTHS[i % 3], codec == "HapA" or i % 2 == 0
            blk_np, bstride = padded_blocks(textures(lib, w, h, c, F, seed=i), 16 * (i % 3))
            blk = dev(blk_np.ravel())
            lpitch, cpitch, fstride = geometry(w, h, sub, n, i)
            out = Out(F, w, h, sub, n, lpitch, cpitch, fstride)
            assert lib.block_decode_planar_batch(blk.data_ptr(), F, bstride, w, h, c, *out.ptrs(alpha, codec != "HapA"), fstride, lpitch,
                                                 cpitch, sub, n, cs) == 0
            out.check_rgba(rgba_of_blocks(lib, blk, F, bstride, w, h, c), codec, cs, alpha, (w, h, codec))


def encode_frames(lib, pics, c, comp, chunks):
    """pictures (F, h, w, 4) uint8 -> (device frames at a common stride, stride, device lengths)"""
    F, h, w = pics.shape[:3]
    ostride = align16(lib.max_encoded_length_rgba(w, h, c, chunks))
    out = torch.zeros(F * ostride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    src = dev(pics)
    if c == L.HapB200Codec_Hap7:
        r = lib.encode_rgba_bc7_batch(src.data_ptr(), F, 4 * w * h, w, h, comp, chunks, out.data_ptr(), ostride, used.data_ptr())
    else:
        r = lib.encode_rgba_batch(src.data_ptr(), F, 4 * w * h, w, h, c, comp, chunks, out.data_ptr(), ostride, used.data_ptr())
    assert r == 0
    return out, ostride, used


def decode_both(lib, frames, F, istride, used, codec, w, h, sub, n, cs, alpha, i=1):
    """HapB200DecodeRGBABatch and HapB200DecodePlanarBatch on the same frames: (RGBA pictures, RGBA results, Out, planar results)"""
    c = CODECS[codec]
    rgba = torch.zeros(F * 4 * w * h, dtype=torch.uint8, device="cuda")
    rres = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_rgba_batch(frames.data_ptr(), F, istride, used.data_ptr(), MAX_CHUNKS, c, w, h, rgba.data_ptr(), 4 * w * h,
                                 rres.data_ptr()) == 0
    lpitch, cpitch, fstride = geometry(w, h, sub, n, i)
    out = Out(F, w, h, sub, n, lpitch, cpitch, fstride)
    pres = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    assert lib.decode_planar_batch(frames.data_ptr(), F, istride, used.data_ptr(), MAX_CHUNKS, c, w, h, *out.ptrs(alpha, codec != "HapA"),
                                   fstride, lpitch, cpitch, sub, n, cs, pres.data_ptr()) == 0
    return rgba.cpu().numpy().reshape(F, h, w, 4), rres.cpu().numpy(), out, pres.cpu().numpy()


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("sub", Q.SUBSAMPLINGS)
def test_decode_planar_batch_equals_rgba(lib, codec, sub):
    w, h, F = 260, 132, 3
    pics = np.stack([synth.frame(w, h, i, kind="video" if i % 2 == 0 else "gradient", alpha="ramp").numpy() for i in range(F)])
    try:
        for k, (comp, chunks, index, offsets) in enumerate([(HapCompressorSnappy, 1, 0, 0), (HapCompressorSnappy, 8, 0, 0),
                                                            (HapCompressorSnappy, 8, 1, 0), (HapCompressorSnappy, 8, 0, 1),
                                                            (HapCompressorNone, 1, 0, 0)]):
            lib.set_option(lib.OPTION_WRITE_INDEX, index)
            lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, offsets)
            frames, istride, used = encode_frames(lib, pics, CODECS[codec], comp, chunks)
            before = frames.cpu().numpy()
            for j, n in enumerate(Q.DEPTHS):
                cs, alpha = (k + j) % 4, codec == "HapA" or (k + j) % 2 == 0
                rgba, rres, out, pres = decode_both(lib, frames, F, istride, used, codec, w, h, sub, n, cs, alpha, k)
                assert (rres == 0).all() and (pres == rres).all(), (comp, chunks, index, offsets, rres, pres)
                out.check_rgba(rgba, codec, cs, alpha, (comp, chunks, index, offsets, n))
            assert (frames.cpu().numpy() == before).all()
    finally:
        lib.set_option(lib.OPTION_WRITE_INDEX, 0)
        lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, 0)


def test_decode_planar_of_the_reference_frames(lib):
    """frames the reference's encoder wrote: 4096 blocks each, decoded as 256 x 256 pictures, batch and single-frame"""
    names = {"dxt1": "Hap1", "dxt5": "Hap5", "ycocg": "HapY", "rgtc1": "HapA", "hapm": "HapM"}
    w = h = 256
    for name, e in golden()["ref_frames"].items():
        codec = names[name]
        fr = np.frombuffer(b64(e["frame_b64"]), np.uint8)
        frames = dev(fr)
        used = torch.tensor([fr.size], dtype=torch.int64, device="cuda")
        for sub in Q.SUBSAMPLINGS:
            for n in Q.DEPTHS:
                cs = (sub + n) % 4
                rgba, rres, out, pres = decode_both(lib, frames, 1, fr.size, used, codec, w, h, sub, n, cs, True, cs)
                assert rres[0] == 0 and pres[0] == 0, (name, rres, pres)
                out.check_rgba(rgba, codec, cs, True, (name, sub, n))
                # the single-frame call, host frame, tight planes allocated by the wrapper
                r, planes = lib.decode_planar(fr.tobytes(), w, h, sub, n, cs)
                want = want_planes(rgba[0], codec, sub, n, cs, True)
                assert r == 0, (name, r)
                for k in range(4):
                    if want[k] is not None:
                        assert planes[k] == want[k].tobytes(), (name, sub, n, k)
                    elif planes[k] is not None:
                        assert not any(planes[k]), (name, sub, n, k)       # allocated zeroed, never written


def test_decode_planar_batch_mixed_good_truncated_wrong_codec_and_hdr(lib):
    w, h = 132, 68
    c = L.HapB200Codec_HapM
    pics = np.stack([synth.frame(w, h, i, alpha="ramp").numpy() for i in range(4)])
    good, gstride, gused = encode_frames(lib, pics, c, HapCompressorSnappy, 4)
    other, ostride_, oused = encode_frames(lib, pics[:1], L.HapB200Codec_Hap1, HapCompressorSnappy, 4)
    half = np.zeros((h, w, 4), np.float16)
    half[..., :3] = 0.25
    r, hdr = lib.encode_rgba_half(half.view(np.uint8), w, h, 0x8E8F)   # HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT
    assert r == 0
    istride = align16(max(gstride, ostride_, len(hdr)))
    F = 7
    buf = torch.zeros(F * istride, dtype=torch.uint8, device="cuda")
    lens = []
    # frames: good, truncated, good, wrong codec (Hap1 in a Hap Q Alpha stream), truncated to a header, Hap HDR, good
    plan = [("good", 0), ("trunc", 1), ("good", 2), ("wrong", 0), ("head", 3), ("hdr", 0), ("good", 3)]
    for f, (kind, src) in enumerate(plan):
        if kind == "wrong":
            n = int(oused[0])
            buf[f * istride: f * istride + n] = other[:n]
        elif kind == "hdr":
            n = len(hdr)
            buf[f * istride: f * istride + n] = dev(np.frombuffer(hdr, np.uint8))
        else:
            n = int(gused[src])
            buf[f * istride: f * istride + n] = good[src * gstride: src * gstride + n]
            n = n // 2 if kind == "trunc" else 8 if kind == "head" else n
        lens.append(n)
    used = torch.tensor(lens, dtype=torch.int64, device="cuda")
    ok = np.array([k == "good" for k, _ in plan])
    for sub in Q.SUBSAMPLINGS:
        for n in Q.DEPTHS:
            cs = (sub + n) % 4
            rgba, rres, out, pres = decode_both(lib, buf, F, istride, used, "HapM", w, h, sub, n, cs, True, cs)
            assert (pres == rres).all(), (rres, pres)
            assert (rres[ok] == 0).all() and (rres[~ok] != 0).all(), rres
            assert (rgba[~ok] == 0).all()
            out.check_rgba(rgba, "HapM", cs, True, (sub, n))
            # failed frames are black and transparent: Y = yOff, Cb = Cr = cOff, alpha 0
            yb, cb = Q.black(n, cs)
            for f in np.flatnonzero(~ok):
                lu, cbp, crp, al = want_planes(np.zeros((h, w, 4), np.uint8), "HapM", sub, n, cs, True)
                assert (lu == yb).all() and (cbp == cb).all() and (crp == cb).all() and (al == 0).all()


def test_planar_decode_batch_of_65537_frames(lib):
    """4x4 pictures, 65537 of them: two launches (65535 + 2 frames)"""
    w, h, F = 4, 4, 65537
    for sub, n in ((Q.S420, 10), (Q.S444, 8), (Q.S422, 12)):
        sb = P.sample_bytes(n)
        lpitch, cpitch, fstride = 16, 16, 96
        for codec in ("Hap1", "Hap7", "HapA"):
            c = CODECS[codec]
            t = textures(lib, w, h, c, F, seed=sub)
            blk = dev(np.pad(t, ((0, 0), (0, 16 - t.shape[1]))).ravel())
            out = Out(F, w, h, sub, n, lpitch, cpitch, fstride)
            assert lib.block_decode_planar_batch(blk.data_ptr(), F, 16, w, h, c, *out.ptrs(True, codec != "HapA"), fstride, lpitch, cpitch,
                                                 sub, n, P.COLOR_SPACES[1]) == 0
            out.check_rgba(rgba_of_blocks(lib, blk, F, 16, w, h, c), codec, P.COLOR_SPACES[1], True, (codec, sub, n))
            del out, blk
        # whole frames, Hap Q: seven distinct pictures repeat
        pics = np.stack([synth.frame(w, h, i).numpy() for i in range(7)])
        frames7, istride, used7 = encode_frames(lib, pics, CODECS["HapY"], HapCompressorSnappy, 1)
        idx = torch.arange(F, device="cuda") % 7
        frames = frames7.view(7, istride)[idx].reshape(-1)
        used = used7[idx]
        rgba, rres, out, pres = decode_both(lib, frames, F, istride, used, "HapY", w, h, sub, n, 2, sb == 2)
        assert (rres == 0).all() and (pres == 0).all()
        out.check_rgba(rgba, "HapY", 2, sb == 2, ("HapY frames", sub, n))
        del out, frames


@pytest.mark.parametrize("codec", list(CODECS))
@pytest.mark.parametrize("sub", Q.SUBSAMPLINGS)
def test_decode_planar_single_frame_host_and_device_unaligned(lib, codec, sub):
    c = CODECS[codec]
    w, h = 132, 68
    pics = synth.frame(w, h, 3, alpha="ramp").numpy()[None]
    frames, _, used = encode_frames(lib, pics, c, HapCompressorSnappy, 4)
    fr = frames[: int(used[0])].cpu().numpy()
    r, rgba = lib.decode_rgba(fr.tobytes(), w, h)
    assert r == 0
    rgba = np.frombuffer(rgba, np.uint8).reshape(h, w, 4)
    for k, n in enumerate(Q.DEPTHS):
        cs, alpha = (k + sub) % 4, codec == "HapA" or k != 1
        sb = P.sample_bytes(n)
        ch, cw = P.chroma_shape(w, h, sub)
        lpitch, cpitch = sb * w + 7, sb * cw + 5                               # odd: the single-frame call copies
        want = want_planes(rgba, codec, sub, n, cs, alpha)
        shapes = [(h, lpitch), (ch, cpitch), (ch, cpitch), (h, lpitch)]
        exp = [np.full(r_ * p_, PAD, np.uint8) if wnt is None else P.Y.pitched(wnt, p_, PAD).ravel() for wnt, (r_, p_) in zip(want, shapes)]
        given = [True, True, True, alpha] if codec != "HapA" else [False, False, False, True]
        # host frame and planes at odd addresses (Hap Alpha-Only: luma, Cb and Cr NULL)
        hf = np.zeros(fr.size + 1, np.uint8)[1:]
        hf[:] = fr
        hp = [np.full(e.size + 1 + j, PAD, np.uint8)[1 + j:] for j, e in enumerate(exp)]
        hosts = dict(zip(("luma", "cb", "cr", "alpha"), [p if g else None for p, g in zip(hp, given)]))
        r, _ = lib.decode_planar(hf, w, h, sub, n, cs, luma_pitch=lpitch, chroma_pitch=cpitch, **hosts)
        assert r == 0, (n, r)
        for j in range(4):
            if given[j]:
                assert (hp[j] == exp[j]).all(), (n, j)
        # device frame and planes at odd addresses
        df = dev(np.concatenate([[0, 0, 0, 0, 0], fr]).astype(np.uint8))
        dp = [torch.full((e.size + 1 + j,), PAD, dtype=torch.uint8, device="cuda") for j, e in enumerate(exp)]
        devs = dict(zip(("luma", "cb", "cr", "alpha"), [(d.data_ptr() + 1 + j, exp[j].size) if g else None for j, (d, g) in enumerate(zip(dp, given))]))
        r, _ = lib.decode_planar((df.data_ptr() + 5, fr.size), w, h, sub, n, cs, luma_pitch=lpitch, chroma_pitch=cpitch, **devs)
        assert r == 0, (n, r)
        for j in range(4):
            got = dp[j].cpu().numpy()
            assert (got[1 + j:] == exp[j]).all() if given[j] else (got == PAD).all(), (n, j)
        assert (df.cpu().numpy()[5:] == fr).all()


def test_decode_planar_answers_as_decode_rgba_for_hap_hdr_and_bad_frames(lib):
    w, h = 16, 8
    half = np.zeros((h, w, 4), np.float16)
    half[..., :3] = 0.5
    r, hdr = lib.encode_rgba_half(half.view(np.uint8), w, h, 0x8E8F)     # HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT
    assert r == 0
    for frame in (hdr, b"\x00\x00\x00\xbb", b"\x01"):
        want, _ = lib.decode_rgba(frame, w, h)
        for sub in Q.SUBSAMPLINGS:
            r, _ = lib.decode_planar(frame, w, h, sub, 10, P.COLOR_SPACES[2])
            assert r == want != 0, (frame[:8], r, want)
    assert lib.decode_rgba(hdr, w, h)[0] == BAD_FRAME


@pytest.mark.parametrize("codec", ["HapY", "HapM"])
def test_yuva444p12le_round_trip_gives_the_rgba_encoders_frames(lib, codec):
    """Hap Q / Hap Q Alpha frames -> yuva444p12le -> the planar encoder: the frames the RGBA8 encoder makes of the RGBA8 decode"""
    c = CODECS[codec]
    w, h, F, n, sub = 516, 260, 3, 12, Q.S444
    pics = np.stack([synth.frame(w, h, i, kind="video" if i % 2 == 0 else "gradient", alpha="ramp").numpy() for i in range(F)])
    frames, istride, used = encode_frames(lib, pics, c, HapCompressorSnappy, 8)
    for cs in Q.COLOR_SPACES:
        rgba, rres, out, pres = decode_both(lib, frames, F, istride, used, codec, w, h, sub, n, cs, True, cs)
        assert (rres == 0).all() and (pres == 0).all()
        ostride = align16(lib.max_encoded_length_rgba(w, h, c, 8))
        got = torch.full((F * ostride,), PAD, dtype=torch.uint8, device="cuda")
        gused = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_planar_batch(*out.ptrs(), F, out.fstride, w, h, out.lpitch, out.cpitch, sub, n, cs, c, HapCompressorSnappy, 8,
                                       got.data_ptr(), ostride, gused.data_ptr()) == 0
        want = torch.full((F * ostride,), PAD, dtype=torch.uint8, device="cuda")
        wused = torch.zeros(F, dtype=torch.int64, device="cuda")
        assert lib.encode_rgba_batch(dev(rgba).data_ptr(), F, 4 * w * h, w, h, c, HapCompressorSnappy, 8, want.data_ptr(), ostride,
                                     wused.data_ptr()) == 0
        assert (gused.cpu().numpy() == wused.cpu().numpy()).all(), cs
        assert (got.cpu().numpy() == want.cpu().numpy()).all(), cs
