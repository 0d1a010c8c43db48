"""The fused Hap Q encoder (hapq_fused.cuh): HapB200EncodeRGBABatch and HapB200EncodeRGBA with HapY must give the frames of
the two-kernel path (HapB200BlockEncodeBatch, then HapB200EncodeBatch) byte for byte, on 4K batches and on geometries where
fragments start mid-row, last fragments are short, chunks are 1, 3, 8 or 64, frames lie wider apart than they are long,
content is flat or noise (the chunk and whole-section fallbacks copy the written-through texture), with the fragment index
and the offset table on and off.  The reference decoder reproduces the texture, and the stage counters show which path ran."""
import numpy as np
import pytest
import torch

import hap_b200
import oracles
from hap_b200 import synth
from hap_b200.abi import HapCompressorNone, HapCompressorSnappy, HapTextureFormat_YCoCg_DXT5
from hap_b200.lib import HapB200Codec_HapM, HapB200Codec_HapY

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    L = hap_b200.load()
    yield L
    for opt in (L.OPTION_WRITE_INDEX, L.OPTION_WRITE_OFFSET_TABLE, L.OPTION_CHROMA_REFINE):
        L.set_option(opt, 0)


def pictures(w, h, frames, kind, seed, pad_row=0, pad_frame=0):
    """frames RGBA8 pictures (rows 4w + pad_row bytes apart, frames h * row + pad_frame apart) on cuda:0."""
    row, rng = 4 * w + pad_row, np.random.default_rng(seed)
    fstride = h * row + pad_frame
    buf = np.full(frames * fstride, 0xA5, dtype=np.uint8)
    for f in range(frames):
        if kind == "noise":
            img = rng.integers(0, 256, size=(h, w, 4), dtype=np.uint8)
        elif kind == "flat":
            img = np.zeros((h, w, 4), dtype=np.uint8)
            img[...] = (16 + 7 * f, 128, 200, 255)
        elif kind == "mixed":   # picture content on top, noise below: chunk fallbacks in a compressed frame
            img = synth.frame(w, h, seed + f).numpy().copy()
            img[h // 2:] = rng.integers(0, 256, size=(h - h // 2, w, 4), dtype=np.uint8)
        else:
            img = synth.frame(w, h, seed + f).numpy()
        v = buf[f * fstride: f * fstride + h * row].reshape(h, row)
        v[:, : 4 * w] = img.reshape(h, 4 * w)
    return torch.from_numpy(buf).cuda(), row, fstride


def encode_both(lib, rgba, frames, fstride, w, h, row, chunks, codec=HapB200Codec_HapY, compressor=HapCompressorSnappy):
    """(frames of HapB200EncodeRGBABatch, frames of block encode + HapB200EncodeBatch, textures, stage launches of the first)"""
    n = lib.texture_bytes(w, h, codec, 0)
    cap = (lib.max_encoded_length_rgba(w, h, codec, chunks) + 15) // 16 * 16
    out = [torch.zeros(frames * cap, dtype=torch.uint8, device="cuda") for _ in range(2)]
    used = [torch.zeros(frames, dtype=torch.int64, device="cuda") for _ in range(2)]
    lib.set_stage_timing(True)
    lib.stage_times()
    assert lib.encode_rgba_batch(rgba.data_ptr(), frames, fstride, w, h, codec, compressor, chunks, out[0].data_ptr(), cap,
                                 used[0].data_ptr(), row_bytes=row) == 0
    launches = {k: v[1] for k, v in lib.stage_times().items()}
    lib.set_stage_timing(False)
    tstride = (n + 15) // 16 * 16
    tex = torch.zeros(frames * tstride, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_batch(rgba.data_ptr(), frames, fstride, w, h, codec, tex.data_ptr(), tstride, row_bytes=row) == 0
    assert lib.encode_batch([tex.data_ptr()], [tstride], [n], [HapTextureFormat_YCoCg_DXT5], [compressor], [chunks], frames,
                            out[1].data_ptr(), cap, used[1].data_ptr()) == 0
    torch.cuda.synchronize()
    u = [x.cpu().numpy() for x in used]
    o = [x.cpu().numpy() for x in out]
    fr = [[o[k][f * cap: f * cap + u[k][f]].tobytes() for f in range(frames)] for k in range(2)]
    t = tex.cpu().numpy()
    return fr[0], fr[1], [t[f * tstride: f * tstride + n].tobytes() for f in range(frames)], launches


CASES = [
    # (w, h, frames, chunks, content, pad_row, pad_frame)
    (3840, 2160, 6, 8, "synth", 0, 0),            # bench.py's frames: 32 fragments per chunk, the last one short
    (3840, 2160, 2, 64, "synth", 0, 4096),
    (1924, 1084, 3, 3, "synth", 48, 272),          # 481 blocks per row: fragments start mid-row
    (1000, 600, 4, 1, "mixed", 16, 0),
    (516, 260, 3, 64, "synth", 0, 16),
    (256, 128, 5, 8, "flat", 0, 0),
    (640, 480, 3, 8, "noise", 0, 0),               # every chunk stored raw: the whole-section fallback
    (1024, 1024, 2, 3, "mixed", 0, 0),
]


@pytest.mark.parametrize("index,offsets", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}x{c[1]}x{c[2]}_{c[3]}ch_{c[4]}" for c in CASES])
def test_fused_batch_matches_two_kernel_path(lib, case, index, offsets):
    w, h, frames, chunks, kind, pad_row, pad_frame = case
    if (w, h) == (3840, 2160) and (index, offsets) not in ((0, 0), (1, 0)):
        pytest.skip("4K runs with the index on and off")
    lib.set_option(lib.OPTION_WRITE_INDEX, index)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, offsets)
    rgba, row, fstride = pictures(w, h, frames, kind, seed=w + chunks, pad_row=pad_row, pad_frame=pad_frame)
    fused, two, tex, launches = encode_both(lib, rgba, frames, fstride, w, h, row, chunks)
    assert launches.get("snappy_encode", 0) == 0 and launches.get("bc_encode", 0) == 1, launches
    for f in range(frames):
        assert fused[f] == two[f], f"frame {f} differs"
    ref = oracles.ref_abi() or oracles.oracle_abi()
    n = lib.texture_bytes(w, h, HapB200Codec_HapY, 0)
    for f in (0, frames - 1):
        r, t, fmt, _ = ref.decode(fused[f], 0, n)
        assert r == 0 and fmt == HapTextureFormat_YCoCg_DXT5 and t == tex[f]


def test_single_picture_entry_point(lib):
    w, h = 1924, 1084
    rgba, row, _ = pictures(w, h, 1, "synth", seed=5)
    host = rgba.cpu().numpy()
    r, frame = lib.encode_rgba(host, w, h, HapB200Codec_HapY, HapCompressorSnappy, 8)
    assert r == 0
    _, two, tex, _ = encode_both(lib, rgba, 1, h * row, w, h, row, 8)
    assert frame == two[0]
    ref = oracles.ref_abi() or oracles.oracle_abi()
    assert ref.decode(frame, 0, len(tex[0]))[1] == tex[0]


@pytest.mark.parametrize("variant", ["no_compressor", "refine", "hapm"])
def test_other_encodes_keep_the_two_kernel_path(lib, variant):
    w, h, frames, chunks = 516, 260, 2, 3
    rgba, row, fstride = pictures(w, h, frames, "synth", seed=9)
    codec = HapB200Codec_HapM if variant == "hapm" else HapB200Codec_HapY
    compressor = HapCompressorNone if variant == "no_compressor" else HapCompressorSnappy
    lib.set_option(lib.OPTION_CHROMA_REFINE, 1 if variant == "refine" else 0)
    try:
        n = lib.texture_bytes(w, h, codec, 0)
        cap = (lib.max_encoded_length_rgba(w, h, codec, chunks) + 15) // 16 * 16
        out = torch.zeros(frames * cap, dtype=torch.uint8, device="cuda")
        used = torch.zeros(frames, dtype=torch.int64, device="cuda")
        lib.set_stage_timing(True)
        lib.stage_times()
        assert lib.encode_rgba_batch(rgba.data_ptr(), frames, fstride, w, h, codec, compressor, chunks, out.data_ptr(), cap,
                                     used.data_ptr(), row_bytes=row) == 0
        launches = {k: v[1] for k, v in lib.stage_times().items()}
        lib.set_stage_timing(False)
        assert launches.get("snappy_encode", 0) == 1 and launches.get("bc_encode", 0) == 1, launches
        frame = out[: int(used[0])].cpu().numpy().tobytes()
        tstride = (lib.texture_bytes(w, h, codec, 0) + lib.texture_bytes(w, h, codec, 1) + 31) // 16 * 16
        tex = torch.zeros(frames * tstride, dtype=torch.uint8, device="cuda")
        assert lib.block_encode_batch(rgba.data_ptr(), frames, fstride, w, h, codec, tex.data_ptr(), tstride, row_bytes=row) == 0
        torch.cuda.synchronize()
        ref = oracles.ref_abi() or oracles.oracle_abi()
        r, t, _, _ = ref.decode(frame, 0, n)
        assert r == 0 and t == tex[:n].cpu().numpy().tobytes()
    finally:
        lib.set_option(lib.OPTION_CHROMA_REFINE, 0)
