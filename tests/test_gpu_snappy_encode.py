"""The GPU Snappy compressor (snappy_encode.cuh) and the frames around its streams, held byte for byte to the numpy model of
its rules (snappy_encode_model.py) on the corpus of snappy_encode_corpus.py: HapEncode on host buffers, HapB200EncodeBatch
over a few hundred mixed two-texture frames (forward and shuffled, fragment index and offset table off and on), Hap Q from
RGBA8 through both fused encoders, one BC7 and one BC6H encode.  A frame that differs is reported per fragment with the rule
step the device's stream first departs from.  The decoder must take every index the encoder writes without its repair pass."""
import random

import numpy as np
import pytest
import torch

import hap_b200
import oracles
import snappy_encode_corpus as ec
import snappy_encode_model as m
from hap_b200 import synth
from hap_b200.lib import HapB200Codec_HapY

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    L = hap_b200.load()
    yield L
    set_options(L, 0)
    L.set_stage_timing(False)


@pytest.fixture(scope="module")
def corpus():
    return ec.corpus()


CACHE = {}


def set_options(lib, options):
    lib.set_option(lib.OPTION_WRITE_INDEX, options & 1)
    lib.set_option(lib.OPTION_WRITE_OFFSET_TABLE, options >> 1)


def model(textures, options):
    return m.encode_frame(textures, index=bool(options & 1), offsets=bool(options & 2), cache=CACHE)


def assert_frames(named):
    """named: [(name, device frame, model FramePlan)]"""
    bad = [f"{name}: {m.explain_frame(plan, got)}" for name, got, plan in named if got != plan.frame]
    assert not bad, f"{len(bad)} of {len(named)} frames differ from the model:\n" + "\n".join(bad[:12])


def host_encode(lib, textures):
    lens = [len(t[0]) for t in textures]
    cap = lib.max_encoded_length(lens, [t[1] for t in textures], [t[3] for t in textures]) + 65536
    r, frame = lib.encode([t[0] for t in textures], [t[1] for t in textures], [t[2] for t in textures],
                          [t[3] for t in textures], out_capacity=cap)
    assert r == 0
    return frame


@pytest.mark.parametrize("options", [0, 1, 2, 3])
def test_hap_encode_host_buffers(lib, corpus, options):
    """every corpus texture through HapEncode, and two-texture frames (YCoCg + RGTC1) built from it"""
    set_options(lib, options)
    try:
        named = [(e.name, host_encode(lib, e.textures), model(e.textures, options)) for e in corpus]
        ycocg = [e.textures[0] for e in corpus if e.textures[0][1] == m.FMT_YCOCG and e.textures[0][2] == 1]
        rgtc = [e.textures[0] for e in corpus if e.textures[0][1] in (m.FMT_RGTC1, m.FMT_DXT1)]
        for k, (a, b) in enumerate(zip(ycocg, rgtc)):
            pair = [a, (b[0], m.FMT_RGTC1, 1, 1 + k % 3)]
            named.append((f"pair {k}", host_encode(lib, pair), model(pair, options)))
    finally:
        set_options(lib, 0)
    assert_frames(named)


# ---- batches ------------------------------------------------------------------------------------------------------------------

BATCH_FRAMES = 320
TEX0 = (5 * m.FRAG_BYTES + 8 * 258, m.FMT_YCOCG, 3)        # 3 chunks of a fragment and 1 451 units
TEX1 = (2 * m.FRAG_BYTES + 8 * 9, m.FMT_RGTC1, 2)


@pytest.fixture(scope="module")
def batch_textures(corpus):
    """BATCH_FRAMES frames of two textures each, cut from the corpus at random 16-byte offsets, with flat and noise frames"""
    rng = random.Random(11)
    pool = b"".join(t[0] for e in corpus for t in e.textures if len(t[0]) >= 4096)
    noise = np.random.default_rng(3).integers(0, 256, TEX0[0], dtype=np.uint8).tobytes()
    frames = []
    for f in range(BATCH_FRAMES):
        tex = []
        for n, fmt, chunks in (TEX0, TEX1):
            if f % 53 == 7:
                data = noise[:n]
            elif f % 41 == 3:
                data = bytes([f & 0xFF]) * n
            else:
                parts, size = [], 0
                while size < n:
                    at = rng.randrange(0, len(pool) - 4096) & ~15
                    k = min(rng.choice((1024, 4096, 40000)), len(pool) - at, n - size)
                    parts.append(pool[at: at + k])
                    size += k
                data = b"".join(parts)
            tex.append((data, fmt, 1, chunks))
        frames.append(tex)
    return frames


def encode_batch(lib, frames):
    """HapB200EncodeBatch over frames of the TEX0 + TEX1 geometry -> device frames (bytes)"""
    F = len(frames)
    strides = [(TEX0[0] + 255) // 256 * 256, (TEX1[0] + 255) // 256 * 256]
    host = [np.zeros(F * s, np.uint8) for s in strides]
    for f, tex in enumerate(frames):
        for i in range(2):
            host[i][f * strides[i]: f * strides[i] + len(tex[i][0])] = np.frombuffer(tex[i][0], np.uint8)
    dev = [torch.from_numpy(h).cuda() for h in host]
    cap = (lib.max_encoded_length([TEX0[0], TEX1[0]], [TEX0[1], TEX1[1]], [TEX0[2], TEX1[2]]) + 65536 + 15) // 16 * 16
    out = torch.zeros(F * cap, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    assert lib.encode_batch([d.data_ptr() for d in dev], strides, [TEX0[0], TEX1[0]], [TEX0[1], TEX1[1]], [1, 1],
                            [TEX0[2], TEX1[2]], F, out.data_ptr(), cap, used.data_ptr()) == 0
    torch.cuda.synchronize()
    o, u = out.cpu().numpy(), used.cpu().numpy()
    return [o[f * cap: f * cap + int(u[f])].tobytes() for f in range(F)]


@pytest.mark.parametrize("options", [0, 1, 2, 3])
@pytest.mark.parametrize("order", ["forward", "shuffled"])
def test_batch_of_mixed_frames(lib, batch_textures, order, options):
    """a few hundred two-texture frames (YCoCg in 3 chunks, RGTC1 in 2, short last fragments) in one call: ~2 500 fragments,
    far more than the resident CTAs; the same call twice gives the same bytes"""
    frames = list(batch_textures)
    if order == "shuffled":
        random.Random(5).shuffle(frames)
    set_options(lib, options)
    try:
        got = encode_batch(lib, frames)
        again = encode_batch(lib, frames) if order == "shuffled" else got
    finally:
        set_options(lib, 0)
    assert got == again
    assert_frames([(f"frame {f}", got[f], model(frames[f], options)) for f in range(len(frames))])


# ---- Hap Q from RGBA8 ---------------------------------------------------------------------------------------------------------

def hapq_pictures(w, h, frames, seed):
    """flat areas, repeated tiles, picture content and one band of noise (a chunk stored raw)"""
    rng = np.random.default_rng(seed)
    out = np.zeros((frames, h, w, 4), np.uint8)
    for f in range(frames):
        img = synth.frame(w, h, seed + f).numpy().copy()
        img[: h // 5] = (30 + f, 60, 90, 255)
        tile = img[h // 5: h // 5 + 32, :64].copy()
        for y in range(2 * h // 5, 3 * h // 5 - 31, 32):
            for x in range(0, w - 63, 64):
                img[y: y + 32, x: x + 64] = tile
        img[4 * h // 5:] = rng.integers(0, 256, size=(h - 4 * h // 5, w, 4), dtype=np.uint8)
        out[f] = img
    return out


@pytest.mark.parametrize("index,offsets", [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize("w,h,chunks", [(1000, 600, 5), (516, 260, 3), (1924, 1084, 8)])
def test_hapq_from_rgba(lib, w, h, chunks, index, offsets):
    """HapB200EncodeRGBABatch with Hap Q: the fused encoders (offset table off: hapq_ws_place_kernel, on:
    hapq_fused_encode_kernel) against the model applied to HapB200BlockEncodeBatch's textures"""
    frames = 3
    pics = hapq_pictures(w, h, frames, seed=w + chunks)
    rgba = torch.from_numpy(pics.reshape(-1)).cuda()
    fstride = h * w * 4
    n = lib.texture_bytes(w, h, HapB200Codec_HapY, 0)
    cap = (lib.max_encoded_length_rgba(w, h, HapB200Codec_HapY, chunks) + 15) // 16 * 16
    out = torch.zeros(frames * cap, dtype=torch.uint8, device="cuda")
    used = torch.zeros(frames, dtype=torch.int64, device="cuda")
    tstride = (n + 15) // 16 * 16
    tex = torch.zeros(frames * tstride, dtype=torch.uint8, device="cuda")
    set_options(lib, index | (offsets << 1))
    try:
        assert lib.encode_rgba_batch(rgba.data_ptr(), frames, fstride, w, h, HapB200Codec_HapY, 1, chunks, out.data_ptr(), cap,
                                     used.data_ptr()) == 0
    finally:
        set_options(lib, 0)
    assert lib.block_encode_batch(rgba.data_ptr(), frames, fstride, w, h, HapB200Codec_HapY, tex.data_ptr(), tstride) == 0
    torch.cuda.synchronize()
    o, u, t = out.cpu().numpy(), used.cpu().numpy(), tex.cpu().numpy()
    named = []
    for f in range(frames):
        textures = [(t[f * tstride: f * tstride + n].tobytes(), m.FMT_YCOCG, 1, chunks)]
        plan = model(textures, index | (offsets << 1))
        named.append((f"frame {f}", o[f * cap: f * cap + int(u[f])].tobytes(), plan))
    assert_frames(named)
    if chunks == 5:
        assert any(not cp.snappy for cp in named[0][2].sections[0].chunk_plans), "the noise band leaves a chunk raw"


# ---- BC7 and BC6H: period 2 on 16-byte blocks -----------------------------------------------------------------------------------

@pytest.mark.parametrize("options", [0, 1])
def test_bc7_encode(lib, options):
    w, h, chunks = 516, 260, 3
    pic = hapq_pictures(w, h, 1, seed=17)[0]
    n = (w // 4) * (h // 4) * 16
    dev = torch.from_numpy(pic.reshape(-1).copy()).cuda()
    blocks = torch.zeros((n + 15) // 16 * 16, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_bc7_batch(dev.data_ptr(), 1, 4 * w * h, w, h, blocks.data_ptr(), blocks.numel()) == 0
    torch.cuda.synchronize()
    set_options(lib, options)
    try:
        r, frame = lib.encode_rgba_bc7(pic.reshape(-1), w, h, 1, chunks)
    finally:
        set_options(lib, 0)
    assert r == 0
    textures = [(blocks.cpu().numpy()[:n].tobytes(), m.FMT_BC7, 1, chunks)]
    assert_frames([("bc7", frame, model(textures, options))])


@pytest.mark.parametrize("options", [0, 1])
def test_bc6h_encode(lib, options):
    w, h, chunks = 260, 132, 2
    pic = hapq_pictures(w, h, 1, seed=23)[0].astype(np.float32) / 64.0
    half = pic.astype(np.float16)
    half[..., 3] = 1.0
    n = (w // 4) * (h // 4) * 16
    dev = torch.from_numpy(half.view(np.uint8).reshape(-1).copy()).cuda()
    blocks = torch.zeros((n + 15) // 16 * 16, dtype=torch.uint8, device="cuda")
    assert lib.block_encode_half_batch(dev.data_ptr(), 1, 8 * w * h, w, h, m.FMT_BC6U, blocks.data_ptr(), blocks.numel()) == 0
    torch.cuda.synchronize()
    set_options(lib, options)
    try:
        r, frame = lib.encode_rgba_half(half.view(np.uint8).reshape(-1), w, h, m.FMT_BC6U, 1, chunks)
    finally:
        set_options(lib, 0)
    assert r == 0
    textures = [(blocks.cpu().numpy()[:n].tobytes(), m.FMT_BC6U, 1, chunks)]
    assert_frames([("bc6h", frame, model(textures, options))])


# ---- the decoder takes the encoder's indexes ------------------------------------------------------------------------------------

def test_decoder_takes_every_index_the_encoder_writes(lib, corpus):
    """a single HapDecode of each indexed corpus frame the GPU wrote runs the windows and index passes once (no repair pass)
    and gives the texture back"""
    set_options(lib, 1)
    try:
        frames = [(e, host_encode(lib, e.textures)) for e in corpus]
    finally:
        set_options(lib, 0)
    checked = 0
    for e, frame in frames:
        plan = model(e.textures, 1)
        assert frame == plan.frame, f"{e.name}: {m.explain_frame(plan, frame)}"
        if not any(cp.entries_at for s in plan.sections for cp in s.chunk_plans):
            continue
        s = plan.sections[0]
        want = e.textures[0][0][: s.chunks * s.chunk_bytes]
        lib.set_stage_timing(True)
        try:
            lib.stage_times()
            r, tex, fmt, _ = lib.decode(frame, 0, len(e.textures[0][0]))
            counts = {k: v[1] for k, v in lib.stage_times().items()}
        finally:
            lib.set_stage_timing(False)
        assert r == 0 and fmt == e.textures[0][1] and tex == want, e.name
        assert (counts["windows"], counts["snappy_index"]) == (1, 1), (e.name, counts)
        checked += 1
    assert checked >= 20
    ref = oracles.ref_abi() or oracles.oracle_abi()
    for e, frame in frames[:: 7]:
        r, tex, _, _ = ref.decode(frame, 0, len(e.textures[0][0]))
        assert r == 0
