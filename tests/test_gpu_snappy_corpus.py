"""The GPU Snappy decoder (snappy_decode.cuh) on the corpus of snappy_corpus.py: streams of every element form written element
by element, wrapped in Hap frames whose chunk outputs start at arbitrary bytes of the texture, decoded singly through HapDecode
(host and device buffers at every 16-byte misalignment) and in batches of a few hundred frames through HapB200DecodeBatch.
The judge of every frame is the reference (oracle/_ref: hap.c over Google Snappy; the CPU oracle where it is not built): the
texture bytes and the result code must be its own, and nothing may be written outside the texture."""
import random

import numpy as np
import pytest
import torch

import hap_b200
import oracles
import snappy_corpus as sc

pytestmark = pytest.mark.gpu

PAT = 0xA5          # fill of every output byte the decoder must not write
GUARD = 4096


@pytest.fixture(scope="module")
def lib():
    lib = hap_b200.load()
    yield lib
    lib.set_option(lib.OPTION_USE_INDEX, 1)
    lib.set_stage_timing(False)


_judged = {}


def judge(frame):
    """(result, texture bytes or None) of the reference; the texture's region for a frame it refuses is what the chunks
    declare"""
    if frame not in _judged:
        ref = oracles.ref_abi() or oracles.oracle_abi()
        region = texture_region(frame)
        r, tex, _, _ = ref.decode(frame, 0, max(region, 1))
        _judged[frame] = (r, tex, region)
    return _judged[frame]


def texture_region(frame):
    """bytes the frame's chunks declare (verbatim sizes and Snappy preambles), or its one section's size"""
    typ = frame[3]
    hdr = 8 if frame[:3] == b"\0\0\0" else 4
    size = int.from_bytes(frame[4:8], "little") if hdr == 8 else int.from_bytes(frame[:3], "little")
    body = frame[hdr: hdr + size]
    if typ >> 4 != 0xC:
        return sc.declared_size(typ >> 4, body)
    di_hdr = 8 if body[:3] == b"\0\0\0" else 4
    di_len = int.from_bytes(body[4:8], "little") if di_hdr == 8 else int.from_bytes(body[:3], "little")
    p, t = di_hdr, {}
    while p < di_hdr + di_len:
        h = 8 if body[p: p + 3] == b"\0\0\0" else 4
        n = int.from_bytes(body[p + 4: p + 8], "little") if h == 8 else int.from_bytes(body[p: p + 3], "little")
        t[body[p + 3]] = body[p + h: p + h + n]
        p += h + n
    comp = list(t[0x02])
    sizes = [int.from_bytes(t[0x03][4 * i: 4 * i + 4], "little") for i in range(len(comp))]
    offs = [int.from_bytes(t[0x04][4 * i: 4 * i + 4], "little") for i in range(len(comp))] if 0x04 in t else \
        [sum(sizes[:i]) for i in range(len(comp))]
    data = di_hdr + di_len
    return sum(sc.declared_size(c, body[data + o: data + o + s]) for c, o, s in zip(comp, offs, sizes))


def family_frames():
    """one frame per family: three chunks of it around a verbatim chunk of odd size, so the second Snappy chunk's output
    starts at an odd byte of the texture"""
    out = {}
    for i, fam in enumerate(sorted(sc.FAMILIES)):
        a = sc.pool_stream(fam, i, 40001)
        b = sc.write_stream(sc.FAMILIES[fam](100 + i, 70001 + 2 * i))
        out[fam] = sc.complex_frame([(sc.SNAPPY, a), (sc.RAW, bytes(range(37)) * 3), (sc.SNAPPY, b), (sc.SNAPPY, a)],
                                    offset_table=i % 2 == 1, long_headers=i % 3 == 0)
    return out


def check_single(lib, frame, decode_into):
    """decode_into(out address getter) -> (result, used); checks bytes, code and guards against the judge"""
    r_want, want, region = judge(frame)
    r, used, tex, front, back = decode_into(max(region, 1))
    assert r == r_want
    if r == 0:
        assert used == len(want) and tex == want
    assert front == bytes([PAT]) * GUARD and back == bytes([PAT]) * GUARD


def host_decode(lib, frame):
    def run(n):
        buf = np.full(n + 2 * GUARD, PAT, np.uint8)
        r, used, _, _ = lib.decode(frame, 0, n, out=(buf.ctypes.data + GUARD, n))
        return r, used, buf[GUARD: GUARD + n].tobytes(), buf[:GUARD].tobytes(), buf[GUARD + n:].tobytes()
    return run


def device_decode(lib, frame, fo, to):
    """the frame at byte fo of a device allocation, the texture at byte to (both 0-15 past a 256-byte boundary)"""
    def run(n):
        fbuf = torch.zeros(len(frame) + 512, dtype=torch.uint8, device="cuda")
        fbuf[256 + fo: 256 + fo + len(frame)] = torch.frombuffer(bytearray(frame), dtype=torch.uint8).cuda()
        out = torch.full((n + 2 * GUARD + 16,), PAT, dtype=torch.uint8, device="cuda")
        r, used, _, _ = lib.decode((fbuf.data_ptr() + 256 + fo, len(frame)), 0, n, out=(out.data_ptr() + GUARD + to, n))
        h = out.cpu().numpy()
        return r, used, h[GUARD + to: GUARD + to + n].tobytes(), h[to: GUARD + to].tobytes(), h[GUARD + to + n: 2 * GUARD + to + n].tobytes()
    return run


def test_single_frames_host(lib):
    """HapDecode, host frame to host texture with guard bytes: one frame per family, and frames around every illegal stream"""
    for fam, frame in family_frames().items():
        check_single(lib, frame, host_decode(lib, frame))
    good = sc.pool_stream("mixed", 5, 4097)
    for name, s in sc.illegal_streams().items():
        for frame in (sc.complex_frame([(sc.SNAPPY, good), (sc.SNAPPY, s)]), sc.simple_frame(sc.SNAPPY, s)):
            assert judge(frame)[0] != 0, name
            check_single(lib, frame, host_decode(lib, frame))


def test_single_frames_device_at_every_misalignment(lib):
    """HapDecode, device frame to device texture, the frame and the texture each at every offset 0-15: the TMA head/tail
    staging of the index and execute kernels and the byte-wise stores at the texture's edges"""
    frames = family_frames()
    for k, (fam, frame) in enumerate(frames.items()):
        for fo in range(16):
            check_single(lib, frame, device_decode(lib, frame, fo, (fo * 7 + k) % 16))


def stage_counts(lib):
    return {k: v[1] for k, v in lib.stage_times().items()}


def run_batch(lib, frames):
    """HapB200DecodeBatch over frames (bytes); checks every frame against the judge and every byte outside the textures
    against the fill.  Returns the stage launch counts of the call."""
    F = len(frames)
    in_stride = (max(len(f) for f in frames) + 63) // 64 * 64
    stride = (max(judge(f)[2] for f in frames) + 16 + 15) // 16 * 16      # at least 16 bytes of slack in every slot
    max_chunks = 8
    host_in = np.zeros(F * in_stride, np.uint8)
    for i, f in enumerate(frames):
        host_in[i * in_stride: i * in_stride + len(f)] = np.frombuffer(f, np.uint8)
    din = torch.from_numpy(host_in).cuda()
    lens = torch.tensor([len(f) for f in frames], dtype=torch.int64, device="cuda")
    out = torch.full((F * stride + 2 * GUARD,), PAT, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    fmts = torch.zeros(F, dtype=torch.int32, device="cuda")
    res = torch.full((F,), 99, dtype=torch.int32, device="cuda")
    lib.stage_times()
    assert lib.decode_batch(din.data_ptr(), F, in_stride, lens.data_ptr(), 0, max_chunks, out.data_ptr() + GUARD, stride,
                            used.data_ptr(), fmts.data_ptr(), res.data_ptr()) == 0
    counts = stage_counts(lib)
    h = out.cpu().numpy()
    res, used = res.tolist(), used.tolist()
    assert (h[:GUARD] == PAT).all() and (h[GUARD + F * stride:] == PAT).all()
    bad = []
    for i, f in enumerate(frames):
        r_want, want, region = judge(f)
        slot = h[GUARD + i * stride: GUARD + (i + 1) * stride]
        if res[i] != r_want:
            bad.append((i, "result", res[i], r_want))
            continue
        if r_want == 0:
            if used[i] != len(want) or slot[: len(want)].tobytes() != want:
                bad.append((i, "bytes", used[i], len(want)))
            if not (slot[len(want):] == PAT).all():
                bad.append((i, "slack written"))
        elif not (slot[min(region, stride):] == PAT).all():
            bad.append((i, "written outside the texture of a refused frame"))
    assert not bad, bad[:10]
    return counts


def indexed_twins():
    """[true-index frame, lying variant, true-index frame, lying variant, ...]"""
    ix = sc.indexed_frames()
    out = []
    for name, (frame, _) in sorted(ix.items()):
        if name != "true":
            out += [ix["true"][0], frame]
    return out


def batch_frames(seed):
    """a few hundred pool frames, the indexed frames next to their true-index twins, frames around every illegal stream
    between good neighbours"""
    frames = [f for f, _ in sc.random_frames(seed, 300, sc.pool(), max_chunks=8, max_texture=3 << 20)]
    frames += indexed_twins()
    good = sc.pool_stream("dense", 1, 40001)
    for s in sc.illegal_streams().values():
        frames += [sc.complex_frame([(sc.SNAPPY, good), (sc.SNAPPY, s), (sc.RAW, b"\x11" * 333)]), frames[len(frames) % 300]]
    return frames


@pytest.mark.parametrize("use_index", [1, 0])
@pytest.mark.parametrize("order", ["forward", "shuffled"])
def test_batch(lib, order, use_index):
    """a few hundred frames per call, far more chunks than there are resident CTAs, forward and in a seeded shuffled order,
    with the embedded indexes used and ignored.  Launch counts show the passes that ran: the on-the-fly index kernel runs in
    both cases, the unit kernel and the repair pass only with OPTION_USE_INDEX 1.  Whether the index kernel's CTAs found
    work cannot be told from the counters: it is launched over every chunk and returns at once for chunks that have an index."""
    frames = batch_frames(1)
    assert len(frames) >= 300
    if order == "shuffled":
        random.Random(7).shuffle(frames)
    lib.set_option(lib.OPTION_USE_INDEX, use_index)
    lib.set_stage_timing(True)
    try:
        counts = run_batch(lib, frames)
    finally:
        lib.set_stage_timing(False)
        lib.set_option(lib.OPTION_USE_INDEX, 1)
    # windows + index + execute, and with the index used: the unit kernel, and the repair pass (requeue, index, execute)
    assert counts["parse"] == 1 and counts["collect"] == 1
    if use_index:
        assert (counts["windows"], counts["snappy_index"], counts["snappy_decode"]) == (2, 2, 3), counts
    else:
        assert (counts["windows"], counts["snappy_index"], counts["snappy_decode"]) == (1, 1, 1), counts


def test_batch_with_a_chunk_of_16_mib(lib):
    """one chunk of more than 16 MiB (~50 windows of the on-the-fly index, each waiting for the ones its copies read) among a
    few dozen frames of the pool, forward and shuffled"""
    big = sc.pool(big=True)[-1][1]
    frames = [sc.complex_frame([(sc.RAW, b"\x5a" * 13), (sc.SNAPPY, big), (sc.SNAPPY, sc.pool_stream("far_copies", 17, 333333))])]
    frames += [f for f, _ in sc.random_frames(2, 40, sc.pool(), max_chunks=4, max_texture=1 << 20)]
    assert judge(frames[0])[2] > 16 << 20
    run_batch(lib, frames)
    random.Random(3).shuffle(frames)
    lib.set_option(lib.OPTION_USE_INDEX, 0)
    try:
        run_batch(lib, frames)
    finally:
        lib.set_option(lib.OPTION_USE_INDEX, 1)


LIES_ALWAYS_REPAIRED = ("entry_into_literal", "entered_piece_none", "repointed_copy")


def test_indexed_frames_single_and_batched(lib):
    """Byte-granular fragments under an embedded index (the execute kernel's general path with win.first == kNoDeps): the
    frame with the true index decodes without the repair pass; the lies that only the execute kernel can see (an entry moved
    into a literal, an entered piece marked empty, a copy that leaves its fragment) are caught there and repaired.  A moved
    boundary or swapped lengths may instead be refused before any window is listed (the record does not add up), in which
    case the chunk is indexed on the fly in the first pass: for those only the bytes are checked."""
    ix = sc.indexed_frames()
    for name, (frame, _) in sorted(ix.items()):
        lib.set_stage_timing(True)
        try:
            check_single(lib, frame, host_decode(lib, frame))
            counts = stage_counts(lib)
        finally:
            lib.set_stage_timing(False)
        if name == "true":
            assert (counts["windows"], counts["snappy_index"]) == (1, 1), counts
        elif name.split("/")[0] in LIES_ALWAYS_REPAIRED:
            assert (counts["windows"], counts["snappy_index"]) == (2, 2), (name, counts)
        lib.set_option(lib.OPTION_USE_INDEX, 0)
        try:
            check_single(lib, frame, host_decode(lib, frame))
        finally:
            lib.set_option(lib.OPTION_USE_INDEX, 1)
    run_batch(lib, indexed_twins())
