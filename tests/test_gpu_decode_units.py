"""The execute kernel's unit path on the device (snappy_decode.cuh: fragments of an embedded index that are 8-byte granular
are decoded as 4096 units of 8 bytes).  Frames of this encoder decode to the reference's bytes with their index, without
it and with it damaged; a frame whose stream copies across a fragment boundary under a correct index (legal Snappy) is
handed to the repair pass and decodes to the reference's bytes through HapDecode and the batch decoder."""
import numpy as np
import pytest
import torch

import hap_b200
import oracles
from hap_b200 import synth
from hap_b200.abi import HapCompressorSnappy, HapTextureFormat_RGB_DXT1

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    lib = hap_b200.load()
    lib.set_option(lib.OPTION_WRITE_INDEX, 1)
    yield lib
    lib.set_option(lib.OPTION_WRITE_INDEX, 0)
    lib.set_option(lib.OPTION_USE_INDEX, 1)


def reference():
    return oracles.ref_abi() or oracles.oracle_abi()


def decode_batch(lib, frames, index, n, k):
    """texture `index` of each frame through HapB200DecodeBatch; returns (results, textures)"""
    F = len(frames)
    bcap = (max(len(f) for f in frames) + 63) // 64 * 64
    buf = torch.zeros(F * bcap, dtype=torch.uint8, device="cuda")
    for f, fr in enumerate(frames):
        buf[f * bcap: f * bcap + len(fr)] = torch.frombuffer(bytearray(fr), dtype=torch.uint8).cuda()
    lens = torch.tensor([len(fr) for fr in frames], dtype=torch.int64, device="cuda")
    stride = (n + 15) // 16 * 16
    tex = torch.zeros(F * stride, dtype=torch.uint8, device="cuda")
    used = torch.zeros(F, dtype=torch.int64, device="cuda")
    fmts = torch.zeros(F, dtype=torch.int32, device="cuda")
    res = torch.full((F,), 9, dtype=torch.int32, device="cuda")
    assert lib.decode_batch(buf.data_ptr(), F, bcap, lens.data_ptr(), index, k, tex.data_ptr(), stride, used.data_ptr(),
                            fmts.data_ptr(), res.data_ptr()) == 0
    assert used.tolist() == [n] * F
    host = tex.cpu().numpy()
    return res.tolist(), [host[f * stride: f * stride + n].tobytes() for f in range(F)]


def check_all_ways(lib, frame, damaged, ntex, texture_bytes, k):
    ref = reference()
    for i in range(ntex):
        n = texture_bytes(i)
        want = ref.decode(frame, i, n)
        assert want[0] == 0 and len(want[1]) == n
        assert lib.decode(frame, i, n)[:3] == want[:3]
        assert lib.decode(damaged, i, n)[:3] == want[:3]
        lib.set_option(lib.OPTION_USE_INDEX, 0)
        try:
            assert lib.decode(frame, i, n)[:3] == want[:3]
        finally:
            lib.set_option(lib.OPTION_USE_INDEX, 1)
        res, tex = decode_batch(lib, [frame, damaged, frame], i, n, k)
        assert res == [0, 0, 0] and tex == [want[1]] * 3


@pytest.mark.parametrize("w,h,codec_name,k", [(1920, 1080, "Hap1", 4), (3840, 2160, "HapY", 8), (1280, 720, "HapM", 3)])
def test_indexed_frames_match_the_reference(lib, w, h, codec_name, k):
    import hap_b200.lib as L
    codec = getattr(L, "HapB200Codec_" + codec_name)
    img = synth.frame(w, h, 5, alpha="ramp" if codec_name == "HapM" else "opaque", device="cuda")
    cap = (lib.max_encoded_length_rgba(w, h, codec, k) + 15) // 16 * 16
    out = torch.zeros(cap, dtype=torch.uint8, device="cuda")
    used = torch.zeros(1, dtype=torch.int64, device="cuda")
    assert lib.encode_rgba_batch(img.data_ptr(), 1, img.numel(), w, h, codec, 1, k, out.data_ptr(), cap, used.data_ptr()) == 0
    frame = out.cpu().numpy()[: int(used[0])].tobytes()
    proper = frame_proper_bytes(frame)
    assert frame[proper + 3] == 0xFB   # the index section follows the frame
    damaged = bytearray(frame)
    rng = np.random.default_rng(11)
    for _ in range(8):
        damaged[proper + 40 + int(rng.integers(0, len(frame) - proper - 40))] ^= 1 << int(rng.integers(0, 8))
    check_all_ways(lib, frame, bytes(damaged), 2 if codec_name == "HapM" else 1, lambda i: lib.texture_bytes(w, h, codec, i), k)


def section_header(b, at):
    size = b[at] | (b[at + 1] << 8) | (b[at + 2] << 16)
    if size == 0:
        return int.from_bytes(b[at + 4: at + 8], "little"), b[at + 3], 8
    return size, b[at + 3], 4


def frame_proper_bytes(frame):
    size, _, hdr = section_header(frame, 0)
    return hdr + size


def test_copy_across_fragments_goes_to_the_repair_pass(lib):
    """One Snappy chunk of three fragments; a copy of fragment 1 is re-pointed into fragment 0.  The index still describes
    every element exactly, so only the copy's reach tells that the fragment is not self-contained."""
    rng = np.random.default_rng(3)
    blocks = 3 * 4096
    data = np.zeros((blocks, 8), np.uint8)
    for b in range(blocks):
        data[b] = data[b - 1] if b and rng.random() < 0.5 else rng.integers(0, 256, 8, dtype=np.uint8)
    n = data.size
    r, frame = lib.encode([data.tobytes()], [HapTextureFormat_RGB_DXT1], [HapCompressorSnappy], [1])
    assert r == 0
    size, typ, hdr = section_header(frame, 0)
    assert typ in (0xBB, 0xCB), hex(typ)   # one Snappy chunk, with or without Decode Instructions
    stream = hdr
    if typ == 0xCB:
        di_size, di_typ, di_hdr = section_header(frame, hdr)
        assert di_typ == 0x01 and frame[hdr + di_hdr + 4] == 0x0B   # one chunk, Snappy
        stream = hdr + di_hdr + di_size
    # the stream's preamble, then the fragments' streams; their lengths are in the index record
    pre = 1
    while frame[stream + pre - 1] & 0x80:
        pre += 1
    isz, ityp, ihdr = section_header(frame, hdr + size)
    body = hdr + size + ihdr
    assert ityp == 0xFB and frame[body: body + 4] == b"HB2I"
    rec = body + int.from_bytes(frame[body + 20: body + 24], "little")
    s0, s1 = (int.from_bytes(frame[rec + 2 * f: rec + 2 * f + 2], "little") for f in range(2))
    p, end, o = stream + pre + s0, stream + pre + s0 + s1, 0
    patched = bytearray(frame)
    while p < end:
        tag = frame[p]
        kind = tag & 3
        if kind == 0:
            m, extra = tag >> 2, 0
            if m >= 60:
                extra = m - 59
                m = int.from_bytes(frame[p + 1: p + 1 + extra], "little")
            p += 1 + extra + m + 1
            o += m + 1
            continue
        length = 4 + ((tag >> 2) & 7) if kind == 1 else (tag >> 2) + 1
        if kind == 2 and o >= 8:
            off = o + 4096   # 4 KiB before the fragment's start
            patched[p + 1], patched[p + 2] = off & 0xFF, off >> 8
            break
        p += 2 if kind == 1 else 3 if kind == 2 else 5
        o += length
    assert p < end, "fragment 1 has no copy"
    patched = bytes(patched)
    want = reference().decode(patched, 0, n)
    assert want[0] == 0 and want[1] != data.tobytes()
    assert lib.decode(patched, 0, n)[:3] == want[:3]
    res, tex = decode_batch(lib, [patched, frame, patched], 0, n, 1)
    assert res == [0, 0, 0] and tex == [want[1], data.tobytes(), want[1]]
    lib.set_option(lib.OPTION_USE_INDEX, 0)
    try:
        assert lib.decode(patched, 0, n)[:3] == want[:3]
    finally:
        lib.set_option(lib.OPTION_USE_INDEX, 1)
