"""Test-only BC7 (BPTC RGBA UNORM) helpers: the mode table, a block writer that lays fields out in the order of the
format, random blocks of a chosen mode, a small picture-like packer (mode 6, per-channel min/max endpoints), the
partition / anchor probes that read those tables back from Pillow's independent "bcn" decoder, and the bindings of the
two CPU decoders: the oracle (tests/bc7_oracle.c, written apart from the kernel) and the host build of the kernel's own
block decoder (tests/emu/bc7_twin.cc)."""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")

# mode: (NS subsets, PB partition bits, RB rotation bits, ISB index-selection bits, CB colour bits, AB alpha bits,
#        EPB p-bit per endpoint, SPB p-bit per subset, IB index bits, IB2 secondary index bits)
MODES = [
    (3, 4, 0, 0, 4, 0, 1, 0, 3, 0),
    (2, 6, 0, 0, 6, 0, 0, 1, 3, 0),
    (3, 6, 0, 0, 5, 0, 0, 0, 2, 0),
    (2, 6, 0, 0, 7, 0, 1, 0, 2, 0),
    (1, 0, 2, 1, 5, 6, 0, 0, 2, 3),
    (1, 0, 2, 0, 7, 8, 0, 0, 2, 2),
    (1, 0, 0, 0, 7, 7, 1, 0, 4, 0),
    (2, 6, 0, 0, 5, 5, 1, 0, 2, 0),
]


class _Writer:
    def __init__(self):
        self.v, self.pos = 0, 0

    def put(self, value: int, n: int):
        assert 0 <= value < (1 << n) or n == 0 and value == 0, (value, n)
        self.v |= value << self.pos
        self.pos += n

    def bytes(self) -> bytes:
        assert self.pos == 128, self.pos
        return self.v.to_bytes(16, "little")


def pack_block(mode, partition=0, rotation=0, isb=0, colour=None, alpha=None, pbits=None, idx1=None, idx2=None,
               anchors=(0,)):
    """Lay out one block.  colour[c][e] (c = R, G, B; e = s0e0 s0e1 s1e0 ...), alpha[e], pbits[k], idx1/idx2[t]: raw field
    values; `anchors`: the texels whose primary index is stored with one bit less (the secondary set has texel 0 alone)."""
    ns, pb, rb, isbb, cb, ab, epb, spb, ib, ib2 = MODES[mode]
    assert len(set(anchors)) == ns and 0 in anchors
    ne = 2 * ns
    colour = colour if colour is not None else [[0] * ne for _ in range(3)]
    alpha = alpha if alpha is not None else [0] * ne
    npb = ne if epb else ns if spb else 0
    pbits = pbits if pbits is not None else [0] * npb
    idx1 = idx1 if idx1 is not None else [0] * 16
    idx2 = idx2 if idx2 is not None else [0] * 16
    w = _Writer()
    w.put(1 << mode, mode + 1)
    w.put(partition, pb)
    w.put(rotation, rb)
    w.put(isb, isbb)
    for c in range(3):
        for e in range(ne):
            w.put(colour[c][e], cb)
    if ab:
        for e in range(ne):
            w.put(alpha[e], ab)
    for k in range(npb):
        w.put(pbits[k], 1)
    for t in range(16):
        w.put(idx1[t], ib - (t in anchors))
    if ib2:
        for t in range(16):
            w.put(idx2[t], ib2 - (t == 0))
    return w.bytes()


def random_blocks(rng, n: int, mode: int) -> np.ndarray:
    """n random blocks whose byte 0 selects `mode` (mode 8: the reserved block, byte 0 = 0) -> (n, 16) uint8"""
    b = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    if mode == 8:
        b[:, 0] = 0
    else:
        b[:, 0] = (b[:, 0] & np.uint8((0xFF << (mode + 1)) & 0xFF)) | np.uint8(1 << mode)
    return b


def mode_of(blocks: np.ndarray) -> np.ndarray:
    """per block of (n, 16) uint8: its mode, 8 for reserved blocks"""
    b0 = blocks.reshape(-1, 16)[:, 0].astype(np.int64)
    m = np.full(b0.shape, 8)
    for k in range(7, -1, -1):
        m[(b0 >> k) & 1 == 1] = k
    return m


def pack_picture(rgba: np.ndarray) -> bytes:
    """A picture (h, w, 4) -> mode-6 blocks: endpoints the per-channel minimum and maximum of the block (7 bits + p-bit),
    one 4-bit index per texel by the texel's position between them.  Not an encoder of any quality: picture-like test
    content that the frame compressor can shrink."""
    h, w = rgba.shape[:2]
    blk = rgba.reshape(h // 4, 4, w // 4, 4, 4).transpose(0, 2, 1, 3, 4).reshape(-1, 16, 4).astype(np.int64)
    lo, hi = blk.min(1), blk.max(1)
    q0, q1 = lo >> 1, np.minimum((hi + 1) >> 1, 127)      # e0 = 2 q0 (p-bit 0), e1 = 2 q1 + 1 (p-bit 1)
    e0, e1 = 2 * q0, 2 * q1 + 1
    span = np.maximum((e1 - e0).sum(1), 1)
    idx = np.clip(((blk - e0[:, None, :]).sum(2) * 15 + span[:, None] // 2) // span[:, None], 0, 15)
    flip = idx[:, 0] >= 8                                  # texel 0 (the anchor) stores 3 bits: swap the endpoints
    idx[flip] = 15 - idx[flip]
    q0[flip], q1[flip] = q1[flip].copy(), q0[flip].copy()
    p0, p1 = np.where(flip, 1, 0), np.where(flip, 0, 1)
    v = np.zeros((len(blk), 2), np.uint64)                 # bits 0..63, 64..127

    def put(pos, n, val):
        val = val.astype(np.uint64)
        for half, shift in ((0, pos), (1, pos - 64)):
            if shift >= 64 or shift + n <= 0:
                continue
            v[:, half] |= (val << np.uint64(shift)) if shift >= 0 else (val >> np.uint64(-shift))

    put(0, 7, np.full(len(blk), 1 << 6))                   # mode bits
    pos = 7
    for c in range(4):
        put(pos, 7, q0[:, c])
        put(pos + 7, 7, q1[:, c])
        pos += 14
    put(pos, 1, p0)
    put(pos + 1, 1, p1)
    pos += 2
    for t in range(16):
        put(pos, 4 - (t == 0), idx[:, t])
        pos += 4 - (t == 0)
    assert pos == 128
    return v.astype("<u8").tobytes()


# ---- Pillow as the independent judge ------------------------------------------------------------------------------------

def pil_decode(blocks: bytes, w: int, h: int) -> np.ndarray:
    from PIL import Image
    return np.asarray(Image.frombytes("RGBA", (w, h), bytes(blocks), "bcn", (7,)))


def probe_partitions() -> tuple[list[int], list[list[int]]]:
    """The 64 two-subset and 64 three-subset partitions as Pillow decodes them: mode-1 blocks with black subset 0 and
    white subset 1 (every index 0) show the two-subset masks; mode-2 blocks with black, red and green subsets the others."""
    # (every index is 0, so where the anchors sit does not matter)
    two = [pack_block(1, p, colour=[[0, 0, 63, 63]] * 3, pbits=[0, 1], anchors=(0, 1)) for p in range(64)]
    three = [pack_block(2, p, colour=[[0, 0, 31, 31, 0, 0], [0, 0, 0, 0, 31, 31], [0] * 6], anchors=(0, 1, 2)) for p in range(64)]
    a = pil_decode(b"".join(two), 4 * 64, 4).reshape(4, 64, 4, 4).transpose(1, 0, 2, 3).reshape(64, 16, 4)
    b = pil_decode(b"".join(three), 4 * 64, 4).reshape(4, 64, 4, 4).transpose(1, 0, 2, 3).reshape(64, 16, 4)
    masks = [int(sum(1 << t for t in range(16) if a[p, t, 0] == 255)) for p in range(64)]
    maps = [[int(1 if b[p, t, 0] == 255 else 2 if b[p, t, 1] == 255 else 0) for t in range(16)] for p in range(64)]
    return masks, maps


def probe_anchors(masks, maps, seed=5) -> tuple[list[int], list[tuple[int, int]]]:
    """Anchor texels as Pillow reads them.  For every partition and every candidate anchor set, one block is written with
    that set; its indices make each texel's value tell its index (endpoints 0 and 255 in every subset).  Only the true set
    reproduces the intended index pattern.  Returns the two-subset anchors and the three-subset (subset 1, subset 2) pairs."""
    rng = np.random.default_rng(seed)
    two_sets = [(a,) for a in range(1, 16)]
    three_sets = [(a, b) for a in range(1, 16) for b in range(a + 1, 16)]

    def run(mode, sets):
        ns, _, _, _, cb, _, _, _, ib, _ = MODES[mode]
        top = (1 << cb) - 1
        colour = [[0, top] * ns for _ in range(3)]
        pbits = [0, 1] * ns if MODES[mode][6] else None      # mode 3: p-bits 0 and 1 make the endpoints 0 and 255
        found = []
        for p in range(64):
            blocks, want = [], []
            for s in sets:
                anchors = (0,) + s
                idx = [int(rng.integers(0, 1 << (ib - 1))) if t in anchors else int(rng.integers(1 << (ib - 1), 1 << ib))
                       for t in range(16)]
                blocks.append(pack_block(mode, p, colour=colour, pbits=pbits, idx1=idx, anchors=anchors))
                want.append(idx)
            px = pil_decode(b"".join(blocks), 4 * len(sets), 4).reshape(4, len(sets), 4, 4).transpose(1, 0, 2, 3)
            px = px.reshape(len(sets), 16, 4)[..., 0].astype(np.int64)
            # value of index i between 0 and 255: the weight table in 8-bit units
            wt = {2: [0, 21, 43, 64], 3: [0, 9, 18, 27, 37, 46, 55, 64]}[ib]
            table = [((64 - x) * 0 + x * 255 + 32) >> 6 for x in wt]
            hits = [s for k, s in enumerate(sets) if [table[i] for i in want[k]] == list(px[k])]
            assert len(hits) == 1, (mode, p, hits)
            found.append(hits[0])
        return found

    two = [s[0] for s in run(3, two_sets)]
    three = []
    for p, s in enumerate(run(2, three_sets)):
        a, b = s
        # the probe finds the set; the partition says which subset each anchor belongs to
        three.append((a, b) if maps[p][a] == 1 else (b, a))
    return two, three


# ---- the CPU decoders ------------------------------------------------------------------------------------------------------

@functools.lru_cache(None)
def _so(name: str):
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "lib%s.so" % name)
    if name == "bc7_oracle":
        cmd = ["gcc", "-std=c11", "-O2", "-Wall", "-fPIC", "-shared", os.path.join(ROOT, "tests", "bc7_oracle.c"), "-o", so]
    else:
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
               "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "bc7_twin.cc"), "-o", so]
    subprocess.run(cmd, check=True)
    return C.CDLL(so)


def _decode(fn, blocks, w: int, h: int) -> np.ndarray:
    b = np.frombuffer(bytes(blocks), dtype=np.uint8)
    assert b.size == (w // 4) * (h // 4) * 16
    out = np.empty((h, w, 4), np.uint8)
    fn(C.c_void_p(b.ctypes.data), C.c_int(w), C.c_int(h), C.c_void_p(out.ctypes.data))
    return out


def oracle_decode(blocks, w: int, h: int) -> np.ndarray:
    """The oracle's BC7 decoding (tests/bc7_oracle.c) -> (h, w, 4) uint8"""
    return _decode(_so("bc7_oracle").bc7_oracle_decode, blocks, w, h)


def twin_decode(blocks, w: int, h: int) -> np.ndarray:
    """The host build of the kernel's BC7 block decoder (bc7_decode.cuh) -> (h, w, 4) uint8"""
    return _decode(_so("bc7_twin").bc7_twin_decode, blocks, w, h)


def twin_tables():
    """The partition maps (2 bits per texel) and anchor masks (bit t: texel t is an anchor) the kernel compiles:
    ([64 two-subset maps], [64 three-subset maps], [64 two-subset masks], [64 three-subset masks])"""
    part = np.empty(128, np.uint32)
    anchors = np.empty(128, np.uint32)
    _so("bc7_twin").bc7_twin_tables(C.c_void_p(part.ctypes.data), C.c_void_p(anchors.ctypes.data))
    return [int(x) for x in part[:64]], [int(x) for x in part[64:]], [int(x) for x in anchors[:64]], [int(x) for x in anchors[64:]]
