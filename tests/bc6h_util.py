"""Test-only BC6H (BPTC RGB UF16 / SF16, "Hap HDR") helpers: the bindings of the two CPU decoders -- the oracle
(tests/bc6h_oracle.c, written apart from the kernel) and the host build of the kernel's own block decoder
(tests/emu/bc6h_twin.cc) -- a block writer that lays fields out by the oracle's per-mode layout, random blocks of a chosen
mode, blocks whose every value lies in [0, 1], a small picture-like packer (mode 11), and Pillow's "bcn" decoder with
its 8-bit projection of the half values."""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")

NMODES = 14                                  # modes 0..13 here are the specification's modes 1..14
RESERVED = (0x13, 0x17, 0x1B, 0x1F)          # the four reserved 5-bit mode values
ONE = 0x3C00                                 # binary16 1.0 (A of every texel)


@functools.lru_cache(None)
def _so(name: str):
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "lib%s.so" % name)
    if name == "bc6h_oracle":
        cmd = ["gcc", "-std=c11", "-O2", "-Wall", "-fPIC", "-shared", os.path.join(ROOT, "tests", "bc6h_oracle.c"), "-o", so]
    else:
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
               "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "bc6h_twin.cc"), "-o", so]
    subprocess.run(cmd, check=True)
    return C.CDLL(so)


class Mode:
    """What the oracle says of one mode: mode bits and value, regions, transformed, precision, delta bits (R, G, B), and
    per header bit its endpoint component (-1: mode or partition bit) and component bit."""

    def __init__(self, m: int):
        info = (C.c_int * 8)()
        comp, bit = (C.c_int8 * 82)(), (C.c_int8 * 82)()
        self.header = _so("bc6h_oracle").bc6h_oracle_layout(m, info, comp, bit)
        self.mode_bits, self.mode_value, self.regions, self.transformed, self.prec = info[:5]
        self.delta = tuple(info[5:8])
        self.comp, self.bit = list(comp)[: self.header], list(bit)[: self.header]
        self.index_bits = 3 if self.regions == 2 else 4


@functools.lru_cache(None)
def mode(m: int) -> Mode:
    return Mode(m)


@functools.lru_cache(None)
def tables():
    """(partitions (32, 16) uint8, anchors (32,) uint8) of the oracle"""
    part, anchor = np.zeros((32, 16), np.uint8), np.zeros(32, np.uint8)
    _so("bc6h_oracle").bc6h_oracle_tables(C.c_void_p(part.ctypes.data), C.c_void_p(anchor.ctypes.data))
    return part, anchor


def random_blocks(rng, n: int, m: int) -> np.ndarray:
    """n random blocks of mode m (0..13), or of reserved mode value RESERVED[m - 14] -> (n, 16) uint8"""
    b = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    bits, value = (5, RESERVED[m - NMODES]) if m >= NMODES else (mode(m).mode_bits, mode(m).mode_value)
    b[:, 0] = (b[:, 0] & np.uint8((0xFF << bits) & 0xFF)) | np.uint8(value)
    return b


def pack_blocks(m: int, ep: np.ndarray, partition: np.ndarray, idx: np.ndarray) -> np.ndarray:
    """Blocks of mode m from raw field values: ep (n, 12) the stored endpoint components r0 g0 b0 r1 ... b3 (deltas as
    stored), partition (n,), idx (n, 16) texel indices (anchors must fit one bit less) -> (n, 16) uint8"""
    md = mode(m)
    n = len(ep)
    ep, idx, partition = np.asarray(ep, np.int64), np.asarray(idx, np.int64), np.asarray(partition, np.int64)
    bits = np.zeros((n, 128), np.uint8)
    for k in range(md.mode_bits):
        bits[:, k] = (md.mode_value >> k) & 1
    for p in range(md.mode_bits, md.header):
        if md.comp[p] >= 0:
            bits[:, p] = (ep[:, md.comp[p]] >> md.bit[p]) & 1
    if md.regions == 2:
        for k in range(5):
            bits[:, md.header - 5 + k] = (partition >> k) & 1
        second = tables()[1][partition]      # the anchor of subset 1 moves with the partition
    else:
        second = np.full(n, -1)
    rows, pos = np.arange(n), np.full(n, md.header)
    for t in range(16):
        nb = np.where((t == 0) | (second == t), md.index_bits - 1, md.index_bits)
        assert (idx[:, t] < (1 << nb)).all()
        for k in range(md.index_bits):
            live = k < nb
            bits[rows[live], pos[live] + k] = (idx[live, t] >> k) & 1
        pos += nb
    assert (pos == 128).all()
    return np.packbits(bits, axis=1, bitorder="little")


def unit_blocks(rng, n: int, m: int, signed: bool) -> np.ndarray:
    """n blocks of mode m whose every decoded value lies in [0, 1] (so Pillow's clamp to [0, 1] hides nothing): endpoints
    drawn below the largest value that decodes to at most 1.0, deltas that keep them there, random partitions and indices"""
    md = mode(m)
    lim = max(v for v in range(1 << min(md.prec, 16)) if _decoded(v, md.prec, signed) <= ONE and v < (1 << (md.prec - signed)))
    ne = 2 * md.regions
    ep = np.zeros((n, 12), np.int64)
    for c in range(3):
        base = rng.integers(0, lim + 1, n)
        ep[:, c] = base
        for e in range(1, ne):
            if md.transformed:
                d = md.delta[c]
                lo, hi = np.maximum(-base, -(1 << (d - 1))), np.minimum(lim - base, (1 << (d - 1)) - 1)
                dv = lo + (rng.random(n) * (hi - lo + 1)).astype(np.int64)
                ep[:, 3 * e + c] = dv & ((1 << d) - 1)
            else:
                ep[:, 3 * e + c] = rng.integers(0, lim + 1, n)
    partition = rng.integers(0, 32, n) if md.regions == 2 else np.zeros(n, np.int64)
    idx = rng.integers(0, 1 << md.index_bits, (n, 16))
    idx[:, 0] >>= 1
    if md.regions == 2:
        _, anchor = tables()
        rows = np.arange(n)
        idx[rows, anchor[partition]] >>= 1
    return pack_blocks(m, ep, partition, idx)


def _decoded(v: int, prec: int, signed: bool) -> int:
    """binary16 bits an endpoint value v >= 0 decodes to (unquantise, then the final scale)"""
    if not signed:
        q = v if prec >= 15 else 0 if v == 0 else 0xFFFF if v == (1 << prec) - 1 else ((v << 16) + 0x8000) >> prec
        return (q * 31) >> 6
    q = v if prec >= 16 else 0 if v == 0 else 0x7FFF if v >= (1 << (prec - 1)) - 1 else ((v << 15) + 0x4000) >> (prec - 1)
    return (q * 31) >> 5


def pack_picture(rgb: np.ndarray, signed: bool = False, peak: float = 4.0) -> bytes:
    """A picture (h, w, >= 3) uint8 -> mode-11 blocks (one region, 10-bit endpoints): the picture is taken as sRGB-like
    values, made linear and scaled to [0, peak]; the endpoints are each block's per-channel minimum and maximum in the
    10-bit code that decodes nearest, one 4-bit index per texel by its position between them.  Not an encoder of any
    quality: picture-like HDR content that the frame compressor can shrink."""
    h, w = rgb.shape[:2]
    lin = (rgb[..., :3].astype(np.float64) / 255.0) ** 2.2 * peak
    halfbits = lin.astype(np.float16).view(np.uint16).astype(np.int64)
    # mode 11 decodes code v to about v * 31 (UF16) or v * 62 (SF16, v < 512) binary16 units
    unit, top = (62.0, 511) if signed else (31.0, 1023)
    code = np.clip(np.rint(halfbits / unit), 0, top).astype(np.int64)
    blk = code.reshape(h // 4, 4, w // 4, 4, 3).transpose(0, 2, 1, 3, 4).reshape(-1, 16, 3)
    e0, e1 = blk.min(1), blk.max(1)
    span = np.maximum((e1 - e0).sum(1), 1)
    idx = np.clip(((blk - e0[:, None, :]).sum(2) * 15 + span[:, None] // 2) // span[:, None], 0, 15)
    flip = idx[:, 0] >= 8                                  # texel 0 stores 3 bits: swap the endpoints
    idx[flip] = 15 - idx[flip]
    e0[flip], e1[flip] = e1[flip].copy(), e0[flip].copy()
    ep = np.zeros((len(blk), 12), np.int64)
    ep[:, 0:3], ep[:, 3:6] = e0, e1
    return pack_blocks(10, ep, np.zeros(len(blk), np.int64), idx).tobytes()


# ---- the CPU decoders ------------------------------------------------------------------------------------------------------

def _decode(fn, blocks, w: int, h: int, signed: bool, *extra) -> np.ndarray:
    b = np.frombuffer(bytes(blocks), dtype=np.uint8)
    assert b.size == (w // 4) * (h // 4) * 16
    out = np.empty((h, w, 4), np.uint16)
    fn(C.c_void_p(b.ctypes.data), C.c_int(w), C.c_int(h), C.c_int(int(signed)), *[C.c_int(x) for x in extra],
       C.c_void_p(out.ctypes.data))
    return out


def oracle_decode(blocks, w: int, h: int, signed: bool, round: int = 32) -> np.ndarray:
    """The oracle's decoding (tests/bc6h_oracle.c) -> (h, w, 4) uint16 binary16 bits.  round: the interpolation's rounding
    term (32 as the specification says, 0 as Pillow does)"""
    return _decode(_so("bc6h_oracle").bc6h_oracle_decode, blocks, w, h, signed, round)


def twin_decode(blocks, w: int, h: int, signed: bool) -> np.ndarray:
    """The host build of the kernel's BC6H block decoder (bc6h_decode.cuh) -> (h, w, 4) uint16 binary16 bits"""
    return _decode(_so("bc6h_twin").bc6h_twin_decode, blocks, w, h, signed)


def twin_tables():
    """The partition maps (2 bits per texel) and anchor masks (bit t: texel t is an anchor) of partitions 0-31 as the
    kernel reads them"""
    part = np.empty(32, np.uint32)
    anchors = np.empty(32, np.uint32)
    _so("bc6h_twin").bc6h_twin_tables(C.c_void_p(part.ctypes.data), C.c_void_p(anchors.ctypes.data))
    return [int(x) for x in part], [int(x) for x in anchors]


# ---- Pillow as the independent judge ------------------------------------------------------------------------------------

def pil_decode(blocks, w: int, h: int, signed: bool) -> np.ndarray:
    """Pillow's BC6H decoding -> (h, w, 3) uint8"""
    from PIL import Image
    return np.asarray(Image.frombytes("RGB", (w, h), bytes(blocks), "bcn", (6, "BC6HS" if signed else "BC6H")))


def project8(half: np.ndarray) -> np.ndarray:
    """binary16 bits -> Pillow's 8-bit projection, uint8(clamp(value, 0, 1) * 255)"""
    v = np.asarray(half, np.uint16).view(np.float16).astype(np.float32)
    return (np.clip(v, 0.0, 1.0) * np.float32(255.0)).astype(np.uint8)
