"""Test-only helpers for the NV12 / P010 encoders: the conversion of include/hap_b200.h restated in numpy integers
(yuv_to_rgba), the same upsampling with the real matrix in float64 (yuv_to_rgb_float), the coefficient table read from the
header, test pictures made from RGBA content (rgba_to_yuv), pitched plane buffers, and the binding of the C++ pixel-by-pixel
conversion (tests/emu/yuv_twin.cc) that the emulated kernel test is built on."""
from __future__ import annotations

import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")

NV12, P010 = 0, 1
BT601_LIMITED, BT601_FULL, BT709_LIMITED, BT709_FULL = range(4)
LAYOUTS = (NV12, P010)
COLOR_SPACES = (BT601_LIMITED, BT601_FULL, BT709_LIMITED, BT709_FULL)
KRKB = {BT601_LIMITED: (0.299, 0.114), BT601_FULL: (0.299, 0.114), BT709_LIMITED: (0.2126, 0.0722), BT709_FULL: (0.2126, 0.0722)}


def bits(layout) -> int:
    return 10 if layout == P010 else 8


def sample_bytes(layout) -> int:
    return 2 if layout == P010 else 1


def is_full(cs) -> bool:
    return cs in (BT601_FULL, BT709_FULL)


@functools.lru_cache(None)
def coefficients() -> np.ndarray:
    """HAPB200_YUV_COEFFICIENTS of include/hap_b200.h: (8, 7) int64, row layout * 4 + colour space"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_COEFFICIENTS"):]
    body = body[: body.index("\n\n")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{\s*(-?\d+(?:\s*,\s*-?\d+){6})\s*\}", body)]
    assert len(rows) == 8
    return np.array(rows, np.int64)


def scales(layout, cs):
    """(luma offset, luma scale, chroma scale, chroma offset) of the definition"""
    n = bits(layout)
    s = 1 << (n - 8)
    if is_full(cs):
        return 0, (1 << n) - 1, (1 << n) - 1, 1 << (n - 1)
    return 16 * s, 219 * s, 224 * s, 1 << (n - 1)


def samples(plane, layout) -> np.ndarray:
    """NV12 bytes as they are; P010 16-bit words >> 6 (the low 6 bits are ignored)"""
    p = np.asarray(plane)
    return (p.astype(np.int64) >> 6) if layout == P010 else p.astype(np.int64)


def upsample8(chroma, w, h, layout):
    """chroma (h/2, w) interleaved Cb, Cr samples -> (Cb8, Cr8): (h, w) int64 in eighths, bilinear at the default siting,
    indices clamped to the plane"""
    c = samples(chroma, layout).reshape(h // 2, w // 2, 2)
    x, y = np.arange(w), np.arange(h)
    i, j = x // 2, y // 2
    rn = np.clip(np.where(y % 2 == 1, j + 1, j - 1), 0, h // 2 - 1)
    cn = np.clip(i + 1, 0, w // 2 - 1)
    wh0 = np.where(x % 2 == 1, 1, 2)
    wh1 = np.where(x % 2 == 1, 1, 0)
    v = 3 * c[j] + c[rn]                                         # (h, w/2, 2): vertical, in quarters
    out = wh0[None, :, None] * v[:, i] + wh1[None, :, None] * v[:, cn]
    return out[..., 0], out[..., 1]


def yuv_to_rgba(luma, chroma, layout, cs) -> np.ndarray:
    """The conversion of include/hap_b200.h in integers: luma (h, w) and chroma (h/2, w) interleaved, uint8 (NV12) or uint16
    words (P010) -> (h, w, 4) uint8 RGBA with A = 255"""
    yv = samples(luma, layout)
    h, w = yv.shape
    cb8, cr8 = upsample8(chroma, w, h, layout)
    cy, crr, cbg, crg, cbb, yoff, coff = (int(v) for v in coefficients()[layout * 4 + cs])
    yd, cb, cr = cy * (yv - yoff), cb8 - 8 * coff, cr8 - 8 * coff
    out = np.empty((h, w, 4), np.uint8)
    out[..., 0] = np.clip((yd + crr * cr + 32768) >> 16, 0, 255)
    out[..., 1] = np.clip((yd + cbg * cb + crg * cr + 32768) >> 16, 0, 255)
    out[..., 2] = np.clip((yd + cbb * cb + 32768) >> 16, 0, 255)
    out[..., 3] = 255
    return out


def yuv_to_rgb_float(luma, chroma, layout, cs) -> np.ndarray:
    """The same upsampling, then the real (Kr, Kb) matrix in float64, scaled to 0..255 and clamped: (h, w, 3) float64"""
    yv = samples(luma, layout).astype(np.float64)
    h, w = yv.shape
    cb8, cr8 = upsample8(chroma, w, h, layout)
    yoff, ys, cs_, coff = scales(layout, cs)
    kr, kb = KRKB[cs]
    kg = 1 - kr - kb
    ey = (yv - yoff) / ys
    pb = (cb8 / 8.0 - coff) / cs_
    pr = (cr8 / 8.0 - coff) / cs_
    r = ey + 2 * (1 - kr) * pr
    g = ey - 2 * kb * (1 - kb) / kg * pb - 2 * kr * (1 - kr) / kg * pr
    b = ey + 2 * (1 - kb) * pb
    return np.clip(np.stack([r, g, b], -1) * 255.0, 0.0, 255.0)


def rgba_to_yuv(rgba, layout, cs):
    """Test pictures: RGBA8 (h, w, 4) -> (luma (h, w), chroma (h/2, w) interleaved), uint8 or uint16 P010 words; chroma is
    the mean of each 2 x 2 quad (any 4:2:0 picture will do: the encoders are held to the conversion, not to this)"""
    rgb = np.asarray(rgba)[..., :3].astype(np.float64) / 255.0
    h, w = rgb.shape[:2]
    kr, kb = KRKB[cs]
    yoff, ys, cs_, coff = scales(layout, cs)
    ey = kr * rgb[..., 0] + (1 - kr - kb) * rgb[..., 1] + kb * rgb[..., 2]
    pb = (rgb[..., 2] - ey) / (2 * (1 - kb))
    pr = (rgb[..., 0] - ey) / (2 * (1 - kr))
    top = (1 << bits(layout)) - 1
    y = np.clip(np.rint(yoff + ys * ey), 0, top).astype(np.int64)
    quad = lambda p: p.reshape(h // 2, 2, w // 2, 2).mean(axis=(1, 3))
    cb = np.clip(np.rint(coff + cs_ * quad(pb)), 0, top).astype(np.int64)
    cr = np.clip(np.rint(coff + cs_ * quad(pr)), 0, top).astype(np.int64)
    chroma = np.stack([cb, cr], -1).reshape(h // 2, w)
    if layout == P010:
        return (y << 6).astype(np.uint16), (chroma << 6).astype(np.uint16)
    return y.astype(np.uint8), chroma.astype(np.uint8)


def pitched(plane, pitch, fill=0xA5) -> np.ndarray:
    """plane (rows, n) uint8 / uint16 -> (rows, pitch) uint8 bytes, the padding of every row set to `fill`"""
    b = np.ascontiguousarray(plane).view(np.uint8).reshape(plane.shape[0], -1)
    out = np.full((plane.shape[0], pitch), fill, np.uint8)
    out[:, : b.shape[1]] = b
    return out


@functools.lru_cache(None)
def _twin():
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libyuv_twin.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
                    "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "yuv_twin.cc"), "-o", so], check=True)
    return C.CDLL(so)


def twin_to_rgba(luma, chroma, layout, cs, pitch=None) -> np.ndarray:
    """tests/emu/yuv_twin.cc on the same planes (written with row pitch `pitch`, default: tight) -> (h, w, 4) uint8"""
    luma, chroma = np.asarray(luma), np.asarray(chroma)
    h, w = luma.shape
    pitch = pitch or w * sample_bytes(layout)
    lb, cb = pitched(luma, pitch), pitched(chroma, pitch)
    out = np.zeros((h, w, 4), np.uint8)
    _twin().yuv_twin_to_rgba(C.c_void_p(lb.ctypes.data), C.c_void_p(cb.ctypes.data), C.c_uint32(w), C.c_uint32(h), C.c_uint64(pitch),
                             C.c_int(layout), C.c_int(cs), C.c_void_p(out.ctypes.data))
    return out


def random_planes(rng, w, h, layout, junk_low_bits=True):
    """uniformly random luma and chroma samples over the whole sample range (P010: random junk in the low 6 bits)"""
    top = 1 << bits(layout)
    y = rng.integers(0, top, (h, w), dtype=np.int64)
    c = rng.integers(0, top, (h // 2, w), dtype=np.int64)
    if layout == P010:
        lo = (lambda s: rng.integers(0, 64, s, dtype=np.int64)) if junk_low_bits else (lambda s: 0)
        return ((y << 6) | lo(y.shape)).astype(np.uint16), ((c << 6) | lo(c.shape)).astype(np.uint16)
    return y.astype(np.uint8), c.astype(np.uint8)
