"""Test-only helpers for the HDR10 encoders (HapB200EncodeYUVPQ*): the conversion of include/hap_b200.h restated in numpy
integers (yuv_pq_to_rgba_half) with the transfer table evaluated by mpmath at 50 digits and rounded once to binary16
(pq_table), the coefficient rows read from the header, the 12-bit matrix in float64 (r12_float), HDR10 test pictures made
from linear BT.2020 light in cd/m2 (hdr10_planes), and the bindings of the library's own table and of the C++
pixel-by-pixel conversion (tests/emu/yuv_pq_twin.cc) that the emulated kernel test is built on."""
from __future__ import annotations

import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np

import yuv_util as Y

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")

BT2020_LIMITED, BT2020_FULL = 4, 5
COLOR_SPACES = (BT2020_LIMITED, BT2020_FULL)
KR, KB = 0.2627, 0.0593
UNITS = (1, 80, 100, 203, 1000, 10000)
ONE = 0x3C00                                          # binary16 1.0
M1, M2, C1, C2, C3 = 2610 / 16384, 2523 / 32, 3424 / 4096, 2413 / 128, 2392 / 128


@functools.lru_cache(None)
def coefficients() -> np.ndarray:
    """HAPB200_YUV_PQ_COEFFICIENTS of include/hap_b200.h: (2, 7) int64, row colour space - BT2020_LIMITED"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_PQ_COEFFICIENTS"):]
    body = body[: body.index("\n\n")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{\s*(-?\d+(?:\s*,\s*-?\d+){6})\s*\}", body)]
    assert len(rows) == 2
    return np.array(rows, np.int64)


def scales(cs):
    """(luma offset, luma scale, chroma scale, chroma offset) of the 10-bit range"""
    return (0, 1023, 1023, 512) if cs == BT2020_FULL else (64, 876, 896, 512)


def half_of(v) -> int:
    """A non-negative number (mpmath or float, below 65520) -> binary16 bits, rounded once, to nearest, ties to even"""
    import mpmath
    v = mpmath.mpf(v)
    if v <= 0:
        return 0
    e = max(int(mpmath.floor(mpmath.log(v, 2))), -14)
    if mpmath.mpf(2) ** e > v:                        # log's own rounding at a power of two
        e = max(e - 1, -14)
    elif mpmath.mpf(2) ** (e + 1) <= v:
        e += 1
    q = v * mpmath.mpf(2) ** (10 - e)
    n = int(mpmath.floor(q))
    d = q - n
    if d > 0.5 or (d == 0.5 and n % 2 == 1):
        n += 1
    return ((e + 15) << 10) + n - 1024


@functools.lru_cache(None)
def _eotf_nits():
    """10000 * EOTF(c / 4095) for c = 0 .. 4095, mpmath at 50 digits"""
    import mpmath
    mpmath.mp.dps = 50
    m1, m2 = mpmath.mpf(2610) / 16384, mpmath.mpf(2523) / 32
    c1, c2, c3 = mpmath.mpf(3424) / 4096, mpmath.mpf(2413) / 128, mpmath.mpf(2392) / 128
    out = []
    for c in range(4096):
        e = (mpmath.mpf(c) / 4095) ** (1 / m2)
        num = max(e - c1, mpmath.mpf(0))
        out.append(10000 * (num / (c2 - c3 * e)) ** (1 / m1))
    return out


@functools.lru_cache(None)
def pq_table(unit_nits: int) -> np.ndarray:
    """T of include/hap_b200.h: (4096,) uint16 binary16 bits of (10000 * EOTF(c / 4095)) / unitNits"""
    import mpmath
    mpmath.mp.dps = 50
    return np.array([half_of(v / unit_nits) for v in _eotf_nits()], np.uint16)


def pq_inverse(nits):
    """ST 2084 inverse EOTF, float64: luminance in cd/m2 -> signal 0 .. 1"""
    y = np.clip(np.asarray(nits, np.float64) / 10000.0, 0.0, 1.0) ** M1
    return ((C1 + C2 * y) / (1 + C3 * y)) ** M2


def r12(luma, chroma, cs):
    """The integer matrix of the definition: P010 planes -> (h, w, 3) int64 12-bit R'G'B', clamped to 0..4095"""
    yv = Y.samples(luma, Y.P010)
    h, w = yv.shape
    cb8, cr8 = Y.upsample8(chroma, w, h, Y.P010)
    cy, crr, cbg, crg, cbb, yoff, coff = (int(v) for v in coefficients()[cs - BT2020_LIMITED])
    yd, cb, cr = cy * (yv - yoff), cb8 - 8 * coff, cr8 - 8 * coff
    out = np.stack([(yd + crr * cr + 32768) >> 16, (yd + cbg * cb + crg * cr + 32768) >> 16, (yd + cbb * cb + 32768) >> 16], -1)
    return np.clip(out, 0, 4095)


def r12_float(luma, chroma, cs):
    """The same upsampling, then the BT.2020 matrix in float64, scaled to 0..4095 and unclamped: (h, w, 3) float64"""
    yv = Y.samples(luma, Y.P010).astype(np.float64)
    h, w = yv.shape
    cb8, cr8 = Y.upsample8(chroma, w, h, Y.P010)
    yoff, ys, csc, coff = scales(cs)
    kg = 1 - KR - KB
    ey = (yv - yoff) / ys
    pb = (cb8 / 8.0 - coff) / csc
    pr = (cr8 / 8.0 - coff) / csc
    r = ey + 2 * (1 - KR) * pr
    g = ey - 2 * KB * (1 - KB) / kg * pb - 2 * KR * (1 - KR) / kg * pr
    b = ey + 2 * (1 - KB) * pb
    return np.stack([r, g, b], -1) * 4095.0


def yuv_pq_to_rgba_half(luma, chroma, cs, unit_nits) -> np.ndarray:
    """The conversion of include/hap_b200.h: P010 luma (h, w) and chroma (h/2, w) words -> (h, w, 4) uint16 binary16 RGBA,
    A = 1.0"""
    rgb = r12(luma, chroma, cs)
    h, w = rgb.shape[:2]
    out = np.empty((h, w, 4), np.uint16)
    out[..., :3] = pq_table(unit_nits)[rgb]
    out[..., 3] = ONE
    return out


def planes_from_rgb_signal(rgb, cs, rng=None):
    """R'G'B' signal (h, w, 3) in 0..1 -> P010 (luma (h, w), chroma (h/2, w) interleaved) uint16 words; chroma is the mean of
    each 2 x 2 quad; rng: random junk in the low 6 bits"""
    rgb = np.asarray(rgb, np.float64)
    h, w = rgb.shape[:2]
    yoff, ys, csc, coff = scales(cs)
    ey = KR * rgb[..., 0] + (1 - KR - KB) * rgb[..., 1] + KB * rgb[..., 2]
    pb = (rgb[..., 2] - ey) / (2 * (1 - KB))
    pr = (rgb[..., 0] - ey) / (2 * (1 - KR))
    quad = lambda p: p.reshape(h // 2, 2, w // 2, 2).mean(axis=(1, 3))
    y = np.clip(np.rint(yoff + ys * ey), 0, 1023).astype(np.int64)
    cb = np.clip(np.rint(coff + csc * quad(pb)), 0, 1023).astype(np.int64)
    cr = np.clip(np.rint(coff + csc * quad(pr)), 0, 1023).astype(np.int64)
    chroma = np.stack([cb, cr], -1).reshape(h // 2, w)
    lo = (lambda s: rng.integers(0, 64, s, dtype=np.int64)) if rng is not None else (lambda s: 0)
    return ((y << 6) | lo(y.shape)).astype(np.uint16), ((chroma << 6) | lo(chroma.shape)).astype(np.uint16)


def hdr10_planes(kind, w, h, cs, index=0, lo=0.005, hi=4000.0, seed=0):
    """HDR10 test pictures: a synth.frame class made linear, (v / 255)^2.2, scaled to lo .. hi cd/m2 of BT.2020 light ->
    PQ inverse EOTF -> BT.2020 matrix -> quantised P010 planes with junk in the low 6 bits"""
    from hap_b200 import synth
    lin = (synth.frame(w, h, index, kind=kind).numpy()[..., :3].astype(np.float64) / 255.0) ** 2.2
    return planes_from_rgb_signal(pq_inverse(lo + (hi - lo) * lin), cs, np.random.default_rng(seed + 7 * index))


def random_planes(rng, w, h):
    """uniformly random 10-bit luma and chroma samples over the whole range, random junk in the low 6 bits"""
    return Y.random_planes(rng, w, h, Y.P010)


@functools.lru_cache(None)
def _twin():
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libyuv_pq_twin.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
                    "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "yuv_pq_twin.cc"), "-o", so], check=True)
    return C.CDLL(so)


def twin_table(unit_nits) -> np.ndarray:
    """the library's own table (yuv_pq_table of hap_b200/csrc/yuv_source.cuh, built on the host) -> (4096,) uint16"""
    out = np.zeros(4096, np.uint16)
    _twin().yuv_pq_twin_table(C.c_uint32(unit_nits), C.c_void_p(out.ctypes.data))
    return out


def twin_to_rgba_half(luma, chroma, cs, unit_nits, pitch=None) -> np.ndarray:
    """tests/emu/yuv_pq_twin.cc on the same planes (written with row pitch `pitch`, default: tight) -> (h, w, 4) uint16"""
    luma, chroma = np.asarray(luma), np.asarray(chroma)
    h, w = luma.shape
    pitch = pitch or 2 * w
    lb, cb = Y.pitched(luma, pitch), Y.pitched(chroma, pitch)
    out = np.zeros((h, w, 4), np.uint16)
    _twin().yuv_pq_twin_to_rgba_half(C.c_void_p(lb.ctypes.data), C.c_void_p(cb.ctypes.data), C.c_uint32(w), C.c_uint32(h),
                                     C.c_uint64(pitch), C.c_int(cs), C.c_uint32(unit_nits), C.c_void_p(out.ctypes.data))
    return out
