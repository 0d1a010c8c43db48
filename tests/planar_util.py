"""Test-only helpers for the planar Y'CbCr encoders (HapB200EncodePlanar*): the conversion of include/hap_b200.h restated in
numpy integers (planar_to_rgba), the same upsampling with the real matrix in float64 (planar_to_rgb_float), the 12-bit
coefficient table read from the header, test pictures made from RGBA content (rgba_to_planar), random planes, and the
binding of the C++ pixel-by-pixel conversion (tests/emu/planar_twin.cc) that the emulated kernel test is built on.  The 8-
and 10-bit matrix rows and the 4:2:0 upsampler are yuv_util's."""
from __future__ import annotations

import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np

import yuv_util as Y

ROOT = Y.ROOT
BUILD = Y.BUILD

S420, S422, S444 = 0, 1, 2
SUBSAMPLINGS = (S420, S422, S444)
DEPTHS = (8, 10, 12)
COLOR_SPACES = Y.COLOR_SPACES


def sample_bytes(n) -> int:
    return 1 if n == 8 else 2


def chroma_shape(w, h, sub):
    """(rows, samples per row) of the Cb and Cr planes"""
    return (h // 2 if sub == S420 else h), (w if sub == S444 else w // 2)


@functools.lru_cache(None)
def coefficients12() -> np.ndarray:
    """HAPB200_YUV_12BIT_COEFFICIENTS of include/hap_b200.h: (4, 7) int64, row colour space"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_12BIT_COEFFICIENTS"):]
    body = body[: body.index("\n\n")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{\s*(-?\d+(?:\s*,\s*-?\d+){6})\s*\}", body)]
    assert len(rows) == 4
    return np.array(rows, np.int64)


def matrix(n, cs):
    """({cy, crR, cbG, crG, cbB, yOff, cOff}, shift) of depth n and colour space cs"""
    if n == 12:
        return [int(v) for v in coefficients12()[cs]], 18
    return [int(v) for v in Y.coefficients()[(Y.P010 if n == 10 else Y.NV12) * 4 + cs]], 16


def scales(n, cs):
    """(luma offset, luma scale, chroma scale, chroma offset) of the definition at depth n"""
    s = 1 << (n - 8)
    if Y.is_full(cs):
        return 0, (1 << n) - 1, (1 << n) - 1, 1 << (n - 1)
    return 16 * s, 219 * s, 224 * s, 1 << (n - 1)


def samples(plane, n) -> np.ndarray:
    """bytes as they are; 16-bit words & (2^n - 1) (higher bits are ignored)"""
    p = np.asarray(plane).astype(np.int64)
    return p if n == 8 else p & ((1 << n) - 1)


def upsample8(cb, cr, w, h, sub):
    """Cb and Cr sample planes (int64) -> (Cb8, Cr8): (h, w) in eighths, as the definition states for each subsampling"""
    if sub == S420:
        return Y.upsample8(np.stack([cb, cr], -1).reshape(h // 2, w), w, h, Y.NV12)
    if sub == S444:
        return 8 * cb, 8 * cr
    x = np.arange(w)
    i, cn = x // 2, np.clip(x // 2 + 1, 0, w // 2 - 1)
    wh0, wh1 = np.where(x % 2 == 1, 1, 2), np.where(x % 2 == 1, 1, 0)
    up = lambda c: 4 * (wh0[None, :] * c[:, i] + wh1[None, :] * c[:, cn])
    return up(cb), up(cr)


def alpha8(a, n) -> np.ndarray:
    """A = (510 a + 2^n - 1) / (2 (2^n - 1)), integer division"""
    m = (1 << n) - 1
    return (510 * np.asarray(a, np.int64) + m) // (2 * m)


def planar_to_rgba(luma, cb, cr, alpha, sub, n, cs) -> np.ndarray:
    """The conversion of include/hap_b200.h in integers: luma (h, w), cb and cr (chroma_shape), alpha (h, w) or None, uint8
    (n = 8) or uint16 words -> (h, w, 4) uint8 RGBA (A = 255 without alpha)"""
    yv = samples(luma, n)
    h, w = yv.shape
    cb8, cr8 = upsample8(samples(cb, n), samples(cr, n), w, h, sub)
    (cy, crr, cbg, crg, cbb, yoff, coff), shift = matrix(n, cs)
    half = 1 << (shift - 1)
    yd, b_, r_ = cy * (yv - yoff), cb8 - 8 * coff, cr8 - 8 * coff
    out = np.empty((h, w, 4), np.uint8)
    out[..., 0] = np.clip((yd + crr * r_ + half) >> shift, 0, 255)
    out[..., 1] = np.clip((yd + cbg * b_ + crg * r_ + half) >> shift, 0, 255)
    out[..., 2] = np.clip((yd + cbb * b_ + half) >> shift, 0, 255)
    out[..., 3] = 255 if alpha is None else alpha8(samples(alpha, n), n)
    return out


def planar_to_rgb_float(luma, cb, cr, sub, n, cs) -> np.ndarray:
    """The same upsampling, then the real (Kr, Kb) matrix in float64, scaled to 0..255 and clamped: (h, w, 3) float64"""
    yv = samples(luma, n).astype(np.float64)
    h, w = yv.shape
    cb8, cr8 = upsample8(samples(cb, n), samples(cr, n), w, h, sub)
    yoff, ys, csc, coff = scales(n, cs)
    kr, kb = Y.KRKB[cs]
    kg = 1 - kr - kb
    ey = (yv - yoff) / ys
    pb = (cb8 / 8.0 - coff) / csc
    pr = (cr8 / 8.0 - coff) / csc
    r = ey + 2 * (1 - kr) * pr
    g = ey - 2 * kb * (1 - kb) / kg * pb - 2 * kr * (1 - kr) / kg * pr
    b = ey + 2 * (1 - kb) * pb
    return np.clip(np.stack([r, g, b], -1) * 255.0, 0.0, 255.0)


def as_plane(s, n, junk=None) -> np.ndarray:
    """int64 samples -> uint8 (n = 8) or uint16 words, with `junk` (int64 of the same shape) in the bits above n"""
    if n == 8:
        return s.astype(np.uint8)
    return (s | ((junk << n) & 0xFFFF if junk is not None else 0)).astype(np.uint16)


def random_planes(rng, w, h, sub, n, alpha=True, junk_high_bits=True):
    """uniformly random samples over the whole range of depth n: (luma, cb, cr, alpha or None); 16-bit words carry random
    junk above the sample"""
    top = 1 << n
    ch, cw = chroma_shape(w, h, sub)
    junk = (lambda s: rng.integers(0, 1 << 16, s, dtype=np.int64)) if junk_high_bits and n > 8 else (lambda s: None)
    plane = lambda s: as_plane(rng.integers(0, top, s, dtype=np.int64), n, junk(s))
    return plane((h, w)), plane((ch, cw)), plane((ch, cw)), (plane((h, w)) if alpha else None)


def rgba_to_planar(rgba, sub, n, cs, alpha=True):
    """Test pictures: RGBA8 (h, w, 4) -> (luma, cb, cr, alpha or None) at depth n; chroma is the mean over each chroma
    sample's luma footprint (any picture will do: the encoders are held to the conversion, not to this)"""
    rgba = np.asarray(rgba)
    rgb = rgba[..., :3].astype(np.float64) / 255.0
    h, w = rgb.shape[:2]
    kr, kb = Y.KRKB[cs]
    yoff, ys, csc, coff = scales(n, cs)
    ey = kr * rgb[..., 0] + (1 - kr - kb) * rgb[..., 1] + kb * rgb[..., 2]
    pb = (rgb[..., 2] - ey) / (2 * (1 - kb))
    pr = (rgb[..., 0] - ey) / (2 * (1 - kr))
    top = (1 << n) - 1
    fy, fx = (2 if sub == S420 else 1), (1 if sub == S444 else 2)
    foot = lambda p: p.reshape(h // fy, fy, w // fx, fx).mean(axis=(1, 3))
    q = lambda v: np.clip(np.rint(v), 0, top).astype(np.int64)
    a = q(rgba[..., 3].astype(np.float64) * top / 255.0) if alpha else None
    return (as_plane(q(yoff + ys * ey), n), as_plane(q(coff + csc * foot(pb)), n), as_plane(q(coff + csc * foot(pr)), n),
            None if a is None else as_plane(a, n))


@functools.lru_cache(None)
def _twin():
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libplanar_twin.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
                    "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "planar_twin.cc"), "-o", so],
                   check=True)
    return C.CDLL(so)


def twin_to_rgba(luma, cb, cr, alpha, sub, n, cs, luma_pad=0, chroma_pad=0) -> np.ndarray:
    """tests/emu/planar_twin.cc on the same planes (rows padded by luma_pad / chroma_pad bytes) -> (h, w, 4) uint8"""
    luma, cb, cr = np.asarray(luma), np.asarray(cb), np.asarray(cr)
    h, w = luma.shape
    lp, cp = w * sample_bytes(n) + luma_pad, cb.shape[1] * sample_bytes(n) + chroma_pad
    planes = [Y.pitched(luma, lp), Y.pitched(cb, cp), Y.pitched(cr, cp), None if alpha is None else Y.pitched(np.asarray(alpha), lp)]
    ptr = lambda b: C.c_void_p(None if b is None else b.ctypes.data)
    out = np.zeros((h, w, 4), np.uint8)
    _twin().planar_twin_to_rgba(*[ptr(b) for b in planes], C.c_uint32(w), C.c_uint32(h), C.c_uint64(lp), C.c_uint64(cp), C.c_int(sub),
                                C.c_int(n), C.c_int(cs), C.c_void_p(out.ctypes.data))
    return out


def kernel_alpha(a, n) -> int:
    """the kernel's alpha mapping (planar_alpha16, yuv_source.cuh) of one 10- or 12-bit sample"""
    return int(_twin().planar_twin_kernel_alpha(C.c_uint32(a), C.c_int(n)))
