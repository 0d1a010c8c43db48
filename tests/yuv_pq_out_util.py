"""Test-only helpers for the HDR10 decoders (HapB200DecodeYUVPQ*): the RGBA16F -> P010 conversion of include/hap_b200.h
restated in numpy integers (rgba_half_to_yuv_pq) with the transfer table P evaluated by mpmath at 50 digits (pq_out_table),
the coefficient rows read from the header and recomputed from their rule, the same filter with the real BT.2020 matrix in
float64, and the bindings of the library's own table and of the C++ sample-by-sample conversion
(tests/emu/yuv_pq_out_twin.cc) that the emulated kernel test is built on."""
from __future__ import annotations

import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np

import yuv_out_util as O
import yuv_pq_util as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
ENTRIES = 0x7C00                                      # the non-negative finite binary16 values


@functools.lru_cache(None)
def coefficients() -> np.ndarray:
    """HAPB200_YUV_PQ_OUT_COEFFICIENTS of include/hap_b200.h: (2, 11) int64, row colour space - BT2020_LIMITED"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_PQ_OUT_COEFFICIENTS"):]
    body = body[: body.index("\n\n")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{\s*(-?\d+(?:\s*,\s*-?\d+){10})\s*\}", body)]
    assert len(rows) == 2
    return np.array(rows, np.int64)


def row(cs) -> list:
    return [int(v) for v in coefficients()[cs - P.BT2020_LIMITED]]


def rule_coefficients(cs) -> list:
    """{yR, yG, yB, cbR, cbG, cbB, crR, crG, crB, yOff, cOff} from the rule the header states (that of
    HAPB200_YUV_OUT_COEFFICIENTS with 4095 for 255)"""
    rnd = lambda v: int(np.floor(v + 0.5))
    yoff, ys, csc, coff = P.scales(cs)
    kg = 1 - P.KR - P.KB
    lum, s = 65536 * ys / 4095, 65536 * csc / 4095
    yr, yb = rnd(lum * P.KR), rnd(lum * P.KB)
    cbr, cbg = rnd(-s * P.KR / (2 * (1 - P.KB))), rnd(-s * kg / (2 * (1 - P.KB)))
    crg, crb = rnd(-s * kg / (2 * (1 - P.KR))), rnd(-s * P.KB / (2 * (1 - P.KR)))
    return [yr, rnd(lum) - yr - yb, yb, cbr, cbg, -(cbr + cbg), -(crg + crb), crg, crb, yoff, coff]


def half_value(h: int):
    """the exact value of a non-negative finite binary16, as an mpmath number"""
    import mpmath
    e, m = h >> 10, h & 1023
    return mpmath.ldexp(m, -24) if e == 0 else mpmath.ldexp(1024 + m, e - 25)


def pq_out_code(h: int, unit_nits: int) -> int:
    """P[h] of include/hap_b200.h at 50 digits: floor(4095 * OETF(min(value(h) * unitNits / 10000, 1)) + 1/2)"""
    import mpmath
    mpmath.mp.dps = 50
    y = min(half_value(h) * unit_nits / 10000, mpmath.mpf(1))
    m1, m2 = mpmath.mpf(2610) / 16384, mpmath.mpf(2523) / 32
    c1, c2, c3 = mpmath.mpf(3424) / 4096, mpmath.mpf(2413) / 128, mpmath.mpf(2392) / 128
    p = y ** m1
    return int(mpmath.floor(4095 * ((c1 + c2 * p) / (1 + c3 * p)) ** m2 + mpmath.mpf(1) / 2))


@functools.lru_cache(None)
def pq_out_table(unit_nits: int) -> np.ndarray:
    """P for every non-negative finite binary16 (ENTRIES,) int64, mpmath at 50 digits; values at or above 10000 / unitNits are
    4095 without evaluation (min(.., 1) makes them so)"""
    out = np.full(ENTRIES, 4095, np.int64)
    for h in range(ENTRIES):
        if half_value(h) * unit_nits >= 10000:
            break
        out[h] = pq_out_code(h, unit_nits)
    return out


def codes(rgba_half, table) -> np.ndarray:
    """(h, w, 4) uint16 binary16 RGBA -> (h, w, 3) int64 12-bit codes: sign bit set -> 0, else table[min(h, 0x7BFF)]"""
    v = np.asarray(rgba_half)[..., :3].astype(np.int64)
    return np.where(v >= 0x8000, 0, np.asarray(table, np.int64)[np.minimum(v, ENTRIES - 1)])


def samples_of_codes(c, cs):
    """(h, w, 3) 12-bit codes -> (luma (h, w), chroma (h/2, w) interleaved Cb, Cr) int64 samples of the integer matrix"""
    k = row(cs)
    c = np.asarray(c, np.int64)
    luma = np.clip(((k[0] * c[..., 0] + k[1] * c[..., 1] + k[2] * c[..., 2] + 32768) >> 16) + k[9], 0, 1023)
    s = O.filtered(c)
    cb = np.clip(((k[3] * s[..., 0] + k[4] * s[..., 1] + k[5] * s[..., 2] + (1 << 18)) >> 19) + k[10], 0, 1023)
    cr = np.clip(((k[6] * s[..., 0] + k[7] * s[..., 1] + k[8] * s[..., 2] + (1 << 18)) >> 19) + k[10], 0, 1023)
    h, w = luma.shape
    return luma, np.stack([cb, cr], -1).reshape(h // 2, w)


def samples_of_codes_float(c, cs):
    """the same filter, then the real BT.2020 matrix in float64 on codes / 4095, clamped to 0..1023: (luma, chroma)"""
    yoff, ys, csc, coff = P.scales(cs)
    kg = 1 - P.KR - P.KB
    p = np.asarray(c, np.float64) / 4095
    luma = yoff + ys * (P.KR * p[..., 0] + kg * p[..., 1] + P.KB * p[..., 2])
    s = O.filtered(c) / (8.0 * 4095)
    ey = P.KR * s[..., 0] + kg * s[..., 1] + P.KB * s[..., 2]
    cb = coff + csc * (s[..., 2] - ey) / (2 * (1 - P.KB))
    cr = coff + csc * (s[..., 0] - ey) / (2 * (1 - P.KR))
    h, w = luma.shape
    return np.clip(luma, 0, 1023), np.clip(np.stack([cb, cr], -1).reshape(h // 2, w), 0, 1023)


def rgba_half_to_yuv_pq(rgba_half, cs, unit_nits, table=None):
    """The conversion of include/hap_b200.h: (h, w, 4) uint16 binary16 RGBA -> (luma (h, w), chroma (h/2, w)) P010 words
    (sample << 6).  table: P of unit_nits (default: the library's own, twin_table)"""
    t = twin_table(unit_nits) if table is None else table
    luma, chroma = samples_of_codes(codes(rgba_half, t), cs)
    return (luma << 6).astype(np.uint16), (chroma << 6).astype(np.uint16)


def black(cs):
    """the (Y, Cb = Cr) samples of codes (0, 0, 0): the planes of a frame that failed"""
    k = row(cs)
    return k[9], k[10]


@functools.lru_cache(None)
def _twin():
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libyuv_pq_out_twin.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
                    "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "yuv_pq_out_twin.cc"), "-o", so], check=True)
    return C.CDLL(so)


@functools.lru_cache(None)
def twin_table(unit_nits) -> np.ndarray:
    """the library's own P (yuv_pq_out_table of hap_b200/csrc/yuv_sink.cuh, built on the host) -> (ENTRIES,) int64"""
    out = np.zeros(ENTRIES, np.uint16)
    _twin().yuv_pq_out_twin_table(C.c_uint32(unit_nits), C.c_void_p(out.ctypes.data))
    return out.astype(np.int64)


def twin_to_yuv(rgba_half, cs, unit_nits, pitch=None):
    """tests/emu/yuv_pq_out_twin.cc on the same picture, planes written with row pitch `pitch` (default: tight) -> (luma, chroma)
    words, the pitch slack dropped (and checked to be untouched)"""
    rgba = np.ascontiguousarray(rgba_half, dtype=np.uint16)
    h, w = rgba.shape[:2]
    pitch = pitch or 2 * w
    lb, cb = np.full((h, pitch), 0xA5, np.uint8), np.full((h // 2, pitch), 0xA5, np.uint8)
    _twin().yuv_pq_out_twin_from_half(C.c_void_p(rgba.ctypes.data), C.c_uint32(w), C.c_uint32(h), C.c_int(cs), C.c_uint32(unit_nits),
                                      C.c_void_p(lb.ctypes.data), C.c_void_p(cb.ctypes.data), C.c_uint64(pitch))
    assert (lb[:, 2 * w:] == 0xA5).all() and (cb[:, 2 * w:] == 0xA5).all()
    return (np.ascontiguousarray(lb[:, : 2 * w]).view(np.uint16).reshape(h, w),
            np.ascontiguousarray(cb[:, : 2 * w]).view(np.uint16).reshape(h // 2, w))


def random_halves(rng, h, w, signed=True) -> np.ndarray:
    """(h, w, 4) uint16 binary16 RGBA as the BC6H decoder writes them: any finite value (UF16: 0 .. 0x7BFF; SF16 also
    negatives and -0), A = 1.0; a third of the pixels small (below 1.0), where P is steepest"""
    v = rng.integers(0, 0x7C00, (h, w, 4), dtype=np.int64)
    small = rng.random((h, w, 1)) < 0.33
    v = np.where(small, v % 0x3C00, v)
    if signed:
        v |= np.where(rng.random((h, w, 4)) < 0.25, 0x8000, 0)
    v[..., 3] = P.ONE
    return v.astype(np.uint16)
