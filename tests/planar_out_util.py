"""Test-only helpers for the planar decoders (HapB200DecodePlanar*): the RGBA8 -> planar Y'CbCr 4:2:0 / 4:2:2 / 4:4:4 (+ alpha)
conversion of include/hap_b200.h restated in numpy integers (rgba_to_planar_out), the same filters with the real matrix in
float64 (rgba_to_planar_out_float), the 12-bit row table read from the header and every row recomputed from its rule
(rule_row), and the binding of the C++ sample-by-sample conversion (tests/emu/planar_out_twin.cc) that the emulated kernel test
is built on.  The 8- and 10-bit rows are yuv_out_util's."""
from __future__ import annotations

import ctypes as C
import functools
import os
import re
import subprocess

import numpy as np

import planar_util as P
import yuv_out_util as O
import yuv_util as Y

ROOT = Y.ROOT
BUILD = Y.BUILD
S420, S422, S444 = P.S420, P.S422, P.S444
SUBSAMPLINGS, DEPTHS, COLOR_SPACES = P.SUBSAMPLINGS, P.DEPTHS, P.COLOR_SPACES


@functools.lru_cache(None)
def coefficients12() -> np.ndarray:
    """HAPB200_YUV_12BIT_OUT_COEFFICIENTS of include/hap_b200.h: (4, 11) int64, row colour space"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_12BIT_OUT_COEFFICIENTS"):]
    body = body[: body.index("\n\n")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{\s*(-?\d+(?:\s*,\s*-?\d+){10})\s*\}", body)]
    assert len(rows) == 4
    return np.array(rows, np.int64)


def row(n, cs) -> list:
    """{yR, yG, yB, cbR, cbG, cbB, crR, crG, crB, yOff, cOff} of depth n and colour space cs, as the header lists it"""
    if n == 12:
        return [int(v) for v in coefficients12()[cs]]
    return [int(v) for v in O.coefficients()[(Y.P010 if n == 10 else Y.NV12) * 4 + cs]]


def rule_row(n, cs) -> list:
    """the same row from the rule the header states, with the scales of depth n"""
    rnd = lambda v: int(np.floor(v + 0.5))
    yoff, ys, csc, coff = P.scales(n, cs)
    kr, kb = Y.KRKB[cs]
    kg = 1 - kr - kb
    lum, s = 65536 * ys / 255, 65536 * csc / 255
    yr, yb = rnd(lum * kr), rnd(lum * kb)
    cbr, cbg = rnd(-s * kr / (2 * (1 - kb))), rnd(-s * kg / (2 * (1 - kb)))
    crg, crb = rnd(-s * kg / (2 * (1 - kr))), rnd(-s * kb / (2 * (1 - kr)))
    return [yr, rnd(lum) - yr - yb, yb, cbr, cbg, -(cbr + cbg), -(crg + crb), crg, crb, yoff, coff]


def sums(rgba, sub) -> np.ndarray:
    """(h, w, 4) RGBA -> (ch, cw, 3) int64 chroma sums of total weight 8: 4:2:0 the NV12 sink's [1 2 1] x [1 1], 4:2:2
    [1 2 1] on the sample's own row times 2, 4:4:4 8 times the pixel; column -1 clamped to 0"""
    p = np.asarray(rgba)[..., :3].astype(np.int64)
    if sub == S420:
        return O.filtered(rgba)
    if sub == S444:
        return 8 * p
    w = p.shape[1]
    i = np.arange(w // 2)
    return 2 * (p[:, np.maximum(2 * i - 1, 0)] + 2 * p[:, 2 * i] + p[:, 2 * i + 1])


def alpha_out(a, n) -> np.ndarray:
    """a = (2 (2^n - 1) A + 255) / 510, integer division"""
    return (2 * ((1 << n) - 1) * np.asarray(a, np.int64) + 255) // 510


def samples(rgba, sub, n, cs, alpha=True):
    """(luma (h, w), cb, cr (P.chroma_shape), alpha (h, w) or None) int64 samples of the integer conversion"""
    k = row(n, cs)
    top = (1 << n) - 1
    p = np.asarray(rgba)[..., :3].astype(np.int64)
    luma = np.clip(((k[0] * p[..., 0] + k[1] * p[..., 1] + k[2] * p[..., 2] + 32768) >> 16) + k[9], 0, top)
    s = sums(rgba, sub)
    cb = np.clip(((k[3] * s[..., 0] + k[4] * s[..., 1] + k[5] * s[..., 2] + (1 << 18)) >> 19) + k[10], 0, top)
    cr = np.clip(((k[6] * s[..., 0] + k[7] * s[..., 1] + k[8] * s[..., 2] + (1 << 18)) >> 19) + k[10], 0, top)
    return luma, cb, cr, (alpha_out(np.asarray(rgba)[..., 3], n) if alpha else None)


def store(plane, n) -> np.ndarray:
    """samples -> the plane's storage: uint8 (n = 8) or uint16 words holding the sample in the low bits"""
    return None if plane is None else plane.astype(np.uint8 if n == 8 else np.uint16)


def rgba_to_planar_out(rgba, sub, n, cs, alpha=True):
    """The conversion of include/hap_b200.h in integers: (h, w, 4) uint8 RGBA -> (luma, cb, cr, alpha or None) as stored"""
    return tuple(store(s, n) for s in samples(rgba, sub, n, cs, alpha))


def rgba_to_planar_out_float(rgba, sub, n, cs):
    """The same filters, then the real (Kr, Kb) matrix in float64, clamped to the sample range: (luma, cb, cr) float64"""
    yoff, ys, csc, coff = P.scales(n, cs)
    kr, kb = Y.KRKB[cs]
    kg = 1 - kr - kb
    top = (1 << n) - 1
    p = np.asarray(rgba)[..., :3].astype(np.float64) / 255
    luma = yoff + ys * (kr * p[..., 0] + kg * p[..., 1] + kb * p[..., 2])
    s = sums(rgba, sub) / (8.0 * 255)
    ey = kr * s[..., 0] + kg * s[..., 1] + kb * s[..., 2]
    cb = coff + csc * (s[..., 2] - ey) / (2 * (1 - kb))
    cr = coff + csc * (s[..., 0] - ey) / (2 * (1 - kr))
    return np.clip(luma, 0, top), np.clip(cb, 0, top), np.clip(cr, 0, top)


def black(n, cs):
    """the (Y, Cb = Cr) samples of RGB (0, 0, 0): the colour planes of a frame that failed (its alpha is 0)"""
    k = row(n, cs)
    return k[9], k[10]


@functools.lru_cache(None)
def _twin():
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libplanar_out_twin.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
                    "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "planar_out_twin.cc"), "-o", so],
                   check=True)
    return C.CDLL(so)


def twin_to_planar(rgba, sub, n, cs, alpha=True, luma_pad=0, chroma_pad=0):
    """tests/emu/planar_out_twin.cc on the same picture, rows padded by luma_pad / chroma_pad bytes -> (luma, cb, cr, alpha or
    None) as stored, the padding dropped (and checked to be untouched)"""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    h, w = rgba.shape[:2]
    sb = P.sample_bytes(n)
    ch, cw = P.chroma_shape(w, h, sub)
    lp, cp = w * sb + luma_pad, cw * sb + chroma_pad
    bufs = [np.full((h, lp), 0xA5, np.uint8), np.full((ch, cp), 0xA5, np.uint8), np.full((ch, cp), 0xA5, np.uint8),
            np.full((h, lp), 0xA5, np.uint8) if alpha else None]
    ptr = lambda b: C.c_void_p(None if b is None else b.ctypes.data)
    _twin().planar_out_twin_from_rgba(C.c_void_p(rgba.ctypes.data), C.c_uint32(w), C.c_uint32(h), *[ptr(b) for b in bufs],
                                      C.c_uint64(lp), C.c_uint64(cp), C.c_int(sub), C.c_int(n), C.c_int(cs))
    dt = np.uint8 if n == 8 else np.uint16
    out = []
    for b, samples_per_row in zip(bufs, (w, cw, cw, w)):
        if b is None:
            out.append(None)
            continue
        assert (b[:, sb * samples_per_row:] == 0xA5).all()
        out.append(np.ascontiguousarray(b[:, : sb * samples_per_row]).view(dt).reshape(b.shape[0], samples_per_row))
    return tuple(out)
