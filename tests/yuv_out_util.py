"""Test-only helpers for the NV12 / P010 decoders: the RGBA8 -> Y'CbCr 4:2:0 conversion of include/hap_b200.h
(HapB200DecodeYUV) restated in numpy integers (rgba_to_yuv_out), the same filter with the real matrix in float64
(rgba_to_yuv_out_float), the coefficient table read from the header and recomputed from its rule, plane helpers, and the
binding of the C++ pixel-by-pixel conversion (tests/emu/yuv_out_twin.cc) that the emulated kernel test is built on."""
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


@functools.lru_cache(None)
def coefficients() -> np.ndarray:
    """HAPB200_YUV_OUT_COEFFICIENTS of include/hap_b200.h: (8, 11) int64, row layout * 4 + colour space"""
    text = open(os.path.join(ROOT, "include", "hap_b200.h")).read()
    body = text[text.index("#define HAPB200_YUV_OUT_COEFFICIENTS"):]
    body = body[: body.index("\n\n")]
    rows = [[int(v) for v in r.split(",")] for r in re.findall(r"\{\s*(-?\d+(?:\s*,\s*-?\d+){10})\s*\}", body)]
    assert len(rows) == 8
    return np.array(rows, np.int64)


def rule_coefficients(layout, cs) -> list:
    """{yR, yG, yB, cbR, cbG, cbB, crR, crG, crB, yOff, cOff} from the rule the header states"""
    rnd = lambda v: int(np.floor(v + 0.5))
    yoff, ys, csc, coff = Y.scales(layout, cs)
    kr, kb = Y.KRKB[cs]
    kg = 1 - kr - kb
    lum, s = 65536 * ys / 255, 65536 * csc / 255
    yr, yb = rnd(lum * kr), rnd(lum * kb)
    cbr, cbg = rnd(-s * kr / (2 * (1 - kb))), rnd(-s * kg / (2 * (1 - kb)))
    crg, crb = rnd(-s * kg / (2 * (1 - kr))), rnd(-s * kb / (2 * (1 - kr)))
    return [yr, rnd(lum) - yr - yb, yb, cbr, cbg, -(cbr + cbg), -(crg + crb), crg, crb, yoff, coff]


def filtered(rgba) -> np.ndarray:
    """(h, w, 4) RGBA -> (h/2, w/2, 3) int64 sums of weight 8 at the chroma sites: columns 2i-1 (clamped), 2i, 2i+1 with
    weights 1 2 1, rows 2j and 2j+1"""
    p = np.asarray(rgba)[..., :3].astype(np.int64)
    h, w = p.shape[:2]
    i = np.arange(w // 2)
    left = np.maximum(2 * i - 1, 0)
    hs = p[:, left] + 2 * p[:, 2 * i] + p[:, 2 * i + 1]          # (h, w/2, 3)
    return hs[0::2] + hs[1::2]


def samples(rgba, layout, cs):
    """(luma (h, w), chroma (h/2, w) interleaved Cb, Cr) int64 samples of the integer conversion"""
    k = [int(v) for v in coefficients()[layout * 4 + cs]]
    top = (1 << Y.bits(layout)) - 1
    p = np.asarray(rgba)[..., :3].astype(np.int64)
    luma = np.clip(((k[0] * p[..., 0] + k[1] * p[..., 1] + k[2] * p[..., 2] + 32768) >> 16) + k[9], 0, top)
    s = filtered(rgba)
    cb = np.clip(((k[3] * s[..., 0] + k[4] * s[..., 1] + k[5] * s[..., 2] + (1 << 18)) >> 19) + k[10], 0, top)
    cr = np.clip(((k[6] * s[..., 0] + k[7] * s[..., 1] + k[8] * s[..., 2] + (1 << 18)) >> 19) + k[10], 0, top)
    h, w = luma.shape
    return luma, np.stack([cb, cr], -1).reshape(h // 2, w)


def store(plane, layout) -> np.ndarray:
    """samples -> the plane's storage: NV12 uint8, P010 uint16 words sample << 6"""
    return (plane << 6).astype(np.uint16) if layout == Y.P010 else plane.astype(np.uint8)


def rgba_to_yuv_out(rgba, layout, cs):
    """The conversion of include/hap_b200.h in integers: (h, w, 4) uint8 RGBA -> (luma (h, w), chroma (h/2, w)) as stored
    (NV12 uint8, P010 uint16 words)"""
    luma, chroma = samples(rgba, layout, cs)
    return store(luma, layout), store(chroma, layout)


def rgba_to_yuv_out_float(rgba, layout, cs):
    """The same filter, then the real (Kr, Kb) matrix in float64, clamped to the sample range: (luma, chroma) float64"""
    yoff, ys, csc, coff = Y.scales(layout, cs)
    kr, kb = Y.KRKB[cs]
    kg = 1 - kr - kb
    top = (1 << Y.bits(layout)) - 1
    p = np.asarray(rgba)[..., :3].astype(np.float64) / 255
    luma = yoff + ys * (kr * p[..., 0] + kg * p[..., 1] + kb * p[..., 2])
    s = filtered(rgba) / (8.0 * 255)
    ey = kr * s[..., 0] + kg * s[..., 1] + kb * s[..., 2]
    cb = coff + csc * (s[..., 2] - ey) / (2 * (1 - kb))
    cr = coff + csc * (s[..., 0] - ey) / (2 * (1 - kr))
    h, w = luma.shape
    return np.clip(luma, 0, top), np.clip(np.stack([cb, cr], -1).reshape(h // 2, w), 0, top)


@functools.lru_cache(None)
def _twin():
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libyuv_out_twin.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
                    "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "yuv_out_twin.cc"), "-o", so], check=True)
    return C.CDLL(so)


def twin_to_yuv(rgba, layout, cs, pitch=None):
    """tests/emu/yuv_out_twin.cc on the same picture, planes written with row pitch `pitch` (default: tight) -> (luma, chroma)
    as stored, the pitch slack dropped (and checked to be untouched)"""
    rgba = np.ascontiguousarray(rgba, dtype=np.uint8)
    h, w = rgba.shape[:2]
    sb = Y.sample_bytes(layout)
    pitch = pitch or w * sb
    lb, cb = np.full((h, pitch), 0xA5, np.uint8), np.full((h // 2, pitch), 0xA5, np.uint8)
    _twin().yuv_out_twin_from_rgba(C.c_void_p(rgba.ctypes.data), C.c_uint32(w), C.c_uint32(h), C.c_int(layout), C.c_int(cs),
                                   C.c_void_p(lb.ctypes.data), C.c_void_p(cb.ctypes.data), C.c_uint64(pitch))
    assert (lb[:, sb * w:] == 0xA5).all() and (cb[:, sb * w:] == 0xA5).all()
    dt = np.uint16 if layout == Y.P010 else np.uint8
    return (np.ascontiguousarray(lb[:, : sb * w]).view(dt).reshape(h, w), np.ascontiguousarray(cb[:, : sb * w]).view(dt).reshape(h // 2, w))


def black(layout, cs):
    """the (Y, Cb = Cr) samples of RGB (0, 0, 0): the planes of a frame that failed"""
    k = coefficients()[layout * 4 + cs]
    return int(k[9]), int(k[10])
