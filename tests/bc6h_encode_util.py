"""Test-only helpers for Hap HDR (BC6H) ENCODING: the bindings of the two CPU encoders -- the oracle encoder
(tests/bc6h_oracle_encode.c, written apart from the kernel) and the host build of the kernel's own block encoder
(tests/emu/bc6h_encode_twin.cc) -- HDR test content (the synth.frame classes made linear, an exposure ramp), the input
rules, PSNR16, per-block errors and a mode-11 baseline packer on half input.  The decoding helpers (the oracle's and the
kernel's decoders, the block writer, Pillow) are tests/bc6h_util.py's."""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

from bc6h_util import BUILD, NMODES, ONE, ROOT, mode, pack_blocks

MAX_HALF = 0x7BFF                            # 65504, the largest finite binary16
CLASSES = ("video", "gradient", "texture", "edges", "noise")


@functools.lru_cache(None)
def _encode_twin(partition_fits: int = 0):
    """the host build of bc6h_encode.cuh (tests/emu/bc6h_encode_twin.cc); partition_fits 0: the kernel's own constant"""
    os.makedirs(BUILD, exist_ok=True)
    name = "bc6h_encode_twin" + ("_%d" % partition_fits if partition_fits else "")
    so = os.path.join(BUILD, "lib%s.so" % name)
    cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
           "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "bc6h_encode_twin.cc"), "-o", so]
    if partition_fits:
        cmd.insert(1, "-DHAPB200_BC6H_PARTITION_FITS=%d" % partition_fits)
    subprocess.run(cmd, check=True)
    return C.CDLL(so)


@functools.lru_cache(None)
def _oracle_encoder():
    """tests/bc6h_oracle_encode.c (the decoder oracle included)"""
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libbc6h_oracle_encode.so")
    subprocess.run(["gcc", "-std=c11", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "tests"),
                    os.path.join(ROOT, "tests", "bc6h_oracle_encode.c"), "-o", so, "-lm"], check=True)
    return C.CDLL(so)


def _rgba_half(img) -> np.ndarray:
    img = np.ascontiguousarray(np.asarray(img, np.uint16))
    assert img.ndim == 3 and img.shape[2] == 4 and img.shape[0] % 4 == 0 and img.shape[1] % 4 == 0
    return img


def twin_encode(img, signed: bool, partition_fits: int = 0):
    """The kernel's block encoder on the host: (h, w, 4) binary16 bits -> (blocks bytes, per-block chosen error uint64)"""
    img = _rgba_half(img)
    h, w = img.shape[:2]
    nb = (w // 4) * (h // 4)
    out, errs = np.zeros(16 * nb, np.uint8), np.zeros(nb, np.uint64)
    _encode_twin(partition_fits).bc6h_twin_encode(C.c_void_p(img.ctypes.data), C.c_int(w), C.c_int(h), C.c_long(4 * w),
                                                  C.c_int(int(signed)), C.c_void_p(out.ctypes.data), C.c_void_p(errs.ctypes.data))
    return out.tobytes(), errs


def twin_partition_fits() -> int:
    return int(_encode_twin().bc6h_twin_partition_fits())


def oracle_encode(img, signed: bool):
    """The oracle encoder (tests/bc6h_oracle.c): (h, w, 4) binary16 bits -> (blocks bytes, per-block chosen error)"""
    img = _rgba_half(img)
    h, w = img.shape[:2]
    nb = (w // 4) * (h // 4)
    out, errs = np.zeros(16 * nb, np.uint8), np.zeros(nb, np.uint64)
    _oracle_encoder().bc6h_oracle_encode(C.c_void_p(img.ctypes.data), C.c_int(w), C.c_int(h), C.c_int(int(signed)),
                                          C.c_void_p(out.ctypes.data), C.c_void_p(errs.ctypes.data))
    return out.tobytes(), errs


def in_blocks(fn, img, signed: bool, rows: int = 16):
    """fn(img, signed) over horizontal bands of `rows` pixel rows on a thread pool (the C encoders release the GIL)"""
    from concurrent.futures import ThreadPoolExecutor
    img = _rgba_half(img)
    fn(img[:4, :4], signed)                  # builds the library once, before the threads
    bands = [img[y:y + rows] for y in range(0, img.shape[0], rows)]
    with ThreadPoolExecutor(max(1, min(len(bands), os.cpu_count() or 1))) as ex:
        parts = list(ex.map(lambda b: fn(b, signed), bands))
    return b"".join(p[0] for p in parts), np.concatenate([p[1] for p in parts])


def to_rgba_half(rgb: np.ndarray) -> np.ndarray:
    """(h, w, 3) float values -> (h, w, 4) binary16 bits, A = 1.0"""
    h, w = rgb.shape[:2]
    out = np.empty((h, w, 4), np.uint16)
    out[..., :3] = np.asarray(rgb, np.float64).astype(np.float16).view(np.uint16)
    out[..., 3] = ONE
    return out


def hdr_content(kind: str, w: int, h: int, peak: float, signed: bool = False, index: int = 0) -> np.ndarray:
    """A synth.frame class made linear, (v / 255)^2.2 x peak; for SF16 centred on zero, (lin - peak / 2) x 2 -> (h, w, 4)
    binary16 bits"""
    from hap_b200 import synth
    lin = (synth.frame(w, h, index, kind=kind).numpy()[..., :3].astype(np.float64) / 255.0) ** 2.2 * peak
    return to_rgba_half((lin - peak / 2) * 2 if signed else lin)


def exposure_ramp(w: int, h: int, signed: bool = False) -> np.ndarray:
    """Values log-uniform from 2^-12 to 2^15 along the picture in reading order, each channel offset by a fraction of a
    stop; for SF16 every other row negative -> (h, w, 4) binary16 bits"""
    pos = np.arange(w * h, dtype=np.float64).reshape(h, w) / (w * h - 1)
    off = np.array([0.0, -0.37, -0.71])
    v = 2.0 ** (-12 + 27 * pos[..., None] + off)
    if signed:
        v = v * np.where(np.arange(h) % 2 == 0, 1.0, -1.0)[:, None, None]
    return to_rgba_half(v)


def source_values(img, signed: bool) -> np.ndarray:
    """the input rules: (h, w, >= 3) binary16 bits -> (h, w, 3) int64 sign-magnitude integers (UF16: negatives, -0 and NaN
    -> 0, +Inf -> 0x7BFF; SF16: NaN -> 0, +-Inf -> +-0x7BFF, -0 -> 0)"""
    b = np.asarray(img, np.uint16)[..., :3].astype(np.int64)
    mag = b & 0x7FFF
    mag = np.where(mag > 0x7C00, 0, np.where(mag == 0x7C00, MAX_HALF, mag))
    neg = (b & 0x8000) != 0
    return np.where(neg, -mag if signed else 0, mag)


def decoded_values(half) -> np.ndarray:
    """decoded binary16 bits -> (h, w, 3) int64 sign-magnitude integers"""
    b = np.asarray(half, np.uint16)[..., :3].astype(np.int64)
    return np.where(b & 0x8000, -(b & 0x7FFF), b)


def psnr16(decoded, img, signed: bool) -> float:
    """10 log10(0x7BFF^2 / MSE), the MSE over R, G, B of the sign-magnitude integers of decoded and clamped source halves"""
    mse = float(np.mean((decoded_values(decoded) - source_values(img, signed)).astype(np.float64) ** 2))
    return float("inf") if mse == 0 else 10 * np.log10(MAX_HALF ** 2 / mse)


def block_errors(decoded, img, signed: bool) -> np.ndarray:
    """per block (row-major) the sum of squared sign-magnitude differences over R, G, B"""
    d = (decoded_values(decoded) - source_values(img, signed)) ** 2
    h, w = d.shape[:2]
    return d.reshape(h // 4, 4, w // 4, 4, 3).transpose(0, 2, 1, 3, 4).reshape(-1, 48).sum(1).astype(np.uint64)


def baseline_encode(img, signed: bool) -> bytes:
    """Mode-11 min / max packer on half input, as pack_picture does on 8-bit pictures: per block and channel the minimum
    and maximum in the 10-bit code that decodes nearest, one 4-bit index per texel by its position between them"""
    img = _rgba_half(img)
    h, w = img.shape[:2]
    x = source_values(img, signed)
    unit, lo, top = (62.0, -511, 511) if signed else (31.0, 0, 1023)
    code = np.clip(np.rint(x / unit), lo, top).astype(np.int64)
    blk = code.reshape(h // 4, 4, w // 4, 4, 3).transpose(0, 2, 1, 3, 4).reshape(-1, 16, 3)
    e0, e1 = blk.min(1), blk.max(1)
    span = np.maximum((e1 - e0).sum(1), 1)
    idx = np.clip(((blk - e0[:, None, :]).sum(2) * 15 + span[:, None] // 2) // span[:, None], 0, 15)
    flip = idx[:, 0] >= 8
    idx[flip] = 15 - idx[flip]
    e0[flip], e1[flip] = e1[flip].copy(), e0[flip].copy()
    ep = np.zeros((len(blk), 12), np.int64)
    ep[:, 0:3], ep[:, 3:6] = e0 & 1023, e1 & 1023
    return pack_blocks(10, ep, np.zeros(len(blk), np.int64), idx).tobytes()


def block_modes(blocks) -> np.ndarray:
    """mode (0-13) of every block, -1 for a reserved mode value"""
    b0 = np.frombuffer(bytes(blocks), np.uint8)[::16].astype(np.int64)
    m5 = b0 & 0x1F
    lut = np.full(32, -1, np.int64)
    for m in range(NMODES):
        if mode(m).mode_bits == 5:
            lut[mode(m).mode_value] = m
    return np.where((b0 & 3) < 2, b0 & 1, lut[m5])
