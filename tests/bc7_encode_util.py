"""Test-only helpers for Hap R (BC7) ENCODING: the bindings of the two CPU encoders -- the oracle encoder
(tests/bc7_oracle_encode.c, written apart from the kernel) and the host build of the kernel's own block encoder
(tests/emu/bc7_encode_twin.cc) -- the test content (the synth.frame classes, opaque and with an alpha ramp, and noise with
random alpha), PSNR over R, G, B and A, per-block errors, block modes and a mode-6 bounding-box baseline.  The decoding
helpers (the oracle's and the kernel's decoders, the block writer, Pillow) are tests/bc7_util.py's."""
from __future__ import annotations

import ctypes as C
import functools
import os
import subprocess

import numpy as np

from bc7_util import BUILD, ROOT, mode_of, pack_picture

CLASSES = ("video", "gradient", "texture", "edges")
# (class, alpha): the four picture classes opaque and with synth's alpha ramp, and noise opaque and with random alpha
CONTENT = [(k, a) for k in CLASSES for a in ("opaque", "ramp")] + [("noise", "opaque"), ("noise", "random")]


@functools.lru_cache(None)
def _encode_twin(fits2: int = 0, fits3: int = 0):
    """the host build of bc7_encode.cuh (tests/emu/bc7_encode_twin.cc); fits 0: the kernel's own constants"""
    os.makedirs(BUILD, exist_ok=True)
    name = "bc7_encode_twin" + ("_%d_%d" % (fits2, fits3) if fits2 or fits3 else "")
    so = os.path.join(BUILD, "lib%s.so" % name)
    cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-w", "-I", os.path.join(ROOT, "hap_b200", "csrc"),
           "-I", os.path.join(ROOT, "tests", "emu"), os.path.join(ROOT, "tests", "emu", "bc7_encode_twin.cc"), "-o", so]
    if fits2:
        cmd.insert(1, "-DHAPB200_BC7_PARTITION_FITS=%d" % fits2)
    if fits3:
        cmd.insert(1, "-DHAPB200_BC7_PARTITION3_FITS=%d" % fits3)
    subprocess.run(cmd, check=True)
    return C.CDLL(so)


@functools.lru_cache(None)
def _oracle_encoder():
    """tests/bc7_oracle_encode.c (the decoder oracle included)"""
    os.makedirs(BUILD, exist_ok=True)
    so = os.path.join(BUILD, "libbc7_oracle_encode.so")
    subprocess.run(["gcc", "-std=c11", "-O2", "-Wall", "-fPIC", "-shared", "-I", os.path.join(ROOT, "tests"),
                    os.path.join(ROOT, "tests", "bc7_oracle_encode.c"), "-o", so, "-lm"], check=True)
    return C.CDLL(so)


def _rgba(img) -> np.ndarray:
    img = np.ascontiguousarray(np.asarray(img, np.uint8))
    assert img.ndim == 3 and img.shape[2] == 4 and img.shape[0] % 4 == 0 and img.shape[1] % 4 == 0
    return img


def twin_encode(img, fits2: int = 0, fits3: int = 0):
    """The kernel's block encoder on the host: (h, w, 4) uint8 -> (blocks bytes, per-block chosen error uint64)"""
    img = _rgba(img)
    h, w = img.shape[:2]
    nb = (w // 4) * (h // 4)
    out, errs = np.zeros(16 * nb, np.uint8), np.zeros(nb, np.uint64)
    _encode_twin(fits2, fits3).bc7_twin_encode(C.c_void_p(img.ctypes.data), C.c_int(w), C.c_int(h), C.c_long(4 * w),
                                               C.c_void_p(out.ctypes.data), C.c_void_p(errs.ctypes.data))
    return out.tobytes(), errs


def twin_partition_fits() -> tuple[int, int]:
    lib = _encode_twin()
    return int(lib.bc7_twin_partition_fits()), int(lib.bc7_twin_partition3_fits())


def oracle_encode(img):
    """The oracle encoder (tests/bc7_oracle_encode.c): (h, w, 4) uint8 -> (blocks bytes, per-block chosen error)"""
    img = _rgba(img)
    h, w = img.shape[:2]
    nb = (w // 4) * (h // 4)
    out, errs = np.zeros(16 * nb, np.uint8), np.zeros(nb, np.uint64)
    _oracle_encoder().bc7_oracle_encode(C.c_void_p(img.ctypes.data), C.c_int(w), C.c_int(h), C.c_void_p(out.ctypes.data),
                                        C.c_void_p(errs.ctypes.data))
    return out.tobytes(), errs


def in_blocks(fn, img, rows: int = 16):
    """fn(img) over horizontal bands of `rows` pixel rows on a thread pool (the C encoders release the GIL)"""
    from concurrent.futures import ThreadPoolExecutor
    img = _rgba(img)
    fn(img[:4, :4])                          # builds the library once, before the threads
    bands = [img[y:y + rows] for y in range(0, img.shape[0], rows)]
    with ThreadPoolExecutor(max(1, min(len(bands), os.cpu_count() or 1))) as ex:
        parts = list(ex.map(fn, bands))
    return b"".join(p[0] for p in parts), np.concatenate([p[1] for p in parts])


def content(kind: str, alpha: str, w: int, h: int, index: int = 0) -> np.ndarray:
    """synth.frame of a class with alpha "opaque" or "ramp"; noise with alpha "random" takes random A -> (h, w, 4) uint8"""
    from hap_b200 import synth
    img = synth.frame(w, h, index, kind=kind, alpha="opaque" if alpha == "random" else alpha).numpy().copy()
    if alpha == "random":
        img[..., 3] = np.random.default_rng(1000 + index).integers(0, 256, (h, w), dtype=np.uint8)
    return img


def psnr(decoded, img) -> float:
    """10 log10(255^2 / MSE), the MSE over R, G, B and A"""
    mse = float(np.mean((np.asarray(decoded, np.float64) - np.asarray(img, np.float64)) ** 2))
    return float("inf") if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


def block_errors(decoded, img) -> np.ndarray:
    """per block (row-major) the sum of squared differences over R, G, B and A"""
    d = (np.asarray(decoded, np.int64) - np.asarray(img, np.int64)) ** 2
    h, w = d.shape[:2]
    return d.reshape(h // 4, 4, w // 4, 4, 4).transpose(0, 2, 1, 3, 4).reshape(-1, 64).sum(1).astype(np.uint64)


def block_modes(blocks) -> np.ndarray:
    """mode (0-7) of every block, 8 for a reserved block"""
    return mode_of(np.frombuffer(bytes(blocks), np.uint8).reshape(-1, 16))


def baseline_encode(img) -> bytes:
    """the mode-6 bounding-box packer of tests/bc7_util.py: per block and channel the minimum and maximum, one 4-bit index
    per texel by its position between them"""
    return pack_picture(_rgba(img))
