"""Deterministic integer-only synthetic RGBA frames (SURVEY.md section 8d).

One implementation on torch integer ops, so the same code produces the host frames the CPU oracle
is fed in tests and the device-resident frame streams bench.py times.  Pinned by a CRC in
tests/test_synth.py.  Kinds:
  video  smooth triangle-wave gradients, hash noise on a 64-px checkerboard of tiles, letterbox bars
         (partly compressible: Snappy ratio ~0.6 on the Hap Q payload)
  flat   constant 0x336699FF (maximum compressibility, exercises the RLE paths)
  noise  hash bytes (incompressible, exercises both raw fallbacks of hap.c:460 and :478)
Content classes for the block-encoder quality bar (tests only; the benchmark stream is `video`):
  gradient  steep two-axis colour ramps without grain (where a 4-colour palette per block hurts most)
  texture   grain of 5 bits on every pixel over slow ramps (camera footage at high gain)
  edges     hard-edged graphics: bars, checkers and 1-pixel lines in saturated colours on flat ground
"""
from __future__ import annotations

import torch

SEED = 20260923
_M32 = 0xFFFFFFFF


def pcg_hash(v: torch.Tensor) -> torch.Tensor:
    """PCG-RXS-M-XS 32-bit output hash on int64 tensors holding uint32 values."""
    state = (v * 747796405 + 2891336453) & _M32
    shift = (state >> 28) + 4
    word = (((state >> shift) ^ state) * 277803737) & _M32
    return ((word >> 22) ^ word) & _M32


def _tri8(t: torch.Tensor) -> torch.Tensor:
    u = t & 511
    return torch.where(u < 256, u, 511 - u)


def frame(width: int, height: int, index: int = 0, kind: str = "video", alpha: str = "opaque",
          seed: int = SEED, noise_bits: int = 3, device="cpu", rows=None) -> torch.Tensor:
    """(height, width, 4) uint8 RGBA frame number `index`; with rows=(y0, y1) only those rows of it, (y1 - y0, width, 4),
    bit-identical to the same rows of the whole frame (the int64 intermediates of a whole 16K frame take 8 GiB each)."""
    dev = torch.device(device)
    y0, y1 = rows if rows is not None else (0, height)
    if kind == "flat":
        px = torch.tensor([0x33, 0x66, 0x99, 0xFF], dtype=torch.uint8, device=dev)
        return px.expand(y1 - y0, width, 4).contiguous()
    y = torch.arange(y0, y1, dtype=torch.int64, device=dev).view(y1 - y0, 1, 1)
    x = torch.arange(width, dtype=torch.int64, device=dev).view(1, width, 1)
    c = torch.arange(4, dtype=torch.int64, device=dev).view(1, 1, 4)
    lin = (((index * height + y) * width + x) * 4 + c) & _M32
    h = pcg_hash(lin ^ (seed & _M32))
    if kind == "noise":
        out = (h >> 24).to(torch.uint8)
        out[..., 3] = 255
        return out
    if kind in ("gradient", "texture", "edges"):
        out = _content_class(kind, x, y, c, h, index, width, height)
        return _apply_alpha(out, alpha, x, y, width, height)
    if kind != "video":
        raise ValueError(kind)
    k1 = torch.tensor([1, 2, 3, 1], dtype=torch.int64, device=dev).view(1, 1, 4)
    k2 = torch.tensor([2, 1, 3, 1], dtype=torch.int64, device=dev).view(1, 1, 4)
    px = (3 * x * k1 * 512) // width + 8 * index
    py = (5 * y * k2 * 512) // height
    half = 1 << (noise_bits - 1) if noise_bits > 0 else 0
    nz = (h >> (32 - noise_bits)) - half if noise_bits > 0 else torch.zeros_like(h)
    # camera-like grain only on every other 64x64 tile: the rest stays clean gradient (graphics-like), so the
    # DXT payload is PARTLY compressible like real footage (Snappy ratio ~0.6) instead of all-or-nothing
    nz = nz * (((x >> 6) + (y >> 6)) & 1)
    v = 43 + _tri8(px) // 3 + _tri8(py) // 3 + nz
    v = v.clamp(0, 255)
    bar = height // 10
    letter = (y < bar) | (y >= height - bar)
    v = torch.where(letter, torch.full_like(v, 16), v)
    out = v.to(torch.uint8)
    return _apply_alpha(out, alpha, x, y, width, height)


def _content_class(kind, x, y, c, h, index, width, height):
    if kind == "gradient":
        k1 = torch.tensor([7, 3, 5, 1], dtype=torch.int64, device=x.device).view(1, 1, 4)
        k2 = torch.tensor([2, 9, 4, 1], dtype=torch.int64, device=x.device).view(1, 1, 4)
        v = (_tri8((x * k1 * 512) // width + 16 * index) + _tri8((y * k2 * 512) // height)) // 2
        return v.clamp(0, 255).to(torch.uint8)
    if kind == "texture":
        k1 = torch.tensor([1, 2, 1, 1], dtype=torch.int64, device=x.device).view(1, 1, 4)
        v = 64 + _tri8((x * k1 * 512) // width) // 4 + _tri8((y * 512) // height) // 4 + (h >> 27) - 16
        return v.clamp(0, 255).to(torch.uint8)
    # edges
    pal = torch.tensor([[230, 30, 30, 255], [30, 200, 60, 255], [40, 60, 230, 255], [240, 240, 240, 255], [20, 20, 20, 255],
                        [250, 200, 20, 255]], dtype=torch.int64, device=x.device)
    cell = ((x // 37) + (y // 23) * 7 + index) % 6
    stripe = ((x + 2 * y) // 5) % 2
    line = ((x % 61) == 0) | ((y % 47) == 0)
    idx = torch.where(line, torch.full_like(cell, 3), torch.where(stripe == 1, cell, torch.full_like(cell, 4)))
    checker = (((x // 3) + (y // 3)) % 2) == 1
    region = (y * 3 // max(height, 1)) == 1
    idx = torch.where(region & checker, (cell + 1) % 6, idx)
    return pal[idx[..., 0]].to(torch.uint8)


def _apply_alpha(out, alpha, x, y, width, height):
    if alpha == "opaque":
        out[..., 3] = 255
    elif alpha == "ramp":
        # horizontal ramp blended with a soft disc (Hap Q Alpha / Hap Alpha configs)
        ramp = (255 * x) // max(width - 1, 1)
        cx, cy = width // 2, height // 2
        r2 = (x - cx) * (x - cx) + (y - cy) * (y - cy)
        rad2 = (min(width, height) // 3) ** 2
        disc = (255 - (255 * r2) // max(rad2, 1)).clamp(0, 255)
        a = torch.maximum(ramp.expand(y.shape[0], width, 1), disc)
        out[..., 3] = a[..., 0].to(torch.uint8)
    else:
        raise ValueError(alpha)
    return out


def frames(width: int, height: int, count: int, start: int = 0, **kw) -> torch.Tensor:
    """(count, height, width, 4) uint8"""
    return torch.stack([frame(width, height, start + i, **kw) for i in range(count)])
