"""The Y'CbCr -> RGBA8 pass of the Hap R encoders from NV12 / P010 and planar pictures (bc_source_to_rgba8_kernel, all eight
sources) under the fiber SIMT emulator at odd block widths, one-block-wide pictures, wide pitches, a chroma pitch different
from the luma pitch, and three strided frames with slack, with and without an alpha plane (tests/emu/test_yuv_bc7_emu.cc).
Every texel must equal the pixel-by-pixel reference conversion, and the bytes between frames keep their sentinel.  Once
plainly and once under AddressSanitizer with exact-size planes and output."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu")]


@pytest.mark.parametrize("asan", [False, True])
def test_yuv_to_rgba8_kernel_for_bc7_emulated(asan):
    os.makedirs(BUILD, exist_ok=True)
    exe = os.path.join(BUILD, "test_yuv_bc7_emu" + ("_asan" if asan else ""))
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + (["-fsanitize=address"] if asan else []) + INC +
                   [os.path.join(ROOT, "tests", "emu", "test_yuv_bc7_emu.cc"), "-ldl", "-lm", "-o", exe], check=True)
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    assert " 0 failures" in p.stdout
