"""The planar sink of the block decoder (bc_decode_planar_kernel, bc_decode_planar_alpha_kernel) under the fiber SIMT emulator:
every instantiation, at block widths around the 31-column warp span, odd heights in blocks, wide and unequal pitches, strided
frames, the alpha plane present and absent, Hap Alpha-Only with no luma, Cb or Cr plane, and a failed frame
(tests/emu/test_planar_out_emu.cc).  Every sample must equal the sample-by-sample conversion applied to the block decoder's
texels, and every other byte must keep its sentinel.  Once plainly and once under AddressSanitizer with exact-size planes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu")]


@pytest.mark.parametrize("asan", [False, True])
def test_planar_block_decode_kernels_emulated(asan):
    os.makedirs(BUILD, exist_ok=True)
    exe = os.path.join(BUILD, "test_planar_out_emu" + ("_asan" if asan else ""))
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + (["-fsanitize=address"] if asan else []) + INC +
                   [os.path.join(ROOT, "tests", "emu", "test_planar_out_emu.cc"), "-ldl", "-lm", "-o", exe], check=True)
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    assert " 0 failures" in p.stdout
