"""The planar instantiations of the block encode kernel (bc_encode_planar_kernel: 4:2:0, 4:2:2 and 4:4:4 on bytes and
16-bit words, every colour kind and RGTC1) under the fiber SIMT emulator at odd block widths, one-block-wide pictures, a
chroma pitch different from the luma pitch, wide pitches and strided frames (tests/emu/test_planar_emu.cc).  Each block must
equal the per-block encoder applied to the reference conversion of its pixels.  Once plainly and once under
AddressSanitizer with exact-size planes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu")]


@pytest.mark.parametrize("asan", [False, True])
def test_planar_block_encode_kernels_emulated(asan):
    os.makedirs(BUILD, exist_ok=True)
    exe = os.path.join(BUILD, "test_planar_emu" + ("_asan" if asan else ""))
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + (["-fsanitize=address"] if asan else []) + INC +
                   [os.path.join(ROOT, "tests", "emu", "test_planar_emu.cc"), "-ldl", "-lm", "-o", exe], check=True)
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    assert " 0 failures" in p.stdout
