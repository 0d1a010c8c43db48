"""The HDR10 instantiation of the BC6H encode kernel (bc6h_encode_kernel with the P010 / BT.2020 / PQ source) under the
fiber SIMT emulator at odd block widths, wide pitches, strided frames, wide block strides and an NVDEC-style chroma plane,
UF16 and SF16, both ranges and several unitNits (tests/emu/test_yuv_pq_emu.cc).  Each block must equal the RGBA16F block
encoder applied to the reference conversion of its pixels.  Once plainly and once under AddressSanitizer with exact-size
planes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu")]


@pytest.mark.parametrize("asan", [False, True])
def test_yuv_pq_encode_kernel_emulated(asan):
    os.makedirs(BUILD, exist_ok=True)
    exe = os.path.join(BUILD, "test_yuv_pq_emu" + ("_asan" if asan else ""))
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + (["-fsanitize=address"] if asan else []) + INC +
                   [os.path.join(ROOT, "tests", "emu", "test_yuv_pq_emu.cc"), "-ldl", "-lm", "-o", exe], check=True)
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    assert " 0 failures" in p.stdout
