"""The Hap R (BC7) encode kernel, bc_encode_kernel<kBcBc7>, under the fiber SIMT emulator at odd block widths, wide row
pitches, strided frames and wide block strides, on random bytes with constant and opaque blocks among them
(tests/emu/test_bc7_encode_emu.cc).  Its blocks must equal the host twin's and the padding must keep its sentinel.  Once
plainly and once under AddressSanitizer with exact-size buffers."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu")]


@pytest.mark.parametrize("asan", [False, True])
def test_bc7_encode_kernel_geometry_emulated(asan):
    os.makedirs(BUILD, exist_ok=True)
    exe = os.path.join(BUILD, "test_bc7_encode_emu" + ("_asan" if asan else ""))
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + (["-fsanitize=address"] if asan else []) + INC +
                   [os.path.join(ROOT, "tests", "emu", "test_bc7_encode_emu.cc"), "-ldl", "-lm", "-o", exe], check=True)
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    assert " 0 failures" in p.stdout
