"""snappy_execute_units_kernel (the Snappy decoder's kernel for 8-byte granular fragments of an embedded index) under the
fiber SIMT emulator, in the library's launch sequence, against the oracle: the unit-path cases of test_decode_units_emu.cc
(this encoder's fragments, 4-byte elements, copies that leave their fragment, lying indexes, every destination
misalignment) must give the same bytes, the windows that took the unit path must be the unit kernel's, and the windows it
declines must reach the execute kernel; in six thread resume orders, and under ASan with exact-size buffers."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu"), "-I", os.path.join(ROOT, "oracle")]
SRC = [os.path.join(ROOT, "tests", "emu", "test_unit_kernel_emu.cc"), os.path.join(ROOT, "oracle", "snappy_oracle.c")]


def _run(exe, flags, modes, env=None):
    os.makedirs(BUILD, exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + flags + INC + SRC + ["-ldl", "-lm", "-o", exe], check=True)
    p = subprocess.run([exe, str(modes)], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    windows = int(p.stdout.split(" unit-kernel windows")[0].rsplit("\n", 1)[-1])
    declined = int(p.stdout.split(" declined")[0].rsplit(" ", 1)[1])
    assert windows > 0 and declined > 0, p.stdout


def test_unit_kernel_emulated():
    _run(os.path.join(BUILD, "test_unit_kernel_emu"), [], 6)


def test_unit_kernel_under_address_sanitizer():
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    _run(os.path.join(BUILD, "test_unit_kernel_emu_asan"), ["-fsanitize=address"], 3, env)
