"""The unit path of the Snappy execute kernel (indexed fragments made of 8-byte units) under the fiber SIMT emulator,
against the oracle: this encoder's fragments, 4-byte elements, copies that leave their fragment, lying indexes and every
destination misalignment; in six thread resume orders, and under ASan with exact-size buffers."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu"), "-I", os.path.join(ROOT, "oracle")]
SRC = [os.path.join(ROOT, "tests", "emu", "test_decode_units_emu.cc"), os.path.join(ROOT, "oracle", "snappy_oracle.c")]


def _run(exe, flags, modes, env=None):
    os.makedirs(BUILD, exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + flags + INC + SRC + ["-ldl", "-lm", "-o", exe], check=True)
    p = subprocess.run([exe, str(modes)], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    # the counter proves the unit path ran (and was not silently replaced by the general path)
    windows = int(p.stdout.split(" unit-path windows")[0].rsplit(" ", 1)[1])
    assert windows > 0, p.stdout


def test_decode_units_emulated():
    _run(os.path.join(BUILD, "test_decode_units_emu"), [], 6)


def test_decode_units_under_address_sanitizer():
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    _run(os.path.join(BUILD, "test_decode_units_emu_asan"), ["-fsanitize=address"], 3, env)
