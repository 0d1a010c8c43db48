"""The fused Hap Q encoder with its fit and compressor in warp groups of their own (hapq_fused.cuh, hapq_ws_place_kernel)
under the fiber SIMT emulator: byte-identical output slots (sentinel-filled, so writes past a frame's end show), frame
lengths, fragment sizes, index entries, scratch slots and written-through textures against hapq_fused_place_kernel, in
every thread resume order, with a grid of one CTA, of three, and of more CTAs than fragments, and under ASan with exact-size
buffers (tests/emu/test_fused_ws_emu.cc)."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu"), "-I", os.path.join(ROOT, "oracle")]
SRC = [os.path.join(ROOT, "tests", "emu", "test_fused_ws_emu.cc")] + [os.path.join(ROOT, "oracle", f) for f in ("snappy_oracle.c", "hap_oracle.c")]


def _run(exe, flags, modes, env=None):
    os.makedirs(BUILD, exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + flags + INC + SRC + ["-ldl", "-lm", "-o", exe], check=True)
    p = subprocess.run([exe, str(modes)], capture_output=True, text=True, timeout=1800, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    assert " 0 failures" in p.stdout, p.stdout


def test_fused_ws_emulated():
    _run(os.path.join(BUILD, "test_fused_ws_emu"), [], 4)   # forward, reverse and two seeded shuffles


def test_fused_ws_under_address_sanitizer():
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    _run(os.path.join(BUILD, "test_fused_ws_emu_asan"), ["-fsanitize=address"], 2, env)
