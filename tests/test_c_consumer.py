"""A compiled C host program that includes the REFERENCE's hap.h and links libhap_b200.so -- the drop-in boundary exercised
the way a C application would.  The reference-header build is oracle/_ref/c_consumer_ref (oracle/Makefile, made by
build() wherever the reference sources are, kept with the reference build); the own-header build is made here."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "c_consumer", "consumer.c")
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
LIBDIR = os.path.join(ROOT, "hap_b200")
REF_EXE = os.path.join(ROOT, "oracle", "_ref", "c_consumer_ref")


def build(which: str) -> str:
    if which == "ref":
        subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "ref"], check=True, capture_output=True)
        return REF_EXE if os.path.exists(REF_EXE) else ""
    exe = os.path.join(BUILD, "c_consumer_own")
    os.makedirs(BUILD, exist_ok=True)
    subprocess.run(["gcc", "-std=c99", "-O1", "-Wall", "-Werror", "-D_GNU_SOURCE", "-I", os.path.join(ROOT, "include"), SRC, "-o", exe,
                    "-L", LIBDIR, "-l:libhap_b200.so", "-Wl,-rpath," + LIBDIR, "-pthread"], check=True)
    return exe


@pytest.mark.parametrize("which", ["ref", "own"])
def test_c_consumer_container_paths(which):
    import hap_b200
    hap_b200.load()
    exe = build(which)
    if not exe:
        pytest.skip("reference build unavailable")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert p.returncode == 0 and "consumer ok" in p.stdout, p.stdout + p.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["ref", "own"])
def test_c_consumer_gpu_paths(which):
    exe = build(which)
    if not exe:
        pytest.skip("reference build unavailable")
    p = subprocess.run([exe, "--gpu"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0 and "GPU paths" in p.stdout, p.stdout + p.stderr
