"""The C symbols libhap_b200.so exports are its declared entry points alone: a host helper exported under a plain C name
would collide with any function of that name in the application that loads the library."""
import os
import re
import subprocess

import pytest

import hap_b200

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from hap_b200 import build
    build.build()
    return hap_b200.load()


def declared_functions():
    names = set()
    for hdr in ("hap.h", "hap_b200.h", "hap_mov.h"):
        text = open(os.path.join(ROOT, "include", hdr)).read()
        names |= set(re.findall(r"\b([A-Za-z_]\w*)\s*\(", text))
    return names


def test_every_unmangled_exported_function_is_declared_in_the_headers(lib):
    out = subprocess.run(["nm", "-D", "--defined-only", hap_b200.lib.library_path()], capture_output=True, text=True, check=True).stdout
    text = {f[2] for f in (line.split() for line in out.splitlines()) if len(f) == 3 and f[1] == "T"}
    # names that start with an underscore are reserved to the implementation: mangled C++ (_Z...) and the toolchain's own
    unmangled = {n for n in text if not n.startswith("_")}
    assert "HapDecode" in unmangled and "HapB200DecodeYUVPQ" in unmangled, sorted(unmangled)
    assert sorted(unmangled - declared_functions()) == []
