"""Pins the exact output bytes of the encode path (K5 fragment compressor, K6 plan + place) under the fiber SIMT
emulator.  K5's decisions do not depend on how units are dealt to threads or how many CTAs stride over the
fragments, so a change to its CTA shape or thread mapping must reproduce these digests exactly.  A change that
alters the Snappy bytes on purpose (fragment size, hash bits, propagation) has to record new digests here."""
import subprocess

from test_kernels_emulated import ORC, compile_emu

# "<case> <digest>" per case of tests/emu/test_encode_emu.cc: FNV-1a 64 over each of the four write-index /
# offset-table variants' frame, fragment sizes and fragment index entries (tests/emu/test_encode_digest_emu.cc).
# Recorded from the kernel that ran one 1024-thread CTA per SM with 4 units per thread.
EXPECTED = """
dxt1_1chunk 442ba9bfa1ba174c
dxt1_3chunks 28ce1f0c0a5a90f7
dxt5_4chunks 814578ca4dc945d4
ycocg_8chunks afee2ee4df23cd3d
ycocg_limit_7_to_x e42b21860bff705b
rgtc_2chunks e87d4244e6984b1a
hapm 180b52017afd986b
hapm_mixed_none c4a9f0ff4c68cf16
none_single aee255ec8ccc3719
none_pair d4886d5fbedb4615
noise_fallback_whole f4792308328ee8e1
flat_rle a7f72315ce730891
big_multi_fragment 76b589a2b0761808
big_1chunk 7f7d22810c0eb3fb
tiny_16 2641318ac0149505
tiny_8 d310ca1cf0b4f601
kat_a_64x55 c3cfc9c6b86f02f7
mixed_chunk_fallback 5a599d070ea128eb
random_0 6be0b311a9af7959
random_1 7470218c8b34eef1
random_2 1e144dc06e1fe19b
random_3 821202b66652a985
random_4 e131185e5075f1a4
random_5 21a63c9a0d3b1dc0
random_6 f8b12e1e402c400b
random_7 f64d3473dc1ca068
"""


def test_encode_bytes_match_recorded_digests():
    exe = compile_emu("test_encode_digest_emu", ORC)
    p = subprocess.run([exe], capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout + p.stderr
    got = dict(line.split() for line in p.stdout.splitlines() if line.strip())
    want = dict(line.split() for line in EXPECTED.strip().splitlines())
    assert got.keys() == want.keys()
    differ = sorted(k for k in want if got[k] != want[k])
    assert not differ, "encoded bytes changed for: " + ", ".join(differ)
