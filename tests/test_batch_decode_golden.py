"""The batch decode path (HapB200DecodeBatch: hap_parse_frames_kernel, the chunk pipeline, hap_collect_status_kernel) on the
golden frames of the unmodified reference: the same result codes, formats and output bytes as the reference.  On the GPU
through the library, and on CPU under the fiber SIMT emulator (tests/emu/test_parse_emu.cc), also under AddressSanitizer.
test_gpu_parity.py checks the same frames through HapDecode."""
import os
import subprocess

import pytest

from golden_util import b64, golden, kat_c_bytes, sha

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "tests", "emu", "_build")
INC = ["-I", os.path.join(ROOT, "hap_b200", "csrc"), "-I", os.path.join(ROOT, "tests", "emu")]
MAX_CHUNKS = 64


def snappy_stream_frames(s):
    """The two frames golden_util.container_checks decodes a raw Snappy stream from: the stream as a whole 0xBE section,
    and as the one chunk of a Complex 0xCE section."""
    n = len(s)
    whole = (n.to_bytes(3, "little") + b"\xbe" + s) if n else (b"\0\0\0\xbe" + (0).to_bytes(4, "little"))
    di = b"\x01\0\0\x02\x0b" + b"\x04\0\0\x03" + n.to_bytes(4, "little")
    body = len(di).to_bytes(3, "little") + b"\x01" + di + s
    return whole, len(body).to_bytes(3, "little") + b"\xce" + body


def golden_frames():
    """(name, frame, texture index, output capacity, (result, format, sha256 of the output)) for every decode case of
    golden_util.container_checks whose texture index the batch entry point takes (it refuses index 2 for the whole call).
    format is None where the golden data does not pin it, the hash None where the reference failed."""
    G = golden()
    out = []
    for key in ("kat_a", "kat_a_none"):
        out.append((key, bytes.fromhex(G[key]["frame"]), 0, 64, (0, 0x83F0, sha(bytes([0x55]) * 64))))
    f = bytes.fromhex(G["kat_d"]["frame"])
    out.append(("kat_d.tex0", f, 0, 4096, (0, 0x01, sha(kat_c_bytes(4096)))))
    out.append(("kat_d.tex1", f, 1, 2048, (0, 0x8DBB, sha(bytes([0x55]) * 2048))))
    for name, e in G["ref_frames"].items():
        fr = b64(e["frame_b64"])
        if name == "hapm":
            for i in (0, 1):
                out.append((f"ref_frames.hapm[{i}]", fr, i, e["payload_len"][i], (0, None, e["payload_sha256"][i])))
        else:
            out.append((f"ref_frames.{name}", fr, 0, e["payload_len"], (0, e["format"], e["payload_sha256"])))
    for name, e in G["snappy_streams"].items():
        whole, cx = snappy_stream_frames(bytes.fromhex(e["stream"]))
        for kind, fr, w in (("whole", whole, e["whole_section"]), ("complex", cx, e["complex_1chunk"])):
            out.append((f"snappy.{name}.{kind}", fr, 0, 4096, (w["result"], None, w["out_sha256"])))
    for name, e in G["container_cases"].items():
        if e["index"] <= 1:
            ok = e["result"] == 0
            out.append((f"case.{name}", bytes.fromhex(e["frame"]), e["index"], e["cap"],
                        (e["result"], e["format"] if ok else None, sha(bytes.fromhex(e["out"])) if ok else None)))
    return out


def mismatches(results):
    """results: (result, format, output bytes) per golden_frames() case, in order."""
    bad = []
    for (name, _, _, _, want), (r, fmt, data) in zip(golden_frames(), results):
        got = (r, fmt if want[1] is not None else None, sha(data) if r == 0 else None)
        if got != want:
            bad.append(f"{name}: got {got!r} want {want!r}")
    return bad


@pytest.mark.gpu
def test_batch_decode_of_the_golden_frames():
    import torch

    import hap_b200
    lib = hap_b200.load()
    results = []
    for _, frame, index, cap, _ in golden_frames():
        dev = torch.tensor(list(frame), dtype=torch.uint8, device="cuda")
        nbytes = torch.tensor([len(frame)], dtype=torch.int64, device="cuda")
        out = torch.zeros(max(cap, 1), dtype=torch.uint8, device="cuda")
        used = torch.zeros(1, dtype=torch.int64, device="cuda")
        fmt = torch.zeros(1, dtype=torch.int32, device="cuda")
        res = torch.full((1,), 99, dtype=torch.int32, device="cuda")
        r = lib.decode_batch(dev.data_ptr(), 1, len(frame), nbytes.data_ptr(), index, MAX_CHUNKS, out.data_ptr(), cap, used.data_ptr(),
                             fmt.data_ptr(), res.data_ptr())
        r = r or int(res[0])
        results.append((r, int(fmt[0]), out[: int(used[0])].cpu().numpy().tobytes() if r == 0 else None))
    assert mismatches(results) == []


@pytest.mark.parametrize("asan", [False, True])
def test_batch_decode_of_the_golden_frames_emulated(asan):
    os.makedirs(BUILD, exist_ok=True)
    exe = os.path.join(BUILD, "test_parse_emu" + ("_asan" if asan else ""))
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-w"] + (["-fsanitize=address"] if asan else []) + INC +
                   [os.path.join(ROOT, "tests", "emu", "test_parse_emu.cc"), "-ldl", "-lm", "-o", exe], check=True)
    with open(exe + ".cases", "w") as fh:
        fh.writelines(f"{index} {cap} {frame.hex()}\n" for _, frame, index, cap, _ in golden_frames())
    env = dict(os.environ, ASAN_OPTIONS="detect_stack_use_after_return=0:detect_leaks=0")
    p = subprocess.run([exe, exe + ".cases", exe + ".results"], capture_output=True, text=True, timeout=900, env=env)
    assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
    results = []
    with open(exe + ".results") as fh:
        for line in fh:
            r, fmt, *data = line.split()
            results.append((int(r), int(fmt), bytes.fromhex(data[0] if data else "")))
    assert len(results) == len(golden_frames())
    assert mismatches(results) == []
