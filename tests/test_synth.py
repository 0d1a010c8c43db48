import zlib

import torch

from hap_b200 import synth


def test_video_frame_is_pinned():
    f = synth.frame(512, 512, 0)
    assert f.shape == (512, 512, 4) and f.dtype == torch.uint8
    assert zlib.crc32(f.numpy().tobytes()) == 954759326
    assert (f[:51] == torch.tensor([16, 16, 16, 255], dtype=torch.uint8)).all()


def test_kinds():
    assert (synth.frame(8, 8, 0, kind="flat") == torch.tensor([0x33, 0x66, 0x99, 0xFF], dtype=torch.uint8)).all()
    n = synth.frame(64, 64, 1, kind="noise")
    assert n[..., :3].float().std() > 60
    a = synth.frame(64, 64, 0, alpha="ramp")
    assert a[..., 3].min() < 10 and a[..., 3].max() == 255
    assert not torch.equal(synth.frame(64, 64, 0), synth.frame(64, 64, 1))


def test_row_bands_equal_the_whole_frame():
    for kind in ("video", "flat", "noise", "gradient", "texture", "edges"):
        whole = synth.frame(96, 80, 2, kind=kind, alpha="ramp" if kind != "noise" else "opaque")
        bands = [synth.frame(96, 80, 2, kind=kind, alpha="ramp" if kind != "noise" else "opaque", rows=(y, min(y + 24, 80)))
                 for y in range(0, 80, 24)]
        assert torch.equal(torch.cat(bands), whole), kind
