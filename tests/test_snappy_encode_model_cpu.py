"""The numpy model of the GPU Snappy compressor (snappy_encode_model.py) against the compressor itself, run under the fiber SIMT
emulator (tests/emu/encode_frames_emu.cc: K5 + plan + place, as the library launches them), on the corpus of
snappy_encode_corpus.py.  The model's frames are also judged on their own: they decode through the CPU oracle and the
reference build (oracle/_ref, when it is built) to their textures, no copy reads outside its fragment, and the trailing
index equals an independent walk of every chunk stream.  So the GPU tests (test_gpu_snappy_encode.py) can hold the device to
the model byte for byte."""
import os
import struct
import subprocess
import tempfile

import numpy as np
import pytest

import oracles
import snappy_corpus as sc
import snappy_encode_corpus as ec
import snappy_encode_model as m
from test_kernels_emulated import compile_emu

OPTIONS = (0, 1, 2, 3)   # bit 0: fragment index, bit 1: chunk offset table


@pytest.fixture(scope="module")
def corpus():
    return ec.corpus()


@pytest.fixture(scope="module")
def models(corpus):
    cache = {}
    return {(e.name, o): m.encode_frame(e.textures, index=bool(o & 1), offsets=bool(o & 2), cache=cache)
            for e in corpus for o in OPTIONS}


def run_emulated(cases, mode, grid):
    """cases: [(textures, options)] -> the emulated kernels' frames"""
    exe = compile_emu("encode_frames_emu", [])
    with tempfile.TemporaryDirectory() as d:
        fin, fout = os.path.join(d, "in"), os.path.join(d, "out")
        with open(fin, "wb") as f:
            for textures, opts in cases:
                f.write(struct.pack("<II", opts, len(textures)))
                for data, fmt, comp, chunks in textures:
                    f.write(struct.pack("<IIII", fmt, comp, chunks, len(data)) + data)
        p = subprocess.run([exe, fin, fout, str(mode), str(grid)], capture_output=True, text=True, timeout=1200)
        assert p.returncode == 0, p.stdout + p.stderr
        blob = open(fout, "rb").read()
    frames, pos = [], 0
    while pos < len(blob):
        n = struct.unpack_from("<I", blob, pos)[0]
        frames.append(blob[pos + 4: pos + 4 + n])
        pos += 4 + n
    assert len(frames) == len(cases)
    return frames


@pytest.mark.parametrize("mode,grid,options", [(0, 1, OPTIONS), (2, 3, (1, 3))])
def test_model_equals_emulated_kernel(corpus, models, mode, grid, options):
    """every corpus texture in every option, under two fiber resume orders and persistent-grid sizes"""
    cases = [(e, o) for e in corpus for o in options]
    frames = run_emulated([(e.textures, o) for e, o in cases], mode, grid)
    bad = [f"{e.name} options {o}: {m.explain_frame(models[(e.name, o)], fr)}"
           for (e, o), fr in zip(cases, frames) if fr != models[(e.name, o)].frame]
    assert not bad, "\n".join(bad[:20])


def _decoded(textures, i, plan):
    s = plan.sections[i]
    data = textures[i][0]
    return data[: s.chunks * s.chunk_bytes] if s.complex else data


def test_model_frames_decode_to_their_textures(corpus, models):
    judges = [oracles.oracle_abi()] + ([oracles.ref_abi()] if oracles.ref_abi() else [])
    for e in corpus:
        for o in OPTIONS:
            plan = models[(e.name, o)]
            for i in range(len(e.textures)):
                want = _decoded(e.textures, i, plan)
                for j in judges:
                    r, tex, fmt, _ = j.decode(plan.frame, i, len(e.textures[i][0]))
                    assert r == 0 and fmt == e.textures[i][1] and tex == want, (e.name, o, i, j.path)


# ---- an independent walk of the frames ----------------------------------------------------------------------------------------

def _header(b, p):
    n = int.from_bytes(b[p: p + 3], "little")
    if n == 0:
        return 8, int.from_bytes(b[p + 4: p + 8], "little"), b[p + 3]
    return 4, n, b[p + 3]


def texture_sections(frame):
    """[(offset of the section body, length, type)] of the frame's textures, and the end of the frame proper"""
    h, n, t = _header(frame, 0)
    if t != 0x0D:
        return [(h, n, t)], h + n
    out, p = [], h
    while p < h + n:
        hh, nn, tt = _header(frame, p)
        out.append((p + hh, nn, tt))
        p += hh + nn
    return out, h + n


def snappy_chunks(frame, body, length):
    """[(chunk index, stream offset in the frame, stream bytes)] of the Snappy chunks of a complex section"""
    dh, dn, _ = _header(frame, body)
    p, tables = body + dh, {}
    while p < body + dh + dn:
        h, n, t = _header(frame, p)
        tables[t] = frame[p + h: p + h + n]
        p += h + n
    comp = list(tables[0x02])
    sizes = [int.from_bytes(tables[0x03][4 * c: 4 * c + 4], "little") for c in range(len(comp))]
    offs = [int.from_bytes(tables[0x04][4 * c: 4 * c + 4], "little") for c in range(len(comp))] if 0x04 in tables else \
        [sum(sizes[:c]) for c in range(len(comp))]
    data = body + dh + dn
    return len(comp), [(c, data + offs[c], sizes[c]) for c in range(len(comp)) if comp[c] == 0x0B]


def walk_chunk(stream):
    """the chunk's fragments as an element walk sees them: [(stream bytes, element starts)]; asserts that no copy reads before
    its fragment's first byte"""
    total, p = sc.parse_varint(stream)
    frags, out, cur_start, starts = [], 0, p, []
    for start, enc, n, kind, length, off in sc.parse_elements(stream, p):
        frag_out = out - (out // sc.FRAG) * sc.FRAG
        if kind:
            assert off <= frag_out, f"copy at {start} reads {off} back, {frag_out} bytes into its fragment"
        starts.append(start - cur_start)
        out += n
        assert out <= total and (out - 1) // sc.FRAG == (out - n) // sc.FRAG, "element crosses a fragment boundary"
        if out % sc.FRAG == 0 or out == total:
            frags.append((start + enc - cur_start, starts))
            cur_start, starts = start + enc, []
    assert out == total
    return frags


def test_copies_stay_in_their_fragments_and_the_index_matches_a_walk(corpus, models):
    for e in corpus:
        for o in (1, 3):
            frame = models[(e.name, o)].frame
            secs, end = texture_sections(frame)
            walked = {}
            counts = [0, 0]
            for i, (body, length, typ) in enumerate(secs):
                if typ >> 4 != 0xC:
                    counts[i] = m.limited_chunk_count(length, e.textures[i][1], e.textures[i][3])
                    continue
                counts[i], chunks = snappy_chunks(frame, body, length)
                for c, at, size in chunks:
                    walked[(i, c)] = walk_chunk(frame[at: at + size])
            if end == len(frame):
                assert not walked or e.textures[0][2] == 0, (e.name, o, "no index section")
                continue
            h, n, t = _header(frame, end)
            assert t == 0xFB and end + h + n == len(frame)
            ib = frame[end + h:]
            assert ib[:8] == b"HB2I\x01\x07" + len(secs).to_bytes(2, "little")
            k = [int.from_bytes(ib[12 + 4 * q: 16 + 4 * q], "little") for q in range(2)]
            assert k[0] == counts[0] and k[1] == (counts[1] if len(secs) == 2 else 0), (e.name, o)
            seen = 0
            for i in range(len(secs)):
                for c in range(k[i]):
                    off = int.from_bytes(ib[20 + 4 * (c + (k[0] if i else 0)): 24 + 4 * (c + (k[0] if i else 0))], "little")
                    if (i, c) not in walked:
                        assert off == 0, (e.name, o, i, c)
                        continue
                    seen += 1
                    frags = walked[(i, c)]
                    nf = len(frags)
                    sizes = [int.from_bytes(ib[off + 2 * j: off + 2 * j + 2], "little") for j in range(nf)]
                    assert sizes == [s for s, _ in frags], (e.name, o, i, c)
                    p = off + 2 * nf
                    for s, starts in frags:
                        ent = list(ib[p: p + (s + sc.SUB - 1) // sc.SUB])
                        assert ent == sc.fragment_entries(starts, s), (e.name, o, i, c)
                        p += len(ent)
            assert seen == len(walked)


# ---- coverage -----------------------------------------------------------------------------------------------------------------

def features(plan, textures):
    """what the model's trace of a frame shows, as a set of names"""
    got = set()
    for s, t in zip(plan.sections, textures):
        for cp in s.chunk_plans:
            d = cp.packed - s.chunk_bytes if cp.fragments else None
            if d in (-1, 0, 1):
                got.add(f"chunk_stream_{d:+d}")
            for f in cp.fragments:
                got |= fragment_features(f)
        if s.want_snappy:
            d = s.body - (s.nbytes + s.top_hdr)
            if d in (-1, 0, 1):
                got.add(f"texture_body_{d:+d}")
        if not s.compress:
            got.add("not_compressed")
        if s.compress and s.chunk_bytes % 16:
            got.add("chunk_bytes_8_mod_16")
    return got


def fragment_features(f):
    got = {f"U{f.U}"} if f.U in (1, 2, 7, 8, 9, 255, 256, 257, 4095) else set()
    idx = np.arange(f.U)
    lits = [n // 8 for _, k, n, _ in f.elements if k == "lit"]
    got |= {f"literal_{n}" for n in lits if n <= 40}
    for _, k, n, _ in f.elements:
        if k == "lit":
            got.add("tag60" if 60 < n <= 256 else "tag61" if n > 256 else "tag1")
    if len(f.stream) == 8 * f.U + 3 and f.U == m.FRAG_UNITS:
        got.add("whole_literal_fragment")
    for s, n, d in f.runs:
        if d in (1, 2, 3):
            got.add(f"copy_run_d{d}_{min(n, 18)}")
        if d == m.FRAG_UNITS - 1:
            got.add("copy_offset_32760")
        if d and s + n == f.U:
            got.add("copy_run_at_fragment_end")
    over = f.dd3 != f.dd2
    for p in (1, 2):
        if f.period == p and over.any():
            got.add(f"block_repeat_p{p}")
            if over[idx % 8 == 0].any():
                got.add(f"block_repeat_p{p}_strip")
            if over[idx % 256 == 0].any():
                got.add(f"block_repeat_p{p}_warp")
    if f.period == 2:
        # a pair where only one unit repeats the pair before
        i = np.arange(2, f.U - 1, 2)
        if ((f.units[i] == f.units[i - 2]) != (f.units[i + 1] == f.units[i - 1])).any():
            got.add("half_pair_repeat")
    coll = (f.first < idx) & (f.units[f.first] != f.units)
    if coll.any():
        got.add("collision")
        later = [i for i in np.flatnonzero(coll).tolist() if (f.units[:i] == f.units[i]).any()]
        if later:
            got.add("collision_hides_match")
    same_h = np.concatenate([[False], (f.h[1:] == f.h[:-1]) & (f.units[1:] != f.units[:-1])])
    if (same_h & (idx % 8 == 0)).any():
        got.add("dup_skip_strip")
    if (same_h & (idx % 256 == 0)).any():
        got.add("dup_skip_warp")
    for v, name in ((1, "prop_left"), (2, "prop_right"), (3, "prop_right_second")):
        if (f.prop == v).any():
            got.add(name)
    # the left neighbour's distance taken where the right one's, nonzero and different, would have matched too
    r = np.concatenate([f.dd3[1:], [0]])
    src = np.where((r != 0) & (idx >= r), idx - r, 0)
    if ((f.prop == 1) & (r != 0) & (r != f.dd4) & (idx >= r) & (f.units[src] == f.units)).any():
        got.add("prop_left_over_right")
    return got


REQUIRED = {
    "literal_runs": {f"literal_{n}" for n in range(1, 41)} | {"tag1", "tag60", "tag61", "whole_literal_fragment"},
    "copy_runs": {f"copy_run_d1_{n}" for n in range(1, 18)} | {f"copy_run_d2_{n}" for n in range(2, 18)}
    | {"copy_run_d3_1", "copy_run_d3_3", "copy_offset_32760", "copy_run_at_fragment_end"},
    "block_repeats": {"block_repeat_p1_strip", "block_repeat_p1_warp", "block_repeat_p2_strip", "block_repeat_p2_warp",
                      "half_pair_repeat"},
    "hash_collisions": {"collision", "collision_hides_match", "dup_skip_strip", "dup_skip_warp"},
    "propagation": {"prop_left", "prop_right", "prop_right_second", "prop_left_over_right"},
    "last_fragments": {f"U{u}" for u in (1, 2, 7, 8, 9, 255, 256, 257, 4095)} | {"chunk_bytes_8_mod_16", "not_compressed"},
    "boundaries": {"chunk_stream_-1", "chunk_stream_+0", "chunk_stream_+1", "texture_body_-1", "texture_body_+0",
                   "texture_body_+1"},
    "real": {"prop_left", "collision", "tag61"},
}


def test_corpus_reaches_every_case(corpus, models):
    """for every family, the model's trace shows each feature the family is there for"""
    assert set(REQUIRED) == set(ec.FAMILIES)
    got = {fam: set() for fam in ec.FAMILIES}
    for e in corpus:
        got[e.family] |= features(models[(e.name, 0)], e.textures)
    missing = {fam: sorted(REQUIRED[fam] - got[fam]) for fam in REQUIRED if REQUIRED[fam] - got[fam]}
    assert not missing, missing
