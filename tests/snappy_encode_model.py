"""A plain numpy restatement of the GPU Snappy compressor (hap_b200/csrc/snappy_encode.cuh, compress_fragment) and of the frame
layout the plan kernel writes around its streams (hap_assemble.cuh, hap_host.h, hap_index.h), without the kernels' thread
mapping: every step works on whole-fragment arrays.  Test-only; it needs no GPU and no library.

A fragment is up to 32 768 bytes of a chunk, read as U 8-byte little-endian units (x, y):
  1. hash     h = ((x * 0x9E3779B1) ^ (y * 0x85EBCA6B)) mod 2^32 >> 19; table[h] = the lowest unit index with that hash
  2. dd[i] = i - c when c = table[h[i]] < i and unit c equals unit i, else 0
  3. block repeats: period 1 (DXT1, RGTC1) dd[i] = 1 when unit i equals unit i - 1; period 2 (DXT5, YCoCg, BC7, BC6H) for even
     i >= 2 with i + 1 < U, dd[i] = dd[i + 1] = 2 when both units of the pair equal the pair before
  4. one propagation round from the values before it (l = dd[i - 1], r = dd[i + 1], 0 at the fragment's ends): a unit that is
     not already dd != 0 with dd == l or dd == r takes cand = l (r when l is 0) if i >= cand and the data match there, else r
     when l != 0, r != 0, r != l and the data match there
  5. every maximal run of equal dd is one literal (dd 0, 8 * len bytes) or copy-2 elements of 8 * min(8, left) bytes at offset
     8 * dd
  6. an index entry per 128 bytes of the stream: offset of the first element start inside it, 0xFF for none
`encode_frame` lays the fragments' streams out into whole Hap frames as the plan kernel does.  Every fragment's trace
(the arrays after each step, the runs, the stream and its entries) is kept for diagnostics and coverage checks."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

FRAG_BYTES = 32768
FRAG_UNITS = FRAG_BYTES // 8
HASH_BITS = 13
SUB_LOG2 = 7
NO_ENTRY = 0xFF
U24_MAX = 0xFFFFFF
MAX_CHUNKS = 3355431

FMT_DXT1, FMT_DXT5, FMT_YCOCG, FMT_RGTC1 = 0x83F0, 0x83F3, 0x01, 0x8DBB
FMT_BC7, FMT_BC6U, FMT_BC6S = 0x8E8C, 0x8E8F, 0x8E8E
NIBBLE = {FMT_DXT1: 0xB, FMT_DXT5: 0xE, FMT_YCOCG: 0xF, FMT_RGTC1: 0x1, FMT_BC7: 0xC, FMT_BC6U: 0x2, FMT_BC6S: 0x3}
RAW, SNAPPY, COMPLEX = 0xA, 0xB, 0xC


def period_units(fmt: int) -> int:
    """block size in 8-byte units"""
    return 1 if fmt in (FMT_DXT1, FMT_RGTC1) else 2


def unit_hash(u: np.ndarray) -> np.ndarray:
    x = (u & 0xFFFFFFFF).astype(np.uint64)
    y = (u >> np.uint64(32)).astype(np.uint64)
    m = np.uint64(0xFFFFFFFF)
    return ((((x * np.uint64(0x9E3779B1)) & m) ^ ((y * np.uint64(0x85EBCA6B)) & m)) >> np.uint64(32 - HASH_BITS)).astype(np.int64)


def literal_header(nbytes: int) -> bytes:
    m = nbytes - 1
    if nbytes <= 60:
        return bytes([m << 2])
    if nbytes <= 256:
        return bytes([60 << 2, m])
    return bytes([61 << 2, m & 0xFF, m >> 8])


def varint(v: int) -> bytes:
    out = bytearray()
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)
    return bytes(out)


@dataclass
class FragmentTrace:
    units: np.ndarray            # uint64 [U]
    period: int
    h: np.ndarray                # step 1: hash per unit
    first: np.ndarray            # step 1: table[h[i]] per unit
    dd2: np.ndarray              # after step 2
    dd3: np.ndarray              # after step 3
    dd4: np.ndarray              # after step 4
    prop: np.ndarray             # step 4: 0 unchanged, 1 took l, 2 took r as first choice (l == 0), 3 took r as second choice
    runs: list                   # step 5: [(first unit, units, dd)]
    elements: list               # [(stream offset, kind "lit" | "copy", bytes of output, offset)]
    stream: bytes
    entries: list                # step 6: one per 128 stream bytes

    @property
    def U(self):
        return len(self.units)


def compress_fragment(frag: bytes, period: int) -> FragmentTrace:
    assert len(frag) % 8 == 0 and 0 < len(frag) <= FRAG_BYTES
    u = np.frombuffer(frag, dtype="<u8").astype(np.uint64)
    U = len(u)
    idx = np.arange(U, dtype=np.int64)
    # 1
    h = unit_hash(u)
    table = np.full(1 << HASH_BITS, U, dtype=np.int64)
    np.minimum.at(table, h, idx)
    first = table[h]
    # 2
    dd = np.where((first < idx) & (u[first] == u), idx - first, 0).astype(np.int64)
    dd2 = dd.copy()
    # 3
    if period == 1:
        rep = np.zeros(U, bool)
        rep[1:] = u[1:] == u[:-1]
        dd[rep] = 1
    else:
        for i in range(2, U - 1, 2):
            if u[i] == u[i - 2] and u[i + 1] == u[i - 1]:
                dd[i] = dd[i + 1] = 2
    dd3 = dd.copy()
    # 4
    l = np.concatenate([[0], dd3[:-1]])
    r = np.concatenate([dd3[1:], [0]])
    keep = (dd3 != 0) & ((dd3 == l) | (dd3 == r))
    cand = np.where(l != 0, l, r)

    def match(dist):
        ok = (dist != 0) & (idx >= dist)
        src = np.where(ok, idx - dist, 0)
        return ok & (u[src] == u)

    first_ok = ~keep & match(cand)
    second_ok = ~keep & ~first_ok & (l != 0) & (r != 0) & (r != l) & match(r)
    dd4 = dd3.copy()
    dd4[first_ok] = cand[first_ok]
    dd4[second_ok] = r[second_ok]
    prop = np.zeros(U, np.int8)
    prop[first_ok & (l != 0)] = 1
    prop[first_ok & (l == 0)] = 2
    prop[second_ok] = 3
    # 5 and 6
    starts = np.flatnonzero(np.concatenate([[True], dd4[1:] != dd4[:-1]]))
    ends = np.concatenate([starts[1:], [U]])
    runs, elements, out = [], [], bytearray()
    for s, e in zip(starts.tolist(), ends.tolist()):
        d = int(dd4[s])
        runs.append((s, e - s, d))
        if d == 0:
            n = 8 * (e - s)
            elements.append((len(out), "lit", n, 0))
            out += literal_header(n) + frag[8 * s: 8 * e]
        else:
            for i in range(s, e, 8):
                n = 8 * min(8, e - i)
                elements.append((len(out), "copy", n, 8 * d))
                out += bytes([2 | ((n - 1) << 2), (8 * d) & 0xFF, (8 * d) >> 8])
    entries = [NO_ENTRY] * ((len(out) + (1 << SUB_LOG2) - 1) >> SUB_LOG2)
    for p, *_ in elements:
        if entries[p >> SUB_LOG2] == NO_ENTRY:
            entries[p >> SUB_LOG2] = p & ((1 << SUB_LOG2) - 1)
    return FragmentTrace(u, period, h, first, dd2, dd3, dd4, prop, runs, elements, bytes(out), entries)


# ---- frames ----------------------------------------------------------------------------------------------------------------

def limited_chunk_count(nbytes: int, fmt: int, k: int) -> int:
    k = min(k, MAX_CHUNKS)
    blocks = nbytes // (8 if period_units(fmt) == 1 else 16)
    while blocks % k:
        k -= 1
    return k


def section_header(hdr: int, length: int, typ: int) -> bytes:
    if hdr == 4:
        return length.to_bytes(3, "little") + bytes([typ])
    return b"\0\0\0" + bytes([typ]) + length.to_bytes(4, "little")


@dataclass
class ChunkPlan:
    texture: int
    chunk: int
    chunk_bytes: int
    fragments: list              # FragmentTrace per fragment, [] when the section is not compressed
    packed: int = 0              # varint + the fragments' streams
    snappy: bool = False         # stored as Snappy (packed < chunk_bytes)
    frag_at: list = field(default_factory=list)    # frame offset of every fragment's stream (Snappy chunks)
    entries_at: list = field(default_factory=list)  # frame offset of every fragment's entries (indexed chunks)


@dataclass
class SectionPlan:
    fmt: int
    nbytes: int
    chunks: int
    chunk_bytes: int
    top_hdr: int
    compress: bool
    want_snappy: bool
    body: int = 0                # would-be complex body length (0 without Snappy)
    complex: bool = False
    chunk_plans: list = field(default_factory=list)


@dataclass
class FramePlan:
    frame: bytes
    sections: list


def section_geometry(nbytes, fmt, compressor, chunks):
    top_hdr = 8 if nbytes > U24_MAX else 4
    k = limited_chunk_count(nbytes, fmt, chunks)
    want = compressor == 1
    if want and nbytes + 5 * k + 8 + 4 > U24_MAX:
        top_hdr = 8
    cb = nbytes // k
    if cb == 0:
        k, cb = 1, nbytes
    return SectionPlan(fmt, nbytes, k, cb, top_hdr, want and cb % 8 == 0, want)


def encode_frame(textures, index=False, offsets=False, cache=None) -> FramePlan:
    """textures: [(bytes, format, compressor, requested chunks)], one or two.  index: the trailing fragment index section;
    offsets: the Chunk Offset Table with 16-byte aligned chunks.  cache: optional dict of fragment traces by (bytes, period)."""
    assert len(textures) in (1, 2)
    secs = [section_geometry(len(t[0]), t[1], t[2], t[3]) for t in textures]
    outer = 0
    if len(textures) == 2:
        worst = sum(len(t[0]) + 5 * t[3] + 8 + 4 for t in textures)
        outer = 8 if worst > U24_MAX else 4
    # fragments and the per-section decisions (pass 1)
    rec_total, sec_off, running = [0, 0], [0, 0], outer
    for si, (s, t) in enumerate(zip(secs, textures)):
        data = t[0]
        per = period_units(s.fmt)
        for c in range(s.chunks):
            cp = ChunkPlan(si, c, s.chunk_bytes, [])
            base = c * s.chunk_bytes
            if s.compress:
                for j in range(0, s.chunk_bytes, FRAG_BYTES):
                    frag = data[base + j: base + min(j + FRAG_BYTES, s.chunk_bytes)]
                    key = (frag, per)
                    if cache is not None and key in cache:
                        tr = cache[key]
                    else:
                        tr = compress_fragment(frag, per)
                        if cache is not None:
                            cache[key] = tr
                    cp.fragments.append(tr)
                cp.packed = len(varint(s.chunk_bytes)) + sum(len(f.stream) for f in cp.fragments)
                cp.snappy = cp.packed < s.chunk_bytes
            s.chunk_plans.append(cp)
        if s.want_snappy:
            sizes = [cp.packed if cp.snappy else s.chunk_bytes for cp in s.chunk_plans]
            if offsets:
                sizes = [(z + 15) & ~15 for z in sizes[:-1]] + sizes[-1:]
            di = 5 * s.chunks + 8 + (4 * s.chunks + 4 if offsets else 0)
            s.body = sum(sizes) + 4 + di
            if offsets:
                s.body += (16 - ((running + s.top_hdr + 4 + di) & 15)) & 15
            s.complex = s.body < s.nbytes + s.top_hdr and s.body < 1 << 31
        if s.complex and index and s.compress:
            rec_total[si] = sum(2 * len(cp.fragments) + sum(len(f.entries) for f in cp.fragments)
                                for cp in s.chunk_plans if cp.snappy)
        sec_off[si] = running
        running += s.top_hdr + (s.body if s.complex else s.nbytes)
    frame_end = running
    k0, k1 = secs[0].chunks, secs[1].chunks if len(secs) == 2 else 0
    index_len = 20 + 4 * (k0 + k1) + sum(rec_total) if sum(rec_total) else 0
    index_hdr = 0 if not index_len else 8 if index_len > U24_MAX else 4
    out = bytearray(frame_end + index_hdr + index_len)
    ibody = frame_end + index_hdr
    if index_len:
        out[frame_end: ibody] = section_header(index_hdr, index_len, 0xFB)
        out[ibody: ibody + 20] = (b"HB2I" + bytes([1, SUB_LOG2, len(secs), 0]) + FRAG_BYTES.to_bytes(4, "little")
                                  + k0.to_bytes(4, "little") + k1.to_bytes(4, "little"))
    # pass 2
    rec_running = 20 + 4 * (k0 + k1)
    for si, (s, t) in enumerate(zip(secs, textures)):
        data, so, hdr, k = t[0], sec_off[si], s.top_hdr, s.chunks
        slots = ibody + 20 + 4 * (k0 if si else 0)
        nib = NIBBLE[s.fmt]
        if not s.complex:
            out[so: so + hdr] = section_header(hdr, s.nbytes, (RAW << 4) | nib)
            out[so + hdr: so + hdr + s.nbytes] = data
            continue
        di = 5 * k + 8 + (4 * k + 4 if offsets else 0)
        p = so + hdr
        ctab, stab = p + 8, p + 8 + k + 4
        otab = stab + 4 * k + 4
        out[so: p] = section_header(hdr, s.body, (COMPLEX << 4) | nib)
        out[p: p + 4] = section_header(4, di, 0x01)
        out[p + 4: p + 8] = section_header(4, k, 0x02)
        out[ctab + k: ctab + k + 4] = section_header(4, 4 * k, 0x03)
        if offsets:
            out[stab + 4 * k: stab + 4 * k + 4] = section_header(4, 4 * k, 0x04)
        data0 = p + 4 + di
        at = (data0 + 15) & ~15 if offsets else data0
        for c, cp in enumerate(s.chunk_plans):
            sz = cp.packed if cp.snappy else s.chunk_bytes
            out[ctab + c] = SNAPPY if cp.snappy else RAW
            out[stab + 4 * c: stab + 4 * c + 4] = sz.to_bytes(4, "little")
            if offsets:
                out[otab + 4 * c: otab + 4 * c + 4] = (at - data0).to_bytes(4, "little")
            rec = cp.snappy and rec_total[si] > 0
            if index_len:
                out[slots + 4 * c: slots + 4 * c + 4] = (rec_running if rec else 0).to_bytes(4, "little")
            if cp.snappy:
                v = varint(s.chunk_bytes)
                out[at: at + len(v)] = v
                o = at + len(v)
                eo = ibody + rec_running + 2 * len(cp.fragments)
                for j, f in enumerate(cp.fragments):
                    out[o: o + len(f.stream)] = f.stream
                    cp.frag_at.append(o)
                    o += len(f.stream)
                    if rec:
                        out[ibody + rec_running + 2 * j: ibody + rec_running + 2 * j + 2] = len(f.stream).to_bytes(2, "little")
                        out[eo: eo + len(f.entries)] = bytes(f.entries)
                        cp.entries_at.append(eo)
                        eo += len(f.entries)
                if rec:
                    rec_running = eo - ibody
            else:
                out[at: at + s.chunk_bytes] = data[c * s.chunk_bytes: (c + 1) * s.chunk_bytes]
            at += (sz + 15) & ~15 if offsets and c + 1 < k else sz
    if len(secs) == 2:
        out[:outer] = section_header(outer, frame_end - outer, 0x0D)
    return FramePlan(bytes(out), secs)


# ---- diagnostics -----------------------------------------------------------------------------------------------------------

def stream_distances(stream: bytes, U: int):
    """the distance per unit a fragment stream implies (literal 0, copy offset / 8), or None when it is not made of whole units"""
    import snappy_corpus as sc
    dd, runs = [], []
    try:
        for _, _, n, kind, length, off in sc.parse_elements(stream):
            if n % 8 or (kind and off % 8):
                return None, None
            runs.append((len(dd), n // 8, 0 if kind == 0 else off // 8))
            dd += [0 if kind == 0 else off // 8] * (n // 8)
    except sc.SnappyError:
        return None, None
    return (np.array(dd, np.int64) if len(dd) == U else None), runs


def explain_fragment(tr: FragmentTrace, got_stream: bytes, got_entries=None) -> str:
    """Which rule step the device's fragment stream (and entries) first departs from: the distances its elements imply are
    compared unit by unit with the model's after steps 2, 3 and 4, then the element split, the bytes and the entries."""
    if got_stream == tr.stream:
        if got_entries is not None and list(got_entries) != tr.entries:
            q = next(i for i, (a, b) in enumerate(zip(list(got_entries), tr.entries)) if a != b)
            return f"step 6 (index entries): entry {q} is {got_entries[q]}, the model's is {tr.entries[q]}"
        return "fragment stream and entries agree"
    dd, runs = stream_distances(got_stream, tr.U)
    if dd is None:
        return (f"step 5 (elements): the stream ({len(got_stream)} bytes, model {len(tr.stream)}) does not cover the fragment's "
                f"{tr.U} units in whole units")
    if not np.array_equal(dd, tr.dd4):
        i = int(np.flatnonzero(dd != tr.dd4)[0])
        where = f"unit {i} of {tr.U}: device distance {dd[i]}, model {tr.dd4[i]}"
        facts = (f"(step 2 gave {tr.dd2[i]}, step 3 {tr.dd3[i]}, step 4 {tr.dd4[i]}; "
                 f"l={tr.dd3[i - 1] if i else 0} r={tr.dd3[i + 1] if i + 1 < tr.U else 0}, first occurrence {tr.first[i]})")
        d = int(dd[i])
        if tr.dd4[i] != tr.dd3[i] or d == tr.dd3[i] or _neighbour_dist(tr, i, d):
            step = "step 4 (propagation)"        # the model's value came from the round, or the device's from a neighbour
        elif tr.dd3[i] != tr.dd2[i] or d == tr.period:
            step = "step 3 (block repeat)"
        else:
            step = "step 2 (candidate distance)"
        return f"{step}: {where} {facts}"
    model_runs = []
    for off, kind, n, o in tr.elements:
        model_runs.append((kind, n, o))
    got = [("lit" if d == 0 else "copy", 8 * n, 8 * d) for _, n, d in runs]
    if got != model_runs:
        q = next((i for i, (a, b) in enumerate(zip(got, model_runs)) if a != b), min(len(got), len(model_runs)))
        return f"step 5 (run split): element {q} is {got[q] if q < len(got) else None}, the model's is " \
               f"{model_runs[q] if q < len(model_runs) else None}"
    q = next((i for i, (a, b) in enumerate(zip(got_stream, tr.stream)) if a != b), min(len(got_stream), len(tr.stream)))
    return f"step 5 (element bytes): byte {q} of the stream differs (literal header or copy tag)"


def _neighbour_dist(tr, i, d):
    return (i and tr.dd3[i - 1] == d) or (i + 1 < tr.U and tr.dd3[i + 1] == d)


def explain_frame(plan: FramePlan, got: bytes) -> str:
    """The first fragment whose stream or entries differ between the device's frame and the model's, with the step that
    breaks; else the first differing byte of the frame layout."""
    if got == plan.frame:
        return "frames agree"
    for s in plan.sections:
        for cp in s.chunk_plans:
            if not cp.snappy:
                continue
            for j, (f, at) in enumerate(zip(cp.fragments, cp.frag_at)):
                g = got[at: at + len(f.stream)]
                ge = None
                if cp.entries_at:
                    e = cp.entries_at[j]
                    ge = got[e: e + len(f.entries)]
                if g != f.stream or (ge is not None and list(ge) != f.entries):
                    # the device's own stream for this fragment runs to the next fragment's start as the device placed it
                    gs = _device_fragment(got, at, f)
                    return (f"texture {cp.texture} chunk {cp.chunk} fragment {j} ({f.U} units, period {f.period}): "
                            + explain_fragment(f, gs, ge))
    q = next((i for i, (a, b) in enumerate(zip(got, plan.frame)) if a != b), min(len(got), len(plan.frame)))
    return f"frame layout: {len(got)} bytes (model {len(plan.frame)}), first difference at byte {q}"


def _device_fragment(got: bytes, at: int, f: FragmentTrace) -> bytes:
    """the elements of the device's frame from `at` that produce the fragment's 8 * U bytes"""
    import snappy_corpus as sc
    want, n, end = 8 * f.U, 0, at
    try:
        for start, enc, out, *_ in sc.parse_elements(got, at):
            if n >= want:
                break
            n += out
            end = start + enc
    except sc.SnappyError:
        pass
    return got[at: end]
