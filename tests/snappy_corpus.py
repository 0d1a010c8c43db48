"""A seeded corpus of raw Snappy streams written element by element, a plain Python decoder of the format, and builders of
the Hap frames (HapVideoDRAFT.md) and trailing fragment indexes (hap_b200/csrc/hap_index.h) that carry them.  Test-only: it
needs no GPU and no library.

An element list is what the writer encodes, with the encoding of every element chosen by the caller:
  ("lit", payload, form)           form None: the shortest tag; 0: the 1-byte tag (payload <= 60 bytes); 60..63: the tag that
                                   stores len - 1 in 1..4 further bytes, also where a shorter form would do (tag 60 for 10 bytes)
  ("copy", length, offset, form)   form 1 (length 4..11, offset < 2048), 2 (length 1..64, offset < 65536) or 4 (length 1..64)
Copies may overlap their own output (offset < length): the bytes repeat with period `offset`."""
from __future__ import annotations

import bisect
import functools
import random

FRAG = 32768            # uncompressed bytes per fragment of the fragment index (hap_index.h)
SUB = 128               # stream bytes per index entry (sub_log2 7)
FRAG_MAX_STREAM = 32800  # the longest fragment stream the decoder takes from an index
NO_ENTRY = 0xFF


class SnappyError(ValueError):
    pass


# ---- writer -----------------------------------------------------------------------------------------------------------

def varint(v: int) -> bytes:
    out = bytearray()
    while True:
        b = v & 0x7F
        v >>= 7
        out.append(b | (0x80 if v else 0))
        if not v:
            return bytes(out)


def lit(payload, form=None):
    return ("lit", bytes(payload), form)


def copy(length, offset, form=None):
    if form is None:
        form = 1 if 4 <= length <= 11 and offset < 2048 else 2 if offset < 65536 else 4
    return ("copy", length, offset, form)


def encode_element(e) -> bytes:
    if e[0] == "lit":
        payload, form = e[1], e[2]
        m = len(payload) - 1
        if m < 0:
            raise ValueError("empty literal")
        if form is None:
            form = 0 if m < 60 else 59 + (m.bit_length() + 7) // 8
        if form == 0:
            if m >= 60:
                raise ValueError("1-byte literal tag holds at most 60 bytes")
            return bytes([m << 2]) + payload
        extra = form - 59
        if not 1 <= extra <= 4 or m >= 1 << (8 * extra):
            raise ValueError(f"literal of {m + 1} bytes in form {form}")
        return bytes([form << 2]) + m.to_bytes(extra, "little") + payload
    _, length, offset, form = e
    if form == 1:
        if not (4 <= length <= 11 and offset < 2048):
            raise ValueError(f"copy-1 of {length} at {offset}")
        return bytes([1 | ((length - 4) << 2) | ((offset >> 8) << 5), offset & 0xFF])
    if not 1 <= length <= 64:
        raise ValueError(f"copy of {length}")
    if form == 2:
        if offset >= 65536:
            raise ValueError(f"copy-2 at {offset}")
        return bytes([2 | ((length - 1) << 2)]) + offset.to_bytes(2, "little")
    return bytes([3 | ((length - 1) << 2)]) + offset.to_bytes(4, "little")


def element_output(e) -> int:
    return len(e[1]) if e[0] == "lit" else e[1]


def write_stream(elements, declared=None) -> bytes:
    """varint(declared, default: what the elements produce) followed by the encoded elements"""
    body = b"".join(encode_element(e) for e in elements)
    if declared is None:
        declared = sum(element_output(e) for e in elements)
    return varint(declared) + body


# ---- the plain decoder ------------------------------------------------------------------------------------------------

def parse_varint(s: bytes):
    """(value, bytes used); SnappyError unless it is a varint32 (at most 5 bytes, the 5th < 16)"""
    v = 0
    for i in range(5):
        if i >= len(s):
            raise SnappyError("preamble cut off")
        b = s[i]
        if i == 4 and b > 15:
            raise SnappyError("preamble overflows 32 bits")
        v |= (b & 0x7F) << (7 * i)
        if not b & 0x80:
            return v, i + 1
    raise SnappyError("preamble overflows 32 bits")


def parse_elements(s: bytes, pos: int = 0, end: int | None = None):
    """Yields (start, encoded bytes, output bytes, kind, length, offset-or-payload position) for each element of s[pos:end]."""
    end = len(s) if end is None else end
    while pos < end:
        tag = s[pos]
        kind = tag & 3
        if kind == 0:
            m = tag >> 2
            hdr = 1
            if m >= 60:
                extra = m - 59
                if pos + 1 + extra > end:
                    raise SnappyError("literal header cut off")
                m = int.from_bytes(s[pos + 1: pos + 1 + extra], "little")
                hdr += extra
            n = m + 1
            if pos + hdr + n > end:
                raise SnappyError("literal runs past the input")
            yield pos, hdr + n, n, 0, n, pos + hdr
            pos += hdr + n
            continue
        hdr = 2 if kind == 1 else 3 if kind == 2 else 5
        if pos + hdr > end:
            raise SnappyError("copy header cut off")
        if kind == 1:
            length, off = 4 + ((tag >> 2) & 7), ((tag >> 5) << 8) | s[pos + 1]
        else:
            length, off = (tag >> 2) + 1, int.from_bytes(s[pos + 1: pos + hdr], "little")
        yield pos, hdr, length, kind, length, off
        pos += hdr


def decode(s: bytes) -> bytes:
    """A raw Snappy stream -> its bytes, or SnappyError"""
    s = bytes(s)
    want, pre = parse_varint(s)
    out = bytearray()
    for pos, _, n, kind, length, aux in parse_elements(s, pre):
        if len(out) + n > want:
            raise SnappyError("element runs past the declared length")
        if kind == 0:
            out += s[aux: aux + n]
            continue
        if aux == 0 or aux > len(out):
            raise SnappyError(f"copy offset {aux} with {len(out)} bytes written")
        start = len(out) - aux
        if length <= aux:
            out += out[start: start + length]
        else:   # overlapping: the last `aux` bytes repeat
            period = out[start:]
            out += (period * (length // aux + 1))[:length]
    if len(out) != want:
        raise SnappyError(f"{len(out)} bytes produced, {want} declared")
    return bytes(out)


def stream_stats(elements):
    """what a family promises: max elements starting in any 16 KiB of the stream, longest literal, copy-4 count, expansion
    ratio, the longest chain of copies that read the output of copies (depth), max copy offset"""
    s = write_stream(elements)
    _, pre = parse_varint(s)
    starts = [pre]
    for e in elements[:-1]:
        starts.append(starts[-1] + len(encode_element(e)))
    per_win = {}
    for p in starts:
        per_win[p // 16384] = per_win.get(p // 16384, 0) + 1
    # depth: per output byte range, the copy generation that wrote it (literals 0); a copy is one more than its source's max
    gen = []   # (end, generation) runs of the output
    pos = depth = 0
    ends = []
    for e in elements:
        n = element_output(e)
        if e[0] == "lit":
            g = 0
        else:
            src0, src1 = pos - e[2], pos - e[2] + min(e[1], e[2])
            i = bisect.bisect_right(ends, src0)
            g = 0
            while i < len(ends) and (i == 0 or ends[i - 1] < src1):
                g = max(g, gen[i][1])
                i += 1
            g += 1
        pos += n
        depth = max(depth, g)
        if gen and gen[-1][1] == g:
            gen[-1] = (pos, g)
            ends[-1] = pos
        else:
            gen.append((pos, g))
            ends.append(pos)
    lits = [len(e[1]) for e in elements if e[0] == "lit"]
    copies = [e for e in elements if e[0] == "copy"]
    return {
        "elements": len(elements),
        "max_elems_per_16k": max(per_win.values()),
        "max_literal": max(lits) if lits else 0,
        "copy4": sum(1 for e in copies if e[3] == 4),
        "expansion": pos / max(len(s), 1),
        "depth": depth,
        "max_offset": max((e[2] for e in copies), default=0),
        "reaches_byte0": any(e[2] == p for e, p in zip(elements, _positions(elements)) if e[0] == "copy"),
        "output": pos,
    }


def _positions(elements):
    p = 0
    for e in elements:
        yield p
        p += element_output(e)


# ---- stream families: each a function of (seed, size) -> element list producing exactly `size` bytes -------------------
# Every copy reads only the output of the same list, so a family's list is also a self-contained fragment.

def _rand_bytes(rng, n):
    return rng.randbytes(n)


def _tagish_bytes(rng, n):
    """bytes that mostly parse as long-literal tags (0xF0-0xFC): they drive the index kernel's per-offset sweep into its far
    list and past it"""
    r = rng.getrandbits
    return bytes(0xF0 + r(4) % 13 if r(3) else r(8) for _ in range(n))


def _fill_copy(rng, out, remaining):
    """a short copy (or literal, at the very start) that produces exactly `remaining` (1..64) bytes"""
    if out == 0:
        return lit(_rand_bytes(rng, remaining))
    return copy(remaining, rng.randint(1, min(out, 65535)), 2)


LONG_LITERALS = (1, 60, 61, 256, 16383, 16384, 65536, 65537, 200000)


def fam_long_literals(seed, size):
    rng = random.Random(seed)
    els, out, i = [], 0, 0
    while out < size:
        n = min(LONG_LITERALS[i % len(LONG_LITERALS)], size - out)
        i += 1
        m = n - 1
        forms = [None] + [f for f in (60, 61, 62, 63) if m < 1 << (8 * (f - 59))] + ([0] if m < 60 else [])
        els.append(lit(_tagish_bytes(rng, n), rng.choice(forms)))
        out += n
        if out < size:   # a short copy between literals, so that a literal's end is an element start
            k = min(rng.randint(4, 11), size - out)
            els.append(copy(k, rng.randint(1, min(out, 2047)), 1 if k >= 4 else 2))
            out += k
    return els


def fam_dense(seed, size):
    """2-byte copy-1 elements: ~8 000 element starts per 16 KiB of stream"""
    rng = random.Random(seed)
    first = min(size, 2048)
    els, out = [lit(_rand_bytes(rng, first))], first
    while out < size:
        left = size - out
        if left < 4:
            els.append(_fill_copy(rng, out, left))
            out += left
            break
        k = left if left <= 11 else rng.randint(4, min(11, left - 4))   # what is left after it is 0 or at least 4
        els.append(copy(k, rng.randint(1, min(out, 2047)), 1))
        out += k
    return els


def fam_expanding(seed, size):
    """3-byte copy-2 elements of 64 bytes: ~21x expansion"""
    rng = random.Random(seed)
    first = min(size, 64)
    els, out = [lit(_rand_bytes(rng, first))], first
    while out < size:
        k = min(64, size - out)
        els.append(copy(k, rng.randint(1, min(out, 65535)), 2))
        out += k
    return els


def fam_deep_chains(seed, size, block=8192):
    """periodic runs at periods 1-19 (each copy reads the one before it), then blocks each made of copies of half of the block
    before it: the output of block k depends on every block before it, over many windows"""
    rng = random.Random(seed)
    els, out = [], 0
    for p in range(1, 20):
        if out >= size:
            break
        n = min(p, size - out)
        els.append(lit(_rand_bytes(rng, n)))
        out += n
        run = min(rng.randint(100, 700), size - out)
        while run > 0:
            k = min(run, 64)
            els.append(copy(k, p, 1 if 4 <= k <= 11 else 2))
            out += k
            run -= k
    if out < size:
        n = min(block, size - out)
        els.append(lit(_rand_bytes(rng, n)))
        out += n
    prev = out - block
    while out < size and prev >= 0:
        start = out
        while out < size and out - start < block:
            k = min(64, size - out, block - (out - start))
            src = prev + block // 2 + ((out - start) // 2) % (block // 2 - 64)   # the second half of the previous block
            els.append(copy(k, out - src, 2))
            out += k
        prev = start
    while out < size:
        k = min(64, size - out)
        els.append(_fill_copy(rng, out, k))
        out += k
    return els


def fam_far_copies(seed, size):
    """copy-2 up to offset 65 535, copy-4 beyond it and at small offsets, and copies that reach exactly byte 0"""
    rng = random.Random(seed)
    first = min(size, 4096)
    els, out = [lit(_rand_bytes(rng, first))], first
    while out < size:
        k = min(rng.randint(1, 64), size - out)
        r = rng.random()
        if r < 0.1:
            els.append(copy(k, out, 2 if out < 65536 else 4))        # byte 0 of the chunk
        elif r < 0.25:
            els.append(copy(k, rng.randint(1, min(out, 300)), 4))    # copy-4 at a small offset
        elif out > 65535 and r < 0.7:
            els.append(copy(k, rng.randint(65536, out), 4))
        elif r < 0.8:
            els.append(copy(k, min(out, 65535), 2))                  # the farthest copy-2
        else:
            els.append(copy(k, rng.randint(max(1, min(out, 65535) - 4096), min(out, 65535)), 2))
        out += k
    return els


def fam_mixed(seed, size):
    """random weights over every element kind and encoding"""
    rng = random.Random(seed)
    w = [rng.random() for _ in range(8)]
    els, out = [], 0
    while out < size:
        left = size - out
        kind = rng.choices(range(8), w)[0] if out else 0
        if kind == 0 or (kind == 1 and left < 61):
            n = min(rng.randint(1, 60), left)
            els.append(lit(_rand_bytes(rng, n), rng.choice([None, 0, 60, 61, 62, 63])))
        elif kind == 1:
            n = min(rng.randint(61, 3000), left)
            els.append(lit(_tagish_bytes(rng, n), rng.choice([None, 61, 62, 63])))
        elif kind == 2 and left >= 4:
            n = min(rng.randint(4, 11), left)
            els.append(copy(n, rng.randint(1, min(out, 2047)), 1))
        elif kind == 3:
            n = min(rng.randint(1, 64), left)
            els.append(copy(n, rng.randint(1, min(out, 65535)), 2))
        elif kind == 4:
            n = min(rng.randint(1, 64), left)
            els.append(copy(n, rng.randint(1, out), 4))
        elif kind == 5:   # a periodic run
            p = rng.randint(1, min(out, 19))
            n = min(rng.randint(20, 64), left)
            els.append(copy(n, p, 2))
        elif kind == 6:
            n = min(rng.randint(1, 64), left)
            els.append(copy(n, out, 4 if out > 65535 else 2))
        else:
            n = min(left, 64)
            els.append(copy(n, rng.randint(1, min(out, 65535)), 2))
        out += element_output(els[-1])
    return els


FAMILIES = {
    "long_literals": fam_long_literals,
    "dense": fam_dense,
    "expanding": fam_expanding,
    "deep_chains": fam_deep_chains,
    "far_copies": fam_far_copies,
    "mixed": fam_mixed,
}


# ---- illegal streams: one or more per error class ----------------------------------------------------------------------

def illegal_streams():
    r = random.Random(99)
    head = _rand_bytes(r, 8)
    L = encode_element
    return {
        "offset_zero": varint(12) + L(lit(head)) + bytes([1 | (0 << 2), 0]),
        "offset_zero_copy4": varint(12) + L(lit(head)) + bytes([3 | (3 << 2)]) + (0).to_bytes(4, "little"),
        "offset_beyond_output": varint(16) + L(lit(head)) + L(copy(8, 9, 2)),
        "offset_beyond_output_copy4": varint(70000) + L(lit(head)) + L(copy(64, 65536, 4)),
        "copy_past_declared": varint(20) + L(lit(head)) + L(copy(16, 8, 2)),
        "literal_past_declared": varint(10) + L(lit(_rand_bytes(r, 16))),
        "literal_past_input": varint(32) + bytes([31 << 2]) + _rand_bytes(r, 10),
        "long_literal_past_input": varint(300) + bytes([60 << 2, 255]) + _rand_bytes(r, 200),
        "copy_header_cut": varint(16) + L(lit(head)) + bytes([2 | (7 << 2), 8]),
        "literal_header_cut": varint(400) + L(lit(head)) + bytes([61 << 2, 0x10]),
        "varint_overflow": bytes([0xFF, 0xFF, 0xFF, 0xFF, 0x1F]) + L(lit(head)),
        "varint_six_bytes": bytes([0x88, 0x80, 0x80, 0x80, 0x80, 0x00]) + L(lit(head)),
        "declared_short": varint(8) + L(lit(head)) + L(copy(8, 8, 1)),
        "declared_long": varint(20) + L(lit(head)) + L(copy(8, 8, 1)),
    }


# ---- Hap frames -------------------------------------------------------------------------------------------------------

TEX_DXT1 = 0xB            # texture-format nibble of RGB DXT1 (HapTextureFormat_RGB_DXT1)
RAW, SNAPPY = 0x0A, 0x0B


def section(typ: int, body: bytes, long: bool = False) -> bytes:
    """a section header (4 bytes, or 8 bytes when asked or when the body needs it) and the body"""
    if long or len(body) > 0xFFFFFF:
        return b"\0\0\0" + bytes([typ]) + len(body).to_bytes(4, "little") + body
    return len(body).to_bytes(3, "little") + bytes([typ]) + body


def declared_size(compressor: int, data: bytes) -> int:
    """the decoded size a chunk claims: its bytes (verbatim) or its preamble (Snappy; 0 when unreadable)"""
    if compressor == RAW:
        return len(data)
    try:
        return parse_varint(data)[0]
    except SnappyError:
        return 0


def complex_frame(chunks, offset_table=False, long_headers=False, gap=0, fmt=TEX_DXT1, index=None) -> bytes:
    """A Complex texture section (HapVideoDRAFT.md: Decode Instructions container with the Second-Stage Compressor Table, the
    Chunk Size Table and optionally the Chunk Offset Table, then the chunk data).  chunks: [(compressor, bytes)].  gap: zero
    bytes left between chunks (only with the offset table).  index: a fragment index body to append behind the frame."""
    subs = section(0x02, bytes(c for c, _ in chunks), long_headers)
    subs += section(0x03, b"".join(len(d).to_bytes(4, "little") for _, d in chunks), long_headers)
    data, offs = bytearray(), []
    for _, d in chunks:
        offs.append(len(data))
        data += d
        if offset_table:
            data += bytes(gap)
    if offset_table:
        subs += section(0x04, b"".join(o.to_bytes(4, "little") for o in offs), long_headers)
    body = section(0x01, subs, long_headers) + bytes(data)
    frame = section(0xC0 | fmt, body, long_headers)
    if index is not None:
        frame += section(0xFB, index)
    return frame


def simple_frame(compressor, data, long_header=False, fmt=TEX_DXT1) -> bytes:
    """a texture section of one chunk without Decode Instructions"""
    return section((compressor << 4) | fmt, data, long_header)


def frame_texture(chunks) -> bytes:
    """what a frame of these legal chunks decodes to: the chunks' bytes one after the other"""
    return b"".join(d if c == RAW else decode(d) for c, d in chunks)


# ---- fragment index (hap_index.h) -------------------------------------------------------------------------------------

def fragment_entries(starts, stream_bytes):
    """entry per 128-byte piece: offset of the first element start inside it, 0xFF for none"""
    ent = [NO_ENTRY] * ((stream_bytes + SUB - 1) // SUB)
    for p in starts:
        if ent[p // SUB] == NO_ENTRY:
            ent[p // SUB] = p % SUB
    return ent


class IndexedChunk:
    """A Snappy chunk cut into self-contained 32 KiB fragments: fragments[f] is the element list of output bytes
    [f * 32768, ...), reading only its own output.  The stream is varint(total) + the fragments' streams."""

    def __init__(self, fragments):
        self.fragments = [list(f) for f in fragments]
        self.encoded = [[encode_element(e) for e in f] for f in self.fragments]
        self.output = sum(element_output(e) for f in self.fragments for e in f)
        for i, f in enumerate(self.fragments):
            got = sum(element_output(e) for e in f)
            if got != (FRAG if i + 1 < len(self.fragments) else self.output - FRAG * i):
                raise ValueError(f"fragment {i} produces {got} bytes")
        self.pre = varint(self.output)

    def stream(self) -> bytes:
        return self.pre + b"".join(b"".join(e) for e in self.encoded)

    def true_layout(self):
        """[(stream bytes, element starts)] per fragment, from the element chain"""
        out = []
        for enc in self.encoded:
            starts, p = [], 0
            for e in enc:
                starts.append(p)
                p += len(e)
            if p > FRAG_MAX_STREAM or starts[-1] >= FRAG:
                raise ValueError("fragment stream too long for the index")
            out.append((p, starts))
        return out


def index_record(layout) -> bytes:
    """a chunk's record: u16 stream_bytes[nf], then the entries of every fragment"""
    rec = bytearray(b"".join(s.to_bytes(2, "little") for s, _ in layout))
    for s, starts in layout:
        rec += bytes(fragment_entries(starts, s))
    return bytes(rec)


def index_body(records, chunk_counts=None) -> bytes:
    """records: one per chunk of texture 0 (None: no record); the trailing index body (hap_index.h)"""
    counts = chunk_counts or (len(records), 0)
    head = b"HB2I" + bytes([1, 7]) + (1).to_bytes(2, "little") + FRAG.to_bytes(4, "little")
    head += b"".join(c.to_bytes(4, "little") for c in counts)
    table_end = len(head) + 4 * (counts[0] + counts[1])
    offs, blob = [], bytearray()
    for r in records:
        if r is None:
            offs.append(0)
        else:
            offs.append(table_end + len(blob))
            blob += r
    offs += [0] * (counts[0] + counts[1] - len(offs))
    return head + b"".join(o.to_bytes(4, "little") for o in offs) + bytes(blob)


def _record_entries(rec, nf):
    lens = [int.from_bytes(rec[2 * f: 2 * f + 2], "little") for f in range(nf)]
    ents, p = [], 2 * nf
    for s in lens:
        k = (s + SUB - 1) // SUB
        ents.append(list(rec[p: p + k]))
        p += k
    return lens, ents


def lying_variants(chunk: IndexedChunk, seed=0):
    """{name: (stream, record, what the lie is)}: the true stream under a targeted false record, or (repointed_copy) a
    stream changed under its otherwise true record.  Every variant is legal Snappy."""
    rng = random.Random(seed)
    lay = chunk.true_layout()
    stream = chunk.stream()
    true = index_record(lay)
    nf = len(lay)
    out = {}
    # an entry moved one byte into the payload of the literal it points at (the byte still parses as a header)
    cands = []
    for f, (s, starts) in enumerate(lay):
        ent = fragment_entries(starts, s)
        for p, e in zip(starts, chunk.encoded[f]):
            if ent[p // SUB] == p % SUB and e[0] & 3 == 0 and p % SUB + 1 < SUB and len(e) > 1:
                cands.append((f, p))
    if cands:
        f, p = rng.choice(cands)
        l2 = [(s, st if g != f else [q if q != p else p + 1 for q in st]) for g, (s, st) in enumerate(lay)]
        out["entry_into_literal"] = (stream, index_record(l2), (f, p))
    # an entered piece marked as having no element start
    f = rng.randrange(nf)
    s, st = lay[f]
    ent = fragment_entries(st, s)
    piece = rng.choice([i for i, v in enumerate(ent) if v != NO_ENTRY])
    rec = bytearray(true)
    rec[2 * nf + sum((lay[g][0] + SUB - 1) // SUB for g in range(f)) + piece] = NO_ENTRY
    out["entered_piece_none"] = (stream, bytes(rec), (f, piece))
    if nf >= 2:
        # one fragment boundary moved by one element (the last element of fragment f opens fragment f + 1)
        # (where the grown fragment still fits the longest stream an index may describe)
        f = rng.choice([g for g in range(nf - 1) if lay[g + 1][0] + len(chunk.encoded[g][-1]) <= FRAG_MAX_STREAM and len(lay[g][1]) > 1])
        moved = len(chunk.encoded[f][-1])
        l2 = list(lay)
        s0, st0 = lay[f]
        s1, st1 = lay[f + 1]
        l2[f] = (s0 - moved, st0[:-1])
        l2[f + 1] = (s1 + moved, [0] + [q + moved for q in st1])
        out["boundary_moved"] = (stream, index_record(l2), (f, moved))
        # two fragment lengths swapped
        pairs = [g for g in range(nf - 1) if lay[g][0] != lay[g + 1][0]]
        if pairs:
            g = rng.choice(pairs)
            rec = bytearray(true)
            rec[2 * g: 2 * g + 2], rec[2 * g + 2: 2 * g + 4] = true[2 * g + 2: 2 * g + 4], true[2 * g: 2 * g + 2]
            out["lengths_swapped"] = (stream, bytes(rec), g)
        # a copy re-pointed before its fragment's start: same encoding size, so the record stays true
        for f in range(1, nf):
            base = len(chunk.pre) + sum(lay[g][0] for g in range(f))
            pos = 0
            for e, enc in zip(chunk.fragments[f], chunk.encoded[f]):
                if e[0] == "copy" and e[3] in (2, 4) and e[2] < 32768:
                    new = e[2] + FRAG    # now reads 32 KiB further back: inside fragment f - 1
                    s2 = bytearray(stream)
                    s2[base + pos + 1: base + pos + (3 if e[3] == 2 else 5)] = new.to_bytes(2 if e[3] == 2 else 4, "little")
                    out["repointed_copy"] = (bytes(s2), true, (f, pos, e[2], new))
                    break
                pos += len(enc)
            if "repointed_copy" in out:
                break
    return out


def indexed_chunk(seed, nfrag, last=FRAG, families=("dense", "expanding", "deep_chains", "mixed", "long_literals")):
    """nfrag fragments, each from a family in turn (the last `last` bytes long)"""
    rng = random.Random(seed)
    frags = []
    for f in range(nfrag):
        fam = families[(seed + f) % len(families)]
        n = FRAG if f + 1 < nfrag else last
        frags.append(FAMILIES[fam](rng.randrange(1 << 30), n))
    return IndexedChunk(frags)


# ---- the shared corpus: a pool of chunk streams, and frames assembled from it ----------------------------------------

POOL_SPECS = [(fam, seed, size) for seed, fam in enumerate(FAMILIES) for size in (1, 61, 4097, 40001)] + [
    ("long_literals", 11, 600007), ("dense", 12, 200003), ("dense", 13, 65537), ("expanding", 14, 300001),
    ("deep_chains", 15, 260005), ("deep_chains", 16, 99999), ("far_copies", 17, 333333), ("far_copies", 18, 70001),
    ("mixed", 19, 150001), ("mixed", 20, 500009), ("expanding", 21, 1000003)]
BIG_SPEC = ("expanding", 22, 16 * 2**20 + 4099)   # one chunk of more than 16 MiB: many windows of one chunk in flight


@functools.lru_cache(None)
def pool_stream(fam, seed, size) -> bytes:
    return write_stream(FAMILIES[fam](seed, size))


def pool(big=False):
    """[(name, stream)] of the pool"""
    specs = POOL_SPECS + ([BIG_SPEC] if big else [])
    return [(f"{fam}/{seed}/{size}", pool_stream(fam, seed, size)) for fam, seed, size in specs]


def random_frames(seed, count, streams, max_chunks=6, max_texture=1 << 22):
    """count frames of 1..max_chunks chunks drawn from streams ([(name, stream)], Snappy) and from verbatim chunks of odd
    sizes, so that chunk outputs start at arbitrary bytes of the texture; Complex frames with and without the Chunk Offset
    Table, with 4- and 8-byte headers, and single-chunk sections without Decode Instructions.  [(frame, chunks)]"""
    rng = random.Random(seed)
    frames = []
    while len(frames) < count:
        k = rng.randint(1, max_chunks)
        chunks, total = [], 0
        for _ in range(k):
            if rng.random() < 0.2:
                d = rng.randbytes(rng.randint(1, 5000))
                chunks.append((RAW, d))
                total += len(d)
            else:
                name, s = rng.choice(streams)
                chunks.append((SNAPPY, s))
                total += parse_varint(s)[0]
        if total > max_texture:
            continue
        if k == 1 and rng.random() < 0.4:
            frames.append((simple_frame(chunks[0][0], chunks[0][1], rng.random() < 0.5), chunks))
            continue
        ot = rng.random() < 0.4
        frames.append((complex_frame(chunks, offset_table=ot, long_headers=rng.random() < 0.4, gap=rng.randint(0, 19) if ot else 0), chunks))
    return frames


def indexed_chunks():
    """chunks of self-contained fragments: several fragments with a short last one, one whole fragment, one of 77 bytes
    past a fragment boundary"""
    return [indexed_chunk(31, 4, 5001), indexed_chunk(32, 1, FRAG), indexed_chunk(33, 3, 77), indexed_chunk(34, 5, 30000)]


def indexed_frames():
    """{name: (frame, chunks)}: one frame with a true fragment index over indexed_chunks() and a verbatim chunk, and one frame
    per lying variant of each chunk, the other chunks keeping their true records"""
    ics = indexed_chunks()
    raw = (RAW, random.Random(5).randbytes(1001))
    true_recs = [index_record(c.true_layout()) for c in ics]

    def frame(streams, recs):
        chunks = [(SNAPPY, streams[0]), raw] + [(SNAPPY, s) for s in streams[1:]]
        records = [recs[0], None] + list(recs[1:])
        return complex_frame(chunks, index=index_body(records)), chunks

    streams = [c.stream() for c in ics]
    out = {"true": frame(streams, true_recs)}
    for i, c in enumerate(ics):
        for name, (s, rec, _) in lying_variants(c, seed=i).items():
            ss, rr = list(streams), list(true_recs)
            ss[i], rr[i] = s, rec
            out[f"{name}/{i}"] = frame(ss, rr)
    return out
