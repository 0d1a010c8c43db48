"""Textures for the GPU Snappy compressor, one generator per shape family its rules have to handle (tests/snappy_encode_model.py
states the rules).  Every generator is seeded and returns Entry objects: a name, the family, and the one or two textures of a
HapEncode call, [(bytes, format, compressor, requested chunks)].  Test-only; it needs no GPU and no library.

Designed units are "fresh": random 8-byte units whose 13-bit hashes are unused so far in their fragment, so the first
occurrence of every hash is the unit the design means, and matches happen only where a family puts them."""
from __future__ import annotations

import functools
from dataclasses import dataclass

import numpy as np

import snappy_encode_model as m

FAMILIES = ("literal_runs", "copy_runs", "block_repeats", "hash_collisions", "propagation", "last_fragments", "boundaries",
            "real")


@dataclass
class Entry:
    name: str
    family: str
    textures: list


class Fragment:
    """a fragment's units under construction; fresh() hands out units with hashes new to the fragment"""

    def __init__(self, rng: np.random.Generator):
        self.rng = rng
        self.units: list[int] = []
        self.used: set[int] = set()

    def fresh(self, n=1):
        out = []
        while len(out) < n:
            cand = self.rng.integers(1, 1 << 63, 64, dtype=np.int64).astype(np.uint64)
            for u, h in zip(cand.tolist(), m.unit_hash(cand).tolist()):
                if h not in self.used and len(out) < n:
                    self.used.add(h)
                    out.append(u)
        return out

    def add(self, units):
        for u in units:
            self.used.add(int(m.unit_hash(np.array([u], np.uint64))[0]))
        self.units += list(units)
        return self

    def fill_to(self, n):
        """fresh units up to n units"""
        return self.add(self.fresh(n - len(self.units))) if n > len(self.units) else self

    def bytes(self) -> bytes:
        return np.array(self.units, dtype="<u8").tobytes()


def _one(name, family, data, fmt, chunks=1):
    return Entry(name, family, [(data, fmt, 1, chunks)])


def _flat(n, unit=0x0123456789ABCDEF):
    return np.full(n, unit, dtype="<u8").tobytes()


# ---- literal runs -------------------------------------------------------------------------------------------------------------

def literal_runs(seed=1):
    out = []
    for fmt in (m.FMT_DXT1, m.FMT_YCOCG):
        f = Fragment(np.random.default_rng(seed + fmt))
        anchor = f.fresh(8)
        f.add(anchor)
        for L in range(1, 41):
            f.add(anchor).add(f.fresh(L))         # an 8-unit copy of the anchor, then L literal units
        f.add(anchor)
        if len(f.units) % 2:
            f.add(f.fresh(1))
        out.append(_one(f"literal_runs/{fmt:x}", "literal_runs", f.bytes(), fmt))
    # a whole literal fragment (stream n + 3) in a chunk that still compresses thanks to its flat second fragment
    f = Fragment(np.random.default_rng(seed + 7)).fill_to(m.FRAG_UNITS)
    out.append(_one("literal_runs/whole_fragment", "literal_runs", f.bytes() + _flat(m.FRAG_UNITS), m.FMT_DXT1))
    return out


# ---- copy runs ----------------------------------------------------------------------------------------------------------------

def copy_runs(seed=2):
    out = []
    rng = np.random.default_rng(seed)
    for d, fmt in ((1, m.FMT_DXT1), (2, m.FMT_YCOCG), (3, m.FMT_DXT1), (2, m.FMT_DXT1), (1, m.FMT_RGTC1)):
        f = Fragment(rng)
        for L in range(1, 18):
            f.add(f.fresh(1 + (len(f.units) + 1) % 2))     # keep every period-d pattern on an even unit
            pat = f.fresh(d)
            f.add(pat).add([pat[i % d] for i in range(L)])
        f.add(f.fresh(3))
        if len(f.units) % 2:
            f.add(f.fresh(1))
        out.append(_one(f"copy_runs/d{d}_{fmt:x}", "copy_runs", f.bytes(), fmt))
    # far copies: a block of L units at the fragment's start again at its end (offset 4096 - L units, up to 4095 = 32760 bytes)
    for L in (1, 2, 5, 8, 9, 16, 17):
        f = Fragment(rng)
        blk = f.fresh(L)
        f.add(blk).fill_to(m.FRAG_UNITS - L).add(blk)
        # the next fragment opens with the first fragment's last and first units: literals, copies never leave a fragment
        g = Fragment(rng).add(f.units[-3:] + f.units[:3]).fill_to(64)
        g.add(g.units[:8] * 4)
        out.append(_one(f"copy_runs/far_{L}", "copy_runs", f.bytes() + g.bytes(), m.FMT_DXT1))
    return out


# ---- block repeats ------------------------------------------------------------------------------------------------------------

def block_repeats(seed=3):
    """period 1 and 2 repeats that start and end on the 8-unit strip and the 256-unit warp boundaries; the repeated block
    also appears far earlier, so the hash alone would give a long distance"""
    out = []
    rng = np.random.default_rng(seed)
    for fmt, per in ((m.FMT_DXT1, 1), (m.FMT_RGTC1, 1), (m.FMT_YCOCG, 2), (m.FMT_DXT5, 2)):
        f = Fragment(rng)
        f.add(f.fresh(4))
        blocks = []
        for _ in range(12):
            b = f.fresh(per)
            blocks.append(b)
            f.add(b).add(f.fresh(2))
        f.fill_to(16)
        for k, at in enumerate((24, 40, 63, 96, 254, 256, 510, 768, 1023, 1280, 1536, 2046)):
            start = at - (at % per)
            f.fill_to(start)
            reps = 1 + (k * 5) % 11
            b = blocks[k]
            f.add(b * reps)
            if per == 2:
                # DXT5 pairs where only one unit repeats: (a, b) (a, c) (d, b)
                a, c = b
                f.add([a] + f.fresh(1) + f.fresh(1) + [c])
            f.add(f.fresh(3))
        f.fill_to(2600)
        if len(f.units) % 2:
            f.add(f.fresh(1))
        out.append(_one(f"block_repeats/{fmt:x}", "block_repeats", f.bytes(), fmt))
    return out


# ---- hash collisions ----------------------------------------------------------------------------------------------------------

@functools.lru_cache(None)
def colliding_units(count=48, seed=4):
    """`count` distinct units with one 13-bit hash, and pairs of distinct units with equal hashes, found by brute force"""
    rng = np.random.default_rng(seed)
    u = rng.integers(1, 1 << 63, 1 << 21, dtype=np.int64).astype(np.uint64)
    h = m.unit_hash(u)
    vals, counts = np.unique(h, return_counts=True)
    best = vals[np.argmax(counts)]
    same = u[h == best][:count]
    assert len(same) == count and len(set(same.tolist())) == count
    order = np.argsort(h, kind="stable")
    hs = h[order]
    pairs = [(int(u[order[i]]), int(u[order[i + 1]])) for i in np.flatnonzero(hs[1:] == hs[:-1])[:64].tolist()
             if u[order[i]] != u[order[i + 1]]]
    return [int(x) for x in same], pairs


def hash_collisions(seed=5):
    out = []
    same, pairs = colliding_units()
    for fmt in (m.FMT_DXT1, m.FMT_YCOCG):
        rng = np.random.default_rng(seed + fmt)
        f = Fragment(rng)
        f.add(f.fresh(6))
        # the colliding unit comes first, so the table's entry for the hash is a different unit: the later repeat of b is
        # not found through the hash
        for k, (a, b) in enumerate(pairs[:16]):
            f.add([a]).add(f.fresh(3)).add([b]).add(f.fresh(2 + k % 3)).add([b])
        # runs of distinct units with one hash across the strip (8-unit) and warp (256-unit) boundaries: the dup-skip
        for at, n in ((253, 7), (509, 6), (1022, 11), (1535, 3)):
            f.fill_to(at)
            f.add(same[:n])
        # equal hashes one and two units back, alternating
        f.fill_to(2044)
        f.add([same[20], f.fresh(1)[0], same[21], same[22], f.fresh(1)[0], same[23]])
        f.add(same[24:40])
        f.fill_to(2304)
        out.append(_one(f"hash_collisions/{fmt:x}", "hash_collisions", f.bytes(), fmt))
    return out


# ---- propagation --------------------------------------------------------------------------------------------------------------

def propagation(seed=6):
    """the three outcomes of the round: the left neighbour's distance, the right one's when the left is 0, and the right one's
    as the second choice; each placed at many strip offsets"""
    out = []
    for fmt in (m.FMT_DXT1, m.FMT_YCOCG):
        rng = np.random.default_rng(seed + fmt)
        f = Fragment(rng)
        f.add(f.fresh(4))
        designs = []
        for k in range(24):
            x, y, z, w, v, y2, z2 = f.fresh(7)
            x3, y3, z3 = f.fresh(3)
            designs.append((x, y, z, w, v, y2, z2, x3, y3, z3))
            # first occurrences: y alone, then the pair (x, y); v alone, then the pair (v, z); w alone; y2 alone, then (y2, z2)
            f.add([y]).add(f.fresh(2)).add([x, y]).add(f.fresh(2)).add([v]).add(f.fresh(1)).add([v, z]).add(f.fresh(2))
            f.add([w]).add(f.fresh(2)).add([y2]).add(f.fresh(2)).add([y2, z2]).add(f.fresh(2))
            # y3 alone, then the pairs (x3, y3) and (y3, z3)
            f.add([y3]).add(f.fresh(2)).add([x3, y3]).add(f.fresh(2)).add([y3, z3]).add(f.fresh(2))
        for k, (x, y, z, w, v, y2, z2, x3, y3, z3) in enumerate(designs):
            f.fill_to(600 + 64 * k + (k % 8))
            f.add([x, y]).add(f.fresh(2))                   # left wins: y takes x's distance
            f.fill_to(len(f.units) + k % 5)
            f.add([v, z]).add(f.fresh(2))                   # right wins: v (first at its lone copy) takes z's distance
            f.add([w, y2, z2]).add(f.fresh(2))              # y2: w's distance fails, z2's distance as the second choice
            f.add([x3, y3, z3]).add(f.fresh(2))             # y3 matches at both neighbours' distances: the left one wins
        f.fill_to(2400)
        out.append(_one(f"propagation/{fmt:x}", "propagation", f.bytes(), fmt))
    return out


# ---- last fragments and odd chunk sizes ---------------------------------------------------------------------------------------

def _mixed_fragment(rng, n):
    f = Fragment(rng)
    blk = f.fresh(8)
    f.add(blk)
    while len(f.units) < n:
        f.add(f.fresh(1 + len(f.units) % 7)).add(blk[: 1 + len(f.units) % 8])
    return f.units[:n]


def last_fragments(seed=7):
    out = []
    rng = np.random.default_rng(seed)
    for U in (1, 2, 7, 8, 9, 255, 256, 257, 4095):
        body = np.array(_mixed_fragment(rng, m.FRAG_UNITS) + _mixed_fragment(rng, U), dtype="<u8").tobytes()
        out.append(_one(f"last_fragments/U{U}", "last_fragments", body, m.FMT_DXT1))
        if U % 2 == 0:
            out.append(_one(f"last_fragments/U{U}_ycocg", "last_fragments", body, m.FMT_YCOCG))
    # DXT1 chunks of 8008 bytes (not a multiple of 16): chunks start at every second 8-byte block of the input
    out.append(_one("last_fragments/dxt1_chunk_8008", "last_fragments",
                    np.array(_mixed_fragment(rng, 3 * 1001), dtype="<u8").tobytes(), m.FMT_DXT1, 3))
    # chunk_bytes % 8 != 0: no compression, the texture is stored verbatim
    out.append(_one("last_fragments/dxt1_1004_bytes", "last_fragments", bytes(rng.integers(0, 3, 1004, dtype=np.uint8)),
                    m.FMT_DXT1))
    out.append(_one("last_fragments/ycocg_148_bytes_3_chunks", "last_fragments", bytes(148), m.FMT_YCOCG, 3))
    return out


# ---- boundaries searched with the model --------------------------------------------------------------------------------------

def _candidate(rng_seed, U, M, s, gap):
    """U units: fresh literals, s single repeats of their predecessor `gap` units apart inside them (each splits the literal
    and costs 2, 3 or 4 bytes less than the unit it replaces, by the literal headers around it), then M repeats of the last
    literal"""
    f = Fragment(np.random.default_rng(rng_seed))
    L = U - M
    lits = f.fresh(L)
    for q in range(1, s + 1):
        if gap * q < L - 1:
            lits[gap * q] = lits[gap * q - 1]
    return lits + [lits[-1]] * M


def _packed(units):
    tr = m.compress_fragment(np.array(units, dtype="<u8").tobytes(), 1)
    return len(m.varint(8 * len(units))) + len(tr.stream)


def search_chunk(U, target, seed):
    """DXT1 units of one chunk (U <= 4096) whose Snappy stream, varint included, is exactly `target` bytes, by the model"""
    for gap in (5, 12, 40):
        for s in range(4):
            lo, hi = 1, U - 1                 # the stream shrinks as M grows: find the largest M with packed >= target
            if _packed(_candidate(seed, U, lo, s, gap)) < target:
                continue
            while lo < hi:
                mid = (lo + hi + 1) // 2
                if _packed(_candidate(seed, U, mid, s, gap)) >= target:
                    lo = mid
                else:
                    hi = mid - 1
            units = _candidate(seed, U, lo, s, gap)
            if _packed(units) == target:
                return units
    raise ValueError(f"no chunk of {U} units packs to {target} bytes")


def boundaries(seed=8):
    out = []
    # a chunk whose stream is chunk_bytes - 1 (Snappy), chunk_bytes and + 1 (both stored raw); 2- and 3-byte preambles
    for U in (20, 100, 1000, 2100, 4096):
        cb = 8 * U
        for delta in (-1, 0, 1):
            try:
                units = search_chunk(U, cb + delta, seed + U)
            except ValueError:
                continue
            out.append(_one(f"boundaries/chunk_{U}_{delta:+d}", "boundaries", np.array(units, dtype="<u8").tobytes(), m.FMT_DXT1))
    # a texture whose complex body is bytes + top_hdr - 1 (complex), equal (verbatim) and + 1: a raw chunk and a searched one
    for U in (300, 4096):
        cb = 8 * U
        noise = Fragment(np.random.default_rng(seed + 99)).fill_to(U).units
        for delta in (-1, 0, 1):
            units = search_chunk(U, cb - 18 + delta, seed + 2 * U)     # body = cb + packed + 4 + (5 * 2 + 8)
            data = np.array(noise + units, dtype="<u8").tobytes()
            out.append(_one(f"boundaries/texture_{U}_{delta:+d}", "boundaries", data, m.FMT_DXT1, 2))
    return out


# ---- real content -------------------------------------------------------------------------------------------------------------

def real(seed=9):
    import twin
    from hap_b200 import synth
    out = []
    for kind, fmt, (w, h), chunks, content in (("bc1", m.FMT_DXT1, (512, 256), 3, "video"),
                                               ("ycocg", m.FMT_YCOCG, (640, 360), 4, "video"),
                                               ("bc4", m.FMT_RGTC1, (256, 128), 1, "video"),
                                               ("bc3", m.FMT_DXT5, (256, 192), 2, "edges"),
                                               ("ycocg", m.FMT_YCOCG, (256, 256), 2, "flat")):
        rgba = synth.frame(w, h, seed, kind=content).numpy()
        out.append(_one(f"real/{kind}_{content}_{w}x{h}", "real", twin.encode(kind, rgba), fmt, chunks))
    return out


def corpus():
    return (literal_runs() + copy_runs() + block_repeats() + hash_collisions() + propagation() + last_fragments() + boundaries()
            + real())
