"""The Snappy corpus of snappy_corpus.py is what it claims to be: every legal stream decodes to the same bytes in the plain
Python decoder, the CPU oracle and Google Snappy (pyarrow's RawUncompress); every illegal stream is rejected by all three; the
built frames decode in the reference to the concatenation of their chunks; the fragment index records describe the element
chains, and each lying variant lies exactly where it says; each stream family has the property it exists for."""
import pytest

import oracles
import snappy_corpus as sc
from hap_b200.abi import HapResult_No_Error, HapTextureFormat_RGB_DXT1

SEEDS_SIZES = [(1, 1), (2, 7), (3, 61), (4, 4097), (5, 40001), (6, 300001)]


def google(stream, size):
    """(True, bytes) or (False, None) from Google Snappy; None when pyarrow is not there"""
    try:
        import pyarrow as pa
    except ImportError:
        return None
    try:
        return True, pa.decompress(stream, decompressed_size=size, codec="snappy").to_pybytes()
    except OSError:
        return False, None


def reference():
    return oracles.ref_abi() or oracles.oracle_abi()


@pytest.mark.parametrize("family", sorted(sc.FAMILIES))
def test_legal_streams_decode_alike_in_three_decoders(family):
    for seed, size in SEEDS_SIZES:
        s = sc.write_stream(sc.FAMILIES[family](seed, size))
        want = sc.decode(s)
        assert len(want) == size
        assert oracles.snappy_uncompress(s) == (0, want), (family, seed, size)
        g = google(s, size)
        if g is not None:
            assert g == (True, want), (family, seed, size)


def test_element_encodings_every_decoder_takes():
    """literals in every tag form, also non-minimal ones; copy-1, copy-2 and copy-4, also copy-4 at small offsets"""
    head = bytes(range(40, 50))
    els = [sc.lit(head, 60), sc.lit(b"x", 0), sc.lit(b"yz", 63), sc.lit(bytes(61), 61), sc.lit(bytes(300), 62),
           sc.copy(4, 1, 1), sc.copy(11, 300, 1), sc.copy(1, 5, 2), sc.copy(64, 3, 2), sc.copy(64, 1, 4),
           sc.copy(7, 7, 4), sc.copy(5, 374 + 4 + 11 + 1 + 64 + 64 + 7, 4)]
    s = sc.write_stream(els)
    pre = sc.parse_varint(s)[1]
    assert s[pre] == 60 << 2 and s[pre + 1] == 9            # tag 60 for a 10-byte literal
    want = sc.decode(s)
    assert want[:10] == head and want[10:13] == b"xyz"
    assert oracles.snappy_uncompress(s) == (0, want)
    g = google(s, len(want))
    if g is not None:
        assert g == (True, want)
    with pytest.raises(ValueError):
        sc.encode_element(sc.lit(bytes(61), 0))
    with pytest.raises(ValueError):
        sc.encode_element(sc.copy(12, 5, 1))


@pytest.mark.parametrize("name", sorted(sc.illegal_streams()))
def test_illegal_streams_are_rejected_by_every_decoder(name):
    s = sc.illegal_streams()[name]
    with pytest.raises(sc.SnappyError):
        sc.decode(s)
    assert oracles.snappy_uncompress(s)[0] != 0
    try:
        size = min(sc.parse_varint(s)[0], 1 << 20)
    except sc.SnappyError:
        size = 64
    g = google(s, size)
    if g is not None:
        assert g == (False, None)


def test_pool_frames_decode_in_the_reference():
    """every frame shape the GPU tests send: Complex frames of verbatim and Snappy chunks at arbitrary output sizes, with and
    without the Chunk Offset Table, 4- and 8-byte headers, and single-chunk sections"""
    ref = reference()
    frames = sc.random_frames(3, 60, sc.pool())
    shapes = set()
    for frame, chunks in frames:
        want = sc.frame_texture(chunks)
        r, tex, fmt, _ = ref.decode(frame, 0, len(want))
        assert (r, fmt) == (HapResult_No_Error, HapTextureFormat_RGB_DXT1) and tex == want
        shapes.add((frame[3] >> 4, frame[:3] == b"\0\0\0", len(chunks) > 1))
    assert {(0xC, False, True), (0xC, True, True), (0xB, False, False), (0xB, True, False)} <= shapes


@pytest.mark.parametrize("name", sorted(sc.illegal_streams()))
def test_frames_around_illegal_streams_fail_in_the_reference(name):
    s = sc.illegal_streams()[name]
    good = sc.pool()[3][1]
    for frame, n in ((sc.complex_frame([(sc.SNAPPY, good), (sc.SNAPPY, s)]), len(sc.decode(good)) + 1024),
                     (sc.simple_frame(sc.SNAPPY, s), 1024)):
        r = reference().decode(frame, 0, n)[0]
        assert r != HapResult_No_Error
        assert oracles.oracle_abi().decode(frame, 0, n)[0] == r


def rebuild_record(stream):
    """the index record of a stream of self-contained fragments, rebuilt by walking its element chain and cutting it every
    32 KiB of output"""
    total, pre = sc.parse_varint(stream)
    frags, starts, out, fstart = [], [], 0, pre
    for pos, size, n, _, _, _ in sc.parse_elements(stream, pre):
        if out and out % sc.FRAG == 0 and out // sc.FRAG == len(frags) + 1:
            frags.append((pos - fstart, starts))
            starts, fstart = [], pos
        starts.append(pos - fstart)
        out += n
    frags.append((len(stream) - fstart, starts))
    assert out == total
    return sc.index_record(frags)


def test_index_records_and_their_lies():
    for i, c in enumerate(sc.indexed_chunks()):
        s = c.stream()
        true = sc.index_record(c.true_layout())
        assert rebuild_record(s) == true
        assert sc.decode(s) == oracles.snappy_uncompress(s)[1]
        nf = len(c.fragments)
        lens, ents = sc._record_entries(true, nf)
        lies = sc.lying_variants(c, seed=i)
        assert {"entry_into_literal", "entered_piece_none"} <= set(lies)
        if nf >= 2:
            assert {"boundary_moved", "lengths_swapped"} <= set(lies)
        for name, (s2, rec, what) in lies.items():
            assert oracles.snappy_uncompress(s2)[0] == 0     # legal Snappy, whatever the index says
            if name == "repointed_copy":
                f, pos, old, new = what
                assert rec == true and s2 != s and new - old == sc.FRAG
                assert sum(a != b for a, b in zip(s, s2)) <= 2
                assert rebuild_record(s2) == true            # the record still describes the element chain
                continue
            assert s2 == s and rec != true
            l2, e2 = sc._record_entries(rec, nf)
            if name == "entry_into_literal":
                f, p = what
                assert l2 == lens
                diff = [(g, k) for g in range(nf) for k in range(len(ents[g])) if ents[g][k] != e2[g][k]]
                assert diff == [(f, p // sc.SUB)] and e2[f][p // sc.SUB] == ents[f][p // sc.SUB] + 1
                assert s[len(c.pre) + sum(lens[:f]) + p] & 3 == 0     # it pointed at a literal
            elif name == "entered_piece_none":
                f, piece = what
                assert l2 == lens and ents[f][piece] != sc.NO_ENTRY and e2[f][piece] == sc.NO_ENTRY
                assert sum(a != b for g in range(nf) for a, b in zip(ents[g], e2[g])) == 1
            elif name == "boundary_moved":
                f, moved = what
                assert sum(l2) == sum(lens) and l2[f] == lens[f] - moved and l2[f + 1] == lens[f + 1] + moved
                assert all(l2[g] == lens[g] for g in range(nf) if g not in (f, f + 1))
            elif name == "lengths_swapped":
                g = what
                assert l2[g] == lens[g + 1] and l2[g + 1] == lens[g] and lens[g] != lens[g + 1]
            else:
                raise AssertionError(name)


def test_indexed_frames_decode_in_the_reference():
    ref = reference()
    for name, (frame, chunks) in sc.indexed_frames().items():
        want = b"".join(d if c == sc.RAW else oracles.snappy_uncompress(d)[1] for c, d in chunks)
        r, tex, _, _ = ref.decode(frame, 0, len(want))
        assert r == 0 and tex == want, name


def test_families_have_their_properties():
    """measured on the streams the pool holds, so that an edit of a generator cannot quietly weaken the corpus"""
    st = {fam: sc.stream_stats(sc.FAMILIES[fam](seed, size)) for fam, seed, size in
          [("long_literals", 11, 600007), ("dense", 12, 200003), ("expanding", 14, 300001), ("deep_chains", 15, 260005),
           ("far_copies", 17, 333333), ("mixed", 20, 500009)]}
    assert st["long_literals"]["max_literal"] == 200000
    lits = {len(e[1]) for e in sc.fam_long_literals(11, 600007) if e[0] == "lit"}
    assert set(sc.LONG_LITERALS) <= lits
    assert st["dense"]["max_elems_per_16k"] > 4 * 800 and st["dense"]["max_elems_per_16k"] >= 7000
    assert st["expanding"]["expansion"] > 20
    assert st["deep_chains"]["depth"] >= 30
    assert st["far_copies"]["copy4"] > 100 and st["far_copies"]["max_offset"] > 65535 and st["far_copies"]["reaches_byte0"]
    assert st["mixed"]["copy4"] > 0 and st["mixed"]["max_literal"] > 60
    big = sc.stream_stats(sc.FAMILIES[sc.BIG_SPEC[0]](sc.BIG_SPEC[1], 1 << 20))
    assert big["expansion"] > 20
    assert sc.BIG_SPEC[2] >= 16 << 20
