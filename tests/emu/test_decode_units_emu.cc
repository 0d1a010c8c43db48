// tests/emu/test_decode_units_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The unit path of snappy_execute_kernel (fragments of an embedded index whose elements are all 8-byte granular) under the
// fiber SIMT emulator, checked against the CPU oracle (oracle/snappy_oracle.c): this encoder's own fragments (K5 run on
// the emulator), fragments with 4-byte elements (general path), copies that leave their fragment under a correct index
// (repair pass), lying indexes, and every destination misalignment 0..15.  Built with -fsanitize=address the source,
// index and destination buffers have their exact sizes.
#define HAPB200_EMU
#include "hap_host.h"
#include "snappy_decode.cuh"
#include "decode_emu.h"

extern "C" {
#include "snappy_oracle.h"
}
#include <random>
#include <string>

#if defined(__SANITIZE_ADDRESS__)
static const size_t kGuard = 0;    // exact-size destination: ASan reports any byte written past it
#else
static const size_t kGuard = 32;   // guard bytes behind the destination, checked below
#endif

using namespace hapb200;
static int g_fail = 0;

struct Chunk {
    std::vector<uint8_t> stream;   // varint(uncompressed) + fragment streams
    std::vector<uint8_t> index;    // the chunk's record (hap_index.h)
    size_t raw_bytes;
};

static void varint(std::vector<uint8_t> &s, uint32_t n)
{
    while (n >= 0x80) { s.push_back((uint8_t)((n & 0x7F) | 0x80)); n >>= 7; }
    s.push_back((uint8_t)n);
}

// record of a chunk from its fragments' element streams: the entries are those of the true element chain
static Chunk assemble(size_t raw_bytes, const std::vector<std::vector<uint8_t>> &frags)
{
    Chunk c;
    c.raw_bytes = raw_bytes;
    varint(c.stream, (uint32_t)raw_bytes);
    for (auto &f : frags) { c.index.push_back((uint8_t)f.size()); c.index.push_back((uint8_t)(f.size() >> 8)); }
    for (auto &f : frags) {
        c.stream.insert(c.stream.end(), f.begin(), f.end());
        std::vector<uint8_t> ent((f.size() + (1u << kIndexSubLog2) - 1) >> kIndexSubLog2, (uint8_t)kIndexNoEntry);
        for (size_t p = 0; p < f.size();) {
            const size_t piece = p >> kIndexSubLog2;
            if (ent[piece] == kIndexNoEntry) ent[piece] = (uint8_t)(p & ((1u << kIndexSubLog2) - 1));
            const uint32_t tag = f[p], kind = tag & 3;
            if (kind == 0) {
                uint32_t m = tag >> 2, hdr = 1;
                if (m >= 60) { const uint32_t extra = m - 59; m = 0; for (uint32_t q = 0; q < extra; q++) m |= (uint32_t)f[p + 1 + q] << (8 * q); hdr += extra; }
                p += hdr + m + 1;
            } else {
                p += kind == 1 ? 2 : kind == 2 ? 3 : 5;
            }
        }
        c.index.insert(c.index.end(), ent.begin(), ent.end());
    }
    return c;
}

// this encoder's fragments of one single-chunk texture (K5 on the emulator)
static Chunk encode_chunk(const std::vector<uint8_t> &raw, unsigned fmt)
{
    TextureArgs ta{raw.size(), fmt, HapCompressorSnappy, 1};
    FrameGeom G;
    if (build_frame_geom(1, &ta, G) != 0 || G.s[0].chunks != 1 || !G.s[0].compress) abort();
    std::vector<uint8_t> scratch((size_t)G.frags_per_frame * kFragCap), fent((size_t)G.frags_per_frame * kFragEntryStride);
    std::vector<uint32_t> fsize(G.frags_per_frame);
    emu::g_order_mode() = 0;
    HAP_LAUNCH(snappy_encode_fragments_kernel, dim3(2), dim3(kEncThreads), sizeof(EncodeSmem), nullptr, raw.data(), G,
               (uint32_t)G.frags_per_frame, scratch.data(), fsize.data(), fent.data());
    std::vector<std::vector<uint8_t>> frags;
    for (uint32_t f = 0; f < G.frags_per_frame; f++) {
        if (fsize[f] == kFragStoredRaw) abort();
        frags.emplace_back(scratch.begin() + (size_t)f * kFragCap, scratch.begin() + (size_t)f * kFragCap + fsize[f]);
    }
    Chunk c = assemble(raw.size(), frags);
    // the encoder's own entries must equal those of the chain (the record above is what its frames carry)
    const uint8_t *e = c.index.data() + 2 * frags.size();
    for (uint32_t f = 0; f < frags.size(); f++) {
        const size_t n = (fsize[f] + (1u << kIndexSubLog2) - 1) >> kIndexSubLog2;
        if (memcmp(e, &fent[(size_t)f * kFragEntryStride], n) != 0) { fprintf(stderr, "encoder entries differ from the chain\n"); g_fail++; }
        e += n;
    }
    return c;
}

// Decodes `c` through the library's launch sequence; expects the oracle's bytes.  expect_units: windows the unit path
// must decode; expect_repaired: chunks requeued after pass 0 (kStatusIndexMismatch).
static void check(const std::string &name, const Chunk &c, int mode, uint32_t dmis, int64_t expect_units, int expect_repaired,
                  bool use_index = true)
{
    std::vector<uint8_t> ref(c.raw_bytes + 1);
    size_t rn = c.raw_bytes;
    const int rs = orc_snappy_uncompress(c.stream.data(), c.stream.size(), ref.data(), &rn);
    if (rs != ORC_SNAPPY_OK || rn != c.raw_bytes) { fprintf(stderr, "FAIL %s: oracle rejects the stream\n", name.c_str()); g_fail++; return; }
    std::vector<uint8_t> src(c.stream), index(c.index);             // exact sizes
    std::vector<uint8_t> out_store(dmis + c.raw_bytes + kGuard, 0xCD);
    uint8_t *got = out_store.data() + dmis;
    ChunkJob job;
    job.src = src.data();
    job.dst = got;
    job.src_bytes = (uint32_t)src.size();
    job.dst_bytes = (uint32_t)c.raw_bytes;
    job.compressor = kHapChunkSnappy;
    job.status = 99;
    job.index = use_index ? index.data() : nullptr;
    job.index_bytes = use_index ? (uint32_t)index.size() : 0;
    job.mode = kJobUndecided;
    job.win_base = 0;
    job.win_count = 0;
    emu::g_order_mode() = mode;
    const uint64_t units0 = emu_unit_windows();
    uint32_t wo[2] = {0, 0};
    decode_jobs_emu(&job, 1, src.size(), c.raw_bytes, 1, 1 + mode % 3, wo);
    const int64_t units = (int64_t)(emu_unit_windows() - units0);
    std::string why;
    if (job.status != HapResult_No_Error) why = "status " + std::to_string(job.status);
    else if (memcmp(got, ref.data(), c.raw_bytes) != 0) why = "bytes differ from the oracle";
    for (uint32_t i = 0; i < dmis; i++) if (out_store[i] != 0xCD) why = "wrote before dst";
    for (size_t i = 0; i < kGuard; i++) if (got[c.raw_bytes + i] != 0xCD) why = "wrote behind dst";
    if (expect_units >= 0 && units != expect_units) why = "unit path decoded " + std::to_string(units) + " windows, expected " + std::to_string(expect_units);
    if (expect_repaired >= 0 && (int)wo[1] != expect_repaired) why = "repaired " + std::to_string(wo[1]) + " chunks, expected " + std::to_string(expect_repaired);
    if (!why.empty()) {
        g_fail++;
        fprintf(stderr, "FAIL %s mode %d dmis %u: %s\n", name.c_str(), mode, dmis, why.c_str());
    }
}

// A hand-built fragment stream: literal runs and copies, as (kind, length, offset or literal bytes).
struct Frag {
    std::vector<uint8_t> s, raw;
    void lit(const std::vector<uint8_t> &b)
    {
        const uint32_t n = (uint32_t)b.size();
        if (n <= 60) s.push_back((uint8_t)((n - 1) << 2));
        else if (n <= 256) { s.push_back(60 << 2); s.push_back((uint8_t)(n - 1)); }
        else { s.push_back(61 << 2); s.push_back((uint8_t)(n - 1)); s.push_back((uint8_t)((n - 1) >> 8)); }
        s.insert(s.end(), b.begin(), b.end());
        raw.insert(raw.end(), b.begin(), b.end());
    }
    // copy with a 2-byte offset; `before` = the chunk's bytes in front of this fragment (for the raw image)
    void copy(uint32_t len, uint32_t off, const std::vector<uint8_t> &before)
    {
        s.push_back((uint8_t)(2 | ((len - 1) << 2)));
        s.push_back((uint8_t)off);
        s.push_back((uint8_t)(off >> 8));
        for (uint32_t i = 0; i < len; i++) {
            const size_t at = before.size() + raw.size();
            raw.push_back(at - off >= before.size() ? raw[at - off - before.size()] : before[at - off]);
        }
    }
};

static std::vector<uint8_t> random_bytes(std::mt19937 &rng, size_t n)
{
    std::vector<uint8_t> v(n);
    for (auto &b : v) b = (uint8_t)rng();
    return v;
}

// fragment of `n` output bytes out of literals and copies of `grain` bytes (8: the unit path; 4: the general path)
static Frag grained_fragment(std::mt19937 &rng, uint32_t n, uint32_t grain)
{
    Frag f;
    static const std::vector<uint8_t> none;
    while (f.raw.size() < n) {
        const uint32_t left = n - (uint32_t)f.raw.size();
        const uint32_t len = std::min<uint32_t>(left, grain * (1 + rng() % (64 / grain)));
        const uint32_t have = (uint32_t)f.raw.size() / grain;
        if (have >= 1 && rng() % 3 != 0) f.copy(len, grain * (1 + rng() % std::min<uint32_t>(have, 400)), none);
        else f.lit(random_bytes(rng, len));
    }
    return f;
}

int main(int argc, char **argv)
{
    const int modes = argc > 1 ? atoi(argv[1]) : 3;
    std::mt19937 rng(777);
    struct Case { std::string name; Chunk c; int64_t units; int repaired; };
    std::vector<Case> cases;

    // ---- this encoder's fragments ----------------------------------------------------------------------------------------
    {
        // DXT1-like (8-byte blocks, period 1): rows of 960 blocks, repeats of the block above and of neighbours, a shorter last fragment
        const size_t blocks = 4 * 4096 + 500;
        std::vector<uint8_t> v(8 * blocks);
        for (size_t b = 0; b < blocks; b++) {
            const int m = rng() % 8;
            for (int k = 0; k < 8; k++)
                v[8 * b + k] = (m < 3 && b >= 960) ? v[8 * (b - 960) + k] : (m < 5 && b >= 1) ? v[8 * (b - 1) + k] : (uint8_t)rng();
        }
        cases.push_back({"enc_dxt1", encode_chunk(v, HapFmt_RGB_DXT1), 5, 0});
    }
    {
        // DXT5-like (16-byte blocks, period 2), 2.5 fragments
        const size_t blocks = 2 * 2048 + 1024;
        std::vector<uint8_t> v(16 * blocks);
        for (size_t b = 0; b < blocks; b++) {
            const int m = rng() % 6;
            for (int k = 0; k < 16; k++)
                v[16 * b + k] = (m < 2 && b >= 480) ? v[16 * (b - 480) + k] : (m < 4 && b >= 1) ? v[16 * (b - 1) + k] : (uint8_t)rng();
        }
        cases.push_back({"enc_dxt5", encode_chunk(v, HapFmt_RGBA_DXT5), 3, 0});
    }
    {
        // whole fragments of one repeated 8-byte block (distance-1 runs) and of one repeated 16-byte block (distance 2)
        std::vector<uint8_t> v(3 * 32768);
        for (size_t i = 0; i < v.size(); i++) v[i] = (uint8_t)(0x31 + (i & 7) * 17);
        cases.push_back({"enc_dist1", encode_chunk(v, HapFmt_RGB_DXT1), 3, 0});
        std::vector<uint8_t> w(2 * 32768 + 4096);
        for (size_t i = 0; i < w.size(); i++) w[i] = (uint8_t)(0x52 + (i & 15) * 29);
        cases.push_back({"enc_dist2", encode_chunk(w, HapFmt_RGBA_DXT5), 3, 0});
    }
    {
        // noise: literals only
        cases.push_back({"enc_noise", encode_chunk(random_bytes(rng, 32768 + 8 * 77), HapFmt_RGB_DXT1), 2, 0});
    }

    // ---- hand-built fragments ------------------------------------------------------------------------------------------
    {
        // granular elements, random offsets inside the fragment, a short last fragment
        std::vector<std::vector<uint8_t>> fs;
        size_t raw = 0;
        for (uint32_t n : {32768u, 32768u, 8u * 123}) { Frag f = grained_fragment(rng, n, 8); fs.push_back(f.s); raw += f.raw.size(); }
        cases.push_back({"hand_units", assemble(raw, fs), 3, 0});
    }
    {
        // 4-byte elements: self-contained, but not 8-byte granular -> general path, no repair
        std::vector<std::vector<uint8_t>> fs;
        size_t raw = 0;
        for (uint32_t n : {32768u, 32768u - 4}) { Frag f = grained_fragment(rng, n, 4); fs.push_back(f.s); raw += f.raw.size(); }
        cases.push_back({"hand_4byte", assemble(raw, fs), 0, 0});
    }
    for (uint32_t grain : {8u, 4u}) {
        // a copy in fragment 1 reads fragment 0 under a correct index: legal Snappy, decoded by the repair pass
        Frag f0 = grained_fragment(rng, 32768, grain);
        Frag f1;
        f1.lit(random_bytes(rng, 64));
        f1.copy(64, 64 + 4096, f0.raw);   // reaches 4096 bytes into fragment 0
        Frag rest = grained_fragment(rng, 32768 - 128 - 3 * grain, grain);
        f1.s.insert(f1.s.end(), rest.s.begin(), rest.s.end());   // (rest's copies stay inside rest)
        f1.raw.insert(f1.raw.end(), rest.raw.begin(), rest.raw.end());
        f1.lit(random_bytes(rng, 3 * grain));
        // fragment 0 keeps its path; fragment 1 is handed over
        cases.push_back({"crossing_copy_" + std::to_string(grain), assemble(f0.raw.size() + f1.raw.size(), {f0.s, f1.s}), grain == 8 ? 1 : 0, 1});
    }

    // ---- lying indexes: every chunk must still decode to the oracle's bytes ------------------------------------------------
    {
        const Chunk base = cases[0].c;   // (a copy: the cases below are appended to the same vector)
        const uint32_t nf = (uint32_t)((base.raw_bytes + 32767) / 32768);
        for (int k = 0; k < 8; k++) {
            Chunk c = base;
            const size_t ent0 = 2 * nf;
            if (k == 0) c.index[ent0 + 1] = (uint8_t)((c.index[ent0 + 1] + 1) & 0x7F);          // entry one byte off
            else if (k == 1) c.index[ent0 + 3] = (uint8_t)kIndexNoEntry;                          // entered piece marked empty
            else if (k == 2) c.index[ent0] = 5;                                                   // first element not at 0
            else if (k == 3) { uint16_t s0 = c.index[0] | (c.index[1] << 8); s0 -= 1; c.index[0] = (uint8_t)s0; c.index[1] = (uint8_t)(s0 >> 8);
                               uint16_t s1 = c.index[2] | (c.index[3] << 8); s1 += 1; c.index[2] = (uint8_t)s1; c.index[3] = (uint8_t)(s1 >> 8); }   // boundary moved
            else c.index[ent0 + 1 + rng() % (c.index.size() - ent0 - 1)] ^= (uint8_t)(1u << (rng() % 7));
            cases.push_back({"lying_" + std::to_string(k), c, -1, -1});
        }
        cases.push_back({"truncated_index", base, -1, -1});
        cases.back().c.index.resize(2 * nf + 3);
    }

    for (int mode = 0; mode < modes; mode++)
        for (auto &c : cases) check(c.name, c.c, mode, 0, c.units, c.repaired);
    // every destination misalignment, for the aligned and the funnel-shifted store paths
    for (uint32_t dm = 0; dm < 16; dm++)
        for (size_t i : {(size_t)0, (size_t)2, (size_t)5}) check(cases[i].name, cases[i].c, 2 + dm % 3, dm, cases[i].units, cases[i].repaired);
    // the same chunks without their index: unit path not taken, same bytes
    for (size_t i : {(size_t)0, (size_t)7}) check(cases[i].name + "_noindex", cases[i].c, 1, 3, 0, 0, false);
    g_fail += g_decode_emu_overflow;
    printf("%zu cases x %d modes, %d failures, %llu unit-path windows\n", cases.size(), modes, g_fail, (unsigned long long)emu_unit_windows());
    return g_fail ? 1 : 0;
}
