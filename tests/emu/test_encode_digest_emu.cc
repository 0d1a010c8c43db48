// tests/emu/test_encode_digest_emu.cc -- TEST INFRASTRUCTURE ONLY.
// Pins the exact bytes of the encode path (K5 fragment compressor, K6 plan + place) under the fiber SIMT emulator.
// Every case of test_encode_emu.cc is encoded in every write-index / offset-table variant, under three fiber resume
// orders and two persistent-grid sizes.  For each encode a 64-bit FNV-1a digest is taken over the frame, every
// fragment's stream size and (when written) every fragment's index entries.  The digest of one variant must not
// depend on the resume order or the grid; the program prints one line per case, "<name> <digest>", combining the
// case's four variants, and the pytest wrapper compares those lines with digests recorded from an earlier kernel.
// So a change to how K5 assigns units to threads, or to its CTA shape, must leave every output byte as it was.
#define HAPB200_EMU
#include "hap_assemble.cuh"
#include "hap_host.h"

extern "C" {
#include "bc_oracle.h"
#include "hap_oracle.h"
}
#include <random>
#include <string>

using namespace hapb200;

struct Tex { std::vector<uint8_t> data; unsigned fmt, compressor, chunks; };

static uint64_t fnv(uint64_t h, const void *p, size_t n)
{
    const uint8_t *b = static_cast<const uint8_t *>(p);
    for (size_t i = 0; i < n; i++) { h ^= b[i]; h *= 0x100000001B3ull; }
    return h;
}

// encodes `tex` and returns the digest of the frame, the fragment sizes and (write_index bit 0) the fragment entries
static uint64_t encode_digest(const std::vector<Tex> &tex, int mode, unsigned grid, uint32_t write_index)
{
    TextureArgs ta[2];
    for (size_t i = 0; i < tex.size(); i++) ta[i] = TextureArgs{tex[i].data.size(), tex[i].fmt, tex[i].compressor, tex[i].chunks};
    FrameGeom G;
    if (build_frame_geom((uint32_t)tex.size(), ta, G) != 0) abort();
    size_t off1 = (tex[0].data.size() + 15) & ~(size_t)15;
    std::vector<uint8_t> in(off1 + (tex.size() > 1 ? tex[1].data.size() : 0));
    memcpy(in.data(), tex[0].data.data(), tex[0].data.size());
    if (tex.size() > 1) { memcpy(in.data() + off1, tex[1].data.data(), tex[1].data.size()); G.s[1].in_offset = off1; }
    unsigned long lens[2], cap;
    unsigned fmts[2], chunks[2];
    for (size_t i = 0; i < tex.size(); i++) { lens[i] = tex[i].data.size(); fmts[i] = tex[i].fmt; chunks[i] = tex[i].chunks; }
    cap = orc_HapMaxEncodedLength((unsigned)tex.size(), lens, fmts, chunks);
    std::vector<uint8_t> scratch((size_t)G.frags_per_frame * kFragCap), out(cap, 0xEE);
    std::vector<uint32_t> fsize(G.frags_per_frame), fdst(G.frags_per_frame), fidx(G.frags_per_frame);
    std::vector<uint8_t> fent((size_t)G.frags_per_frame * kFragEntryStride, 0xDD);
    unsigned long long used = 0;
    emu::g_order_mode() = mode;
    const unsigned k5_grid = G.frags_per_frame < grid ? G.frags_per_frame : grid;
    uint8_t *ent = (write_index & 1) ? fent.data() : nullptr;
    HAP_LAUNCH(snappy_encode_fragments_kernel, dim3(k5_grid), dim3(kEncThreads), sizeof(EncodeSmem), nullptr,
               in.data(), G, (uint32_t)G.frags_per_frame, scratch.data(), fsize.data(), ent);
    HAP_LAUNCH(hap_plan_frames_kernel, dim3(1), dim3(kPlanThreads), 0, nullptr, G, in.data(), fsize.data(), fdst.data(), fidx.data(),
               write_index, out.data(), (uint64_t)cap, &used);
    HAP_LAUNCH(hap_place_fragments_kernel, dim3(G.frags_per_frame), dim3(kPlaceThreads), 0, nullptr, G, in.data(),
               scratch.data(), fsize.data(), fdst.data(), fidx.data(), (const uint8_t *)ent, out.data(), (uint64_t)cap);
    if (used > cap) { fprintf(stderr, "used %llu > cap %lu\n", used, cap); abort(); }
    uint64_t h = 0xCBF29CE484222325ull;
    h = fnv(h, &used, sizeof used);
    h = fnv(h, out.data(), (size_t)used);
    h = fnv(h, fsize.data(), fsize.size() * 4);
    if (ent) h = fnv(h, fent.data(), fent.size());
    return h;
}

int main()
{
    // the case list of test_encode_emu.cc, built from the same seed in the same order
    std::mt19937 rng(777);
    const int W = 256, H = 128;
    std::vector<uint8_t> img(W * H * 4);
    for (int y = 0; y < H; y++)
        for (int x = 0; x < W; x++) {
            uint8_t *p = &img[4 * (y * W + x)];
            bool bar = y < 16 || y >= H - 16;
            for (int c = 0; c < 3; c++) p[c] = bar ? 16 : (uint8_t)(40 + (x * (c + 1)) % 160 + (y * 3) % 40 + (rng() % 4));
            p[3] = (uint8_t)(x);
        }
    auto blocks = [&](int kind) {
        std::vector<uint8_t> b((W / 4) * (H / 4) * (kind == 0 || kind == 3 ? 8 : 16));
        if (kind == 0) orc_bc1_encode_clusterfit(img.data(), W, H, b.data(), 1);
        else if (kind == 1) orc_bc3_encode_clusterfit(img.data(), W, H, b.data(), 1);
        else if (kind == 2) orc_ycocg_dxt5_encode_clusterfit(img.data(), W, H, b.data(), 1);
        else orc_bc4_encode_squish(img.data(), W, H, 3, b.data());
        return b;
    };
    std::vector<uint8_t> dxt1 = blocks(0), dxt5 = blocks(1), ycocg = blocks(2), rgtc = blocks(3);
    std::vector<uint8_t> noise(70000 - 70000 % 16), flat(16 * 5000);
    for (auto &b : noise) b = (uint8_t)rng();
    for (size_t i = 0; i < flat.size(); i++) flat[i] = (uint8_t)(0x30 + (i % 16));
    std::vector<uint8_t> big;
    for (int r = 0; r < 5; r++) big.insert(big.end(), ycocg.begin(), ycocg.end());
    for (size_t i = 0; i < big.size(); i += 977) big[i] ^= (uint8_t)rng();

    struct Case { std::string name; std::vector<Tex> tex; };
    std::vector<Case> cases = {
        {"dxt1_1chunk", {{dxt1, 0x83F0, 1, 1}}},
        {"dxt1_3chunks", {{dxt1, 0x83F0, 1, 3}}},
        {"dxt5_4chunks", {{dxt5, 0x83F3, 1, 4}}},
        {"ycocg_8chunks", {{ycocg, 0x01, 1, 8}}},
        {"ycocg_limit_7_to_x", {{ycocg, 0x01, 1, 7}}},
        {"rgtc_2chunks", {{rgtc, 0x8DBB, 1, 2}}},
        {"hapm", {{ycocg, 0x01, 1, 4}, {rgtc, 0x8DBB, 1, 2}}},
        {"hapm_mixed_none", {{ycocg, 0x01, 0, 4}, {rgtc, 0x8DBB, 1, 2}}},
        {"none_single", {{dxt5, 0x83F3, 0, 5}}},
        {"none_pair", {{ycocg, 0x01, 0, 1}, {rgtc, 0x8DBB, 0, 1}}},
        {"noise_fallback_whole", {{noise, 0x83F3, 1, 2}}},
        {"flat_rle", {{flat, 0x01, 1, 2}}},
        {"big_multi_fragment", {{big, 0x01, 1, 2}}},
        {"big_1chunk", {{big, 0x8E8C, 1, 1}}},
        {"tiny_16", {{std::vector<uint8_t>(16, 0x55), 0x01, 1, 1}}},
        {"tiny_8", {{std::vector<uint8_t>(8, 0x11), 0x83F0, 1, 1}}},
        {"kat_a_64x55", {{std::vector<uint8_t>(64, 0x55), 0x83F0, 1, 1}}},
    };
    {
        std::vector<uint8_t> mix(ycocg.begin(), ycocg.begin() + 16384);
        mix.insert(mix.end(), noise.begin(), noise.begin() + 16384);
        cases.push_back({"mixed_chunk_fallback", {{mix, 0x01, 1, 2}}});
    }
    for (int r = 0; r < 8; r++) {
        const size_t blocks16 = 200 + rng() % 12000;
        std::vector<uint8_t> v;
        while (v.size() < blocks16 * 16) {
            const int what = rng() % 5;
            const size_t n = 16 * (1 + rng() % 700);
            if (what == 0) { size_t at = (rng() % (ycocg.size() / 16 - n / 16 - 1)) * 16; v.insert(v.end(), ycocg.begin() + at, ycocg.begin() + at + n); }
            else if (what == 1 && v.size() >= 4096) { size_t at = v.size() - 16 * (1 + rng() % 200); for (size_t i = 0; i < n; i++) v.push_back(v[at + i % 16]); }
            else if (what == 2) { uint8_t b16[16]; for (auto &b : b16) b = (uint8_t)rng(); for (size_t i = 0; i < n; i++) v.push_back(b16[i % 16]); }
            else if (what == 3) { for (size_t i = 0; i < n; i++) v.push_back((uint8_t)rng()); }
            else { for (size_t i = 0; i < n; i++) v.push_back((uint8_t)((i / 16) & 0xFF)); }
        }
        v.resize(blocks16 * 16);
        cases.push_back({"random_" + std::to_string(r), {{v, 0x01, 1, (unsigned)(1 + rng() % 9)}}});
    }

    // resume order (forward, reverse, shuffled) x persistent grid (one CTA, or three striding CTAs)
    const int modes[3] = {0, 1, 2};
    const unsigned grids[2] = {1, 3};
    int fail = 0;
    for (auto &c : cases) {
        uint64_t all = 0xCBF29CE484222325ull;
        for (uint32_t wi = 0; wi < 4; wi++) {
            uint64_t first = 0;
            bool have = false;
            for (int m : modes)
                for (unsigned g : grids) {
                    const uint64_t h = encode_digest(c.tex, m, g, wi);
                    if (!have) { first = h; have = true; }
                    else if (h != first) { fprintf(stderr, "FAIL %s variant %u: mode %d grid %u gives %016llx, mode 0 grid 1 %016llx\n",
                                                   c.name.c_str(), wi, m, g, (unsigned long long)h, (unsigned long long)first); fail++; }
                }
            all = fnv(all, &first, sizeof first);
        }
        printf("%s %016llx\n", c.name.c_str(), (unsigned long long)all);
    }
    return fail ? 1 : 0;
}
