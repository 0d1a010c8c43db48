// tests/emu/test_fused_hapq_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The fused Hap Q encoder (hapq_fused.cuh) under the fiber SIMT emulator against the two-kernel path it replaces:
// bc_encode_kernel<kBcYCoCg> into a texture, then snappy_encode_fragments_kernel (K5), each followed by the plan and place
// kernels.  The frame, the fragment sizes, the fragment index entries and the texture the fused kernel writes through must
// be byte-identical to the two-kernel path's, for every frame of the batch, with the fragment index and the offset table
// each on and off, in several fiber resume orders and with a persistent grid of 1 or 3 CTAs.  The cases put fragment
// starts mid-row, leave last fragments short, use 1, 3, 8 and 64 chunks, lay frames out wider than they are, and include
// flat content and noise (the chunk and whole-section fallbacks, which copy the written-through texture).  Buffers are
// exactly as long as the last frame needs (under ASan, any access outside them fails).  The selection rule
// (fused_hapq_geometry) is checked on geometries just outside it.
#define HAPB200_EMU
#include "hap_assemble.cuh"
#include "hap_host.h"
#include "hapq_fused.cuh"

extern "C" {
#include "hap_oracle.h"
}
#include <string>
#include <vector>

using namespace hapb200;

namespace {

int g_fail = 0;
uint64_t g_rng = 0x2545F4914F6CDD1Dull;
uint32_t rnd()
{
    g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17;
    return (uint32_t)(g_rng >> 11);
}

void fail(const std::string &what)
{
    if (g_fail++ < 20) fprintf(stderr, "FAIL %s\n", what.c_str());
}

struct Case {
    std::string name;
    uint32_t w, h, frames, chunks;
    int content;            // 0 picture, 1 flat, 2 noise, 3 picture on top and noise below
    uint32_t pad_row, pad_frame;
};

struct Encoded {
    std::vector<uint8_t> out, tex, ent;
    std::vector<uint32_t> fsize;
    std::vector<unsigned long long> used;
};

// The pictures of a case: exactly as long as the last frame's last row
std::vector<uint8_t> pictures(const Case &c, uint32_t row, uint64_t fstride)
{
    std::vector<uint8_t> b((c.frames - 1) * fstride + (uint64_t)(c.h - 1) * row + 4ull * c.w, 0xA5);
    for (uint32_t f = 0; f < c.frames; f++)
        for (uint32_t y = 0; y < c.h; y++)
            for (uint32_t x = 0; x < c.w; x++) {
                uint8_t *p = &b[f * fstride + (uint64_t)y * row + 4ull * x];
                const bool noise = c.content == 2 || (c.content == 3 && y >= c.h / 2);
                if (noise) { const uint32_t r = rnd(); memcpy(p, &r, 4); }
                else if (c.content == 1) { p[0] = (uint8_t)(16 + 9 * f); p[1] = 128; p[2] = 200; p[3] = 255; }
                else {
                    const bool bar = y < 8 || y + 8 >= c.h;
                    for (int k = 0; k < 3; k++) p[k] = bar ? 16 : (uint8_t)(40 + (x * (k + 1) + f * 5) % 160 + (y * 3) % 40 + (rnd() % 3));
                    p[3] = (uint8_t)x;
                }
            }
    return b;
}

// fused: one launch of hapq_fused_encode_kernel; else bc_encode_kernel<kBcYCoCg>, then K5.  Then plan and place.
Encoded encode(const Case &c, const std::vector<uint8_t> &rgba, uint32_t row, uint64_t fstride, bool fused, uint32_t flags, unsigned grid,
               int mode)
{
    const uint64_t n = (uint64_t)(c.w / 4) * (c.h / 4) * 16, stride = (n + 15) & ~15ull;
    TextureArgs ta{n, HapFmt_YCoCg_DXT5, HapCompressorSnappy, c.chunks};
    FrameGeom G;
    if (build_frame_geom(1, &ta, G) != 0) abort();
    G.s[0].in_offset = 0;
    G.s[0].in_stride = stride;
    if (!fused_hapq_geometry(G)) { fail(c.name + ": outside the selection rule"); return {}; }
    unsigned long lens[1] = {(unsigned long)n};
    unsigned fmts[1] = {HapFmt_YCoCg_DXT5}, chunks[1] = {c.chunks};
    const unsigned long cap = orc_HapMaxEncodedLength(1, lens, fmts, chunks);
    const uint32_t nfrag = c.frames * G.frags_per_frame;
    Encoded e;
    e.tex.assign((c.frames - 1) * stride + n, 0xEE);
    e.out.assign((c.frames - 1) * (uint64_t)cap + cap, 0xEE);
    e.fsize.assign(nfrag, 0);
    e.ent.assign((size_t)nfrag * kFragEntryStride, 0xDD);
    e.used.assign(c.frames, 0);
    std::vector<uint8_t> scratch((size_t)nfrag * kFragCap);
    std::vector<uint32_t> fdst(nfrag), fidx(nfrag);
    uint8_t *ent = (flags & kPlanWriteIndex) ? e.ent.data() : nullptr;
    const BcGeom B = bc_encode_geom(c.w, c.h, row, fstride, stride, 0);
    emu::g_order_mode() = mode;
    const unsigned g = nfrag < grid ? nfrag : grid;
    if (fused) {
        HAP_LAUNCH(hapq_fused_encode_kernel, dim3(g), dim3(kEncThreads), sizeof(EncodeSmem), nullptr, rgba.data(), B, e.tex.data(), G, nfrag,
                   scratch.data(), e.fsize.data(), ent);
    } else {
        HAP_LAUNCH((bc_encode_kernel<kBcYCoCg>), dim3(bc_ctas(B.blocks_x, B.blocks_y), c.frames), dim3(kBcThreads), 0, nullptr, rgba.data(), B,
                   e.tex.data());
        HAP_LAUNCH(snappy_encode_fragments_kernel, dim3(g), dim3(kEncThreads), sizeof(EncodeSmem), nullptr, e.tex.data(), G, nfrag,
                   scratch.data(), e.fsize.data(), ent);
    }
    HAP_LAUNCH(hap_plan_frames_kernel, dim3(c.frames), dim3(kPlanThreads), 0, nullptr, G, e.tex.data(), e.fsize.data(), fdst.data(),
               fidx.data(), flags, e.out.data(), (uint64_t)cap, e.used.data());
    HAP_LAUNCH(hap_place_fragments_kernel, dim3(nfrag), dim3(kPlaceThreads), 0, nullptr, G, e.tex.data(), scratch.data(), e.fsize.data(),
               fdst.data(), fidx.data(), (const uint8_t *)ent, e.out.data(), (uint64_t)cap);
    for (uint32_t f = 0; f < c.frames; f++)
        if (e.used[f] > cap) fail(c.name + ": frame longer than its bound");
    return e;
}

}  // namespace

int main(int argc, char **argv)
{
    const int modes = argc > 1 ? atoi(argv[1]) : 3;
    const Case cases[] = {
        {"one_fragment_short", 132, 132, 1, 1, 0, 0, 0},        // 1 089 blocks: one short fragment
        {"mid_row_starts", 260, 200, 2, 1, 0, 16, 272},          // 65 blocks per row: the second fragment starts mid-row
        {"three_chunks", 516, 132, 2, 3, 3, 0, 0},               // 129 x 33 blocks, chunk and fragment fallbacks
        {"eight_chunks_wide_frames", 512, 256, 3, 8, 0, 48, 4096},
        {"sixtyfour_chunks", 520, 520, 1, 64, 0, 0, 0},          // 16 900 blocks: 64 requested, 52 chunks of 5 200 bytes
        {"flat", 256, 128, 2, 8, 1, 0, 0},
        {"noise_whole_section", 256, 256, 1, 1, 2, 0, 0},
        {"noise_chunks", 512, 256, 1, 8, 3, 0, 16},
        {"big_two_fragments_per_chunk", 1028, 256, 1, 3, 0, 0, 0},
    };
    int runs = 0;
    for (const Case &c : cases) {
        const uint32_t row = 4 * c.w + c.pad_row;
        const uint64_t fstride = (uint64_t)c.h * row + c.pad_frame;
        const std::vector<uint8_t> rgba = pictures(c, row, fstride);
        for (uint32_t flags : {0u, kPlanWriteIndex, kPlanWriteOffsets, kPlanWriteIndex | kPlanWriteOffsets}) {
            const Encoded want = encode(c, rgba, row, fstride, false, flags, 3, 0);
            for (int mode = 0; mode < modes; mode++)
                for (unsigned grid : {1u, 3u}) {
                    if (mode > 0 && grid == 1 && flags != 0) continue;   // (every order and grid once, every variant at grid 3)
                    const Encoded got = encode(c, rgba, row, fstride, true, flags, grid, mode);
                    const std::string what = c.name + " flags " + std::to_string(flags) + " mode " + std::to_string(mode) + " grid " + std::to_string(grid);
                    if (got.used != want.used) fail(what + ": frame sizes differ");
                    else if (got.out != want.out) fail(what + ": frames differ");
                    if (got.fsize != want.fsize) fail(what + ": fragment sizes differ");
                    if ((flags & kPlanWriteIndex) && got.ent != want.ent) fail(what + ": fragment index entries differ");
                    if (got.tex != want.tex) fail(what + ": written-through texture differs");
                    runs++;
                }
        }
    }
    // the selection rule: the two-texture layout, an uncompressed section and 8-byte blocks whose chunks end mid-block fall outside it
    {
        TextureArgs y{16 * 4096, HapFmt_YCoCg_DXT5, HapCompressorSnappy, 4}, a{8 * 4096, HapFmt_A_RGTC1, HapCompressorSnappy, 2};
        TextureArgs pair[2] = {y, a};
        FrameGeom G;
        if (build_frame_geom(1, &y, G) != 0 || !fused_hapq_geometry(G)) fail("rule: a Hap Q texture in whole chunks");
        if (build_frame_geom(2, pair, G) != 0 || fused_hapq_geometry(G)) fail("rule: two textures");
        TextureArgs none{16 * 4096, HapFmt_YCoCg_DXT5, HapCompressorNone, 4};
        if (build_frame_geom(1, &none, G) != 0 || fused_hapq_geometry(G)) fail("rule: no compressor");
        TextureArgs odd{8 * 3, HapFmt_RGB_DXT1, HapCompressorSnappy, 3};    // chunks of one 8-byte block
        if (build_frame_geom(1, &odd, G) != 0 || fused_hapq_geometry(G)) fail("rule: chunks of 8 bytes");
    }
    printf("%d fused encodes compared, %d failures\n", runs, g_fail);
    return g_fail ? 1 : 0;
}
