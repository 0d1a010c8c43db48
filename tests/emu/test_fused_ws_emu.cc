// tests/emu/test_fused_ws_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The fused Hap Q encoder with its fit and its compressor in warp groups of their own (hapq_ws_place_kernel: 1 024 threads,
// two shared-memory images, named barriers) under the fiber SIMT emulator, against hapq_fused_place_kernel on the same
// pictures; both are followed by hap_plan_placed_frames_kernel and hap_place_listed_kernel.  Every byte of every output slot
// (filled with a sentinel first, so a write past a frame's end shows), the frame lengths, the fragment sizes, the index
// entries, the written-through texture and the scratch slots must be identical, with the fragment index on and off, in every
// fiber resume order (forward, reverse, seeded shuffles), with a grid of one CTA (it holds every ticket, so both fragments
// of its pipeline meet the look-back) and of three CTAs, and launched with more CTAs than fragments.  The cases: one short
// fragment; partial last fragments and fragments that start mid-row; 1 to 64 chunks; one noise chunk at the first, a middle
// and the last chunk position (per-chunk raw fallback, hap.c:460); all-noise frames (whole-section fallback, hap.c:478);
// frames whose compressed body ends past where a verbatim section would end.  Buffers are exactly as long as the last frame
// needs (under ASan, any access outside them fails).
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

constexpr uint8_t kSentinel = 0xEE, kScratchSentinel = 0xCC;

struct Case {
    std::string name;
    uint32_t w, h, frames, chunks;
    int content;            // 0 picture, 1 flat, 2 noise, 3 picture with chunk `arg` noise, 4 noise but `arg` flat blocks opening the last chunk
    int arg;
    uint32_t pad_row, pad_frame;
};

struct Encoded {
    std::vector<uint8_t> out, tex, ent, scratch;
    std::vector<uint32_t> fsize, fdst;
    std::vector<unsigned long long> used;
    uint32_t listed = 0;   // fragments listed for the place kernel
};

// The pictures of a case: exactly as long as the last frame's last row
std::vector<uint8_t> pictures(const Case &c, uint32_t row, uint64_t fstride)
{
    std::vector<uint8_t> b((c.frames - 1) * fstride + (uint64_t)(c.h - 1) * row + 4ull * c.w, 0xA5);
    g_rng = 0x2545F4914F6CDD1Dull;   // (every case's content is its own, whatever runs before it)
    const uint64_t nblk = (uint64_t)(c.w / 4) * (c.h / 4);
    for (uint32_t f = 0; f < c.frames; f++)
        for (uint32_t y = 0; y < c.h; y++)
            for (uint32_t x = 0; x < c.w; x++) {
                uint8_t *p = &b[f * fstride + (uint64_t)y * row + 4ull * x];
                const uint64_t blk = (uint64_t)(y / 4) * (c.w / 4) + x / 4;
                bool noise = c.content == 2;
                if (c.content == 3) noise = (int)(blk * c.chunks / nblk) == c.arg;
                if (c.content == 4) noise = blk < (c.chunks - 1) * nblk / c.chunks || blk >= (c.chunks - 1) * nblk / c.chunks + (uint64_t)c.arg;
                if (noise) { const uint32_t r = rnd(); memcpy(p, &r, 4); }
                else if (c.content == 1 || c.content == 4) { p[0] = (uint8_t)(16 + 9 * f); p[1] = 128; p[2] = 200; p[3] = 255; }
                else {
                    const bool bar = y < 8 || y + 8 >= c.h;
                    for (int k = 0; k < 3; k++) p[k] = bar ? 16 : (uint8_t)(40 + (x * (k + 1) + f * 5) % 160 + (y * 3) % 40 + (rnd() % 3));
                    p[3] = (uint8_t)x;
                }
            }
    return b;
}

// ws: hapq_ws_place_kernel on `grid` CTAs (not clamped to the fragments), else hapq_fused_place_kernel; then
// hap_plan_placed_frames_kernel and hap_place_listed_kernel.
Encoded encode(const Case &c, const std::vector<uint8_t> &rgba, uint32_t row, uint64_t fstride, bool ws, uint32_t flags, unsigned grid, int mode)
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
    e.tex.assign((c.frames - 1) * stride + n, kSentinel);
    e.out.assign((c.frames - 1) * (uint64_t)cap + cap, kSentinel);
    e.fsize.assign(nfrag, 0);
    e.ent.assign((size_t)nfrag * kFragEntryStride, 0xDD);
    e.used.assign(c.frames, 0);
    e.scratch.assign((size_t)nfrag * kFragCap, kScratchSentinel);
    e.fdst.assign(nfrag, 0);
    std::vector<uint32_t> fidx(nfrag);
    uint8_t *ent = (flags & kPlanWriteIndex) ? e.ent.data() : nullptr;
    const BcGeom B = bc_encode_geom(c.w, c.h, row, fstride, stride, 0);
    emu::g_order_mode() = mode;
    std::vector<uint32_t> sync(2 + 2 * (size_t)nfrag, 0), work(nfrag, 0xFFFFFFFFu);
    const FusedPlaceArgs P{e.out.data(), (uint64_t)cap, sync.data(), sync.data() + 2, sync.data() + 2 + nfrag};
    if (ws)
        HAP_LAUNCH(hapq_ws_place_kernel, dim3(grid), dim3(kWsThreads), sizeof(WsSmem), nullptr, rgba.data(), B, e.tex.data(), G, nfrag,
                   e.scratch.data(), e.fsize.data(), ent, P);
    else
        HAP_LAUNCH(hapq_fused_place_kernel, dim3(nfrag < grid ? nfrag : grid), dim3(kEncThreads), sizeof(EncodeSmem), nullptr, rgba.data(), B,
                   e.tex.data(), G, nfrag, e.scratch.data(), e.fsize.data(), ent, P);
    if (sync[0] < nfrag) fail(c.name + ": tickets left");
    HAP_LAUNCH(hap_plan_placed_frames_kernel, dim3(c.frames), dim3(kPlanThreads), 0, nullptr, G, e.tex.data(), e.fsize.data(),
               e.fdst.data(), fidx.data(), flags, e.out.data(), (uint64_t)cap, e.used.data(),
               PlanPlaced{e.scratch.data(), ent, work.data(), sync.data() + 1});
    HAP_LAUNCH(hap_place_listed_kernel, dim3(grid), dim3(kPlaceThreads), 0, nullptr, G, e.tex.data(), e.fsize.data(), e.fdst.data(),
               work.data(), sync.data() + 1, e.out.data(), (uint64_t)cap);
    e.listed = sync[1];
    for (uint32_t f = 0; f < c.frames; f++)
        if (e.used[f] > cap) fail(c.name + ": frame longer than its bound");
    return e;
}

}  // namespace

int main(int argc, char **argv)
{
    const int modes = argc > 1 ? atoi(argv[1]) : 3;
    const Case cases[] = {
        {"one_fragment_short", 132, 132, 1, 1, 0, 0, 0, 0},          // 1 089 blocks: one short fragment, fewer fragments than CTAs
        {"two_fragments", 260, 200, 1, 1, 0, 0, 16, 272},             // 65 blocks per row: the second fragment starts mid-row
        {"eight_chunks_wide_frames", 512, 256, 3, 8, 0, 0, 48, 4096},
        {"sixtyfour_chunks", 520, 520, 1, 64, 0, 0, 0, 0},            // 16 900 blocks: 64 requested, 52 chunks of 5 200 bytes
        {"flat", 256, 128, 2, 8, 1, 0, 0, 0},
        {"noise_first_chunk", 512, 256, 2, 8, 3, 0, 0, 16},
        {"noise_middle_chunk", 512, 256, 1, 8, 3, 3, 0, 0},
        {"noise_last_chunk", 512, 256, 2, 8, 3, 7, 0, 0},
        {"noise_whole_section", 256, 256, 2, 1, 2, 0, 0, 0},
        {"big_two_fragments_per_chunk", 1028, 256, 1, 3, 0, 0, 0, 0},   // a full and a partial fragment per chunk
        {"body_past_verbatim_end_three_chunks", 256, 128, 1, 3, 4, 3, 0, 0},
    };
    int runs = 0;
    for (const Case &c : cases) {
        const uint32_t row = 4 * c.w + c.pad_row;
        const uint64_t fstride = (uint64_t)c.h * row + c.pad_frame;
        const std::vector<uint8_t> rgba = pictures(c, row, fstride);
        for (uint32_t flags : {0u, kPlanWriteIndex}) {
            const Encoded want = encode(c, rgba, row, fstride, false, flags, 3, 0);
            for (int mode = 0; mode < modes; mode++)
                for (unsigned grid : {1u, 3u}) {
                    if (mode > 1 && flags != 0) continue;   // (every order with the index off, forward and reverse with it on)
                    const Encoded got = encode(c, rgba, row, fstride, true, flags, grid, mode);
                    const std::string what = c.name + " flags " + std::to_string(flags) + " mode " + std::to_string(mode) + " grid " + std::to_string(grid);
                    if (got.used != want.used) fail(what + ": frame sizes differ");
                    else if (got.out != want.out) fail(what + ": frames (or the bytes behind them) differ");
                    if (got.fsize != want.fsize) fail(what + ": fragment sizes differ");
                    if ((flags & kPlanWriteIndex) && got.ent != want.ent) fail(what + ": fragment index entries differ");
                    if (got.tex != want.tex) fail(what + ": written-through texture differs");
                    if (got.scratch != want.scratch) fail(what + ": scratch slots differ");
                    if (got.listed != want.listed) fail(what + ": " + std::to_string(got.listed) + " fragments listed, not " + std::to_string(want.listed));
                    runs++;
                }
        }
    }
    printf("%d warp-group encodes compared, %d failures\n", runs, g_fail);
    return g_fail ? 1 : 0;
}
