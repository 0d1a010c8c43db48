// tests/emu/test_fused_place_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The fused Hap Q encoder that writes its element streams into the frames itself (hapq_fused_place_kernel, then
// hap_plan_placed_frames_kernel and hap_place_listed_kernel) under the fiber SIMT emulator, against the fused kernel that
// leaves them in scratch for hap_plan_frames_kernel and hap_place_fragments_kernel.  Every byte of every output slot
// (filled with a sentinel first, so a write past a frame's end shows), the frame lengths, the fragment sizes, the index
// entries and the written-through texture must be identical, with the fragment index on and off, in several fiber resume
// orders and with a persistent grid of 1 or 3 CTAs.  The cases: compressible frames; one noise chunk at the first, a middle
// and the last chunk position (per-chunk raw fallback, hap.c:460); all-noise frames (whole-section fallback, hap.c:478);
// frames whose compressed body ends in [bytes, bytes + top_hdr), past where a verbatim section would end; 1 to 64 chunks,
// short last fragments, fragments that start mid-row, frames laid out wider than they are.  Buffers are exactly as long as
// the last frame needs (under ASan, any access outside them fails).  That the streams did not go through scratch is
// checked too: in frames without raw chunks only a fragment that ends past a verbatim section's end touches its scratch
// slot, and exactly the raw fragments are listed for the place kernel.
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
    std::vector<uint8_t> out, tex, ent;
    std::vector<uint32_t> fsize, fdst;
    std::vector<unsigned long long> used;
    uint32_t listed = 0, kept = 0;   // fragments listed for the place kernel; fragments that touched their scratch slot
    uint32_t top_hdr = 0, bytes = 0;
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

// placed: hapq_fused_place_kernel, hap_plan_placed_frames_kernel, hap_place_listed_kernel; else hapq_fused_encode_kernel,
// hap_plan_frames_kernel, hap_place_fragments_kernel.
Encoded encode(const Case &c, const std::vector<uint8_t> &rgba, uint32_t row, uint64_t fstride, bool placed, uint32_t flags, unsigned grid,
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
    e.top_hdr = G.s[0].top_hdr;
    e.bytes = G.s[0].bytes;
    e.tex.assign((c.frames - 1) * stride + n, kSentinel);
    e.out.assign((c.frames - 1) * (uint64_t)cap + cap, kSentinel);
    e.fsize.assign(nfrag, 0);
    e.ent.assign((size_t)nfrag * kFragEntryStride, 0xDD);
    e.used.assign(c.frames, 0);
    std::vector<uint8_t> scratch((size_t)nfrag * kFragCap, kScratchSentinel);
    e.fdst.assign(nfrag, 0);
    std::vector<uint32_t> fidx(nfrag);
    uint8_t *ent = (flags & kPlanWriteIndex) ? e.ent.data() : nullptr;
    const BcGeom B = bc_encode_geom(c.w, c.h, row, fstride, stride, 0);
    emu::g_order_mode() = mode;
    const unsigned g = nfrag < grid ? nfrag : grid;
    if (placed) {
        std::vector<uint32_t> sync(2 + 2 * (size_t)nfrag, 0), work(nfrag, 0xFFFFFFFFu);
        const FusedPlaceArgs P{e.out.data(), (uint64_t)cap, sync.data(), sync.data() + 2, sync.data() + 2 + nfrag};
        HAP_LAUNCH(hapq_fused_place_kernel, dim3(g), dim3(kEncThreads), sizeof(EncodeSmem), nullptr, rgba.data(), B, e.tex.data(), G, nfrag,
                   scratch.data(), e.fsize.data(), ent, P);
        HAP_LAUNCH(hap_plan_placed_frames_kernel, dim3(c.frames), dim3(kPlanThreads), 0, nullptr, G, e.tex.data(), e.fsize.data(),
                   e.fdst.data(), fidx.data(), flags, e.out.data(), (uint64_t)cap, e.used.data(),
                   PlanPlaced{scratch.data(), ent, work.data(), sync.data() + 1});
        HAP_LAUNCH(hap_place_listed_kernel, dim3(grid), dim3(kPlaceThreads), 0, nullptr, G, e.tex.data(), e.fsize.data(), e.fdst.data(),
                   work.data(), sync.data() + 1, e.out.data(), (uint64_t)cap);
        e.listed = sync[1];
        for (uint32_t i = 0; i < e.listed; i++)
            if (work[i] >= nfrag || !(e.fdst[work[i]] & kPlaceRawFlag)) fail(c.name + ": a listed fragment is not raw");
        if (sync[0] < nfrag) fail(c.name + ": tickets left");
    } else {
        HAP_LAUNCH(hapq_fused_encode_kernel, dim3(g), dim3(kEncThreads), sizeof(EncodeSmem), nullptr, rgba.data(), B, e.tex.data(), G, nfrag,
                   scratch.data(), e.fsize.data(), ent);
        HAP_LAUNCH(hap_plan_frames_kernel, dim3(c.frames), dim3(kPlanThreads), 0, nullptr, G, e.tex.data(), e.fsize.data(), e.fdst.data(),
                   fidx.data(), flags, e.out.data(), (uint64_t)cap, e.used.data());
        HAP_LAUNCH(hap_place_fragments_kernel, dim3(nfrag), dim3(kPlaceThreads), 0, nullptr, G, e.tex.data(), scratch.data(), e.fsize.data(),
                   e.fdst.data(), fidx.data(), (const uint8_t *)ent, e.out.data(), (uint64_t)cap);
    }
    for (uint32_t i = 0; i < nfrag; i++)
        for (uint32_t q = 0; q < (uint32_t)kFragCap; q++)
            if (scratch[(size_t)i * kFragCap + q] != kScratchSentinel) { e.kept++; break; }
    for (uint32_t f = 0; f < c.frames; f++)
        if (e.used[f] > cap) fail(c.name + ": frame longer than its bound");
    return e;
}

}  // namespace

int main(int argc, char **argv)
{
    const int modes = argc > 1 ? atoi(argv[1]) : 3;
    // content 4: the number of flat blocks puts the compressed body of the frame (index off) between `bytes` and
    // `bytes + top_hdr`: the frame ends past where the verbatim section would have ended (checked below)
    const Case cases[] = {
        {"one_fragment_short", 132, 132, 1, 1, 0, 0, 0, 0},          // 1 089 blocks: one short fragment
        {"mid_row_starts", 260, 200, 2, 1, 0, 0, 16, 272},            // 65 blocks per row: the second fragment starts mid-row
        {"eight_chunks_wide_frames", 512, 256, 3, 8, 0, 0, 48, 4096},
        {"sixtyfour_chunks", 520, 520, 1, 64, 0, 0, 0, 0},            // 16 900 blocks: 64 requested, 52 chunks of 5 200 bytes
        {"flat", 256, 128, 2, 8, 1, 0, 0, 0},
        {"noise_first_chunk", 512, 256, 2, 8, 3, 0, 0, 16},
        {"noise_middle_chunk", 512, 256, 1, 8, 3, 3, 0, 0},
        {"noise_last_chunk", 512, 256, 2, 8, 3, 7, 0, 0},
        {"noise_one_of_three", 516, 132, 1, 3, 3, 1, 0, 0},           // 129 x 33 blocks
        {"noise_whole_section", 256, 256, 2, 1, 2, 0, 0, 0},
        {"noise_whole_section_eight_chunks", 512, 256, 1, 8, 2, 0, 0, 0},
        {"big_two_fragments_per_chunk", 1028, 256, 1, 3, 0, 0, 0, 0},
        {"body_past_verbatim_end_three_chunks", 256, 128, 1, 3, 4, 3, 0, 0},
        {"body_past_verbatim_end_six_chunks", 96, 96, 1, 6, 4, 4, 0, 0},
    };
    int runs = 0;
    for (const Case &c : cases) {
        const uint32_t row = 4 * c.w + c.pad_row;
        const uint64_t fstride = (uint64_t)c.h * row + c.pad_frame;
        const std::vector<uint8_t> rgba = pictures(c, row, fstride);
        for (uint32_t flags : {0u, kPlanWriteIndex}) {
            const Encoded want = encode(c, rgba, row, fstride, false, flags, 3, 0);
            uint32_t raw = 0;
            for (uint32_t d : want.fdst) raw += (d & kPlaceRawFlag) ? 1u : 0u;
            bool past_verbatim_end = false;
            for (unsigned long long u : want.used) past_verbatim_end = past_verbatim_end || u > (unsigned long long)want.top_hdr + want.bytes;
            if (c.content == 4 && flags == 0 && !past_verbatim_end) fail(c.name + ": the frame does not end past the verbatim end");
            for (int mode = 0; mode < modes; mode++)
                for (unsigned grid : {1u, 3u}) {
                    if (mode > 0 && grid == 1 && flags != 0) continue;   // (every order and grid once, every variant at grid 3)
                    const Encoded got = encode(c, rgba, row, fstride, true, flags, grid, mode);
                    const std::string what = c.name + " flags " + std::to_string(flags) + " mode " + std::to_string(mode) + " grid " + std::to_string(grid);
                    if (got.used != want.used) fail(what + ": frame sizes differ");
                    else if (got.out != want.out) fail(what + ": frames (or the bytes behind them) differ");
                    if (got.fsize != want.fsize) fail(what + ": fragment sizes differ");
                    if ((flags & kPlanWriteIndex) && got.ent != want.ent) fail(what + ": fragment index entries differ");
                    if (got.tex != want.tex) fail(what + ": written-through texture differs");
                    if (got.listed != raw) fail(what + ": " + std::to_string(got.listed) + " fragments listed, " + std::to_string(raw) + " raw");
                    // (a fragment of a raw chunk may keep back bytes that are never used)
                    if (raw == 0 && got.kept > (past_verbatim_end ? c.frames : 0u)) fail(what + ": " + std::to_string(got.kept) + " streams went through scratch");
                    if (c.content == 4 && flags == 0 && got.kept == 0) fail(what + ": no stream bytes kept back past the verbatim end");
                    runs++;
                }
        }
    }
    printf("%d placed encodes compared, %d failures\n", runs, g_fail);
    return g_fail ? 1 : 0;
}
