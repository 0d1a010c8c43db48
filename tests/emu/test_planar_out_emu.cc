// tests/emu/test_planar_out_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The planar sink of K8 (bc_decode_planar_kernel and bc_decode_planar_alpha_kernel, planar_sink.cuh) under the fiber SIMT
// emulator: every instantiation (DXT1, DXT5, scaled YCoCg with and without its RGTC1 alpha texture, BC7 x 4:2:0 / 4:2:2 /
// 4:4:4 x bytes / 16-bit words, and RGTC1 to the alpha plane alone on bytes and words), at block widths 1, 2, 30, 31, 32, 33,
// 62, 63, 64 and 129 (the halo lane at row starts, row ends and warp-span boundaries), heights of 1, 2 and 3 block rows, luma
// and chroma pitches wider than their rows and different from each other, three frames with slack between them, and a failed
// middle frame.  Depth (10 / 12 for words), colour space and the alpha plane's presence alternate with the shapes.  Every plane
// is a buffer of its own that ends with the last frame's last sample, so a store past a plane leaves every buffer under ASan;
// Hap Alpha-Only runs with no luma, Cb or Cr buffer at all.  Every sample must equal the sample-by-sample conversion of
// planar_out_twin.h applied to decode_block's texels (zeros for the failed frame), and every other byte must keep its sentinel.
#define HAPB200_EMU
#include "planar_out_twin.h"

#include <string>
#include <vector>

using namespace hapb200;

namespace {

constexpr uint32_t kFrames = 3;
constexpr uint8_t kPad = 0xA5;
int g_fail = 0;
int g_runs = 0;

uint64_t g_rng = 0x243F6A8885A308D3ull;
uint32_t rnd()
{
    g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17;
    return (uint32_t)(g_rng >> 11);
}

void fail(const std::string &what)
{
    if (g_fail++ < 20) fprintf(stderr, "FAIL %s\n", what.c_str());
}

struct Shape {
    uint32_t bw, bh, lpad, cpad, n, cs;
    bool alpha;
};

// KIND kBcRgtc1: Hap Alpha-Only (the alpha kernel); kBcYCoCgPlusAlpha: Hap Q Alpha (the YCoCg kernel merging its RGTC1 texture
// when there is an alpha plane)
template <int KIND, int SUB, bool WIDE>
void check(const Shape &s)
{
    const bool alpha_only = KIND == kBcRgtc1, alpha = s.alpha || alpha_only;
    const uint32_t w = 4 * s.bw, h = 4 * s.bh, sb = WIDE ? 2 : 1, n = WIDE ? s.n : 8;
    const uint32_t cw = SUB == HapB200Chroma_444 ? w : w / 2, ch = SUB == HapB200Chroma_420 ? h / 2 : h;
    const uint32_t lpitch = sb * w + s.lpad, cpitch = sb * cw + s.cpad;
    const uint64_t block_bytes = KIND == kBcDxt1 || KIND == kBcRgtc1 ? 8 : 16;
    const uint64_t nblk = (uint64_t)s.bw * s.bh, first = (nblk * block_bytes + 15) / 16 * 16;
    const uint64_t in_stride = first + (KIND == kBcYCoCgPlusAlpha ? (nblk * 8 + 15) / 16 * 16 : 0) + 32;
    std::vector<uint8_t> in(kFrames * in_stride);
    for (auto &b : in) b = (uint8_t)rnd();
    const uint64_t luma_rows = (uint64_t)h * lpitch, chroma_rows = (uint64_t)ch * cpitch;
    const uint64_t frame_bytes = (luma_rows > chroma_rows ? luma_rows : chroma_rows) + 48;
    auto plane_end = [&](uint32_t rows, uint32_t pitch, uint32_t samples) {
        return (kFrames - 1) * frame_bytes + (uint64_t)(rows - 1) * pitch + (uint64_t)sb * samples;
    };
    const uint64_t lsize = plane_end(h, lpitch, w), csize = plane_end(ch, cpitch, cw);
    std::vector<uint8_t> lbuf(alpha_only ? 0 : lsize, kPad), cbbuf(alpha_only ? 0 : csize, kPad), crbuf(alpha_only ? 0 : csize, kPad),
        abuf(alpha ? lsize : 0, kPad);
    const uint32_t results[kFrames] = {0, 7 /* a failed frame */, 0};
    PlanarOut P;
    P.g = yuv_out_geom(w, h, lpitch, in_stride, frame_bytes, planar_out_coeffs(n, s.cs));
    P.cb = alpha_only ? nullptr : cbbuf.data();
    P.cr = alpha_only ? nullptr : crbuf.data();
    P.alpha = alpha ? abuf.data() : nullptr;
    P.chroma_pitch = cpitch;
    P.merge_alpha = KIND == kBcYCoCgPlusAlpha && alpha ? 1u : 0u;
    P.second_offset = first;
    if (alpha_only) {
        HAP_LAUNCH((bc_decode_planar_alpha_kernel<WIDE>), dim3(bc_ctas(s.bw, s.bh), kFrames), dim3(kBcThreads), 0, nullptr, in.data(), P, results);
    } else {
        constexpr int kKind = KIND == kBcYCoCgPlusAlpha ? kBcYCoCg : KIND;
        const unsigned ctas = SUB == HapB200Chroma_444 ? bc_ctas(s.bw, s.bh) : (unsigned)yuv_out_ctas(P.g);
        HAP_LAUNCH((bc_decode_planar_kernel<kKind, SUB, WIDE>), dim3(ctas, kFrames), dim3(kBcThreads), 0, nullptr, in.data(), P, lbuf.data(),
                   results);
    }
    // expected: the twin on the decoded picture, written into sentinel buffers of the same shape
    std::vector<uint8_t> wl(lbuf.size(), kPad), wcb(cbbuf.size(), kPad), wcr(crbuf.size(), kPad), wa(abuf.size(), kPad);
    std::vector<uint8_t> rgba(4ull * w * h);
    for (uint32_t f = 0; f < kFrames; f++) {
        for (uint32_t by = 0; by < s.bh; by++)
            for (uint32_t bx = 0; bx < s.bw; bx++) {
                uint32_t px[16] = {0};
                const uint64_t bi = (uint64_t)by * s.bw + bx;
                if (results[f] == 0) {
                    uint32_t v[4] = {0, 0, 0, 0};
                    memcpy(v, &in[f * in_stride + bi * block_bytes], block_bytes);
                    decode_block(KIND == kBcYCoCgPlusAlpha ? kBcYCoCg : KIND, v[0], v[1], v[2], v[3], px);
                    if (KIND == kBcYCoCgPlusAlpha && alpha) {
                        uint32_t a[2], rows[4];
                        memcpy(a, &in[f * in_stride + first + bi * 8], 8);
                        bc4_rows(a[0], a[1], rows);
                        for (int t = 0; t < 16; t++) px[t] = (px[t] & 0x00FFFFFFu) | (uint32_t)byte_of(rows[t / 4], t % 4) << 24;
                    }
                    if (alpha_only)   // the matte is the value decode_block writes to R, G and B
                        for (int t = 0; t < 16; t++) px[t] = (px[t] & 0x00FFFFFFu) | (px[t] & 0xFFu) << 24;
                }
                for (int t = 0; t < 16; t++) memcpy(&rgba[4 * ((uint64_t)(4 * by + t / 4) * w + 4 * bx + t % 4)], &px[t], 4);
            }
        const uint64_t o = f * frame_bytes;
        planar_out_twin::picture(rgba.data(), w, h, alpha_only ? nullptr : wl.data() + o, alpha_only ? nullptr : wcb.data() + o,
                                 alpha_only ? nullptr : wcr.data() + o, alpha ? wa.data() + o : nullptr, lpitch, cpitch, SUB, n, s.cs);
    }
    const std::string what = "kind " + std::to_string(KIND) + " sub " + std::to_string(SUB) + " depth " + std::to_string(n) + " cs " +
                             std::to_string(s.cs) + " " + std::to_string(w) + "x" + std::to_string(h) + " pitches " + std::to_string(lpitch) +
                             "/" + std::to_string(cpitch) + (alpha ? " alpha" : "");
    const std::pair<const std::vector<uint8_t> *, const std::vector<uint8_t> *> planes[4] = {{&lbuf, &wl}, {&cbbuf, &wcb}, {&crbuf, &wcr}, {&abuf, &wa}};
    const char *names[4] = {"luma", "cb", "cr", "alpha"};
    for (int p = 0; p < 4; p++)
        for (size_t i = 0; i < planes[p].first->size(); i++)
            if ((*planes[p].first)[i] != (*planes[p].second)[i]) { fail(what + ": " + names[p] + " byte " + std::to_string(i)); break; }
    g_runs++;
}

template <int SUB, bool WIDE>
void check_kinds(const Shape &s)
{
    check<kBcDxt1, SUB, WIDE>(s);
    check<kBcDxt5, SUB, WIDE>(s);
    check<kBcYCoCg, SUB, WIDE>(s);
    check<kBcYCoCgPlusAlpha, SUB, WIDE>(s);
    check<kBcBc7, SUB, WIDE>(s);
    if (SUB == HapB200Chroma_420) check<kBcRgtc1, SUB, WIDE>(s);   // (the alpha kernel has no subsampling)
}

}  // namespace

int main()
{
    const uint32_t widths[] = {1, 2, 30, 31, 32, 33, 62, 63, 64, 129};
    int shapes = 0;
    for (uint32_t bw : widths)
        for (uint32_t bh : {1u, 2u, 3u}) {
            const Shape s{bw, bh, 16u * (shapes % 3), 16u * ((shapes + 1) % 3), shapes % 2 ? 12u : 10u, (uint32_t)(shapes % 4), shapes % 3 != 1};
            check_kinds<HapB200Chroma_420, false>(s);
            check_kinds<HapB200Chroma_420, true>(s);
            check_kinds<HapB200Chroma_422, false>(s);
            check_kinds<HapB200Chroma_422, true>(s);
            check_kinds<HapB200Chroma_444, false>(s);
            check_kinds<HapB200Chroma_444, true>(s);
            shapes++;
        }
    printf("%d shapes, %d runs x %u frames, %d failures\n", shapes, g_runs, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
