// tests/emu/test_yuv_pq_out_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The HDR10 sink of K8 (bc6h_decode_yuv_kernel, yuv_sink.cuh: BC6H -> P010, BT.2020, PQ) under the fiber SIMT emulator, at
// block widths 1, 2, 30, 31, 32, 33, 62, 63 and 64 (the halo lane at row starts, row ends and warp-span boundaries), heights
// of 1, 2 and 3 block rows, pitches wider than the row, four frames with slack between them, a block stride wider than the
// texture, both ranges and several unitNits.  Random block bytes reach every mode and the reserved ones.  The frames mix
// UF16 and SF16 through per-frame formats, one frame has failed, and the signedness from the call is checked as well.  Two
// placements of the chroma plane: its own exact-size buffer, and NVDEC's, inside the luma buffer at pitch * surfaceHeight;
// either buffer ends with the last frame's last sample, so a store past a plane leaves every buffer.  Every sample must equal
// the sample-by-sample conversion of yuv_pq_out_twin.h applied to bc6h_decode_block's texels (zeros for the failed frame),
// and every other byte must keep its sentinel.
#define HAPB200_EMU
#include "yuv_pq_out_twin.h"

#include <string>
#include <vector>

using namespace hapb200;

namespace {

constexpr uint32_t kFrames = 4;
constexpr uint8_t kPad = 0xA5;
int g_fail = 0;

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

// how: 0 = UF16 from the call, 1 = SF16 from the call, 2 = per-frame formats (UF16, SF16, SF16, UF16) with frame 2 failed
void check(uint32_t bw, uint32_t bh, uint32_t pad, bool nvdec, int cs, uint32_t unit, int how)
{
    const uint32_t w = 4 * bw, h = 4 * bh, pitch = 2 * w + pad;
    const uint64_t nblk = (uint64_t)bw * bh, in_stride = nblk * 16 + 32;
    std::vector<uint8_t> in(kFrames * in_stride);
    for (auto &b : in) b = (uint8_t)rnd();
    const uint64_t surface_rows = h + (nvdec ? 8 : 0);
    const uint64_t frame_bytes = nvdec ? (surface_rows + h / 2) * pitch + 32 : (uint64_t)h * pitch + 48;
    const uint64_t chroma_at = nvdec ? surface_rows * pitch : 0;
    auto plane_end = [&](uint32_t rows) { return (kFrames - 1) * frame_bytes + (uint64_t)(rows - 1) * pitch + 2ull * w; };
    std::vector<uint8_t> lbuf(nvdec ? chroma_at + plane_end(h / 2) : plane_end(h), kPad), cbuf(nvdec ? 0 : plane_end(h / 2), kPad);
    uint8_t *luma = lbuf.data(), *chroma = nvdec ? lbuf.data() + chroma_at : cbuf.data();
    const uint32_t formats[kFrames] = {HapFmt_RGB_BPTC_UFLOAT, HapFmt_RGB_BPTC_SFLOAT, HapFmt_RGB_BPTC_SFLOAT, HapFmt_RGB_BPTC_UFLOAT};
    const uint32_t results[kFrames] = {0, 0, 7 /* a failed frame */, 0};
    std::vector<uint16_t> table(kPqOutEntries);
    yuv_pq_out_table(unit, table.data());
    const YuvOutGeom g = yuv_out_geom(w, h, pitch, in_stride, frame_bytes, yuv_pq_out_coeffs(cs));
    HAP_LAUNCH(bc6h_decode_yuv_kernel, dim3((unsigned)yuv_out_ctas(g), kFrames), dim3(kBcThreads), 0, nullptr, in.data(), g, luma, chroma,
               how == 2 ? results : nullptr, how == 2 ? formats : nullptr, how == 1 ? 1u : 0u, table.data());
    // expected: the twin on the decoded picture, written into sentinel buffers of the same shape
    std::vector<uint8_t> wl(lbuf.size(), kPad), wc(cbuf.size(), kPad);
    uint8_t *want_luma = wl.data(), *want_chroma = nvdec ? wl.data() + chroma_at : wc.data();
    std::vector<uint16_t> rgba(4ull * w * h);
    for (uint32_t f = 0; f < kFrames; f++) {
        const bool sgn = how == 2 ? formats[f] == HapFmt_RGB_BPTC_SFLOAT : how == 1;
        for (uint32_t by = 0; by < bh; by++)
            for (uint32_t bx = 0; bx < bw; bx++) {
                uint32_t px[32] = {0};
                if (how != 2 || results[f] == 0) {
                    uint32_t v[4];
                    memcpy(v, &in[f * in_stride + ((uint64_t)by * bw + bx) * 16], 16);
                    bc6h_decode_block(v[0], v[1], v[2], v[3], sgn, px);
                }
                for (int t = 0; t < 16; t++) memcpy(&rgba[4 * ((uint64_t)(4 * by + t / 4) * w + 4 * bx + t % 4)], &px[2 * t], 8);
            }
        yuv_pq_out_twin::picture(rgba.data(), w, h, cs, table.data(), want_luma + f * frame_bytes, want_chroma + f * frame_bytes, pitch);
    }
    const std::string what = "cs " + std::to_string(cs) + " unit " + std::to_string(unit) + " how " + std::to_string(how) + " " +
                             std::to_string(w) + "x" + std::to_string(h) + " pitch " + std::to_string(pitch) + (nvdec ? " nvdec" : "");
    for (size_t i = 0; i < lbuf.size(); i++)
        if (lbuf[i] != wl[i]) { fail(what + ": luma buffer byte " + std::to_string(i)); break; }
    for (size_t i = 0; i < cbuf.size(); i++)
        if (cbuf[i] != wc[i]) { fail(what + ": chroma buffer byte " + std::to_string(i)); break; }
}

}  // namespace

int main()
{
    const uint32_t widths[] = {1, 2, 30, 31, 32, 33, 62, 63, 64};
    const uint32_t units[] = {1, 100, 203, 1000, 10000};
    int shapes = 0;
    for (uint32_t bw : widths)
        for (uint32_t bh : {1u, 2u, 3u})
            for (bool nvdec : {false, true}) {
                const int cs = HapB200YUV_BT2020_Limited + shapes % 2;
                const uint32_t pad = 16 * (shapes % 3), unit = units[shapes % 5];
                for (int how = 0; how < 3; how++) check(bw, bh, pad, nvdec, cs, unit, how);
                shapes++;
            }
    printf("%d shapes x 3 signedness modes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
