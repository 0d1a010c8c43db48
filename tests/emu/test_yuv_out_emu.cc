// tests/emu/test_yuv_out_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The NV12 / P010 sink of K8 (bc_decode_yuv_kernel, yuv_sink.cuh) under the fiber SIMT emulator, every kind x layout, at
// block widths 1, 2, 30, 31, 32, 33, 62, 63, 64 and 129 (the halo lane at row starts, row ends and warp-span boundaries),
// heights of 1, 2 and 3 block rows, pitches wider than the row, three frames with slack between them, and a failed middle
// frame.  Two placements of the chroma plane: its own exact-size buffer, and NVDEC's, inside the luma buffer at
// pitch * surfaceHeight; either buffer ends with the last frame's last sample, so a store past a plane leaves every buffer.
// Every sample must equal the pixel-by-pixel conversion of yuv_out_twin.h applied to decode_block's texels (zeros for the
// failed frame), and every other byte must keep its sentinel.
#define HAPB200_EMU
#include "yuv_out_twin.h"

#include <string>
#include <vector>

using namespace hapb200;

namespace {

constexpr uint32_t kFrames = 3;
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

template <int KIND, int LAYOUT>
void check(uint32_t bw, uint32_t bh, uint32_t pad, bool nvdec, int cs)
{
    const uint32_t w = 4 * bw, h = 4 * bh, sb = LAYOUT == HapB200YUV_P010 ? 2 : 1;
    const uint32_t pitch = sb * w + pad;
    const uint64_t block_bytes = KIND == kBcDxt1 || KIND == kBcRgtc1 ? 8 : 16;
    const uint64_t nblk = (uint64_t)bw * bh, in_stride = (nblk * block_bytes + 15) / 16 * 16 + 32;
    std::vector<uint8_t> in(kFrames * in_stride);
    for (auto &b : in) b = (uint8_t)rnd();
    const uint64_t surface_rows = h + (nvdec ? 8 : 0);
    const uint64_t frame_bytes = nvdec ? (surface_rows + h / 2) * pitch + 32 : (uint64_t)h * pitch + 48;
    const uint64_t chroma_at = nvdec ? surface_rows * pitch : 0;
    auto plane_end = [&](uint32_t rows) { return (kFrames - 1) * frame_bytes + (uint64_t)(rows - 1) * pitch + (uint64_t)sb * w; };
    std::vector<uint8_t> lbuf(nvdec ? chroma_at + plane_end(h / 2) : plane_end(h), kPad), cbuf(nvdec ? 0 : plane_end(h / 2), kPad);
    uint8_t *luma = lbuf.data(), *chroma = nvdec ? lbuf.data() + chroma_at : cbuf.data();
    const uint32_t results[kFrames] = {0, 7 /* a failed frame */, 0};
    const YuvOutGeom g = yuv_out_geom(w, h, pitch, in_stride, frame_bytes, LAYOUT, cs);
    HAP_LAUNCH((bc_decode_yuv_kernel<KIND, LAYOUT>), dim3((unsigned)yuv_out_ctas(g), kFrames), dim3(kBcThreads), 0, nullptr, in.data(), g,
               luma, chroma, results);
    // expected: the twin on the decoded picture, written into sentinel buffers of the same shape
    std::vector<uint8_t> wl(lbuf.size(), kPad), wc(cbuf.size(), kPad);
    uint8_t *want_luma = wl.data(), *want_chroma = nvdec ? wl.data() + chroma_at : wc.data();
    std::vector<uint8_t> rgba(4ull * w * h);
    for (uint32_t f = 0; f < kFrames; f++) {
        for (uint32_t by = 0; by < bh; by++)
            for (uint32_t bx = 0; bx < bw; bx++) {
                uint32_t px[16] = {0};
                if (results[f] == 0) {
                    uint32_t v[4] = {0, 0, 0, 0};
                    memcpy(v, &in[f * in_stride + ((uint64_t)by * bw + bx) * block_bytes], block_bytes);
                    decode_block(KIND, v[0], v[1], v[2], v[3], px);
                }
                for (int t = 0; t < 16; t++) memcpy(&rgba[4 * ((uint64_t)(4 * by + t / 4) * w + 4 * bx + t % 4)], &px[t], 4);
            }
        yuv_out_twin::picture(rgba.data(), w, h, LAYOUT, cs, want_luma + f * frame_bytes, want_chroma + f * frame_bytes, pitch);
    }
    const std::string what = "kind " + std::to_string(KIND) + (LAYOUT ? " P010" : " NV12") + " cs " + std::to_string(cs) + " " +
                             std::to_string(w) + "x" + std::to_string(h) + " pitch " + std::to_string(pitch) + (nvdec ? " nvdec" : "");
    for (size_t i = 0; i < lbuf.size(); i++)
        if (lbuf[i] != wl[i]) { fail(what + ": luma buffer byte " + std::to_string(i)); break; }
    for (size_t i = 0; i < cbuf.size(); i++)
        if (cbuf[i] != wc[i]) { fail(what + ": chroma buffer byte " + std::to_string(i)); break; }
}

template <int LAYOUT>
void check_kinds(uint32_t bw, uint32_t bh, uint32_t pad, bool nvdec, int cs)
{
    check<kBcDxt1, LAYOUT>(bw, bh, pad, nvdec, cs);
    check<kBcDxt5, LAYOUT>(bw, bh, pad, nvdec, cs);
    check<kBcYCoCg, LAYOUT>(bw, bh, pad, nvdec, cs);
    check<kBcRgtc1, LAYOUT>(bw, bh, pad, nvdec, cs);
    check<kBcBc7, LAYOUT>(bw, bh, pad, nvdec, cs);
}

}  // namespace

int main()
{
    const uint32_t widths[] = {1, 2, 30, 31, 32, 33, 62, 63, 64, 129};
    int shapes = 0;
    for (uint32_t bw : widths)
        for (uint32_t bh : {1u, 2u, 3u})
            for (bool nvdec : {false, true}) {
                const int cs = shapes % 4;
                const uint32_t pad = 16 * (shapes % 3);
                check_kinds<HapB200YUV_NV12>(bw, bh, pad, nvdec, cs);
                check_kinds<HapB200YUV_P010>(bw, bh, pad, nvdec, cs);
                shapes++;
            }
    printf("%d shapes x 5 kinds x 2 layouts x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
