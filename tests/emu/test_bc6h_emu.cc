// tests/emu/test_bc6h_emu.cc -- TEST INFRASTRUCTURE ONLY.
// bc6h_decode_kernel (Hap HDR -> RGBA16F) under the fiber SIMT emulator at the geometries the batch entry points accept: odd
// block widths (warps that straddle block rows), row pitches wider than the picture, three frames with slack between them
// and a block stride wider than the texture.  Signedness once from the call (UF16, then SF16 for every frame) and once from
// a per-frame format array (UF16, SF16, UF16), with and without per-frame results (frame 1 failed: its picture must be
// zeros).  The blocks are random bytes with every mode and the reserved mode values forced in turn along each frame, so
// neighbouring lanes of a warp decode different modes.  Every buffer is exactly as long as the last frame needs and its
// padding holds a sentinel: each pixel is compared with bc6h_decode_block, and every padding byte must keep the sentinel.
#define HAPB200_EMU
#include "bc6h_decode.cuh"

#include <string>
#include <vector>

using namespace hapb200;

namespace {

constexpr uint32_t kFrames = 3;
constexpr uint8_t kPad = 0xA5;
const uint8_t kModeValues[18] = {0x00, 0x01, 0x02, 0x06, 0x0A, 0x0E, 0x12, 0x16, 0x1A, 0x1E, 0x03, 0x07, 0x0B, 0x0F,
                                 0x13, 0x17, 0x1B, 0x1F};   // modes 1..14, then the reserved values
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

struct Shape {
    uint32_t w, h, row_bytes;
    uint64_t frame_bytes;
    std::string name() const
    {
        return std::to_string(w) + "x" + std::to_string(h) + " pitch " + std::to_string(row_bytes) + " frame " + std::to_string(frame_bytes);
    }
    uint64_t out_bytes() const { return (kFrames - 1) * frame_bytes + (uint64_t)(h - 1) * row_bytes + 8ull * w; }
    bool is_pixel(uint64_t off) const
    {
        const uint64_t f = off / frame_bytes, in = off % frame_bytes;
        return f < kFrames && in / row_bytes < h && in % row_bytes < 8ull * w;
    }
    uint64_t pixel(uint32_t f, uint32_t x, uint32_t y) const { return f * frame_bytes + (uint64_t)y * row_bytes + 8ull * x; }
};

// how: 0 = UF16 from the call, 1 = SF16 from the call, 2 = per-frame formats (UF16, SF16, UF16)
void check_decode(const Shape &s, int how, bool with_results)
{
    const uint64_t nblk = (uint64_t)(s.w / 4) * (s.h / 4), t0 = 16 * nblk;
    const uint64_t stride = ((t0 + 15) & ~15ull) + 32;
    std::vector<uint8_t> blocks((kFrames - 1) * stride + t0, kPad);
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint64_t b = 0; b < nblk; b++) {
            uint8_t *blk = &blocks[f * stride + 16 * b];
            for (int k = 0; k < 16; k++) blk[k] = (uint8_t)rnd();
            const uint8_t v = kModeValues[(b + 5 * f) % 18];
            const uint8_t bits = v < 2 ? 0x03 : 0x1F;
            blk[0] = (uint8_t)((blk[0] & ~bits) | v);
        }
    std::vector<uint8_t> out(s.out_bytes(), kPad);
    const uint32_t results[kFrames] = {0u, 7u /* a frame whose decode failed */, 0u};
    const uint32_t formats[kFrames] = {HapFmt_RGB_BPTC_UFLOAT, HapFmt_RGB_BPTC_SFLOAT, HapFmt_RGB_BPTC_UFLOAT};
    const BcDecodeGeom g = bc_decode_geom(s.w, s.h, s.row_bytes, false, stride, 0, s.frame_bytes);
    HAP_LAUNCH(bc6h_decode_kernel, dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, blocks.data(), g, out.data(),
               with_results ? results : (const uint32_t *)nullptr, how == 2 ? formats : (const uint32_t *)nullptr, how == 1 ? 1u : 0u);
    const std::string what = std::string("decode bc6h how ") + std::to_string(how) + (with_results ? " results " : " ") + s.name();
    int bad = 0;
    for (uint32_t f = 0; f < kFrames && !bad; f++) {
        const bool sgn = how == 1 || (how == 2 && f == 1);
        for (uint32_t by = 0; by < s.h / 4 && !bad; by++)
            for (uint32_t bx = 0; bx < s.w / 4 && !bad; bx++) {
                const uint64_t bi = (uint64_t)by * (s.w / 4) + bx;
                uint32_t v[4], px[32];
                memcpy(v, &blocks[f * stride + 16 * bi], 16);
                bc6h_decode_block(v[0], v[1], v[2], v[3], sgn, px);
                if (with_results && results[f] != 0)
                    for (int k = 0; k < 32; k++) px[k] = 0;
                for (int t = 0; t < 16 && !bad; t++) {
                    uint32_t got[2];
                    memcpy(got, &out[s.pixel(f, 4 * bx + t % 4, 4 * by + t / 4)], 8);
                    if (got[0] != px[2 * t] || got[1] != px[2 * t + 1]) {
                        fail(what + ": frame " + std::to_string(f) + " block " + std::to_string(bx) + "," + std::to_string(by) + " texel " + std::to_string(t));
                        bad = 1;
                    }
                }
            }
    }
    for (uint64_t i = 0; i < out.size(); i++)
        if (!s.is_pixel(i) && out[i] != kPad) { fail(what + ": padding byte " + std::to_string(i) + " of the pictures changed"); break; }
}

}  // namespace

int main()
{
    const uint32_t widths[] = {4, 8, 12, 20, 36, 132, 516}, heights[] = {4, 8, 20}, pads[] = {0, 16, 48};
    int shapes = 0;
    for (uint32_t w : widths)
        for (uint32_t h : heights)
            for (uint32_t pad : pads) {
                Shape s{w, h, 8 * w + pad, 0};
                s.frame_bytes = (uint64_t)h * s.row_bytes + 16 * (1 + shapes % 3);   // slack between frames
                for (int how = 0; how < 3; how++) {
                    check_decode(s, how, false);
                    check_decode(s, how, true);
                }
                shapes++;
            }
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
