// tests/emu/test_bc7_emu.cc -- TEST INFRASTRUCTURE ONLY.
// bc_decode_kernel<kBcBc7> (Hap R) under the fiber SIMT emulator at the geometries the batch entry points accept: odd block
// widths (warps that straddle block rows), row pitches wider than the picture, three frames with slack between them and a
// block stride wider than the texture, with and without per-frame results (frame 1 failed: its picture must be zeros).  The
// blocks are random bytes with every mode forced in turn along each frame, reserved blocks included, so neighbouring lanes
// of a warp decode different modes.  Every buffer is exactly as long as the last frame needs and its padding holds a
// sentinel: each pixel is compared with bc7_decode_block, and every padding byte must still hold the sentinel.
#define HAPB200_EMU
#include "bc_decode.cuh"

#include <string>
#include <vector>

using namespace hapb200;

namespace {

constexpr uint32_t kFrames = 3;
constexpr uint8_t kPad = 0xA5;
int g_fail = 0;

uint64_t g_rng = 0x13198A2E03707344ull;
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
    uint64_t rgba_bytes() const { return (kFrames - 1) * frame_bytes + (uint64_t)(h - 1) * row_bytes + 4ull * w; }
    bool is_pixel(uint64_t off) const
    {
        const uint64_t f = off / frame_bytes, in = off % frame_bytes;
        return f < kFrames && in / row_bytes < h && in % row_bytes < 4ull * w;
    }
    uint64_t pixel(uint32_t f, uint32_t x, uint32_t y) const { return f * frame_bytes + (uint64_t)y * row_bytes + 4ull * x; }
};

void check_decode(const Shape &s, bool with_results)
{
    const uint64_t nblk = (uint64_t)(s.w / 4) * (s.h / 4), t0 = 16 * nblk;
    const uint64_t stride = ((t0 + 15) & ~15ull) + 32;
    std::vector<uint8_t> blocks((kFrames - 1) * stride + t0, kPad);
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint64_t b = 0; b < nblk; b++) {
            uint8_t *blk = &blocks[f * stride + 16 * b];
            for (int k = 0; k < 16; k++) blk[k] = (uint8_t)rnd();
            const uint32_t mode = (uint32_t)((b + 3 * f) % 9);   // 8: reserved (byte 0 = 0)
            blk[0] = mode == 8 ? 0 : (uint8_t)((blk[0] & (0xFFu << (mode + 1))) | (1u << mode));
        }
    std::vector<uint8_t> rgba(s.rgba_bytes(), kPad);
    const uint32_t results[kFrames] = {0u, 7u /* a frame whose decode failed */, 0u};
    const BcDecodeGeom g = bc_decode_geom(s.w, s.h, s.row_bytes, false, stride, 0, s.frame_bytes);
    HAP_LAUNCH(bc_decode_kernel<kBcBc7>, dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, blocks.data(),
               (const uint8_t *)nullptr, g, rgba.data(), with_results ? results : (const uint32_t *)nullptr);
    const std::string what = std::string("decode bc7") + (with_results ? " results " : " ") + s.name();
    int bad = 0;
    for (uint32_t f = 0; f < kFrames && !bad; f++)
        for (uint32_t by = 0; by < s.h / 4 && !bad; by++)
            for (uint32_t bx = 0; bx < s.w / 4 && !bad; bx++) {
                const uint64_t bi = (uint64_t)by * (s.w / 4) + bx;
                uint32_t v[4], px[16];
                memcpy(v, &blocks[f * stride + 16 * bi], 16);
                bc7_decode_block(v[0], v[1], v[2], v[3], px);
                if (with_results && results[f] != 0)
                    for (int t = 0; t < 16; t++) px[t] = 0;
                for (int t = 0; t < 16 && !bad; t++) {
                    uint32_t got;
                    memcpy(&got, &rgba[s.pixel(f, 4 * bx + t % 4, 4 * by + t / 4)], 4);
                    if (got != px[t]) {
                        fail(what + ": frame " + std::to_string(f) + " block " + std::to_string(bx) + "," + std::to_string(by) + " texel " + std::to_string(t));
                        bad = 1;
                    }
                }
            }
    for (uint64_t i = 0; i < rgba.size(); i++)
        if (!s.is_pixel(i) && rgba[i] != kPad) { fail(what + ": padding byte " + std::to_string(i) + " of the pictures changed"); break; }
}

}  // namespace

int main()
{
    const uint32_t widths[] = {4, 8, 12, 20, 36, 132, 516}, heights[] = {4, 8, 12, 20}, pads[] = {0, 16, 48};
    int shapes = 0;
    for (uint32_t w : widths)
        for (uint32_t h : heights)
            for (uint32_t pad : pads) {
                Shape s{w, h, 4 * w + pad, 0};
                s.frame_bytes = (uint64_t)h * s.row_bytes + 16 * (1 + shapes % 3);   // slack between frames
                check_decode(s, false);
                check_decode(s, true);
                shapes++;
            }
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
