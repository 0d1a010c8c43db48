// tests/emu/test_bc7_encode_emu.cc -- TEST INFRASTRUCTURE ONLY.
// bc_encode_kernel<kBcBc7> (RGBA8 -> Hap R blocks) under the fiber SIMT emulator at the geometries the batch entry points
// accept: odd block widths (warps that straddle block rows), row pitches wider than the picture, three frames with slack
// between them and a block stride wider than the texture.  Pixels are random bytes, every tenth block constant and every
// seventh opaque.  Every buffer is exactly as long as the last frame needs; the block buffer's padding holds a sentinel.
// Each block must equal bc7_encode_block's (the host twin) and the padding must keep the sentinel.
#define HAPB200_EMU
#include "bc_encode.cuh"

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

uint8_t *texel(std::vector<uint8_t> &rgba, uint32_t f, uint64_t frame_bytes, uint32_t row_bytes, uint32_t bx, uint32_t by, int t)
{
    return &rgba[f * frame_bytes + (uint64_t)(4 * by + t / 4) * row_bytes + 16u * bx + 4 * (t % 4)];
}

void check_encode(uint32_t w, uint32_t h, uint32_t pad, uint64_t slack)
{
    const uint32_t row_bytes = 4 * w + pad;
    const uint64_t frame_bytes = (uint64_t)h * row_bytes + slack;
    const uint64_t nblk = (uint64_t)(w / 4) * (h / 4), t0 = 16 * nblk, stride = t0 + 48;
    std::vector<uint8_t> rgba((kFrames - 1) * frame_bytes + (uint64_t)(h - 1) * row_bytes + 4ull * w);
    for (auto &b : rgba) b = (uint8_t)rnd();
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint64_t b = 0; b < nblk; b++) {
            const uint32_t by = (uint32_t)(b / (w / 4)), bx = (uint32_t)(b % (w / 4));
            uint8_t first[4];
            memcpy(first, texel(rgba, f, frame_bytes, row_bytes, bx, by, 0), 4);
            for (int t = 0; t < 16; t++) {
                uint8_t *p = texel(rgba, f, frame_bytes, row_bytes, bx, by, t);
                if (b % 10 == 0) memcpy(p, first, 4);   // constant
                if (b % 7 == 3) p[3] = 255;              // opaque
            }
        }
    std::vector<uint8_t> out((kFrames - 1) * stride + t0, kPad);
    const BcGeom g = bc_encode_geom(w, h, row_bytes, frame_bytes, stride, 0);
    HAP_LAUNCH(bc_encode_kernel<kBcBc7>, dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, rgba.data(), g,
               out.data());
    const std::string what = std::to_string(w) + "x" + std::to_string(h) + " pad " + std::to_string(pad);
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint64_t b = 0; b < nblk; b++) {
            const uint32_t by = (uint32_t)(b / (w / 4)), bx = (uint32_t)(b % (w / 4));
            uint32_t px[16], want[4];
            for (int t = 0; t < 16; t++) memcpy(&px[t], texel(rgba, f, frame_bytes, row_bytes, bx, by, t), 4);
            bc7_encode_block(px, want);
            if (memcmp(want, &out[f * stride + 16 * b], 16)) {
                fail(what + ": frame " + std::to_string(f) + " block " + std::to_string(b));
                return;
            }
        }
    for (uint32_t f = 0; f + 1 < kFrames; f++)
        for (uint64_t i = t0; i < stride; i++)
            if (out[f * stride + i] != kPad) { fail(what + ": padding after frame " + std::to_string(f) + " changed"); return; }
}

}  // namespace

int main()
{
    const uint32_t widths[] = {4, 12, 36, 132}, heights[] = {4, 8}, pads[] = {0, 16, 48};
    int shapes = 0;
    for (uint32_t w : widths)
        for (uint32_t h : heights)
            for (uint32_t pad : pads) {
                check_encode(w, h, pad, 16 * (1 + shapes % 3));
                shapes++;
            }
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
