// tests/emu/test_bc6h_encode_emu.cc -- TEST INFRASTRUCTURE ONLY.
// bc6h_encode_kernel (RGBA16F -> Hap HDR blocks) under the fiber SIMT emulator at the geometries the batch entry points
// accept: odd block widths (warps that straddle block rows), row pitches wider than the picture, three frames with slack
// between them and a block stride wider than the texture, UF16 and SF16.  Pixels are random halves, every tenth block
// constant, with NaN, Inf, -0 and negatives among them.  Every buffer is exactly as long as the last frame needs; the block
// buffer's padding holds a sentinel.  Each block must equal bc6h_encode_block's (the host twin) and the padding must keep
// the sentinel.
#define HAPB200_EMU
#include "bc6h_encode.cuh"

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

uint16_t random_half()
{
    const uint32_t r = rnd();
    switch (r % 16) {
    case 0: return 0x7C00;                                  // +Inf
    case 1: return 0xFC00;                                  // -Inf
    case 2: return (uint16_t)(0x7C01 + (r >> 8) % 0x3FF);   // NaN
    case 3: return 0x8000;                                  // -0
    default: return (uint16_t)(r >> 4) & ((r >> 20) & 1 ? 0xFBFF : 0x7BFF);   // finite, half of them negative
    }
}

void check_encode(uint32_t w, uint32_t h, uint32_t pad, uint64_t slack, bool sgn)
{
    const uint32_t row_bytes = 8 * w + pad;
    const uint64_t frame_bytes = (uint64_t)h * row_bytes + slack;
    const uint64_t nblk = (uint64_t)(w / 4) * (h / 4), t0 = 16 * nblk, stride = t0 + 48;
    std::vector<uint8_t> rgba((kFrames - 1) * frame_bytes + (uint64_t)(h - 1) * row_bytes + 8ull * w);
    for (size_t i = 0; i + 1 < rgba.size(); i += 2) {
        const uint16_t v = random_half();
        memcpy(&rgba[i], &v, 2);
    }
    for (uint32_t f = 0; f < kFrames; f++)   // every tenth block constant
        for (uint64_t b = 0; b < nblk; b += 10) {
            const uint32_t by = (uint32_t)(b / (w / 4)), bx = (uint32_t)(b % (w / 4));
            const uint8_t *c = &rgba[f * frame_bytes + (uint64_t)(4 * by) * row_bytes + 32u * bx];
            uint8_t texel[8];
            memcpy(texel, c, 8);
            for (int t = 0; t < 16; t++) memcpy(&rgba[f * frame_bytes + (uint64_t)(4 * by + t / 4) * row_bytes + 32u * bx + 8 * (t % 4)], texel, 8);
        }
    std::vector<uint8_t> out((kFrames - 1) * stride + t0, kPad);
    const BcGeom g = bc_encode_geom(w, h, row_bytes, frame_bytes, stride, 0);
    HAP_LAUNCH(bc6h_encode_kernel, dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, rgba.data(), g, out.data(),
               sgn ? 1u : 0u);
    const std::string what = std::string(sgn ? "SF16 " : "UF16 ") + std::to_string(w) + "x" + std::to_string(h) + " pad " + std::to_string(pad);
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint64_t b = 0; b < nblk; b++) {
            const uint32_t by = (uint32_t)(b / (w / 4)), bx = (uint32_t)(b % (w / 4));
            uint32_t px[32], want[4];
            for (int t = 0; t < 16; t++) memcpy(&px[2 * t], &rgba[f * frame_bytes + (uint64_t)(4 * by + t / 4) * row_bytes + 32u * bx + 8 * (t % 4)], 8);
            bc6h_encode_block(px, sgn, want);
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
                for (int sgn = 0; sgn < 2; sgn++) check_encode(w, h, pad, 16 * (1 + shapes % 3), sgn != 0);
                shapes++;
            }
    printf("%d shapes x %u frames x 2 formats, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
