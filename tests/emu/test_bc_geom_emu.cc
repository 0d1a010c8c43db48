// tests/emu/test_bc_geom_emu.cc -- TEST INFRASTRUCTURE ONLY.
// bc_encode_kernel and bc_decode_kernel under the fiber SIMT emulator at the geometries the batch entry points accept:
// odd block widths (warps that straddle block rows, a non-exact inv_blocks_x), row pitches wider than the picture, three
// frames with slack between them, and a block stride wider than the texture.  The launch geometry comes from the library's
// own helpers (bc_encode_geom, bc_decode_geom, bc_ctas).  Every buffer is exactly as long as the last frame needs and its
// padding is filled with a sentinel: each block / pixel is compared with the per-block functions of bc_block.cuh and
// bc_decode.cuh, and every padding byte, inside a row, between rows and between frames, must still hold the sentinel.
#define HAPB200_EMU
#include "bc_decode.cuh"

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

struct Shape {
    uint32_t w, h, row_bytes;
    uint64_t frame_bytes;
    std::string name() const
    {
        return std::to_string(w) + "x" + std::to_string(h) + " pitch " + std::to_string(row_bytes) + " frame " + std::to_string(frame_bytes);
    }
    // bytes of the picture buffer: the last frame's last row ends the buffer
    uint64_t rgba_bytes() const { return (kFrames - 1) * frame_bytes + (uint64_t)(h - 1) * row_bytes + 4ull * w; }
    bool is_pixel(uint64_t off) const
    {
        const uint64_t f = off / frame_bytes, in = off % frame_bytes;
        return f < kFrames && in / row_bytes < h && in % row_bytes < 4ull * w;
    }
    uint64_t pixel(uint32_t f, uint32_t x, uint32_t y) const { return f * frame_bytes + (uint64_t)y * row_bytes + 4ull * x; }
};

// frame 0 noise, frame 1 smooth ramps (the chroma refinement's case), frame 2 flat 8x8 tiles with noisy alpha
std::vector<uint8_t> make_pictures(const Shape &s)
{
    std::vector<uint8_t> b(s.rgba_bytes(), kPad);
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint32_t y = 0; y < s.h; y++)
            for (uint32_t x = 0; x < s.w; x++) {
                uint8_t *p = &b[s.pixel(f, x, y)];
                const uint32_t r = rnd();
                if (f == 0) memcpy(p, &r, 4);
                else if (f == 1) { p[0] = (uint8_t)(x * 3 + y); p[1] = (uint8_t)(128 + x / 4); p[2] = (uint8_t)(200 - y * 2); p[3] = (uint8_t)(x ^ y); }
                else { const uint32_t t = (x / 8) * 31 + (y / 8) * 17; p[0] = (uint8_t)(t * 5); p[1] = (uint8_t)(t * 11); p[2] = (uint8_t)(t * 23); p[3] = (uint8_t)r; }
            }
    return b;
}

void gather(const std::vector<uint8_t> &b, const Shape &s, uint32_t f, uint32_t bx, uint32_t by, uint32_t px[16])
{
    for (int t = 0; t < 16; t++) memcpy(&px[t], &b[s.pixel(f, 4 * bx + t % 4, 4 * by + t / 4)], 4);
}

// ---- encode --------------------------------------------------------------------------------------------------------------

// the bytes of block (bx, by) of plane `plane` the per-block functions give (plane 1: the RGTC1 plane of kBcYCoCgPlusAlpha)
template <int KIND, bool REFINE>
int expected_block(const uint32_t px[16], int plane, uint8_t out[16])
{
    Block8 a, c;
    if (plane == 1 || KIND == kBcRgtc1) { a = encode_rgtc1_alpha(px); memcpy(out, &a, 8); return 8; }
    if (KIND == kBcDxt1) { c = encode_dxt1(px); memcpy(out, &c, 8); return 8; }
    if (KIND == kBcDxt5) encode_dxt5(px, a, c);
    else encode_ycocg_dxt5<REFINE>(px, a, c);
    memcpy(out, &a, 8);
    memcpy(out + 8, &c, 8);
    return 16;
}

template <int KIND, bool REFINE = false>
void check_encode(const Shape &s, const std::vector<uint8_t> &rgba)
{
    const uint64_t nblk = (uint64_t)(s.w / 4) * (s.h / 4);
    const uint64_t t0 = nblk * (KIND == kBcDxt1 || KIND == kBcRgtc1 ? 8 : 16), t1 = KIND == kBcYCoCgPlusAlpha ? nblk * 8 : 0;
    const uint64_t stride = ((t0 + t1 + 15) & ~15ull) + 48;          // wider than the frame's blocks
    std::vector<uint8_t> out((kFrames - 1) * stride + t0 + t1, kPad);
    const BcGeom g = bc_encode_geom(s.w, s.h, s.row_bytes, s.frame_bytes, stride, t0);
    HAP_LAUNCH((bc_encode_kernel<KIND, REFINE>), dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, rgba.data(), g,
               out.data());
    std::vector<bool> written(out.size(), false);
    const std::string what = "encode kind " + std::to_string(KIND) + (REFINE ? " refine " : " ") + s.name();
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint32_t by = 0; by < s.h / 4; by++)
            for (uint32_t bx = 0; bx < s.w / 4; bx++) {
                uint32_t px[16];
                gather(rgba, s, f, bx, by, px);
                const uint64_t bi = (uint64_t)by * (s.w / 4) + bx;
                for (int plane = 0; plane < (t1 ? 2 : 1); plane++) {
                    uint8_t want[16];
                    const int n = expected_block<KIND, REFINE>(px, plane, want);
                    const uint64_t at = f * stride + (plane ? t0 : 0) + bi * n;
                    if (memcmp(&out[at], want, n) != 0)
                        fail(what + ": frame " + std::to_string(f) + " block " + std::to_string(bx) + "," + std::to_string(by) + " plane " + std::to_string(plane));
                    for (int k = 0; k < n; k++) written[at + k] = true;
                }
            }
    for (size_t i = 0; i < out.size(); i++)
        if (!written[i] && out[i] != kPad) { fail(what + ": padding byte " + std::to_string(i) + " of the blocks changed"); break; }
}

// ---- decode --------------------------------------------------------------------------------------------------------------

template <int KIND>
void check_decode(const Shape &s, bool merge_alpha, bool with_results)
{
    const uint64_t nblk = (uint64_t)(s.w / 4) * (s.h / 4);
    const uint32_t bb = KIND == kBcDxt1 || KIND == kBcRgtc1 ? 8 : 16;
    const uint64_t t0 = nblk * bb, t1 = merge_alpha ? nblk * 8 : 0;
    const uint64_t stride = ((t0 + t1 + 15) & ~15ull) + 32;
    std::vector<uint8_t> blocks((kFrames - 1) * stride + t0 + t1, kPad);
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint64_t i = 0; i < t0 + t1; i++) blocks[f * stride + i] = (uint8_t)rnd();
    std::vector<uint8_t> rgba(s.rgba_bytes(), kPad);
    const uint32_t results[kFrames] = {0u, 7u /* a frame whose decode failed */, 0u};
    const BcDecodeGeom g = bc_decode_geom(s.w, s.h, s.row_bytes, merge_alpha, stride, stride, s.frame_bytes);
    HAP_LAUNCH(bc_decode_kernel<KIND>, dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, blocks.data(),
               blocks.data() + t0, g, rgba.data(), with_results ? results : (const uint32_t *)nullptr);
    const std::string what = "decode kind " + std::to_string(KIND) + (merge_alpha ? " merge" : "") + (with_results ? " results " : " ") + s.name();
    int bad = 0;
    for (uint32_t f = 0; f < kFrames && !bad; f++)
        for (uint32_t by = 0; by < s.h / 4 && !bad; by++)
            for (uint32_t bx = 0; bx < s.w / 4 && !bad; bx++) {
                const uint64_t bi = (uint64_t)by * (s.w / 4) + bx;
                uint32_t v[4] = {0, 0, 0, 0}, px[16];
                memcpy(v, &blocks[f * stride + bi * bb], bb);
                decode_block(KIND, v[0], v[1], v[2], v[3], px);
                if (merge_alpha) {
                    uint32_t a[2], al[16];
                    memcpy(a, &blocks[f * stride + t0 + bi * 8], 8);
                    decode_block(kBcRgtc1, a[0], a[1], 0, 0, al);
                    for (int t = 0; t < 16; t++) px[t] = (px[t] & 0x00FFFFFFu) | ((al[t] & 0xFFu) << 24);
                }
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
                const std::vector<uint8_t> rgba = make_pictures(s);
                check_encode<kBcDxt1>(s, rgba);
                check_encode<kBcDxt5>(s, rgba);
                check_encode<kBcYCoCg>(s, rgba);
                check_encode<kBcYCoCg, true>(s, rgba);
                check_encode<kBcRgtc1>(s, rgba);
                check_encode<kBcYCoCgPlusAlpha>(s, rgba);
                check_encode<kBcYCoCgPlusAlpha, true>(s, rgba);
                for (bool with_results : {false, true}) {
                    check_decode<kBcDxt1>(s, false, with_results);
                    check_decode<kBcRgtc1>(s, false, with_results);
                    for (bool merge : {false, true}) {
                        check_decode<kBcDxt5>(s, merge, with_results);
                        check_decode<kBcYCoCg>(s, merge, with_results);
                    }
                }
                shapes++;
            }
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
