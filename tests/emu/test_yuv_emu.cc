// tests/emu/test_yuv_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The NV12 / P010 instantiations of bc_encode_kernel under the fiber SIMT emulator, at the geometries of test_bc_geom_emu.cc:
// odd block widths, pitches wider than the row, three frames with slack between them, and a block stride wider than the
// texture.  Two placements of the chroma plane: its own exact-size buffer (a read above the first chroma row or past the
// last is outside any buffer), and NVDEC's, inside one buffer with the luma plane at pitch * surfaceHeight, the buffer ending
// with the last frame's last chroma sample.  Bytes of the input rows past the picture hold junk.  Each block must equal the
// per-block encoder of bc_block.cuh applied to the pixel-by-pixel conversion of yuv_twin.h (which tests/test_yuv_cpu.py holds
// to the numpy definition), and every padding byte of the output must keep its sentinel.
#define HAPB200_EMU
#include "bc_encode.cuh"
#include "yuv_twin.h"

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
    uint32_t w, h, pitch, sb;   // sb: bytes per sample
    uint64_t frame_bytes;       // frame stride of both planes
    uint64_t chroma_at;         // offset of the chroma plane from luma when the two share a buffer (NVDEC); 0: buffers of their own
    std::string name() const
    {
        return std::to_string(w) + "x" + std::to_string(h) + " pitch " + std::to_string(pitch) + " frame " + std::to_string(frame_bytes) +
               (chroma_at ? " chroma at " + std::to_string(chroma_at) : " separate planes");
    }
    uint64_t plane_bytes(uint32_t rows) const { return (kFrames - 1) * frame_bytes + (uint64_t)(rows - 1) * pitch + (uint64_t)sb * w; }
};

// frame 0 random samples, frame 1 ramps, frame 2 flat 8x8 tiles; P010 words carry junk in their low 6 bits
void fill_plane(uint8_t *p, const Shape &s, uint32_t f, uint32_t rows, uint32_t samples_per_row)
{
    const uint32_t top = s.sb == 2 ? 1024 : 256;
    for (uint32_t y = 0; y < rows; y++)
        for (uint32_t x = 0; x < samples_per_row; x++) {
            uint32_t v = f == 0 ? rnd() % top : f == 1 ? (x * 7 + y * 3) % top : (((x / 8) * 31 + (y / 8) * 17) * 5) % top;
            uint8_t *at = p + f * s.frame_bytes + (uint64_t)y * s.pitch + (uint64_t)s.sb * x;
            if (s.sb == 2) { const uint16_t word = (uint16_t)(v << 6 | (rnd() & 63)); memcpy(at, &word, 2); }
            else *at = (uint8_t)v;
        }
}

template <int KIND, bool REFINE>
int expected_block(const uint32_t px[16], int plane, uint8_t out[16])
{
    Block8 a, c;
    if (plane == 1) { a = encode_rgtc1_alpha(px); memcpy(out, &a, 8); return 8; }
    if (KIND == kBcDxt1) { c = encode_dxt1(px); memcpy(out, &c, 8); return 8; }
    if (KIND == kBcDxt5) encode_dxt5(px, a, c);
    else encode_ycocg_dxt5<REFINE>(px, a, c);
    memcpy(out, &a, 8);
    memcpy(out + 8, &c, 8);
    return 16;
}

template <int KIND, bool REFINE, int SRC>
void check_encode(const Shape &s, const uint8_t *luma, const uint8_t *chroma, int cs, const std::vector<std::vector<uint8_t>> &rgba)
{
    const uint64_t nblk = (uint64_t)(s.w / 4) * (s.h / 4);
    const uint64_t t0 = nblk * (KIND == kBcDxt1 ? 8 : 16), t1 = KIND == kBcYCoCgPlusAlpha ? nblk * 8 : 0;
    const uint64_t stride = ((t0 + t1 + 15) & ~15ull) + 48;
    std::vector<uint8_t> out((kFrames - 1) * stride + t0 + t1, kPad);
    const BcGeom g = bc_encode_geom(s.w, s.h, s.pitch, s.frame_bytes, stride, t0);
    const YuvSrc y = yuv_src(SRC == kSrcP010 ? HapB200YUV_P010 : HapB200YUV_NV12, cs, chroma);
    HAP_LAUNCH((bc_encode_kernel<KIND, REFINE, SRC>), dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, luma, g,
               out.data(), y);
    std::vector<bool> written(out.size(), false);
    const std::string what = "kind " + std::to_string(KIND) + (REFINE ? " refine" : "") + (SRC == kSrcP010 ? " P010" : " NV12") + " cs " +
                             std::to_string(cs) + " " + s.name();
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint32_t by = 0; by < s.h / 4; by++)
            for (uint32_t bx = 0; bx < s.w / 4; bx++) {
                uint32_t px[16];
                for (int t = 0; t < 16; t++) memcpy(&px[t], &rgba[f][4 * ((uint64_t)(4 * by + t / 4) * s.w + 4 * bx + t % 4)], 4);
                const uint64_t bi = (uint64_t)by * (s.w / 4) + bx;
                for (int plane = 0; plane < (t1 ? 2 : 1); plane++) {
                    uint8_t want[16];
                    const int n = expected_block<KIND, REFINE>(px, plane, want);
                    const uint64_t at = f * stride + (plane ? t0 : 0) + bi * n;
                    if (memcmp(&out[at], want, n) != 0)
                        fail(what + ": frame " + std::to_string(f) + " block " + std::to_string(bx) + "," + std::to_string(by) + " plane " +
                             std::to_string(plane));
                    for (int k = 0; k < n; k++) written[at + k] = true;
                }
            }
    for (size_t i = 0; i < out.size(); i++)
        if (!written[i] && out[i] != kPad) { fail(what + ": padding byte " + std::to_string(i) + " of the blocks changed"); break; }
}

template <int SRC>
void check_shape(const Shape &s, int cs)
{
    // the planes: one buffer each, or one buffer for both with chroma at chroma_at; either ends with the last sample
    std::vector<uint8_t> lbuf, cbuf;
    const uint8_t *luma, *chroma;
    if (s.chroma_at) {
        lbuf.resize(s.chroma_at + s.plane_bytes(s.h / 2));
        for (auto &b : lbuf) b = (uint8_t)rnd();
        luma = lbuf.data();
        chroma = lbuf.data() + s.chroma_at;
    } else {
        lbuf.resize(s.plane_bytes(s.h));
        cbuf.resize(s.plane_bytes(s.h / 2));
        for (auto &b : lbuf) b = (uint8_t)rnd();
        for (auto &b : cbuf) b = (uint8_t)rnd();
        luma = lbuf.data();
        chroma = cbuf.data();
    }
    for (uint32_t f = 0; f < kFrames; f++) {
        fill_plane(const_cast<uint8_t *>(luma), s, f, s.h, s.w);
        fill_plane(const_cast<uint8_t *>(chroma), s, f, s.h / 2, s.w);
    }
    const int layout = SRC == kSrcP010 ? HapB200YUV_P010 : HapB200YUV_NV12;
    std::vector<std::vector<uint8_t>> rgba(kFrames, std::vector<uint8_t>(4ull * s.w * s.h));
    for (uint32_t f = 0; f < kFrames; f++)
        yuv_twin::picture(luma + f * s.frame_bytes, chroma + f * s.frame_bytes, s.w, s.h, s.pitch, layout, cs, rgba[f].data());
    check_encode<kBcDxt1, false, SRC>(s, luma, chroma, cs, rgba);
    check_encode<kBcDxt5, false, SRC>(s, luma, chroma, cs, rgba);
    check_encode<kBcYCoCg, false, SRC>(s, luma, chroma, cs, rgba);
    check_encode<kBcYCoCg, true, SRC>(s, luma, chroma, cs, rgba);
    check_encode<kBcYCoCgPlusAlpha, false, SRC>(s, luma, chroma, cs, rgba);
    check_encode<kBcYCoCgPlusAlpha, true, SRC>(s, luma, chroma, cs, rgba);
}

}  // namespace

int main()
{
    const uint32_t widths[] = {4, 8, 12, 20, 36, 132}, heights[] = {4, 8, 12, 20}, pads[] = {0, 16, 48};
    int shapes = 0;
    for (uint32_t sb : {1u, 2u})
        for (uint32_t w : widths)
            for (uint32_t h : heights)
                for (uint32_t pad : pads)
                    for (bool nvdec : {false, true}) {
                        Shape s{w, h, sb * w + pad, sb, 0, 0};
                        const uint64_t surface_rows = h + (nvdec ? 8 : 0);   // NVDEC: chroma after a taller surface
                        s.frame_bytes = nvdec ? (surface_rows + h / 2) * s.pitch + 16 * (1 + shapes % 3)
                                              : (uint64_t)h * s.pitch + 16 * (1 + shapes % 3);
                        s.chroma_at = nvdec ? surface_rows * s.pitch : 0;
                        const int cs = shapes % 4;
                        if (sb == 2) check_shape<kSrcP010>(s, cs);
                        else check_shape<kSrcNv12>(s, cs);
                        shapes++;
                    }
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
