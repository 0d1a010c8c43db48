// tests/emu/test_yuv_pq_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The HDR10 instantiation of bc6h_encode_kernel (P010, BT.2020, PQ -> Hap HDR blocks) under the fiber SIMT emulator: odd
// block widths, pitches wider than the row, three frames with slack between them, a block stride wider than the texture,
// UF16 and SF16, both ranges and several unitNits.  Two placements of the chroma plane: its own exact-size buffer (a read
// above the first chroma row or past the last is outside any buffer), and NVDEC's, inside one buffer with the luma plane at
// pitch * surfaceHeight, the buffer ending with the last frame's last chroma sample.  Bytes of the input rows past the
// picture hold junk, and P010 words carry junk in their low 6 bits.  Each block must equal bc6h_encode_block (the host twin
// of the RGBA16F encoder) applied to the pixel-by-pixel conversion of yuv_pq_twin.h, and every padding byte of the output
// must keep its sentinel.  Pictures are small: the BC6H search is slow on a CPU.
#define HAPB200_EMU
#include "bc6h_encode.cuh"
#include "yuv_pq_twin.h"

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
    uint32_t w, h, pitch;
    uint64_t frame_bytes;       // frame stride of both planes
    uint64_t chroma_at;         // offset of the chroma plane from luma when the two share a buffer (NVDEC); 0: buffers of their own
    std::string name() const
    {
        return std::to_string(w) + "x" + std::to_string(h) + " pitch " + std::to_string(pitch) + " frame " + std::to_string(frame_bytes) +
               (chroma_at ? " chroma at " + std::to_string(chroma_at) : " separate planes");
    }
    uint64_t plane_bytes(uint32_t rows) const { return (kFrames - 1) * frame_bytes + (uint64_t)(rows - 1) * pitch + 2ull * w; }
};

// frame 0 random 10-bit samples, frame 1 ramps, frame 2 flat 8x8 tiles (constant blocks); junk in the low 6 bits
void fill_plane(uint8_t *p, const Shape &s, uint32_t f, uint32_t rows)
{
    for (uint32_t y = 0; y < rows; y++)
        for (uint32_t x = 0; x < s.w; x++) {
            const uint32_t v = f == 0 ? rnd() % 1024 : f == 1 ? (x * 37 + y * 11) % 1024 : (((x / 8) * 31 + (y / 8) * 17) * 29) % 1024;
            const uint16_t word = (uint16_t)(v << 6 | (rnd() & 63));
            memcpy(p + f * s.frame_bytes + (uint64_t)y * s.pitch + 2ull * x, &word, 2);
        }
}

void check_shape(const Shape &s, int cs, uint32_t unit_nits, bool sgn)
{
    std::vector<uint8_t> lbuf, cbuf;
    uint8_t *luma, *chroma;
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
        fill_plane(luma, s, f, s.h);
        fill_plane(chroma, s, f, s.h / 2);
    }
    std::vector<uint16_t> table(4096);
    yuv_pq_table(unit_nits, table.data());

    const uint64_t nblk = (uint64_t)(s.w / 4) * (s.h / 4), t0 = 16 * nblk, stride = ((t0 + 15) & ~15ull) + 48;
    std::vector<uint8_t> out((kFrames - 1) * stride + t0, kPad);
    const BcGeom g = bc_encode_geom(s.w, s.h, s.pitch, s.frame_bytes, stride, 0);
    const YuvPqSrc k = yuv_pq_src(cs, chroma, table.data());
    HAP_LAUNCH(bc6h_encode_kernel<kSrcP010Pq>, dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, luma, g,
               out.data(), sgn ? 1u : 0u, k);
    const std::string what = std::string(sgn ? "SF16" : "UF16") + " cs " + std::to_string(cs) + " unit " + std::to_string(unit_nits) + " " +
                             s.name();
    std::vector<uint16_t> rgba(4ull * s.w * s.h);
    for (uint32_t f = 0; f < kFrames; f++) {
        yuv_pq_twin::picture(luma + f * s.frame_bytes, chroma + f * s.frame_bytes, s.w, s.h, s.pitch, cs, table.data(), rgba.data());
        for (uint64_t b = 0; b < nblk; b++) {
            const uint32_t by = (uint32_t)(b / (s.w / 4)), bx = (uint32_t)(b % (s.w / 4));
            uint32_t px[32], want[4];
            for (int t = 0; t < 16; t++) memcpy(&px[2 * t], &rgba[4 * ((uint64_t)(4 * by + t / 4) * s.w + 4 * bx + t % 4)], 8);
            bc6h_encode_block(px, sgn, want);
            if (memcmp(want, &out[f * stride + 16 * b], 16)) {
                fail(what + ": frame " + std::to_string(f) + " block " + std::to_string(bx) + "," + std::to_string(by));
                return;
            }
        }
    }
    for (uint32_t f = 0; f + 1 < kFrames; f++)
        for (uint64_t i = t0; i < stride; i++)
            if (out[f * stride + i] != kPad) { fail(what + ": padding after frame " + std::to_string(f) + " changed"); return; }
}

}  // namespace

int main()
{
    const uint32_t widths[] = {4, 12, 36}, heights[] = {4, 8, 12}, pads[] = {0, 48}, units[] = {1, 80, 100, 203, 1000, 10000};
    int shapes = 0;
    for (uint32_t w : widths)
        for (uint32_t h : heights)
            for (uint32_t pad : pads)
                for (bool nvdec : {false, true}) {
                    Shape s{w, h, 2 * w + pad, 0, 0};
                    const uint64_t surface_rows = h + (nvdec ? 8 : 0);   // NVDEC: chroma after a taller surface
                    s.frame_bytes = nvdec ? (surface_rows + h / 2) * s.pitch + 16 * (1 + shapes % 3) : (uint64_t)h * s.pitch + 16 * (1 + shapes % 3);
                    s.chroma_at = nvdec ? surface_rows * s.pitch : 0;
                    check_shape(s, HapB200YUV_BT2020_Limited + shapes % 2, units[shapes % 6], (shapes / 2) % 2 != 0);
                    shapes++;
                }
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
