// tests/emu/test_yuv_bc7_emu.cc -- TEST INFRASTRUCTURE ONLY.
// bc_source_to_rgba8_kernel, the first of BC7's two passes from a Y'CbCr picture, under the fiber SIMT emulator: all eight
// sources (NV12, P010, and 4:2:0 / 4:2:2 / 4:4:4 on bytes and 16-bit words).  Shapes: odd block widths and one-block-wide
// pictures, pitches wider than the row (and, for the planar sources, a chroma pitch different from the luma pitch), and three
// frames with slack between them, in the input and in the RGBA8 output.  Every plane is a buffer of its own that ends with
// the last frame's last sample, and the output ends with the last frame's last texel, so under ASan a read or write past
// any of them is outside every buffer.  Input bytes past the picture and the unused bits of 16-bit words hold junk.  The
// planar depth (10 / 12) and alpha (present or NULL) alternate with the shapes.  Every texel must equal the pixel-by-pixel
// conversion of yuv_twin.h or planar_twin.h (which tests/test_yuv_cpu.py and tests/test_planar_cpu.py hold to the numpy
// definitions), with A = 255 for NV12 / P010 and for a NULL alpha plane, and every byte between frames must keep its sentinel.
#define HAPB200_EMU
#include "bc_encode.cuh"
#include "planar_twin.h"
#include "yuv_twin.h"

#include <string>
#include <vector>

using namespace hapb200;

namespace {

constexpr uint32_t kFrames = 3;
constexpr uint8_t kPad = 0xA5;
int g_fail = 0;

uint64_t g_rng = 0x452821E638D01377ull;
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
    uint32_t w, h, lpitch, cpitch, n, sub;   // n: sample depth; sub: HapB200ChromaSubsampling (NV12 / P010: 4:2:0, cpitch = lpitch)
    uint64_t frame_bytes;                    // frame stride of every plane
    bool alpha;
    uint32_t sb() const { return n == 8 ? 1 : 2; }
    std::string name() const
    {
        return std::to_string(w) + "x" + std::to_string(h) + " depth " + std::to_string(n) + " pitches " + std::to_string(lpitch) + "/" +
               std::to_string(cpitch) + " frame " + std::to_string(frame_bytes) + (alpha ? " alpha" : "");
    }
    uint64_t plane_bytes(uint32_t rows, uint32_t pitch, uint64_t row_bytes) const
    {
        return (kFrames - 1) * frame_bytes + (uint64_t)(rows - 1) * pitch + row_bytes;
    }
};

// bytes of one row: random samples (frame 0), ramps (frame 1) or flat 8x8 tiles (frame 2) of depth n in bytes or in
// 16-bit words whose other bits are junk (P010: the sample in the top 10 bits; planar: in the low n bits)
void fill_plane(uint8_t *p, const Shape &s, uint32_t f, uint32_t rows, uint32_t pitch, uint32_t samples, bool p010)
{
    const uint32_t top = 1u << s.n;
    for (uint32_t y = 0; y < rows; y++)
        for (uint32_t x = 0; x < samples; x++) {
            const uint32_t v = f == 0 ? rnd() % top : f == 1 ? (x * 7 + y * 3) % top : (((x / 8) * 31 + (y / 8) * 17) * 5) % top;
            uint8_t *at = p + f * s.frame_bytes + (uint64_t)y * pitch + (uint64_t)s.sb() * x;
            if (s.sb() == 2) {
                const uint16_t word = p010 ? (uint16_t)(v << 6 | (rnd() & 63)) : (uint16_t)(v | (rnd() << s.n));
                memcpy(at, &word, 2);
            } else {
                *at = (uint8_t)v;
            }
        }
}

std::vector<uint8_t> junk_buffer(uint64_t bytes)
{
    std::vector<uint8_t> b(bytes);
    for (auto &v : b) v = (uint8_t)rnd();
    return b;
}

// Run the kernel on the planes (luma, P / Y) and hold its RGBA8 frames to the twin's pictures `want`
template <int SRC>
void run_and_check(const Shape &s, const uint8_t *luma, const YuvSrc &y, const PlanarSrc &p, const std::vector<std::vector<uint8_t>> &want,
                   const std::string &what)
{
    const uint64_t frame_rgba = 4ull * s.w * s.h, stride = frame_rgba + 16 * (1 + s.w % 3);   // slack between frames
    std::vector<uint8_t> out((kFrames - 1) * stride + frame_rgba, kPad);                       // exact: ends with the last texel
    BcGeom g = bc_encode_geom(s.w, s.h, s.lpitch, s.frame_bytes, stride, 0);
    HAP_LAUNCH((bc_source_to_rgba8_kernel<SRC>), dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr, luma, g,
               out.data(), y, p);
    for (uint32_t f = 0; f < kFrames; f++) {
        for (uint64_t i = 0; i < frame_rgba; i += 4)
            if (memcmp(&out[f * stride + i], &want[f][i], 4) != 0) {
                const uint64_t px = i / 4;
                fail(what + ": frame " + std::to_string(f) + " texel " + std::to_string(px % s.w) + "," + std::to_string(px / s.w));
                break;
            }
        if (f + 1 < kFrames)
            for (uint64_t i = frame_rgba; i < stride; i++)
                if (out[f * stride + i] != kPad) { fail(what + ": slack byte " + std::to_string(i) + " after frame " + std::to_string(f)); break; }
    }
}

template <int SRC>
void check_yuv(const Shape &s, int cs)
{
    constexpr bool kP010 = SRC == kSrcP010;
    std::vector<uint8_t> lbuf = junk_buffer(s.plane_bytes(s.h, s.lpitch, (uint64_t)s.sb() * s.w));
    std::vector<uint8_t> cbuf = junk_buffer(s.plane_bytes(s.h / 2, s.lpitch, (uint64_t)s.sb() * s.w));
    for (uint32_t f = 0; f < kFrames; f++) {
        fill_plane(lbuf.data(), s, f, s.h, s.lpitch, s.w, kP010);
        fill_plane(cbuf.data(), s, f, s.h / 2, s.lpitch, s.w, kP010);
    }
    const int layout = kP010 ? HapB200YUV_P010 : HapB200YUV_NV12;
    std::vector<std::vector<uint8_t>> want(kFrames, std::vector<uint8_t>(4ull * s.w * s.h));
    for (uint32_t f = 0; f < kFrames; f++)
        yuv_twin::picture(lbuf.data() + f * s.frame_bytes, cbuf.data() + f * s.frame_bytes, s.w, s.h, s.lpitch, layout, cs, want[f].data());
    run_and_check<SRC>(s, lbuf.data(), yuv_src(layout, cs, cbuf.data()), PlanarSrc(), want,
                       std::string(kP010 ? "P010" : "NV12") + " cs " + std::to_string(cs) + " " + s.name());
}

template <int SRC>
void check_planar(const Shape &s, int cs)
{
    const uint32_t cw = s.sub == HapB200Chroma_444 ? s.w : s.w / 2, ch = s.sub == HapB200Chroma_420 ? s.h / 2 : s.h;
    std::vector<uint8_t> bufs[4] = {junk_buffer(s.plane_bytes(s.h, s.lpitch, (uint64_t)s.sb() * s.w)),
                                    junk_buffer(s.plane_bytes(ch, s.cpitch, (uint64_t)s.sb() * cw)),
                                    junk_buffer(s.plane_bytes(ch, s.cpitch, (uint64_t)s.sb() * cw)),
                                    junk_buffer(s.plane_bytes(s.h, s.lpitch, (uint64_t)s.sb() * s.w))};
    for (uint32_t f = 0; f < kFrames; f++) {
        fill_plane(bufs[0].data(), s, f, s.h, s.lpitch, s.w, false);
        fill_plane(bufs[1].data(), s, f, ch, s.cpitch, cw, false);
        fill_plane(bufs[2].data(), s, f, ch, s.cpitch, cw, false);
        fill_plane(bufs[3].data(), s, f, s.h, s.lpitch, s.w, false);
    }
    const uint8_t *alpha = s.alpha ? bufs[3].data() : nullptr;
    std::vector<std::vector<uint8_t>> want(kFrames, std::vector<uint8_t>(4ull * s.w * s.h));
    for (uint32_t f = 0; f < kFrames; f++) {
        const uint64_t o = f * s.frame_bytes;
        planar_twin::picture(bufs[0].data() + o, bufs[1].data() + o, bufs[2].data() + o, alpha ? alpha + o : nullptr, s.w, s.h, s.lpitch,
                             s.cpitch, s.sub, s.n, cs, want[f].data());
    }
    const PlanarSrc p = planar_src_args(s.n, cs, bufs[1].data(), bufs[2].data(), alpha, s.cpitch);
    run_and_check<SRC>(s, bufs[0].data(), YuvSrc(), p, want,
                       "planar src " + std::to_string(SRC) + " cs " + std::to_string(cs) + " " + s.name());
}

template <int SRC>
void check_source(int &shapes)
{
    constexpr bool kYuv = SRC == kSrcNv12 || SRC == kSrcP010;
    const uint32_t widths[] = {4, 12, 20, 36, 132}, heights[] = {4, 8, 20};
    const uint32_t pads[][2] = {{0, 0}, {16, 48}, {48, 0}};   // luma and chroma row padding (NV12 / P010: luma's for both)
    for (uint32_t w : widths)
        for (uint32_t h : heights)
            for (const auto &pad : pads) {
                Shape s{w, h, 0, 0, 8, HapB200Chroma_420, 0, false};
                if (SRC == kSrcP010) s.n = 10;
                if (!kYuv) {
                    s.sub = (uint32_t)planar_subsampling(SRC);
                    s.n = planar_wide(SRC) ? (shapes % 2 ? 12u : 10u) : 8u;
                    s.alpha = shapes % 3 != 2;
                }
                const uint32_t cw = s.sub == HapB200Chroma_444 ? w : w / 2;
                s.lpitch = s.sb() * w + pad[0];
                s.cpitch = kYuv ? s.lpitch : s.sb() * cw + pad[1];
                s.frame_bytes = (uint64_t)h * (s.lpitch > s.cpitch ? s.lpitch : s.cpitch) + 16 * (1 + shapes % 3);
                s.frame_bytes = (s.frame_bytes + 15) & ~15ull;
                if (kYuv) check_yuv<SRC>(s, shapes % 4);
                else check_planar<SRC>(s, shapes % 4);
                shapes++;
            }
}

}  // namespace

int main()
{
    int shapes = 0;
    check_source<kSrcNv12>(shapes);
    check_source<kSrcP010>(shapes);
    check_source<kSrcPlanar420x8>(shapes);
    check_source<kSrcPlanar420x16>(shapes);
    check_source<kSrcPlanar422x8>(shapes);
    check_source<kSrcPlanar422x16>(shapes);
    check_source<kSrcPlanar444x8>(shapes);
    check_source<kSrcPlanar444x16>(shapes);
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
