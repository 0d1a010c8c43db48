// tests/emu/test_planar_emu.cc -- TEST INFRASTRUCTURE ONLY.
// Every planar instantiation of bc_encode_planar_kernel (three subsamplings x bytes / 16-bit words x six colour kinds, and
// RGTC1 on bytes and words) under the fiber SIMT emulator.  Shapes: odd block widths and one-block-wide pictures, a
// chroma pitch different from the luma pitch, rows wider than the picture, and three frames with slack between them.
// Every plane is a buffer of its own that ends with the last frame's last sample, so a read past a plane's edge (above the
// first chroma row, past the last, right of the last column) is outside any buffer under ASan.  Bytes of the rows past the
// picture, and the bits above the sample in 16-bit words, hold junk.  Depth (10 / 12) and alpha (present or not) alternate
// with the shapes.  Each block must equal the per-block encoder of bc_block.cuh applied to the pixel-by-pixel conversion of
// planar_twin.h (which tests/test_planar_cpu.py holds to the numpy definition), and every padding byte of the output must
// keep its sentinel.
#define HAPB200_EMU
#include "bc_encode.cuh"
#include "planar_twin.h"

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
    uint32_t w, h, lpitch, cpitch, n, sub;   // n: sample depth
    uint64_t frame_bytes;                    // frame stride of every plane
    bool alpha;
    uint32_t sb() const { return n == 8 ? 1 : 2; }
    uint32_t cw() const { return sub == HapB200Chroma_444 ? w : w / 2; }
    uint32_t ch() const { return sub == HapB200Chroma_420 ? h / 2 : h; }
    std::string name() const
    {
        return std::to_string(w) + "x" + std::to_string(h) + " sub " + std::to_string(sub) + " depth " + std::to_string(n) + " pitches " +
               std::to_string(lpitch) + "/" + std::to_string(cpitch) + " frame " + std::to_string(frame_bytes) + (alpha ? " alpha" : "");
    }
    uint64_t plane_bytes(uint32_t rows, uint32_t pitch, uint32_t samples) const
    {
        return (kFrames - 1) * frame_bytes + (uint64_t)(rows - 1) * pitch + (uint64_t)sb() * samples;
    }
};

// frame 0 random samples, frame 1 ramps, frame 2 flat 8x8 tiles; 16-bit words carry junk above the sample
void fill_plane(uint8_t *p, const Shape &s, uint32_t f, uint32_t rows, uint32_t pitch, uint32_t samples)
{
    const uint32_t top = 1u << s.n;
    for (uint32_t y = 0; y < rows; y++)
        for (uint32_t x = 0; x < samples; x++) {
            uint32_t v = f == 0 ? rnd() % top : f == 1 ? (x * 7 + y * 3) % top : (((x / 8) * 31 + (y / 8) * 17) * 5) % top;
            uint8_t *at = p + f * s.frame_bytes + (uint64_t)y * pitch + (uint64_t)s.sb() * x;
            if (s.sb() == 2) { const uint16_t word = (uint16_t)(v | (rnd() << s.n)); memcpy(at, &word, 2); }
            else *at = (uint8_t)v;
        }
}

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

struct Planes {
    const uint8_t *luma, *cb, *cr, *alpha;
};

template <int KIND, bool REFINE, int SRC>
void check_encode(const Shape &s, const Planes &pl, int cs, const std::vector<std::vector<uint8_t>> &rgba)
{
    const uint64_t nblk = (uint64_t)(s.w / 4) * (s.h / 4);
    const uint64_t t0 = nblk * (KIND == kBcDxt1 || KIND == kBcRgtc1 ? 8 : 16), t1 = KIND == kBcYCoCgPlusAlpha ? nblk * 8 : 0;
    const uint64_t stride = ((t0 + t1 + 15) & ~15ull) + 48;
    std::vector<uint8_t> out((kFrames - 1) * stride + t0 + t1, kPad);
    const BcGeom g = bc_encode_geom(s.w, s.h, s.lpitch, s.frame_bytes, stride, t0);
    // as the library passes them: Hap1 and HapY get no alpha plane; RGTC1 gets the alpha plane in place of the others
    const bool reads_alpha = KIND == kBcDxt5 || KIND == kBcYCoCgPlusAlpha || KIND == kBcRgtc1;
    const uint8_t *alpha = reads_alpha ? pl.alpha : nullptr;
    const bool alpha_only = KIND == kBcRgtc1;
    const PlanarSrc p = planar_src_args(s.n, cs, alpha_only ? alpha : pl.cb, alpha_only ? alpha : pl.cr, alpha, s.cpitch);
    HAP_LAUNCH((bc_encode_planar_kernel<KIND, REFINE, SRC>), dim3(bc_ctas(g.blocks_x, g.blocks_y), kFrames), dim3(kBcThreads), 0, nullptr,
               alpha_only ? alpha : pl.luma, g, out.data(), p);
    std::vector<bool> written(out.size(), false);
    const std::string what = "kind " + std::to_string(KIND) + (REFINE ? " refine" : "") + " src " + std::to_string(SRC) + " cs " +
                             std::to_string(cs) + " " + s.name();
    for (uint32_t f = 0; f < kFrames; f++)
        for (uint32_t by = 0; by < s.h / 4; by++)
            for (uint32_t bx = 0; bx < s.w / 4; bx++) {
                uint32_t px[16];
                for (int t = 0; t < 16; t++) {
                    memcpy(&px[t], &rgba[f][4 * ((uint64_t)(4 * by + t / 4) * s.w + 4 * bx + t % 4)], 4);
                    if (!reads_alpha) px[t] |= 0xFF000000u;
                }
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
    std::vector<uint8_t> bufs[4];
    const uint64_t sizes[4] = {s.plane_bytes(s.h, s.lpitch, s.w), s.plane_bytes(s.ch(), s.cpitch, s.cw()), s.plane_bytes(s.ch(), s.cpitch, s.cw()),
                               s.plane_bytes(s.h, s.lpitch, s.w)};
    for (int i = 0; i < 4; i++) {
        bufs[i].resize(sizes[i]);
        for (auto &b : bufs[i]) b = (uint8_t)rnd();
    }
    for (uint32_t f = 0; f < kFrames; f++) {
        fill_plane(bufs[0].data(), s, f, s.h, s.lpitch, s.w);
        fill_plane(bufs[1].data(), s, f, s.ch(), s.cpitch, s.cw());
        fill_plane(bufs[2].data(), s, f, s.ch(), s.cpitch, s.cw());
        fill_plane(bufs[3].data(), s, f, s.h, s.lpitch, s.w);
    }
    const Planes pl{bufs[0].data(), bufs[1].data(), bufs[2].data(), s.alpha ? bufs[3].data() : nullptr};
    std::vector<std::vector<uint8_t>> rgba(kFrames, std::vector<uint8_t>(4ull * s.w * s.h));
    for (uint32_t f = 0; f < kFrames; f++) {
        const uint64_t o = f * s.frame_bytes;
        planar_twin::picture(pl.luma + o, pl.cb + o, pl.cr + o, pl.alpha ? pl.alpha + o : nullptr, s.w, s.h, s.lpitch, s.cpitch, s.sub, s.n,
                             cs, rgba[f].data());
    }
    check_encode<kBcDxt1, false, SRC>(s, pl, cs, rgba);
    check_encode<kBcDxt5, false, SRC>(s, pl, cs, rgba);
    check_encode<kBcYCoCg, false, SRC>(s, pl, cs, rgba);
    check_encode<kBcYCoCg, true, SRC>(s, pl, cs, rgba);
    check_encode<kBcYCoCgPlusAlpha, false, SRC>(s, pl, cs, rgba);
    check_encode<kBcYCoCgPlusAlpha, true, SRC>(s, pl, cs, rgba);
    // Hap Alpha-Only: the library instantiates RGTC1 on the 4:2:0 sources only (it reads alpha alone)
    if (s.alpha && (SRC == kSrcPlanar420x8 || SRC == kSrcPlanar420x16)) check_encode<kBcRgtc1, false, SRC>(s, pl, cs, rgba);
}

template <int SRC>
void check_source(int &shapes, uint32_t n0)
{
    const uint32_t widths[] = {4, 12, 20, 36}, heights[] = {4, 8, 20};
    const uint32_t pads[][2] = {{0, 0}, {16, 48}, {48, 0}};   // luma and chroma row padding
    for (uint32_t w : widths)
        for (uint32_t h : heights)
            for (const auto &pad : pads) {
                Shape s{w, h, 0, 0, planar_wide(SRC) ? (shapes % 2 ? 12u : 10u) : n0, (uint32_t)planar_subsampling(SRC), 0, shapes % 3 != 2};
                s.lpitch = s.sb() * w + pad[0];
                s.cpitch = s.sb() * s.cw() + pad[1];
                s.frame_bytes = (uint64_t)h * (s.lpitch > s.cpitch ? s.lpitch : s.cpitch) + 16 * (1 + shapes % 3);
                s.frame_bytes = (s.frame_bytes + 15) & ~15ull;
                check_shape<SRC>(s, shapes % 4);
                shapes++;
            }
}

}  // namespace

int main()
{
    int shapes = 0;
    check_source<kSrcPlanar420x8>(shapes, 8);
    check_source<kSrcPlanar420x16>(shapes, 10);
    check_source<kSrcPlanar422x8>(shapes, 8);
    check_source<kSrcPlanar422x16>(shapes, 10);
    check_source<kSrcPlanar444x8>(shapes, 8);
    check_source<kSrcPlanar444x16>(shapes, 10);
    printf("%d shapes x %u frames, %d failures\n", shapes, kFrames, g_fail);
    return g_fail ? 1 : 0;
}
