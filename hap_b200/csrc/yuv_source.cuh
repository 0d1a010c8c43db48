// hap_b200/csrc/yuv_source.cuh -- the NV12 / P010 source of the K1-K4 block encoders: 4:2:0 Y'CbCr -> RGBA8 in registers.
//
// The conversion is defined exactly, in integers, in include/hap_b200.h (HapB200EncodeYUV): bilinear chroma upsampling at
// the MPEG-2 / H.264 / HEVC default siting, then one fixed-point dot product per channel with the coefficients of
// HAPB200_YUV_COEFFICIENTS.  The thread that owns a 4x4 block (bc_encode.cuh) reads its 16 luma samples and the 4 x 3 chroma
// pairs around them, converts, and hands px[16] to the unchanged block fit, so a YUV picture encodes to exactly the bytes of
// the RGBA8 picture this conversion makes of it.  Every load stays inside the two planes: the chroma row above, the row
// below and the column to the right are clamped at the picture's edges, as the definition clamps them.
//
// The planar sources (load_block_planar; HapB200EncodePlanar: 4:2:0, 4:2:2 and 4:4:4, 8, 10 or 12 bits, optional alpha)
// feed bc_encode_planar_kernel the same way: 4:2:0 through the same filter (upsample_block_420), 4:2:2 through its
// horizontal half (upsample_row_h), 4:4:4 as it is.
//
// The NV12 / P010 gather also feeds the HDR10 source of the BC6H encoder (bc6h_encode.cuh, HapB200EncodeYUVPQ): P010 BT.2020 -> 12-bit
// R'G'B' (HAPB200_YUV_PQ_COEFFICIENTS) -> linear binary16 through the PQ table T, built on the host (yuv_pq_table).
#pragma once
#include "bc_block.cuh"
#include "../../include/hap_b200.h"

namespace hapb200 {

// The picture a block encoder reads (the SRC parameter of bc_encode_kernel: RGBA8, NV12, P010; of bc6h_encode_kernel:
// RGBA16F, HDR10 P010; of bc_encode_planar_kernel: the planar pictures, one per subsampling and sample width, x8 bytes and
// x16 little-endian 16-bit words holding 10- or 12-bit samples in their low bits)
enum BcSource : int {
    kSrcRgba8 = 0, kSrcNv12 = 1, kSrcP010 = 2, kSrcRgbaHalf = 3, kSrcP010Pq = 4,
    kSrcPlanar420x8 = 5, kSrcPlanar420x16 = 6, kSrcPlanar422x8 = 7, kSrcPlanar422x16 = 8, kSrcPlanar444x8 = 9, kSrcPlanar444x16 = 10
};

// What a YUV source adds to BcGeom: the chroma plane (frame f at chroma + f*frame_bytes, rows row_bytes apart, as luma)
// and the row of HAPB200_YUV_COEFFICIENTS.  Unused by the RGBA8 source.
struct YuvSrc {
    const uint8_t *chroma;
    int32_t cy, cr_r, cb_g, cr_g, cb_b, y_off, c_off8;   // c_off8 = 8 * cOff: the chroma offset in eighths
};

// the coefficients of layout (HapB200YUVLayout) and colorSpace (HapB200YUVColorSpace); both in range
inline YuvSrc yuv_src(unsigned layout, unsigned color_space, const uint8_t *chroma)
{
    static const int32_t kCoeffs[8][7] = HAPB200_YUV_COEFFICIENTS;
    const int32_t *k = kCoeffs[layout * 4 + color_space];
    return YuvSrc{chroma, k[0], k[1], k[2], k[3], k[4], k[5], 8 * k[6]};
}

HAP_HD uint32_t yuv_clamp8(int32_t v) { return (uint32_t)(v < 0 ? 0 : v > 255 ? 255 : v); }

// one pixel: luma sample y, upsampled chroma cb8 / cr8 in eighths -> RGBA8 (R in the low byte, A = 255)
HAP_HD uint32_t yuv_pixel(int32_t y, int32_t cb8, int32_t cr8, const YuvSrc &k)
{
    const int32_t l = k.cy * (y - k.y_off), cb = cb8 - k.c_off8, cr = cr8 - k.c_off8;
    const uint32_t r = yuv_clamp8((l + k.cr_r * cr + 32768) >> 16);
    const uint32_t g = yuv_clamp8((l + k.cb_g * cb + k.cr_g * cr + 32768) >> 16);
    const uint32_t b = yuv_clamp8((l + k.cb_b * cb + 32768) >> 16);
    return r | g << 8 | b << 16 | 0xFF000000u;
}

// Local chroma row r (0..3) of block row by: chroma row 2by-1+r, clamped to the 4:2:0 plane's rows
HAP_HD uint32_t yuv420_chroma_row(int r, uint32_t by, uint32_t blocks_y)
{
    return r == 0 ? (by > 0 ? 2 * by - 1 : 0) : r == 3 ? (by + 1 < blocks_y ? 2 * by + 2 : 2 * by + 1) : 2 * by + r - 1;
}

// Luma row yl of a block with vertically filtered chroma vb / vr (columns 2bx .. 2bx+2, in quarters) -> pixel(t, Y, Cb8, Cr8)
// for its four texels: columns 4bx+xl have chroma column i = 2bx + xl/2, local column xl/2; odd columns average it with the
// next one.
template <class Pixel>
HAP_HD void upsample_row_h(int yl, const int32_t y[4], const int32_t vb[3], const int32_t vr[3], const Pixel &pixel)
{
    pixel(4 * yl + 0, y[0], 2 * vb[0], 2 * vr[0]);
    pixel(4 * yl + 1, y[1], vb[0] + vb[1], vr[0] + vr[1]);
    pixel(4 * yl + 2, y[2], 2 * vb[1], 2 * vr[1]);
    pixel(4 * yl + 3, y[3], vb[1] + vb[2], vr[1] + vr[2]);
}

// The 4:2:0 filter of a block: cb[r][c], cr[r][c] are chroma rows 2by-1+r and columns 2bx+c, clamped; luma(yl, y[4]) loads
// luma row yl.  Shared by the NV12 / P010 gather (interleaved chroma) and the planar 4:2:0 gather (load_block_planar).
template <class Luma, class Pixel>
HAP_HD void upsample_block_420(const int32_t cb[4][3], const int32_t cr[4][3], const Luma &luma, const Pixel &pixel)
{
#pragma unroll
    for (int yl = 0; yl < 4; yl++) {
        // luma row 4by+yl: chroma row j = 2by + yl/2 is local row 1 + yl/2; its neighbour is the row above (y even) or below
        const int rj = 1 + yl / 2, rn = (yl & 1) ? rj + 1 : rj - 1;
        int32_t vb[3], vr[3];   // vertically filtered chroma of the three columns, in quarters
#pragma unroll
        for (int c = 0; c < 3; c++) { vb[c] = 3 * cb[rj][c] + cb[rn][c]; vr[c] = 3 * cr[rj][c] + cr[rn][c]; }
        int32_t y[4];
        luma(yl, y);
        upsample_row_h(yl, y, vb, vr, pixel);
    }
}

// The 4:2:0 gather of block (bx, by) of a blocks_x x blocks_y picture: pixel(t, Y, Cb8, Cr8) for its texels t = 4*row + column,
// Cb8 / Cr8 upsampled in eighths.  luma / chroma: this frame's planes, rows `pitch` bytes apart.  Luma: 4 rows of 4 samples.
// Chroma: rows 2by-1 .. 2by+2 and pair columns 2bx .. 2bx+2, clamped (so at the edges the row above, the row below and the
// right column are the block's own outermost ones, and are not loaded).  Shared by the RGBA8 (load_block_yuv) and the
// HDR10 (load_block_yuv_pq) conversions.
template <int SRC, class Pixel>
HAP_HD void gather_block_yuv(const uint8_t *luma, const uint8_t *chroma, uint32_t pitch, uint32_t bx, uint32_t by, uint32_t blocks_x,
                             uint32_t blocks_y, const Pixel &pixel)
{
    constexpr bool kP010 = SRC == kSrcP010;
    constexpr uint32_t kPair = kP010 ? 4 : 2;            // bytes of one Cb, Cr pair
    const bool right = bx + 1 < blocks_x;                // chroma column 2bx+2 exists
    // cb[r][c], cr[r][c]: chroma rows 2by-1+r, columns 2bx+c
    int32_t cb[4][3], cr[4][3];
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const uint32_t row = yuv420_chroma_row(r, by, blocks_y);
        const uint8_t *c = chroma + (uint64_t)row * pitch + (uint64_t)(2 * bx) * kPair;
        if (kP010) {
            const uint2 v = *reinterpret_cast<const uint2 *>(c);
            const uint32_t n = right ? *reinterpret_cast<const uint32_t *>(c + 8) : v.y;
            cb[r][0] = (v.x & 0xFFFF) >> 6; cr[r][0] = v.x >> 22;
            cb[r][1] = (v.y & 0xFFFF) >> 6; cr[r][1] = v.y >> 22;
            cb[r][2] = (n & 0xFFFF) >> 6;   cr[r][2] = n >> 22;
        } else {
            const uint32_t v = *reinterpret_cast<const uint32_t *>(c);
            const uint32_t n = right ? *reinterpret_cast<const uint16_t *>(c + 4) : v >> 16;
            cb[r][0] = v & 0xFF;         cr[r][0] = (v >> 8) & 0xFF;
            cb[r][1] = (v >> 16) & 0xFF; cr[r][1] = v >> 24;
            cb[r][2] = n & 0xFF;         cr[r][2] = (n >> 8) & 0xFF;
        }
    }
    upsample_block_420(cb, cr, [&](int yl, int32_t y[4]) {
        const uint8_t *l = luma + (uint64_t)(4 * by + yl) * pitch;
        if (kP010) {
            const uint2 v = *reinterpret_cast<const uint2 *>(l + 8ull * bx);
            y[0] = (v.x & 0xFFFF) >> 6; y[1] = v.x >> 22; y[2] = (v.y & 0xFFFF) >> 6; y[3] = v.y >> 22;
        } else {
            const uint32_t v = *reinterpret_cast<const uint32_t *>(l + 4ull * bx);
            y[0] = v & 0xFF; y[1] = (v >> 8) & 0xFF; y[2] = (v >> 16) & 0xFF; y[3] = v >> 24;
        }
    }, pixel);
}

struct YuvRgba8Pixel {
    const YuvSrc &k;
    uint32_t *px;
    HAP_HD void operator()(int t, int32_t y, int32_t cb8, int32_t cr8) const { px[t] = yuv_pixel(y, cb8, cr8, k); }
};

// Block (bx, by) -> px[16], RGBA8 (bc_encode_kernel's YUV source)
template <int SRC>
HAP_HD void load_block_yuv(const uint8_t *luma, const uint8_t *chroma, uint32_t pitch, uint32_t bx, uint32_t by, uint32_t blocks_x,
                           uint32_t blocks_y, const YuvSrc &k, uint32_t px[16])
{
    gather_block_yuv<SRC>(luma, chroma, pitch, bx, by, blocks_x, blocks_y, YuvRgba8Pixel{k, px});
}

// ---- planar Y'CbCr 4:2:0 / 4:2:2 / 4:4:4 with an optional alpha plane (bc_encode_planar_kernel; HapB200EncodePlanar) ------

// The planar sources (BcSource) by subsampling (HapB200ChromaSubsampling) and sample width
constexpr bool is_planar_src(int src) { return src >= kSrcPlanar420x8 && src <= kSrcPlanar444x16; }
constexpr int planar_src(unsigned subsampling, bool wide) { return kSrcPlanar420x8 + 2 * (int)subsampling + (wide ? 1 : 0); }
constexpr int planar_subsampling(int src) { return (src - kSrcPlanar420x8) / 2; }
constexpr bool planar_wide(int src) { return (src - kSrcPlanar420x8) % 2 == 1; }

// What a planar source adds to BcGeom (luma is the kernel's picture pointer): the Cb plane (m.chroma) and the row of the
// matrix (m), the Cr and alpha planes (alpha nullptr: A = 255), all frame_bytes apart per frame; the chroma planes' pitch;
// the sample mask 2^n - 1 and the matrix's shift (16, or 18 at n = 12); and alpha_mul = ceil(2^42 / (2 (2^n - 1))), which
// makes A = ((510 a + 2^n - 1) * alpha_mul) >> 42 the definition's integer division for n = 10 and 12 (the numerator is
// below 2^21, so the reciprocal's error, below 2^-21, never reaches the next multiple of the divisor).  Uniform per launch.
struct PlanarSrc {
    YuvSrc m;
    const uint8_t *cr, *alpha;
    uint32_t chroma_pitch, mask, shift, alpha_mul;
};

// bit_depth 8, 10 or 12; color_space BT.601 / BT.709 limited / full (both in range)
inline PlanarSrc planar_src_args(unsigned bit_depth, unsigned color_space, const uint8_t *cb, const uint8_t *cr, const uint8_t *alpha,
                                 uint32_t chroma_pitch)
{
    static const int32_t k12[4][7] = HAPB200_YUV_12BIT_COEFFICIENTS;
    YuvSrc m = yuv_src(bit_depth == 8 ? HapB200YUV_NV12 : HapB200YUV_P010, color_space, cb);
    if (bit_depth == 12) {
        const int32_t *k = k12[color_space];
        m = YuvSrc{cb, k[0], k[1], k[2], k[3], k[4], k[5], 8 * k[6]};
    }
    const uint32_t mask = (1u << bit_depth) - 1, d = 2 * mask;
    const uint32_t alpha_mul = bit_depth == 8 ? 0u : (uint32_t)(((1ull << 42) + d - 1) / d);   // (8-bit alpha is taken as it is)
    return PlanarSrc{m, cr, alpha, chroma_pitch, mask, bit_depth == 12 ? 18u : 16u, alpha_mul};
}

// one pixel: sample y, upsampled chroma cb8 / cr8 in eighths -> R | G << 8 | B << 16 (A = 0)
HAP_HD uint32_t planar_rgb(int32_t y, int32_t cb8, int32_t cr8, const PlanarSrc &p)
{
    const YuvSrc &k = p.m;
    const int32_t l = k.cy * (y - k.y_off), cb = cb8 - k.c_off8, cr = cr8 - k.c_off8, half = 1 << (p.shift - 1);
    const uint32_t r = yuv_clamp8((l + k.cr_r * cr + half) >> p.shift);
    const uint32_t g = yuv_clamp8((l + k.cb_g * cb + k.cr_g * cr + half) >> p.shift);
    const uint32_t b = yuv_clamp8((l + k.cb_b * cb + half) >> p.shift);
    return r | g << 8 | b << 16;
}

// an alpha sample of 10 or 12 bits -> A (the integer division of include/hap_b200.h)
HAP_HD uint32_t planar_alpha16(uint32_t a, const PlanarSrc &p) { return (uint32_t)(((uint64_t)(510 * a + p.mask) * p.alpha_mul) >> 42); }

// Row `row` of a plane, samples 4bx .. 4bx+3 (one 4- or 8-byte load), the 16-bit ones masked
template <bool WIDE>
HAP_HD void planar_load4(const uint8_t *plane, uint64_t row, uint32_t pitch, uint32_t bx, uint32_t mask, int32_t s[4])
{
    const uint8_t *l = plane + row * pitch;
    if (WIDE) {
        const uint2 v = *reinterpret_cast<const uint2 *>(l + 8ull * bx);
        s[0] = v.x & mask; s[1] = (v.x >> 16) & mask; s[2] = v.y & mask; s[3] = (v.y >> 16) & mask;
    } else {
        const uint32_t v = *reinterpret_cast<const uint32_t *>(l + 4ull * bx);
        s[0] = v & 0xFF; s[1] = (v >> 8) & 0xFF; s[2] = (v >> 16) & 0xFF; s[3] = v >> 24;
    }
}

// Row `row` of a half-width chroma plane, samples 2bx, 2bx+1 and 2bx+2 (clamped to 2bx+1 when `right` is false: the block
// is the rightmost and column 2bx+2 is past the plane, so it is not loaded)
template <bool WIDE>
HAP_HD void planar_load3(const uint8_t *plane, uint64_t row, uint32_t pitch, uint32_t bx, bool right, uint32_t mask, int32_t s[3])
{
    const uint8_t *c = plane + row * pitch;
    if (WIDE) {
        const uint32_t v = *reinterpret_cast<const uint32_t *>(c + 4ull * bx);
        const uint32_t n = right ? *reinterpret_cast<const uint16_t *>(c + 4ull * bx + 4) : v >> 16;
        s[0] = v & mask; s[1] = (v >> 16) & mask; s[2] = n & mask;
    } else {
        const uint32_t v = *reinterpret_cast<const uint16_t *>(c + 2ull * bx);
        const uint32_t n = right ? c[2ull * bx + 2] : v >> 8;
        s[0] = v & 0xFF; s[1] = v >> 8; s[2] = n;
    }
}

// Block (bx, by) of planar picture SRC (this frame's luma plane `luma`, rows `pitch` apart; the other planes in p, already
// offset to this frame) -> px[16], RGBA8.  ALPHA: the kind encodes alpha (DXT5, YCoCg + RGTC1, RGTC1); otherwise, or when
// p.alpha is nullptr, A = 255.  COLOUR: the kind encodes colour (all but RGTC1, which reads the alpha plane alone).
template <int SRC, bool COLOUR, bool ALPHA>
HAP_HD void load_block_planar(const uint8_t *luma, uint32_t pitch, uint32_t bx, uint32_t by, uint32_t blocks_x, uint32_t blocks_y,
                              const PlanarSrc &p, uint32_t px[16])
{
    constexpr bool kWide = planar_wide(SRC);
    constexpr int kSub = planar_subsampling(SRC);
    const auto pixel = [&](int t, int32_t y, int32_t cb8, int32_t cr8) { px[t] = planar_rgb(y, cb8, cr8, p); };
    const auto luma_row = [&](int yl, int32_t y[4]) { planar_load4<kWide>(luma, 4 * by + yl, pitch, bx, p.mask, y); };
    if (!COLOUR) {
#pragma unroll
        for (int t = 0; t < 16; t++) px[t] = 0;
    } else if (kSub == HapB200Chroma_420) {
        const bool right = bx + 1 < blocks_x;
        int32_t cb[4][3], cr[4][3];
#pragma unroll
        for (int r = 0; r < 4; r++) {
            const uint32_t row = yuv420_chroma_row(r, by, blocks_y);
            planar_load3<kWide>(p.m.chroma, row, p.chroma_pitch, bx, right, p.mask, cb[r]);
            planar_load3<kWide>(p.cr, row, p.chroma_pitch, bx, right, p.mask, cr[r]);
        }
        upsample_block_420(cb, cr, luma_row, pixel);
    } else if (kSub == HapB200Chroma_422) {
        const bool right = bx + 1 < blocks_x;
#pragma unroll
        for (int yl = 0; yl < 4; yl++) {
            int32_t vb[3], vr[3], y[4];   // vertical weight 4: the row's own chroma in quarters
            planar_load3<kWide>(p.m.chroma, 4 * by + yl, p.chroma_pitch, bx, right, p.mask, vb);
            planar_load3<kWide>(p.cr, 4 * by + yl, p.chroma_pitch, bx, right, p.mask, vr);
#pragma unroll
            for (int c = 0; c < 3; c++) { vb[c] *= 4; vr[c] *= 4; }
            luma_row(yl, y);
            upsample_row_h(yl, y, vb, vr, pixel);
        }
    } else {
#pragma unroll
        for (int yl = 0; yl < 4; yl++) {
            int32_t cb[4], cr[4], y[4];
            planar_load4<kWide>(p.m.chroma, 4 * by + yl, p.chroma_pitch, bx, p.mask, cb);
            planar_load4<kWide>(p.cr, 4 * by + yl, p.chroma_pitch, bx, p.mask, cr);
            luma_row(yl, y);
#pragma unroll
            for (int xl = 0; xl < 4; xl++) pixel(4 * yl + xl, y[xl], 8 * cb[xl], 8 * cr[xl]);
        }
    }
    if (ALPHA && p.alpha) {
#pragma unroll
        for (int yl = 0; yl < 4; yl++) {
            int32_t a[4];
            planar_load4<kWide>(p.alpha, 4 * by + yl, pitch, bx, p.mask, a);
#pragma unroll
            for (int xl = 0; xl < 4; xl++) px[4 * yl + xl] |= (kWide ? planar_alpha16((uint32_t)a[xl], p) : (uint32_t)a[xl]) << 24;
        }
    } else {
#pragma unroll
        for (int t = 0; t < 16; t++) px[t] |= 0xFF000000u;
    }
}

// ---- HDR10: P010, BT.2020, PQ -> linear RGBA16F (bc6h_encode_kernel's kSrcP010Pq source; HapB200EncodeYUVPQ) ----------

// What the HDR10 source adds to BcGeom: the chroma plane (as YuvSrc), the row of HAPB200_YUV_PQ_COEFFICIENTS and the
// transfer table T (4096 binary16 values in device memory, read with __ldg: the index is lane-dependent, so a __constant__
// or parameter table would serialise; 8 KiB stay in L1).  Unused by the RGBA16F source.
struct YuvPqSrc {
    YuvSrc m;
    const uint16_t *table;
};

// colorSpace HapB200YUV_BT2020_Limited or _Full
inline YuvPqSrc yuv_pq_src(unsigned color_space, const uint8_t *chroma, const uint16_t *table)
{
    static const int32_t kCoeffs[2][7] = HAPB200_YUV_PQ_COEFFICIENTS;
    const int32_t *k = kCoeffs[color_space - HapB200YUV_BT2020_Limited];
    return YuvPqSrc{YuvSrc{chroma, k[0], k[1], k[2], k[3], k[4], k[5], 8 * k[6]}, table};
}

#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD uint32_t yuv_pq_lookup(const uint16_t *table, uint32_t c) { return table[c]; }
#else
__device__ __forceinline__ uint32_t yuv_pq_lookup(const uint16_t *table, uint32_t c) { return __ldg(table + c); }
#endif

HAP_HD uint32_t yuv_clamp12(int32_t v) { return (uint32_t)(v < 0 ? 0 : v > 4095 ? 4095 : v); }

// one pixel: luma sample y, upsampled chroma cb8 / cr8 in eighths -> R | G << 16 and B | 1.0 << 16 in binary16
HAP_HD void yuv_pq_pixel(int32_t y, int32_t cb8, int32_t cr8, const YuvPqSrc &p, uint32_t &rg, uint32_t &ba)
{
    const YuvSrc &k = p.m;
    const int32_t l = k.cy * (y - k.y_off), cb = cb8 - k.c_off8, cr = cr8 - k.c_off8;
    const uint32_t r = yuv_clamp12((l + k.cr_r * cr + 32768) >> 16);
    const uint32_t g = yuv_clamp12((l + k.cb_g * cb + k.cr_g * cr + 32768) >> 16);
    const uint32_t b = yuv_clamp12((l + k.cb_b * cb + 32768) >> 16);
    rg = yuv_pq_lookup(p.table, r) | yuv_pq_lookup(p.table, g) << 16;
    ba = yuv_pq_lookup(p.table, b) | 0x3C000000u;
}

struct YuvPqPixel {
    const YuvPqSrc &k;
    uint32_t *px;
    HAP_HD void operator()(int t, int32_t y, int32_t cb8, int32_t cr8) const { yuv_pq_pixel(y, cb8, cr8, k, px[2 * t], px[2 * t + 1]); }
};

// Block (bx, by) of a P010 picture -> px[32], the RGBA16F texels bc6h_encode_block takes
HAP_HD void load_block_yuv_pq(const uint8_t *luma, const uint8_t *chroma, uint32_t pitch, uint32_t bx, uint32_t by, uint32_t blocks_x,
                              uint32_t blocks_y, const YuvPqSrc &k, uint32_t px[32])
{
    gather_block_yuv<kSrcP010>(luma, chroma, pitch, bx, by, blocks_x, blocks_y, YuvPqPixel{k, px});
}

// Non-negative finite v (below 65520) -> binary16 bits, rounded once, to nearest, ties to even
inline uint16_t yuv_half_rne(double v)
{
    if (!(v > 0)) return 0;
    int e;
    frexp(v, &e);                                        // v = f * 2^e, 0.5 <= f < 1
    const int ex = e - 1 < -14 ? -14 : e - 1;            // the binade (subnormals share -14's quantum, 2^-24)
    const double q = ldexp(v, 10 - ex);                  // v in quanta of its binade: exact, below 2048
    double n = floor(q);
    const double d = q - n;                              // exact
    if (d > 0.5 || (d == 0.5 && fmod(n, 2.0) != 0)) n += 1;
    return (uint16_t)(((ex + 15) << 10) + (int)n - 1024);   // n = 2048 carries into the next binade
}

// T of include/hap_b200.h for unitNits (1 .. 10000), in double precision: T[c] = half((10000 * EOTF(c / 4095)) / unitNits)
inline void yuv_pq_table(uint32_t unit_nits, uint16_t table[4096])
{
    const double m1 = 2610.0 / 16384, m2 = 2523.0 / 32, c1 = 3424.0 / 4096, c2 = 2413.0 / 128, c3 = 2392.0 / 128;
    for (uint32_t c = 0; c < 4096; c++) {
        const double e = pow((double)c / 4095, 1 / m2);
        const double num = e - c1 > 0 ? e - c1 : 0;
        table[c] = yuv_half_rne(10000 * pow(num / (c2 - c3 * e), 1 / m1) / unit_nits);
    }
}

}  // namespace hapb200
