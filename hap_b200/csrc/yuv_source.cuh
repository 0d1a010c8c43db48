// hap_b200/csrc/yuv_source.cuh -- the NV12 / P010 source of the K1-K4 block encoders: 4:2:0 Y'CbCr -> RGBA8 in registers.
//
// The conversion is defined exactly, in integers, in include/hap_b200.h (HapB200EncodeYUV): bilinear chroma upsampling at
// the MPEG-2 / H.264 / HEVC default siting, then one fixed-point dot product per channel with the coefficients of
// HAPB200_YUV_COEFFICIENTS.  The thread that owns a 4x4 block (bc_encode.cuh) reads its 16 luma samples and the 4 x 3 chroma
// pairs around them, converts, and hands px[16] to the unchanged block fit, so a YUV picture encodes to exactly the bytes of
// the RGBA8 picture this conversion makes of it.  Every load stays inside the two planes: the chroma row above, the row
// below and the column to the right are clamped at the picture's edges, as the definition clamps them.
//
// The same gather feeds the HDR10 source of the BC6H encoder (bc6h_encode.cuh, HapB200EncodeYUVPQ): P010 BT.2020 -> 12-bit
// R'G'B' (HAPB200_YUV_PQ_COEFFICIENTS) -> linear binary16 through the PQ table T, built on the host (yuv_pq_table).
#pragma once
#include "bc_block.cuh"
#include "../../include/hap_b200.h"

namespace hapb200 {

// The picture a block encoder reads (the SRC parameter of bc_encode_kernel: RGBA8, NV12, P010; of bc6h_encode_kernel:
// RGBA16F, HDR10 P010)
enum BcSource : int { kSrcRgba8 = 0, kSrcNv12 = 1, kSrcP010 = 2, kSrcRgbaHalf = 3, kSrcP010Pq = 4 };

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
        const uint32_t row = r == 0 ? (by > 0 ? 2 * by - 1 : 0) : r == 3 ? (by + 1 < blocks_y ? 2 * by + 2 : 2 * by + 1) : 2 * by + r - 1;
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
#pragma unroll
    for (int yl = 0; yl < 4; yl++) {
        // luma row 4by+yl: chroma row j = 2by + yl/2 is local row 1 + yl/2; its neighbour is the row above (y even) or below
        const int rj = 1 + yl / 2, rn = (yl & 1) ? rj + 1 : rj - 1;
        int32_t vb[3], vr[3];   // vertically filtered chroma of the three columns, in quarters
#pragma unroll
        for (int c = 0; c < 3; c++) { vb[c] = 3 * cb[rj][c] + cb[rn][c]; vr[c] = 3 * cr[rj][c] + cr[rn][c]; }
        const uint8_t *l = luma + (uint64_t)(4 * by + yl) * pitch;
        int32_t y[4];
        if (kP010) {
            const uint2 v = *reinterpret_cast<const uint2 *>(l + 8ull * bx);
            y[0] = (v.x & 0xFFFF) >> 6; y[1] = v.x >> 22; y[2] = (v.y & 0xFFFF) >> 6; y[3] = v.y >> 22;
        } else {
            const uint32_t v = *reinterpret_cast<const uint32_t *>(l + 4ull * bx);
            y[0] = v & 0xFF; y[1] = (v >> 8) & 0xFF; y[2] = (v >> 16) & 0xFF; y[3] = v >> 24;
        }
        // columns 4bx+xl: chroma column i = 2bx + xl/2 is local column xl/2; odd columns average it with the next one
        pixel(4 * yl + 0, y[0], 2 * vb[0], 2 * vr[0]);
        pixel(4 * yl + 1, y[1], vb[0] + vb[1], vr[0] + vr[1]);
        pixel(4 * yl + 2, y[2], 2 * vb[1], 2 * vr[1]);
        pixel(4 * yl + 3, y[3], vb[1] + vb[2], vr[1] + vr[2]);
    }
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
