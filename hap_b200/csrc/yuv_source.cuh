// hap_b200/csrc/yuv_source.cuh -- the NV12 / P010 source of the K1-K4 block encoders: 4:2:0 Y'CbCr -> RGBA8 in registers.
//
// The conversion is defined exactly, in integers, in include/hap_b200.h (HapB200EncodeYUV): bilinear chroma upsampling at
// the MPEG-2 / H.264 / HEVC default siting, then one fixed-point dot product per channel with the coefficients of
// HAPB200_YUV_COEFFICIENTS.  The thread that owns a 4x4 block (bc_encode.cuh) reads its 16 luma samples and the 4 x 3 chroma
// pairs around them, converts, and hands px[16] to the unchanged block fit, so a YUV picture encodes to exactly the bytes of
// the RGBA8 picture this conversion makes of it.  Every load stays inside the two planes: the chroma row above, the row
// below and the column to the right are clamped at the picture's edges, as the definition clamps them.
#pragma once
#include "bc_block.cuh"
#include "../../include/hap_b200.h"

namespace hapb200 {

// The picture a block encoder reads (the SRC parameter of bc_encode_kernel)
enum BcSource : int { kSrcRgba8 = 0, kSrcNv12 = 1, kSrcP010 = 2 };

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

// Block (bx, by) of a blocks_x x blocks_y picture -> px[16].  luma / chroma: this frame's planes, rows `pitch` bytes apart.
// Luma: 4 rows of 4 samples.  Chroma: rows 2by-1 .. 2by+2 and pair columns 2bx .. 2bx+2, clamped (so at the edges the row
// above, the row below and the right column are the block's own outermost ones, and are not loaded).
template <int SRC>
HAP_HD void load_block_yuv(const uint8_t *luma, const uint8_t *chroma, uint32_t pitch, uint32_t bx, uint32_t by, uint32_t blocks_x,
                           uint32_t blocks_y, const YuvSrc &k, uint32_t px[16])
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
        px[4 * yl + 0] = yuv_pixel(y[0], 2 * vb[0], 2 * vr[0], k);
        px[4 * yl + 1] = yuv_pixel(y[1], vb[0] + vb[1], vr[0] + vr[1], k);
        px[4 * yl + 2] = yuv_pixel(y[2], 2 * vb[1], 2 * vr[1], k);
        px[4 * yl + 3] = yuv_pixel(y[3], vb[1] + vb[2], vr[1] + vr[2], k);
    }
}

}  // namespace hapb200
