// tests/emu/planar_twin.h -- TEST INFRASTRUCTURE ONLY.
// The planar Y'CbCr -> RGBA8 conversion of include/hap_b200.h (HapB200EncodePlanar) written pixel by pixel: chroma
// indices clamped one at a time, the upsampling weights of each subsampling as the definition states them, the alpha
// mapping as its integer division, then the kernel's own matrix function (planar_rgb, hap_b200/csrc/yuv_source.cuh).  It
// shares no loads or index arithmetic with load_block_planar, the kernel's block loader: tests/test_planar_cpu.py holds it
// to the numpy restatement (tests/planar_util.py), and tests/emu/test_planar_emu.cc holds the kernel to it.
#pragma once
#define HAPB200_EMU
#include "yuv_source.cuh"

#include <cstring>

namespace planar_twin {

using namespace hapb200;

// sample i of a row: bytes (n = 8), or 16-bit words & (2^n - 1)
inline int32_t sample(const uint8_t *row, uint32_t i, int n)
{
    if (n == 8) return row[i];
    uint16_t w;
    memcpy(&w, row + 2 * i, 2);
    return w & ((1 << n) - 1);
}

// the RGBA8 pixel (x, y) of a width x height picture: luma and alpha rows lpitch bytes apart, Cb and Cr rows cpitch apart
inline uint32_t pixel(const uint8_t *luma, const uint8_t *cb, const uint8_t *cr, const uint8_t *alpha, uint32_t width, uint32_t height,
                      uint64_t lpitch, uint64_t cpitch, int sub, int n, int color_space, uint32_t x, uint32_t y)
{
    const PlanarSrc k = planar_src_args(n, color_space, cb, cr, alpha, (uint32_t)cpitch);
    const int32_t cw = sub == HapB200Chroma_444 ? (int32_t)width : (int32_t)width / 2;
    const int32_t ch = sub == HapB200Chroma_420 ? (int32_t)height / 2 : (int32_t)height;
    int32_t rows[2], wv[2], cols[2], wh[2];
    if (sub == HapB200Chroma_420) {
        const int32_t j = (int32_t)y / 2;
        rows[0] = j; rows[1] = (y % 2) ? j + 1 : j - 1; wv[0] = 3; wv[1] = 1;
    } else {
        rows[0] = rows[1] = (int32_t)y; wv[0] = 4; wv[1] = 0;
    }
    if (sub == HapB200Chroma_444) {
        cols[0] = cols[1] = (int32_t)x; wh[0] = 2; wh[1] = 0;
    } else {
        const int32_t i = (int32_t)x / 2;
        cols[0] = i; cols[1] = i + 1; wh[0] = (x % 2) ? 1 : 2; wh[1] = (x % 2) ? 1 : 0;
    }
    int32_t cb8 = 0, cr8 = 0;
    for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2; b++) {
            const int32_t r = rows[a] < 0 ? 0 : rows[a] >= ch ? ch - 1 : rows[a];
            const int32_t c = cols[b] >= cw ? cw - 1 : cols[b];
            cb8 += wv[a] * wh[b] * sample(cb + (uint64_t)r * cpitch, c, n);
            cr8 += wv[a] * wh[b] * sample(cr + (uint64_t)r * cpitch, c, n);
        }
    uint32_t A = 255;
    if (alpha) {
        const int64_t m = (1 << n) - 1;
        A = (uint32_t)((510 * (int64_t)sample(alpha + (uint64_t)y * lpitch, x, n) + m) / (2 * m));
    }
    return planar_rgb(sample(luma + (uint64_t)y * lpitch, x, n), cb8, cr8, k) | A << 24;
}

// the whole picture -> RGBA8 rows 4*width bytes apart
inline void picture(const uint8_t *luma, const uint8_t *cb, const uint8_t *cr, const uint8_t *alpha, uint32_t width, uint32_t height,
                    uint64_t lpitch, uint64_t cpitch, int sub, int n, int color_space, uint8_t *rgba)
{
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const uint32_t p = pixel(luma, cb, cr, alpha, width, height, lpitch, cpitch, sub, n, color_space, x, y);
            memcpy(rgba + 4 * ((uint64_t)y * width + x), &p, 4);
        }
}

}  // namespace planar_twin
