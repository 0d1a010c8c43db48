// tests/emu/yuv_twin.h -- TEST INFRASTRUCTURE ONLY.
// The NV12 / P010 -> RGBA8 conversion of include/hap_b200.h written pixel by pixel: chroma indices clamped one at a time,
// the upsampling weights as the definition states them, then the kernel's own per-pixel function (yuv_pixel,
// hap_b200/csrc/yuv_source.cuh).  It shares no loads or index arithmetic with load_block_yuv, the kernel's block loader:
// tests/test_yuv_cpu.py holds it to the numpy restatement (tests/yuv_util.py), and tests/emu/test_yuv_emu.cc holds the
// kernel to it.
#pragma once
#define HAPB200_EMU
#include "yuv_source.cuh"

#include <cstring>

namespace yuv_twin {

using namespace hapb200;

// sample i of a row: NV12 bytes, P010 16-bit words >> 6
inline int32_t sample(const uint8_t *row, uint32_t i, int layout)
{
    if (layout == HapB200YUV_NV12) return row[i];
    uint16_t w;
    memcpy(&w, row + 2 * i, 2);
    return w >> 6;
}

// the RGBA8 pixel (x, y) of a width x height picture whose planes have rows `pitch` bytes apart
inline uint32_t pixel(const uint8_t *luma, const uint8_t *chroma, uint32_t width, uint32_t height, uint64_t pitch, int layout,
                      int color_space, uint32_t x, uint32_t y)
{
    const YuvSrc k = yuv_src(layout, color_space, chroma);
    const int32_t cw = (int32_t)width / 2, ch = (int32_t)height / 2;
    const int32_t i = (int32_t)x / 2, j = (int32_t)y / 2;
    const int32_t rows[2] = {j, (y % 2) ? j + 1 : j - 1}, wv[2] = {3, 1};
    const int32_t cols[2] = {i, i + 1}, wh[2] = {(x % 2) ? 1 : 2, (x % 2) ? 1 : 0};
    int32_t cb8 = 0, cr8 = 0;
    for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2; b++) {
            const int32_t r = rows[a] < 0 ? 0 : rows[a] >= ch ? ch - 1 : rows[a];
            const int32_t c = cols[b] >= cw ? cw - 1 : cols[b];
            const uint8_t *row = chroma + (uint64_t)r * pitch;
            cb8 += wv[a] * wh[b] * sample(row, 2 * c, layout);
            cr8 += wv[a] * wh[b] * sample(row, 2 * c + 1, layout);
        }
    return yuv_pixel(sample(luma + (uint64_t)y * pitch, x, layout), cb8, cr8, k);
}

// the whole picture -> RGBA8 rows 4*width bytes apart
inline void picture(const uint8_t *luma, const uint8_t *chroma, uint32_t width, uint32_t height, uint64_t pitch, int layout, int color_space,
                    uint8_t *rgba)
{
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const uint32_t p = pixel(luma, chroma, width, height, pitch, layout, color_space, x, y);
            memcpy(rgba + 4 * ((uint64_t)y * width + x), &p, 4);
        }
}

}  // namespace yuv_twin
