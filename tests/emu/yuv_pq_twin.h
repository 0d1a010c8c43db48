// tests/emu/yuv_pq_twin.h -- TEST INFRASTRUCTURE ONLY.
// The HDR10 P010 -> RGBA16F conversion of include/hap_b200.h (HapB200EncodeYUVPQ) written pixel by pixel: the chroma
// upsampling of yuv_twin.h (indices clamped one at a time), then the 12-bit matrix and the library's own table
// (yuv_pq_table, hap_b200/csrc/yuv_source.cuh) through the kernel's per-pixel function (yuv_pq_pixel).  It shares no loads
// or index arithmetic with gather_block_yuv, the kernel's block loader: tests/test_yuv_pq_cpu.py holds it to the numpy
// restatement (tests/yuv_pq_util.py), and tests/emu/test_yuv_pq_emu.cc holds the kernel to it.
#pragma once
#include "yuv_twin.h"

namespace yuv_pq_twin {

using namespace hapb200;

// the whole picture -> RGBA16F rows 4*width halves apart; table: yuv_pq_table of the unitNits wanted
inline void picture(const uint8_t *luma, const uint8_t *chroma, uint32_t width, uint32_t height, uint64_t pitch, int color_space,
                    const uint16_t *table, uint16_t *rgba)
{
    const YuvPqSrc k = yuv_pq_src(color_space, chroma, table);
    const int32_t cw = (int32_t)width / 2, ch = (int32_t)height / 2;
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) {
            const int32_t i = (int32_t)x / 2, j = (int32_t)y / 2;
            const int32_t rows[2] = {j, (y % 2) ? j + 1 : j - 1}, wv[2] = {3, 1};
            const int32_t cols[2] = {i, i + 1}, wh[2] = {(x % 2) ? 1 : 2, (x % 2) ? 1 : 0};
            int32_t cb8 = 0, cr8 = 0;
            for (int a = 0; a < 2; a++)
                for (int b = 0; b < 2; b++) {
                    const int32_t r = rows[a] < 0 ? 0 : rows[a] >= ch ? ch - 1 : rows[a];
                    const int32_t c = cols[b] >= cw ? cw - 1 : cols[b];
                    const uint8_t *row = chroma + (uint64_t)r * pitch;
                    cb8 += wv[a] * wh[b] * yuv_twin::sample(row, 2 * c, HapB200YUV_P010);
                    cr8 += wv[a] * wh[b] * yuv_twin::sample(row, 2 * c + 1, HapB200YUV_P010);
                }
            uint32_t px[2];
            yuv_pq_pixel(yuv_twin::sample(luma + (uint64_t)y * pitch, x, HapB200YUV_P010), cb8, cr8, k, px[0], px[1]);
            memcpy(rgba + 4 * ((uint64_t)y * width + x), px, 8);
        }
}

}  // namespace yuv_pq_twin
