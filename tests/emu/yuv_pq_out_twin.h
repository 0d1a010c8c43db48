// tests/emu/yuv_pq_out_twin.h -- TEST INFRASTRUCTURE ONLY.
// The RGBA16F -> HDR10 P010 conversion of include/hap_b200.h (HapB200DecodeYUVPQ) written sample by sample: each of R, G and
// B through the library's own table P (yuv_pq_out_table, hap_b200/csrc/yuv_sink.cuh) with the sign and clamp rules restated
// here, then every chroma sample sums its six neighbours with the weights as the definition states them, column -1 clamped
// one at a time, and the kernel's own per-sample functions (yuv_out_luma_rgb, yuv_out_cb, yuv_out_cr).  It shares no loads,
// halo exchange or index arithmetic with bc6h_decode_yuv_kernel: tests/test_yuv_pq_out_cpu.py holds it to the numpy
// restatement (tests/yuv_pq_out_util.py), and tests/emu/test_yuv_pq_out_emu.cc holds the kernel to it.
#pragma once
#define HAPB200_EMU
#include "yuv_sink.cuh"

#include <cstring>

namespace yuv_pq_out_twin {

using namespace hapb200;

inline void put(uint8_t *row, uint32_t i, uint32_t s)
{
    const uint16_t w = (uint16_t)(s << 6);
    memcpy(row + 2 * i, &w, 2);
}

// channel ch (0 R, 1 G, 2 B) of pixel (x, y) of a tight width x height RGBA16F picture -> its 12-bit code
inline int32_t code(const uint16_t *rgba, const uint16_t *table, uint32_t width, uint32_t x, uint32_t y, int ch)
{
    const uint16_t h = rgba[4 * ((uint64_t)y * width + x) + ch];
    if (h >= 0x8000) return 0;                       // sign bit set: SF16 negatives and -0
    return table[h > 0x7BFF ? 0x7BFF : h];
}

// the whole picture -> luma and chroma planes whose rows are `pitch` bytes apart; only each row's samples are written.
// table: yuv_pq_out_table of the unitNits wanted
inline void picture(const uint16_t *rgba, uint32_t width, uint32_t height, int color_space, const uint16_t *table, uint8_t *luma,
                    uint8_t *chroma, uint64_t pitch)
{
    const YuvOutCoeffs k = yuv_pq_out_coeffs(color_space);
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++)
            put(luma + y * pitch, x,
                yuv_out_luma_rgb(code(rgba, table, width, x, y, 0), code(rgba, table, width, x, y, 1), code(rgba, table, width, x, y, 2), k));
    const int32_t wh[3] = {1, 2, 1};
    for (uint32_t j = 0; j < height / 2; j++)
        for (uint32_t i = 0; i < width / 2; i++) {
            int32_t s[3] = {0, 0, 0};
            for (int dy = 0; dy < 2; dy++)
                for (int dx = -1; dx <= 1; dx++) {
                    const int32_t col = (int32_t)(2 * i) + dx;
                    const uint32_t x = col < 0 ? 0 : (uint32_t)col;
                    for (int ch = 0; ch < 3; ch++) s[ch] += wh[dx + 1] * code(rgba, table, width, x, 2 * j + dy, ch);
                }
            put(chroma + j * pitch, 2 * i, yuv_out_cb(s[0], s[1], s[2], k));
            put(chroma + j * pitch, 2 * i + 1, yuv_out_cr(s[0], s[1], s[2], k));
        }
}

}  // namespace yuv_pq_out_twin
