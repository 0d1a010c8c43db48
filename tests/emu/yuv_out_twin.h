// tests/emu/yuv_out_twin.h -- TEST INFRASTRUCTURE ONLY.
// The RGBA8 -> NV12 / P010 conversion of include/hap_b200.h (HapB200DecodeYUV) written sample by sample: every chroma sample
// sums its six neighbours with the weights as the definition states them, column -1 clamped one at a time, then the kernel's own
// per-sample functions (yuv_out_luma, yuv_out_cb, yuv_out_cr, hap_b200/csrc/yuv_sink.cuh).  It shares no loads, halo exchange
// or index arithmetic with bc_decode_yuv_kernel: tests/test_yuv_out_cpu.py holds it to the numpy restatement
// (tests/yuv_out_util.py), and tests/emu/test_yuv_out_emu.cc holds the kernel to it.
#pragma once
#define HAPB200_EMU
#include "yuv_sink.cuh"

#include <cstring>

namespace yuv_out_twin {

using namespace hapb200;

// stores sample s (0..2^n-1) at index i of a row: NV12 byte, P010 16-bit word s << 6
inline void put(uint8_t *row, uint32_t i, uint32_t s, int layout)
{
    if (layout == HapB200YUV_NV12) { row[i] = (uint8_t)s; return; }
    const uint16_t w = (uint16_t)(s << 6);
    memcpy(row + 2 * i, &w, 2);
}

// channel ch (0 R, 1 G, 2 B) of pixel (x, y) of a tight width x height RGBA8 picture
inline int32_t chan(const uint8_t *rgba, uint32_t width, uint32_t x, uint32_t y, int ch) { return rgba[4 * ((uint64_t)y * width + x) + ch]; }

// the whole picture -> luma and chroma planes whose rows are `pitch` bytes apart; only each row's samples are written
inline void picture(const uint8_t *rgba, uint32_t width, uint32_t height, int layout, int color_space, uint8_t *luma, uint8_t *chroma,
                    uint64_t pitch)
{
    const YuvOutCoeffs k = yuv_out_coeffs(layout, color_space);
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) {
            uint32_t p;
            memcpy(&p, rgba + 4 * ((uint64_t)y * width + x), 4);
            put(luma + y * pitch, x, yuv_out_luma(p, k), layout);
        }
    const int32_t wh[3] = {1, 2, 1};
    for (uint32_t j = 0; j < height / 2; j++)
        for (uint32_t i = 0; i < width / 2; i++) {
            int32_t s[3] = {0, 0, 0};
            for (int dy = 0; dy < 2; dy++)
                for (int dx = -1; dx <= 1; dx++) {
                    const int32_t col = (int32_t)(2 * i) + dx;
                    const uint32_t x = col < 0 ? 0 : (uint32_t)col;
                    for (int ch = 0; ch < 3; ch++) s[ch] += wh[dx + 1] * chan(rgba, width, x, 2 * j + dy, ch);
                }
            put(chroma + j * pitch, 2 * i, yuv_out_cb(s[0], s[1], s[2], k), layout);
            put(chroma + j * pitch, 2 * i + 1, yuv_out_cr(s[0], s[1], s[2], k), layout);
        }
}

}  // namespace yuv_out_twin
