// tests/emu/planar_out_twin.h -- TEST INFRASTRUCTURE ONLY.
// The RGBA8 -> planar Y'CbCr (+ alpha) conversion of include/hap_b200.h (HapB200DecodePlanar) written sample by sample: every
// chroma sample sums its neighbours with the weights of its subsampling as the definition states them, column -1 clamped one
// at a time, alpha as the definition's integer division, then the kernel's own per-sample functions (yuv_out_luma, yuv_out_cb,
// yuv_out_cr, hap_b200/csrc/yuv_sink.cuh) with the row of planar_out_coeffs.  It shares no loads, halo exchange or index
// arithmetic with bc_decode_planar_kernel: tests/test_planar_out_cpu.py holds it to the numpy restatement
// (tests/planar_out_util.py), and tests/emu/test_planar_out_emu.cc holds the kernel to it.
#pragma once
#define HAPB200_EMU
#include "planar_sink.cuh"

#include <cstring>

namespace planar_out_twin {

using namespace hapb200;

// stores sample s at index i of a row: a byte (n = 8) or a little-endian 16-bit word
inline void put(uint8_t *row, uint32_t i, uint32_t s, int n)
{
    if (n == 8) { row[i] = (uint8_t)s; return; }
    const uint16_t w = (uint16_t)s;
    memcpy(row + 2 * i, &w, 2);
}

// byte ch (0 R, 1 G, 2 B, 3 A) of pixel (x, y) of a tight width x height RGBA8 picture
inline int32_t chan(const uint8_t *rgba, uint32_t width, uint32_t x, uint32_t y, int ch) { return rgba[4 * ((uint64_t)y * width + x) + ch]; }

// the whole picture -> its planes: luma and alpha rows lpitch bytes apart, Cb and Cr rows cpitch apart; luma, cb and cr
// nullptr: not written (Hap Alpha-Only); alpha nullptr: not written.  Only each row's samples are written.
inline void picture(const uint8_t *rgba, uint32_t width, uint32_t height, uint8_t *luma, uint8_t *cb, uint8_t *cr, uint8_t *alpha,
                    uint64_t lpitch, uint64_t cpitch, int sub, int n, int color_space)
{
    const YuvOutCoeffs k = planar_out_coeffs(n, color_space);
    const int64_t top = (1 << n) - 1;
    for (uint32_t y = 0; y < height; y++)
        for (uint32_t x = 0; x < width; x++) {
            uint32_t p;
            memcpy(&p, rgba + 4 * ((uint64_t)y * width + x), 4);
            if (luma) put(luma + y * lpitch, x, yuv_out_luma(p, k), n);
            if (alpha) put(alpha + y * lpitch, x, (uint32_t)((2 * top * (p >> 24) + 255) / 510), n);
        }
    if (!cb) return;
    const uint32_t cw = sub == HapB200Chroma_444 ? width : width / 2, ch = sub == HapB200Chroma_420 ? height / 2 : height;
    for (uint32_t j = 0; j < ch; j++)
        for (uint32_t i = 0; i < cw; i++) {
            int32_t s[3] = {0, 0, 0};
            if (sub == HapB200Chroma_444) {
                for (int c = 0; c < 3; c++) s[c] = 8 * chan(rgba, width, i, j, c);
            } else {
                // weights 1 2 1 over columns 2i-1 .. 2i+1; rows 2j and 2j+1 (4:2:0) or row j twice (4:2:2)
                const int32_t wh[3] = {1, 2, 1};
                for (int dy = 0; dy < 2; dy++)
                    for (int dx = -1; dx <= 1; dx++) {
                        const int32_t col = (int32_t)(2 * i) + dx;
                        const uint32_t x = col < 0 ? 0 : (uint32_t)col, y = sub == HapB200Chroma_420 ? 2 * j + dy : j;
                        for (int c = 0; c < 3; c++) s[c] += wh[dx + 1] * chan(rgba, width, x, y, c);
                    }
            }
            put(cb + j * cpitch, i, yuv_out_cb(s[0], s[1], s[2], k), n);
            put(cr + j * cpitch, i, yuv_out_cr(s[0], s[1], s[2], k), n);
        }
}

}  // namespace planar_out_twin
