// hap_b200/csrc/yuv_sink.cuh -- K8 with an NV12 / P010 sink: DXT1 / DXT5 / scaled-YCoCg-DXT5 / RGTC1 / BC7 blocks -> 4:2:0
// Y'CbCr planes, with no RGBA picture in between.
//
// The conversion is defined exactly, in integers, in include/hap_b200.h (HapB200DecodeYUV): per pixel a luma dot product with
// the coefficients of HAPB200_YUV_OUT_COEFFICIENTS; per chroma sample a [1 2 1] x [1 1] filter over the RGB around it (default
// siting: co-sited with even luma columns, midway between the two rows), then one dot product per chroma channel.  The
// texels come from K8's own block decoders (decode_block, bc_decode.cuh), so the planes are the conversion of exactly the
// RGBA8 picture bc_decode_kernel writes.
//
// Shape: K8's, one thread per 4x4 block, kBcThreads per CTA, frames on blockIdx.y in slices of kBcFramesPerLaunch.  A thread
// writes its block's 4 luma row pieces (NV12: one 32-bit store per row; P010: 64-bit) and its 2 x 2 chroma pairs (one 32- or
// 64-bit store per chroma row).
// Halo: chroma column 2bx filters luma columns 4bx-1 .. 4bx+1, and column 4bx-1 is column 3 of the block to the left.  Each
// warp owns one block row and kYuvOutSpan = 31 consecutive block columns of it: lanes 1-31 decode and write those blocks, lane
// 0 decodes the block to the left of them, and every lane hands its column 3 (4 RGBA words) one lane up by __shfl_up_sync.
// One extra decode per 31 blocks and no divergence, which matters for BC7, where a per-lane extra decode would serialise the
// warp.  At the picture's left edge the clamp makes the neighbour column the block's own column 0.
#pragma once
#include "bc_decode.cuh"
#include "yuv_source.cuh"

namespace hapb200 {

constexpr uint32_t kYuvOutSpan = 31;   // block columns a warp writes

// a row of HAPB200_YUV_OUT_COEFFICIENTS and the largest sample of the layout
struct YuvOutCoeffs {
    int32_t y_r, y_g, y_b, cb_r, cb_g, cb_b, cr_r, cr_g, cr_b, y_off, c_off, top;
};

// the coefficients of layout (HapB200YUVLayout) and colorSpace (BT.601 / BT.709, limited / full); both in range
inline YuvOutCoeffs yuv_out_coeffs(unsigned layout, unsigned color_space)
{
    static const int32_t kCoeffs[8][11] = HAPB200_YUV_OUT_COEFFICIENTS;
    const int32_t *k = kCoeffs[layout * 4 + color_space];
    return YuvOutCoeffs{k[0], k[1], k[2], k[3], k[4], k[5], k[6], k[7], k[8], k[9], k[10], layout == HapB200YUV_P010 ? 1023 : 255};
}

HAP_HD uint32_t yuv_out_clamp(int32_t v, int32_t top) { return (uint32_t)(v < 0 ? 0 : v > top ? top : v); }

// one pixel, packed RGBA8 (R in the low byte) -> its luma sample
HAP_HD uint32_t yuv_out_luma(uint32_t rgba, const YuvOutCoeffs &k)
{
    const int32_t r = (int32_t)(rgba & 0xFF), g = (int32_t)((rgba >> 8) & 0xFF), b = (int32_t)((rgba >> 16) & 0xFF);
    return yuv_out_clamp(((k.y_r * r + k.y_g * g + k.y_b * b + 32768) >> 16) + k.y_off, k.top);
}

// the filtered sums of one chroma sample (total weight 8) -> its Cb and Cr samples
HAP_HD uint32_t yuv_out_cb(int32_t rs, int32_t gs, int32_t bs, const YuvOutCoeffs &k)
{
    return yuv_out_clamp(((k.cb_r * rs + k.cb_g * gs + k.cb_b * bs + (1 << 18)) >> 19) + k.c_off, k.top);
}
HAP_HD uint32_t yuv_out_cr(int32_t rs, int32_t gs, int32_t bs, const YuvOutCoeffs &k)
{
    return yuv_out_clamp(((k.cr_r * rs + k.cr_g * gs + k.cr_b * bs + (1 << 18)) >> 19) + k.c_off, k.top);
}

struct YuvOutGeom {
    uint32_t blocks_x, blocks_y;
    uint32_t spans;          // warps per block row: ceil(blocks_x / kYuvOutSpan)
    uint32_t pitch;          // row pitch of both planes, bytes
    uint64_t in_stride;      // block bytes per frame
    uint64_t frame_bytes;    // frame stride of both planes
    YuvOutCoeffs k;
};

inline YuvOutGeom yuv_out_geom(uint32_t width, uint32_t height, uint32_t pitch, uint64_t in_stride, uint64_t frame_bytes, unsigned layout,
                               unsigned color_space)
{
    YuvOutGeom g;
    g.blocks_x = width / 4;
    g.blocks_y = height / 4;
    g.spans = (g.blocks_x + kYuvOutSpan - 1) / kYuvOutSpan;
    g.pitch = pitch;
    g.in_stride = in_stride;
    g.frame_bytes = frame_bytes;
    g.k = yuv_out_coeffs(layout, color_space);
    return g;
}

// CTAs of one frame: kBcThreads / 32 warps each, one warp per span of a block row
inline uint64_t yuv_out_ctas(const YuvOutGeom &g) { return ((uint64_t)g.blocks_y * g.spans + kBcThreads / 32 - 1) / (kBcThreads / 32); }

// one luma row piece or chroma row pair of 4 samples -> NV12 bytes (one 32-bit word) or P010 words (two 32-bit words)
template <int LAYOUT>
HAP_HD void yuv_out_store4(uint8_t *p, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3)
{
    if (LAYOUT == HapB200YUV_P010) *reinterpret_cast<uint2 *>(p) = make_uint2(s0 << 6 | s1 << 22, s2 << 6 | s3 << 22);
    else *reinterpret_cast<uint32_t *>(p) = s0 | s1 << 8 | s2 << 16 | s3 << 24;
}

// grid = (yuv_out_ctas, frames).  KIND: kBcDxt1, kBcDxt5, kBcYCoCg (Hap Q and Hap Q Alpha: alpha is dropped), kBcRgtc1
// (Hap Alpha-Only: (v, v, v, 255)), kBcBc7.  LAYOUT: HapB200YUV_NV12 / _P010.  frame_results (optional): a frame whose entry
// is not HapResult_No_Error is converted from zeros, as K8 writes it.
template <int KIND, int LAYOUT>
__global__ void __launch_bounds__(kBcThreads) bc_decode_yuv_kernel(const uint8_t *__restrict__ blocks, YuvOutGeom G,
                                                                    uint8_t *__restrict__ luma, uint8_t *__restrict__ chroma,
                                                                    const uint32_t *__restrict__ frame_results)
{
    constexpr uint32_t kSample = LAYOUT == HapB200YUV_P010 ? 2 : 1;
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t warp = (uint64_t)blockIdx.x * (kBcThreads / 32) + (threadIdx.x >> 5);
    const uint64_t by64 = warp / G.spans;
    if (by64 >= G.blocks_y) return;   // (whole warps)
    const uint32_t by = (uint32_t)by64, span = (uint32_t)(warp - by64 * G.spans);
    // lanes 1-31: blocks span*31 .. span*31+30 of the row; lane 0: the block left of them (none at the left edge).  Lanes
    // past the row's end decode its last block again and write nothing.
    const uint32_t bx = span * kYuvOutSpan + lane - 1;   // (lane 0 of span 0: wraps, writes nothing)
    const uint32_t bxr = (lane == 0 && span == 0) ? 0 : bx < G.blocks_x ? bx : G.blocks_x - 1;
    uint32_t px[16];
    if (frame_results && frame_results[blockIdx.y] != 0u /* HapResult_No_Error */) {
#pragma unroll
        for (int t = 0; t < 16; t++) px[t] = 0;
    } else {
        const uint8_t *in = blocks + (uint64_t)blockIdx.y * G.in_stride;
        const uint32_t bi = by * G.blocks_x + bxr;
        if (KIND == kBcDxt1 || KIND == kBcRgtc1) {
            const uint2 v = reinterpret_cast<const uint2 *>(in)[bi];
            decode_block(KIND, v.x, v.y, 0, 0, px);
        } else {
            const uint4 v = reinterpret_cast<const uint4 *>(in)[bi];
            decode_block(KIND, v.x, v.y, v.z, v.w, px);
        }
    }
    // column 4bx-1 of rows 0..3: column 3 of the lane below; at the left edge column 0 (the clamp)
    uint32_t left[4];
#pragma unroll
    for (int r = 0; r < 4; r++) {
        left[r] = __shfl_up_sync(0xFFFFFFFFu, px[4 * r + 3], 1);
        if (bx == 0) left[r] = px[4 * r];
    }
    if (lane == 0 || bx >= G.blocks_x) return;
    const YuvOutCoeffs &k = G.k;
    uint8_t *lrow = luma + (uint64_t)blockIdx.y * G.frame_bytes + (uint64_t)(4 * by) * G.pitch + (uint64_t)(4 * kSample) * bx;
#pragma unroll
    for (int r = 0; r < 4; r++)
        yuv_out_store4<LAYOUT>(lrow + (uint64_t)r * G.pitch, yuv_out_luma(px[4 * r], k), yuv_out_luma(px[4 * r + 1], k),
                               yuv_out_luma(px[4 * r + 2], k), yuv_out_luma(px[4 * r + 3], k));
    uint8_t *crow = chroma + (uint64_t)blockIdx.y * G.frame_bytes + (uint64_t)(2 * by) * G.pitch + (uint64_t)(4 * kSample) * bx;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        // s[c][ch]: chroma column 2bx+c, channel ch (R, G, B): luma columns 4bx+2c-1 .. 4bx+2c+1, weights 1 2 1, rows 2j, 2j+1
        int32_t s[2][3] = {{0, 0, 0}, {0, 0, 0}};
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
            const int r = 2 * j + rr;
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                const int32_t l = (int32_t)byte_of(left[r], ch), p0 = (int32_t)byte_of(px[4 * r], ch), p1 = (int32_t)byte_of(px[4 * r + 1], ch);
                const int32_t p2 = (int32_t)byte_of(px[4 * r + 2], ch), p3 = (int32_t)byte_of(px[4 * r + 3], ch);
                s[0][ch] += l + 2 * p0 + p1;
                s[1][ch] += p1 + 2 * p2 + p3;
            }
        }
        yuv_out_store4<LAYOUT>(crow + (uint64_t)j * G.pitch, yuv_out_cb(s[0][0], s[0][1], s[0][2], k), yuv_out_cr(s[0][0], s[0][1], s[0][2], k),
                               yuv_out_cb(s[1][0], s[1][1], s[1][2], k), yuv_out_cr(s[1][0], s[1][1], s[1][2], k));
    }
}

}  // namespace hapb200
