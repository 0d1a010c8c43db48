// hap_b200/csrc/planar_sink.cuh -- K8 with a planar sink: DXT1 / DXT5 / scaled-YCoCg-DXT5 (+ RGTC1 alpha) / BC7 blocks ->
// planar Y'CbCr 4:2:0, 4:2:2 or 4:4:4 with an optional alpha plane, and RGTC1 blocks (Hap Alpha-Only) -> the alpha plane
// alone, with no RGBA picture in between.
//
// The conversion is defined exactly, in integers, in include/hap_b200.h (HapB200DecodePlanar).  It is the NV12 / P010 sink's
// (yuv_sink.cuh) with a chroma filter per subsampling, a row per depth (8: NV12's, 10: P010's, 12: HAPB200_YUV_12BIT_OUT_
// COEFFICIENTS) and an alpha mapping.  The texels come from K8's own block decoders (decode_block, bc_decode.cuh), and Hap Q
// Alpha's alpha texture is merged as bc_decode_kernel merges it, so the planes are the conversion of exactly the RGBA8 picture
// bc_decode_kernel writes.
//
// Shape.  4:2:0 and 4:2:2 filter luma columns 4bx-1 .. 4bx+3 for the block's chroma, so they take bc_decode_yuv_kernel's
// layout and halo unchanged: a warp per span of kYuvOutSpan block columns, lane 0 decoding the block to their left, column 3
// handed one lane up by __shfl_up_sync (yuv_out_lane).  4:4:4 has no filter, hence no halo: it takes K8's one-block-per-thread
// layout, which spends no extra decode on a halo lane (1 in 32 lanes of the span layout, most costly for BC7) and keeps each
// warp's row stores contiguous over 32 blocks.
// Stores per block: 4 luma row pieces of 4 samples; Cb and Cr each 2 rows of 2 samples (4:2:0), 4 rows of 2 (4:2:2) or 4 rows
// of 4 (4:4:4); 4 alpha row pieces when there is an alpha plane.  Samples are bytes or 16-bit words (WIDE), so every store is
// one 16-, 32- or 64-bit word at a multiple of its size under the batch rules (16-byte aligned planes and pitches) and in the
// single-frame call's scratch.  Depth (10 or 12 for words) and the alpha plane's presence are runtime values.
#pragma once
#include "yuv_sink.cuh"

namespace hapb200 {

// the row of the conversion for bit_depth 8 / 10 / 12 and colorSpace BT.601 / BT.709 limited / full (both in range); top 2^n-1
inline YuvOutCoeffs planar_out_coeffs(unsigned bit_depth, unsigned color_space)
{
    if (bit_depth != 12) return yuv_out_coeffs(bit_depth == 8 ? HapB200YUV_NV12 : HapB200YUV_P010, color_space);
    static const int32_t kCoeffs[4][11] = HAPB200_YUV_12BIT_OUT_COEFFICIENTS;
    const int32_t *k = kCoeffs[color_space];
    return YuvOutCoeffs{k[0], k[1], k[2], k[3], k[4], k[5], k[6], k[7], k[8], k[9], k[10], 4095};
}

// What the planar sink adds to YuvOutGeom (G.pitch: the luma and alpha pitch; G.k: the row, k.top = 2^n - 1): the Cb, Cr and
// alpha planes (alpha nullptr: none is written), all G.frame_bytes apart per frame like luma; the chroma planes' pitch; and,
// for Hap Q Alpha with an alpha plane, merge_alpha = 1 and the RGTC1 texture second_offset bytes behind each frame's blocks.
// Uniform per launch.
struct PlanarOut {
    YuvOutGeom g;
    uint8_t *cb, *cr, *alpha;
    uint32_t chroma_pitch, merge_alpha;
    uint64_t second_offset;
};

// A of RGBA8 -> the alpha sample of depth top = 2^n - 1: (2 top A + 255) / 510, integer division (A itself at n = 8)
HAP_HD uint32_t planar_out_alpha(uint32_t a, uint32_t top) { return (2 * top * a + 255) / 510; }

// 4 samples -> bytes (one 32-bit word) or 16-bit words (one 64-bit word); 2 samples -> one 16- or 32-bit word
template <bool WIDE>
HAP_HD void planar_out_store4(uint8_t *p, uint32_t s0, uint32_t s1, uint32_t s2, uint32_t s3)
{
    if (WIDE) *reinterpret_cast<uint2 *>(p) = make_uint2(s0 | s1 << 16, s2 | s3 << 16);
    else *reinterpret_cast<uint32_t *>(p) = s0 | s1 << 8 | s2 << 16 | s3 << 24;
}
template <bool WIDE>
HAP_HD void planar_out_store2(uint8_t *p, uint32_t s0, uint32_t s1)
{
    if (WIDE) *reinterpret_cast<uint32_t *>(p) = s0 | s1 << 16;
    else *reinterpret_cast<uint16_t *>(p) = (uint16_t)(s0 | s1 << 8);
}

// The store half of the planar sink: block (bx, by) of frame f, texels px[16] (RGBA8, R in the low byte) and the column to its
// left, left[4] (4:2:0 and 4:2:2 only) -> its luma, Cb, Cr and alpha pieces.  luma: frame 0's luma plane.
template <int SUB, bool WIDE>
HAP_HD void planar_out_store_block(const PlanarOut &P, uint32_t f, uint32_t bx, uint32_t by, uint8_t *luma, const uint32_t px[16],
                                   const uint32_t left[4])
{
    constexpr uint32_t kSample = WIDE ? 2 : 1;
    const YuvOutCoeffs &k = P.g.k;
    const uint64_t frame = (uint64_t)f * P.g.frame_bytes, lrow = frame + (uint64_t)(4 * by) * P.g.pitch + (uint64_t)(4 * kSample) * bx;
#pragma unroll
    for (int r = 0; r < 4; r++)
        planar_out_store4<WIDE>(luma + lrow + (uint64_t)r * P.g.pitch, yuv_out_luma(px[4 * r], k), yuv_out_luma(px[4 * r + 1], k),
                                yuv_out_luma(px[4 * r + 2], k), yuv_out_luma(px[4 * r + 3], k));
    const auto ch = [&](int r, int c, int chan) { return (int32_t)byte_of(c < 0 ? left[r] : px[4 * r + c], chan); };
    if (SUB == HapB200Chroma_444) {
        const uint64_t crow = frame + (uint64_t)(4 * by) * P.chroma_pitch + (uint64_t)(4 * kSample) * bx;
#pragma unroll
        for (int r = 0; r < 4; r++) {
            uint32_t cb[4], cr[4];
#pragma unroll
            for (int c = 0; c < 4; c++) {
                const int32_t R = 8 * ch(r, c, 0), G = 8 * ch(r, c, 1), B = 8 * ch(r, c, 2);
                cb[c] = yuv_out_cb(R, G, B, k);
                cr[c] = yuv_out_cr(R, G, B, k);
            }
            planar_out_store4<WIDE>(P.cb + crow + (uint64_t)r * P.chroma_pitch, cb[0], cb[1], cb[2], cb[3]);
            planar_out_store4<WIDE>(P.cr + crow + (uint64_t)r * P.chroma_pitch, cr[0], cr[1], cr[2], cr[3]);
        }
    } else {
        // chroma rows of the block: 4:2:0 two (each the sum of texel rows 2j, 2j+1), 4:2:2 four (each texel row twice)
        constexpr int kRows = SUB == HapB200Chroma_420 ? 2 : 4;
        const uint64_t crow = frame + (uint64_t)(kRows * by) * P.chroma_pitch + (uint64_t)(2 * kSample) * bx;
#pragma unroll
        for (int j = 0; j < kRows; j++) {
            // s[c][chan]: chroma column 2bx+c: luma columns 4bx+2c-1 .. 4bx+2c+1, weights 1 2 1
            int32_t s[2][3] = {{0, 0, 0}, {0, 0, 0}};
#pragma unroll
            for (int rr = 0; rr < 2; rr++) {
                const int r = kRows == 2 ? 2 * j + rr : j;
#pragma unroll
                for (int c3 = 0; c3 < 3; c3++) {
                    const int32_t l = ch(r, -1, c3), p0 = ch(r, 0, c3), p1 = ch(r, 1, c3), p2 = ch(r, 2, c3), p3 = ch(r, 3, c3);
                    s[0][c3] += l + 2 * p0 + p1;
                    s[1][c3] += p1 + 2 * p2 + p3;
                }
            }
            planar_out_store2<WIDE>(P.cb + crow + (uint64_t)j * P.chroma_pitch, yuv_out_cb(s[0][0], s[0][1], s[0][2], k),
                                    yuv_out_cb(s[1][0], s[1][1], s[1][2], k));
            planar_out_store2<WIDE>(P.cr + crow + (uint64_t)j * P.chroma_pitch, yuv_out_cr(s[0][0], s[0][1], s[0][2], k),
                                    yuv_out_cr(s[1][0], s[1][1], s[1][2], k));
        }
    }
    if (P.alpha) {
#pragma unroll
        for (int r = 0; r < 4; r++) {
            uint32_t a[4];
#pragma unroll
            for (int c = 0; c < 4; c++) a[c] = WIDE ? planar_out_alpha(px[4 * r + c] >> 24, (uint32_t)k.top) : px[4 * r + c] >> 24;
            planar_out_store4<WIDE>(P.alpha + lrow + (uint64_t)r * P.g.pitch, a[0], a[1], a[2], a[3]);
        }
    }
}

// grid: 4:4:4 (bc_ctas, frames), 4:2:0 and 4:2:2 (yuv_out_ctas, frames).  KIND: kBcDxt1, kBcDxt5, kBcYCoCg (Hap Q; Hap Q Alpha
// when P.merge_alpha, whose RGTC1 texture then becomes A), kBcBc7.  SUB: HapB200ChromaSubsampling.  WIDE: 16-bit samples.
// frame_results (optional): a frame whose entry is not HapResult_No_Error is converted from zeros, as K8 writes it.
template <int KIND, int SUB, bool WIDE>
__global__ void __launch_bounds__(kBcThreads) bc_decode_planar_kernel(const uint8_t *__restrict__ blocks, PlanarOut P,
                                                                       uint8_t *__restrict__ luma, const uint32_t *__restrict__ frame_results)
{
    const YuvOutGeom &G = P.g;
    uint32_t bx, by, bxr;
    YuvOutLane L;
    if (SUB == HapB200Chroma_444) {
        const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
        if (bi >= G.blocks_x * G.blocks_y) return;
        by = bi / G.blocks_x;
        bx = bxr = bi - by * G.blocks_x;
    } else {
        if (!yuv_out_lane(G, blockIdx.x, threadIdx.x, L)) return;
        bx = L.bx;
        by = L.by;
        bxr = L.bxr;
    }
    uint32_t px[16];
    if (frame_results && frame_results[blockIdx.y] != 0u /* HapResult_No_Error */) {
#pragma unroll
        for (int t = 0; t < 16; t++) px[t] = 0;
    } else {
        const uint8_t *in = blocks + (uint64_t)blockIdx.y * G.in_stride;
        const uint32_t bi = by * G.blocks_x + bxr;
        if (KIND == kBcDxt1) {
            const uint2 v = reinterpret_cast<const uint2 *>(in)[bi];
            decode_block(KIND, v.x, v.y, 0, 0, px);
        } else {
            const uint4 v = reinterpret_cast<const uint4 *>(in)[bi];
            decode_block(KIND, v.x, v.y, v.z, v.w, px);
            if (KIND == kBcYCoCg && P.merge_alpha) {
                const uint2 a = reinterpret_cast<const uint2 *>(in + P.second_offset)[bi];
                uint32_t al[4];
                bc4_rows(a.x, a.y, al);
#pragma unroll
                for (int t = 0; t < 16; t++) px[t] = hap_prmt(px[t], al[t >> 2], 0x4210u + ((uint32_t)(t & 3) << 12));   // as bc_decode_kernel
            }
        }
    }
    uint32_t left[4] = {0, 0, 0, 0};
    if (SUB != HapB200Chroma_444) {
        // column 4bx-1 of rows 0..3: column 3 of the lane below; at the left edge column 0 (the clamp)
#pragma unroll
        for (int r = 0; r < 4; r++) {
            left[r] = __shfl_up_sync(0xFFFFFFFFu, px[4 * r + 3], 1);
            if (bx == 0) left[r] = px[4 * r];
        }
        if (L.lane == 0 || bx >= G.blocks_x) return;
    }
    planar_out_store_block<SUB, WIDE>(P, blockIdx.y, bx, by, luma, px, left);
}

// Hap Alpha-Only: grid = (bc_ctas, frames), RGTC1 blocks -> the alpha plane P.alpha alone (the matte v, mapped as A), rows
// P.g.pitch apart.  One thread per block; frame_results as bc_decode_planar_kernel (a failed frame's alpha is 0).
template <bool WIDE>
__global__ void __launch_bounds__(kBcThreads) bc_decode_planar_alpha_kernel(const uint8_t *__restrict__ blocks, PlanarOut P,
                                                                             const uint32_t *__restrict__ frame_results)
{
    const YuvOutGeom &G = P.g;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= G.blocks_x * G.blocks_y) return;
    const uint32_t by = bi / G.blocks_x, bx = bi - by * G.blocks_x;
    uint32_t rows[4] = {0, 0, 0, 0};   // row r: the values of texels 4r .. 4r+3, one per byte
    if (!(frame_results && frame_results[blockIdx.y] != 0u /* HapResult_No_Error */)) {
        const uint2 v = reinterpret_cast<const uint2 *>(blocks + (uint64_t)blockIdx.y * G.in_stride)[bi];
        bc4_rows(v.x, v.y, rows);
    }
    uint8_t *a = P.alpha + (uint64_t)blockIdx.y * G.frame_bytes + (uint64_t)(4 * by) * G.pitch + (uint64_t)(WIDE ? 8 : 4) * bx;
    const uint32_t top = (uint32_t)G.k.top;
#pragma unroll
    for (int r = 0; r < 4; r++) {
        if (WIDE)
            planar_out_store4<true>(a + (uint64_t)r * G.pitch, planar_out_alpha(byte_of(rows[r], 0), top), planar_out_alpha(byte_of(rows[r], 1), top),
                                    planar_out_alpha(byte_of(rows[r], 2), top), planar_out_alpha(byte_of(rows[r], 3), top));
        else
            *reinterpret_cast<uint32_t *>(a + (uint64_t)r * G.pitch) = rows[r];
    }
}

}  // namespace hapb200
