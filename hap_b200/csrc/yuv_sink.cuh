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
//
// The HDR10 sink (bc6h_decode_yuv_kernel, HapB200DecodeYUVPQ) has the same shape and the same store half
// (yuv_out_store_block): BC6H blocks (bc6h_decode_block, bc6h_decode.cuh) -> RGBA16F texels in registers -> 12-bit PQ codes
// through the table P (yuv_pq_out_table, built on the host) -> the matrix of HAPB200_YUV_PQ_OUT_COEFFICIENTS -> P010.
#pragma once
#include "bc6h_decode.cuh"
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

// the row of HAPB200_YUV_PQ_OUT_COEFFICIENTS of colorSpace (HapB200YUV_BT2020_Limited / _Full), for P010
inline YuvOutCoeffs yuv_pq_out_coeffs(unsigned color_space)
{
    static const int32_t kCoeffs[2][11] = HAPB200_YUV_PQ_OUT_COEFFICIENTS;
    const int32_t *k = kCoeffs[color_space - HapB200YUV_BT2020_Limited];
    return YuvOutCoeffs{k[0], k[1], k[2], k[3], k[4], k[5], k[6], k[7], k[8], k[9], k[10], 1023};
}

// one pixel's R, G, B (8-bit values, or 12-bit codes with a PQ row) -> its luma sample
HAP_HD uint32_t yuv_out_luma_rgb(int32_t r, int32_t g, int32_t b, const YuvOutCoeffs &k)
{
    return yuv_out_clamp(((k.y_r * r + k.y_g * g + k.y_b * b + 32768) >> 16) + k.y_off, k.top);
}

// one pixel, packed RGBA8 (R in the low byte) -> its luma sample
HAP_HD uint32_t yuv_out_luma(uint32_t rgba, const YuvOutCoeffs &k)
{
    return yuv_out_luma_rgb((int32_t)(rgba & 0xFF), (int32_t)((rgba >> 8) & 0xFF), (int32_t)((rgba >> 16) & 0xFF), k);
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

inline YuvOutGeom yuv_out_geom(uint32_t width, uint32_t height, uint32_t pitch, uint64_t in_stride, uint64_t frame_bytes, const YuvOutCoeffs &k)
{
    YuvOutGeom g;
    g.blocks_x = width / 4;
    g.blocks_y = height / 4;
    g.spans = (g.blocks_x + kYuvOutSpan - 1) / kYuvOutSpan;
    g.pitch = pitch;
    g.in_stride = in_stride;
    g.frame_bytes = frame_bytes;
    g.k = k;
    return g;
}

inline YuvOutGeom yuv_out_geom(uint32_t width, uint32_t height, uint32_t pitch, uint64_t in_stride, uint64_t frame_bytes, unsigned layout,
                               unsigned color_space)
{
    return yuv_out_geom(width, height, pitch, in_stride, frame_bytes, yuv_out_coeffs(layout, color_space));
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

// The block a lane of a sink decodes (see the file comment): lanes 1-31 blocks span*31 .. span*31+30 of block row `by`, lane
// 0 the block left of them (none at the left edge).  Lanes past the row's end decode its last block again and write nothing.
// false: the warp is past the last block row (whole warps).
struct YuvOutLane {
    uint32_t lane, by, bx, bxr;   // bx: the block the lane writes (lane 0 of span 0: wraps, writes nothing); bxr: the one it decodes
};
HAP_HD bool yuv_out_lane(const YuvOutGeom &G, uint32_t cta, uint32_t thread, YuvOutLane &l)
{
    l.lane = thread & 31;
    const uint64_t warp = (uint64_t)cta * (kBcThreads / 32) + (thread >> 5);
    const uint64_t by64 = warp / G.spans;
    if (by64 >= G.blocks_y) return false;
    l.by = (uint32_t)by64;
    const uint32_t span = (uint32_t)(warp - by64 * G.spans);
    l.bx = span * kYuvOutSpan + l.lane - 1;
    l.bxr = (l.lane == 0 && span == 0) ? 0 : l.bx < G.blocks_x ? l.bx : G.blocks_x - 1;
    return true;
}

// The store half of the sinks: block (bx, by) of frame f -> its 4 luma row pieces and its 2 x 2 chroma pairs.  chan(r, c, ch):
// channel ch (0 R, 1 G, 2 B) of the block's texel row r, column c (0 .. 3, or -1: the column to the block's left);
// chan.luma(r, c, k): that texel's luma sample.  The channels are RGBA8 bytes or 12-bit PQ codes; G.k is the row for their
// range.
template <int LAYOUT, class Chan>
HAP_HD void yuv_out_store_block(const YuvOutGeom &G, uint32_t f, uint32_t bx, uint32_t by, uint8_t *luma, uint8_t *chroma, const Chan &chan)
{
    constexpr uint32_t kSample = LAYOUT == HapB200YUV_P010 ? 2 : 1;
    const YuvOutCoeffs &k = G.k;
    uint8_t *lrow = luma + (uint64_t)f * G.frame_bytes + (uint64_t)(4 * by) * G.pitch + (uint64_t)(4 * kSample) * bx;
#pragma unroll
    for (int r = 0; r < 4; r++)
        yuv_out_store4<LAYOUT>(lrow + (uint64_t)r * G.pitch, chan.luma(r, 0, k), chan.luma(r, 1, k), chan.luma(r, 2, k), chan.luma(r, 3, k));
    uint8_t *crow = chroma + (uint64_t)f * G.frame_bytes + (uint64_t)(2 * by) * G.pitch + (uint64_t)(4 * kSample) * bx;
#pragma unroll
    for (int j = 0; j < 2; j++) {
        // s[c][ch]: chroma column 2bx+c, channel ch (R, G, B): luma columns 4bx+2c-1 .. 4bx+2c+1, weights 1 2 1, rows 2j, 2j+1
        int32_t s[2][3] = {{0, 0, 0}, {0, 0, 0}};
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
            const int r = 2 * j + rr;
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                const int32_t l = chan(r, -1, ch), p0 = chan(r, 0, ch), p1 = chan(r, 1, ch), p2 = chan(r, 2, ch), p3 = chan(r, 3, ch);
                s[0][ch] += l + 2 * p0 + p1;
                s[1][ch] += p1 + 2 * p2 + p3;
            }
        }
        yuv_out_store4<LAYOUT>(crow + (uint64_t)j * G.pitch, yuv_out_cb(s[0][0], s[0][1], s[0][2], k), yuv_out_cr(s[0][0], s[0][1], s[0][2], k),
                               yuv_out_cb(s[1][0], s[1][1], s[1][2], k), yuv_out_cr(s[1][0], s[1][1], s[1][2], k));
    }
}

// RGBA8 texels px[16] (R in the low byte) and the left column left[4]
struct YuvOutRgba8 {
    const uint32_t *px, *left;
    HAP_HD int32_t operator()(int r, int c, int ch) const { return (int32_t)byte_of(c < 0 ? left[r] : px[4 * r + c], ch); }
    HAP_HD uint32_t luma(int r, int c, const YuvOutCoeffs &k) const { return yuv_out_luma(px[4 * r + c], k); }
};

// grid = (yuv_out_ctas, frames).  KIND: kBcDxt1, kBcDxt5, kBcYCoCg (Hap Q and Hap Q Alpha: alpha is dropped), kBcRgtc1
// (Hap Alpha-Only: (v, v, v, 255)), kBcBc7.  LAYOUT: HapB200YUV_NV12 / _P010.  frame_results (optional): a frame whose entry
// is not HapResult_No_Error is converted from zeros, as K8 writes it.
template <int KIND, int LAYOUT>
__global__ void __launch_bounds__(kBcThreads) bc_decode_yuv_kernel(const uint8_t *__restrict__ blocks, YuvOutGeom G,
                                                                    uint8_t *__restrict__ luma, uint8_t *__restrict__ chroma,
                                                                    const uint32_t *__restrict__ frame_results)
{
    YuvOutLane L;
    if (!yuv_out_lane(G, blockIdx.x, threadIdx.x, L)) return;
    uint32_t px[16];
    if (frame_results && frame_results[blockIdx.y] != 0u /* HapResult_No_Error */) {
#pragma unroll
        for (int t = 0; t < 16; t++) px[t] = 0;
    } else {
        const uint8_t *in = blocks + (uint64_t)blockIdx.y * G.in_stride;
        const uint32_t bi = L.by * G.blocks_x + L.bxr;
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
        if (L.bx == 0) left[r] = px[4 * r];
    }
    if (L.lane == 0 || L.bx >= G.blocks_x) return;
    yuv_out_store_block<LAYOUT>(G, blockIdx.y, L.bx, L.by, luma, chroma, YuvOutRgba8{px, left});
}

// ---- HDR10: BC6H -> RGBA16F -> PQ -> BT.2020 P010 (HapB200DecodeYUVPQ) -----------------------------------------------------

constexpr uint32_t kPqOutEntries = 0x7C00;   // P's index: the non-negative finite binary16 values 0x0000 .. 0x7BFF

// P of include/hap_b200.h for unitNits (1 .. 10000), in double precision:
// P[h] = floor(4095 * OETF(min(value(h) * unitNits / 10000, 1)) + 1/2), OETF the inverse of ST 2084's EOTF
inline void yuv_pq_out_table(uint32_t unit_nits, uint16_t table[kPqOutEntries])
{
    const double m1 = 2610.0 / 16384, m2 = 2523.0 / 32, c1 = 3424.0 / 4096, c2 = 2413.0 / 128, c3 = 2392.0 / 128;
    for (uint32_t h = 0; h < kPqOutEntries; h++) {
        const int e = (int)(h >> 10), m = (int)(h & 1023);
        const double v = e ? ldexp(1024 + m, e - 25) : ldexp(m, -24);   // exact
        const double y = v * unit_nits / 10000;
        const double p = pow(y < 1 ? y : 1, m1);
        table[h] = (uint16_t)floor(4095 * pow((c1 + c2 * p) / (1 + c3 * p), m2) + 0.5);
    }
}

// one binary16 value -> its 12-bit code: a set sign bit (SF16 negatives, -0) gives 0; the index is clamped to 0x7BFF (the
// block decoder writes no Inf or NaN)
HAP_HD uint32_t yuv_pq_code(const uint16_t *table, uint32_t h)
{
    return (h & 0x8000u) ? 0u : yuv_pq_lookup(table, h < kPqOutEntries - 1 ? h : kPqOutEntries - 1);
}

// 12-bit codes of texels px[32] (texel t: R | G << 16 in px[2t], B in px[2t + 1]) and of the left column (row r: left[2r],
// left[2r + 1])
struct YuvOutCodes {
    const uint32_t *px, *left;
    HAP_HD int32_t operator()(int r, int c, int ch) const
    {
        const uint32_t *p = c < 0 ? left + 2 * r : px + 2 * (4 * r + c);
        return (int32_t)(ch == 0 ? p[0] & 0xFFFFu : ch == 1 ? p[0] >> 16 : p[1]);
    }
    HAP_HD uint32_t luma(int r, int c, const YuvOutCoeffs &k) const { return yuv_out_luma_rgb((*this)(r, c, 0), (*this)(r, c, 1), (*this)(r, c, 2), k); }
};

// grid = (yuv_out_ctas, frames), G.k a row of HAPB200_YUV_PQ_OUT_COEFFICIENTS; P010 only.  Signedness per frame: SF16 when
// frame_formats[f] is the signed BC6H format, else UF16; without frame_formats, is_signed for every frame (as
// bc6h_decode_kernel).  frame_results (optional): a frame that failed is converted from zeros.  table: P (kPqOutEntries
// codes, device memory, read with __ldg: lane-dependent indices).
__global__ void __launch_bounds__(kBcThreads) bc6h_decode_yuv_kernel(const uint8_t *__restrict__ blocks, YuvOutGeom G,
                                                                     uint8_t *__restrict__ luma, uint8_t *__restrict__ chroma,
                                                                     const uint32_t *__restrict__ frame_results,
                                                                     const uint32_t *__restrict__ frame_formats, uint32_t is_signed,
                                                                     const uint16_t *__restrict__ table)
{
    YuvOutLane L;
    if (!yuv_out_lane(G, blockIdx.x, threadIdx.x, L)) return;
    uint32_t px[32];
    if (frame_results && frame_results[blockIdx.y] != 0u /* HapResult_No_Error */) {
#pragma unroll
        for (int k = 0; k < 32; k++) px[k] = 0;
    } else {
        const bool sgn = frame_formats ? frame_formats[blockIdx.y] == HapFmt_RGB_BPTC_SFLOAT : is_signed != 0u;
        const uint4 v = reinterpret_cast<const uint4 *>(blocks + (uint64_t)blockIdx.y * G.in_stride)[L.by * G.blocks_x + L.bxr];
        bc6h_decode_block(v.x, v.y, v.z, v.w, sgn, px);
    }
    // halves -> codes in place (A dropped)
#pragma unroll
    for (int t = 0; t < 16; t++) {
        px[2 * t] = yuv_pq_code(table, px[2 * t] & 0xFFFFu) | yuv_pq_code(table, px[2 * t] >> 16) << 16;
        px[2 * t + 1] = yuv_pq_code(table, px[2 * t + 1] & 0xFFFFu);
    }
    // column 4bx-1 of rows 0..3 from the lane below (R | G << 16 per row; B of rows 0, 1 and of rows 2, 3 share a word); at
    // the left edge column 0 (the clamp)
    uint32_t left[8];
#pragma unroll
    for (int r = 0; r < 4; r++) left[2 * r] = __shfl_up_sync(0xFFFFFFFFu, px[2 * (4 * r + 3)], 1);
#pragma unroll
    for (int h = 0; h < 2; h++) {
        const uint32_t b = __shfl_up_sync(0xFFFFFFFFu, px[2 * (8 * h + 3) + 1] | px[2 * (8 * h + 7) + 1] << 16, 1);
        left[4 * h + 1] = b & 0xFFFFu;
        left[4 * h + 3] = b >> 16;
    }
    if (L.bx == 0) {
#pragma unroll
        for (int r = 0; r < 4; r++) { left[2 * r] = px[8 * r]; left[2 * r + 1] = px[8 * r + 1]; }
    }
    if (L.lane == 0 || L.bx >= G.blocks_x) return;
    yuv_out_store_block<HapB200YUV_P010>(G, blockIdx.y, L.bx, L.by, luma, chroma, YuvOutCodes{px, left});
}

}  // namespace hapb200
