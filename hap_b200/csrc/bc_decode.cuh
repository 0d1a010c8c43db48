// hap_b200/csrc/bc_decode.cuh -- K8: DXT1 / DXT5 / scaled-YCoCg-DXT5 / RGTC1 / BC7 blocks -> RGBA8.
//
// The step AFTER HapDecode in every player: in the reference's world it is the GPU texture unit plus
// a YCoCg fragment shader (/root/reference/README.md:4, documentation/HapVideoDRAFT.md:8,81).  Here it
// is an optional tail kernel so a decoded frame can be handed on as plain RGBA.  Integer arithmetic
// throughout (truncating S3TC interpolation, exact quarter-unit YCoCg), bit-exact against
// oracle/bc_oracle.c, which is itself cross-checked against Pillow's bcn decoder.
// One thread per block: reads 8/16 contiguous bytes, writes four 16-byte row pieces; a warp therefore
// writes 512 contiguous bytes per pixel row.
#pragma once
#include "bc7_decode.cuh"
#include "bc_encode.cuh"

namespace hapb200 {

// ---- palette look-ups by byte permute --------------------------------------------------------------------------
// A block's palette has 4 (colour) or 8 (BC4) byte-sized entries per channel: they fit one or two registers, and
// PRMT picks four of them at once when its selector holds the four texel indices of a block row, one per nibble.
// The indices arrive 2 or 3 bits apart; two mask-shift-or steps spread them to nibbles.
// (hap_prmt: bc_block.cuh)
#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD int hap_min_relu(int a, int b) { int m = a < b ? a : b; return m < 0 ? 0 : m; }
#else
__device__ __forceinline__ int hap_min_relu(int a, int b) { return __vimin_s32_relu(a, b); }   // clamp(a, 0, b) for b >= 0
#endif
HAP_HD uint32_t spread3_to_nibbles(uint32_t x)   // i0 | i1<<3 | i2<<6 | i3<<9  ->  i0 | i1<<4 | i2<<8 | i3<<12
{
    x = (x & 0x3Fu) | ((x & 0xFC0u) << 2);
    return (x & 0x0707u) | ((x & 0x3838u) << 1);
}
HAP_HD uint32_t spread2_to_nibbles(uint32_t x)   // i0 | i1<<2 | i2<<4 | i3<<6  ->  i0 | i1<<4 | i2<<8 | i3<<12
{
    x = (x & 0x0Fu) | ((x & 0xF0u) << 4);
    return (x & 0x0303u) | ((x & 0x0C0Cu) << 2);
}
HAP_HD uint32_t byte_of(uint32_t x, int k) { return hap_prmt(x, 0, 0x4440u + (uint32_t)k); }   // zero-extended byte k

// BC4 block (w0, w1) -> its 16 values, four per register (row r = texels 4r .. 4r+3)
HAP_HD void bc4_rows(uint32_t w0, uint32_t w1, uint32_t rows[4])
{
    const uint32_t a0 = w0 & 0xFF, a1 = (w0 >> 8) & 0xFF;
    uint32_t p[8];
    p[0] = a0;
    p[1] = a1;
    if (a0 > a1) {
        // ((8-i) a0 + (i-1) a1) / 7, truncating; the numerators stay below 1786, where q/7 == (q * 9363) >> 16
#pragma unroll
        for (uint32_t i = 2; i < 8; i++) p[i] = (((8 - i) * a0 + (i - 1) * a1) * 9363u) >> 16;
    } else {
        // ((6-i) a0 + (i-1) a1) / 5: numerators below 1276, where q/5 == (q * 13108) >> 16
#pragma unroll
        for (uint32_t i = 2; i < 6; i++) p[i] = (((6 - i) * a0 + (i - 1) * a1) * 13108u) >> 16;
        p[6] = 0;
        p[7] = 255;
    }
    const uint32_t plo = p[0] | (p[1] << 8) | (p[2] << 16) | (p[3] << 24), phi = p[4] | (p[5] << 8) | (p[6] << 16) | (p[7] << 24);
    const uint32_t lo = (w0 >> 16) | (w1 << 16), hi = w1 >> 16;   // the 48 index bits
    rows[0] = hap_prmt(plo, phi, spread3_to_nibbles(lo & 0xFFFu));
    rows[1] = hap_prmt(plo, phi, spread3_to_nibbles((lo >> 12) & 0xFFFu));
    rows[2] = hap_prmt(plo, phi, spread3_to_nibbles(((lo >> 24) | (hi << 8)) & 0xFFFu));
    rows[3] = hap_prmt(plo, phi, spread3_to_nibbles((hi >> 4) & 0xFFFu));
}

// BC1 colour block (w0 = endpoints, w1 = indices) -> per channel its 16 values, four per register.
// force4: DXT5-style blocks are always in 4-colour mode.  ch[0..3] = R, G, B, A planes, [r] = row.
HAP_HD void bc1_rows(uint32_t w0, uint32_t w1, bool force4, uint32_t ch[4][4])
{
    const uint32_t c0 = w0 & 0xFFFF, c1 = w0 >> 16;
    const uint32_t e0[3] = {expand5(c0 >> 11), expand6((c0 >> 5) & 63), expand5(c0 & 31)};
    const uint32_t e1[3] = {expand5(c1 >> 11), expand6((c1 >> 5) & 63), expand5(c1 & 31)};
    const bool four = force4 || c0 > c1;
    uint32_t pal[4];
#pragma unroll
    for (int c = 0; c < 3; c++) {
        // thirds, truncating: numerators below 766, where q/3 == (q * 21846) >> 16; or the average and 0
        const uint32_t p2 = four ? ((2 * e0[c] + e1[c]) * 21846u) >> 16 : (e0[c] + e1[c]) >> 1;
        const uint32_t p3 = four ? ((e0[c] + 2 * e1[c]) * 21846u) >> 16 : 0u;
        pal[c] = e0[c] | (e1[c] << 8) | (p2 << 16) | (p3 << 24);
    }
    pal[3] = four ? 0xFFFFFFFFu : 0x00FFFFFFu;   // 3-colour mode: index 3 is transparent black
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const uint32_t sel = spread2_to_nibbles((w1 >> (8 * r)) & 0xFFu);
#pragma unroll
        for (int c = 0; c < 4; c++) ch[c][r] = hap_prmt(pal[c], 0, sel);
    }
}

// four planar rows -> the 16 packed RGBA texels
HAP_HD void interleave_rows(const uint32_t R[4], const uint32_t G[4], const uint32_t B[4], const uint32_t A[4], uint32_t out[16])
{
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const uint32_t rg_lo = hap_prmt(R[r], G[r], 0x5140u), rg_hi = hap_prmt(R[r], G[r], 0x7362u);   // R0 G0 R1 G1 | R2 G2 R3 G3
        const uint32_t ba_lo = hap_prmt(B[r], A[r], 0x5140u), ba_hi = hap_prmt(B[r], A[r], 0x7362u);
        out[4 * r + 0] = hap_prmt(rg_lo, ba_lo, 0x5410u);
        out[4 * r + 1] = hap_prmt(rg_lo, ba_lo, 0x7632u);
        out[4 * r + 2] = hap_prmt(rg_hi, ba_hi, 0x5410u);
        out[4 * r + 3] = hap_prmt(rg_hi, ba_hi, 0x7632u);
    }
}

// texel t of a decoded block; out[16] packed RGBA (kBcRgtc1: the value in every colour channel, A = 255)
HAP_HD void decode_block(int kind, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t out[16])
{
    if (kind == kBcBc7) {
        bc7_decode_block(w0, w1, w2, w3, out);
        return;
    }
    const uint32_t ones[4] = {0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu};
    if (kind == kBcDxt1) {
        uint32_t ch[4][4];
        bc1_rows(w0, w1, false, ch);
        interleave_rows(ch[0], ch[1], ch[2], ch[3], out);
        return;
    }
    uint32_t a[4];
    bc4_rows(w0, w1, a);
    if (kind == kBcRgtc1) {
        interleave_rows(a, a, a, ones, out);
        return;
    }
    uint32_t ch[4][4];
    bc1_rows(w2, w3, true, ch);
    if (kind == kBcDxt5) {
        interleave_rows(ch[0], ch[1], ch[2], a, out);
        return;
    }
    // scaled YCoCg: (R',G',B',A) = (Co', Cg', scale bits, Y); exact quarter units, round half up.
    // quarter units per stored chroma step from the texel's B': B' >> 3 = 0 -> 4, 1 -> 2, else 1.
    // Only the palette's four B' values occur, so the step is looked up per palette entry, then per texel by PRMT.
    const uint32_t c0 = w2 & 0xFFFF, c1 = w2 >> 16;
    const uint32_t b0 = expand5(c0 & 31), b1 = expand5(c1 & 31);
    const uint32_t bp[4] = {b0, b1, ((2 * b0 + b1) * 21846u) >> 16, ((b0 + 2 * b1) * 21846u) >> 16};
    uint32_t qpal = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t sc = bp[i] >> 3;
        qpal |= (sc == 0 ? 4u : sc == 1 ? 2u : 1u) << (8 * i);
    }
#pragma unroll
    for (int r = 0; r < 4; r++) {
        const uint32_t q4 = hap_prmt(qpal, 0, spread2_to_nibbles((w3 >> (8 * r)) & 0xFFu));
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const int q = (int)byte_of(q4, k);
            const int co4 = ((int)byte_of(ch[0][r], k) - 128) * q, cg4 = ((int)byte_of(ch[1][r], k) - 128) * q;
            const int y4 = 4 * (int)byte_of(a[r], k) + 2;
            const uint32_t R = (uint32_t)hap_min_relu((y4 + co4 - cg4) >> 2, 255);
            const uint32_t G = (uint32_t)hap_min_relu((y4 + cg4) >> 2, 255);
            const uint32_t B = (uint32_t)hap_min_relu((y4 - co4 - cg4) >> 2, 255);
            out[4 * r + k] = R | (G << 8) | (B << 16) | 0xFF000000u;
        }
    }
}

struct BcDecodeGeom {
    uint32_t blocks_x, blocks_y;
    uint32_t row_bytes;      // RGBA row stride
    uint32_t merge_alpha;    // 1: `alpha_blocks` holds an RGTC1 plane to merge into A (Hap Q Alpha)
    uint64_t in_stride;      // DXT bytes per frame
    uint64_t alpha_stride;
    uint64_t frame_bytes;    // RGBA frame stride
};

HAP_HD BcDecodeGeom bc_decode_geom(uint32_t width, uint32_t height, uint32_t row_bytes, bool merge_alpha, uint64_t in_stride,
                                   uint64_t alpha_stride, uint64_t frame_bytes)
{
    BcDecodeGeom g;
    g.blocks_x = width / 4;
    g.blocks_y = height / 4;
    g.row_bytes = row_bytes;
    g.merge_alpha = merge_alpha ? 1u : 0u;
    g.in_stride = in_stride;
    g.alpha_stride = alpha_stride;
    g.frame_bytes = frame_bytes;
    return g;
}

// grid = (bc_ctas, frames).  kBcRgtc1 alone writes the value to all of R,G,B with A=255.  kBcBc7 never merges alpha.
template <int KIND>
__global__ void __launch_bounds__(kBcThreads) bc_decode_kernel(const uint8_t *__restrict__ blocks,
                                                                const uint8_t *__restrict__ alpha_blocks,
                                                                BcDecodeGeom G, uint8_t *__restrict__ rgba,
                                                                const uint32_t *__restrict__ frame_results)
{
    const uint32_t nblocks = G.blocks_x * G.blocks_y;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= nblocks) return;
    const uint32_t by = bi / G.blocks_x, bx = bi - by * G.blocks_x;
    const uint8_t *in = blocks + (uint64_t)blockIdx.y * G.in_stride;
    uint32_t px[16];
    // frame_results (optional): HapResult per frame of the decode that filled `blocks`.  A frame that failed has no
    // texture in its slot (the slot holds whatever the memory pool handed out): its picture is written as zeros.
    if (frame_results && frame_results[blockIdx.y] != 0u /* HapResult_No_Error */) {
#pragma unroll
        for (int t = 0; t < 16; t++) px[t] = 0;
    } else if (KIND == kBcDxt1 || KIND == kBcRgtc1) {
        uint2 v = reinterpret_cast<const uint2 *>(in)[bi];
        decode_block(KIND, v.x, v.y, 0, 0, px);
    } else if (KIND == kBcBc7) {
        uint4 v = reinterpret_cast<const uint4 *>(in)[bi];
        bc7_decode_block(v.x, v.y, v.z, v.w, px);
    } else {
        uint4 v = reinterpret_cast<const uint4 *>(in)[bi];
        decode_block(KIND, v.x, v.y, v.z, v.w, px);
        if (G.merge_alpha) {
            uint2 a = reinterpret_cast<const uint2 *>(alpha_blocks + (uint64_t)blockIdx.y * G.alpha_stride)[bi];
            uint32_t al[4];
            bc4_rows(a.x, a.y, al);
#pragma unroll
            for (int t = 0; t < 16; t++) px[t] = hap_prmt(px[t], al[t >> 2], 0x4210u + ((uint32_t)(t & 3) << 12));   // alpha byte t%4 of its row
        }
    }
    uint8_t *dst = rgba + (uint64_t)blockIdx.y * G.frame_bytes + (uint64_t)(4 * by) * G.row_bytes + 16u * bx;
#pragma unroll
    for (int row = 0; row < 4; row++)
        *reinterpret_cast<uint4 *>(dst + (uint64_t)row * G.row_bytes) =
            make_uint4(px[4 * row], px[4 * row + 1], px[4 * row + 2], px[4 * row + 3]);
}

}  // namespace hapb200
