// hap_b200/csrc/bc6h_decode.cuh -- K8: BPTC / BC6H (RGB UF16 and SF16, "Hap HDR") blocks -> RGBA16F, bc6h_decode_kernel.
//
// Output: four IEEE binary16 values per pixel, R G B A, 8 bytes; A is always 1.0 (0x3C00).  Integer arithmetic only, as
// the BPTC specification states the decoder: endpoints unquantised to 16 bits, interpolated with (a (64 - w) + b w + 32) >> 6,
// then scaled by 31/64 (UF16) or, on the magnitude, 31/32 (SF16) into the bits of a half.  Finite by construction: UF16
// tops out at 0x7BFF, and an SF16 endpoint of -32768 (mode 14) is taken as -32767, so no value reaches the +-Inf of
// 31/32 x 32768 = 0x7C00.  A negative value whose magnitude scales to 0 gives +0 (0x0000), as the specification's integer
// form does.  The four reserved 5-bit mode values decode to (0, 0, 0, 1.0).
//
// Every endpoint component of BC6H is scattered over the block in a mode-specific order: a contiguous run for its low bits
// and, in most modes, a few single bits elsewhere; modes 13 and 14 store their base's high bits reversed.  Neighbouring
// blocks of real content use different modes, so as for BC7 (bc7_decode.cuh) the decoder is TABLE-DRIVEN and every lane
// runs one instruction stream: the mode's row of kBc6hLayout lists, for each of the 12 components, the pieces it is made
// of (source bit, length, destination bit, reversed or not), at most 25 pieces in fixed slots, so the destination register
// of every slot is known at compile time.  A row is 64 bytes, read as four 128-bit __ldg loads; the 14 rows (896 bytes)
// stay in L1.  Partitions 0-31 and their anchors are the first 32 two-subset entries of BC7's tables (bc7_partition,
// bc7_anchors).
#pragma once
#include "bc_decode.cuh"
#include "hap_codes.h"

namespace hapb200 {

// Row of mode m (the specification's mode m + 1), 32 halves: the mode's parameters (two halves), then its pieces in slots
//   r0 r0 | g0 g0 | b0 b0 | r1 | g1 | b1 | r2 | g2 g2 g2 | b2 b2 b2 | r3 | g3 g3 g3 | b3 b3 b3 b3 b3
// (component c of endpoint e; endpoints 0 and 1 belong to region 0, 2 and 3 to region 1; an empty slot is 0), then padding.
//   BC6H_MODE(precision, delta bits R, G, B, transformed, regions)
//   BC6H_F(pos, hi, lo): bits hi..lo of the component are stored from block bit pos on, lowest first;
//   BC6H_R(pos, hi, lo): the same bits stored reversed, bit hi first.
#define BC6H_MODE(prec, dr, dg, db, tr, regions) \
    (uint16_t)((prec) | (dr) << 5 | (dg) << 10), (uint16_t)((db) | (tr) << 5 | ((regions) - 1) << 6)
#define BC6H_F(pos, hi, lo) (uint16_t)((pos) | ((hi) - (lo) + 1) << 7 | (lo) << 11)
#define BC6H_R(pos, hi, lo) (uint16_t)(BC6H_F(pos, hi, lo) | 0x8000u)
#define HAP_BC6H_LAYOUT \
    /*  1 */ BC6H_MODE(10, 5, 5, 5, 1, 2), BC6H_F(5, 9, 0), 0, BC6H_F(15, 9, 0), 0, BC6H_F(25, 9, 0), 0, BC6H_F(35, 4, 0), \
    BC6H_F(45, 4, 0), BC6H_F(55, 4, 0), BC6H_F(65, 4, 0), BC6H_F(2, 4, 4), BC6H_F(41, 3, 0), 0, BC6H_F(3, 4, 4), BC6H_F(61, 3, 0), 0, \
    BC6H_F(71, 4, 0), BC6H_F(40, 4, 4), BC6H_F(51, 3, 0), 0, BC6H_F(4, 4, 4), BC6H_F(50, 0, 0), BC6H_F(60, 1, 1), BC6H_F(70, 2, 2), \
    BC6H_F(76, 3, 3), 0, 0, 0, 0, 0, \
    /*  2 */ BC6H_MODE(7, 6, 6, 6, 1, 2), BC6H_F(5, 6, 0), 0, BC6H_F(15, 6, 0), 0, BC6H_F(25, 6, 0), 0, BC6H_F(35, 5, 0), \
    BC6H_F(45, 5, 0), BC6H_F(55, 5, 0), BC6H_F(65, 5, 0), BC6H_F(2, 5, 5), BC6H_F(24, 4, 4), BC6H_F(41, 3, 0), BC6H_F(14, 4, 4), \
    BC6H_F(22, 5, 5), BC6H_F(61, 3, 0), BC6H_F(71, 5, 0), BC6H_F(3, 5, 4), BC6H_F(51, 3, 0), 0, BC6H_F(12, 1, 0), BC6H_F(23, 2, 2), \
    BC6H_F(32, 3, 3), BC6H_R(33, 5, 4), 0, 0, 0, 0, 0, 0, \
    /*  3 */ BC6H_MODE(11, 5, 4, 4, 1, 2), BC6H_F(5, 9, 0), BC6H_F(40, 10, 10), BC6H_F(15, 9, 0), BC6H_F(49, 10, 10), BC6H_F(25, 9, 0), \
    BC6H_F(59, 10, 10), BC6H_F(35, 4, 0), BC6H_F(45, 3, 0), BC6H_F(55, 3, 0), BC6H_F(65, 4, 0), BC6H_F(41, 3, 0), 0, 0, \
    BC6H_F(61, 3, 0), 0, 0, BC6H_F(71, 4, 0), BC6H_F(51, 3, 0), 0, 0, BC6H_F(50, 0, 0), BC6H_F(60, 1, 1), BC6H_F(70, 2, 2), \
    BC6H_F(76, 3, 3), 0, 0, 0, 0, 0, 0, \
    /*  4 */ BC6H_MODE(11, 4, 5, 4, 1, 2), BC6H_F(5, 9, 0), BC6H_F(39, 10, 10), BC6H_F(15, 9, 0), BC6H_F(50, 10, 10), BC6H_F(25, 9, 0), \
    BC6H_F(59, 10, 10), BC6H_F(35, 3, 0), BC6H_F(45, 4, 0), BC6H_F(55, 3, 0), BC6H_F(65, 3, 0), BC6H_F(41, 3, 0), BC6H_F(75, 4, 4), 0, \
    BC6H_F(61, 3, 0), 0, 0, BC6H_F(71, 3, 0), BC6H_F(40, 4, 4), BC6H_F(51, 3, 0), 0, BC6H_F(60, 1, 1), BC6H_F(69, 0, 0), \
    BC6H_F(70, 2, 2), BC6H_F(76, 3, 3), 0, 0, 0, 0, 0, 0, \
    /*  5 */ BC6H_MODE(11, 4, 4, 5, 1, 2), BC6H_F(5, 9, 0), BC6H_F(39, 10, 10), BC6H_F(15, 9, 0), BC6H_F(49, 10, 10), BC6H_F(25, 9, 0), \
    BC6H_F(60, 10, 10), BC6H_F(35, 3, 0), BC6H_F(45, 3, 0), BC6H_F(55, 4, 0), BC6H_F(65, 3, 0), BC6H_F(41, 3, 0), 0, 0, \
    BC6H_F(40, 4, 4), BC6H_F(61, 3, 0), 0, BC6H_F(71, 3, 0), BC6H_F(51, 3, 0), 0, 0, BC6H_F(50, 0, 0), BC6H_F(69, 2, 1), \
    BC6H_R(75, 4, 3), 0, 0, 0, 0, 0, 0, 0, \
    /*  6 */ BC6H_MODE(9, 5, 5, 5, 1, 2), BC6H_F(5, 8, 0), 0, BC6H_F(15, 8, 0), 0, BC6H_F(25, 8, 0), 0, BC6H_F(35, 4, 0), \
    BC6H_F(45, 4, 0), BC6H_F(55, 4, 0), BC6H_F(65, 4, 0), BC6H_F(24, 4, 4), BC6H_F(41, 3, 0), 0, BC6H_F(14, 4, 4), BC6H_F(61, 3, 0), 0, \
    BC6H_F(71, 4, 0), BC6H_F(40, 4, 4), BC6H_F(51, 3, 0), 0, BC6H_F(34, 4, 4), BC6H_F(50, 0, 0), BC6H_F(60, 1, 1), BC6H_F(70, 2, 2), \
    BC6H_F(76, 3, 3), 0, 0, 0, 0, 0, \
    /*  7 */ BC6H_MODE(8, 6, 5, 5, 1, 2), BC6H_F(5, 7, 0), 0, BC6H_F(15, 7, 0), 0, BC6H_F(25, 7, 0), 0, BC6H_F(35, 5, 0), \
    BC6H_F(45, 4, 0), BC6H_F(55, 4, 0), BC6H_F(65, 5, 0), BC6H_F(24, 4, 4), BC6H_F(41, 3, 0), 0, BC6H_F(14, 4, 4), BC6H_F(61, 3, 0), 0, \
    BC6H_F(71, 5, 0), BC6H_F(13, 4, 4), BC6H_F(51, 3, 0), 0, BC6H_F(23, 2, 2), BC6H_F(33, 4, 3), BC6H_F(50, 0, 0), BC6H_F(60, 1, 1), \
    0, 0, 0, 0, 0, 0, \
    /*  8 */ BC6H_MODE(8, 5, 6, 5, 1, 2), BC6H_F(5, 7, 0), 0, BC6H_F(15, 7, 0), 0, BC6H_F(25, 7, 0), 0, BC6H_F(35, 4, 0), \
    BC6H_F(45, 5, 0), BC6H_F(55, 4, 0), BC6H_F(65, 4, 0), BC6H_R(23, 5, 4), BC6H_F(41, 3, 0), 0, BC6H_F(14, 4, 4), BC6H_F(61, 3, 0), 0, \
    BC6H_F(71, 4, 0), BC6H_F(33, 5, 5), BC6H_F(40, 4, 4), BC6H_F(51, 3, 0), BC6H_F(13, 0, 0), BC6H_F(34, 4, 4), BC6H_F(60, 1, 1), \
    BC6H_F(70, 2, 2), BC6H_F(76, 3, 3), 0, 0, 0, 0, 0, \
    /*  9 */ BC6H_MODE(8, 5, 5, 6, 1, 2), BC6H_F(5, 7, 0), 0, BC6H_F(15, 7, 0), 0, BC6H_F(25, 7, 0), 0, BC6H_F(35, 4, 0), \
    BC6H_F(45, 4, 0), BC6H_F(55, 5, 0), BC6H_F(65, 4, 0), BC6H_F(24, 4, 4), BC6H_F(41, 3, 0), 0, BC6H_F(14, 4, 4), BC6H_F(23, 5, 5), \
    BC6H_F(61, 3, 0), BC6H_F(71, 4, 0), BC6H_F(40, 4, 4), BC6H_F(51, 3, 0), 0, BC6H_F(13, 1, 1), BC6H_R(33, 5, 4), BC6H_F(50, 0, 0), \
    BC6H_F(70, 2, 2), BC6H_F(76, 3, 3), 0, 0, 0, 0, 0, \
    /* 10 */ BC6H_MODE(6, 6, 6, 6, 0, 2), BC6H_F(5, 5, 0), 0, BC6H_F(15, 5, 0), 0, BC6H_F(25, 5, 0), 0, BC6H_F(35, 5, 0), \
    BC6H_F(45, 5, 0), BC6H_F(55, 5, 0), BC6H_F(65, 5, 0), BC6H_F(21, 5, 5), BC6H_F(24, 4, 4), BC6H_F(41, 3, 0), BC6H_F(14, 4, 4), \
    BC6H_F(22, 5, 5), BC6H_F(61, 3, 0), BC6H_F(71, 5, 0), BC6H_F(11, 4, 4), BC6H_F(31, 5, 5), BC6H_F(51, 3, 0), BC6H_F(12, 1, 0), \
    BC6H_F(23, 2, 2), BC6H_F(32, 3, 3), BC6H_R(33, 5, 4), 0, 0, 0, 0, 0, 0, \
    /* 11 */ BC6H_MODE(10, 10, 10, 10, 0, 1), BC6H_F(5, 9, 0), 0, BC6H_F(15, 9, 0), 0, BC6H_F(25, 9, 0), 0, BC6H_F(35, 9, 0), \
    BC6H_F(45, 9, 0), BC6H_F(55, 9, 0), 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, \
    /* 12 */ BC6H_MODE(11, 9, 9, 9, 1, 1), BC6H_F(5, 9, 0), BC6H_F(44, 10, 10), BC6H_F(15, 9, 0), BC6H_F(54, 10, 10), BC6H_F(25, 9, 0), \
    BC6H_F(64, 10, 10), BC6H_F(35, 8, 0), BC6H_F(45, 8, 0), BC6H_F(55, 8, 0), 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, \
    /* 13 */ BC6H_MODE(12, 8, 8, 8, 1, 1), BC6H_F(5, 9, 0), BC6H_R(43, 11, 10), BC6H_F(15, 9, 0), BC6H_R(53, 11, 10), BC6H_F(25, 9, 0), \
    BC6H_R(63, 11, 10), BC6H_F(35, 7, 0), BC6H_F(45, 7, 0), BC6H_F(55, 7, 0), 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, \
    /* 14 */ BC6H_MODE(16, 4, 4, 4, 1, 1), BC6H_F(5, 9, 0), BC6H_R(39, 15, 10), BC6H_F(15, 9, 0), BC6H_R(49, 15, 10), BC6H_F(25, 9, 0), \
    BC6H_R(59, 15, 10), BC6H_F(35, 3, 0), BC6H_F(45, 3, 0), BC6H_F(55, 3, 0), 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0

constexpr uint32_t kBc6hModes = 14, kBc6hSlots = 25;

#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
alignas(16) static const uint16_t kBc6hLayoutHost[] = {HAP_BC6H_LAYOUT};
static_assert(sizeof(kBc6hLayoutHost) == kBc6hModes * 64, "a row of kBc6hLayout is 32 halves");
#endif
#ifndef HAPB200_EMU
__device__ __align__(16) const uint16_t kBc6hLayout[kBc6hModes * 32] = {HAP_BC6H_LAYOUT};
#endif
#undef BC6H_MODE
#undef BC6H_F
#undef BC6H_R

// 16 bytes k (0..3) of the row of mode m, and the bit reversal
#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD uint4 bc6h_layout(uint32_t m, uint32_t k)
{
    uint4 v;
    memcpy(&v, &kBc6hLayoutHost[32 * m + 8 * k], 16);
    return v;
}
HAP_HD uint32_t hap_brev(uint32_t x)
{
    uint32_t r = 0;
    for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i);
    return r;
}
#else
__device__ __forceinline__ uint4 bc6h_layout(uint32_t m, uint32_t k) { return __ldg(reinterpret_cast<const uint4 *>(kBc6hLayout) + 4 * m + k); }
__device__ __forceinline__ uint32_t hap_brev(uint32_t x) { return __brev(x); }
#endif

// component (r0 g0 b0 r1 ... b3 = 0 .. 11) that piece slot s builds (the slot order of the rows above)
HAP_HD constexpr uint32_t bc6h_slot_component(uint32_t s)
{
    return s < 6 ? s / 2 : s < 10 ? s - 3 : s < 13 ? 7 : s < 16 ? 8 : s == 16 ? 9 : s < 20 ? 10 : 11;
}

// the low n bits of v sign-extended (4 <= n <= 16)
HAP_HD int32_t bc6h_sext(uint32_t v, uint32_t n) { return (int32_t)(v << (32 - n)) >> (32 - n); }

// an endpoint component of `prec` bits -> 16 bits (UF16: 0 .. 0xFFFF; SF16: -32767 .. 32767)
HAP_HD int32_t bc6h_unquantize(int32_t x, uint32_t prec, bool sgn)
{
    if (!sgn) {
        const uint32_t u = (uint32_t)x;
        return prec >= 15 ? x : u == 0 ? 0 : u == (1u << prec) - 1u ? 0xFFFF : (int32_t)(((u << 16) + 0x8000u) >> prec);
    }
    const uint32_t a = (uint32_t)(x < 0 ? -x : x);
    const uint32_t q = prec >= 16 ? (a > 0x7FFFu ? 0x7FFFu : a)
                       : a == 0 ? 0u : a >= (1u << (prec - 1)) - 1u ? 0x7FFFu : ((a << 15) + 0x4000u) >> (prec - 1);
    return x < 0 ? -(int32_t)q : (int32_t)q;
}

// an interpolated value -> binary16 bits: x 31/64 (UF16), or x 31/32 on the magnitude with the sign apart (SF16)
HAP_HD uint32_t bc6h_finish(int32_t c, bool sgn)
{
    const uint32_t a = (uint32_t)(c < 0 ? -c : c);
    const uint32_t m = (a * 31u) >> (sgn ? 5 : 6);
    return c < 0 && m ? 0x8000u | m : m;
}

// One block -> its 16 texels, RGBA16F: texel t in out[2t] (R | G << 16) and out[2t + 1] (B | 1.0 << 16)
HAP_HD void bc6h_decode_block(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, bool sgn, uint32_t out[32])
{
    // mode: 2 bits (00, 01: modes 1, 2), else 5 bits: xxx10 = modes 3..10, 0xx11 = modes 11..14, 1xx11 reserved
    const uint32_t lo2 = w0 & 3u, m5 = (w0 >> 2) & 7u;
    const bool reserved = lo2 == 3u && m5 >= 4u;
    const uint32_t mi = lo2 < 2u ? lo2 : lo2 == 2u ? 2u + m5 : 10u + (m5 & 3u);   // (a reserved block reads a row, then is replaced)
    uint32_t row[16];
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        const uint4 v = bc6h_layout(mi, k);
        row[4 * k] = v.x; row[4 * k + 1] = v.y; row[4 * k + 2] = v.z; row[4 * k + 3] = v.w;
    }
    const uint32_t par = row[0], prec = par & 31u, transformed = (par >> 21) & 1u, two = (par >> 22) & 1u;

    // the stored components, piece by piece
    uint32_t raw[12];
#pragma unroll
    for (uint32_t c = 0; c < 12; c++) raw[c] = 0;
#pragma unroll
    for (uint32_t s = 0; s < kBc6hSlots; s++) {
        const uint32_t e = (row[1 + s / 2] >> (16 * (s & 1))) & 0xFFFFu, n = (e >> 7) & 15u;
        uint32_t v = bc7_bits(w0, w1, w2, w3, e & 127u, n);
        v = (e & 0x8000u) ? hap_brev(v) >> ((32u - n) & 31u) : v;
        raw[bc6h_slot_component(s)] |= v << ((e >> 11) & 15u);
    }

    // endpoints: the base sign-extended (SF16); the others deltas from it (transformed modes: sign-extended, added to the
    // base, wrapped to its precision, then sign-extended as well in SF16) or values of their own; all unquantised
    const uint32_t mask = (1u << prec) - 1u;
    int32_t ep[12];
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) {
        const uint32_t db = (par >> (c == 0 ? 5 : c == 1 ? 10 : 16)) & 31u;
        ep[c] = bc6h_unquantize(sgn ? bc6h_sext(raw[c], prec) : (int32_t)raw[c], prec, sgn);
#pragma unroll
        for (uint32_t e = 1; e < 4; e++) {
            const uint32_t x = transformed ? ((uint32_t)bc6h_sext(raw[3 * e + c], db) + raw[c]) & mask : raw[3 * e + c];
            ep[3 * e + c] = bc6h_unquantize(sgn ? bc6h_sext(x, prec) : (int32_t)x, prec, sgn);
        }
    }

    // two regions: partition (5 bits after the endpoints), 3-bit indices from bit 82; one region: 4-bit indices from bit 65.
    // Texel 0 and the anchor of region 1 store one index bit less.
    const uint32_t part = bc7_bits(w0, w1, w2, w3, 77, 5);
    const uint32_t map = two ? bc7_partition(part) : 0u, amask = two ? bc7_anchors(part) : 1u;
    const uint32_t ib = two ? 3u : 4u, p_idx = two ? 82u : 65u;
    uint32_t before = 0;   // anchors before texel t
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const uint32_t anchor = (amask >> t) & 1u;
        const uint32_t i = bc7_bits(w0, w1, w2, w3, p_idx + t * ib - before, ib - anchor);
        before += anchor;
        const int32_t w = (int32_t)bc7_weight(i, ib);
        const bool r1 = ((map >> (2 * t)) & 1u) != 0;
        uint32_t h[3];
#pragma unroll
        for (uint32_t c = 0; c < 3; c++) {
            const int32_t a = r1 ? ep[6 + c] : ep[c], b = r1 ? ep[9 + c] : ep[3 + c];
            h[c] = bc6h_finish((a * (64 - w) + b * w + 32) >> 6, sgn);
        }
        out[2 * t] = reserved ? 0u : h[0] | (h[1] << 16);
        out[2 * t + 1] = (reserved ? 0u : h[2]) | 0x3C000000u;
    }
}

// grid = (bc_ctas, frames), G as for bc_decode_kernel (row_bytes >= 8 * width).  Signedness per frame: SF16 when
// frame_formats[f] is the signed BC6H format, else UF16; without frame_formats, is_signed for every frame.
// frame_results (optional): HapResult per frame of the decode that filled `blocks`; a frame that failed is written as zeros.
__global__ void __launch_bounds__(kBcThreads) bc6h_decode_kernel(const uint8_t *__restrict__ blocks, BcDecodeGeom G,
                                                                 uint8_t *__restrict__ rgba, const uint32_t *__restrict__ frame_results,
                                                                 const uint32_t *__restrict__ frame_formats, uint32_t is_signed)
{
    const uint32_t nblocks = G.blocks_x * G.blocks_y;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= nblocks) return;
    const uint32_t by = bi / G.blocks_x, bx = bi - by * G.blocks_x;
    uint32_t px[32];
    if (frame_results && frame_results[blockIdx.y] != 0u /* HapResult_No_Error */) {
#pragma unroll
        for (int k = 0; k < 32; k++) px[k] = 0;
    } else {
        const bool sgn = frame_formats ? frame_formats[blockIdx.y] == HapFmt_RGB_BPTC_SFLOAT : is_signed != 0u;
        const uint4 v = reinterpret_cast<const uint4 *>(blocks + (uint64_t)blockIdx.y * G.in_stride)[bi];
        bc6h_decode_block(v.x, v.y, v.z, v.w, sgn, px);
    }
    // a block row is 32 bytes: two 16-byte stores, so a warp writes 1 KiB contiguous per pixel row
    uint8_t *dst = rgba + (uint64_t)blockIdx.y * G.frame_bytes + (uint64_t)(4 * by) * G.row_bytes + 32u * bx;
#pragma unroll
    for (int row = 0; row < 4; row++) {
        uint4 *d = reinterpret_cast<uint4 *>(dst + (uint64_t)row * G.row_bytes);
        d[0] = make_uint4(px[8 * row], px[8 * row + 1], px[8 * row + 2], px[8 * row + 3]);
        d[1] = make_uint4(px[8 * row + 4], px[8 * row + 5], px[8 * row + 6], px[8 * row + 7]);
    }
}

}  // namespace hapb200
