// hap_b200/csrc/bc7_decode.cuh -- BPTC / BC7 (RGBA UNORM, "Hap R") blocks -> RGBA8, for bc_decode_kernel<kBcBc7> (K8).
//
// Every field of a BC7 block sits at a place that depends on the block's mode (eight layouts).  Neighbouring blocks of real
// content use different modes, so a branch per mode would split every warp eight ways.  The decoder is TABLE-DRIVEN instead:
// the mode's field widths come out of packed immediates (one nibble per mode, no memory access), one bit reader extracts any
// field of the 128 bits, and every lane runs the same instruction stream whatever its mode.  Fields a mode lacks are read
// with width 0 and come out as 0.
//
// Partition and anchor tables (768 bytes, indexed by a lane-dependent partition number): read with __ldg from global
// memory, not from __constant__ (divergent constant-bank reads are serialised, one address per pass) and not from a
// shared-memory copy (every 128-thread CTA would have to fill it and wait on a barrier before its one block per thread;
// a 4K frame has ~4 000 such CTAs).  The tables span six 128-byte lines, which stay in L1 after the first touch.
//
// Reserved blocks (byte 0 = 0) decode to (0, 0, 0, 0) in every texel, as the format specification says.  (Some software
// decoders, Pillow's among them, write A = 255 there.)
#pragma once
#include "bc_block.cuh"

namespace hapb200 {

// Partitions [0, 64) two subsets, [64, 128) three subsets: subset of texel t in bits 2t, 2t+1.
#define HAP_BC7_PARTITIONS \
    0x50505050u, 0x40404040u, 0x54545454u, 0x54505040u, 0x50404000u, 0x55545450u, 0x55545040u, 0x54504000u, \
    0x50400000u, 0x55555450u, 0x55544000u, 0x54400000u, 0x55555440u, 0x55550000u, 0x55555500u, 0x55000000u, \
    0x55150100u, 0x00004054u, 0x15010000u, 0x00405054u, 0x00004050u, 0x15050100u, 0x05010000u, 0x40505054u, \
    0x00404050u, 0x05010100u, 0x14141414u, 0x05141450u, 0x01155440u, 0x00555500u, 0x15014054u, 0x05414150u, \
    0x44444444u, 0x55005500u, 0x11441144u, 0x05055050u, 0x05500550u, 0x11114444u, 0x41144114u, 0x44111144u, \
    0x15055054u, 0x01055040u, 0x05041050u, 0x05455150u, 0x14414114u, 0x50050550u, 0x41411414u, 0x00141400u, \
    0x00041504u, 0x00105410u, 0x10541000u, 0x04150400u, 0x50410514u, 0x41051450u, 0x05415014u, 0x14054150u, \
    0x41050514u, 0x41505014u, 0x40011554u, 0x54150140u, 0x50505500u, 0x00555050u, 0x15151010u, 0x54540404u, \
    0xAA685050u, 0x6A5A5040u, 0x5A5A4200u, 0x5450A0A8u, 0xA5A50000u, 0xA0A05050u, 0x5555A0A0u, 0x5A5A5050u, \
    0xAA550000u, 0xAA555500u, 0xAAAA5500u, 0x90909090u, 0x94949494u, 0xA4A4A4A4u, 0xA9A59450u, 0x2A0A4250u, \
    0xA5945040u, 0x0A425054u, 0xA5A5A500u, 0x55A0A0A0u, 0xA8A85454u, 0x6A6A4040u, 0xA4A45000u, 0x1A1A0500u, \
    0x0050A4A4u, 0xAAA59090u, 0x14696914u, 0x69691400u, 0xA08585A0u, 0xAA821414u, 0x50A4A450u, 0x6A5A0200u, \
    0xA9A58000u, 0x5090A0A8u, 0xA8A09050u, 0x24242424u, 0x00AA5500u, 0x24924924u, 0x24499224u, 0x50A50A50u, \
    0x500AA550u, 0xAAAA4444u, 0x66660000u, 0xA5A0A5A0u, 0x50A050A0u, 0x69286928u, 0x44AAAA44u, 0x66666600u, \
    0xAA444444u, 0x54A854A8u, 0x95809580u, 0x96969600u, 0xA85454A8u, 0x80959580u, 0xAA141414u, 0x96960000u, \
    0xAAAA1414u, 0xA05050A0u, 0xA0A5A5A0u, 0x96000000u, 0x40804080u, 0xA9A8A9A8u, 0xAAAAAA44u, 0x2A4A5254u
// Anchor texels (those whose primary index is stored with one bit less) of the same partitions, one bit per texel: texel 0
// and the anchors of subsets 1 and 2.
#define HAP_BC7_ANCHORS \
    0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, \
    0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, \
    0x8001u, 0x0005u, 0x0101u, 0x0005u, 0x0005u, 0x0101u, 0x0101u, 0x8001u, \
    0x0005u, 0x0101u, 0x0005u, 0x0005u, 0x0101u, 0x0101u, 0x0005u, 0x0005u, \
    0x8001u, 0x8001u, 0x0041u, 0x0101u, 0x0005u, 0x0101u, 0x8001u, 0x8001u, \
    0x0005u, 0x0101u, 0x0005u, 0x0005u, 0x0005u, 0x8001u, 0x8001u, 0x0041u, \
    0x0041u, 0x0005u, 0x0041u, 0x0101u, 0x8001u, 0x8001u, 0x0005u, 0x0005u, \
    0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x8001u, 0x0005u, 0x0005u, 0x8001u, \
    0x8009u, 0x0109u, 0x8101u, 0x8009u, 0x8101u, 0x8009u, 0x8009u, 0x8101u, \
    0x8101u, 0x8101u, 0x8041u, 0x8041u, 0x8041u, 0x8021u, 0x8009u, 0x0109u, \
    0x8009u, 0x0109u, 0x8101u, 0x8009u, 0x8009u, 0x0109u, 0x8041u, 0x0501u, \
    0x0029u, 0x8101u, 0x0141u, 0x0441u, 0x8101u, 0x8021u, 0x8401u, 0x8101u, \
    0x8101u, 0x8009u, 0x8009u, 0x0421u, 0x0441u, 0x0501u, 0x0301u, 0x8401u, \
    0x8041u, 0x8009u, 0x8101u, 0x8021u, 0x8009u, 0x8041u, 0x8041u, 0x8101u, \
    0x8009u, 0x8009u, 0x8021u, 0x8021u, 0x8021u, 0x8101u, 0x8021u, 0x8401u, \
    0x8021u, 0x8401u, 0x8101u, 0xA001u, 0x8009u, 0x9001u, 0x8009u, 0x0109u

#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
static const uint32_t kBc7PartitionHost[128] = {HAP_BC7_PARTITIONS};
static const uint16_t kBc7AnchorsHost[128] = {HAP_BC7_ANCHORS};
#endif
#ifndef HAPB200_EMU
__device__ const uint32_t kBc7Partition[128] = {HAP_BC7_PARTITIONS};
__device__ const uint16_t kBc7Anchors[128] = {HAP_BC7_ANCHORS};
#endif

// (hi:lo) >> s for s < 32, the lowest set bit of x != 0, and the table reads
#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD uint32_t hap_funnel_r(uint32_t lo, uint32_t hi, uint32_t s) { return (uint32_t)((((uint64_t)hi << 32) | lo) >> (s & 31)); }
HAP_HD uint32_t hap_ctz(uint32_t x) { return (uint32_t)__builtin_ctz(x); }
HAP_HD uint32_t bc7_partition(uint32_t i) { return kBc7PartitionHost[i]; }
HAP_HD uint32_t bc7_anchors(uint32_t i) { return kBc7AnchorsHost[i]; }
#else
__device__ __forceinline__ uint32_t hap_funnel_r(uint32_t lo, uint32_t hi, uint32_t s) { return __funnelshift_r(lo, hi, s); }
__device__ __forceinline__ uint32_t hap_ctz(uint32_t x) { return (uint32_t)__ffs((int)x) - 1u; }
__device__ __forceinline__ uint32_t bc7_partition(uint32_t i) { return __ldg(&kBc7Partition[i]); }
__device__ __forceinline__ uint32_t bc7_anchors(uint32_t i) { return __ldg(&kBc7Anchors[i]); }
#endif

// The mode table, one nibble per mode (mode m in bits 4m .. 4m+3), read with bc7_field(table, m)
constexpr uint32_t kBc7Subsets = 0x21112323u;      // NS   3 2 3 2 1 1 1 2
constexpr uint32_t kBc7PartBits = 0x60006664u;     // PB   4 6 6 6 0 0 0 6
constexpr uint32_t kBc7RotBits = 0x00220000u;      // RB   0 0 0 0 2 2 0 0
constexpr uint32_t kBc7SelBits = 0x00010000u;      // ISB  0 0 0 0 1 0 0 0
constexpr uint32_t kBc7ColourBits = 0x57757564u;   // CB   4 6 5 7 5 7 7 5
constexpr uint32_t kBc7AlphaBits = 0x57860000u;    // AB   0 0 0 0 6 8 7 5
constexpr uint32_t kBc7EndpointP = 0x11001001u;    // EPB  1 0 0 1 0 0 1 1
constexpr uint32_t kBc7SubsetP = 0x00000010u;      // SPB  0 1 0 0 0 0 0 0
constexpr uint32_t kBc7IndexBits = 0x24222233u;    // IB   3 3 2 2 2 2 4 2
constexpr uint32_t kBc7Index2Bits = 0x00230000u;   // IB2  0 0 0 0 3 2 0 0
HAP_HD uint32_t bc7_field(uint32_t table, uint32_t mode) { return (table >> (4 * mode)) & 0xFu; }

// n (<= 8) bits of the block (w0 = bits 0..31, ... w3 = bits 96..127) from bit `pos` on; 0 when n = 0
HAP_HD uint32_t bc7_bits(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t pos, uint32_t n)
{
    const uint32_t k = pos >> 5;
    const uint32_t lo = k == 0 ? w0 : k == 1 ? w1 : k == 2 ? w2 : w3;
    const uint32_t hi = k == 0 ? w1 : k == 1 ? w2 : k == 2 ? w3 : 0u;
    return hap_funnel_r(lo, hi, pos) & ((1u << n) - 1u);
}

// An n-bit endpoint value (5 <= n <= 8) -> 8 bits, its top bits repeated below it
HAP_HD uint32_t bc7_expand(uint32_t v, uint32_t n) { return (v << (8 - n)) | (v >> (2 * n - 8)); }

// Interpolation weight (of 64) of index i of a b-bit index set.  The tables of the format ({0,21,43,64}, {0,9,18,27,37,46,55,
// 64}, {0,4,9,...,60,64}) are i * 64 / (2^b - 1) rounded to nearest, which is (i replicated to 12 bits + 32) >> 6:
// i * 4095 / (2^b - 1) = i * {1365, 585, 273}.
HAP_HD uint32_t bc7_weight(uint32_t i, uint32_t b) { return (i * (b == 2 ? 1365u : b == 3 ? 585u : 273u) + 32u) >> 6; }

// One 8-bit channel between endpoint values e0 and e1 at weight w (of 64), as the format interpolates: the expression
// bc7_decode_block evaluates for G and A (and for R and B two at a time in 16-bit lanes), for the encoder's error
HAP_HD uint32_t bc7_interp(uint32_t e0, uint32_t e1, uint32_t w) { return ((64 - w) * e0 + w * e1 + 32u) >> 6; }

// One block -> its 16 texels, packed RGBA (texel t = row t/4, column t%4)
HAP_HD void bc7_decode_block(uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t out[16])
{
    const uint32_t mode = hap_ctz((w0 & 0xFFu) | 0x100u);   // 8: reserved block
    const uint32_t m = mode > 7 ? 7u : mode;               // (a reserved block is decoded as mode 7, then zeroed)
    const uint32_t ns = bc7_field(kBc7Subsets, m), pb = bc7_field(kBc7PartBits, m), rb = bc7_field(kBc7RotBits, m);
    const uint32_t sb = bc7_field(kBc7SelBits, m), cb = bc7_field(kBc7ColourBits, m), ab = bc7_field(kBc7AlphaBits, m);
    const uint32_t epb = bc7_field(kBc7EndpointP, m), spb = bc7_field(kBc7SubsetP, m);
    const uint32_t ib = bc7_field(kBc7IndexBits, m), ib2 = bc7_field(kBc7Index2Bits, m);

    // fields in the order of the format: mode, partition, rotation, index selection, R G B A endpoints, p-bits, indices
    const uint32_t p_part = m + 1, p_rot = p_part + pb, p_sel = p_rot + rb, p_col = p_sel + sb;
    const uint32_t part = bc7_bits(w0, w1, w2, w3, p_part, pb), rot = bc7_bits(w0, w1, w2, w3, p_rot, rb);
    const uint32_t sel = bc7_bits(w0, w1, w2, w3, p_sel, sb);
    const uint32_t ne = 2 * ns, p_alpha = p_col + 3 * ne * cb, p_pbits = p_alpha + ne * ab;
    const uint32_t has_p = epb | spb, p_idx = p_pbits + (epb ? ne : spb ? ns : 0u);

    // the partition: subset per texel, anchor texels (one subset: every texel in subset 0, texel 0 the only anchor)
    const uint32_t ti = (part & 63u) + (ns == 3 ? 64u : 0u);
    const uint32_t map = ns == 1 ? 0u : bc7_partition(ti), amask = ns == 1 ? 1u : bc7_anchors(ti);

    // endpoints e = 0 .. 2 ns - 1 (subset s: 2s, 2s+1), expanded to 8 bits and packed RGBA; modes without alpha: A = 255
    uint32_t ep[6];
#pragma unroll
    for (uint32_t e = 0; e < 6; e++) {
        const uint32_t live = e < ne ? 1u : 0u;
        const uint32_t p = bc7_bits(w0, w1, w2, w3, p_pbits + (epb ? e : e >> 1), has_p & live);
        uint32_t v = 0;
#pragma unroll
        for (uint32_t c = 0; c < 3; c++) {
            const uint32_t raw = bc7_bits(w0, w1, w2, w3, p_col + (c * ne + e) * cb, live ? cb : 0u);
            v |= bc7_expand((raw << has_p) | p, cb + has_p) << (8 * c);
        }
        const uint32_t araw = bc7_bits(w0, w1, w2, w3, p_alpha + e * ab, live ? ab : 0u);
        v |= (ab ? bc7_expand((araw << has_p) | p, ab + has_p) : 255u) << 24;
        ep[e] = v;
    }

    // texels: primary index (ib bits, one less at the anchors), secondary index (modes 4, 5: ib2 bits, one less at texel 0)
    const uint32_t p_idx2 = p_idx + 16 * ib - (ns == 1 ? 1u : ns == 2 ? 2u : 3u);
    // colour takes the primary set, alpha the secondary one where there is one; index selection 1 swaps them
    const uint32_t cbits = sel ? ib2 : ib, abits = ib2 ? (sel ? ib : ib2) : ib;
    // rotation: 1 swaps A with R, 2 with G, 3 with B (byte-permute selectors)
    const uint32_t rsel = rot == 0 ? 0x3210u : rot == 1 ? 0x0213u : rot == 2 ? 0x1230u : 0x2310u;
    uint32_t before = 0;   // anchors before texel t
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const uint32_t anchor = (amask >> t) & 1u;
        const uint32_t i1 = bc7_bits(w0, w1, w2, w3, p_idx + t * ib - before, ib - anchor);
        before += anchor;
        const uint32_t i2 = bc7_bits(w0, w1, w2, w3, p_idx2 + t * ib2 - (t ? 1u : 0u), t || !ib2 ? ib2 : ib2 - 1u);
        const uint32_t wc = bc7_weight(sel ? i2 : i1, cbits), wa = bc7_weight(ib2 && !sel ? i2 : i1, abits);
        const uint32_t s = (map >> (2 * t)) & 3u;
        const uint32_t e0 = s == 0 ? ep[0] : s == 1 ? ep[2] : ep[4], e1 = s == 0 ? ep[1] : s == 1 ? ep[3] : ep[5];
        // R and B side by side in 16-bit lanes (each sum < 2^14), then G and A
        const uint32_t rb2 = (((64 - wc) * (e0 & 0x00FF00FFu) + wc * (e1 & 0x00FF00FFu) + 0x00200020u) >> 6) & 0x00FF00FFu;
        const uint32_t g = ((64 - wc) * ((e0 >> 8) & 0xFFu) + wc * ((e1 >> 8) & 0xFFu) + 32u) >> 6;
        const uint32_t a = ((64 - wa) * (e0 >> 24) + wa * (e1 >> 24) + 32u) >> 6;
        const uint32_t px = hap_prmt(rb2 | (g << 8) | (a << 24), 0, rsel);
        out[t] = mode > 7 ? 0u : px;
    }
}

}  // namespace hapb200
