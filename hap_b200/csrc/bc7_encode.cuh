// hap_b200/csrc/bc7_encode.cuh -- K1-K4 family: RGBA8 pictures -> BPTC / BC7 blocks (RGBA UNORM, "Hap R"), the block math
// of bc_encode_kernel<kBcBc7> (bc_encode.cuh).
//
// Error.  Every candidate is scored by its EXACT error: its endpoints are quantised to the mode's bits and p-bits, expanded
// with the decoder's bc7_expand, interpolated with the decoder's bc7_weight and bc7_interp, and every texel takes the index
// whose decoded value is nearest (all 4, 8 or 16 tried).  The error is the sum over R, G, B and A of the squared 8-bit
// differences of decoded and source texels, unweighted.  Rotations (modes 4, 5) swap A with a colour channel in the source
// before the search, which leaves that sum unchanged.
//
// Search.
//   * one subset: mode 6; mode 5 under rotations 0-3; mode 4 under rotations 0-3 and both index selections.  Modes 4 and 5
//     fit colour and alpha apart, each with its own index set;
//   * two subsets: modes 1, 3 and 7 on the kBc7PartitionFits best of the 64 partitions;
//   * three subsets: modes 0 and 2 on the kBc7Partition3Fits best of their 16 and 64 partitions.
//   Partitions are ranked by a pre-score, the sum over their subsets of each subset's squared distance from its principal
//   line (bc7_line_residual; the method of bc6h_line_residual, over four channels).  Each candidate starts from its subsets'
//   bounding boxes (per channel minimum and maximum, the diagonal chosen by covariance signs), is quantised under every p-bit
//   choice of the mode, refitted by least squares on the indices it got (a 2x2 normal system per channel in 64-bit integers)
//   and quantised again under every p-bit choice.  Subsets are independent, so each subset keeps its own best p-bits.
//   * last, the best candidate of each subset count is refitted once more the same way, then gets +-1 nudges of each of its
//     quantised endpoint components, each kept when it lowers the error.
//
// Rules (include/hap_b200.h).  A block of one colour takes mode 5, rotation 0, colour index 1 (weight 21) between two 7-bit
// endpoints per channel from bc7_const_pair (every 8-bit value is reachable so) and both 8-bit alpha endpoints at A: it
// decodes bit-exactly.  In a block whose texels all have A = 255, modes 4-7 keep the endpoints of the channel that decodes to
// A at the top code (in modes 6 and 7 with p-bits 1), so every decoded texel has A = 255; modes 0-3 always decode A = 255.
// Every block has a mode bit, so no reserved block is written.
//
// Packing is the inverse of bc7_decode_block's field order.  At an anchor texel whose index has its top bit set, the subset's
// endpoints (the channels that index drives) are swapped and its indices inverted: the weight tables are symmetric
// (w(2^b - 1 - i) = 64 - w(i)), so the decoded block and its error do not change.
//
// All arithmetic is integer but the pre-score's, which is float written with hap_fma (the library is built -fmad=false), so
// the host build (tests/emu/bc7_encode_twin.cc) is bit-exact with the device.  The search visits modes, partitions, rotations
// and p-bits in one fixed order, so the lanes of a warp walk the same loops.
#pragma once
#include "bc7_decode.cuh"

namespace hapb200 {

// partitions fully fitted per block in the two-subset modes (of 64) and the three-subset modes (of 16 / 64), best
// pre-scores first (DESIGN.md section 1: the quality / time trade-off they were chosen from)
#ifndef HAPB200_BC7_PARTITION_FITS
#define HAPB200_BC7_PARTITION_FITS 8
#endif
#ifndef HAPB200_BC7_PARTITION3_FITS
#define HAPB200_BC7_PARTITION3_FITS 4
#endif
constexpr uint32_t kBc7PartitionFits = HAPB200_BC7_PARTITION_FITS;
constexpr uint32_t kBc7Partition3Fits = HAPB200_BC7_PARTITION3_FITS;

// For an 8-bit value v: two 7-bit codes a | b << 8 with bc7_interp(bc7_expand(a, 7), bc7_expand(b, 7), 21) == v, the mode-5
// colour at index 1.  The first match of a in {v / 2, v / 2 - 1}, b in {a, a + 1, a - 1} exists for every v (checked by
// enumeration, and by the constant-block tests for all 256 values).
HAP_HD uint32_t bc7_const_pair(uint32_t v)
{
    uint32_t pair = 0;
    bool found = false;
#pragma unroll
    for (int32_t k = 0; k < 6; k++) {
        const int32_t a = (int32_t)(v >> 1) - (k / 3), b = a + (k % 3 == 0 ? 0 : k % 3 == 1 ? 1 : -1);
        const bool ok = !found && a >= 0 && b >= 0 && b < 128 &&
                        bc7_interp(bc7_expand((uint32_t)a, 7), bc7_expand((uint32_t)b, 7), 21) == v;
        pair = ok ? (uint32_t)a | ((uint32_t)b << 8) : pair;
        found = found || ok;
    }
    return pair;
}

// byte c of a packed RGBA texel
HAP_HD uint32_t bc7_ch(uint32_t p, uint32_t c) { return (p >> (8 * c)) & 0xFFu; }

// the byte-permute selector of rotation r (1 swaps A with R, 2 with G, 3 with B; its own inverse), as bc7_decode_block's
HAP_HD uint32_t bc7_rot_sel(uint32_t r) { return r == 0 ? 0x3210u : r == 1 ? 0x0213u : r == 2 ? 0x1230u : 0x2310u; }

// the stored channel that decodes to A under rotation r
HAP_HD uint32_t bc7_alpha_slot(uint32_t r) { return r == 0 ? 3u : r - 1u; }

// A candidate: mode, partition (0-63), rotation, index selection, the raw endpoint codes of endpoint e (subset e / 2) as
// R | G << 8 | B << 16 | A << 24 in the mode's bits, p-bit of endpoint e in bit e, the indices of texel t in bits 4t.. of i1
// (the primary set) and i2 (the secondary set of modes 4 and 5), as the search found them (anchors not yet satisfied), and
// the error of the whole block.
struct Bc7Pick {
    uint32_t err;
    uint32_t mode, part, rot, sel, pbits;
    uint32_t ep[6];
    uint64_t i1, i2;
};

// the subset map of a candidate, 2 bits per texel (one subset: all 0)
HAP_HD uint32_t bc7_map(uint32_t ns, uint32_t part) { return ns == 1 ? 0u : bc7_partition((part & 63u) + (ns == 3 ? 64u : 0u)); }

// texel mask of subset s of a map
HAP_HD uint32_t bc7_subset_mask(uint32_t map, uint32_t s)
{
    uint32_t in = 0;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) in |= (((map >> (2 * t)) & 3u) == s ? 1u : 0u) << t;
    return in;
}

// a texel mask with 4 bits per texel
HAP_HD uint64_t bc7_nibbles(uint32_t in)
{
    uint64_t m = 0;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) m |= ((in >> t) & 1u) ? 15ull << (4 * t) : 0ull;
    return m;
}

// raw codes of one endpoint (mode m, p-bit p) -> RGBA8 as the decoder expands them; modes without alpha: A = 255
HAP_HD uint32_t bc7_unquantize(uint32_t raw, uint32_t p, uint32_t m)
{
    const uint32_t cb = bc7_field(kBc7ColourBits, m), ab = bc7_field(kBc7AlphaBits, m);
    const uint32_t has_p = bc7_field(kBc7EndpointP, m) | bc7_field(kBc7SubsetP, m);
    uint32_t v = 0;
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) v |= bc7_expand((bc7_ch(raw, c) << has_p) | p, cb + has_p) << (8 * c);
    v |= (ab ? bc7_expand((bc7_ch(raw, 3) << has_p) | p, ab + has_p) : 255u) << 24;
    return v;
}

// an 8-bit value -> the n-bit code (with p-bit p below it when has_p) whose expansion is nearest (ties: the lower)
HAP_HD uint32_t bc7_quantize(int32_t v, uint32_t n, uint32_t has_p, uint32_t p)
{
    const uint32_t tb = n + has_p, top = (1u << n) - 1u;
    const int32_t u = v < 0 ? 0 : v > 255 ? 255 : v;
    const int32_t r = (int32_t)((((uint32_t)u * ((1u << tb) - 1u) + 127u) / 255u) >> has_p);
    uint32_t best = 0, bd = ~0u;
#pragma unroll
    for (int32_t d = -1; d <= 1; d++) {
        const int32_t c = r + d;
        const uint32_t q = c < 0 ? 0u : (uint32_t)c > top ? top : (uint32_t)c;
        const int32_t e = (int32_t)bc7_expand((q << has_p) | p, tb) - u;
        const uint32_t ad = (uint32_t)(e < 0 ? -e : e);
        best = ad < bd ? q : best;
        bd = ad < bd ? ad : bd;
    }
    return best;
}

// Endpoint fits are held as ends[8 s + 4 j + c]: channel c of endpoint j of subset s, 8-bit domain.
// Endpoints of the texels of `in` from their bounding box over the channels of cmask: per channel the minimum and the
// maximum, in the order of the channel of widest range or the reverse, as the channel's covariance with it has the sign
HAP_HD void bc7_bbox(const uint32_t x[16], uint32_t in, uint32_t cmask, int32_t e[8])
{
    int32_t lo[4] = {255, 255, 255, 255}, hi[4] = {0, 0, 0, 0};
    int32_t s[4] = {0, 0, 0, 0}, n = 0;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool on = ((in >> t) & 1u) != 0;
        n += on ? 1 : 0;
#pragma unroll
        for (uint32_t c = 0; c < 4; c++) {
            const int32_t v = (int32_t)bc7_ch(x[t], c);
            lo[c] = on && v < lo[c] ? v : lo[c];
            hi[c] = on && v > hi[c] ? v : hi[c];
            s[c] += on ? v : 0;
        }
    }
    uint32_t p = 0;
    int32_t wide = -1;
#pragma unroll
    for (uint32_t c = 0; c < 4; c++) {
        const bool live = ((cmask >> c) & 1u) != 0 && hi[c] - lo[c] > wide;
        p = live ? c : p;
        wide = live ? hi[c] - lo[c] : wide;
    }
    int32_t cov[4] = {0, 0, 0, 0};
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool on = ((in >> t) & 1u) != 0;
        const int32_t vp = n * (int32_t)bc7_ch(x[t], p) - s[p];
#pragma unroll
        for (uint32_t c = 0; c < 4; c++) cov[c] += on ? vp * (n * (int32_t)bc7_ch(x[t], c) - s[c]) : 0;   // |sum| < 2^29
    }
#pragma unroll
    for (uint32_t c = 0; c < 4; c++) {
        const bool live = ((cmask >> c) & 1u) != 0;
        e[c] = live ? (cov[c] < 0 ? hi[c] : lo[c]) : e[c];
        e[4 + c] = live ? (cov[c] < 0 ? lo[c] : hi[c]) : e[4 + c];
    }
}

// n / d rounded to nearest, halves away from zero (d > 0)
HAP_HD int64_t bc7_div_round(int64_t n, int64_t d) { return n >= 0 ? (n + d / 2) / d : -((-n + d / 2) / d); }

// Least-squares endpoints of the texels of `in` over the channels of cmask, with their indices (idx, b-bit) held: a and b
// minimise sum ((64 - w) a + w b - 64 x)^2.  e is left alone when every texel has the same weight.
HAP_HD void bc7_refit(const uint32_t x[16], uint32_t in, uint64_t idx, uint32_t b, uint32_t cmask, int32_t e[8])
{
    int64_t aa = 0, ab = 0, bb = 0, ax[4] = {0, 0, 0, 0}, bx[4] = {0, 0, 0, 0};
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool on = ((in >> t) & 1u) != 0;
        const int64_t w = on ? (int64_t)bc7_weight((uint32_t)(idx >> (4 * t)) & 15u, b) : 0, v = on ? 64 - w : 0;
        aa += v * v;
        ab += v * w;
        bb += w * w;
#pragma unroll
        for (uint32_t c = 0; c < 4; c++) {
            const int64_t xv = (int64_t)bc7_ch(x[t], c);
            ax[c] += v * xv;
            bx[c] += w * xv;
        }
    }
    const int64_t det = aa * bb - ab * ab, den = det > 0 ? det : 1;
#pragma unroll
    for (uint32_t c = 0; c < 4; c++) {
        int64_t a = bc7_div_round(64 * (bb * ax[c] - ab * bx[c]), den), bv = bc7_div_round(64 * (aa * bx[c] - ab * ax[c]), den);
        a = a < 0 ? 0 : a > 255 ? 255 : a;
        bv = bv < 0 ? 0 : bv > 255 ? 255 : bv;
        const bool live = det > 0 && ((cmask >> c) & 1u) != 0;
        e[c] = live ? (int32_t)a : e[c];
        e[4 + c] = live ? (int32_t)bv : e[4 + c];
    }
}

// The exact error of endpoints ep (expanded RGBA8, endpoint e of subset e / 2) on the (rotated) texels x of a mode-m block
// with subset map `map` and index selection sel: every texel takes its nearest index (ties: the lowest).  Returns the
// indices (i1, i2 as in Bc7Pick) and the error of each subset in serr.
HAP_HD void bc7_score(uint32_t m, uint32_t map, uint32_t sel, const uint32_t ep[6], const uint32_t x[16], uint64_t &i1,
                      uint64_t &i2, uint32_t serr[3])
{
    const uint32_t ib = bc7_field(kBc7IndexBits, m), ib2 = bc7_field(kBc7Index2Bits, m);
    const uint32_t cbits = sel ? ib2 : ib, abits = ib2 ? (sel ? ib : ib2) : ib;
    const uint32_t cn = ib2 ? 1u << cbits : 1u << ib, an = ib2 ? 1u << abits : 0u, cch = ib2 ? 3u : 4u;
    serr[0] = serr[1] = serr[2] = 0;
    i1 = i2 = 0;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const uint32_t s = (map >> (2 * t)) & 3u;
        const uint32_t e0 = s == 0 ? ep[0] : s == 1 ? ep[2] : ep[4], e1 = s == 0 ? ep[1] : s == 1 ? ep[3] : ep[5];
        uint32_t bc = ~0u, ci = 0, ba = ib2 ? ~0u : 0u, ai = 0;
#pragma unroll 1
        for (uint32_t i = 0; i < cn; i++) {
            const uint32_t w = bc7_weight(i, ib2 ? cbits : ib);
            uint32_t d2 = 0;
#pragma unroll
            for (uint32_t c = 0; c < 4; c++) {
                const int32_t d = (int32_t)bc7_interp(bc7_ch(e0, c), bc7_ch(e1, c), w) - (int32_t)bc7_ch(x[t], c);
                d2 += c < cch ? (uint32_t)(d * d) : 0u;
            }
            ci = d2 < bc ? i : ci;
            bc = d2 < bc ? d2 : bc;
        }
#pragma unroll 1
        for (uint32_t i = 0; i < an; i++) {
            const int32_t d = (int32_t)bc7_interp(e0 >> 24, e1 >> 24, bc7_weight(i, abits)) - (int32_t)(x[t] >> 24);
            const uint32_t d2 = (uint32_t)(d * d);
            ai = d2 < ba ? i : ai;
            ba = d2 < ba ? d2 : ba;
        }
        const uint32_t e = bc + ba;
        serr[0] += s == 0 ? e : 0u;
        serr[1] += s == 1 ? e : 0u;
        serr[2] += s == 2 ? e : 0u;
        i1 |= (uint64_t)(ib2 && sel ? ai : ci) << (4 * t);
        i2 |= (uint64_t)(ib2 ? (sel ? ci : ai) : 0u) << (4 * t);
    }
}

// The fits `ends` quantised to mode m under every p-bit choice and scored; each subset of `cur` takes the choice that lowers
// its error (cur.err: the sum of serr).  opaque: the channel that decodes to A stays at the top code (p-bits 1 in modes 6, 7).
HAP_HD void bc7_quantize_all(const Bc7Pick &shape, const int32_t ends[24], const uint32_t x[16], bool opaque, const uint64_t nib[3],
                             Bc7Pick &cur, uint32_t serr[3])
{
    const uint32_t m = shape.mode, ns = bc7_field(kBc7Subsets, m), cb = bc7_field(kBc7ColourBits, m), ab = bc7_field(kBc7AlphaBits, m);
    const uint32_t epb = bc7_field(kBc7EndpointP, m), spb = bc7_field(kBc7SubsetP, m), has_p = epb | spb;
    const uint32_t map = bc7_map(ns, shape.part), aslot = bc7_alpha_slot(shape.rot);
    const bool pin = opaque && m >= 4, pin_p = opaque && m >= 6;
    const uint32_t choices = pin_p ? 1u : epb ? 4u : spb ? 2u : 1u;
#pragma unroll 1
    for (uint32_t k = 0; k < choices; k++) {
        uint32_t raw[6], ex[6], pbits = 0;
#pragma unroll
        for (uint32_t e = 0; e < 6; e++) {
            const uint32_t p = pin_p ? 1u : epb ? (k >> (e & 1u)) & 1u : spb ? k & 1u : 0u;
            uint32_t r = 0;
#pragma unroll
            for (uint32_t c = 0; c < 4; c++) {
                const uint32_t n = c < 3 ? cb : ab;
                uint32_t q = n ? bc7_quantize(ends[4 * e + c], n, has_p, p) : 0u;
                q = pin && c == aslot ? (1u << n) - 1u : q;
                r |= q << (8 * c);
            }
            raw[e] = r;
            ex[e] = bc7_unquantize(r, p, m);
            pbits |= (e < 2 * ns ? p : 0u) << e;
        }
        uint64_t i1, i2;
        uint32_t se[3];
        bc7_score(m, map, shape.sel, ex, x, i1, i2, se);
#pragma unroll
        for (uint32_t s = 0; s < 3; s++) {
            const bool take = s < ns && se[s] < serr[s];
            serr[s] = take ? se[s] : serr[s];
            cur.ep[2 * s] = take ? raw[2 * s] : cur.ep[2 * s];
            cur.ep[2 * s + 1] = take ? raw[2 * s + 1] : cur.ep[2 * s + 1];
            const uint32_t pm = 3u << (2 * s);
            cur.pbits = take ? (cur.pbits & ~pm) | (pbits & pm) : cur.pbits;
            cur.i1 = take ? (cur.i1 & ~nib[s]) | (i1 & nib[s]) : cur.i1;
            cur.i2 = take ? (cur.i2 & ~nib[s]) | (i2 & nib[s]) : cur.i2;
        }
    }
    cur.err = serr[0] + serr[1] + serr[2];
}

// least-squares fits of every subset of a candidate on its indices (modes 4, 5: colour and alpha apart, each on its set)
HAP_HD void bc7_refit_pick(const Bc7Pick &p, const uint32_t x[16], int32_t ends[24])
{
    const uint32_t m = p.mode, ns = bc7_field(kBc7Subsets, m), ib = bc7_field(kBc7IndexBits, m), ib2 = bc7_field(kBc7Index2Bits, m);
    const uint32_t map = bc7_map(ns, p.part);
#pragma unroll
    for (uint32_t s = 0; s < 3; s++) {
        const uint32_t in = s < ns ? bc7_subset_mask(map, s) : 0u;
        if (ib2) {
            bc7_refit(x, in, p.sel ? p.i2 : p.i1, p.sel ? ib2 : ib, 0x7u, ends + 8 * s);
            bc7_refit(x, in, p.sel ? p.i1 : p.i2, p.sel ? ib : ib2, 0x8u, ends + 8 * s);
        } else {
            bc7_refit(x, in, p.i1, ib, 0xFu, ends + 8 * s);
        }
    }
}

// One candidate shape (mode, partition, rotation, index selection) from the fits `ends`: quantised under every p-bit choice,
// refitted on the indices it got and quantised again; kept in `best` when its error is lower
HAP_HD void bc7_fit(const Bc7Pick &shape, int32_t ends[24], const uint32_t x[16], bool opaque, Bc7Pick &best)
{
    const uint32_t ns = bc7_field(kBc7Subsets, shape.mode), map = bc7_map(ns, shape.part);
    uint64_t nib[3];
#pragma unroll
    for (uint32_t s = 0; s < 3; s++) nib[s] = s < ns ? bc7_nibbles(bc7_subset_mask(map, s)) : 0ull;
    Bc7Pick cur = shape;
    uint32_t serr[3] = {~0u, ~0u, ~0u};
    serr[1] = ns > 1 ? ~0u : 0u;
    serr[2] = ns > 2 ? ~0u : 0u;
    bc7_quantize_all(shape, ends, x, opaque, nib, cur, serr);
    bc7_refit_pick(cur, x, ends);
    bc7_quantize_all(shape, ends, x, opaque, nib, cur, serr);
    const bool take = cur.err < best.err;
    best = take ? cur : best;
}

// the bounding-box fits of every subset of mode m on partition part (modes 4, 5: colour and alpha apart)
HAP_HD void bc7_bbox_all(uint32_t m, uint32_t part, const uint32_t x[16], int32_t ends[24])
{
    const uint32_t ns = bc7_field(kBc7Subsets, m), map = bc7_map(ns, part);
    const bool apart = bc7_field(kBc7Index2Bits, m) != 0;
#pragma unroll
    for (uint32_t k = 0; k < 24; k++) ends[k] = 0;
#pragma unroll
    for (uint32_t s = 0; s < 3; s++) {
        const uint32_t in = s < ns ? bc7_subset_mask(map, s) : 0u;
        bc7_bbox(x, in, apart ? 0x7u : 0xFu, ends + 8 * s);
        if (apart) bc7_bbox(x, in, 0x8u, ends + 8 * s);
    }
}

// bc7_fit of a shape from its subsets' bounding boxes
HAP_HD void bc7_try(uint32_t m, uint32_t part, uint32_t rot, uint32_t sel, const uint32_t x[16], bool opaque, Bc7Pick &best)
{
    int32_t ends[24];
    bc7_bbox_all(m, part, x, ends);
    Bc7Pick shape = best;
    shape.mode = m;
    shape.part = part;
    shape.rot = rot;
    shape.sel = sel;
    bc7_fit(shape, ends, x, opaque, best);
}

// +-1 nudges of each quantised endpoint component of a pick, each kept when it lowers the error (pinned channels of opaque
// blocks stay)
HAP_HD void bc7_nudge(const uint32_t x[16], bool opaque, Bc7Pick &p)
{
    const uint32_t m = p.mode, ns = bc7_field(kBc7Subsets, m), cb = bc7_field(kBc7ColourBits, m), ab = bc7_field(kBc7AlphaBits, m);
    const uint32_t map = bc7_map(ns, p.part), aslot = bc7_alpha_slot(p.rot);
#pragma unroll 1
    for (uint32_t k = 0; k < 2 * 4 * 2 * ns; k++) {
        const uint32_t e = k >> 3, c = (k >> 1) & 3u, n = c < 3 ? cb : ab;
        if (n == 0 || (opaque && m >= 4 && c == aslot)) continue;
        const int32_t v = (int32_t)bc7_ch(p.ep[e], c) + ((k & 1u) ? 1 : -1);
        if (v < 0 || v > (int32_t)((1u << n) - 1u)) continue;
        uint32_t raw[6], ex[6];
#pragma unroll
        for (uint32_t j = 0; j < 6; j++) {
            raw[j] = j == e ? (p.ep[j] & ~(0xFFu << (8 * c))) | ((uint32_t)v << (8 * c)) : p.ep[j];
            ex[j] = bc7_unquantize(raw[j], (p.pbits >> j) & 1u, m);
        }
        uint64_t i1, i2;
        uint32_t se[3];
        bc7_score(m, map, p.sel, ex, x, i1, i2, se);
        const uint32_t err = se[0] + se[1] + se[2];
        const bool take = err < p.err;
        p.err = take ? err : p.err;
        p.i1 = take ? i1 : p.i1;
        p.i2 = take ? i2 : p.i2;
#pragma unroll
        for (uint32_t j = 0; j < 6; j++) p.ep[j] = take ? raw[j] : p.ep[j];
    }
}

// The partition pre-score of one subset (the texels of `in`): its squared distance from the line through its mean along its
// principal axis, the trace of its scatter matrix less the largest eigenvalue, the eigenvalue estimated by two steps of power
// iteration from the column of the widest channel (as bc6h_line_residual, over R, G, B and A).  Exact integer moments, then
// float (hap_fma).
HAP_HD float bc7_line_residual(const uint32_t x[16], uint32_t in)
{
    int32_t n = 0, s[4] = {0, 0, 0, 0}, ss[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};   // ss: 00 11 22 33 01 02 03 12 13 23
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool on = ((in >> t) & 1u) != 0;
        const int32_t r = on ? (int32_t)bc7_ch(x[t], 0) : 0, g = on ? (int32_t)bc7_ch(x[t], 1) : 0;
        const int32_t b = on ? (int32_t)bc7_ch(x[t], 2) : 0, a = on ? (int32_t)bc7_ch(x[t], 3) : 0;
        n += on ? 1 : 0;
        s[0] += r; s[1] += g; s[2] += b; s[3] += a;
        ss[0] += r * r; ss[1] += g * g; ss[2] += b * b; ss[3] += a * a;
        ss[4] += r * g; ss[5] += r * b; ss[6] += r * a; ss[7] += g * b; ss[8] += g * a; ss[9] += b * a;
    }
    // n^2 x the covariance (each term < 2^31: n <= 16, values < 256)
    float c[4][4];
    const uint32_t pi[10] = {0, 1, 2, 3, 0, 0, 0, 1, 1, 2}, pj[10] = {0, 1, 2, 3, 1, 2, 3, 2, 3, 3};
#pragma unroll
    for (uint32_t k = 0; k < 10; k++) {
        const float v = (float)(n * ss[k] - s[pi[k]] * s[pj[k]]);
        c[pi[k]][pj[k]] = v;
        c[pj[k]][pi[k]] = v;
    }
    float v[4], widest = c[0][0];
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) v[k] = c[0][k];
#pragma unroll
    for (uint32_t r = 1; r < 4; r++) {
        const bool w = c[r][r] > widest;
        widest = w ? c[r][r] : widest;
#pragma unroll
        for (uint32_t k = 0; k < 4; k++) v[k] = w ? c[r][k] : v[k];
    }
    float a[4];
#pragma unroll
    for (int it = 0; it < 3; it++) {
        const float mx = fmaxf(hap_fmax3(fabsf(v[0]), fabsf(v[1]), fabsf(v[2])), fabsf(v[3]));
        const float k = mx > 0.0f ? 1.0f / mx : 0.0f;
#pragma unroll
        for (uint32_t r = 0; r < 4; r++) a[r] = v[r] * k;
#pragma unroll
        for (uint32_t r = 0; r < 4; r++) v[r] = hap_fma(c[r][0], a[0], hap_fma(c[r][1], a[1], hap_fma(c[r][2], a[2], c[r][3] * a[3])));
    }
    // after two steps a is the axis and v = C a: the Rayleigh quotient
    const float vv = hap_fma(a[0], a[0], hap_fma(a[1], a[1], hap_fma(a[2], a[2], a[3] * a[3])));
    const float lambda = vv > 0.0f ? hap_fma(a[0], v[0], hap_fma(a[1], v[1], hap_fma(a[2], v[2], a[3] * v[3]))) / vv : 0.0f;
    return (c[0][0] + c[1][1] + c[2][2] + c[3][3] - lambda) / (float)(n > 0 ? n * n : 1);
}

// keep (score, part) among the K lowest of top_score / top_part (ascending)
template <uint32_t K>
HAP_HD void bc7_rank(float score, uint32_t part, float top_score[K], uint32_t top_part[K])
{
#pragma unroll
    for (uint32_t k = 0; k < K; k++) {
        const bool lower = score < top_score[k];
        const float ts = top_score[k];
        const uint32_t tp = top_part[k];
        top_score[k] = lower ? score : ts;
        top_part[k] = lower ? part : tp;
        score = lower ? ts : score;
        part = lower ? tp : part;
    }
}

// n bits of v into the block (w[0] = bits 0..31, ... w[3] = bits 96..127) from bit pos on (pos + n <= 128, n <= 16)
HAP_HD void bc7_put(uint32_t w[4], uint32_t pos, uint32_t n, uint32_t v)
{
    const uint64_t s = (uint64_t)(v & ((1u << n) - 1u)) << (pos & 31u);
    const uint32_t k = pos >> 5;
#pragma unroll
    for (uint32_t j = 0; j < 4; j++) w[j] |= j == k ? (uint32_t)s : j == k + 1u ? (uint32_t)(s >> 32) : 0u;
}

// A pick -> its 128 bits, fields in bc7_decode_block's order.  An index set whose anchor texel has its top bit set gets its
// subset's endpoints swapped (the channels that set drives, and the p-bits with them) and the subset's indices inverted.
HAP_HD void bc7_pack(Bc7Pick p, uint32_t out[4])
{
    const uint32_t m = p.mode, ns = bc7_field(kBc7Subsets, m), pb = bc7_field(kBc7PartBits, m), rb = bc7_field(kBc7RotBits, m);
    const uint32_t sb = bc7_field(kBc7SelBits, m), cb = bc7_field(kBc7ColourBits, m), ab = bc7_field(kBc7AlphaBits, m);
    const uint32_t epb = bc7_field(kBc7EndpointP, m), spb = bc7_field(kBc7SubsetP, m);
    const uint32_t ib = bc7_field(kBc7IndexBits, m), ib2 = bc7_field(kBc7Index2Bits, m);
    const uint32_t ti = (p.part & 63u) + (ns == 3 ? 64u : 0u);
    const uint32_t map = bc7_map(ns, p.part), amask = ns == 1 ? 1u : bc7_anchors(ti);
    // channels the primary set drives (modes 4, 5: colour, or alpha under index selection 1), and the secondary set
    const uint32_t c1 = ib2 ? (p.sel ? 0xFF000000u : 0x00FFFFFFu) : 0xFFFFFFFFu, c2 = ~c1;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        if (!((amask >> t) & 1u)) continue;
        const uint32_t s = (map >> (2 * t)) & 3u;
        if ((((uint32_t)(p.i1 >> (4 * t)) & 15u) >> (ib - 1u)) == 0) continue;
        const uint32_t a = p.ep[2 * s], b = p.ep[2 * s + 1];
        p.ep[2 * s] = (a & ~c1) | (b & c1);
        p.ep[2 * s + 1] = (b & ~c1) | (a & c1);
        const uint32_t pa = (p.pbits >> (2 * s)) & 1u, pbb = (p.pbits >> (2 * s + 1)) & 1u;
        p.pbits = (p.pbits & ~(3u << (2 * s))) | (pbb << (2 * s)) | (pa << (2 * s + 1));
        const uint64_t nib = bc7_nibbles(bc7_subset_mask(map, s)), top = (1ull << ib) - 1u;
#pragma unroll
        for (uint32_t u = 0; u < 16; u++)
            if ((nib >> (4 * u)) & 1u) p.i1 = (p.i1 & ~(15ull << (4 * u))) | ((top - ((p.i1 >> (4 * u)) & 15u)) << (4 * u));
    }
    if (ib2 && ((p.i2 & 15u) >> (ib2 - 1u))) {
        const uint32_t a = p.ep[0], b = p.ep[1];
        p.ep[0] = (a & ~c2) | (b & c2);
        p.ep[1] = (b & ~c2) | (a & c2);
        const uint64_t top = (1ull << ib2) - 1u;
#pragma unroll
        for (uint32_t u = 0; u < 16; u++) p.i2 = (p.i2 & ~(15ull << (4 * u))) | ((top - ((p.i2 >> (4 * u)) & 15u)) << (4 * u));
    }
    uint32_t w[4] = {1u << m, 0u, 0u, 0u};
    uint32_t pos = m + 1;
    bc7_put(w, pos, pb, p.part);
    pos += pb;
    bc7_put(w, pos, rb, p.rot);
    pos += rb;
    bc7_put(w, pos, sb, p.sel);
    pos += sb;
    const uint32_t ne = 2 * ns;
#pragma unroll 1
    for (uint32_t c = 0; c < 4; c++) {
        const uint32_t n = c < 3 ? cb : ab;
#pragma unroll 1
        for (uint32_t e = 0; e < ne; e++) {
            bc7_put(w, pos, n, bc7_ch(p.ep[e], c));
            pos += n;
        }
    }
#pragma unroll 1
    for (uint32_t e = 0; e < ne; e++) {
        const uint32_t live = epb ? 1u : spb && !(e & 1u) ? 1u : 0u;
        bc7_put(w, pos, live, (p.pbits >> e) & 1u);
        pos += live;
    }
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const uint32_t nb = ib - ((amask >> t) & 1u);
        bc7_put(w, pos, nb, (uint32_t)(p.i1 >> (4 * t)) & 15u);
        pos += nb;
    }
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const uint32_t nb = ib2 ? ib2 - (t == 0 ? 1u : 0u) : 0u;
        bc7_put(w, pos, nb, (uint32_t)(p.i2 >> (4 * t)) & 15u);
        pos += nb;
    }
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) out[k] = w[k];
}

// One block: texel t in px[t] (RGBA8, R in the low byte) -> 16 bytes of BC7 in out[0..3].  Returns the error the block was
// chosen by (the sum over the texels and R, G, B, A of the squared difference of decoded and source values).
HAP_HD uint32_t bc7_encode_block(const uint32_t px[16], uint32_t out[4])
{
    bool flat = true, opaque = true;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        flat = flat && px[t] == px[0];
        opaque = opaque && (px[t] >> 24) == 255u;
    }
    Bc7Pick best;
    best.err = ~0u;
    best.mode = 5u;
    best.part = best.rot = best.sel = best.pbits = 0u;
    best.i1 = best.i2 = 0ull;
#pragma unroll
    for (uint32_t e = 0; e < 6; e++) best.ep[e] = 0u;

    if (flat) {
        // mode 5, rotation 0: colour index 1 between the pair of bc7_const_pair, alpha endpoints both A (index 0)
        uint32_t a = 0, b = 0;
#pragma unroll
        for (uint32_t c = 0; c < 3; c++) {
            const uint32_t q = bc7_const_pair(bc7_ch(px[0], c));
            a |= (q & 0xFFu) << (8 * c);
            b |= (q >> 8) << (8 * c);
        }
        best.ep[0] = a | (px[0] & 0xFF000000u);
        best.ep[1] = b | (px[0] & 0xFF000000u);
        best.i1 = 0x1111111111111111ull;
        best.err = 0;
        bc7_pack(best, out);
        return 0;
    }

    Bc7Pick pick[3];
    pick[0] = pick[1] = pick[2] = best;
    pick[1].mode = 1u;
    pick[2].mode = 2u;

    // one subset: mode 6; modes 4 (both index selections) and 5 under every rotation
    uint32_t xr[16];
    bc7_try(6, 0, 0, 0, px, opaque, pick[0]);
#pragma unroll 1
    for (uint32_t rot = 0; rot < 4; rot++) {
        const uint32_t rs = bc7_rot_sel(rot);
#pragma unroll
        for (uint32_t t = 0; t < 16; t++) xr[t] = hap_prmt(px[t], 0, rs);
        bc7_try(5, 0, rot, 0, xr, opaque, pick[0]);
        bc7_try(4, 0, rot, 0, xr, opaque, pick[0]);
        bc7_try(4, 0, rot, 1, xr, opaque, pick[0]);
    }

    // two subsets: the partitions whose subsets lie closest to one line each
    float top2[kBc7PartitionFits], top3a[kBc7Partition3Fits], top3b[kBc7Partition3Fits];
    uint32_t part2[kBc7PartitionFits], part3a[kBc7Partition3Fits], part3b[kBc7Partition3Fits];
#pragma unroll
    for (uint32_t k = 0; k < kBc7PartitionFits; k++) { top2[k] = 3.0e38f; part2[k] = 0; }
#pragma unroll
    for (uint32_t k = 0; k < kBc7Partition3Fits; k++) { top3a[k] = top3b[k] = 3.0e38f; part3a[k] = part3b[k] = 0; }
#pragma unroll 1
    for (uint32_t part = 0; part < 64; part++) {
        const uint32_t map2 = bc7_partition(part), map3 = bc7_partition(64 + part);
        const float s2 = bc7_line_residual(px, bc7_subset_mask(map2, 0)) + bc7_line_residual(px, bc7_subset_mask(map2, 1));
        bc7_rank<kBc7PartitionFits>(s2, part, top2, part2);
        const float s3 = bc7_line_residual(px, bc7_subset_mask(map3, 0)) + bc7_line_residual(px, bc7_subset_mask(map3, 1)) +
                         bc7_line_residual(px, bc7_subset_mask(map3, 2));
        if (part < 16) bc7_rank<kBc7Partition3Fits>(s3, part, top3a, part3a);
        bc7_rank<kBc7Partition3Fits>(s3, part, top3b, part3b);
    }
#pragma unroll 1
    for (uint32_t k = 0; k < kBc7PartitionFits; k++) {
        bc7_try(1, part2[k], 0, 0, px, opaque, pick[1]);
        bc7_try(3, part2[k], 0, 0, px, opaque, pick[1]);
        bc7_try(7, part2[k], 0, 0, px, opaque, pick[1]);
    }
    // three subsets: mode 0 (partitions 0-15) and mode 2
#pragma unroll 1
    for (uint32_t k = 0; k < kBc7Partition3Fits; k++) {
        bc7_try(0, part3a[k], 0, 0, px, opaque, pick[2]);
        bc7_try(2, part3b[k], 0, 0, px, opaque, pick[2]);
    }

    // the best of each subset count: refitted once more, then nudged
#pragma unroll 1
    for (uint32_t n = 0; n < 3; n++) {
        Bc7Pick p = pick[n];
        const uint32_t rs = bc7_rot_sel(p.rot);
#pragma unroll
        for (uint32_t t = 0; t < 16; t++) xr[t] = hap_prmt(px[t], 0, rs);
        int32_t ends[24];
        bc7_bbox_all(p.mode, p.part, xr, ends);
        bc7_refit_pick(p, xr, ends);
        bc7_fit(p, ends, xr, opaque, p);
        bc7_nudge(xr, opaque, p);
        const bool take = p.err < best.err;
        best = take ? p : best;
    }
    bc7_pack(best, out);
    return best.err;
}

}  // namespace hapb200
