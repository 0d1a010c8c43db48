// hap_b200/csrc/bc6h_encode.cuh -- K1-K4 family: RGBA16F (or HDR10 P010) pictures -> BPTC / BC6H blocks (UF16 or SF16,
// "Hap HDR"), bc6h_encode_kernel.
//
// Shape as the other block encoders (bc_encode.cuh): one thread per 4x4 block, kBcThreads per CTA, frames on blockIdx.y in
// slices of kBcFramesPerLaunch.  A block row of RGBA16F is 32 bytes, read as two 128-bit loads, so a warp reads 1 KiB
// contiguous per pixel row; the block is written with one 16-byte store.  A is ignored.
//
// Input rules (include/hap_b200.h): UF16 takes negative values, -0 and NaN as 0 and +Inf as 65504 (0x7BFF); SF16 takes NaN
// as 0, +-Inf as +-65504 and -0 as +0.  Each value is then held as the sign-magnitude integer of its half (UF16: 0 .. 0x7BFF;
// SF16: -0x7BFF .. 0x7BFF), the domain in which BC6H interpolates.
//
// Search.  Every candidate is scored by its TRUE error: its endpoints are quantised to the mode's precision, unquantised and
// interpolated with the decoder's own functions (bc6h_unquantize, the (a (64 - w) + b w + 32) >> 6 interpolation and
// bc6h_finish of bc6h_decode.cuh), every texel takes the index whose decoded value is nearest (all 8 or 16 tried), and the
// error is the sum over R, G and B of the squared differences of decoded and source sign-magnitude integers.  Candidates:
//   * one region, modes 11-14, endpoints from the block's bounding box (per channel min / max, the diagonal picked by the
//     sign of each channel's covariance with the channel of widest range);
//   * two regions, modes 1-10, on the kBc6hPartitionFits partitions of 32 whose regions lie closest to one line each (the
//     pre-score, bc6h_line_residual), endpoints from each region's bounding box;
//   * every candidate once more with least-squares endpoints for the indices it got, in the integer domain with the
//     indices held (a 2x2 normal system per channel, 64-bit integers);
//   * then, twice, the best one-region and the best two-region candidate refitted so and tried again in every mode of that
//     region count, and last +-1 nudges of each of their quantised endpoint components.
// In the transformed modes a candidate whose deltas do not fit their bits after the wrap to the base's precision is
// skipped.  Mode 11 (untransformed) always fits, so a block is never left without a mode and no reserved mode is written.
// A constant block decodes bit-exactly: its endpoint is the smallest interpolated value that bc6h_finish maps to the colour,
// and mode 14 (16-bit base, zero deltas) holds it.
//
// All arithmetic is integer but the pre-score's, which is float written with hap_fma (the library is built -fmad=false),
// so the host build (tests/emu) is bit-exact with the device.  Every lane runs one instruction
// stream whatever its block ends in: fixed trip counts, mode parameters from the decoder's kBc6hLayout rows, and packing
// through those rows' pieces (the inverse of the decoder's piece reader), with partitions and anchors from bc7_partition and
// bc7_anchors, so the encoder and the decoder cannot disagree on a layout.
#pragma once
#include "bc6h_decode.cuh"
#include "bc_encode.cuh"

namespace hapb200 {

// partitions of 32 fully fitted in the two-region modes, best pre-scores first (DESIGN.md section 1: the quality / time
// trade-off this was chosen from)
#ifndef HAPB200_BC6H_PARTITION_FITS
#define HAPB200_BC6H_PARTITION_FITS 8
#endif
constexpr uint32_t kBc6hPartitionFits = HAPB200_BC6H_PARTITION_FITS;

// the mode value in the low bits of a block of mode m (0-based): 2 bits for modes 0, 1, else 5 bits xxx10 / 0xx11
HAP_HD constexpr uint32_t bc6h_mode_value(uint32_t m) { return m < 2 ? m : m < 10 ? 2u + 4u * (m - 2u) : 3u + 4u * (m - 10u); }

// a half of the input -> its sign-magnitude integer after the input rules
HAP_HD int32_t bc6h_source(uint32_t h, bool sgn)
{
    const uint32_t a = h & 0x7FFFu;
    const int32_t m = a > 0x7C00u ? 0 : a == 0x7C00u ? 0x7BFF : (int32_t)a;   // NaN -> 0, Inf -> the largest finite half
    return (h & 0x8000u) ? (sgn ? -m : 0) : m;
}

// decoded binary16 bits (bc6h_finish) -> their sign-magnitude integer
HAP_HD int32_t bc6h_value(uint32_t h) { return (h & 0x8000u) ? -(int32_t)(h & 0x7FFFu) : (int32_t)h; }

// the interpolated value of least magnitude that bc6h_finish maps to the sign-magnitude integer x
HAP_HD int32_t bc6h_target(int32_t x, bool sgn)
{
    const int32_t a = x < 0 ? -x : x;
    const int32_t c = ((sgn ? 32 : 64) * a + 30) / 31;
    return x < 0 ? -c : c;
}

// an interpolated-domain endpoint -> the prec-bit endpoint whose unquantised value (bc6h_unquantize) is nearest it: the
// code below it or the next one (ties: the lower)
HAP_HD int32_t bc6h_quantize(int32_t c, uint32_t prec, bool sgn)
{
    if (!sgn) {
        const int32_t u = c < 0 ? 0 : c > 0xFFFF ? 0xFFFF : c, top = prec >= 16 ? 0xFFFF : (1 << prec) - 1;
        const int32_t q = prec >= 16 ? u : (int32_t)(((uint32_t)u << prec) >> 16), q1 = q < top ? q + 1 : q;
        const int32_t d0 = u - bc6h_unquantize(q, prec, false), d1 = bc6h_unquantize(q1, prec, false) - u;
        return d1 < d0 ? q1 : q;
    }
    const int32_t a = c < 0 ? (c < -0x7FFF ? 0x7FFF : -c) : (c > 0x7FFF ? 0x7FFF : c);
    const int32_t top = prec >= 16 ? 0x7FFF : (1 << (prec - 1)) - 1;
    int32_t q = prec >= 16 ? a : (int32_t)(((uint32_t)a << (prec - 1)) >> 15);
    q = q > top ? top : q;
    const int32_t q1 = q < top ? q + 1 : q;
    const int32_t d0 = a - bc6h_unquantize(q, prec, true), d1 = bc6h_unquantize(q1, prec, true) - a;
    const int32_t m = d1 < d0 ? q1 : q;
    return c < 0 ? -m : m;
}

// the best candidate of one region count so far: its error, mode (0-13), partition, quantised endpoints r0 g0 b0 r1 .. b3
// (in the order stored, anchors already satisfied) and 16 indices of 4 bits
struct Bc6hPick {
    uint64_t err, idx;
    int32_t q[12];
    uint32_t mode, part;
};

// the texel mask of region 1 of partition part (bit t: texel t)
HAP_HD uint32_t bc6h_region1(uint32_t part)
{
    const uint32_t map = bc7_partition(part);
    uint32_t in = 0;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) in |= ((map >> (2 * t)) & 1u) << t;
    return in;
}

// Endpoints of the texels of `in` from their bounding box: per channel the minimum and the maximum, in the order of the
// channel of widest range or the reverse, as the channel's covariance with it has the sign; ends = a r g b, b r g b (the
// interpolated domain)
HAP_HD void bc6h_bbox(const int32_t x[48], uint32_t in, bool sgn, int32_t ends[6])
{
    int32_t lo[3] = {0x7FFFFFFF, 0x7FFFFFFF, 0x7FFFFFFF}, hi[3] = {-0x7FFFFFFF, -0x7FFFFFFF, -0x7FFFFFFF};
    int64_t s[3] = {0, 0, 0}, s01 = 0, s02 = 0, s12 = 0, n = 0;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool on = ((in >> t) & 1u) != 0;
#pragma unroll
        for (uint32_t c = 0; c < 3; c++) {
            const int32_t v = x[3 * t + c];
            lo[c] = on && v < lo[c] ? v : lo[c];
            hi[c] = on && v > hi[c] ? v : hi[c];
            s[c] += on ? v : 0;
        }
        s01 += on ? (int64_t)x[3 * t] * x[3 * t + 1] : 0;
        s02 += on ? (int64_t)x[3 * t] * x[3 * t + 2] : 0;
        s12 += on ? (int64_t)x[3 * t + 1] * x[3 * t + 2] : 0;
        n += on ? 1 : 0;
    }
    const int32_t r0 = hi[0] - lo[0], r1 = hi[1] - lo[1], r2 = hi[2] - lo[2];
    const uint32_t p = r0 >= r1 && r0 >= r2 ? 0u : r1 >= r2 ? 1u : 2u;
    const int64_t c01 = n * s01 - s[0] * s[1], c02 = n * s02 - s[0] * s[2], c12 = n * s12 - s[1] * s[2];
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) {
        const int64_t cov = c == p ? 1 : (c == 0 || p == 0) && (c == 1 || p == 1) ? c01 : (c == 0 || p == 0) ? c02 : c12;
        ends[c] = bc6h_target(cov < 0 ? hi[c] : lo[c], sgn);
        ends[3 + c] = bc6h_target(cov < 0 ? lo[c] : hi[c], sgn);
    }
}

// n / d rounded to nearest, halves away from zero (d > 0)
HAP_HD int64_t bc6h_div_round(int64_t n, int64_t d) { return n >= 0 ? (n + d / 2) / d : -((-n + d / 2) / d); }

// Least-squares endpoints of the texels of `in` with their indices held: per channel, a and b minimise
// sum (a (64 - w) + b w - 64 c)^2 over the texels, c the interpolated-domain value of the source (64 x / 31 in UF16,
// 32 x / 31 in SF16).  ends is left alone when every texel has the same weight.
HAP_HD void bc6h_refit(const int32_t x[48], uint32_t in, uint64_t idx, uint32_t ib, bool sgn, int32_t ends[6])
{
    int64_t aa = 0, ab = 0, bb = 0, ax[3] = {0, 0, 0}, bx[3] = {0, 0, 0};
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool on = ((in >> t) & 1u) != 0;
        const int64_t w = on ? (int64_t)bc7_weight((uint32_t)(idx >> (4 * t)) & 15u, ib) : 0, v = on ? 64 - w : 0;
        aa += v * v;
        ab += v * w;
        bb += w * w;
#pragma unroll
        for (uint32_t c = 0; c < 3; c++) {
            ax[c] += v * x[3 * t + c];
            bx[c] += w * x[3 * t + c];
        }
    }
    const int64_t det = aa * bb - ab * ab, k = sgn ? 2048 : 4096, den = 31 * (det > 0 ? det : 1);
    const int64_t lo = sgn ? -32767 : 0, hi = sgn ? 32767 : 0xFFFF;
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) {
        int64_t a = bc6h_div_round(k * (bb * ax[c] - ab * bx[c]), den), b = bc6h_div_round(k * (aa * bx[c] - ab * ax[c]), den);
        a = a < lo ? lo : a > hi ? hi : a;
        b = b < lo ? lo : b > hi ? hi : b;
        ends[c] = det > 0 ? (int32_t)a : ends[c];
        ends[3 + c] = det > 0 ? (int32_t)b : ends[3 + c];
    }
}

// One candidate: mode m (0-13; TWO: modes 0-9 on partition `part`, else modes 10-13) with the quantised endpoints q (a0,
// b0, then a1, b1 of region 1).  Every texel is given its nearest index by the decoder's arithmetic (raw: those indices,
// for a refit), the anchors are made to fit by swapping a region's endpoints and mirroring its indices (exact: the weights
// are symmetric), and the candidate is kept in `best` when its deltas fit and its error is lower.
template <bool TWO>
HAP_HD void bc6h_eval(uint32_t m, uint32_t part, const int32_t qin[12], const int32_t x[48], bool sgn, Bc6hPick &best, uint64_t &raw)
{
    const uint32_t par = bc6h_layout(m, 0).x, prec = par & 31u, transformed = (par >> 21) & 1u;
    constexpr uint32_t kEnds = TWO ? 12 : 6, kLevels = TWO ? 8 : 16, kIb = TWO ? 3 : 4;
    int32_t q[12], e[12];
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) {
        q[k] = k < kEnds ? qin[k] : 0;
        e[k] = bc6h_unquantize(q[k], prec, sgn);
    }
    const uint32_t map = TWO ? bc7_partition(part) : 0u;
    uint64_t err = 0, idx = 0;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool r1 = TWO && ((map >> (2 * t)) & 1u) != 0;
        int32_t a[3], b[3];
#pragma unroll
        for (uint32_t c = 0; c < 3; c++) {
            a[c] = r1 ? e[6 + c] : e[c];
            b[c] = r1 ? e[9 + c] : e[3 + c];
        }
        uint64_t be = ~0ull;
        uint32_t bi = 0;
#pragma unroll
        for (uint32_t i = 0; i < kLevels; i++) {
            const int32_t w = (int32_t)bc7_weight(i, kIb);
            uint64_t s = 0;
#pragma unroll
            for (uint32_t c = 0; c < 3; c++) {
                const int32_t d = bc6h_value(bc6h_finish((a[c] * (64 - w) + b[c] * w + 32) >> 6, sgn)) - x[3 * t + c];
                const uint32_t ad = (uint32_t)(d < 0 ? -d : d);
                s += (uint64_t)(ad * ad);
            }
            bi = s < be ? i : bi;
            be = s < be ? s : be;
        }
        err += be;
        idx |= (uint64_t)bi << (4 * t);
    }
    raw = idx;
    // anchors: texel 0 (region 0) and, with two regions, the partition's second anchor store one index bit less
    const uint32_t in1 = TWO ? bc6h_region1(part) : 0u;
    const uint32_t t1 = TWO ? hap_ctz(bc7_anchors(part) & ~1u) : 0u;
    const bool sw0 = (idx & 15u) >= kLevels / 2, sw1 = TWO && ((idx >> (4 * t1)) & 15u) >= kLevels / 2;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool flip = ((in1 >> t) & 1u) ? sw1 : sw0;
        const uint64_t f = (idx >> (4 * t)) & 15u;
        idx = flip ? (idx & ~(15ull << (4 * t))) | ((kLevels - 1u - f) << (4 * t)) : idx;
    }
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) {
        const int32_t a0 = q[c], b0 = q[3 + c], a1 = q[6 + c], b1 = q[9 + c];
        q[c] = sw0 ? b0 : a0;
        q[3 + c] = sw0 ? a0 : b0;
        q[6 + c] = sw1 ? b1 : a1;
        q[9 + c] = sw1 ? a1 : b1;
    }
    // transformed modes: each other endpoint as a delta from the base, wrapped to the base's precision, must fit its bits
    bool fits = true;
    const uint32_t mask = (1u << prec) - 1u;
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) {
        const uint32_t db = (par >> (c == 0 ? 5 : c == 1 ? 10 : 16)) & 31u;
        const int32_t lim = 1 << (db - 1);
#pragma unroll
        for (uint32_t k = 1; k < kEnds / 3; k++) {
            const int32_t d = bc6h_sext((uint32_t)(q[3 * k + c] - q[c]) & mask, prec);
            fits = fits && (!transformed || (d >= -lim && d < lim));
        }
    }
    const bool take = fits && err < best.err;
    best.err = take ? err : best.err;
    best.idx = take ? idx : best.idx;
    best.mode = take ? m : best.mode;
    best.part = take ? part : best.part;
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) best.q[k] = take ? q[k] : best.q[k];
}

// bc6h_eval of interpolated-domain endpoints `ends` quantised to mode m, then again of the least-squares endpoints of
// the indices they got
template <bool TWO>
HAP_HD void bc6h_try(uint32_t m, uint32_t part, const int32_t ends[12], const int32_t x[48], bool sgn, Bc6hPick &best)
{
    const uint32_t prec = bc6h_layout(m, 0).x & 31u;
    int32_t q[12], fit[12];
    uint64_t idx;
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) { q[k] = bc6h_quantize(ends[k], prec, sgn); fit[k] = ends[k]; }
    bc6h_eval<TWO>(m, part, q, x, sgn, best, idx);
    const uint32_t in1 = TWO ? bc6h_region1(part) : 0u;
    bc6h_refit(x, 0xFFFFu & ~in1, idx, TWO ? 3u : 4u, sgn, fit);
    if (TWO) bc6h_refit(x, in1, idx, 3u, sgn, fit + 6);
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) q[k] = bc6h_quantize(fit[k], prec, sgn);
    bc6h_eval<TWO>(m, part, q, x, sgn, best, idx);
}

// +-1 nudges of each quantised endpoint component of the pick, in its own mode, each kept when it lowers the error
template <bool TWO>
HAP_HD void bc6h_nudge(const int32_t x[48], bool sgn, Bc6hPick &best)
{
    const uint32_t m = best.mode, part = best.part, prec = bc6h_layout(m, 0).x & 31u;
    const int32_t lo = sgn ? -(prec >= 16 ? 0x7FFF : (1 << (prec - 1)) - 1) : 0;
    const int32_t hi = sgn ? (prec >= 16 ? 0x7FFF : (1 << (prec - 1)) - 1) : (prec >= 16 ? 0xFFFF : (1 << prec) - 1);
    uint64_t idx;
#pragma unroll 1
    for (uint32_t k = 0; k < (TWO ? 24u : 12u); k++) {
        int32_t q[12];
#pragma unroll
        for (uint32_t j = 0; j < 12; j++) q[j] = best.q[j];
        const int32_t v = q[k >> 1] + ((k & 1u) ? 1 : -1);
        q[k >> 1] = v < lo ? lo : v > hi ? hi : v;
        bc6h_eval<TWO>(m, part, q, x, sgn, best, idx);
    }
}

// n bits of v into the block (w0 = bits 0..31, ... w3 = bits 96..127) from bit pos on (pos + n <= 128, n <= 16)
HAP_HD void bc6h_put(uint32_t w[4], uint32_t pos, uint32_t n, uint32_t v)
{
    const uint64_t s = (uint64_t)(v & ((1u << n) - 1u)) << (pos & 31u);
    const uint32_t k = pos >> 5;
#pragma unroll
    for (uint32_t j = 0; j < 4; j++) w[j] |= j == k ? (uint32_t)s : j == k + 1u ? (uint32_t)(s >> 32) : 0u;
}

// A pick -> its 128 bits: the mode value, each endpoint component through the pieces of the mode's kBc6hLayout row (the
// inverse of bc6h_decode_block's reader), the partition, the indices
HAP_HD void bc6h_pack(const Bc6hPick &p, uint32_t out[4])
{
    uint32_t row[16];
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        const uint4 v = bc6h_layout(p.mode, k);
        row[4 * k] = v.x; row[4 * k + 1] = v.y; row[4 * k + 2] = v.z; row[4 * k + 3] = v.w;
    }
    const uint32_t par = row[0], prec = par & 31u, transformed = (par >> 21) & 1u, two = (par >> 22) & 1u;
    const uint32_t mask = (1u << prec) - 1u;
    uint32_t raw[12];
#pragma unroll
    for (uint32_t c = 0; c < 3; c++) {
        const uint32_t db = (par >> (c == 0 ? 5 : c == 1 ? 10 : 16)) & 31u;
        raw[c] = (uint32_t)p.q[c] & mask;
#pragma unroll
        for (uint32_t e = 1; e < 4; e++) {
            const uint32_t d = (uint32_t)(p.q[3 * e + c] - p.q[c]) & mask;
            raw[3 * e + c] = transformed ? (uint32_t)bc6h_sext(d, prec) & ((1u << db) - 1u) : (uint32_t)p.q[3 * e + c] & mask;
        }
    }
    uint32_t w[4] = {bc6h_mode_value(p.mode), 0u, 0u, 0u};
#pragma unroll
    for (uint32_t s = 0; s < kBc6hSlots; s++) {
        const uint32_t e = (row[1 + s / 2] >> (16 * (s & 1))) & 0xFFFFu, n = (e >> 7) & 15u;
        uint32_t v = (raw[bc6h_slot_component(s)] >> ((e >> 11) & 15u)) & ((1u << n) - 1u);
        v = (e & 0x8000u) ? hap_brev(v) >> ((32u - n) & 31u) : v;
        bc6h_put(w, e & 127u, n, v);
    }
    bc6h_put(w, 77, two ? 5u : 0u, p.part);
    const uint32_t amask = two ? bc7_anchors(p.part) : 1u, ib = two ? 3u : 4u;
    uint32_t pos = two ? 82u : 65u;
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const uint32_t nb = ib - ((amask >> t) & 1u);
        bc6h_put(w, pos, nb, (uint32_t)(p.idx >> (4 * t)) & 15u);
        pos += nb;
    }
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) out[k] = w[k];
}

// The partition pre-score of one region (the texels of `in`): its squared distance from the line through its mean along
// its principal axis, i.e. the trace of its scatter matrix less the largest eigenvalue, the eigenvalue estimated by two
// steps of power iteration from the column of the widest channel.  Exact integer moments, then float (hap_fma).
HAP_HD float bc6h_line_residual(const int32_t x[48], uint32_t in)
{
    int64_t n = 0, s[3] = {0, 0, 0}, ss[6] = {0, 0, 0, 0, 0, 0};   // ss: 00 11 22 01 02 12
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        const bool on = ((in >> t) & 1u) != 0;
        const int64_t r = on ? x[3 * t] : 0, g = on ? x[3 * t + 1] : 0, b = on ? x[3 * t + 2] : 0;
        n += on ? 1 : 0;
        s[0] += r; s[1] += g; s[2] += b;
        ss[0] += r * r; ss[1] += g * g; ss[2] += b * b; ss[3] += r * g; ss[4] += r * b; ss[5] += g * b;
    }
    // n^2 x the covariance
    const float c00 = (float)(n * ss[0] - s[0] * s[0]), c11 = (float)(n * ss[1] - s[1] * s[1]), c22 = (float)(n * ss[2] - s[2] * s[2]);
    const float c01 = (float)(n * ss[3] - s[0] * s[1]), c02 = (float)(n * ss[4] - s[0] * s[2]), c12 = (float)(n * ss[5] - s[1] * s[2]);
    float v0 = c00 >= c11 && c00 >= c22 ? c00 : c11 >= c22 ? c01 : c02;
    float v1 = c00 >= c11 && c00 >= c22 ? c01 : c11 >= c22 ? c11 : c12;
    float v2 = c00 >= c11 && c00 >= c22 ? c02 : c11 >= c22 ? c12 : c22;
#pragma unroll
    for (int it = 0; it < 2; it++) {
        const float m = hap_fmax3(fabsf(v0), fabsf(v1), fabsf(v2));
        const float k = m > 0.0f ? 1.0f / m : 0.0f;
        const float a = v0 * k, b = v1 * k, c = v2 * k;
        v0 = hap_fma(c00, a, hap_fma(c01, b, c02 * c));
        v1 = hap_fma(c01, a, hap_fma(c11, b, c12 * c));
        v2 = hap_fma(c02, a, hap_fma(c12, b, c22 * c));
    }
    const float m = hap_fmax3(fabsf(v0), fabsf(v1), fabsf(v2));
    const float k = m > 0.0f ? 1.0f / m : 0.0f;
    const float a = v0 * k, b = v1 * k, c = v2 * k;
    const float cv0 = hap_fma(c00, a, hap_fma(c01, b, c02 * c)), cv1 = hap_fma(c01, a, hap_fma(c11, b, c12 * c));
    const float cv2 = hap_fma(c02, a, hap_fma(c12, b, c22 * c));
    const float vv = hap_fma(a, a, hap_fma(b, b, c * c));
    const float lambda = vv > 0.0f ? hap_fma(a, cv0, hap_fma(b, cv1, c * cv2)) / vv : 0.0f;
    return (c00 + c11 + c22 - lambda) / (float)(n > 0 ? n * n : 1);
}

// One block: texel t of the picture in px[2t] (R | G << 16) and px[2t + 1] (B | A << 16), RGBA16F -> 16 bytes of BC6H in
// out[0..3].  Returns the error the block was chosen by (sum over the texels and R, G, B of the squared difference of
// decoded and source sign-magnitude integers, after the input rules).
HAP_HD uint64_t bc6h_encode_block(const uint32_t px[32], bool sgn, uint32_t out[4])
{
    int32_t x[48];
#pragma unroll
    for (uint32_t t = 0; t < 16; t++) {
        x[3 * t] = bc6h_source(px[2 * t] & 0xFFFFu, sgn);
        x[3 * t + 1] = bc6h_source(px[2 * t] >> 16, sgn);
        x[3 * t + 2] = bc6h_source(px[2 * t + 1] & 0xFFFFu, sgn);
    }
    Bc6hPick one, two;
    one.err = two.err = ~0ull;
    one.idx = two.idx = 0;
    one.mode = 10u;
    two.mode = 0u;
    one.part = two.part = 0u;
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) one.q[k] = two.q[k] = 0;
    int32_t ends[12];
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) ends[k] = 0;

    // one region
    bc6h_bbox(x, 0xFFFFu, sgn, ends);
#pragma unroll 1
    for (uint32_t m = 10; m < 14; m++) bc6h_try<false>(m, 0, ends, x, sgn, one);

    // two regions: pre-score the 32 partitions by how far each region's texels lie from one line, keep the best few
    float top_score[kBc6hPartitionFits];
    uint32_t top_part[kBc6hPartitionFits];
#pragma unroll
    for (uint32_t k = 0; k < kBc6hPartitionFits; k++) { top_score[k] = 3.0e38f; top_part[k] = 0; }
#pragma unroll 1
    for (uint32_t part = 0; part < 32; part++) {
        const uint32_t in1 = bc6h_region1(part);
        float score = bc6h_line_residual(x, in1) + bc6h_line_residual(x, 0xFFFFu & ~in1);
        uint32_t p = part;
#pragma unroll
        for (uint32_t k = 0; k < kBc6hPartitionFits; k++) {
            const bool lower = score < top_score[k];
            const float ts = top_score[k];
            const uint32_t tp = top_part[k];
            top_score[k] = lower ? score : ts;
            top_part[k] = lower ? p : tp;
            score = lower ? ts : score;
            p = lower ? tp : p;
        }
    }
#pragma unroll 1
    for (uint32_t k = 0; k < kBc6hPartitionFits; k++) {
        const uint32_t part = top_part[k], in1 = bc6h_region1(part);
        bc6h_bbox(x, 0xFFFFu & ~in1, sgn, ends);
        bc6h_bbox(x, in1, sgn, ends + 6);
#pragma unroll 1
        for (uint32_t m = 0; m < 10; m++) bc6h_try<true>(m, part, ends, x, sgn, two);
    }

    // refinement: least squares on the indices of the best candidate of each region count, tried again in every mode
#pragma unroll 1
    for (uint32_t it = 0; it < 2; it++) {
        bc6h_bbox(x, 0xFFFFu, sgn, ends);
        bc6h_refit(x, 0xFFFFu, one.idx, 4, sgn, ends);
#pragma unroll 1
        for (uint32_t m = 10; m < 14; m++) bc6h_try<false>(m, 0, ends, x, sgn, one);
        const uint32_t part = two.part, in1 = bc6h_region1(part);
        bc6h_bbox(x, 0xFFFFu & ~in1, sgn, ends);
        bc6h_bbox(x, in1, sgn, ends + 6);
        bc6h_refit(x, 0xFFFFu & ~in1, two.idx, 3, sgn, ends);
        bc6h_refit(x, in1, two.idx, 3, sgn, ends + 6);
#pragma unroll 1
        for (uint32_t m = 0; m < 10; m++) bc6h_try<true>(m, part, ends, x, sgn, two);
    }

    bc6h_nudge<false>(x, sgn, one);
    bc6h_nudge<true>(x, sgn, two);

    const bool use_two = two.err < one.err;
    Bc6hPick p;
    p.err = use_two ? two.err : one.err;
    p.idx = use_two ? two.idx : one.idx;
    p.mode = use_two ? two.mode : one.mode;
    p.part = use_two ? two.part : one.part;
#pragma unroll
    for (uint32_t k = 0; k < 12; k++) p.q[k] = use_two ? two.q[k] : one.q[k];
    bc6h_pack(p, out);
    return p.err;
}

// grid = (bc_ctas, frames), G as for bc_encode_kernel with 8 bytes per pixel (row_bytes >= 8 * width, out_stride >= 16 per
// block).  is_signed: SF16, else UF16.  SRC (BcSource): kSrcRgbaHalf reads `rgba` as RGBA16F rows; kSrcP010Pq reads it as
// the luma plane of an HDR10 P010 picture and P.m.chroma as its chroma plane, both frame_bytes apart per frame and rows
// row_bytes apart, and converts them to RGBA16F (yuv_source.cuh) before the search.  P comes last so that the parameters of
// the RGBA16F instantiation keep their offsets.
template <int SRC = kSrcRgbaHalf>
__global__ void __launch_bounds__(kBcThreads) bc6h_encode_kernel(const uint8_t *__restrict__ rgba, BcGeom G, uint8_t *__restrict__ out,
                                                                 uint32_t is_signed, YuvPqSrc P = YuvPqSrc())
{
    const uint32_t nblocks = G.blocks_x * G.blocks_y;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= nblocks) return;
    uint32_t by = __umulhi(bi, G.inv_blocks_x), bx = bi - by * G.blocks_x;  // the estimate is exact or one short
    if (bx >= G.blocks_x) { by++; bx -= G.blocks_x; }
    uint32_t px[32];
    if (SRC == kSrcRgbaHalf) {
        const uint8_t *src = rgba + (uint64_t)blockIdx.y * G.frame_bytes + (uint64_t)(4 * by) * G.row_bytes + 32u * bx;
#pragma unroll
        for (int row = 0; row < 4; row++) {
            const uint4 *s = reinterpret_cast<const uint4 *>(src + (uint64_t)row * G.row_bytes);
            const uint4 v0 = s[0], v1 = s[1];
            px[8 * row] = v0.x; px[8 * row + 1] = v0.y; px[8 * row + 2] = v0.z; px[8 * row + 3] = v0.w;
            px[8 * row + 4] = v1.x; px[8 * row + 5] = v1.y; px[8 * row + 6] = v1.z; px[8 * row + 7] = v1.w;
        }
    } else {
        const uint64_t f = (uint64_t)blockIdx.y * G.frame_bytes;
        load_block_yuv_pq(rgba + f, P.m.chroma + f, G.row_bytes, bx, by, G.blocks_x, G.blocks_y, P, px);
    }
    uint32_t w[4];
    bc6h_encode_block(px, is_signed != 0u, w);
    reinterpret_cast<uint4 *>(out + (uint64_t)blockIdx.y * G.out_stride)[bi] = make_uint4(w[0], w[1], w[2], w[3]);
}

}  // namespace hapb200
