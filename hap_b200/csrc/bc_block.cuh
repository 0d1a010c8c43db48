// hap_b200/csrc/bc_block.cuh -- K1-K4 block math: one 4x4 RGBA block -> one 8/16-byte S3TC/RGTC block.
//
// The block compressors sit UPSTREAM of the reference (which takes already-compressed DXT bytes,
// /root/reference/source/hap.h:82-104; formats per documentation/HapVideoDRAFT.md:22-27); the
// north star makes them the encode hot kernel.  Quality bar: PSNR within 0.1 dB of a squish-HIGH
// (iterative cluster fit) encode, which oracle/bc_oracle.c restates.
//
// Work decomposition: ONE THREAD PER BLOCK.  SURVEY.md H1: at the bandwidth target a 4x4 block has
// ~13 warp-instructions if a warp owns it but ~420 thread-instructions if a thread owns it; all 16
// texels live in registers, every reduction is a private serial sum (no shuffles, no idle lanes),
// and the four 16-byte row pieces of neighbouring threads are contiguous, so the loads are coalesced as
// they are (bc_encode.cuh).
//
// The fits, all on the same pattern -- principal axis of the block's covariance, 4 clusters by projection,
// the 2x2 least-squares system for the two endpoints given those clusters (the normal equations cluster
// fit solves, for the partition the axis implies instead of all 969), endpoints onto the 5:6:5 grid by a
// small search with the decoder's expanded values, indices against the decoder's palette:
//   * scaled YCoCg chroma (encode_ycocg_chroma): 2-D, closed-form axis, one start, ~600 instructions;
//   * RGB (encode_rgb_block): 3-D, power iteration, 2 x 2 starts scored after grid snapping, one Lloyd
//     round on the winner, exact nearest-palette indices, ~2 600 instructions;
//   * BC4 (encode_bc4_scaled): endpoints = min / max, indices by one biased fixed-point rounding per texel.
// Instruction counts are the currency here: the kernels are bound by instruction issue, and every step was
// held to the PSNR bar on the host build of this very source before it went to the GPU.
//
// Floating point is written with explicit fused multiply-adds (hap_fma) and the translation unit is
// built with -fmad=false, so the CPU twin used by the tests (tests/emu/bc_twin.cc) reproduces the
// GPU result bit for bit: IEEE add/mul/div/sqrt and fma are exact on both sides.
#pragma once
#include "simt.h"
#include <math.h>

namespace hapb200 {

#ifdef HAPB200_EMU
#define HAP_HD inline
static inline float hap_fma(float a, float b, float c) { return fmaf(a, b, c); }
#else
#define HAP_HD __host__ __device__ __forceinline__
HAP_HD float hap_fma(float a, float b, float c) { return fmaf(a, b, c); }
#endif


struct Block8 { uint32_t lo, hi; };

// sum over the four bytes of a (unsigned) times the four bytes of b (signed), plus c: one DP4A instruction
#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD int hap_dp4a_us(uint32_t a, uint32_t b, int c)
{
    for (int k = 0; k < 4; k++) c += (int)((a >> (8 * k)) & 0xFF) * (int)(int8_t)((b >> (8 * k)) & 0xFF);
    return c;
}
#else
__device__ __forceinline__ int hap_dp4a_us(uint32_t a, uint32_t b, int c)
{
    int d;
    asm("dp4a.u32.s32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
#endif

// unsigned x unsigned bytes, and the byte permute (selector nibble n picks byte n of the result from the 8 bytes {a, b})
#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD uint32_t hap_dp4a_uu(uint32_t a, uint32_t b, uint32_t c)
{
    for (int k = 0; k < 4; k++) c += ((a >> (8 * k)) & 0xFF) * ((b >> (8 * k)) & 0xFF);
    return c;
}
HAP_HD uint32_t hap_prmt(uint32_t a, uint32_t b, uint32_t sel)
{
    const uint64_t v = (uint64_t)a | ((uint64_t)b << 32);
    uint32_t r = 0;
    for (int k = 0; k < 4; k++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * k)) & 7))) & 0xFF) << (8 * k);
    return r;
}
#else
__device__ __forceinline__ uint32_t hap_dp4a_uu(uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t d;
    asm("dp4a.u32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}
__device__ __forceinline__ uint32_t hap_prmt(uint32_t a, uint32_t b, uint32_t sel) { return __byte_perm(a, b, sel); }
#endif

HAP_HD int hap_clampi(int v, int lo, int hi) { return v < lo ? lo : v > hi ? hi : v; }

// Three-input min/max, clamp(a+b, 0, c) and saturate: CUDA intrinsics on the device (sm_90a lowers each to a few
// IMNMX / IADD / FMNMX instructions); plain C++ on the host so that the CPU twin computes the same values.
#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD int hap_max3(int a, int b, int c) { int m = a > b ? a : b; return m > c ? m : c; }
HAP_HD int hap_min3(int a, int b, int c) { int m = a < b ? a : b; return m < c ? m : c; }
HAP_HD int hap_addmin_relu(int a, int b, int c) { int s = a + b; s = s < c ? s : c; return s < 0 ? 0 : s; }
#else
__device__ __forceinline__ int hap_max3(int a, int b, int c) { return __vimax3_s32(a, b, c); }
__device__ __forceinline__ int hap_min3(int a, int b, int c) { return __vimin3_s32(a, b, c); }
__device__ __forceinline__ int hap_addmin_relu(int a, int b, int c) { return __viaddmin_s32_relu(a, b, c); }
#endif
HAP_HD float hap_fmax3(float a, float b, float c) { return fmaxf(a, fmaxf(b, c)); }
HAP_HD float hap_fmin3(float a, float b, float c) { return fminf(a, fminf(b, c)); }
HAP_HD float hap_sat(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }
#if defined(HAPB200_EMU) || !defined(__CUDA_ARCH__)
HAP_HD uint32_t hap_float_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
#else
__device__ __forceinline__ uint32_t hap_float_bits(float f) { return __float_as_uint(f); }
#endif
constexpr float kRoundMagic = 12582912.0f;      // 1.5 * 2^23: x + magic rounds x to the nearest integer (ties to even) ...
constexpr uint32_t kRoundMagicBits = 0x4B400000u;  // ... which then sits in the low mantissa bits

// ---- BC4 / RGTC1: 16 values -> 8 bytes ------------------------------------------------------------
// 8-value mode (a0 > a1): palette a0, a1, then 6 interpolants (decoder: ((8-i)a0 + (i-1)a1)/7).
// Endpoints are the block's max/min (a least-squares refinement of them was measured to change nothing);
// each texel takes the nearest of the decoder's truncating palette values.
// decoder palette, truncating: ((7-L)*a1 + L*a0)/7 = a1 + floor(L*(a0-a1)/7); L*(a0-a1) <= 1785, where
// floor(q/7) == (q*9363)>>16 exactly (checked exhaustively)
HAP_HD int bc4_level_value(int L, int a0, int a1) { return a1 + (int)(((uint32_t)(L * (a0 - a1)) * 9363u) >> 16); }

// ---- BC4 ------------------------------------------------------------------------------------------
// v[t] = the value in 1/UNIT steps, UNIT a multiple of 7 (UNIT = 7: 7 * alpha; UNIT = 28: 7 * (R + 2G + B), luma
// with the two bits kept that rounding Y to 8 bits throws away -- the factors ride for free in the DP4A weights);
// vmax / vmin = max / min of v.  Endpoints = the rounded max and min of the block (a least-squares refinement of
// them was measured to change nothing).
// A texel's level L (0 = the min end ... 7 = the max end) is the nearest of the 8 palette values.  The decoder's
// palette truncates: value(L) = min + floor(L d / 7), i.e. the ideal ramp minus 0/7 .. 6/7 of a grey level, 3/7 on
// average -- so the texel is moved UP by 3/7 (exactly 3 UNIT/7 here) before it is rounded onto the ideal ramp.
// That is one VIADDMNMX (clamp(v - UNIT min + 3 UNIT/7, 0, range)), one fixed-point multiply and one shift per
// texel instead of seven threshold compares (measured against the exhaustive choice: see test_block_quality_cpu).
// Levels are packed 8 to a word and turned into DXT index numbering on all eight 3-bit fields at once.
HAP_HD uint32_t bc4_levels_to_indices8(uint32_t levels)
{
    const uint32_t x = levels ^ 0xFFFFFFu;                            // M = 7 - L: 0 = the max end (a0)
    const uint32_t m0 = 0x249249u;                                     // bit 0 of each of the eight fields
    const uint32_t x1 = x >> 1, x2 = x >> 2;
    const uint32_t sevens = x & x1 & x2 & m0, zeros = ~(x | x1 | x2) & m0;
    return (x & ~(sevens * 7u)) + m0 - zeros;                         // M: 0 -> 0, 7 -> 1, else M + 1
}

template <int UNIT>
HAP_HD Block8 encode_bc4_scaled(const int v[16], int vmax, int vmin)
{
    static_assert(UNIT % 7 == 0, "UNIT carries the factor 7");
    const int mx = (int)((uint32_t)(vmax + UNIT / 2) / (uint32_t)UNIT), mn = (int)((uint32_t)(vmin + UNIT / 2) / (uint32_t)UNIT);
    Block8 out;
    out.lo = (uint32_t)mx | ((uint32_t)mn << 8);
    out.hi = 0;
    if (mx == mn) return out;  // a0 == a1 selects the 6-value mode; index 0 decodes to a0 in both modes
    const int d = mx - mn, range = UNIT * d;
    const int r7 = d - 7 * (int)(((uint32_t)d * 9363u) >> 16);                       // d mod 7 (d <= 255)
    // integer inputs (UNIT = 7): 3/7 is exact for every d.  Quarter-step inputs: the best constant per d mod 7,
    // 0, 8, 9, 11, 11, 9, 8 twenty-eighths (0 when d is a multiple of 7: nothing is truncated then)
    const int bias = UNIT % 28 == 0 ? (int)((0x89BB980u >> (4 * r7)) & 15u) * (UNIT / 28) : 3 * (UNIT / 7);
    const int c0 = bias - UNIT * mn;
    // 7 * 2^20 / range, rounded: (t * mul + 2^19) >> 20 is round(7 t / range) for every t <= range (<= 7140)
    const int mul = (int)(7340032.0f * (1.0f / (float)range) + 0.5f);
    uint32_t a = 0, b = 0;
#pragma unroll
    for (int t = 0; t < 8; t++) {
        const uint32_t La = (uint32_t)(hap_addmin_relu(v[t], c0, range) * mul + (1 << 19)) >> 20;
        const uint32_t Lb = (uint32_t)(hap_addmin_relu(v[t + 8], c0, range) * mul + (1 << 19)) >> 20;
        a += La << (3 * t);
        b += Lb << (3 * t);
    }
    a = bc4_levels_to_indices8(a);
    b = bc4_levels_to_indices8(b);
    out.lo |= a << 16;
    out.hi = (a >> 16) | (b << 8);
    return out;
}

// ---- BC1 colour block: 16 (r,g,b) in 0..255 -> 8 bytes, always 4-colour mode ---------------------
HAP_HD uint32_t expand5(uint32_t c) { return (c << 3) | (c >> 2); }
HAP_HD uint32_t expand6(uint32_t c) { return (c << 2) | (c >> 4); }

// ---- scaled YCoCg (van Waveren & Castano 2007) ----------------------------------------------------
// Per block: co = (R-B)/2, cg = (-R+2G-B)/4 kept as exact half/quarter integers; scale = largest of
// {4,2,1} with |co*scale|,|cg*scale| <= 127; stored texel (Co', Cg', (scale-1)*8, Y).
// RGB error of a chroma error (dCo, dCg): (dCo-dCg)^2 + dCg^2 + (dCo+dCg)^2 = 2 dCo^2 + 3 dCg^2
#ifndef HAP_YCOCG_FIT
#define HAP_YCOCG_FIT 1, 0, true
#endif
constexpr float kYCoCgMetricCo = 1.41421356f, kYCoCgMetricCg = 1.73205081f;

// One channel of the endpoint pair onto its 5- or 6-bit grid.  For fixed clusters the squared error separates per
// channel, E(a,b) = a^2 A2 + b^2 B2 + 2ab AB - 2a AX - 2b BX, so floor/ceil of both ends are tried (4 candidates)
// with the values the DECODER expands them to.  a, b: storage units 0..255; the sums are taken about `off`.
HAP_HD void snap_pair(float a, float b, float off, float A2, float B2, float AB, float AX, float BX, float levels,
                      uint32_t &ga_out, uint32_t &gb_out)
{
    const float to_grid = levels * (1.0f / 255.0f), from_grid = 255.0f / levels;
    const float ga0 = floorf(a * to_grid), gb0 = floorf(b * to_grid);
    const float ga1 = fminf(ga0 + 1.0f, levels), gb1 = fminf(gb0 + 1.0f, levels);
    // the decoder expands by bit replication, which equals round(g * 255 / levels) for 5 and 6 bits
    const float ca0 = floorf(hap_fma(ga0, from_grid, 0.5f)) - off, ca1 = floorf(hap_fma(ga1, from_grid, 0.5f)) - off;
    const float cb0 = floorf(hap_fma(gb0, from_grid, 0.5f)) - off, cb1 = floorf(hap_fma(gb1, from_grid, 0.5f)) - off;
    const float m2AX = -2.0f * AX, m2BX = -2.0f * BX, AB2 = 2.0f * AB;
    const float ua0 = ca0 * hap_fma(ca0, A2, m2AX), ua1 = ca1 * hap_fma(ca1, A2, m2AX);
    const float ub0 = cb0 * hap_fma(cb0, B2, m2BX), ub1 = cb1 * hap_fma(cb1, B2, m2BX);
    const float e00 = hap_fma(AB2 * ca0, cb0, ua0 + ub0), e10 = hap_fma(AB2 * ca1, cb0, ua1 + ub0);
    const float e01 = hap_fma(AB2 * ca0, cb1, ua0 + ub1), e11 = hap_fma(AB2 * ca1, cb1, ua1 + ub1);
    float best = e00, ga = ga0, gb = gb0;
    if (e10 < best) { best = e10; ga = ga1; gb = gb0; }
    if (e01 < best) { best = e01; ga = ga0; gb = gb1; }
    if (e11 < best) { ga = ga1; gb = gb1; }
    ga_out = (uint32_t)(int)ga;
    gb_out = (uint32_t)(int)gb;
}

// ---- endpoint refinement where the grid is coarse against the data ---------------------------------------------
// snap_pair scores grid candidates with the clusters of the unquantised fit held fixed.  That is right while the
// grid step is small against the block's extent; when the Co' endpoints lie less than one 5-bit cell (8.2 storage
// units) apart, putting them on the grid stretches or collapses the segment so much that texels change cluster, and the
// fixed-partition score picks the wrong candidate about half the time (-0.47 dB on slow colour ramps against the
// oracle's search over all partitions).  There, the four floor/ceil candidates of the Co' pair are scored by their TRUE
// error instead: every texel re-assigned to the nearest of the candidate's four palette points.
//   sum |x - p0 - r e|^2 = sum |x - p0|^2 + |e|^2 sum r (r - 2u),  u = (x - p0).e / |e|^2,  r = round(3 sat(u)) / 3:
// the first sum follows from the block moments, the second costs 7 instructions per texel.
// It doubles the cost of the blocks it touches (half of the blocks of a smooth 4K picture), so it is an encoder OPTION
// (HAPB200_OPTION_CHROMA_REFINE, include/hap_b200.h) and a template parameter here: off costs nothing.
HAP_HD float chroma_true_error(const float x[16], const float y[16], float Sx, float Sy, float Sxx, float Syy, float p0x, float p0y, float p1x, float p1y)
{
    const float ex = p1x - p0x, ey = p1y - p0y;
    const float ee = hap_fma(ex, ex, ey * ey);
    const float iee = ee > 1e-9f ? 1.0f / ee : 0.0f;      // both endpoints on one grid point: every texel decodes to p0
    const float wx = ex * iee, wy = ey * iee, w0 = -hap_fma(p0x, wx, p0y * wy);
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < 16; t++) {
        const float u = hap_fma(x[t], wx, hap_fma(y[t], wy, w0));
        const float r3 = hap_fma(hap_sat(u), 3.0f, kRoundMagic) - kRoundMagic;     // 3 r = 0, 1, 2, 3
        acc = hap_fma(r3, hap_fma(u, -6.0f, r3), acc);                            // 9 r (r - 2u)
    }
    const float P = hap_fma(16.0f, hap_fma(p0x, p0x, p0y * p0y), hap_fma(-2.0f * p0x, Sx, hap_fma(-2.0f * p0y, Sy, Sxx + Syy)));
    return hap_fma(ee * (1.0f / 9.0f), acc, P);
}

// The chroma half of a scaled-YCoCg block: 16 (Co, Cg) pairs -> BC1 colour block (R' = Co', G' = Cg', B' = scale
// code).  co2 = R - B (half units), cg4 = -R + 2G - B (quarter units), with their max / min over the block.
//
// Everything is a fit in the 2-D plane of (Co', Cg') weighted by the metric above, done on the UNROUNDED chroma
// (the stored texel would be its rounding; the fit is against what the decoder should reproduce) and about the
// centre of the block's bounding box, which keeps the fp32 moment sums exact enough for a one-pass covariance:
//   moments -> 2x2 covariance -> principal axis in closed form -> extent along it -> 4 clusters by projection
//   -> the 2x2 least-squares system for the two endpoints given those clusters (the normal equations cluster
//   fit solves, for the partition the axis implies) -> per-channel grid search (snap_pair) -> indices by
//   projection onto the decoder's palette segment.
// Cluster sums are kept in terms of q = 0..3 (the cluster number): with beta = q/3, alpha = 1 - beta all nine
// sums of the normal equations follow from sum(q), sum(q^2), sum(q x), sum(q y) and the plain moments.
template <bool REFINE>
HAP_HD Block8 encode_ycocg_chroma(const int co2[16], const int cg4[16], int co_hi, int co_lo, int cg_hi, int cg_lo)
{
    const int m2 = co_hi > -co_lo ? co_hi : -co_lo, m4 = cg_hi > -cg_lo ? cg_hi : -cg_lo;
    int scale = 1;
    if (m2 * 4 <= 254 && m4 * 4 <= 508) scale = 4;
    else if (m2 * 2 <= 254 && m4 * 2 <= 508) scale = 2;
    const uint32_t blue5 = (uint32_t)(scale - 1);  // 5-bit code 0, 1 or 3: expands to B' = 0, 8, 24
    const float fs = (float)scale;
    // x = (Co' - offx) * metric, Co' = co2 * scale / 2 + 128
    const float cx = 0.5f * (float)(co_hi + co_lo), cy = 0.5f * (float)(cg_hi + cg_lo);
    const float kx = fs * (0.5f * kYCoCgMetricCo), ky = fs * (0.25f * kYCoCgMetricCg);
    const float bx0 = -cx * kx, by0 = -cy * ky;
    const float offx = hap_fma(cx, 0.5f * fs, 128.0f), offy = hap_fma(cy, 0.25f * fs, 128.0f);
    const float imx = 1.0f / kYCoCgMetricCo, imy = 1.0f / kYCoCgMetricCg;
    float x[16], y[16];
    float Sx = 0.f, Sy = 0.f, Sxx = 0.f, Sxy = 0.f, Syy = 0.f;
#pragma unroll
    for (int t = 0; t < 16; t++) {
        x[t] = hap_fma((float)co2[t], kx, bx0);
        y[t] = hap_fma((float)cg4[t], ky, by0);
        Sx += x[t]; Sy += y[t];
        Sxx = hap_fma(x[t], x[t], Sxx); Sxy = hap_fma(x[t], y[t], Sxy); Syy = hap_fma(y[t], y[t], Syy);
    }
    const float cxx = hap_fma(-0.0625f * Sx, Sx, Sxx), cxy = hap_fma(-0.0625f * Sx, Sy, Sxy), cyy = hap_fma(-0.0625f * Sy, Sy, Syy);

    uint32_t a5r, a6g, b5r, b6g;
    bool fitted = false;
    if (cxx + cyy >= 0.5f) {
        // principal axis of [[cxx, cxy], [cxy, cyy]]: eigenvector of the larger eigenvalue, closed form
        const float hd = 0.5f * (cxx - cyy);
        const float rad = sqrtf(hap_fma(hd, hd, cxy * cxy));
        float vx = hd >= 0.f ? hd + rad : cxy, vy = hd >= 0.f ? cxy : rad - hd;
        const float vv0 = hap_fma(vx, vx, vy * vy);
        if (vv0 < 1e-12f) { vx = 1.0f; vy = 0.0f; }  // isotropic spread: any axis
        // extent along the axis
        float d[16];
#pragma unroll
        for (int t = 0; t < 16; t++) d[t] = hap_fma(x[t], vx, y[t] * vy);
        float tmin = d[0], tmax = d[0];
#pragma unroll
        for (int t = 1; t < 15; t += 2) { tmin = hap_fmin3(tmin, d[t], d[t + 1]); tmax = hap_fmax3(tmax, d[t], d[t + 1]); }
        tmin = fminf(tmin, d[15]); tmax = fmaxf(tmax, d[15]);
        const float ext = tmax - tmin;
        if (ext > 1e-6f) {
            // clusters: q = round(3 (d - tmin) / ext) is 0..3 by construction, no clamp
            const float sc = 3.0f * (1.0f / ext);
            const float c0 = -tmin * sc;
            float Sq = 0.f, Sqq = 0.f, Sqx = 0.f, Sqy = 0.f;
#pragma unroll
            for (int t = 0; t < 16; t++) {
                const float q = rintf(hap_fma(d[t], sc, c0));
                Sq += q; Sqq = hap_fma(q, q, Sqq); Sqx = hap_fma(q, x[t], Sqx); Sqy = hap_fma(q, y[t], Sqy);
            }
            const float B2 = Sqq * (1.0f / 9.0f), AB = hap_fma(Sq, 1.0f / 3.0f, -B2), A2 = 16.0f - hap_fma(Sq, 2.0f / 3.0f, -B2);
            const float BXx = Sqx * (1.0f / 3.0f), BXy = Sqy * (1.0f / 3.0f), AXx = Sx - BXx, AXy = Sy - BXy;
            const float det = hap_fma(A2, B2, -(AB * AB));
            float eax, eay, ebx, eby;  // endpoints, metric space about the centre
            if (det >= 1e-4f) {
                const float idet = 1.0f / det;
                eax = hap_fma(AXx, B2, -(BXx * AB)) * idet; ebx = hap_fma(BXx, A2, -(AXx * AB)) * idet;
                eay = hap_fma(AXy, B2, -(BXy * AB)) * idet; eby = hap_fma(BXy, A2, -(AXy * AB)) * idet;
            } else {
                const float ivv = 1.0f / hap_fma(vx, vx, vy * vy);
                eax = vx * (tmin * ivv); eay = vy * (tmin * ivv); ebx = vx * (tmax * ivv); eby = vy * (tmax * ivv);
            }
            // storage units, then the grid
            const float ar = fminf(fmaxf(hap_fma(eax, imx, offx), 0.f), 255.f), br = fminf(fmaxf(hap_fma(ebx, imx, offx), 0.f), 255.f);
            const float ag = fminf(fmaxf(hap_fma(eay, imy, offy), 0.f), 255.f), bg = fminf(fmaxf(hap_fma(eby, imy, offy), 0.f), 255.f);
            if (det >= 1e-4f) {
                a6g = (uint32_t)(int)floorf(hap_fma(ag, 63.0f / 255.0f, 0.5f)); b6g = (uint32_t)(int)floorf(hap_fma(bg, 63.0f / 255.0f, 0.5f));
                if (REFINE && fabsf(ar - br) < 255.0f / 31.0f) {
                    const float p0y = ((float)expand6(a6g) - offy) * kYCoCgMetricCg, p1y = ((float)expand6(b6g) - offy) * kYCoCgMetricCg;
                    const uint32_t fa = (uint32_t)(int)floorf(ar * (31.0f / 255.0f)), fb = (uint32_t)(int)floorf(br * (31.0f / 255.0f));
                    float best = 3.0e38f;
                    a5r = fa; b5r = fb;
#pragma unroll 1
                    for (uint32_t c = 0; c < 4; c++) {
                        const uint32_t ca = fa + (c & 1u) < 31u ? fa + (c & 1u) : 31u, cb = fb + (c >> 1) < 31u ? fb + (c >> 1) : 31u;
                        const float e = chroma_true_error(x, y, Sx, Sy, Sxx, Syy, ((float)expand5(ca) - offx) * kYCoCgMetricCo, p0y,
                                                          ((float)expand5(cb) - offx) * kYCoCgMetricCo, p1y);
                        if (e < best) { best = e; a5r = ca; b5r = cb; }
                    }
                } else {
                    snap_pair(ar, br, offx, A2, B2, AB, AXx * imx, BXx * imx, 31.0f, a5r, b5r);
                }
            } else {
                a5r = (uint32_t)(int)floorf(hap_fma(ar, 31.0f / 255.0f, 0.5f)); b5r = (uint32_t)(int)floorf(hap_fma(br, 31.0f / 255.0f, 0.5f));
                a6g = (uint32_t)(int)floorf(hap_fma(ag, 63.0f / 255.0f, 0.5f)); b6g = (uint32_t)(int)floorf(hap_fma(bg, 63.0f / 255.0f, 0.5f));
            }
            fitted = true;
        }
    }
    if (!fitted) {
        // (nearly) one chroma: bracket it with its grid neighbours so the 4 palette entries straddle it
        const float fr = fminf(fmaxf(hap_fma(Sx * 0.0625f, imx, offx), 0.f), 255.f), fg = fminf(fmaxf(hap_fma(Sy * 0.0625f, imy, offy), 0.f), 255.f);
        a5r = (uint32_t)(int)floorf(fr * (31.0f / 255.0f)); b5r = (uint32_t)(int)ceilf(fr * (31.0f / 255.0f));
        a6g = (uint32_t)(int)floorf(fg * (63.0f / 255.0f)); b6g = (uint32_t)(int)ceilf(fg * (63.0f / 255.0f));
    }
    uint32_t c0 = (a5r << 11) | (a6g << 5) | blue5, c1 = (b5r << 11) | (b6g << 5) | blue5;
    Block8 out;
    out.lo = c0 | (c1 << 16);
    out.hi = 0;  // index 0 = c0 in either mode
    if (c0 == c1) return out;
    if (c0 < c1) {
        uint32_t tmp;
        tmp = c0; c0 = c1; c1 = tmp;
        tmp = a5r; a5r = b5r; b5r = tmp;
        tmp = a6g; a6g = b6g; b6g = tmp;
        out.lo = c0 | (c1 << 16);
    }
    // indices: position along the decoder's palette segment P0 -> P1, saturated to its ends, rounded to thirds.
    // The rounded level k = 0..3 sits in the low mantissa bits of (3w + magic); all sixteen are summed into one word
    // as k << 2t (the magic's own bits add up to a constant that is taken off once).
    const float p0x = ((float)expand5(a5r) - offx) * kYCoCgMetricCo, p0y = ((float)expand6(a6g) - offy) * kYCoCgMetricCg;
    const float p1x = ((float)expand5(b5r) - offx) * kYCoCgMetricCo, p1y = ((float)expand6(b6g) - offy) * kYCoCgMetricCg;
    const float ex = p1x - p0x, ey = p1y - p0y;
    const float iee = 1.0f / hap_fma(ex, ex, ey * ey);
    const float wx = ex * iee, wy = ey * iee, w0 = -hap_fma(p0x, wx, p0y * wy);
    uint32_t acc = 0;
#pragma unroll
    for (int t = 0; t < 16; t++) {
        const float w = hap_sat(hap_fma(x[t], wx, hap_fma(y[t], wy, w0)));
        acc += hap_float_bits(hap_fma(w, 3.0f, kRoundMagic)) << (2 * t);
    }
    const uint32_t k = acc - kRoundMagicBits * 0x55555555u;
    // level along the segment -> DXT numbering (0 = c0, 1 = c1, 2, 3 in between): 0,1,2,3 -> 0,2,3,1
    out.hi = (((k ^ (k >> 1)) & 0x55555555u) << 1) | ((k >> 1) & 0x55555555u);
    return out;
}

// A block whose 16 texels are one colour (letterbox bars, graphics, clipped highlights -- common in real
// footage): no statistics needed.  Endpoints bracket the colour on the 5:6:5 grid, the single index is the
// nearest of the four decoder palette entries under the metric (wr,wg,wb = squared channel weights).
HAP_HD Block8 encode_flat_colour(int R, int G, int B, int fixed_blue5, float wr, float wg, float wb)
{
    uint32_t a5r = (uint32_t)(R * 31) / 255u, a6g = (uint32_t)(G * 63) / 255u, a5b = (uint32_t)(B * 31) / 255u;
    uint32_t b5r = a5r + (expand5(a5r) != (uint32_t)R && a5r < 31 ? 1u : 0u);
    uint32_t b6g = a6g + (expand6(a6g) != (uint32_t)G && a6g < 63 ? 1u : 0u);
    uint32_t b5b = a5b + (expand5(a5b) != (uint32_t)B && a5b < 31 ? 1u : 0u);
    if (fixed_blue5 >= 0) a5b = b5b = (uint32_t)fixed_blue5;
    // c0 > c1 required for 4-colour mode: the "ceil" triple is the larger 565 word unless they are equal
    const uint32_t c0 = (b5r << 11) | (b6g << 5) | b5b, c1 = (a5r << 11) | (a6g << 5) | a5b;
    Block8 out;
    out.lo = c0 | (c1 << 16);
    out.hi = 0;
    if (c0 == c1) return out;
    if (c0 < c1) {
        // cannot happen (each field of c0 is >= the field of c1), kept for safety: index 0 still decodes to c0
        return out;
    }
    const int p0[3] = {(int)expand5(b5r), (int)expand6(b6g), (int)expand5(b5b)};
    const int p1[3] = {(int)expand5(a5r), (int)expand6(a6g), (int)expand5(a5b)};
    const int px3[3] = {R, G, B};
    const float wv[3] = {wr, wg, wb};
    float best = 1e30f;
    uint32_t bi = 0;
#pragma unroll
    for (uint32_t k = 0; k < 4; k++) {
        float e = 0.f;
#pragma unroll
        for (int c = 0; c < 3; c++) {
            int v = k == 0 ? p0[c] : k == 1 ? p1[c] : k == 2 ? (2 * p0[c] + p1[c]) / 3 : (p0[c] + 2 * p1[c]) / 3;
            float dlt = (float)(px3[c] - v);
            e = hap_fma(dlt * wv[c], dlt, e);
        }
        if (e < best) { best = e; bi = k; }
    }
    out.hi = bi * 0x55555555u;
    return out;
}

// ---- RGB colour block (DXT1 / the colour half of DXT5), the short way ----------------------------------------
// Principal axis of the covariance, then a small multi-start search along it that stands in for cluster fit's
// search over all 969 ordered partitions: N starts = placements of the two ends of the extent; per start 4 clusters
// by projection, the 2x2 least-squares system for the endpoints, endpoints onto the 5:6:5 grid (4 candidates per
// channel) and the error there; the best start gets one more Lloyd round on the quantised problem, then exact
// nearest-palette indices.  (A single start was measured at -0.39 dB against the cluster-fit oracle, this at
// -0.09 ... +0.03 dB.)  Arranged so that a start costs ~330 instructions:
//  * everything is done about the block mean (sum of the centred texels = 0, so alpha.x = -beta.x for every channel);
//  * texels are projected on the axis ONCE; a start only rescales the projection;
//  * cluster sums are over the cluster NUMBER q (sum q, sum q^2, sum q x): with beta = q/3 all normal-equation
//    terms follow;
//  * the grid search returns its error, which is the start's score.
#ifndef HAP_RGB_STARTS
#define HAP_RGB_STARTS 4
#endif
#ifndef HAP_RGB_RESNAP
#define HAP_RGB_RESNAP 1
#endif
struct RgbFit {
    float A2, B2, AB, BXr, BXg, BXb;     // normal-equation sums about the mean (AX = -BX)
};

// grid value (0..levels) nearest to storage value v (0..255), and what the decoder expands it to
HAP_HD float grid_round(float v, float levels) { return floorf(hap_fma(v, levels * (1.0f / 255.0f), 0.5f)); }
HAP_HD float grid_expand(float gq, float levels) { return floorf(hap_fma(gq, 255.0f / levels, 0.5f)); }

// error (up to the constant sum of squares) of endpoints ca, cb (about the mean) for one channel
HAP_HD float pair_error(float ca, float cb, float A2, float B2, float AB, float BX)
{
    // E = ca^2 A2 + cb^2 B2 + 2 ca cb AB - 2 ca AX - 2 cb BX with AX = -BX
    return hap_fma(ca, hap_fma(ca, A2, 2.0f * BX), hap_fma(cb, hap_fma(cb, B2, -2.0f * BX), (2.0f * AB) * ca * cb));
}

// 4-candidate search of one channel: floor/ceil of both ends on the grid; returns grid values
HAP_HD float snap_pair_centred(float a, float b, float mean, float A2, float B2, float AB, float BX, float levels, float &ga_out, float &gb_out)
{
    const float to_grid = levels * (1.0f / 255.0f);
    const float ga0 = floorf(a * to_grid), gb0 = floorf(b * to_grid);
    const float ga1 = fminf(ga0 + 1.0f, levels), gb1 = fminf(gb0 + 1.0f, levels);
    const float ca0 = grid_expand(ga0, levels) - mean, ca1 = grid_expand(ga1, levels) - mean;
    const float cb0 = grid_expand(gb0, levels) - mean, cb1 = grid_expand(gb1, levels) - mean;
    // E = ua(ca) + ub(cb) + 2 AB ca cb with ua(c) = c (c A2 + 2 BX), ub(c) = c (c B2 - 2 BX)  (AX = -BX)
    const float BX2 = 2.0f * BX, AB2 = 2.0f * AB;
    const float ua0 = ca0 * hap_fma(ca0, A2, BX2), ua1 = ca1 * hap_fma(ca1, A2, BX2);
    const float ub0 = cb0 * hap_fma(cb0, B2, -BX2), ub1 = cb1 * hap_fma(cb1, B2, -BX2);
    const float e00 = hap_fma(AB2 * ca0, cb0, ua0 + ub0), e10 = hap_fma(AB2 * ca1, cb0, ua1 + ub0);
    const float e01 = hap_fma(AB2 * ca0, cb1, ua0 + ub1), e11 = hap_fma(AB2 * ca1, cb1, ua1 + ub1);
    float best = e00, ga = ga0, gb = gb0;
    if (e10 < best) { best = e10; ga = ga1; gb = gb0; }
    if (e01 < best) { best = e01; ga = ga0; gb = gb1; }
    if (e11 < best) { best = e11; ga = ga1; gb = gb1; }
    ga_out = ga;
    gb_out = gb;
    return best;
}

// Texel data never leaves the integer domain: the sixteen texels are kept as RGBA words (px) and as three PLANES of
// packed bytes (four texels per word), so that every sum over texels is a handful of DP4A instructions --
//   moments:        sum R, sum R^2, sum R G ...      = DP4A(plane, 0x01010101), DP4A(plane, plane')          (36 for all nine)
//   projections:    d_t = texel . axis                = DP4A(px[t], axis as four signed bytes)                 (1 per texel)
//   cluster sums:   sum q, sum q^2, sum q R ...       = DP4A(q bytes, ...) with the cluster numbers q packed 4 to a word (20)
//   palette search: texel . (P_k - 128)               = DP4A(px[t], palette point as signed bytes)              (4 per texel)
// -- where the float formulation spends 3 to 6 instructions per texel and channel.  All sums are exact integers below 2^24,
// so the conversion to float for the 2x2 solve loses nothing.
struct RgbPlanes { uint32_t r[4], g[4], b[4]; };

// cluster numbers (0..3, one byte each, texel t in byte t%4 of word t/4) along [lo, hi] of the projections d[] -> sums
HAP_HD bool rgb_cluster_sums(const float d[16], const RgbPlanes &P, float mr, float mg, float mb, float lo, float hi, RgbFit &F)
{
    const float ext = hi - lo;
    if (!(ext > 1e-6f)) return false;
    const float sc = 1.0f / ext, c0 = -lo * sc;
    uint32_t sq = 0, sqq = 0, sqr = 0, sqg = 0, sqb = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        uint32_t w = 0;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            // q = round(3 sat((d - lo) / ext)) sits in the low mantissa bits of (3 w + magic); four of them share a word
            // (the magic's own bits add up to a constant that is taken off once)
            const float q = hap_fma(hap_sat(hap_fma(d[4 * i + j], sc, c0)), 3.0f, kRoundMagic);
            w += hap_float_bits(q) << (8 * j);
        }
        w -= kRoundMagicBits * 0x01010101u;
        sq = hap_dp4a_uu(w, 0x01010101u, sq); sqq = hap_dp4a_uu(w, w, sqq);
        sqr = hap_dp4a_uu(w, P.r[i], sqr); sqg = hap_dp4a_uu(w, P.g[i], sqg); sqb = hap_dp4a_uu(w, P.b[i], sqb);
    }
    const float Sq = (float)sq, Sqq = (float)sqq;
    F.B2 = Sqq * (1.0f / 9.0f);
    F.AB = hap_fma(Sq, 1.0f / 3.0f, -F.B2);
    F.A2 = 16.0f - hap_fma(Sq, 2.0f / 3.0f, -F.B2);
    // sums about the mean: sum q (R - mr) = sum q R - mr sum q
    F.BXr = hap_fma(-mr, Sq, (float)sqr) * (1.0f / 3.0f); F.BXg = hap_fma(-mg, Sq, (float)sqg) * (1.0f / 3.0f); F.BXb = hap_fma(-mb, Sq, (float)sqb) * (1.0f / 3.0f);
    return hap_fma(F.A2, F.B2, -(F.AB * F.AB)) >= 1e-4f;
}

// least-squares endpoints (about the mean) of one channel: AX = -BX
HAP_HD void rgb_solve(const RgbFit &F, float idet, float BX, float &a, float &b)
{
    a = -BX * (F.B2 + F.AB) * idet;
    b = BX * (F.A2 + F.AB) * idet;
}

// endpoints of fit F in storage units, put on the 5:6:5 grid (4 candidates per channel); returns the error there
HAP_HD float rgb_solve_and_snap(const RgbFit &F, float mr, float mg, float mb, float &gar, float &gag, float &gab, float &gbr, float &gbg, float &gbb)
{
    const float idet = 1.0f / hap_fma(F.A2, F.B2, -(F.AB * F.AB));
    float ar, br, ag, bg, ab, bb;
    rgb_solve(F, idet, F.BXr, ar, br); rgb_solve(F, idet, F.BXg, ag, bg); rgb_solve(F, idet, F.BXb, ab, bb);
    ar = fminf(fmaxf(ar + mr, 0.f), 255.f); br = fminf(fmaxf(br + mr, 0.f), 255.f);
    ag = fminf(fmaxf(ag + mg, 0.f), 255.f); bg = fminf(fmaxf(bg + mg, 0.f), 255.f);
    ab = fminf(fmaxf(ab + mb, 0.f), 255.f); bb = fminf(fmaxf(bb + mb, 0.f), 255.f);
    return snap_pair_centred(ar, br, mr, F.A2, F.B2, F.AB, F.BXr, 31.f, gar, gbr) +
           snap_pair_centred(ag, bg, mg, F.A2, F.B2, F.AB, F.BXg, 63.f, gag, gbg) +
           snap_pair_centred(ab, bb, mb, F.A2, F.B2, F.AB, F.BXb, 31.f, gab, gbb);
}

// (r, g, b) small signed integers -> the DP4A operand that multiplies a texel word's R, G, B bytes by them (A by 0)
HAP_HD uint32_t pack_s8x3(int r, int g, int b) { return ((uint32_t)r & 0xFFu) | (((uint32_t)g & 0xFFu) << 8) | (((uint32_t)b & 0xFFu) << 16); }

HAP_HD Block8 encode_rgb_block(const uint32_t px[16])
{
    RgbPlanes P;
    uint32_t sr = 0, sg = 0, sb = 0, rr = 0, rg = 0, rb = 0, gg = 0, gb = 0, bb2 = 0;
#pragma unroll
    for (int i = 0; i < 4; i++) {
        const uint32_t t0 = hap_prmt(px[4 * i], px[4 * i + 1], 0x5140u), t1 = hap_prmt(px[4 * i + 2], px[4 * i + 3], 0x5140u);
        const uint32_t t2 = hap_prmt(px[4 * i], px[4 * i + 1], 0x6262u), t3 = hap_prmt(px[4 * i + 2], px[4 * i + 3], 0x6262u);
        P.r[i] = hap_prmt(t0, t1, 0x5410u); P.g[i] = hap_prmt(t0, t1, 0x7632u); P.b[i] = hap_prmt(t2, t3, 0x5410u);
        sr = hap_dp4a_uu(P.r[i], 0x01010101u, sr); sg = hap_dp4a_uu(P.g[i], 0x01010101u, sg); sb = hap_dp4a_uu(P.b[i], 0x01010101u, sb);
        rr = hap_dp4a_uu(P.r[i], P.r[i], rr); rg = hap_dp4a_uu(P.r[i], P.g[i], rg); rb = hap_dp4a_uu(P.r[i], P.b[i], rb);
        gg = hap_dp4a_uu(P.g[i], P.g[i], gg); gb = hap_dp4a_uu(P.g[i], P.b[i], gb); bb2 = hap_dp4a_uu(P.b[i], P.b[i], bb2);
    }
    const float fsr = (float)sr, fsg = (float)sg, fsb = (float)sb;
    const float mr = fsr * 0.0625f, mg = fsg * 0.0625f, mb = fsb * 0.0625f;
    // covariance * 16 (exact: every term is an integer below 2^24, the products with 1/16 are exact too)
    const float crr = hap_fma(-mr, fsr, (float)rr), crg = hap_fma(-mr, fsg, (float)rg), crb = hap_fma(-mr, fsb, (float)rb);
    const float cgg = hap_fma(-mg, fsg, (float)gg), cgb = hap_fma(-mg, fsb, (float)gb), cbb = hap_fma(-mb, fsb, (float)bb2);
    float gar, gag, gab, gbr, gbg, gbb;   // endpoints on the 5:6:5 grid
    if (crr + cgg + cbb < 0.5f) {
        // flat block: bracket the colour with its grid neighbours so the 4 palette entries straddle it
        gar = floorf(mr * (31.0f / 255.0f)); gbr = ceilf(mr * (31.0f / 255.0f));
        gag = floorf(mg * (63.0f / 255.0f)); gbg = ceilf(mg * (63.0f / 255.0f));
        gab = floorf(mb * (31.0f / 255.0f)); gbb = ceilf(mb * (31.0f / 255.0f));
    } else {
        // principal axis: power iteration from the covariance row with the largest diagonal
        float vr, vg, vb;
        if (crr >= cgg && crr >= cbb) { vr = crr; vg = crg; vb = crb; }
        else if (cgg >= cbb) { vr = crg; vg = cgg; vb = cgb; }
        else { vr = crb; vg = cgb; vb = cbb; }
#pragma unroll
        for (int it = 0; it < 4; it++) {
            const float nr = hap_fma(crr, vr, hap_fma(crg, vg, crb * vb));
            const float ng = hap_fma(crg, vr, hap_fma(cgg, vg, cgb * vb));
            const float nb = hap_fma(crb, vr, hap_fma(cgb, vg, cbb * vb));
            const float inv = 1.0f / fmaxf(fabsf(nr), fmaxf(fabsf(ng), fabsf(nb)));
            vr = nr * inv; vg = ng * inv; vb = nb * inv;
        }
        // the axis in 7 bits + sign (its largest component is +-127): a texel's projection is one DP4A.  Only the ORDER and
        // spacing of the projections matter (they choose the clusters; the endpoints come from the least-squares solve).
        const int ar8 = (int)rintf(vr * 127.0f), ag8 = (int)rintf(vg * 127.0f), ab8 = (int)rintf(vb * 127.0f);
        const uint32_t axis = pack_s8x3(ar8, ag8, ab8);
        float d[16];
        int dmin = 0x7FFFFFFF, dmax = -0x7FFFFFFF;
#pragma unroll
        for (int t = 0; t < 16; t += 2) {
            const int d0 = hap_dp4a_us(px[t], axis, 0), d1 = hap_dp4a_us(px[t + 1], axis, 0);
            d[t] = (float)d0; d[t + 1] = (float)d1;
            dmin = hap_min3(dmin, d0, d1); dmax = hap_max3(dmax, d0, d1);
        }
        const float tmin = (float)dmin, tmax = (float)dmax;
        // starts: both ends of the extent moved independently outwards or inwards by 1/5 of its length (2 x 2).
        // (A 3 x 3 grid that also tried 3/5 inwards was measured: its five extra starts win almost never,
        // +0.005 dB for more than twice the work.)
        const float step = 0.2f * (tmax - tmin);
        bool have = false;
        float best_e = 1e30f;
#pragma unroll 1
        for (int st = 0; st < HAP_RGB_STARTS; st++) {
            const float lo = HAP_RGB_STARTS == 1 ? tmin : tmin + ((float)(st & 1) * 2.0f - 1.0f) * step;
            const float hi = HAP_RGB_STARTS == 1 ? tmax : tmax - ((float)(st >> 1) * 2.0f - 1.0f) * step;
            RgbFit F;
            if (!rgb_cluster_sums(d, P, mr, mg, mb, lo, hi, F)) continue;
            // scored AFTER the endpoints are put on the grid (4 candidates per channel): scoring the unquantised or the
            // plainly rounded endpoints picks the wrong start often enough to cost 0.01 ... 0.06 dB
            float s_ar, s_br, s_ag, s_bg, s_ab, s_bb;
            const float e = rgb_solve_and_snap(F, mr, mg, mb, s_ar, s_ag, s_ab, s_br, s_bg, s_bb);
            if (e < best_e) {
                best_e = e; have = true;
                gar = s_ar; gag = s_ag; gab = s_ab; gbr = s_br; gbg = s_bg; gbb = s_bb;
            }
        }
        if (!have) {
            // no start had two usable clusters: the ends of the extent, rounded (t = projection / |axis|^2 along the axis)
            const float fr8 = (float)ar8, fg8 = (float)ag8, fb8 = (float)ab8;
            const float ivv = 1.0f / fmaxf(hap_fma(fr8, fr8, hap_fma(fg8, fg8, fb8 * fb8)), 1.0f);
            const float m_ax = hap_fma(mr, fr8, hap_fma(mg, fg8, mb * fb8));
            const float t0 = (tmin - m_ax) * ivv, t1 = (tmax - m_ax) * ivv;
            gar = grid_round(fminf(fmaxf(hap_fma(fr8, t0, mr), 0.f), 255.f), 31.f); gbr = grid_round(fminf(fmaxf(hap_fma(fr8, t1, mr), 0.f), 255.f), 31.f);
            gag = grid_round(fminf(fmaxf(hap_fma(fg8, t0, mg), 0.f), 255.f), 63.f); gbg = grid_round(fminf(fmaxf(hap_fma(fg8, t1, mg), 0.f), 255.f), 63.f);
            gab = grid_round(fminf(fmaxf(hap_fma(fb8, t0, mb), 0.f), 255.f), 31.f); gbb = grid_round(fminf(fmaxf(hap_fma(fb8, t1, mb), 0.f), 255.f), 31.f);
        } else {
            // Lloyd rounds on the quantised problem: re-cluster against the snapped segment, re-solve, re-snap
#pragma unroll 1
            for (int rs = 0; rs < HAP_RGB_RESNAP; rs++) {
                const int ear = (int)expand5((uint32_t)(int)gar), eag = (int)expand6((uint32_t)(int)gag), eab = (int)expand5((uint32_t)(int)gab);
                const int sr_ = (int)expand5((uint32_t)(int)gbr) - ear, sg_ = (int)expand6((uint32_t)(int)gbg) - eag, sb_ = (int)expand5((uint32_t)(int)gbb) - eab;
                // projection of the texels on the snapped segment, p = ((x - ea) . s') / (s . s') with s' = s / 2 as signed
                // bytes (p is 0 at ea and 1 at eb exactly; the direction is off by half a unit per channel at most)
                const int hr = sr_ / 2, hg = sg_ / 2, hb = sb_ / 2;
                const int ss = sr_ * hr + sg_ * hg + sb_ * hb;
                if (ss > 0) {
                    const uint32_t seg = pack_s8x3(hr, hg, hb);
                    const int base = -(ear * hr + eag * hg + eab * hb);
                    float p[16];
#pragma unroll
                    for (int t = 0; t < 16; t++) p[t] = (float)hap_dp4a_us(px[t], seg, base);
                    RgbFit N;
                    if (rgb_cluster_sums(p, P, mr, mg, mb, 0.0f, (float)ss, N)) rgb_solve_and_snap(N, mr, mg, mb, gar, gag, gab, gbr, gbg, gbb);
                }
            }
        }
    }
    uint32_t a5r = (uint32_t)(int)gar, a6g = (uint32_t)(int)gag, a5b = (uint32_t)(int)gab;
    uint32_t b5r = (uint32_t)(int)gbr, b6g = (uint32_t)(int)gbg, b5b = (uint32_t)(int)gbb;
    uint32_t c0 = (a5r << 11) | (a6g << 5) | a5b, c1 = (b5r << 11) | (b6g << 5) | b5b;
    Block8 out;
    out.lo = c0 | (c1 << 16);
    out.hi = 0;  // index 0 = c0 in either mode
    if (c0 == c1) return out;
    if (c0 < c1) {
        uint32_t tmp;
        tmp = c0; c0 = c1; c1 = tmp;
        tmp = a5r; a5r = b5r; b5r = tmp;
        tmp = a6g; a6g = b6g; b6g = tmp;
        tmp = a5b; a5b = b5b; b5b = tmp;
        out.lo = c0 | (c1 << 16);
    }
    // exact indices: nearest of the decoder's four palette colours (truncating thirds), DXT numbering 0 = c0, 1 = c1, 2, 3.
    // |x - P|^2 = |x|^2 - 2 x.P + |P|^2 and x.P = x.(P - 128) + 128 (R + G + B): the first and the last term are the same for
    // all four colours, so compare  |P|^2 - 2 x.(P - 128), the dot product being one DP4A with P - 128 as signed bytes
    const int e0r = (int)expand5(a5r), e0g = (int)expand6(a6g), e0b = (int)expand5(a5b);
    const int e1r = (int)expand5(b5r), e1g = (int)expand6(b6g), e1b = (int)expand5(b5b);
    const int q2r = (int)((uint32_t)(2 * e0r + e1r) / 3u), q2g = (int)((uint32_t)(2 * e0g + e1g) / 3u), q2b = (int)((uint32_t)(2 * e0b + e1b) / 3u);
    const int q3r = (int)((uint32_t)(e0r + 2 * e1r) / 3u), q3g = (int)((uint32_t)(e0g + 2 * e1g) / 3u), q3b = (int)((uint32_t)(e0b + 2 * e1b) / 3u);
    const uint32_t w0 = pack_s8x3(e0r - 128, e0g - 128, e0b - 128), w1 = pack_s8x3(e1r - 128, e1g - 128, e1b - 128);
    const uint32_t w2 = pack_s8x3(q2r - 128, q2g - 128, q2b - 128), w3 = pack_s8x3(q3r - 128, q3g - 128, q3b - 128);
    const int n0 = e0r * e0r + e0g * e0g + e0b * e0b, n1 = e1r * e1r + e1g * e1g + e1b * e1b;
    const int n2 = q2r * q2r + q2g * q2g + q2b * q2b, n3 = q3r * q3r + q3g * q3g + q3b * q3b;
    uint32_t bits = 0;
#pragma unroll
    for (int t = 0; t < 16; t++) {
        const int d0 = n0 - 2 * hap_dp4a_us(px[t], w0, 0), d1 = n1 - 2 * hap_dp4a_us(px[t], w1, 0);
        const int d2 = n2 - 2 * hap_dp4a_us(px[t], w2, 0), d3 = n3 - 2 * hap_dp4a_us(px[t], w3, 0);
        const uint32_t i01 = d1 < d0 ? 1u : 0u, i23 = d3 < d2 ? 3u : 2u;
        const int m01 = d1 < d0 ? d1 : d0, m23 = d3 < d2 ? d3 : d2;
        bits |= (m23 < m01 ? i23 : i01) << (2 * t);
    }
    out.hi = bits;
    return out;
}

// ---- whole-block encoders: px = 16 RGBA8 texels, row-major inside the block, little-endian ------
HAP_HD bool block_is_flat_rgb(const uint32_t px[16])
{
    uint32_t diff = 0;
#pragma unroll
    for (int t = 1; t < 16; t++) diff |= px[t] ^ px[0];
    return (diff & 0x00FFFFFFu) == 0;
}

HAP_HD Block8 encode_dxt1(const uint32_t px[16])
{
    if (block_is_flat_rgb(px))
        return encode_flat_colour((int)(px[0] & 0xFF), (int)((px[0] >> 8) & 0xFF), (int)((px[0] >> 16) & 0xFF), -1, 1.f, 1.f, 1.f);
    return encode_rgb_block(px);
}

HAP_HD Block8 encode_rgtc1_alpha(const uint32_t px[16])
{
    int a7[16];
#pragma unroll
    for (int t = 0; t < 16; t++) a7[t] = hap_dp4a_us(px[t], 0x07000000u, 0);  // 7 * alpha
    int hi = a7[0], lo = a7[0];
#pragma unroll
    for (int t = 1; t < 15; t += 2) { hi = hap_max3(hi, a7[t], a7[t + 1]); lo = hap_min3(lo, a7[t], a7[t + 1]); }
    hi = hap_max3(hi, a7[15], a7[15]); lo = hap_min3(lo, a7[15], a7[15]);
    return encode_bc4_scaled<7>(a7, hi, lo);
}

HAP_HD void encode_dxt5(const uint32_t px[16], Block8 &alpha, Block8 &colour)
{
    alpha = encode_rgtc1_alpha(px);
    colour = encode_dxt1(px);
}

template <bool REFINE = false>
HAP_HD void encode_ycocg_dxt5(const uint32_t px[16], Block8 &alpha, Block8 &colour)
{
    if (block_is_flat_rgb(px)) {
        const int R = (int)(px[0] & 0xFF), G = (int)((px[0] >> 8) & 0xFF), B = (int)((px[0] >> 16) & 0xFF);
        const int co2 = R - B, cg4 = -R + 2 * G - B;
        const int a2 = co2 < 0 ? -co2 : co2, a4 = cg4 < 0 ? -cg4 : cg4;
        const int scale = (a2 * 4 <= 254 && a4 * 4 <= 508) ? 4 : (a2 * 2 <= 254 && a4 * 2 <= 508) ? 2 : 1;
        const int co = hap_clampi(((co2 * scale + 1) >> 1) + 128, 0, 255), cg = hap_clampi(((cg4 * scale + 2) >> 2) + 128, 0, 255);
        const uint32_t Y = (uint32_t)((R + 2 * G + B + 2) >> 2);
        alpha.lo = Y | (Y << 8);
        alpha.hi = 0;
        colour = encode_flat_colour(co, cg, (scale - 1) << 3, scale - 1, 2.0f, 3.0f, 1.0f);
        return;
    }
    // texel bytes are R,G,B,A: weights (1,0,-1,0), (-1,2,-1,0) and 7 * (1,2,1,0) as signed bytes, one DP4A each
    int co2[16], cg4[16], y28[16];
#pragma unroll
    for (int t = 0; t < 16; t++) {
        co2[t] = hap_dp4a_us(px[t], 0x00FF0001u, 0);
        cg4[t] = hap_dp4a_us(px[t], 0x00FF02FFu, 0);
        y28[t] = hap_dp4a_us(px[t], 0x00070E07u, 0);  // 7 (R + 2G + B) = 28 * luma
    }
    int co_hi = co2[0], co_lo = co2[0], cg_hi = cg4[0], cg_lo = cg4[0], y_hi = y28[0], y_lo = y28[0];
#pragma unroll
    for (int t = 1; t < 15; t += 2) {
        co_hi = hap_max3(co_hi, co2[t], co2[t + 1]); co_lo = hap_min3(co_lo, co2[t], co2[t + 1]);
        cg_hi = hap_max3(cg_hi, cg4[t], cg4[t + 1]); cg_lo = hap_min3(cg_lo, cg4[t], cg4[t + 1]);
        y_hi = hap_max3(y_hi, y28[t], y28[t + 1]); y_lo = hap_min3(y_lo, y28[t], y28[t + 1]);
    }
    co_hi = hap_max3(co_hi, co2[15], co2[15]); co_lo = hap_min3(co_lo, co2[15], co2[15]);
    cg_hi = hap_max3(cg_hi, cg4[15], cg4[15]); cg_lo = hap_min3(cg_lo, cg4[15], cg4[15]);
    y_hi = hap_max3(y_hi, y28[15], y28[15]); y_lo = hap_min3(y_lo, y28[15], y28[15]);
    alpha = encode_bc4_scaled<28>(y28, y_hi, y_lo);
    colour = encode_ycocg_chroma<REFINE>(co2, cg4, co_hi, co_lo, cg_hi, cg_lo);
}

}  // namespace hapb200
