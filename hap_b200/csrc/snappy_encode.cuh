// hap_b200/csrc/snappy_encode.cuh -- K5: second-stage compressor for one fragment of a Hap chunk.
//
// Replaces snappy_compress as the reference calls it from the chunk loop of hap_encode_texture
// (/root/reference/source/hap.c:448-476, call site :453).  The reference's loop is serial over chunks
// and Snappy is serial inside a chunk; here a chunk is cut into independent 32 KiB FRAGMENTS (a raw
// Snappy stream is varint(length) followed by elements, so fragment element streams concatenate
// into one legal chunk stream as long as copies never reach outside their fragment), a persistent grid
// of CTAs (two per SM) striding over the fragments, and inside a fragment every 8-byte unit is handled on its own:
//   1. first-occurrence hash of every aligned word (shared-memory table, atomicMin => deterministic);
//   2. each word picks a source: the word one DXT block back when its whole block repeats the
//      previous block (block RLE, decodes as one periodic fill), else the first earlier occurrence
//      of the same word.  Choosing FIRST occurrences makes copies point at literal data, so the
//      decoder's dependency depth stays ~1 (see snappy_decode.cuh);
//   3. runs of words with one distance become copy elements (<= 64 bytes each), everything else
//      literal runs; element sizes are prefix-summed and every word writes its own bytes (for this
//      last step the words are re-dealt so that the lanes of a warp write neighbouring bytes).
// The output differs from Google's encoder byte-for-byte (the reference pins no Snappy bytes,
// SURVEY.md 8c); parity is: the reference's HapDecode reproduces the input exactly.
#pragma once
#include "hap_codes.h"
#include "hap_index.h"
#include "simt.h"

namespace hapb200 {

constexpr int kEncThreads = 512;        // two CTAs per SM: 2 x 512 threads x 64 registers fill the register file
constexpr int kEncWarps = kEncThreads / 32;
constexpr int kFragBytes = 32768;
constexpr int kFragCap = kFragBytes + 32;   // element stream of a fragment never exceeds n + 3
constexpr int kEncHashBits = 13;
constexpr uint32_t kFragStoredRaw = 0xFFFFFFFFu;  // fragment size marker: chunk must be stored raw
constexpr int kFragEntryPieces = (kFragCap + (1 << kIndexSubLog2) - 1) >> kIndexSubLog2;   // 128-byte pieces of a fragment's stream (hap_index.h)
constexpr int kFragEntryStride = 272;             // bytes reserved per fragment in the entries scratch (multiple of 16)
static_assert(kFragEntryPieces <= kFragEntryStride, "entries of one fragment fit their scratch slot");

// Shared memory of one fragment.  The unit of every decision is 8 BYTES (a DXT1 / RGTC1 block, half a DXT5 block): thread t
// owns the 8 consecutive units [8t, 8t+8) and keeps them (and every per-unit quantity) in registers; shared memory only
// carries what OTHER threads read: the data (random match verification), the hash table, the strip-boundary values of the
// per-unit arrays, and -- for the last step, which re-distributes the units over the threads -- positions, run starts and
// distances.  (Round 1 decided per 4-byte word: twice the elements in every step, and 4-byte matches that were demoted
// again because a copy element costs 3 bytes.  Matches that start at an odd word are lost; DXT payloads hardly have any.)
constexpr int kFragUnits = kFragBytes / 8;        // 4096
constexpr int kUnitStrip = kFragUnits / kEncThreads;   // 8 units per thread
static_assert(kUnitStrip == 8, "the strip code below moves 8 uint16 values per thread as one 16-byte access");
struct EncodeSmem {
    uint2 data[kFragUnits + 2];                     // input units
    union {
        uint32_t table[1 << kEncHashBits];          // first occurrence of every hashed unit
        struct {
            uint16_t a[kFragUnits];                 // final distance per unit (written by the propagation once the table is dead)
            uint16_t b[kFragUnits];                 // run start per unit
            uint16_t c[kFragUnits];                 // stream position per unit
        } h;
    } u;
    uint16_t da[kFragUnits];                        // candidate distances, then the run ends (stored at the run start)
    uint32_t warp_tot[kEncWarps];
    uint32_t entry[kFragEntryStride];               // fragment index: offset of the first element start in every 128 bytes of the stream
    uint32_t total;
    alignas(16) uint32_t out[(kFragCap + 3) / 4 + 6];   // the element stream (copied out in 16-byte words)
    uint32_t place[6];                              // hapq_fused_place_kernel: ticket and the fragment waiting in `out`
};
// Two CTAs per SM: an H100 SM has 228 KiB of shared memory for CTAs and reserves 1 KiB of it per CTA, so each of two CTAs
// may use (233,472 - 2 x 1,024) / 2 = 115,712 bytes.
static_assert(sizeof(EncodeSmem) <= 115712, "two encode CTAs fit the shared memory of one SM");

// -DHAPB200_ENC_PHASE_CLOCKS=1 (measurement builds only, tools/measure_enc_phases.py): thread 0 of the compressor (and,
// in hapq_ws_place_kernel, thread 0 of the fit group, thread kEncThreads) adds up clock64() per phase of the fused Hap Q
// encoders in shared memory, and thread 0 folds the sums into g_enc_phase_clocks when the CTA ends.  Phases end at barriers
// where there is one, so a phase's clocks are those of its warp group, not of one thread alone.
#ifndef HAPB200_ENC_PHASE_CLOCKS
#define HAPB200_ENC_PHASE_CLOCKS 0
#endif
enum : int {
    kEpFit = 0,          // the fit
    kEpFitWait,          // the barrier behind the fit (hapq_ws_place_kernel: the compressor waits for a fitted image)
    kEpHash, kEpCandidates, kEpPropagate, kEpRunScan, kEpSizeScan, kEpWrite,   // compress_fragment's steps 1 .. 5
    kEpLookBack,         // the look-back of the fragment whose stream waits in shared memory, and the barrier behind it
    kEpStore,            // its stream to the frame
    kEpOther,            // table clear, strip load, ticket, size publication
    kEpGroupFit,         // hapq_ws_place_kernel's fit group: fitting
    kEpGroupEmptyWait,   // ... waiting for the compressor to release an image
    kEpGroupTicket,      // ... handing out the ticket inside the group
    kEpCount
};
enum : int { kEpFragments = kEpCount, kEpSlots };   // fragments compressed, kept behind the phase clocks
#if HAPB200_ENC_PHASE_CLOCKS && !defined(HAPB200_EMU)
__device__ unsigned long long g_enc_phase_clocks[kEpSlots];
__shared__ unsigned long long s_enc_phase[kEpSlots + 2];   // [kEpSlots + w]: clock of warp group w's last mark
#define HAP_EPHASE_BEGIN()                                                                \
    do {                                                                                  \
        if (threadIdx.x == 0)                                                             \
            for (int q_ = 0; q_ < kEpSlots; q_++) s_enc_phase[q_] = 0;                    \
        __syncthreads();                                                                  \
        if ((threadIdx.x & (kEncThreads - 1)) == 0) s_enc_phase[kEpSlots + threadIdx.x / kEncThreads] = clock64(); \
    } while (0)
#define HAP_EPHASE_MARK(ph)                                                               \
    do {                                                                                  \
        if ((threadIdx.x & (kEncThreads - 1)) == 0) {                                     \
            const unsigned long long c_ = clock64();                                      \
            unsigned long long &l_ = s_enc_phase[kEpSlots + threadIdx.x / kEncThreads];   \
            s_enc_phase[ph] += c_ - l_;                                                   \
            l_ = c_;                                                                      \
        }                                                                                 \
    } while (0)
#define HAP_EPHASE_COUNT(slot)                                                            \
    do {                                                                                  \
        if (threadIdx.x == 0) s_enc_phase[slot]++;                                        \
    } while (0)
#define HAP_EPHASE_END()                                                                  \
    do {                                                                                  \
        __syncthreads();                                                                  \
        if (threadIdx.x == 0)                                                             \
            for (int q_ = 0; q_ < kEpSlots; q_++) atomicAdd(&g_enc_phase_clocks[q_], s_enc_phase[q_]); \
    } while (0)
#else
#define HAP_EPHASE_BEGIN() do {} while (0)
#define HAP_EPHASE_MARK(ph) do {} while (0)
#define HAP_EPHASE_COUNT(slot) do {} while (0)
#define HAP_EPHASE_END() do {} while (0)
#endif

__device__ __forceinline__ uint32_t enc_hash(uint2 u) { return ((u.x * 0x9E3779B1u) ^ (u.y * 0x85EBCA6Bu)) >> (32 - kEncHashBits); }
__device__ __forceinline__ bool same_unit(uint2 a, uint2 b) { return a.x == b.x && a.y == b.y; }

__device__ __forceinline__ uint32_t literal_header_bytes(uint32_t len) { return len <= 60 ? 1u : len <= 256 ? 2u : 3u; }

__device__ __forceinline__ void store_strip16(uint16_t *arr, uint32_t base, const uint32_t v[kUnitStrip])
{
    *reinterpret_cast<uint4 *>(arr + base) = make_uint4(v[0] | (v[1] << 16), v[2] | (v[3] << 16), v[4] | (v[5] << 16), v[6] | (v[7] << 16));
}

// The barrier the compressor's kEncThreads threads meet at: the whole CTA (K5, the fused kernels), or a named barrier of
// the compressor's warp group when the CTA has other warps too (hapq_ws_place_kernel).
struct CtaBarrier {
    __device__ static __forceinline__ void sync() { __syncthreads(); }
};
template <int ID>
struct GroupBarrier {
    __device__ static __forceinline__ void sync() { hap_bar_sync(ID, kEncThreads); }
};

// Inclusive max / sum over the block of one value per thread; returns the exclusive prefix for this thread and
// the block total.  Two barriers.  The warp totals are scanned by every warp with shuffles (lane w holds the
// total of warp w; lanes past the last warp hold the identity, 0 for both) instead of a loop over shared memory.
template <class Bar = CtaBarrier>
__device__ __forceinline__ uint32_t enc_block_excl(uint32_t v, bool is_max, uint32_t *total, uint32_t *warp_tot)
{
    static_assert(kEncWarps <= 32, "one warp total per lane");
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t o = __shfl_up_sync(HAP_FULL_MASK, incl, d);
        if (lane >= d) incl = is_max ? (incl > o ? incl : o) : incl + o;
    }
    uint32_t prev = __shfl_up_sync(HAP_FULL_MASK, incl, 1);
    if (lane == 0) prev = 0;
    if (lane == 31) warp_tot[warp] = incl;
    Bar::sync();
    uint32_t wi = lane < kEncWarps ? warp_tot[lane] : 0u;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t o = __shfl_up_sync(HAP_FULL_MASK, wi, d);
        if (lane >= d) wi = is_max ? (wi > o ? wi : o) : wi + o;
    }
    const uint32_t tot = __shfl_sync(HAP_FULL_MASK, wi, 31);
    uint32_t base = __shfl_sync(HAP_FULL_MASK, wi, warp > 0 ? warp - 1 : 0);
    if (warp == 0) base = 0;
    Bar::sync();
    *total = tot;
    return is_max ? (base > prev ? base : prev) : base + prev;
}

// One fragment: U units (8 bytes each; U <= kFragUnits) already in the shared-memory image `data` (S.data, or a second
// image of the same size) AND in the caller's registers d[8] (units 8t..8t+7) -> element stream written to `out` (S.out,
// or a second buffer of the same size) as bytes; returns its size (all threads).
// period_units = DXT block size in units (1 or 2).
// FULL = the fragment has all kFragUnits units (31 of 32 fragments of a 1 MiB chunk): every per-unit bounds test
// folds away at compile time.  Bar: the barrier of the kEncThreads threads that run it.
template <bool FULL, class Bar = CtaBarrier>
__device__ __forceinline__ uint32_t compress_fragment(EncodeSmem &S, const uint2 *data, uint32_t *out_words, const uint2 d[kUnitStrip],
                                                      uint32_t Udyn, uint32_t period_units)
{
    const uint32_t t = threadIdx.x;
    const uint32_t U = FULL ? (uint32_t)kFragUnits : Udyn;
    const uint32_t i0 = t * kUnitStrip;              // first unit of my strip
    const uint32_t nv = FULL ? (uint32_t)kUnitStrip : (i0 >= U ? 0u : (U - i0 < (uint32_t)kUnitStrip ? U - i0 : (uint32_t)kUnitStrip));  // my valid units

    // 1. first occurrence of every unit (the table was initialised by the caller, before the barrier).  A unit whose hash
    //    equals that of one of the two units before it leaves the atomicMin to that lower unit: the table ends the same,
    //    and on flat content (letterbox bars, repeated blocks) a warp no longer sends 32 lanes to one address.
    uint32_t hsh[kUnitStrip];
#pragma unroll
    for (int k = 0; k < kUnitStrip; k++) hsh[k] = enc_hash(d[k]);
    {
        const uint32_t lane = t & 31;
        const uint32_t p1 = __shfl_up_sync(HAP_FULL_MASK, hsh[kUnitStrip - 1], 1), p2 = __shfl_up_sync(HAP_FULL_MASK, hsh[kUnitStrip - 2], 1);
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) {
            const bool has1 = k >= 1 || lane > 0, has2 = k >= 2 || lane > 0;
            const uint32_t h1 = k >= 1 ? hsh[k - 1] : p1, h2 = k >= 2 ? hsh[k - 2] : k == 1 ? p1 : p2;
            const bool dup = (has1 && h1 == hsh[k]) || (has2 && h2 == hsh[k]);
            if ((uint32_t)k < nv && !dup) atomicMin(&S.u.table[hsh[k]], i0 + k);
        }
    }
    Bar::sync();
    HAP_EPHASE_MARK(kEpHash);

    // 2. candidate distance per unit: first earlier occurrence, or one block back when the whole block repeats
    uint32_t dd[kUnitStrip];
#pragma unroll
    for (int k = 0; k < kUnitStrip; k++) {
        dd[k] = 0;
        if ((uint32_t)k < nv) {
            const uint32_t c = S.u.table[hsh[k]];
            if (c < i0 + k && same_unit(data[c], d[k])) dd[k] = i0 + k - c;
        }
    }
    if (period_units == 2) {
        // DXT5-sized blocks: units (2b, 2b+1); the block repeats when both of its units exist and equal the block before
        const uint2 p0 = i0 >= 2 ? data[i0 - 2] : make_uint2(0, 0), p1 = i0 >= 2 ? data[i0 - 1] : make_uint2(0, 0);
        if (i0 >= 2 && nv >= 2 && same_unit(p0, d[0]) && same_unit(p1, d[1])) { dd[0] = 2; dd[1] = 2; }
#pragma unroll
        for (int k = 2; k < kUnitStrip; k += 2)
            if ((uint32_t)k + 2 <= nv && same_unit(d[k - 2], d[k]) && same_unit(d[k - 1], d[k + 1])) { dd[k] = 2; dd[k + 1] = 2; }
    } else {
        const uint2 p = i0 >= 1 ? data[i0 - 1] : make_uint2(0, 0);
        if (i0 >= 1 && nv >= 1 && same_unit(p, d[0])) dd[0] = 1;
#pragma unroll
        for (int k = 1; k < kUnitStrip; k++)
            if ((uint32_t)k < nv && same_unit(d[k - 1], d[k])) dd[k] = 1;
    }
    store_strip16(S.da, i0, dd);
    Bar::sync();
    HAP_EPHASE_MARK(kEpCandidates);

    // 2b. propagation (one round): a unit that is not yet part of a run adopts its left (else right) neighbour's
    //     distance when its own data also matches there.  First occurrences of neighbouring units often point at
    //     different earlier blocks; this re-aligns them and recovers most of what a greedy match extension finds.
    //     Every unit decides from the distances before the round (S.da), so the result does not depend on the order
    //     in which threads run.  (Measured on the emulator cases: with 8-byte units ONE round recovers what two did --
    //     frame sizes equal on picture content, +0.1 .. 0.5 % on the stitched random cases; none costs 5 .. 16 %.)
    {
        const uint32_t lb = i0 > 0 ? S.da[i0 - 1] : 0u;
        const uint32_t rb = i0 + kUnitStrip < U ? S.da[i0 + kUnitStrip] : 0u;
        uint32_t l = lb;   // the left neighbour's distance before the round
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) {
            const uint32_t r = k < kUnitStrip - 1 ? dd[k + 1] : rb;
            const uint32_t cd = dd[k], i = i0 + k;
            if ((uint32_t)k < nv && !(cd != 0 && (cd == l || cd == r))) {
                // one look-up decides: the left neighbour's distance if there is one, else the right one's
                const uint32_t cand = l != 0 ? l : r;
                if (cand != 0 && i >= cand && same_unit(data[i - cand], d[k])) dd[k] = cand;
                else if (l != 0 && r != 0 && r != l && i >= r && same_unit(data[i - r], d[k])) dd[k] = r;
            }
            l = cd;
        }
    }
    // The hash table is dead since the barrier above: its space takes the final distances (read across strip boundaries
    // below and by the re-dealt output step); S.da is free once every thread has read its neighbours there, and takes
    // the run ends.  (A single matching unit is kept: an 8-byte copy costs 3 bytes.)
    store_strip16(S.u.h.a, i0, dd);
    Bar::sync();
    HAP_EPHASE_MARK(kEpPropagate);
    const uint16_t *fin = S.u.h.a;
    uint16_t *ends = S.da;

    // 3. run start of every unit (max-scan of "i+1 where a run starts") and run ends (stored at the run start)
    uint32_t rs[kUnitStrip];
    {
        const uint32_t lb = i0 > 0 ? fin[i0 - 1] : 0u;
        uint32_t last = 0;  // (index + 1) of the last run start inside my strip so far
        uint32_t loc[kUnitStrip];
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) {
            const uint32_t prev = k > 0 ? dd[k - 1] : lb;
            if ((uint32_t)k < nv && (i0 + k == 0 || dd[k] != prev)) last = i0 + k + 1;
            loc[k] = last;
        }
        uint32_t unused;
        const uint32_t carry = enc_block_excl<Bar>(last, true, &unused, S.warp_tot);
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) rs[k] = (loc[k] ? loc[k] : carry) - 1;
        const uint32_t rb = i0 + kUnitStrip < U ? fin[i0 + kUnitStrip] : 0xFFFFFFFFu;
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) {
            const uint32_t nx = k < kUnitStrip - 1 ? dd[k + 1] : rb;
            if ((uint32_t)k < nv && (i0 + k + 1 == U || nx != dd[k])) ends[rs[k]] = (uint16_t)(i0 + k);
        }
    }
    Bar::sync();
    HAP_EPHASE_MARK(kEpRunScan);

    // 4. bytes each unit contributes and their exclusive prefix sum
    uint32_t pos[kUnitStrip];
    {
        uint32_t run = 0;
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) {
            uint32_t c = 0;
            if ((uint32_t)k < nv) {
                const uint32_t i = i0 + k;
                if (dd[k] == 0) {
                    c = 8;
                    if (i == rs[k]) c += literal_header_bytes(8u * (ends[i] - i + 1));
                } else if (((i - rs[k]) & 7) == 0) {
                    c = 3;      // one copy element per 64 bytes of the run
                }
            }
            pos[k] = run;
            run += c;
        }
        uint32_t tot;
        const uint32_t base = enc_block_excl<Bar>(run, false, &tot, S.warp_tot);
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) pos[k] += base;
        if (t == 0) S.total = tot;
    }

    // 5. every unit writes its own bytes.  Ownership changes for this step: thread t takes units t, t + 512, ... so that
    //    the lanes of a warp write neighbouring bytes of the stream (with the strip layout they sit 64 bytes apart: bank
    //    conflicts on every store).  Positions, run starts and distances travel through shared memory as 16-bit strips.
    //    Inside a literal run the stream is the input shifted by (p & 3) bytes, so a unit writes TWO aligned 32-bit words
    //    made of its own bytes and the next unit's first bytes; only the two ends of a run, headers and copy elements are
    //    written bytewise.
    store_strip16(S.u.h.c, i0, pos);
    store_strip16(S.u.h.b, i0, rs);
    Bar::sync();
    HAP_EPHASE_MARK(kEpSizeScan);
    uint8_t *out = reinterpret_cast<uint8_t *>(out_words);
#pragma unroll 1
    for (int j = 0; j < kUnitStrip; j++) {
        const uint32_t i = t + (uint32_t)j * kEncThreads;
        if (!FULL && i >= U) continue;
        const uint32_t dist = S.u.h.a[i], rs_i = S.u.h.b[i];
        uint32_t p = S.u.h.c[i];
        if (dist == 0) {
            const uint2 w = data[i];
            const uint32_t e = ends[rs_i];   // last unit of this literal run
            if (i == rs_i) {
                const uint32_t len = 8u * (e - i + 1);
                atomicMin(&S.entry[p >> kIndexSubLog2], p & ((1u << kIndexSubLog2) - 1u));   // an element starts here
                if (len <= 60) {
                    out[p++] = (uint8_t)((len - 1) << 2);
                } else if (len <= 256) {
                    out[p++] = (uint8_t)(60 << 2);
                    out[p++] = (uint8_t)(len - 1);
                } else {
                    out[p++] = (uint8_t)(61 << 2);
                    out[p++] = (uint8_t)(len - 1);
                    out[p++] = (uint8_t)((len - 1) >> 8);
                }
            }
            const uint32_t sh = p & 3u;
            if (sh == 0) {
                *reinterpret_cast<uint32_t *>(out + p) = w.x;
                *reinterpret_cast<uint32_t *>(out + p + 4) = w.y;
            } else {
                const uint32_t a1 = (p & ~3u) + 4u;   // the first aligned word behind p
                if (i == rs_i)
                    for (uint32_t q = 0; q < 4u - sh; q++) out[p + q] = (uint8_t)(w.x >> (8 * q));   // the run's first bytes
                *reinterpret_cast<uint32_t *>(out + a1) = __funnelshift_r(w.x, w.y, 8 * (4u - sh));
                if (i < e) {
                    *reinterpret_cast<uint32_t *>(out + a1 + 4) = __funnelshift_r(w.y, data[i + 1].x, 8 * (4u - sh));
                } else {
                    for (uint32_t q = 0; q < sh; q++) out[a1 + 4 + q] = (uint8_t)(w.y >> (8 * (4u - sh + q)));   // the run's last bytes
                }
            }
        } else if (((i - rs_i) & 7) == 0) {
            const uint32_t left = ends[rs_i] - i + 1;          // units left in the run
            const uint32_t len = 8u * (left < 8 ? left : 8);    // 8..64 bytes
            const uint32_t off = 8u * dist;
            atomicMin(&S.entry[p >> kIndexSubLog2], p & ((1u << kIndexSubLog2) - 1u));       // an element starts here
            out[p] = (uint8_t)(2u | ((len - 1) << 2));          // copy with 2-byte offset
            out[p + 1] = (uint8_t)off;
            out[p + 2] = (uint8_t)(off >> 8);
        }
    }
    Bar::sync();
    HAP_EPHASE_MARK(kEpWrite);
    return S.total;
}

// Geometry of one texture section of a batch of identical frames (host fills it once per call).
struct SectionGeom {
    uint32_t bytes;            // texture bytes (hap.c: inputBufferBytes)
    uint32_t chunks;           // limited chunk count (hap.c:277-300)
    uint32_t chunk_bytes;      // bytes / chunks (hap.c:433)
    uint32_t frags_per_chunk;  // ceil(chunk_bytes / kFragBytes)
    uint32_t period_words;     // DXT block size in 4-byte words (2 or 4)
    uint32_t compress;         // 1 = HapCompressorSnappy requested and chunk_bytes % 8 == 0
    uint32_t inv_frags_per_chunk;  // floor(2^32 / frags_per_chunk), 0xFFFFFFFF for 1 (fast_divmod)
    uint32_t frag_base;        // index of this section's first fragment inside a frame
    uint32_t fmt_nibble;       // wire format id (hap.c:45-51)
    uint32_t top_hdr;          // 4 or 8 (hap.c:398-405, :425-428)
    uint32_t want_snappy;      // caller passed HapCompressorSnappy
    uint64_t in_offset;        // this texture's bytes of frame f start at dxt + in_offset + f * in_stride
    uint64_t in_stride;
};

struct FrameGeom {
    uint32_t sections;         // 1 or 2
    uint32_t outer_hdr;        // 0 (single texture), 4 or 8 (hap.c:563-576)
    uint32_t frags_per_frame;
    uint32_t inv_frags_per_frame;  // floor(2^32 / frags_per_frame), 0xFFFFFFFF for 1
    SectionGeom s[2];
};

// Where fragment `gfrag` of the batch lives and how long it is.
struct FragRef {
    const uint8_t *in;
    bool second;         // fragment of the frame's second texture
    uint32_t units;      // 8-byte units; 0: the section is not compressed (fragment stored raw)
    uint32_t frame;      // frame of the batch
    uint32_t tex_off;    // byte offset of the fragment inside its texture
};
// x / d and x % d with a multiplication: magic = floor(2^32 / d) (0xFFFFFFFF for d = 1), one correction step
__device__ __forceinline__ uint32_t fast_divmod(uint32_t x, uint32_t d, uint32_t magic, uint32_t &rem)
{
#ifdef HAPB200_EMU
    rem = x % d;
    (void)magic;
    return x / d;
#else
    uint32_t q = __umulhi(x, magic);
    uint32_t r = x - q * d;
    while (r >= d) { q++; r -= d; }
    rem = r;
    return q;
#endif
}
__device__ __forceinline__ FragRef locate_fragment(const uint8_t *dxt, const FrameGeom &G, uint32_t gfrag)
{
    uint32_t f;
    const uint32_t frame = fast_divmod(gfrag, G.frags_per_frame, G.inv_frags_per_frame, f);
    const bool second = G.sections == 2 && f >= G.s[1].frag_base;
    const uint32_t frag_base = second ? G.s[1].frag_base : G.s[0].frag_base, fpc = second ? G.s[1].frags_per_chunk : G.s[0].frags_per_chunk;
    const uint32_t inv_fpc = second ? G.s[1].inv_frags_per_chunk : G.s[0].inv_frags_per_chunk;
    const uint32_t chunk_bytes = second ? G.s[1].chunk_bytes : G.s[0].chunk_bytes, compress = second ? G.s[1].compress : G.s[0].compress;
    const uint64_t in_stride = second ? G.s[1].in_stride : G.s[0].in_stride, in_offset = second ? G.s[1].in_offset : G.s[0].in_offset;
    uint32_t j;
    const uint32_t chunk = fast_divmod(f - frag_base, fpc, inv_fpc, j);
    FragRef r;
    r.in = dxt + (uint64_t)frame * in_stride + in_offset + (uint64_t)chunk * chunk_bytes + (uint64_t)j * kFragBytes;
    const uint32_t left = chunk_bytes - j * kFragBytes;
    r.units = compress ? (left < (uint32_t)kFragBytes ? left : (uint32_t)kFragBytes) >> 3 : 0u;
    r.second = second;
    r.frame = frame;
    r.tex_off = chunk * chunk_bytes + j * (uint32_t)kFragBytes;   // (a section is under 2 GiB: build_frame_geom)
    return r;
}

// A thread's 8 units of a fragment, from global memory: four 16-byte loads when possible
__device__ __forceinline__ void load_strip(const FragRef &fr, uint32_t i0, uint2 d[kUnitStrip])
{
    if ((((uintptr_t)fr.in) & 15) == 0 && i0 + kUnitStrip <= fr.units) {
        const uint4 *in4 = reinterpret_cast<const uint4 *>(fr.in) + (i0 >> 1);
#pragma unroll
        for (int k = 0; k < kUnitStrip / 2; k++) {
            const uint4 a = in4[k];
            d[2 * k] = make_uint2(a.x, a.y);
            d[2 * k + 1] = make_uint2(a.z, a.w);
        }
    } else {
#pragma unroll
        for (int k = 0; k < kUnitStrip; k++) {
            const uint32_t i = i0 + k;
            d[k] = make_uint2(0, 0);
            if (i < fr.units) {
                const uint8_t *b = fr.in + 8 * (size_t)i;
                d[k].x = b[0] | (b[1] << 8) | (b[2] << 16) | ((uint32_t)b[3] << 24);
                d[k].y = b[4] | (b[5] << 8) | (b[6] << 16) | ((uint32_t)b[7] << 24);
            }
        }
    }
}

// Copies fragment gfrag's element stream (`total` bytes in S.out) and index entries out of shared memory, records its size,
// and waits until every thread is done with the fragment's shared memory.
__device__ __forceinline__ void store_fragment(const EncodeSmem &S, uint32_t total, uint32_t gfrag, uint8_t *__restrict__ scratch,
                                               uint32_t *__restrict__ frag_size, uint8_t *__restrict__ frag_entries)
{
    const uint32_t t = threadIdx.x;
    uint8_t *o = scratch + (uint64_t)gfrag * kFragCap;
    const uint4 *o4s = reinterpret_cast<const uint4 *>(S.out);
    uint4 *o4 = reinterpret_cast<uint4 *>(o);       // (scratch slots are kFragCap = 32800 bytes apart: 16-byte aligned)
    for (uint32_t i = t; i < (total + 15) / 16; i += kEncThreads) o4[i] = o4s[i];
    if (frag_entries != nullptr && t < kFragEntryStride) frag_entries[(uint64_t)gfrag * kFragEntryStride + t] = (uint8_t)S.entry[t];
    if (t == 0) frag_size[gfrag] = total;
    __syncthreads();   // S.out, S.data and the tables are rewritten by the next fragment
}

// The table and the index entries of a fragment start empty (before the barrier in front of compress_fragment).
__device__ __forceinline__ void init_fragment_tables(EncodeSmem &S)
{
    const int t = threadIdx.x;
    uint4 *tb = reinterpret_cast<uint4 *>(S.u.table);
    const uint4 ones = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
    for (int q = t; q < (1 << kEncHashBits) / 4; q += kEncThreads) tb[q] = ones;
    if (t < kFragEntryStride) S.entry[t] = kIndexNoEntry;
}

// A persistent grid (as many CTAs as fit on the device at once: two per SM, the kernel needs 108 KB of shared memory)
// strides over the nfrag = frames * frags_per_frame fragments of the batch.  While one CTA of an SM waits at a barrier
// or for the HBM latency of its next fragment's input, the other one computes.
// dxt: base pointer of the texture bytes; scratch: [nfrag][kFragCap]; frag_size: [nfrag] (kFragStoredRaw when the
// fragment was not compressed); frag_entries: [nfrag][kFragEntryStride] or nullptr (fragment index, hap_index.h).
__global__ void __launch_bounds__(kEncThreads, 2) snappy_encode_fragments_kernel(
    const uint8_t *__restrict__ dxt, FrameGeom G, uint32_t nfrag, uint8_t *__restrict__ scratch, uint32_t *__restrict__ frag_size,
    uint8_t *__restrict__ frag_entries)
{
    HAP_DYN_SMEM(smem_raw);
    EncodeSmem &S = *reinterpret_cast<EncodeSmem *>(smem_raw);
    const int t = threadIdx.x;
    const uint32_t i0 = (uint32_t)t * kUnitStrip;
    for (uint32_t gfrag = blockIdx.x; gfrag < nfrag; gfrag += gridDim.x) {
        const FragRef cur = locate_fragment(dxt, G, gfrag);
        if (cur.units == 0) {
            if (t == 0) frag_size[gfrag] = kFragStoredRaw;
            continue;
        }
        const uint32_t U = cur.units;
        uint2 d[kUnitStrip];
        load_strip(cur, i0, d);
#pragma unroll
        for (int k = 0; k < kUnitStrip; k += 2) *reinterpret_cast<uint4 *>(&S.data[i0 + k]) = make_uint4(d[k].x, d[k].y, d[k + 1].x, d[k + 1].y);
        init_fragment_tables(S);
        __syncthreads();
        const uint32_t period_units = (cur.second ? G.s[1].period_words : G.s[0].period_words) >> 1;   // 8-byte blocks: 1, 16-byte blocks: 2
        const uint32_t total = U == (uint32_t)kFragUnits ? compress_fragment<true>(S, S.data, S.out, d, U, period_units)
                                                         : compress_fragment<false>(S, S.data, S.out, d, U, period_units);
        store_fragment(S, total, gfrag, scratch, frag_size, frag_entries);
    }
}

}  // namespace hapb200
