// hap_b200/csrc/snappy_decode.cuh -- K7: the second-stage decompressor, as three kernels.
//
// Replaces hap_decode_chunk + snappy_uncompress (/root/reference/source/hap.c:606-642, call sites :612 and :899): a chunk
// of a Hap frame -> its decoded DXT bytes at a fixed destination.  A chunk is one raw Snappy stream (compressor byte
// 0x0B) or a verbatim copy (0x0A).
//
// Snappy is serial twice over: an element's position depends on the length of every element before it, and copies read
// earlier output.  Round 1 broke both chains inside ONE kernel, one CTA per chunk, window after window; every phase of a
// window waited for the slowest thread of the one before it (8 barrier-separated phases, 5.7 % of the HBM roofline).
// Here the two chains are separated, so that only what is serial by nature stays serial:
//
//   snappy_index_kernel (one CTA per chunk that has no index yet; light: 50 KB of shared memory, 4 CTAs per SM)
//       finds the ELEMENT CHAIN and nothing else.  Per 16 KiB of compressed bytes: the bytes arrive by a TMA bulk copy
//       (double buffered: the next window lands while this one is parsed); thread t owns 64 bytes and computes, for EVERY
//       offset o inside them, where an element chain entering at o leaves them (one backward sweep, x[o] = x[o+size(o)],
//       branch-free); one thread hops sub-block to sub-block along the true chain with one table look-up per hop; entered
//       sub-blocks add up their output bytes.  Result: one byte per 64 compressed bytes ("first element start in this
//       sub-block") and the output offset of every window -- the same index this repo's encoder can write into the frame
//       (hap_index.h), in which case this kernel does not run at all.
//   hap_build_windows_kernel (one thread per chunk) turns chunks into WINDOWS: fragments of an indexed chunk, 64 KiB
//       pieces of a verbatim chunk; chunks without an index are left to the kernel above.
//   snappy_execute_kernel (persistent CTAs draw windows from a counter) does everything that touches bytes, window
//       by window in parallel: walk the sub-blocks from their entries, scan element counts / output bytes, describe the
//       elements, flatten copy-of-copy chains (pointer jumping), then produce the OUTPUT-CENTRIC: thread g assembles
//       the 16 aligned output bytes of group g from the one to three elements that cover them and writes them with one
//       128-bit store, so every lane moves the same number of bytes whatever the element lengths are.  Groups whose
//       source bytes are not final yet wait for a later round; windows of an on-the-fly index wait (one acquire) for
//       the earlier windows their copies reach into.  Fragments of an embedded index made of 8-byte elements (this
//       encoder's) skip the descriptors and tiles: they are decoded as 4096 eight-byte units (execute_units).
//   snappy_execute_units_kernel runs before it and decodes those fragments in a kernel of their own that keeps more
//       windows resident per SM; the execute kernel then takes only the windows it left.
// Every decision is taken on device; the host reads one status word per chunk.
#pragma once
#include "block_primitives.cuh"
#include "hap_codes.h"
#include "hap_index.h"
#include "simt.h"

namespace hapb200 {

struct ChunkJob {
    const uint8_t *src;   // compressed (0x0B) or raw (0x0A) chunk bytes
    uint8_t *dst;         // decoded bytes go here
    uint32_t src_bytes;
    uint32_t dst_bytes;   // decoded size the container arithmetic expects (hap.c:813, :833)
    uint32_t compressor;  // kHapCompressorNone 0x0A | kHapCompressorSnappy 0x0B (hap.c:41-42); 0 = unused slot
    uint32_t status;      // out: HapResult of this chunk (hap.c:617-640)
    const uint8_t *index; // this chunk's record inside the frame's fragment index (hap_index.h), or nullptr
    uint32_t index_bytes; // bytes readable at `index`
    uint32_t mode;        // internal, see kJob*
    uint32_t win_base;    // internal: the chunk's windows are wins[win_base .. win_base + win_count)
    uint32_t win_count;
};
// kJobReady: windows listed, first execute pass takes them.  kJobNeedsIndex: waits for the index kernel.  kJobRepaired: indexed
// again after its embedded index failed the execute kernel's checks; the second execute pass takes it.
enum : uint32_t { kJobUndecided = 0, kJobReady = 1, kJobNeedsIndex = 2, kJobRepaired = 3, kJobFinished = 4 };
constexpr uint32_t kStatusIndexMismatch = 0x100;  // internal: the embedded index does not describe the stream -> decode again without it

enum : uint32_t { kWinSnappy = 0, kWinRaw = 1, kWinSkip = 2 };
constexpr uint32_t kNoDeps = 0xFFFFFFFFu;
struct DecWin {                // one unit of work of the execute kernel
    uint32_t job;
    uint32_t kind;
    uint32_t in_off, in_len;   // bytes [in_off, in_off + in_len) of the chunk's stream hold this window's element STARTS
    uint32_t out_off, out_len; // its elements write job.dst[out_off, out_off + out_len)
    const uint8_t *entries;    // first element start per sub-block (kIndexNoEntry: none)
    uint32_t sub_log2;         // sub-block = 1 << sub_log2 stream bytes (6: index kernel, 7: embedded index)
    uint32_t first;            // list position of the chunk's first window when copies may reach into earlier windows, else kNoDeps
};
struct DecodeCtl {
    uint32_t n_windows;        // windows in the list (device-side counter)
    uint32_t n_entry_slots;    // 256-entry slots of the on-the-fly index handed out so far
    uint32_t overflow;         // a chunk did not fit the list (cannot happen with the host's sizing; checked)
    uint32_t ticket[2];        // per execute pass: next ticket.  Ticket T = window (T / njobs) of chunk (T % njobs): the
    uint32_t max_k[2];         //   k-th windows of ALL chunks come before any (k+1)-th, so that a window rarely has to wait for
                               //   its predecessor and 444 resident CTAs work on 444 different chunks.  max_k: most windows any chunk has.
    uint32_t unit_ticket;      // snappy_execute_units_kernel: next ticket (window k = T / njobs of chunk T % njobs, k < max_k_units)
    uint32_t max_k_units;      //   most windows any chunk with an embedded index has
    uint32_t units_ran;        // nonzero once that kernel ran: pass 0 of the execute kernel then draws max_k_rest * njobs tickets and
    uint32_t max_k_rest;       //   skips the windows it finished (done[w] != 0).  max_k_rest: (k + 1) of the last pass-0 window that
                               //   is not an embedded-index fragment, or that the unit kernel left undone
};

constexpr uint32_t kSrcIn = 0u << 30, kSrcOut = 1u << 30, kSrcRun = 2u << 30, kSrcMask = 3u << 30, kPosMask = (1u << 30) - 1;
constexpr uint32_t kRawWindow = 65536;

// ---- element headers --------------------------------------------------------------------------------------------------
// p = the element's first byte (readable for 5 bytes; bytes past the stream's end may hold anything: they are only
// interpreted after the length checks below passed).  pos/in_end are positions inside the chunk's stream.
__device__ __forceinline__ bool read_element_header(const uint8_t *p, uint32_t pos, uint32_t in_end, uint32_t &len, uint32_t &aux,
                                                    uint32_t &hdr, uint32_t &kind)
{
    uint32_t tag = p[0];
    kind = tag & 3;
    if (kind == 0) {
        uint32_t m = tag >> 2;
        hdr = 1;
        if (m >= 60) {
            uint32_t extra = m - 59;
            if ((uint64_t)pos + 1 + extra > in_end) return false;
            uint32_t v = p[1] | (p[2] << 8) | (p[3] << 16) | ((uint32_t)p[4] << 24);
            m = extra == 4 ? v : (v & ((1u << (8 * extra)) - 1));
            hdr = 1 + extra;
        }
        if (m == 0xFFFFFFFFu) return false;
        len = m + 1;
        aux = pos + hdr;  // payload position
        return (uint64_t)pos + hdr + len <= in_end;
    }
    if (kind == 1) {
        hdr = 2;
        len = 4 + ((tag >> 2) & 7);
        aux = ((tag >> 5) << 8) | p[1];
    } else if (kind == 2) {
        hdr = 3;
        len = 1 + (tag >> 2);
        aux = p[1] | (p[2] << 8);
    } else {
        hdr = 5;
        len = 1 + (tag >> 2);
        aux = p[1] | (p[2] << 8) | (p[3] << 16) | ((uint32_t)p[4] << 24);
    }
    return (uint64_t)pos + hdr <= in_end;
}

// varint32 preamble of a raw Snappy stream; returns its length in bytes, 0 when malformed
__device__ __forceinline__ uint32_t read_preamble(const uint8_t *src, uint32_t n, uint64_t &value)
{
    uint64_t v = 0;
    for (uint32_t i = 0; i < 5 && i < n; i++) {
        const uint32_t b = src[i];
        v |= (uint64_t)(b & 0x7F) << (7 * i);
        if (!(b & 0x80)) { value = v; return i + 1; }
    }
    return 0;
}

// ---- staging: `len` bytes at global address g -> shared memory such that base[a + i] = g[i], a = g & 15 ------------------
// The 16-byte units that lie wholly inside [g, g + len) travel by ONE bulk copy (TMA; completes on `bar`); the at most
// 15 bytes in front of and behind them are fetched by single threads, so nothing outside [g, g + len) is ever read.
// Call with all threads of the CTA; the data is complete after hap_mbar_wait(bar, parity) + __syncthreads().
__device__ __forceinline__ void stage_bytes(uint8_t *base, const uint8_t *g, uint32_t len, hap_mbar_t *bar, int t)
{
    const uint32_t a = (uint32_t)((uintptr_t)g & 15);
    const uint32_t head = len < ((16 - a) & 15) ? len : ((16 - a) & 15);   // bytes before the first aligned unit
    const uint32_t body = (len - head) & ~15u;
    const uint32_t tail = len - head - body;
    if (t == 0) {
        hap_mbar_expect_tx(bar, body);   // with body == 0 this arrival alone completes the phase
        if (body) hap_tma_load_1d(base + a + head, g + head, body, bar);
    }
    if ((uint32_t)t < head) base[a + t] = g[t];
    if ((uint32_t)t >= 32 && (uint32_t)t < 32 + tail) base[a + head + body + (t - 32)] = g[head + body + (t - 32)];
}

// =====================================================================================================================
//  index kernel
// =====================================================================================================================
constexpr int kIdxThreads = 256;
constexpr int kIdxSub = 64;                          // compressed bytes owned by one thread per window
constexpr int kIdxWin = kIdxThreads * kIdxSub;       // 16 KiB of compressed input per window
constexpr int kIdxLook = 32;                         // staged beyond the window: header look-ahead of its last elements
constexpr int kTblStride = kIdxThreads + 4;          // row stride of the exit table: rows 65 words apart, so that the 32 lanes'
                                                     // look-ups of DIFFERENT rows spread over the banks (256 put four lanes on one)
constexpr uint32_t kExitMaxRel = 186;                // tbl value <= this: exit = sub-block end + value
constexpr uint32_t kExitFarList = 187;               // kExitFarList + i (i = 0..3): the chain leaves through a long literal; where to is
constexpr uint32_t kFarSlots = 4;                    //   entry i of the sub-block's far list (the sweep fills it: no header to re-read)
constexpr uint32_t kExitFarBase = 191;               // kExitFarBase + o (o = 0..63): the same, but the far list was full: the literal's
                                                     // header sits at offset o of the sub-block; its end is read from that header
constexpr uint32_t kExitInvalid = 255;               // the chain runs into an invalid element header
constexpr uint32_t kIdxParts = 4;                    // a 16 KiB window with many elements is listed as up to 4 execute windows ...
constexpr uint32_t kIdxPartElems = 800;              // ... of about this many elements each (the execute kernel holds 1024 per pass)

struct IndexSmem {
    uint8_t cin[2][kIdxWin + kIdxLook + 32];         // staged windows (double buffered), cin[b][a + i] = byte i of the window
    uint8_t tbl[kIdxSub * kTblStride];               // tbl[o][t]: where the chain entering sub-block t at offset o leaves it
    uint16_t entry[kIdxThreads];                     // true entry offset of each sub-block, 0xFFFF = no element starts there
    uint32_t far[kFarSlots][kIdxThreads];            // window-relative positions long literals of a sub-block lead to
    uint32_t split_sub[kIdxParts + 1], split_out[kIdxParts + 1];   // sub-block / output offset where part q of the window starts
    uint32_t scratch[kIdxThreads / 32];
    hap_mbar_t bar[2];
    unsigned long long saddr_box;
    uint32_t next_rel;
    int fail;
};

// jobs with mode == kJobNeedsIndex are indexed: entries (one byte per 64 stream bytes) and one to kIdxParts DecWin per 16 KiB
// of stream are appended to the lists; the job then waits for execute pass `pass` (0: kJobReady, 1: kJobRepaired).
// entries_pool: [entry_slots][256], one slot per 16 KiB of stream.
__global__ void __launch_bounds__(kIdxThreads, 4) snappy_index_kernel(ChunkJob *jobs, int njobs, uint32_t pass, DecWin *wins,
                                                                      uint32_t win_cap, uint8_t *entries_pool, uint32_t entry_slots,
                                                                      DecodeCtl *ctl)
{
    HAP_DYN_SMEM(smem_raw);
    IndexSmem &S = *reinterpret_cast<IndexSmem *>(smem_raw);
    const int t = threadIdx.x;
    if ((int)blockIdx.x >= njobs) return;
    ChunkJob &job = jobs[blockIdx.x];
    if (job.mode != kJobNeedsIndex || job.compressor != kHapChunkSnappy) return;
    const uint32_t done_mode = pass == 0 ? (uint32_t)kJobReady : (uint32_t)kJobRepaired;
    const uint8_t *__restrict__ src = job.src;
    const uint32_t n = job.src_bytes;
    const uint32_t expected = job.dst_bytes;
    const uint32_t nwin = (n + kIdxWin - 1) / kIdxWin;

    if (t == 0) {
        uint64_t v = 0;
        const uint32_t pre = read_preamble(src, n, v);
        S.fail = (pre == 0 || v != (uint64_t)expected) ? 1 : 0;
        S.next_rel = pre;
        uint32_t base = 0, base_e = 0;
        if (!S.fail) {
            base = atomicAdd(&ctl->n_windows, kIdxParts * nwin);
            base_e = atomicAdd(&ctl->n_entry_slots, nwin);
            if (base + kIdxParts * nwin > win_cap || base + kIdxParts * nwin < base || base_e + nwin > entry_slots) { S.fail = 2; atomicExch(&ctl->overflow, 1u); }
        }
        S.scratch[0] = base;
        S.scratch[1] = base_e;
        hap_mbar_init(&S.bar[0], 1);
        hap_mbar_init(&S.bar[1], 1);
    }
    __syncthreads();
    if (S.fail) {
        if (t == 0) { job.status = S.fail == 2 ? HapResult_Internal_Error : HapResult_Bad_Frame; job.mode = kJobFinished; job.win_count = 0; }
        return;
    }
    const uint32_t base = S.scratch[0], base_e = S.scratch[1];
    uint32_t emitted = 0;     // execute windows listed so far (thread 0 keeps the count)
    const uint32_t a = (uint32_t)((uintptr_t)src & 15);   // the same for every window: windows are 16 KiB apart
    __syncthreads();

    auto window_len = [&](uint32_t k) { return n - k * kIdxWin < (uint32_t)kIdxWin ? n - k * kIdxWin : (uint32_t)kIdxWin; };
    auto staged_len = [&](uint32_t k) { return n - k * kIdxWin < (uint32_t)(kIdxWin + kIdxLook) ? n - k * kIdxWin : (uint32_t)(kIdxWin + kIdxLook); };

    stage_bytes(S.cin[0], src, staged_len(0), &S.bar[0], t);
    uint64_t d0 = 0;        // output bytes of earlier windows
    uint32_t k = 0;
    for (; k < nwin; k++) {
        const uint32_t buf = k & 1;
        // the next window's bytes start travelling now (its buffer was last read two windows ago; the barrier that
        // closed the previous iteration ordered those reads before this copy)
        if (k + 1 < nwin) stage_bytes(S.cin[buf ^ 1], src + (size_t)(k + 1) * kIdxWin, staged_len(k + 1), &S.bar[buf ^ 1], t);
        S.entry[t] = 0xFFFFu;
        hap_mbar_wait(&S.bar[buf], (k >> 1) & 1);
        __syncthreads();
        const uint8_t *cin = S.cin[buf] + a;
        const uint32_t wl = window_len(k);
        const uint32_t wpos = k * kIdxWin;                 // stream position of the window's first byte

        // ---- (a) every thread: for EACH of the 64 offsets of its sub-block, where does an element chain entering
        //      there leave the sub-block?  One backward sweep: x[o] = x[o + size(o)], branch-free ------------------
        if ((uint32_t)t * kIdxSub < wl) {
            const uint32_t blk_len = wl - t * kIdxSub < (uint32_t)kIdxSub ? wl - t * kIdxSub : (uint32_t)kIdxSub;
            const uint32_t limit = n - (wpos + t * kIdxSub);   // a chain position may not pass this
            const uint32_t bi = a + (uint32_t)t * kIdxSub;     // byte index inside S.cin[buf]
            const uint32_t *c32 = reinterpret_cast<const uint32_t *>(S.cin[buf]) + (bi >> 2);
            const uint32_t sh = 8 * (bi & 3);
            uint8_t *col = S.tbl + t;
            uint32_t nfar = 0;
#pragma unroll 1
            for (int g = kIdxSub / 16 - 1; g >= 0; g--) {
                uint32_t raw[7], w[6];
#pragma unroll
                for (int q = 0; q < 7; q++) raw[q] = c32[4 * g + q];
#pragma unroll
                for (int q = 0; q < 6; q++) w[q] = __funnelshift_r(raw[q], raw[q + 1], sh);
#pragma unroll
                for (int oo = 15; oo >= 0; oo--) {
                    const uint32_t o = (uint32_t)(16 * g + oo);
                    const uint32_t tag = (w[oo >> 2] >> (8 * (oo & 3))) & 0xFFu;
                    const uint32_t kind = tag & 3u, m = tag >> 2;
                    const uint32_t v4 = __funnelshift_r(w[(oo + 1) >> 2], w[((oo + 1) >> 2) + 1], 8 * ((oo + 1) & 3));  // the 4 bytes after the tag
                    const uint32_t extra = m - 59u;                                  // 1..4 when m >= 60
                    const uint32_t mm = extra >= 4u ? v4 : (v4 & ((1u << (8 * (extra & 3))) - 1u));
                    const uint32_t lit_long = mm >= 0x3FFFFFFFu ? 0x7FFFFFFFu : o + 2u + extra + mm;   // cannot fit a < 1 GiB chunk
                    const uint32_t lit = m < 60u ? o + m + 2u : lit_long;
                    const uint32_t nxt = kind != 0u ? o + ((0x5320u >> (4 * kind)) & 0xFu) : lit;     // copy headers: 2, 3 or 5 bytes
                    const uint32_t inside = nxt < blk_len ? nxt : o;                 // a row this thread has already written
                    const uint32_t chained = col[inside * kTblStride];
                    const bool is_far = nxt >= blk_len && nxt - blk_len > kExitMaxRel && nxt <= limit;   // (only long literals get this far)
                    const uint32_t beyond = !is_far ? nxt - blk_len : (nfar < kFarSlots ? kExitFarList + nfar : kExitFarBase + o);
                    if (is_far && nfar < kFarSlots) {
                        S.far[nfar][t] = (uint32_t)t * kIdxSub + nxt;               // window-relative position the literal ends at
                        nfar++;
                    }
                    uint32_t x = nxt < blk_len ? chained : beyond;
                    x = nxt > limit ? kExitInvalid : x;                              // header or payload runs past the input
                    col[o * kTblStride] = (uint8_t)x;
                }
            }
        }
        __syncthreads();
        // ---- (b) one thread hops sub-block to sub-block along the true chain ---------------------------------------------
        if (t == 0) {
            uint32_t rel = S.next_rel;       // window-relative position of the next true element start
            // The table's shared-window address, read back through a volatile word: ptxas otherwise re-derives it from
            // the CTA-in-cluster id (an S2R, tens of cycles on this thread's critical path) in EVERY iteration of the hop.
            volatile hap_saddr_t *base_box = reinterpret_cast<volatile hap_saddr_t *>(&S.saddr_box);
            *base_box = hap_smem_addr(S.tbl);
            const hap_saddr_t tbl_s = *base_box, entry_s = tbl_s + (hap_saddr_t)((const uint8_t *)S.entry - (const uint8_t *)S.tbl);
            while (rel < wl) {
                const uint32_t blk = rel >> 6, o = rel & 63;
                const uint32_t x = hap_lds_u8(tbl_s + (o * kTblStride + blk));
                hap_sts_u16(entry_s + 2 * blk, o);
                uint32_t bend = (blk + 1) << 6;
                bend = bend < wl ? bend : wl;
                if (x <= kExitMaxRel) {
                    rel = bend + x;
                } else if (x < kExitFarBase) {
                    rel = S.far[x - kExitFarList][blk];
                } else if (x == kExitInvalid) {
                    S.fail = 1;
                    break;
                } else {
                    // a long literal leaves this sub-block by more than a byte can hold: the table names its header
                    const uint32_t p2 = (blk << 6) + (x - kExitFarBase);
                    uint32_t len, aux, hdr, kind;
                    if (!read_element_header(cin + p2, wpos + p2, n, len, aux, hdr, kind) || kind != 0) { S.fail = 1; break; }
                    rel = p2 + hdr + len;
                }
            }
            S.next_rel = rel - wl;           // (garbage when the hop failed: nobody reads it then)
            if (k + 1 == nwin && rel != wl) S.fail = 1;   // the chain must end exactly at the end of the stream
        }
        __syncthreads();
        // ---- (c) every entered sub-block adds up the output of the elements that start in it ----------------------------
        uint32_t out_bytes = 0, count = 0;
        int invalid = 0;
        const uint32_t ent = S.entry[t];
        if (ent != 0xFFFFu) {
            uint32_t pos = t * kIdxSub + ent;
            const uint32_t end = (t + 1) * kIdxSub < wl ? (t + 1) * kIdxSub : wl;
            while (pos < end) {
                uint32_t len, aux, hdr, kind;
                if (!read_element_header(cin + pos, wpos + pos, n, len, aux, hdr, kind)) { invalid = 1; break; }
                out_bytes += len;                      // (cannot wrap: <= 64 elements of <= 2^30 + ... checked against `expected` below)
                count++;
                pos += hdr + (kind == 0 ? len : 0);
            }
        }
        uint32_t total_o, total_e;
        const uint32_t obase = block_excl_sum<kIdxThreads>(out_bytes > 0x40000000u ? 0x40000000u : out_bytes, &total_o, S.scratch);
        const uint32_t ebase = block_excl_sum<kIdxThreads>(count, &total_e, S.scratch);
        if (invalid) S.fail = 1;
        if (t == 0 && d0 + total_o > (uint64_t)expected) S.fail = 1;
        // A window with many elements is listed as several execute windows over consecutive sub-block ranges, so that each
        // fits the execute kernel's descriptor arrays in one pass and more CTAs share the work: part q starts behind the
        // sub-block in which the (q * total_e / parts)-th element starts.
        const uint32_t parts = total_e <= kIdxPartElems ? 1u : ((total_e + kIdxPartElems - 1) / kIdxPartElems < kIdxParts ? (total_e + kIdxPartElems - 1) / kIdxPartElems : kIdxParts);
        for (uint32_t q = 1; q < parts; q++) {
            const uint32_t thr = (uint32_t)(((unsigned long long)total_e * q) / parts);    // 0 < thr < total_e
            if (ebase < thr && thr <= ebase + count) { S.split_sub[q] = (uint32_t)t + 1; S.split_out[q] = obase + out_bytes; }
        }
        __syncthreads();
        if (S.fail) break;
        entries_pool[(size_t)(base_e + k) * kIdxThreads + t] = ent == 0xFFFFu ? (uint8_t)kIndexNoEntry : (uint8_t)ent;
        if (t == 0) {
            const uint32_t nsub = (wl + kIdxSub - 1) / kIdxSub;
            S.split_sub[0] = 0; S.split_out[0] = 0;
            S.split_sub[parts] = nsub; S.split_out[parts] = total_o;
            for (uint32_t q = 0; q < parts; q++) {
                DecWin w;
                w.job = blockIdx.x;
                w.kind = kWinSnappy;
                w.in_off = wpos + S.split_sub[q] * kIdxSub;
                w.in_len = (q + 1 == parts ? wl : S.split_sub[q + 1] * kIdxSub) - S.split_sub[q] * kIdxSub;
                w.out_off = (uint32_t)d0 + S.split_out[q];
                w.out_len = S.split_out[q + 1] - S.split_out[q];
                w.entries = entries_pool + (size_t)(base_e + k) * kIdxThreads + S.split_sub[q];
                w.sub_log2 = 6;
                w.first = base;
                wins[base + emitted + q] = w;
            }
            emitted += parts;
        }
        d0 += total_o;
    }
    if (t == 0) {
        // an invalid stream keeps the windows listed so far (they decode what was valid) and reports Bad_Frame
        if (k < nwin || d0 != (uint64_t)expected) job.status = HapResult_Bad_Frame;
        job.win_base = base;
        job.win_count = emitted;
        atomicMax(&ctl->max_k[pass], emitted);
        if (pass == 0) atomicMax(&ctl->max_k_rest, emitted);
        job.mode = done_mode;
    }
}

// =====================================================================================================================
//  chunks -> windows (one thread per chunk)
// =====================================================================================================================
constexpr uint32_t kFragMaxStream = 32768 + 32;      // an element stream of one fragment (snappy_encode.cuh: at most n + 3)
constexpr uint32_t kIndexFragBytes = 32768;

__device__ __forceinline__ uint32_t rd16(const uint8_t *p) { return p[0] | (p[1] << 8); }

// use_index = 0: ignore embedded indexes (every Snappy chunk goes to the index kernel).
__global__ void hap_build_windows_kernel(ChunkJob *jobs, uint32_t njobs, uint32_t use_index, DecWin *wins, uint32_t win_cap, DecodeCtl *ctl)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= njobs) return;
    ChunkJob &job = jobs[j];
    if (job.compressor == 0) return;   // unused slot of a batched frame (hap_parse.cuh)
    job.status = HapResult_No_Error;
    job.mode = kJobFinished;    // nothing to execute, unless windows are listed below
    job.win_base = 0;
    job.win_count = 0;
    const uint32_t n = job.src_bytes, expected = job.dst_bytes;
    if (job.compressor == kHapChunkRaw) {
        // hap.c:630-636: verbatim chunk
        if (n != expected) { job.status = HapResult_Bad_Frame; return; }
        const uint32_t cnt = (n + kRawWindow - 1) / kRawWindow;
        if (cnt == 0) return;
        const uint32_t base = atomicAdd(&ctl->n_windows, cnt);
        if (base + cnt > win_cap || base + cnt < base) { job.status = HapResult_Internal_Error; atomicExch(&ctl->overflow, 1u); return; }
        job.win_base = base; job.win_count = cnt; job.mode = kJobReady;
        atomicMax(&ctl->max_k[0], cnt);
        atomicMax(&ctl->max_k_rest, cnt);
        for (uint32_t i = 0; i < cnt; i++) {
            DecWin w;
            w.job = j; w.kind = kWinRaw; w.in_off = i * kRawWindow; w.in_len = n - i * kRawWindow < kRawWindow ? n - i * kRawWindow : kRawWindow;
            w.out_off = w.in_off; w.out_len = w.in_len; w.entries = nullptr; w.sub_log2 = 6; w.first = kNoDeps;
            wins[base + i] = w;
        }
        return;
    }
    if (job.compressor != kHapChunkSnappy || n > kPosMask || expected > kPosMask) {
        // hap.c:637-640; also chunks of 1 GiB and more, whose positions do not fit the packed descriptors
        job.status = HapResult_Bad_Frame;
        return;
    }
    uint64_t v = 0;
    const uint32_t pre = read_preamble(job.src, n, v);
    if (pre == 0 || v != (uint64_t)expected) { job.status = HapResult_Bad_Frame; return; }
    job.mode = kJobNeedsIndex;
    if (!use_index || job.index == nullptr) return;
    // embedded index (hap_index.h): u16 stream_bytes[nf], then the entries of every fragment
    const uint32_t nf = (expected + kIndexFragBytes - 1) / kIndexFragBytes;
    if (nf == 0 || (uint64_t)2 * nf > job.index_bytes) return;
    uint64_t stream = pre, ent_bytes = 0;
    for (uint32_t f = 0; f < nf; f++) {
        const uint32_t s = rd16(job.index + 2 * f);
        if (s == 0 || s > kFragMaxStream) return;
        stream += s;
        ent_bytes += (s + (1u << kIndexSubLog2) - 1) >> kIndexSubLog2;
    }
    if (stream != n || 2ull * nf + ent_bytes > job.index_bytes) return;
    const uint32_t base = atomicAdd(&ctl->n_windows, nf);
    if (base + nf > win_cap || base + nf < base) { job.status = HapResult_Internal_Error; job.mode = kJobFinished; atomicExch(&ctl->overflow, 1u); return; }
    job.win_base = base; job.win_count = nf;
    atomicMax(&ctl->max_k[0], nf);
    atomicMax(&ctl->max_k_units, nf);
    uint32_t in_off = pre;
    const uint8_t *ent = job.index + 2 * nf;
    for (uint32_t f = 0; f < nf; f++) {
        const uint32_t s = rd16(job.index + 2 * f);
        DecWin w;
        w.job = j; w.kind = kWinSnappy; w.in_off = in_off; w.in_len = s;
        w.out_off = f * kIndexFragBytes;
        w.out_len = expected - w.out_off < kIndexFragBytes ? expected - w.out_off : kIndexFragBytes;
        w.entries = ent; w.sub_log2 = kIndexSubLog2; w.first = kNoDeps;
        wins[base + f] = w;
        in_off += s;
        ent += (s + (1u << kIndexSubLog2) - 1) >> kIndexSubLog2;
    }
    job.mode = kJobReady;
}

// After the first execute pass: chunks whose embedded index did not hold up are handed to the index kernel (mode
// kJobNeedsIndex, status cleared); *any_left counts them.
__global__ void hap_requeue_mismatched_kernel(ChunkJob *jobs, uint32_t njobs, uint32_t *any_left)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= njobs) return;
    if (jobs[j].compressor != 0 && jobs[j].status == kStatusIndexMismatch) {
        jobs[j].status = HapResult_No_Error;
        jobs[j].mode = kJobNeedsIndex;
        atomicAdd(any_left, 1u);
    }
}

// =====================================================================================================================
//  execute kernel
// =====================================================================================================================
#ifndef HAPB200_EX_MAX_ELEMS
#define HAPB200_EX_MAX_ELEMS 1024
#endif
#ifndef HAPB200_EX_TILE
#define HAPB200_EX_TILE 16384
#endif
#ifndef HAPB200_EX_MIN_BLOCKS
#define HAPB200_EX_MIN_BLOCKS 4
#endif
// 1024 descriptors / 16 KiB tiles at 4 CTAs per SM (54 KB, 64 registers; sm_90a spills 108 bytes) against 3 CTAs per SM
// (80 registers, 40 bytes of spills), this kernel's time on 444 4K Hap Q frames with index, H100 80GB HBM3 at a 400 W
// power limit, four alternating runs each: 6.94-7.12 ms at 4, 7.07-7.43 ms at 3.  Outputs are identical.
constexpr int kExThreads = 256;
constexpr int kExMaxElems = HAPB200_EX_MAX_ELEMS;    // descriptors held in shared memory per pass
constexpr int kExMaxIn = 32768 + 64;                 // stream bytes of one window the staging buffer holds
constexpr int kExLook = 16;                          // staged beyond the window: header look-ahead
constexpr int kExTile = HAPB200_EX_TILE;             // output bytes produced per tile
constexpr int kExGroups = kExTile / 16 + 1;          // a tile that does not start on a 16-byte address touches one group more
constexpr int kFlattenHops = 12;
#ifndef HAPB200_EX_UNIT_PATH
#define HAPB200_EX_UNIT_PATH 1
#endif
// -DHAPB200_EX_PHASE_CLOCKS=1 (measurement builds only, tools/measure_unit_phases.py): thread 0 of every CTA adds up
// clock64() per phase of the unit path in shared memory and folds its sums into g_ex_phase_clocks when the CTA ends.
// Phases end at barriers where there is one, so a phase's clocks are those of the CTA, not of thread 0 alone.
#ifndef HAPB200_EX_PHASE_CLOCKS
#define HAPB200_EX_PHASE_CLOCKS 0
#endif
enum : int { kPhStage = 0, kPhWalk, kPhScan, kPhRecords, kPhMap, kPhRounds, kPhWrite, kPhOther, kPhCount };
enum : int { kPhUnitWindows = kPhCount, kPhRoundCount, kPhSlots };   // counters kept behind the phase clocks
#if HAPB200_EX_PHASE_CLOCKS && !defined(HAPB200_EMU)
__device__ unsigned long long g_ex_phase_clocks[kPhSlots];
__shared__ unsigned long long s_ex_phase[kPhSlots + 1];   // [kPhSlots]: clock of the last mark
#define HAP_PHASE_BEGIN()                                                                 \
    do {                                                                                  \
        if (threadIdx.x == 0) {                                                           \
            for (int q_ = 0; q_ < kPhSlots; q_++) s_ex_phase[q_] = 0;                     \
            s_ex_phase[kPhSlots] = clock64();                                             \
        }                                                                                 \
    } while (0)
#define HAP_PHASE_MARK(ph)                                                                \
    do {                                                                                  \
        if (threadIdx.x == 0) {                                                           \
            const unsigned long long c_ = clock64();                                      \
            s_ex_phase[ph] += c_ - s_ex_phase[kPhSlots];                                  \
            s_ex_phase[kPhSlots] = c_;                                                    \
        }                                                                                 \
    } while (0)
#define HAP_PHASE_COUNT(slot)                                                             \
    do {                                                                                  \
        if (threadIdx.x == 0) s_ex_phase[slot]++;                                         \
    } while (0)
#define HAP_PHASE_END()                                                                   \
    do {                                                                                  \
        if (threadIdx.x == 0)                                                             \
            for (int q_ = 0; q_ < kPhSlots; q_++) atomicAdd(&g_ex_phase_clocks[q_], s_ex_phase[q_]); \
    } while (0)
#else
#define HAP_PHASE_BEGIN() do {} while (0)
#define HAP_PHASE_MARK(ph) do {} while (0)
#define HAP_PHASE_COUNT(slot) do {} while (0)
#define HAP_PHASE_END() do {} while (0)
#endif

constexpr uint32_t kExUnits = kIndexFragBytes / 8;   // 8-byte output units of a fragment (unit path)
constexpr uint32_t kUnitLit = kExUnits;              // unit map value >= this: literal bytes at window byte (value - kUnitLit)
constexpr int kUnitMaxRounds = 24;                   // pointer jumping over chains of <= 4096 units ends within 13 rounds
constexpr int kUnitStripLen = 16;                    // units per thread in the unit path's map step

struct ExecSmem {
    uint8_t cin[32 + kExMaxIn + kExLook + 48];       // staged window, cin[32 + a + i] = byte i of the window (32 spare bytes in front)
    union {
        struct {
            uint32_t e_dst[kExMaxElems];             // output position inside the chunk
            uint32_t e_len[kExMaxElems];
            uint32_t e_a[kExMaxElems];               // packed source: kSrcIn|input position, kSrcOut|output position, kSrcRun|offset
            uint32_t e_b[kExMaxElems];               // destination of the head of the element's same-offset run (its own, if alone)
        };
        uint16_t umap[2 * kExUnits];                 // unit path: element records, then the source of every 8-byte unit of the fragment
    };
    uint16_t gfirst[kExGroups + 7];                  // (element + 1) that holds the first byte of an output group
    uint16_t gdone[kExGroups + 7];                   // round in which a group was written (0: not yet)
    uint8_t landed[kExThreads];                      // a chain exit lands in this sub-block
    uint32_t scratch[kExThreads / 32];
    uint32_t red[3][kExThreads / 32];
    // the window being worked on, two slots used alternately: thread 0 fills the slot of the next iteration while slower
    // threads may still be reading this iteration's (some paths reach the top of the loop without passing a barrier)
    struct Slot {
        DecWin win;
        uint32_t ticket;
    } slot[2];
    hap_mbar_t bar;
    // per-window flags, two sets used alternately: the set of the NEXT window is cleared while this one is being worked on
    // (clearing the current set at the top of the loop would race with threads that still test it on their way there)
    struct Flags {
        uint32_t min_src;
        int fail;         // walk stage
        int fail_desc;    // descriptor stage
        int mismatch;     // embedded index does not describe the chain, or a copy of the fragment reads before it
    } flags[2];
};

// three block reductions at once: minimum of a, minimum of b, maximum of c (two barriers)
__device__ __forceinline__ void block_min_min_max(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t (*red)[kExThreads / 32])
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
        const uint32_t oa = __shfl_xor_sync(HAP_FULL_MASK, a, d), ob = __shfl_xor_sync(HAP_FULL_MASK, b, d), oc = __shfl_xor_sync(HAP_FULL_MASK, c, d);
        a = a < oa ? a : oa;
        b = b < ob ? b : ob;
        c = c > oc ? c : oc;
    }
    if (lane == 0) { red[0][warp] = a; red[1][warp] = b; red[2][warp] = c; }
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kExThreads / 32; w++) {
        a = a < red[0][w] ? a : red[0][w];
        b = b < red[1][w] ? b : red[1][w];
        c = c > red[2][w] ? c : red[2][w];
    }
    __syncthreads();
}

__device__ __forceinline__ unsigned long long low_bytes_mask(uint32_t k) { return k >= 8 ? ~0ull : ((1ull << (8 * k)) - 1ull); }

// One aligned 32-bit word at `wa`, of which only the bytes inside [need_lo, need_hi) are wanted, fetched byte by byte:
// the first and last word of a chunk or of the output buffer, where a whole-word load would touch bytes outside it.
__device__ __noinline__ uint32_t edge_word(uintptr_t wa, uintptr_t need_lo, uintptr_t need_hi)
{
    uint32_t v = 0;
    for (uint32_t q = 0; q < 4; q++)
        if (wa + q >= need_lo && wa + q < need_hi) v |= (uint32_t) * reinterpret_cast<const uint8_t *>(wa + q) << (8 * q);
    return v;
}

// n (1..16) bytes at `ptr` -> bytes [q, 16) of the 16-byte group held in (lo64, hi64); bytes below q are kept.  (What lands
// behind q + n is overwritten by the pieces that follow, or lies beyond the group's last byte and is never stored.)
// `safe`: the five aligned words around the piece may be read whole (shared memory, or well inside a global buffer).
__device__ __forceinline__ void gather_into_group(const uint8_t *ptr, uint32_t n, uint32_t q, bool safe, unsigned long long &lo64,
                                                  unsigned long long &hi64)
{
    const uintptr_t p = (uintptr_t)ptr;
    // the address that corresponds to byte 0 of the group, its aligned base and the shift between the two
    const uintptr_t g0 = p - q;
    const uint32_t mis = (uint32_t)(g0 & 3);
    const uintptr_t b0 = g0 - mis;
    uint32_t s[5];
    if (safe) {
#pragma unroll
        for (int k = 0; k < 5; k++) s[k] = reinterpret_cast<const uint32_t *>(b0)[k];
    } else {
#pragma unroll
        for (int k = 0; k < 5; k++) s[k] = edge_word(b0 + 4 * k, p, p + n);
    }
    const uint32_t sh = 8 * mis;
    const uint32_t c0 = __funnelshift_r(s[0], s[1], sh), c1 = __funnelshift_r(s[1], s[2], sh);
    const uint32_t c2 = __funnelshift_r(s[2], s[3], sh), c3 = __funnelshift_r(s[3], s[4], sh);
    const unsigned long long cl = c0 | ((unsigned long long)c1 << 32), ch = c2 | ((unsigned long long)c3 << 32);
    const unsigned long long kl = low_bytes_mask(q), kh = q > 8 ? low_bytes_mask(q - 8) : 0ull;   // the bytes to keep
    lo64 = (lo64 & kl) | (cl & ~kl);
    hi64 = (hi64 & kh) | (ch & ~kh);
}

__device__ __forceinline__ uint32_t group_byte(unsigned long long lo64, unsigned long long hi64, uint32_t i)
{
    const unsigned long long h = (i & 8) ? hi64 : lo64;
    return (uint32_t)(h >> (8 * (i & 7))) & 0xFFu;
}
__device__ __forceinline__ void set_group_byte(unsigned long long &lo64, unsigned long long &hi64, uint32_t i, uint32_t b)
{
    const unsigned long long m = 0xFFull << (8 * (i & 7)), v = (unsigned long long)b << (8 * (i & 7));
    if (i & 8) hi64 = (hi64 & ~m) | v;
    else lo64 = (lo64 & ~m) | v;
}

// Everything one tile of output needs to know.
struct TileCtx {
    const uint8_t *src;        // the chunk's stream
    uint8_t *dst;              // the chunk's output
    uint32_t src_bytes, dst_bytes;
    const uint8_t *cin;        // staged window: cin[i] = stream byte wb + i for i < staged
    uint32_t wb, staged;
    int32_t gbase;             // output position of byte 0 of group 0 (may lie before T0: group 0 can be partial)
    uint32_t T0, T1;           // the tile's output positions
};

// Assemble the bytes [max(gstart, T0), min(gstart + 16, T1)) of group g and write them.  false: a source is not final yet.
__device__ __forceinline__ bool assemble_group(ExecSmem &S, const TileCtx &C, uint32_t g, uint32_t round)
{
    const int32_t gstart = C.gbase + 16 * (int32_t)g;
    const uint32_t lo = gstart > (int32_t)C.T0 ? (uint32_t)gstart : C.T0;
    const uint32_t hi = (uint32_t)(gstart + 16) < C.T1 ? (uint32_t)(gstart + 16) : C.T1;
    uint32_t e = (uint32_t)S.gfirst[g] - 1u;
    unsigned long long lo64 = 0, hi64 = 0;
    uint32_t pos = lo;
    while (pos < hi) {
        const uint32_t d = S.e_dst[e], l = S.e_len[e];
        const uint32_t seg_end = d + l < hi ? d + l : hi;
        uint32_t n = seg_end - pos;
        const uint32_t q = (uint32_t)((int32_t)pos - gstart);
        const uint32_t a = S.e_a[e], kind = a & kSrcMask, ap = a & kPosMask;
        const uint8_t *ptr;
        bool safe;
        if (kind == kSrcIn) {
            const uint32_t ip = ap + (pos - d);
            const bool staged = ip >= C.wb && ip + n <= C.wb + C.staged;
            ptr = staged ? C.cin + (ip - C.wb) : C.src + ip;
            // (the staging buffer has 32 spare bytes in front of and behind the window: whole words around a piece are always readable)
            safe = staged || (ip >= 20u && ip + 20u <= C.src_bytes);
        } else {
            uint32_t sp;
            if (kind == kSrcOut) {
                sp = ap + (pos - d);
            } else {
                // periodic fill of the run's base period: the bytes [base - off, base)
                const uint32_t off = ap, base = S.e_b[e];
                const uint32_t r = (pos - base) % off;
                if (n > off - r) n = off - r;
                sp = base - off + r;
            }
            if (sp >= lo) {
                // the source bytes are earlier bytes of this very group (offsets below 16): they are in the registers
                for (uint32_t i = 0; i < n; i++) set_group_byte(lo64, hi64, q + i, group_byte(lo64, hi64, (uint32_t)((int32_t)(sp + i) - gstart)));
                pos += n;
                if (pos >= d + l) e++;
                continue;
            }
            if (sp + n > lo) n = lo - sp;             // the rest of the piece comes from the registers next time round
            if (sp + n > C.T0) {
                // bytes this tile produces: their groups must have been written in an earlier round
                const int32_t rel0 = (int32_t)sp - C.gbase, rel1 = (int32_t)(sp + n - 1) - C.gbase;
                const uint32_t g0 = rel0 < 0 ? 0u : (uint32_t)rel0 >> 4, g1 = (uint32_t)rel1 >> 4;
                const uint32_t r0 = S.gdone[g0], r1 = S.gdone[g1];
                if (r0 == 0 || r0 >= round || r1 == 0 || r1 >= round) return false;
            }
            ptr = C.dst + sp;
            safe = sp >= 20u && sp + 20u <= C.dst_bytes;
        }
        gather_into_group(ptr, n, q, safe, lo64, hi64);
        pos += n;
        if (pos >= d + l) e++;
    }
    uint8_t *out = C.dst + gstart;   // 16-byte aligned by construction of gbase
    if (lo == (uint32_t)gstart && hi == (uint32_t)(gstart + 16)) {
        *reinterpret_cast<uint4 *>(out) = make_uint4((uint32_t)lo64, (uint32_t)(lo64 >> 32), (uint32_t)hi64, (uint32_t)(hi64 >> 32));
    } else {
        for (uint32_t i = (uint32_t)((int32_t)lo - gstart); i < (uint32_t)((int32_t)hi - gstart); i++) out[i] = (uint8_t)group_byte(lo64, hi64, i);
    }
    S.gdone[g] = (uint16_t)round;
    return true;
}

// walk the elements that start in stream bytes [pos, end) of the window; positions are relative to the window
struct WalkResult {
    uint32_t exit, count, out_bytes;
    int invalid;
    uint32_t coarse;   // nonzero: an element's length, or a copy's offset, is not a nonzero multiple of 8
};
__device__ __forceinline__ WalkResult walk_piece(const uint8_t *cin, uint32_t wb, uint32_t pos, uint32_t end, uint32_t in_end)
{
    WalkResult r;
    r.count = 0;
    r.out_bytes = 0;
    r.invalid = 0;
    r.coarse = 0;
    while (pos < end) {
        uint32_t len, aux, hdr, kind;
        if (!read_element_header(cin + pos, wb + pos, in_end, len, aux, hdr, kind)) { r.invalid = 1; break; }
        r.count++;
        r.out_bytes += len;
        r.coarse |= (len | (kind == 0 ? 0u : aux)) & 7u;
        if (kind != 0 && aux == 0) r.coarse = 1;
        pos += hdr + (kind == 0 ? len : 0);
    }
    r.exit = pos;
    return r;
}

// The next ticket that names an existing window (window k = T / njobs of chunk T % njobs) and that window's record, fetched
// by thread 0 one window AHEAD, right after the current window's bulk copy has been issued: the atomic and the global
// loads then overlap the copy instead of standing alone in front of a barrier.  (Not inlined: one thread's cold path.)
// finished: the unit kernel's per-window flags (done[]) when it ran before this pass, else nullptr.
__device__ __noinline__ void fetch_next_window(const ChunkJob *jobs, uint32_t njobs, uint32_t pass, uint32_t want_mode, unsigned long long n_tickets,
                                               const DecWin *wins, DecodeCtl *ctl, DecWin *win_out, uint32_t *ticket_out, const uint32_t *finished)
{
    uint32_t w = 0xFFFFFFFFu;
    for (;;) {
        const unsigned long long T = atomicAdd(&ctl->ticket[pass], 1u);
        if (T >= n_tickets) break;
        const uint32_t k = (uint32_t)(T / njobs), j = (uint32_t)(T % njobs);
        if (jobs[j].compressor != 0 && jobs[j].mode == want_mode && k < jobs[j].win_count) {
            w = jobs[j].win_base + k;
            if (finished && finished[w] != 0) { w = 0xFFFFFFFFu; continue; }
            break;
        }
    }
    *ticket_out = w;
    if (w != 0xFFFFFFFFu) *win_out = wins[w];
}

#ifdef HAPB200_EMU
inline uint64_t &emu_unit_windows() { static uint64_t n = 0; return n; }   // windows the unit path decoded (tests only)
#endif

// The unit path: a fragment of an embedded index whose elements are all 8-byte granular (every length and copy offset a
// nonzero multiple of 8: what this repo's encoder writes) is 4096 units of 8 bytes, each either 8 literal bytes of the
// staged stream or a copy of an earlier unit.  No descriptors, passes, runs or output-centric rounds are needed:
//   records: every piece's walk writes one 16-bit record at the first unit of each element (kUnitLit + stream position of a
//            literal, the distance in units of a copy; 0 = no element starts at this unit);
//   map:     thread t owns units 16t .. 16t + 15; a max-scan finds the element each unit lies in, and the unit gets
//            kUnitLit + its stream position (literal) or the earlier unit it copies (the element's period for overlapping
//            copies): every lane does the same work whatever the element lengths are;
//   resolve: map[u] = map[map[u]] in rounds until every unit names stream bytes (sources are strictly earlier units of the
//            fragment, so every chain ends at a literal; a racing update only skips hops);
//   write:   thread g assembles destination-aligned 16-byte group g from two or three units of the staged window.
// Called by all threads behind the walk checks (total_o == out_len <= 32 KiB).  Returns false (uniform) when a copy reads
// before the fragment or before the chunk: the caller hands the chunk to the repair pass.  `coff`: cin byte of window byte 0;
// `crossing`: the window's flag that is not tested behind the walk's barrier (set here by the thread that finds such a copy).
__device__ __noinline__ bool execute_units(ExecSmem &S, int &crossing, uint32_t coff, uint32_t wb, uint32_t in_end, bool entered,
                                           uint32_t pos, uint32_t end, uint32_t obase, uint8_t *out, uint32_t out_len)
{
    static_assert(kExUnits == kUnitStripLen * kExThreads, "16 units per thread");
    const int t = threadIdx.x;
    uint16_t *rec = S.umap, *map = S.umap + kExUnits;
    const uint8_t *cin = S.cin + coff;
    uint4 *rec4 = reinterpret_cast<uint4 *>(rec), *map4 = reinterpret_cast<uint4 *>(map);
    rec4[2 * t] = make_uint4(0, 0, 0, 0);
    rec4[2 * t + 1] = make_uint4(0, 0, 0, 0);
    __syncthreads();
    if (entered) {
        uint32_t u = obase >> 3;   // (a multiple of 8: every element before this piece is)
        while (pos < end) {
            uint32_t len, aux, hdr, kind;
            read_element_header(cin + pos, wb + pos, in_end, len, aux, hdr, kind);   // (the walk checked every header)
            if (kind == 0) {
                rec[u] = (uint16_t)(kUnitLit + (aux - wb));
                pos += hdr + len;
            } else {
                const uint32_t d = aux >> 3;
                if (d > u) { crossing = 1; break; }
                rec[u] = (uint16_t)d;
                pos += hdr;
            }
            u += len >> 3;
        }
    }
    __syncthreads();
    HAP_PHASE_MARK(kPhRecords);
    if (crossing) return false;
    const uint32_t U = out_len >> 3, u0 = kUnitStripLen * (uint32_t)t;
    uint32_t r[kUnitStripLen];
    {
        const uint4 a = rec4[2 * t], b = rec4[2 * t + 1];
        const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int k = 0; k < kUnitStripLen; k++) r[k] = (w[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
    }
    uint32_t last = 0;   // (unit + 1) of the last element start in this strip
#pragma unroll
    for (int k = 0; k < kUnitStripLen; k++) last = r[k] != 0 ? u0 + k + 1 : last;
    uint32_t unused;
    const uint32_t carry = block_excl_max<kExThreads>(last, &unused, S.scratch);   // the element running into this strip
    uint32_t start = carry ? carry - 1 : 0, rs = carry ? rec[carry - 1] : 0;
    int pending = 0;   // a unit still names another unit
    uint32_t v[kUnitStripLen];
#pragma unroll
    for (int k = 0; k < kUnitStripLen; k++) {
        const uint32_t u = u0 + k;
        if (r[k] != 0) { start = u; rs = r[k]; }
        const uint32_t q = u - start;
        v[k] = rs >= kUnitLit ? rs + 8 * q : start - rs + (q < rs || rs == 0 ? q : q % rs);   // (rs == 0: only past unit U)
        pending |= u < U && v[k] < kUnitLit;
    }
#pragma unroll
    for (int h = 0; h < 2; h++)
        map4[2 * t + h] = make_uint4((v[8 * h] & 0xFFFFu) | (v[8 * h + 1] << 16), (v[8 * h + 2] & 0xFFFFu) | (v[8 * h + 3] << 16),
                                     (v[8 * h + 4] & 0xFFFFu) | (v[8 * h + 5] << 16), (v[8 * h + 6] & 0xFFFFu) | (v[8 * h + 7] << 16));
    pending = __syncthreads_or(pending);
    HAP_PHASE_MARK(kPhMap);
    for (int round = 0; pending; round++) {
        pending = 0;
        for (uint32_t u = t; u < U; u += kExThreads) {
            const uint32_t v = map[u];
            if (v < kUnitLit) {
                const uint32_t v2 = map[v];
                map[u] = (uint16_t)v2;
                pending |= v2 < kUnitLit;
            }
        }
        pending = __syncthreads_or(pending);
        HAP_PHASE_MARK(kPhRounds);
        HAP_PHASE_COUNT(kPhRoundCount);
        if (pending && round == kUnitMaxRounds) return false;   // (cannot happen: chains are at most 4096 units deep)
    }
    // group g = destination bytes [16g - m, 16g - m + 16) of the fragment, m = misalignment of its first byte
    const uint32_t *c32 = reinterpret_cast<const uint32_t *>(S.cin);
    const uint32_t m = (uint32_t)((uintptr_t)out & 15);
    const uint32_t ngroups = (m + out_len + 15) >> 4;
    for (uint32_t g = t; g < ngroups; g += kExThreads) {
        const int32_t x = 16 * (int32_t)g - (int32_t)m;
        const int32_t ua = x >> 3;   // (floor: -2 or -1 for the first group of a misaligned fragment)
        const uint32_t r = (uint32_t)x & 7u;
        uint32_t w[6];
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const int32_t u = ua + k;
            w[2 * k] = 0;
            w[2 * k + 1] = 0;
            if (u >= 0 && (uint32_t)u < U && (k < 2 || r != 0)) {
                const uint32_t b = coff + (uint32_t)map[u] - kUnitLit, i = b >> 2, sh = 8 * (b & 3);
                const uint32_t s0 = c32[i], s1 = c32[i + 1], s2 = c32[i + 2];
                w[2 * k] = __funnelshift_r(s0, s1, sh);
                w[2 * k + 1] = __funnelshift_r(s1, s2, sh);
            }
        }
        const uint32_t q = r >> 2, sh = 8 * (r & 3);
        const uint32_t o0 = __funnelshift_r(w[q], w[q + 1], sh), o1 = __funnelshift_r(w[q + 1], w[q + 2], sh);
        const uint32_t o2 = __funnelshift_r(w[q + 2], w[q + 3], sh), o3 = __funnelshift_r(w[q + 3], w[q + 4], sh);
        if (x >= 0 && (uint32_t)x + 16 <= out_len) {
            *reinterpret_cast<uint4 *>(out + x) = make_uint4(o0, o1, o2, o3);   // 16-byte aligned by the choice of m
        } else {
            const uint32_t ow[4] = {o0, o1, o2, o3};
            for (int i = 0; i < 16; i++)
                if (x + i >= 0 && (uint32_t)(x + i) < out_len) out[x + i] = (uint8_t)(ow[i >> 2] >> (8 * (i & 3)));
        }
    }
    return true;
}

// pass 0 executes the chunks in mode kJobReady, pass 1 (repair) those in mode kJobRepaired.
__global__ void __launch_bounds__(kExThreads, HAPB200_EX_MIN_BLOCKS) snappy_execute_kernel(ChunkJob *jobs, uint32_t njobs, uint32_t pass, const DecWin *wins,
                                                                       DecodeCtl *ctl, uint32_t *done)
{
    HAP_DYN_SMEM(smem_raw);
    ExecSmem &S = *reinterpret_cast<ExecSmem *>(smem_raw);
    const int t = threadIdx.x;
    // final: every kernel that lists windows ran before this one.  Behind the unit kernel, pass 0 takes only the chunks
    // whose windows it did not all finish, and skips the windows it did.
    const bool behind_units = pass == 0 && ctl->units_ran != 0;
    const uint32_t max_k = behind_units ? ctl->max_k_rest : ctl->max_k[pass];
    const uint32_t *finished = behind_units ? done : nullptr;
    const uint32_t want_mode = pass == 0 ? (uint32_t)kJobReady : (uint32_t)kJobRepaired;
    const unsigned long long n_tickets = (unsigned long long)max_k * njobs;
    if (t == 0) {
        hap_mbar_init(&S.bar, 1);
        for (int q = 0; q < 2; q++) { S.flags[q].min_src = 0xFFFFFFFFu; S.flags[q].fail = 0; S.flags[q].fail_desc = 0; S.flags[q].mismatch = 0; }
    }
    uint32_t phase = 0;
    HAP_PHASE_BEGIN();
    __syncthreads();
    auto fetch_window = [&](uint32_t slot) { fetch_next_window(jobs, njobs, pass, want_mode, n_tickets, wins, ctl, &S.slot[slot & 1].win, &S.slot[slot & 1].ticket, finished); };
    if (t == 0) fetch_window(0);
    for (uint32_t it = 0;; it++) {
        ExecSmem::Flags &F = S.flags[it & 1];
        __syncthreads();
        const uint32_t w = S.slot[it & 1].ticket;
        if (w == 0xFFFFFFFFu) break;
        if (t == 0) { ExecSmem::Flags &N = S.flags[(it + 1) & 1]; N.min_src = 0xFFFFFFFFu; N.fail = 0; N.fail_desc = 0; N.mismatch = 0; }
        S.landed[t] = 0;    // (written by the walk behind the staging barrier below; last read before the previous window's scans ended)
        const DecWin win = S.slot[it & 1].win;
        if (win.kind == kWinSkip) {
            if (t == 0) { hap_st_release(&done[w], 1u); fetch_window(it + 1); }
            continue;
        }
        ChunkJob &job = jobs[win.job];
        const uint8_t *__restrict__ src = job.src;
        uint8_t *__restrict__ dst = job.dst;
        const uint32_t in_end = job.src_bytes, expected = job.dst_bytes;
        if (win.kind == kWinRaw) {
            const uint8_t *s = src + win.in_off;
            uint8_t *d = dst + win.out_off;
            if ((((uintptr_t)s | (uintptr_t)d) & 15) == 0) {
                const uint4 *s4 = reinterpret_cast<const uint4 *>(s);
                uint4 *d4 = reinterpret_cast<uint4 *>(d);
                const uint32_t n4 = win.in_len >> 4;
                for (uint32_t i = t; i < n4; i += kExThreads) d4[i] = s4[i];
                for (uint32_t i = (n4 << 4) + t; i < win.in_len; i += kExThreads) d[i] = s[i];
            } else {
                for (uint32_t i = t; i < win.in_len; i += kExThreads) d[i] = s[i];
            }
            if (t == 0) fetch_window(it + 1);
            HAP_PHASE_MARK(kPhOther);
            continue;   // nobody waits for a verbatim window
        }
        const bool embedded = win.first == kNoDeps;     // entries come from the frame: nothing in them is trusted
        const uint32_t sub = 1u << win.sub_log2;
        const uint32_t nsub_all = (win.in_len + sub - 1) >> win.sub_log2;
        const uint32_t nsub = nsub_all < (uint32_t)kExThreads ? nsub_all : (uint32_t)kExThreads;   // the last thread walks to the window's end
        const bool fits = win.in_len <= (uint32_t)kExMaxIn && win.in_off <= in_end && win.in_len <= in_end - win.in_off &&
                          win.out_off <= expected && win.out_len <= expected - win.out_off;
        if (!fits) {   // (uniform: every thread computed it from the same window and chunk records)
            if (t == 0) { job.status = embedded ? kStatusIndexMismatch : (uint32_t)HapResult_Bad_Frame; __threadfence(); hap_st_release(&done[w], 1u); fetch_window(it + 1); }
            continue;
        }
        // ---- stage the window (TMA bulk copy), read the entries meanwhile ---------------------------------------------
        uint32_t ent = kIndexNoEntry;
        const uint32_t staged = in_end - win.in_off < win.in_len + (uint32_t)kExLook ? in_end - win.in_off : win.in_len + (uint32_t)kExLook;
        stage_bytes(S.cin + 32, src + win.in_off, staged, &S.bar, t);
        if (t == 0) fetch_window(it + 1);
        if ((uint32_t)t < nsub) ent = win.entries[t];
        if (embedded && (uint32_t)t + kExThreads < nsub_all && win.entries[t + kExThreads] != kIndexNoEntry) F.mismatch = 1;  // no starts beyond piece 255
        hap_mbar_wait(&S.bar, phase);
        phase ^= 1;
        __syncthreads();
        HAP_PHASE_MARK(kPhStage);
        const uint32_t a_sh = (uint32_t)((uintptr_t)(src + win.in_off) & 15);
        const uint8_t *cin = S.cin + 32 + a_sh;
        const uint32_t wb = win.in_off;

        // ---- walk: every entered piece from its entry to its end ---------------------------------------------------------------
        const uint32_t my_lo = (uint32_t)t * sub;
        const uint32_t my_hi = ((uint32_t)t + 1 == nsub) ? win.in_len : ((uint32_t)t + 1) * sub;
        const bool entered = (uint32_t)t < nsub && ent != kIndexNoEntry;
        WalkResult wr;
        wr.exit = 0; wr.count = 0; wr.out_bytes = 0; wr.invalid = 0; wr.coarse = 0;
        if (entered) {
            if (my_lo + ent >= my_hi) {
                wr.invalid = 1;
            } else {
                wr = walk_piece(cin, wb, my_lo + ent, my_hi, in_end);
                // an element that starts in the window may END beyond it (its payload belongs to the next window of an
                // on-the-fly index); a fragment of an embedded index is self-contained
                if (!wr.invalid && wr.exit < win.in_len) {
                    uint32_t b = wr.exit >> win.sub_log2;
                    b = b < (uint32_t)kExThreads ? b : (uint32_t)kExThreads - 1;
                    S.landed[b] = 1;
                }
                if (embedded && wr.exit > win.in_len) wr.invalid = 1;
            }
        }
        if (wr.invalid) F.fail = 1;
        HAP_PHASE_MARK(kPhWalk);
        uint32_t total_e, total_o;
        const uint32_t ebase = block_excl_sum<kExThreads>(wr.count, &total_e, S.scratch);
        const uint32_t obase = block_excl_sum<kExThreads>(wr.out_bytes > 0x40000000u ? 0x40000000u : wr.out_bytes, &total_o, S.scratch);
        if (embedded) {
            // the entries must describe exactly the chain that starts at byte 0 of the fragment: a piece is entered if and
            // only if an exit lands in it (piece 0: the fragment's first element), at the entry's very offset
            const bool should = (uint32_t)t < nsub && (t == 0 || S.landed[t]);
            if (should != entered) F.mismatch = 1;
            if (t == 0 && (!entered || ent != 0)) F.mismatch = 1;
            if (entered && !wr.invalid && wr.exit < win.in_len) {
                uint32_t b = wr.exit >> win.sub_log2;
                b = b < (uint32_t)kExThreads ? b : (uint32_t)kExThreads - 1;
                if (b * sub + win.entries[b] != wr.exit) F.mismatch = 1;
            }
        }
        if (t == 0 && total_o != win.out_len) F.fail = 1;
#if HAPB200_EX_UNIT_PATH
        const bool coarse = __syncthreads_or(wr.coarse != 0) != 0;   // the barrier the checks below need, OR-ing the walk's grain test
#else
        __syncthreads();
#endif
        HAP_PHASE_MARK(kPhScan);
        if (F.fail || F.mismatch) {
            if (t == 0) { job.status = embedded ? kStatusIndexMismatch : (uint32_t)HapResult_Bad_Frame; __threadfence(); hap_st_release(&done[w], 1u); }
            continue;
        }
#if HAPB200_EX_UNIT_PATH
        if (embedded && !coarse) {
            // A copy that reads before the fragment is flagged in fail_desc, the descriptor stage's flag: mismatch may still be
            // tested by slower threads behind the barrier above.  Either way the chunk ends as kStatusIndexMismatch (repair).
            int &crossing = F.fail_desc;
            const bool ok = execute_units(S, crossing, 32 + a_sh, wb, in_end, entered, my_lo + ent, my_hi, obase, dst + win.out_off, win.out_len);
            __syncthreads();
            HAP_PHASE_MARK(kPhWrite);
            HAP_PHASE_COUNT(kPhUnitWindows);
            if (t == 0) {
                if (!ok) job.status = kStatusIndexMismatch;
#ifdef HAPB200_EMU
                else emu_unit_windows()++;
#endif
                __threadfence();
                hap_st_release(&done[w], 1u);
            }
            continue;
        }
#endif

        // ---- passes: as many pieces as the descriptor arrays hold -------------------------------------------------------------
        uint32_t pbase_e = 0;
        bool waited = embedded;     // windows of an on-the-fly index wait once for the earlier windows their copies read
        bool bad = false;
        while (pbase_e < total_e) {
            bool keep;
            uint32_t next_e, P0, P1;
            if (total_e <= (uint32_t)kExMaxElems) {
                keep = entered;
                next_e = total_e;
                P0 = win.out_off;
                P1 = win.out_off + total_o;
            } else {
                const bool cand = entered && ebase >= pbase_e;
                keep = cand && ebase + wr.count - pbase_e <= (uint32_t)kExMaxElems;
                uint32_t m_next = cand && !keep ? ebase : 0xFFFFFFFFu;
                uint32_t m_p0 = keep ? obase : 0xFFFFFFFFu;
                uint32_t m_p1 = keep ? obase + wr.out_bytes : 0u;
                block_min_min_max(m_next, m_p0, m_p1, S.red);
                next_e = m_next == 0xFFFFFFFFu ? total_e : m_next;
                P0 = win.out_off + m_p0;
                P1 = win.out_off + m_p1;
            }
            const uint32_t pass_e = next_e - pbase_e;

            // ---- descriptors.  e_a packs the SOURCE of an element as (kind << 30) | position:
            //      kSrcIn  : bytes of the compressed input at `position` (literals, and copies flattened onto them)
            //      kSrcOut : bytes of the output at `position` (plain copies; offset >= length)
            //      kSrcRun : periodic fill with period `position` (= the offset) of the e_b[e] - offset .. e_b[e] bytes
            if (keep) {
                uint32_t pos = my_lo + ent, e = ebase - pbase_e, o = win.out_off + obase, msrc = 0xFFFFFFFFu;
                while (pos < my_hi) {
                    uint32_t len, aux, hdr, kind;
                    read_element_header(cin + pos, wb + pos, in_end, len, aux, hdr, kind);
                    S.e_dst[e] = o;
                    S.e_len[e] = len;
                    if (kind == 0) {
                        S.e_a[e] = kSrcIn | aux;
                        S.e_b[e] = 0;  // literals break same-offset runs (a copy's offset is never 0)
                        pos += hdr + len;
                    } else {
                        if (aux == 0 || aux > o) F.fail_desc = 1;  // offset 0 or before the start of the output
                        else if (o - aux < msrc) msrc = o - aux;
                        S.e_a[e] = aux >= len ? (kSrcOut | (o - aux)) : (kSrcRun | aux);
                        S.e_b[e] = aux;  // the offset, for run detection below; becomes the run base afterwards
                        pos += hdr;
                    }
                    o += len;
                    e++;
                }
                if (!waited && msrc < win.out_off) atomicMin(&F.min_src, msrc);
                // a fragment of an embedded index is decoded without waiting for the others: a copy that reads before it
                // is legal Snappy, but only the repair pass (on-the-fly index, with waits) may execute it
                // (fail_desc, not mismatch: slower threads may still be testing mismatch behind the walk's barrier)
                if (embedded && msrc < win.out_off) F.fail_desc = 1;
            }
            __syncthreads();
            if (F.fail_desc) { bad = true; break; }

            // ---- same-offset runs: a copy with the offset of the copy right before it continues that copy's
            //      match, so it is a periodic fill of the run head's base period, independent of its neighbours --
            {
                const uint32_t strip = (pass_e + kExThreads - 1) / kExThreads;
                const uint32_t lo = t * strip < pass_e ? t * strip : pass_e;
                const uint32_t hi = lo + strip < pass_e ? lo + strip : pass_e;
                // Pass 1: flag continuations in the spare top bit of e_len (copies are at most 64 long) and find
                // the last run head of the strip.
                uint32_t last_head = 0;  // index + 1
                for (uint32_t e = lo; e < hi; e++) {
                    const uint32_t off = S.e_b[e];
                    const bool cont = e > 0 && off != 0 && off == S.e_b[e - 1];
                    if (cont) S.e_len[e] |= 0x80000000u;
                    else last_head = e + 1;
                }
                uint32_t unused;
                uint32_t head = block_excl_max<kExThreads>(last_head, &unused, S.scratch);  // ends with a barrier
                // Pass 2: e_b becomes the base (destination of the run head); continuations become periodic fills.
                for (uint32_t e = lo; e < hi; e++) {
                    const uint32_t off = S.e_b[e];
                    if (S.e_len[e] & 0x80000000u) {
                        S.e_len[e] &= 0x7FFFFFFFu;
                        S.e_a[e] = kSrcRun | off;
                        S.e_b[e] = S.e_dst[head - 1];
                    } else {
                        head = e + 1;
                        S.e_b[e] = S.e_dst[e];
                    }
                }
            }
            __syncthreads();

            // ---- flatten copy-of-copy chains.  DXT payloads are full of "same as the previous block except a few
            //      bytes": a copy whose source is itself a copy, hundreds deep.  A plain copy whose source bytes lie
            //      inside ONE earlier element of this pass takes over that element's source (pointer jumping on
            //      the packed e_a words; a racing update only makes the hop longer, never wrong).  Chains end at
            //      literals (-> read the input instead) or before this pass (-> already written). --------------
            for (uint32_t e = t; e < pass_e; e += kExThreads) {
                uint32_t a = S.e_a[e];
                if ((a & kSrcMask) != kSrcOut) continue;
                const uint32_t len = S.e_len[e];
                bool changed = false;
#pragma unroll 1
                for (int hop = 0; hop < kFlattenHops; hop++) {
                    const uint32_t sp = a & kPosMask;
                    if (sp < P0) break;                        // reads (at least partly) what earlier passes / windows wrote
                    uint32_t lo2 = 0, hi2 = e;                 // last element with e_dst <= sp (it is before e)
                    while (hi2 - lo2 > 1) {
                        const uint32_t m = (lo2 + hi2) >> 1;
                        if (S.e_dst[m] <= sp) lo2 = m; else hi2 = m;
                    }
                    const uint32_t f = lo2, fd = S.e_dst[f];
                    if (sp + len > fd + S.e_len[f]) break;     // spans several producers
                    const uint32_t fa = S.e_a[f];
                    if ((fa & kSrcMask) == kSrcRun) break;     // periodic producer: stay dependent on it
                    a = (fa & kSrcMask) | ((fa & kPosMask) + (sp - fd));
                    changed = true;
                    if ((fa & kSrcMask) == kSrcIn) break;      // landed on input bytes: fully resolved
                }
                if (changed) S.e_a[e] = a;
            }
            __syncthreads();

            // ---- earlier windows of the chunk this window's copies read (on-the-fly index only): wait for them once ----
            if (!waited) {
                waited = true;
                if (t == 0 && F.min_src < win.out_off) {
                    const uint32_t need = F.min_src;
                    for (uint32_t j = w; j > win.first;) {
                        j--;
                        const uint32_t jo = wins[j].out_off, jl = wins[j].out_len;
                        if (wins[j].kind == kWinSnappy) {
                            uint32_t spins = 0;
                            while (hap_ld_acquire(&done[j]) == 0) { if (++spins > 64) hap_nanosleep(200); }
                        }
                        if (jo <= need || jo + jl <= need) break;   // this window starts at or before the earliest byte needed
                    }
                }
                __syncthreads();
            }

            // ---- execute, output-centric: tiles of 32 KiB, groups of 16 aligned bytes ---------------------------------------------
            for (uint32_t T0 = P0; T0 < P1; T0 += kExTile) {
                TileCtx C;
                C.src = src; C.dst = dst; C.src_bytes = in_end; C.dst_bytes = expected;
                C.cin = cin; C.wb = wb; C.staged = staged;
                C.T0 = T0;
                C.T1 = T0 + kExTile < P1 ? T0 + kExTile : P1;
                const uint32_t shift = (uint32_t)((uintptr_t)(dst + T0) & 15);
                C.gbase = (int32_t)T0 - (int32_t)shift;
                const uint32_t ngroups = (uint32_t)((int32_t)C.T1 - C.gbase + 15) >> 4;
                for (uint32_t g = t; g < ngroups; g += kExThreads) { S.gfirst[g] = 0; S.gdone[g] = 0; }
                __syncthreads();
                // the element that holds the first byte of each group: elements mark the first group whose first byte they hold ...
                for (uint32_t e = t; e < pass_e; e += kExThreads) {
                    const uint32_t d = S.e_dst[e], l = S.e_len[e];
                    if (d + l <= C.T0 || d >= C.T1) continue;
                    uint32_t gs = 0;
                    if (d > C.T0) gs = (uint32_t)((int32_t)d - C.gbase + 15) >> 4;
                    const int32_t first_byte = gs == 0 ? (int32_t)C.T0 : C.gbase + 16 * (int32_t)gs;
                    if (gs < ngroups && first_byte < (int32_t)(d + l)) S.gfirst[gs] = (uint16_t)(e + 1);
                }
                __syncthreads();
                // ... and a running maximum fills in the groups that lie inside one long element
                {
                    const uint32_t per = (ngroups + kExThreads - 1) / kExThreads;
                    const uint32_t glo = t * per < ngroups ? t * per : ngroups, ghi = glo + per < ngroups ? glo + per : ngroups;
                    uint32_t local = 0;
                    for (uint32_t g = glo; g < ghi; g++) local = S.gfirst[g] > local ? S.gfirst[g] : local;
                    uint32_t unused;
                    uint32_t run = block_excl_max<kExThreads>(local, &unused, S.scratch);
                    for (uint32_t g = glo; g < ghi; g++) {
                        run = S.gfirst[g] > run ? S.gfirst[g] : run;
                        S.gfirst[g] = (uint16_t)run;
                    }
                }
                __syncthreads();
                for (uint32_t round = 1;; round++) {
                    int pending = 0;
                    for (uint32_t g = t; g < ngroups; g += kExThreads)
                        if (S.gdone[g] == 0 && !assemble_group(S, C, g, round)) pending = 1;
                    if (round >= 65000u) { F.fail_desc = 1; pending = 0; }   // (a dependency chain deeper than any window has groups)
                    if (!__syncthreads_or(pending)) break;
                }
            }
            pbase_e = next_e;
            __syncthreads();
        }
        __syncthreads();
        if (t == 0) {
            if (bad || F.fail_desc) job.status = embedded ? kStatusIndexMismatch : (uint32_t)HapResult_Bad_Frame;
            __threadfence();
            hap_st_release(&done[w], 1u);
        }
        HAP_PHASE_MARK(kPhOther);
    }
    HAP_PHASE_END();
}

// =====================================================================================================================
//  unit kernel: the unit path on its own, ahead of the execute kernel
// =====================================================================================================================
// snappy_execute_units_kernel decodes the pass-0 fragments of embedded indexes (win.first == kNoDeps) whose elements are
// all 8-byte granular, with the decisions of the execute kernel's unit path (execute_units), in a kernel that holds only
// what that path needs: the staged window and one 16-bit unit map built in place over the records, 41 KB of shared memory
// against the execute kernel's 54 KB, so that 5 windows are resident per SM instead of 4.  Per window: one scan (output
// bytes) instead of two, the element owning each unit found by one max-scan over packed (unit, record) keys, and the
// period of an overlapping copy followed by a counter instead of a modulo per unit.  Fragments of an embedded index never
// wait for each other, so windows are taken in list order.  A window it finishes (decoded, or found not to match its
// index: kStatusIndexMismatch, the repair pass decodes the chunk) gets done[w] = 1; a window it declines (an element that
// is not 8-byte granular) is left to the execute kernel, which then skips the finished ones (DecodeCtl::units_ran).
#ifndef HAPB200_EX_UNIT_KERNEL
#define HAPB200_EX_UNIT_KERNEL 1
#endif
#ifndef HAPB200_UX_MIN_BLOCKS
#define HAPB200_UX_MIN_BLOCKS 5
#endif
constexpr int kUxThreads = 256;

struct UnitSmem {
    uint8_t cin[kExMaxIn + kExLook + 48];            // staged window, cin[a + i] = byte i of the window (a = its address & 15)
    uint16_t map[kExUnits];                          // records, then (in place) the source of every 8-byte unit
    uint8_t landed[kUxThreads];                      // a chain exit lands in this piece
    uint32_t scratch[kUxThreads / 32];
    DecWin win[2];                                   // the window being worked on and the next one (fetched by thread 0)
    uint32_t ticket[2];
    hap_mbar_t bar;
    int mismatch[2];                                 // per window, two sets used alternately (as ExecSmem::flags)
};

#ifdef HAPB200_EMU
inline uint64_t &emu_unit_kernel_windows() { static uint64_t n = 0; return n; }   // windows this kernel decoded (tests only)
inline uint64_t &emu_unit_kernel_declined() { static uint64_t n = 0; return n; }  // windows it left to the execute kernel
#endif

// thread 0: the next window this kernel takes, and its record.  Only windows a chunk lists are looked at (the list has
// reserved slots that were never written).
__device__ __noinline__ void fetch_unit_window(const ChunkJob *jobs, uint32_t njobs, unsigned long long n_tickets, const DecWin *wins, DecodeCtl *ctl,
                                               DecWin *win_out, uint32_t *ticket_out)
{
    uint32_t w = 0xFFFFFFFFu;
    for (;;) {
        const unsigned long long T = atomicAdd(&ctl->unit_ticket, 1u);
        if (T >= n_tickets) break;
        const uint32_t k = (uint32_t)(T / njobs), j = (uint32_t)(T % njobs);
        if (jobs[j].compressor == 0 || jobs[j].mode != kJobReady || k >= jobs[j].win_count) continue;
        const DecWin x = wins[jobs[j].win_base + k];
        if (x.kind == kWinSnappy && x.first == kNoDeps) { *win_out = x; w = jobs[j].win_base + k; break; }
    }
    *ticket_out = w;
}

__global__ void __launch_bounds__(kUxThreads, HAPB200_UX_MIN_BLOCKS) snappy_execute_units_kernel(ChunkJob *jobs, uint32_t njobs, const DecWin *wins,
                                                                                                DecodeCtl *ctl, uint32_t *done)
{
    static_assert(kExUnits == kUnitStripLen * kUxThreads, "16 units per thread");
    HAP_DYN_SMEM(smem_raw);
    UnitSmem &S = *reinterpret_cast<UnitSmem *>(smem_raw);
    const int t = threadIdx.x;
    const unsigned long long n_tickets = (unsigned long long)ctl->max_k_units * njobs;   // (final: the listing kernels ran before)
    uint4 *map4 = reinterpret_cast<uint4 *>(S.map);
    if (t == 0) {
        hap_mbar_init(&S.bar, 1);
        S.mismatch[0] = 0;
        S.mismatch[1] = 0;
        if (blockIdx.x == 0) ctl->units_ran = 1;   // (read by the execute kernel, which runs behind this one)
        fetch_unit_window(jobs, njobs, n_tickets, wins, ctl, &S.win[0], &S.ticket[0]);
    }
    uint32_t phase = 0;
    HAP_PHASE_BEGIN();
    for (uint32_t it = 0;; it++) {
        __syncthreads();   // the previous window's reads of the staging buffer and the map are over; slot it & 1 is filled
        const uint32_t w = S.ticket[it & 1];
        if (w == 0xFFFFFFFFu) break;
        int &mismatch = S.mismatch[it & 1];
        if (t == 0) S.mismatch[(it + 1) & 1] = 0;
        const DecWin win = S.win[it & 1];
        ChunkJob &job = jobs[win.job];
        const uint8_t *__restrict__ src = job.src;
        uint8_t *__restrict__ out = job.dst + win.out_off;
        const uint32_t in_end = job.src_bytes, expected = job.dst_bytes;
        const uint32_t sub = 1u << win.sub_log2;
        const uint32_t nsub_all = (win.in_len + sub - 1) >> win.sub_log2;
        const uint32_t nsub = nsub_all < (uint32_t)kUxThreads ? nsub_all : (uint32_t)kUxThreads;   // the last thread walks to the window's end
        const bool fits = win.in_len <= (uint32_t)kExMaxIn && win.in_off <= in_end && win.in_len <= in_end - win.in_off &&
                          win.out_off <= expected && win.out_len <= expected - win.out_off && win.out_len <= kIndexFragBytes;
        if (!fits) {   // (uniform)
            if (t == 0) {
                job.status = kStatusIndexMismatch;
                done[w] = 1u;
                fetch_unit_window(jobs, njobs, n_tickets, wins, ctl, &S.win[(it + 1) & 1], &S.ticket[(it + 1) & 1]);
            }
            continue;
        }
        const uint32_t staged = in_end - win.in_off < win.in_len + (uint32_t)kExLook ? in_end - win.in_off : win.in_len + (uint32_t)kExLook;
        stage_bytes(S.cin, src + win.in_off, staged, &S.bar, t);
        if (t == 0) fetch_unit_window(jobs, njobs, n_tickets, wins, ctl, &S.win[(it + 1) & 1], &S.ticket[(it + 1) & 1]);
        const uint32_t ent = (uint32_t)t < nsub ? win.entries[t] : (uint32_t)kIndexNoEntry;
        if ((uint32_t)t + kUxThreads < nsub_all && win.entries[t + kUxThreads] != kIndexNoEntry) mismatch = 1;   // no starts beyond piece 255
        S.landed[t] = 0;
        map4[2 * t] = make_uint4(0, 0, 0, 0);
        map4[2 * t + 1] = make_uint4(0, 0, 0, 0);
        hap_mbar_wait(&S.bar, phase);
        phase ^= 1;
        __syncthreads();
        HAP_PHASE_MARK(kPhStage);
        const uint32_t coff = (uint32_t)((uintptr_t)(src + win.in_off) & 15);
        const uint8_t *cin = S.cin + coff;
        const uint32_t wb = win.in_off;

        // ---- walk: every entered piece from its entry to its end (as the execute kernel's walk, for a self-contained fragment)
        const uint32_t my_lo = (uint32_t)t * sub;
        const uint32_t my_hi = ((uint32_t)t + 1 == nsub) ? win.in_len : ((uint32_t)t + 1) * sub;
        const bool entered = (uint32_t)t < nsub && ent != kIndexNoEntry;
        WalkResult wr;
        wr.exit = 0; wr.count = 0; wr.out_bytes = 0; wr.invalid = 0; wr.coarse = 0;
        if (entered) {
            if (my_lo + ent >= my_hi) {
                wr.invalid = 1;
            } else {
                wr = walk_piece(cin, wb, my_lo + ent, my_hi, in_end);
                if (!wr.invalid && wr.exit < win.in_len) {
                    uint32_t b = wr.exit >> win.sub_log2;
                    b = b < (uint32_t)kUxThreads ? b : (uint32_t)kUxThreads - 1;
                    S.landed[b] = 1;
                    if (b * sub + win.entries[b] != wr.exit) mismatch = 1;
                }
                if (wr.exit > win.in_len) wr.invalid = 1;
            }
        }
        HAP_PHASE_MARK(kPhWalk);
        uint32_t total_o;
        const uint32_t obase = block_excl_sum<kUxThreads>(wr.out_bytes > 0x40000000u ? 0x40000000u : wr.out_bytes, &total_o, S.scratch);
        // the entries must describe exactly the chain that starts at byte 0 of the fragment (see the execute kernel)
        const bool should = (uint32_t)t < nsub && (t == 0 || S.landed[t]);
        int bad = wr.invalid || should != entered || (t == 0 && (!entered || ent != 0)) || total_o != win.out_len;
        bad = __syncthreads_or(bad || mismatch);
        const bool coarse = __syncthreads_or(wr.coarse != 0) != 0;
        HAP_PHASE_MARK(kPhScan);
        if (bad) {
            if (t == 0) { job.status = kStatusIndexMismatch; done[w] = 1u; }
            continue;
        }
        if (coarse) {
            // not 8-byte granular: the execute kernel decodes this window (its tickets reach chunk window k)
            if (t == 0) {
                atomicMax(&ctl->max_k_rest, w - job.win_base + 1);
#ifdef HAPB200_EMU
                emu_unit_kernel_declined()++;
#endif
            }
            continue;
        }

        // ---- records: one per element at its first unit (kUnitLit + stream position of a literal, the copy's distance in units)
        int crossing = 0;
        if (entered) {
            uint32_t u = obase >> 3, pos = my_lo + ent;   // (obase is a multiple of 8: every element before this piece is)
            while (pos < my_hi) {
                uint32_t len, aux, hdr, kind;
                read_element_header(cin + pos, wb + pos, in_end, len, aux, hdr, kind);   // (the walk checked every header)
                if (kind == 0) {
                    S.map[u] = (uint16_t)(kUnitLit + (aux - wb));
                    pos += hdr + len;
                } else {
                    const uint32_t d = aux >> 3;
                    if (d > u) { crossing = 1; break; }   // reads before the fragment: the repair pass decodes the chunk
                    S.map[u] = (uint16_t)d;
                    pos += hdr;
                }
                u += len >> 3;
            }
        }
        if (__syncthreads_or(crossing)) {
            if (t == 0) { job.status = kStatusIndexMismatch; done[w] = 1u; }
            continue;
        }
        HAP_PHASE_MARK(kPhRecords);

        // ---- map: thread t owns units 16t .. 16t + 15.  The element running into the strip comes from a max-scan over
        //      (unit + 1) << 16 | record of the strip's last element start; the unit's source then follows by counting.
        const uint32_t U = win.out_len >> 3, u0 = kUnitStripLen * (uint32_t)t;
        uint32_t r[kUnitStripLen];
        {
            const uint4 a = map4[2 * t], b = map4[2 * t + 1];
            const uint32_t wd[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
            for (int k = 0; k < kUnitStripLen; k++) r[k] = (wd[k >> 1] >> (16 * (k & 1))) & 0xFFFFu;
        }
        uint32_t last = 0;
#pragma unroll
        for (int k = 0; k < kUnitStripLen; k++) last = r[k] != 0 ? ((u0 + k + 1) << 16) | r[k] : last;
        uint32_t unused;
        const uint32_t carry = block_excl_max<kUxThreads>(last, &unused, S.scratch);   // ends with a barrier: the records are read
        // v: the source of the current unit; per: the copy's period (distance), 0 for a literal; q: units since the period began
        uint32_t v = 0, per = 0, q = 0, step = 0;
        if (carry) {
            const uint32_t start = (carry >> 16) - 1, rs = carry & 0xFFFFu, d = u0 - start;
            if (rs >= kUnitLit) { v = rs + 8 * d; step = 8; per = 0; }
            else { per = rs; q = d % rs; v = start - rs + q; step = 1; }
        }
        int pending = 0;
        uint32_t m[kUnitStripLen];
#pragma unroll
        for (int k = 0; k < kUnitStripLen; k++) {
            const uint32_t u = u0 + k;
            if (r[k] != 0) {
                if (r[k] >= kUnitLit) { v = r[k]; step = 8; per = 0; }
                else { per = r[k]; q = 0; v = u - per; step = 1; }
            } else if (k > 0) {   // (k == 0: v, q are those of unit u0 already)
                v += step;
                if (per != 0 && ++q == per) { q = 0; v -= per; }
            }
            m[k] = v;
            pending |= u < U && v < kUnitLit;
        }
#pragma unroll
        for (int h = 0; h < 2; h++)
            map4[2 * t + h] = make_uint4((m[8 * h] & 0xFFFFu) | (m[8 * h + 1] << 16), (m[8 * h + 2] & 0xFFFFu) | (m[8 * h + 3] << 16),
                                         (m[8 * h + 4] & 0xFFFFu) | (m[8 * h + 5] << 16), (m[8 * h + 6] & 0xFFFFu) | (m[8 * h + 7] << 16));
        pending = __syncthreads_or(pending);
        HAP_PHASE_MARK(kPhMap);

        // ---- resolve: map[u] = map[map[u]] until every unit names stream bytes (sources are strictly earlier units)
        for (int round = 0; pending; round++) {
            pending = 0;
            for (uint32_t u = t; u < U; u += kUxThreads) {
                const uint32_t x = S.map[u];
                if (x < kUnitLit) {
                    const uint32_t x2 = S.map[x];
                    S.map[u] = (uint16_t)x2;
                    pending |= x2 < kUnitLit;
                }
            }
            pending = __syncthreads_or(pending);
            HAP_PHASE_MARK(kPhRounds);
            HAP_PHASE_COUNT(kPhRoundCount);
            if (pending && round == kUnitMaxRounds) { crossing = 1; break; }   // (cannot happen: chains are at most 4096 units deep)
        }
        if (crossing) {
            if (t == 0) { job.status = kStatusIndexMismatch; done[w] = 1u; }
            continue;
        }

        // ---- write: thread g assembles destination-aligned 16-byte group g from two or three units of the staged window
        const uint32_t *c32 = reinterpret_cast<const uint32_t *>(S.cin);
        const uint32_t mis = (uint32_t)((uintptr_t)out & 15);
        const uint32_t ngroups = (mis + win.out_len + 15) >> 4;
        for (uint32_t g = t; g < ngroups; g += kUxThreads) {
            const int32_t x = 16 * (int32_t)g - (int32_t)mis;
            const int32_t ua = x >> 3;   // (floor: -2 or -1 for the first group of a misaligned fragment)
            const uint32_t rr = (uint32_t)x & 7u;
            uint32_t wv[6];
#pragma unroll
            for (int k = 0; k < 3; k++) {
                const int32_t u = ua + k;
                wv[2 * k] = 0;
                wv[2 * k + 1] = 0;
                if (u >= 0 && (uint32_t)u < U && (k < 2 || rr != 0)) {
                    const uint32_t b = coff + (uint32_t)S.map[u] - kUnitLit, i = b >> 2, sh = 8 * (b & 3);
                    const uint32_t s0 = c32[i], s1 = c32[i + 1], s2 = c32[i + 2];
                    wv[2 * k] = __funnelshift_r(s0, s1, sh);
                    wv[2 * k + 1] = __funnelshift_r(s1, s2, sh);
                }
            }
            const uint32_t qq = rr >> 2, sh = 8 * (rr & 3);
            const uint32_t o0 = __funnelshift_r(wv[qq], wv[qq + 1], sh), o1 = __funnelshift_r(wv[qq + 1], wv[qq + 2], sh);
            const uint32_t o2 = __funnelshift_r(wv[qq + 2], wv[qq + 3], sh), o3 = __funnelshift_r(wv[qq + 3], wv[qq + 4], sh);
            if (x >= 0 && (uint32_t)x + 16 <= win.out_len) {
                *reinterpret_cast<uint4 *>(out + x) = make_uint4(o0, o1, o2, o3);   // 16-byte aligned by the choice of mis
            } else {
                const uint32_t ow[4] = {o0, o1, o2, o3};
                for (int i = 0; i < 16; i++)
                    if (x + i >= 0 && (uint32_t)(x + i) < win.out_len) out[x + i] = (uint8_t)(ow[i >> 2] >> (8 * (i & 3)));
            }
        }
        if (t == 0) {
            done[w] = 1u;
#ifdef HAPB200_EMU
            emu_unit_kernel_windows()++;
#endif
        }
        HAP_PHASE_MARK(kPhWrite);
        HAP_PHASE_COUNT(kPhUnitWindows);
    }
    HAP_PHASE_END();
}

}  // namespace hapb200
