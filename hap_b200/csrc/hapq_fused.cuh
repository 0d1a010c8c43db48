// hap_b200/csrc/hapq_fused.cuh -- Hap Q from RGBA8 in one kernel: the scaled-YCoCg block fit of K1-K4 in front of K5.
//
// The two-kernel path writes the DXT texture to HBM (bc_encode_kernel<kBcYCoCg>) and reads it back (K5).  Here the CTA
// that compresses a fragment fits the fragment's blocks itself, straight into the fragment's shared-memory image: one launch
// instead of two, the texture is not read back, and the barrier-free fit of one resident CTA can issue while the other
// waits on the compressor's barriers and shared-memory round trips (DESIGN.md §4 and §6 give what that bought: 0.6 ms of
// 12.9 per 444 4K frames).  The blocks are still written through to
// the texture scratch, because the plan and place kernels copy a chunk (hap.c:460) or the whole section (hap.c:478) from
// it when compression does not pay.  Same shape as K5 (persistent grid, 512 threads, two CTAs per SM, EncodeSmem), same
// block fit (encode_ycocg_dxt5), same compressor: the frames are byte-identical to those of the two-kernel path.
//
// hapq_fused_place_kernel goes one step further: it writes each element stream from shared memory to its final place in
// the frame, so the streams no longer go through scratch and hap_place_fragments_kernel only copies raw fallbacks.
// hapq_ws_place_kernel does the same with the fit and the compressor in warp groups of their own (the library's choice).
#pragma once
#include "bc_encode.cuh"
#include "hap_assemble.cuh"
#include "snappy_encode.cuh"

#ifndef HAPB200_FUSED_HAPQ
#define HAPB200_FUSED_HAPQ 1   // 0: the library never selects the fused kernel (A/B builds)
#endif
#ifndef HAPB200_FUSED_PLACE
#define HAPB200_FUSED_PLACE 1  // 0: the fused kernel never writes the frames itself (fused kernel, plan, place: A/B builds)
#endif
#ifndef HAPB200_FUSED_WS
#define HAPB200_FUSED_WS 1     // 0: hapq_fused_place_kernel writes the frames, not hapq_ws_place_kernel (A/B builds)
#endif

namespace hapb200 {

// The texture geometries the fused kernel takes: one compressed section cut into whole chunks of whole 16-byte blocks, so that
// every block lies in exactly one fragment and every fragment starts at a block.
HAP_HD bool fused_hapq_geometry(const FrameGeom &G)
{
    const SectionGeom &s = G.s[0];
    return G.sections == 1 && s.compress && (uint64_t)s.chunks * s.chunk_bytes == s.bytes && s.chunk_bytes % 16 == 0;
}

// The fit of fragment gfrag by the kEncThreads threads t = 0 .. 511 of a warp group: block blk0 + lb (lb = t, t + 512, ...
// < nblk) is fitted, stored to the shared-memory image `img` and written through to the texture.  Lanes take neighbouring
// blocks, so the four 16-byte row loads of a warp are coalesced as in bc_encode_kernel, and so are the 16-byte stores.
// The fit alone needs more than 64 registers (bc_encode_kernel gives it 72; capped at 64 it spills even in a kernel that
// does nothing else, here 7 values per block), so nothing else may live across it: only lb, nblk, blk0 and frame do, and
// the picture and texture addresses are derived from them for every block (the empty asm keeps the compiler from hoisting
// them out of the loop, where they would be spilled too).
__device__ __forceinline__ void fused_fit_blocks(uint2 *img, uint32_t t, const uint8_t *__restrict__ rgba, const BcGeom &B,
                                                 uint8_t *__restrict__ tex, const FrameGeom &G, uint32_t gfrag)
{
    const FragRef cur = locate_fragment(tex, G, gfrag);
    const uint32_t nblk = cur.units >> 1, blk0 = cur.tex_off >> 4;
    uint32_t frame = cur.frame;
#pragma unroll 1
    for (uint32_t lb = t; lb < nblk; lb += kEncThreads) {
        asm volatile("" : "+r"(frame));
        const uint32_t bi = blk0 + lb;
        uint32_t bx, by, px[16];
        block_xy(bi, B.blocks_x, B.inv_blocks_x, bx, by);
        load_block_rgba8(rgba + (uint64_t)frame * B.frame_bytes, B.row_bytes, bx, by, px);
        Block8 a, c;
        encode_ycocg_dxt5<false>(px, a, c);
        const uint4 v = make_uint4(a.lo, a.hi, c.lo, c.hi);
        reinterpret_cast<uint4 *>(img)[lb] = v;
        reinterpret_cast<uint4 *>(tex + (uint64_t)frame * G.s[0].in_stride + G.s[0].in_offset)[bi] = v;
    }
}

// The fit by the whole CTA into S.data; then the compressor's tables are cleared.
__device__ __forceinline__ void fused_fit_fragment(unsigned char *smem_raw, const uint8_t *__restrict__ rgba, const BcGeom &B,
                                                   uint8_t *__restrict__ tex, const FrameGeom &G, uint32_t gfrag)
{
    EncodeSmem &S = *reinterpret_cast<EncodeSmem *>(smem_raw);
    fused_fit_blocks(S.data, threadIdx.x, rgba, B, tex, G, gfrag);
    init_fragment_tables(S);
}

// The compressor on the fitted fragment in `img` (after the barrier behind the fit): each thread reloads its own strip from
// it; returns the size of the element stream now in `out`.
template <class Bar = CtaBarrier>
__device__ __forceinline__ uint32_t fused_compress_fragment(EncodeSmem &S, const uint2 *img, uint32_t *out, uint8_t *tex,
                                                            const FrameGeom &G, uint32_t gfrag)
{
    const uint32_t U = locate_fragment(tex, G, gfrag).units;
    const uint32_t i0 = threadIdx.x * kUnitStrip;
    uint2 d[kUnitStrip];
#pragma unroll
    for (int k = 0; k < kUnitStrip; k += 2) {
        const uint4 v = i0 + k < U ? *reinterpret_cast<const uint4 *>(&img[i0 + k]) : make_uint4(0, 0, 0, 0);   // (U is even)
        d[k] = make_uint2(v.x, v.y);
        d[k + 1] = make_uint2(v.z, v.w);
    }
    return U == (uint32_t)kFragUnits ? compress_fragment<true, Bar>(S, img, out, d, U, 2)
                                     : compress_fragment<false, Bar>(S, img, out, d, U, 2);
}

// rgba: RGBA8 pictures (geometry B: B.frame_bytes apart, rows B.row_bytes apart; B.out_stride is not used); tex: the texture
// scratch that G describes (16-byte aligned), written through; the other arguments are those of snappy_encode_fragments_kernel.
__global__ void __launch_bounds__(kEncThreads, 2) hapq_fused_encode_kernel(
    const uint8_t *__restrict__ rgba, BcGeom B, uint8_t *__restrict__ tex, FrameGeom G, uint32_t nfrag, uint8_t *__restrict__ scratch,
    uint32_t *__restrict__ frag_size, uint8_t *__restrict__ frag_entries)
{
    HAP_DYN_SMEM(smem_raw);
    for (uint32_t gfrag = blockIdx.x; gfrag < nfrag; gfrag += gridDim.x) {
        fused_fit_fragment(smem_raw, rgba, B, tex, G, gfrag);
        __syncthreads();
        // the fragment again, recomputed rather than kept live across the fit.  The compressor's shared-memory addresses are
        // derived after the fit too: the empty asm hides that `off` is 0, so the compiler cannot hoist them to the top of the
        // kernel, where they would be spilled around the fit.
        uint32_t off = 0;
        asm volatile("" : "+r"(off));
        EncodeSmem &S = *reinterpret_cast<EncodeSmem *>(smem_raw + off);
        const uint32_t total = fused_compress_fragment(S, S.data, S.out, tex, G, gfrag);
        store_fragment(S, total, gfrag, scratch, frag_size, frag_entries);
    }
}

// ---- the fused kernel that writes the frames ---------------------------------------------------------------------------
//
// A fragment's place in its frame follows from the sizes of the fragments before it (hap_plan_frames_kernel, pass 2):
// chunk 0 starts at data0 = outer_hdr + top_hdr + 4 + di (di = 5k + 8, hap.c:265-275), fragment j of chunk c at
// start_c + varint(chunk_bytes) + the sizes of fragments 0 .. j-1 of the chunk, and start_{c+1} = start_c + min(packed_c,
// chunk_bytes) with packed_c = varint(chunk_bytes) + the chunk's sizes (hap.c:460: a chunk that does not shrink is stored
// raw, in chunk_bytes).  Each fragment publishes its size as soon as it is compressed; the last fragment of a chunk, once
// it knows its place, publishes start_{c+1} too.  A fragment's look-back (one warp) adds the sizes of the earlier fragments
// of its chunk, then walks back over the earlier chunks of its frame: a published start ends the walk, else the chunk's
// size follows from its fragments' sizes.  It only ever waits for the SIZES of fragments with smaller tickets.
//
// The look-back and the store of a fragment are deferred until its CTA has fitted its next fragment (S.out is untouched by
// the fit), so the fragments before it have had a whole fit's time to publish their sizes.  Tickets (one atomic counter)
// hand out the fragments in order, as snappy_execute_kernel's windows: a CTA that waits holds a larger ticket than every
// fragment it waits for, and a fragment's size only waits for the look-back of its CTA's previous, smaller ticket; tickets
// are only taken by CTAs that run, so the smallest unfinished ticket never waits and nothing can deadlock, whatever share
// of the device the kernel gets.
//
// What a fragment writes, so that every byte ends right whatever the plan kernel decides afterwards: only bytes below
// start_c + chunk_bytes (past it the chunk is certainly raw, and the place kernel overwrites all of its bytes), and only
// bytes below top_hdr + bytes, where a verbatim section (hap.c:478) would end.  A complex frame can end up to top_hdr - 1
// bytes past that; those few bytes go to the fragment's scratch slot, at their offset in the stream, and the plan kernel
// copies them once it knows the section is complex.  The plan kernel writes the headers, tables, varints, index and
// lengths and lists the raw fragments; the place kernel then copies those, on the same stream.

// Where the fused kernel publishes what the look-back reads (zeroed before every launch)
struct FusedPlaceArgs {
    uint8_t *out;              // frames, out_stride apart
    uint64_t out_stride;
    uint32_t *ticket;          // next fragment to take
    uint32_t *size_flag;       // [nfrag]: 1 + the fragment's stream size, 0 until published
    uint32_t *next_start;      // [nfrag]: at the last fragment of a chunk, 1 + the next chunk's start, 0 until published
};
enum { kPlTicket = 0, kPlPend, kPlPendTotal, kPlOff, kPlStart };   // EncodeSmem::place
constexpr uint32_t kNoFragment = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t fused_wait_size(const uint32_t *size_flag, uint32_t g)
{
    uint32_t v, spins = 0;
    while ((v = hap_ld_acquire(size_flag + g)) == 0)
        if (++spins > 16) hap_nanosleep(100);
    return v - 1;
}

// sum of the published sizes of fragments g0 .. g0 + n - 1 (one warp; every lane gets it)
__device__ __forceinline__ uint32_t fused_size_sum(const uint32_t *size_flag, uint32_t g0, uint32_t n)
{
    uint32_t s = 0;
    for (uint32_t i = threadIdx.x & 31; i < n; i += 32) s += fused_wait_size(size_flag, g0 + i);
    return __reduce_add_sync(HAP_FULL_MASK, s);
}

// Warp 0: the place of fragment gfrag (`total` stream bytes) in its frame -> S.place[kPlOff], its chunk's start ->
// S.place[kPlStart]; the last fragment of a chunk publishes the next chunk's start.
__device__ __forceinline__ void fused_look_back(EncodeSmem &S, const FrameGeom &G, const FusedPlaceArgs &P, uint32_t gfrag, uint32_t total)
{
    const SectionGeom &s = G.s[0];
    uint32_t f, j;
    fast_divmod(gfrag, G.frags_per_frame, G.inv_frags_per_frame, f);
    const uint32_t c = fast_divmod(f, s.frags_per_chunk, s.inv_frags_per_chunk, j);
    const uint32_t fpc = s.frags_per_chunk, cb = s.chunk_bytes, vb = varint_bytes(cb);
    const uint32_t g_chunk = gfrag - j;   // my chunk's first fragment
    const uint32_t own = fused_size_sum(P.size_flag, g_chunk, j);
    uint32_t start = G.outer_hdr + s.top_hdr + 4u + 5u * s.chunks + 8u, acc = 0;   // data0, then the chunks walked over
    for (uint32_t cc = c; cc-- > 0;) {
        const uint32_t g0 = g_chunk - (c - cc) * fpc;
        const uint32_t e = __shfl_sync(HAP_FULL_MASK, (threadIdx.x & 31) == 0 ? hap_ld_acquire(P.next_start + g0 + fpc - 1) : 0u, 0);
        if (e != 0) { start = e - 1; break; }
        const uint32_t packed = vb + fused_size_sum(P.size_flag, g0, fpc);
        acc += packed < cb ? packed : cb;
    }
    start += acc;
    const uint32_t o = start + vb + own;
    if ((threadIdx.x & 31) == 0) {
        S.place[kPlOff] = o;
        S.place[kPlStart] = start;
        if (j == fpc - 1) {
            const uint32_t end = o + total, lim = start + cb;
            hap_st_release(P.next_start + gfrag, (end < lim ? end : lim) + 1u);
        }
    }
}

// All threads: fragment gfrag's stream (`n` bytes in `out`, S.out or a second buffer of its size) to its place (S.place, after
// the barrier behind the look-back).
// Destination-aligned 16-byte groups, each from five shared-memory words and four funnel shifts, one 16-byte store; the
// partial groups at either end are written bytewise, since the neighbouring fragments own their other bytes.
__device__ __forceinline__ void fused_store(const EncodeSmem &S, const uint32_t *out, const FrameGeom &G, const FusedPlaceArgs &P,
                                            uint8_t *__restrict__ scratch, uint32_t gfrag, uint32_t n)
{
    const uint32_t t = threadIdx.x;
    const SectionGeom &s = G.s[0];
    uint32_t f;
    const uint32_t frame = fast_divmod(gfrag, G.frags_per_frame, G.inv_frags_per_frame, f);
    const uint32_t o = S.place[kPlOff], lim_chunk = S.place[kPlStart] + s.chunk_bytes;
    const uint32_t lim_verbatim = G.outer_hdr + s.top_hdr + s.bytes;
    const uint32_t lim = lim_chunk < lim_verbatim ? lim_chunk : lim_verbatim;
    const uint32_t nf = o >= lim ? 0u : (lim - o < n ? lim - o : n);                  // bytes that go to the frame
    const uint32_t nk = o >= lim_chunk ? 0u : (lim_chunk - o < n ? lim_chunk - o : n);   // ... and up to here to scratch
    const uint8_t *src = reinterpret_cast<const uint8_t *>(out);
    uint8_t *dst = P.out + (uint64_t)frame * P.out_stride + o;
    uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (head > nf) head = nf;
    if (t < head) dst[t] = src[t];
    const uint32_t ng = (nf - head) >> 4, w0 = head >> 2, bs = 8 * (head & 3);
    uint4 *d16 = reinterpret_cast<uint4 *>(dst + head);
    for (uint32_t i = t; i < ng; i += kEncThreads) {
        const uint32_t *w = out + w0 + 4 * i;   // (the buffer has 6 words of slack behind the longest stream)
        d16[i] = make_uint4(__funnelshift_r(w[0], w[1], bs), __funnelshift_r(w[1], w[2], bs), __funnelshift_r(w[2], w[3], bs),
                            __funnelshift_r(w[3], w[4], bs));
    }
    const uint32_t done = head + (ng << 4);
    if (t < nf - done) dst[done + t] = src[done + t];
    for (uint32_t i = nf + t; i < nk; i += kEncThreads) scratch[(uint64_t)gfrag * kFragCap + i] = src[i];
}

// hapq_fused_encode_kernel's arguments, and P.  G must pass fused_hapq_geometry; the frames carry no Chunk Offset Table.
// Follow it with hap_plan_placed_frames_kernel and hap_place_listed_kernel.
__global__ void __launch_bounds__(kEncThreads, 2) hapq_fused_place_kernel(
    const uint8_t *__restrict__ rgba, BcGeom B, uint8_t *__restrict__ tex, FrameGeom G, uint32_t nfrag, uint8_t *__restrict__ scratch,
    uint32_t *__restrict__ frag_size, uint8_t *__restrict__ frag_entries, FusedPlaceArgs P)
{
    HAP_DYN_SMEM(smem_raw);
    const uint32_t t = threadIdx.x;
    HAP_EPHASE_BEGIN();
    if (t == 0) {
        EncodeSmem &S0 = *reinterpret_cast<EncodeSmem *>(smem_raw);
        S0.place[kPlTicket] = atomicAdd(P.ticket, 1u);
        S0.place[kPlPend] = kNoFragment;
    }
    __syncthreads();
    uint32_t gfrag = reinterpret_cast<const EncodeSmem *>(smem_raw)->place[kPlTicket];
    for (;;) {
        if (gfrag < nfrag) fused_fit_fragment(smem_raw, rgba, B, tex, G, gfrag);
        HAP_EPHASE_MARK(kEpFit);
        uint32_t off = 0;   // (as in hapq_fused_encode_kernel)
        asm volatile("" : "+r"(off));
        EncodeSmem &S = *reinterpret_cast<EncodeSmem *>(smem_raw + off);
        const uint32_t pend = S.place[kPlPend];   // the previous fragment, its stream still in S.out
        if (pend != kNoFragment && t < 32) fused_look_back(S, G, P, pend, S.place[kPlPendTotal]);
        HAP_EPHASE_MARK(kEpLookBack);
        __syncthreads();
        HAP_EPHASE_MARK(kEpFitWait);
        if (pend != kNoFragment) fused_store(S, S.out, G, P, scratch, pend, S.place[kPlPendTotal]);
        HAP_EPHASE_MARK(kEpStore);
        if (gfrag >= nfrag) break;
        HAP_EPHASE_COUNT(kEpFragments);
        // (compress_fragment passes barriers before it writes S.out: every thread is done with the store by then)
        const uint32_t total = fused_compress_fragment(S, S.data, S.out, tex, G, gfrag);
        if (frag_entries != nullptr && t < kFragEntryStride) frag_entries[(uint64_t)gfrag * kFragEntryStride + t] = (uint8_t)S.entry[t];
        if (t == 0) {
            frag_size[gfrag] = total;
            hap_st_release(P.size_flag + gfrag, total + 1u);
            S.place[kPlPend] = gfrag;
            S.place[kPlPendTotal] = total;
            S.place[kPlTicket] = atomicAdd(P.ticket, 1u);
        }
        __syncthreads();
        HAP_EPHASE_MARK(kEpOther);
        gfrag = S.place[kPlTicket];
    }
    HAP_EPHASE_END();
}

// ---- the same, with the fit and the compressor in warp groups of their own -----------------------------------------
//
// In hapq_fused_place_kernel every thread fits, then compresses, and the hope that one CTA of an SM fits while the other
// waits at the compressor's barriers mostly does not come true: both run the same loop and drift into the same phase.
// hapq_ws_place_kernel runs one CTA of 1 024 threads per SM, in two warp groups of kEncThreads threads:
//   warps 16-31 (the fit group) fit fragment k+1 into one of two shared-memory images while
//   warps  0-15 (the compressor group, compress_fragment's strip layout unchanged) compress fragment k from the other,
// so the fit's instructions issue while the compressor waits at its barriers, on its shared-memory atomics and on the
// look-back.  The fit and the compressor are those of hapq_fused_place_kernel; the frames are byte-identical.
// Shared memory: EncodeSmem, a second image and a second stream buffer, 169 KiB.
//
// Barriers (named, bar.sync / bar.arrive; 0 is __syncthreads, which this kernel does not use):
//   kWsBarComp      the compressor group's own barrier (compress_fragment's GroupBarrier)
//   kWsBarFit       the fit group's own barrier (the ticket hand-out)
//   kWsBarFull + b  image b holds a fitted fragment: the fit group arrives, the compressor group syncs
//   kWsBarEmpty + b image b may be fitted again: the compressor group arrives, the fit group syncs
// The fit group's i-th fragment goes to image i & 1, with its ticket in WsSmem::frag[i & 1]; a ticket past the last
// fragment ends both groups.  Every arrival is matched by a sync of the other group (a fit group that stops waits for the
// release of the last image it filled), so no barrier is left half-way when the CTA exits.
//
// Tickets and placement as in hapq_fused_place_kernel, with four tickets per CTA at most: the fragment whose stream waits
// for its look-back, the one being compressed, the one being fitted, and the next one, which the fit group takes while it
// fits.  The compressor publishes a fragment's size as soon as it has compressed it, and looks back for it and stores it
// only after it has compressed the CTA's next fragment, into the other of two stream buffers (S.out, WsSmem::out1): the
// fragments before it have had a compression's time to publish their sizes.  (Looking back right after the compression,
// with one stream buffer, left the compressor waiting a quarter of its time, as the phase clocks show.)  Deadlock freedom:
// take the smallest ticket m whose size is not published.  Its fit waits only for the release of an image by the
// compression of an earlier ticket of its CTA, which is published, so done; its compression waits only for its fit and for
// the look-back of its CTA's ticket two back, which waits only for sizes of smaller tickets, all published.  So m's size is
// published after all, whatever share of the device the kernel gets.
constexpr int kWsThreads = 2 * kEncThreads;
enum : int { kWsBarComp = 1, kWsBarFit = 2, kWsBarFull = 3, kWsBarEmpty = 5 };   // kWsBarFull + b, kWsBarEmpty + b: b = 0, 1
struct WsSmem {
    EncodeSmem S;                      // the compressor's shared memory; S.data is image 0
    alignas(16) uint2 data1[kFragUnits + 2];   // image 1
    alignas(16) uint32_t out1[(kFragCap + 3) / 4 + 6];   // stream buffer 1 (0 is S.out)
    uint32_t frag[2];                  // the ticket fitted into image b (fit group -> compressor group)
    uint32_t next[2];                  // the fit group's next ticket (thread 0 of the group -> the group)
};
// One CTA per SM: an H100 SM gives one CTA up to 227 KiB of shared memory.
static_assert(sizeof(WsSmem) <= 232448, "the two images, the two stream buffers and the compressor's tables fit one SM");

// Warps 16-31.  The fit is the same as hapq_fused_place_kernel's (4 blocks per thread of a full fragment); only the
// iteration count and the image's base live across it.
__device__ __forceinline__ void ws_fit_group(WsSmem &W, const uint8_t *__restrict__ rgba, const BcGeom &B, uint8_t *__restrict__ tex,
                                             const FrameGeom &G, uint32_t nfrag, uint32_t *ticket)
{
    const uint32_t ft = threadIdx.x - kEncThreads;
    if (ft == 0) W.next[0] = atomicAdd(ticket, 1u);
#pragma unroll 1
    for (uint32_t i = 0;; i++) {
        const uint32_t b = i & 1;
        if (i >= 2) hap_bar_sync(kWsBarEmpty + b, kWsThreads);   // the compressor is done with the fragment two back
        HAP_EPHASE_MARK(kEpGroupEmptyWait);
        hap_bar_sync(kWsBarFit, kEncThreads);                    // W.next[b] is there
        const uint32_t g = W.next[b];
        if (ft == 0) {
            W.frag[b] = g;
            if (g < nfrag) W.next[b ^ 1] = atomicAdd(ticket, 1u);   // (read behind the next iteration's barrier)
        }
        HAP_EPHASE_MARK(kEpGroupTicket);
        if (g < nfrag) fused_fit_blocks(b ? W.data1 : W.S.data, ft, rgba, B, tex, G, g);
        HAP_EPHASE_MARK(kEpGroupFit);
        hap_bar_arrive(kWsBarFull + b, kWsThreads);
        if (g >= nfrag) {
            if (i >= 1) hap_bar_sync(kWsBarEmpty + (b ^ 1), kWsThreads);   // the release of the last fitted image
            break;
        }
    }
}

// Warps 0-15: compress_fragment on its own named barrier, then the look-back and the store of hapq_fused_place_kernel
// for the fragment compressed before.
__device__ __forceinline__ void ws_compress_group(WsSmem &W, uint8_t *__restrict__ tex, const FrameGeom &G, uint32_t nfrag,
                                                  uint8_t *__restrict__ scratch, uint32_t *__restrict__ frag_size,
                                                  uint8_t *__restrict__ frag_entries, const FusedPlaceArgs &P)
{
    using Bar = GroupBarrier<kWsBarComp>;
    EncodeSmem &S = W.S;
    const uint32_t t = threadIdx.x;
    uint32_t pend = kNoFragment, pend_total = 0;   // the fragment compressed before, its stream in buffer (i - 1) & 1
#pragma unroll 1
    for (uint32_t i = 0;; i++) {
        const uint32_t b = i & 1;
        hap_bar_sync(kWsBarFull + b, kWsThreads);   // (every compressor thread is past the previous store too)
        HAP_EPHASE_MARK(kEpFitWait);
        const uint32_t g = W.frag[b];
        uint32_t total = 0;
        if (g < nfrag) {
            HAP_EPHASE_COUNT(kEpFragments);
            // (the table shares its space with the last step's arrays, and the index entries were copied out before the
            // barrier behind the last look-back; compress_fragment passes barriers before it writes buffer b, whose store
            // was done in the previous iteration)
            init_fragment_tables(S);
            Bar::sync();
            HAP_EPHASE_MARK(kEpOther);
            total = fused_compress_fragment<Bar>(S, b ? W.data1 : S.data, b ? W.out1 : S.out, tex, G, g);
            hap_bar_arrive(kWsBarEmpty + b, kWsThreads);
            if (frag_entries != nullptr && t < kFragEntryStride) frag_entries[(uint64_t)g * kFragEntryStride + t] = (uint8_t)S.entry[t];
            if (t == 0) {
                frag_size[g] = total;
                hap_st_release(P.size_flag + g, total + 1u);
            }
            HAP_EPHASE_MARK(kEpOther);
        }
        if (pend != kNoFragment) {
            if (t < 32) fused_look_back(S, G, P, pend, pend_total);
            Bar::sync();
            HAP_EPHASE_MARK(kEpLookBack);
            fused_store(S, b ? S.out : W.out1, G, P, scratch, pend, pend_total);
            HAP_EPHASE_MARK(kEpStore);
        }
        if (g >= nfrag) break;
        pend = g;
        pend_total = total;
    }
}

// hapq_fused_place_kernel's arguments and contract, kWsThreads threads and sizeof(WsSmem) bytes of shared memory per CTA.
__global__ void __launch_bounds__(kWsThreads, 1) hapq_ws_place_kernel(
    const uint8_t *__restrict__ rgba, BcGeom B, uint8_t *__restrict__ tex, FrameGeom G, uint32_t nfrag, uint8_t *__restrict__ scratch,
    uint32_t *__restrict__ frag_size, uint8_t *__restrict__ frag_entries, FusedPlaceArgs P)
{
    HAP_DYN_SMEM(smem_raw);
    WsSmem &W = *reinterpret_cast<WsSmem *>(smem_raw);
    HAP_EPHASE_BEGIN();
    if (threadIdx.x >= kEncThreads) ws_fit_group(W, rgba, B, tex, G, nfrag, P.ticket);
    else ws_compress_group(W, tex, G, nfrag, scratch, frag_size, frag_entries, P);
    HAP_EPHASE_END();
}

}  // namespace hapb200
