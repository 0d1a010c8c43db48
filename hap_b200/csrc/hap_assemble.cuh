// hap_b200/csrc/hap_assemble.cuh -- K6: frame assembly on device.
//
// Everything hap_encode_texture / HapEncode (/root/reference/source/hap.c:355-604) decides AFTER
// compression -- chunk sizes, the per-chunk raw fallback (:460-466), the whole-texture fallback
// (:478-487), section lengths, the two tables of the Decode Instructions container (:430-442) and the
// 4/8-byte section headers (:189-212, :497-499, :598) -- is decided here from the fragment sizes K5
// produced, without a host round trip:
//   hap_plan_frames_kernel   one CTA per frame: sizes -> layout, writes headers + tables + varints and
//                            the destination of every fragment;
//   hap_place_fragments_kernel  one CTA per fragment: copies its element stream (or its raw DXT bytes
//                            on a fallback) to the final position.  Chunks end up back to back with no
//                            padding, exactly as hap.c:473 lays them out.
// Behind the fused Hap Q encoder that writes its streams into the frames itself (hapq_fused_place_kernel), the plan
// kernel's twin hap_plan_placed_frames_kernel lists the raw fragments instead, and hap_place_listed_kernel copies them.
#pragma once
#include "block_primitives.cuh"
#include "hap_wire.h"
#include "snappy_encode.cuh"

namespace hapb200 {

constexpr int kPlanThreads = 256;
constexpr uint32_t kPlanWriteIndex = 1, kPlanWriteOffsets = 2;
constexpr uint32_t kPlaceRawFlag = 0x80000000u;

__device__ __forceinline__ uint32_t varint_bytes(uint32_t v) { return v < (1u << 7) ? 1 : v < (1u << 14) ? 2 : v < (1u << 21) ? 3 : v < (1u << 28) ? 4 : 5; }

// Sum of the fragment sizes of one chunk; returns false when any fragment was not compressed.
__device__ __forceinline__ bool chunk_packed_size(const uint32_t *fs, uint32_t fpc, uint32_t chunk_bytes, uint32_t &packed)
{
    uint64_t sum = varint_bytes(chunk_bytes);
    bool ok = true;
    for (uint32_t j = 0; j < fpc; j++) {
        uint32_t s = fs[j];
        if (s == kFragStoredRaw) ok = false;
        sum += s;
    }
    packed = ok && sum < chunk_bytes ? (uint32_t)sum : chunk_bytes;  // hap.c:460: packed >= chunk -> raw
    return ok && sum < chunk_bytes;
}

// bytes of the index record of one chunk (hap_index.h): u16 stream size per fragment + one entry per 128 stream bytes
__device__ __forceinline__ uint32_t chunk_index_record_bytes(const uint32_t *fs, uint32_t fpc)
{
    uint32_t b = 2u * fpc;
    for (uint32_t j = 0; j < fpc; j++) b += (fs[j] + (1u << kIndexSubLog2) - 1u) >> kIndexSubLog2;
    return b;
}

__device__ __forceinline__ void put_le32(uint8_t *p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

// sum over the block of a value that may exceed 16 bits per thread (the 32-bit block scan adds halves separately)
__device__ __forceinline__ uint32_t plan_excl_sum(uint32_t v, uint64_t *total, uint32_t *scratch)
{
    uint32_t tl, th;
    const uint32_t el = block_excl_sum<kPlanThreads>(v & 0xFFFFu, &tl, scratch);
    const uint32_t eh = block_excl_sum<kPlanThreads>(v >> 16, &th, scratch);
    *total = (uint64_t)tl + ((uint64_t)th << 16);
    return el + (eh << 16);
}

// What the fused Hap Q encoder that writes its streams into the frames (hapq_fused.cuh, hapq_fused_place_kernel) leaves
// to the plan kernel: the stream bytes at or past the end a verbatim section would have (they wait in the fragment's
// scratch slot, at their offset in the stream), the fragments' index entries, and a list of the fragments whose raw bytes
// the place kernel must copy (work[0 .. *work_count)).
struct PlanPlaced {
    const uint8_t *scratch;        // [nfrag][kFragCap]
    const uint8_t *frag_entries;   // [nfrag][kFragEntryStride] or nullptr
    uint32_t *work, *work_count;
};

// out: [frames][out_stride]; frag_size / frag_dst / frag_idx_dst: [frames][G.frags_per_frame]; out_used: [frames].
// flags & kPlanWriteIndex: a frame with at least one compressed chunk gets the trailing fragment index section
// (hap_index.h); frag_idx_dst[f] then says where fragment f's entries go (0: nowhere).
// flags & kPlanWriteOffsets: Complex sections carry the optional Chunk Offset Table (HapVideoDRAFT.md:126-128, honoured by
// hap.c:697-700 and :800-803) and every chunk starts on a 16-byte boundary of the frame; the up to 15 bytes between two
// chunks are zero.  The reference's own encoder never writes this table (hap.c:430-442), hence an option.
// PLACED: the compressed fragments are already in the frames (PlanPlaced above; no offset table): compressed fragments get
// no destination, raw ones are listed for the place kernel.
template <bool PLACED>
__device__ __forceinline__ void plan_frames(
    const FrameGeom &G, const uint8_t *__restrict__ dxt, const uint32_t *__restrict__ frag_size,
    uint32_t *__restrict__ frag_dst, uint32_t *__restrict__ frag_idx_dst, uint32_t flags, uint8_t *__restrict__ out,
    uint64_t out_stride, unsigned long long *__restrict__ out_used, const PlanPlaced &pp)
{
    __shared__ uint32_t scratch[kPlanThreads / 32];
    const uint32_t write_index = flags & kPlanWriteIndex, write_offsets = flags & kPlanWriteOffsets;
    const int t = threadIdx.x;
    const uint32_t frame = blockIdx.x;
    uint8_t *fo = out + (uint64_t)frame * out_stride;
    const uint32_t *fs_frame = frag_size + (uint64_t)frame * G.frags_per_frame;
    uint32_t *fd_frame = frag_dst + (uint64_t)frame * G.frags_per_frame;
    uint32_t *fi_frame = frag_idx_dst + (uint64_t)frame * G.frags_per_frame;
    for (uint32_t i = t; i < G.frags_per_frame; i += kPlanThreads) fi_frame[i] = 0;

    // ---- pass 1, every section: would-be complex body length (hap.c:446-476) -> storage decision (hap.c:478), section
    //      lengths, and the size of the chunks' index records --------------------------------------------------------------
    bool complex_storage[2] = {false, false};
    uint64_t body[2] = {0, 0}, rec_total[2] = {0, 0};
    uint32_t sec_off[2] = {0, 0}, sec_len[2] = {0, 0};
    uint32_t running_off = G.outer_hdr;
    for (uint32_t si = 0; si < G.sections; si++) {
        const SectionGeom &sec = G.s[si];
        const uint32_t k = sec.chunks, fpc = sec.frags_per_chunk;
        const uint32_t *fs = fs_frame + sec.frag_base;
        if (sec.want_snappy) {
            const bool indexed = write_index != 0 && sec.compress != 0;
            for (uint32_t c0 = 0; c0 < k; c0 += kPlanThreads) {
                uint32_t c = c0 + t, sz = 0, rec = 0;
                if (c < k && chunk_packed_size(fs + (uint64_t)c * fpc, fpc, sec.chunk_bytes, sz) && indexed)
                    rec = chunk_index_record_bytes(fs + (uint64_t)c * fpc, fpc);
                if (write_offsets && c + 1 < k) sz = (sz + 15u) & ~15u;   // every chunk but the last is padded to the next chunk's aligned start
                uint64_t ts, tr;
                plan_excl_sum(c < k ? sz : 0u, &ts, scratch);
                plan_excl_sum(rec, &tr, scratch);
                body[si] += ts;
                rec_total[si] += tr;
            }
            const uint32_t di1 = 5u * k + 8u + (write_offsets ? 4u * k + 4u : 0u);   // hap.c:265-275 (+ the offset table)
            body[si] += 4u + di1;
            if (write_offsets) body[si] += (16u - ((running_off + sec.top_hdr + 4u + di1) & 15u)) & 15u;   // chunk 0 starts aligned too
            complex_storage[si] = body[si] < (uint64_t)sec.bytes + sec.top_hdr && body[si] < (1ull << 31);  // hap.c:478
        }
        if (!complex_storage[si]) rec_total[si] = 0;
        sec_off[si] = running_off;
        sec_len[si] = complex_storage[si] ? (uint32_t)body[si] : sec.bytes;
        running_off += sec.top_hdr + sec_len[si];
    }
    const uint32_t frame_end = running_off;   // end of the frame proper (hap.c:499 / :598)
    // trailing index section
    const uint32_t k0 = G.s[0].chunks, k1 = G.sections == 2 ? G.s[1].chunks : 0u;
    const uint64_t index_len = rec_total[0] + rec_total[1] > 0 ? (uint64_t)kIndexHeaderBytes + 4ull * (k0 + k1) + rec_total[0] + rec_total[1] : 0;
    const uint32_t index_hdr = index_len == 0 ? 0u : (index_len > kU24Max ? 8u : 4u);
    uint8_t *ibody = fo + frame_end + index_hdr;
    if (index_len && t == 0) {
        put_section_header(fo + frame_end, index_hdr, (uint32_t)index_len, kSecFragmentIndex);
        put_le32(ibody, kIndexMagic);
        ibody[4] = (uint8_t)kIndexVersion; ibody[5] = (uint8_t)kIndexSubLog2; ibody[6] = (uint8_t)G.sections; ibody[7] = 0;
        put_le32(ibody + 8, (uint32_t)kFragBytes);
        put_le32(ibody + 12, k0);
        put_le32(ibody + 16, k1);
    }

    // ---- pass 2, every section: headers, tables, varints, destinations ----------------------------------------------------------
    uint32_t rec_running = kIndexHeaderBytes + 4u * (k0 + k1);   // offset of the next chunk record inside the index body
    for (uint32_t si = 0; si < G.sections; si++) {
        const SectionGeom &sec = G.s[si];
        const uint32_t k = sec.chunks, fpc = sec.frags_per_chunk, hdr = sec.top_hdr;
        const uint32_t di = 5u * k + 8u + (write_offsets ? 4u * k + 4u : 0u);  // hap.c:265-275 (+ the offset table)
        const uint32_t *fs = fs_frame + sec.frag_base;
        uint32_t *fd = fd_frame + sec.frag_base;
        uint32_t *fi = fi_frame + sec.frag_base;
        uint8_t *so = fo + sec_off[si];
        uint8_t *slots = ibody + kIndexHeaderBytes + 4u * (si ? k0 : 0u);   // this texture's record offsets
        const uint32_t verbatim_end = sec_off[si] + hdr + sec.bytes;   // where the section would end stored verbatim (hap.c:490-495)
        if (complex_storage[si]) {
            uint8_t *p = so + hdr;
            uint8_t *ctab = p + 8, *stab = p + 8 + k + 4, *otab = stab + 4u * k + 4;
            if (t == 0) {
                put_section_header(so, hdr, sec_len[si], (kHapComplex << 4) | sec.fmt_nibble);
                put_section_header(p, 4, di, kSecDecodeInstructions);        // hap.c:436
                put_section_header(p + 4, 4, k, kSecCompressorTable);        // hap.c:438
                put_section_header(ctab + k, 4, 4u * k, kSecSizeTable);      // hap.c:440
                if (write_offsets) put_section_header(stab + 4u * k, 4, 4u * k, kSecOffsetTable);   // HapVideoDRAFT.md:126-128
            }
            const uint32_t data0 = sec_off[si] + hdr + 4u + di;   // "frame data": what the offset table counts from (hap.c:672)
            uint32_t running = write_offsets ? (data0 + 15u) & ~15u : data0;  // offset of chunk 0 inside the frame
            if (write_offsets && (uint32_t)t < running - data0) fo[data0 + t] = 0;
            for (uint32_t c0 = 0; c0 < k; c0 += kPlanThreads) {
                uint32_t c = c0 + t, sz = 0, rec = 0;
                bool snappy = false;
                if (c < k) snappy = chunk_packed_size(fs + (uint64_t)c * fpc, fpc, sec.chunk_bytes, sz);
                if (snappy && rec_total[si]) rec = chunk_index_record_bytes(fs + (uint64_t)c * fpc, fpc);
                uint64_t ts, tr;
                const uint32_t szp = c >= k ? 0u : (write_offsets && c + 1 < k ? (sz + 15u) & ~15u : sz);   // with its padding
                const uint32_t start = running + plan_excl_sum(szp, &ts, scratch);
                const uint32_t rec_off = rec_running + plan_excl_sum(rec, &tr, scratch);
                if (c < k) {
                    ctab[c] = snappy ? kHapChunkSnappy : kHapChunkRaw;
                    put_le32(stab + 4 * c, sz);
                    if (write_offsets) {
                        put_le32(otab + 4 * c, start - data0);
                        for (uint32_t z = sz; z < szp; z++) fo[start + z] = 0;   // the gap in front of the next chunk
                    }
                    if (index_len) put_le32(slots + 4 * c, rec ? rec_off : 0u);
                    if (snappy) {
                        uint32_t v = sec.chunk_bytes, o = start;
                        while (v >= 0x80) { fo[o++] = (uint8_t)(v | 0x80); v >>= 7; }
                        fo[o++] = (uint8_t)v;
                        uint32_t eo = rec_off + 2u * fpc;   // entries follow the u16 sizes of the record
                        for (uint32_t j = 0; j < fpc; j++) {
                            const uint32_t s = fs[(uint64_t)c * fpc + j];
                            if (!PLACED) {
                                fd[(uint64_t)c * fpc + j] = o;
                            } else if (o + s > verbatim_end) {
                                // the bytes the fused encoder kept back (fewer than top_hdr: the section is complex)
                                const uint8_t *ks = pp.scratch + ((uint64_t)frame * G.frags_per_frame + sec.frag_base + (uint64_t)c * fpc + j) * kFragCap;
                                for (uint32_t q = o > verbatim_end ? o : verbatim_end; q < o + s; q++) fo[q] = ks[q - o];
                            }
                            o += s;
                            if (rec) {
                                ibody[rec_off + 2 * j] = (uint8_t)s;
                                ibody[rec_off + 2 * j + 1] = (uint8_t)(s >> 8);
                                fi[(uint64_t)c * fpc + j] = frame_end + index_hdr + eo;
                                eo += (s + (1u << kIndexSubLog2) - 1u) >> kIndexSubLog2;
                            }
                        }
                    } else {
                        for (uint32_t j = 0; j < fpc; j++) fd[(uint64_t)c * fpc + j] = (start + j * kFragBytes) | kPlaceRawFlag;
                        if (PLACED) {
                            const uint32_t w = atomicAdd(pp.work_count, fpc);
                            for (uint32_t j = 0; j < fpc; j++) pp.work[w + j] = frame * G.frags_per_frame + sec.frag_base + c * fpc + j;
                        }
                    }
                }
                running += (uint32_t)ts;
                rec_running += (uint32_t)tr;
            }
        } else {
            // hap.c:490-495: the whole texture verbatim
            if (t == 0) put_section_header(so, hdr, sec_len[si], (kHapChunkRaw << 4) | sec.fmt_nibble);
            if (index_len) for (uint32_t c = t; c < k; c += kPlanThreads) put_le32(slots + 4 * c, 0u);
            const uint32_t data0 = sec_off[si] + hdr;
            for (uint64_t i = t; i < (uint64_t)k * fpc; i += kPlanThreads) {
                uint32_t c = (uint32_t)(i / fpc), j = (uint32_t)(i % fpc);
                fd[i] = (data0 + c * sec.chunk_bytes + j * kFragBytes) | kPlaceRawFlag;
            }
            if (PLACED) {
                __shared__ uint32_t work_base;
                if (t == 0) work_base = atomicAdd(pp.work_count, k * fpc);
                __syncthreads();
                for (uint32_t i = t; i < k * fpc; i += kPlanThreads) pp.work[work_base + i] = frame * G.frags_per_frame + sec.frag_base + i;
                __syncthreads();   // (work_base is taken again by the next section)
            }
            // bytes / chunks truncates (hap.c:433); the verbatim path still copies every byte (hap.c:492)
            const uint32_t covered = k * sec.chunk_bytes;
            const uint8_t *in = dxt + (uint64_t)frame * sec.in_stride + sec.in_offset;
            for (uint32_t i = covered + t; i < sec.bytes; i += kPlanThreads) fo[data0 + i] = in[i];
        }
    }
    if (PLACED && index_len) {
        // the compressed fragments' index entries (a warp per fragment; frag_idx_dst was written by other threads)
        __syncthreads();
        const uint32_t lane = t & 31;
        for (uint32_t f = t >> 5; f < G.frags_per_frame; f += kPlanThreads / 32) {
            const uint32_t id = fi_frame[f];
            if (id == 0) continue;
            const uint8_t *e = pp.frag_entries + ((uint64_t)frame * G.frags_per_frame + f) * kFragEntryStride;
            const uint32_t pieces = (fs_frame[f] + (1u << kIndexSubLog2) - 1u) >> kIndexSubLog2;
            for (uint32_t q = lane; q < pieces; q += 32) fo[id + q] = e[q];
        }
    }
    if (t == 0) {
        if (G.sections == 2) put_section_header(fo, G.outer_hdr, frame_end - G.outer_hdr, kSecMultipleImages);  // hap.c:598
        out_used[frame] = frame_end + index_hdr + index_len;
    }
}

__global__ void __launch_bounds__(kPlanThreads) hap_plan_frames_kernel(
    FrameGeom G, const uint8_t *__restrict__ dxt, const uint32_t *__restrict__ frag_size,
    uint32_t *__restrict__ frag_dst, uint32_t *__restrict__ frag_idx_dst, uint32_t flags, uint8_t *__restrict__ out,
    uint64_t out_stride, unsigned long long *__restrict__ out_used)
{
    plan_frames<false>(G, dxt, frag_size, frag_dst, frag_idx_dst, flags, out, out_stride, out_used, PlanPlaced{});
}

// The plan kernel behind hapq_fused_place_kernel (flags without kPlanWriteOffsets).
__global__ void __launch_bounds__(kPlanThreads) hap_plan_placed_frames_kernel(
    FrameGeom G, const uint8_t *__restrict__ dxt, const uint32_t *__restrict__ frag_size,
    uint32_t *__restrict__ frag_dst, uint32_t *__restrict__ frag_idx_dst, uint32_t flags, uint8_t *__restrict__ out,
    uint64_t out_stride, unsigned long long *__restrict__ out_used, PlanPlaced pp)
{
    plan_frames<true>(G, dxt, frag_size, frag_dst, frag_idx_dst, flags, out, out_stride, out_used, pp);
}

constexpr int kPlaceThreads = 256;

// One fragment's bytes to their place in the frame: its element stream from scratch, or its raw bytes on a fallback.
__device__ __forceinline__ void place_fragment(
    uint32_t gfrag, const FrameGeom &G, const uint8_t *__restrict__ dxt, const uint8_t *__restrict__ scratch,
    const uint32_t *__restrict__ frag_size, const uint32_t *__restrict__ frag_dst, const uint32_t *__restrict__ frag_idx_dst,
    const uint8_t *__restrict__ frag_entries, uint8_t *__restrict__ out, uint64_t out_stride)
{
    const int t = threadIdx.x;
    const uint32_t frame = gfrag / G.frags_per_frame;
    const uint32_t f = gfrag % G.frags_per_frame;
    const SectionGeom &sec = (G.sections == 2 && f >= G.s[1].frag_base) ? G.s[1] : G.s[0];
    const uint32_t fl = f - sec.frag_base;
    const uint32_t chunk = fl / sec.frags_per_chunk, j = fl % sec.frags_per_chunk;
    const uint32_t d = frag_dst[gfrag];
    const uint8_t *src;
    uint32_t n;
    if (d & kPlaceRawFlag) {
        src = dxt + (uint64_t)frame * sec.in_stride + sec.in_offset + (uint64_t)chunk * sec.chunk_bytes + (uint64_t)j * kFragBytes;
        const uint32_t left = sec.chunk_bytes - j * kFragBytes;
        n = left < (uint32_t)kFragBytes ? left : (uint32_t)kFragBytes;
    } else {
        src = scratch + (uint64_t)gfrag * kFragCap;
        n = frag_size[gfrag];
    }
    uint8_t *dst = out + (uint64_t)frame * out_stride + (d & ~kPlaceRawFlag);
    // the fragment's entries of the frame's index section (hap_index.h), when the plan gave them a place
    if (frag_entries != nullptr && !(d & kPlaceRawFlag)) {
        const uint32_t id = frag_idx_dst[gfrag];
        const uint32_t pieces = (n + (1u << kIndexSubLog2) - 1u) >> kIndexSubLog2;
        if (id != 0 && (uint32_t)t < pieces) out[(uint64_t)frame * out_stride + id + t] = frag_entries[(uint64_t)gfrag * kFragEntryStride + t];
        if (id != 0 && (uint32_t)t + kPlaceThreads < pieces) out[(uint64_t)frame * out_stride + id + t + kPlaceThreads] = frag_entries[(uint64_t)gfrag * kFragEntryStride + t + kPlaceThreads];
    }
    // destination alignment is arbitrary (headers, tables and earlier chunks are byte-sized): byte-copy to the first 16-byte
    // boundary of the DESTINATION, then whole 16-byte groups, each assembled from the two aligned 16-byte source cells that
    // hold its bytes (two LDG.128, four funnel shifts, one STG.128; the shift is the same for the whole fragment), then a
    // byte tail of at most 31 bytes.
    uint32_t head = (uint32_t)((16 - ((uintptr_t)dst & 15)) & 15);
    if (head > n) head = n;
    if ((uint32_t)t < head) dst[t] = src[t];
    const uint32_t rem = n - head;
    const uint8_t *s2 = src + head;
    uint4 *d16 = reinterpret_cast<uint4 *>(dst + head);
    const uint32_t mis = (uint32_t)((uintptr_t)s2 & 15);
    const uint4 *s16 = reinterpret_cast<const uint4 *>(s2 - mis);   // (s2 - mis >= the buffer's start: buffers are 16-byte aligned)
    uint32_t ng = rem >> 4;
    if (mis != 0) {
        // group i reads cells i and i+1: keep cell i+1 wholly inside the source bytes (a caller's texture buffer may end with them)
        const uint32_t whole = (mis + rem) >> 4;
        const uint32_t lim = whole ? whole - 1 : 0;
        ng = ng < lim ? ng : lim;
    }
    if (mis == 0) {
        for (uint32_t i = t; i < ng; i += kPlaceThreads) d16[i] = s16[i];
    } else {
        const uint32_t ws = mis >> 2, bs = 8 * (mis & 3);
        for (uint32_t i = t; i < ng; i += kPlaceThreads) {
            const uint4 a = s16[i], b = s16[i + 1];    // group i = bytes mis+16i .. mis+16i+15 of the cells: cell i+1 holds at least one of them
            uint32_t w0, w1, w2, w3, w4;
            if (ws == 0) { w0 = a.x; w1 = a.y; w2 = a.z; w3 = a.w; w4 = b.x; }
            else if (ws == 1) { w0 = a.y; w1 = a.z; w2 = a.w; w3 = b.x; w4 = b.y; }
            else if (ws == 2) { w0 = a.z; w1 = a.w; w2 = b.x; w3 = b.y; w4 = b.z; }
            else { w0 = a.w; w1 = b.x; w2 = b.y; w3 = b.z; w4 = b.w; }
            d16[i] = make_uint4(__funnelshift_r(w0, w1, bs), __funnelshift_r(w1, w2, bs), __funnelshift_r(w2, w3, bs), __funnelshift_r(w3, w4, bs));
        }
    }
    const uint32_t done = head + (ng << 4);
    if ((uint32_t)t < n - done) dst[done + t] = src[done + t];
}

// grid.x = frames * frags_per_frame
__global__ void __launch_bounds__(kPlaceThreads) hap_place_fragments_kernel(
    FrameGeom G, const uint8_t *__restrict__ dxt, const uint8_t *__restrict__ scratch,
    const uint32_t *__restrict__ frag_size, const uint32_t *__restrict__ frag_dst, const uint32_t *__restrict__ frag_idx_dst,
    const uint8_t *__restrict__ frag_entries, uint8_t *__restrict__ out, uint64_t out_stride)
{
    place_fragment(blockIdx.x, G, dxt, scratch, frag_size, frag_dst, frag_idx_dst, frag_entries, out, out_stride);
}

// The raw fragments hap_plan_placed_frames_kernel listed (work[0 .. *work_count)), a persistent grid striding over them: on
// content that compresses the list is empty and the launch costs next to nothing.
__global__ void __launch_bounds__(kPlaceThreads) hap_place_listed_kernel(
    FrameGeom G, const uint8_t *__restrict__ dxt, const uint32_t *__restrict__ frag_size, const uint32_t *__restrict__ frag_dst,
    const uint32_t *__restrict__ work, const uint32_t *__restrict__ work_count, uint8_t *__restrict__ out, uint64_t out_stride)
{
    const uint32_t n = *work_count;
    for (uint32_t i = blockIdx.x; i < n; i += gridDim.x)
        place_fragment(work[i], G, dxt, nullptr, frag_size, frag_dst, nullptr, nullptr, out, out_stride);
}

}  // namespace hapb200
