// hap_b200/csrc/hap_parse.cuh -- the decode prepass: one texture of one frame -> its chunk jobs.
//
// hap_decode_single_texture's serial prepass (/root/reference/source/hap.c:748-843: section type ->
// compressor/format, Decode-Instructions tables -> one HapChunkDecodeInfo per chunk, the running
// source/destination offsets and the output-size check), written once for both decode paths:
// HapDecode runs it on the host, and hap_parse_frames_kernel runs it with one thread per frame, so a
// batch of device-resident frames is decoded without the host ever reading a header.
#pragma once
#include "hap_wire.h"
#include "snappy_decode.cuh"

namespace hapb200 {

constexpr uint32_t kHapChunkSkip = 0;  // ChunkJob.compressor of an unused slot

// One chunk job, in offsets from the frame start (source, fragment index record) or from the texture's output (dst_off).
struct PlannedJob {
    uint32_t src_off, src_bytes;
    uint64_t dst_off;
    uint32_t dst_bytes;
    uint32_t compressor;                // 0x0A, 0x0B, or 0xFF for any other: the decode kernels report Bad_Frame for it
    uint32_t index_off, index_bytes;    // the chunk's record in the frame's fragment index; index_bytes == 0 when none
};

struct TexturePlan {
    bool located = false;   // the texture section was found: loc and format are set
    Located loc;
    uint32_t format = 0;
    bool whole = false;     // the texture is one 0xB? stream: its errors map to Internal_Error (hap.c:891-903)
    uint64_t produced = 0;  // bytes the jobs decode
    FragmentIndex ix;       // the frame's fragment index, when a job has a record in it
};

// Texture `index` of the frame [frame, frame+n): hands one PlannedJob per chunk to emit() and returns the HapResult of the
// prepass.  At most max_jobs jobs (more -> Bad_Arguments); a chunk's output may start at most max_dst_off bytes into the
// texture (further -> Buffer_Too_Small); all of them may decode at most `capacity` bytes.  On an error, jobs emitted
// before it are void.  Every byte the walk reads is asked of rd.need() first.
HAP_HD_TEMPLATE
template <class Reader, class Sink>
HAP_HD uint32_t plan_texture(const uint8_t *frame, uint32_t n, uint32_t index, uint64_t capacity, uint32_t max_jobs, uint64_t max_dst_off,
                             Reader &&rd, TexturePlan &p, Sink &&emit)
{
    uint32_t r = locate_texture(frame, n, index, p.loc, rd);
    if (r != HapResult_No_Error) return r;
    const Located &loc = p.loc;
    const uint8_t *sec = frame + loc.offset;
    const uint32_t compressor = (loc.type >> 4) & 0xF;
    p.located = true;
    p.format = format_from_nibble(loc.type & 0xF);
    if (p.format == 0) return HapResult_Bad_Frame;
    if (compressor == kHapComplex) {
        ChunkTables t;
        t.count = 0;
        r = parse_decode_instructions(sec, loc.len, t, rd);
        if (r != HapResult_No_Error) return r;
        const bool have_ix = locate_fragment_index(frame, n, p.ix, rd);
        if (t.count == 0) return HapResult_No_Error;
        if ((uint32_t)t.count > max_jobs) return HapResult_Bad_Arguments;
        uint64_t in_run = 0, out_run = 0;
        for (int i = 0; i < t.count; i++) {
            const uint32_t cc = sec[t.compressors + i];
            const uint32_t sz = rd_le32(sec + t.sizes + 4 * i);
            const uint64_t start = t.data + (t.offsets != 0xFFFFFFFFu ? (uint64_t)rd_le32(sec + t.offsets + 4 * i) : in_run);
            in_run += sz;
            if (start + sz > loc.len) return HapResult_Bad_Frame;  // SURVEY.md Q9: the reference reads out of bounds here
            uint32_t usz = sz;
            if (cc == kHapChunkSnappy) {
                if (!rd.need(sec + start, 5)) return HapResult_Internal_Error;
                if (!snappy_preamble(sec + start, sz, usz)) return HapResult_Bad_Frame;  // hap.c:817-829
            }
            if (out_run > max_dst_off) return HapResult_Buffer_Too_Small;
            PlannedJob j = {loc.offset + (uint32_t)start, sz, out_run, usz, (cc == kHapChunkSnappy || cc == kHapChunkRaw) ? cc : 0xFFu, 0, 0};
            if (cc == kHapChunkSnappy && have_ix) fragment_index_record(frame, p.ix, index, (uint32_t)t.count, (uint32_t)i, j.index_off, j.index_bytes);
            emit(j);
            out_run += usz;
        }
        if (out_run > capacity) return HapResult_Buffer_Too_Small;  // hap.c:840-843
        p.produced = out_run;
        return HapResult_No_Error;
    }
    if (compressor == kHapChunkSnappy) {
        uint32_t usz = 0;
        p.whole = true;
        if (!rd.need(sec, 5) || !snappy_preamble(sec, loc.len, usz)) return HapResult_Internal_Error;  // hap.c:890-894
        if (usz > capacity) return HapResult_Buffer_Too_Small;
        emit(PlannedJob{loc.offset, loc.len, 0, usz, kHapChunkSnappy, 0, 0});
        p.produced = usz;
        return HapResult_No_Error;
    }
    if (compressor == kHapChunkRaw) {
        if (loc.len > capacity) return HapResult_Buffer_Too_Small;
        emit(PlannedJob{loc.offset, loc.len, 0, loc.len, kHapChunkRaw, 0, 0});
        p.produced = loc.len;
        return HapResult_No_Error;
    }
    return HapResult_Bad_Frame;
}

// frame f: in + f*in_stride, in_bytes[f] bytes.  jobs: [frames][max_chunks].
// Frame f's texture goes to out + f*out_stride and may use out_capacity bytes there (the slot of a batch is often
// wider than what one texture may fill: two textures of a Hap Q Alpha frame share a slot).
// results[f] = HapResult of the prepass; whole_section[f] = TexturePlan::whole.
__global__ void hap_parse_frames_kernel(const uint8_t *__restrict__ in, uint64_t in_stride,
                                        const unsigned long long *__restrict__ in_bytes, uint32_t frames,
                                        uint32_t index, uint32_t max_chunks, uint8_t *__restrict__ out,
                                        uint64_t out_stride, uint64_t out_capacity, ChunkJob *__restrict__ jobs,
                                        unsigned long long *__restrict__ used, uint32_t *__restrict__ formats,
                                        uint32_t *__restrict__ results, uint32_t *__restrict__ whole_section)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= frames) return;
    const uint8_t *frame = in + (uint64_t)f * in_stride;
    uint8_t *dst = out + (uint64_t)f * out_stride;
    ChunkJob *fj = jobs + (uint64_t)f * max_chunks;
    for (uint32_t c = 0; c < max_chunks; c++) fj[c].compressor = kHapChunkSkip;
    uint32_t emitted = 0;
    TexturePlan p;
    const uint32_t r = index > 1 ? (uint32_t)HapResult_Bad_Arguments
                                 : plan_texture(frame, (uint32_t)in_bytes[f], index, out_capacity, max_chunks, ~0ull, NoFetch(), p, [&](const PlannedJob &j) {
                                       ChunkJob &c = fj[emitted++];
                                       c.src = frame + j.src_off; c.src_bytes = j.src_bytes;
                                       c.dst = dst + j.dst_off; c.dst_bytes = j.dst_bytes;
                                       c.compressor = j.compressor;
                                       c.index = j.index_bytes ? frame + j.index_off : nullptr; c.index_bytes = j.index_bytes;
                                   });
    if (r != HapResult_No_Error)
        for (uint32_t c = 0; c < emitted; c++) fj[c].compressor = kHapChunkSkip;
    results[f] = r;
    formats[f] = p.format;
    used[f] = r == HapResult_No_Error ? p.produced : 0;
    whole_section[f] = p.whole;
}

// hap.c:867-875: the first chunk error wins
__global__ void hap_collect_status_kernel(const ChunkJob *__restrict__ jobs, uint32_t frames, uint32_t max_chunks,
                                          const uint32_t *__restrict__ whole_section, uint32_t *__restrict__ results,
                                          unsigned long long *__restrict__ used)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= frames) return;
    if (results[f] != HapResult_No_Error) return;
    const ChunkJob *fj = jobs + (uint64_t)f * max_chunks;
    for (uint32_t c = 0; c < max_chunks; c++) {
        if (fj[c].compressor != kHapChunkSkip && fj[c].status != HapResult_No_Error) {
            results[f] = whole_section[f] ? (uint32_t)HapResult_Internal_Error : fj[c].status;
            used[f] = 0;
            return;
        }
    }
}

// RGBA decode path: a texture must have the format and size the caller's codec implies; the first
// failing texture of a frame decides that frame's result (merged into `merged`, which may alias `res`).
__global__ void hap_check_texture_kernel(uint32_t frames, const unsigned long long *__restrict__ used,
                                         const uint32_t *__restrict__ formats, const uint32_t *res,
                                         unsigned long long want_bytes, uint32_t want_format, uint32_t *merged)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= frames) return;
    uint32_t r = res[f];
    if (r == HapResult_No_Error && (formats[f] != want_format || used[f] != want_bytes)) r = HapResult_Bad_Frame;
    if (res == merged) merged[f] = r;
    else if (merged[f] == HapResult_No_Error) merged[f] = r;
}

// RGBA16F decode path (Hap HDR): texture 0 of every frame was decoded into room of exactly want_bytes.  A frame must be
// one BC6H texture of that size: a texture larger than the room (the prepass's Buffer_Too_Small: capacity is the only
// limit the batch prepass sets), of another size or format, or a frame that has a texture 1 reports Bad_Frame.  Other
// failures keep their code.
__global__ void hap_check_bc6h_frames_kernel(const uint8_t *__restrict__ in, uint64_t in_stride,
                                             const unsigned long long *__restrict__ in_bytes, uint32_t frames,
                                             const unsigned long long *__restrict__ used, const uint32_t *__restrict__ formats,
                                             unsigned long long want_bytes, uint32_t *results)
{
    const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= frames) return;
    uint32_t r = results[f];
    if (r == HapResult_Buffer_Too_Small) {
        r = HapResult_Bad_Frame;
    } else if (r == HapResult_No_Error) {
        Located second;
        const bool bc6h = formats[f] == HapFmt_RGB_BPTC_UFLOAT || formats[f] == HapFmt_RGB_BPTC_SFLOAT;
        if (!bc6h || used[f] != want_bytes || locate_texture(in + (uint64_t)f * in_stride, (uint32_t)in_bytes[f], 1, second) == HapResult_No_Error)
            r = HapResult_Bad_Frame;
    }
    results[f] = r;
}

}  // namespace hapb200
