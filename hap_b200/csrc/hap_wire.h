// hap_b200/csrc/hap_wire.h -- the Hap section / Decode-Instructions byte layout, shared by the host
// entry points and the device-side frame parser (every function is host+device).
//
// Follows documentation/HapVideoDRAFT.md:36-128 and the behaviour of /root/reference/source/hap.c
// (function-level citations below).  One deliberate tightening (SURVEY.md Q9): chunk source ranges
// are checked against the section, where hap.c:798-807 trusts the tables.
#pragma once
#include "bc_block.cuh"  // HAP_HD
#include "hap_codes.h"
#include "hap_index.h"

namespace hapb200 {

HAP_HD uint32_t rd_le24(const uint8_t *p) { return p[0] | (p[1] << 8) | ((uint32_t)p[2] << 16); }
HAP_HD uint32_t rd_le32(const uint8_t *p) { return rd_le24(p) | ((uint32_t)p[3] << 24); }

struct Section {
    uint32_t hdr, len, type;
};

// The header walks below call need(p, len) before they read [p, p+len) of a frame; false means the bytes could not be
// fetched (the walk then fails with Internal_Error).  Frames the caller can read directly use NoFetch; the host entry
// points reading a device frame pass a reader that copies the bytes over on demand (hap_api.cu HeaderView).
struct NoFetch {
    HAP_HD bool need(const uint8_t *, uint64_t) const { return true; }
};
// Precedes the templates that call their reader (or a sink, hap_parse.cuh): instantiated for the host, they may call
// host-only code.
#if defined(__CUDACC__) && !defined(HAPB200_EMU)
#define HAP_HD_TEMPLATE _Pragma("nv_exec_check_disable")
#else
#define HAP_HD_TEMPLATE
#endif

// hap.c:189-212: a 4- or 8-byte section header at p
HAP_HD void put_section_header(uint8_t *p, uint32_t hdr, uint32_t len, uint32_t type)
{
    if (hdr == 4) {
        p[0] = (uint8_t)len; p[1] = (uint8_t)(len >> 8); p[2] = (uint8_t)(len >> 16);
    } else {
        p[0] = p[1] = p[2] = 0;
        p[4] = (uint8_t)len; p[5] = (uint8_t)(len >> 8); p[6] = (uint8_t)(len >> 16); p[7] = (uint8_t)(len >> 24);
    }
    p[3] = (uint8_t)type;
}

// hap.c:137-187.  The reference does this arithmetic in 32 bits (hap.c:181); `avail` is truncated
// the same way by the callers (hap.c:1022 -> :932).
HAP_HD uint32_t read_section_header(const uint8_t *p, uint32_t avail, Section &s)
{
    if (avail < 4) return HapResult_Bad_Frame;
    s.len = rd_le24(p);
    s.hdr = 4;
    if (s.len == 0) {
        if (avail < 8) return HapResult_Bad_Frame;
        s.len = rd_le32(p + 4);
        s.hdr = 8;
    }
    s.type = p[3];
    if ((uint32_t)(s.hdr + s.len) > avail) return HapResult_Bad_Frame;
    // tightening: hdr+len wrapping past 2^32 must not pass the test above
    if ((uint64_t)s.hdr + s.len > avail) return HapResult_Bad_Frame;
    return HapResult_No_Error;
}

// hap.c:215-261
HAP_HD uint32_t format_from_nibble(uint32_t nib)
{
    switch (nib) {
    case 0xB: return HapFmt_RGB_DXT1;
    case 0xE: return HapFmt_RGBA_DXT5;
    case 0xF: return HapFmt_YCoCg_DXT5;
    case 0x1: return HapFmt_A_RGTC1;
    case 0xC: return HapFmt_RGBA_BPTC_UNORM;
    case 0x2: return HapFmt_RGB_BPTC_UFLOAT;
    case 0x3: return HapFmt_RGB_BPTC_SFLOAT;
    default: return 0;
    }
}
HAP_HD uint32_t nibble_from_format(uint32_t fmt)
{
    switch (fmt) {
    case HapFmt_RGB_DXT1: return 0xB;
    case HapFmt_RGBA_DXT5: return 0xE;
    case HapFmt_YCoCg_DXT5: return 0xF;
    case HapFmt_A_RGTC1: return 0x1;
    case HapFmt_RGBA_BPTC_UNORM: return 0xC;
    case HapFmt_RGB_BPTC_UFLOAT: return 0x2;
    case HapFmt_RGB_BPTC_SFLOAT: return 0x3;
    default: return 0;
    }
}

// hap.c:932-991: the texture section at `index` (offset relative to the frame start)
struct Located {
    uint32_t offset, len, type;
};
HAP_HD_TEMPLATE
template <class Reader = NoFetch>
HAP_HD uint32_t locate_texture(const uint8_t *in, uint32_t n, uint32_t index, Located &out, Reader &&rd = Reader())
{
    Section top;
    if (!rd.need(in, 8)) return HapResult_Internal_Error;
    uint32_t r = read_section_header(in, n, top);
    if (r != HapResult_No_Error) return r;
    if (top.type == kSecMultipleImages) {
        uint64_t off = 0;
        Section cur;
        cur.hdr = 0; cur.len = 0; cur.type = 0;
        for (uint32_t i = 0; i <= index; i++) {
            off += (uint64_t)cur.hdr + cur.len;
            if (off >= top.len) return HapResult_Bad_Arguments;
            if (!rd.need(in + top.hdr + off, 8)) return HapResult_Internal_Error;
            r = read_section_header(in + top.hdr + off, (uint32_t)(top.len - off), cur);
            if (r != HapResult_No_Error) return r;
        }
        out.offset = (uint32_t)(top.hdr + off + cur.hdr);
        out.len = cur.len;
        out.type = cur.type;
        return HapResult_No_Error;
    }
    if (index == 0) {
        out.offset = top.hdr;
        out.len = top.len;
        out.type = top.type;
        return HapResult_No_Error;
    }
    return HapResult_Bad_Arguments;
}

// hap.c:644-730: tables of a Complex texture section; offsets relative to the section start
struct ChunkTables {
    uint32_t compressors, sizes, offsets;  // offsets == 0xFFFFFFFF when absent
    uint32_t data;                         // first byte of frame data
    int count;
    bool has_compressors, has_sizes;
};
HAP_HD_TEMPLATE
template <class Reader = NoFetch>
HAP_HD uint32_t parse_decode_instructions(const uint8_t *sec, uint32_t sec_len, ChunkTables &t, Reader &&rd = Reader())
{
    // t.count is an in/out accumulator exactly like the reference's int *chunk_count
    t.has_compressors = t.has_sizes = false;
    t.offsets = 0xFFFFFFFFu;
    Section s;
    if (!rd.need(sec, 8)) return HapResult_Internal_Error;
    uint32_t r = read_section_header(sec, sec_len, s);
    if (r == HapResult_No_Error && s.type != kSecDecodeInstructions) r = HapResult_Bad_Frame;
    if (r != HapResult_No_Error) return r;
    if (!rd.need(sec, (uint64_t)s.hdr + s.len)) return HapResult_Internal_Error;   // the whole container: tables included
    t.data = s.hdr + s.len;
    uint32_t pos = s.hdr, left = s.len;
    // byte lengths of the tables as found (0xFFFFFFFF = table absent): the entry counts derived from them must all
    // describe `count` chunks EXACTLY.  hap.c:709-716 only compares counts that are non-zero, so a compressor table of
    // length 0 or a size table shorter than 4 bytes would leave `count` to the other table and the per-chunk reads
    // (hap.c:794-807) would run past the short table; that inherited hole is closed here (-> Bad_Frame).
    uint32_t comp_len = 0xFFFFFFFFu, size_len = 0xFFFFFFFFu, offs_len = 0xFFFFFFFFu;
    while (left > 0) {
        Section in;
        r = read_section_header(sec + pos, left, in);
        if (r != HapResult_No_Error) return r;
        pos += in.hdr;
        uint32_t c = 0;
        if (in.type == kSecCompressorTable) { t.compressors = pos; t.has_compressors = true; c = in.len; comp_len = in.len; }
        else if (in.type == kSecSizeTable) { t.sizes = pos; t.has_sizes = true; c = in.len / 4; size_len = in.len; }
        else if (in.type == kSecOffsetTable) { t.offsets = pos; c = in.len / 4; offs_len = in.len; }
        // any other type: ignored, like hap.c:701-704
        if (c != 0) {
            if (t.count != 0 && (int)c != t.count) return HapResult_Bad_Frame;
            t.count = (int)c;
        }
        pos += in.len;
        left -= in.hdr + in.len;
    }
    if (!t.has_compressors || !t.has_sizes) return HapResult_Bad_Frame;
    if (t.count < 0) return HapResult_Bad_Frame;
    const uint64_t k = (uint64_t)t.count;
    if (comp_len != k || size_len / 4 != k) return HapResult_Bad_Frame;
    if (offs_len != 0xFFFFFFFFu && offs_len / 4 != k) return HapResult_Bad_Frame;
    return HapResult_No_Error;
}

// The body of the trailing fragment index section of a frame (hap_index.h): offset from the frame start and length;
// false when the frame has none (or it is not one this decoder understands).
struct FragmentIndex {
    uint32_t body, len;
    uint32_t chunks[2];
};
HAP_HD_TEMPLATE
template <class Reader = NoFetch>
HAP_HD bool locate_fragment_index(const uint8_t *frame, uint32_t n, FragmentIndex &ix, Reader &&rd = Reader())
{
    Section top;
    if (!rd.need(frame, 8) || read_section_header(frame, n, top) != HapResult_No_Error) return false;
    const uint64_t end = (uint64_t)top.hdr + top.len;
    if (end + 4 > n || !rd.need(frame + end, 8 + kIndexHeaderBytes)) return false;
    Section s;
    if (read_section_header(frame + end, (uint32_t)(n - end), s) != HapResult_No_Error || s.type != kSecFragmentIndex) return false;
    if (s.len < kIndexHeaderBytes) return false;
    const uint8_t *b = frame + end + s.hdr;
    if (rd_le32(b) != kIndexMagic || b[4] != kIndexVersion || b[5] != kIndexSubLog2 || rd_le32(b + 8) != 32768u) return false;
    ix.body = (uint32_t)(end + s.hdr);
    ix.len = s.len;
    ix.chunks[0] = rd_le32(b + 12);
    ix.chunks[1] = rd_le32(b + 16);
    const uint64_t table = (uint64_t)kIndexHeaderBytes + 4ull * ((uint64_t)ix.chunks[0] + ix.chunks[1]);
    return table <= s.len && rd.need(b, table);     // fragment_index_record reads the record-offset table
}
// The record of chunk `i` of texture `texture` (which has `count` chunks by its own tables): offset from the frame start
// and the bytes readable from there; false when there is no record for it.
HAP_HD bool fragment_index_record(const uint8_t *frame, const FragmentIndex &ix, uint32_t texture, uint32_t count, uint32_t i, uint32_t &off,
                                  uint32_t &bytes)
{
    if (texture > 1 || ix.chunks[texture] != count || i >= count) return false;
    const uint32_t slot = (texture ? ix.chunks[0] : 0u) + i;
    const uint32_t o = rd_le32(frame + ix.body + kIndexHeaderBytes + 4 * slot);
    if (o < kIndexHeaderBytes + 4u * (ix.chunks[0] + ix.chunks[1]) || o >= ix.len) return false;
    off = ix.body + o;
    bytes = ix.len - o;
    return true;
}

// varint32 preamble of a raw Snappy stream (snappy_uncompressed_length, hap.c:813, :890)
HAP_HD bool snappy_preamble(const uint8_t *p, uint32_t n, uint32_t &value)
{
    uint64_t v = 0;
    for (uint32_t i = 0; i < 5 && i < n; i++) {
        uint32_t b = p[i];
        v |= (uint64_t)(b & 0x7F) << (7 * i);
        if (!(b & 0x80)) {
            if (v > 0xFFFFFFFFull) return false;
            value = (uint32_t)v;
            return true;
        }
    }
    return false;
}

// hap.c:277-300
HAP_HD uint32_t limited_chunk_count(uint64_t bytes, uint32_t fmt, uint32_t k)
{
    if (k > kMaxChunkCount) k = kMaxChunkCount;
    uint64_t blocks = (fmt == HapFmt_RGB_DXT1 || fmt == HapFmt_A_RGTC1) ? bytes / 8 : bytes / 16;
    while (blocks % k != 0) k--;
    return k;
}

HAP_HD uint64_t snappy_max_compressed(uint64_t n) { return 32 + n + n / 6; }   // snappy_max_compressed_length
HAP_HD uint64_t decode_instructions_length(uint32_t k) { return 5ull * k + 8; }  // hap.c:265-275

// hap.c:302-322
HAP_HD uint64_t max_encoded_length_one(uint64_t bytes, uint32_t fmt, uint32_t compressor, uint32_t k)
{
    k = limited_chunk_count(bytes, fmt, k);
    uint64_t payload = compressor == HapCompressorSnappy ? snappy_max_compressed(bytes / k) * k : bytes;
    return payload + 8 + decode_instructions_length(k) + 4;
}

}  // namespace hapb200
