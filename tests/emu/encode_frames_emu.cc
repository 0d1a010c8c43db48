// tests/emu/encode_frames_emu.cc -- TEST INFRASTRUCTURE ONLY.
// Encodes frames with the library's encode path (K5 fragment compressor, K6 plan + place) under the fiber SIMT emulator, for
// tests/test_snappy_encode_model_cpu.py, which compares them with the numpy model of the compressor (tests/snappy_encode_model.py).
//
//   encode_frames_emu <cases in> <frames out> <resume order mode> <K5 grid>
//
// Cases in, one after the other until the end of the file (little endian):
//   u32 options (bit 0: fragment index section, bit 1: chunk offset table), u32 textures (1 or 2), then per texture
//   u32 format, u32 compressor, u32 requested chunks, u32 bytes, the texture's bytes.
// Frames out: u32 bytes and the frame, one per case in order.
#define HAPB200_EMU
#include "hap_assemble.cuh"
#include "hap_host.h"

#include <string>

using namespace hapb200;

struct Tex { std::vector<uint8_t> data; uint32_t fmt, compressor, chunks; };

static std::vector<uint8_t> encode(const std::vector<Tex> &tex, uint32_t options, int mode, unsigned grid)
{
    TextureArgs ta[2];
    for (size_t i = 0; i < tex.size(); i++) ta[i] = TextureArgs{tex[i].data.size(), tex[i].fmt, tex[i].compressor, tex[i].chunks};
    FrameGeom G;
    if (build_frame_geom((uint32_t)tex.size(), ta, G) != 0) { fprintf(stderr, "frame geometry refused\n"); exit(2); }
    // one input buffer holding both textures at 16-byte aligned offsets, exact size, no slack (as test_encode_emu.cc)
    const size_t off1 = (tex[0].data.size() + 15) & ~(size_t)15;
    std::vector<uint8_t> in(off1 + (tex.size() > 1 ? tex[1].data.size() : 0));
    memcpy(in.data(), tex[0].data.data(), tex[0].data.size());
    if (tex.size() > 1) { memcpy(in.data() + off1, tex[1].data.data(), tex[1].data.size()); G.s[1].in_offset = off1; }
    // room for the frame (HapMaxEncodedLength of every texture and the outer header) and the trailing index section
    uint64_t cap = 8 + 64;
    for (size_t i = 0; i < tex.size(); i++) {
        cap += max_encoded_length_one(tex[i].data.size(), tex[i].fmt, tex[i].compressor, tex[i].chunks) + 16 * (uint64_t)G.s[i].chunks;
        cap += 4ull * G.s[i].chunks + (uint64_t)G.s[i].chunks * G.s[i].frags_per_chunk * (2 + kFragEntryStride);
    }
    std::vector<uint8_t> scratch((size_t)G.frags_per_frame * kFragCap), out(cap, 0xEE);
    std::vector<uint32_t> fsize(G.frags_per_frame), fdst(G.frags_per_frame), fidx(G.frags_per_frame);
    std::vector<uint8_t> fent((size_t)G.frags_per_frame * kFragEntryStride, 0xDD);
    uint8_t *ent = (options & 1) ? fent.data() : nullptr;
    unsigned long long used = 0;
    emu::g_order_mode() = mode;
    const unsigned k5_grid = G.frags_per_frame < grid ? G.frags_per_frame : grid;
    HAP_LAUNCH(snappy_encode_fragments_kernel, dim3(k5_grid), dim3(kEncThreads), sizeof(EncodeSmem), nullptr,
               in.data(), G, (uint32_t)G.frags_per_frame, scratch.data(), fsize.data(), ent);
    HAP_LAUNCH(hap_plan_frames_kernel, dim3(1), dim3(kPlanThreads), 0, nullptr, G, in.data(), fsize.data(), fdst.data(), fidx.data(),
               options, out.data(), (uint64_t)cap, &used);
    HAP_LAUNCH(hap_place_fragments_kernel, dim3(G.frags_per_frame), dim3(kPlaceThreads), 0, nullptr, G, in.data(),
               scratch.data(), fsize.data(), fdst.data(), fidx.data(), (const uint8_t *)ent, out.data(), (uint64_t)cap);
    if (used > cap) { fprintf(stderr, "used %llu > cap %llu\n", used, (unsigned long long)cap); exit(2); }
    out.resize(used);
    return out;
}

static bool rd32(FILE *f, uint32_t &v) { uint8_t b[4]; if (fread(b, 1, 4, f) != 4) return false; v = rd_le32(b); return true; }

int main(int argc, char **argv)
{
    if (argc != 5) { fprintf(stderr, "usage: %s <cases in> <frames out> <mode> <grid>\n", argv[0]); return 2; }
    FILE *fi = fopen(argv[1], "rb"), *fo = fopen(argv[2], "wb");
    if (!fi || !fo) { perror("open"); return 2; }
    const int mode = atoi(argv[3]);
    const unsigned grid = (unsigned)atoi(argv[4]);
    uint32_t options, count, n = 0;
    while (rd32(fi, options)) {
        if (!rd32(fi, count) || count < 1 || count > 2) { fprintf(stderr, "bad case %u\n", n); return 2; }
        std::vector<Tex> tex(count);
        for (auto &t : tex) {
            uint32_t bytes;
            if (!rd32(fi, t.fmt) || !rd32(fi, t.compressor) || !rd32(fi, t.chunks) || !rd32(fi, bytes)) { fprintf(stderr, "bad case %u\n", n); return 2; }
            t.data.resize(bytes);
            if (fread(t.data.data(), 1, bytes, fi) != bytes) { fprintf(stderr, "short case %u\n", n); return 2; }
        }
        const std::vector<uint8_t> frame = encode(tex, options, mode, grid);
        uint8_t len[4] = {(uint8_t)frame.size(), (uint8_t)(frame.size() >> 8), (uint8_t)(frame.size() >> 16), (uint8_t)(frame.size() >> 24)};
        fwrite(len, 1, 4, fo);
        fwrite(frame.data(), 1, frame.size(), fo);
        n++;
    }
    fclose(fo);
    fclose(fi);
    printf("%u frames\n", n);
    return 0;
}
