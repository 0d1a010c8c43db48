// tests/emu/test_parse_emu.cc -- TEST INFRASTRUCTURE ONLY.
// hap_api.cu's launch_decode_batch under the fiber SIMT emulator, one frame at a time, in buffers of exactly the frame's and
// the capacity's size: hap_parse_frames_kernel, the chunk pipeline (decode_emu.h), hap_collect_status_kernel.
// usage: test_parse_emu CASES RESULTS.  CASES holds "index capacity frame-hex" lines; RESULTS gets one "result format
// output-hex" line per case (tests/test_batch_decode_golden.py compares them with the reference's answers).
#define HAPB200_EMU
#include "hap_parse.cuh"
#include "decode_emu.h"

#include <fstream>
#include <string>

using namespace hapb200;

int main(int argc, char **argv)
{
    if (argc < 3) { fprintf(stderr, "usage: %s CASES RESULTS\n", argv[0]); return 2; }
    std::ifstream in(argv[1]);
    FILE *out = fopen(argv[2], "w");
    if (!in || !out) { fprintf(stderr, "cannot open %s or %s\n", argv[1], argv[2]); return 2; }
    const uint32_t max_chunks = 64;
    uint32_t index;
    unsigned long long cap;
    std::string hex;
    int cases = 0;
    while (in >> index >> cap >> hex) {
        std::vector<uint8_t> frame(hex.size() / 2), dst(cap);
        for (size_t i = 0; i < frame.size(); i++) frame[i] = (uint8_t)std::stoul(hex.substr(2 * i, 2), nullptr, 16);
        std::vector<ChunkJob> jobs(max_chunks);
        unsigned long long nbytes = frame.size(), used = 0;
        uint32_t fmt = 0, res = 0, whole = 0;
        HAP_LAUNCH(hap_parse_frames_kernel, dim3(1), dim3(128), 0, nullptr, frame.data(), (uint64_t)frame.size(), &nbytes, 1u, index,
                   max_chunks, dst.data(), (uint64_t)cap, (uint64_t)cap, jobs.data(), &used, &fmt, &res, &whole);
        decode_jobs_emu(jobs.data(), max_chunks, frame.size(), cap, 1);
        HAP_LAUNCH(hap_collect_status_kernel, dim3(1), dim3(128), 0, nullptr, jobs.data(), 1u, max_chunks, &whole, &res, &used);
        fprintf(out, "%u %u ", res, fmt);
        for (unsigned long long i = 0; res == HapResult_No_Error && i < used; i++) fprintf(out, "%02x", dst[i]);
        fprintf(out, "\n");
        cases++;
    }
    fclose(out);
    printf("%d frames, %d window-list overflows\n", cases, g_decode_emu_overflow);
    return g_decode_emu_overflow ? 1 : 0;
}
