// tests/emu/bc7_encode_twin.cc -- TEST INFRASTRUCTURE ONLY.
// Host build of the BC7 block encoder the Hap R encode kernel compiles (hap_b200/csrc/bc7_encode.cuh), exported as plain C:
// the CPU tests hold its blocks to the oracle's decoding and the quality bars, and the GPU tests hold the device's blocks to
// it byte for byte.  Built by tests/bc7_encode_util.py (HAPB200_BC7_PARTITION_FITS and HAPB200_BC7_PARTITION3_FITS may be set
// for trade-off studies).
#define HAPB200_EMU
#include "bc7_encode.cuh"

using namespace hapb200;

// RGBA8 picture (rows row_bytes apart) -> blocks row-major over (w/4) x (h/4), 16 bytes each, and per block the error it was
// chosen by (errs may be NULL)
extern "C" void bc7_twin_encode(const uint8_t *rgba, int w, int h, long row_bytes, uint8_t *blocks, uint64_t *errs)
{
    for (int by = 0; by < h / 4; by++)
        for (int bx = 0; bx < w / 4; bx++) {
            uint32_t px[16], out[4];
            for (int t = 0; t < 16; t++) memcpy(&px[t], rgba + (size_t)(4 * by + t / 4) * row_bytes + 4 * (4 * bx + t % 4), 4);
            const size_t b = (size_t)by * (w / 4) + bx;
            const uint32_t e = bc7_encode_block(px, out);
            memcpy(blocks + 16 * b, out, 16);
            if (errs) errs[b] = e;
        }
}

// the partitions fully fitted per block: two subsets (kBc7PartitionFits) and three (kBc7Partition3Fits)
extern "C" int bc7_twin_partition_fits(void) { return (int)kBc7PartitionFits; }
extern "C" int bc7_twin_partition3_fits(void) { return (int)kBc7Partition3Fits; }
