// tests/emu/bc6h_encode_twin.cc -- TEST INFRASTRUCTURE ONLY.
// Host build of the BC6H block encoder the Hap HDR encode kernel compiles (hap_b200/csrc/bc6h_encode.cuh), exported as
// plain C: the CPU tests hold its blocks to the oracle's decoding and the quality bars, and the GPU tests hold the device's
// blocks to it byte for byte.  Built by tests/bc6h_encode_util.py (HAPB200_BC6H_PARTITION_FITS may be set for trade-off studies).
#define HAPB200_EMU
#include "bc6h_encode.cuh"

using namespace hapb200;

// RGBA16F picture (4*w halves per row, rows row_halves apart) -> blocks row-major over (w/4) x (h/4), 16 bytes each, and
// per block the error it was chosen by (errs may be NULL)
extern "C" void bc6h_twin_encode(const uint16_t *rgba, int w, int h, long row_halves, int is_signed, uint8_t *blocks, uint64_t *errs)
{
    for (int by = 0; by < h / 4; by++)
        for (int bx = 0; bx < w / 4; bx++) {
            uint32_t px[32], out[4];
            for (int t = 0; t < 16; t++) memcpy(&px[2 * t], rgba + (size_t)(4 * by + t / 4) * row_halves + 4 * (4 * bx + t % 4), 8);
            const size_t b = (size_t)by * (w / 4) + bx;
            const uint64_t e = bc6h_encode_block(px, is_signed != 0, out);
            memcpy(blocks + 16 * b, out, 16);
            if (errs) errs[b] = e;
        }
}

// the partitions fully fitted per block (kBc6hPartitionFits)
extern "C" int bc6h_twin_partition_fits(void) { return (int)kBc6hPartitionFits; }
