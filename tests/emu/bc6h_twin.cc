// tests/emu/bc6h_twin.cc -- TEST INFRASTRUCTURE ONLY.
// Host build of the BC6H block decoder the Hap HDR kernel compiles (hap_b200/csrc/bc6h_decode.cuh), exported as plain C:
// the CPU tests hold it bit for bit to the oracle (tests/bc6h_oracle.c) and read back the partition and anchor tables it
// uses.  Built by tests/bc6h_util.py.
#define HAPB200_EMU
#include "bc6h_decode.cuh"

using namespace hapb200;

// blocks (row-major over (w/4) x (h/4), 16 bytes each) -> RGBA16F, 4*w halves per row
extern "C" void bc6h_twin_decode(const uint8_t *blocks, int w, int h, int is_signed, uint16_t *rgba)
{
    for (int by = 0; by < h / 4; by++)
        for (int bx = 0; bx < w / 4; bx++) {
            uint32_t v[4], px[32];
            memcpy(v, blocks + 16 * ((size_t)by * (w / 4) + bx), 16);
            bc6h_decode_block(v[0], v[1], v[2], v[3], is_signed != 0, px);
            for (int t = 0; t < 16; t++) memcpy(rgba + 4 * ((size_t)(4 * by + t / 4) * w + 4 * bx + t % 4), &px[2 * t], 8);
        }
}

// the partition maps (2 bits per texel) and anchor masks of partitions 0-31 as the decoder reads them
extern "C" void bc6h_twin_tables(uint32_t *partitions, uint32_t *anchors)
{
    for (uint32_t i = 0; i < 32; i++) {
        partitions[i] = bc7_partition(i);
        anchors[i] = bc7_anchors(i);
    }
}
