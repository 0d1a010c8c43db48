// tests/emu/bc7_twin.cc -- TEST INFRASTRUCTURE ONLY.
// Host build of the BC7 block decoder the Hap R kernel compiles (hap_b200/csrc/bc7_decode.cuh, through bc_decode.cuh's
// decode_block), exported as plain C: the CPU tests hold it byte for byte to the oracle (tests/bc7_oracle.c) and read
// back its partition and anchor tables.  Built by tests/bc7_util.py.
#define HAPB200_EMU
#include "bc_decode.cuh"

using namespace hapb200;

// blocks (row-major over (w/4) x (h/4), 16 bytes each) -> RGBA8, stride 4*w
extern "C" void bc7_twin_decode(const uint8_t *blocks, int w, int h, uint8_t *rgba)
{
    for (int by = 0; by < h / 4; by++)
        for (int bx = 0; bx < w / 4; bx++) {
            uint32_t v[4], px[16];
            memcpy(v, blocks + 16 * ((size_t)by * (w / 4) + bx), 16);
            decode_block(kBcBc7, v[0], v[1], v[2], v[3], px);
            for (int t = 0; t < 16; t++) memcpy(rgba + 4 * ((size_t)(4 * by + t / 4) * w + 4 * bx + t % 4), &px[t], 4);
        }
}

// the 128 partition maps (2 bits per texel) and 128 anchor masks the decoder compiles
extern "C" void bc7_twin_tables(uint32_t *partitions, uint32_t *anchors)
{
    for (uint32_t i = 0; i < 128; i++) {
        partitions[i] = bc7_partition(i);
        anchors[i] = bc7_anchors(i);
    }
}
