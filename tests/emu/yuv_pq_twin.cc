// tests/emu/yuv_pq_twin.cc -- TEST INFRASTRUCTURE ONLY.
// The library's PQ table (yuv_pq_table) and tests/emu/yuv_pq_twin.h exported as plain C for tests/yuv_pq_util.py (built with
// g++ into tests/emu/_build).
#include "yuv_pq_twin.h"

using namespace hapb200;

extern "C" void yuv_pq_twin_table(uint32_t unit_nits, uint16_t *table) { yuv_pq_table(unit_nits, table); }

extern "C" void yuv_pq_twin_to_rgba_half(const uint8_t *luma, const uint8_t *chroma, uint32_t width, uint32_t height, uint64_t pitch,
                                         int color_space, uint32_t unit_nits, uint16_t *rgba)
{
    uint16_t table[4096];
    yuv_pq_table(unit_nits, table);
    yuv_pq_twin::picture(luma, chroma, width, height, pitch, color_space, table, rgba);
}
