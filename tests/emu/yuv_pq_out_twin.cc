// tests/emu/yuv_pq_out_twin.cc -- TEST INFRASTRUCTURE ONLY.
// The library's table P (yuv_pq_out_table) and tests/emu/yuv_pq_out_twin.h exported as plain C for tests/yuv_pq_out_util.py
// (built with g++ into tests/emu/_build).
#include "yuv_pq_out_twin.h"

#include <vector>

using namespace hapb200;

extern "C" void yuv_pq_out_twin_table(uint32_t unit_nits, uint16_t *table) { yuv_pq_out_table(unit_nits, table); }

extern "C" void yuv_pq_out_twin_from_half(const uint16_t *rgba, uint32_t width, uint32_t height, int color_space, uint32_t unit_nits,
                                          uint8_t *luma, uint8_t *chroma, uint64_t pitch)
{
    std::vector<uint16_t> table(kPqOutEntries);
    yuv_pq_out_table(unit_nits, table.data());
    yuv_pq_out_twin::picture(rgba, width, height, color_space, table.data(), luma, chroma, pitch);
}
