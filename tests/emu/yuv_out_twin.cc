// tests/emu/yuv_out_twin.cc -- TEST INFRASTRUCTURE ONLY.
// tests/emu/yuv_out_twin.h exported as plain C for tests/yuv_out_util.py (built with g++ into tests/emu/_build).
#include "yuv_out_twin.h"

extern "C" void yuv_out_twin_from_rgba(const uint8_t *rgba, uint32_t width, uint32_t height, int layout, int color_space, uint8_t *luma,
                                       uint8_t *chroma, uint64_t pitch)
{
    yuv_out_twin::picture(rgba, width, height, layout, color_space, luma, chroma, pitch);
}
