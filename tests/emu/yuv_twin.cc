// tests/emu/yuv_twin.cc -- TEST INFRASTRUCTURE ONLY.
// tests/emu/yuv_twin.h exported as plain C for tests/yuv_util.py (built with g++ into tests/emu/_build).
#include "yuv_twin.h"

extern "C" void yuv_twin_to_rgba(const uint8_t *luma, const uint8_t *chroma, uint32_t width, uint32_t height, uint64_t pitch, int layout,
                                 int color_space, uint8_t *rgba)
{
    yuv_twin::picture(luma, chroma, width, height, pitch, layout, color_space, rgba);
}
