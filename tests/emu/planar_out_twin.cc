// tests/emu/planar_out_twin.cc -- TEST INFRASTRUCTURE ONLY.
// tests/emu/planar_out_twin.h exported as plain C for tests/planar_out_util.py (built with g++ into tests/emu/_build).
#include "planar_out_twin.h"

extern "C" void planar_out_twin_from_rgba(const uint8_t *rgba, uint32_t width, uint32_t height, uint8_t *luma, uint8_t *cb, uint8_t *cr,
                                          uint8_t *alpha, uint64_t lpitch, uint64_t cpitch, int sub, int n, int color_space)
{
    planar_out_twin::picture(rgba, width, height, luma, cb, cr, alpha, lpitch, cpitch, sub, n, color_space);
}
