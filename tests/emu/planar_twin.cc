// tests/emu/planar_twin.cc -- TEST INFRASTRUCTURE ONLY.
// tests/emu/planar_twin.h exported as plain C for tests/planar_util.py (built with g++ into tests/emu/_build), and the
// kernel's alpha mapping, which tests/test_planar_cpu.py holds to the definition over every sample value.
#include "planar_twin.h"

extern "C" void planar_twin_to_rgba(const uint8_t *luma, const uint8_t *cb, const uint8_t *cr, const uint8_t *alpha, uint32_t width,
                                    uint32_t height, uint64_t lpitch, uint64_t cpitch, int sub, int n, int color_space, uint8_t *rgba)
{
    planar_twin::picture(luma, cb, cr, alpha, width, height, lpitch, cpitch, sub, n, color_space, rgba);
}

extern "C" uint32_t planar_twin_kernel_alpha(uint32_t a, int n)
{
    const hapb200::PlanarSrc k = hapb200::planar_src_args(n, 0, nullptr, nullptr, nullptr, 0);
    return hapb200::planar_alpha16(a, k);
}
