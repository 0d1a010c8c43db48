// tests/emu/test_unit_kernel_emu.cc -- TEST INFRASTRUCTURE ONLY.
// The cases of test_decode_units_emu.cc (this encoder's fragments, hand-built 8-byte and 4-byte fragments, copies that
// leave their fragment, lying and truncated indexes, every destination misalignment) through the launch sequence of
// hap_api.cu's DecodePasses with snappy_execute_units_kernel ahead of the execute kernel, against the CPU oracle.  The
// windows the cases expect on the unit path must be decoded by the unit kernel (counted), the execute kernel's own unit
// path must not run at all, and the 4-byte windows the unit kernel declines must reach the execute kernel (counted).
#define HAPB200_EMU
#include "hap_host.h"
#include "snappy_decode.cuh"
#include "decode_emu.h"

static uint64_t g_execute_unit_path = 0;   // windows the execute kernel's own unit path decoded behind the unit kernel

static inline void decode_jobs_unit_kernel_emu(hapb200::ChunkJob *jobs, uint32_t njobs, uint64_t in_bound, uint64_t out_bound, uint32_t use_index,
                                               unsigned ex_grid = 3, uint32_t *windows_out = nullptr)
{
    using namespace hapb200;
    const uint32_t entry_slots = (uint32_t)(2 * (in_bound / kIdxWin + njobs) + 16);
    const uint32_t win_cap = (uint32_t)(kIdxParts * (uint64_t)entry_slots + out_bound / kIndexFragBytes + 2ull * njobs + 16);
    std::vector<DecWin> wins(win_cap);
    std::vector<uint8_t> entries((size_t)entry_slots * kIdxThreads, 0xEE);
    std::vector<uint32_t> done(win_cap, 0);
    DecodeCtl ctl;
    memset(&ctl, 0, sizeof ctl);
    uint32_t any_left = 0;
    const uint64_t exec_units0 = emu_unit_windows();
    HAP_LAUNCH(hap_build_windows_kernel, dim3((njobs + 127) / 128), dim3(128), 0, nullptr, jobs, njobs, use_index, wins.data(), win_cap, &ctl);
    HAP_LAUNCH(snappy_index_kernel, dim3(njobs), dim3(kIdxThreads), sizeof(IndexSmem), nullptr, jobs, (int)njobs, 0u, wins.data(),
               win_cap, entries.data(), entry_slots, &ctl);
    if (use_index)
        HAP_LAUNCH(snappy_execute_units_kernel, dim3(ex_grid), dim3(kUxThreads), sizeof(UnitSmem), nullptr, jobs, njobs, wins.data(), &ctl,
                   done.data());
    HAP_LAUNCH(snappy_execute_kernel, dim3(ex_grid), dim3(kExThreads), sizeof(ExecSmem), nullptr, jobs, njobs, 0u, wins.data(), &ctl, done.data());
    if (use_index) {
        HAP_LAUNCH(hap_requeue_mismatched_kernel, dim3((njobs + 127) / 128), dim3(128), 0, nullptr, jobs, njobs, &any_left);
        HAP_LAUNCH(snappy_index_kernel, dim3(njobs), dim3(kIdxThreads), sizeof(IndexSmem), nullptr, jobs, (int)njobs, 1u, wins.data(),
                   win_cap, entries.data(), entry_slots, &ctl);
        HAP_LAUNCH(snappy_execute_kernel, dim3(ex_grid), dim3(kExThreads), sizeof(ExecSmem), nullptr, jobs, njobs, 1u, wins.data(), &ctl, done.data());
    }
    g_execute_unit_path += emu_unit_windows() - exec_units0;
    if (ctl.overflow) g_decode_emu_overflow++;
    if (windows_out) { windows_out[0] = ctl.n_windows; windows_out[1] = any_left; }
}

// the cases, their checks and their main, with the launch sequence above and the unit kernel's counter
#define decode_jobs_emu decode_jobs_unit_kernel_emu
#define emu_unit_windows emu_unit_kernel_windows
#define main unit_cases_main
#include "test_decode_units_emu.cc"
#undef main
#undef emu_unit_windows
#undef decode_jobs_emu

int main(int argc, char **argv)
{
    int r = unit_cases_main(argc, argv);
    if (g_execute_unit_path != 0) {
        fprintf(stderr, "FAIL: the execute kernel's unit path decoded %llu windows behind the unit kernel\n", (unsigned long long)g_execute_unit_path);
        r = 1;
    }
    if (hapb200::emu_unit_kernel_declined() == 0) {
        fprintf(stderr, "FAIL: no window was left to the execute kernel (the 4-byte cases must be)\n");
        r = 1;
    }
    printf("%llu unit-kernel windows, %llu declined\n", (unsigned long long)hapb200::emu_unit_kernel_windows(),
           (unsigned long long)hapb200::emu_unit_kernel_declined());
    return r;
}
