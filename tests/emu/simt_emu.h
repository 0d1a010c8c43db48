// tests/emu/simt_emu.h -- TEST INFRASTRUCTURE ONLY (g++; never compiled into libhap_b200.so).
//
// A small SIMT emulator: one CUDA block = a set of ucontext fibers on one OS thread, switched only
// at synchronisation points (__syncthreads, __syncwarp, warp collectives).  Blocks of a grid run
// one after another.  The resume ORDER of fibers is selectable (forward / reverse / seeded random)
// so that code relying on an accidental thread order between barriers (a missing __syncthreads)
// fails in at least one mode.  It exists because the build container has no GPU: kernel logic is
// debugged here against the oracle, then confirmed on the H100 with pytest -m gpu.
#pragma once

#include <algorithm>
#include <cassert>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <vector>

struct uint3 { unsigned x, y, z; };
struct uint2 { unsigned x, y; };
struct uint4 { unsigned x, y, z, w; };
struct uchar4 { unsigned char x, y, z, w; };
struct dim3 {
    unsigned x, y, z;
    dim3(unsigned a = 1, unsigned b = 1, unsigned c = 1) : x(a), y(b), z(c) {}
};
static inline uint4 make_uint4(unsigned a, unsigned b, unsigned c, unsigned d) { return uint4{a, b, c, d}; }
static inline uint2 make_uint2(unsigned a, unsigned b) { return uint2{a, b}; }
typedef void *cudaStream_t;

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline
#define __noinline__
#define __restrict__
#define __shared__ static
#define __align__(n) alignas(n)
#define __launch_bounds__(...)

// Minimal x86-64 context switch (callee-saved registers + stack pointer).  glibc's swapcontext does
// a sigprocmask system call per switch, which made barrier-heavy kernels take minutes.
extern "C" void hap_emu_swap(void **save_sp, void *load_sp);
asm(".text\n.globl hap_emu_swap\n.type hap_emu_swap,@function\nhap_emu_swap:\n"
    "pushq %rbp\npushq %rbx\npushq %r12\npushq %r13\npushq %r14\npushq %r15\n"
    "movq %rsp, (%rdi)\nmovq %rsi, %rsp\n"
    "popq %r15\npopq %r14\npopq %r13\npopq %r12\npopq %rbx\npopq %rbp\nret\n"
    ".size hap_emu_swap,.-hap_emu_swap\n");

namespace emu {

struct Warp {
    int arrived = 0;
    unsigned gen = 0;
    unsigned alive_mask = 0;
    uint64_t xchg[32];
};

struct Fiber {
    void *sp = nullptr;
    char *stack = nullptr;
    bool done = false;
    uint3 tid{0, 0, 0};
    int linear = 0;
    unsigned or_phase = 0;
};

struct NamedBar {
    int arrived = 0;
    unsigned gen = 0;
    int acc = 0;
    int res[2] = {0, 0};
};

struct Block {
    NamedBar named[16];
    std::vector<Fiber> fibers;
    std::vector<Warp> warps;
    int arrived = 0;
    unsigned gen = 0;
    int alive = 0;
    int current = -1;
    void *sched_sp = nullptr;
    unsigned char *dyn_smem = nullptr;
    int or_acc[2] = {0, 0};
    const std::function<void()> *body = nullptr;
};

inline Block *&g_block() { static Block *b = nullptr; return b; }
inline uint3 &g_block_idx() { static uint3 v{0, 0, 0}; return v; }
inline dim3 &g_block_dim() { static dim3 v; return v; }
inline dim3 &g_grid_dim() { static dim3 v; return v; }
// 0 forward, 1 reverse, >=2 seeded shuffle
inline int &g_order_mode() { static int m = 0; return m; }
inline uint64_t &g_barriers() { static uint64_t n = 0; return n; }

inline const uint3 &cur_tid() { Block *B = g_block(); return B->fibers[B->current].tid; }
inline int cur_linear() { Block *B = g_block(); return B->fibers[B->current].linear; }
inline int cur_lane() { return cur_linear() & 31; }
inline Warp &cur_warp() { Block *B = g_block(); return B->warps[cur_linear() >> 5]; }

inline void yield() {
    Block *B = g_block();
    hap_emu_swap(&B->fibers[B->current].sp, B->sched_sp);
}

inline void syncthreads() {
    Block &B = *g_block();
    g_barriers()++;
    unsigned g = B.gen;
    if (++B.arrived >= B.alive) {
        B.arrived = 0;
        B.gen++;
    } else {
        while (B.gen == g) yield();
    }
}

// bar.sync / bar.arrive / bar.red.or with a barrier number and a participant count
inline void bar_sync(int id, int n) {
    NamedBar &N = g_block()->named[id];
    g_barriers()++;
    unsigned g = N.gen;
    if (++N.arrived >= n) { N.res[g & 1] = N.acc; N.acc = 0; N.arrived = 0; N.gen++; }
    else while (N.gen == g) yield();
}
inline void bar_arrive(int id, int n) {
    NamedBar &N = g_block()->named[id];
    unsigned g = N.gen;
    if (++N.arrived >= n) { N.res[g & 1] = N.acc; N.acc = 0; N.arrived = 0; N.gen++; }
}
inline int bar_or(int id, int n, int pred) {
    NamedBar &N = g_block()->named[id];
    g_barriers()++;
    unsigned g = N.gen;
    if (pred) N.acc = 1;
    if (++N.arrived >= n) { N.res[g & 1] = N.acc; N.acc = 0; N.arrived = 0; N.gen++; }
    else while (N.gen == g) yield();
    return N.res[g & 1];
}

inline void warp_barrier(unsigned mask) {
    Warp &W = cur_warp();
    unsigned g = W.gen;
    int need = __builtin_popcount(mask & W.alive_mask);
    if (++W.arrived >= need) {
        W.arrived = 0;
        W.gen++;
    } else {
        while (W.gen == g) yield();
    }
}

inline void trampoline() {
    Block *B = g_block();
    Fiber &F = B->fibers[B->current];
    (*B->body)();
    F.done = true;
    B->alive--;
    B->warps[F.linear >> 5].alive_mask &= ~(1u << (F.linear & 31));
    if (B->arrived > 0 && B->arrived >= B->alive) {
        fprintf(stderr, "emu: thread exited while others wait at __syncthreads (divergent barrier)\n");
        abort();
    }
    hap_emu_swap(&F.sp, B->sched_sp);
    abort();
}

inline void run_block(dim3 block, size_t smem, const std::function<void()> &body) {
    Block B;
    int n = (int)(block.x * block.y * block.z);
    B.fibers.resize(n);
    B.warps.resize((n + 31) / 32);
    B.alive = n;
    B.body = &body;
    std::vector<unsigned char> dyn(smem + 64);
    B.dyn_smem = (unsigned char *)(((uintptr_t)dyn.data() + 15) & ~(uintptr_t)15);
    const size_t STACK = 256 * 1024;
    g_block() = &B;
    for (int i = 0; i < n; i++) {
        Fiber &F = B.fibers[i];
        F.linear = i;
        F.tid = uint3{(unsigned)i % block.x, ((unsigned)i / block.x) % block.y, (unsigned)i / (block.x * block.y)};
        F.stack = (char *)malloc(STACK);
        uintptr_t top = ((uintptr_t)F.stack + STACK) & ~(uintptr_t)15;
        void **sp = (void **)top;
        *--sp = nullptr;                      // fake return address of trampoline
        *--sp = (void *)&trampoline;          // `ret` target of the first switch
        for (int r = 0; r < 6; r++) *--sp = nullptr;
        F.sp = (void *)sp;
        B.warps[i >> 5].alive_mask |= 1u << (i & 31);
    }
    std::vector<int> order(n);
    for (int i = 0; i < n; i++) order[i] = i;
    uint64_t rng = 0x9E3779B97F4A7C15ull * (uint64_t)(g_order_mode() + 1);
    int remaining = n;
    while (remaining > 0) {
        int mode = g_order_mode();
        if (mode == 1) {
            for (int i = 0; i < n; i++) order[i] = n - 1 - i;
        } else if (mode >= 2) {
            for (int i = n - 1; i > 0; i--) {
                rng ^= rng << 13; rng ^= rng >> 7; rng ^= rng << 17;
                std::swap(order[i], order[(int)(rng % (uint64_t)(i + 1))]);
            }
        }
        int progressed = 0;
        for (int k = 0; k < n; k++) {
            int i = order[k];
            if (B.fibers[i].done) continue;
            B.current = i;
            hap_emu_swap(&B.sched_sp, B.fibers[i].sp);
            progressed++;
            if (B.fibers[i].done) remaining--;
        }
        if (!progressed) break;
    }
    for (int i = 0; i < n; i++) free(B.fibers[i].stack);
    g_block() = nullptr;
}

inline void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()> &body) {
    g_grid_dim() = grid;
    g_block_dim() = block;
    for (unsigned z = 0; z < grid.z; z++)
        for (unsigned y = 0; y < grid.y; y++)
            for (unsigned x = 0; x < grid.x; x++) {
                g_block_idx() = uint3{x, y, z};
                run_block(block, smem, body);
            }
}

template <class T> inline uint64_t to_bits(T v) { uint64_t b = 0; memcpy(&b, &v, sizeof(T)); return b; }
template <class T> inline T from_bits(uint64_t b) { T v; memcpy(&v, &b, sizeof(T)); return v; }

template <class T, class F> inline T collective(unsigned mask, T v, F pick) {
    Warp &W = cur_warp();
    int lane = cur_lane();
    W.xchg[lane] = to_bits(v);
    warp_barrier(mask);
    T r = pick(W, lane);
    warp_barrier(mask);
    return r;
}

}  // namespace emu

#define threadIdx (emu::cur_tid())
#define blockIdx (emu::g_block_idx())
#define blockDim (emu::g_block_dim())
#define gridDim (emu::g_grid_dim())

#define HAP_LAUNCH(kernel, grid, block, smem, stream, ...) \
    emu::launch((grid), (block), (smem), [&]() { kernel(__VA_ARGS__); })
#define HAP_DYN_SMEM(name) unsigned char *name = emu::g_block()->dyn_smem

static inline void __syncthreads() { emu::syncthreads(); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::warp_barrier(mask); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
typedef uintptr_t hap_saddr_t;
static inline hap_saddr_t hap_smem_addr(const void *p) { return (hap_saddr_t)p; }
static inline uint32_t hap_lds_u8(hap_saddr_t a) { return *(const uint8_t *)a; }
static inline void hap_sts_u16(hap_saddr_t a, uint32_t v) { *(uint16_t *)a = (uint16_t)v; }
typedef unsigned long long hap_mbar_t;
static inline void hap_mbar_init(hap_mbar_t *bar, uint32_t) { *bar = 0; }
static inline void hap_mbar_expect_tx(hap_mbar_t *, uint32_t) {}
static inline void hap_tma_load_1d(void *smem_dst, const void *gmem_src, uint32_t bytes, hap_mbar_t *)
{
    // the real unit requires 16-byte alignment of both addresses and of the size: keep the emulated kernels honest
    if (((uintptr_t)smem_dst | (uintptr_t)gmem_src | bytes) & 15) { fprintf(stderr, "emu: misaligned bulk copy\n"); abort(); }
    memcpy(smem_dst, gmem_src, bytes);
}
static inline void hap_mbar_wait(hap_mbar_t *, uint32_t) {}
static inline void hap_fence_proxy_async() {}
static inline uint32_t hap_ld_acquire(const uint32_t *p) { return *p; }
static inline void hap_st_release(uint32_t *p, uint32_t v) { *p = v; }
static inline void hap_nanosleep(uint32_t) {}
static inline void hap_bar_sync(int id, int n) { emu::bar_sync(id, n); }
static inline void hap_bar_arrive(int id, int n) { emu::bar_arrive(id, n); }
static inline int hap_bar_or(int id, int n, int pred) { return emu::bar_or(id, n, pred); }

static inline int __syncthreads_or(int pred) {
    emu::Block *B = emu::g_block();
    unsigned ph = B->fibers[B->current].or_phase++ & 1;
    if (pred) B->or_acc[ph] = 1;
    emu::syncthreads();
    int r = B->or_acc[ph];
    emu::syncthreads();
    B->or_acc[ph] = 0;  // the slot is not reused before every thread has passed the next call's barriers
    return r;
}

template <class T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32) {
    return emu::collective(mask, v, [&](emu::Warp &W, int lane) {
        int base = lane & ~(width - 1);
        return emu::from_bits<T>(W.xchg[base + (src & (width - 1))]);
    });
}
template <class T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    return emu::collective(mask, v, [&](emu::Warp &W, int lane) {
        int base = lane & ~(width - 1);
        int s = lane - (int)delta;
        return emu::from_bits<T>(W.xchg[s < base ? lane : s]);
    });
}
template <class T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32) {
    return emu::collective(mask, v, [&](emu::Warp &W, int lane) {
        int base = lane & ~(width - 1);
        int s = lane + (int)delta;
        return emu::from_bits<T>(W.xchg[s >= base + width ? lane : s]);
    });
}
template <class T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32) {
    return emu::collective(mask, v, [&](emu::Warp &W, int lane) {
        (void)width;
        return emu::from_bits<T>(W.xchg[lane ^ lanemask]);
    });
}
static inline unsigned __ballot_sync(unsigned mask, int pred) {
    return emu::collective(mask, (unsigned)(pred != 0), [&](emu::Warp &W, int) {
        unsigned r = 0;
        for (int l = 0; l < 32; l++)
            if ((mask & W.alive_mask) >> l & 1) r |= (unsigned)(W.xchg[l] & 1) << l;
        return r;
    });
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) {
    unsigned b = __ballot_sync(mask, pred);
    return b == (mask & emu::cur_warp().alive_mask);
}
#define EMU_REDUCE(name, T, init, op)                                                   \
    static inline T name(unsigned mask, T v) {                                          \
        return emu::collective(mask, v, [&](emu::Warp &W, int) {                        \
            T r = init;                                                                 \
            for (int l = 0; l < 32; l++)                                                \
                if ((mask & W.alive_mask) >> l & 1) { T o = emu::from_bits<T>(W.xchg[l]); r = op; } \
            return r;                                                                   \
        });                                                                             \
    }
EMU_REDUCE(__reduce_add_sync, unsigned, 0u, r + o)
EMU_REDUCE(__reduce_max_sync, unsigned, 0u, (r > o ? r : o))
EMU_REDUCE(__reduce_min_sync, unsigned, 0xffffffffu, (r < o ? r : o))
EMU_REDUCE(__reduce_or_sync, unsigned, 0u, r | o)
EMU_REDUCE(__reduce_and_sync, unsigned, 0xffffffffu, r & o)
#undef EMU_REDUCE

template <class T> static inline T atomicAdd(T *p, T v) { T o = *p; *p = o + v; return o; }
template <class T> static inline T atomicMin(T *p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T atomicMax(T *p, T v) { T o = *p; if (v > o) *p = v; return o; }
template <class T> static inline T atomicOr(T *p, T v) { T o = *p; *p = o | v; return o; }
template <class T> static inline T atomicAnd(T *p, T v) { T o = *p; *p = o & v; return o; }
template <class T> static inline T atomicExch(T *p, T v) { T o = *p; *p = v; return o; }
template <class T> static inline T atomicCAS(T *p, T cmp, T v) { T o = *p; if (o == cmp) *p = v; return o; }

static inline int __popc(unsigned x) { return __builtin_popcount(x); }
static inline int __popcll(unsigned long long x) { return __builtin_popcountll(x); }
static inline int __clz(int x) { return x ? __builtin_clz((unsigned)x) : 32; }
static inline int __ffs(int x) { return __builtin_ffs(x); }
static inline unsigned __brev(unsigned x) {
    unsigned r = 0;
    for (int i = 0; i < 32; i++) r |= ((x >> i) & 1u) << (31 - i);
    return r;
}
static inline unsigned __byte_perm(unsigned x, unsigned y, unsigned s) {
    uint64_t v = ((uint64_t)y << 32) | x;
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        unsigned sel = (s >> (4 * i)) & 0xF;
        unsigned b = (unsigned)(v >> (8 * (sel & 7))) & 0xFF;
        if (sel & 8) b = (b & 0x80) ? 0xFF : 0x00;
        r |= b << (8 * i);
    }
    return r;
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned shift) {
    return (unsigned)((((uint64_t)hi << 32) | lo) >> (shift & 31));
}
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned shift) {
    return (unsigned)(((((uint64_t)hi << 32) | lo) << (shift & 31)) >> 32);
}
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
template <class T> static inline T __ldg(const T *p) { return *p; }
template <class T> static inline T __ldcg(const T *p) { return *p; }
template <class T> static inline T __ldcs(const T *p) { return *p; }
template <class T> static inline void __stcg(T *p, T v) { *p = v; }
template <class T> static inline void __stcs(T *p, T v) { *p = v; }
static inline int __float2int_rn(float f) { return (int)lrintf(f); }
static inline float __saturatef(float f) { return f < 0.f ? 0.f : f > 1.f ? 1.f : f; }
static inline float __fdividef(float a, float b) { return a / b; }
static inline float rsqrtf(float a) { return 1.0f / sqrtf(a); }
static inline float __frcp_rn(float a) { return 1.0f / a; }
static inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
static inline float __fmul_rn(float a, float b) { return a * b; }
static inline float __fadd_rn(float a, float b) { return a + b; }
static inline unsigned __vabsdiffu4(unsigned a, unsigned b) {
    unsigned r = 0;
    for (int i = 0; i < 4; i++) {
        int x = (a >> (8 * i)) & 0xFF, y = (b >> (8 * i)) & 0xFF;
        r |= (unsigned)(x > y ? x - y : y - x) << (8 * i);
    }
    return r;
}
using std::max;
using std::min;
static inline unsigned umin(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned umax(unsigned a, unsigned b) { return a > b ? a : b; }
