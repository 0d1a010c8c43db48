// hap_b200/csrc/hap_api.cu -- the C-ABI of libhap_b200.so: the six entry points of include/hap.h
// (same signatures and behaviour as /root/reference/source/hap.h:76-152) and the extensions of
// include/hap_b200.h.  Host code here only validates arguments, walks section headers, moves
// buffers and launches kernels; all compression, decompression, block coding and frame assembly
// runs in the kernels of this directory.  There is no CPU implementation of any of those steps in
// this library: without a CUDA device the compute entry points return HapResult_Internal_Error.
#include "../../include/hap_b200.h"

#include "bc6h_decode.cuh"
#include "bc6h_encode.cuh"
#include "bc_decode.cuh"
#include "bc_encode.cuh"
#include "hap_assemble.cuh"
#include "hap_host.h"
#include "hap_mov.h"
#include "hap_parse.cuh"
#include "hapq_fused.cuh"
#include "planar_sink.cuh"
#include "snappy_decode.cuh"
#include "snappy_encode.cuh"
#include "yuv_sink.cuh"

#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <vector>

using namespace hapb200;

namespace {

std::atomic<unsigned long long> g_launches{0};
// Options (HapB200SetOption).  g_use_index: the decoder uses a frame's embedded fragment index when it has one
// (hap_index.h).  g_write_index: the encoder writes that section into Complex texture sections.
std::atomic<int> g_use_index{1};
std::atomic<int> g_write_index{0};
std::atomic<int> g_write_offsets{0};
std::atomic<int> g_chroma_refine{0};   // HAPB200_OPTION_CHROMA_REFINE

// Optional per-stage device timing (HapB200SetStageTiming): CUDA events around every kernel, on the
// stream the kernel is launched on.  Off by default; bench.py turns it on for its roofline pass only.
enum Stage { kStBcEncode = 0, kStSnappyEncode, kStPlan, kStPlace, kStParse, kStSnappyDecode, kStCollect, kStBcDecode, kStSnappyIndex, kStWindows, kStCount };
struct StageTimer {
    std::mutex mu;
    bool on = false;
    struct Rec { int stage; cudaEvent_t a, b; };
    std::vector<Rec> recs;
    double ms[kStCount] = {0};
    unsigned long long n[kStCount] = {0};
};
StageTimer g_timer;

struct StageScope {
    cudaEvent_t a = nullptr, b = nullptr;
    cudaStream_t st;
    int stage;
    bool live;
    StageScope(int stage_, cudaStream_t st_) : st(st_), stage(stage_), live(g_timer.on)
    {
        if (live) { cudaEventCreate(&a); cudaEventCreate(&b); cudaEventRecord(a, st); }
    }
    ~StageScope()
    {
        if (!live) return;
        cudaEventRecord(b, st);
        std::lock_guard<std::mutex> l(g_timer.mu);
        g_timer.recs.push_back({stage, a, b});
    }
};

#define HAP_KLAUNCH(stage, kernel, grid, block, smem, stream, ...)         \
    do {                                                                   \
        StageScope hap_scope_(stage, stream);                              \
        HAP_LAUNCH(kernel, grid, block, smem, stream, __VA_ARGS__);        \
        g_launches.fetch_add(1, std::memory_order_relaxed);                \
    } while (0)

// ---- devices ------------------------------------------------------------------------------------------------------------
// The library can drive every GPU of the box from one process (or one GPU per process under torchrun -- both work):
//   * a call that has a DEVICE pointer among its buffers runs on that pointer's device;
//   * a call with host pointers only runs on the process's default device: the device that was current in the thread that
//     made the library's first call, or the one named by HapB200SetDevice (a new host thread starts on device 0, so "the
//     calling thread's current device" would send the worker threads of a process that drives GPU 3 to GPU 0);
//   * the caller's current device is restored when the call returns.
// Per-device state (SM count, kernel attributes, memory-pool threshold) is set up on a device's first use.
constexpr int kMaxDevices = 64;
struct DeviceState {
    std::once_flag once;
    bool ready = false;
    int sm_count = 132;
    int k5_ctas_per_sm = 1;   // resident CTAs of the fragment compressor per SM (its persistent grid is this x sm_count)
    int fused_ctas_per_sm = 1;   // the same for the fused Hap Q encoder (hapq_fused.cuh)
    int fused_place_ctas_per_sm = 1;   // ... and for its variant that writes the frames itself
    int ws_place_ctas_per_sm = 1;   // ... and for that variant with its fit and compressor in warp groups of their own
    int units_ctas_per_sm = 1;   // ... and for the Snappy decoder's unit kernel (snappy_execute_units_kernel)
};
DeviceState g_dev[kMaxDevices];
std::atomic<int> g_default_device{-1};
std::mutex g_legacy_mu;   // serialises the calls that run on the legacy default stream (those with a device pointer among their buffers)
thread_local int t_device = 0;   // device of the library call running on this thread

void device_init(int dev)
{
    DeviceState &d = g_dev[dev];
    if (cudaDeviceGetAttribute(&d.sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || d.sm_count <= 0) { cudaGetLastError(); d.sm_count = 132; }
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        unsigned long long keep = ~0ull;  // keep freed scratch in the pool: steady-state calls never hit the OS
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    // (function attributes are per device: set them on each device's first use)
    bool ok = cudaFuncSetAttribute(snappy_execute_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ExecSmem)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(snappy_index_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(IndexSmem)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(snappy_encode_fragments_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                    (int)sizeof(EncodeSmem)) == cudaSuccess;
    ok = ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.k5_ctas_per_sm, snappy_encode_fragments_kernel, kEncThreads,
                                                             sizeof(EncodeSmem)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(hapq_fused_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(EncodeSmem)) == cudaSuccess;
    ok = ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.fused_ctas_per_sm, hapq_fused_encode_kernel, kEncThreads,
                                                             sizeof(EncodeSmem)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(hapq_fused_place_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(EncodeSmem)) == cudaSuccess;
    ok = ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.fused_place_ctas_per_sm, hapq_fused_place_kernel, kEncThreads,
                                                             sizeof(EncodeSmem)) == cudaSuccess;
    ok = ok && cudaFuncSetAttribute(hapq_ws_place_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(WsSmem)) == cudaSuccess;
    ok = ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.ws_place_ctas_per_sm, hapq_ws_place_kernel, kWsThreads, sizeof(WsSmem)) ==
                   cudaSuccess;
#if HAPB200_EX_UNIT_KERNEL
    ok = ok && cudaFuncSetAttribute(snappy_execute_units_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(UnitSmem)) == cudaSuccess;
    ok = ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&d.units_ctas_per_sm, snappy_execute_units_kernel, kUxThreads,
                                                             sizeof(UnitSmem)) == cudaSuccess;
#endif
    if (!ok) { cudaGetLastError(); return; }
    if (d.units_ctas_per_sm < 1) d.units_ctas_per_sm = 1;
    if (d.fused_place_ctas_per_sm < 1) d.fused_place_ctas_per_sm = 1;
    if (d.ws_place_ctas_per_sm < 1) d.ws_place_ctas_per_sm = 1;
    if (d.k5_ctas_per_sm < 1) d.k5_ctas_per_sm = 1;
    if (d.fused_ctas_per_sm < 1) d.fused_ctas_per_sm = 1;
    d.ready = true;
}

int pointer_device(const void *p)   // device ordinal of a device / managed pointer, -1 for host memory
{
    cudaPointerAttributes a;
    if (!p || cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return -1; }
    return (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) ? a.device : -1;
}
inline bool is_device(const void *p) { return pointer_device(p) >= 0; }

// The device of a codec call.  `hints`: the call's buffers; the first device pointer among them decides the device,
// else the process default.  -1 when there is none.
int call_device(std::initializer_list<const void *> hints)
{
    static std::once_flag env_once;
    std::call_once(env_once, [] {
        // process-wide defaults of the options (HapB200SetOption overrides them)
        if (const char *e = getenv("HAPB200_WRITE_INDEX")) g_write_index.store(atoi(e) != 0);
        if (const char *e = getenv("HAPB200_USE_INDEX")) g_use_index.store(atoi(e) != 0);
        if (const char *e = getenv("HAPB200_WRITE_OFFSET_TABLE")) g_write_offsets.store(atoi(e) != 0);
        if (const char *e = getenv("HAPB200_CHROMA_REFINE")) g_chroma_refine.store(atoi(e) != 0);
    });
    for (const void *h : hints)
        if (const int d = pointer_device(h); d >= 0) return d;
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess) { cudaGetLastError(); return -1; }
    int expected = -1;
    g_default_device.compare_exchange_strong(expected, cur);   // first call: this thread's device becomes the default
    return g_default_device.load();
}

// One per entry point: runs the call on `device` (set up on its first use) and restores the caller's device.
struct DeviceGuard {
    int saved = -1;
    bool ok = false;
    explicit DeviceGuard(int device)
    {
        if (cudaGetDevice(&saved) != cudaSuccess) { cudaGetLastError(); saved = -1; return; }
        if (device < 0 || device >= kMaxDevices) return;
        if (device != saved && cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return; }
        std::call_once(g_dev[device].once, device_init, device);
        t_device = device;
        ok = g_dev[device].ready;
    }
    ~DeviceGuard()
    {
        int cur = -1;
        if (saved >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != saved) cudaSetDevice(saved);
        cudaGetLastError();
    }
};
#define HAP_ENTER(...)                                           \
    DeviceGuard hap_device_guard_(call_device({__VA_ARGS__}));   \
    if (!hap_device_guard_.ok) return HapResult_Internal_Error

inline int sm_count() { return g_dev[t_device].sm_count; }
#if HAPB200_EX_UNIT_KERNEL
inline int units_ctas_per_sm() { return g_dev[t_device].units_ctas_per_sm; }
#endif
const cudaStream_t kLegacyStream = cudaStreamLegacy;
// NULL-stream calls and the host-pointer entry points that touch caller-owned device buffers run on the LEGACY default
// stream: it orders itself against every blocking stream of the process, so buffers a caller produced on its own (blocking)
// stream -- torch's current stream, cudaMemset, ... -- are complete before our kernels touch them.

// Stream of one host-pointer call.  When every buffer of the call is host memory nothing outside the call can
// be ordered against it, so it takes a private non-blocking stream from a pool and concurrent calls from
// different host threads overlap their copies and kernels (the reference is re-entrant, hap.c has no globals).
// With any device pointer among the arguments the call uses the legacy default stream under a mutex, which
// orders it after whatever produced those buffers on the caller's (blocking) streams.
// A pooled stream brings its own memory pool: scratch freed by one host-pointer call is handed to the next call
// on the SAME stream.  With the device's default pool, memory freed on one stream and re-used on another makes the
// second stream wait for the first, which chained concurrent calls from different host threads one behind the other.
struct PooledStream {
    cudaStream_t st = nullptr;
    cudaMemPool_t mem = nullptr;
};
thread_local cudaMemPool_t g_call_mem = nullptr;   // pool of the host-pointer call running on this thread, if any

struct CallStream {
    cudaStream_t st = nullptr;
    bool pooled = false;
    PooledStream ps;
    std::unique_lock<std::mutex> serial;
    static std::mutex &pool_mu() { static std::mutex m; return m; }
    static std::vector<PooledStream> &pool() { static std::vector<PooledStream> v[kMaxDevices]; return v[t_device]; }
    explicit CallStream(bool all_host)
    {
        if (all_host) {
            {
                std::lock_guard<std::mutex> l(pool_mu());
                if (!pool().empty()) { ps = pool().back(); pool().pop_back(); }
            }
            if (!ps.st) {
                if (cudaStreamCreateWithFlags(&ps.st, cudaStreamNonBlocking) != cudaSuccess) { cudaGetLastError(); ps.st = nullptr; }
                int dev = 0;
                cudaMemPoolProps props;
                memset(&props, 0, sizeof props);
                props.allocType = cudaMemAllocationTypePinned;
                props.handleTypes = cudaMemHandleTypeNone;
                props.location.type = cudaMemLocationTypeDevice;
                if (ps.st && cudaGetDevice(&dev) == cudaSuccess) {
                    props.location.id = dev;
                    if (cudaMemPoolCreate(&ps.mem, &props) == cudaSuccess) {
                        unsigned long long keep = ~0ull;
                        cudaMemPoolSetAttribute(ps.mem, cudaMemPoolAttrReleaseThreshold, &keep);
                    } else {
                        cudaGetLastError();
                        ps.mem = nullptr;   // fall back to the default pool
                    }
                }
            }
            st = ps.st;
            pooled = st != nullptr;
            if (pooled) g_call_mem = ps.mem;
        }
        if (!pooled) {
            serial = std::unique_lock<std::mutex>(g_legacy_mu);
            st = kLegacyStream;
        }
    }
    ~CallStream()
    {
        if (pooled) {
            g_call_mem = nullptr;
            std::lock_guard<std::mutex> l(pool_mu());
            pool().push_back(ps);   // (t_device is still this call's device: the guard outlives the stream)
        }
    }
};

// stream-ordered scratch
struct DevBuf {
    void *p = nullptr;
    cudaStream_t s;
    explicit DevBuf(cudaStream_t st) : s(st) {}
    bool alloc(size_t n)
    {
        n = (n + 31) & ~(size_t)15;   // whole 16-byte cells + one: kernels read their inputs in aligned 16-byte cells
        if (g_call_mem) return cudaMallocFromPoolAsync(&p, n, g_call_mem, s) == cudaSuccess;
        return cudaMallocAsync(&p, n, s) == cudaSuccess;
    }
    ~DevBuf() { if (p) cudaFreeAsync(p, s); }
    template <class T> T *as() { return reinterpret_cast<T *>(p); }
};

inline uint64_t align16(uint64_t v) { return (v + 15) & ~15ull; }

// ---- codec tables ------------------------------------------------------------------------------
struct CodecInfo {
    uint32_t textures;
    uint32_t fmt[2];
    uint32_t block_bytes[2];
    int bc_kind;
};
bool codec_info(unsigned codec, CodecInfo &c)
{
    switch (codec) {
    case HapB200Codec_Hap1: c = {1, {HapFmt_RGB_DXT1, 0}, {8, 0}, kBcDxt1}; return true;
    case HapB200Codec_Hap5: c = {1, {HapFmt_RGBA_DXT5, 0}, {16, 0}, kBcDxt5}; return true;
    case HapB200Codec_HapY: c = {1, {HapFmt_YCoCg_DXT5, 0}, {16, 0}, kBcYCoCg}; return true;
    case HapB200Codec_HapM: c = {2, {HapFmt_YCoCg_DXT5, HapFmt_A_RGTC1}, {16, 8}, kBcYCoCgPlusAlpha}; return true;
    case HapB200Codec_HapA: c = {1, {HapFmt_A_RGTC1, 0}, {8, 0}, kBcRgtc1}; return true;
    case HapB200Codec_Hap7: c = {1, {HapFmt_RGBA_BPTC_UNORM, 0}, {16, 0}, kBcBc7}; return true;
    default: return false;
    }
}
// the codecs the RGBA encode entry points take: every one with a block compressor (BC7 has none)
bool codec_encodes(const CodecInfo &c) { return c.bc_kind != kBcBc7; }

// Hap HDR: one BC6H texture, UF16 or SF16 as textureFormat.  No codec value names it (codec_info refuses it): the Hap HDR entry
// points take the texture format instead.
constexpr int kBcBc6h = kBcBc7 + 1;
bool bc6h_codec(unsigned textureFormat, CodecInfo &c)
{
    if (textureFormat != HapFmt_RGB_BPTC_UFLOAT && textureFormat != HapFmt_RGB_BPTC_SFLOAT) return false;
    c = {1, {textureFormat, 0}, {16, 0}, kBcBc6h};
    return true;
}

unsigned long texture_bytes(unsigned width, unsigned height, const CodecInfo &ci, unsigned index)
{
    if (index >= ci.textures || width % 4 || height % 4) return 0;
    return (unsigned long)(width / 4) * (height / 4) * ci.block_bytes[index];
}

unsigned long max_encoded_length_rgba(unsigned width, unsigned height, const CodecInfo &ci, unsigned chunkCount)
{
    unsigned long lens[2] = {texture_bytes(width, height, ci, 0), texture_bytes(width, height, ci, 1)};
    unsigned fmts[2] = {ci.fmt[0], ci.fmt[1]}, chunks[2] = {chunkCount, chunkCount};
    if (lens[0] == 0) return 0;
    return HapMaxEncodedLength(ci.textures, lens, fmts, chunks);
}

// hap.c:551-559 (SURVEY.md Q5): of two textures, one must be scaled YCoCg DXT5 or alpha RGTC1
bool texture_formats_ok(unsigned count, const unsigned *f)
{
    return count != 2 || f[0] == HapFmt_YCoCg_DXT5 || f[1] == HapFmt_YCoCg_DXT5 || f[0] == HapFmt_A_RGTC1 || f[1] == HapFmt_A_RGTC1;
}

// width x height pictures of `bpp` bytes per pixel (4: RGBA8, 8: RGBA16F), rows rowBytes apart.  aligned: the batch entry
// points' rules besides (16-byte aligned rows, picture address and picture stride).  The block kernels hold the row pitch and
// the block index in 32 bits.
bool rgba_geometry_ok(const void *rgba, unsigned width, unsigned height, unsigned long rowBytes, unsigned long frameStride, bool aligned,
                      unsigned long bpp = 4)
{
    if (!rgba || width == 0 || height == 0 || width % 4 || height % 4 || rowBytes < bpp * width) return false;
    if (rowBytes > HAPB200_MAX_ROW_BYTES || (unsigned long)(width / 4) * (height / 4) > HAPB200_MAX_BLOCKS) return false;
    return !aligned || (rowBytes % 16 == 0 && ((uintptr_t)rgba | frameStride) % 16 == 0);
}

// The batch entry points run `work` on the caller's stream, or on the legacy stream when the caller gave none; then they
// return only once the work is done.
template <class Work>
uint32_t on_batch_stream(void *stream, Work &&work)
{
    const cudaStream_t st = stream ? (cudaStream_t)stream : kLegacyStream;
    uint32_t r = work(st);
    if (r == HapResult_No_Error && !stream && cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); r = HapResult_Internal_Error; }
    return r;
}

// ---- device pipelines (all asynchronous on `st`) -------------------------------------------------

// The RGBA8 pictures the fused Hap Q encoder fits its blocks from (geometry g: g.frame_bytes apart, rows g.row_bytes apart).
struct FusedPictures {
    const uint8_t *rgba;
    BcGeom g;
};

// textures of `frames` frames (device, described by G.s[i].in_offset/in_stride relative to `base`) ->
// frames at out + f*out_stride, lengths in used[f].
// fused: the textures are not there yet; the fused Hap Q encoder fits them from these pictures, writes them to `base` and
// compresses them in one kernel, in place of the fragment compressor (G must pass fused_hapq_geometry).  Without the offset
// table it also writes the streams into the frames (hapq_ws_place_kernel, or hapq_fused_place_kernel in -DHAPB200_FUSED_WS=0
// builds), and the place kernel copies raw fragments only.
uint32_t launch_encode(const uint8_t *base, const FrameGeom &G, uint32_t frames, uint8_t *out, uint64_t out_stride,
                       unsigned long long *used, cudaStream_t st, const FusedPictures *fused = nullptr)
{
    const uint64_t nfrag = (uint64_t)frames * G.frags_per_frame;
    if (nfrag == 0 || nfrag >= (1ull << 31)) return HapResult_Bad_Arguments;
    DevBuf scratch(st), fsize(st), fdst(st), fidx(st), fent(st);
    bool any_compress = false;
    for (uint32_t i = 0; i < G.sections; i++) any_compress = any_compress || G.s[i].compress;
    const uint32_t write_index = any_compress && g_write_index.load() ? 1u : 0u;
    if (!scratch.alloc(any_compress ? nfrag * kFragCap : 16) || !fsize.alloc(nfrag * 4) || !fdst.alloc(nfrag * 4) || !fidx.alloc(nfrag * 4) ||
        !fent.alloc(write_index ? nfrag * kFragEntryStride : 16)) {
        cudaGetLastError();
        return HapResult_Internal_Error;
    }
    const bool write_offsets = g_write_offsets.load();
    const uint32_t plan_flags = (write_index ? kPlanWriteIndex : 0u) | (write_offsets ? kPlanWriteOffsets : 0u);
    uint8_t *entries = write_index ? fent.as<uint8_t>() : (uint8_t *)nullptr;
    if (HAPB200_FUSED_PLACE && fused && !write_offsets) {
        // The fused encoder writes the element streams into the frames itself; the plan kernel lists the raw fragments
        // for the place kernel.  sync = ticket, raw-fragment count, published sizes [nfrag], next-chunk starts [nfrag].
        DevBuf sync(st), work(st);
        const size_t sync_bytes = (2 + 2 * nfrag) * 4;
        if (!sync.alloc(sync_bytes) || !work.alloc(nfrag * 4) || cudaMemsetAsync(sync.p, 0, sync_bytes, st) != cudaSuccess) {
            cudaGetLastError();
            return HapResult_Internal_Error;
        }
        uint32_t *sy = sync.as<uint32_t>();
        const FusedPlaceArgs P{out, out_stride, sy, sy + 2, sy + 2 + nfrag};
        if (HAPB200_FUSED_WS) {
            const uint64_t resident = (uint64_t)sm_count() * (uint64_t)g_dev[t_device].ws_place_ctas_per_sm;
            HAP_KLAUNCH(kStBcEncode, hapq_ws_place_kernel, dim3((unsigned)(nfrag < resident ? nfrag : resident)), dim3(kWsThreads),
                        sizeof(WsSmem), st, fused->rgba, fused->g, const_cast<uint8_t *>(base), G, (uint32_t)nfrag, scratch.as<uint8_t>(),
                        fsize.as<uint32_t>(), entries, P);
        } else {
            const uint64_t resident = (uint64_t)sm_count() * (uint64_t)g_dev[t_device].fused_place_ctas_per_sm;
            HAP_KLAUNCH(kStBcEncode, hapq_fused_place_kernel, dim3((unsigned)(nfrag < resident ? nfrag : resident)), dim3(kEncThreads),
                        sizeof(EncodeSmem), st, fused->rgba, fused->g, const_cast<uint8_t *>(base), G, (uint32_t)nfrag, scratch.as<uint8_t>(),
                        fsize.as<uint32_t>(), entries, P);
        }
        HAP_KLAUNCH(kStPlan, hap_plan_placed_frames_kernel, dim3(frames), dim3(kPlanThreads), 0, st, G, base, fsize.as<uint32_t>(),
                    fdst.as<uint32_t>(), fidx.as<uint32_t>(), plan_flags, out, out_stride, used,
                    PlanPlaced{scratch.as<uint8_t>(), entries, work.as<uint32_t>(), sy + 1});
        const uint64_t place_grid = (uint64_t)sm_count() * 8;   // 8 CTAs of 256 threads fill an SM
        HAP_KLAUNCH(kStPlace, hap_place_listed_kernel, dim3((unsigned)(nfrag < place_grid ? nfrag : place_grid)), dim3(kPlaceThreads), 0, st,
                    G, base, fsize.as<uint32_t>(), fdst.as<uint32_t>(), work.as<uint32_t>(), sy + 1, out, out_stride);
        return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
    }
    // every CTA that can be resident at once (two per SM with the kernel's 108 KB of shared memory) strides over the fragments
    const uint64_t k5_resident = (uint64_t)sm_count() * (uint64_t)(fused ? g_dev[t_device].fused_ctas_per_sm : g_dev[t_device].k5_ctas_per_sm);
    const unsigned k5_grid = (unsigned)(nfrag < k5_resident ? nfrag : k5_resident);
    if (fused)   // (counted as block encoding: the fit is most of its work)
        HAP_KLAUNCH(kStBcEncode, hapq_fused_encode_kernel, dim3(k5_grid), dim3(kEncThreads), sizeof(EncodeSmem), st, fused->rgba, fused->g,
                    const_cast<uint8_t *>(base), G, (uint32_t)nfrag, scratch.as<uint8_t>(), fsize.as<uint32_t>(), entries);
    else
        HAP_KLAUNCH(kStSnappyEncode, snappy_encode_fragments_kernel, dim3(k5_grid), dim3(kEncThreads), sizeof(EncodeSmem), st, base, G,
                    (uint32_t)nfrag, scratch.as<uint8_t>(), fsize.as<uint32_t>(), entries);
    HAP_KLAUNCH(kStPlan, hap_plan_frames_kernel, dim3(frames), dim3(kPlanThreads), 0, st, G, base, fsize.as<uint32_t>(),
                fdst.as<uint32_t>(), fidx.as<uint32_t>(), plan_flags, out, out_stride, used);
    HAP_KLAUNCH(kStPlace, hap_place_fragments_kernel, dim3((unsigned)nfrag), dim3(kPlaceThreads), 0, st, G, base,
                scratch.as<uint8_t>(), fsize.as<uint32_t>(), fdst.as<uint32_t>(), fidx.as<uint32_t>(),
                write_index ? fent.as<uint8_t>() : (const uint8_t *)nullptr, out, out_stride);
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

// the scaled-YCoCg kinds have a chroma-refining variant (HAPB200_OPTION_CHROMA_REFINE)
template <int KIND, int SRC>
void launch_bc_encode_slice(const dim3 &grid, cudaStream_t st, const uint8_t *src, const BcGeom &g, uint8_t *dst, bool refine, const YuvSrc &yuv)
{
    constexpr bool kRefines = KIND == kBcYCoCg || KIND == kBcYCoCgPlusAlpha;
    if (kRefines && refine) HAP_KLAUNCH(kStBcEncode, (bc_encode_kernel<KIND, kRefines, SRC>), grid, dim3(kBcThreads), 0, st, src, g, dst, yuv);
    else HAP_KLAUNCH(kStBcEncode, (bc_encode_kernel<KIND, false, SRC>), grid, dim3(kBcThreads), 0, st, src, g, dst, yuv);
}

// the planar sources' kernel (bc_encode_planar_kernel), as launch_bc_encode_slice
template <int KIND, int SRC>
void launch_bc_encode_planar_slice(const dim3 &grid, cudaStream_t st, const uint8_t *luma, const BcGeom &g, uint8_t *dst, bool refine,
                                   const PlanarSrc &p)
{
    constexpr bool kRefines = KIND == kBcYCoCg || KIND == kBcYCoCgPlusAlpha;
    if (kRefines && refine) HAP_KLAUNCH(kStBcEncode, (bc_encode_planar_kernel<KIND, kRefines, SRC>), grid, dim3(kBcThreads), 0, st, luma, g, dst, p);
    else HAP_KLAUNCH(kStBcEncode, (bc_encode_planar_kernel<KIND, false, SRC>), grid, dim3(kBcThreads), 0, st, luma, g, dst, p);
}

// RGTC1 (Hap Alpha-Only) reads the alpha plane alone, so only the sample width picks its instantiation
template <int KIND>
void launch_bc_encode_planar(const dim3 &grid, cudaStream_t st, const uint8_t *luma, const BcGeom &g, uint8_t *dst, bool refine, int src,
                             const PlanarSrc &p)
{
    if constexpr (KIND == kBcRgtc1) {
        if (planar_wide(src)) launch_bc_encode_planar_slice<KIND, kSrcPlanar420x16>(grid, st, luma, g, dst, refine, p);
        else launch_bc_encode_planar_slice<KIND, kSrcPlanar420x8>(grid, st, luma, g, dst, refine, p);
    } else {
        switch (src) {
        case kSrcPlanar420x8: launch_bc_encode_planar_slice<KIND, kSrcPlanar420x8>(grid, st, luma, g, dst, refine, p); break;
        case kSrcPlanar420x16: launch_bc_encode_planar_slice<KIND, kSrcPlanar420x16>(grid, st, luma, g, dst, refine, p); break;
        case kSrcPlanar422x8: launch_bc_encode_planar_slice<KIND, kSrcPlanar422x8>(grid, st, luma, g, dst, refine, p); break;
        case kSrcPlanar422x16: launch_bc_encode_planar_slice<KIND, kSrcPlanar422x16>(grid, st, luma, g, dst, refine, p); break;
        case kSrcPlanar444x8: launch_bc_encode_planar_slice<KIND, kSrcPlanar444x8>(grid, st, luma, g, dst, refine, p); break;
        default: launch_bc_encode_planar_slice<KIND, kSrcPlanar444x16>(grid, st, luma, g, dst, refine, p); break;
        }
    }
}

// One launch per kBcFramesPerLaunch frames.  The kinds that encode colour (not RGTC1 alone, not BC7) also read NV12 / P010;
// the planar sources serve every kind but BC7.
template <int KIND>
void launch_bc_encode(uint32_t frames, cudaStream_t st, const uint8_t *rgba, const BcGeom &g, uint8_t *blocks, bool refine, int src,
                      const YuvSrc &yuv, const PlanarSrc &planar)
{
    constexpr bool kTakesYuv = KIND != kBcRgtc1 && KIND != kBcBc7;
    for (uint32_t f0 = 0; f0 < frames; f0 += kBcFramesPerLaunch) {
        const dim3 grid(bc_ctas(g.blocks_x, g.blocks_y), frames - f0 < kBcFramesPerLaunch ? frames - f0 : kBcFramesPerLaunch);
        const uint8_t *s = rgba + f0 * g.frame_bytes;
        uint8_t *dst = blocks + f0 * g.out_stride;
        if constexpr (KIND != kBcBc7) {
            if (is_planar_src(src)) {
                PlanarSrc p = planar;
                p.m.chroma += f0 * g.frame_bytes;
                p.cr += f0 * g.frame_bytes;
                if (p.alpha) p.alpha += f0 * g.frame_bytes;
                launch_bc_encode_planar<KIND>(grid, st, s, g, dst, refine, src, p);
                continue;
            }
        }
        YuvSrc y = yuv;
        if (y.chroma) y.chroma += f0 * g.frame_bytes;
        if constexpr (kTakesYuv) {
            if (src == kSrcNv12) { launch_bc_encode_slice<KIND, kSrcNv12>(grid, st, s, g, dst, refine, y); continue; }
            if (src == kSrcP010) { launch_bc_encode_slice<KIND, kSrcP010>(grid, st, s, g, dst, refine, y); continue; }
        }
        launch_bc_encode_slice<KIND, kSrcRgba8>(grid, st, s, g, dst, refine, y);
    }
}

// The PQ tables of the HDR10 converters per (device, direction, unitNits): T of the encoders (kPqIn: yuv_pq_table, 4096
// halves, 8 KiB) and P of the decoders (kPqOut: yuv_pq_out_table, kPqOutEntries codes, 62 KiB), both of include/hap_b200.h.
// Built on the host and uploaded by the first call that needs one, which waits for the copy; kept for the life of the
// process, so later calls (batches among them) find it without touching the host.  nullptr when the upload fails.
enum PqDirection : uint32_t { kPqIn = 0, kPqOut = 1 };
const uint16_t *pq_table(uint32_t unit_nits, PqDirection dir)
{
    static std::mutex mu;
    static std::map<uint32_t, uint16_t *> tables[kMaxDevices];
    std::lock_guard<std::mutex> l(mu);
    std::map<uint32_t, uint16_t *> &mine = tables[t_device];
    const uint32_t key = unit_nits << 1 | dir;
    const auto it = mine.find(key);
    if (it != mine.end()) return it->second;
    const size_t bytes = (dir == kPqOut ? kPqOutEntries : 4096) * sizeof(uint16_t);
    std::vector<uint16_t> host(bytes / sizeof(uint16_t));
    if (dir == kPqOut) yuv_pq_out_table(unit_nits, host.data());
    else yuv_pq_table(unit_nits, host.data());
    void *d = nullptr;
    cudaStream_t s = nullptr;
    bool ok = cudaMalloc(&d, bytes) == cudaSuccess && cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(d, host.data(), bytes, cudaMemcpyHostToDevice, s) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(s) == cudaSuccess;
    if (s) cudaStreamDestroy(s);
    if (!ok) {
        cudaGetLastError();
        if (d) cudaFree(d);
        return nullptr;
    }
    return mine[key] = (uint16_t *)d;
}

// The picture an encoder reads: an RGBA8 picture (kSrcRgba8), the luma and chroma planes of an NV12 / P010 picture
// (kSrcNv12 / kSrcP010, yuv_source.cuh), an RGBA16F picture (kSrcRgbaHalf), an HDR10 P010 picture (kSrcP010Pq) or a planar
// picture (kSrcPlanar*).  Rows of the luma (and alpha) plane are `pitch` bytes apart; rows of the NV12 / P010 chroma plane
// too, rows of the planar chroma planes chroma_pitch bytes apart.
struct PictureSrc {
    int kind;                 // BcSource
    const void *pixels;       // the RGBA8 / RGBA16F picture, or the luma plane
    const void *chroma;       // the interleaved CbCr plane, or the planar Cb plane
    unsigned color_space;     // HapB200YUVColorSpace
    unsigned unit_nits = 0;   // kSrcP010Pq: the luminance of 1.0
    // kSrcPlanar*: the Cr and alpha planes (alpha nullptr: A = 255), the chroma planes' pitch and the sample depth.
    // alpha_only (Hap Alpha-Only): only the alpha plane is read, and pixels, chroma and cr point at it too.
    const void *cr = nullptr, *alpha = nullptr;
    uint64_t chroma_pitch = 0;
    unsigned bit_depth = 0;
    bool alpha_only = false;
    uint64_t sample_bytes() const   // per pixel of a luma / RGBA row
    {
        if (is_planar_src(kind)) return planar_wide(kind) ? 2 : 1;
        return kind == kSrcRgba8 ? 4 : kind == kSrcRgbaHalf ? 8 : kind == kSrcNv12 ? 1 : 2;
    }
    uint32_t planes() const { return kind == kSrcRgba8 || kind == kSrcRgbaHalf ? 1 : is_planar_src(kind) ? 4 : 2; }
    bool is_planar() const { return is_planar_src(kind); }
    YuvSrc yuv() const
    {
        return kind == kSrcNv12 || kind == kSrcP010 ? yuv_src(kind - kSrcNv12, color_space, (const uint8_t *)chroma) : YuvSrc();
    }
    PlanarSrc planar() const
    {
        return is_planar_src(kind) ? planar_src_args(bit_depth, color_space, (const uint8_t *)chroma, (const uint8_t *)cr,
                                                     (const uint8_t *)alpha, (uint32_t)chroma_pitch)
                                   : PlanarSrc();
    }
    // the chroma planes' samples per row and rows of a width x height picture
    uint32_t chroma_width(uint32_t width) const { return planar_subsampling(kind) == HapB200Chroma_444 ? width : width / 2; }
    uint32_t chroma_height(uint32_t height) const { return planar_subsampling(kind) == HapB200Chroma_420 ? height / 2 : height; }
};
PictureSrc rgba_picture(const void *rgba) { return {kSrcRgba8, rgba, nullptr, 0}; }
PictureSrc rgba_half_picture(const void *rgba) { return {kSrcRgbaHalf, rgba, nullptr, 0}; }

// The BC6H kind (Hap HDR) of launch_block_encode: RGBA16F pictures (kSrcRgbaHalf) or HDR10 P010 ones (kSrcP010Pq, converted
// through pq) -> blocks, SF16 when is_signed, else UF16.  One launch per kBcFramesPerLaunch frames.
void launch_bc6h_slices(uint32_t frames, cudaStream_t st, const uint8_t *rgba, const BcGeom &g, uint8_t *blocks, uint32_t is_signed, int src,
                        const YuvPqSrc &pq)
{
    for (uint32_t f0 = 0; f0 < frames; f0 += kBcFramesPerLaunch) {
        const dim3 grid(bc_ctas(g.blocks_x, g.blocks_y), frames - f0 < kBcFramesPerLaunch ? frames - f0 : kBcFramesPerLaunch);
        if (src == kSrcP010Pq) {
            YuvPqSrc y = pq;
            y.m.chroma += f0 * g.frame_bytes;
            HAP_KLAUNCH(kStBcEncode, bc6h_encode_kernel<kSrcP010Pq>, grid, dim3(kBcThreads), 0, st, rgba + f0 * g.frame_bytes, g,
                        blocks + f0 * g.out_stride, is_signed, y);
        } else {
            HAP_KLAUNCH(kStBcEncode, bc6h_encode_kernel<>, grid, dim3(kBcThreads), 0, st, rgba + f0 * g.frame_bytes, g, blocks + f0 * g.out_stride,
                        is_signed, pq);
        }
    }
}

// The RGBA8 scratch of BC7 from a Y'CbCr picture holds at most this many bytes, or one frame when a frame is larger
constexpr uint64_t kBc7ScratchBytes = 256ull << 20;

// The BC7 kind of launch_block_encode from NV12 / P010 or planar pictures (g: their geometry, out_stride the blocks' frame
// stride), in two passes per slice of frames: bc_source_to_rgba8_kernel converts the slice into a tight RGBA8 picture in
// scratch, then the RGBA8 BC7 kernel encodes it, so no BC7 search is instantiated per source (bc_encode.cuh).  Whole frames
// per slice, as many as kBc7ScratchBytes holds (at least one); stream order lets each slice reuse the scratch.
uint32_t launch_bc7_from_yuv(uint32_t frames, cudaStream_t st, const uint8_t *luma, const BcGeom &g, uint8_t *blocks, int src,
                             const YuvSrc &yuv, const PlanarSrc &planar)
{
    const uint64_t row = 16ull * g.blocks_x, frame_rgba = row * 4 * g.blocks_y;   // (the entry points: 4 * width < 2^32)
    uint64_t slice = kBc7ScratchBytes / frame_rgba;
    slice = slice < 1 ? 1 : slice > kBcFramesPerLaunch ? kBcFramesPerLaunch : slice;
    if (slice > frames) slice = frames;
    DevBuf rgba(st);
    if (!rgba.alloc(slice * frame_rgba)) { cudaGetLastError(); return HapResult_Internal_Error; }
    BcGeom cg = g;   // the source read, the RGBA8 picture written
    cg.out_stride = frame_rgba;
    const BcGeom rg = bc_encode_geom(4 * g.blocks_x, 4 * g.blocks_y, (uint32_t)row, frame_rgba, g.out_stride, 0);
    for (uint32_t f0 = 0; f0 < frames; f0 += (uint32_t)slice) {
        const uint32_t n = frames - f0 < slice ? frames - f0 : (uint32_t)slice;
        const dim3 grid(bc_ctas(g.blocks_x, g.blocks_y), n);
        const uint8_t *s = luma + f0 * g.frame_bytes;
        YuvSrc y = yuv;
        PlanarSrc p = planar;
        if (y.chroma) y.chroma += f0 * g.frame_bytes;
        if (is_planar_src(src)) {
            p.m.chroma += f0 * g.frame_bytes;
            p.cr += f0 * g.frame_bytes;
            if (p.alpha) p.alpha += f0 * g.frame_bytes;
        }
        uint8_t *o = rgba.as<uint8_t>();
        switch (src) {
        case kSrcNv12: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcNv12>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        case kSrcP010: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcP010>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        case kSrcPlanar420x8: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcPlanar420x8>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        case kSrcPlanar420x16: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcPlanar420x16>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        case kSrcPlanar422x8: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcPlanar422x8>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        case kSrcPlanar422x16: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcPlanar422x16>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        case kSrcPlanar444x8: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcPlanar444x8>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        case kSrcPlanar444x16: HAP_KLAUNCH(kStBcEncode, bc_source_to_rgba8_kernel<kSrcPlanar444x16>, grid, dim3(kBcThreads), 0, st, s, cg, o, y, p); break;
        default: return HapResult_Bad_Arguments;
        }
        launch_bc_encode<kBcBc7>(n, st, o, rg, blocks + f0 * g.out_stride, false, kSrcRgba8, YuvSrc(), PlanarSrc());
    }
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

// The pictures p (frame f's planes frame_stride apart, luma / RGBA rows row_bytes apart) -> blocks of ci, frame f's at
// blocks + f*blocks_stride, its second texture (Hap Q Alpha) second_offset behind them.  BC6H signedness: ci.fmt[0].
uint32_t launch_block_encode(const CodecInfo &ci, const PictureSrc &p, uint32_t frames, uint64_t frame_stride, uint32_t width,
                             uint32_t height, uint64_t row_bytes, uint8_t *blocks, uint64_t blocks_stride, uint64_t second_offset,
                             cudaStream_t st)
{
    const BcGeom g = bc_encode_geom(width, height, (uint32_t)row_bytes, frame_stride, blocks_stride, second_offset);   // (rgba_geometry_ok: row_bytes < 2^32)
    const uint8_t *rgba = (const uint8_t *)p.pixels;
    const int src = p.kind;
    const YuvSrc yuv = p.yuv();
    const PlanarSrc planar = p.planar();
    const bool refine = g_chroma_refine.load() != 0;
    if (ci.bc_kind == kBcBc7 && (src == kSrcNv12 || src == kSrcP010 || is_planar_src(src)))
        return launch_bc7_from_yuv(frames, st, rgba, g, blocks, src, yuv, planar);
    if (src != kSrcRgba8 && ci.bc_kind == kBcBc7) return HapResult_Bad_Arguments;
    if ((src == kSrcNv12 || src == kSrcP010) && ci.bc_kind == kBcRgtc1) return HapResult_Bad_Arguments;
    switch (ci.bc_kind) {
    case kBcDxt1: launch_bc_encode<kBcDxt1>(frames, st, rgba, g, blocks, refine, src, yuv, planar); break;
    case kBcDxt5: launch_bc_encode<kBcDxt5>(frames, st, rgba, g, blocks, refine, src, yuv, planar); break;
    case kBcYCoCg: launch_bc_encode<kBcYCoCg>(frames, st, rgba, g, blocks, refine, src, yuv, planar); break;
    case kBcRgtc1: launch_bc_encode<kBcRgtc1>(frames, st, rgba, g, blocks, refine, src, yuv, planar); break;
    case kBcYCoCgPlusAlpha: launch_bc_encode<kBcYCoCgPlusAlpha>(frames, st, rgba, g, blocks, refine, src, yuv, planar); break;
    case kBcBc7: launch_bc_encode<kBcBc7>(frames, st, rgba, g, blocks, refine, src, yuv, planar); break;
    case kBcBc6h: {
        YuvPqSrc pq = YuvPqSrc();
        if (src == kSrcP010Pq) {
            const uint16_t *table = pq_table(p.unit_nits, kPqIn);
            if (!table) return HapResult_Internal_Error;
            pq = yuv_pq_src(p.color_space, (const uint8_t *)p.chroma, table);
        }
        launch_bc6h_slices(frames, st, rgba, g, blocks, ci.fmt[0] == HapFmt_RGB_BPTC_SFLOAT ? 1u : 0u, src, pq);
        break;
    }
    default: return HapResult_Bad_Arguments;
    }
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

// The tail of the picture batch encoders: encode_blocks(textures, stride) fills the textures of every frame into device
// scratch (frame f at textures + f*stride, texture 1 at align16(t[0]) inside it), then the frames are laid out from them at
// out + f*out_stride, lengths in used[f].  fused: Hap Q pictures the fused encoder may take (hapq_fused.cuh); it does when the
// texture's chunks pass fused_hapq_geometry, and encode_blocks is not called then.
template <class EncodeBlocks>
uint32_t encode_frames_from_blocks(uint32_t frames, uint32_t count, const uint64_t t[2], const uint32_t fmt[2], unsigned compressor,
                                   unsigned chunk_count, uint8_t *out, uint64_t out_stride, unsigned long long *used, cudaStream_t st,
                                   EncodeBlocks &&encode_blocks, const FusedPictures *fused = nullptr)
{
    const uint64_t stride = align16(t[0]) + align16(t[1]);
    DevBuf tex(st);
    if (!tex.alloc(stride * frames + 16)) { cudaGetLastError(); return (uint32_t)HapResult_Internal_Error; }
    TextureArgs ta[2] = {{t[0], fmt[0], compressor, chunk_count}, {t[1], fmt[1], compressor, chunk_count}};
    FrameGeom G;
    uint32_t r = build_frame_geom(count, ta, G);
    if (r != HapResult_No_Error) return r;
    for (unsigned i = 0; i < count; i++) {
        G.s[i].in_offset = i ? align16(t[0]) : 0;
        G.s[i].in_stride = stride;
    }
    if (fused && !fused_hapq_geometry(G)) fused = nullptr;
    if (!fused) {
        r = encode_blocks(tex.as<uint8_t>(), stride);
        if (r != HapResult_No_Error) return r;
    }
    return launch_encode(tex.as<uint8_t>(), G, frames, out, out_stride, used, st, fused);
}

// The picture a decoder writes: an RGBA8 picture (kDstRgba8), an RGBA16F picture (kDstRgbaHalf), the luma and chroma planes of
// an NV12 / P010 picture (kDstNv12 / kDstP010, yuv_sink.cuh) or of an HDR10 P010 picture (kDstP010Pq, BT.2020 PQ), or a planar
// picture (kDstPlanar*, planar_sink.cuh: one per subsampling and sample width, x8 bytes and x16 16-bit words).  The NV12 / P010
// chroma plane's rows are as many bytes apart as luma's; rows of the planar chroma planes are chroma_pitch bytes apart, rows of
// the alpha plane `pitch` bytes apart, as luma's.
enum DstKind {
    kDstRgba8, kDstRgbaHalf, kDstNv12, kDstP010, kDstP010Pq,
    kDstPlanar420x8, kDstPlanar420x16, kDstPlanar422x8, kDstPlanar422x16, kDstPlanar444x8, kDstPlanar444x16
};
constexpr bool is_planar_dst(int kind) { return kind >= kDstPlanar420x8 && kind <= kDstPlanar444x16; }
constexpr int planar_dst(unsigned subsampling, bool wide) { return kDstPlanar420x8 + 2 * (int)subsampling + (wide ? 1 : 0); }
constexpr int planar_dst_subsampling(int kind) { return (kind - kDstPlanar420x8) / 2; }
constexpr bool planar_dst_wide(int kind) { return (kind - kDstPlanar420x8) % 2 == 1; }
struct PictureDst {
    int kind;                 // DstKind
    void *pixels;             // the RGBA8 / RGBA16F picture, or the luma plane
    void *chroma;             // the interleaved CbCr plane, or the planar Cb plane
    unsigned color_space;     // HapB200YUVColorSpace
    unsigned unit_nits = 0;   // kDstP010Pq: the luminance of 1.0
    // kDstPlanar*: the Cr and alpha planes (alpha nullptr: no alpha is written), the chroma planes' pitch and the sample depth.
    // alpha_only (Hap Alpha-Only): only the alpha plane is written, and pixels, chroma and cr point at it too.
    void *cr = nullptr, *alpha = nullptr;
    uint64_t chroma_pitch = 0;
    unsigned bit_depth = 0;
    bool alpha_only = false;
    uint64_t sample_bytes() const   // per pixel of a luma / RGBA row
    {
        if (is_planar_dst(kind)) return planar_dst_wide(kind) ? 2 : 1;
        return kind == kDstRgba8 ? 4 : kind == kDstRgbaHalf ? 8 : kind == kDstNv12 ? 1 : 2;
    }
    uint32_t planes() const { return kind == kDstRgba8 || kind == kDstRgbaHalf ? 1 : is_planar_dst(kind) ? 4 : 2; }
    bool is_planar() const { return is_planar_dst(kind); }
    bool hdr() const { return kind == kDstRgbaHalf || kind == kDstP010Pq; }   // the sinks of Hap HDR (BC6H) frames
    // the chroma planes' samples per row and rows of a width x height picture
    uint32_t chroma_width(uint32_t width) const { return planar_dst_subsampling(kind) == HapB200Chroma_444 ? width : width / 2; }
    uint32_t chroma_height(uint32_t height) const { return planar_dst_subsampling(kind) == HapB200Chroma_420 ? height / 2 : height; }
};

// The planar sink's launches (planar_sink.cuh): Hap Alpha-Only (kBcRgtc1) writes its alpha plane alone
// (bc_decode_planar_alpha_kernel), the colour kinds every plane (bc_decode_planar_kernel).
template <int KIND>
void launch_planar_decode_slice(int dst_kind, const dim3 &grid, cudaStream_t st, const uint8_t *blocks, const PlanarOut &p, uint8_t *luma,
                                const uint32_t *results)
{
    if constexpr (KIND == kBcRgtc1) {
        if (planar_dst_wide(dst_kind)) HAP_KLAUNCH(kStBcDecode, bc_decode_planar_alpha_kernel<true>, grid, dim3(kBcThreads), 0, st, blocks, p, results);
        else HAP_KLAUNCH(kStBcDecode, bc_decode_planar_alpha_kernel<false>, grid, dim3(kBcThreads), 0, st, blocks, p, results);
    } else {
#define HAPB200_PLANAR_DECODE(SUB, WIDE) \
    HAP_KLAUNCH(kStBcDecode, (bc_decode_planar_kernel<KIND, SUB, WIDE>), grid, dim3(kBcThreads), 0, st, blocks, p, luma, results)
        switch (dst_kind) {
        case kDstPlanar420x8: HAPB200_PLANAR_DECODE(HapB200Chroma_420, false); break;
        case kDstPlanar420x16: HAPB200_PLANAR_DECODE(HapB200Chroma_420, true); break;
        case kDstPlanar422x8: HAPB200_PLANAR_DECODE(HapB200Chroma_422, false); break;
        case kDstPlanar422x16: HAPB200_PLANAR_DECODE(HapB200Chroma_422, true); break;
        case kDstPlanar444x8: HAPB200_PLANAR_DECODE(HapB200Chroma_444, false); break;
        default: HAPB200_PLANAR_DECODE(HapB200Chroma_444, true); break;
        }
#undef HAPB200_PLANAR_DECODE
    }
}

// launch_block_decode for the planar pictures (its arguments; d.alpha_only exactly when ci is Hap Alpha-Only).  Hap Q Alpha
// merges its alpha texture, second_offset behind the blocks, when d has an alpha plane.  4:4:4 and Hap Alpha-Only run one
// thread per block, 4:2:0 and 4:2:2 the warp spans of the NV12 sink.
uint32_t launch_planar_decode(const CodecInfo &ci, const PictureDst &d, const uint8_t *blocks, uint64_t second_offset, uint32_t frames,
                              uint64_t blocks_stride, uint32_t width, uint32_t height, uint64_t frame_stride, uint64_t pitch,
                              const uint32_t *frame_results, cudaStream_t st)
{
    if ((ci.bc_kind == kBcRgtc1) != d.alpha_only || ci.bc_kind == kBcBc6h) return HapResult_Bad_Arguments;
    PlanarOut p;
    p.g = yuv_out_geom(width, height, (uint32_t)pitch, blocks_stride, frame_stride, planar_out_coeffs(d.bit_depth, d.color_space));
    p.chroma_pitch = (uint32_t)d.chroma_pitch;   // (planar_geometry_ok: both pitches < 2^32)
    p.merge_alpha = ci.textures == 2 && d.alpha ? 1u : 0u;
    p.second_offset = second_offset;
    const bool per_block = d.alpha_only || planar_dst_subsampling(d.kind) == HapB200Chroma_444;
    const unsigned ctas = per_block ? bc_ctas(p.g.blocks_x, p.g.blocks_y) : (unsigned)yuv_out_ctas(p.g);
    for (uint32_t f0 = 0; f0 < frames; f0 += kBcFramesPerLaunch) {
        const dim3 grid(ctas, frames - f0 < kBcFramesPerLaunch ? frames - f0 : kBcFramesPerLaunch);
        const uint64_t o = f0 * frame_stride;
        const uint8_t *b = blocks + f0 * blocks_stride;
        PlanarOut s = p;
        s.cb = (uint8_t *)d.chroma + o;
        s.cr = (uint8_t *)d.cr + o;
        s.alpha = d.alpha ? (uint8_t *)d.alpha + o : nullptr;
        uint8_t *luma = (uint8_t *)d.pixels + o;
        const uint32_t *res = frame_results ? frame_results + f0 : nullptr;
        switch (ci.bc_kind) {
        case kBcDxt1: launch_planar_decode_slice<kBcDxt1>(d.kind, grid, st, b, s, luma, res); break;
        case kBcDxt5: launch_planar_decode_slice<kBcDxt5>(d.kind, grid, st, b, s, luma, res); break;
        case kBcRgtc1: launch_planar_decode_slice<kBcRgtc1>(d.kind, grid, st, b, s, luma, res); break;
        case kBcYCoCg:
        case kBcYCoCgPlusAlpha: launch_planar_decode_slice<kBcYCoCg>(d.kind, grid, st, b, s, luma, res); break;
        case kBcBc7: launch_planar_decode_slice<kBcBc7>(d.kind, grid, st, b, s, luma, res); break;
        default: return HapResult_Internal_Error;
        }
    }
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

// The launches of launch_block_decode for the BC kinds: to RGBA8 (bc_decode_kernel; Hap Q Alpha merges its alpha texture) or
// to NV12 / P010 (bc_decode_yuv_kernel; Hap Q Alpha decodes its YCoCg texture only, alpha is dropped).
template <int KIND>
void launch_bc_decode_slice(int dst_kind, const dim3 &grid, cudaStream_t st, const uint8_t *blocks, const uint8_t *alpha,
                            const BcDecodeGeom &g, const YuvOutGeom &yg, uint8_t *pixels, uint8_t *chroma, const uint32_t *results)
{
    if (dst_kind == kDstRgba8)
        HAP_KLAUNCH(kStBcDecode, bc_decode_kernel<KIND>, grid, dim3(kBcThreads), 0, st, blocks, alpha, g, pixels, results);
    else if (dst_kind == kDstP010)
        HAP_KLAUNCH(kStBcDecode, (bc_decode_yuv_kernel<KIND, HapB200YUV_P010>), grid, dim3(kBcThreads), 0, st, blocks, yg, pixels, chroma, results);
    else
        HAP_KLAUNCH(kStBcDecode, (bc_decode_yuv_kernel<KIND, HapB200YUV_NV12>), grid, dim3(kBcThreads), 0, st, blocks, yg, pixels, chroma, results);
}

// Blocks of ci (frame f's at blocks + f*blocks_stride, its second texture, Hap Q Alpha's alpha, second_offset behind them) ->
// the pictures d (frame f's planes at d's + f*frame_stride, rows `pitch` apart).  The kernel follows ci.bc_kind and the sink:
// launch_bc_decode_slice for the BC kinds, bc6h_decode_kernel (RGBA16F) or bc6h_decode_yuv_kernel (HDR10 P010) for BC6H,
// launch_planar_decode for the planar pictures.
// frame_results (optional): HapResult per frame; a frame that failed is written as zeros.  BC6H signedness per frame from
// frame_formats, or from ci.fmt[0] for every frame without them.  One launch per kBcFramesPerLaunch frames, counted as bc_decode.
uint32_t launch_block_decode(const CodecInfo &ci, const PictureDst &d, const uint8_t *blocks, uint64_t second_offset, uint32_t frames,
                             uint64_t blocks_stride, uint32_t width, uint32_t height, uint64_t frame_stride, uint64_t pitch,
                             const uint32_t *frame_results, const uint32_t *frame_formats, cudaStream_t st)
{
    if (d.is_planar())
        return launch_planar_decode(ci, d, blocks, second_offset, frames, blocks_stride, width, height, frame_stride, pitch, frame_results, st);
    const bool two_planes = d.planes() == 2;
    const uint16_t *table = nullptr;
    if (d.kind == kDstP010Pq && !(table = pq_table(d.unit_nits, kPqOut))) return HapResult_Internal_Error;
    BcDecodeGeom g = BcDecodeGeom();
    YuvOutGeom yg = YuvOutGeom();
    if (!two_planes) g = bc_decode_geom(width, height, (uint32_t)pitch, ci.textures == 2, blocks_stride, blocks_stride, frame_stride);
    else if (d.kind == kDstP010Pq) yg = yuv_out_geom(width, height, (uint32_t)pitch, blocks_stride, frame_stride, yuv_pq_out_coeffs(d.color_space));
    else yg = yuv_out_geom(width, height, (uint32_t)pitch, blocks_stride, frame_stride, d.kind == kDstP010 ? HapB200YUV_P010 : HapB200YUV_NV12, d.color_space);
    const unsigned ctas = two_planes ? (unsigned)yuv_out_ctas(yg) : bc_ctas(g.blocks_x, g.blocks_y);   // (pitch < 2^32)
    const uint32_t is_signed = ci.fmt[0] == HapFmt_RGB_BPTC_SFLOAT ? 1u : 0u;
    for (uint32_t f0 = 0; f0 < frames; f0 += kBcFramesPerLaunch) {
        const dim3 grid(ctas, frames - f0 < kBcFramesPerLaunch ? frames - f0 : kBcFramesPerLaunch);
        const uint8_t *b = blocks + f0 * blocks_stride;
        uint8_t *pixels = (uint8_t *)d.pixels + f0 * frame_stride, *chroma = two_planes ? (uint8_t *)d.chroma + f0 * frame_stride : nullptr;
        const uint32_t *res = frame_results ? frame_results + f0 : nullptr, *fmts = frame_formats ? frame_formats + f0 : nullptr;
        switch (ci.bc_kind) {
        case kBcDxt1: launch_bc_decode_slice<kBcDxt1>(d.kind, grid, st, b, b + second_offset, g, yg, pixels, chroma, res); break;
        case kBcDxt5: launch_bc_decode_slice<kBcDxt5>(d.kind, grid, st, b, b + second_offset, g, yg, pixels, chroma, res); break;
        case kBcRgtc1: launch_bc_decode_slice<kBcRgtc1>(d.kind, grid, st, b, b + second_offset, g, yg, pixels, chroma, res); break;
        case kBcYCoCg:
        case kBcYCoCgPlusAlpha: launch_bc_decode_slice<kBcYCoCg>(d.kind, grid, st, b, b + second_offset, g, yg, pixels, chroma, res); break;
        case kBcBc7: launch_bc_decode_slice<kBcBc7>(d.kind, grid, st, b, b + second_offset, g, yg, pixels, chroma, res); break;
        case kBcBc6h:
            if (two_planes)
                HAP_KLAUNCH(kStBcDecode, bc6h_decode_yuv_kernel, grid, dim3(kBcThreads), 0, st, b, yg, pixels, chroma, res, fmts, is_signed, table);
            else
                HAP_KLAUNCH(kStBcDecode, bc6h_decode_kernel, grid, dim3(kBcThreads), 0, st, b, g, pixels, res, fmts, is_signed);
            break;
        default: return HapResult_Internal_Error;
        }
    }
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

// The decode of a list of chunk jobs (a device array): first pass (windows -> on-the-fly index for chunks without one -> execute) and the repair
// pass for chunks whose embedded index did not describe their stream (decoded again as if they had none).  Batch calls queue
// both passes (the second finds nothing to do on honest frames); HapDecode, which reads the statuses on the host anyway, only
// launches the repair pass when a chunk asks for it.
struct DecodePasses {
    DevBuf wins, entries, done, ctl;
    ChunkJob *jobs = nullptr;
    uint32_t njobs = 0, win_cap = 0, entry_slots = 0;
    cudaStream_t st;
    explicit DecodePasses(cudaStream_t s) : wins(s), entries(s), done(s), ctl(s), st(s) {}

    // in_bound / out_bound: upper bounds of the jobs' total compressed / decoded bytes (they size the window list; a list
    // that turns out too short makes the affected chunks report Internal_Error, never overruns)
    uint32_t first(ChunkJob *j, uint32_t n, uint64_t in_bound, uint64_t out_bound)
    {
        jobs = j; njobs = n;
        // windows: up to kIdxParts per 16 KiB of stream from the index kernel (twice: a chunk may be indexed again by the repair
        // pass), one per fragment of an indexed chunk, one per 64 KiB of a verbatim chunk
        const uint64_t slots64 = 2 * (in_bound / kIdxWin + njobs) + 16;
        const uint64_t cap64 = kIdxParts * slots64 + out_bound / kIndexFragBytes + 2ull * njobs + 16;
        if (cap64 >= (1ull << 31)) return HapResult_Bad_Arguments;
        win_cap = (uint32_t)cap64; entry_slots = (uint32_t)slots64;
        if (!wins.alloc((size_t)win_cap * sizeof(DecWin)) || !entries.alloc((size_t)entry_slots * kIdxThreads) || !done.alloc((size_t)win_cap * 4) ||
            !ctl.alloc(sizeof(DecodeCtl) + 16)) {
            cudaGetLastError();
            return HapResult_Internal_Error;
        }
        if (cudaMemsetAsync(ctl.p, 0, sizeof(DecodeCtl) + 16, st) != cudaSuccess || cudaMemsetAsync(done.p, 0, (size_t)win_cap * 4, st) != cudaSuccess) {
            cudaGetLastError();
            return HapResult_Internal_Error;
        }
        DecodeCtl *c = ctl.as<DecodeCtl>();
        const unsigned ex_grid = (unsigned)sm_count() * (unsigned)HAPB200_EX_MIN_BLOCKS;
        HAP_KLAUNCH(kStWindows, hap_build_windows_kernel, dim3((njobs + 127) / 128), dim3(128), 0, st, jobs, njobs, (uint32_t)g_use_index.load(),
                    wins.as<DecWin>(), win_cap, c);
        HAP_KLAUNCH(kStSnappyIndex, snappy_index_kernel, dim3(njobs), dim3(kIdxThreads), sizeof(IndexSmem), st, jobs, (int)njobs, 0u,
                    wins.as<DecWin>(), win_cap, entries.as<uint8_t>(), entry_slots, c);
#if HAPB200_EX_UNIT_KERNEL
        // the fragments of embedded indexes first (without the index there are none); the execute kernel takes the rest
        if (g_use_index.load())
            HAP_KLAUNCH(kStSnappyDecode, snappy_execute_units_kernel, dim3((unsigned)sm_count() * (unsigned)units_ctas_per_sm()), dim3(kUxThreads),
                        sizeof(UnitSmem), st, jobs, njobs, wins.as<DecWin>(), c, done.as<uint32_t>());
#endif
        HAP_KLAUNCH(kStSnappyDecode, snappy_execute_kernel, dim3(ex_grid), dim3(kExThreads), sizeof(ExecSmem), st, jobs, njobs, 0u, wins.as<DecWin>(), c,
                    done.as<uint32_t>());
        return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
    }

    // chunks whose embedded index did not describe their stream: decode them again as if they had none
    uint32_t repair()
    {
        DecodeCtl *c = ctl.as<DecodeCtl>();
        uint32_t *any_left = reinterpret_cast<uint32_t *>(ctl.as<uint8_t>() + sizeof(DecodeCtl));
        const unsigned ex_grid = (unsigned)sm_count() * (unsigned)HAPB200_EX_MIN_BLOCKS;
        HAP_KLAUNCH(kStWindows, hap_requeue_mismatched_kernel, dim3((njobs + 127) / 128), dim3(128), 0, st, jobs, njobs, any_left);
        HAP_KLAUNCH(kStSnappyIndex, snappy_index_kernel, dim3(njobs), dim3(kIdxThreads), sizeof(IndexSmem), st, jobs, (int)njobs, 1u,
                    wins.as<DecWin>(), win_cap, entries.as<uint8_t>(), entry_slots, c);
        HAP_KLAUNCH(kStSnappyDecode, snappy_execute_kernel, dim3(ex_grid), dim3(kExThreads), sizeof(ExecSmem), st, jobs, njobs, 1u, wins.as<DecWin>(),
                    c, done.as<uint32_t>());
        return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
    }
};

uint32_t launch_decode_jobs(ChunkJob *jobs, uint32_t njobs, uint64_t in_bound, uint64_t out_bound, cudaStream_t st, bool may_have_index = true)
{
    DecodePasses P(st);
    uint32_t r = P.first(jobs, njobs, in_bound, out_bound);
    if (r == HapResult_No_Error && g_use_index.load() && may_have_index) r = P.repair();
    return r;
}

// device frames -> texture `index` of each; jobs scratch is allocated here
uint32_t launch_decode_batch(const uint8_t *in, uint32_t frames, uint64_t in_stride, const unsigned long long *in_bytes,
                             uint32_t index, uint32_t max_chunks, uint8_t *out, uint64_t out_stride, uint64_t out_capacity,
                             unsigned long long *used, uint32_t *formats, uint32_t *results, cudaStream_t st)
{
    const uint64_t njobs = (uint64_t)frames * max_chunks;
    if (njobs == 0 || njobs >= (1ull << 31)) return HapResult_Bad_Arguments;
    DevBuf jobs(st), whole(st);
    if (!jobs.alloc(njobs * sizeof(ChunkJob)) || !whole.alloc((size_t)frames * 4)) { cudaGetLastError(); return HapResult_Internal_Error; }
    HAP_KLAUNCH(kStParse, hap_parse_frames_kernel, dim3((frames + 127) / 128), dim3(128), 0, st, in, in_stride, in_bytes, frames, index,
                max_chunks, out, out_stride, out_capacity, jobs.as<ChunkJob>(), used, formats, results, whole.as<uint32_t>());
    uint32_t r = launch_decode_jobs(jobs.as<ChunkJob>(), (uint32_t)njobs, (uint64_t)frames * in_stride, (uint64_t)frames * out_capacity, st);
    if (r != HapResult_No_Error) return r;
    HAP_KLAUNCH(kStCollect, hap_collect_status_kernel, dim3((frames + 127) / 128), dim3(128), 0, st, jobs.as<ChunkJob>(), frames,
                max_chunks, whole.as<uint32_t>(), results, used);
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

// host-side view of a frame whose bytes may live on the device.  Header walks read a few hundred bytes at data-dependent
// places (section headers, the Decode Instructions tables, five bytes at the head of every chunk, the trailing index header), so
// a device frame is mirrored LAZILY: `p` points at a zero-page-backed image of the whole frame and need(q, len) fetches the
// 4 KiB pages under [q, q+len) that are not there yet.  A 4K Hap Q frame costs ~10 small copies instead of 5 MB.  It is the
// reader the header walks of hap_wire.h take.
struct HeaderView {
    static constexpr uint64_t kPage = 4096;
    uint8_t *mirror = nullptr;
    const uint8_t *dev = nullptr;
    const uint8_t *p = nullptr;
    uint64_t bytes = 0;
    std::vector<bool> have;
    bool ok = true;
    HeaderView(const void *frame, unsigned long n) : bytes(n)
    {
        if (!is_device(frame)) { p = (const uint8_t *)frame; return; }
        dev = (const uint8_t *)frame;
        mirror = (uint8_t *)calloc(n ? n : 1, 1);     // untouched pages stay uncommitted
        if (!mirror) { ok = false; return; }
        p = mirror;
        have.assign((size_t)((n + kPage - 1) / kPage), false);
        need(p, kPage);
    }
    ~HeaderView() { free(mirror); }
    HeaderView(const HeaderView &) = delete;
    HeaderView &operator=(const HeaderView &) = delete;
    // make [q, q+len) of the frame readable through p (clamped to the frame); false after a failed copy
    bool need(const uint8_t *q, uint64_t len)
    {
        const uint64_t off = (uint64_t)(q - p);
        if (!dev || !ok || off >= bytes || len == 0) return ok;
        if (len > bytes - off) len = bytes - off;
        uint64_t a = off / kPage;
        const uint64_t b = (off + len - 1) / kPage;
        while (a <= b) {
            if (have[(size_t)a]) { a++; continue; }
            uint64_t e = a;
            while (e <= b && !have[(size_t)e]) have[(size_t)e++] = true;
            const uint64_t lo = a * kPage, hi = e * kPage < bytes ? e * kPage : bytes;
            if (cudaMemcpy(mirror + lo, dev + lo, hi - lo, cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); ok = false; return false; }
            a = e;
        }
        return true;
    }
};

struct WorkState {
    std::atomic<unsigned> claimed{0};
};
void work_function(void *p, unsigned int)
{
    // every chunk was submitted to the GPU before the callback ran (hap.h contract: the callee calls
    // this once per chunk, from any threads, and returns when all calls returned)
    reinterpret_cast<WorkState *>(p)->claimed.fetch_add(1, std::memory_order_relaxed);
}

// ---- the picture encoders and decoders behind the picture entry points ---------------------------------------------------

// width x height NV12 (bpp 1) / P010 (bpp 2) planes with one pitch: the chroma plane's rows hold as many bytes as luma's.
// aligned: the batch entry points' rules besides (16-byte aligned pitch, planes and frame stride).
bool yuv_geometry_ok(const void *luma, const void *chroma, unsigned width, unsigned height, unsigned long pitch, unsigned long frameStride,
                     bool aligned, unsigned long bpp)
{
    return chroma && rgba_geometry_ok(luma, width, height, pitch, frameStride, aligned, bpp) && (!aligned || (uintptr_t)chroma % 16 == 0);
}

// A planar picture's four planes (PictureSrc read by the encoders, PictureDst written by the decoders): luma (and alpha) as
// rgba_geometry_ok with `pitch`; Cb and Cr of p.chroma_width(width) samples per row, rows p.chroma_pitch apart.  Alpha-only
// pictures are checked as their alpha plane.
template <class Picture>
bool planar_geometry_ok(const Picture &p, unsigned width, unsigned height, unsigned long pitch, unsigned long frameStride, bool aligned)
{
    if (!rgba_geometry_ok(p.pixels, width, height, pitch, frameStride, aligned, p.sample_bytes())) return false;
    if (p.alpha_only) return true;
    if (!p.chroma || !p.cr || p.chroma_pitch < p.sample_bytes() * p.chroma_width(width) || p.chroma_pitch > HAPB200_MAX_ROW_BYTES) return false;
    return !aligned || (((uintptr_t)p.chroma | (uintptr_t)p.cr | (uintptr_t)p.alpha | p.chroma_pitch) % 16 == 0);
}

bool picture_geometry_ok(const PictureSrc &p, unsigned width, unsigned height, unsigned long pitch, unsigned long frameStride, bool aligned)
{
    if (is_planar_src(p.kind)) return planar_geometry_ok(p, width, height, pitch, frameStride, aligned);
    if (p.planes() == 1) return rgba_geometry_ok(p.pixels, width, height, pitch, frameStride, aligned, p.sample_bytes());
    return yuv_geometry_ok(p.pixels, p.chroma, width, height, pitch, frameStride, aligned, p.sample_bytes());
}

bool picture_geometry_ok(const PictureDst &d, unsigned width, unsigned height, unsigned long pitch, unsigned long frameStride, bool aligned)
{
    if (d.is_planar()) return planar_geometry_ok(d, width, height, pitch, frameStride, aligned);
    if (d.planes() == 1) return rgba_geometry_ok(d.pixels, width, height, pitch, frameStride, aligned, d.sample_bytes());
    return yuv_geometry_ok(d.pixels, d.chroma, width, height, pitch, frameStride, aligned, d.sample_bytes());
}

// The picture encoders of every codec with a block compressor and of Hap HDR, behind the codec-taking RGBA8 entry points (which
// refuse Hap7), the BC7 ones (which ask for it by name), the YUV, planar, RGBA16F and HDR10 ones
unsigned block_encode_picture_batch(const CodecInfo &ci, const PictureSrc &p, unsigned frames, unsigned long frameStride, unsigned width,
                                    unsigned height, unsigned long pitch, void *blocks, unsigned long blocksStride, void *stream)
{
    if (!blocks || frames == 0 || !picture_geometry_ok(p, width, height, pitch, frameStride, true) || ((uintptr_t)blocks | blocksStride) % 16)
        return HapResult_Bad_Arguments;
    HAP_ENTER(p.pixels, blocks);
    return on_batch_stream(stream, [&](cudaStream_t st) -> uint32_t {
        return launch_block_encode(ci, p, frames, frameStride, width, height, pitch, (uint8_t *)blocks, blocksStride,
                                   texture_bytes(width, height, ci, 0), st);
    });
}

unsigned encode_picture_batch(const CodecInfo &ci, const PictureSrc &p, unsigned frames, unsigned long frameStride, unsigned width,
                              unsigned height, unsigned long pitch, unsigned compressor, unsigned chunkCount, void *out,
                              unsigned long outStride, unsigned long long *used, void *stream)
{
    if (!out || !used || frames == 0 || chunkCount == 0 || !picture_geometry_ok(p, width, height, pitch, frameStride, true) ||
        (compressor != HapCompressorNone && compressor != HapCompressorSnappy))
        return HapResult_Bad_Arguments;
    if (outStride < max_encoded_length_rgba(width, height, ci, chunkCount)) return HapResult_Buffer_Too_Small;
    HAP_ENTER(p.pixels, out);
    // Hap Q from RGBA8 without the chroma refinement, Snappy: the fused encoder (hapq_fused.cuh) when the chunks allow it
    const FusedPictures fp = {(const uint8_t *)p.pixels, bc_encode_geom(width, height, (uint32_t)pitch, frameStride, 0, 0)};
    const bool fuse = HAPB200_FUSED_HAPQ && ci.bc_kind == kBcYCoCg && p.kind == kSrcRgba8 && g_chroma_refine.load() == 0 &&
                      compressor == HapCompressorSnappy;
    return on_batch_stream(stream, [&](cudaStream_t st) -> uint32_t {
        const uint64_t t[2] = {texture_bytes(width, height, ci, 0), texture_bytes(width, height, ci, 1)};
        return encode_frames_from_blocks(
            frames, ci.textures, t, ci.fmt, compressor, chunkCount, (uint8_t *)out, outStride, used, st,
            [&](uint8_t *tex, uint64_t stride) {
                return launch_block_encode(ci, p, frames, frameStride, width, height, pitch, tex, stride, align16(t[0]), st);
            },
            fuse ? &fp : nullptr);
    });
}

// The planes the single-frame calls copy between the caller's picture and tight device scratch: the picture's pointer to the
// plane (field), the caller's pitch, the bytes and rows it holds, and the scratch pitch (align16 of the row bytes).  Luma (or
// the RGBA picture), then the NV12 / P010 chroma plane, or the planar Cb, Cr and (when given) alpha planes; alpha-only
// pictures their alpha plane alone.  Returns the count.
template <class Picture>
struct PicturePlane {
    decltype(Picture::pixels) Picture::*field;
    uint64_t pitch, row, rows, tight;
};
template <class Picture>
int picture_planes(const Picture &p, uint32_t width, uint32_t height, uint64_t pitch, PicturePlane<Picture> planes[4])
{
    const uint64_t row = p.sample_bytes() * width, tight = align16(row);   // (RGBA8, RGBA16F: tight = row, width is a multiple of 4)
    int n = 0;
    if (p.is_planar()) {
        const uint64_t crow = p.sample_bytes() * (p.alpha_only ? 0 : p.chroma_width(width)), ctight = align16(crow);
        if (p.alpha_only) {
            planes[n++] = {&Picture::alpha, pitch, row, height, tight};
        } else {
            planes[n++] = {&Picture::pixels, pitch, row, height, tight};
            planes[n++] = {&Picture::chroma, p.chroma_pitch, crow, p.chroma_height(height), ctight};
            planes[n++] = {&Picture::cr, p.chroma_pitch, crow, p.chroma_height(height), ctight};
            if (p.alpha) planes[n++] = {&Picture::alpha, pitch, row, height, tight};
        }
    } else {
        planes[n++] = {&Picture::pixels, pitch, row, height, tight};
        if (p.planes() == 2) planes[n++] = {&Picture::chroma, pitch, row, height / 2, tight};
    }
    return n;
}

// One picture in host or device memory, its arguments checked: its planes (picture_planes) are copied into tight device
// scratch, one behind the other, and encoded as a batch of one by encode_picture_batch.  cap: the frame's size bound.
unsigned encode_picture(const CodecInfo &ci, const PictureSrc &p, unsigned width, unsigned height, unsigned long pitch, unsigned compressor,
                        unsigned chunkCount, void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    if (!outputBuffer || !outputBufferBytesUsed || chunkCount == 0 || !picture_geometry_ok(p, width, height, pitch, 0, false) ||
        (compressor != HapCompressorNone && compressor != HapCompressorSnappy))
        return HapResult_Bad_Arguments;
    const unsigned long cap = max_encoded_length_rgba(width, height, ci, chunkCount);
    if (outputBufferBytes < cap) return HapResult_Buffer_Too_Small;
    HAP_ENTER(p.pixels, outputBuffer);
    CallStream call(!is_device(p.pixels) && !is_device(p.chroma) && !is_device(p.cr) && !is_device(p.alpha) && !is_device(outputBuffer));
    cudaStream_t st = call.st;
    DevBuf img(st), frame(st), used(st);
    const uint64_t tight = align16(p.sample_bytes() * width);
    PictureSrc dev = p;
    if (p.is_planar()) dev.chroma_pitch = align16(p.sample_bytes() * (p.alpha_only ? 0 : p.chroma_width(width)));
    PicturePlane<PictureSrc> planes[4];
    const int n = picture_planes(p, width, height, pitch, planes);
    uint64_t plane_bytes = 0;
    for (int i = 0; i < n; i++) plane_bytes += planes[i].tight * planes[i].rows;
    if (!img.alloc(plane_bytes) || !frame.alloc(align16(cap)) || !used.alloc(32)) { cudaGetLastError(); return HapResult_Internal_Error; }
    uint64_t at = 0;
    for (int i = 0; i < n; i++) {
        const PicturePlane<PictureSrc> &q = planes[i];
        dev.*q.field = img.as<uint8_t>() + at;
        if (cudaMemcpy2DAsync(img.as<uint8_t>() + at, q.tight, p.*q.field, q.pitch, q.row, q.rows, cudaMemcpyDefault, st) != cudaSuccess) {
            cudaGetLastError();
            return HapResult_Internal_Error;
        }
        at += q.tight * q.rows;
    }
    if (dev.alpha_only) dev.pixels = dev.chroma = dev.cr = dev.alpha;
    uint32_t r = encode_picture_batch(ci, dev, 1, align16(plane_bytes), width, height, tight, compressor, chunkCount, frame.p, align16(cap),
                                      used.as<unsigned long long>(), st);
    if (r != HapResult_No_Error) return r;
    unsigned long long total = 0;
    if (cudaMemcpyAsync(&total, used.p, sizeof total, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess ||
        total > outputBufferBytes || cudaMemcpyAsync(outputBuffer, frame.p, total, cudaMemcpyDefault, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
    *outputBufferBytesUsed = (unsigned long)total;
    return HapResult_No_Error;
}

// ---- the families' own arguments and pictures ----

CodecInfo bc7_codec()
{
    CodecInfo ci;
    codec_info(HapB200Codec_Hap7, ci);
    return ci;
}

// the layouts and colour spaces the YUV encoders take (BC7 from Y'CbCr too)
bool yuv_format_ok(unsigned layout, unsigned colorSpace) { return layout <= HapB200YUV_P010 && colorSpace <= HapB200YUV_BT709_Full; }

// the codecs the YUV encoders take (every one with a block compressor that encodes colour) and the layouts and colour spaces
bool yuv_args_ok(unsigned layout, unsigned colorSpace, unsigned codec, CodecInfo &ci)
{
    return yuv_format_ok(layout, colorSpace) && codec_info(codec, ci) && codec_encodes(ci) && ci.bc_kind != kBcRgtc1;
}

PictureSrc yuv_picture(const void *luma, const void *chroma, unsigned layout, unsigned colorSpace)
{
    return {layout == HapB200YUV_P010 ? kSrcP010 : kSrcNv12, luma, chroma, colorSpace};
}

// the subsamplings, depths and colour spaces the planar encoders take (BC7 from Y'CbCr too)
bool planar_format_ok(unsigned subsampling, unsigned bitDepth, unsigned colorSpace)
{
    return subsampling <= HapB200Chroma_444 && (bitDepth == 8 || bitDepth == 10 || bitDepth == 12) && colorSpace <= HapB200YUV_BT709_Full;
}

// ... and the codecs they take: every one with a block compressor, HapA only with an alpha plane
bool planar_args_ok(const void *alpha, unsigned subsampling, unsigned bitDepth, unsigned colorSpace, unsigned codec, CodecInfo &ci)
{
    return planar_format_ok(subsampling, bitDepth, colorSpace) && codec_info(codec, ci) && codec_encodes(ci) && (ci.bc_kind != kBcRgtc1 || alpha);
}

// BC7 from a Y'CbCr picture encodes the RGBA8 picture made of it (launch_bc7_from_yuv), so that picture's rows, 4 * width
// bytes, must be rows the RGBA8 encoders take
bool bc7_rgba_width_ok(unsigned width) { return 4ul * width <= HAPB200_MAX_ROW_BYTES; }

// Hap1 and HapY do not read alpha; HapA reads alpha alone (the picture's other planes are the alpha plane, never read)
PictureSrc planar_picture(const CodecInfo &ci, const void *luma, const void *cb, const void *cr, const void *alpha, unsigned long chromaPitch,
                          unsigned subsampling, unsigned bitDepth, unsigned colorSpace)
{
    PictureSrc p{planar_src(subsampling, bitDepth > 8), luma, cb, colorSpace};
    p.cr = cr;
    p.alpha = ci.bc_kind == kBcDxt1 || ci.bc_kind == kBcYCoCg ? nullptr : alpha;
    p.chroma_pitch = chromaPitch;
    p.bit_depth = bitDepth;
    if (ci.bc_kind == kBcRgtc1) {
        p.alpha_only = true;
        p.pixels = p.chroma = p.cr = alpha;
    }
    return p;
}

// HapB200YUV_BT2020_Limited or _Full, and a unitNits of 1 .. 10000 cd/m2
bool yuv_pq_args_ok(unsigned colorSpace, unsigned unitNits)
{
    return (colorSpace == HapB200YUV_BT2020_Limited || colorSpace == HapB200YUV_BT2020_Full) && unitNits >= 1 && unitNits <= 10000;
}

PictureSrc yuv_pq_picture(const void *luma, const void *chroma, unsigned colorSpace, unsigned unitNits)
{
    return {kSrcP010Pq, luma, chroma, colorSpace, unitNits};
}

// the layouts and colour spaces the YUV decoders take (BT.601 / BT.709; no BT.2020)
bool yuv_out_args_ok(unsigned layout, unsigned colorSpace) { return layout <= HapB200YUV_P010 && colorSpace <= HapB200YUV_BT709_Full; }

PictureDst yuv_out_picture(void *luma, void *chroma, unsigned layout, unsigned colorSpace)
{
    return {layout == HapB200YUV_P010 ? kDstP010 : kDstNv12, luma, chroma, colorSpace};
}

// the subsamplings, depths and colour spaces the planar decoders take (BT.601 / BT.709; no BT.2020)
bool planar_out_args_ok(unsigned subsampling, unsigned bitDepth, unsigned colorSpace)
{
    return subsampling <= HapB200Chroma_444 && (bitDepth == 8 || bitDepth == 10 || bitDepth == 12) && colorSpace <= HapB200YUV_BT709_Full;
}

PictureDst planar_out_picture(void *luma, void *cb, void *cr, void *alpha, unsigned long chromaPitch, unsigned subsampling, unsigned bitDepth,
                              unsigned colorSpace)
{
    PictureDst d{planar_dst(subsampling, bitDepth > 8), luma, cb, colorSpace};
    d.cr = cr;
    d.alpha = alpha;
    d.chroma_pitch = chromaPitch;
    d.bit_depth = bitDepth;
    return d;
}

// Hap Alpha-Only's form of a planar picture: its alpha plane alone (pixels, chroma and cr point at it; nullptr without one)
PictureDst alpha_only_picture(const PictureDst &d)
{
    PictureDst a = d;
    a.alpha_only = true;
    a.pixels = a.chroma = a.cr = d.alpha;
    return a;
}

// the Hap HDR batch decoders' codec: each frame's signedness comes from its own texture format (frame_formats)
CodecInfo hap_hdr_batch_codec()
{
    CodecInfo ci;
    bc6h_codec(HapFmt_RGB_BPTC_UFLOAT, ci);
    return ci;
}

// ---- decoding ----

// The blocks of every frame (frame f's at blocks + f*blocksStride, Hap Q Alpha's alpha texture texture_bytes(.., 0) behind
// them) -> the pictures d, frameStride apart
unsigned block_decode_picture_batch(const CodecInfo &ci, const PictureDst &d, const void *blocks, unsigned frames, unsigned long blocksStride,
                                    unsigned width, unsigned height, unsigned long frameStride, unsigned long pitch, void *stream)
{
    if (!blocks || frames == 0 || !picture_geometry_ok(d, width, height, pitch, frameStride, true) || ((uintptr_t)blocks | blocksStride) % 16)
        return HapResult_Bad_Arguments;
    HAP_ENTER(blocks, d.pixels);
    return on_batch_stream(stream, [&](cudaStream_t st) -> uint32_t {
        return launch_block_decode(ci, d, (const uint8_t *)blocks, texture_bytes(width, height, ci, 0), frames, blocksStride, width, height,
                                   frameStride, pitch, nullptr, nullptr, st);
    });
}

// The texture half of the picture batch decoders: every texture of every frame decoded into device scratch `tex` (frame f at
// f * (align16(t[0]) + align16(t[1])), texture 1 at align16(t[0]) inside it) and texture 0's format into `formats`, both
// allocated here, and results[f] set as the batch decoders report it.  The decoded size must equal the texture size: each
// texture is offered exactly that much room per frame (the slot stride is wider: both textures of a frame share a slot, so a
// texture that over-declares its size must not reach its neighbour or the next frame's slot).  Then a frame whose textures are
// not ci's reports Bad_Frame (Hap HDR: hap_check_bc6h_frames_kernel, which takes either signedness; the others:
// hap_check_texture_kernel per texture), other failures keep the decoder's code.
uint32_t decode_textures_batch(const CodecInfo &ci, const void *in, unsigned frames, unsigned long inStride, const unsigned long long *inBytes,
                               unsigned maxChunks, const uint64_t t[2], DevBuf &tex, DevBuf &formats, unsigned *results, cudaStream_t st)
{
    const bool bc6h = ci.bc_kind == kBcBc6h;
    const uint64_t stride = align16(t[0]) + align16(t[1]);
    DevBuf used(st), res1(st);
    if (!tex.alloc(stride * frames + 16) || !used.alloc(8ull * frames) || !formats.alloc(4ull * frames) || (!bc6h && !res1.alloc(4ull * frames))) {
        cudaGetLastError();
        return HapResult_Internal_Error;
    }
    for (uint32_t ti = 0; ti < ci.textures; ti++) {
        uint32_t *res = ti == 0 ? results : res1.as<uint32_t>();
        const uint32_t r = launch_decode_batch((const uint8_t *)in, frames, inStride, inBytes, ti, maxChunks, tex.as<uint8_t>() + (ti ? align16(t[0]) : 0),
                                               stride, t[ti], used.as<unsigned long long>(), formats.as<uint32_t>(), res, st);
        if (r != HapResult_No_Error) return r;
        if (bc6h)
            HAP_KLAUNCH(kStCollect, hap_check_bc6h_frames_kernel, dim3((frames + 127) / 128), dim3(128), 0, st, (const uint8_t *)in,
                        (uint64_t)inStride, inBytes, frames, used.as<unsigned long long>(), formats.as<uint32_t>(), (unsigned long long)t[0], results);
        else
            HAP_KLAUNCH(kStCollect, hap_check_texture_kernel, dim3((frames + 127) / 128), dim3(128), 0, st, frames, used.as<unsigned long long>(),
                        formats.as<uint32_t>(), res, (unsigned long long)t[ti], ci.fmt[ti], results);
    }
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

unsigned decode_picture_batch(const CodecInfo &ci, const PictureDst &d, const void *in, unsigned frames, unsigned long inStride,
                              const unsigned long long *inBytes, unsigned maxChunks, unsigned width, unsigned height, unsigned long frameStride,
                              unsigned long pitch, unsigned *results, void *stream)
{
    if (!in || !inBytes || !results || frames == 0 || maxChunks == 0 || !picture_geometry_ok(d, width, height, pitch, frameStride, true))
        return HapResult_Bad_Arguments;
    HAP_ENTER(in, d.pixels);
    return on_batch_stream(stream, [&](cudaStream_t st) -> uint32_t {
        const uint64_t t[2] = {texture_bytes(width, height, ci, 0), texture_bytes(width, height, ci, 1)};
        DevBuf tex(st), formats(st);
        const uint32_t r = decode_textures_batch(ci, in, frames, inStride, inBytes, maxChunks, t, tex, formats, results, st);
        if (r != HapResult_No_Error) return r;
        return launch_block_decode(ci, d, tex.as<uint8_t>(), align16(t[0]), frames, align16(t[0]) + align16(t[1]), width, height, frameStride,
                                   pitch, results, formats.as<uint32_t>(), st);
    });
}

// One frame in host or device memory -> the picture d.  The frame's codec comes from its headers: Hap HDR frames decode to the
// RGBA16F and HDR10 sinks only, the other flavours to the others (Bad_Frame otherwise).  A planar picture takes Hap Alpha-Only's
// form (alpha_only_picture) for a Hap Alpha-Only frame, so before the headers are read its planes need only pass as either
// form, and after it as the frame's (Bad_Arguments: a Hap Alpha-Only frame without an alpha plane, another without luma, Cb or
// Cr).  The frame's textures, t[i] bytes each, are decoded by HapDecode into device scratch (a texture that does not fill its
// room: Bad_Frame; the HDR sinks answer Bad_Frame for one too large for it as well, the others what HapDecode answers); then
// launch_block_decode writes a tight picture (picture_planes), which is copied to the caller's planes.
uint32_t decode_picture(const PictureDst &dst, const void *inputBuffer, unsigned long inputBufferBytes, unsigned width, unsigned height,
                        unsigned long pitch)
{
    if (!inputBuffer || !(picture_geometry_ok(dst, width, height, pitch, 0, false) ||
                          (dst.is_planar() && picture_geometry_ok(alpha_only_picture(dst), width, height, pitch, 0, false))))
        return HapResult_Bad_Arguments;
    unsigned count = 0, f0 = 0, f1 = 0;
    uint32_t r = HapGetFrameTextureCount(inputBuffer, inputBufferBytes, &count);
    if (r != HapResult_No_Error) return r;
    r = HapGetFrameTextureFormat(inputBuffer, inputBufferBytes, 0, &f0);
    if (r != HapResult_No_Error) return r;
    CodecInfo ci;
    if (dst.hdr()) {
        if (count != 1 || !bc6h_codec(f0, ci)) return HapResult_Bad_Frame;
    } else {
        if (count == 2 && (r = HapGetFrameTextureFormat(inputBuffer, inputBufferBytes, 1, &f1)) != HapResult_No_Error) return r;
        unsigned codec = 0;
        while (codec_info(codec, ci) && (ci.textures != count || ci.fmt[0] != f0 || (count == 2 && ci.fmt[1] != f1))) codec++;
        if (!codec_info(codec, ci)) return HapResult_Bad_Frame;
    }
    const PictureDst d = dst.is_planar() && ci.bc_kind == kBcRgtc1 ? alpha_only_picture(dst) : dst;
    if (d.is_planar() && !picture_geometry_ok(d, width, height, pitch, 0, false)) return HapResult_Bad_Arguments;
    HAP_ENTER(inputBuffer, d.pixels, d.chroma);
    const uint64_t t[2] = {texture_bytes(width, height, ci, 0), texture_bytes(width, height, ci, 1)};
    PicturePlane<PictureDst> planes[4];
    const int n = picture_planes(d, width, height, pitch, planes);
    uint64_t plane_bytes = 0;
    for (int i = 0; i < n; i++) plane_bytes += planes[i].tight * planes[i].rows;
    // scratch from the device's stream-ordered pool on the legacy stream (the nested HapDecode calls below write it on
    // that stream, or on a pooled stream they synchronise before returning): no cudaMalloc/cudaFree, no device-wide sync
    DevBuf texb(kLegacyStream), imgb(kLegacyStream);
    if (!texb.alloc(align16(t[0]) + align16(t[1]) + 16) || !imgb.alloc(plane_bytes)) { cudaGetLastError(); return HapResult_Internal_Error; }
    if (cudaStreamSynchronize(kLegacyStream) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }   // the allocations are real now
    auto serial = [](HapDecodeWorkFunction fn, void *p, unsigned n, void *) { for (unsigned i = 0; i < n; i++) fn(p, i); };
    for (unsigned i = 0; i < ci.textures && r == HapResult_No_Error; i++) {
        unsigned long used = 0;
        unsigned fmt = 0;
        r = HapDecode(inputBuffer, inputBufferBytes, i, serial, nullptr, texb.as<uint8_t>() + (i ? align16(t[0]) : 0), t[i], &used, &fmt);
        if (r == HapResult_No_Error && used != t[i]) r = HapResult_Bad_Frame;
    }
    // the room offered is the picture's texture size: to the HDR sinks, a texture too large for it (HapDecode: Buffer_Too_Small)
    // is not this picture's texture either
    if (r != HapResult_No_Error) return d.hdr() && r == HapResult_Buffer_Too_Small ? (uint32_t)HapResult_Bad_Frame : r;
    CallStream call(false);  // the scratch buffers are device memory filled on the legacy stream by HapDecode above
    cudaStream_t st = call.st;
    PictureDst img = d;
    uint64_t at = 0;
    for (int i = 0; i < n; i++) {
        img.*planes[i].field = imgb.as<uint8_t>() + at;
        at += planes[i].tight * planes[i].rows;
    }
    if (img.alpha_only) img.pixels = img.chroma = img.cr = img.alpha;
    if (img.is_planar()) img.chroma_pitch = align16(d.sample_bytes() * (d.alpha_only ? 0 : d.chroma_width(width)));
    r = launch_block_decode(ci, img, texb.as<uint8_t>(), align16(t[0]), 1, 0, width, height, 0, align16(d.sample_bytes() * width), nullptr,
                            nullptr, st);
    for (int i = 0; i < n && r == HapResult_No_Error; i++) {
        const PicturePlane<PictureDst> &q = planes[i];
        if (cudaMemcpy2DAsync(d.*q.field, q.pitch, img.*q.field, q.tight, q.row, q.rows, cudaMemcpyDefault, st) != cudaSuccess) {
            cudaGetLastError();
            r = HapResult_Internal_Error;
        }
    }
    if (r == HapResult_No_Error && cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); r = HapResult_Internal_Error; }
    return r;
}

}  // namespace

// ---- delivery rings: helpers ----
namespace {
__global__ void ring_publish_kernel(unsigned int *flag, unsigned int value)
{
    // the kernels queued before this one have completed, their stores to the peer are performed; the fence orders this
    // thread's view, the release store makes the flag the last thing the consumer can see
    __threadfence_system();
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(flag), "r"(value) : "memory");
}
__global__ void ring_wait_kernel(const unsigned int *flag, unsigned int value, unsigned long long timeout_ns)
{
    unsigned int v;
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    for (;;) {
        asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
        if ((int)(v - value) >= 0) break;
        hap_nanosleep(500);
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        if (timeout_ns && t1 - t0 > timeout_ns) break;     // a producer that died must not hang the consumer's GPU for ever
    }
}
}  // namespace

// =====================================================================================================
extern "C" {

const char *HapB200Version(void) { return "hap-b200 0.1 (sm_90a)"; }
unsigned long long HapB200KernelLaunchCount(void) { return g_launches.load(); }

// The device host-pointer calls run on (device-pointer calls run where their buffers live).  -1: forget it; the next
// host-pointer call takes its thread's current device.
int HapB200SetDevice(int device)
{
    if (device < -1 || device >= kMaxDevices) return -1;
    g_default_device.store(device);
    return 0;
}
int HapB200GetDevice(void) { return g_default_device.load(); }

// ---- delivery rings (include/hap_b200.h) ---------------------------------------------------------------------------
unsigned int HapB200RingCreate(int device, unsigned long bytes, void **ring, void *handle)
{
    if (!ring || bytes == 0) return HapResult_Bad_Arguments;
    DeviceGuard on(device);
    if (!on.ok) return HapResult_Internal_Error;
    void *p = nullptr;
    // plain cudaMalloc: memory of a stream-ordered pool cannot be exported
    if (cudaMalloc(&p, bytes) != cudaSuccess || cudaMemset(p, 0, bytes) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) {
        cudaGetLastError();
        if (p) cudaFree(p);
        return HapResult_Internal_Error;
    }
    if (handle) {
        static_assert(sizeof(cudaIpcMemHandle_t) == HAPB200_RING_HANDLE_BYTES, "handle size");
        cudaIpcMemHandle_t h;
        if (cudaIpcGetMemHandle(&h, p) != cudaSuccess) { cudaGetLastError(); cudaFree(p); return HapResult_Internal_Error; }
        memcpy(handle, &h, sizeof h);
    }
    *ring = p;
    return HapResult_No_Error;
}

unsigned int HapB200RingDestroy(int device, void *ring)
{
    if (!ring) return HapResult_Bad_Arguments;
    DeviceGuard on(device);
    if (!on.ok) return HapResult_Internal_Error;
    cudaDeviceSynchronize();
    const bool ok = cudaFree(ring) == cudaSuccess;
    cudaGetLastError();
    return ok ? HapResult_No_Error : HapResult_Internal_Error;
}

unsigned int HapB200RingOpen(int device, const void *handle, void **ring)
{
    if (!handle || !ring) return HapResult_Bad_Arguments;
    DeviceGuard on(device);
    if (!on.ok) return HapResult_Internal_Error;
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, sizeof h);
    void *p = nullptr;
    if (cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
    *ring = p;
    return HapResult_No_Error;
}

unsigned int HapB200RingClose(int device, void *ring)
{
    if (!ring) return HapResult_Bad_Arguments;
    DeviceGuard on(device);
    if (!on.ok) return HapResult_Internal_Error;
    cudaDeviceSynchronize();
    const bool ok = cudaIpcCloseMemHandle(ring) == cudaSuccess;
    cudaGetLastError();
    return ok ? HapResult_No_Error : HapResult_Internal_Error;
}

unsigned int HapB200RingAttach(int device, int ringDevice)
{
    if (ringDevice < 0 || ringDevice >= kMaxDevices) return HapResult_Bad_Arguments;
    if (device == ringDevice) return HapResult_No_Error;
    DeviceGuard on(device);
    if (!on.ok) return HapResult_Internal_Error;
    int can = 0;
    if (cudaDeviceCanAccessPeer(&can, device, ringDevice) != cudaSuccess || !can) { cudaGetLastError(); return HapResult_Internal_Error; }
    const cudaError_t e = cudaDeviceEnablePeerAccess(ringDevice, 0);
    cudaGetLastError();
    return (e == cudaSuccess || e == cudaErrorPeerAccessAlreadyEnabled) ? HapResult_No_Error : HapResult_Internal_Error;
}

unsigned int HapB200RingPublish(int device, void *flag, unsigned int value, void *stream)
{
    if (!flag || ((uintptr_t)flag & 3)) return HapResult_Bad_Arguments;
    DeviceGuard on(device);
    if (!on.ok) return HapResult_Internal_Error;
    cudaStream_t st = stream ? (cudaStream_t)stream : kLegacyStream;
    ring_publish_kernel<<<1, 1, 0, st>>>((unsigned int *)flag, value);
    g_launches.fetch_add(1);
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

unsigned int HapB200RingWait(int device, const void *flag, unsigned int value, unsigned int timeoutMs, void *stream)
{
    if (!flag || ((uintptr_t)flag & 3)) return HapResult_Bad_Arguments;
    DeviceGuard on(device);
    if (!on.ok) return HapResult_Internal_Error;
    cudaStream_t st = stream ? (cudaStream_t)stream : kLegacyStream;
    if (timeoutMs == 0) {
        // No timeout asked for: a stream memory operation of the driver (cuStreamWaitValue32, "flag - value >= 0" compared as
        // signed), which holds the stream WITHOUT occupying an SM.  (A polling kernel resident on one SM keeps the encoder's
        // one-CTA-per-SM fragment kernel from getting that SM, so the last CTA of that grid runs as a second wave.)
        typedef int (*WaitValue32)(cudaStream_t, unsigned long long, unsigned int, unsigned int);
        static WaitValue32 wait_value = [] {
            void *fn = nullptr;
            cudaDriverEntryPointQueryResult q;
            if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &fn, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) { cudaGetLastError(); fn = nullptr; }
            return (WaitValue32)fn;
        }();
        if (wait_value && wait_value(st, (unsigned long long)(uintptr_t)flag, value, 0u /* CU_STREAM_WAIT_VALUE_GEQ */) == 0) return HapResult_No_Error;
        // (driver without stream memory operations: the polling kernel below, waiting for ever)
    }
    ring_wait_kernel<<<1, 1, 0, st>>>((const unsigned int *)flag, value, 1000000ull * timeoutMs);
    g_launches.fetch_add(1);
    return cudaGetLastError() == cudaSuccess ? HapResult_No_Error : HapResult_Internal_Error;
}

int HapB200SetOption(int option, int value)
{
    switch (option) {
    case HAPB200_OPTION_USE_INDEX: g_use_index.store(value != 0); return 0;
    case HAPB200_OPTION_WRITE_INDEX: g_write_index.store(value != 0); return 0;
    case HAPB200_OPTION_WRITE_OFFSET_TABLE: g_write_offsets.store(value != 0); return 0;
    case HAPB200_OPTION_CHROMA_REFINE: g_chroma_refine.store(value != 0); return 0;
    default: return -1;
    }
}

void HapB200SetStageTiming(int enabled)
{
    std::lock_guard<std::mutex> l(g_timer.mu);
    g_timer.on = enabled != 0;
}

// Synchronises the device, folds the recorded events into per-stage totals and returns them:
// ms[i], launches[i] for i < n (stage order: bc_encode, snappy_encode, plan, place, parse, snappy_decode,
// collect, bc_decode, snappy_index, windows).  Totals are reset by the call.
int HapB200StageTimes(double *ms, unsigned long long *launches, int n)
{
    cudaDeviceSynchronize();
    std::lock_guard<std::mutex> l(g_timer.mu);
    for (auto &r : g_timer.recs) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) { g_timer.ms[r.stage] += t; g_timer.n[r.stage]++; }
        cudaEventDestroy(r.a);
        cudaEventDestroy(r.b);
    }
    g_timer.recs.clear();
    for (int i = 0; i < n && i < kStCount; i++) { ms[i] = g_timer.ms[i]; launches[i] = g_timer.n[i]; }
    for (int i = 0; i < kStCount; i++) { g_timer.ms[i] = 0; g_timer.n[i] = 0; }
    cudaGetLastError();
    return kStCount;
}

#if HAPB200_ENC_PHASE_CLOCKS
// Measurement builds only (-DHAPB200_ENC_PHASE_CLOCKS=1): the fused Hap Q encoders' clocks per phase summed over every CTA
// of the current device since the last call, then the fragments compressed (snappy_encode.cuh, kEp*).  Synchronises the
// device and resets the sums.  Returns the number of slots.
int HapB200EncodePhaseClocks(unsigned long long *out, int n)
{
    cudaDeviceSynchronize();
    unsigned long long v[kEpSlots] = {};
    if (cudaMemcpyFromSymbol(v, g_enc_phase_clocks, sizeof v) != cudaSuccess) { cudaGetLastError(); return -1; }
    const unsigned long long zero[kEpSlots] = {};
    cudaMemcpyToSymbol(g_enc_phase_clocks, zero, sizeof zero);
    for (int i = 0; i < n && i < kEpSlots; i++) out[i] = v[i];
    return kEpSlots;
}
#endif

#if HAPB200_EX_PHASE_CLOCKS
// Measurement builds only (-DHAPB200_EX_PHASE_CLOCKS=1): the unit path's clocks per phase summed over every CTA of the
// current device since the last call, then the unit windows and the pointer-jumping rounds (snappy_decode.cuh, kPh*).
// Synchronises the device and resets the sums.  Returns the number of slots.
int HapB200UnitPhaseClocks(unsigned long long *out, int n)
{
    cudaDeviceSynchronize();
    unsigned long long v[kPhSlots] = {};
    if (cudaMemcpyFromSymbol(v, g_ex_phase_clocks, sizeof v) != cudaSuccess) { cudaGetLastError(); return -1; }
    const unsigned long long zero[kPhSlots] = {};
    cudaMemcpyToSymbol(g_ex_phase_clocks, zero, sizeof zero);
    for (int i = 0; i < n && i < kPhSlots; i++) out[i] = v[i];
    return kPhSlots;
}
#endif

// hap.c:324-353
unsigned long HapMaxEncodedLength(unsigned int count, unsigned long *lengths, unsigned int *textureFormats,
                                  unsigned int *chunkCounts)
{
    if (count == 0 || count > 2 || !lengths || !textureFormats || !chunkCounts) return 0;
    unsigned long total = 8;
    for (unsigned i = 0; i < count; i++) {
        if (chunkCounts[i] == 0) return 0;
        total += (unsigned long)max_encoded_length_one(lengths[i], textureFormats[i], HapCompressorSnappy, chunkCounts[i]);
    }
    return total;
}

// hap.c:1042-1087
unsigned int HapGetFrameTextureCount(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int *outputTextureCount)
{
    HeaderView hv(inputBuffer, inputBufferBytes);
    if (!hv.ok) return HapResult_Internal_Error;
    const uint8_t *in = hv.p;
    Section top;
    uint32_t r = read_section_header(in, (uint32_t)inputBufferBytes, top);
    if (r != HapResult_No_Error) return r;
    if (top.type != kSecMultipleImages) { *outputTextureCount = 1; return HapResult_No_Error; }
    uint32_t off = top.hdr;
    *outputTextureCount = 0;
    while (off < top.len) {  // hap.c:1064 compares against the body length, as here
        Section s;
        if (!hv.need(in + off, 8)) return HapResult_Internal_Error;
        r = read_section_header(in + off, (uint32_t)(inputBufferBytes - off), s);
        if (r != HapResult_No_Error) return r;
        off += s.hdr + s.len;
        *outputTextureCount += 1;
    }
    return HapResult_No_Error;
}

// hap.c:1089-1126
unsigned int HapGetFrameTextureFormat(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int index,
                                      unsigned int *outputBufferTextureFormat)
{
    if (!inputBuffer || index > 1 || !outputBufferTextureFormat) return HapResult_Bad_Arguments;
    HeaderView hv(inputBuffer, inputBufferBytes);
    if (!hv.ok) return HapResult_Internal_Error;
    Located loc;
    uint32_t r = locate_texture(hv.p, (uint32_t)inputBufferBytes, index, loc, hv);
    if (r != HapResult_No_Error) return r;
    *outputBufferTextureFormat = format_from_nibble(loc.type & 0xF);
    return *outputBufferTextureFormat ? HapResult_No_Error : HapResult_Bad_Frame;
}

// hap.c:1128-1188
unsigned int HapGetFrameTextureChunkCount(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int index,
                                          int *chunk_count)
{
    *chunk_count = 0;  // before validation, like hap.c:1134
    if (!inputBuffer || index > 1) return HapResult_Bad_Arguments;
    HeaderView hv(inputBuffer, inputBufferBytes);
    if (!hv.ok) return HapResult_Internal_Error;
    Located loc;
    uint32_t r = locate_texture(hv.p, (uint32_t)inputBufferBytes, index, loc, hv);
    if (r != HapResult_No_Error) return r;
    const uint32_t compressor = (loc.type >> 4) & 0xF;
    if (compressor == kHapComplex) {
        ChunkTables t;
        t.count = 0;
        r = parse_decode_instructions(hv.p + loc.offset, loc.len, t, hv);
        *chunk_count = t.count;
        return r;
    }
    if (compressor == kHapChunkSnappy || compressor == kHapChunkRaw) { *chunk_count = 1; return HapResult_No_Error; }
    return HapResult_Bad_Frame;
}

// hap.c:506-604 + :355-504
unsigned int HapEncode(unsigned int count, const void **inputBuffers, unsigned long *inputBuffersBytes,
                       unsigned int *textureFormats, unsigned int *compressors, unsigned int *chunkCounts,
                       void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    if (count == 0 || count > 2 || !inputBuffers || !inputBuffersBytes || !textureFormats || !compressors || !chunkCounts ||
        !outputBuffer || outputBufferBytes == 0 || !outputBufferBytesUsed)
        return HapResult_Bad_Arguments;
    for (unsigned i = 0; i < count; i++)
        if (chunkCounts[i] == 0) return HapResult_Bad_Arguments;
    if (!texture_formats_ok(count, textureFormats)) return HapResult_Bad_Arguments;

    TextureArgs ta[2];
    for (unsigned i = 0; i < count; i++) ta[i] = TextureArgs{inputBuffersBytes[i], textureFormats[i], compressors[i], chunkCounts[i]};
    // hap.c:563-576: outer header from the worst case, with the REQUESTED chunk counts (SURVEY.md Q6)
    uint64_t outer = 0;
    if (count == 2) {
        uint64_t worst = 0;
        for (unsigned i = 0; i < 2; i++) worst += ta[i].bytes + decode_instructions_length(ta[i].chunks) + 4;
        outer = worst > kU24Max ? 8 : 4;
    }
    // Errors surface in texture order: the reference encodes texture 0 completely before it looks at
    // texture 1 (hap.c:580-596).  The capacity test of texture 1 is made against what section 0 really
    // used (hap.c:589), which is only known after compression: checked further down.
    if (!inputBuffers[0] || validate_texture_args(ta[0]) != HapResult_No_Error) return HapResult_Bad_Arguments;
    if (outputBufferBytes < outer ||
        outputBufferBytes - outer < max_encoded_length_one(ta[0].bytes, ta[0].format, ta[0].compressor, ta[0].chunks))
        return HapResult_Buffer_Too_Small;
    if (count == 2 && (!inputBuffers[1] || validate_texture_args(ta[1]) != HapResult_No_Error)) return HapResult_Bad_Arguments;
    FrameGeom G;
    {
        uint32_t gr = build_frame_geom(count, ta, G);
        if (gr != HapResult_No_Error) return gr;
    }

    bool all_host_verbatim = !is_device(outputBuffer);
    for (unsigned i = 0; i < count; i++)
        all_host_verbatim = all_host_verbatim && ta[i].compressor == HapCompressorNone && !is_device(inputBuffers[i]);
    if (all_host_verbatim) {
        // hap.c:490-501 for every texture: headers plus a copy, nothing to compute and nothing for a GPU to do
        uint8_t *o = (uint8_t *)outputBuffer;
        uint64_t pos = outer;
        for (unsigned i = 0; i < count; i++) {
            const uint32_t hdr = G.s[i].top_hdr;
            if (i == 1 && (outputBufferBytes < pos ||
                           outputBufferBytes - pos < max_encoded_length_one(ta[1].bytes, ta[1].format, ta[1].compressor, ta[1].chunks)))
                return HapResult_Buffer_Too_Small;
            put_section_header(o + pos, hdr, (uint32_t)ta[i].bytes, (kHapChunkRaw << 4) | G.s[i].fmt_nibble);
            memcpy(o + pos + hdr, inputBuffers[i], ta[i].bytes);
            pos += hdr + ta[i].bytes;
        }
        if (count == 2) put_section_header(o, (uint32_t)outer, (uint32_t)(pos - outer), kSecMultipleImages);
        *outputBufferBytesUsed = (unsigned long)pos;
        return HapResult_No_Error;
    }

    HAP_ENTER(outputBuffer, inputBuffers[0], count == 2 ? inputBuffers[1] : nullptr);
    bool enc_all_host = !is_device(outputBuffer);
    for (unsigned i = 0; i < count; i++) enc_all_host = enc_all_host && !is_device(inputBuffers[i]);
    CallStream call(enc_all_host);
    cudaStream_t st = call.st;

    // worst-case frame in device scratch; textures staged into 16-byte aligned device memory
    unsigned long lens[2] = {ta[0].bytes, count == 2 ? ta[1].bytes : 0};
    unsigned fmts[2] = {ta[0].format, ta[1].format}, chunks[2] = {ta[0].chunks, ta[1].chunks};
    const unsigned long cap = HapMaxEncodedLength(count, lens, fmts, chunks);
    DevBuf tex(st), frame(st), used(st);
    const uint64_t off1 = align16(ta[0].bytes);
    const uint64_t tex_bytes = off1 + (count == 2 ? align16(ta[1].bytes) : 0) + 16;
    if (!tex.alloc(tex_bytes) || !frame.alloc(cap) || !used.alloc(sizeof(unsigned long long) * 4)) { cudaGetLastError(); return HapResult_Internal_Error; }
    for (unsigned i = 0; i < count; i++) {
        uint8_t *d = tex.as<uint8_t>() + (i ? off1 : 0);
        cudaMemcpyKind kind = is_device(inputBuffers[i]) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
        if (cudaMemcpyAsync(d, inputBuffers[i], ta[i].bytes, kind, st) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
        G.s[i].in_offset = i ? off1 : 0;
        G.s[i].in_stride = 0;
    }
    uint32_t r = launch_encode(tex.as<uint8_t>(), G, 1, frame.as<uint8_t>(), cap, used.as<unsigned long long>(), st);
    if (r != HapResult_No_Error) return r;
    unsigned long long total = 0;
    if (cudaMemcpyAsync(&total, used.p, sizeof total, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
        cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
    if (total > outputBufferBytes) return HapResult_Buffer_Too_Small;
    if (count == 2) {
        // hap.c:589: capacity left for texture 1 = outputBufferBytes - (outer header + actual section 0)
        Section s0;
        uint8_t head[16];
        if (cudaMemcpy(head, frame.as<uint8_t>() + outer, 8, cudaMemcpyDeviceToHost) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
        if (read_section_header(head, 0xFFFFFFFFu, s0) == HapResult_No_Error) {
            uint64_t before = outer + s0.hdr + s0.len;
            if (outputBufferBytes < before ||
                outputBufferBytes - before < max_encoded_length_one(ta[1].bytes, ta[1].format, ta[1].compressor, ta[1].chunks))
                return HapResult_Buffer_Too_Small;
        }
    }
    cudaMemcpyKind okind = is_device(outputBuffer) ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost;
    if (cudaMemcpyAsync(outputBuffer, frame.p, total, okind, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess) {
        cudaGetLastError();
        return HapResult_Internal_Error;
    }
    *outputBufferBytesUsed = (unsigned long)total;
    return HapResult_No_Error;
}

// hap.c:993-1040 + :732-930
unsigned int HapDecode(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int index,
                       HapDecodeCallback callback, void *info, void *outputBuffer, unsigned long outputBufferBytes,
                       unsigned long *outputBufferBytesUsed, unsigned int *outputBufferTextureFormat)
{
    if (!inputBuffer || index > 1 || !callback || !outputBuffer || !outputBufferTextureFormat) return HapResult_Bad_Arguments;
    const bool in_dev = is_device(inputBuffer), out_dev = is_device(outputBuffer);
    HeaderView hv(inputBuffer, inputBufferBytes);
    if (!hv.ok) return HapResult_Internal_Error;
    // chunk offsets fit the 32-bit fields of hap.c's HapChunkDecodeInfo
    TexturePlan plan;
    std::vector<PlannedJob> planned;
    uint32_t r = plan_texture(hv.p, (uint32_t)inputBufferBytes, index, outputBufferBytes, ~0u, 0xFFFFFFFFull, hv, plan,
                              [&](const PlannedJob &j) { planned.push_back(j); });
    if (plan.located) *outputBufferTextureFormat = plan.format;
    if (r != HapResult_No_Error) return r;
    const Located &loc = plan.loc;
    const uint8_t *sec = hv.p + loc.offset;
    if (((loc.type >> 4) & 0xF) == kHapChunkRaw) {
        // hap.c:905-916: a verbatim texture is a copy; nothing to compute
        if (!in_dev && !out_dev) {
            memcpy(outputBuffer, sec, loc.len);
        } else {
            HAP_ENTER(inputBuffer, outputBuffer);
            const uint8_t *src = in_dev ? (const uint8_t *)inputBuffer + loc.offset : sec;
            if (cudaMemcpy(outputBuffer, src, loc.len, cudaMemcpyDefault) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
        }
        if (outputBufferBytesUsed) *outputBufferBytesUsed = loc.len;
        return HapResult_No_Error;
    }

    if (!planned.empty()) {
        HAP_ENTER(inputBuffer, outputBuffer);
        CallStream call(!in_dev && !out_dev);
        cudaStream_t st = call.st;
        DevBuf din(st), dout(st), djobs(st);
        const uint8_t *dsec;
        const uint8_t *dindex = nullptr;    // device address of byte 0 of the fragment index body (hap_index.h), when a chunk has a record
        bool any_index = false;
        for (auto &j : planned) any_index = any_index || j.index_bytes != 0;
        if (in_dev) {
            dsec = (const uint8_t *)inputBuffer + loc.offset;
            if (any_index) dindex = (const uint8_t *)inputBuffer + plan.ix.body;
        } else {
            // the texture section, and behind it (16-byte aligned) the body of the frame's trailing index section
            const uint64_t ioff = align16(loc.len);
            if (!din.alloc(ioff + (any_index ? plan.ix.len : 0)) || cudaMemcpyAsync(din.p, sec, loc.len, cudaMemcpyHostToDevice, st) != cudaSuccess ||
                (any_index && cudaMemcpyAsync(din.as<uint8_t>() + ioff, hv.p + plan.ix.body, plan.ix.len, cudaMemcpyHostToDevice, st) != cudaSuccess)) {
                cudaGetLastError();
                return HapResult_Internal_Error;
            }
            dsec = din.as<uint8_t>();
            if (any_index) dindex = din.as<uint8_t>() + ioff;
        }
        uint8_t *ddst;
        if (out_dev) ddst = (uint8_t *)outputBuffer;
        else {
            if (!dout.alloc(plan.produced)) { cudaGetLastError(); return HapResult_Internal_Error; }
            ddst = dout.as<uint8_t>();
        }
        std::vector<ChunkJob> jobs(planned.size());   // (the fields the decode kernels set start zeroed)
        uint64_t in_sum = 0;
        for (size_t i = 0; i < planned.size(); i++) {
            const PlannedJob &j = planned[i];
            jobs[i].src = dsec + (j.src_off - loc.offset);
            jobs[i].dst = ddst + j.dst_off;
            jobs[i].src_bytes = j.src_bytes;
            jobs[i].dst_bytes = j.dst_bytes;
            jobs[i].compressor = j.compressor;
            jobs[i].index = j.index_bytes ? dindex + (j.index_off - plan.ix.body) : nullptr;
            jobs[i].index_bytes = j.index_bytes;
            in_sum += j.src_bytes;
        }
        if (!djobs.alloc(jobs.size() * sizeof(ChunkJob)) ||
            cudaMemcpyAsync(djobs.p, jobs.data(), jobs.size() * sizeof(ChunkJob), cudaMemcpyHostToDevice, st) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
        DecodePasses passes(st);
        r = passes.first(djobs.as<ChunkJob>(), (uint32_t)jobs.size(), in_sum, plan.produced);
        if (r != HapResult_No_Error) return r;
        if (!plan.whole && jobs.size() > 1) {
            WorkState ws;
            callback(work_function, &ws, (unsigned)jobs.size(), info);  // hap.c:861
        }
        if (cudaMemcpyAsync(jobs.data(), djobs.p, jobs.size() * sizeof(ChunkJob), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
            cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
        bool mismatch = false;     // a chunk whose embedded index failed the execute kernel's checks: the repair pass, then the statuses again
        for (size_t i = 0; i < jobs.size(); i++) mismatch = mismatch || jobs[i].status == kStatusIndexMismatch;
        if (mismatch) {
            r = passes.repair();
            if (r != HapResult_No_Error) return r;
            if (cudaMemcpyAsync(jobs.data(), djobs.p, jobs.size() * sizeof(ChunkJob), cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
        }
        for (size_t i = 0; i < jobs.size(); i++)
            if (jobs[i].status != HapResult_No_Error) return plan.whole ? (uint32_t)HapResult_Internal_Error : jobs[i].status;  // hap.c:867-875, :899-903
        if (!out_dev && plan.produced) {
            if (cudaMemcpyAsync(outputBuffer, ddst, plan.produced, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                cudaStreamSynchronize(st) != cudaSuccess) { cudaGetLastError(); return HapResult_Internal_Error; }
        }
    }
    if (outputBufferBytesUsed) *outputBufferBytesUsed = (unsigned long)plan.produced;
    return HapResult_No_Error;
}

// ---- extensions ----------------------------------------------------------------------------------

unsigned long HapB200TextureBytes(unsigned int width, unsigned int height, unsigned int codec, unsigned int index)
{
    CodecInfo ci;
    if (!codec_info(codec, ci)) return 0;
    return texture_bytes(width, height, ci, index);
}

unsigned long HapB200MaxEncodedLengthRGBA(unsigned int width, unsigned int height, unsigned int codec, unsigned int chunkCount)
{
    CodecInfo ci;
    if (!codec_info(codec, ci)) return 0;
    return max_encoded_length_rgba(width, height, ci, chunkCount);
}

unsigned int HapB200BlockEncodeBatch(const void *rgba, unsigned int frames, unsigned long frameStride, unsigned int width,
                                     unsigned int height, unsigned long rowBytes, unsigned int codec, void *blocks,
                                     unsigned long blocksStride, void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci) || !codec_encodes(ci)) return HapResult_Bad_Arguments;
    return block_encode_picture_batch(ci, rgba_picture(rgba), frames, frameStride, width, height, rowBytes, blocks, blocksStride, stream);
}

unsigned int HapB200BlockDecodeBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                     unsigned int height, unsigned int codec, void *rgba, unsigned long frameStride,
                                     unsigned long rowBytes, void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci)) return HapResult_Bad_Arguments;
    return block_decode_picture_batch(ci, {kDstRgba8, rgba, nullptr, 0}, blocks, frames, blocksStride, width, height, frameStride, rowBytes,
                                      stream);
}

unsigned int HapB200EncodeBatch(unsigned int count, const void **textures, unsigned long *textureStrides,
                                unsigned long *textureBytes, unsigned int *textureFormats, unsigned int *compressors,
                                unsigned int *chunkCounts, unsigned int frames, void *out, unsigned long outStride,
                                unsigned long long *used, void *stream)
{
    if (count == 0 || count > 2 || !textures || !textureStrides || !textureBytes || !textureFormats || !compressors ||
        !chunkCounts || frames == 0 || !out || !used)
        return HapResult_Bad_Arguments;
    TextureArgs ta[2];
    for (unsigned i = 0; i < count; i++) {
        if (chunkCounts[i] == 0 || !textures[i] || ((uintptr_t)textures[i] | textureStrides[i]) % 16) return HapResult_Bad_Arguments;
        ta[i] = TextureArgs{textureBytes[i], textureFormats[i], compressors[i], chunkCounts[i]};
        if (validate_texture_args(ta[i]) != HapResult_No_Error) return HapResult_Bad_Arguments;
    }
    if (!texture_formats_ok(count, textureFormats)) return HapResult_Bad_Arguments;
    if (outStride < HapMaxEncodedLength(count, textureBytes, textureFormats, chunkCounts)) return HapResult_Buffer_Too_Small;
    FrameGeom G;
    uint32_t r = build_frame_geom(count, ta, G);
    if (r != HapResult_No_Error) return r;
    HAP_ENTER(out, textures[0]);
    const uint8_t *base = (const uint8_t *)textures[0];
    for (unsigned i = 0; i < count; i++) {
        G.s[i].in_offset = (uint64_t)((const uint8_t *)textures[i] - base);  // wraps for i = 1 when below base; 64-bit add undoes it
        G.s[i].in_stride = textureStrides[i];
    }
    return on_batch_stream(stream, [&](cudaStream_t st) -> uint32_t { return launch_encode(base, G, frames, (uint8_t *)out, outStride, used, st); });
}

unsigned int HapB200EncodeRGBABatch(const void *rgba, unsigned int frames, unsigned long frameStride, unsigned int width,
                                    unsigned int height, unsigned long rowBytes, unsigned int codec, unsigned int compressor,
                                    unsigned int chunkCount, void *out, unsigned long outStride, unsigned long long *used,
                                    void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci) || !codec_encodes(ci)) return HapResult_Bad_Arguments;
    return encode_picture_batch(ci, rgba_picture(rgba), frames, frameStride, width, height, rowBytes, compressor, chunkCount, out, outStride, used, stream);
}

unsigned int HapB200EncodeRGBA(const void *rgba, unsigned int width, unsigned int height, unsigned long rowBytes,
                               unsigned int codec, unsigned int compressor, unsigned int chunkCount, void *outputBuffer,
                               unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    CodecInfo ci;
    if (!codec_info(codec, ci) || !codec_encodes(ci)) return HapResult_Bad_Arguments;
    return encode_picture(ci, rgba_picture(rgba), width, height, rowBytes, compressor, chunkCount, outputBuffer, outputBufferBytes, outputBufferBytesUsed);
}

// ---- Hap R encoding: RGBA8 -> BC7 (bc7_encode.cuh), the RGBA8 encoders' plumbing with the Hap7 codec -------------------

unsigned int HapB200EncodeRGBABC7(const void *rgba, unsigned int width, unsigned int height, unsigned long rowBytes,
                                  unsigned int compressor, unsigned int chunkCount, void *outputBuffer,
                                  unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    return encode_picture(bc7_codec(), rgba_picture(rgba), width, height, rowBytes, compressor, chunkCount, outputBuffer, outputBufferBytes, outputBufferBytesUsed);
}

unsigned int HapB200EncodeRGBABC7Batch(const void *rgba, unsigned int frames, unsigned long frameStride, unsigned int width,
                                       unsigned int height, unsigned long rowBytes, unsigned int compressor, unsigned int chunkCount,
                                       void *out, unsigned long outStride, unsigned long long *used, void *stream)
{
    return encode_picture_batch(bc7_codec(), rgba_picture(rgba), frames, frameStride, width, height, rowBytes, compressor, chunkCount, out, outStride, used,
                             stream);
}

unsigned int HapB200BlockEncodeBC7Batch(const void *rgba, unsigned int frames, unsigned long frameStride, unsigned int width,
                                        unsigned int height, unsigned long rowBytes, void *blocks, unsigned long blocksStride, void *stream)
{
    return block_encode_picture_batch(bc7_codec(), rgba_picture(rgba), frames, frameStride, width, height, rowBytes, blocks, blocksStride, stream);
}

// ---- NV12 / P010 -> Hap, Hap Alpha, Hap Q, Hap Q Alpha: the picture encoders with a YUV source (yuv_source.cuh) ----------

unsigned int HapB200EncodeYUV(const void *luma, const void *chroma, unsigned int width, unsigned int height, unsigned long pitch,
                              unsigned int layout, unsigned int colorSpace, unsigned int codec, unsigned int compressor,
                              unsigned int chunkCount, void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    CodecInfo ci;
    if (!yuv_args_ok(layout, colorSpace, codec, ci)) return HapResult_Bad_Arguments;
    return encode_picture(ci, yuv_picture(luma, chroma, layout, colorSpace), width, height, pitch, compressor, chunkCount, outputBuffer,
                          outputBufferBytes, outputBufferBytesUsed);
}

unsigned int HapB200EncodeYUVBatch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride, unsigned int width,
                                   unsigned int height, unsigned long pitch, unsigned int layout, unsigned int colorSpace, unsigned int codec,
                                   unsigned int compressor, unsigned int chunkCount, void *out, unsigned long outStride,
                                   unsigned long long *used, void *stream)
{
    CodecInfo ci;
    if (!yuv_args_ok(layout, colorSpace, codec, ci)) return HapResult_Bad_Arguments;
    return encode_picture_batch(ci, yuv_picture(luma, chroma, layout, colorSpace), frames, frameStride, width, height, pitch, compressor,
                                chunkCount, out, outStride, used, stream);
}

unsigned int HapB200BlockEncodeYUVBatch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                        unsigned int width, unsigned int height, unsigned long pitch, unsigned int layout,
                                        unsigned int colorSpace, unsigned int codec, void *blocks, unsigned long blocksStride, void *stream)
{
    CodecInfo ci;
    if (!yuv_args_ok(layout, colorSpace, codec, ci)) return HapResult_Bad_Arguments;
    return block_encode_picture_batch(ci, yuv_picture(luma, chroma, layout, colorSpace), frames, frameStride, width, height, pitch, blocks,
                                      blocksStride, stream);
}

// ---- planar Y'CbCr 4:2:0 / 4:2:2 / 4:4:4 (+ alpha) -> Hap, Hap Alpha, Hap Q, Hap Q Alpha, Hap Alpha-Only: the picture
// encoders with a planar source (yuv_source.cuh) ----------------------------------------------------------------------------

unsigned int HapB200EncodePlanar(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int width, unsigned int height,
                                 unsigned long lumaPitch, unsigned long chromaPitch, unsigned int subsampling, unsigned int bitDepth,
                                 unsigned int colorSpace, unsigned int codec, unsigned int compressor, unsigned int chunkCount,
                                 void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    CodecInfo ci;
    if (!planar_args_ok(alpha, subsampling, bitDepth, colorSpace, codec, ci)) return HapResult_Bad_Arguments;
    return encode_picture(ci, planar_picture(ci, luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace), width, height, lumaPitch,
                          compressor, chunkCount, outputBuffer, outputBufferBytes, outputBufferBytesUsed);
}

unsigned int HapB200EncodePlanarBatch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                      unsigned long frameStride, unsigned int width, unsigned int height, unsigned long lumaPitch,
                                      unsigned long chromaPitch, unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace,
                                      unsigned int codec, unsigned int compressor, unsigned int chunkCount, void *out, unsigned long outStride,
                                      unsigned long long *used, void *stream)
{
    CodecInfo ci;
    if (!planar_args_ok(alpha, subsampling, bitDepth, colorSpace, codec, ci)) return HapResult_Bad_Arguments;
    return encode_picture_batch(ci, planar_picture(ci, luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace), frames, frameStride,
                                width, height, lumaPitch, compressor, chunkCount, out, outStride, used, stream);
}

unsigned int HapB200BlockEncodePlanarBatch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                           unsigned long frameStride, unsigned int width, unsigned int height, unsigned long lumaPitch,
                                           unsigned long chromaPitch, unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace,
                                           unsigned int codec, void *blocks, unsigned long blocksStride, void *stream)
{
    CodecInfo ci;
    if (!planar_args_ok(alpha, subsampling, bitDepth, colorSpace, codec, ci)) return HapResult_Bad_Arguments;
    return block_encode_picture_batch(ci, planar_picture(ci, luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace), frames,
                                      frameStride, width, height, lumaPitch, blocks, blocksStride, stream);
}

// ---- NV12 / P010 and planar Y'CbCr (+ alpha) -> Hap R: the picture encoders with a YUV or planar source and the Hap7 codec;
// launch_block_encode converts to RGBA8, then runs the RGBA8 BC7 kernel (launch_bc7_from_yuv) ------------------------------

unsigned int HapB200EncodeYUVBC7(const void *luma, const void *chroma, unsigned int width, unsigned int height, unsigned long pitch,
                                 unsigned int layout, unsigned int colorSpace, unsigned int compressor, unsigned int chunkCount,
                                 void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    if (!yuv_format_ok(layout, colorSpace) || !bc7_rgba_width_ok(width)) return HapResult_Bad_Arguments;
    return encode_picture(bc7_codec(), yuv_picture(luma, chroma, layout, colorSpace), width, height, pitch, compressor, chunkCount, outputBuffer,
                          outputBufferBytes, outputBufferBytesUsed);
}

unsigned int HapB200EncodeYUVBC7Batch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride, unsigned int width,
                                      unsigned int height, unsigned long pitch, unsigned int layout, unsigned int colorSpace,
                                      unsigned int compressor, unsigned int chunkCount, void *out, unsigned long outStride,
                                      unsigned long long *used, void *stream)
{
    if (!yuv_format_ok(layout, colorSpace) || !bc7_rgba_width_ok(width)) return HapResult_Bad_Arguments;
    return encode_picture_batch(bc7_codec(), yuv_picture(luma, chroma, layout, colorSpace), frames, frameStride, width, height, pitch, compressor,
                                chunkCount, out, outStride, used, stream);
}

unsigned int HapB200BlockEncodeYUVBC7Batch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                           unsigned int width, unsigned int height, unsigned long pitch, unsigned int layout,
                                           unsigned int colorSpace, void *blocks, unsigned long blocksStride, void *stream)
{
    if (!yuv_format_ok(layout, colorSpace) || !bc7_rgba_width_ok(width)) return HapResult_Bad_Arguments;
    return block_encode_picture_batch(bc7_codec(), yuv_picture(luma, chroma, layout, colorSpace), frames, frameStride, width, height, pitch,
                                      blocks, blocksStride, stream);
}

unsigned int HapB200EncodePlanarBC7(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int width,
                                    unsigned int height, unsigned long lumaPitch, unsigned long chromaPitch, unsigned int subsampling,
                                    unsigned int bitDepth, unsigned int colorSpace, unsigned int compressor, unsigned int chunkCount,
                                    void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    if (!planar_format_ok(subsampling, bitDepth, colorSpace) || !bc7_rgba_width_ok(width)) return HapResult_Bad_Arguments;
    const CodecInfo ci = bc7_codec();
    return encode_picture(ci, planar_picture(ci, luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace), width, height, lumaPitch,
                          compressor, chunkCount, outputBuffer, outputBufferBytes, outputBufferBytesUsed);
}

unsigned int HapB200EncodePlanarBC7Batch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                         unsigned long frameStride, unsigned int width, unsigned int height, unsigned long lumaPitch,
                                         unsigned long chromaPitch, unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace,
                                         unsigned int compressor, unsigned int chunkCount, void *out, unsigned long outStride,
                                         unsigned long long *used, void *stream)
{
    if (!planar_format_ok(subsampling, bitDepth, colorSpace) || !bc7_rgba_width_ok(width)) return HapResult_Bad_Arguments;
    const CodecInfo ci = bc7_codec();
    return encode_picture_batch(ci, planar_picture(ci, luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace), frames, frameStride,
                                width, height, lumaPitch, compressor, chunkCount, out, outStride, used, stream);
}

unsigned int HapB200BlockEncodePlanarBC7Batch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                              unsigned long frameStride, unsigned int width, unsigned int height, unsigned long lumaPitch,
                                              unsigned long chromaPitch, unsigned int subsampling, unsigned int bitDepth,
                                              unsigned int colorSpace, void *blocks, unsigned long blocksStride, void *stream)
{
    if (!planar_format_ok(subsampling, bitDepth, colorSpace) || !bc7_rgba_width_ok(width)) return HapResult_Bad_Arguments;
    const CodecInfo ci = bc7_codec();
    return block_encode_picture_batch(ci, planar_picture(ci, luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace), frames,
                                      frameStride, width, height, lumaPitch, blocks, blocksStride, stream);
}

unsigned int HapB200DecodeBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                unsigned int index, unsigned int maxChunks, void *out, unsigned long outStride,
                                unsigned long long *used, unsigned int *formats, unsigned int *results, void *stream)
{
    if (!in || !inBytes || !out || !used || !formats || !results || frames == 0 || maxChunks == 0 || index > 1)
        return HapResult_Bad_Arguments;
    HAP_ENTER(in, out);
    return on_batch_stream(stream, [&](cudaStream_t st) -> uint32_t {
        return launch_decode_batch((const uint8_t *)in, frames, inStride, inBytes, index, maxChunks, (uint8_t *)out, outStride, outStride,
                                   used, formats, results, st);
    });
}

unsigned int HapB200DecodeRGBABatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                    unsigned int maxChunks, unsigned int codec, unsigned int width, unsigned int height, void *rgba,
                                    unsigned long frameStride, unsigned long rowBytes, unsigned int *results, void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci)) return HapResult_Bad_Arguments;
    return decode_picture_batch(ci, {kDstRgba8, rgba, nullptr, 0}, in, frames, inStride, inBytes, maxChunks, width, height, frameStride, rowBytes,
                                results, stream);
}

unsigned int HapB200DecodeRGBA(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height,
                               void *rgba, unsigned long rowBytes)
{
    return decode_picture({kDstRgba8, rgba, nullptr, 0}, inputBuffer, inputBufferBytes, width, height, rowBytes);
}

// ---- Hap, Hap Alpha, Hap Q, Hap Q Alpha, Hap Alpha-Only, Hap R -> NV12 / P010: K8 with a YUV sink (yuv_sink.cuh) ----------

unsigned int HapB200BlockDecodeYUVBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                        unsigned int height, unsigned int codec, void *luma, void *chroma, unsigned long frameStride,
                                        unsigned long pitch, unsigned int layout, unsigned int colorSpace, void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci) || !yuv_out_args_ok(layout, colorSpace)) return HapResult_Bad_Arguments;
    return block_decode_picture_batch(ci, yuv_out_picture(luma, chroma, layout, colorSpace), blocks, frames, blocksStride, width, height,
                                      frameStride, pitch, stream);
}

unsigned int HapB200DecodeYUVBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                   unsigned int maxChunks, unsigned int codec, unsigned int width, unsigned int height, void *luma,
                                   void *chroma, unsigned long frameStride, unsigned long pitch, unsigned int layout, unsigned int colorSpace,
                                   unsigned int *results, void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci) || !yuv_out_args_ok(layout, colorSpace)) return HapResult_Bad_Arguments;
    return decode_picture_batch(ci, yuv_out_picture(luma, chroma, layout, colorSpace), in, frames, inStride, inBytes, maxChunks, width, height,
                                frameStride, pitch, results, stream);
}

unsigned int HapB200DecodeYUV(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height, void *luma,
                              void *chroma, unsigned long pitch, unsigned int layout, unsigned int colorSpace)
{
    if (!yuv_out_args_ok(layout, colorSpace)) return HapResult_Bad_Arguments;
    return decode_picture(yuv_out_picture(luma, chroma, layout, colorSpace), inputBuffer, inputBufferBytes, width, height, pitch);
}

// ---- Hap, Hap Alpha, Hap Q, Hap Q Alpha, Hap Alpha-Only, Hap R -> planar Y'CbCr 4:2:0 / 4:2:2 / 4:4:4 (+ alpha): K8 with a
// planar sink (planar_sink.cuh); Hap Alpha-Only writes its alpha plane alone --------------------------------------------------

unsigned int HapB200BlockDecodePlanarBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                           unsigned int height, unsigned int codec, void *luma, void *cb, void *cr, void *alpha,
                                           unsigned long frameStride, unsigned long lumaPitch, unsigned long chromaPitch,
                                           unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace, void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci) || !planar_out_args_ok(subsampling, bitDepth, colorSpace)) return HapResult_Bad_Arguments;
    const PictureDst d = planar_out_picture(luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace);
    return block_decode_picture_batch(ci, ci.bc_kind == kBcRgtc1 ? alpha_only_picture(d) : d, blocks, frames, blocksStride, width, height,
                                      frameStride, lumaPitch, stream);
}

unsigned int HapB200DecodePlanarBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                      unsigned int maxChunks, unsigned int codec, unsigned int width, unsigned int height,
                                      void *luma, void *cb, void *cr, void *alpha, unsigned long frameStride,
                                      unsigned long lumaPitch, unsigned long chromaPitch, unsigned int subsampling,
                                      unsigned int bitDepth, unsigned int colorSpace, unsigned int *results, void *stream)
{
    CodecInfo ci;
    if (!codec_info(codec, ci) || !planar_out_args_ok(subsampling, bitDepth, colorSpace)) return HapResult_Bad_Arguments;
    const PictureDst d = planar_out_picture(luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace);
    return decode_picture_batch(ci, ci.bc_kind == kBcRgtc1 ? alpha_only_picture(d) : d, in, frames, inStride, inBytes, maxChunks, width,
                                height, frameStride, lumaPitch, results, stream);
}

unsigned int HapB200DecodePlanar(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height,
                                 void *luma, void *cb, void *cr, void *alpha, unsigned long lumaPitch, unsigned long chromaPitch,
                                 unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace)
{
    if (!planar_out_args_ok(subsampling, bitDepth, colorSpace)) return HapResult_Bad_Arguments;
    return decode_picture(planar_out_picture(luma, cb, cr, alpha, chromaPitch, subsampling, bitDepth, colorSpace), inputBuffer,
                          inputBufferBytes, width, height, lumaPitch);
}

// ---- Hap HDR -> RGBA16F: BC6H (bc6h_decode.cuh) ----

unsigned int HapB200BlockDecodeHalfBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                         unsigned int height, unsigned int textureFormat, void *rgbaHalf, unsigned long frameStride,
                                         unsigned long rowBytes, void *stream)
{
    CodecInfo ci;
    if (!bc6h_codec(textureFormat, ci)) return HapResult_Bad_Arguments;
    return block_decode_picture_batch(ci, {kDstRgbaHalf, rgbaHalf, nullptr, 0}, blocks, frames, blocksStride, width, height, frameStride,
                                      rowBytes, stream);
}

unsigned int HapB200DecodeRGBAHalfBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                        unsigned int maxChunks, unsigned int width, unsigned int height, void *rgbaHalf,
                                        unsigned long frameStride, unsigned long rowBytes, unsigned int *results, void *stream)
{
    return decode_picture_batch(hap_hdr_batch_codec(), {kDstRgbaHalf, rgbaHalf, nullptr, 0}, in, frames, inStride, inBytes, maxChunks, width,
                                height, frameStride, rowBytes, results, stream);
}

unsigned int HapB200DecodeRGBAHalf(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height,
                                   void *rgbaHalf, unsigned long rowBytes)
{
    return decode_picture({kDstRgbaHalf, rgbaHalf, nullptr, 0}, inputBuffer, inputBufferBytes, width, height, rowBytes);
}

// ---- Hap HDR encoding: RGBA16F -> BC6H (bc6h_encode.cuh) ----

unsigned int HapB200BlockEncodeHalfBatch(const void *rgbaHalf, unsigned int frames, unsigned long frameStride, unsigned int width,
                                         unsigned int height, unsigned long rowBytes, unsigned int textureFormat, void *blocks,
                                         unsigned long blocksStride, void *stream)
{
    CodecInfo ci;
    if (!bc6h_codec(textureFormat, ci)) return HapResult_Bad_Arguments;
    return block_encode_picture_batch(ci, rgba_half_picture(rgbaHalf), frames, frameStride, width, height, rowBytes, blocks, blocksStride,
                                      stream);
}

// (the Hap HDR batch encoders alone refuse an `out` or outStride that is not 16-byte aligned)
unsigned int HapB200EncodeRGBAHalfBatch(const void *rgbaHalf, unsigned int frames, unsigned long frameStride, unsigned int width,
                                        unsigned int height, unsigned long rowBytes, unsigned int textureFormat, unsigned int compressor,
                                        unsigned int chunkCount, void *out, unsigned long outStride, unsigned long long *used, void *stream)
{
    CodecInfo ci;
    if (!bc6h_codec(textureFormat, ci) || ((uintptr_t)out | outStride) % 16) return HapResult_Bad_Arguments;
    return encode_picture_batch(ci, rgba_half_picture(rgbaHalf), frames, frameStride, width, height, rowBytes, compressor, chunkCount, out,
                                outStride, used, stream);
}

unsigned int HapB200EncodeRGBAHalf(const void *rgbaHalf, unsigned int width, unsigned int height, unsigned long rowBytes,
                                   unsigned int textureFormat, unsigned int compressor, unsigned int chunkCount, void *outputBuffer,
                                   unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    CodecInfo ci;
    if (!bc6h_codec(textureFormat, ci)) return HapResult_Bad_Arguments;
    return encode_picture(ci, rgba_half_picture(rgbaHalf), width, height, rowBytes, compressor, chunkCount, outputBuffer, outputBufferBytes,
                          outputBufferBytesUsed);
}

// ---- Hap HDR encoding from HDR10: P010, BT.2020, PQ -> BC6H, the Hap HDR encoders with the kSrcP010Pq source (yuv_source.cuh) ----

unsigned int HapB200EncodeYUVPQ(const void *luma, const void *chroma, unsigned int width, unsigned int height, unsigned long pitch,
                                unsigned int colorSpace, unsigned int unitNits, unsigned int textureFormat, unsigned int compressor,
                                unsigned int chunkCount, void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed)
{
    CodecInfo ci;
    if (!yuv_pq_args_ok(colorSpace, unitNits) || !bc6h_codec(textureFormat, ci)) return HapResult_Bad_Arguments;
    return encode_picture(ci, yuv_pq_picture(luma, chroma, colorSpace, unitNits), width, height, pitch, compressor, chunkCount, outputBuffer,
                          outputBufferBytes, outputBufferBytesUsed);
}

unsigned int HapB200EncodeYUVPQBatch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride, unsigned int width,
                                     unsigned int height, unsigned long pitch, unsigned int colorSpace, unsigned int unitNits,
                                     unsigned int textureFormat, unsigned int compressor, unsigned int chunkCount, void *out,
                                     unsigned long outStride, unsigned long long *used, void *stream)
{
    CodecInfo ci;
    if (!yuv_pq_args_ok(colorSpace, unitNits) || !bc6h_codec(textureFormat, ci) || ((uintptr_t)out | outStride) % 16)
        return HapResult_Bad_Arguments;
    return encode_picture_batch(ci, yuv_pq_picture(luma, chroma, colorSpace, unitNits), frames, frameStride, width, height, pitch, compressor,
                                chunkCount, out, outStride, used, stream);
}

unsigned int HapB200BlockEncodeYUVPQBatch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                          unsigned int width, unsigned int height, unsigned long pitch, unsigned int colorSpace,
                                          unsigned int unitNits, unsigned int textureFormat, void *blocks, unsigned long blocksStride,
                                          void *stream)
{
    CodecInfo ci;
    if (!yuv_pq_args_ok(colorSpace, unitNits) || !bc6h_codec(textureFormat, ci)) return HapResult_Bad_Arguments;
    return block_encode_picture_batch(ci, yuv_pq_picture(luma, chroma, colorSpace, unitNits), frames, frameStride, width, height, pitch, blocks,
                                      blocksStride, stream);
}

// ---- Hap HDR -> HDR10: BC6H -> P010, BT.2020, PQ, K8 with the HDR10 sink (yuv_sink.cuh) ----

unsigned int HapB200BlockDecodeYUVPQBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                          unsigned int height, unsigned int textureFormat, void *luma, void *chroma, unsigned long frameStride,
                                          unsigned long pitch, unsigned int colorSpace, unsigned int unitNits, void *stream)
{
    CodecInfo ci;
    if (!bc6h_codec(textureFormat, ci) || !yuv_pq_args_ok(colorSpace, unitNits)) return HapResult_Bad_Arguments;
    return block_decode_picture_batch(ci, {kDstP010Pq, luma, chroma, colorSpace, unitNits}, blocks, frames, blocksStride, width, height,
                                      frameStride, pitch, stream);
}

unsigned int HapB200DecodeYUVPQBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                     unsigned int maxChunks, unsigned int width, unsigned int height, void *luma, void *chroma,
                                     unsigned long frameStride, unsigned long pitch, unsigned int colorSpace, unsigned int unitNits,
                                     unsigned int *results, void *stream)
{
    if (!yuv_pq_args_ok(colorSpace, unitNits)) return HapResult_Bad_Arguments;
    return decode_picture_batch(hap_hdr_batch_codec(), {kDstP010Pq, luma, chroma, colorSpace, unitNits}, in, frames, inStride, inBytes,
                                maxChunks, width, height, frameStride, pitch, results, stream);
}

unsigned int HapB200DecodeYUVPQ(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height, void *luma,
                                void *chroma, unsigned long pitch, unsigned int colorSpace, unsigned int unitNits)
{
    if (!yuv_pq_args_ok(colorSpace, unitNits)) return HapResult_Bad_Arguments;
    return decode_picture({kDstP010Pq, luma, chroma, colorSpace, unitNits}, inputBuffer, inputBufferBytes, width, height, pitch);
}

// ---- include/hap_mov.h: QuickTime sample tables around Hap frames (host code only) -------------------------

unsigned int HapB200MovFourCCForFrame(const void *frame, unsigned long frameBytes, unsigned int *fourcc)
{
    if (!frame || !fourcc) return HapResult_Bad_Arguments;
    unsigned int count = 0, f0 = 0, f1 = 0;
    if (HapGetFrameTextureCount(frame, frameBytes, &count) != HapResult_No_Error || count < 1 || count > 2) return HapResult_Bad_Frame;
    if (HapGetFrameTextureFormat(frame, frameBytes, 0, &f0) != HapResult_No_Error) return HapResult_Bad_Frame;
    if (count == 2 && HapGetFrameTextureFormat(frame, frameBytes, 1, &f1) != HapResult_No_Error) return HapResult_Bad_Frame;
    // HapVideoDRAFT.md:132-142
    char c = 0;
    if (count == 1) {
        switch (f0) {
        case HapTextureFormat_RGB_DXT1: c = '1'; break;
        case HapTextureFormat_RGBA_DXT5: c = '5'; break;
        case HapTextureFormat_YCoCg_DXT5: c = 'Y'; break;
        case HapTextureFormat_A_RGTC1: c = 'A'; break;
        case HapTextureFormat_RGBA_BPTC_UNORM: c = '7'; break;
        case HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT:
        case HapTextureFormat_RGB_BPTC_SIGNED_FLOAT: c = 'H'; break;
        default: break;
        }
    } else if ((f0 == HapTextureFormat_YCoCg_DXT5 && f1 == HapTextureFormat_A_RGTC1) ||
               (f1 == HapTextureFormat_YCoCg_DXT5 && f0 == HapTextureFormat_A_RGTC1)) {
        c = 'M';
    }
    if (!c) return HapResult_Bad_Frame;
    *fourcc = HAPB200_FOURCC('H', 'a', 'p', c);
    return HapResult_No_Error;
}

HapB200Mov *HapB200MovOpen(const char *path) { return hapmov::open_read(path); }

unsigned int HapB200MovInfo(const HapB200Mov *mov, unsigned int *fourcc, unsigned int *width, unsigned int *height,
                            unsigned long *frameCount, unsigned int *timescale, unsigned long *duration)
{
    if (!mov) return HapResult_Bad_Arguments;
    if (fourcc) *fourcc = mov->fourcc;
    if (width) *width = mov->width;
    if (height) *height = mov->height;
    if (frameCount) *frameCount = (unsigned long)mov->size.size();
    if (timescale) *timescale = mov->timescale;
    if (duration) *duration = (unsigned long)mov->duration;
    return HapResult_No_Error;
}

unsigned long HapB200MovFrameBytes(const HapB200Mov *mov, unsigned long index)
{
    return (mov && index < mov->size.size()) ? mov->size[index] : 0;
}

unsigned int HapB200MovReadFrame(HapB200Mov *mov, unsigned long index, void *buffer, unsigned long bufferBytes,
                                 unsigned long *bytesUsed, unsigned int *durationTicks)
{
    if (!mov || mov->writing || !buffer || index >= mov->size.size()) return HapResult_Bad_Arguments;
    const unsigned long n = mov->size[index];
    if (n > bufferBytes) return HapResult_Buffer_Too_Small;
    if (fseeko(mov->f, (off_t)mov->offset[index], SEEK_SET) != 0 || fread(buffer, 1, n, mov->f) != n) return HapResult_Internal_Error;
    if (bytesUsed) *bytesUsed = n;
    if (durationTicks) *durationTicks = mov->ticks[index];
    return HapResult_No_Error;
}

HapB200Mov *HapB200MovCreate(const char *path, unsigned int fourcc, unsigned int width, unsigned int height, unsigned int timescale)
{
    return hapmov::create(path, fourcc, width, height, timescale);
}

unsigned int HapB200MovWriteFrame(HapB200Mov *mov, const void *frame, unsigned long frameBytes, unsigned int durationTicks)
{
    return hapmov::write_frame(mov, frame, frameBytes, durationTicks);
}

unsigned int HapB200MovClose(HapB200Mov *mov)
{
    if (!mov) return HapResult_No_Error;
    unsigned int r = HapResult_No_Error;
    if (mov->writing) r = hapmov::finish(mov);
    if (mov->f && fclose(mov->f) != 0 && r == HapResult_No_Error) r = HapResult_Internal_Error;
    delete mov;
    return r;
}

}  // extern "C"
