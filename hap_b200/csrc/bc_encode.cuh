// hap_b200/csrc/bc_encode.cuh -- K1-K4 kernels: RGBA8 (or NV12 / P010, or planar Y'CbCr) frames -> DXT1 / DXT5 /
// scaled-YCoCg-DXT5 / RGTC1 / BC7 blocks, and the Y'CbCr -> RGBA8 pass that BC7 takes from Y'CbCr pictures.
//
// One thread per 4x4 block (see bc_block.cuh for why).  Memory shape: thread t of a warp owns block
// column bx0+t, so for each of the four pixel rows the warp reads 32 x 16 B = 512 contiguous bytes
// (LDG.128, fully coalesced) and writes 32 x 8/16 B contiguous block bytes (STG.64 / STG.128): HBM sees
// each RGBA byte once and each DXT byte once, no shared-memory staging needed for coalescing.
// Block order is row-major over (width/4) x (height/4), the order S3TC textures are uploaded in and
// the order hap.c:450 slices into chunks.
#pragma once
#include "bc_block.cuh"
#include "bc7_encode.cuh"
#include "yuv_source.cuh"

namespace hapb200 {

// kBcBc7: BPTC RGBA UNORM (Hap R), block math in bc7_encode.cuh (encode) and bc7_decode.cuh (decode).  The codec-taking RGBA
// encode entry points refuse it; the BC7 entry points ask for it by name.
enum BcKind : int { kBcDxt1 = 0, kBcDxt5 = 1, kBcYCoCg = 2, kBcRgtc1 = 3, kBcYCoCgPlusAlpha = 4, kBcBc7 = 5 };

constexpr int kBcThreads = 128;
#ifndef HAPB200_BC_MIN_BLOCKS
#define HAPB200_BC_MIN_BLOCKS 1      // resident CTAs asked for (= register cap).  Hap Q: 7 = the 72 registers the kernel needs anyway (without the bound the
                                     // compiler takes 76 and loses a CTA); RGB kinds: 5, a cap of 102 registers (sm_90a: 95-96 used, no spills)
#endif

struct BcGeom {
    uint32_t blocks_x, blocks_y;   // width/4, height/4
    uint32_t row_bytes;            // RGBA row stride in bytes (>= 16*blocks_x, multiple of 16)
    uint32_t inv_blocks_x;         // floor(2^32 / blocks_x): row index by multiply-high + one correction (no division)
    uint64_t frame_bytes;          // RGBA frame stride
    uint64_t out_stride;           // DXT bytes per frame in `out`
    uint64_t second_offset;        // kBcYCoCgPlusAlpha: offset of the RGTC1 plane inside a frame's output
};

// The geometry of width x height pictures (multiples of 4, at most 2^32 - 1 blocks), rows row_bytes apart.
HAP_HD BcGeom bc_encode_geom(uint32_t width, uint32_t height, uint32_t row_bytes, uint64_t frame_bytes, uint64_t out_stride,
                             uint64_t second_offset)
{
    BcGeom g;
    g.blocks_x = width / 4;
    g.blocks_y = height / 4;
    g.row_bytes = row_bytes;
    const uint64_t inv = 0x100000000ull / g.blocks_x;          // 2^32 when the image is one block wide
    g.inv_blocks_x = inv > 0xFFFFFFFFull ? 0xFFFFFFFFu : (uint32_t)inv;
    g.frame_bytes = frame_bytes;
    g.out_stride = out_stride;
    g.second_offset = second_offset;
    return g;
}

// CTAs per frame of the block kernels (encode and decode): one thread per block
HAP_HD uint32_t bc_ctas(uint32_t blocks_x, uint32_t blocks_y) { return (uint32_t)(((uint64_t)blocks_x * blocks_y + kBcThreads - 1) / kBcThreads); }

// Column and row of block bi (row-major) without a division: the multiply-high estimate of the row is exact or one short.
__device__ __forceinline__ void block_xy(uint32_t bi, uint32_t blocks_x, uint32_t inv_blocks_x, uint32_t &bx, uint32_t &by)
{
    by = __umulhi(bi, inv_blocks_x);
    bx = bi - by * blocks_x;
    if (bx >= blocks_x) { by++; bx -= blocks_x; }
}

// The 16 texels of block (bx, by) of the RGBA8 picture at `pic`: one 16-byte load per pixel row.
__device__ __forceinline__ void load_block_rgba8(const uint8_t *pic, uint32_t row_bytes, uint32_t bx, uint32_t by, uint32_t px[16])
{
    const uint8_t *src = pic + (uint64_t)(4 * by) * row_bytes + 16u * bx;
#pragma unroll
    for (int row = 0; row < 4; row++) {
        uint4 v = *reinterpret_cast<const uint4 *>(src + (uint64_t)row * row_bytes);
        px[4 * row + 0] = v.x; px[4 * row + 1] = v.y; px[4 * row + 2] = v.z; px[4 * row + 3] = v.w;
    }
}

// The frame is blockIdx.y, and gridDim.y is at most 65535: batches of more frames are launched in slices of this many.
constexpr uint32_t kBcFramesPerLaunch = 65535;

// Resident CTAs each kind asks for (= its register cap).  kBcBc7 asks for one (a cap of 255 registers): its exact-error
// search holds more state than any register cap would keep.
constexpr int bc_encode_min_ctas(int kind, bool refine)
{
    return (kind == kBcYCoCg && !refine) ? 7 : (kind == kBcDxt1 || kind == kBcDxt5) ? 5 : kind == kBcBc7 ? 1 : HAPB200_BC_MIN_BLOCKS;
}

// The fit of block bi from its texels px and its store into this frame's output o (both encode kernels)
template <int KIND, bool REFINE>
__device__ __forceinline__ void bc_encode_store(const uint32_t px[16], const BcGeom &G, uint8_t *o, uint32_t bi)
{
    if (KIND == kBcDxt1) {
        Block8 c = encode_dxt1(px);
        reinterpret_cast<uint2 *>(o)[bi] = make_uint2(c.lo, c.hi);
    } else if (KIND == kBcRgtc1) {
        Block8 a = encode_rgtc1_alpha(px);
        reinterpret_cast<uint2 *>(o)[bi] = make_uint2(a.lo, a.hi);
    } else if (KIND == kBcDxt5) {
        Block8 a, c;
        encode_dxt5(px, a, c);
        reinterpret_cast<uint4 *>(o)[bi] = make_uint4(a.lo, a.hi, c.lo, c.hi);
    } else if (KIND == kBcBc7) {
        uint32_t w[4];
        bc7_encode_block(px, w);
        reinterpret_cast<uint4 *>(o)[bi] = make_uint4(w[0], w[1], w[2], w[3]);
    } else {
        Block8 a, c;
        encode_ycocg_dxt5<REFINE>(px, a, c);
        reinterpret_cast<uint4 *>(o)[bi] = make_uint4(a.lo, a.hi, c.lo, c.hi);
        if (KIND == kBcYCoCgPlusAlpha) {
            Block8 al = encode_rgtc1_alpha(px);
            reinterpret_cast<uint2 *>(o + G.second_offset)[bi] = make_uint2(al.lo, al.hi);
        }
    }
}

// grid = (bc_ctas, frames).  REFINE: the chroma endpoint refinement of the YCoCg kinds (bc_block.cuh).
// SRC (BcSource): kSrcRgba8 reads `rgba` as RGBA8 rows; kSrcNv12 / kSrcP010 read it as the luma plane and Y.chroma as the
// chroma plane (yuv_source.cuh), both frame_bytes apart per frame, and convert before the fit.  Y comes last so that the
// parameters of the RGBA8 instantiations keep their offsets.
template <int KIND, bool REFINE = false, int SRC = kSrcRgba8>
__global__ void __launch_bounds__(kBcThreads, bc_encode_min_ctas(KIND, REFINE)) bc_encode_kernel(const uint8_t *__restrict__ rgba, BcGeom G,
                                                                uint8_t *__restrict__ out, YuvSrc Y = YuvSrc())
{
    const uint32_t nblocks = G.blocks_x * G.blocks_y;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= nblocks) return;
    uint32_t bx, by;
    block_xy(bi, G.blocks_x, G.inv_blocks_x, bx, by);
    uint32_t px[16];
    if (SRC == kSrcRgba8) {
        load_block_rgba8(rgba + (uint64_t)blockIdx.y * G.frame_bytes, G.row_bytes, bx, by, px);
    } else {
        const uint64_t f = (uint64_t)blockIdx.y * G.frame_bytes;
        load_block_yuv<SRC>(rgba + f, Y.chroma + f, G.row_bytes, bx, by, G.blocks_x, G.blocks_y, Y, px);
    }
    bc_encode_store<KIND, REFINE>(px, G, out + (uint64_t)blockIdx.y * G.out_stride, bi);
}

// The same kernel for the planar sources (SRC: kSrcPlanar*, yuv_source.cuh): `luma` is the luma plane, P holds the chroma
// and alpha planes, all frame_bytes apart per frame.  A kernel of its own, so that the parameters, and so the -Xptxas -v
// lines, of bc_encode_kernel's instantiations stay as they are.  KIND kBcRgtc1 reads the alpha plane alone.
template <int KIND, bool REFINE, int SRC>
__global__ void __launch_bounds__(kBcThreads, bc_encode_min_ctas(KIND, REFINE)) bc_encode_planar_kernel(const uint8_t *__restrict__ luma, BcGeom G,
                                                                       uint8_t *__restrict__ out, PlanarSrc P)
{
    const uint32_t nblocks = G.blocks_x * G.blocks_y;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= nblocks) return;
    uint32_t bx, by;
    block_xy(bi, G.blocks_x, G.inv_blocks_x, bx, by);
    const uint64_t f = (uint64_t)blockIdx.y * G.frame_bytes;
    PlanarSrc p = P;
    p.m.chroma += f;
    p.cr += f;
    if (p.alpha) p.alpha += f;
    uint32_t px[16];
    constexpr bool kAlpha = KIND == kBcDxt5 || KIND == kBcYCoCgPlusAlpha || KIND == kBcRgtc1;
    load_block_planar<SRC, KIND != kBcRgtc1, kAlpha>(luma + f, G.row_bytes, bx, by, G.blocks_x, G.blocks_y, p, px);
    bc_encode_store<KIND, REFINE>(px, G, out + (uint64_t)blockIdx.y * G.out_stride, bi);
}

// The first of BC7's two passes from a Y'CbCr picture (Hap R from NV12 / P010 or planar pictures): the picture -> a tight
// RGBA8 picture, which bc_encode_kernel<kBcBc7> then encodes unchanged.  The DXT kinds fuse the conversion into their fit;
// BC7 does not, because each source would instantiate the whole BC7 search again (minutes of build and more spills each),
// and the RGBA8 round trip costs three orders of magnitude less than the search (DESIGN.md section 4).
// grid = (bc_ctas, frames), one thread per 4x4 block.  The block encoders' own loaders convert (load_block_yuv for
// kSrcNv12 / kSrcP010, load_block_planar with alpha for kSrcPlanar*), so the picture is exactly the one the DXT encoders fit
// from.  G: the source (luma rows row_bytes apart, every plane frame_bytes apart per frame); out_stride is the RGBA8 frame
// stride, its rows 16*blocks_x bytes apart.  Y: the NV12 / P010 chroma plane and matrix; P: the planar ones (alpha nullptr:
// A = 255).  Each pixel row of the block is one 16-byte store.
template <int SRC>
__global__ void __launch_bounds__(kBcThreads) bc_source_to_rgba8_kernel(const uint8_t *__restrict__ luma, BcGeom G, uint8_t *__restrict__ rgba,
                                                                       YuvSrc Y, PlanarSrc P)
{
    const uint32_t nblocks = G.blocks_x * G.blocks_y;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= nblocks) return;
    uint32_t bx, by;
    block_xy(bi, G.blocks_x, G.inv_blocks_x, bx, by);
    const uint64_t f = (uint64_t)blockIdx.y * G.frame_bytes;
    uint32_t px[16];
    if constexpr (SRC == kSrcNv12 || SRC == kSrcP010) {
        load_block_yuv<SRC>(luma + f, Y.chroma + f, G.row_bytes, bx, by, G.blocks_x, G.blocks_y, Y, px);
    } else {
        PlanarSrc p = P;
        p.m.chroma += f;
        p.cr += f;
        if (p.alpha) p.alpha += f;
        load_block_planar<SRC, true, true>(luma + f, G.row_bytes, bx, by, G.blocks_x, G.blocks_y, p, px);
    }
    const uint64_t row = 16ull * G.blocks_x;
    uint8_t *o = rgba + (uint64_t)blockIdx.y * G.out_stride + 4 * by * row + 16ull * bx;
#pragma unroll
    for (int r = 0; r < 4; r++)
        *reinterpret_cast<uint4 *>(o + r * row) = make_uint4(px[4 * r + 0], px[4 * r + 1], px[4 * r + 2], px[4 * r + 3]);
}

}  // namespace hapb200
