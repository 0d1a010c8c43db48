// hap_b200/csrc/bc_encode.cuh -- K1-K4 kernels: RGBA8 frames -> DXT1 / DXT5 / scaled-YCoCg-DXT5 / RGTC1 blocks.
//
// One thread per 4x4 block (see bc_block.cuh for why).  Memory shape: thread t of a warp owns block
// column bx0+t, so for each of the four pixel rows the warp reads 32 x 16 B = 512 contiguous bytes
// (LDG.128, fully coalesced) and writes 32 x 8/16 B contiguous block bytes (STG.64 / STG.128): HBM sees
// each RGBA byte once and each DXT byte once, no shared-memory staging needed for coalescing.
// Block order is row-major over (width/4) x (height/4), the order S3TC textures are uploaded in and
// the order hap.c:450 slices into chunks.
#pragma once
#include "bc_block.cuh"

namespace hapb200 {

enum BcKind : int { kBcDxt1 = 0, kBcDxt5 = 1, kBcYCoCg = 2, kBcRgtc1 = 3, kBcYCoCgPlusAlpha = 4 };

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

// grid = (ceil(blocks/kBcThreads), frames).  REFINE: the chroma endpoint refinement of the YCoCg kinds (bc_block.cuh).
template <int KIND, bool REFINE = false>
__global__ void __launch_bounds__(kBcThreads, (KIND == kBcYCoCg && !REFINE) ? 7 : (KIND == kBcDxt1 || KIND == kBcDxt5) ? 5 : HAPB200_BC_MIN_BLOCKS) bc_encode_kernel(const uint8_t *__restrict__ rgba, BcGeom G,
                                                                uint8_t *__restrict__ out)
{
    const uint32_t nblocks = G.blocks_x * G.blocks_y;
    const uint32_t bi = blockIdx.x * kBcThreads + threadIdx.x;
    if (bi >= nblocks) return;
    uint32_t by = __umulhi(bi, G.inv_blocks_x), bx = bi - by * G.blocks_x;  // the estimate is exact or one short
    if (bx >= G.blocks_x) { by++; bx -= G.blocks_x; }
    const uint8_t *src = rgba + (uint64_t)blockIdx.y * G.frame_bytes + (uint64_t)(4 * by) * G.row_bytes + 16u * bx;
    uint32_t px[16];
#pragma unroll
    for (int row = 0; row < 4; row++) {
        uint4 v = *reinterpret_cast<const uint4 *>(src + (uint64_t)row * G.row_bytes);
        px[4 * row + 0] = v.x; px[4 * row + 1] = v.y; px[4 * row + 2] = v.z; px[4 * row + 3] = v.w;
    }
    uint8_t *o = out + (uint64_t)blockIdx.y * G.out_stride;
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

}  // namespace hapb200
