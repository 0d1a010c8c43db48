// hap_b200/csrc/hapq_fused.cuh -- Hap Q from RGBA8 in one kernel: the scaled-YCoCg block fit of K1-K4 in front of K5.
//
// The two-kernel path writes the DXT texture to HBM (bc_encode_kernel<kBcYCoCg>) and reads it back (K5).  Here the CTA
// that compresses a fragment fits the fragment's blocks itself, straight into the fragment's shared-memory image: one launch
// instead of two, the texture is not read back, and the barrier-free fit of one resident CTA can issue while the other
// waits on the compressor's barriers and shared-memory round trips (DESIGN.md §4 and §6 give what that bought: 0.6 ms of
// 12.9 per 444 4K frames).  The blocks are still written through to
// the texture scratch, because the plan and place kernels copy a chunk (hap.c:460) or the whole section (hap.c:478) from
// it when compression does not pay.  Same shape as K5 (persistent grid, 512 threads, two CTAs per SM, EncodeSmem), same
// block fit (encode_ycocg_dxt5), same compressor: the frames are byte-identical to those of the two-kernel path.
#pragma once
#include "bc_encode.cuh"
#include "snappy_encode.cuh"

#ifndef HAPB200_FUSED_HAPQ
#define HAPB200_FUSED_HAPQ 1   // 0: the library never selects the fused kernel (A/B builds)
#endif

namespace hapb200 {

// The texture geometries the fused kernel takes: one compressed section cut into whole chunks of whole 16-byte blocks, so that
// every block lies in exactly one fragment and every fragment starts at a block.
HAP_HD bool fused_hapq_geometry(const FrameGeom &G)
{
    const SectionGeom &s = G.s[0];
    return G.sections == 1 && s.compress && (uint64_t)s.chunks * s.chunk_bytes == s.bytes && s.chunk_bytes % 16 == 0;
}

// rgba: RGBA8 pictures (geometry B: B.frame_bytes apart, rows B.row_bytes apart; B.out_stride is not used); tex: the texture
// scratch that G describes (16-byte aligned), written through; the other arguments are those of snappy_encode_fragments_kernel.
__global__ void __launch_bounds__(kEncThreads, 2) hapq_fused_encode_kernel(
    const uint8_t *__restrict__ rgba, BcGeom B, uint8_t *__restrict__ tex, FrameGeom G, uint32_t nfrag, uint8_t *__restrict__ scratch,
    uint32_t *__restrict__ frag_size, uint8_t *__restrict__ frag_entries)
{
    HAP_DYN_SMEM(smem_raw);
    const uint32_t t = threadIdx.x;
    for (uint32_t gfrag = blockIdx.x; gfrag < nfrag; gfrag += gridDim.x) {
        {
            EncodeSmem &S = *reinterpret_cast<EncodeSmem *>(smem_raw);
            // The fit: block blk0 + lb (lb = t, t + 512, ... < nblk) is fitted, stored to S.data and written through.  Lanes
            // take neighbouring blocks, so the four 16-byte row loads of a warp are coalesced as in bc_encode_kernel, and so
            // are the 16-byte stores.  The fit alone needs more than 64 registers (bc_encode_kernel gives it 72; capped at
            // 64 it spills even in a kernel that does nothing else, here 7 values per block), so nothing else may live across it: only lb,
            // nblk, blk0 and frame do, and the picture and texture addresses are derived from them for every block (the
            // empty asm keeps the compiler from hoisting them out of the loop, where they would be spilled too).
            const FragRef cur = locate_fragment(tex, G, gfrag);
            const uint32_t nblk = cur.units >> 1, blk0 = cur.tex_off >> 4;
            uint32_t frame = cur.frame;
#pragma unroll 1
            for (uint32_t lb = t; lb < nblk; lb += kEncThreads) {
                asm volatile("" : "+r"(frame));
                const uint32_t bi = blk0 + lb;
                uint32_t bx, by, px[16];
                block_xy(bi, B.blocks_x, B.inv_blocks_x, bx, by);
                load_block_rgba8(rgba + (uint64_t)frame * B.frame_bytes, B.row_bytes, bx, by, px);
                Block8 a, c;
                encode_ycocg_dxt5<false>(px, a, c);
                const uint4 v = make_uint4(a.lo, a.hi, c.lo, c.hi);
                reinterpret_cast<uint4 *>(S.data)[lb] = v;
                reinterpret_cast<uint4 *>(tex + (uint64_t)frame * G.s[0].in_stride + G.s[0].in_offset)[bi] = v;
            }
            init_fragment_tables(S);
        }
        __syncthreads();
        // the fragment again, recomputed rather than kept live across the fit; each thread reloads its own strip.  The
        // compressor's shared-memory addresses are derived after the fit too: the empty asm hides that `off` is 0, so the
        // compiler cannot hoist them to the top of the kernel, where they would be spilled around the fit.
        uint32_t off = 0;
        asm volatile("" : "+r"(off));
        EncodeSmem &S = *reinterpret_cast<EncodeSmem *>(smem_raw + off);
        const uint32_t U = locate_fragment(tex, G, gfrag).units;
        const uint32_t i0 = t * kUnitStrip;
        uint2 d[kUnitStrip];
#pragma unroll
        for (int k = 0; k < kUnitStrip; k += 2) {
            const uint4 v = i0 + k < U ? *reinterpret_cast<const uint4 *>(&S.data[i0 + k]) : make_uint4(0, 0, 0, 0);   // (U is even)
            d[k] = make_uint2(v.x, v.y);
            d[k + 1] = make_uint2(v.z, v.w);
        }
        const uint32_t total = U == (uint32_t)kFragUnits ? compress_fragment<true>(S, d, U, 2) : compress_fragment<false>(S, d, U, 2);
        store_fragment(S, total, gfrag, scratch, frag_size, frag_entries);
    }
}

}  // namespace hapb200
