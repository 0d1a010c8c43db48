// hap_b200/csrc/hap_index.h -- the private "fragment index" section this encoder can append to a frame, and that this
// decoder uses when it finds one.
//
// Why it exists.  A raw Snappy stream is serial: an element's position depends on the length of every element before
// it.  This encoder compresses a chunk as independent 32 KiB FRAGMENTS (snappy_encode.cuh) whose element streams are
// simply concatenated, so the chunk is an ordinary Snappy stream for every other decoder -- but a decoder that knows
// where each fragment's stream starts, and at which byte of every 128-byte piece of it the first element begins, can
// decode all pieces in parallel without walking the chain first.  That knowledge is ~1 % of the compressed size.
//
// Where it travels.  BEHIND the frame: a frame is one top-level section (a texture section, or the 0x0D wrapper around two
// of them, HapVideoDRAFT.md:36-85); the index is one more section of a type the format does not define, appended after it.
// Every decoder reads the first section header, works inside the length it states and never looks further: the reference
// (/root/reference/source/hap.c:932-991 walks [0, header + length) only; HapDecode's inputBufferBytes may exceed it),
// FFmpeg's hap decoder likewise (checked in tests/test_mov_cpu.py: frames with a trailing section decode to the same
// picture; a section INSIDE the Decode Instructions container, which hap.c:701-704 would skip, makes FFmpeg's parser
// lose its place, so the index does not go there).  A frame that carries the index decodes to the same bytes everywhere; a
// frame without it (every frame the reference writes) is indexed on the fly by snappy_index_kernel.
// Nothing in the index is trusted: the execute kernel checks that the entries describe exactly the element chain it
// walks (snappy_decode.cuh), and a chunk whose index does not hold up is decoded again as if it had none.  The fragments of
// an indexed chunk are decoded independently, without waiting for one another, so the index also claims that every copy
// reads inside its own fragment.  A copy that reaches before its fragment's start is legal Snappy (every other decoder
// follows it), so such a chunk is not an error: it is decoded again without the index, where windows wait for the windows
// their copies read.
//
// Layout: a section header (4 or 8 bytes, hap.c:137-187) of type kSecFragmentIndex, then the body (little endian, unaligned):
//   0   'H' 'B' '2' 'I'          magic
//   4   u8  version (1)
//   5   u8  sub_log2 (7)         an entry per 2^sub_log2 stream bytes of a fragment
//   6   u16 texture_count (1 or 2)
//   8   u32 frag_bytes (32768)   uncompressed bytes per fragment (the last fragment of a chunk may be shorter)
//   12  u32 chunk_count[2]       chunks of texture 0 / texture 1 (0 when absent); must equal the textures' own tables
//   20  u32 record_offset[chunk_count[0] + chunk_count[1]]   offset of a chunk's record from the start of the body;
//                                0 = no record (the chunk is stored raw, or the texture is not chunked at all)
//   ..  records.  Record of a chunk with nf = ceil(uncompressed / frag_bytes) fragments:
//         u16 stream_bytes[nf]                       length of each fragment's element stream
//         u8  entry[ ceil(stream_bytes[j] / 2^sub_log2) ]  for j = 0..nf-1, back to back:
//                                offset of the first element START inside that piece of the fragment's stream, 0xFF = none
//       The chunk's stream is varint(uncompressed) followed by the fragments' streams in order.
#pragma once
#include <stdint.h>

namespace hapb200 {

constexpr uint32_t kSecFragmentIndex = 0xFB;   // top-level section type of the trailing index (not a type the format defines)
constexpr uint32_t kIndexMagic = 0x49324248u;  // "HB2I" read as little-endian u32
constexpr uint32_t kIndexVersion = 1;
constexpr uint32_t kIndexSubLog2 = 7;
constexpr uint32_t kIndexHeaderBytes = 20;
constexpr uint32_t kIndexNoEntry = 0xFF;

}  // namespace hapb200
