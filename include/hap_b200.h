/*
 * include/hap_b200.h -- extensions of libhap_b200.so beyond the reference's hap.h.
 *
 * The reference API starts at DXT bytes and moves one frame per call through host memory
 * (Vidvox/hap source/hap.h:98-137).  A GPU is only busy when whole streams of frames stay in
 * HBM, so these entry points add (a) the RGBA side of the path -- the block compressors that sit
 * upstream of HapEncode and the block decoder downstream of HapDecode -- and (b) batched,
 * device-resident, stream-ordered variants.  Plain C ABI: pointers, sizes, no CUDA types (a stream is
 * passed as void*, NULL = the library's own stream; the call then returns after the work finished).
 * Results are HapResult values (hap.h).
 */
#ifndef hap_b200_h
#define hap_b200_h
#include "hap.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Hap flavours by FourCC (reference documentation/HapVideoDRAFT.md:132-142) */
enum HapB200Codec {
    HapB200Codec_Hap1 = 0, /* RGB DXT1                         "Hap"            */
    HapB200Codec_Hap5 = 1, /* RGBA DXT5                        "Hap Alpha"      */
    HapB200Codec_HapY = 2, /* scaled YCoCg DXT5                "Hap Q"          */
    HapB200Codec_HapM = 3, /* scaled YCoCg DXT5 + alpha RGTC1  "Hap Q Alpha"    */
    HapB200Codec_HapA = 4, /* alpha RGTC1                      "Hap Alpha-Only" */
    HapB200Codec_Hap7 = 5  /* RGBA BPTC (BC7) UNORM            "Hap R"          */
};
/* Hap R (Hap7): the codec-taking encoders HapB200EncodeRGBA, HapB200EncodeRGBABatch and HapB200BlockEncodeBatch refuse it
 * with HapResult_Bad_Arguments (a BC7 search costs far more per block than the DXT encoders, so a caller asks for it by
 * name): HapB200EncodeRGBABC7, HapB200EncodeRGBABC7Batch and HapB200BlockEncodeBC7Batch encode it.  HapEncode and
 * HapB200EncodeBatch wrap BC7 textures that were compressed elsewhere.  The RGBA decoders turn BC7 blocks into RGBA8 exactly as the BPTC specification defines them,
 * reserved blocks (first byte 0) included: those decode to (0, 0, 0, 0) in all 16 texels. */

const char *HapB200Version(void);
/* kernels launched by this library in this process so far (bench.py reports the delta) */
unsigned long long HapB200KernelLaunchCount(void);
/* Devices.  One process can drive every GPU of the box: a call with a device pointer among its buffers runs on that
 * pointer's device; a call with host pointers only runs on the default device -- the device that was current in the
 * thread that made the library's first call, or the one set here (-1: forget it).  The caller's current device is
 * restored before a call returns.  HapB200SetDevice returns 0, or -1 for an ordinal out of range. */
int HapB200SetDevice(int device);
int HapB200GetDevice(void);

/* Delivery rings: frames encoded on one GPU written STRAIGHT into memory of another GPU of the box.
 * Frames of a stream are independent (HapVideoDRAFT.md:29-34), so N GPUs encode N frames at once; the consumer (a muxer, a
 * file writer) sits next to ONE of them.  A ring is device memory on the consumer's GPU.  Producers -- other processes
 * (CUDA IPC) or other threads of this process -- pass an address inside it as the `out` (and `used`) argument of
 * HapB200EncodeRGBABatch / HapB200EncodeBatch: the kernel that lays the frame out stores it over NVLink / NVSwitch into the
 * consumer's memory, so there is no second pass over the encoded bytes (no staging copy, no collective).
 *   consumer:  HapB200RingCreate(device, bytes, &ring, handle)        -- handle: 64 bytes to hand to the producers
 *   producer:  HapB200RingOpen(device, handle, &ring)                 -- other process; maps the ring, enables peer access
 *              HapB200RingAttach(device, ringDevice)                  -- same process: enables peer access, use `ring` as is
 *              ... HapB200EncodeRGBABatch(..., out = ring + slot, ..., stream) ...
 *              HapB200RingPublish(device, ring + flagOffset, value, stream)  -- after everything queued on `stream` so far
 *   consumer:  HapB200RingWait(device, ring + flagOffset, value, timeoutMs, stream)  -- work queued on `stream` afterwards sees
 *              the frames.  timeoutMs 0: wait for ever, as a stream memory operation (cuStreamWaitValue32: no SM is occupied);
 *              timeoutMs > 0: a one-thread polling kernel that gives up after that long (a dead producer cannot hold the GPU).
 *              Queue a wait BEHIND the work of its own device that it depends on (a producer on the consumer's GPU publishes
 *              first, then the wait is queued): streams can share a hardware queue, and a wait at its head holds back what
 *              follows in it.  Producers on other GPUs are independent of the consumer's queues.
 * Layout inside the ring (slots, flags, lengths) is the caller's; flags are 4-byte words, 4-byte aligned, that only grow.
 * Results: HapResult values (hap.h).  Close / Destroy synchronise the device. */
#define HAPB200_RING_HANDLE_BYTES 64
unsigned int HapB200RingCreate(int device, unsigned long bytes, void **ring, void *handle);
unsigned int HapB200RingDestroy(int device, void *ring);
unsigned int HapB200RingOpen(int device, const void *handle, void **ring);
unsigned int HapB200RingClose(int device, void *ring);
unsigned int HapB200RingAttach(int device, int ringDevice);
unsigned int HapB200RingPublish(int device, void *flag, unsigned int value, void *stream);
unsigned int HapB200RingWait(int device, const void *flag, unsigned int value, unsigned int timeoutMs, void *stream);

/* Options.  HAPB200_OPTION_USE_INDEX: the decoder uses a frame's embedded fragment index when it finds one (default 1;
 * 0 = always derive the index from the Snappy streams, as for every frame another encoder wrote).
 * HAPB200_OPTION_WRITE_INDEX: the encoder adds a private "fragment index" section to the Decode Instructions container
 * of the texture sections it compresses (default 0: frames are laid out byte for byte as hap.c:430-442 lays them out).
 * The section is skipped by the reference decoder (hap.c:701-704) and by FFmpeg; it lets this decoder start at every
 * 32 KiB fragment without walking the chunk's element chain first (hap_b200/csrc/hap_index.h; ~1 % of the frame size).
 * Returns 0, or -1 for an unknown option. */
#define HAPB200_OPTION_USE_INDEX 1
#define HAPB200_OPTION_WRITE_INDEX 2
/* HAPB200_OPTION_WRITE_OFFSET_TABLE: Complex texture sections carry the optional Chunk Offset Table (reference
 * documentation/HapVideoDRAFT.md:126-128; honoured by the reference decoder, hap.c:697-700 and :800-803, and by FFmpeg) and
 * every chunk starts on a 16-byte boundary of the frame, the few bytes between chunks being zero.  Default 0: the
 * reference's encoder never writes this table and packs chunks back to back (hap.c:473). */
#define HAPB200_OPTION_WRITE_OFFSET_TABLE 3
/* HAPB200_OPTION_CHROMA_REFINE: the scaled-YCoCg block encoders (Hap Q, Hap Q Alpha) score the 5-bit Co' endpoint
 * candidates of blocks with less than one grid cell of Co' extent by their true error (every texel re-assigned) instead of
 * with the clusters of the unquantised fit held fixed.  Closes the encoder's one deficit against the cluster-fit oracle
 * beyond the 0.1 dB bar (slow colour ramps, 1080p: -0.47 dB -> -0.06 dB; video content +0.61 -> +0.65 dB) for +60-70 % block-encode
 * time on 4K footage (half of its blocks qualify).  Default 0.  Environment: HAPB200_CHROMA_REFINE. */
#define HAPB200_OPTION_CHROMA_REFINE 4
int HapB200SetOption(int option, int value);

/* Per-stage device timing for profiling runs: when enabled every kernel launch is bracketed by CUDA
 * events on its own stream.  HapB200StageTimes synchronises, returns milliseconds and launch counts
 * per stage (bc_encode, snappy_encode, plan, place, parse, snappy_decode, collect, bc_decode, snappy_index, windows) and
 * resets them; its return value is the number of stages. */
void HapB200SetStageTiming(int enabled);
int HapB200StageTimes(double *ms, unsigned long long *launches, int n);

/* worst-case frame size for a width x height frame of `codec` (HapMaxEncodedLength on its textures) */
unsigned long HapB200MaxEncodedLengthRGBA(unsigned int width, unsigned int height, unsigned int codec,
                                          unsigned int chunkCount);
/* bytes of texture `index` (0 or 1) of a width x height frame of `codec`; 0 when absent */
unsigned long HapB200TextureBytes(unsigned int width, unsigned int height, unsigned int codec, unsigned int index);

/* Limits of every RGBA picture below (HapB200EncodeRGBA .. HapB200BlockDecodeBatch): rowBytes is at most
 * HAPB200_MAX_ROW_BYTES and (width/4)*(height/4) at most HAPB200_MAX_BLOCKS; larger values are refused with
 * HapResult_Bad_Arguments.  A batch may hold any number of frames. */
#define HAPB200_MAX_ROW_BYTES 0xFFFFFFFFul
#define HAPB200_MAX_BLOCKS 0xFFFFFFFFul

/* One RGBA8 frame (row-major, rowBytes stride, width/height multiples of 4) -> one Hap frame.
 * Host or device pointers.  Fuses block compression, Snappy and frame assembly on the GPU. */
unsigned int HapB200EncodeRGBA(const void *rgba, unsigned int width, unsigned int height, unsigned long rowBytes,
                               unsigned int codec, unsigned int compressor, unsigned int chunkCount,
                               void *outputBuffer, unsigned long outputBufferBytes,
                               unsigned long *outputBufferBytesUsed);

/* One Hap frame -> RGBA8 (all textures of the frame combined; YCoCg converted, alpha merged).  Hap HDR (BC6H) frames
 * decode to half floats instead (HapB200DecodeRGBAHalf below); here they return HapResult_Bad_Frame. */
unsigned int HapB200DecodeRGBA(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width,
                               unsigned int height, void *rgba, unsigned long rowBytes);

/* ---- device-resident batches: every pointer below is a DEVICE pointer, 16-byte aligned ---------- */

/* frames x RGBA8 -> frames x Hap frame at out + f*outStride, encoded length in used[f] (device). */
unsigned int HapB200EncodeRGBABatch(const void *rgba, unsigned int frames, unsigned long frameStride,
                                    unsigned int width, unsigned int height, unsigned long rowBytes,
                                    unsigned int codec, unsigned int compressor, unsigned int chunkCount,
                                    void *out, unsigned long outStride, unsigned long long *used, void *stream);

/* HapEncode over a batch: texture t of frame f at textures[t] + f*textureStrides[t]. */
unsigned int HapB200EncodeBatch(unsigned int count, const void **textures, unsigned long *textureStrides,
                                unsigned long *textureBytes, unsigned int *textureFormats,
                                unsigned int *compressors, unsigned int *chunkCounts, unsigned int frames,
                                void *out, unsigned long outStride, unsigned long long *used, void *stream);

/* HapDecode over a batch: frame f at in + f*inStride with inBytes[f] bytes -> texture `index` at
 * out + f*outStride; per frame used[f], formats[f], results[f] (HapResult) are device arrays.
 * maxChunks bounds the chunk count of any frame (frames with more report Bad_Arguments). */
unsigned int HapB200DecodeBatch(const void *in, unsigned int frames, unsigned long inStride,
                                const unsigned long long *inBytes, unsigned int index, unsigned int maxChunks,
                                void *out, unsigned long outStride, unsigned long long *used,
                                unsigned int *formats, unsigned int *results, void *stream);

/* Decode straight to RGBA8: HapDecode of every texture + block decode (+ YCoCg, + alpha merge).
 * codec = the HapB200Codec of the stream (its FourCC); frames of another flavour report Bad_Frame. */
unsigned int HapB200DecodeRGBABatch(const void *in, unsigned int frames, unsigned long inStride,
                                    const unsigned long long *inBytes, unsigned int maxChunks,
                                    unsigned int codec, unsigned int width, unsigned int height, void *rgba,
                                    unsigned long frameStride, unsigned long rowBytes, unsigned int *results,
                                    void *stream);

/* Block codecs alone (K1-K4 / K8), batched: kind = HapB200Codec; HapM writes/reads the YCoCg plane at
 * blocks and the RGTC1 plane at blocks + HapB200TextureBytes(.., 0).  Hap7 (BC7) decodes only here (encode: HapB200BlockEncodeBC7Batch).  BC6H blocks: see
 * HapB200BlockDecodeHalfBatch. */
unsigned int HapB200BlockEncodeBatch(const void *rgba, unsigned int frames, unsigned long frameStride,
                                     unsigned int width, unsigned int height, unsigned long rowBytes,
                                     unsigned int codec, void *blocks, unsigned long blocksStride, void *stream);
unsigned int HapB200BlockDecodeBatch(const void *blocks, unsigned int frames, unsigned long blocksStride,
                                     unsigned int width, unsigned int height, unsigned int codec, void *rgba,
                                     unsigned long frameStride, unsigned long rowBytes, void *stream);

/* ---- Hap HDR (BC6H, "HapH") -> RGBA16F ---------------------------------------------------------------------------------
 * BC6H decodes to half floats: every pixel is 8 bytes, four IEEE binary16 values R, G, B, A, with A = 1.0 (0x3C00).
 * Blocks decode exactly as the BPTC specification defines them, UF16 (HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT) or SF16
 * (HapTextureFormat_RGB_BPTC_SIGNED_FLOAT), interpolation rounding (+32) included.  Every output is finite: an SF16
 * endpoint of -32768 (mode 14) is taken as -32767, whose scaled magnitude is the largest finite half.  A negative value
 * whose magnitude scales to 0 is written as +0 (0x0000), as the specification's integer form gives it.  The four reserved
 * mode values decode to (0, 0, 0, 1.0).  Geometry as for the RGBA8 entry points with 8 bytes per pixel: width and height
 * multiples of 4, 8 * width <= rowBytes <= HAPB200_MAX_ROW_BYTES, at most HAPB200_MAX_BLOCKS blocks; the batch entry points
 * take device pointers, 16-byte aligned rows, pictures and strides, and any number of frames. */

/* One Hap HDR frame (host or device pointers) -> RGBA16F.  A frame that is not one BC6H texture of exactly
 * (width/4)*(height/4)*16 bytes returns HapResult_Bad_Frame. */
unsigned int HapB200DecodeRGBAHalf(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width,
                                   unsigned int height, void *rgbaHalf, unsigned long rowBytes);
/* HapB200DecodeRGBABatch for Hap HDR: each frame decodes as its own texture says (UF16 or SF16).  A frame that is not one
 * BC6H texture of exactly (width/4)*(height/4)*16 bytes (another format, a larger or smaller texture, a second texture)
 * reports Bad_Frame in results[f], as HapB200DecodeRGBAHalf answers for it; other failures keep the chunk decoder's code;
 * the picture of a failed frame is all zero bytes. */
unsigned int HapB200DecodeRGBAHalfBatch(const void *in, unsigned int frames, unsigned long inStride,
                                        const unsigned long long *inBytes, unsigned int maxChunks, unsigned int width,
                                        unsigned int height, void *rgbaHalf, unsigned long frameStride,
                                        unsigned long rowBytes, unsigned int *results, void *stream);
/* HapB200BlockDecodeBatch for BC6H blocks: textureFormat = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT or
 * HapTextureFormat_RGB_BPTC_SIGNED_FLOAT (anything else: HapResult_Bad_Arguments). */
unsigned int HapB200BlockDecodeHalfBatch(const void *blocks, unsigned int frames, unsigned long blocksStride,
                                         unsigned int width, unsigned int height, unsigned int textureFormat,
                                         void *rgbaHalf, unsigned long frameStride, unsigned long rowBytes, void *stream);

/* ---- Hap HDR (BC6H, "HapH") <- RGBA16F --------------------------------------------------------------------------------
 * The encoders take RGBA16F pictures (8 bytes per pixel, binary16 R, G, B, A; A is ignored) and write BC6H blocks of
 * textureFormat = HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT (UF16) or HapTextureFormat_RGB_BPTC_SIGNED_FLOAT (SF16);
 * anything else is refused with HapResult_Bad_Arguments.  A frame holds one BC6H texture, whose section type is
 * textureFormat (HapGetFrameTextureFormat reports it).  Geometry as for the RGBA16F decoders: width and height multiples of
 * 4, 8 * width <= rowBytes <= HAPB200_MAX_ROW_BYTES, at most HAPB200_MAX_BLOCKS blocks; the batch entry points take device
 * pointers, with rows, pictures, strides, out and blocks 16-byte aligned, and any number of frames.  compressor and
 * chunkCount as for HapB200EncodeRGBA.  The output of a frame needs
 *     HapMaxEncodedLength(1, {(width/4)*(height/4)*16}, {textureFormat}, {chunkCount})
 * bytes (outputBufferBytes, outStride); less is refused with HapResult_Buffer_Too_Small.
 * Input rules, applied to R, G and B before the search:
 *   UF16: negative values, -0 and NaN encode as 0; +Inf as 65504 (0x7BFF).
 *   SF16: NaN encodes as 0; +-Inf as +-65504; -0 as +0.
 * After them, a block whose 16 texels hold one colour decodes bit-exactly to that colour (mode 14, a 16-bit base with zero
 * deltas, represents every finite half of either signedness).  Each block is chosen by its exact error after decoding:
 * the squared difference of decoded and source halves taken as sign-magnitude integers, summed over R, G and B. */

/* one RGBA16F picture (host or device pointers) -> one Hap HDR frame */
unsigned int HapB200EncodeRGBAHalf(const void *rgbaHalf, unsigned int width, unsigned int height, unsigned long rowBytes,
                                   unsigned int textureFormat, unsigned int compressor, unsigned int chunkCount,
                                   void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);
/* frames x RGBA16F (device) -> frames x Hap HDR frame at out + f*outStride, encoded length in used[f] (device) */
unsigned int HapB200EncodeRGBAHalfBatch(const void *rgbaHalf, unsigned int frames, unsigned long frameStride,
                                        unsigned int width, unsigned int height, unsigned long rowBytes,
                                        unsigned int textureFormat, unsigned int compressor, unsigned int chunkCount,
                                        void *out, unsigned long outStride, unsigned long long *used, void *stream);
/* frames x RGBA16F (device) -> bare BC6H textures at blocks + f*blocksStride */
unsigned int HapB200BlockEncodeHalfBatch(const void *rgbaHalf, unsigned int frames, unsigned long frameStride,
                                         unsigned int width, unsigned int height, unsigned long rowBytes,
                                         unsigned int textureFormat, void *blocks, unsigned long blocksStride, void *stream);

/* ---- Hap R (BC7, "Hap7") <- RGBA8 ----------------------------------------------------------------------------------------
 * The encoders take RGBA8 pictures and write BPTC (BC7) RGBA UNORM blocks.  Geometry, alignment, compressor and chunkCount as
 * for HapB200EncodeRGBA / HapB200EncodeRGBABatch / HapB200BlockEncodeBatch.  A frame holds one texture of format
 * HapTextureFormat_RGBA_BPTC_UNORM and needs HapB200MaxEncodedLengthRGBA(width, height, HapB200Codec_Hap7, chunkCount)
 * bytes (outputBufferBytes, outStride); less is refused with HapResult_Buffer_Too_Small.  Arguments are checked before
 * anything touches the GPU.
 * Each block is chosen by its exact error after decoding: the sum over R, G, B and A of the squared differences of decoded
 * and source 8-bit values, unweighted.  Rules:
 *   - a block whose 16 texels hold one RGBA colour decodes bit-exactly to that colour (mode 5, rotation 0, colour index 1
 *     between two 7-bit endpoints per channel, both alpha endpoints at A);
 *   - a block whose texels all have A = 255 decodes with A = 255 in all 16 texels (modes 0-3 always do; modes 4-7 keep the
 *     channel that decodes to A at its top code, in modes 6 and 7 with p-bits 1);
 *   - no reserved block (first byte 0) is ever written.
 * A BC7 search costs orders of magnitude more per block than the DXT encoders (DESIGN.md section 6). */

/* one RGBA8 picture (host or device pointers) -> one Hap R frame */
unsigned int HapB200EncodeRGBABC7(const void *rgba, unsigned int width, unsigned int height, unsigned long rowBytes,
                                  unsigned int compressor, unsigned int chunkCount,
                                  void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);
/* frames x RGBA8 (device) -> frames x Hap R frame at out + f*outStride, encoded length in used[f] (device) */
unsigned int HapB200EncodeRGBABC7Batch(const void *rgba, unsigned int frames, unsigned long frameStride,
                                       unsigned int width, unsigned int height, unsigned long rowBytes,
                                       unsigned int compressor, unsigned int chunkCount,
                                       void *out, unsigned long outStride, unsigned long long *used, void *stream);
/* frames x RGBA8 (device) -> bare BC7 textures at blocks + f*blocksStride */
unsigned int HapB200BlockEncodeBC7Batch(const void *rgba, unsigned int frames, unsigned long frameStride,
                                        unsigned int width, unsigned int height, unsigned long rowBytes,
                                        void *blocks, unsigned long blocksStride, void *stream);

#ifdef __cplusplus
}
#endif
#endif
