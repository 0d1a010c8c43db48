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
 * name): HapB200EncodeRGBABC7, HapB200EncodeRGBABC7Batch and HapB200BlockEncodeBC7Batch encode it, and
 * HapB200Encode{YUV,Planar}BC7* encode it from NV12 / P010 and planar Y'CbCr pictures.  HapEncode and
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

/* ---- Hap, Hap Alpha, Hap Q, Hap Q Alpha <- NV12 / P010 ----------------------------------------------------------------------
 * The encoders take the 4:2:0 pictures a video decoder writes (NVDEC surfaces) and convert them to RGBA8 inside the block
 * encoder, so no RGBA picture is ever written.  Encoding a YUV picture gives exactly the bytes HapB200EncodeRGBA* gives for
 * the RGBA8 picture the conversion below makes of it.
 * Planes:
 *   HapB200YUV_NV12: luma is one byte per pixel; chroma is interleaved Cb, Cr byte pairs, width/2 pairs per row, height/2 rows.
 *   HapB200YUV_P010: the same shape in little-endian 16-bit words; the sample is word >> 6 (the low 6 bits are ignored).
 *   Both planes have the same row pitch (bytes), as NVDEC surfaces do.  chroma is a pointer of its own: NVDEC places it at
 *   pitch * surfaceHeight, not at pitch * height.  In a batch frame f's planes start at luma + f*frameStride and
 *   chroma + f*frameStride.
 * Geometry: width and height multiples of 4, width * (bytes per sample) <= pitch <= HAPB200_MAX_ROW_BYTES, at most
 * HAPB200_MAX_BLOCKS blocks.  The batch entry points take device pointers; luma, chroma, pitch, frameStride, out, outStride,
 * blocks and blocksStride are 16-byte aligned; a batch may hold any number of frames.
 * Codecs: HapB200Codec_Hap1, _Hap5, _HapY and _HapM, with A = 255.  HapB200Codec_HapA (the picture has no alpha) and
 * HapB200Codec_Hap7 (as for every codec-taking encoder) are refused with HapResult_Bad_Arguments, as are an unknown layout
 * or colour space.  Every argument is checked before anything touches the GPU.  Sizes (HapB200MaxEncodedLengthRGBA),
 * compressor, chunkCount, HapResult_Buffer_Too_Small and the index, offset-table and chroma-refine options behave exactly
 * as for HapB200EncodeRGBA*.
 * The conversion, exactly (n = 8 for NV12, 10 for P010):
 *   Chroma upsampling: bilinear, MPEG-2 / H.264 / HEVC default siting (chroma_sample_loc_type 0): chroma is co-sited with
 *   even luma columns and midway between luma rows 2j and 2j+1.  For luma (x, y), i = x/2 and j = y/2 (rounded down); the
 *   upsampled value in eighths is C8 = sum of wh*wv*C over: vertical weight 3 on row j and 1 on row j-1 (y even) or j+1
 *   (y odd); horizontal weight 2 on column i (x even), or 1 and 1 on columns i and i+1 (x odd).  Row and column indices are
 *   clamped to the chroma plane.
 *   Matrix: the Y'CbCr -> R'G'B' matrix of (Kr, Kb) = BT.601 (0.299, 0.114) or BT.709 (0.2126, 0.0722).  Limited range:
 *   luma offset 16 * 2^(n-8), luma scale 219 * 2^(n-8), chroma scale 224 * 2^(n-8); full range: luma offset 0, both
 *   scales 2^n - 1.  Chroma offset 2^(n-1).
 *   Fixed point: with the row {cy, crR, cbG, crG, cbB, yOff, cOff} of HAPB200_YUV_COEFFICIENTS below (each coefficient
 *   round(65536 * 255 * matrix entry / scale), the chroma ones divided by 8 more for the eighths; in limited range the NV12
 *   coefficients are 4 times the P010 ones, so a P010 picture whose samples are 4 times an NV12 picture's converts to the
 *   same RGBA), Yd = Y - yOff,
 *   Cb8d = Cb8 - 8*cOff and Cr8d = Cr8 - 8*cOff:
 *     R = (cy*Yd + crR*Cr8d + 32768) >> 16,  G = (cy*Yd + cbG*Cb8d + crG*Cr8d + 32768) >> 16,  B = (cy*Yd + cbB*Cb8d + 32768) >> 16,
 *   the shift arithmetic, each result clamped to 0..255 (samples outside the nominal range are not clamped first); A = 255. */
enum HapB200YUVLayout { HapB200YUV_NV12 = 0, HapB200YUV_P010 = 1 };
/* BT.2020 (non-constant luminance) is taken only by the HDR10 encoders below (HapB200EncodeYUVPQ*); HapB200EncodeYUV*
 * refuse it: BT.2020 into 8-bit Hap would need tone mapping. */
enum HapB200YUVColorSpace {
    HapB200YUV_BT601_Limited = 0,
    HapB200YUV_BT601_Full = 1,
    HapB200YUV_BT709_Limited = 2,
    HapB200YUV_BT709_Full = 3,
    HapB200YUV_BT2020_Limited = 4,
    HapB200YUV_BT2020_Full = 5
};
/* row layout * 4 + colorSpace: {cy, crR, cbG, crG, cbB, yOff, cOff} */
#define HAPB200_YUV_COEFFICIENTS                                                                                           \
    {                                                                                                                      \
        {76308, 13076, -3208, -6660, 16524, 16, 128},  /* NV12 BT.601 limited */                                           \
        {65536, 11485, -2819, -5850, 14516, 0, 128},   /* NV12 BT.601 full    */                                           \
        {76308, 14688, -1748, -4364, 17304, 16, 128},  /* NV12 BT.709 limited */                                           \
        {65536, 12901, -1535, -3835, 15201, 0, 128},   /* NV12 BT.709 full    */                                           \
        {19077, 3269, -802, -1665, 4131, 64, 512},     /* P010 BT.601 limited */                                           \
        {16336, 2863, -703, -1458, 3618, 0, 512},      /* P010 BT.601 full    */                                           \
        {19077, 3672, -437, -1091, 4326, 64, 512},     /* P010 BT.709 limited */                                           \
        {16336, 3216, -383, -956, 3789, 0, 512}        /* P010 BT.709 full    */                                           \
    }

/* one picture (host or device pointers) -> one Hap frame */
unsigned int HapB200EncodeYUV(const void *luma, const void *chroma, unsigned int width, unsigned int height,
                              unsigned long pitch, unsigned int layout, unsigned int colorSpace, unsigned int codec,
                              unsigned int compressor, unsigned int chunkCount,
                              void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);
/* frames x picture (device) -> frames x Hap frame at out + f*outStride, encoded length in used[f] (device) */
unsigned int HapB200EncodeYUVBatch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                   unsigned int width, unsigned int height, unsigned long pitch, unsigned int layout,
                                   unsigned int colorSpace, unsigned int codec, unsigned int compressor, unsigned int chunkCount,
                                   void *out, unsigned long outStride, unsigned long long *used, void *stream);
/* frames x picture (device) -> bare textures, as HapB200BlockEncodeBatch (HapM: the RGTC1 plane at blocks + HapB200TextureBytes(.., 0)) */
unsigned int HapB200BlockEncodeYUVBatch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                        unsigned int width, unsigned int height, unsigned long pitch, unsigned int layout,
                                        unsigned int colorSpace, unsigned int codec, void *blocks, unsigned long blocksStride,
                                        void *stream);

/* ---- Hap, Hap Alpha, Hap Q, Hap Q Alpha, Hap Alpha-Only <- planar Y'CbCr 4:2:0 / 4:2:2 / 4:4:4 (+ alpha) ---------------------
 * The encoders take the planar pictures software decoders and mastering formats give (FFmpeg's yuv420p, yuv422p10le,
 * yuva444p12le and their kin) and convert them to RGBA8 inside the block encoder, so no RGBA picture is ever written.
 * The arguments follow FFmpeg's AVFrame: luma, cb, cr and alpha are data[0], data[1], data[2] and data[3]; lumaPitch is
 * linesize[0] and chromaPitch is linesize[1] (= linesize[2]; alpha's rows are lumaPitch apart, as linesize[3] is).
 * Encoding a planar picture gives exactly the bytes HapB200EncodeRGBA* / HapB200BlockEncodeBatch give for the RGBA8 picture
 * the conversion below makes of it.
 * Planes:
 *   Luma and alpha: width x height samples, rows lumaPitch bytes apart.
 *   Cb and Cr: cw x ch samples, rows chromaPitch bytes apart; cw = width/2 for 4:2:0 and 4:2:2, width for 4:4:4; ch =
 *   height/2 for 4:2:0, height otherwise.
 *   In a batch, each of the four planes of frame f starts at its pointer + f*frameStride.
 * Samples: bitDepth 8: bytes.  bitDepth 10 or 12: little-endian 16-bit words with the sample in the low bits, as in FFmpeg's
 *   *p10le / *p12le; the sample is word & (2^n - 1), so higher bits are ignored.  Any other depth is refused.
 * Geometry: width and height multiples of 4, width*bytes <= lumaPitch <= HAPB200_MAX_ROW_BYTES, cw*bytes <= chromaPitch <=
 *   HAPB200_MAX_ROW_BYTES (bytes: 1 per sample at 8 bits, else 2), at most HAPB200_MAX_BLOCKS blocks.  The batch entry points
 *   take device pointers; the planes, both pitches, frameStride, out, outStride, blocks and blocksStride are 16-byte aligned.
 *   The single-frame call takes host or device memory at any alignment and pitch.
 * Codecs: HapB200Codec_Hap1 and _HapY do not read alpha.  _Hap5 and _HapM use alpha; a NULL alpha means A = 255.  _HapA
 *   requires alpha and reads only that plane: luma, cb and cr are neither read nor checked, and may be NULL.  _Hap7 (as for
 *   every codec-taking encoder) and unknown codecs are refused with HapResult_Bad_Arguments.
 * Colour spaces: BT.601 and BT.709, limited and full range; BT.2020 is refused, as for HapB200EncodeYUV*.
 * Every argument is checked before anything touches the GPU.  Sizes (HapB200MaxEncodedLengthRGBA), HapResult_Buffer_Too_Small,
 * compressor, chunkCount and the index, offset-table and chroma-refine options behave exactly as for HapB200EncodeRGBA*.
 * The conversion, exactly (n = bitDepth), extending that of HapB200EncodeYUV; chroma keeps its default siting (co-sited
 * with even luma columns; in 4:2:0 midway between luma rows):
 *   1. Chroma to eighths, C8 for luma (x, y), row and column indices clamped to the chroma plane:
 *      4:2:0: exactly HapB200EncodeYUV's upsampler (vertical weights 3 and 1, horizontal weights 2, or 1 and 1).
 *      4:2:2: vertical weight 4 on row y; for even x weight 2 on column i = x/2, for odd x weight 1 on columns i and i+1.
 *      4:4:4: C8 = 8*C.
 *   2. Matrix: n = 8: the NV12 rows of HAPB200_YUV_COEFFICIENTS with shift 16; n = 10: the P010 rows with shift 16 (a 10-bit
 *      sample has the value P010's word >> 6 has, so both are unchanged).  n = 12: the rows of HAPB200_YUV_12BIT_COEFFICIENTS
 *      below, each coefficient round(2^18 * 255 * matrix entry / scale), the chroma ones divided by 8 more (limited range:
 *      luma offset 256, luma scale 3504, chroma scale 3584; full range: offset 0, both scales 4095; chroma offset 2048), with
 *      R = (cy*Yd + crR*Cr8d + 2^17) >> 18, G and B likewise, each clamped to 0..255.  Every intermediate stays below 2^31.
 *      The limited rows equal the P010 rows, so 12-bit samples that are 4 times 10-bit ones convert identically.
 *   3. Alpha: A = (510*a + 2^n - 1) / (2*(2^n - 1)), integer division: 255*a / (2^n - 1) rounded half up (A = a at n = 8).
 *      Alpha is taken as given: no premultiplication is added or removed. */
enum HapB200ChromaSubsampling { HapB200Chroma_420 = 0, HapB200Chroma_422 = 1, HapB200Chroma_444 = 2 };
/* row colorSpace: {cy, crR, cbG, crG, cbB, yOff, cOff}, shift 18 */
#define HAPB200_YUV_12BIT_COEFFICIENTS                                                                                     \
    {                                                                                                                      \
        {19077, 3269, -802, -1665, 4131, 256, 2048},  /* BT.601 limited */                                                 \
        {16324, 2861, -702, -1457, 3616, 0, 2048},    /* BT.601 full    */                                                 \
        {19077, 3672, -437, -1091, 4326, 256, 2048},  /* BT.709 limited */                                                 \
        {16324, 3213, -382, -955, 3786, 0, 2048}      /* BT.709 full    */                                                 \
    }

/* one picture (host or device pointers, any alignment, any pitches) -> one Hap frame */
unsigned int HapB200EncodePlanar(const void *luma, const void *cb, const void *cr, const void *alpha,
                                 unsigned int width, unsigned int height, unsigned long lumaPitch, unsigned long chromaPitch,
                                 unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace, unsigned int codec,
                                 unsigned int compressor, unsigned int chunkCount,
                                 void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);
/* frames x picture (device) -> frames x Hap frame at out + f*outStride, encoded length in used[f] (device) */
unsigned int HapB200EncodePlanarBatch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                      unsigned long frameStride, unsigned int width, unsigned int height, unsigned long lumaPitch,
                                      unsigned long chromaPitch, unsigned int subsampling, unsigned int bitDepth,
                                      unsigned int colorSpace, unsigned int codec, unsigned int compressor, unsigned int chunkCount,
                                      void *out, unsigned long outStride, unsigned long long *used, void *stream);
/* frames x picture (device) -> bare textures, as HapB200BlockEncodeBatch (HapM: RGTC1 plane at blocks + HapB200TextureBytes(.., 0)) */
unsigned int HapB200BlockEncodePlanarBatch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                           unsigned long frameStride, unsigned int width, unsigned int height,
                                           unsigned long lumaPitch, unsigned long chromaPitch, unsigned int subsampling,
                                           unsigned int bitDepth, unsigned int colorSpace, unsigned int codec,
                                           void *blocks, unsigned long blocksStride, void *stream);

/* ---- Hap R (BC7, "Hap7") <- NV12 / P010 and planar Y'CbCr 4:2:0 / 4:2:2 / 4:4:4 (+ alpha) ----------------------------------
 * The BC7 forms of the YUV and planar encoders above, asking for BC7 by name as HapB200EncodeRGBABC7 does: the same
 * arguments without the codec.  A picture encodes to exactly the bytes HapB200EncodeRGBABC7* / HapB200BlockEncodeBC7Batch
 * give for the RGBA8 picture made of it by the conversion of HapB200EncodeYUV (NV12 / P010) or of HapB200EncodePlanar
 * (planar, its alpha rule included).
 * Alpha: NV12 / P010 give A = 255.  A planar picture's alpha plane is read when it is non-NULL; a NULL alpha means A = 255, and
 *   then every decoded texel has A = 255 (the BC7 encoder's opaque rule).  There is no alpha-only form: luma, cb and cr are
 *   always read.
 * Planes, layouts, subsamplings, depths, colour spaces, geometry and alignment: those of HapB200EncodeYUV* and
 *   HapB200EncodePlanar*.  In addition, the RGBA8 picture must be one the RGBA8 encoders take: 4 * width <=
 *   HAPB200_MAX_ROW_BYTES.  BT.2020, unknown layouts, subsamplings, depths or colour spaces, NULL planes and bad geometry are
 *   refused with HapResult_Bad_Arguments before anything touches the GPU.
 * Sizes, options: a frame needs HapB200MaxEncodedLengthRGBA(width, height, HapB200Codec_Hap7, chunkCount) bytes
 *   (outputBufferBytes, outStride); less is refused with HapResult_Buffer_Too_Small.  compressor, chunkCount and the index and
 *   offset-table options behave as for HapB200EncodeRGBABC7*.
 * The conversion runs as a pass of its own into device scratch of at most max(4 * width * height, 256 MiB) bytes, whatever
 * the number of frames; the BC7 search costs orders of magnitude more (DESIGN.md sections 4 and 6). */

/* one picture (host or device pointers) -> one Hap R frame */
unsigned int HapB200EncodeYUVBC7(const void *luma, const void *chroma, unsigned int width, unsigned int height,
                                 unsigned long pitch, unsigned int layout, unsigned int colorSpace,
                                 unsigned int compressor, unsigned int chunkCount,
                                 void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);
/* frames x picture (device) -> frames x Hap R frame at out + f*outStride, encoded length in used[f] (device) */
unsigned int HapB200EncodeYUVBC7Batch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                      unsigned int width, unsigned int height, unsigned long pitch, unsigned int layout,
                                      unsigned int colorSpace, unsigned int compressor, unsigned int chunkCount,
                                      void *out, unsigned long outStride, unsigned long long *used, void *stream);
/* frames x picture (device) -> bare BC7 textures at blocks + f*blocksStride */
unsigned int HapB200BlockEncodeYUVBC7Batch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                           unsigned int width, unsigned int height, unsigned long pitch, unsigned int layout,
                                           unsigned int colorSpace, void *blocks, unsigned long blocksStride, void *stream);
/* one planar picture (host or device pointers, any alignment, any pitches) -> one Hap R frame */
unsigned int HapB200EncodePlanarBC7(const void *luma, const void *cb, const void *cr, const void *alpha,
                                    unsigned int width, unsigned int height, unsigned long lumaPitch, unsigned long chromaPitch,
                                    unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace,
                                    unsigned int compressor, unsigned int chunkCount,
                                    void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);
/* frames x planar picture (device) -> frames x Hap R frame at out + f*outStride, encoded length in used[f] (device) */
unsigned int HapB200EncodePlanarBC7Batch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                         unsigned long frameStride, unsigned int width, unsigned int height, unsigned long lumaPitch,
                                         unsigned long chromaPitch, unsigned int subsampling, unsigned int bitDepth,
                                         unsigned int colorSpace, unsigned int compressor, unsigned int chunkCount,
                                         void *out, unsigned long outStride, unsigned long long *used, void *stream);
/* frames x planar picture (device) -> bare BC7 textures at blocks + f*blocksStride */
unsigned int HapB200BlockEncodePlanarBC7Batch(const void *luma, const void *cb, const void *cr, const void *alpha, unsigned int frames,
                                              unsigned long frameStride, unsigned int width, unsigned int height,
                                              unsigned long lumaPitch, unsigned long chromaPitch, unsigned int subsampling,
                                              unsigned int bitDepth, unsigned int colorSpace,
                                              void *blocks, unsigned long blocksStride, void *stream);

/* ---- Hap, Hap Alpha, Hap Q, Hap Q Alpha, Hap Alpha-Only, Hap R -> NV12 / P010------------------------------------------------
 * The decoders write the 4:2:0 pictures a video encoder takes (NVENC surfaces).  The conversion is fused into the block
 * decoder, so no RGBA picture is ever written.  The planes are exactly the conversion below applied to the RGBA8 picture that
 * HapB200DecodeRGBA / HapB200DecodeRGBABatch / HapB200BlockDecodeBatch give for the same input; alpha is ignored.
 * Planes, pitch and layouts: those of the YUV encoders above (HapB200YUV_NV12: bytes; HapB200YUV_P010: little-endian 16-bit
 * words holding sample << 6, the low 6 bits zero).  One pitch for both planes; chroma is a pointer of its own.  In a batch frame
 * f's planes start at luma + f*frameStride and chroma + f*frameStride.  The only bytes written are the width * (bytes per
 * sample) bytes of each of the height luma rows and height/2 chroma rows: pitch slack and whatever lies between planes and
 * frames stays as it was.
 * Geometry: that of the YUV encoders (width and height multiples of 4, width * (bytes per sample) <= pitch <=
 * HAPB200_MAX_ROW_BYTES, at most HAPB200_MAX_BLOCKS blocks).  The batch entry points take device pointers; luma, chroma, pitch,
 * frameStride, blocks and blocksStride are 16-byte aligned; a batch may hold any number of frames.  The single-frame call takes
 * host or device pointers at any alignment and any pitch.
 * Codecs: every HapB200Codec.  Hap Alpha-Only (HapA) decodes to (v, v, v, 255), so its matte comes out as a grey luma picture
 * with neutral chroma: a key signal.  Colour spaces: BT.601 and BT.709, limited and full range; BT.2020 is refused with
 * HapResult_Bad_Arguments (8-bit Hap into BT.2020 would be a gamut decision), as are an unknown layout or colour space.  Every
 * argument is checked before anything touches the GPU.
 * Results: HapB200DecodeYUV answers exactly as HapB200DecodeRGBA does (Hap HDR (BC6H) frames: HapResult_Bad_Frame);
 * HapB200DecodeYUVBatch reports in results[f] exactly what HapB200DecodeRGBABatch reports.  A failed frame's RGBA picture is
 * all zero bytes, so its planes are the conversion of zeros: black, Y = yOff and Cb = Cr = cOff.
 * The conversion, exactly (n = 8 for NV12, 10 for P010; scales and offsets those of the encoders' definition: limited range
 * luma offset 16 * 2^(n-8), luma scale 219 * 2^(n-8), chroma scale 224 * 2^(n-8); full range offset 0 and both scales
 * 2^n - 1; chroma offset 2^(n-1)):
 *   Coefficients: L = 65536 * lumaScale / 255 and S = 65536 * chromaScale / 255, (Kr, Kb) = BT.601 (0.299, 0.114) or BT.709
 *   (0.2126, 0.0722), Kg = 1 - Kr - Kb, round() to nearest, halves up:
 *     yR = round(L*Kr), yB = round(L*Kb), yG = round(L) - yR - yB;
 *     cbR = round(-S*Kr / (2(1-Kb))), cbG = round(-S*Kg / (2(1-Kb))), cbB = -(cbR + cbG);
 *     crG = round(-S*Kg / (2(1-Kr))), crB = round(-S*Kb / (2(1-Kr))), crR = -(crG + crB).
 *   The derived entries make every grey map to exactly neutral chroma, and 0 and 255 to the nominal black and white codes.
 *   They are the rows of HAPB200_YUV_OUT_COEFFICIENTS below.
 *   Luma, per pixel: Y = ((yR*R + yG*G + yB*B + 32768) >> 16) + yOff, clamped to 0..2^n-1.
 *   Chroma, 4:2:0 at the default siting the encoders' upsampler assumes (chroma_sample_loc_type 0: co-sited with even luma
 *   columns, midway between luma rows 2j and 2j+1): for chroma sample (i, j), Rs, Gs and Bs are the sums of R, G and B over
 *   luma columns 2i-1, 2i, 2i+1 with weights 1, 2, 1 (column -1 clamped to 0) and rows 2j and 2j+1 with weight 1 each, a
 *   total weight of 8; then
 *     Cb = ((cbR*Rs + cbG*Gs + cbB*Bs + 2^18) >> 19) + cOff,  Cr = ((crR*Rs + crG*Gs + crB*Bs + 2^18) >> 19) + cOff,
 *   the shift arithmetic, each clamped to 0..2^n-1.  Every intermediate is below 2^31.
 *   A flat colour converted to P010 here and back by the YUV encoders' conversion returns exactly, for all 2^24 colours. */
/* row layout * 4 + colorSpace: {yR, yG, yB, cbR, cbG, cbB, crR, crG, crB, yOff, cOff} */
#define HAPB200_YUV_OUT_COEFFICIENTS                                                                                       \
    {                                                                                                                      \
        {16829, 33039, 6416, -9714, -19071, 28785, 28784, -24103, -4681, 16, 128},        /* NV12 BT.601 limited */        \
        {19595, 38470, 7471, -11058, -21710, 32768, 32768, -27439, -5329, 0, 128},        /* NV12 BT.601 full    */        \
        {11966, 40254, 4064, -6596, -22189, 28785, 28784, -26145, -2639, 16, 128},        /* NV12 BT.709 limited */        \
        {13933, 46871, 4732, -7509, -25259, 32768, 32768, -29763, -3005, 0, 128},         /* NV12 BT.709 full    */        \
        {67315, 132155, 25665, -38856, -76282, 115138, 115137, -96413, -18724, 64, 512},  /* P010 BT.601 limited */        \
        {78612, 154331, 29972, -44363, -87094, 131457, 131457, -110079, -21378, 0, 512},  /* P010 BT.601 full    */        \
        {47864, 161016, 16255, -26383, -88755, 115138, 115137, -104580, -10557, 64, 512}, /* P010 BT.709 limited */        \
        {55896, 188037, 18982, -30123, -101335, 131458, 131458, -119404, -12054, 0, 512}  /* P010 BT.709 full    */        \
    }

/* one Hap frame (host or device pointers, any alignment) -> one NV12 / P010 picture */
unsigned int HapB200DecodeYUV(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height,
                              void *luma, void *chroma, unsigned long pitch, unsigned int layout, unsigned int colorSpace);
/* frames x Hap frame (device, as HapB200DecodeRGBABatch) -> frames x picture (device): frame f's planes at luma + f*frameStride,
 * chroma + f*frameStride */
unsigned int HapB200DecodeYUVBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                   unsigned int maxChunks, unsigned int codec, unsigned int width, unsigned int height,
                                   void *luma, void *chroma, unsigned long frameStride, unsigned long pitch,
                                   unsigned int layout, unsigned int colorSpace, unsigned int *results, void *stream);
/* bare textures (device, as HapB200BlockDecodeBatch; HapM: the RGTC1 plane at blocks + HapB200TextureBytes(.., 0), which is
 * not read, alpha being dropped) -> pictures */
unsigned int HapB200BlockDecodeYUVBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                        unsigned int height, unsigned int codec, void *luma, void *chroma, unsigned long frameStride,
                                        unsigned long pitch, unsigned int layout, unsigned int colorSpace, void *stream);

/* ---- Hap, Hap Alpha, Hap Q, Hap Q Alpha, Hap Alpha-Only, Hap R -> planar Y'CbCr 4:2:0 / 4:2:2 / 4:4:4 (+ alpha) ------------
 * The decoders write the planar pictures software encoders and mastering formats take (FFmpeg's yuv420p, yuv422p10le,
 * yuva444p12le, gray12le and their kin): the inverse of the planar encoders above.  The conversion is fused into the block
 * decoder, so no RGBA picture is ever written.  The planes are exactly the conversion below applied to the RGBA8 picture that
 * HapB200DecodeRGBA / HapB200DecodeRGBABatch / HapB200BlockDecodeBatch give for the same input, alpha included.
 * Arguments, planes, samples and geometry: those of the planar encoders (luma, cb, cr and alpha are AVFrame's data[0..3],
 * lumaPitch and chromaPitch its linesize[0] and linesize[1]; alpha rows are lumaPitch apart; cw x ch chroma samples; bitDepth
 * 8: bytes, 10 or 12: little-endian 16-bit words holding the sample in the low bits, the high bits written as zero; width and
 * height multiples of 4, width*bytes <= lumaPitch <= HAPB200_MAX_ROW_BYTES, cw*bytes <= chromaPitch <= HAPB200_MAX_ROW_BYTES,
 * at most HAPB200_MAX_BLOCKS blocks).  In a batch, each plane of frame f starts at its pointer + f*frameStride.  The batch
 * entry points take device pointers; the planes, both pitches, frameStride, blocks and blocksStride are 16-byte aligned.  The
 * single-frame call takes host or device memory at any alignment and pitch.  Only each row's samples are written: pitch
 * slack and whatever lies between planes and frames stays as it was.
 * Codecs: every HapB200Codec.  A non-NULL alpha receives the picture's A (Hap Alpha: DXT5 alpha; Hap Q Alpha: its RGTC1
 * texture; Hap R: BC7 alpha; Hap: 255, or 0 on DXT1's transparent texels; Hap Q: 255); a NULL alpha writes no alpha.  Hap
 * Alpha-Only writes its matte v to the alpha plane alone, which it requires: luma, cb and cr are neither written nor checked,
 * and may be NULL.  A Hap Alpha-Only frame (the batch calls: codec HapB200Codec_HapA) with a NULL alpha is refused with
 * HapResult_Bad_Arguments; the single-frame call learns the codec from the frame's headers and answers this after reading
 * them, still before anything touches the GPU.  Colour spaces: BT.601 and BT.709, limited and full range.  BT.2020, unknown
 * subsamplings, depths, colour spaces or codecs and bad geometry are refused with HapResult_Bad_Arguments before anything
 * touches the GPU.
 * Results: HapB200DecodePlanar answers exactly as HapB200DecodeRGBA does (Hap HDR (BC6H) frames: HapResult_Bad_Frame);
 * HapB200DecodePlanarBatch reports in results[f] exactly what HapB200DecodeRGBABatch reports.  A failed frame's RGBA picture is
 * all zero bytes, so its planes are the conversion of zeros: Y = yOff, Cb = Cr = cOff, alpha 0.
 * The conversion, exactly (n = bitDepth), extending that of HapB200DecodeYUV; chroma keeps the default siting the planar
 * encoders' upsampler assumes:
 *   1. Chroma sums of total weight 8, Rs, Gs and Bs the weighted sums of R, G and B around chroma sample (i, j), column -1
 *      clamped to 0:
 *        4:2:0: HapB200DecodeYUV's, weights 1 2 1 over luma columns 2i-1 .. 2i+1 times 1 1 over rows 2j and 2j+1;
 *        4:2:2: weights 1 2 1 over columns 2i-1 .. 2i+1 on row j alone, times 2;
 *        4:4:4: 8*R, 8*G, 8*B of pixel (i, j).
 *      Then Cb = ((cbR*Rs + cbG*Gs + cbB*Bs + 2^18) >> 19) + cOff, Cr likewise; luma is HapB200DecodeYUV's,
 *      Y = ((yR*R + yG*G + yB*B + 32768) >> 16) + yOff; each result clamped to 0..2^n-1.  Every intermediate is below 2^31.
 *   2. Rows: n = 8: the NV12 rows of HAPB200_YUV_OUT_COEFFICIENTS; n = 10: its P010 rows (the samples stored unshifted);
 *      n = 12: the rows of HAPB200_YUV_12BIT_OUT_COEFFICIENTS below, from the same rule with the 12-bit scales of
 *      HAPB200_YUV_12BIT_COEFFICIENTS (limited range luma offset 256, luma scale 3504, chroma scale 3584; full range offset 0,
 *      both scales 4095; chroma offset 2048).  Greys map to exactly neutral chroma, 0 and 255 to the nominal black and white.
 *   3. Alpha: a = (2*(2^n - 1)*A + 255) / 510, integer division: (2^n - 1)*A / 255 rounded to nearest (no tie occurs),
 *      so 255 gives 2^n - 1; a = A at n = 8.
 * Round trips: a flat RGB colour converted to 10- or 12-bit Y'CbCr here and back by the planar encoders' conversion returns
 * exactly, for all 2^24 colours, in all four colour spaces (at 8 bits it does not, as for NV12).  4:4:4 has no chroma filter,
 * so any RGBA8 picture decoded to 4:4:4 at 10 or 12 bits with alpha converts back through HapB200EncodePlanar*'s conversion to
 * the identical RGBA8 picture: yuva444p10le and yuva444p12le are lossless against the RGBA8 decoders.  The planar encoders'
 * alpha rule inverts step 3 exactly at every depth. */
/* row colorSpace: {yR, yG, yB, cbR, cbG, cbB, crR, crG, crB, yOff, cOff} */
#define HAPB200_YUV_12BIT_OUT_COEFFICIENTS                                                                                 \
    {                                                                                                                      \
        {269262, 528618, 102662, -155423, -305128, 460551, 460551, -385654, -74897, 256, 2048}, /* BT.601 limited */       \
        {314677, 617777, 119977, -177583, -348633, 526216, 526216, -440640, -85576, 0, 2048},   /* BT.601 full    */       \
        {191455, 644068, 65019, -105533, -355018, 460551, 460551, -418321, -42230, 256, 2048},  /* BT.709 limited */       \
        {223747, 752698, 75986, -120579, -405636, 526215, 526216, -477965, -48251, 0, 2048}     /* BT.709 full    */       \
    }

/* one Hap frame (host or device pointers, any alignment, any pitches) -> one planar picture */
unsigned int HapB200DecodePlanar(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height,
                                 void *luma, void *cb, void *cr, void *alpha, unsigned long lumaPitch, unsigned long chromaPitch,
                                 unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace);
/* frames x Hap frame (device, as HapB200DecodeRGBABatch) -> frames x picture (device), each plane at its pointer + f*frameStride */
unsigned int HapB200DecodePlanarBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                      unsigned int maxChunks, unsigned int codec, unsigned int width, unsigned int height,
                                      void *luma, void *cb, void *cr, void *alpha, unsigned long frameStride,
                                      unsigned long lumaPitch, unsigned long chromaPitch, unsigned int subsampling,
                                      unsigned int bitDepth, unsigned int colorSpace, unsigned int *results, void *stream);
/* bare textures (device, as HapB200BlockDecodeBatch; HapM: RGTC1 plane at blocks + HapB200TextureBytes(.., 0)) -> pictures */
unsigned int HapB200BlockDecodePlanarBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                           unsigned int height, unsigned int codec, void *luma, void *cb, void *cr, void *alpha,
                                           unsigned long frameStride, unsigned long lumaPitch, unsigned long chromaPitch,
                                           unsigned int subsampling, unsigned int bitDepth, unsigned int colorSpace, void *stream);

/* ---- Hap HDR (BC6H, "HapH") <- HDR10 P010 (BT.2020, SMPTE ST 2084 / PQ) --------------------------------------------------
 * The encoders take the P010 pictures a video decoder writes for HEVC Main10 HDR10 and convert them to linear RGBA16F inside
 * the BC6H encoder, so no RGBA16F picture is ever written.  A P010 picture encodes to exactly the bytes
 * HapB200EncodeRGBAHalf* give for the RGBA16F picture the conversion below makes of it.
 * Planes, pitch, geometry and alignment: those of HapB200YUV_P010 for HapB200EncodeYUV* (HDR10 is always 10-bit, so there
 * is no layout argument).  colorSpace: HapB200YUV_BT2020_Limited or HapB200YUV_BT2020_Full; any other is refused with
 * HapResult_Bad_Arguments.  textureFormat, compressor, chunkCount, sizes (HapMaxEncodedLength of the one BC6H texture) and
 * HapResult_Buffer_Too_Small: as for HapB200EncodeRGBAHalf*.  unitNits: the luminance in cd/m2 that the output value 1.0
 * stands for, an integer from 1 to 10000 (80 for scRGB, 100, or 203 for the BT.2408 HDR reference white are usual); there
 * is no convention for it shared across tools, so the caller names its working space.  Every argument is checked before
 * anything touches the GPU.  The first call with a unitNits on a device builds its table (8 KiB) on the host and uploads
 * it, waiting for the copy; later calls reuse it.
 * The conversion, exactly:
 *   1. Chroma upsampling: that of HapB200EncodeYUV, unchanged (Cb8, Cr8 in eighths, default siting, indices clamped).
 *   2. Matrix to 12-bit R'G'B': the BT.2020 matrix (Kr = 0.2627, Kb = 0.0593), limited range (luma offset 64, luma scale
 *      876, chroma scale 896) or full range (offset 0, scales 1023), chroma offset 512.  With the row {cy, crR, cbG, crG,
 *      cbB, yOff, cOff} of HAPB200_YUV_PQ_COEFFICIENTS below (each coefficient round(65536 * 4095 * matrix entry / scale),
 *      the chroma ones divided by 8 more: the rule of HAPB200_YUV_COEFFICIENTS with 4095 for 255), Yd = Y - yOff,
 *      Cb8d = Cb8 - 8*cOff and Cr8d = Cr8 - 8*cOff:
 *        R12 = (cy*Yd + crR*Cr8d + 32768) >> 16,  G12 = (cy*Yd + cbG*Cb8d + crG*Cr8d + 32768) >> 16,
 *        B12 = (cy*Yd + cbB*Cb8d + 32768) >> 16,
 *      the shift arithmetic, each clamped to 0..4095 (every intermediate is below 2^30).  12 bits are four times the source's
 *      resolution, so this rounding adds at most 1/8 of a source code.
 *   3. Transfer: T[c] is the binary16 of (10000 * EOTF(c / 4095)) / unitNits, rounded once, to nearest, ties to even, where
 *      EOTF is SMPTE ST 2084's: EOTF(E) = (max(E^(1/m2) - c1, 0) / (c2 - c3 * E^(1/m2)))^(1/m1), m1 = 2610/16384,
 *      m2 = 2523/32, c1 = 3424/4096, c2 = 2413/128, c3 = 2392/128.  T[0] = 0, T[4095] = the half of 10000 / unitNits;
 *      every value is finite and non-negative.
 *   4. The pixel is (T[R12], T[G12], T[B12], 1.0): linear light, in units of unitNits cd/m2, with the BT.2020 primaries
 *      kept.  Mapping to BT.709 / scRGB primaries (which gives negative values) is left to the caller. */
/* row colorSpace - HapB200YUV_BT2020_Limited: {cy, crR, cbG, crG, cbB, yOff, cOff} */
#define HAPB200_YUV_PQ_COEFFICIENTS                                                                                        \
    {                                                                                                                      \
        {306358, 55209, -6161, -21391, 70440, 64, 512},  /* P010 BT.2020 limited */                                        \
        {262336, 48355, -5396, -18736, 61695, 0, 512}    /* P010 BT.2020 full    */                                        \
    }

/* one P010 picture (host or device pointers) -> one Hap HDR frame */
unsigned int HapB200EncodeYUVPQ(const void *luma, const void *chroma, unsigned int width, unsigned int height,
                                unsigned long pitch, unsigned int colorSpace, unsigned int unitNits,
                                unsigned int textureFormat, unsigned int compressor, unsigned int chunkCount,
                                void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);
/* frames x P010 picture (device) -> frames x Hap HDR frame at out + f*outStride, encoded length in used[f] (device) */
unsigned int HapB200EncodeYUVPQBatch(const void *luma, const void *chroma, unsigned int frames, unsigned long frameStride,
                                     unsigned int width, unsigned int height, unsigned long pitch, unsigned int colorSpace,
                                     unsigned int unitNits, unsigned int textureFormat, unsigned int compressor,
                                     unsigned int chunkCount, void *out, unsigned long outStride,
                                     unsigned long long *used, void *stream);
/* frames x P010 picture (device) -> bare BC6H textures at blocks + f*blocksStride */
unsigned int HapB200BlockEncodeYUVPQBatch(const void *luma, const void *chroma, unsigned int frames,
                                          unsigned long frameStride, unsigned int width, unsigned int height,
                                          unsigned long pitch, unsigned int colorSpace, unsigned int unitNits,
                                          unsigned int textureFormat, void *blocks, unsigned long blocksStride, void *stream);

/* ---- Hap HDR (BC6H, "HapH") -> HDR10 P010 (BT.2020, SMPTE ST 2084 / PQ) --------------------------------------------------
 * The decoders write the P010 pictures a video encoder takes for HEVC Main10 HDR10 (NVENC surfaces): the inverse of the HDR10
 * encoders above.  The conversion is fused into the BC6H block decoder, so no RGBA16F picture is ever written.  The planes are
 * exactly the conversion below applied to the RGBA16F picture that HapB200DecodeRGBAHalf / HapB200DecodeRGBAHalfBatch /
 * HapB200BlockDecodeHalfBatch give for the same input; alpha is ignored.
 * Planes, pitch, geometry, alignment and bytes written: those of HapB200DecodeYUV* with HapB200YUV_P010 (little-endian 16-bit
 * words holding sample << 6; only the 2 * width bytes of each of the height luma rows and height/2 chroma rows are written:
 * pitch slack and whatever lies between planes and frames stays as it was).  HDR10 is always 10-bit, so there is no layout
 * argument.  colorSpace: HapB200YUV_BT2020_Limited or HapB200YUV_BT2020_Full.  unitNits: as for the HDR10 encoders, the
 * luminance in cd/m2 that the value 1.0 stands for, 1 to 10000.  textureFormat (HapB200BlockDecodeYUVPQBatch): UF16 or SF16.
 * Any other value, and any bad geometry, is refused with HapResult_Bad_Arguments before anything touches the GPU.  The first
 * call with a unitNits on a device builds its table (62 KiB) on the host and uploads it, waiting for the copy; later calls
 * reuse it.
 * Results: HapB200DecodeYUVPQ answers exactly as HapB200DecodeRGBAHalf does (a frame that is not one BC6H texture of
 * (width/4)*(height/4)*16 bytes: HapResult_Bad_Frame); HapB200DecodeYUVPQBatch reports in results[f] exactly what
 * HapB200DecodeRGBAHalfBatch reports.  Each frame decodes as its own texture format says (UF16 or SF16).  A failed frame's
 * RGBA16F picture is all zero, so its planes are black: Y = yOff, Cb = Cr = 512.
 * The conversion, exactly:
 *   1. Transfer, the inverse of the encoders' step 3: each of R, G and B, a binary16 h, becomes the 12-bit code P[h], where
 *        P[h] = floor(4095 * OETF(min(value(h) * unitNits / 10000, 1)) + 1/2),
 *        OETF(Y) = ((c1 + c2 * Y^m1) / (1 + c3 * Y^m1))^m2
 *      with the ST 2084 constants of the encoders, for every non-negative finite h (0x0000 .. 0x7BFF).  A value whose sign
 *      bit is set (SF16 negatives and -0) gives code 0.  P[0] = 0, every value at or above 10000 / unitNits gives 4095, and
 *      P never decreases.  The block decoder writes no Inf or NaN.
 *   2. Matrix, 12-bit R'G'B' to BT.2020 Y'CbCr (non-constant luminance): the rule of HAPB200_YUV_OUT_COEFFICIENTS with 4095
 *      for 255 (L = 65536 * lumaScale / 4095, S = 65536 * chromaScale / 4095; Kr = 0.2627, Kb = 0.0593; limited range luma
 *      offset 64, luma scale 876, chroma scale 896; full range offset 0, both scales 1023; chroma offset 512), which gives
 *      the rows of HAPB200_YUV_PQ_OUT_COEFFICIENTS below; the derived entries make greys exactly neutral.  Then, as for
 *      HapB200DecodeYUV with the codes for R, G and B:
 *        Y = ((yR*R + yG*G + yB*B + 32768) >> 16) + yOff, clamped to 0..1023;
 *        chroma at the default siting, Rs, Gs, Bs the [1 2 1] x [1 1] sums of the codes (column -1 clamped to 0),
 *        Cb = ((cbR*Rs + cbG*Gs + cbB*Bs + 2^18) >> 19) + cOff,  Cr = ((crR*Rs + crG*Gs + crB*Bs + 2^18) >> 19) + cOff,
 *      the shift arithmetic, each clamped to 0..1023.  Every intermediate is below 2^29.  Codes 4095 and 0 land on the
 *      nominal white and black (Y = 940 / 64 limited, 1023 / 0 full).  12 bits are four times the output's resolution, so
 *      the matrix adds at most about 0.1 of a code before its final rounding.
 * Round trip: a flat P010 colour converted to R'G'B' by HAPB200_YUV_PQ_COEFFICIENTS and back by the rows below returns
 * exactly wherever its R'G'B' is not clamped, and P[T[c]] = c for every code c at unitNits up to 123 (above, only the lowest
 * codes, whose halves cannot tell neighbours apart, miss: c = 1 at 203; some codes below 16 at 1000, below 180 at 10000).  So a flat HDR10
 * picture encoded by HapB200EncodeYUVPQ and decoded here at the same colorSpace and unitNits comes back byte for byte
 * within those bounds. */
/* row colorSpace - HapB200YUV_BT2020_Limited: {yR, yG, yB, cbR, cbG, cbB, crR, crG, crB, yOff, cOff} */
#define HAPB200_YUV_PQ_OUT_COEFFICIENTS                                                                                    \
    {                                                                                                                      \
        {3683, 9505, 831, -2002, -5168, 7170, 7170, -6593, -577, 64, 512},  /* P010 BT.2020 limited */                     \
        {4301, 11100, 971, -2286, -5900, 8186, 8186, -7528, -658, 0, 512}   /* P010 BT.2020 full    */                     \
    }

/* one Hap HDR frame (host or device pointers, any alignment, any pitch) -> one HDR10 P010 picture */
unsigned int HapB200DecodeYUVPQ(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int width, unsigned int height,
                                void *luma, void *chroma, unsigned long pitch, unsigned int colorSpace, unsigned int unitNits);
/* frames x Hap HDR frame (device, as HapB200DecodeRGBAHalfBatch) -> frames x picture (device): frame f's planes at
 * luma + f*frameStride, chroma + f*frameStride */
unsigned int HapB200DecodeYUVPQBatch(const void *in, unsigned int frames, unsigned long inStride, const unsigned long long *inBytes,
                                     unsigned int maxChunks, unsigned int width, unsigned int height, void *luma, void *chroma,
                                     unsigned long frameStride, unsigned long pitch, unsigned int colorSpace, unsigned int unitNits,
                                     unsigned int *results, void *stream);
/* bare BC6H textures (device, textureFormat UF16 or SF16, as HapB200BlockDecodeHalfBatch) -> pictures */
unsigned int HapB200BlockDecodeYUVPQBatch(const void *blocks, unsigned int frames, unsigned long blocksStride, unsigned int width,
                                          unsigned int height, unsigned int textureFormat, void *luma, void *chroma,
                                          unsigned long frameStride, unsigned long pitch, unsigned int colorSpace,
                                          unsigned int unitNits, void *stream);

#ifdef __cplusplus
}
#endif
#endif
