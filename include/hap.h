/*
 * include/hap.h -- the Hap frame API exported by libhap_b200.so.
 *
 * Drop-in boundary: same six entry points, enum values, callback types and argument meaning as the
 * reference header /root/reference/source/hap.h:40-152 (Vidvox/hap), so a host codec or player that
 * includes the reference's hap.h and links hap.c can link this library instead, unchanged.
 * Behind the boundary the second-stage (Snappy) compression and decompression run as sm_90a CUDA
 * kernels; see include/hap_b200.h for the device-resident batch extensions and INTEGRATION.md for
 * linking.  Every pointer argument may be a host pointer or a CUDA device pointer.
 */
#ifndef hap_h
#define hap_h

#ifdef __cplusplus
extern "C" {
#endif

/* texture formats: the GL constants of EXT_texture_compression_s3tc / ARB_..._rgtc / ARB_..._bptc
 * (reference hap.h:40-48) */
enum HapTextureFormat {
    HapTextureFormat_RGB_DXT1 = 0x83F0,
    HapTextureFormat_RGBA_DXT5 = 0x83F3,
    HapTextureFormat_YCoCg_DXT5 = 0x01,
    HapTextureFormat_A_RGTC1 = 0x8DBB,
    HapTextureFormat_RGBA_BPTC_UNORM = 0x8E8C,
    HapTextureFormat_RGB_BPTC_UNSIGNED_FLOAT = 0x8E8F,
    HapTextureFormat_RGB_BPTC_SIGNED_FLOAT = 0x8E8E,
};

/* second-stage compressors (reference hap.h:50-53) */
enum HapCompressor { HapCompressorNone, HapCompressorSnappy };

/* results (reference hap.h:55-61) */
enum HapResult {
    HapResult_No_Error = 0,
    HapResult_Bad_Arguments,
    HapResult_Buffer_Too_Small,
    HapResult_Bad_Frame,
    HapResult_Internal_Error
};

/* decode work fan-out (reference hap.h:66-67, contract hap.h:113-128) */
typedef void (*HapDecodeWorkFunction)(void *p, unsigned int index);
typedef void (*HapDecodeCallback)(HapDecodeWorkFunction function, void *p, unsigned int count, void *info);

/* reference hap.h:76-79 (hap.c:324-353): worst-case frame size for 1 or 2 textures, 0 on error */
unsigned long HapMaxEncodedLength(unsigned int count, unsigned long *lengths, unsigned int *textureFormats,
                                  unsigned int *chunkCounts);

/* reference hap.h:98-104 (hap.c:506-604): DXT/RGTC/BPTC bytes of 1 or 2 textures -> one Hap frame */
unsigned int HapEncode(unsigned int count, const void **inputBuffers, unsigned long *inputBuffersBytes,
                       unsigned int *textureFormats, unsigned int *compressors, unsigned int *chunkCounts,
                       void *outputBuffer, unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed);

/* reference hap.h:132-137 (hap.c:993-1040): texture `index` of a Hap frame -> its DXT/RGTC/BPTC bytes.
 * callback is required (non-NULL), is invoked exactly once and only when the texture has more than
 * one chunk, with count = chunk count; it must call function(p, i) for every i in [0, count) and
 * return when all calls have returned.  The GPU has already been given every chunk when the callback
 * runs; function(p, i) waits for chunk i. */
unsigned int HapDecode(const void *inputBuffer, unsigned long inputBufferBytes, unsigned int index,
                       HapDecodeCallback callback, void *info, void *outputBuffer,
                       unsigned long outputBufferBytes, unsigned long *outputBufferBytesUsed,
                       unsigned int *outputBufferTextureFormat);

/* reference hap.h:142-152 (hap.c:1042-1188): header walks only, never touch the GPU */
unsigned int HapGetFrameTextureCount(const void *inputBuffer, unsigned long inputBufferBytes,
                                     unsigned int *outputTextureCount);
unsigned int HapGetFrameTextureFormat(const void *inputBuffer, unsigned long inputBufferBytes,
                                      unsigned int index, unsigned int *outputBufferTextureFormat);
unsigned int HapGetFrameTextureChunkCount(const void *inputBuffer, unsigned long inputBufferBytes,
                                          unsigned int index, int *chunk_count);

#ifdef __cplusplus
}
#endif
#endif
