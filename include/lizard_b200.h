/* lizard_b200.h -- C ABI of liblizard_b200.so: the Lizard block codec hot path on NVIDIA H100 (sm_90a).
 *
 * Two groups of entry points:
 *
 *  (1) DROP-IN symbols: same names, argument meaning, return values and error conventions as the
 *      reference library, so an application (or the reference's own frame layer / bench / CLI) can be
 *      relinked against this library unchanged.  All pointers are HOST pointers, as in the reference.
 *        reference declaration                              replaced implementation
 *        lib/lizard_compress.h:82    Lizard_versionNumber
 *        lib/lizard_compress.h:97    Lizard_compress          lib/lizard_compress.c:596-606
 *        lib/lizard_compress.h:136   Lizard_compressBound     lib/lizard_compress.c:67
 *        lib/lizard_compress.h:146   Lizard_sizeofState       lib/lizard_compress.c:311-323
 *        lib/lizard_compress.h:147   Lizard_compress_extState lib/lizard_compress.c:583-593
 *        lib/lizard_decompress.h:73  Lizard_decompress_safe   lib/lizard_decompress.c:267-270
 *        lib/lizard_decompress.h:89  Lizard_decompress_safe_partial lib/lizard_decompress.c:272-275
 *        lib/lizard_decompress.h:145 Lizard_decompress_safe_usingDict lib/lizard_decompress.c:351-360
 *        lib/lizard_decompress.h:135 Lizard_decompress_safe_continue  lib/lizard_decompress.c:322-344 (see (1a))
 *      Compression output is byte-identical to the reference built with -DLIZARD_RESET_MEM
 *      (hash table empty at the start of every call), for the levels whose parsers are implemented on
 *      the GPU: 10, 11, 30, 31 (fastSmall / fast), 13-17, 34-38 (hashChain), 20, 40 (fastBig), 21, 22, 41, 42 (priceFast)
 *      23-25, 43-45 (lowestPrice) and 18, 19, 39 (the binary-tree optimal parser, LZ4 codewords).  Any other level (12,
 *      26-29, 32-33, 46-49) makes the compress entry points return 0 ("failed"), never a CPU fallback.
 *      Decompression accepts every level 10..49 (the block format only has two codeword flavours).
 *
 *  (2) BATCH symbols (LizardB200_*): what the reference's per-block loops
 *      (lib/lizard_frame.c:544-556 compressUpdate, :1148-1169 decodeCBlock, programs/bench.c:231-286)
 *      turn into: n independent units per call, one GPU launch.  Host-pointer and device-pointer variants.
 *
 * A unit's compressed form is exactly what one Lizard_compress call returns; a unit's decoded size is
 * exactly what Lizard_decompress_safe returns (negative values are the reference's error codes).
 *
 * There is no CPU fallback anywhere: if no usable CUDA device exists every entry point fails
 * (compress -> 0, decompress -> LIZARDB200_ERR_NO_DEVICE, batch calls -> negative status).
 */
#ifndef LIZARD_B200_H
#define LIZARD_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__cplusplus)
extern "C" {
#endif

#define LIZARD_B200_VERSION_NUMBER 10000          /* same numbering as LIZARD_VERSION_NUMBER 1.0.0 */
#define LIZARD_MIN_CLEVEL   10
#define LIZARD_MAX_CLEVEL   49
#define LIZARD_BLOCK_SIZE   (1 << 17)
#define LIZARD_MAX_INPUT_SIZE 0x7E000000
#define LIZARD_COMPRESSBOUND(isize) \
    ((unsigned)(isize) > (unsigned)LIZARD_MAX_INPUT_SIZE ? 0 : (isize) + 1 + 1 + (((isize) / LIZARD_BLOCK_SIZE) + 1) * 4)

/* status codes of the batch API (all negative); per-unit results use the reference's conventions */
#define LIZARDB200_OK               0
#define LIZARDB200_ERR_NO_DEVICE   (-1001)   /* no CUDA device / driver, or kernels not built for this GPU */
#define LIZARDB200_ERR_CUDA        (-1002)   /* a CUDA call failed; see LizardB200_lastError() */
#define LIZARDB200_ERR_ARGUMENT    (-1003)
#define LIZARDB200_ERR_LEVEL       (-1004)   /* compression level whose parser is not implemented on the GPU */
#define LIZARDB200_ERR_MEMORY      (-1005)

/* ---------------------------------------------------------------------------------------------
 * (1) drop-in symbols
 * ------------------------------------------------------------------------------------------- */
int Lizard_versionNumber(void);
int Lizard_compressBound(int inputSize);
int Lizard_sizeofState(int compressionLevel);
/* returns compressed size, or 0 when it failed / did not fit maxDstSize */
int Lizard_compress(const char* src, char* dst, int srcSize, int maxDstSize, int compressionLevel);
/* `state` is accepted for signature compatibility (must be pointer-aligned, else 0); the device keeps its own */
int Lizard_compress_extState(void* state, const char* src, char* dst, int srcSize, int maxDstSize, int compressionLevel);
/* returns decoded size (>= 0) or a negative error exactly as the reference:
 * -1 for a bad level byte / block header / stream, -(tokenIndex)-1 from the token loops.
 * Two deliberate differences, both on streams no encoder produces (DESIGN.md 3.5): a match offset below 8 is decoded with
 * byte-serial semantics (the reference's 8-byte granule copies give bytes that depend on stale memory), and a call whose
 * raw inner block is followed by a compressed one, decoded into less room than it needs, returns a negative value -- the
 * reference does not charge raw inner blocks against maxDecompressedSize (lib/lizard_decompress.c:164-180), decodes the
 * following block past dst + maxDecompressedSize and reports success.  This library never writes outside
 * [dst, dst + maxDecompressedSize): it is the safer of the two. */
int Lizard_decompress_safe(const char* src, char* dst, int compressedSize, int maxDecompressedSize);
/* decodes until at least targetOutputSize bytes are out, then stops; returns the decoded size (which may exceed the target),
 * or a negative error, exactly as the reference (lib/lizard_decompress.c:115-264 with partialDecoding), quirks included:
 * each inner block's token loop measures the target from the START OF THAT BLOCK (so a target inside the second block of a
 * unit decodes that block whole), the fastLZ4 codewords stop after a token's literals or its match (a block that stops after
 * its last match does not copy its last literals), the LIZv1 codewords stop in front of a token.  Nothing behind the
 * stopping point is read: damage there is not reported.  Bytes behind the returned size are unspecified.  With
 * targetOutputSize >= the decoded size this is Lizard_decompress_safe. */
int Lizard_decompress_safe_partial(const char* source, char* dest, int compressedSize, int targetOutputSize, int maxDecompressedSize);
/* Lizard_decompress_safe with the dictSize bytes at dictStart in front of the output: matches may reach that far below dest.
 * The reference's three modes, chosen as it chooses them: dictSize == 0 is Lizard_decompress_safe; a dictionary that ends at
 * dest (dictStart + dictSize == dest) is read in place; any other is an external dictionary (a match running past its end
 * continues at dest).  Return values as Lizard_decompress_safe, the same two differences included; a match that starts
 * further below dest than the dictionary reaches returns the reference's token error.  A negative dictSize returns -1 (the
 * reference has no defined behaviour there).  The dictionary is only read, and only its last 65535 bytes (levels 10-19,
 * 30-39) or 2^24 - 1 bytes (LIZv1 levels) can be reached. */
int Lizard_decompress_safe_usingDict(const char* source, char* dest, int compressedSize, int maxDecompressedSize,
                                     const char* dictStart, int dictSize);

/* ---------------------------------------------------------------------------------------------
 * (1a) the rest of the reference's export list (lib/dll/liblizard.def:3-19), so that its own callers link:
 *      lib/lizard_frame.c and the sources under programs/ reference every one of these.
 *      Stream objects are functional: lib/lizard_frame.c:379-401 creates one per compression context and hands it to
 *      Lizard_compress_extState.  Of the streaming / dictionary family (linked blocks, cross-call windows;
 *      lib/lizard_compress.h:178-198, lib/lizard_decompress.h:89-145) the DECODE side is implemented on the GPU:
 *      Lizard_setStreamDecode and Lizard_decompress_safe_continue keep the reference's window state (an external
 *      dictionary plus the prefix decoded in place, lib/lizard_decompress.c:303-344) and decode one unit per call against
 *      it, like Lizard_decompress_safe_usingDict (1).  On the COMPRESS side, Lizard_loadDict records the dictionary in the
 *      stream object and returns the reference's value (the size, trimmed to the last 2^24 bytes); the stream's next
 *      Lizard_compress_continue is Lizard_loadDict + Lizard_compress_continue of the reference, byte for byte, in one launch
 *      (LizardB200_compress_dict_batch; levels 13-17, 21, 22, 34-38, 41 and 42, other levels return 0).  Lizard_compress_continue on
 *      a fresh or reset stream is Lizard_compress, at every GPU level.  Any later Lizard_compress_continue on the same stream
 *      would need the tables the previous call left behind: it returns 0, as Lizard_saveDict always does.  No CPU code path
 *      behind any.
 * ------------------------------------------------------------------------------------------- */
typedef struct Lizard_stream_s Lizard_stream_t;                 /* lib/lizard_compress.h:72 */
typedef struct Lizard_streamDecode_s Lizard_streamDecode_t;     /* lib/lizard_decompress.h:100 */
Lizard_stream_t* Lizard_createStream(int compressionLevel);
int              Lizard_freeStream(Lizard_stream_t* streamPtr);
Lizard_stream_t* Lizard_resetStream(Lizard_stream_t* streamPtr, int compressionLevel);
int Lizard_loadDict(Lizard_stream_t* streamPtr, const char* dictionary, int dictSize);
int Lizard_saveDict(Lizard_stream_t* streamPtr, char* safeBuffer, int dictSize);
int Lizard_compress_continue(Lizard_stream_t* streamPtr, const char* src, char* dst, int srcSize, int maxDstSize);
Lizard_streamDecode_t* Lizard_createStreamDecode(void);
int Lizard_freeStreamDecode(Lizard_streamDecode_t* streamPtr);
int Lizard_setStreamDecode(Lizard_streamDecode_t* streamPtr, const char* dictionary, int dictSize);
int Lizard_decompress_safe_continue(Lizard_streamDecode_t* streamPtr, const char* source, char* dest, int compressedSize, int maxDecompressedSize);

/* ---------------------------------------------------------------------------------------------
 * (1b) drop-in frame layer: same names, types and error values as lib/lizard_frame.h:57-297 and
 *      lib/lizard_frame_static.h:56-67.  Frame format: doc/lizard_Frame_format.md (magic 0x184D2206).
 *      All full blocks handed to one LizardF_compressUpdate / LizardF_compressFrame / LizardF_decompress
 *      call are processed by ONE batch on the GPU (reference loops: lib/lizard_frame.c:544-556, 1010-1320).
 *      Only LizardF_blockIndependent is supported (linked blocks need the out-of-scope streaming dictionary
 *      API): a linked request / frame returns -LizardF_ERROR_blockMode_invalid.  NOTE that, as in the
 *      reference, a zeroed LizardF_preferences_t means blockLinked: set blockMode = LizardF_blockIndependent
 *      (the reference CLI does, programs/lizardio.c:109).
 * ------------------------------------------------------------------------------------------- */
typedef size_t LizardF_errorCode_t;
typedef enum { LizardF_default = 0, LizardF_max128KB = 1, LizardF_max256KB = 2, LizardF_max1MB = 3, LizardF_max4MB = 4,
               LizardF_max16MB = 5, LizardF_max64MB = 6, LizardF_max256MB = 7 } LizardF_blockSizeID_t;
typedef enum { LizardF_blockLinked = 0, LizardF_blockIndependent } LizardF_blockMode_t;
typedef enum { LizardF_noContentChecksum = 0, LizardF_contentChecksumEnabled } LizardF_contentChecksum_t;
typedef enum { LizardF_frame = 0, LizardF_skippableFrame } LizardF_frameType_t;
typedef struct {
    LizardF_blockSizeID_t     blockSizeID;
    LizardF_blockMode_t       blockMode;
    LizardF_contentChecksum_t contentChecksumFlag;
    LizardF_frameType_t       frameType;
    unsigned long long        contentSize;
    unsigned                  reserved[2];
} LizardF_frameInfo_t;
typedef struct {
    LizardF_frameInfo_t frameInfo;
    int      compressionLevel;
    unsigned autoFlush;
    unsigned reserved[4];
} LizardF_preferences_t;
typedef struct { unsigned stableSrc; unsigned reserved[3]; } LizardF_compressOptions_t;
typedef struct { unsigned stableDst; unsigned reserved[3]; } LizardF_decompressOptions_t;
typedef struct LizardF_cctx_s* LizardF_compressionContext_t;
typedef struct LizardF_dctx_s* LizardF_decompressionContext_t;
#define LIZARDF_VERSION 100

unsigned    LizardF_isError(LizardF_errorCode_t code);
const char* LizardF_getErrorName(LizardF_errorCode_t code);
size_t LizardF_compressFrameBound(size_t srcSize, const LizardF_preferences_t* preferencesPtr);
size_t LizardF_compressFrame(void* dstBuffer, size_t dstMaxSize, const void* srcBuffer, size_t srcSize,
                             const LizardF_preferences_t* preferencesPtr);
LizardF_errorCode_t LizardF_createCompressionContext(LizardF_compressionContext_t* cctxPtr, unsigned version);
LizardF_errorCode_t LizardF_freeCompressionContext(LizardF_compressionContext_t cctx);
size_t LizardF_compressBegin(LizardF_compressionContext_t cctx, void* dstBuffer, size_t dstMaxSize, const LizardF_preferences_t* prefsPtr);
size_t LizardF_compressBound(size_t srcSize, const LizardF_preferences_t* prefsPtr);
size_t LizardF_compressUpdate(LizardF_compressionContext_t cctx, void* dstBuffer, size_t dstMaxSize, const void* srcBuffer,
                              size_t srcSize, const LizardF_compressOptions_t* cOptPtr);
size_t LizardF_flush(LizardF_compressionContext_t cctx, void* dstBuffer, size_t dstMaxSize, const LizardF_compressOptions_t* cOptPtr);
size_t LizardF_compressEnd(LizardF_compressionContext_t cctx, void* dstBuffer, size_t dstMaxSize, const LizardF_compressOptions_t* cOptPtr);
LizardF_errorCode_t LizardF_createDecompressionContext(LizardF_decompressionContext_t* dctxPtr, unsigned version);
LizardF_errorCode_t LizardF_freeDecompressionContext(LizardF_decompressionContext_t dctx);
size_t LizardF_getFrameInfo(LizardF_decompressionContext_t dctx, LizardF_frameInfo_t* frameInfoPtr,
                            const void* srcBuffer, size_t* srcSizePtr);
size_t LizardF_decompress(LizardF_decompressionContext_t dctx, void* dstBuffer, size_t* dstSizePtr,
                          const void* srcBuffer, size_t* srcSizePtr, const LizardF_decompressOptions_t* dOptPtr);

/* ---------------------------------------------------------------------------------------------
 * (2) batch symbols
 * ------------------------------------------------------------------------------------------- */
/* Select the CUDA device used by this thread's subsequent calls (default 0). Returns LIZARDB200_OK or error. */
int LizardB200_setDevice(int device);
/* 1 if a usable sm_90 device is present and the context could be created, else 0 */
int LizardB200_available(void);
const char* LizardB200_lastError(void);

/* Host-pointer batch: unit i = src[i][0..srcSize[i]) -> dst[i][0..dstCapacity[i]); result[i] as Lizard_compress
 * (0 = failed / did not fit).  Inputs are staged through pinned memory, one launch for the whole batch. */
int LizardB200_compress_batch(const void* const* src, const int* srcSize,
                              void* const* dst, const int* dstCapacity, int* result,
                              int nUnits, int compressionLevel);
/* result[i] as Lizard_decompress_safe */
int LizardB200_decompress_batch(const void* const* src, const int* compressedSize,
                                void* const* dst, const int* dstCapacity, int* result, int nUnits);
/* result[i] as Lizard_decompress_safe_partial(src[i], dst[i], compressedSize[i], targetOutputSize[i], dstCapacity[i]):
 * a warp stops at its unit's target and takes the next unit.  One launch of the partial-decode kernel, whatever
 * LizardB200_setDecodeVariant says (it never runs the pre-passes, which expand or parse whole streams). */
int LizardB200_decompress_partial_batch(const void* const* src, const int* compressedSize,
                                        void* const* dst, const int* dstCapacity, const int* targetOutputSize,
                                        int* result, int nUnits);
/* result[i] as Lizard_decompress_safe_usingDict(src[i], dst[i], compressedSize[i], dstCapacity[i], dict[i], dictSize[i]),
 * the in-place mode included (dict[i] + dictSize[i] == dst[i]).  Units whose dictionaries end at the same address (e.g. one
 * shared dictionary) share one staged copy of it.  One launch of the dictionary-decode kernel, behind the Huffman pre-pass
 * kernels when LizardB200_setDecodeVariant enables them and the batch has at least 32 units; never the token pre-pass or the
 * second generation. */
int LizardB200_decompress_dict_batch(const void* const* src, const int* compressedSize,
                                     void* const* dst, const int* dstCapacity,
                                     const void* const* dict, const int* dictSize, int* result, int nUnits);
/* result[i] as Lizard_createStream(level) + Lizard_loadDict(dict[i], dictSize[i]) + Lizard_compress_continue(src[i], dst[i],
 * srcSize[i], dstCapacity[i]) of the reference, byte for byte; dictSize[i] == 0 means no dictionary (then as Lizard_compress).
 * The dictionary is a prefix when dict[i] + dictSize[i] == src[i], as in the reference; an input that overlaps its dictionary
 * limits the window as the reference does.  Units whose dictionaries end at the same address with the same size share one
 * staged and loaded copy.  Levels 13-17 and 34-38 (hashChain), 21, 22, 41 and 42 (priceFast); LIZARDB200_ERR_LEVEL at every
 * other level.
 * LIZARDB200_ERR_MEMORY when the call has more distinct dictionaries of 8 bytes or more than the encode workspace holds slots
 * for (each takes 1.125 MiB: 1883 for 5000 units on an 80 GB H100; LizardB200_lastError says how many).  One kernel launch
 * (lizard_encode_dict_kernel: the first unit of each dictionary loads its table, the others wait for it), behind a memset of
 * the dictionary map. */
int LizardB200_compress_dict_batch(const void* const* src, const int* srcSize,
                                   void* const* dst, const int* dstCapacity,
                                   const void* const* dict, const int* dictSize, int* result, int nUnits, int compressionLevel);

/* Contiguous host buffers, units described by offset/size arrays (what a frame or a file splitter has).
 * dstStride: unit i is written at dst + i*dstStride with capacity dstCapacityEach. */
int LizardB200_compress_blocks(const void* src, size_t srcSize, int blockSize,
                               void* dst, size_t dstStride, int dstCapacityEach, int* result,
                               int compressionLevel);
/* Inverse: unit i = src + i*srcStride, compressedSize[i] bytes -> dst + i*blockSize (capacity blockSize). */
int LizardB200_decompress_blocks(const void* src, size_t srcStride, const int* compressedSize, size_t nUnits,
                                 void* dst, int blockSize, int* result);

/* Device-pointer variants: everything (payload, offset/size tables, results) already lives in device memory
 * of the current device; the call only enqueues kernels on `cudaStream` (a cudaStream_t, may be NULL) and
 * returns without synchronising.  Workspace is owned by the library, shared by all calls on a device and grown on demand
 * (growing it -- the first call, or a batch larger than any before -- is the one case in which these calls synchronise the
 * stream and allocate; do not capture that call in a CUDA graph).  Calls on DIFFERENT streams are serialised against each
 * other on the device (each launch waits for the previous launch's completion event when the stream changes), so results
 * do not depend on how the caller spreads calls over streams; calls on one stream run in stream order.  The exception: a call
 * made while its stream is being captured into a CUDA graph neither waits for nor records that event (an event recorded
 * outside a capture cannot be waited on inside it), so the graph's launches are not serialised against the library's other
 * calls; the caller orders graph launches against them. */
int LizardB200_decompress_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                 void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                 int* dResult, unsigned nUnits, void* cudaStream);
/* partial decode of every unit, dTarget[i] = its targetOutputSize (device memory); same workspace and stream rules */
int LizardB200_decompress_partial_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                         void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                         const int* dTarget, int* dResult, unsigned nUnits, void* cudaStream);
/* every unit against its dictionary, the dDictLen[i] bytes at dDict + dDictOff[i] (device memory, 0 = none), as
 * Lizard_decompress_safe_usingDict; the in-place mode applies when dDict + dDictOff[i] + dDictLen[i] == dDst + dDstOff[i].
 * Dictionaries are only read, and may be shared by any number of units; same workspace and stream rules */
int LizardB200_decompress_dict_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                      void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                      const void* dDict, const uint64_t* dDictOff, const uint32_t* dDictLen,
                                      int* dResult, unsigned nUnits, void* cudaStream);
int LizardB200_compress_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                               void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                               int* dResult, unsigned nUnits, int compressionLevel, void* cudaStream);
/* LizardB200_compress_dict_batch on device arrays: unit i's dictionary is dDictLen[i] bytes at dDict + dDictOff[i] (0 = none);
 * it is a prefix when dDict + dDictOff[i] + dDictLen[i] == dSrc + dSrcOff[i].  Enqueue-only, with the workspace and stream
 * rules of LizardB200_compress_device.  A unit whose dictionary finds no slot in the workspace (more distinct dictionaries
 * than the bound above) is not compressed and gets dResult[i] = -1; slots go to dictionaries in the order warps meet them, so
 * which units those are depends on scheduling and may change from call to call.  Like the input, a dictionary may be read up to 8 bytes
 * past its end. */
int LizardB200_compress_dict_device(const void* dSrc, const uint64_t* dSrcOff, const uint32_t* dSrcLen,
                                    void* dDst, const uint64_t* dDstOff, const uint32_t* dDstCap,
                                    const void* dDict, const uint64_t* dDictOff, const uint32_t* dDictLen,
                                    int* dResult, unsigned nUnits, int compressionLevel, void* cudaStream);
/* Concatenation step of a block writer on the device (what lib/lizard_frame.c:544-549 does by advancing dstPtr block by
 * block): segment i = dSrc + dSrcOff[i], dLen[i] bytes (entries <= 0 are skipped, e.g. failed units) is copied to
 * dDst + dDstOff[i].  With dLen = the result array of LizardB200_compress_device and dDstOff = its exclusive prefix sum this
 * packs the units of a batch back to back.  Enqueue-only, like the calls above. */
int LizardB200_gather_device(const void* dSrc, const uint64_t* dSrcOff, const int* dLen,
                             void* dDst, const uint64_t* dDstOff, unsigned nUnits, void* cudaStream);
/* LizardF frames in device memory (DESIGN.md 3.4a).  Payload in DEVICE memory of the current device: frame i is the srcSize[i]
 * bytes at dSrc + srcOff[i] and goes to dDst + dstOff[i] with room for dstCap[i] bytes.  Tables and results are in HOST memory.
 * Unlike the enqueue-only calls above these SYNCHRONISE `cudaStream` and return when their work is done: where a frame's blocks
 * lie, and which verdict a frame gets, is only known once its headers and block results have been read back from the device.
 * Same workspace and stream rules as the calls above.  Nothing is written outside [dDst + dstOff[i], dDst + dstOff[i] + dstCap[i]).
 * The return value is LIZARDB200_OK or a negative batch status; result[i] is a size_t that LizardF_isError tests.
 *
 * LizardB200_compressFrames: frame i equals LizardF_compressFrame(dst, dstCap[i], src, srcSize[i], prefs) of this library on host
 * copies, byte for byte and in its return value (errors included, when nothing is written).  One difference, where the host call
 * writes past dstMaxSize: a 1-byte input whose header carries the content size, given 25 to 28 bytes of room (25 to 32 with the
 * content checksum; LizardF_compressFrameBound says 24 / 28), gets LizardF_ERROR_dstMaxSize_tooSmall here.  Its 1-byte block
 * takes 10 bytes, 5 more than the bound counts.  A fixed number of launches however many frames: one encode launch over every block of every frame, then the content
 * checksums and the frame assembly.
 *
 * LizardB200_decompressFrames: result[i] is what LizardF_decompress on a fresh context returns for frame i handed its whole
 * srcSize[i] bytes and dstCap[i] bytes of room in one call: the decoded size if that call finishes the frame, the same error code
 * if it fails; LizardF_ERROR_frameSize_wrong if it would end having read all input without finishing the frame (a truncated
 * frame) or finish it with input left (more bytes behind the frame); LizardF_ERROR_dstMaxSize_tooSmall if it would stop because
 * the output is full, with input left; 0 for a skippable
 * frame (nothing written); LizardF_ERROR_blockMode_invalid for a linked frame.  Damage in one frame changes no other frame's
 * result or bytes; after an error the frame's own dst range holds unspecified bytes.  The decoder stages every compressed block
 * in a workspace slot of its frame's maximum block size, at most 4 GiB of slots at a time: frames of many blocks far smaller
 * than their maximum take several decode rounds (more launches), never a failure of the call.  LIZARDB200_ERR_MEMORY only when
 * the device cannot hold one slot of the call's largest maximum block size.
 * The content checksum of one frame is computed by one warp (about 1.2 GB/s on an H100): for a single large checksummed frame
 * the host frame API, which hashes on a host thread, is faster. */
int LizardB200_compressFrames(const void* dSrc, const uint64_t* srcOff, const uint64_t* srcSize,
                              void* dDst, const uint64_t* dstOff, const uint64_t* dstCap,
                              size_t* result, unsigned nFrames, const LizardF_preferences_t* prefs, void* cudaStream);
int LizardB200_decompressFrames(const void* dSrc, const uint64_t* srcOff, const uint64_t* srcSize,
                                void* dDst, const uint64_t* dstOff, const uint64_t* dstCap,
                                size_t* result, unsigned nFrames, void* cudaStream);
/* LizardB200_decompressFrames with EVERYTHING in device memory -- payload, the offset, size and capacity tables and the results
 * dResult[i] (a size_t that LizardF_isError tests) -- and enqueue-only (DESIGN.md 3.4b).  nFrames, maxBlocks and stageBytes are
 * host values; they fix the grids and the workspace.  Frames are admitted in index order, as a prefix: frame i is admitted while
 * the complete blocks of frames 0..i number at most maxBlocks and their compressed blocks' staging slots (the frame's maximum
 * block size each) take at most stageBytes.  A frame whose header check fails, a skippable frame and an empty one take
 * nothing.  An admitted frame gets exactly what LizardB200_decompressFrames gives it, in result and bytes; a frame that is not
 * admitted gets LizardF_ERROR_allocation_failed and nothing is written to its range.  There is one decode round: the caller
 * chooses the bounds.
 * Stream and capture rules.  The workspace (tables for nFrames and maxBlocks, stageBytes of slots) is library-owned and grows on
 * demand; the growing call synchronises `cudaStream` and allocates.  A call that needs no growth issues no host<->device copy,
 * no synchronisation and no allocation: it enqueues a sequence of launches that depends only on (nFrames, maxBlocks,
 * stageBytes, decode variant), so after one call of the same or a larger shape it can be captured in a CUDA graph, and each
 * replay decodes whatever frames the tables then point at.  A captured call neither waits for nor signals the other streams'
 * use of the shared workspace (the exception above): order the graph's launches against the library's other calls on the
 * device yourself, and capture again after any call grows the workspace (a larger shape, or another device call with a larger
 * batch).  A capture that would have to grow the workspace -- the frame tables, the staging arena or the decoder's pre-pass
 * workspaces -- returns LIZARDB200_ERR_ARGUMENT and enqueues nothing.  stageBytes above maxBlocks slots of the largest maximum
 * block size (256 MiB) admits the same frames as that bound, and the arena is never sized above it, so SIZE_MAX means "no
 * staging bound".  LIZARDB200_ERR_ARGUMENT also for null tables when nFrames > 0; LIZARDB200_ERR_MEMORY when the workspace
 * cannot grow. */
int LizardB200_decompressFramesAsync(const void* dSrc, const uint64_t* dSrcOff, const uint64_t* dSrcSize,
                                     void* dDst, const uint64_t* dDstOff, const uint64_t* dDstCap,
                                     size_t* dResult, unsigned nFrames,
                                     unsigned maxBlocks, size_t stageBytes, void* cudaStream);
/* LizardB200_compressFrames with the offset, size and capacity tables and the results dResult[i] in device memory, and
 * enqueue-only (DESIGN.md 3.4c).  prefs is a host pointer: one set of preferences for the whole call (NULL: zeroed).  nFrames,
 * maxBlocks, stageBytes and prefs are host values; they fix the grids, the workspace and the launch sequence.  Frames are
 * admitted in index order, as a prefix: frame i is admitted while the blocks of frames 0..i number at most maxBlocks and their
 * staging bytes (each block's input length rounded up to 16) stay within stageBytes.  A frame that fails
 * LizardF_compressFrame's checks (bound, block size ID, block mode, level) and an empty frame take nothing.  An admitted frame
 * gets exactly what LizardB200_compressFrames gives it, in result and bytes (the 1-byte content-size case above included); a
 * frame that is not admitted gets LizardF_ERROR_allocation_failed and nothing is written to its range.  stageBytes above
 * maxBlocks blocks of the preferences' block size (256 MiB for an invalid block size ID) admits the same frames as that bound,
 * and the arena is never sized above it, so SIZE_MAX means "no staging bound".
 * Stream and capture rules as for LizardB200_decompressFramesAsync: the workspace (tables for nFrames and maxBlocks, stageBytes
 * of encoded blocks) grows on demand and the growing call synchronises `cudaStream`; a call that needs no growth issues no
 * host<->device copy, no synchronisation and no allocation, and can be captured in a CUDA graph after one call of the same or a
 * larger shape; each replay compresses whatever the tables then point at.  A capture that would have to grow the workspace
 * returns LIZARDB200_ERR_ARGUMENT and enqueues nothing.  Its workspace is its own: no other call of the library moves it.
 * LIZARDB200_ERR_ARGUMENT also for null tables when nFrames > 0; LIZARDB200_ERR_MEMORY when the workspace cannot grow.
 * The encoder's grid holds every SM while it runs: the call does not overlap other kernels during the encode. */
int LizardB200_compressFramesAsync(const void* dSrc, const uint64_t* dSrcOff, const uint64_t* dSrcSize,
                                   void* dDst, const uint64_t* dDstOff, const uint64_t* dDstCap,
                                   size_t* dResult, unsigned nFrames, const LizardF_preferences_t* prefs,
                                   unsigned maxBlocks, size_t stageBytes, void* cudaStream);
/* Streaming decompression of LizardF data held in device memory (DESIGN.md 3.4d): LizardF_decompress on device buffers.
 * A stream is bound to the device current when it is created; create and free return LIZARDB200_OK or an error status.
 * LizardB200_decompressStream takes device pointers dSrc / dDst and host pointers srcSizePtr / dstSizePtr.  For any sequence of
 * calls, each call returns what this library's LizardF_decompress returns when a fresh context is handed host copies of the
 * same chunks and capacities in the same order: the hint or error code, *srcSizePtr, *dstSizePtr and the bytes in
 * [dDst, dDst + *dstSizePtr).  Its rules all carry over: skippable frames, concatenated frames (a call ends at the end of a
 * frame, hint 0), LizardF_ERROR_srcPtr_wrong when dSrc is not where the previous call stopped while it left input unconsumed,
 * LizardF_ERROR_blockMode_invalid for linked blocks.  Nothing is written outside [dDst, dDst + *dstSizePtr on entry); bytes
 * behind the produced size are unspecified, as on the host.  The stream keeps the carried bytes of an incomplete block and a
 * one-block output buffer in device memory (up to the frame's maximum block size each, allocated when a header names it and
 * freed with the stream) and the running content checksum.
 * The call waits for earlier work on `cudaStream`, works on it (workspace hand-over between streams as for the other device
 * calls) and synchronises it before it returns, because it returns sizes: it is neither enqueue-only nor capturable.  A chunk
 * of many complete blocks costs a fixed number of launches whatever it holds: a walk over the block records, one decode of the
 * compressed blocks (at most 1 GiB of staging slots of the maximum block size per round; blocks decoding far below that size
 * can take further rounds), one placement and, with the content checksum, one checksum launch.  The checksum runs on one
 * warp, about 0.7 GB/s on an H100 (DESIGN.md 3.4d), which bounds a checksummed stream: there the host LizardF_decompress is
 * faster.  Device memory: the staging arena of a round is the device context's, shared by its streams and kept until the
 * process ends; it holds one slot of the maximum block size per decode unit, up to 1 GiB + one block (plus the allocator's
 * 25% when it grows) after a call with a large chunk into a large output, e.g. about 1.25 GiB for 64 MiB chunks of 128 KiB
 * blocks and about 1.6 GiB for frames of 256 MiB blocks; the units are bounded by the output's room too.  After
 * LizardF_ERROR_contentChecksum_invalid the stream is where the host context is after that error, so further calls still
 * answer alike.  A CUDA failure gives LizardF_ERROR_GENERIC, no device memory LizardF_ERROR_allocation_failed. */
typedef struct LizardB200_dstream_s LizardB200_dstream_t;
int LizardB200_createDecompressionStream(LizardB200_dstream_t** out);
int LizardB200_freeDecompressionStream(LizardB200_dstream_t* ds);
size_t LizardB200_decompressStream(LizardB200_dstream_t* ds, void* dDst, size_t* dstSizePtr,
                                   const void* dSrc, size_t* srcSizePtr, void* cudaStream);
/* Streaming compression into LizardF frames in device memory (DESIGN.md 3.4e): LizardF_compressBegin / Update / flush / End on
 * device buffers, enqueue-only.  A stream is bound to the device current when it is created; create and free return
 * LIZARDB200_OK or an error status.  dDst, dSrc and dWritten are device pointers; prefs, dstMax and srcSize host values;
 * dWritten may be NULL.
 * Same answers as the host API: for any sequence of calls, call k writes to *dWritten, in stream order, what this library's
 * LizardF_compressBegin / LizardF_compressUpdate / LizardF_flush / LizardF_compressEnd return when a fresh context is handed
 * host copies of the same preferences, chunks and capacities in the same order (a size or an error code), and writes the same
 * bytes to [dDst, dDst + size).  That covers every refusal of the host calls: refused levels and linked blocks at Begin,
 * dstMax below LizardF_compressBound, the flush's capacity check, calls in the wrong stage, and the contentSize check at End,
 * which writes the end mark and the checksum first and then the error code to *dWritten, as the host call returns it.  One
 * difference: with autoFlush, no content checksum and dstMax exactly LizardF_compressBound, an Update whose last block is 1 byte
 * long (its record is 10 bytes, 5 more than the bound counts) and whose other blocks all are stored raw does not fit; the host
 * call writes records up to its capacity and returns ERROR_dstMaxSize_tooSmall, keeping its total, while the device call
 * writes ERROR_dstMaxSize_tooSmall to *dWritten and its stream goes on as after a call that fitted.
 * A new stream answers as a fresh host context does, also before any successful Begin.
 * Host return value: the error code when the host call's result is an error, which every error here can be decided on the host;
 * otherwise 0, "enqueued".  A call refused before it does any work enqueues nothing, leaves *dWritten unwritten and leaves the
 * stream where the host context would be.
 * Enqueue-only: a call that does not grow a buffer issues no host<->device copy, no allocation and no synchronisation, and its
 * launches depend only on its host arguments and the stream's host state.  Growing synchronises `cudaStream`: the first Begin
 * for a block size (the carried block) and an Update larger than any before it, up to the round bound (a round's block table and
 * encoder slots).  Inside a capture a call that would have to grow returns LizardF_ERROR_GENERIC (LizardB200_lastError says
 * why), enqueues nothing and leaves the stream unchanged.  After one uncaptured run of the same sizes, a Begin, Update..., Flush,
 * End sequence can be captured in a CUDA graph; each replay writes a complete frame of what the source buffers then hold
 * (Begin's kernel resets the device-side state).
 * Streams: the calls on one stream object must be on one CUDA stream, or ordered by the caller (its device state is read and
 * written in stream order).  The encoder's workspace is shared by the device's calls with the hand-over of the other device calls.
 * Device memory per stream, kept until it is freed: the carried partial block (one block of the frame's block size: up to
 * 256 MiB at block size ID 7), the running XXH32 state and the call's record offset, and a round's block table and encoder slots
 * (a round takes at most 1 GiB of blocks, at least one block: for 128 KiB blocks up to 8192 blocks and 1 GiB; a chunk of more
 * blocks runs several rounds, each with the same launches).  An Update enqueues: a device-to-device copy completing the carried
 * block, per round a planning kernel, the encoder, a scan and an assembly kernel, with the content checksum one checksum
 * kernel over the chunk, a device-to-device copy of the remainder to the carried block, and a result kernel.  The checksum runs
 * on one warp, about 0.7 GB/s on an H100 (DESIGN.md 3.4d), which bounds a checksummed stream. */
typedef struct LizardB200_cstream_s LizardB200_cstream_t;
int    LizardB200_createCompressionStream(LizardB200_cstream_t** out);
int    LizardB200_freeCompressionStream(LizardB200_cstream_t* cs);
size_t LizardB200_compressStreamBegin (LizardB200_cstream_t* cs, void* dDst, size_t dstMax,
                                       const LizardF_preferences_t* prefs, size_t* dWritten, void* cudaStream);
size_t LizardB200_compressStreamUpdate(LizardB200_cstream_t* cs, void* dDst, size_t dstMax,
                                       const void* dSrc, size_t srcSize, size_t* dWritten, void* cudaStream);
size_t LizardB200_compressStreamFlush (LizardB200_cstream_t* cs, void* dDst, size_t dstMax, size_t* dWritten, void* cudaStream);
size_t LizardB200_compressStreamEnd   (LizardB200_cstream_t* cs, void* dDst, size_t dstMax, size_t* dWritten, void* cudaStream);
/* diagnostics: launch shape of the encode kernel for a level (no device needed): warps per CTA, how many of them keep their
 * hash table in shared memory, CTAs per SM (an upper bound: a launch holds no more than fit), dynamic shared memory per CTA.
 * The level's default, or LIZARDB200_ENC_SHAPE="warps,tables,ctas" when that is set and valid, exactly as the encoder
 * launches it.  Levels 23-25 / 43-45 run a kernel of their own with no shared-memory tables (4 warps, 0 tables, 5 CTAs, 0
 * bytes; LIZARDB200_ENC_SHAPE does not apply).  There the encode workspace binds first: on 132 SMs a launch holds 453 CTAs
 * (about 3.4 per SM).  Levels 18, 19 and 39 run a kernel of their own with the same shape (4, 0, 5, 0), where the workspace
 * holds 445 CTAs on 132 SMs.  LIZARDB200_ERR_LEVEL for levels whose parser is not implemented. */
int LizardB200_encodeShape(int compressionLevel, int* warpsPerCta, int* smemTables, int* ctasPerSM, int* smemBytes);
/* diagnostics (no device needed): pipeline chunk of a unit in a host-buffer call of nUnits units with unitsPerChunk units per
 * chunk (ramp != 0: the decoder's doubling ramp of small first chunks), computed by the host code and by the kernels'
 * arithmetic; returns the number of chunks, -1 if the two disagree. */
int LizardB200_chunkPlan(unsigned nUnits, unsigned unitsPerChunk, int ramp, unsigned unit, unsigned* chunk, unsigned* first, unsigned* count);
/* number of kernel launches issued by this library since load (bench.py reports it as gpu_launches) */
unsigned long long LizardB200_launchCount(void);
/* diagnostics: how this thread's device decodes, four bits: 1 = pooled copy sweeps, 2 = compact length-extension chain,
 * 4 = Huffman pre-pass kernels, 8 = token pre-pass kernel ahead of the token kernel, 16 = second-generation kernel (one CTA
 * per unit: a parser warp and a copier warp, literals stream staged through shared memory by TMA bulk copies; slower than the
 * first generation: on an H100, 1 GiB at level 10, 4.75 against 2.52 ms).  Default 7.  Results are identical for every value;
 * tools/dec_bench.py times them against each other. */
int LizardB200_setDecodeVariant(int variant);

#if defined(__cplusplus)
}
#endif
#endif /* LIZARD_B200_H */
