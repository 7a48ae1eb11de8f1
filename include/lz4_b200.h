/*
 * lz4_b200.h -- C ABI of liblz4_b200.so: an H100 (sm_90a) LZ4 block codec.
 *
 * Two layers, both plain C (pointers and sizes only, no torch / C++ types):
 *
 *  1. DROP-IN layer: the one-shot block API of the reference's lib/lz4.h and lib/lz4hc.h, same names, argument
 *     meaning, return values and error behaviour, host pointers, synchronous.  A program built
 *     against the reference's own lz4.h links against this library unchanged for these symbols
 *     (each declaration cites the lz4.h / lz4.c line it replaces; v1.10.0).
 *
 *  2. BATCH layer (additive, prefix LZ4B200_): many independent blocks per call, device pointers,
 *     asynchronous on a CUDA stream -- the measured path (SURVEY.md section 8b).  `stream` is a
 *     cudaStream_t passed as void* so that this header needs no CUDA include.
 *
 * There is no CPU fallback: without a usable CUDA device every codec entry point fails
 * (compress -> 0, decompress -> negative, batch -> LZ4B200_ERR_CUDA).
 *
 * Threads and devices: every entry point is re-entrant (the host-pointer calls share one context
 * behind a mutex).  The host-pointer calls (layers 1, 3, 4) run on the CUDA device that is current
 * in the calling thread at their FIRST use in the process; the device-pointer calls (layer 2) run
 * on the current device / the given stream, and calls that overlap in time must use different
 * workspaces.  The device-pointer calls do no host synchronisation: they only enqueue work on
 * `stream`, from any thread, and can be captured into a CUDA graph (the first call of a process
 * included).
 */
#ifndef LZ4_B200_H
#define LZ4_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#  define LZ4B200_API __attribute__((visibility("default")))
#else
#  define LZ4B200_API
#endif

/* ---------------------------------------------------------------------------------------------
 * 1. Drop-in layer  (replaces lib/lz4.c behind lib/lz4.h)
 * ------------------------------------------------------------------------------------------- */

#define LZ4B200_VERSION_NUMBER 11000          /* == LZ4_VERSION_NUMBER, lz4.h:131-135 */
#define LZ4B200_MAX_INPUT_SIZE 0x7E000000     /* == LZ4_MAX_INPUT_SIZE, lz4.h:214 */
#define LZ4B200_STATE_BYTES    16416          /* == sizeof(LZ4_stream_t), lz4.h:729-733 */
#define LZ4B200_STATEHC_BYTES  262200         /* == sizeof(LZ4_streamHC_t) == LZ4_STREAMHC_MINSIZE, lz4hc.h:252-256 */

/* lz4.h:142 / lz4.c:749 */
LZ4B200_API int LZ4_versionNumber(void);
/* lz4.h:143 / lz4.c:750 */
LZ4B200_API const char* LZ4_versionString(void);
/* lz4.h:226 / lz4.c:751: srcSize + srcSize/255 + 16, or 0 when srcSize > LZ4_MAX_INPUT_SIZE */
LZ4B200_API int LZ4_compressBound(int inputSize);
/* lz4.h:245 / lz4.c:752 */
LZ4B200_API int LZ4_sizeofState(void);

/* lz4.h:191 / lz4.c:1472.  Returns the number of bytes written into dst, 0 on failure (dst too
 * small or srcSize > LZ4_MAX_INPUT_SIZE).  Output is byte-identical to the reference's. */
LZ4B200_API int LZ4_compress_default(const char* src, char* dst, int srcSize, int dstCapacity);
/* lz4.h:236 / lz4.c:1453.  acceleration <= 0 -> 1; > 65537 -> 65537 (lz4.c:1386-1387). */
LZ4B200_API int LZ4_compress_fast(const char* src, char* dst, int srcSize, int dstCapacity, int acceleration);
/* lz4.h:246 / lz4.c:1382.  `state` is validated the way LZ4_initStream does (lz4.c:1552-1560:
 * non-NULL, 8-byte aligned) but not otherwise used: the match table lives in GPU shared memory.
 * Returns 0 for an invalid state (the reference dereferences it). */
LZ4B200_API int LZ4_compress_fast_extState(void* state, const char* src, char* dst, int srcSize, int dstCapacity, int acceleration);
/* lz4.h:611 / lz4.c:1414 -- the symbol lz4frame dispatches to (lz4frame.c:919).  Always starts
 * from a clean table, i.e. behaves like LZ4_compress_fast_extState. */
LZ4B200_API int LZ4_compress_fast_extState_fastReset(void* state, const char* src, char* dst, int srcSize, int dstCapacity, int acceleration);

/* lz4.h:248-272 / lz4.c:1506-1522.  Compresses as much of src as fits into targetDstSize bytes: returns the bytes written
 * (<= targetDstSize) and sets *srcSizePtr to the input bytes they hold; the output decodes with a capacity of exactly
 * that count.  Output, return value and *srcSizePtr are identical to the reference's:
 *   targetDstSize >= LZ4_compressBound(*srcSizePtr): LZ4_compress_fast's result, *srcSizePtr left as it is (lz4.c:1486);
 *   *srcSizePtr outside 0 .. LZ4_MAX_INPUT_SIZE: 0;  *srcSizePtr == 0: 0 if targetDstSize <= 0, else 1 (one 0x00 byte);
 *   targetDstSize < 1: 0;  otherwise the fill parse (lz4.c:1118-1122, 1147-1152, 1187-1211, 1304-1333).
 * Only the returned bytes are written to dst, never a byte at or past dst + targetDstSize.
 * Deviations: a NULL srcSizePtr or dst returns 0 (the reference dereferences them), and so does a NULL src with
 * *srcSizePtr > 0.  Without a CUDA device the call returns 0 and leaves *srcSizePtr untouched (no CPU fallback). */
LZ4B200_API int LZ4_compress_destSize(const char* src, char* dst, int* srcSizePtr, int targetDstSize);
/* lz4.h:613-617 / lz4.c:1497-1503.  LZ4_compress_destSize with an acceleration: on the compress_fast route it is clamped
 * to 1 .. 65537 (lz4.c:1386-1387); the fill parse takes it unclamped (lz4.c:1490-1493) and gives the reference's result
 * for every value from 1 to 2^25 - 1.  Deviations: acceleration <= 0 is treated as 1 there (the reference asserts, and its
 * release build can emit offset-0 matches) and values of 2^25 and above as 2^25 - 1 (beyond it the reference's
 * `acceleration << 6` overflows int).  `state` is validated as for LZ4_compress_fast_extState: an invalid state returns
 * 0 and leaves *srcSizePtr untouched. */
LZ4B200_API int LZ4_compress_destSize_extState(void* state, const char* src, char* dst, int* srcSizePtr, int targetDstSize,
                                               int acceleration);

/* The one-shot API of the reference's lib/lz4hc.h at every level, each call one block through the batched HC calls of
 * section 2: levels <= 9 (below 1 means 9) through LZ4B200_compress_blocks_hc(_destSize), levels >= 10 (above 12 means
 * 12) through LZ4B200_compress_blocks_hc_opt(_destSize).  Return values, written bytes and *srcSizePtr are the
 * reference's for every size, capacity and level.  The whole input is on the device before any byte is written back, so
 * src and dst may overlap (in-place calls); only the returned bytes are written to dst (nothing for a 0 result), never a
 * byte at or past dst + dstCapacity (targetDstSize).  Decided on the host without a launch: a size outside
 * 0 .. LZ4_MAX_INPUT_SIZE and a capacity (target) below 1 give 0; an empty input gives the one byte 0x00.
 * Cost: one GPU thread parses the block, which is far slower than the reference on one CPU core at levels 10 and up
 * (INTEGRATION.md section 1); batches belong on the section 2 calls.
 * Without a CUDA device the calls that would launch return 0 and leave dst and *srcSizePtr untouched. */
/* lz4hc.h:79 / lz4hc.c:1486 */
LZ4B200_API int LZ4_sizeofStateHC(void);
/* lz4hc.h:66 / lz4hc.c:1519-1535.  Routed as LZ4_compress_HC_extStateHC_fastReset (lz4hc.c:1506-1509): dstCapacity below
 * LZ4_compressBound(srcSize) limits the output, 0 when the block does not fit. */
LZ4B200_API int LZ4_compress_HC(const char* src, char* dst, int srcSize, int dstCapacity, int compressionLevel);
/* lz4hc.h:80 / lz4hc.c:1512-1517.  `state` is checked as LZ4_initStreamHC checks it (lz4hc.c:1573-1586): NULL or not
 * aligned like LZ4_streamHC_t (8 bytes, lz4hc.c:1488-1496) returns 0 and is not written.  A valid state is left as
 * LZ4_initStreamHC leaves it (its first 262 192 bytes zero but the compression level, 9), so the reference's
 * LZ4_resetStreamHC_fast / LZ4_compress_HC_continue accept it afterwards (lz4hc.h:373-382).  Deviation: the reference's
 * state also keeps the block just compressed, which a following LZ4_compress_HC_continue uses as its dictionary; a
 * stream continued from this state starts without one. */
LZ4B200_API int LZ4_compress_HC_extStateHC(void* state, const char* src, char* dst, int srcSize, int dstCapacity,
                                           int compressionLevel);
/* lz4hc.h:392-406 / lz4hc.c:1500-1510.  Only the alignment of `state` is checked, and the state is neither read nor
 * written.  Deviation: a NULL state returns 0 (the reference dereferences it). */
LZ4B200_API int LZ4_compress_HC_extStateHC_fastReset(void* state, const char* src, char* dst, int srcSize, int dstCapacity,
                                                     int compressionLevel);
/* lz4hc.h:83-94 / lz4hc.c:1538-1545.  The fill parse at every targetDstSize from 1 up, the bound and above included:
 * returns the bytes written (<= targetDstSize) and sets *srcSizePtr to the input bytes they hold.  `state` is checked
 * and initialised as for LZ4_compress_HC_extStateHC.  targetDstSize < 1 or *srcSizePtr outside 0 .. LZ4_MAX_INPUT_SIZE:
 * 0 with *srcSizePtr left alone.  Deviations: a NULL srcSizePtr or dst returns 0 (the reference dereferences them), and
 * so does a NULL src with *srcSizePtr > 0. */
LZ4B200_API int LZ4_compress_HC_destSize(void* state, const char* src, char* dst, int* srcSizePtr, int targetDstSize,
                                         int cLevel);

/* lz4.h:208 / lz4.c:2451.  Returns the number of bytes decoded into dst (<= dstCapacity), or a
 * negative value for malformed input / too small dst -- the same value -(position)-1 as the
 * reference's x86-64 build (lz4.c:2443).  Never reads outside src[0,compressedSize) nor writes
 * outside dst[0,dstCapacity). */
LZ4B200_API int LZ4_decompress_safe(const char* src, char* dst, int compressedSize, int dstCapacity);
/* lz4.h:274-308 / lz4.c:2459-2465.  Decodes the first min(targetOutputSize, dstCapacity) bytes (outputSize) of the block
 * and returns how many it wrote (<= outputSize), or the same negative value -(position)-1 as the reference (lz4.c:2443).
 * The return value and the bytes are the reference's: outputSize < 0 or a NULL src -> -1, outputSize == 0 -> 0 whatever
 * the input, srcSize == 0 -> -1 (lz4.c:2036, :2066, :2069); a valid block given at its exact size -> min(targetOutputSize,
 * decoded size); bytes past the block's end inside srcSize are parsed as further sequences (lz4.h:299-306).  Only
 * dst[0, return value) is written, nothing for a rejected block.
 * Deviations: a NULL dst with outputSize > 0 and a negative srcSize return -1 (undefined in the reference); an offset-0
 * match that reaches the last 12 bytes of outputSize writes zeros, as LZ4_decompress_safe does (lz4.c:2407), where the
 * reference copies whatever dst held at those bytes (lz4.c:2392-2404). */
LZ4B200_API int LZ4_decompress_safe_partial(const char* src, char* dst, int srcSize, int targetOutputSize, int dstCapacity);
/* lz4.h:546 / lz4.c:2717.  The call lz4frame makes per block (lz4frame.c:1901,1946).  dictSize == 0
 * routes to LZ4_decompress_safe exactly as lz4.c:2721-2722 does; a non-empty dictionary is out
 * of scope for the GPU path (SURVEY.md section 8 f-4) and returns -1. */
LZ4B200_API int LZ4_decompress_safe_usingDict(const char* src, char* dst, int compressedSize, int dstCapacity,
                                              const char* dictStart, int dictSize);

/* ---------------------------------------------------------------------------------------------
 * 2. Batch layer  (device pointers, asynchronous)
 * ------------------------------------------------------------------------------------------- */

#define LZ4B200_OK            0
#define LZ4B200_ERR_ARG      (-1)   /* bad argument (NULL pointer, negative count, workspace too small) */
#define LZ4B200_ERR_CUDA     (-2)   /* CUDA runtime error; see LZ4B200_last_cuda_error() */

/* Library / device introspection. */
LZ4B200_API int LZ4B200_device_count(void);
LZ4B200_API const char* LZ4B200_last_cuda_error(void);
/* Number of kernel launches issued by this library since load (bench.py's gpu_launches).  A call captured into a
 * CUDA graph counts when it is captured; replays of the graph do not count. */
LZ4B200_API uint64_t LZ4B200_launch_count(void);

/* Bytes of device workspace LZ4B200_decompress_blocks needs for nBlocks blocks of ANY capacity
 * (worst case: 32 KB of sequence marks per block). */
LZ4B200_API size_t LZ4B200_decompress_workspace_bytes(int64_t nBlocks);
/* The workspace one call wants: perBlockCaps != 0 when d_dstCap is passed, else the uniform dstCap.
 * Marks are sized by the capacity (dstCap/4 + 2 slots, at most 8192), so batches of small blocks need little
 * workspace (<= LZ4B200_decompress_workspace_bytes(nBlocks)).  A batch of blocks ABOVE 64 KB with a uniform capacity
 * of at most 64 MB (lz4frame's 256 KB .. 4 MB blocks) is decoded in 60 KB output tiles and wants two words per possible
 * sequence, i.e. about 2 x dstCap bytes per block; with a smaller workspace (at least
 * LZ4B200_decompress_workspace_bytes(nBlocks)) such a batch is still decoded, by the slow one-warp-per-block kernel. */
LZ4B200_API size_t LZ4B200_decompress_workspace_bytes_for(int64_t nBlocks, int perBlockCaps, int32_t dstCap);

/*
 * Decompress nBlocks independent LZ4 blocks (the batched LZ4_decompress_safe; replaces the serial
 * per-block loops of bench.c:514-555 and lz4frame.c:1901).
 *   block i input : d_src + d_srcOff[i], d_srcSize[i] bytes
 *   block i output: d_dst + (d_dstOff ? d_dstOff[i] : i*dstStride), capacity (d_dstCap ? d_dstCap[i] : dstCap)
 *   d_outSize[i]  : LZ4_decompress_safe's return value for block i (negative = that block is
 *                   malformed; other blocks are unaffected)
 * Output regions of different blocks must not overlap.  Enqueued on `stream`; returns LZ4B200_OK
 * once enqueued.
 * Readable padding: blocks of up to 65 535 bytes are staged by 16-byte-granular bulk loads, so the 16-byte
 * granules that hold the first and the last byte of every block are read in full -- up to 15 bytes before
 * d_src + d_srcOff[i] and after the block's end must be readable device memory (e.g. 16 bytes of slack at both
 * ends of d_src; bytes of neighbouring blocks are fine).  Nothing outside a block influences its result.
 */
LZ4B200_API int LZ4B200_decompress_blocks(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                                          void* d_dst, const int64_t* d_dstOff, int64_t dstStride,
                                          const int32_t* d_dstCap, int32_t dstCap,
                                          int32_t* d_outSize, int64_t nBlocks,
                                          void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * The same call split in its two phases (phases: 1 = scan only -- validate every block and fill
 * d_outSize with the decoded sizes / error codes without moving data, the batched equivalent of
 * asking "what would LZ4_decompress_safe return"; 2 = expand only -- move the bytes of the
 * blocks a previous scan accepted, same arguments and workspace; 3 = both).  An expand consumes what
 * its scan left in the workspace (sizes, sequence marks, the list of blocks for the generic kernel): one
 * expand per scan.
 */
LZ4B200_API int LZ4B200_decompress_blocks_phased(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                                                 void* d_dst, const int64_t* d_dstOff, int64_t dstStride,
                                                 const int32_t* d_dstCap, int32_t dstCap,
                                                 int32_t* d_outSize, int64_t nBlocks,
                                                 void* d_workspace, size_t workspaceBytes, int phases, void* stream);

/*
 * Decode a prefix of every block (the batched LZ4_decompress_safe_partial): block i is
 *   LZ4_decompress_safe_partial(src_i, dst_i, d_srcSize[i], t_i, t_i),  t_i = d_target ? d_target[i] : targetOutputSize
 * with src_i / dst_i as in LZ4B200_decompress_blocks (the target is the capacity too, lz4.h:289-296).  d_outSize[i] is its
 * return value; only dst_i[0, d_outSize[i]) is written.  Same readable padding as LZ4B200_decompress_blocks.  The workspace
 * is sized by LZ4B200_decompress_workspace_bytes_for(nBlocks, d_target != NULL, targetOutputSize).  Three kernel launches
 * (scan, shared-memory expand, one-warp expand); nBlocks == 0 returns LZ4B200_OK without one.  LZ4B200_ERR_ARG: nBlocks < 0,
 * a NULL d_src, d_srcOff, d_srcSize, d_dst, d_outSize or d_workspace, or a workspace smaller than the call needs (for a
 * uniform target above 64 KB that is less than LZ4B200_decompress_workspace_bytes_for asks: those blocks never use the
 * wide marks).  Targets of at most 64 KB are decoded in shared memory; larger ones by one warp per block.
 */
LZ4B200_API int LZ4B200_decompress_blocks_partial(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                                                  void* d_dst, const int64_t* d_dstOff, int64_t dstStride,
                                                  const int32_t* d_target, int32_t targetOutputSize,
                                                  int32_t* d_outSize, int64_t nBlocks,
                                                  void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * Decode nFrames LZ4 frames that are already in device memory (the batched LZ4B200_decompressFrame_host of section 4):
 *   frame f input : d_src + d_srcOff[f], d_srcSize[f] bytes
 *   frame f output: d_dst + d_dstOff[f], capacity d_dstCap[f]
 *   d_result[f]   : what LZ4B200_decompressFrame_host(src_f, d_srcSize[f], dst_f, d_dstCap[f], &c) returns for that frame
 *                   alone -- the decoded byte count, or its error code in its order: argument (LZ4B200_ERR_ARG: a negative
 *                   size or capacity), header, chain, then per block in order (decode failure, LZ4B200_ERR_DSTSIZE
 *                   against the capacity, the content size) -- or LZ4B200_ERR_LIMIT (below)
 *   d_consumed[f] : (may be NULL) the frame's length when its header and chain of blocks are valid, else 0 (0 as well
 *                   for a frame with LZ4B200_ERR_LIMIT)
 * The decoded bytes are the host call's: blocks are placed one after the other, short middle blocks closed up.  Nothing
 * is written outside [dst_f, dst_f + d_dstCap[f]); inside a failed frame's region the bytes are unspecified.  Output
 * regions must not overlap.  Frames are accepted exactly where the host call accepts them: independent blocks, no
 * checksums, no dictID, no skippable frames; stored-raw blocks and the content size are supported.  Same readable
 * padding as LZ4B200_decompress_blocks: 16 bytes before and after every frame.
 *
 * The budget: maxBlocks (a host array) bounds the blocks the call decodes from frames of block size ID 4 + c
 * (maxBlocks[0 .. 3]: 64 KB, 256 KB, 1 MB, 4 MB blocks); the workspace is sized by it, so that the host plans every
 * step and the call never synchronises (it can be captured into a CUDA graph).  A frame gets LZ4B200_ERR_LIMIT when the
 * blocks of the earlier frames (lower index) of its class that passed the header and chain checks, plus its own, exceed
 * maxBlocks[c] -- whatever the scheduling.  A frame's chain walk stops after maxBlocks[c] + 1 blocks, which bounds the
 * work of an untrusted frame of empty blocks; the order is therefore: header errors, then chain errors within the first
 * maxBlocks[c] + 1 blocks, then LZ4B200_ERR_LIMIT.
 *
 * Kernel launches: 5, plus 3 for maxBlocks[0] > 0 and 4 for each of maxBlocks[1 .. 3] > 0 (the two phases of
 * LZ4B200_decompress_blocks_phased per class).  nFrames == 0 returns LZ4B200_OK without one.  LZ4B200_ERR_ARG: nFrames < 0,
 * a NULL maxBlocks or an entry outside 0 .. 2^31 - 1, a NULL pointer other than d_consumed, or a workspace smaller than
 * LZ4B200_decompress_frames_workspace_bytes asks (0 for arguments the call rejects).  The workspace is about
 * 2 x maxBlocks[c] x the block size for classes 1 .. 3 (the tiles kernel's marks) and 48 bytes per frame.
 */
#define LZ4B200_ERR_LIMIT (-6)   /* per-frame result: the frame needs more blocks than the call's budget for its block size */
LZ4B200_API size_t LZ4B200_decompress_frames_workspace_bytes(int64_t nFrames, const int64_t maxBlocks[4]);
LZ4B200_API int LZ4B200_decompress_frames(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                          void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                          int64_t* d_result, int64_t* d_consumed,
                                          int64_t nFrames, const int64_t maxBlocks[4],
                                          void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * LZ4B200_decompress_frames for frames that may carry XXH32 checksums -- what the reference `lz4` tool writes by default
 * (a content checksum) and any producer with blockChecksumFlag or contentChecksumFlag set.  Same arguments, budget,
 * LZ4B200_ERR_LIMIT rule, readable padding, argument errors and workspace (LZ4B200_decompress_frames_workspace_bytes);
 * it never synchronises and can be captured into a CUDA graph.
 *
 * Frames: everything LZ4B200_decompress_frames accepts, plus FLG bit 4 (block checksums), bit 2 (content checksum) or
 * both; linked blocks, dictID and skippable frames stay LZ4B200_ERR_UNSUPPORTED.  On a frame without checksum flags the
 * result, bytes and consumed length are LZ4B200_decompress_frames's, whatever skipChecksums.
 *   - With bit 4, every block, compressed or stored raw, is followed by 4 checksum bytes; with bit 2, the EndMark is
 *     followed by 4.  They belong to the chain: a frame that ends inside one is LZ4B200_ERR_FRAME, and d_consumed[f]
 *     counts them.
 *   - skipChecksums == 0: a block checksum is XXH32(seed 0) of the block's payload as stored (the compressed bytes, or
 *     a stored-raw block's bytes), the content checksum XXH32(seed 0) of the frame's decoded content.  A mismatch gives
 *     LZ4B200_ERR_CHECKSUM, in LZ4F_decompress's order: a compressed block's checksum before its decode (decode
 *     failure, room, content size), a stored-raw block's after its room and content size, and the content checksum
 *     after the content-size check at the end of the frame.  The header checksum stays LZ4B200_ERR_FRAME.
 *   - skipChecksums != 0 (LZ4F_decompressOptions_t.skipChecksums): the fields are parsed but not compared, and the call
 *     issues exactly the launches of LZ4B200_decompress_frames.  (The reference's LZ4F_decompress still compares a
 *     compressed block's checksum under skipChecksums, lz4frame.c:1871-1883; this call compares none.)
 *
 * Reads: besides the readable padding of the frames, the content checksum reads each passing frame's decoded bytes in
 * aligned 16-byte granules, every one of which holds at least one byte of [dst_f, dst_f + d_result[f]).
 *
 * Cost: XXH32 is serial within each of its four lanes, so one thread hashes one block (the block checksums); a frame's
 * content checksum is hashed by one thread when its content is shorter than 256 KiB and otherwise by a warp that stages the
 * content through shared memory for the lane that hashes it (DESIGN sections 3.11 and 3.14 have the measured rates).
 * Kernel launches: those of LZ4B200_decompress_frames, plus 2 when skipChecksums == 0.
 */
#define LZ4B200_ERR_CHECKSUM (-7)   /* per-frame result: a block checksum or the content checksum does not match */
LZ4B200_API int LZ4B200_decompress_frames_checksummed(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                                      void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                                      int64_t* d_result, int64_t* d_consumed,
                                                      int64_t nFrames, const int64_t maxBlocks[4], int skipChecksums,
                                                      void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * Decode nFiles whole .lz4 files that are already in device memory, as `lz4 -d -c` decodes each of them piped to its
 * standard input (LZ4IO_decompressSrcFile and selectDecoder, lz4io.c:2349-2436).  "File" is the bytes of one .lz4 file:
 *   file f input : d_src + d_srcOff[f], d_srcSize[f] bytes
 *   file f output: d_dst + d_dstOff[f], d_dstCap[f] bytes of room
 * A file is a sequence of units, read from offset p with r bytes left:
 *   - r == 0 ends the file (an empty file decodes to 0 bytes); 1 <= r < 4 is LZ4B200_ERR_FRAME;
 *   - magic 0x184D2204, an LZ4 frame: the rules of LZ4B200_decompress_frames_checksummed, unchanged -- header, chain,
 *     block and content checksums (skipChecksums as there: `lz4 -d --no-frame-crc`), stored-raw blocks, content size,
 *     LZ4B200_ERR_UNSUPPORTED for linked blocks and dictID.  The unit ends after its EndMark and content checksum; a frame
 *     cut short is LZ4B200_ERR_FRAME;
 *   - magic 0x184D2A50 .. 0x184D2A5F, a skippable frame: an LE32 size, then that many bytes; it decodes to nothing.
 *     Fewer than 8 bytes, or a size that runs past the file's end, is LZ4B200_ERR_FRAME (`lz4 -d` on a pipe);
 *   - magic 0x184C2102, a legacy stream (`lz4 -l`): words w, each followed by a block of w compressed bytes decoded as
 *     LZ4_decompress_safe(block, out, w, 8 MiB), the blocks' output back to back.  The unit ends with the file or at a
 *     word above LZ4_COMPRESSBOUND(8 MiB) = 8 421 520, which is the next unit's magic.  1 .. 3 bytes where a word is due,
 *     a block cut short, or a block that fails to decode (w == 0 included) is LZ4B200_ERR_FRAME;
 *   - any other magic is LZ4B200_ERR_FRAME, at the start of a file or after other units.
 * Results:
 *   d_result[f]  : the file's decoded size, or the code of its first failing unit in file order: LZ4B200_ERR_ARG (a
 *                  negative size, or a negative room when decoding), LZ4B200_ERR_FRAME, LZ4B200_ERR_UNSUPPORTED,
 *                  LZ4B200_ERR_DSTSIZE (the unit's bytes do not fit the room left after the units before it),
 *                  LZ4B200_ERR_CHECKSUM or LZ4B200_ERR_LIMIT (below).  Inside one LZ4 frame the order is the frames call's.
 *   d_consumed[f]: (may be NULL) d_srcSize[f] on success, else the offset in the file of the failing unit's first byte
 *                  (0 for LZ4B200_ERR_ARG)
 *   d_prefix[f]  : (may be NULL) the decoded bytes of the units before the failing unit; d_result[f] on success
 * On success [dst_f, dst_f + d_result[f]) holds what `lz4 -d` writes; on failure [dst_f, dst_f + d_prefix[f]) holds the
 * output of the units before the failing one, a prefix of what `lz4 -d` writes before it fails, and the bytes after it
 * are unspecified.  Nothing is written outside [dst_f, dst_f + d_dstCap[f]); output regions must not overlap.  Readable
 * padding: 16 bytes before and after every file.
 *
 * The budget: maxUnits bounds the units the call takes (LZ4 frames, skippable frames and legacy streams over all files),
 * maxBlocks[c] the blocks of class c: maxBlocks[0 .. 3] the blocks of frames of block size ID 4 + c (64 KB .. 4 MB),
 * maxBlocks[4] legacy blocks.  Units and blocks are counted in file order, then in unit order.  A unit whose index
 * reaches maxUnits, or whose blocks with those of the earlier units of its class exceed maxBlocks[c], gets
 * LZ4B200_ERR_LIMIT, after its own header errors and its chain errors within maxBlocks[c] + 1 blocks (the frames calls'
 * rule).  A file's walk stops at its first unit that fails its header or chain rules or stops short on its budget, and
 * after maxUnits + 1 units, which bounds the work a file of tiny skippable frames can cause; only the units it took are
 * counted.  Results do not depend on scheduling.  The host plans every step from the budget and the call never
 * synchronises, so it can be captured into a CUDA graph.
 *
 * sizeOnly != 0: d_dst, d_dstOff and d_dstCap may be NULL and are not read, the room is unlimited and no byte is written.
 * The results are the decoded sizes; block checksums are still verified unless skipChecksums, content checksums are not
 * compared (no bytes are produced).  The allocate-then-decode companion for files without a content size, which is how
 * `lz4` writes them by default.
 *
 * Deviations from `lz4 -d`: linked blocks and dictID are LZ4B200_ERR_UNSUPPORTED (`lz4 -d` decodes them); under
 * skipChecksums a compressed block's checksum is not compared (the frames call's rule); a skippable frame that runs past
 * the end is LZ4B200_ERR_FRAME (the pipe behaviour, not the seekable file's); the pass-through of non-LZ4 input
 * (`lz4 -dcf`) is not offered.
 *
 * Kernel launches: 4 (the walk, the unit scan, the unit records, the fold), plus, when maxUnits > 0: 3 (the frame
 * decode's budget scan and table fill, the totals); the phases of LZ4B200_decompress_blocks_phased for every class with
 * a budget (3 for maxBlocks[0] and 4 for each of maxBlocks[1 .. 4], or only the scans when sizeOnly: 1 and 2); 1 for the
 * block checksums unless skipChecksums; and, unless sizeOnly, 3 (place, verdict, raw blocks) and 1
 * for the content checksums unless skipChecksums.  nFiles == 0 returns LZ4B200_OK without one.
 * LZ4B200_ERR_ARG: nFiles < 0, a NULL maxBlocks, maxUnits or a budget entry outside 0 .. 2^31 - 1; then, with files
 * present, a NULL d_src, d_srcOff, d_srcSize, d_result or d_workspace, a NULL d_dst, d_dstOff or d_dstCap unless
 * sizeOnly, or a workspace smaller than LZ4B200_decompress_files_workspace_bytes asks (0 for arguments the call
 * rejects).  The workspace is that of LZ4B200_decompress_frames for maxUnits frames with a fifth class of 8 MiB blocks
 * (about 2 x 8 MiB per budgeted legacy block, the tiles kernel's marks), plus 40 bytes per unit and 32 per file.
 */
#define LZ4B200_FILE_CLASSES 5   /* maxBlocks[0..3]: frame blocks of 64 KB .. 4 MB (block size ID 4 + c); [4]: legacy 8 MiB blocks */
LZ4B200_API size_t LZ4B200_decompress_files_workspace_bytes(int64_t nFiles, int64_t maxUnits,
                                                            const int64_t maxBlocks[LZ4B200_FILE_CLASSES]);
LZ4B200_API int LZ4B200_decompress_files(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                         void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                         int64_t* d_result, int64_t* d_consumed, int64_t* d_prefix,
                                         int64_t nFiles, int64_t maxUnits, const int64_t maxBlocks[LZ4B200_FILE_CLASSES],
                                         int skipChecksums, int sizeOnly,
                                         void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * Write nFrames LZ4 frames from sources in device memory (the batched LZ4F_compressFrame, lz4frame.h:224 /
 * lz4frame.c:425-498), at every compression level:
 *   frame f input : d_src + d_srcOff[f], n_f = d_srcSize[f] bytes
 *   frame f output: d_dst + d_dstOff[f], capacity d_dstCap[f]
 *   d_result[f]   : in this order, LZ4B200_ERR_ARG (n_f < 0 or d_dstCap[f] < 0), LZ4B200_ERR_DSTSIZE (d_dstCap[f] below
 *                   LZ4F_compressFrameBound(n_f, &prefs) at the frame's block size ID, 19 + 4 x blocks + n_f + 4: the
 *                   reference's dstMaxSize_tooSmall), LZ4B200_ERR_LIMIT (below), else the frame's length
 * With parallel == 0 frame f is, byte for byte, what LZ4F_compressFrame(dst_f, d_dstCap[f], src_f, n_f, &prefs) writes for
 *   prefs = { frameInfo = { blockSizeID, LZ4F_blockIndependent, noContentChecksum, LZ4F_frame,
 *                           contentSize = contentSizeFlag ? n_f : 0, dictID 0, noBlockChecksum },
 *             compressionLevel, autoFlush 1, favorDecSpeed 0 }:
 * the block size ID (0 means 4, else 4 .. 7) is shrunk per frame as LZ4F_optimalBSID does (lz4frame.c:362-373), so the
 * frames of one call can fall in different classes; an empty frame has no content-size field (lz4frame.c:445-446); a
 * block that does not compress into size - 1 bytes is stored raw (LZ4F_makeBlock, lz4frame.c:883-908).  Levels below 2
 * use LZ4_compress_fast with acceleration -level + 1 for negative levels (below -65 536 as -65 536), 1 otherwise
 * (lz4frame.c:911-921); levels 2 and up use LZ4_compress_HC_extStateHC_fastReset (lz4frame.c:931-937): 2 .. 9 through
 * the hash-chain kernel of LZ4B200_compress_blocks_hc, 10 .. 12 (above 12 reads as 12) through the optimal parser.
 * parallel != 0 (levels below 2 only; LZ4B200_ERR_ARG at the others): every block goes through LZ4B200_PARSE_PARALLEL,
 * routed by size as LZ4B200_compress_blocks_indexed routes it, with capacity size - 1; the header, block headers,
 * stored-raw rule, EndMark and results are as above.  The frame is valid and deterministic, not the reference's bytes.
 *
 * Memory: only [dst_f, dst_f + d_result[f]) is written, nothing for a failed frame; outputs may abut, and must not overlap
 * one another, any source or the workspace.  Destinations are byte-aligned anywhere.  With parallel, the 16-byte granules
 * holding the first and the last byte of every frame's source must be readable (the parse's readable padding); at levels
 * 2 and up, the aligned 4-byte words holding its bytes.
 *
 * The budget: maxBlocks (a host array) bounds the blocks the call compresses from frames of block size ID 4 + c
 * (maxBlocks[0 .. 3]: 64 KB, 256 KB, 1 MB, 4 MB blocks), the rule of LZ4B200_decompress_frames word for word: a frame
 * gets LZ4B200_ERR_LIMIT when the blocks of the earlier frames of its class that passed the checks above, plus its own,
 * exceed maxBlocks[c].  The host sizes everything from it, so the call never synchronises and can be captured into a
 * CUDA graph.  The workspace (LZ4B200_compress_frames_workspace_bytes; 0 for arguments the call rejects) holds 48 bytes
 * per frame, 48 per budgeted block, one slot of blockSize - 1 bytes rounded up to 16 per budgeted block -- about as much
 * memory as the budgeted source -- and, at levels 2 and up, the workspace of LZ4B200_compress_blocks_hc (levels 2 .. 9)
 * or LZ4B200_compress_blocks_hc_opt (10 and up) for the sum of maxBlocks.
 *
 * Kernel launches: 7 (8 with parallel); 5 when every maxBlocks[c] is 0.  nFrames == 0 returns LZ4B200_OK without one.
 * LZ4B200_ERR_ARG: nFrames < 0, a NULL maxBlocks or an entry outside 0 .. 2^31 - 1, blockSizeID outside {0, 4 .. 7},
 * parallel with compressionLevel >= 2, then (with frames present) a NULL pointer or a workspace smaller than the size
 * function asks.
 */
LZ4B200_API size_t LZ4B200_compress_frames_workspace_bytes(int64_t nFrames, const int64_t maxBlocks[4], int compressionLevel);
LZ4B200_API int LZ4B200_compress_frames(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                        void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                        int64_t* d_result, int64_t nFrames,
                                        int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                                        const int64_t maxBlocks[4],
                                        void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * LZ4B200_compress_frames with XXH32 checksums -- the frames the reference `lz4` tool writes by default (a content
 * checksum, programs/lz4io.c:223-227) and with --BX (block checksums).  The arguments, levels, parallel parse, budget,
 * LZ4B200_ERR_LIMIT rule, workspace (LZ4B200_compress_frames_workspace_bytes) and argument errors are those of
 * LZ4B200_compress_frames; the call never synchronises and can be captured into a CUDA graph.  A nonzero flag means on.
 *
 * With parallel == 0 frame f is, byte for byte, what LZ4F_compressFrame writes for the prefs of LZ4B200_compress_frames
 * with blockChecksumFlag and contentChecksumFlag set as given:
 *   - FLG bit 4 (block checksums) and bit 2 (content checksum) are set, and the header checksum byte follows from them;
 *   - with block checksums, every block is followed by the LE32 XXH32(payload, 0) of its stored payload: the compressed
 *     bytes, or a stored-raw block's source bytes (LZ4F_makeBlock, lz4frame.c:883-908);
 *   - with a content checksum, the EndMark is followed by the LE32 XXH32(source, 0) (lz4frame.c:1225-1229); an empty
 *     frame gets XXH32("", 0).
 * d_result[f] is the frame's length, checksums included.  LZ4B200_ERR_DSTSIZE applies exactly below the reference's
 * LZ4F_compressFrameBound for those prefs (lz4frame.c:376-417): 19 + (4 + 4 B) x blocks + n_f + 4 + 4 C, with B and C
 * 1 when the flag is on.  With both flags 0 the call is LZ4B200_compress_frames: the same results, bytes and launches.
 * With parallel != 0 the frames are valid, and their checksums are those of the bytes written.
 *
 * Memory: what LZ4B200_compress_frames writes and reads, and, with either flag on, the aligned 16-byte granules that
 * hold a byte of a frame's source, which the checksums read whole (at levels below 2 without parallel this is a
 * readable-padding rule the call without checksums does not have).  The block checksums hash a compressed payload in the
 * workspace, where the encoder left it, and a stored-raw block's in the source; nothing reads the destination.
 *
 * Cost: one thread hashes each block; each frame's content is hashed by one thread when it is shorter than 256 KiB and by
 * a warp that stages it through shared memory otherwise (DESIGN section 3.14 has the measured rates).  Kernel launches:
 * those of LZ4B200_compress_frames, plus 1 with block checksums and 1 with a content checksum -- 7, 8 or 9 (8, 9 or 10
 * with parallel; 5, 6 or 7 when every maxBlocks[c] is 0).
 */
LZ4B200_API int LZ4B200_compress_frames_checksummed(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                                    void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                                    int64_t* d_result, int64_t nFrames,
                                                    int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                                                    int blockChecksumFlag, int contentChecksumFlag,
                                                    const int64_t maxBlocks[4],
                                                    void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * Write nFiles `lz4 -l` legacy streams -- the format the reference tool's help calls "Linux kernel compression" -- from
 * sources in device memory, at every compression level (LZ4IO_compressLegacy_internal, programs/lz4io.c:766-910):
 *   file f input : d_src + d_srcOff[f], n_f = d_srcSize[f] bytes
 *   file f output: d_dst + d_dstOff[f], capacity d_dstCap[f]
 *   d_result[f]  : in this order, LZ4B200_ERR_ARG (n_f < 0 or d_dstCap[f] < 0), LZ4B200_ERR_DSTSIZE (d_dstCap[f] below
 *                  LZ4B200_compressLegacyBound(n_f)), LZ4B200_ERR_LIMIT (below), else the stream's length
 * File f's output is, byte for byte, what `lz4 -l -c -<level>` (`--fast=N` for level -N) writes for src_f piped to its
 * standard input: the LE32 magic 0x184C2102, then for every 8 MiB chunk of the source (the last one may be short) the LE32
 * compressed size and the compressed block.  There is no EndMark, no checksum and no stored-raw block: an incompressible
 * chunk is written compressed, larger than its input.  An empty source gives the 4-byte magic alone.  The level mapping is
 * the tool's, not LZ4B200_compress_frames's: levels below 3 use LZ4_compress_fast with acceleration -level for negative
 * levels (above 65 537 as 65 537; --fast=N is acceleration N, where a frame gets N + 1) and 1 otherwise, so level 2 is
 * the fast parse; levels 3 and up use LZ4_compress_HC (above 12 read as 12): 3 .. 9 through the hash-chain kernel of
 * LZ4B200_compress_blocks_hc, 10 .. 12 through the optimal parser.  Every chunk is compressed with capacity
 * LZ4_compressBound(chunk), as the tool's room of LZ4_compressBound(8 MiB) + 4 never limits it.  No parallel parse is
 * offered: it takes blocks of at most 64 KB, and every chunk but a short last one is 8 MiB.
 *
 * LZ4B200_compressLegacyBound(n) = 4 + the sum over the chunks of 4 + LZ4_compressBound(chunk); the tool has no capacity
 * of its own, so LZ4B200_ERR_DSTSIZE follows LZ4B200_compress_frames's convention: it is decided before encoding.  Only
 * [dst_f, dst_f + d_result[f]) is written, nothing for a failed file; outputs may abut, and must not overlap one another,
 * any source or the workspace.  Destinations are byte-aligned anywhere.  Readable padding is that of the encoder that
 * runs: at levels 3 and up, the aligned 4-byte words holding a source's bytes.
 *
 * The budget: maxBlocks bounds the 8 MiB chunks the call compresses, with LZ4B200_compress_frames's rule word for word
 * over one class: a file gets LZ4B200_ERR_LIMIT when the chunks of the earlier files that passed the checks above, plus
 * its own, exceed maxBlocks.  The host sizes everything from it, so the call never synchronises and can be captured into
 * a CUDA graph.  The workspace (LZ4B200_compress_legacy_workspace_bytes; 0 for arguments the call rejects) holds 48 bytes
 * per file, 48 per budgeted chunk, a slot of LZ4_compressBound(8 MiB) per budgeted chunk and, at levels 3 and up, the
 * workspace of LZ4B200_compress_blocks_hc (levels 3 .. 9) or LZ4B200_compress_blocks_hc_opt (10 and up) for maxBlocks
 * blocks.
 *
 * Cost: one warp parses each chunk at the fast levels, one thread at levels 3 and up, so a single large file is few
 * lanes of work; DESIGN section 3.16 has the measured times.  Kernel launches: 7; 5 when maxBlocks is 0.  nFiles == 0
 * returns LZ4B200_OK without one.  LZ4B200_ERR_ARG: nFiles < 0 or maxBlocks outside 0 .. 2^31 - 1, then (with files
 * present) a NULL pointer or a workspace smaller than the size function asks.
 */
LZ4B200_API int64_t LZ4B200_compressLegacyBound(int64_t srcSize);      /* LZ4B200_ERR_ARG for srcSize < 0 */
LZ4B200_API size_t LZ4B200_compress_legacy_workspace_bytes(int64_t nFiles, int64_t maxBlocks, int compressionLevel);
LZ4B200_API int LZ4B200_compress_legacy(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                        void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                        int64_t* d_result, int64_t nFiles, int compressionLevel, int64_t maxBlocks,
                                        void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * Compress nBlocks independent blocks (the batched LZ4_compress_fast; replaces bench.c:464-493 and
 * lz4frame.c:1046-1055).
 *   block i input : d_src + i*srcStride, size (d_srcSize ? d_srcSize[i] : srcSize)
 *   block i output: d_dst + i*dstStride, capacity dstCap  (use LZ4_compressBound(srcSize) for the
 *                   reference's notLimited behaviour)
 *   d_outSize[i]  : LZ4_compress_fast's return value for block i (0 = did not fit)
 * Each block's bytes are identical to the reference's LZ4_compress_fast output.
 */
LZ4B200_API int LZ4B200_compress_blocks(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                        void* d_dst, int64_t dstStride, int32_t dstCap, int acceleration,
                                        int32_t* d_outSize, int64_t nBlocks, void* stream);

/*
 * Compress every block into a fixed-size destination (the batched LZ4_compress_destSize_extState, lz4.c:1497):
 *   block i input : d_src + i*srcStride, size n_i = (d_srcSize ? d_srcSize[i] : srcSize)
 *   block i output: d_dst + i*dstStride; at most min(targetDstSize, LZ4_compressBound(n_i)) bytes are written, never a
 *                   byte at or past targetDstSize
 *   d_outSize[i]    : LZ4_compress_destSize_extState(state, src_i, dst_i, &n_i, targetDstSize, acceleration)
 *   d_srcConsumed[i]: what that call leaves in n_i -- the input bytes block i's output holds, or n_i itself where the
 *                     reference leaves it alone (the compress_fast route, bad sizes, failures)
 * The bytes and both values are identical to the reference's, with the acceleration rules of
 * LZ4_compress_destSize_extState above.  One kernel launch; nBlocks == 0 returns LZ4B200_OK without one.  LZ4B200_ERR_ARG:
 * nBlocks < 0, a NULL d_dst, d_outSize or d_srcConsumed, or a NULL d_src with blocks present.
 */
LZ4B200_API int LZ4B200_compress_blocks_destSize(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                                 void* d_dst, int64_t dstStride, int32_t targetDstSize, int acceleration,
                                                 int32_t* d_outSize, int32_t* d_srcConsumed, int64_t nBlocks, void* stream);

/*
 * Compress every block at an HC level (the batched LZ4_compress_HC, lz4hc.h:63 / lz4hc.c:1519-1535):
 *   block i input : d_src + i*srcStride, size n_i = (d_srcSize ? d_srcSize[i] : srcSize), any size the reference takes
 *   block i output: d_dst + i*dstStride, capacity dstCap
 *   d_outSize[i]  : LZ4_compress_HC(src_i, dst_i, n_i, dstCap, compressionLevel); block i's bytes are the reference's
 * Levels follow LZ4HC_getCLevelParams (lz4hc.c:92-116): below 1 means 9; 1 and 2 take the lz4mid parse (lz4hc.c:522-773);
 * 3 .. 9 the hash-chain parse (lz4hc.c:1121-1362) with 4 .. 256 searches, and pattern analysis at 9.  Routing is that of
 * LZ4_compress_HC_extStateHC_fastReset (lz4hc.c:1500-1510): dstCap < LZ4_compressBound(n_i) limits the output (0 when the
 * block does not fit); a size outside 0 .. LZ4_MAX_INPUT_SIZE gives 0; n_i == 0 gives the one byte 0x00 when dstCap >= 1.
 * Nothing at or past dst_i + dstCap is written; a block that returns 0 may have written its slot below dstCap.  Every
 * block starts from a fresh state, so the result does not depend on the batch, the order or the workspace.
 * The input is read in aligned 4-byte words, each of which holds at least one byte of the block.
 * The workspace is at least LZ4B200_compress_blocks_hc_workspace_bytes(nBlocks) bytes (256 KB per block, for at most
 * 16 384 blocks); a larger one lets more blocks run at once.  One kernel launch; nBlocks == 0 returns LZ4B200_OK without
 * one.  LZ4B200_ERR_ARG: compressionLevel >= 10 (the optimal parser of levels 10 .. 12 is not built), nBlocks < 0, a NULL
 * d_dst, d_outSize or d_workspace, a NULL d_src with blocks present, or a workspace smaller than the size function asks.
 */
LZ4B200_API size_t LZ4B200_compress_blocks_hc_workspace_bytes(int64_t nBlocks);
LZ4B200_API int LZ4B200_compress_blocks_hc(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                           void* d_dst, int64_t dstStride, int32_t dstCap, int compressionLevel,
                                           int32_t* d_outSize, int64_t nBlocks,
                                           void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * Compress as much of every block as fits a fixed-size destination at an HC level (the batched LZ4_compress_HC_destSize,
 * lz4hc.h:83-94 / lz4hc.c:1538-1545):
 *   block i input : d_src + i*srcStride, size n_i = (d_srcSize ? d_srcSize[i] : srcSize)
 *   block i output: d_dst + i*dstStride; nothing at or past dst_i + min(targetDstSize, LZ4_compressBound(n_i)) is
 *                   written, and the slot's bytes past d_outSize[i] below that limit are unspecified
 *   d_outSize[i]    : LZ4_compress_HC_destSize(state, src_i, dst_i, &n_i, targetDstSize, compressionLevel)
 *   d_srcConsumed[i]: what that call leaves in n_i -- the input bytes block i's output holds, or n_i itself where the
 *                     reference leaves it alone (targetDstSize < 1, a size outside 0 .. LZ4_MAX_INPUT_SIZE)
 * The bytes and both values are the reference's.  Levels are those of LZ4B200_compress_blocks_hc; unlike
 * LZ4_compress_destSize there is no unlimited route: the fill parse (fillOutput, lz4hc.c:1340-1359 and 747-772) runs at
 * every target from 1 up, the bound and above included.  Every block starts from a fresh state.
 * The input is read in aligned 4-byte words, each of which holds at least one byte of the block.
 * The workspace is at least LZ4B200_compress_blocks_hc_workspace_bytes(nBlocks) bytes, as for LZ4B200_compress_blocks_hc.
 * One kernel launch; nBlocks == 0 returns LZ4B200_OK without one.  LZ4B200_ERR_ARG: compressionLevel >= 10, nBlocks < 0,
 * a NULL d_dst, d_outSize, d_srcConsumed or d_workspace, a NULL d_src with blocks present, or a workspace smaller than
 * the size function asks.
 */
LZ4B200_API int LZ4B200_compress_blocks_hc_destSize(const void* d_src, int64_t srcStride, const int32_t* d_srcSize,
                                                    int32_t srcSize, void* d_dst, int64_t dstStride, int32_t targetDstSize,
                                                    int compressionLevel, int32_t* d_outSize, int32_t* d_srcConsumed,
                                                    int64_t nBlocks, void* d_workspace, size_t workspaceBytes,
                                                    void* stream);

/*
 * The two calls above at LZ4HC levels 10 .. 12, the optimal parser (LZ4HC_compress_optimal, lz4hc.c:1823-2123):
 *   LZ4B200_compress_blocks_hc_opt          takes the arguments of LZ4B200_compress_blocks_hc:
 *       d_outSize[i] = LZ4_compress_HC(src_i, dst_i, n_i, dstCap, compressionLevel), routed as there (a capacity below
 *       LZ4_compressBound(n_i) limits the output, 0 when the block does not fit); nothing at or past dst_i + dstCap
 *       is written
 *   LZ4B200_compress_blocks_hc_opt_destSize takes the arguments of LZ4B200_compress_blocks_hc_destSize:
 *       d_outSize[i] = LZ4_compress_HC_destSize(state, src_i, dst_i, &n_i, targetDstSize, compressionLevel) and
 *       d_srcConsumed[i] what it leaves in n_i, as there; nothing at or past dst_i + min(targetDstSize,
 *       LZ4_compressBound(n_i)) is written
 * The bytes and values are the reference's, from a fresh state per block.  Levels: 10 (96 searches, matches over 64
 * bytes taken at once), 11 (512, 128) and 12 (16 384 searches, every position searched); above 12 reads as 12.  Levels
 * below 10, including <= 0 (which the reference reads as 9), belong to the calls above and give LZ4B200_ERR_ARG here.
 * The input is read in aligned 4-byte words, each of which holds at least one byte of the block.
 * The workspace is at least LZ4B200_compress_blocks_hc_opt_workspace_bytes(nBlocks) bytes: 327 728 bytes per slot (the
 * 256 KB of tables and 4 099 x 16 bytes of prices) for min(nBlocks, 16 384) slots; a larger one gets up to one slot
 * per block.  One kernel launch; nBlocks == 0 returns LZ4B200_OK without one.  LZ4B200_ERR_ARG: compressionLevel < 10
 * (checked first), then the rules of the matching call above.
 * Cost: one thread parses a block, so a call takes as long as its slowest block, and large blocks at levels 11 and 12
 * take a long time.
 */
LZ4B200_API size_t LZ4B200_compress_blocks_hc_opt_workspace_bytes(int64_t nBlocks);
LZ4B200_API int LZ4B200_compress_blocks_hc_opt(const void* d_src, int64_t srcStride, const int32_t* d_srcSize,
                                               int32_t srcSize, void* d_dst, int64_t dstStride, int32_t dstCap,
                                               int compressionLevel, int32_t* d_outSize, int64_t nBlocks,
                                               void* d_workspace, size_t workspaceBytes, void* stream);
LZ4B200_API int LZ4B200_compress_blocks_hc_opt_destSize(const void* d_src, int64_t srcStride, const int32_t* d_srcSize,
                                                        int32_t srcSize, void* d_dst, int64_t dstStride,
                                                        int32_t targetDstSize, int compressionLevel, int32_t* d_outSize,
                                                        int32_t* d_srcConsumed, int64_t nBlocks, void* d_workspace,
                                                        size_t workspaceBytes, void* stream);

/*
 * The same call with the PARALLEL PARSE (throughput mode): every block is a valid LZ4 block that
 * LZ4_decompress_safe expands to the input, the result is deterministic, but it is NOT byte-identical to
 * LZ4_compress_fast: every position is a match candidate (no skipping), matches are chosen by the same greedy
 * rule, and the compression ratio is within 2 % of the reference's at acceleration 1 (usually above it).
 * acceleration 1..4 probe every position, 5..12 every 2nd, 13..20 every 3rd, ... (faster, lower ratio -- monotone
 * like the reference's parameter, not the same curve).  Blocks above 65 536 bytes are compressed by the
 * byte-identical encoder; with d_srcSize every block is routed by its own size and srcSize is not used.
 * d_outSize[i] == 0: block i did not fit dstCap (as LZ4_compress_fast); when it is 0, the first dstCap bytes of
 * block i's slot may have been written, the bytes past them never are.
 * Readable padding: a block of up to 65 536 bytes is staged by 16-byte-granular bulk loads, as in
 * LZ4B200_decompress_blocks, so up to 15 bytes before d_src + i*srcStride and after the block's end must be readable
 * device memory.
 */
LZ4B200_API int LZ4B200_compress_blocks_parallel(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                        void* d_dst, int64_t dstStride, int32_t dstCap, int acceleration,
                                        int32_t* d_outSize, int64_t nBlocks, void* stream);

/*
 * Pack per-block slots into one contiguous stream (what the CPU does implicitly by writing blocks
 * back to back, lz4frame.c:1046-1055): d_outOff[i] = sum_{k<i} max(d_sizes[k],0) + i*headerBytes,
 * d_outOff[nBlocks] = total; block i's bytes are copied to d_packed + d_outOff[i] + headerBytes.
 * With headerBytes == 4 a little-endian block header (the size) is written before each block, as
 * LZ4F_makeBlock does (lz4frame.c:896-907); use 0 for a bare stream.
 */
LZ4B200_API int LZ4B200_pack_blocks(const void* d_slots, int64_t slotStride, const int32_t* d_sizes, int64_t nBlocks,
                                    void* d_packed, int64_t* d_outOff, int headerBytes, void* stream);

/*
 * Compress nBlocks buffers of any sizes at any places in device memory in one call (the tensors of a checkpoint, column
 * chunks, KV-cache pages, message payloads), with the parse of one of the strided calls above:
 *   block i input : d_src + d_srcOff[i], n_i = d_srcSize[i] bytes
 *   block i output: d_dst + d_dstOff[i], capacity cap_i = d_dstCap[i]
 *   d_outSize[i]  : what the matching one-block call returns, and its bytes:
 *     LZ4B200_PARSE_FAST     LZ4_compress_fast(src_i, dst_i, n_i, cap_i, param)
 *     LZ4B200_PARSE_PARALLEL the parallel parse of LZ4B200_compress_blocks_parallel for n_i <= 65 536, and
 *                            LZ4_compress_fast(src_i, dst_i, n_i, cap_i, param) above, routed as that call routes them
 *     LZ4B200_PARSE_HC       LZ4_compress_HC(src_i, dst_i, n_i, cap_i, param): levels up to 9 (below 1 reads as 9) by the
 *                            hash-chain kernel of LZ4B200_compress_blocks_hc, 10 .. 12 (above 12 reads as 12) by the
 *                            optimal parser of LZ4B200_compress_blocks_hc_opt
 *   Sizes outside 0 .. LZ4_MAX_INPUT_SIZE, empty blocks and capacities of 0 or below give what those calls give.  Each
 *   block's capacity alone decides between limited and unlimited output.
 * Memory: nothing outside [dst_i, dst_i + cap_i) is written, so outputs may abut one another; they must not overlap one
 * another or any source.  The readable padding is that of the strided call, per block: the 16-byte granules holding a
 * block's first and last byte for PARSE_PARALLEL, the aligned 4-byte words holding its bytes for PARSE_HC.
 * Workspace: none for PARSE_FAST and PARSE_PARALLEL (the size function returns 0 and d_workspace may be NULL); for
 * PARSE_HC what LZ4B200_compress_blocks_hc_workspace_bytes or, at levels 10 and above,
 * LZ4B200_compress_blocks_hc_opt_workspace_bytes asks for nBlocks.  LZ4B200_compress_blocks_indexed_workspace_bytes
 * returns 0 for an unknown parse.
 * Launches: one for PARSE_FAST and PARSE_HC, two for PARSE_PARALLEL (blocks up to 64 KB and above, as
 * LZ4B200_compress_blocks_parallel with d_srcSize); nBlocks == 0 returns LZ4B200_OK without one.  The call does no host
 * synchronisation and can be captured into a CUDA graph.  LZ4B200_ERR_ARG: nBlocks < 0, an unknown parse, a NULL
 * d_srcOff, d_srcSize, d_dstOff, d_dstCap or d_outSize, a PARSE_HC call with a NULL d_workspace, then (with blocks
 * present) a NULL d_src or d_dst, or a PARSE_HC workspace smaller than the size function asks.
 */
#define LZ4B200_PARSE_FAST      0   /* LZ4_compress_fast, byte for byte; param = acceleration (clamped as LZ4_compress_fast) */
#define LZ4B200_PARSE_PARALLEL  1   /* the parallel parse of LZ4B200_compress_blocks_parallel; param = acceleration */
#define LZ4B200_PARSE_HC        2   /* LZ4_compress_HC, byte for byte; param = level (< 1 -> 9, > 12 -> 12) */
LZ4B200_API size_t LZ4B200_compress_blocks_indexed_workspace_bytes(int64_t nBlocks, int parse, int param);
LZ4B200_API int LZ4B200_compress_blocks_indexed(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                                                void* d_dst, const int64_t* d_dstOff, const int32_t* d_dstCap,
                                                int32_t* d_outSize, int64_t nBlocks, int parse, int param,
                                                void* d_workspace, size_t workspaceBytes, void* stream);

/*
 * LZ4B200_pack_blocks with block i's slot at d_slots + d_slotOff[i] in place of d_slots + i*slotStride: the same
 * d_outOff, headers, launches and argument rules, and LZ4B200_ERR_ARG for a NULL d_slotOff with blocks present.  It packs
 * the output of LZ4B200_compress_blocks_indexed (d_slotOff = its d_dstOff, d_sizes = its d_outSize) into one stream.
 */
LZ4B200_API int LZ4B200_pack_blocks_indexed(const void* d_slots, const int64_t* d_slotOff, const int32_t* d_sizes,
                                            int64_t nBlocks, void* d_packed, int64_t* d_outOff, int headerBytes,
                                            void* stream);

/*
 * The body of an LZ4 frame of independent blocks, assembled on the device (LZ4F_makeBlock, lz4frame.c:883-908):
 * for every block [LE32 header][payload]; a block whose compressed size d_sizes[i] is 0 (it did not fit size - 1) or
 * not smaller than its source is stored raw (payload = its source bytes from d_src + i*srcStride, bit 31 of the
 * header set).  Block i has blockSize source bytes, the last one lastSize if lastSize > 0.  d_outOff[nBlocks] = body bytes.
 */
LZ4B200_API int LZ4B200_pack_frame_blocks(const void* d_slots, int64_t slotStride, const int32_t* d_sizes,
                                          const void* d_src, int64_t srcStride, int32_t blockSize, int32_t lastSize,
                                          int64_t nBlocks, void* d_body, int64_t* d_outOff, void* stream);

/*
 * Multi-GPU reassembly (the ordered-writer role of programs/lz4io.c:594-635 when every GPU decodes a shard of a frame):
 * enqueue on `stream` the copy of `bytes` device bytes from d_src (current device) to d_dstPeer, memory of device
 * `peerDevice` that is mapped into this process (cudaIpcOpenMemHandle / a same-process allocation).  Peer access is
 * enabled on first use (a call with bytes == 0 only does that: a probe); the copy runs on a copy engine over NVLink and
 * takes no SM from the codec kernels.
 * Returns LZ4B200_OK, LZ4B200_ERR_ARG (the devices cannot reach each other directly) or LZ4B200_ERR_CUDA.
 */
LZ4B200_API int LZ4B200_peer_copy_async(void* d_dstPeer, int peerDevice, const void* d_src, size_t bytes, void* stream);

/* ---------------------------------------------------------------------------------------------
 * 3. Host-buffer batch calls (synchronous): the batch layer with the host<->device copies inside,
 *    pipelined over chunks.  h_* are host pointers (pinned memory gives full PCIe speed).
 * ------------------------------------------------------------------------------------------- */
LZ4B200_API int LZ4B200_decompress_blocks_host(const void* h_src, const int64_t* h_srcOff, const int32_t* h_srcSize,
                                               void* h_dst, int64_t dstStride, int32_t dstCap,
                                               int32_t* h_outSize, int64_t nBlocks);
LZ4B200_API int LZ4B200_compress_blocks_host(const void* h_src, int64_t srcStride, int32_t srcSize, int64_t lastSize,
                                             void* h_dst, int64_t dstStride, int32_t dstCap, int acceleration,
                                             int32_t* h_outSize, int64_t nBlocks);

/*
 * Decode nFiles whole .lz4 files in host memory, as LZ4B200_decompress_files (section 2) decodes them in device memory,
 * with no budget and no workspace: file f is h_src + h_srcOff[f], h_srcSize[f] bytes, and decodes to h_dst +
 * h_dstOff[f] with h_dstCap[f] bytes of room.
 *   h_result[f], h_consumed[f], h_prefix[f] (the last two optional): what LZ4B200_decompress_files returns for the same
 *   files with a budget that covers them all -- the same grammar, unit order, error order inside a frame, skipChecksums
 *   and sizeOnly rules and the same deviations from `lz4 -d` -- so never LZ4B200_ERR_LIMIT.
 * On success [dst_f, dst_f + result) holds what `lz4 -d` writes; on failure [dst_f, dst_f + prefix) holds the output of
 * the units before the failing one.  Nothing outside [dst_f, dst_f + cap_f) is written.  sizeOnly != 0: no byte is
 * written and h_dst, h_dstOff and h_dstCap may be NULL.  Host regions must not overlap each other or the source; no
 * readable padding is needed (the call stages the bytes itself).
 * The files are walked on the host and their blocks cut into groups of at most 64 MiB of decode capacity (one block at
 * least; small files share a group, a large frame spans many).  Each group goes through the device on one of the
 * pipeline's streams -- its source pieces up, one decode per block class, the block checksums, its output assembled in
 * file order, the content hashes (a frame's hash state carried from group to group in device memory), its bytes down --
 * with four groups in flight, so device memory is bounded by the pipeline, not by the files.  DESIGN section 3.17.
 * Returns LZ4B200_OK, LZ4B200_ERR_ARG (nFiles < 0; with files, a NULL h_src, h_srcOff, h_srcSize or h_result, or a NULL
 * h_dst, h_dstOff or h_dstCap unless sizeOnly; or host memory for the walk ran out, which LZ4B200_last_cuda_error()
 * then says) or LZ4B200_ERR_CUDA (no device
 * included: there is no CPU fallback).  nFiles == 0 returns LZ4B200_OK without touching the device.  Synchronous; one
 * host-buffer call runs at a time.
 */
LZ4B200_API int LZ4B200_decompress_files_host(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                              void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                              int64_t* h_result, int64_t* h_consumed, int64_t* h_prefix,
                                              int64_t nFiles, int skipChecksums, int sizeOnly);

/*
 * Write nFiles whole .lz4 files from host memory, as LZ4B200_compress_frames_checksummed (frames) and
 * LZ4B200_compress_legacy (`lz4 -l` streams) write them in device memory, with no budget, no workspace and no stream:
 * file f is h_src + h_srcOff[f], h_srcSize[f] bytes, and is written to h_dst + h_dstOff[f] with h_dstCap[f] bytes of
 * room.
 *   h_result[f]: what the device call returns for the same file with the same arguments and a budget that covers every
 *   file -- the file's length, or LZ4B200_ERR_ARG (a negative size or capacity), or LZ4B200_ERR_DSTSIZE, in the device
 *   call's order; never LZ4B200_ERR_LIMIT.  The bytes are the device call's, so with parallel == 0 they are the reference
 *   tool's: `lz4 -c -<level> [-B4..7] [--BX] [--no-frame-crc] [--content-size]` and `lz4 -l -c -<level>`.  Each call
 *   keeps the device call's level mapping: level 2 is lz4mid's HC parse for a frame and the fast parse for a legacy
 *   stream.
 * LZ4B200_ERR_DSTSIZE is decided before encoding, against the device call's bound: LZ4B200_compressFrameBound_checksummed
 * for frames (capacity == bound succeeds, bound - 1 fails; LZ4B200_compressFrameBound, which has no checksums and some
 * slack, is not this threshold), LZ4B200_compressLegacyBound for legacy streams.  Only [dst_f, dst_f + h_result[f]) is
 * written, nothing for a failed file.  Host regions must not overlap each other or the source; no readable padding is
 * needed (the call stages the bytes itself, 16-byte aligned with slack).
 * The files' blocks are cut into groups of at most G source bytes (LZ4B200_HOST_WRITE_MB, default 512 MiB) and B blocks
 * (2 048 at HC levels, 65 536 otherwise), one block at least; small files share a group, a large file spans many.  Each
 * group goes through the device on one of the pipeline's four streams -- its source pieces up, one encode, the body
 * assembled with stored-raw blocks and block checksums, the content checksums (a frame's hash state carried from group to
 * group in device memory), its offsets down -- and its body goes to each file's place when it retires; the host writes
 * headers, EndMarks and digests.  Device memory held at most, over the four slots: 4 x (the staged source, 2 G + 16 B;
 * the encode's slots, G + G/255 + 32 B; the body, G + G/255 + 24 B; the table, 56 B + 8; at HC levels the HC
 * workspace, 256 KB x B at levels 2 .. 9 and 320 KB x B at 10 .. 12; each buffer rounded up by at most 1 MiB + 16
 * bytes), plus 5 x 40 bytes of carried hash state, where G stands for the larger of G and the largest block.  The slots
 * are shared with the other host-buffer calls and kept between calls.
 * DESIGN section 3.18.
 * Returns LZ4B200_OK, LZ4B200_ERR_ARG (nFiles < 0; for frames blockSizeID outside {0, 4 .. 7}, 0 meaning 4, or parallel
 * with compressionLevel >= 2; then, with files, a NULL pointer; or host memory for the plan ran out, which
 * LZ4B200_last_cuda_error() then says) or LZ4B200_ERR_CUDA (no device included: there is no CPU fallback).  nFiles == 0
 * returns LZ4B200_OK without touching the device.  Synchronous; one host-buffer call runs at a time.
 */
LZ4B200_API int LZ4B200_compress_frames_host(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                             void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                             int64_t* h_result, int64_t nFiles,
                                             int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                                             int blockChecksumFlag, int contentChecksumFlag);
LZ4B200_API int LZ4B200_compress_legacy_host(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                             void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                             int64_t* h_result, int64_t nFiles, int compressionLevel);

/*
 * Decode nFiles whole .lz4 files in host memory into device memory: LZ4B200_decompress_files_host with the output in
 * device memory.  File f is h_src + h_srcOff[f], h_srcSize[f] bytes, and decodes to d_dst + h_dstOff[f] with h_dstCap[f]
 * bytes of room; d_dst is one device base pointer, the offset, size and capacity arrays are host arrays.
 *   h_result[f], h_consumed[f], h_prefix[f] (the last two optional): what LZ4B200_decompress_files_host returns for the
 *   same files and arguments with sizeOnly == 0 -- the same grammar, unit order, verdict order, skipChecksums rule and
 *   deviations from `lz4 -d`.  There is no size-only mode: LZ4B200_decompress_files_host answers it from the same bytes.
 * On success [d_dst + h_dstOff[f], + result) holds the host call's bytes; on failure [.., + prefix) does.  Nothing
 * outside [d_dst + h_dstOff[f], + h_dstCap[f]) is written; destinations are byte-aligned anywhere and must not overlap
 * one another.  Only compressed bytes cross PCIe, in one direction: each group's output is copied from the pipeline's
 * buffer to the files in device memory by one scatter kernel per group (DESIGN section 3.19).
 * Device memory held at most: section 3.17's four slots, plus per slot a run table of 24 bytes x (the group's blocks +
 * 64 MiB / 256 KiB + 1) in device and pinned memory.
 * Ordering: the call's device work starts after the work enqueued on `stream` (a cudaStream_t, NULL for the legacy
 * default stream) before the call, and every write to d_dst is complete when it returns.  Synchronous; one host-buffer
 * call runs at a time.
 * Returns LZ4B200_OK, LZ4B200_ERR_ARG (in this order: nFiles < 0; then, with files, a NULL pointer other than h_consumed
 * and h_prefix; d_dst not device or managed memory of the pipeline's device, or an h_ pointer that is device memory,
 * which LZ4B200_last_cuda_error() names; host memory for the walk ran out) or LZ4B200_ERR_CUDA (no device included:
 * there is no CPU fallback).  nFiles == 0 returns LZ4B200_OK without touching the device.
 */
LZ4B200_API int LZ4B200_decompress_files_to_device(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                                   void* d_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                                   int64_t* h_result, int64_t* h_consumed, int64_t* h_prefix,
                                                   int64_t nFiles, int skipChecksums, void* stream);

/*
 * Write nFiles whole .lz4 files from device memory into host memory: LZ4B200_compress_frames_host and
 * LZ4B200_compress_legacy_host with the source in device memory.  File f is d_src + h_srcOff[f], h_srcSize[f] bytes (d_src
 * one device base pointer, the arrays host arrays), written to h_dst + h_dstOff[f] with h_dstCap[f] bytes of room.
 *   h_result[f] and the bytes: exactly what the host writer returns and writes for the same sources and arguments -- so
 *   the reference tool's bytes with parallel == 0, the same LZ4B200_ERR_DSTSIZE thresholds and level mappings, never
 *   LZ4B200_ERR_LIMIT.  Only [dst_f, dst_f + h_result[f]) is written.
 * The source is read where it lies, so its readable padding is the device calls': the aligned 16-byte granules holding
 * a byte of a file (LZ4B200_compress_frames_checksummed; with neither checksum, the encoder's rule), and at HC levels
 * the aligned 4-byte words holding one (LZ4B200_compress_legacy).  Only compressed bytes cross PCIe, in one direction.
 * Device memory held at most: that of the host writers above without the staged source (2 G + 16 bytes per slot).
 * Ordering: the call's device work starts after the work enqueued on `stream` before the call.  Synchronous; one
 * host-buffer call runs at a time.  DESIGN section 3.19.
 * Returns LZ4B200_OK or, in this order: LZ4B200_ERR_ARG for nFiles < 0; LZ4B200_OK for nFiles == 0 without touching the
 * device; LZ4B200_ERR_ARG for a NULL pointer, for frames blockSizeID outside {0, 4 .. 7} or parallel with
 * compressionLevel >= 2, d_src not device or managed memory of the pipeline's device, or an h_ pointer that is device
 * memory (LZ4B200_last_cuda_error() names it), or host memory for the plan ran out; LZ4B200_ERR_CUDA (no device
 * included: there is no CPU fallback).
 */
LZ4B200_API int LZ4B200_compress_frames_from_device(const void* d_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                                    void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                                    int64_t* h_result, int64_t nFiles,
                                                    int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                                                    int blockChecksumFlag, int contentChecksumFlag, void* stream);
LZ4B200_API int LZ4B200_compress_legacy_from_device(const void* d_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                                    void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                                    int64_t* h_result, int64_t nFiles, int compressionLevel, void* stream);

/* The capacity below which LZ4B200_compress_frames_checksummed and LZ4B200_compress_frames_host give a frame of srcSize
 * bytes LZ4B200_ERR_DSTSIZE: LZ4F_compressFrameBound for the checksums at the frame's own block size ID (blockSizeID
 * shrunk as LZ4F_optimalBSID does), 19 + (4 + 4 B) x blocks + srcSize + 4 + 4 C.  LZ4B200_ERR_ARG for srcSize < 0 or
 * blockSizeID outside {0, 4 .. 7}. */
LZ4B200_API int64_t LZ4B200_compressFrameBound_checksummed(int64_t srcSize, int blockSizeID, int blockChecksumFlag,
                                                           int contentChecksumFlag);

/* ---------------------------------------------------------------------------------------------
 * 4. Frame layer (SURVEY.md section 8 f-1): one-shot LZ4 frames of INDEPENDENT blocks, host buffers.
 *    The container logic (header, block headers, EndMark) runs on the host, every block goes through
 *    the batch layer in one pipeline instead of lz4frame.c's serial per-block loop
 *    (lz4frame.c:1046-1055 / :1839-1919).
 * ------------------------------------------------------------------------------------------- */
#define LZ4B200_ERR_FRAME        (-3)   /* malformed frame (bad magic / header checksum / block size / truncated) */
#define LZ4B200_ERR_UNSUPPORTED  (-4)   /* valid LZ4 frame feature outside this layer: linked blocks, block or
                                           content checksums, dictID, skippable frames, HC levels */
#define LZ4B200_ERR_DSTSIZE      (-5)   /* destination buffer too small */

/* Upper bound of the frame LZ4B200_compressFrame_host can produce (>= LZ4F_compressFrameBound, lz4frame.c:406). */
LZ4B200_API int64_t LZ4B200_compressFrameBound(int64_t srcSize, int blockSizeID);

/*
 * LZ4F_compressFrame (lz4frame.h:224 / lz4frame.c:484) for preferences
 *   { frameInfo = { blockSizeID, LZ4F_blockIndependent, noContentChecksum, LZ4F_frame,
 *                   contentSize = contentSizeFlag ? srcSize : 0, dictID 0, noBlockChecksum },
 *     compressionLevel <= 1 (0/1: acceleration 1; negative: acceleration -level+1, lz4frame.c:913) }.
 * blockSizeID: 0 (default = 4) or 4..7 = 64 KB / 256 KB / 1 MB / 4 MB; shrunk for small inputs exactly like
 * LZ4F_optimalBSID (lz4frame.c:362-373).  The frame is byte-identical to the reference's.
 * Returns the frame size, or a negative LZ4B200_ERR_* value.
 */
LZ4B200_API int64_t LZ4B200_compressFrame_host(const void* h_src, int64_t srcSize, void* h_dst, int64_t dstCapacity,
                                               int blockSizeID, int compressionLevel, int contentSizeFlag);

/*
 * Decode ONE whole frame (the one-shot use of LZ4F_decompress, lz4frame.c:1613): header checks as
 * LZ4F_decodeHeader (lz4frame.c:1340-1425), then all blocks in one batch (stored-raw blocks are copied).
 * Returns the number of decoded bytes, or a negative LZ4B200_ERR_* value (LZ4B200_ERR_FRAME also when a
 * block fails to decode or the content size field disagrees).  *consumed (optional) = frame length.
 */
LZ4B200_API int64_t LZ4B200_decompressFrame_host(const void* h_src, int64_t srcSize, void* h_dst, int64_t dstCapacity,
                                                 int64_t* consumed);

#ifdef __cplusplus
}
#endif
#endif /* LZ4_B200_H */
