/*
 * oracle/lz4_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement of the reference LZ4 block codec (lz4/lz4 v1.10.0, lib/lz4.c) used as the
 * parity checker for the CUDA path.  Nothing in the product (lz4_b200/, include/) may include,
 * link or call this; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs do.
 *
 * lz4_oracle.c holds the block codec: one parse for LZ4_compress_fast and LZ4_compress_destSize,
 * one decoder for LZ4_decompress_safe and LZ4_decompress_safe_partial.  datagen_oracle.c holds the
 * data generator and cpu_harness.c the timing harness.  oracle/pyoracle.py wraps them all
 * (`Oracle`) and the reference's matching entry points (`Reference`).
 *
 * Parity pin: oracle/_ref/libref_lz4.so (the unmodified reference lib/lz4.c compiled in place
 * by oracle/Makefile) -- tests/test_oracle_vs_ref.py, tests/test_destsize_oracle.py and
 * tests/test_partial_oracle.py check identical return values and bytes against it, and
 * tests/golden/ holds vectors generated from it (make_golden.py, make_golden_destsize.py,
 * make_golden_partial.py).
 */
#ifndef LZ4_ORACLE_H
#define LZ4_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* lz4.h:214-215, lz4.c:751 */
int oracle_lz4_compress_bound(int srcSize);

/* lz4.c:1453 (LZ4_compress_fast) -> :1382 (extState) -> :1344 (generic) -> :930 (generic_validated),
 * noDict / noDictIssue instantiation, 64-bit little-endian host. Byte-identical output. */
int oracle_lz4_compress_fast(const uint8_t* src, uint8_t* dst, int srcSize, int dstCapacity, int acceleration);

/* lz4.c:2451 (LZ4_decompress_safe) -> :2022 (LZ4_decompress_generic, decode_full_block, noDict),
 * x86-64 build (LZ4_FAST_DEC_LOOP=1): same accepted set, same return value (size or -(ip)-1),
 * same bytes in dst[0, ret). */
int oracle_lz4_decompress_safe(const uint8_t* src, uint8_t* dst, int compressedSize, int dstCapacity);

/* *path of oracle_lz4_compress_destSize_extState: the route taken and, in the fill parse, the first
 * output limit met */
enum oracle_ds_path {
    ORACLE_DS_PATH_FAST = 0,          /* target >= LZ4_compressBound(n): LZ4_compress_fast_extState (lz4.c:1486-1487) */
    ORACLE_DS_PATH_EMPTY = 1,         /* n == 0 (lz4.c:1361-1371) */
    ORACLE_DS_PATH_NO_ROOM = 2,       /* target < 1 (lz4.c:985) */
    ORACLE_DS_PATH_LITERALS = 3,      /* the literal check dropped a token (lz4.c:1118-1122) */
    ORACLE_DS_PATH_NEXT_MATCH = 4,    /* the _next_match check rewound to a token (lz4.c:1147-1152) */
    ORACLE_DS_PATH_REDUCED = 5,       /* a match was shortened (lz4.c:1187-1207) */
    ORACLE_DS_PATH_LAST_LITERALS = 6, /* the last literal run was cut (lz4.c:1305-1311) */
    ORACLE_DS_PATH_FILLED = 7,        /* the whole input fit without meeting a limit */
    ORACLE_DS_PATH_BAD_SIZE = 8       /* n outside 0 .. LZ4_MAX_INPUT_SIZE below the bound (lz4.c:1360) */
};

/* lz4.c:1481-1503 (LZ4_compress_destSize_extState, and LZ4_compress_destSize at acceleration 1)
 * -> :1344 / :930 with fillOutput; the route where success is guaranteed is
 * oracle_lz4_compress_fast.  Byte-identical output, return value and *srcSizePtr.  The acceleration
 * reaches the fill parse unclamped (lz4.c:1490-1493); values below 1 (the reference asserts) are
 * taken as 1 and values of 2^25 and above (where the reference's `acceleration << 6` overflows int)
 * as 2^25 - 1.  *path (may be NULL) receives an oracle_ds_path code.  The names differ from the
 * restatement this replaced (oracle_lz4_compress_destSize, ORACLE_DS_*), which older test trees
 * still compile next to this file. */
int oracle_lz4_compress_destSize_extState(const uint8_t* src, uint8_t* dst, int* srcSizePtr, int targetDstSize,
                                          int acceleration, int* path);

/* lz4.c:2459-2465 (LZ4_decompress_safe_partial) -> :2022 (partial_decode, noDict): same return
 * value and bytes.  Documented deviations: a negative srcSize returns -1, and an offset-0 match
 * writes zeros everywhere (lz4.c:2407, :500), also on the cut path of lz4.c:2392-2404, where the
 * reference copies dst onto itself (bytes that depend on what dst held, including what its own
 * over-long copies left there).  *lastPath: bit 0 = stopped after literals, bit 1 = stopped
 * inside a match, bit 2 = such an offset-0 cut was taken. */
int oracle_lz4_decompress_safe_partial(const uint8_t* src, uint8_t* dst, int srcSize, int targetOutputSize,
                                       int dstCapacity, int* lastPath);

/* tests/datagen.c:154-160 (RDG_genBuffer): synthetic compressible data, byte-identical. */
void oracle_datagen(uint8_t* buffer, size_t size, double matchProba, double litProba, unsigned seed);

/* Walk a valid block and report sequence statistics (used by tests / DESIGN numbers). */
typedef struct {
    uint32_t n_sequences;      /* tokens, including the final literal-only one */
    uint32_t literal_bytes;
    uint32_t match_bytes;
    uint32_t overlap_matches;  /* offset < match length */
} oracle_block_stats;
int oracle_lz4_block_stats(const uint8_t* src, int compressedSize, oracle_block_stats* st);

/* ---- CPU timing harness (bench.py cpu_baseline / --impl reference) ------------------------- */
typedef int (*oracle_decomp_fn)(const char* src, char* dst, int compressedSize, int dstCapacity);
typedef int (*oracle_comp_fn)(const char* src, char* dst, int srcSize, int dstCapacity, int acceleration);

/* Decompress nBlocks blocks (src + srcOff[i], size srcSize[i]) into dst + i*dstStride with
 * `threads` pthreads (static partition, as BASELINE.md section 3); returns wall seconds of the
 * pass, or <0 if any block failed.  outSizes[i] receives each return value. */
double oracle_time_decompress(oracle_decomp_fn fn, const uint8_t* src, const int64_t* srcOff,
                              const int32_t* srcSize, uint8_t* dst, int64_t dstStride, int32_t dstCap,
                              int32_t* outSizes, int64_t nBlocks, int threads);
double oracle_time_compress(oracle_comp_fn fn, const uint8_t* src, int64_t srcStride, int32_t srcSize,
                            int64_t lastSize, uint8_t* dst, int64_t dstStride, int32_t dstCap, int accel,
                            int32_t* outSizes, int64_t nBlocks, int threads);
/* multi-threaded datagen: segment k of segBytes gets seed seed0+k */
void oracle_first_touch(uint8_t* dst, int64_t dstStride, int64_t nBlocks, int threads);
void oracle_pack(const uint8_t* slots, int64_t slotStride, const int32_t* sizes, const int64_t* packOff,
                 uint8_t* packed, int64_t nBlocks, int threads);
void oracle_datagen_mt(uint8_t* buffer, size_t size, size_t segBytes, double matchProba, unsigned seed0, int threads);

#ifdef __cplusplus
}
#endif
#endif
