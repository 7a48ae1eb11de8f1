/*
 * lz4_kernels.h -- the thin extern "C" FFI between the C host layer (lz4_api.c) and the CUDA
 * kernels (lz4_kernels.cu).  Launchers only enqueue work on `stream`; they return a cudaError_t
 * value as int.
 */
#ifndef LZ4_KERNELS_H
#define LZ4_KERNELS_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    const uint8_t* src;        /* base of compressed bytes */
    const int64_t* srcOff;     /* [n] */
    const int32_t* srcSize;    /* [n] */
    uint8_t* dst;
    const int64_t* dstOff;     /* [n] or NULL -> i*dstStride */
    int64_t dstStride;
    const int32_t* dstCapArr;  /* [n] or NULL -> dstCap */
    int32_t dstCap;
    int32_t* outSize;          /* [n] */
    int64_t nBlocks;
    void* workspace;
    size_t workspaceBytes;
} lz4k_decode_args;

typedef struct {
    const uint8_t* src;
    const int64_t* srcOff;     /* [n] or NULL -> i*srcStride */
    int64_t srcStride;
    const int32_t* srcSizeArr; /* [n] or NULL -> srcSize */
    int32_t srcSize;
    uint8_t* dst;
    const int64_t* dstOff;     /* [n] or NULL -> i*dstStride */
    int64_t dstStride;
    const int32_t* dstCapArr;  /* [n] or NULL -> dstCap */
    int32_t dstCap;
    int32_t acceleration;
    int32_t* outSize;
    int64_t nBlocks;
    int32_t minSize, maxSize;  /* only blocks of minSize .. maxSize bytes are compressed; the others (slot and outSize)
                                  are left to another launch */
} lz4k_encode_args;

/* the workspace a decode call of per-block capacities (perBlockCaps != 0) or one capacity dstCap for every block uses when
 * it is given workspaceBytes: SIZE_MAX gives the size that enables the tiles kernel, 0 the smallest a call accepts (the
 * partial call's layout) */
size_t lz4k_decode_workspace_bytes(int64_t nBlocks, int perBlockCaps, int32_t dstCap, size_t workspaceBytes);
/* phases: bit 0 = scan (validate, sizes), bit 1 = expand (move bytes; needs a prior scan's outSize).  partial:
 * LZ4_decompress_safe_partial per block with outputSize = (dstCapArr ? dstCapArr[i] : dstCap), both phases */
int lz4k_launch_decode(const lz4k_decode_args* a, int phases, int partial, void* stream);
int lz4k_launch_encode(const lz4k_encode_args* a, void* stream);       /* byte-identical to LZ4_compress_fast */
int lz4k_launch_encode_par(const lz4k_encode_args* a, void* stream);   /* parallel parse; blocks of <= 65 536 bytes */
/* byte-identical to LZ4_compress_destSize_extState with targetDstSize = dstCap: outSize[i] its return value,
 * srcConsumed[i] what it leaves in *srcSizePtr (block i's own size where it leaves it alone) */
int lz4k_launch_encode_dest(const lz4k_encode_args* a, int32_t* srcConsumed, void* stream);
/* byte-identical to LZ4_compress_HC(src_i, dst_i, n_i, dstCap, level) for level <= 9 (the caller rejects the others);
 * the workspace holds lz4k_encode_hc_workspace_bytes(nBlocks) bytes or more, one launch */
size_t lz4k_encode_hc_workspace_bytes(int64_t nBlocks);
int lz4k_launch_encode_hc(const lz4k_encode_args* a, int level, void* workspace, size_t workspaceBytes, void* stream);
/* byte-identical to LZ4_compress_HC_destSize(state, src_i, dst_i, &n_i, dstCap, level) for level <= 9: outSize[i] its
 * return value, srcConsumed[i] what it leaves in n_i; the workspace as for lz4k_launch_encode_hc, one launch */
int lz4k_launch_encode_hc_dest(const lz4k_encode_args* a, int32_t* srcConsumed, int level, void* workspace,
                               size_t workspaceBytes, void* stream);
/* the two calls above for level >= 10 (the caller rejects the others), the optimal parser; the workspace holds
 * lz4k_encode_hc_opt_workspace_bytes(nBlocks) bytes or more, one launch */
size_t lz4k_encode_hc_opt_workspace_bytes(int64_t nBlocks);
int lz4k_launch_encode_hc_opt(const lz4k_encode_args* a, int level, void* workspace, size_t workspaceBytes, void* stream);
int lz4k_launch_encode_hc_opt_dest(const lz4k_encode_args* a, int32_t* srcConsumed, int level, void* workspace,
                                   size_t workspaceBytes, void* stream);
/* block i's bytes are at slots + (slotOff ? slotOff[i] : i*slotStride) */
int lz4k_launch_pack(const uint8_t* slots, const int64_t* slotOff, int64_t slotStride, const int32_t* sizes,
                     int64_t nBlocks, uint8_t* packed, int64_t* outOff, int headerBytes, void* stream);
/* the body of an LZ4 frame: [LE32 block header][payload] per block; blocks whose compression did not gain are stored raw */
int lz4k_launch_pack_frame(const uint8_t* slots, int64_t slotStride, const int32_t* sizes, const uint8_t* src, int64_t srcStride,
                           int32_t blockSize, int32_t lastSize, int64_t nBlocks, uint8_t* packed, int64_t* outOff, void* stream);
/* the batched frame decode's own steps (lz4_frame_core.h); the decode of the blocks between them is the caller's */
typedef struct {
    const uint8_t* src;        /* the call's frames: frame f is src + srcOff[f], srcSize[f] bytes */
    const int64_t* srcOff;
    const int64_t* srcSize;
    uint8_t* dst;              /* frame f decodes to dst + dstOff[f], dstCap[f] bytes of room */
    const int64_t* dstOff;
    const int64_t* dstCap;
    int64_t* result;           /* [nFrames] */
    int64_t* consumed;         /* [nFrames] or NULL */
    int64_t nFrames;
    int64_t maxBlocks[5];      /* the budget of every class (FC_CLASSES; the frames calls give class 4 none) */
    int64_t tabBase[5];        /* class c's entries of the block table start at tabBase[c] */
    int64_t nEntries;          /* entries of the block table (sum of maxBlocks) */
    int mode;                  /* FC_SUMS_* (lz4_frame_core.h): the checksum flags rejected, skipped or verified */
    void* frames;              /* fc_frame_rec[nFrames] */
    int64_t* tabSrcOff; int64_t* tabDstOff; int32_t* tabSrcSize; int32_t* tabOutSize; int32_t* tabRawLen;
} lz4k_frames_args;

/* pass 1 (index), the per-class scan with the budget rule, then the table cleared and filled (pass 2) */
int lz4k_launch_frames_index(const lz4k_frames_args* a, void* stream);
/* the verdict on every frame, once the scans of every class have run; the expands follow it */
int lz4k_launch_frames_verdict(const lz4k_frames_args* a, void* stream);
/* the stored-raw blocks of the frames that passed, to their place */
int lz4k_launch_frames_raw(const lz4k_frames_args* a, void* stream);
/* FC_SUMS_VERIFY: every marked block's checksum, before the verdict */
int lz4k_launch_frames_block_sums(const lz4k_frames_args* a, void* stream);
/* FC_SUMS_VERIFY: the content checksum of every frame that passed, after the raw blocks */
int lz4k_launch_frames_content_sums(const lz4k_frames_args* a, void* stream);
/* the batched file decode's own steps (lz4_frame_core.h): its units run through the frame decode's steps as the frames
 * of `u`, whose per-frame tables (srcOff, srcSize, dstOff, dstCap, result) are the units' own, in the workspace */
typedef struct {
    const int64_t* srcOff;     /* file f is u.src + srcOff[f], srcSize[f] bytes */
    const int64_t* srcSize;
    const int64_t* dstOff;     /* file f decodes to u.dst + dstOff[f], dstCap[f] bytes of room (NULL when sizing) */
    const int64_t* dstCap;
    int64_t* result;           /* [nFiles] */
    int64_t* consumed;         /* [nFiles] or NULL */
    int64_t* prefix;           /* [nFiles] or NULL */
    int64_t nFiles;
    int64_t maxUnits;          /* records of u (u.nFrames) */
    int sizeOnly;
    void* files;               /* fc_file_rec[nFiles] */
    lz4k_frames_args u;
} lz4k_files_args;

/* the walk of every file, the scan of the unit counts, the unit records (fill), then the frame decode's budget scan and
 * table fill on them (as lz4k_launch_frames_index) */
int lz4k_launch_files_index(const lz4k_files_args* a, void* stream);
/* after the scans of the blocks (and the block checksums): every unit's totals into u.result */
int lz4k_launch_files_totals(const lz4k_files_args* a, void* stream);
/* after the totals: every unit's place and room (u.dstOff, u.dstCap); the frame verdict follows */
int lz4k_launch_files_place(const lz4k_files_args* a, void* stream);
/* last: every file's result, consumed and prefix from the unit results */
int lz4k_launch_files_fold(const lz4k_files_args* a, void* stream);
/* The content checksums of one group of the host-buffer file reader and writers (LZ4B200_decompress_files_host,
 * LZ4B200_compress_frames_host).  A group is a run of consecutive blocks of the call's files; a segment is the run of
 * one frame's blocks in the group, when the frame carries a content checksum.  Its blocks' bytes lie back to back:
 * block k's are base + off[k], size[k] bytes, so a segment's run from base + off[first] to base + off[end - 1] +
 * size[end - 1]. */
#define LZ4K_SEG_CONTINUES 1   /* the frame began in an earlier group: the hash starts from the carried state */
#define LZ4K_SEG_ENDS      2   /* the frame's last block is in this group: its digest is written */
typedef struct {
    int32_t first, end;        /* blocks [first, end) of the group, in file order */
    int32_t flags;             /* LZ4K_SEG_* */
    int32_t pad;
} lz4k_seg;

typedef struct {
    const uint8_t* base;
    const int64_t* off;        /* [n] block k's bytes: base + off[k], size[k] bytes */
    const int32_t* size;
    const lz4k_seg* segs;      /* [nSegs], in file order */
    int64_t nSegs;
    uint32_t* digest;          /* [nSegs] the content checksum of every frame that ends in the group */
    const void* carryIn;       /* fc_xxh32_state of the frame the first segment continues */
    void* carryOut;            /* .. of the frame the last segment leaves open */
} lz4k_seg_args;

/* the digest of every segment that begins and ends its frame in the group; carry: the first or the last segment
 * continues or leaves its frame open */
int lz4k_launch_seg_content(const lz4k_seg_args* a, int carry, void* stream);

/* The steps of one group of LZ4B200_decompress_files_host around the decode of its blocks (one lz4k_launch_decode per
 * class, by the caller).  Its table lists the blocks by class (entry e), and ord gives the entry of the k-th block in
 * file order. */
typedef struct {
    uint8_t* base;             /* the decode's slots and the staged source bytes, in one buffer */
    uint8_t* packed;           /* the group's output, block after block in file order */
    int64_t n;                 /* blocks */
    const int64_t* srcOff;     /* [n] entry e's stored bytes at base + srcOff[e] */
    const int64_t* gatherOff;  /* [n] its output: base + gatherOff[e] (its decode slot, or its stored bytes if raw) */
    const int32_t* srcSize;    /* [n] stored bytes given to the decode (0 for a stored-raw block) */
    const int32_t* rawLen;     /* [n] a stored-raw block's size, -1 for a compressed one */
    const int32_t* ord;        /* [n] the entry of block k */
    int32_t* sum;              /* [n] FC_SUM_PENDING: the block checksum to compare; the kernel writes NONE or BAD */
    const int32_t* outSize;    /* [n] the decode's results */
    int32_t* blockSize;        /* [n] output bytes of block k: its rawLen, or its decoded size (0 if it failed) */
    int64_t* blockFrom;        /* [n] block k's output before the gather: base + the gatherOff of its entry */
    int64_t* blockOff;         /* [n + 1] where block k goes in packed; blockOff[n] = the group's output bytes */
} lz4k_group_args;

/* every block checksum marked FC_SUM_PENDING, over the staged stored bytes */
int lz4k_launch_group_block_sums(const lz4k_group_args* a, void* stream);
/* after the decode: each block's output size and place in file order, their scan (the pack scan), the gather into
 * packed (the pack gather) */
int lz4k_launch_group_assemble(const lz4k_group_args* a, void* stream);
/* The copy of one group's output to its files in device memory (LZ4B200_decompress_files_to_device): run r is runs[r].len
 * bytes from packed + runs[r].src to dst + runs[r].dst, byte-aligned anywhere; nothing outside the runs is written. */
typedef struct { int64_t src, dst, len; } lz4k_run;
typedef struct {
    const uint8_t* packed;     /* the group's output (lz4k_group_args.packed); read up to 4 bytes past a run's end */
    uint8_t* dst;
    const lz4k_run* runs;      /* [nRuns] */
    int64_t nRuns;
} lz4k_scatter_args;

/* one launch, a CTA per run at a time (runs of at most LZ4K_SCATTER_RUN bytes, which the caller cuts, keep the CTAs'
 * work alike); none for nRuns == 0 */
#define LZ4K_SCATTER_RUN (256 << 10)
int lz4k_launch_group_scatter(const lz4k_scatter_args* a, void* stream);
/* The steps of one group of LZ4B200_compress_frames_host and LZ4B200_compress_legacy_host after the encode of its blocks
 * (by the caller), in file order. */
typedef struct {
    const uint8_t* src;        /* the group's staged source */
    const uint8_t* slots;      /* the encode's output */
    uint8_t* packed;           /* the group's body: [LE32 header][payload]([LE32 block checksum]) per block */
    int64_t n;                 /* blocks */
    const int64_t* srcOff;     /* [n] block k's source: src + srcOff[k], srcSize[k] bytes */
    const int32_t* srcSize;
    const int64_t* slotOff;    /* [n] its encode: slots + slotOff[k], outSize[k] bytes */
    const int32_t* outSize;
    int64_t* bodyOff;          /* [n + 1] where block k goes in packed; bodyOff[n] = the group's body bytes */
    int legacy;                /* legacy chunks: never stored raw */
    int blockSums;             /* a block checksum follows every payload */
} lz4k_wgroup_args;

/* the body: the pack scan (4-byte header, a 4-byte trailer with block checksums) and the gather, frame blocks that did
 * not gain stored raw from the staged source; then the block checksums */
int lz4k_launch_wgroup_body(const lz4k_wgroup_args* a, void* stream);
/* the batched frame and legacy encode's own steps (lz4_frame_core.h); the encode of the block table between them is the
 * caller's */
typedef struct {
    const uint8_t* src;        /* frame f's source is src + srcOff[f], srcSize[f] bytes */
    const int64_t* srcOff;
    const int64_t* srcSize;
    uint8_t* dst;              /* frame f is written at dst + dstOff[f], dstCap[f] bytes of room */
    const int64_t* dstOff;
    const int64_t* dstCap;
    int64_t* result;           /* [nFrames] */
    int64_t nFrames;
    int64_t maxBlocks[5];      /* the budget of every class (FC_CLASSES; the frames calls give class 4 none, the legacy
                                  call classes 0 .. 3 none) */
    int64_t tabBase[5];        /* class c's entries of the block table start at tabBase[c] */
    int64_t nEntries;          /* entries of the block table (sum of maxBlocks) */
    int legacy;                /* `lz4 -l` legacy streams (LZ4B200_compress_legacy) instead of frames */
    int bsid;                  /* the requested block size ID, 4 .. 7 (frames) */
    int contentSizeFlag;
    int sums;                  /* the checksums every frame is written with: FC_BLOCK_SUM | FC_CONTENT_SUM */
    void* frames;              /* fc_frame_rec[nFrames] */
    uint8_t* slots;            /* block b is compressed to slots + tabSlotOff[b] */
    int64_t slotBase[5];       /* class c's slots: slotBase[c] + k * slotStride[c] from `slots` */
    int64_t slotStride[5];
    int64_t* tabSrcOff; int32_t* tabSrcSize; int64_t* tabSlotOff; int32_t* tabCap; int32_t* tabOutSize;
    int64_t* tabBodyOff;       /* [nEntries + 1]: the pack scan of 4 + payload (+ 4 with block checksums) over the table */
    int64_t* tabPackOff;       /* where block b's header goes in dst, -1 for an unused entry */
} lz4k_cframes_args;

/* pass 1 (index), the budget scan of the frame decode, then the table cleared and filled (pass 2) */
int lz4k_launch_cframes_index(const lz4k_cframes_args* a, void* stream);
/* after the encode (tabOutSize): the pack scan, the frame headers, places, EndMarks and results (legacy: the magic, the
 * places and the results), then the gather */
int lz4k_launch_cframes_assemble(const lz4k_cframes_args* a, void* stream);
/* FC_BLOCK_SUM, after the assembly: the block checksums, one thread per placed table entry */
int lz4k_launch_cframes_block_sums(const lz4k_cframes_args* a, void* stream);
/* FC_CONTENT_SUM, after the assembly: the content checksum of every frame that passed, in one launch */
int lz4k_launch_cframes_content_sums(const lz4k_cframes_args* a, void* stream);
uint64_t lz4k_launch_count(void);
int lz4k_debug_poison_smem(uint32_t pattern, int lo, int hi, void* stream);   /* developer tool */
int lz4k_launch_ceiling(const lz4k_decode_args* a, int mode, void* stream);   /* developer tool: skeleton of the rows kernel without the decode */
int lz4k_debug_phase_cycles(unsigned long long* out8);

#ifdef __cplusplus
}
#endif
#endif
