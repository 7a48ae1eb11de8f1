/*
 * lz4_api.c -- host side of liblz4_b200.so, in C (as the reference's lib/lz4.c is).
 *
 * Implements include/lz4_b200.h: the drop-in one-shot block API of lib/lz4.h over host pointers,
 * the batched device-pointer API, and the host-buffer batch calls.  Every codec call runs the
 * CUDA kernels of lz4_kernels.cu through the extern "C" launchers of lz4_kernels.h; there is no
 * CPU implementation of the codec in this library.
 */
#include "../../include/lz4_b200.h"
#include "lz4_kernels.h"
#include "lz4_frame_core.h"
#include "lz4_files_plan.h"
#include "lz4_cfiles_plan.h"

#include <cuda_runtime_api.h>
#include <pthread.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------------------------ */
/* trivial host-only entry points (lz4.c:749-752)                                              */
/* ------------------------------------------------------------------------------------------ */
int LZ4_versionNumber(void) { return LZ4B200_VERSION_NUMBER; }
const char* LZ4_versionString(void) { return "1.10.0"; }
int LZ4_sizeofState(void) { return LZ4B200_STATE_BYTES; }
int LZ4_compressBound(int inputSize)
{
    if ((unsigned)inputSize > (unsigned)LZ4B200_MAX_INPUT_SIZE) return 0;
    return inputSize + inputSize / 255 + 16;
}

/* ------------------------------------------------------------------------------------------ */
/* CUDA context shared by the host-pointer calls                                               */
/* ------------------------------------------------------------------------------------------ */
static pthread_mutex_t g_lock = PTHREAD_MUTEX_INITIALIZER;
static char g_cuda_error[256] = "";

static int cuda_fail(cudaError_t e, const char* where)
{
    snprintf(g_cuda_error, sizeof(g_cuda_error), "%s: %s", where, cudaGetErrorString(e));
    return LZ4B200_ERR_CUDA;
}
#define CU(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { rc = cuda_fail(e_, #call); goto done; } } while (0)

const char* LZ4B200_last_cuda_error(void) { return g_cuda_error; }
uint64_t LZ4B200_launch_count(void) { return lz4k_launch_count(); }
/* not part of the public header: developer hook used by tests/perf/phase_timing.py */
__attribute__((visibility("default"))) int LZ4B200_debug_phase_cycles(unsigned long long* out8) { return lz4k_debug_phase_cycles(out8); }
int LZ4B200_peer_copy_async(void* d_dstPeer, int peerDevice, const void* d_src, size_t bytes, void* stream)
{
    static unsigned char enabled[64][64];
    int cur = 0;
    cudaError_t e;
    if (peerDevice < 0 || peerDevice >= 64 || (bytes && (!d_dstPeer || !d_src))) return LZ4B200_ERR_ARG;
    e = cudaGetDevice(&cur);
    if (e != cudaSuccess) return cuda_fail(e, "cudaGetDevice");
    if (cur >= 64) return LZ4B200_ERR_ARG;
    if (cur != peerDevice && !enabled[cur][peerDevice]) {
        int can = 0;
        e = cudaDeviceCanAccessPeer(&can, cur, peerDevice);
        if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceCanAccessPeer");
        if (!can) return LZ4B200_ERR_ARG;
        e = cudaDeviceEnablePeerAccess(peerDevice, 0);
        if (e == cudaErrorPeerAccessAlreadyEnabled) cudaGetLastError();
        else if (e != cudaSuccess) return cuda_fail(e, "cudaDeviceEnablePeerAccess");
        enabled[cur][peerDevice] = 1;
    }
    if (bytes == 0) return LZ4B200_OK;                   /* (a zero-byte call is the probe: peer access is enabled or refused) */
    e = cudaMemcpyAsync(d_dstPeer, d_src, bytes, cudaMemcpyDefault, (cudaStream_t)stream);
    return e == cudaSuccess ? LZ4B200_OK : cuda_fail(e, "cudaMemcpyAsync (peer)");
}

/* not part of the public header: developer hook used by tests/perf/enc_determinism.py */
__attribute__((visibility("default"))) int LZ4B200_debug_poison_smem(uint32_t pattern, int lo, int hi, void* stream)
{
    return lz4k_debug_poison_smem(pattern, lo, hi, stream);
}
/* not part of the public header: developer hook used by bench.py --ceiling (the rows kernel's skeleton without the decode) */
__attribute__((visibility("default"))) int LZ4B200_debug_ceiling(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                                                                  void* d_dst, int64_t dstStride, int64_t nBlocks, int mode, void* stream)
{
    lz4k_decode_args a;
    memset(&a, 0, sizeof a);
    a.src = (const uint8_t*)d_src; a.srcOff = d_srcOff; a.srcSize = d_srcSize;
    a.dst = (uint8_t*)d_dst; a.dstStride = dstStride; a.nBlocks = nBlocks;
    return lz4k_launch_ceiling(&a, mode, stream);
}
int LZ4B200_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

#define N_PIPE 4   /* chunks in flight for the host-buffer batch calls */

typedef struct { void* p; size_t cap; } buf_t;   /* a growable buffer */

/* One pipeline slot: the stream a chunk runs on, the chunk's buffers, and the return values it still owes the caller. */
typedef struct {
    cudaStream_t stream;
    buf_t in, out, ws, pack;   /* device: input, output, decode workspace, frame bodies assembled on the device */
    /* the chunk's per-block tables on the device and their pinned host staging, so that every copy of a chunk is truly
     * asynchronous (a pageable cudaMemcpyAsync blocks the host and serialises the pipeline) */
    buf_t d_tab, h_tab;
    const int32_t* pend_ret;   /* pinned return values still to be handed over: pend_cnt of them to pend_dst */
    int32_t* pend_dst;
    int64_t pend_cnt;
} slot_t;

static struct { int ready, device; slot_t slot[N_PIPE]; } g_ctx;   /* device: the one the slots' streams belong to */

static int ctx_init(void)
{
    int rc = LZ4B200_OK, i;
    if (g_ctx.ready) return LZ4B200_OK;
    if (LZ4B200_device_count() <= 0) {
        snprintf(g_cuda_error, sizeof(g_cuda_error), "no CUDA device: liblz4_b200 has no CPU fallback");
        return LZ4B200_ERR_CUDA;
    }
    CU(cudaGetDevice(&g_ctx.device));
    for (i = 0; i < N_PIPE; i++) CU(cudaStreamCreateWithFlags(&g_ctx.slot[i].stream, cudaStreamNonBlocking));
    g_ctx.ready = 1;
done:
    return rc;
}

/* grow b to at least need bytes: device memory to the next 1 MiB above need, pinned host memory to a multiple of 64 KiB */
static int reserve(buf_t* b, size_t need, int pinned)
{
    int rc = LZ4B200_OK;
    if (need <= b->cap) return rc;
    if (b->p && pinned) CU(cudaFreeHost(b->p));
    if (b->p && !pinned) CU(cudaFree(b->p));
    b->p = NULL; b->cap = 0;
    if (pinned) {
        need = (need + 65535) & ~(size_t)65535;
        CU(cudaHostAlloc(&b->p, need, cudaHostAllocDefault));
    } else {
        need = (need + (size_t)(1 << 20)) & ~(size_t)((1 << 20) - 1);
        CU(cudaMalloc(&b->p, need));
    }
    b->cap = need;
done:
    return rc;
}

/* Wait for the chunk that last used slot s, then hand its return values to the caller. */
static int slot_wait(slot_t* s)
{
    cudaError_t e = cudaStreamSynchronize(s->stream);
    if (e == cudaSuccess && s->pend_dst) memcpy(s->pend_dst, s->pend_ret, (size_t)s->pend_cnt * sizeof(int32_t));
    s->pend_dst = NULL;
    return e == cudaSuccess ? LZ4B200_OK : cuda_fail(e, "cudaStreamSynchronize");
}

/* Make slot s ready for the next chunk: wait for the last one, then grow the buffers to the chunk's sizes (0: a buffer the
 * chunk does not use).  The input, output and body buffers keep 16 bytes of slack, as the kernels read and write whole
 * 16-byte granules at the ends of a block; the host table has the device table's size. */
static int slot_take(slot_t* s, size_t inBytes, size_t outBytes, size_t wsBytes, size_t packBytes, size_t tabBytes)
{
    int rc = slot_wait(s);
    if (rc == LZ4B200_OK) rc = reserve(&s->in, inBytes + 16, 0);
    if (rc == LZ4B200_OK) rc = reserve(&s->out, outBytes + 16, 0);
    if (rc == LZ4B200_OK && wsBytes) rc = reserve(&s->ws, wsBytes, 0);
    if (rc == LZ4B200_OK && packBytes) rc = reserve(&s->pack, packBytes + 16, 0);
    if (rc == LZ4B200_OK) rc = reserve(&s->d_tab, tabBytes, 0);
    if (rc == LZ4B200_OK) rc = reserve(&s->h_tab, tabBytes, 1);
    return rc;
}

/* Queue the copy of a chunk's cnt return values from d_ret to h_ret (both in the slot's tables); the next slot_wait of s
 * hands them to dst. */
static int slot_return(slot_t* s, int32_t* h_ret, const int32_t* d_ret, int32_t* dst, int64_t cnt)
{
    int rc = LZ4B200_OK;
    CU(cudaMemcpyAsync(h_ret, d_ret, (size_t)cnt * sizeof(int32_t), cudaMemcpyDeviceToHost, s->stream));
    s->pend_ret = h_ret; s->pend_dst = dst; s->pend_cnt = cnt;
done:
    return rc;
}

/* Every host-pointer call that runs on the device is bracketed by host_begin and host_end: one call at a time owns the
 * slots.  host_end(LZ4B200_OK) waits for every slot and hands over its results; host_end(error) drains every stream,
 * drops what the slots still owe and keeps that first error.  Both unlock. */
static int host_begin(void)
{
    pthread_mutex_lock(&g_lock);
    return ctx_init();
}

static int host_end(int rc)
{
    int i;
    for (i = 0; i < N_PIPE && g_ctx.ready; i++) {
        if (rc == LZ4B200_OK) rc = slot_wait(&g_ctx.slot[i]);
        else { cudaStreamSynchronize(g_ctx.slot[i].stream); g_ctx.slot[i].pend_dst = NULL; }
    }
    pthread_mutex_unlock(&g_lock);
    return rc;
}

/* ------------------------------------------------------------------------------------------ */
/* batch layer: device pointers                                                                */
/* ------------------------------------------------------------------------------------------ */
size_t LZ4B200_decompress_workspace_bytes(int64_t nBlocks) { return lz4k_decode_workspace_bytes(nBlocks, 1, 0, SIZE_MAX); }
size_t LZ4B200_decompress_workspace_bytes_for(int64_t nBlocks, int perBlockCaps, int32_t dstCap)
{
    return lz4k_decode_workspace_bytes(nBlocks, perBlockCaps, dstCap, SIZE_MAX);
}

/* a launcher's result: LZ4B200_OK, or LZ4B200_ERR_CUDA with the error recorded under `where` */
static int launched(int e, const char* where)
{
    return e == cudaSuccess ? LZ4B200_OK : cuda_fail((cudaError_t)e, where);
}

/* the device decode calls (partial: LZ4_decompress_safe_partial, d_dstCap / dstCap hold the targets) */
static int decode_call(int partial, const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize, void* d_dst,
                       const int64_t* d_dstOff, int64_t dstStride, const int32_t* d_dstCap, int32_t dstCap, int32_t* d_outSize,
                       int64_t nBlocks, void* d_workspace, size_t workspaceBytes, int phases, void* stream)
{
    lz4k_decode_args a;
    if (nBlocks < 0) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_src || !d_srcOff || !d_srcSize || !d_dst || !d_outSize || !d_workspace) return LZ4B200_ERR_ARG;
    if (workspaceBytes < lz4k_decode_workspace_bytes(nBlocks, d_dstCap != NULL, dstCap, 0)) return LZ4B200_ERR_ARG;
    if (phases < 1 || phases > 3) return LZ4B200_ERR_ARG;
    a.src = (const uint8_t*)d_src; a.srcOff = d_srcOff; a.srcSize = d_srcSize;
    a.dst = (uint8_t*)d_dst; a.dstOff = d_dstOff; a.dstStride = dstStride;
    a.dstCapArr = d_dstCap; a.dstCap = dstCap; a.outSize = d_outSize; a.nBlocks = nBlocks;
    a.workspace = d_workspace; a.workspaceBytes = workspaceBytes;
    return launched(lz4k_launch_decode(&a, phases, partial, stream), "lz4k_launch_decode");
}

int LZ4B200_decompress_blocks_phased(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                              void* d_dst, const int64_t* d_dstOff, int64_t dstStride,
                              const int32_t* d_dstCap, int32_t dstCap,
                              int32_t* d_outSize, int64_t nBlocks,
                              void* d_workspace, size_t workspaceBytes, int phases, void* stream)
{
    return decode_call(0, d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, dstStride, d_dstCap, dstCap, d_outSize, nBlocks,
                       d_workspace, workspaceBytes, phases, stream);
}

int LZ4B200_decompress_blocks(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                              void* d_dst, const int64_t* d_dstOff, int64_t dstStride,
                              const int32_t* d_dstCap, int32_t dstCap,
                              int32_t* d_outSize, int64_t nBlocks,
                              void* d_workspace, size_t workspaceBytes, void* stream)
{
    return decode_call(0, d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, dstStride, d_dstCap, dstCap, d_outSize, nBlocks,
                       d_workspace, workspaceBytes, 3, stream);
}

int LZ4B200_decompress_blocks_partial(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                                      void* d_dst, const int64_t* d_dstOff, int64_t dstStride,
                                      const int32_t* d_target, int32_t targetOutputSize,
                                      int32_t* d_outSize, int64_t nBlocks,
                                      void* d_workspace, size_t workspaceBytes, void* stream)
{
    return decode_call(1, d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, dstStride, d_target, targetOutputSize, d_outSize,
                       nBlocks, d_workspace, workspaceBytes, 3, stream);
}

/* The workspace of LZ4B200_decompress_frames, from the budget alone: the frame records, the block table of every class
 * (entries tabBase[c] .. tabBase[c] + maxBlocks[c] - 1), then one decode workspace per class with a budget, each the
 * size that gives the class's uniform capacity its own route (LZ4B200_decompress_workspace_bytes_for(maxBlocks[c], 0,
 * fc_class_bytes(c))).  Regions start on 256 bytes from a base rounded up to 256 (the 256 bytes of slack in `bytes`).
 * The frames calls plan 4 classes, LZ4B200_decompress_files all FC_CLASSES (class 4: legacy blocks); it puts its own
 * regions after these, from `end`. */
#define FRAMES_MAX_BUDGET 0x7FFFFFFF
typedef struct {
    size_t frames, srcOff, dstOff, srcSize, outSize, rawLen, decode[FC_CLASSES], decodeBytes[FC_CLASSES], end, bytes;
    int64_t maxBlocks[FC_CLASSES], tabBase[FC_CLASSES], nEntries;
} frames_plan_t;

static size_t up256(size_t x) { return (x + 255) & ~(size_t)255; }

/* 0 for arguments the call rejects (nFrames < 0, a NULL budget, an entry outside 0 .. FRAMES_MAX_BUDGET) */
static int frames_plan(int64_t nFrames, const int64_t* maxBlocks, int classes, frames_plan_t* p)
{
    size_t at = 0;
    int c;
    if (nFrames < 0 || !maxBlocks) return 0;
    p->nEntries = 0;
    for (c = 0; c < FC_CLASSES; c++) {
        p->maxBlocks[c] = c < classes ? maxBlocks[c] : 0;
        if (p->maxBlocks[c] < 0 || p->maxBlocks[c] > FRAMES_MAX_BUDGET) return 0;
        p->tabBase[c] = p->nEntries;
        p->nEntries += p->maxBlocks[c];
    }
    p->frames = at;  at = up256(at + (size_t)nFrames * sizeof(fc_frame_rec));
    p->srcOff = at;  at = up256(at + (size_t)p->nEntries * sizeof(int64_t));
    p->dstOff = at;  at = up256(at + (size_t)p->nEntries * sizeof(int64_t));
    p->srcSize = at; at = up256(at + (size_t)p->nEntries * sizeof(int32_t));
    p->outSize = at; at = up256(at + (size_t)p->nEntries * sizeof(int32_t));
    p->rawLen = at;  at = up256(at + (size_t)p->nEntries * sizeof(int32_t));
    for (c = 0; c < FC_CLASSES; c++) {
        p->decodeBytes[c] = p->maxBlocks[c] ? lz4k_decode_workspace_bytes(p->maxBlocks[c], 0, (int32_t)fc_class_bytes(c), SIZE_MAX) : 0;
        p->decode[c] = at;
        at = up256(at + p->decodeBytes[c]);
    }
    p->end = at;
    p->bytes = at + 256;
    return 1;
}

size_t LZ4B200_decompress_frames_workspace_bytes(int64_t nFrames, const int64_t maxBlocks[4])
{
    frames_plan_t p;
    return frames_plan(nFrames, maxBlocks, 4, &p) ? p.bytes : 0;
}

/* the frame decode's arguments on the planned workspace ws (aligned to 256) */
static void frames_args(lz4k_frames_args* a, const frames_plan_t* p, uint8_t* ws, int mode)
{
    int c;
    for (c = 0; c < FC_CLASSES; c++) { a->maxBlocks[c] = p->maxBlocks[c]; a->tabBase[c] = p->tabBase[c]; }
    a->nEntries = p->nEntries;
    a->mode = mode;
    a->frames = ws + p->frames;
    a->tabSrcOff = (int64_t*)(ws + p->srcOff); a->tabDstOff = (int64_t*)(ws + p->dstOff);
    a->tabSrcSize = (int32_t*)(ws + p->srcSize); a->tabOutSize = (int32_t*)(ws + p->outSize); a->tabRawLen = (int32_t*)(ws + p->rawLen);
}

/* one phase (1: scan, 2: expand) of the decode of every class's table with a budget, at the class's uniform capacity
 * on its planned workspace (the launches of LZ4B200_decompress_blocks_phased; the scans read no destination, which
 * LZ4B200_decompress_files does not have when it only sizes) */
static int frames_decode_phase(const lz4k_frames_args* a, const frames_plan_t* p, uint8_t* ws, int ph, void* stream)
{
    lz4k_decode_args d;
    int c, rc;
    for (c = 0; c < FC_CLASSES; c++) {
        const int64_t t = p->tabBase[c];
        if (!p->maxBlocks[c]) continue;
        memset(&d, 0, sizeof d);
        d.src = a->src; d.srcOff = a->tabSrcOff + t; d.srcSize = a->tabSrcSize + t;
        d.dst = a->dst; d.dstOff = a->tabDstOff + t; d.dstCap = (int32_t)fc_class_bytes(c);
        d.outSize = a->tabOutSize + t; d.nBlocks = p->maxBlocks[c];
        d.workspace = ws + p->decode[c]; d.workspaceBytes = p->decodeBytes[c];
        if ((rc = launched(lz4k_launch_decode(&d, ph, 0, stream), "lz4k_launch_decode")) != LZ4B200_OK) return rc;
    }
    return LZ4B200_OK;
}

/* index -> per class: scan (phase 1) -> [block checksums] -> verdict -> per class: expand (phase 2) -> raw blocks ->
 * [content checksums].  Every class decodes its whole table (maxBlocks[c] entries, unused ones with size 0) at the
 * uniform capacity of its block size, the capacity lz4frame.c:1901-1904 and LZ4B200_decompressFrame_host decode with.
 * mode: FC_SUMS_* (lz4_frame_core.h); the bracketed steps run under FC_SUMS_VERIFY only. */
static int decompress_frames_mode(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                  void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                  int64_t* d_result, int64_t* d_consumed,
                                  int64_t nFrames, const int64_t maxBlocks[4], int mode,
                                  void* d_workspace, size_t workspaceBytes, void* stream)
{
    frames_plan_t p;
    lz4k_frames_args a;
    uint8_t* ws;
    int ph, rc;
    if (!frames_plan(nFrames, maxBlocks, 4, &p)) return LZ4B200_ERR_ARG;
    if (nFrames == 0) return LZ4B200_OK;
    if (!d_src || !d_srcOff || !d_srcSize || !d_dst || !d_dstOff || !d_dstCap || !d_result || !d_workspace)
        return LZ4B200_ERR_ARG;
    if (workspaceBytes < p.bytes) return LZ4B200_ERR_ARG;
    ws = (uint8_t*)(((uintptr_t)d_workspace + 255) & ~(uintptr_t)255);
    memset(&a, 0, sizeof a);
    a.src = (const uint8_t*)d_src; a.srcOff = d_srcOff; a.srcSize = d_srcSize;
    a.dst = (uint8_t*)d_dst; a.dstOff = d_dstOff; a.dstCap = d_dstCap;
    a.result = d_result; a.consumed = d_consumed; a.nFrames = nFrames;
    frames_args(&a, &p, ws, mode);

    if ((rc = launched(lz4k_launch_frames_index(&a, stream), "lz4k_launch_frames_index")) != LZ4B200_OK) return rc;
    for (ph = 1; ph <= 2; ph++) {
        if (ph == 2 && mode == FC_SUMS_VERIFY &&
            (rc = launched(lz4k_launch_frames_block_sums(&a, stream), "lz4k_launch_frames_block_sums")) != LZ4B200_OK)
            return rc;
        if (ph == 2 && (rc = launched(lz4k_launch_frames_verdict(&a, stream), "lz4k_launch_frames_verdict")) != LZ4B200_OK)
            return rc;
        if ((rc = frames_decode_phase(&a, &p, ws, ph, stream)) != LZ4B200_OK) return rc;
    }
    if ((rc = launched(lz4k_launch_frames_raw(&a, stream), "lz4k_launch_frames_raw")) != LZ4B200_OK) return rc;
    if (mode == FC_SUMS_VERIFY) return launched(lz4k_launch_frames_content_sums(&a, stream), "lz4k_launch_frames_content_sums");
    return LZ4B200_OK;
}

int LZ4B200_decompress_frames(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                              void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                              int64_t* d_result, int64_t* d_consumed,
                              int64_t nFrames, const int64_t maxBlocks[4],
                              void* d_workspace, size_t workspaceBytes, void* stream)
{
    return decompress_frames_mode(d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, d_dstCap, d_result, d_consumed, nFrames,
                                  maxBlocks, FC_SUMS_REJECT, d_workspace, workspaceBytes, stream);
}

int LZ4B200_decompress_frames_checksummed(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                          void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                          int64_t* d_result, int64_t* d_consumed,
                                          int64_t nFrames, const int64_t maxBlocks[4], int skipChecksums,
                                          void* d_workspace, size_t workspaceBytes, void* stream)
{
    return decompress_frames_mode(d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, d_dstCap, d_result, d_consumed, nFrames,
                                  maxBlocks, skipChecksums ? FC_SUMS_SKIP : FC_SUMS_VERIFY, d_workspace, workspaceBytes,
                                  stream);
}

/* The workspace of LZ4B200_decompress_files: the frame decode's plan for maxUnits unit records and all FC_CLASSES
 * classes, then the file records and the units' source offsets, lengths, places, rooms and results. */
typedef struct {
    frames_plan_t f;
    size_t files, uSrcOff, uSrcSize, uDstOff, uDstCap, uResult, bytes;
} files_plan_t;

/* 0 for arguments the call rejects (nFiles < 0, maxUnits or a budget entry outside 0 .. FRAMES_MAX_BUDGET, a NULL
 * budget) */
static int files_plan(int64_t nFiles, int64_t maxUnits, const int64_t* maxBlocks, files_plan_t* p)
{
    size_t at, u;
    if (nFiles < 0 || maxUnits < 0 || maxUnits > FRAMES_MAX_BUDGET) return 0;
    if (!frames_plan(maxUnits, maxBlocks, FC_CLASSES, &p->f)) return 0;
    u = (size_t)maxUnits * sizeof(int64_t);
    at = p->f.end;
    p->files = at;    at = up256(at + (size_t)nFiles * sizeof(fc_file_rec));
    p->uSrcOff = at;  at = up256(at + u);
    p->uSrcSize = at; at = up256(at + u);
    p->uDstOff = at;  at = up256(at + u);
    p->uDstCap = at;  at = up256(at + u);
    p->uResult = at;  at = up256(at + u);
    p->bytes = at + 256;
    return 1;
}

size_t LZ4B200_decompress_files_workspace_bytes(int64_t nFiles, int64_t maxUnits, const int64_t maxBlocks[LZ4B200_FILE_CLASSES])
{
    files_plan_t p;
    return files_plan(nFiles, maxUnits, maxBlocks, &p) ? p.bytes : 0;
}

/* files index -> files scan -> files fill -> frames scan and fill on the units -> per class: scan (phase 1) -> [block
 * checksums] -> totals, then either the fold (sizeOnly) or place -> verdict -> per class: expand (phase 2) -> raw blocks
 * -> [content checksums] -> fold.  The unit steps are skipped when maxUnits is 0. */
int LZ4B200_decompress_files(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                             void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                             int64_t* d_result, int64_t* d_consumed, int64_t* d_prefix,
                             int64_t nFiles, int64_t maxUnits, const int64_t maxBlocks[LZ4B200_FILE_CLASSES],
                             int skipChecksums, int sizeOnly,
                             void* d_workspace, size_t workspaceBytes, void* stream)
{
    files_plan_t p;
    lz4k_files_args a;
    uint8_t* ws;
    int rc;
    const int mode = skipChecksums ? FC_SUMS_SKIP : FC_SUMS_VERIFY;
    if (!files_plan(nFiles, maxUnits, maxBlocks, &p)) return LZ4B200_ERR_ARG;
    if (nFiles == 0) return LZ4B200_OK;
    if (!d_src || !d_srcOff || !d_srcSize || !d_result || !d_workspace) return LZ4B200_ERR_ARG;
    if (!sizeOnly && (!d_dst || !d_dstOff || !d_dstCap)) return LZ4B200_ERR_ARG;
    if (workspaceBytes < p.bytes) return LZ4B200_ERR_ARG;
    ws = (uint8_t*)(((uintptr_t)d_workspace + 255) & ~(uintptr_t)255);
    memset(&a, 0, sizeof a);
    a.srcOff = d_srcOff; a.srcSize = d_srcSize;
    a.dstOff = sizeOnly ? NULL : d_dstOff; a.dstCap = sizeOnly ? NULL : d_dstCap;
    a.result = d_result; a.consumed = d_consumed; a.prefix = d_prefix;
    a.nFiles = nFiles; a.maxUnits = maxUnits; a.sizeOnly = sizeOnly != 0;
    a.files = ws + p.files;
    a.u.src = (const uint8_t*)d_src; a.u.dst = sizeOnly ? NULL : (uint8_t*)d_dst;
    a.u.srcOff = (const int64_t*)(ws + p.uSrcOff); a.u.srcSize = (const int64_t*)(ws + p.uSrcSize);
    a.u.dstOff = (const int64_t*)(ws + p.uDstOff); a.u.dstCap = (const int64_t*)(ws + p.uDstCap);
    a.u.result = (int64_t*)(ws + p.uResult); a.u.consumed = NULL; a.u.nFrames = maxUnits;
    frames_args(&a.u, &p.f, ws, mode);

    if ((rc = launched(lz4k_launch_files_index(&a, stream), "lz4k_launch_files_index")) != LZ4B200_OK) return rc;
    if (maxUnits) {
        if ((rc = frames_decode_phase(&a.u, &p.f, ws, 1, stream)) != LZ4B200_OK) return rc;
        if (mode == FC_SUMS_VERIFY &&
            (rc = launched(lz4k_launch_frames_block_sums(&a.u, stream), "lz4k_launch_frames_block_sums")) != LZ4B200_OK)
            return rc;
        if ((rc = launched(lz4k_launch_files_totals(&a, stream), "lz4k_launch_files_totals")) != LZ4B200_OK) return rc;
        if (!sizeOnly) {
            if ((rc = launched(lz4k_launch_files_place(&a, stream), "lz4k_launch_files_place")) != LZ4B200_OK) return rc;
            if ((rc = launched(lz4k_launch_frames_verdict(&a.u, stream), "lz4k_launch_frames_verdict")) != LZ4B200_OK)
                return rc;
            if ((rc = frames_decode_phase(&a.u, &p.f, ws, 2, stream)) != LZ4B200_OK) return rc;
            if ((rc = launched(lz4k_launch_frames_raw(&a.u, stream), "lz4k_launch_frames_raw")) != LZ4B200_OK) return rc;
            if (mode == FC_SUMS_VERIFY &&
                (rc = launched(lz4k_launch_frames_content_sums(&a.u, stream), "lz4k_launch_frames_content_sums")) != LZ4B200_OK)
                return rc;
        }
    }
    return launched(lz4k_launch_files_fold(&a, stream), "lz4k_launch_files_fold");
}

/* the encode launch arguments, every block size included (a split launch narrows minSize .. maxSize) */
static lz4k_encode_args encode_args(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                    void* d_dst, int64_t dstStride, int32_t dstCap, int acceleration,
                                    int32_t* d_outSize, int64_t nBlocks)
{
    lz4k_encode_args a;
    a.src = (const uint8_t*)d_src; a.srcOff = NULL; a.srcStride = srcStride; a.srcSizeArr = d_srcSize; a.srcSize = srcSize;
    a.dst = (uint8_t*)d_dst; a.dstOff = NULL; a.dstStride = dstStride; a.dstCapArr = NULL; a.dstCap = dstCap;
    a.acceleration = acceleration; a.outSize = d_outSize; a.nBlocks = nBlocks; a.minSize = INT32_MIN; a.maxSize = INT32_MAX;
    return a;
}

int LZ4B200_compress_blocks(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                            void* d_dst, int64_t dstStride, int32_t dstCap, int acceleration,
                            int32_t* d_outSize, int64_t nBlocks, void* stream)
{
    lz4k_encode_args a;
    if (nBlocks < 0) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_dst || !d_outSize) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, srcStride, d_srcSize, srcSize, d_dst, dstStride, dstCap, acceleration, d_outSize, nBlocks);
    return launched(lz4k_launch_encode(&a, stream), "lz4k_launch_encode");
}

size_t LZ4B200_compress_blocks_hc_workspace_bytes(int64_t nBlocks)
{
    return lz4k_encode_hc_workspace_bytes(nBlocks);
}

int LZ4B200_compress_blocks_hc(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                               void* d_dst, int64_t dstStride, int32_t dstCap, int compressionLevel,
                               int32_t* d_outSize, int64_t nBlocks,
                               void* d_workspace, size_t workspaceBytes, void* stream)
{
    lz4k_encode_args a;
    if (compressionLevel >= 10) return LZ4B200_ERR_ARG;     /* the optimal parser (lz4hc.c:1823-) is not built */
    if (nBlocks < 0 || !d_dst || !d_outSize || !d_workspace) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_src || workspaceBytes < lz4k_encode_hc_workspace_bytes(nBlocks)) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, srcStride, d_srcSize, srcSize, d_dst, dstStride, dstCap, 0, d_outSize, nBlocks);
    return launched(lz4k_launch_encode_hc(&a, compressionLevel, d_workspace, workspaceBytes, stream), "lz4k_launch_encode_hc");
}

int LZ4B200_compress_blocks_hc_destSize(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                        void* d_dst, int64_t dstStride, int32_t targetDstSize, int compressionLevel,
                                        int32_t* d_outSize, int32_t* d_srcConsumed, int64_t nBlocks,
                                        void* d_workspace, size_t workspaceBytes, void* stream)
{
    lz4k_encode_args a;
    if (compressionLevel >= 10) return LZ4B200_ERR_ARG;     /* the optimal parser (lz4hc.c:1823-) is not built */
    if (nBlocks < 0 || !d_dst || !d_outSize || !d_srcConsumed || !d_workspace) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_src || workspaceBytes < lz4k_encode_hc_workspace_bytes(nBlocks)) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, srcStride, d_srcSize, srcSize, d_dst, dstStride, targetDstSize, 0, d_outSize, nBlocks);
    return launched(lz4k_launch_encode_hc_dest(&a, d_srcConsumed, compressionLevel, d_workspace, workspaceBytes, stream),
                    "lz4k_launch_encode_hc_dest");
}

size_t LZ4B200_compress_blocks_hc_opt_workspace_bytes(int64_t nBlocks)
{
    return lz4k_encode_hc_opt_workspace_bytes(nBlocks);
}

int LZ4B200_compress_blocks_hc_opt(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                   void* d_dst, int64_t dstStride, int32_t dstCap, int compressionLevel,
                                   int32_t* d_outSize, int64_t nBlocks,
                                   void* d_workspace, size_t workspaceBytes, void* stream)
{
    lz4k_encode_args a;
    if (compressionLevel < 10) return LZ4B200_ERR_ARG;      /* levels 1 .. 9 (and <= 0, read as 9): the hash-chain calls */
    if (nBlocks < 0 || !d_dst || !d_outSize || !d_workspace) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_src || workspaceBytes < lz4k_encode_hc_opt_workspace_bytes(nBlocks)) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, srcStride, d_srcSize, srcSize, d_dst, dstStride, dstCap, 0, d_outSize, nBlocks);
    return launched(lz4k_launch_encode_hc_opt(&a, compressionLevel, d_workspace, workspaceBytes, stream),
                    "lz4k_launch_encode_hc_opt");
}

int LZ4B200_compress_blocks_hc_opt_destSize(const void* d_src, int64_t srcStride, const int32_t* d_srcSize,
                                            int32_t srcSize, void* d_dst, int64_t dstStride, int32_t targetDstSize,
                                            int compressionLevel, int32_t* d_outSize, int32_t* d_srcConsumed,
                                            int64_t nBlocks, void* d_workspace, size_t workspaceBytes, void* stream)
{
    lz4k_encode_args a;
    if (compressionLevel < 10) return LZ4B200_ERR_ARG;      /* levels 1 .. 9 (and <= 0, read as 9): the hash-chain calls */
    if (nBlocks < 0 || !d_dst || !d_outSize || !d_srcConsumed || !d_workspace) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_src || workspaceBytes < lz4k_encode_hc_opt_workspace_bytes(nBlocks)) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, srcStride, d_srcSize, srcSize, d_dst, dstStride, targetDstSize, 0, d_outSize, nBlocks);
    return launched(lz4k_launch_encode_hc_opt_dest(&a, d_srcConsumed, compressionLevel, d_workspace, workspaceBytes,
                                                   stream), "lz4k_launch_encode_hc_opt_dest");
}

int LZ4B200_compress_blocks_destSize(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                     void* d_dst, int64_t dstStride, int32_t targetDstSize, int acceleration,
                                     int32_t* d_outSize, int32_t* d_srcConsumed, int64_t nBlocks, void* stream)
{
    lz4k_encode_args a;
    if (nBlocks < 0 || !d_dst || !d_outSize || !d_srcConsumed) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_src) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, srcStride, d_srcSize, srcSize, d_dst, dstStride, targetDstSize, acceleration, d_outSize, nBlocks);
    return launched(lz4k_launch_encode_dest(&a, d_srcConsumed, stream), "lz4k_launch_encode_dest");
}

/* the parallel parse stages a whole block in shared memory: blocks above 64 KB take the byte-identical encoder.  With
 * per-block sizes each block goes by its own size (srcSize is not used): both kernels run, each on its blocks. */
static int encode_parallel(lz4k_encode_args* a, void* stream)
{
    int rc;
    if (!a->srcSizeArr && a->srcSize <= 65536) return launched(lz4k_launch_encode_par(a, stream), "lz4k_launch_encode_par");
    if (!a->srcSizeArr) return launched(lz4k_launch_encode(a, stream), "lz4k_launch_encode");
    a->maxSize = 65536;
    if ((rc = launched(lz4k_launch_encode_par(a, stream), "lz4k_launch_encode_par")) != LZ4B200_OK) return rc;
    a->minSize = 65537; a->maxSize = INT32_MAX;
    return launched(lz4k_launch_encode(a, stream), "lz4k_launch_encode");
}

int LZ4B200_compress_blocks_parallel(const void* d_src, int64_t srcStride, const int32_t* d_srcSize, int32_t srcSize,
                                     void* d_dst, int64_t dstStride, int32_t dstCap, int acceleration,
                                     int32_t* d_outSize, int64_t nBlocks, void* stream)
{
    lz4k_encode_args a;
    if (nBlocks < 0) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_dst || !d_outSize) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, srcStride, d_srcSize, srcSize, d_dst, dstStride, dstCap, acceleration, d_outSize, nBlocks);
    return encode_parallel(&a, stream);
}

/* LZ4B200_compress_blocks_indexed's workspace: the HC or optimal-parser slots of its level, none for the other parses */
size_t LZ4B200_compress_blocks_indexed_workspace_bytes(int64_t nBlocks, int parse, int param)
{
    if (parse != LZ4B200_PARSE_HC) return 0;
    return param >= 10 ? lz4k_encode_hc_opt_workspace_bytes(nBlocks) : lz4k_encode_hc_workspace_bytes(nBlocks);
}

int LZ4B200_compress_blocks_indexed(const void* d_src, const int64_t* d_srcOff, const int32_t* d_srcSize,
                                    void* d_dst, const int64_t* d_dstOff, const int32_t* d_dstCap,
                                    int32_t* d_outSize, int64_t nBlocks, int parse, int param,
                                    void* d_workspace, size_t workspaceBytes, void* stream)
{
    lz4k_encode_args a;
    if (nBlocks < 0 || parse < LZ4B200_PARSE_FAST || parse > LZ4B200_PARSE_HC) return LZ4B200_ERR_ARG;
    if (!d_srcOff || !d_srcSize || !d_dstOff || !d_dstCap || !d_outSize) return LZ4B200_ERR_ARG;
    if (parse == LZ4B200_PARSE_HC && !d_workspace) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!d_src || !d_dst) return LZ4B200_ERR_ARG;
    if (workspaceBytes < LZ4B200_compress_blocks_indexed_workspace_bytes(nBlocks, parse, param)) return LZ4B200_ERR_ARG;
    a = encode_args(d_src, 0, d_srcSize, 0, d_dst, 0, 0, parse == LZ4B200_PARSE_HC ? 0 : param, d_outSize, nBlocks);
    a.srcOff = d_srcOff; a.dstOff = d_dstOff; a.dstCapArr = d_dstCap;
    if (parse == LZ4B200_PARSE_FAST) return launched(lz4k_launch_encode(&a, stream), "lz4k_launch_encode");
    if (parse == LZ4B200_PARSE_PARALLEL) return encode_parallel(&a, stream);
    if (param >= 10)
        return launched(lz4k_launch_encode_hc_opt(&a, param, d_workspace, workspaceBytes, stream), "lz4k_launch_encode_hc_opt");
    return launched(lz4k_launch_encode_hc(&a, param, d_workspace, workspaceBytes, stream), "lz4k_launch_encode_hc");
}

int LZ4B200_pack_blocks(const void* d_slots, int64_t slotStride, const int32_t* d_sizes, int64_t nBlocks,
                        void* d_packed, int64_t* d_outOff, int headerBytes, void* stream)
{
    if (nBlocks < 0 || !d_outOff || (headerBytes != 0 && headerBytes != 4)) return LZ4B200_ERR_ARG;
    if (nBlocks > 0 && (!d_slots || !d_sizes || !d_packed)) return LZ4B200_ERR_ARG;
    return launched(lz4k_launch_pack((const uint8_t*)d_slots, NULL, slotStride, d_sizes, nBlocks, (uint8_t*)d_packed,
                                     d_outOff, headerBytes, stream), "lz4k_launch_pack");
}

int LZ4B200_pack_blocks_indexed(const void* d_slots, const int64_t* d_slotOff, const int32_t* d_sizes, int64_t nBlocks,
                                void* d_packed, int64_t* d_outOff, int headerBytes, void* stream)
{
    if (nBlocks < 0 || !d_outOff || (headerBytes != 0 && headerBytes != 4)) return LZ4B200_ERR_ARG;
    if (nBlocks > 0 && (!d_slots || !d_slotOff || !d_sizes || !d_packed)) return LZ4B200_ERR_ARG;
    return launched(lz4k_launch_pack((const uint8_t*)d_slots, d_slotOff, 0, d_sizes, nBlocks, (uint8_t*)d_packed,
                                     d_outOff, headerBytes, stream), "lz4k_launch_pack");
}

int LZ4B200_pack_frame_blocks(const void* d_slots, int64_t slotStride, const int32_t* d_sizes, const void* d_src, int64_t srcStride,
                              int32_t blockSize, int32_t lastSize, int64_t nBlocks, void* d_body, int64_t* d_outOff, void* stream)
{
    if (nBlocks < 0 || !d_outOff || blockSize <= 0 || lastSize < 0 || lastSize > blockSize) return LZ4B200_ERR_ARG;
    if (nBlocks > 0 && (!d_slots || !d_sizes || !d_src || !d_body)) return LZ4B200_ERR_ARG;
    return launched(lz4k_launch_pack_frame((const uint8_t*)d_slots, slotStride, d_sizes, (const uint8_t*)d_src, srcStride,
                                           blockSize, lastSize, nBlocks, (uint8_t*)d_body, d_outOff, stream),
                    "lz4k_launch_pack_frame");
}

/* The workspace of the frame-encode calls (LZ4B200_compress_frames, LZ4B200_compress_frames_checksummed,
 * LZ4B200_compress_legacy), from the budget of every class and the encode alone: the frame records, the block table of
 * every class (entries tabBase[c] .. tabBase[c] + maxBlocks[c] - 1: source offset, size, slot offset, capacity, result,
 * the pack scan, the place), one slot per budgeted block -- blockSize - 1 bytes for a frame block, LZ4_compressBound(8 MiB)
 * for a legacy block, rounded up to 16 -- and, when the encode is an HC one (hcLevel > 0), the HC encoder's workspace for
 * the whole table.  Regions start on 256 bytes, as in frames_plan. */
typedef struct {
    size_t frames, srcOff, srcSize, slotOff, cap, outSize, bodyOff, packOff, slots, hc, hcBytes, bytes;
    int64_t tabBase[FC_CLASSES], slotBase[FC_CLASSES], slotStride[FC_CLASSES], nEntries;
} cframes_plan_t;

/* 0 for arguments the call rejects (nFrames < 0, a NULL budget, an entry outside 0 .. FRAMES_MAX_BUDGET).  maxBlocks:
 * FC_CLASSES entries. */
static int cframes_plan(int64_t nFrames, const int64_t* maxBlocks, int hcLevel, cframes_plan_t* p)
{
    size_t at = 0;
    int64_t slotBytes = 0;
    int c;
    if (nFrames < 0 || !maxBlocks) return 0;
    p->nEntries = 0;
    for (c = 0; c < FC_CLASSES; c++) {
        if (maxBlocks[c] < 0 || maxBlocks[c] > FRAMES_MAX_BUDGET) return 0;
        p->tabBase[c] = p->nEntries;
        p->nEntries += maxBlocks[c];
        p->slotStride[c] = ((c == FC_LEGACY_CLASS ? FC_LEGACY_BOUND : fc_block_bytes(4 + c) - 1) + 15) & ~(int64_t)15;
        p->slotBase[c] = slotBytes;
        slotBytes += maxBlocks[c] * p->slotStride[c];
    }
    p->frames = at;  at = up256(at + (size_t)nFrames * sizeof(fc_frame_rec));
    p->srcOff = at;  at = up256(at + (size_t)p->nEntries * sizeof(int64_t));
    p->srcSize = at; at = up256(at + (size_t)p->nEntries * sizeof(int32_t));
    p->slotOff = at; at = up256(at + (size_t)p->nEntries * sizeof(int64_t));
    p->cap = at;     at = up256(at + (size_t)p->nEntries * sizeof(int32_t));
    p->outSize = at; at = up256(at + (size_t)p->nEntries * sizeof(int32_t));
    p->bodyOff = at; at = up256(at + (size_t)(p->nEntries + 1) * sizeof(int64_t));
    p->packOff = at; at = up256(at + (size_t)p->nEntries * sizeof(int64_t));
    p->slots = at;   at = up256(at + (size_t)slotBytes);
    p->hcBytes = hcLevel <= 0 ? 0 : hcLevel >= 10 ? lz4k_encode_hc_opt_workspace_bytes(p->nEntries)
                                                  : lz4k_encode_hc_workspace_bytes(p->nEntries);
    p->hc = at;      at = up256(at + p->hcBytes);
    p->bytes = at + 256;
    return 1;
}

/* The frames calls' budget over FC_CLASSES in mb: theirs for block size IDs 4 .. 7, none for legacy blocks (NULL stays
 * NULL, for cframes_plan to reject) */
static const int64_t* cframes_budget(const int64_t* maxBlocks, int64_t mb[FC_CLASSES])
{
    int c;
    if (!maxBlocks) return NULL;
    for (c = 0; c < 4; c++) mb[c] = maxBlocks[c];
    mb[FC_LEGACY_CLASS] = 0;
    return mb;
}

/* The encode of a frame-writing call at `level` (lz4frame.c:911-937): *hcLevel 0 and LZ4_compress_fast with acceleration
 * -level + 1 below level 1 (LZ4_compress_fast clamps it to 65537; this also keeps -INT_MIN out) below level 2, else
 * LZ4_compress_HC_extStateHC_fastReset at *hcLevel = level */
static void frames_levels(int level, int* hcLevel, int* accel)
{
    *hcLevel = level >= 2 ? level : 0;
    *accel = level >= 0 ? 1 : level < -65536 ? 65537 : -level + 1;
}

/* The encode of `lz4 -l` at `level` (lz4io.c:788-837): below 3, LZ4_compress_fast with acceleration -level for negative
 * levels and 0, read as 1, otherwise (above 65537 as 65537); from 3 on, LZ4_compress_HC at *hcLevel = level (above 12
 * read as 12) */
static void legacy_levels(int level, int* hcLevel, int* accel)
{
    *hcLevel = level >= 3 ? level : 0;
    *accel = level >= 0 ? 1 : level < -65537 ? 65537 : -level;
}

size_t LZ4B200_compress_frames_workspace_bytes(int64_t nFrames, const int64_t maxBlocks[4], int compressionLevel)
{
    cframes_plan_t p;
    int64_t mb[FC_CLASSES];
    int hcLevel, accel;
    frames_levels(compressionLevel, &hcLevel, &accel);
    return cframes_plan(nFrames, cframes_budget(maxBlocks, mb), hcLevel, &p) ? p.bytes : 0;
}

/* The encode of a frame-writing call's block table e at hcLevel / e->acceleration (frames_levels, legacy_levels): the
 * optimal parser, the HC parse, the parallel parse routed by block size, or the fast parse.  hc: hcBytes of workspace. */
static int encode_table(lz4k_encode_args* e, int hcLevel, int parallel, void* hc, size_t hcBytes, void* stream)
{
    if (hcLevel >= 10)
        return launched(lz4k_launch_encode_hc_opt(e, hcLevel, hc, hcBytes, stream), "lz4k_launch_encode_hc_opt");
    if (hcLevel > 0) return launched(lz4k_launch_encode_hc(e, hcLevel, hc, hcBytes, stream), "lz4k_launch_encode_hc");
    if (parallel) return encode_parallel(e, stream);
    return launched(lz4k_launch_encode(e, stream), "lz4k_launch_encode");
}

/* The body of the frame-writing calls: index (+ budget scan, fill) -> one encode of the whole table -> pack scan ->
 * headers, places, EndMarks, results -> gather -> [block checksums] -> [content checksums].  A frame block is compressed
 * into its slot with capacity size - 1, as LZ4F_makeBlock does (lz4frame.c:883-908); a legacy block with capacity
 * LZ4_compressBound(size).  legacy: `lz4 -l` streams (blockSizeID, contentSizeFlag, parallel and sums unused).  sums:
 * FC_BLOCK_SUM | FC_CONTENT_SUM; the bracketed steps run for the checksums the frames carry.  maxBlocks: FC_CLASSES
 * entries; hcLevel, accel: the encode (frames_levels, legacy_levels). */
static int cframes_run(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                       void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                       int64_t* d_result, int64_t nFrames, const int64_t* maxBlocks, int legacy,
                       int blockSizeID, int contentSizeFlag, int parallel, int sums, int hcLevel, int accel,
                       void* d_workspace, size_t workspaceBytes, void* stream)
{
    cframes_plan_t p;
    lz4k_cframes_args a;
    lz4k_encode_args e;
    uint8_t* ws;
    int c, rc;
    if (!cframes_plan(nFrames, maxBlocks, hcLevel, &p)) return LZ4B200_ERR_ARG;
    if (nFrames == 0) return LZ4B200_OK;
    if (!d_src || !d_srcOff || !d_srcSize || !d_dst || !d_dstOff || !d_dstCap || !d_result || !d_workspace)
        return LZ4B200_ERR_ARG;
    if (workspaceBytes < p.bytes) return LZ4B200_ERR_ARG;
    ws = (uint8_t*)(((uintptr_t)d_workspace + 255) & ~(uintptr_t)255);
    memset(&a, 0, sizeof a);
    a.src = (const uint8_t*)d_src; a.srcOff = d_srcOff; a.srcSize = d_srcSize;
    a.dst = (uint8_t*)d_dst; a.dstOff = d_dstOff; a.dstCap = d_dstCap;
    a.result = d_result; a.nFrames = nFrames;
    for (c = 0; c < FC_CLASSES; c++) {
        a.maxBlocks[c] = maxBlocks[c]; a.tabBase[c] = p.tabBase[c];
        a.slotBase[c] = p.slotBase[c]; a.slotStride[c] = p.slotStride[c];
    }
    a.nEntries = p.nEntries;
    a.legacy = legacy;
    a.bsid = blockSizeID;
    a.contentSizeFlag = contentSizeFlag != 0;
    a.sums = sums;
    a.frames = ws + p.frames;
    a.slots = ws + p.slots;
    a.tabSrcOff = (int64_t*)(ws + p.srcOff); a.tabSrcSize = (int32_t*)(ws + p.srcSize);
    a.tabSlotOff = (int64_t*)(ws + p.slotOff); a.tabCap = (int32_t*)(ws + p.cap); a.tabOutSize = (int32_t*)(ws + p.outSize);
    a.tabBodyOff = (int64_t*)(ws + p.bodyOff); a.tabPackOff = (int64_t*)(ws + p.packOff);

    if ((rc = launched(lz4k_launch_cframes_index(&a, stream), "lz4k_launch_cframes_index")) != LZ4B200_OK) return rc;
    e = encode_args(d_src, 0, a.tabSrcSize, 0, a.slots, 0, 0, accel, a.tabOutSize, p.nEntries);
    e.srcOff = a.tabSrcOff; e.dstOff = a.tabSlotOff; e.dstCapArr = a.tabCap;
    if ((rc = encode_table(&e, hcLevel, parallel, ws + p.hc, p.hcBytes, stream)) != LZ4B200_OK) return rc;
    if ((rc = launched(lz4k_launch_cframes_assemble(&a, stream), "lz4k_launch_cframes_assemble")) != LZ4B200_OK) return rc;
    if ((sums & FC_BLOCK_SUM) &&
        (rc = launched(lz4k_launch_cframes_block_sums(&a, stream), "lz4k_launch_cframes_block_sums")) != LZ4B200_OK)
        return rc;
    if (sums & FC_CONTENT_SUM) return launched(lz4k_launch_cframes_content_sums(&a, stream), "lz4k_launch_cframes_content_sums");
    return LZ4B200_OK;
}

/* the two frames calls: their own argument rules, then the body with their budget and levels */
static int compress_frames_sums(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                int64_t* d_result, int64_t nFrames,
                                int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel, int sums,
                                const int64_t maxBlocks[4],
                                void* d_workspace, size_t workspaceBytes, void* stream)
{
    int64_t mb[FC_CLASSES];
    int hcLevel, accel;
    if (blockSizeID == 0) blockSizeID = 4;
    if (blockSizeID < 4 || blockSizeID > 7) return LZ4B200_ERR_ARG;
    if (parallel && compressionLevel >= 2) return LZ4B200_ERR_ARG;
    frames_levels(compressionLevel, &hcLevel, &accel);
    return cframes_run(d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, d_dstCap, d_result, nFrames,
                       cframes_budget(maxBlocks, mb), 0, blockSizeID, contentSizeFlag, parallel, sums, hcLevel, accel,
                       d_workspace, workspaceBytes, stream);
}

int LZ4B200_compress_frames(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                            void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                            int64_t* d_result, int64_t nFrames,
                            int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                            const int64_t maxBlocks[4],
                            void* d_workspace, size_t workspaceBytes, void* stream)
{
    return compress_frames_sums(d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, d_dstCap, d_result, nFrames, blockSizeID,
                                compressionLevel, contentSizeFlag, parallel, 0, maxBlocks, d_workspace, workspaceBytes,
                                stream);
}

int LZ4B200_compress_frames_checksummed(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                                        void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                                        int64_t* d_result, int64_t nFrames,
                                        int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                                        int blockChecksumFlag, int contentChecksumFlag,
                                        const int64_t maxBlocks[4],
                                        void* d_workspace, size_t workspaceBytes, void* stream)
{
    return compress_frames_sums(d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, d_dstCap, d_result, nFrames, blockSizeID,
                                compressionLevel, contentSizeFlag, parallel,
                                (blockChecksumFlag ? FC_BLOCK_SUM : 0) | (contentChecksumFlag ? FC_CONTENT_SUM : 0),
                                maxBlocks, d_workspace, workspaceBytes, stream);
}

int64_t LZ4B200_compressLegacyBound(int64_t srcSize)
{
    return srcSize < 0 ? LZ4B200_ERR_ARG : fc_legacy_bound(srcSize);
}

int64_t LZ4B200_compressFrameBound_checksummed(int64_t srcSize, int blockSizeID, int blockChecksumFlag,
                                               int contentChecksumFlag)
{
    if (srcSize < 0) return LZ4B200_ERR_ARG;
    if (blockSizeID == 0) blockSizeID = 4;
    if (blockSizeID < 4 || blockSizeID > 7) return LZ4B200_ERR_ARG;
    return fc_frame_bound_sums(srcSize, fc_optimal_bsid(blockSizeID, srcSize),
                               (blockChecksumFlag ? FC_BLOCK_SUM : 0) | (contentChecksumFlag ? FC_CONTENT_SUM : 0));
}

/* the legacy call's budget over FC_CLASSES in mb: maxBlocks legacy blocks, no frame blocks */
static const int64_t* legacy_budget(int64_t maxBlocks, int64_t mb[FC_CLASSES])
{
    int c;
    for (c = 0; c < 4; c++) mb[c] = 0;
    mb[FC_LEGACY_CLASS] = maxBlocks;
    return mb;
}

size_t LZ4B200_compress_legacy_workspace_bytes(int64_t nFiles, int64_t maxBlocks, int compressionLevel)
{
    cframes_plan_t p;
    int64_t mb[FC_CLASSES];
    int hcLevel, accel;
    legacy_levels(compressionLevel, &hcLevel, &accel);
    return cframes_plan(nFiles, legacy_budget(maxBlocks, mb), hcLevel, &p) ? p.bytes : 0;
}

int LZ4B200_compress_legacy(const void* d_src, const int64_t* d_srcOff, const int64_t* d_srcSize,
                            void* d_dst, const int64_t* d_dstOff, const int64_t* d_dstCap,
                            int64_t* d_result, int64_t nFiles, int compressionLevel, int64_t maxBlocks,
                            void* d_workspace, size_t workspaceBytes, void* stream)
{
    int64_t mb[FC_CLASSES];
    int hcLevel, accel;
    legacy_levels(compressionLevel, &hcLevel, &accel);
    return cframes_run(d_src, d_srcOff, d_srcSize, d_dst, d_dstOff, d_dstCap, d_result, nFiles,
                       legacy_budget(maxBlocks, mb), 1, 0, 0, 0, 0, hcLevel, accel, d_workspace, workspaceBytes, stream);
}

/* ------------------------------------------------------------------------------------------ */
/* host-buffer batch calls: H2D -> kernels -> D2H, N_PIPE chunks in flight                     */
/* ------------------------------------------------------------------------------------------ */
/* target uncompressed bytes per pipeline chunk: large enough that a chunk's kernels run at batch speed, small enough that
 * the first H2D and the last D2H (which nothing overlaps) are a small part of the call.  LZ4B200_HOST_CHUNK_MB overrides
 * it (developer knob for tests/perf). */
static int64_t chunk_out_bytes(void)
{
    static int64_t v = 0;
    if (v == 0) {
        const char* e = getenv("LZ4B200_HOST_CHUNK_MB");
        long mb = e ? atol(e) : 0;
        v = (int64_t)((mb >= 1 && mb <= 4096) ? mb : 64) << 20;
    }
    return v;
}
#define CHUNK_OUT_BYTES chunk_out_bytes()

int LZ4B200_decompress_blocks_host(const void* h_src, const int64_t* h_srcOff, const int32_t* h_srcSize,
                                   void* h_dst, int64_t dstStride, int32_t dstCap,
                                   int32_t* h_outSize, int64_t nBlocks)
{
    int rc;
    int64_t perChunk, first;
    int slot = 0;
    if (nBlocks < 0 || dstCap < 0 || dstStride < dstCap) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!h_src || !h_srcOff || !h_srcSize || !h_dst || !h_outSize) return LZ4B200_ERR_ARG;
    if ((rc = host_begin()) != LZ4B200_OK) goto done;

    perChunk = CHUNK_OUT_BYTES / (dstStride > 0 ? dstStride : 1);
    if (perChunk < 1) perChunk = 1;
    for (first = 0; first < nBlocks; first += perChunk, slot = (slot + 1) % N_PIPE) {
        const int64_t cnt = (nBlocks - first < perChunk) ? nBlocks - first : perChunk;
        slot_t* s = &g_ctx.slot[slot];
        int64_t lo = h_srcOff[first], hi = lo, k;
        int64_t *h_off, *d_off;
        int32_t *h_size, *d_size;
        /* the chunk's compressed bytes span [lo, hi) of h_src (blocks may be in any order) */
        for (k = first; k < first + cnt; k++) {
            if (h_srcSize[k] < 0) { rc = LZ4B200_ERR_ARG; goto done; }
            if (h_srcOff[k] < lo) lo = h_srcOff[k];
            if (h_srcOff[k] + h_srcSize[k] > hi) hi = h_srcOff[k] + h_srcSize[k];
        }
        rc = slot_take(s, (size_t)(hi - lo), (size_t)(cnt * dstStride), LZ4B200_decompress_workspace_bytes_for(cnt, 0, dstCap), 0,
                       (size_t)cnt * (sizeof(int64_t) + 2 * sizeof(int32_t)));
        if (rc != LZ4B200_OK) goto done;
        /* tables: [offsets i64 | sizes i32 | return values i32] */
        h_off = (int64_t*)s->h_tab.p; h_size = (int32_t*)(h_off + cnt);
        d_off = (int64_t*)s->d_tab.p; d_size = (int32_t*)(d_off + cnt);
        for (k = 0; k < cnt; k++) h_off[k] = h_srcOff[first + k] - lo;   /* relative to the chunk's first byte */
        memcpy(h_size, h_srcSize + first, (size_t)cnt * sizeof(int32_t));
        CU(cudaMemcpyAsync(d_off, h_off, (size_t)cnt * (sizeof(int64_t) + sizeof(int32_t)), cudaMemcpyHostToDevice, s->stream));
        CU(cudaMemcpyAsync(s->in.p, (const char*)h_src + lo, (size_t)(hi - lo), cudaMemcpyHostToDevice, s->stream));
        rc = LZ4B200_decompress_blocks(s->in.p, d_off, d_size, s->out.p, NULL, dstStride, NULL, dstCap, d_size + cnt, cnt,
                                       s->ws.p, s->ws.cap, s->stream);
        if (rc != LZ4B200_OK) goto done;
        CU(cudaMemcpyAsync((char*)h_dst + first * dstStride, s->out.p, (size_t)(cnt * dstStride), cudaMemcpyDeviceToHost, s->stream));
        if ((rc = slot_return(s, h_size + cnt, d_size + cnt, h_outSize + first, cnt)) != LZ4B200_OK) goto done;
    }
done:
    return host_end(rc);
}

int LZ4B200_compress_blocks_host(const void* h_src, int64_t srcStride, int32_t srcSize, int64_t lastSize,
                                 void* h_dst, int64_t dstStride, int32_t dstCap, int acceleration,
                                 int32_t* h_outSize, int64_t nBlocks)
{
    int rc;
    int64_t perChunk, first;
    int slot = 0;
    if (nBlocks < 0 || srcSize < 0 || lastSize < 0 || lastSize > srcSize || srcStride < srcSize) return LZ4B200_ERR_ARG;
    if (nBlocks == 0) return LZ4B200_OK;
    if (!h_dst || !h_outSize || (!h_src && srcSize > 0)) return LZ4B200_ERR_ARG;
    if ((rc = host_begin()) != LZ4B200_OK) goto done;

    perChunk = CHUNK_OUT_BYTES / (srcStride > 0 ? srcStride : 1);
    if (perChunk < 1) perChunk = 1;
    for (first = 0; first < nBlocks; first += perChunk, slot = (slot + 1) % N_PIPE) {
        const int64_t cnt = (nBlocks - first < perChunk) ? nBlocks - first : perChunk;
        const int isLast = (first + cnt == nBlocks);
        const int ragged = isLast && lastSize != srcSize;   /* a per-block size table only for the short final block */
        slot_t* s = &g_ctx.slot[slot];
        const size_t inBytes = (size_t)((cnt - 1) * srcStride + (isLast ? lastSize : srcSize));
        int32_t *h_size, *d_size;
        int64_t k;
        rc = slot_take(s, inBytes, (size_t)(cnt * dstStride), 0, 0, (size_t)cnt * 2 * sizeof(int32_t));
        if (rc != LZ4B200_OK) goto done;
        h_size = (int32_t*)s->h_tab.p;                       /* tables: [source sizes i32 | return values i32] */
        d_size = (int32_t*)s->d_tab.p;
        if (inBytes) CU(cudaMemcpyAsync(s->in.p, (const char*)h_src + first * srcStride, inBytes, cudaMemcpyHostToDevice, s->stream));
        if (ragged) {
            for (k = 0; k < cnt; k++) h_size[k] = srcSize;
            h_size[cnt - 1] = (int32_t)lastSize;
            CU(cudaMemcpyAsync(d_size, h_size, (size_t)cnt * sizeof(int32_t), cudaMemcpyHostToDevice, s->stream));
        }
        rc = LZ4B200_compress_blocks(s->in.p, srcStride, ragged ? d_size : NULL, srcSize, s->out.p, dstStride, dstCap,
                                     acceleration, d_size + cnt, cnt, s->stream);
        if (rc != LZ4B200_OK) goto done;
        CU(cudaMemcpyAsync((char*)h_dst + first * dstStride, s->out.p, (size_t)(cnt * dstStride), cudaMemcpyDeviceToHost, s->stream));
        if ((rc = slot_return(s, h_size + cnt, d_size + cnt, h_outSize + first, cnt)) != LZ4B200_OK) goto done;
    }
done:
    return host_end(rc);
}

/* ------------------------------------------------------------------------------------------ */
/* drop-in layer: one block, host pointers, synchronous                                        */
/* ------------------------------------------------------------------------------------------ */
/* srcSizePtr == NULL: LZ4_compress_fast_extState (lz4.c:1382).  Otherwise LZ4_compress_destSize_extState (lz4.c:1481-1503)
 * with srcSize = *srcSizePtr and targetDstSize = dstCapacity: *srcSizePtr receives the consumed input where the reference
 * writes it (the fill route, lz4.c:1332 and :1369), and is left alone on the compress_fast route (lz4.c:1486-1487). */
static int one_block_compress(const char* src, char* dst, int srcSize, int dstCapacity, int acceleration, int* srcSizePtr)
{
    int rc, bound;
    int32_t res[2] = {0, 0};                 /* return value, consumed input */
    slot_t* s = &g_ctx.slot[0];
    int32_t* d_res;
    /* argument rules of LZ4_compress_generic, lz4.c:1360-1372, decided on the host so that a bad
     * size never reaches the device */
    if ((unsigned)srcSize > (unsigned)LZ4B200_MAX_INPUT_SIZE) return 0;
    if (dstCapacity <= 0) return 0;          /* nothing can be written (lz4.c:1362, :985 and the limited checks) */
    if (dst == NULL) return 0;
    if (srcSize > 0 && src == NULL) return 0;
    bound = LZ4_compressBound(srcSize);
    if ((rc = host_begin()) != LZ4B200_OK) goto done;
    rc = slot_take(s, (size_t)srcSize, (size_t)(dstCapacity < bound ? dstCapacity : bound), 0, 0, sizeof(res));
    if (rc != LZ4B200_OK) goto done;
    d_res = (int32_t*)s->d_tab.p;
    /* copy-in completes before any output is produced: in-place calls (lz4.h:619-678) are safe */
    if (srcSize) CU(cudaMemcpyAsync(s->in.p, src, (size_t)srcSize, cudaMemcpyHostToDevice, s->stream));
    if (srcSizePtr)
        rc = LZ4B200_compress_blocks_destSize(s->in.p, 0, NULL, srcSize, s->out.p, 0, dstCapacity, acceleration,
                                              d_res, d_res + 1, 1, s->stream);
    else
        rc = LZ4B200_compress_blocks(s->in.p, 0, NULL, srcSize, s->out.p, 0, dstCapacity, acceleration, d_res, 1, s->stream);
    if (rc == LZ4B200_OK) rc = slot_return(s, (int32_t*)s->h_tab.p, d_res, res, srcSizePtr ? 2 : 1);
    if (rc == LZ4B200_OK) rc = slot_wait(s);
    if (rc == LZ4B200_OK && res[0] > 0) CU(cudaMemcpyAsync(dst, s->out.p, (size_t)res[0], cudaMemcpyDeviceToHost, s->stream));
done:
    if (host_end(rc) != LZ4B200_OK) return 0;
    if (srcSizePtr && res[0] > 0 && dstCapacity < bound) *srcSizePtr = res[1];
    return res[0];
}

int LZ4_compress_fast(const char* src, char* dst, int srcSize, int dstCapacity, int acceleration)
{
    return one_block_compress(src, dst, srcSize, dstCapacity, acceleration, NULL);
}

int LZ4_compress_default(const char* src, char* dst, int srcSize, int dstCapacity)
{
    return one_block_compress(src, dst, srcSize, dstCapacity, 1, NULL);
}

static int state_is_valid(const void* state)
{
    /* LZ4_initStream, lz4.c:1552-1560: non-NULL and aligned like LZ4_stream_t (8 bytes) */
    return state != NULL && (((uintptr_t)state) & 7u) == 0;
}

int LZ4_compress_fast_extState(void* state, const char* src, char* dst, int srcSize, int dstCapacity, int acceleration)
{
    if (!state_is_valid(state)) return 0;
    return one_block_compress(src, dst, srcSize, dstCapacity, acceleration, NULL);
}

int LZ4_compress_fast_extState_fastReset(void* state, const char* src, char* dst, int srcSize, int dstCapacity, int acceleration)
{
    if (!state_is_valid(state)) return 0;
    return one_block_compress(src, dst, srcSize, dstCapacity, acceleration, NULL);
}

int LZ4_compress_destSize(const char* src, char* dst, int* srcSizePtr, int targetDstSize)
{
    if (srcSizePtr == NULL) return 0;
    return one_block_compress(src, dst, *srcSizePtr, targetDstSize, 1, srcSizePtr);
}

int LZ4_compress_destSize_extState(void* state, const char* src, char* dst, int* srcSizePtr, int targetDstSize, int acceleration)
{
    if (!state_is_valid(state) || srcSizePtr == NULL) return 0;
    return one_block_compress(src, dst, *srcSizePtr, targetDstSize, acceleration, srcSizePtr);
}

/* ------------------------------------------------------------------------------------------ */
/* drop-in HC layer (lz4hc.c:1486-1545): one block, host pointers, synchronous                 */
/* ------------------------------------------------------------------------------------------ */
/* LZ4_initStreamHC (lz4hc.c:1573-1586) zeroes the LZ4HC_CCtx_internal at the head of LZ4_streamHC_t (lz4hc.h:235-250:
 * 262 192 bytes on LP64 targets; the union's last 8 bytes are left alone) and sets its compressionLevel (offset
 * 262 180) to LZ4HC_CLEVEL_DEFAULT.  The alignment is LZ4_streamHC_t's (lz4hc.c:1488-1496), 8 bytes: pointer members. */
#define HC_STATE_INIT_BYTES   262192
#define HC_STATE_LEVEL_OFFSET 262180
#define HC_STATE_ALIGN        8u

static int hc_state_is_aligned(const void* state) { return (((uintptr_t)state) & (HC_STATE_ALIGN - 1)) == 0; }

/* LZ4_initStreamHC's checks and writes: 1 for a state that is non-NULL, aligned and now initialised, else 0 */
static int hc_state_init(void* state)
{
    const short level = 9;
    if (state == NULL || !hc_state_is_aligned(state)) return 0;
    memset(state, 0, HC_STATE_INIT_BYTES);
    memcpy((char*)state + HC_STATE_LEVEL_OFFSET, &level, sizeof level);
    return 1;
}

int LZ4_sizeofStateHC(void) { return LZ4B200_STATEHC_BYTES; }

/* srcSizePtr == NULL: LZ4_compress_HC_extStateHC_fastReset's routing (lz4hc.c:1506-1509: a capacity below the bound
 * limits the output).  Otherwise LZ4_compress_HC_destSize's fill parse (lz4hc.c:1544) with srcSize = *srcSizePtr and
 * targetDstSize = dstCapacity; *srcSizePtr receives the consumed input.  Levels <= 9 go to the hash-chain launchers,
 * levels >= 10 to the optimal parser's.  Like one_block_compress: the whole input is on the device before any byte is
 * written back, only the returned bytes are copied to dst, and the rules the reference decides without parsing are
 * decided here without a launch (lz4hc.c:1388-1389; an empty input is one 0x00 token). */
static int one_block_compress_hc(const char* src, char* dst, int srcSize, int dstCapacity, int level, int* srcSizePtr)
{
    int rc, bound;
    int32_t res[2] = {0, 0};                 /* return value, consumed input */
    slot_t* s = &g_ctx.slot[0];
    int32_t* d_res;
    void* ws;
    size_t wsBytes;
    if ((unsigned)srcSize > (unsigned)LZ4B200_MAX_INPUT_SIZE) return 0;
    if (dstCapacity < 1) return 0;           /* fillOutput: lz4hc.c:1388; limited output: not even a token fits */
    if (dst == NULL) return 0;
    if (srcSize > 0 && src == NULL) return 0;
    if (srcSize == 0) { dst[0] = 0; return 1; }   /* the last-literals token of an empty block; *srcSizePtr stays 0 */
    bound = LZ4_compressBound(srcSize);
    if ((rc = host_begin()) != LZ4B200_OK) goto done;
    rc = slot_take(s, (size_t)srcSize, (size_t)(dstCapacity < bound ? dstCapacity : bound),
                   LZ4B200_compress_blocks_hc_opt_workspace_bytes(1), 0, sizeof(res));
    if (rc != LZ4B200_OK) goto done;
    d_res = (int32_t*)s->d_tab.p;
    ws = s->ws.p; wsBytes = s->ws.cap;
    /* copy-in completes before any output is produced: in-place and overlapping buffers are safe */
    CU(cudaMemcpyAsync(s->in.p, src, (size_t)srcSize, cudaMemcpyHostToDevice, s->stream));
    if (srcSizePtr && level >= 10)
        rc = LZ4B200_compress_blocks_hc_opt_destSize(s->in.p, 0, NULL, srcSize, s->out.p, 0, dstCapacity, level,
                                                     d_res, d_res + 1, 1, ws, wsBytes, s->stream);
    else if (srcSizePtr)
        rc = LZ4B200_compress_blocks_hc_destSize(s->in.p, 0, NULL, srcSize, s->out.p, 0, dstCapacity, level,
                                                 d_res, d_res + 1, 1, ws, wsBytes, s->stream);
    else if (level >= 10)
        rc = LZ4B200_compress_blocks_hc_opt(s->in.p, 0, NULL, srcSize, s->out.p, 0, dstCapacity, level, d_res, 1,
                                            ws, wsBytes, s->stream);
    else
        rc = LZ4B200_compress_blocks_hc(s->in.p, 0, NULL, srcSize, s->out.p, 0, dstCapacity, level, d_res, 1,
                                        ws, wsBytes, s->stream);
    if (rc == LZ4B200_OK) rc = slot_return(s, (int32_t*)s->h_tab.p, d_res, res, srcSizePtr ? 2 : 1);
    if (rc == LZ4B200_OK) rc = slot_wait(s);
    if (rc == LZ4B200_OK && res[0] > 0) CU(cudaMemcpyAsync(dst, s->out.p, (size_t)res[0], cudaMemcpyDeviceToHost, s->stream));
done:
    if (host_end(rc) != LZ4B200_OK) return 0;
    if (srcSizePtr) *srcSizePtr = res[1];
    return res[0];
}

int LZ4_compress_HC(const char* src, char* dst, int srcSize, int dstCapacity, int compressionLevel)
{
    return one_block_compress_hc(src, dst, srcSize, dstCapacity, compressionLevel, NULL);
}

int LZ4_compress_HC_extStateHC(void* state, const char* src, char* dst, int srcSize, int dstCapacity, int compressionLevel)
{
    if (!hc_state_init(state)) return 0;
    return one_block_compress_hc(src, dst, srcSize, dstCapacity, compressionLevel, NULL);
}

int LZ4_compress_HC_extStateHC_fastReset(void* state, const char* src, char* dst, int srcSize, int dstCapacity,
                                         int compressionLevel)
{
    if (state == NULL || !hc_state_is_aligned(state)) return 0;
    return one_block_compress_hc(src, dst, srcSize, dstCapacity, compressionLevel, NULL);
}

int LZ4_compress_HC_destSize(void* state, const char* src, char* dst, int* srcSizePtr, int targetDstSize, int cLevel)
{
    if (!hc_state_init(state) || srcSizePtr == NULL) return 0;
    return one_block_compress_hc(src, dst, *srcSizePtr, targetDstSize, cLevel, srcSizePtr);
}

/* One block through the batch layer: LZ4_decompress_safe (partial == 0) or LZ4_decompress_safe_partial with outputSize =
 * dstCapacity.  The caller has decided the argument rules (compressedSize > 0, dstCapacity > 0, src and dst non-NULL).
 * Only the returned bytes are copied back: dst is untouched for a rejected block. */
static int one_block_decompress(const char* src, char* dst, int compressedSize, int dstCapacity, int partial)
{
    int rc, ret = -1;
    slot_t* s = &g_ctx.slot[0];
    int64_t *h_off, *d_off;
    int32_t *h_size, *d_size;
    if ((rc = host_begin()) != LZ4B200_OK) goto done;
    rc = slot_take(s, (size_t)compressedSize, (size_t)dstCapacity, LZ4B200_decompress_workspace_bytes_for(1, 0, dstCapacity), 0,
                   sizeof(int64_t) + 2 * sizeof(int32_t));
    if (rc != LZ4B200_OK) goto done;
    /* tables: [offset i64 | size i32 | return value i32], as in LZ4B200_decompress_blocks_host */
    h_off = (int64_t*)s->h_tab.p; h_size = (int32_t*)(h_off + 1);
    d_off = (int64_t*)s->d_tab.p; d_size = (int32_t*)(d_off + 1);
    *h_off = 0;
    *h_size = compressedSize;
    CU(cudaMemcpyAsync(d_off, h_off, sizeof(int64_t) + sizeof(int32_t), cudaMemcpyHostToDevice, s->stream));
    /* the whole input is on the device before the first output byte is written back: in-place
     * decompression (lz4.h:619-678, tests/fuzzer.c:1177-1187) needs no special handling */
    CU(cudaMemcpyAsync(s->in.p, src, (size_t)compressedSize, cudaMemcpyHostToDevice, s->stream));
    if (partial)
        rc = LZ4B200_decompress_blocks_partial(s->in.p, d_off, d_size, s->out.p, NULL, 0, NULL, dstCapacity,
                                               d_size + 1, 1, s->ws.p, s->ws.cap, s->stream);
    else
        rc = LZ4B200_decompress_blocks(s->in.p, d_off, d_size, s->out.p, NULL, 0, NULL, dstCapacity,
                                       d_size + 1, 1, s->ws.p, s->ws.cap, s->stream);
    if (rc == LZ4B200_OK) rc = slot_return(s, h_size + 1, d_size + 1, &ret, 1);
    if (rc == LZ4B200_OK) rc = slot_wait(s);
    if (rc == LZ4B200_OK && ret > 0) CU(cudaMemcpyAsync(dst, s->out.p, (size_t)ret, cudaMemcpyDeviceToHost, s->stream));
done:
    return host_end(rc) == LZ4B200_OK ? ret : -1;
}

int LZ4_decompress_safe(const char* src, char* dst, int compressedSize, int dstCapacity)
{
    /* lz4.c:2036, :2064-2069 decided on the host */
    if (src == NULL || dstCapacity < 0) return -1;
    if (dstCapacity == 0) return (compressedSize == 1 && src[0] == 0) ? 0 : -1;
    if (compressedSize <= 0) return -1;
    if (dst == NULL) return -1;
    return one_block_decompress(src, dst, compressedSize, dstCapacity, 0);
}

int LZ4_decompress_safe_partial(const char* src, char* dst, int srcSize, int targetOutputSize, int dstCapacity)
{
    const int outputSize = targetOutputSize < dstCapacity ? targetOutputSize : dstCapacity;   /* lz4.c:2461 */
    /* lz4.c:2036, :2066, :2069 decided on the host; a negative srcSize (undefined in the reference) and a NULL dst with
     * room to write are rejected */
    if (src == NULL || outputSize < 0) return -1;
    if (outputSize == 0) return 0;
    if (srcSize <= 0) return -1;
    if (dst == NULL) return -1;
    return one_block_decompress(src, dst, srcSize, outputSize, 1);
}

int LZ4_decompress_safe_usingDict(const char* src, char* dst, int compressedSize, int dstCapacity,
                                  const char* dictStart, int dictSize)
{
    (void)dictStart;
    if (dictSize == 0) return LZ4_decompress_safe(src, dst, compressedSize, dstCapacity);   /* lz4.c:2721-2722 */
    return -1;   /* prefix / external dictionaries: SURVEY.md section 8 (f-4), not on the GPU path */
}

/* ------------------------------------------------------------------------------------------ */
/* frame layer (SURVEY section 8 f-1): independent-block LZ4 frames over host buffers          */
/* ------------------------------------------------------------------------------------------ */
static void wr_le32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24); }

int64_t LZ4B200_compressFrameBound(int64_t srcSize, int blockSizeID)
{
    int64_t bs, nBlocks;
    if (srcSize < 0) return LZ4B200_ERR_ARG;
    if (blockSizeID == 0) blockSizeID = 4;
    if (blockSizeID < 4 || blockSizeID > 7) return LZ4B200_ERR_ARG;
    bs = fc_block_bytes(blockSizeID);
    nBlocks = srcSize / bs + 1;
    return 19 + nBlocks * 4 + srcSize + 4 + 4;     /* max header + block headers + data + EndMark (+ slack) */
}

int64_t LZ4B200_compressFrame_host(const void* h_src, int64_t srcSize, void* h_dst, int64_t dstCapacity,
                                   int blockSizeID, int compressionLevel, int contentSizeFlag)
{
    const uint8_t* src = (const uint8_t*)h_src;
    uint8_t* dst = (uint8_t*)h_dst;
    int64_t bs, nFull, lastSize, nBlocks, op = 0;
    int accel, bsid;
    if (srcSize < 0 || (!h_src && srcSize > 0) || !h_dst) return LZ4B200_ERR_ARG;
    if (blockSizeID == 0) blockSizeID = 4;
    if (blockSizeID < 4 || blockSizeID > 7) return LZ4B200_ERR_ARG;
    if (compressionLevel >= 2) return LZ4B200_ERR_UNSUPPORTED;          /* LZ4HC levels (lz4frame.c:952-962) */
    if (dstCapacity < LZ4B200_compressFrameBound(srcSize, blockSizeID)) return LZ4B200_ERR_DSTSIZE;
    accel = compressionLevel < 0 ? -compressionLevel + 1 : 1;           /* lz4frame.c:913 */
    bsid = fc_optimal_bsid(blockSizeID, srcSize);                        /* lz4frame.c:447 */
    bs = fc_block_bytes(bsid);
    op = fc_frame_header_bytes(dst, bsid, contentSizeFlag ? srcSize : 0);   /* lz4frame.c:781-809 */

    nFull = srcSize / bs;
    lastSize = srcSize - nFull * bs;
    nBlocks = nFull + (lastSize > 0);
    if (nBlocks > 0) {
        /* Groups of ~256 MiB of source go through the device: H2D, one compress launch (dstCapacity = blockSize - 1; a
         * result of 0 or >= the block's size means "store raw", LZ4F_makeBlock lz4frame.c:883-908), the frame body
         * ([LE32 header][payload] per block) is assembled ON THE DEVICE, and one D2H per group lands it in h_dst.  Group
         * g+1 is issued before group g is retired, so its copies and kernels overlap g's D2H. */
        int64_t group = ((int64_t)256 << 20) / bs, nGroups, g;
        const int64_t slotStride = (bs + 15) & ~(int64_t)15;
        int rc;
        if (group < 1) group = 1;
        nGroups = (nBlocks + group - 1) / group;
        if ((rc = host_begin()) != LZ4B200_OK) goto done;
        for (g = 0; g <= nGroups; g++) {
            if (g < nGroups) {                                         /* ---- issue group g ---- */
                slot_t* s = &g_ctx.slot[g % N_PIPE];
                const int64_t firstB = g * group;
                const int64_t cnt = (nBlocks - firstB < group) ? nBlocks - firstB : group;
                const int hasLast = (firstB + cnt == nBlocks) && lastSize > 0;
                const int64_t inBytes = (cnt - 1) * bs + (hasLast ? lastSize : bs);
                int64_t* d_off; int32_t* d_sz; int32_t* d_ssz;
                rc = slot_take(s, (size_t)inBytes, (size_t)(cnt * slotStride), 0, (size_t)(cnt * (bs + 4)),
                               (size_t)(cnt + 1) * sizeof(int64_t) + (size_t)cnt * 2 * sizeof(int32_t));
                if (rc != LZ4B200_OK) goto done;
                /* tables: [body offsets i64 (cnt + 1) | compressed sizes i32 | source sizes i32]; the host's first word
                 * receives the body size */
                d_off = (int64_t*)s->d_tab.p;
                d_sz = (int32_t*)(d_off + cnt + 1);
                d_ssz = d_sz + cnt;
                CU(cudaMemcpyAsync(s->in.p, src + firstB * bs, (size_t)inBytes, cudaMemcpyHostToDevice, s->stream));
                if (hasLast) {                                           /* per-block sizes only for the group with the ragged block */
                    int32_t* h_ssz = (int32_t*)((int64_t*)s->h_tab.p + cnt + 1) + cnt;
                    int64_t k;
                    for (k = 0; k < cnt; k++) h_ssz[k] = (int32_t)bs;
                    h_ssz[cnt - 1] = (int32_t)lastSize;
                    CU(cudaMemcpyAsync(d_ssz, h_ssz, (size_t)cnt * sizeof(int32_t), cudaMemcpyHostToDevice, s->stream));
                }
                rc = LZ4B200_compress_blocks(s->in.p, bs, hasLast ? d_ssz : NULL, (int32_t)bs, s->out.p, slotStride,
                                             (int32_t)(bs - 1), accel, d_sz, cnt, s->stream);
                if (rc != LZ4B200_OK) goto done;
                rc = LZ4B200_pack_frame_blocks(s->out.p, slotStride, d_sz, s->in.p, bs, (int32_t)bs,
                                               hasLast ? (int32_t)lastSize : 0, cnt, s->pack.p, d_off, s->stream);
                if (rc != LZ4B200_OK) goto done;
                CU(cudaMemcpyAsync(s->h_tab.p, d_off + cnt, sizeof(int64_t), cudaMemcpyDeviceToHost, s->stream));
            }
            if (g > 0) {                                               /* ---- retire group g-1: its size is known once its stream is idle ---- */
                slot_t* s = &g_ctx.slot[(g - 1) % N_PIPE];
                int64_t total;
                if ((rc = slot_wait(s)) != LZ4B200_OK) goto done;
                total = *(const int64_t*)s->h_tab.p;
                if (op + total + 4 > dstCapacity) { rc = LZ4B200_ERR_DSTSIZE; goto done; }
                CU(cudaMemcpyAsync(dst + op, s->pack.p, (size_t)total, cudaMemcpyDeviceToHost, s->stream));
                op += total;
            }
        }
    done:
        if ((rc = host_end(rc)) != LZ4B200_OK) return rc;
    }
    wr_le32(dst + op, 0); op += 4;                                        /* EndMark, lz4frame.c:1222 */
    return op;
}

int64_t LZ4B200_decompressFrame_host(const void* h_src, int64_t srcSize, void* h_dst, int64_t dstCapacity,
                                     int64_t* consumed)
{
    const uint8_t* src = (const uint8_t*)h_src;
    uint8_t* dst = (uint8_t*)h_dst;
    int64_t ip, at, sz, bs, nBlocks = 0, capBlocks = 0, k, total = 0, contentSize;
    int64_t* off = NULL; int32_t* csz = NULL; int32_t* rets = NULL; uint8_t* raw = NULL;
    int64_t result = LZ4B200_ERR_FRAME;
    fc_header_t hdr;
    int isRaw, step;
    if (!h_src || (!h_dst && dstCapacity > 0)) return LZ4B200_ERR_ARG;
    if ((step = fc_frame_header(src, srcSize, dstCapacity, FC_SUMS_REJECT, &hdr)) != LZ4B200_OK) return step;   /* lz4frame.c:1340-1425 */
    contentSize = hdr.contentSize;
    bs = fc_block_bytes(hdr.bsid);

    /* walk the chain of block headers (serial, O(#blocks)), lz4frame.c:1729-1758 */
    ip = hdr.hdrLen;
    while ((step = fc_next_block(src, srcSize, bs, 0, &ip, &at, &sz, &isRaw)) == 1) {
        if (nBlocks == capBlocks) {
            int64_t* o2; int32_t* c2; uint8_t* r2;
            capBlocks = capBlocks ? capBlocks * 2 : 1024;
            o2 = (int64_t*)realloc(off, (size_t)capBlocks * sizeof(int64_t));
            if (o2) off = o2;
            c2 = (int32_t*)realloc(csz, (size_t)capBlocks * sizeof(int32_t));
            if (c2) csz = c2;
            r2 = (uint8_t*)realloc(raw, (size_t)capBlocks);
            if (r2) raw = r2;
            if (!o2 || !c2 || !r2) { result = LZ4B200_ERR_ARG; goto done; }     /* (the old blocks are freed at `done`) */
        }
        off[nBlocks] = at; csz[nBlocks] = (int32_t)sz; raw[nBlocks] = (uint8_t)isRaw;
        nBlocks++;
    }
    if (step < 0) goto done;
    if (consumed) *consumed = ip;
    if (nBlocks == 0) { result = fc_frame_result(0, contentSize); goto done; }

    /* Every block is decoded with dstCapacity = maxBlockSize like lz4frame.c:1901-1904 does.  The frame is untrusted
     * input, so memory is bounded whatever it claims: blocks are decoded in GROUPS of at most ~256 MiB of block slots,
     * straight into h_dst while a group's slots (count x maxBlockSize) fit behind the bytes written so far -- short
     * blocks are then closed up in place -- and through one reusable bounce buffer otherwise (the tail of the caller's
     * buffer, or a flushed stream of many short blocks); the running total is checked after every group. */
    rets = (int32_t*)malloc((size_t)nBlocks * sizeof(int32_t));
    if (!rets) { result = LZ4B200_ERR_ARG; goto done; }
    {
        int64_t G = ((int64_t)256 << 20) / bs, g0;
        uint8_t* bounce = NULL;
        int32_t* tmpSz = NULL;
        if (G < 1) G = 1;
        if (G > nBlocks) G = nBlocks;
        tmpSz = (int32_t*)malloc((size_t)G * sizeof(int32_t));
        if (!tmpSz) { result = LZ4B200_ERR_ARG; goto done; }
        for (g0 = 0; g0 < nBlocks; g0 += G) {
            const int64_t cnt = (nBlocks - g0 < G) ? nBlocks - g0 : G;
            const int direct = (total + cnt * bs <= dstCapacity);
            uint8_t* base;
            int64_t pos = total;
            int anyGpu = 0, rc = LZ4B200_OK;
            if (!direct && !bounce) {
                bounce = (uint8_t*)malloc((size_t)(G * bs));
                if (!bounce) { free(tmpSz); result = LZ4B200_ERR_ARG; goto done; }
            }
            base = direct ? dst + total : bounce;
            /* stored-raw blocks need no GPU: they enter the batch with size 0 (rejected there) and are copied here */
            for (k = 0; k < cnt; k++) { tmpSz[k] = raw[g0 + k] ? 0 : csz[g0 + k]; anyGpu |= !raw[g0 + k]; }
            if (anyGpu) rc = LZ4B200_decompress_blocks_host(src, off + g0, tmpSz, base, bs, (int32_t)bs, rets + g0, cnt);
            if (rc != LZ4B200_OK) { free(bounce); free(tmpSz); result = rc; goto done; }
            for (k = 0; k < cnt; k++) {
                int64_t r;
                if (raw[g0 + k]) { memcpy(base + k * bs, src + off[g0 + k], (size_t)csz[g0 + k]); rets[g0 + k] = csz[g0 + k]; }
                r = rets[g0 + k];
                if ((step = fc_block_verdict(pos, r, dstCapacity, contentSize)) != LZ4B200_OK) {
                    free(bounce); free(tmpSz);
                    result = step;
                    goto done;
                }
                if (dst + pos != base + k * bs) memmove(dst + pos, base + k * bs, (size_t)r);      /* close the gap (moves left) */
                pos += r;
            }
            total = pos;
        }
        free(bounce); free(tmpSz);
    }
    result = fc_frame_result(total, contentSize);                        /* lz4frame.c: frameSize_wrong */
done:
    free(off); free(csz); free(raw); free(rets);
    return result;
}

/* ------------------------------------------------------------------------------------------ */
/* whole .lz4 files over host buffers: LZ4B200_decompress_files's results, pipelined in groups  */
/* ------------------------------------------------------------------------------------------ */
/* The content hash of a frame whose blocks span groups is carried in device memory from one group's carry kernel to the
 * next group's: group g writes slot g % FH_CARRIES of the ring and group g + 1 reads it after g's event.  Group
 * g + FH_CARRIES writes the same slot only after its pipeline slot, last used by group g + 1, is idle. */
#define FH_CARRIES (N_PIPE + 1)
#define FH_GAP     (64 << 10)   /* source pieces at most this far apart in h_src go over in one copy */
/* A group is retired (its results read, its bytes sent down) FH_LAG groups after it is issued, so that the copies down
 * of the groups before it run beside its kernels and the copies up of the groups after it.  Its slot is taken again
 * N_PIPE groups after it: FH_LAG < N_PIPE. */
#define FH_LAG     (N_PIPE - 1)
/* entered: the caller's stream at the start of a call that reads or writes the caller's device memory */
static struct { int ready; cudaEvent_t hashed[N_PIPE], entered; void* carry; } g_fh;

static int fh_init(void)
{
    int rc = LZ4B200_OK, i;
    if (g_fh.ready) return rc;
    for (i = 0; i < N_PIPE; i++) CU(cudaEventCreateWithFlags(&g_fh.hashed[i], cudaEventDisableTiming));
    CU(cudaEventCreateWithFlags(&g_fh.entered, cudaEventDisableTiming));
    CU(cudaMalloc(&g_fh.carry, FH_CARRIES * sizeof(fc_xxh32_state)));
    g_fh.ready = 1;
done:
    return rc;
}

static int64_t up16(int64_t x) { return (x + 15) & ~(int64_t)15; }

/* The checks of a call whose d_ pointers arrive from outside the library (under the host lock, after ctx_init):
 * LZ4B200_ERR_ARG, with LZ4B200_last_cuda_error() naming the pointer, for a d_ pointer that is not device or managed
 * memory of the pipeline's device, or an h_ pointer (NULL: not given) that is device memory, which the host would fault
 * on. */
static int ptr_check(const char* call, const char* name, const void* p, int device)
{
    struct cudaPointerAttributes at;
    int ok;
    if (!p) return LZ4B200_OK;
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
    ok = device ? (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) && at.device == g_ctx.device
                : at.type != cudaMemoryTypeDevice;
    if (ok) return LZ4B200_OK;
    snprintf(g_cuda_error, sizeof(g_cuda_error), "%s: %s is %s", call, name,
             device ? "not device memory of the pipeline's device" : "device memory, which the host cannot reach");
    return LZ4B200_ERR_ARG;
}

/* Every slot stream waits for the work enqueued on the caller's stream before the call (the slot streams do not
 * synchronise with the legacy default stream). */
static int enter_after(void* stream)
{
    int rc = LZ4B200_OK, i;
    CU(cudaEventRecord(g_fh.entered, (cudaStream_t)stream));
    for (i = 0; i < N_PIPE; i++) CU(cudaStreamWaitEvent(g_ctx.slot[i].stream, g_fh.entered, 0));
done:
    return rc;
}

/* Source pieces: [hostOff, devOff, bytes] triples in copies (room for one per block).  A block's bytes [lo, hi) join
 * the last piece when they begin in it or at most FH_GAP past its end, while the group's gaps stay within budget. */
static void piece_add(int64_t* copies, int64_t* nCopies, int64_t* gaps, int64_t lo, int64_t hi, int64_t budget)
{
    int64_t* cp = *nCopies ? copies + 3 * (*nCopies - 1) : NULL;
    const int64_t gap = cp ? lo - (cp[0] + cp[2]) : 0;
    if (cp && lo >= cp[0] && gap <= FH_GAP && *gaps + (gap > 0 ? gap : 0) <= budget) {
        if (gap > 0) *gaps += gap;
        if (hi > cp[0] + cp[2]) cp[2] = hi - cp[0];
    } else {
        cp = copies + 3 * (*nCopies)++; cp[0] = lo; cp[2] = hi - lo;
    }
}

/* where a block's bytes [lo, hi) are staged: the pieces are searched from *piece on, blocks in the order they were
 * added */
static int64_t piece_at(const int64_t* copies, int64_t* piece, int64_t lo, int64_t hi)
{
    const int64_t* cp = copies + 3 * *piece;
    while (!(lo >= cp[0] && hi <= cp[0] + cp[2])) cp = copies + 3 * ++*piece;
    return cp[1] + (lo - cp[0]);
}

/* segment q begins at block i of the group [first, end), for a frame of the blocks [base, base + count) */
static void seg_open(lz4k_seg* q, int64_t i, int64_t base, int64_t count, int64_t first, int64_t end)
{
    q->first = (int32_t)i; q->end = (int32_t)i + 1; q->pad = 0;
    q->flags = (base < first ? LZ4K_SEG_CONTINUES : 0) | (base + count <= end ? LZ4K_SEG_ENDS : 0);
}

/* The content checksums of group g's segments on slot s (seg: their host copy).  Only the first and the last segment
 * can be carried: the first continues the state the group before left in the ring, after that group's event; the last
 * leaves its state in the ring for the group after and records the event that group waits on. */
static int seg_content(slot_t* s, int64_t g, const lz4k_seg* seg, lz4k_seg_args* a)
{
    int32_t f0, fl;
    int rc = LZ4B200_OK;
    if (!a->nSegs) return rc;
    f0 = seg[0].flags; fl = seg[a->nSegs - 1].flags;
    a->carryIn = (const fc_xxh32_state*)g_fh.carry + (g + FH_CARRIES - 1) % FH_CARRIES;
    a->carryOut = (fc_xxh32_state*)g_fh.carry + g % FH_CARRIES;
    if (f0 & LZ4K_SEG_CONTINUES) CU(cudaStreamWaitEvent(s->stream, g_fh.hashed[(g + N_PIPE - 1) % N_PIPE], 0));
    rc = lz4k_launch_seg_content(a, f0 != LZ4K_SEG_ENDS || fl != LZ4K_SEG_ENDS, s->stream);
    if ((rc = launched(rc, "lz4k_launch_seg_content")) != LZ4B200_OK) return rc;
    if (!(fl & LZ4K_SEG_ENDS)) CU(cudaEventRecord(g_fh.hashed[g % N_PIPE], s->stream));
done:
    return rc;
}

/* a run of bytes contiguous in slot s's packed buffer and in the host output, copied down in one piece */
typedef struct { uint8_t* host; int64_t dev, len; } run_t;

static int run_flush(slot_t* s, run_t* r)
{
    int rc = LZ4B200_OK;
    if (r->len) CU(cudaMemcpyAsync(r->host, (uint8_t*)s->pack.p + r->dev, (size_t)r->len, cudaMemcpyDeviceToHost, s->stream));
    r->len = 0;
done:
    return rc;
}

/* len bytes at dev in the packed buffer to host: they extend the run, or the run goes down and theirs begins */
static int run_add(slot_t* s, run_t* r, int64_t dev, uint8_t* host, int64_t len)
{
    int rc = LZ4B200_OK;
    if (r->len && r->dev + r->len == dev && r->host + r->len == host) r->len += len;
    else if ((rc = run_flush(s, r)) == LZ4B200_OK) { r->dev = dev; r->host = host; r->len = len; }
    return rc;
}

/* A group's table in its slot (the host copy pinned, the device copy the kernels use), for n blocks and nSegs segments:
 * [srcOff, gatherOff, dstOff: i64 n | segments | srcSize, rawLen, ord, sum: i32 n] go up, [sum, outSize: i32 n |
 * digest: u32 nSegs] come back, [blockSize: i32 n | blockFrom: i64 n | blockOff: i64 n + 1] stay on the device;
 * [runs: lz4k_run nRuns] go up at retire when the output goes to device memory. */
typedef struct { size_t srcOff, gatherOff, dstOff, segs, srcSize, rawLen, ord, sum, outSize, digest, blockSize, blockFrom, blockOff, runs, bytes; } fh_tab_t;

static fh_tab_t fh_tab(int64_t n, int64_t nSegs, int64_t nRuns)
{
    fh_tab_t t;
    const size_t w8 = (size_t)n * 8, w4 = (size_t)n * 4;
    t.srcOff = 0; t.gatherOff = w8; t.dstOff = 2 * w8; t.segs = 3 * w8;
    t.srcSize = t.segs + (size_t)nSegs * sizeof(lz4k_seg);
    t.rawLen = t.srcSize + w4; t.ord = t.rawLen + w4; t.sum = t.ord + w4; t.outSize = t.sum + w4; t.digest = t.outSize + w4;
    t.blockSize = t.digest + (size_t)nSegs * 4;
    t.blockFrom = (t.blockSize + w4 + 7) & ~(size_t)7;
    t.blockOff = t.blockFrom + w8;
    t.runs = t.blockOff + w8 + 8;
    t.bytes = t.runs + (size_t)nRuns * sizeof(lz4k_run);
    return t;
}

/* what the host keeps of a group in flight: its blocks, segments and room for runs (the rest is in its slot's pinned
 * table) */
typedef struct { int64_t first, end, nSegs, nRuns; } fh_group_t;

/* Issue group gr on slot s (group index g): the table, the source pieces, the decode per class, the block checksums,
 * and unless sizeOnly the assembly and the content hash; then the results back to the pinned table.  devDst: the table
 * keeps room for the runs of the group's output, cut at LZ4K_SCATTER_RUN bytes. */
static int fh_issue(const fp_plan* p, const uint8_t* src, int64_t g, slot_t* s, fh_group_t* gr, int sizeOnly, int verify,
                    int devDst, int64_t* copies)
{
    const int64_t n = gr->end - gr->first;
    const int hash = verify && !sizeOnly;               /* the content checksums (none when the call only sizes) */
    int64_t nc[FC_CLASSES] = {0, 0, 0, 0, 0}, cb[FC_CLASSES], fill[FC_CLASSES], k, e, nSegs = 0, nCopies = 0, gaps = 0;
    int64_t slotBytes = 0, inBytes = 0, at;
    size_t wsBytes = 0;
    int c, rc = LZ4B200_OK, anySum = 0;
    fh_tab_t t;
    uint8_t* h;
    uint8_t* d;
    lz4k_group_args a;
    lz4k_seg_args sa;
    lz4k_seg* seg;
    /* the classes, their slots, the segments and the source pieces */
    for (k = gr->first; k < gr->end; k++) nc[(int)p->blocks[k].cls]++;
    for (c = 0, at = 0; c < FC_CLASSES; c++) {
        cb[c] = at; fill[c] = at; at += nc[c];
        slotBytes += nc[c] * fc_class_bytes(c);
        if (nc[c]) {
            const size_t w = lz4k_decode_workspace_bytes(nc[c], 0, (int32_t)fc_class_bytes(c), SIZE_MAX);
            if (w > wsBytes) wsBytes = w;
        }
    }
    for (k = gr->first; k < gr->end; k++) {
        const fp_unit* u = &p->units[p->blocks[k].unit];
        if (hash && fp_content(u) && (k == gr->first || p->blocks[k - 1].unit != p->blocks[k].unit)) nSegs++;
    }
    /* the pieces, staged after the slots; a group of at most CHUNK_OUT_BYTES of 64 KB or larger slots has fewer gaps
     * of FH_GAP than that, so the budget never binds */
    for (k = gr->first; k < gr->end; k++) {
        const fp_block* b = &p->blocks[k];
        piece_add(copies, &nCopies, &gaps, b->srcOff, b->srcOff + b->size + b->sumBytes, CHUNK_OUT_BYTES);
    }
    at = sizeOnly ? 0 : (slotBytes + 255) & ~(int64_t)255;              /* (the scan alone writes no slot) */
    for (k = 0; k < nCopies; k++) { copies[3 * k + 1] = at; at = up16(at + copies[3 * k + 2]); }
    inBytes = at;
    gr->nRuns = devDst ? n + slotBytes / LZ4K_SCATTER_RUN + 1 : 0;
    t = fh_tab(n, nSegs, gr->nRuns);
    if ((rc = slot_take(s, 0, (size_t)inBytes, wsBytes, sizeOnly ? 0 : (size_t)slotBytes, t.bytes)) != LZ4B200_OK)
        return rc;
    h = (uint8_t*)s->h_tab.p;
    seg = (lz4k_seg*)(h + t.segs);
    gr->nSegs = 0;
    /* the table: entries by class, blocks in file order */
    {
        int64_t* srcOff = (int64_t*)(h + t.srcOff);
        int64_t* gatherOff = (int64_t*)(h + t.gatherOff);
        int64_t* dstOff = (int64_t*)(h + t.dstOff);
        int32_t* srcSize = (int32_t*)(h + t.srcSize);
        int32_t* rawLen = (int32_t*)(h + t.rawLen);
        int32_t* ord = (int32_t*)(h + t.ord);
        int32_t* sum = (int32_t*)(h + t.sum);
        int64_t slotAt[FC_CLASSES], piece = 0, u = -1;
        for (c = 0, at = 0; c < FC_CLASSES; c++) { slotAt[c] = at; at += nc[c] * fc_class_bytes(c); }
        for (k = gr->first; k < gr->end; k++) {
            const fp_block* b = &p->blocks[k];
            e = fill[(int)b->cls]++;
            ord[k - gr->first] = (int32_t)e;
            srcOff[e] = piece_at(copies, &piece, b->srcOff, b->srcOff + b->size + b->sumBytes);
            dstOff[e] = slotAt[(int)b->cls] + (e - cb[(int)b->cls]) * fc_class_bytes(b->cls);
            gatherOff[e] = b->raw ? srcOff[e] : dstOff[e];
            srcSize[e] = b->raw ? 0 : b->size;
            rawLen[e] = b->raw ? b->size : -1;
            sum[e] = (verify && b->verify) ? FC_SUM_PENDING : FC_SUM_NONE;
            anySum |= verify && b->verify;
            if (b->unit != u) {
                const fp_unit* un = &p->units[b->unit];
                u = b->unit;
                if (hash && fp_content(un))
                    seg_open(&seg[gr->nSegs++], k - gr->first, un->r.base, un->r.count, gr->first, gr->end);
            } else if (hash && fp_content(&p->units[u])) {
                seg[gr->nSegs - 1].end++;
            }
        }
    }
    /* up: the table and the pieces */
    d = (uint8_t*)s->d_tab.p;
    CU(cudaMemcpyAsync(d, h, t.outSize, cudaMemcpyHostToDevice, s->stream));
    for (k = 0; k < nCopies; k++)
        CU(cudaMemcpyAsync((uint8_t*)s->out.p + copies[3 * k + 1], src + copies[3 * k], (size_t)copies[3 * k + 2],
                           cudaMemcpyHostToDevice, s->stream));
    memset(&a, 0, sizeof a);
    a.base = (uint8_t*)s->out.p; a.packed = (uint8_t*)s->pack.p; a.n = n;
    a.srcOff = (const int64_t*)(d + t.srcOff); a.gatherOff = (const int64_t*)(d + t.gatherOff);
    a.srcSize = (const int32_t*)(d + t.srcSize); a.rawLen = (const int32_t*)(d + t.rawLen);
    a.ord = (const int32_t*)(d + t.ord); a.sum = (int32_t*)(d + t.sum); a.outSize = (const int32_t*)(d + t.outSize);
    a.blockSize = (int32_t*)(d + t.blockSize); a.blockFrom = (int64_t*)(d + t.blockFrom); a.blockOff = (int64_t*)(d + t.blockOff);
    /* the decode of every class at its uniform capacity (the scan alone when sizing) */
    for (c = 0; c < FC_CLASSES; c++) {
        lz4k_decode_args dd;
        if (!nc[c]) continue;
        memset(&dd, 0, sizeof dd);
        dd.src = a.base; dd.srcOff = a.srcOff + cb[c]; dd.srcSize = a.srcSize + cb[c];
        dd.dst = a.base; dd.dstOff = (const int64_t*)(d + t.dstOff) + cb[c]; dd.dstCap = (int32_t)fc_class_bytes(c);
        dd.outSize = (int32_t*)(d + t.outSize) + cb[c]; dd.nBlocks = nc[c];
        dd.workspace = s->ws.p; dd.workspaceBytes = s->ws.cap;
        if ((rc = launched(lz4k_launch_decode(&dd, sizeOnly ? 1 : 3, 0, s->stream), "lz4k_launch_decode")) != LZ4B200_OK)
            return rc;
    }
    if (anySum && (rc = launched(lz4k_launch_group_block_sums(&a, s->stream), "lz4k_launch_group_block_sums")) != LZ4B200_OK)
        return rc;
    if (!sizeOnly) {
        if ((rc = launched(lz4k_launch_group_assemble(&a, s->stream), "lz4k_launch_group_assemble")) != LZ4B200_OK) return rc;
        memset(&sa, 0, sizeof sa);                        /* the content hash of the output, block after block */
        sa.base = a.packed; sa.off = a.blockOff; sa.size = a.blockSize;
        sa.segs = (const lz4k_seg*)(d + t.segs); sa.nSegs = gr->nSegs; sa.digest = (uint32_t*)(d + t.digest);
        if ((rc = seg_content(s, g, seg, &sa)) != LZ4B200_OK) return rc;
    }
    /* down: the block checksums' outcomes, the decode's results and the segments' */
    CU(cudaMemcpyAsync(h + t.sum, d + t.sum, t.blockSize - t.sum, cudaMemcpyDeviceToHost, s->stream));
done:
    return rc;
}

/* Retire the group gr that ran on slot s: its results into the plan, then (unless sizeOnly) its bytes from the slot's
 * packed output to the files as fp_place places them.  Into host memory (dst, devDst 0): one copy down per run of bytes
 * contiguous on both sides.  Into device memory (devDst 1): the runs, cut at LZ4K_SCATTER_RUN bytes, in the slot's
 * table and one scatter on its stream (the slot is taken again only after this, as FH_LAG < N_PIPE).  runs: room for
 * the group's blocks. */
static int fh_retire(fp_plan* p, slot_t* s, const fh_group_t* gr, int sizeOnly, uint8_t* dst, int devDst,
                     const int64_t* dstOff, const int64_t* dstCap, int64_t* filePos, uint8_t* fileStop, fp_run* runs)
{
    const int64_t n = gr->end - gr->first;
    const fh_tab_t t = fh_tab(n, gr->nSegs, gr->nRuns);
    int64_t k, r, nRuns;
    run_t run = {NULL, 0, 0};
    uint8_t* h;
    const int32_t *ord, *sum, *out;
    const uint32_t* digest;
    const lz4k_seg* seg;
    int rc = slot_wait(s);
    if (rc != LZ4B200_OK) return rc;
    h = (uint8_t*)s->h_tab.p;
    ord = (const int32_t*)(h + t.ord); sum = (const int32_t*)(h + t.sum); out = (const int32_t*)(h + t.outSize);
    digest = (const uint32_t*)(h + t.digest); seg = (const lz4k_seg*)(h + t.segs);
    for (k = 0; k < n; k++) {
        p->outSize[gr->first + k] = out[ord[k]];
        p->sumState[gr->first + k] = sum[ord[k]] == FC_SUM_BAD ? FC_SUM_BAD : FC_SUM_NONE;
    }
    for (k = 0; k < gr->nSegs; k++)
        if (seg[k].flags & LZ4K_SEG_ENDS) {
            const int64_t u = p->blocks[gr->first + seg[k].first].unit;
            p->contentBad[u] = digest[k] != p->units[u].contentSum;
        }
    if (sizeOnly) return rc;
    nRuns = fp_place(p, gr->first, gr->end, dstCap, filePos, fileStop, runs);
    if (!devDst) {
        for (r = 0; r < nRuns; r++)
            if ((rc = run_add(s, &run, runs[r].packed, dst + dstOff[runs[r].file] + runs[r].fileOff, runs[r].len)) != LZ4B200_OK)
                return rc;
        return run_flush(s, &run);
    }
    {
        lz4k_run* dr = (lz4k_run*)(h + t.runs);
        lz4k_scatter_args a;
        int64_t m = 0, at;
        for (r = 0; r < nRuns; r++)
            for (at = 0; at < runs[r].len; at += LZ4K_SCATTER_RUN, m++) {
                dr[m].src = runs[r].packed + at;
                dr[m].dst = dstOff[runs[r].file] + runs[r].fileOff + at;
                dr[m].len = runs[r].len - at < LZ4K_SCATTER_RUN ? runs[r].len - at : LZ4K_SCATTER_RUN;
            }
        if (!m) return rc;
        CU(cudaMemcpyAsync((uint8_t*)s->d_tab.p + t.runs, dr, (size_t)m * sizeof(lz4k_run), cudaMemcpyHostToDevice, s->stream));
        a.packed = (const uint8_t*)s->pack.p; a.dst = dst; a.runs = (const lz4k_run*)((uint8_t*)s->d_tab.p + t.runs); a.nRuns = m;
        rc = launched(lz4k_launch_group_scatter(&a, s->stream), "lz4k_launch_group_scatter");
    }
done:
    return rc;
}

/* LZ4B200_ERR_ARG, with LZ4B200_last_cuda_error() saying that the host's memory ran out (under the host lock) */
static int out_of_host_memory(const char* call)
{
    snprintf(g_cuda_error, sizeof(g_cuda_error), "%s: out of host memory", call);
    return LZ4B200_ERR_ARG;
}

/* walk (host) -> per group, N_PIPE in flight: issue group g, then retire group g - FH_LAG -> fold (host).  devDst: dst is
 * the caller's device memory, written after the work on `stream` before the call. */
static int decompress_files_run(const char* call, const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                void* dst, int devDst, const int64_t* h_dstOff, const int64_t* h_dstCap, int64_t* h_result,
                                int64_t* h_consumed, int64_t* h_prefix, int64_t nFiles, int skipChecksums, int sizeOnly,
                                void* stream)
{
    const int verify = !skipChecksums;
    fp_plan p;
    fh_group_t grs[N_PIPE];
    int64_t *copies = NULL, *filePos = NULL, first, g, nGroups = 0;
    uint8_t* fileStop = NULL;
    fp_run* runs = NULL;
    int rc;
    memset(&p, 0, sizeof p);
    if ((rc = host_begin()) != LZ4B200_OK) goto done;
    if ((rc = fh_init()) != LZ4B200_OK) goto done;
    if (devDst) {
        const void* hp[8] = {h_src, h_srcOff, h_srcSize, h_dstOff, h_dstCap, h_result, h_consumed, h_prefix};
        const char* hn[8] = {"h_src", "h_srcOff", "h_srcSize", "h_dstOff", "h_dstCap", "h_result", "h_consumed", "h_prefix"};
        int i;
        if ((rc = ptr_check(call, "d_dst", dst, 1)) != LZ4B200_OK) goto done;
        for (i = 0; i < 8; i++)
            if ((rc = ptr_check(call, hn[i], hp[i], 0)) != LZ4B200_OK) goto done;
        if ((rc = enter_after(stream)) != LZ4B200_OK) goto done;
    }
    if (!fp_build((const uint8_t*)h_src, h_srcOff, h_srcSize, sizeOnly ? NULL : h_dstCap, nFiles,
                  verify ? FC_SUMS_VERIFY : FC_SUMS_SKIP, &p)) { rc = out_of_host_memory(call); goto done; }
    copies = (int64_t*)malloc((size_t)(p.nBlocks ? p.nBlocks : 1) * 3 * sizeof(int64_t));
    runs = (fp_run*)malloc((size_t)(p.nBlocks ? p.nBlocks : 1) * sizeof(fp_run));
    filePos = (int64_t*)calloc((size_t)nFiles, sizeof(int64_t));
    fileStop = (uint8_t*)calloc((size_t)nFiles, 1);
    if (!copies || !runs || !filePos || !fileStop) { rc = out_of_host_memory(call); goto done; }
    for (first = 0; first < p.nBlocks; nGroups++) first = fp_group_end(&p, first, CHUNK_OUT_BYTES);
    for (g = 0, first = 0; g < nGroups + FH_LAG; g++) {
        if (g < nGroups) {
            fh_group_t* gr = &grs[g % N_PIPE];
            gr->first = first;
            gr->end = fp_group_end(&p, first, CHUNK_OUT_BYTES);
            first = gr->end;
            if ((rc = fh_issue(&p, (const uint8_t*)h_src, g, &g_ctx.slot[g % N_PIPE], gr, sizeOnly, verify, devDst,
                               copies)) != LZ4B200_OK)
                goto done;
        }
        if (g >= FH_LAG && (rc = fh_retire(&p, &g_ctx.slot[(g - FH_LAG) % N_PIPE], &grs[(g - FH_LAG) % N_PIPE], sizeOnly,
                                           (uint8_t*)dst, devDst, h_dstOff, h_dstCap, filePos, fileStop, runs)) != LZ4B200_OK)
            goto done;
    }
    /* every group has retired: the results are in the plan (the last copies down or scatters may still run) */
    if (!fp_fold(&p, h_srcSize, sizeOnly ? NULL : h_dstCap, h_result, h_consumed, h_prefix))
        rc = out_of_host_memory(call);
done:
    rc = host_end(rc);
    fp_free(&p);
    free(copies); free(runs); free(filePos); free(fileStop);
    return rc;
}

int LZ4B200_decompress_files_host(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                  void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                  int64_t* h_result, int64_t* h_consumed, int64_t* h_prefix,
                                  int64_t nFiles, int skipChecksums, int sizeOnly)
{
    if (nFiles < 0) return LZ4B200_ERR_ARG;
    if (nFiles == 0) return LZ4B200_OK;
    if (!h_src || !h_srcOff || !h_srcSize || !h_result) return LZ4B200_ERR_ARG;
    if (!sizeOnly && (!h_dst || !h_dstOff || !h_dstCap)) return LZ4B200_ERR_ARG;
    return decompress_files_run(__func__, h_src, h_srcOff, h_srcSize, h_dst, 0, h_dstOff, h_dstCap, h_result, h_consumed,
                                h_prefix, nFiles, skipChecksums, sizeOnly, NULL);
}

int LZ4B200_decompress_files_to_device(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                       void* d_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                       int64_t* h_result, int64_t* h_consumed, int64_t* h_prefix,
                                       int64_t nFiles, int skipChecksums, void* stream)
{
    if (nFiles < 0) return LZ4B200_ERR_ARG;
    if (nFiles == 0) return LZ4B200_OK;
    if (!h_src || !h_srcOff || !h_srcSize || !d_dst || !h_dstOff || !h_dstCap || !h_result) return LZ4B200_ERR_ARG;
    return decompress_files_run(__func__, h_src, h_srcOff, h_srcSize, d_dst, 1, h_dstOff, h_dstCap, h_result, h_consumed,
                                h_prefix, nFiles, skipChecksums, 0, stream);
}

/* ------------------------------------------------------------------------------------------ */
/* whole .lz4 files written from host buffers: LZ4B200_compress_frames_checksummed's and       */
/* LZ4B200_compress_legacy's bytes, pipelined in groups                                        */
/* ------------------------------------------------------------------------------------------ */
/* Source bytes per group (G).  One warp encodes one block, so a group costs about one block's encode whatever its size
 * until the SMs fill, and the rate grows with G: DESIGN section 3.18 has the sweep that chose the default.
 * LZ4B200_HOST_WRITE_MB overrides it (developer knob for tests/perf), read once per process. */
#define CW_DEFAULT_MB 512
/* Blocks per group (B): at HC levels each block holds an HC workspace slot of 256 KB (320 KB for the optimal parser),
 * so B bounds that workspace; the other parses need no workspace and B only bounds the group's table. */
#define CW_HC_BLOCKS  2048
#define CW_BLOCKS     65536

static int64_t write_group_bytes(void)
{
    static int64_t v = 0;
    if (v == 0) {
        const char* e = getenv("LZ4B200_HOST_WRITE_MB");
        long mb = e ? atol(e) : 0;
        v = (int64_t)((mb >= 1 && mb <= 4096) ? mb : CW_DEFAULT_MB) << 20;
    }
    return v;
}

/* A group's table in its slot, for n blocks and nSegs segments: [srcOff, slotOff: i64 n | segments | srcSize, cap: i32 n]
 * go up, [outSize: i32 n] stays on the device, [bodyOff: i64 n + 1 | digest: u32 nSegs] come back. */
typedef struct { size_t srcOff, slotOff, segs, srcSize, cap, outSize, bodyOff, digest, bytes; } cw_tab_t;

static cw_tab_t cw_tab(int64_t n, int64_t nSegs)
{
    cw_tab_t t;
    const size_t w8 = (size_t)n * 8, w4 = (size_t)n * 4;
    t.srcOff = 0; t.slotOff = w8; t.segs = 2 * w8;
    t.srcSize = t.segs + (size_t)nSegs * sizeof(lz4k_seg);
    t.cap = t.srcSize + w4; t.outSize = t.cap + w4;
    t.bodyOff = (t.outSize + w4 + 7) & ~(size_t)7;
    t.digest = t.bodyOff + w8 + 8;
    t.bytes = t.digest + (size_t)nSegs * 4;
    return t;
}

/* the encode of a writer call: its parse and level, and the checksums its frames carry (none for legacy streams) */
typedef struct { int hcLevel, accel, parallel, sums; } cw_enc_t;

/* Issue group gr on slot s (group index g): the table and the source pieces up, the encode, the body, the block
 * checksums, the content checksums; then the body's offsets and the digests back to the pinned table.  devSrc: src is
 * the caller's device memory, which every step reads where it lies (no pieces, no input buffer). */
static int cw_issue(const cp_plan* p, const uint8_t* src, int devSrc, int64_t g, slot_t* s, fh_group_t* gr,
                    const cw_enc_t* c, int64_t* copies)
{
    const int64_t n = gr->end - gr->first, G = write_group_bytes();
    const int hash = !p->legacy && (c->sums & FC_CONTENT_SUM);
    int64_t k, f = -1, nCopies = 0, gaps = 0, nSegs = 0, slotBytes = 0, packBytes = 0, at;
    size_t hcBytes = 0;
    int rc = LZ4B200_OK;
    cw_tab_t t;
    uint8_t *h, *d;
    const uint8_t* base;                                  /* where the steps read the source */
    lz4k_seg* seg;
    lz4k_encode_args e;
    lz4k_wgroup_args a;
    lz4k_seg_args sa;
    /* the pieces, with the group's gaps within G, so that the staged bytes stay within 2 G (plus alignment) */
    for (k = gr->first; k < gr->end; k++) {
        if (!devSrc) piece_add(copies, &nCopies, &gaps, p->srcOff[k], p->srcOff[k] + p->size[k], G);
        slotBytes += up16(p->cap[k]);
        packBytes += 8 + (p->legacy ? p->cap[k] : p->size[k]);
        if (hash && p->file[k] != f) { nSegs++; f = p->file[k]; }
    }
    for (k = 0, at = 0; k < nCopies; k++) { copies[3 * k + 1] = at; at = up16(at + copies[3 * k + 2]); }
    if (c->hcLevel > 0) hcBytes = c->hcLevel >= 10 ? lz4k_encode_hc_opt_workspace_bytes(n) : lz4k_encode_hc_workspace_bytes(n);
    t = cw_tab(n, nSegs);
    if ((rc = slot_take(s, (size_t)at, (size_t)slotBytes, hcBytes, (size_t)packBytes, t.bytes)) != LZ4B200_OK) return rc;
    h = (uint8_t*)s->h_tab.p;
    d = (uint8_t*)s->d_tab.p;
    base = devSrc ? src : (const uint8_t*)s->in.p;
    seg = (lz4k_seg*)(h + t.segs);
    gr->nSegs = 0;
    /* the table: blocks in file order, each frame's blocks one segment */
    {
        int64_t* srcOff = (int64_t*)(h + t.srcOff);
        int64_t* slotOff = (int64_t*)(h + t.slotOff);
        int32_t* srcSize = (int32_t*)(h + t.srcSize);
        int32_t* cap = (int32_t*)(h + t.cap);
        int64_t piece = 0;
        for (k = gr->first, at = 0, f = -1; k < gr->end; k++) {
            const int64_t i = k - gr->first;
            srcOff[i] = devSrc ? p->srcOff[k] : piece_at(copies, &piece, p->srcOff[k], p->srcOff[k] + p->size[k]);
            srcSize[i] = p->size[k];
            cap[i] = p->cap[k];
            slotOff[i] = at;
            at += up16(p->cap[k]);
            if (!hash) continue;
            if (p->file[k] != f) {
                const fc_frame_rec* r = &p->files[p->file[k]];
                f = p->file[k];
                seg_open(&seg[gr->nSegs++], i, r->base, r->count, gr->first, gr->end);
            } else {
                seg[gr->nSegs - 1].end++;                    /* a file's blocks lie together in one piece */
            }
        }
    }
    /* up: the table and the pieces */
    CU(cudaMemcpyAsync(d, h, t.outSize, cudaMemcpyHostToDevice, s->stream));
    for (k = 0; k < nCopies; k++)
        CU(cudaMemcpyAsync((uint8_t*)s->in.p + copies[3 * k + 1], src + copies[3 * k], (size_t)copies[3 * k + 2],
                           cudaMemcpyHostToDevice, s->stream));
    /* the encode of every block into its slot at its capacity */
    e = encode_args(base, 0, (const int32_t*)(d + t.srcSize), 0, s->out.p, 0, 0, c->accel, (int32_t*)(d + t.outSize), n);
    e.srcOff = (const int64_t*)(d + t.srcOff); e.dstOff = (const int64_t*)(d + t.slotOff); e.dstCapArr = (const int32_t*)(d + t.cap);
    if ((rc = encode_table(&e, c->hcLevel, c->parallel, s->ws.p, s->ws.cap, s->stream)) != LZ4B200_OK) return rc;
    /* the body, the block checksums, the content checksums */
    memset(&a, 0, sizeof a);
    a.src = base; a.slots = (const uint8_t*)s->out.p; a.packed = (uint8_t*)s->pack.p; a.n = n;
    a.srcOff = e.srcOff; a.srcSize = e.srcSizeArr; a.slotOff = e.dstOff; a.outSize = e.outSize;
    a.bodyOff = (int64_t*)(d + t.bodyOff);
    a.legacy = p->legacy;
    a.blockSums = !p->legacy && (c->sums & FC_BLOCK_SUM);
    if ((rc = launched(lz4k_launch_wgroup_body(&a, s->stream), "lz4k_launch_wgroup_body")) != LZ4B200_OK) return rc;
    memset(&sa, 0, sizeof sa);                            /* the content hash of the source */
    sa.base = a.src; sa.off = a.srcOff; sa.size = a.srcSize;
    sa.segs = (const lz4k_seg*)(d + t.segs); sa.nSegs = gr->nSegs; sa.digest = (uint32_t*)(d + t.digest);
    if ((rc = seg_content(s, g, seg, &sa)) != LZ4B200_OK) return rc;
    /* down: the body's offsets and the digests */
    CU(cudaMemcpyAsync(h + t.bodyOff, d + t.bodyOff, t.bytes - t.bodyOff, cudaMemcpyDeviceToHost, s->stream));
done:
    return rc;
}

/* File f's end at byte pos of its output at: a frame's EndMark and, with the content checksum, its digest; returns the
 * file's length */
static int64_t cw_end(const cp_plan* p, int64_t f, uint8_t* at, int64_t pos, uint32_t digest)
{
    if (p->legacy) return pos;
    wr_le32(at + pos, 0);
    if (p->files[f].sums & FC_CONTENT_SUM) { wr_le32(at + pos + 4, digest); return pos + 8; }
    return pos + 4;
}

/* Retire the group gr that ran on slot s: its body from the slot's packed buffer to each file's running position, one
 * copy per run of bytes contiguous on both sides, and the end of every file whose last block it holds. */
static int cw_retire(const cp_plan* p, slot_t* s, const fh_group_t* gr, uint8_t* dst, const int64_t* dstOff,
                     int64_t* filePos, int64_t* result)
{
    const int64_t n = gr->end - gr->first;
    const cw_tab_t t = cw_tab(n, gr->nSegs);
    int64_t k, f = -1, sg = -1;
    run_t run = {NULL, 0, 0};
    const int64_t* bodyOff;
    const uint32_t* digest;
    int rc = slot_wait(s);
    if (rc != LZ4B200_OK) return rc;
    bodyOff = (const int64_t*)((const uint8_t*)s->h_tab.p + t.bodyOff);
    digest = (const uint32_t*)((const uint8_t*)s->h_tab.p + t.digest);
    for (k = 0; k < n; k++) {
        const int64_t b = gr->first + k, len = bodyOff[k + 1] - bodyOff[k];
        const fc_frame_rec* r;
        if (p->file[b] != f) { f = p->file[b]; sg++; }      /* (segment sg, when the frames carry content checksums) */
        r = &p->files[f];
        if ((rc = run_add(s, &run, bodyOff[k], dst + dstOff[f] + filePos[f], len)) != LZ4B200_OK) return rc;
        filePos[f] += len;
        if (b == r->base + r->count - 1)
            result[f] = cw_end(p, f, dst + dstOff[f], filePos[f], sg < gr->nSegs ? digest[sg] : 0);
    }
    return run_flush(s, &run);
}

/* plan (host: verdicts, headers, empty files) -> per group, N_PIPE in flight: issue group g, then retire group
 * g - FH_LAG (bodies, EndMarks, digests, results).  devSrc: src is the caller's device memory, read after the work on
 * `stream` before the call. */
static int compress_files_host(const char* call, const void* src, int devSrc, const int64_t* h_srcOff,
                               const int64_t* h_srcSize, void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                               int64_t* h_result, int64_t nFiles, int legacy, int bsid, int contentSizeFlag,
                               const cw_enc_t* c, void* stream)
{
    uint8_t* dst = (uint8_t*)h_dst;
    cp_plan p;
    fh_group_t grs[N_PIPE];
    int64_t *copies = NULL, *filePos = NULL, first, g, f, nGroups = 0, maxBlocks = c->hcLevel > 0 ? CW_HC_BLOCKS : CW_BLOCKS;
    int rc;
    memset(&p, 0, sizeof p);
    if ((rc = host_begin()) != LZ4B200_OK) goto done;
    if ((rc = fh_init()) != LZ4B200_OK) goto done;
    if (devSrc) {
        const void* hp[6] = {h_srcOff, h_srcSize, h_dst, h_dstOff, h_dstCap, h_result};
        const char* hn[6] = {"h_srcOff", "h_srcSize", "h_dst", "h_dstOff", "h_dstCap", "h_result"};
        int i;
        if ((rc = ptr_check(call, "d_src", src, 1)) != LZ4B200_OK) goto done;
        for (i = 0; i < 6; i++)
            if ((rc = ptr_check(call, hn[i], hp[i], 0)) != LZ4B200_OK) goto done;
        if ((rc = enter_after(stream)) != LZ4B200_OK) goto done;
    }
    if (!cp_build(h_srcOff, h_srcSize, h_dstCap, nFiles, legacy, bsid, contentSizeFlag, c->sums, &p)) {
        rc = out_of_host_memory(call); goto done;
    }
    copies = (int64_t*)malloc((size_t)(p.nBlocks ? p.nBlocks : 1) * 3 * sizeof(int64_t));
    filePos = (int64_t*)calloc((size_t)nFiles, sizeof(int64_t));
    if (!copies || !filePos) { rc = out_of_host_memory(call); goto done; }
    for (f = 0; f < nFiles; f++) {                  /* the headers; a file of no blocks ends here */
        const fc_frame_rec* r = &p.files[f];
        if (r->status != LZ4B200_OK) { h_result[f] = r->status; continue; }
        filePos[f] = cp_header(&p, f, dst + h_dstOff[f]);
        if (r->count == 0) h_result[f] = cw_end(&p, f, dst + h_dstOff[f], filePos[f], fc_xxh32(dst, 0, 0));
    }
    for (first = 0; first < p.nBlocks; nGroups++) first = cp_group_end(&p, first, write_group_bytes(), maxBlocks);
    for (g = 0, first = 0; g < nGroups + FH_LAG; g++) {
        if (g < nGroups) {
            fh_group_t* gr = &grs[g % N_PIPE];
            gr->first = first;
            gr->end = cp_group_end(&p, first, write_group_bytes(), maxBlocks);
            first = gr->end;
            if ((rc = cw_issue(&p, (const uint8_t*)src, devSrc, g, &g_ctx.slot[g % N_PIPE], gr, c, copies)) != LZ4B200_OK)
                goto done;
        }
        if (g >= FH_LAG && (rc = cw_retire(&p, &g_ctx.slot[(g - FH_LAG) % N_PIPE], &grs[(g - FH_LAG) % N_PIPE], dst,
                                           h_dstOff, filePos, h_result)) != LZ4B200_OK)
            goto done;
    }
done:
    rc = host_end(rc);                              /* (the last copies down end here) */
    cp_free(&p);
    free(copies); free(filePos);
    return rc;
}

/* the frame writers' arguments: LZ4B200_ERR_ARG or LZ4B200_OK with *c set; nFiles == 0 is the caller's */
static int frames_enc(int64_t nFiles, int* blockSizeID, int compressionLevel, int parallel, int blockChecksumFlag,
                      int contentChecksumFlag, cw_enc_t* c)
{
    if (nFiles < 0) return LZ4B200_ERR_ARG;
    if (*blockSizeID == 0) *blockSizeID = 4;
    if (*blockSizeID < 4 || *blockSizeID > 7) return LZ4B200_ERR_ARG;
    if (parallel && compressionLevel >= 2) return LZ4B200_ERR_ARG;
    frames_levels(compressionLevel, &c->hcLevel, &c->accel);
    c->parallel = parallel != 0;
    c->sums = (blockChecksumFlag ? FC_BLOCK_SUM : 0) | (contentChecksumFlag ? FC_CONTENT_SUM : 0);
    return LZ4B200_OK;
}

int LZ4B200_compress_frames_host(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                 void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                 int64_t* h_result, int64_t nFiles,
                                 int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                                 int blockChecksumFlag, int contentChecksumFlag)
{
    cw_enc_t c;
    if (frames_enc(nFiles, &blockSizeID, compressionLevel, parallel, blockChecksumFlag, contentChecksumFlag, &c) != LZ4B200_OK)
        return LZ4B200_ERR_ARG;
    if (nFiles == 0) return LZ4B200_OK;
    if (!h_src || !h_srcOff || !h_srcSize || !h_dst || !h_dstOff || !h_dstCap || !h_result) return LZ4B200_ERR_ARG;
    return compress_files_host(__func__, h_src, 0, h_srcOff, h_srcSize, h_dst, h_dstOff, h_dstCap,
                               h_result, nFiles, 0, blockSizeID, contentSizeFlag, &c, NULL);
}

int LZ4B200_compress_frames_from_device(const void* d_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                        void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                        int64_t* h_result, int64_t nFiles,
                                        int blockSizeID, int compressionLevel, int contentSizeFlag, int parallel,
                                        int blockChecksumFlag, int contentChecksumFlag, void* stream)
{
    cw_enc_t c;
    if (nFiles < 0) return LZ4B200_ERR_ARG;
    if (nFiles == 0) return LZ4B200_OK;
    if (frames_enc(nFiles, &blockSizeID, compressionLevel, parallel, blockChecksumFlag, contentChecksumFlag, &c) != LZ4B200_OK)
        return LZ4B200_ERR_ARG;
    if (!d_src || !h_srcOff || !h_srcSize || !h_dst || !h_dstOff || !h_dstCap || !h_result) return LZ4B200_ERR_ARG;
    return compress_files_host(__func__, d_src, 1, h_srcOff, h_srcSize, h_dst, h_dstOff, h_dstCap,
                               h_result, nFiles, 0, blockSizeID, contentSizeFlag, &c, stream);
}

int LZ4B200_compress_legacy_host(const void* h_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                 void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                 int64_t* h_result, int64_t nFiles, int compressionLevel)
{
    cw_enc_t c;
    if (nFiles < 0) return LZ4B200_ERR_ARG;
    if (nFiles == 0) return LZ4B200_OK;
    if (!h_src || !h_srcOff || !h_srcSize || !h_dst || !h_dstOff || !h_dstCap || !h_result) return LZ4B200_ERR_ARG;
    legacy_levels(compressionLevel, &c.hcLevel, &c.accel);
    c.parallel = 0;
    c.sums = 0;
    return compress_files_host(__func__, h_src, 0, h_srcOff, h_srcSize, h_dst, h_dstOff, h_dstCap,
                               h_result, nFiles, 1, 0, 0, &c, NULL);
}

int LZ4B200_compress_legacy_from_device(const void* d_src, const int64_t* h_srcOff, const int64_t* h_srcSize,
                                        void* h_dst, const int64_t* h_dstOff, const int64_t* h_dstCap,
                                        int64_t* h_result, int64_t nFiles, int compressionLevel, void* stream)
{
    cw_enc_t c;
    if (nFiles < 0) return LZ4B200_ERR_ARG;
    if (nFiles == 0) return LZ4B200_OK;
    if (!d_src || !h_srcOff || !h_srcSize || !h_dst || !h_dstOff || !h_dstCap || !h_result) return LZ4B200_ERR_ARG;
    legacy_levels(compressionLevel, &c.hcLevel, &c.accel);
    c.parallel = 0;
    c.sums = 0;
    return compress_files_host(__func__, d_src, 1, h_srcOff, h_srcSize, h_dst, h_dstOff, h_dstCap,
                               h_result, nFiles, 1, 0, 0, &c, stream);
}
