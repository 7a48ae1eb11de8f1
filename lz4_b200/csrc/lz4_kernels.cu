/*
 * lz4_kernels.cu -- hand-written sm_90a (H100) CUDA kernels of the LZ4 block codec.
 *
 * Decode = two kernels (DESIGN.md section 3):
 *   scan   : one THREAD per block walks the token chain and applies every acceptance rule of the
 *            reference decoder (lz4.c:2022-2445, x86-64 control flow incl. the fast loop), giving
 *            the exact return value, and leaves a 4-byte mark per sequence.  No data is moved.
 *   expand : moves the bytes of blocks the scan accepted (literal + match copies).
 * Encode = one WARP per block replaying the reference's greedy parse (lz4.c:930-1338) with the
 *   32 lanes probing 32 consecutive search positions per step; output is byte-identical.
 * pack   = exclusive scan of block sizes + gather into one contiguous stream.
 *
 * All arithmetic is integer/byte; no tensor cores (this is an HBM/latency-bound scan codec).
 */
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <stddef.h>
#include "lz4_kernels.h"

namespace {

constexpr int kMinMatch = 4;
constexpr int kLastLiterals = 5;
constexpr int kMfLimit = 12;
constexpr int kMinLength = 13;
constexpr uint32_t kMaxDistance = 65535;
constexpr int kSmallLimit = 65536 + 11;          // lz4.c:710
constexpr int kSkipTrigger = 6;                  // lz4.c:711
constexpr int kAccelMax = 65537;                 // lz4.c:58
constexpr uint32_t kMaxInput = 0x7E000000u;      // lz4.h:214
constexpr unsigned kFull = 0xFFFFFFFFu;

unsigned long long g_launches = 0;

/* optional phase timing of the fast expand kernel (thread 0 of each CTA; enabled with -DLZ4K_PHASE_TIMING) */
__device__ unsigned long long g_phaseCycles[8];
__device__ unsigned long long g_loopStats[4];    // phase B: warp iterations, lane-iterations with a piece, blocked lane-iterations, pieces done
#ifdef LZ4K_PHASE_TIMING
#define PHASE_MARK(i) do { if (tid == 0) { const long long t_ = clock64(); atomicAdd(&g_phaseCycles[i], (unsigned long long)(t_ - tPhase)); tPhase = t_; } } while (0)
#else
#define PHASE_MARK(i) do { } while (0)
#endif

/* byte readers + the per-block scan (scan_front / scan_tail / scan_block): shared with the CPU
 * emulators under tests/emul/, see the header */
#define LZ4_SCAN_CORE_CONSTANTS
#include "lz4_scan_core.h"
#include "lz4_scan_par.h"
#include "lz4_scan_split.h"
#include "lz4_rows_core.h"
#include "lz4_decode_plan.h"     /* a decode call's workspace layout (WsView), scan choice and block predicates */

/* low 5 bytes at p (for the 5-byte hash, lz4.c:785-791) */
__device__ __forceinline__ uint64_t ld40u(const uint8_t* p)
{
    uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* w = reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3));
    uint32_t sh = (uint32_t)(a & 3) * 8;
    uint32_t lo = __ldg(w);
    uint32_t hi = __ldg(w + 1);
    uint32_t v = __funnelshift_r(lo, hi, sh);
    uint32_t b4 = (hi >> sh) & 0xFFu;
    return (uint64_t)v | ((uint64_t)b4 << 32);
}

constexpr int kInBytes = 65536 + 64;           /* staged compressed block: <= 65535 bytes + 16-byte phase + rounding */

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
/* wait for the phase with the given parity; the hardware may suspend the warp for up to kWaitHintNs per attempt, so that
 * waiting warps do not take issue slots from the warps they are waiting for */
constexpr uint32_t kWaitHintNs = 2000;
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n selp.u32 %0, 1, 0, p;\n}\n"
                     : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(kWaitHintNs) : "memory");
    } while (!ok);
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void tma_load_1d(void* smemDst, const void* gsrc, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(smemDst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void tma_store_1d(void* gdst, const void* smemSrc, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                 ::"l"(gdst), "r"(smem_u32(smemSrc)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_wait_all0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void fence_acq_rel_cta() { asm volatile("fence.acq_rel.cta;" ::: "memory"); }

/* TMA bulk load of the n bytes at src into shared memory at dst, completing on `bar`.  The load starts at the 16-byte
 * boundary below src and is rounded up to 16 bytes, so dst needs room for head + n + 15 bytes; byte i of the block lands
 * at dst[head + i].  Only `issuer` issues the load; every caller gets the head. */
__device__ __forceinline__ int tma_stage(uint8_t* dst, const uint8_t* src, int n, uint64_t* bar, bool issuer = true)
{
    const int head = (int)(reinterpret_cast<uintptr_t>(src) & 15);
    if (issuer) {
        const uint32_t loadBytes = (uint32_t)((head + n + 15) & ~15);
        mbar_expect_tx(bar, loadBytes);
        for (uint32_t o = 0; o < loadBytes; o += 16384u) tma_load_1d(dst + o, src - head + o, min(16384u, loadBytes - o), bar);
    }
    return head;
}


/* a scan kernel's result for block b: the decoder's return value and the sequence count; an accepted block that neither
 * the rows kernel nor (`tiled`) the tiles kernel takes goes on the generic kernel's list */
__device__ __forceinline__ void scan_result(const lz4k_decode_args& a, const WsView& w, int64_t b, int n, int cap, int r,
                                            uint32_t ns, bool tiled = false)
{
    a.outSize[b] = r;
    w.nSeq[b] = ns;
    if (r > 0 && !tiled && !rows_eligible(n, cap, ns, w.markStride)) w.slowList[atomicAdd(&w.hdr->slowCount, 1u)] = (uint32_t)b;
}

/* ---- scan, one THREAD per block: reads through the read-only data cache with L1 prefetch hints, marks in 32-byte chunks ---- */

__global__ void __launch_bounds__(128) lz4_scan_kernel(lz4k_decode_args a, WsView w)
{
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.nBlocks) return;
    const uint8_t* src = a.src + a.srcOff[b];
    const int n = a.srcSize[b];
    int cap = a.dstCapArr ? a.dstCapArr[b] : a.dstCap;
    uint32_t ns = 0;
    MemPtr<true> mem{src};
    const int r = scan_block(mem, n, cap, &ns, block_marks(w, b, n, cap, kMarksNarrow), w.markStride);
    scan_result(a, w, b, n, cap, r, ns);
}

/* ---- scan of the partial call, one THREAD per block: LZ4_decompress_safe_partial with outputSize = the block's target ----
 * The walk ends at the target, so its chain of dependent steps grows with the decoded prefix, not the block.  Marks are
 * written for every target of at most 64 KB, whatever the input size: the rows kernel stages only the consumed prefix.
 * Route P1 (lz4_expand_rows_partial_kernel): rows_eligible on (consumed, target); P2 (the generic kernel): the rest. */
__global__ void __launch_bounds__(128) lz4_scan_partial_kernel(lz4k_decode_args a, WsView w)
{
    int64_t b = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= a.nBlocks) return;
    const uint8_t* src = a.src + a.srcOff[b];
    const int n = a.srcSize[b];
    const int cap = a.dstCapArr ? a.dstCapArr[b] : a.dstCap;
    uint32_t ns = 0, used = 0;
    MemPtr<true> mem{src};
    const int r = scan_block<MemPtr<true>, true>(mem, n, cap, &ns, block_marks(w, b, n, cap, kMarksPartial), w.markStride, &used);
    if (w.used) w.used[b] = used;
    scan_result(a, w, b, (int)used, cap, r, ns);
}

/* ---- scan, kSsLanes lanes per block that merge (lz4_scan_split.h): the chain of dependent steps is kSsLanes times shorter ----
 * The lanes of a block are neighbours in a warp (32 / kSsLanes blocks per warp); phases are separated by __syncwarp.
 * Lists go to the scratch part of the workspace (2 x markStride words per block), the per-block records to shared memory. */
constexpr int kSplitThreads = 128;
constexpr int kSplitBlocksPerCta = kSplitThreads / kSsLanes;

__global__ void __launch_bounds__(kSplitThreads, 10) lz4_scan_split_kernel(lz4k_decode_args a, WsView w)
{
    __shared__ SsBlock sh[kSplitBlocksPerCta];
    const int lane = threadIdx.x % kSsLanes, slot = threadIdx.x / kSsLanes;
    const int64_t b = (int64_t)blockIdx.x * kSplitBlocksPerCta + slot;
    if (b >= a.nBlocks) return;                                 /* (whole groups of kSsLanes lanes leave together) */
    const unsigned grp = ((1u << kSsLanes) - 1u) << ((threadIdx.x & 31) / kSsLanes * kSsLanes);   /* this block's lanes in the warp */
    const uint8_t* src = a.src + a.srcOff[b];
    const int n = a.srcSize[b];
    const int cap = a.dstCapArr ? a.dstCapArr[b] : a.dstCap;
    uint32_t* marks = block_marks(w, b, n, cap, kMarksNarrow);
    SsBlock& S = sh[slot];
    MemPtr<true> mem{src};
    int r = 0;
    uint32_t ns = 0;
    bool serial = !(marks && cap >= 64 && n >= kSsMinBytes);
    if (!serial) {
        const uint32_t R = w.markStride / kSsLanes;
        uint32_t* sc = w.scratch + b * 2 * (int64_t)w.markStride;
        uint32_t* A = sc + (size_t)lane * R;
        uint32_t* B = sc + w.markStride + (size_t)lane * R;
        ss_p1(lane, S, mem, n, A, B, R);
        __syncwarp(grp);
        ss_p2(lane, S, mem, n, A, B, R, [&](int t) { return sc + w.markStride + (size_t)t * R; });
        __syncwarp(grp);
        if (lane == 0) ss_p3(S, [&](int t) { return sc + (size_t)t * R; });
        __syncwarp(grp);
        serial = S.fallback != 0;
        if (!serial) {
            uint32_t e, c, co;
            ss_p4(lane, S, cap, A, B, marks, w.markStride, e, c, co);
            #pragma unroll
            for (int m = 1; m < kSsLanes; m <<= 1) {
                const uint32_t e2 = __shfl_xor_sync(grp, e, m), c2 = __shfl_xor_sync(grp, c, m), co2 = __shfl_xor_sync(grp, co, m);
                if (e2 < e) e = e2;
                if (c2 < c) { c = c2; co = co2; }
            }
            if (lane == 0) { S.errIdx = e; S.capIdx = c; S.capOpn = co; }
            __syncwarp(grp);                                        /* the final marks of every lane are written */
            if (lane == 0) r = ss_p5(S, mem, n, cap, &ns, marks, w.markStride);
        }
    }
    if (serial && lane == 0) r = scan_block(mem, n, cap, &ns, marks, w.markStride);
    if (lane == 0) scan_result(a, w, b, n, cap, r, ns);
}

/* ---- scan, one CTA of NL lanes per block (lz4_scan_par.h): same outputs as lz4_scan_kernel ----
 * Blocks of up to 65 535 bytes are staged in shared memory by one TMA bulk load (the walks are chains of
 * dependent 4-byte reads: ~30 cycles each from shared memory instead of an L2 / HBM round trip); larger
 * blocks (lz4frame's 4 MB blocks) are walked in global memory by the same lanes. */
constexpr int kScanLanes = 128;
static_assert(kScanLanes % 32 == 0 && kScanLanes <= kSpMaxLanes, "scan lanes");

struct ScanParSmem {
    alignas(16) uint8_t in[65536 + 64];
    SpShared sp;
    uint32_t warpCnt[kSpMaxLanes / 32], warpLen[kSpMaxLanes / 32];
    int first;
    alignas(8) uint64_t mbar;
};

template <class M>
__device__ __forceinline__ void scan_par_block(ScanParSmem& S, M& mem, int n, int cap, uint32_t* marks, uint32_t markCap,
                                               int& ret, uint32_t& nseq)
{
    const int lane = threadIdx.x, nl = kScanLanes;
    if (cap < 64 || n < kSpMinBytes) {
        if (lane == 0) { uint32_t ns = 0; S.sp.ret = scan_block(mem, n, cap, &ns, marks, markCap); S.sp.nseq = ns; }
        __syncthreads();
        ret = S.sp.ret; nseq = S.sp.nseq;
        __syncthreads();
        return;
    }
    SpLane L;
    sp_phase0(lane, nl, L, S.sp, mem, n, cap);
    __syncthreads();
    for (;;) {
        sp_decide(lane, L, S.sp);
        __syncthreads();                                   /* everybody has read S.changed's previous value and its neighbour's result */
        if (lane == 0) S.sp.changed = 0;
        __syncthreads();
        sp_redo(lane, L, S.sp, mem, n, cap);
        __syncthreads();
        if (!S.sp.changed) break;
    }
    /* exclusive sums of (count, olen) over the lanes */
    uint32_t c = S.sp.res[lane].count, o = S.sp.res[lane].olen, ci = c, oi = o;
    #pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t yc = __shfl_up_sync(kFull, ci, d), yo = __shfl_up_sync(kFull, oi, d);
        if ((lane & 31) >= d) { ci += yc; oi += yo; }
    }
    if ((lane & 31) == 31) { S.warpCnt[lane >> 5] = ci; S.warpLen[lane >> 5] = oi; }
    if (lane == 0) S.first = nl - 1;
    __syncthreads();
    uint32_t cb = ci - c, ob = oi - o;
    for (int wq = 0; wq < (lane >> 5); wq++) { cb += S.warpCnt[wq]; ob += S.warpLen[wq]; }
    sp_write(lane, L, S.sp, mem, n, cap, cb, ob, marks, markCap);
    if (S.sp.end[lane].kind != SP_RAN) atomicMin(&S.first, lane);
    __syncthreads();
    sp_finish(lane, S.first, S.sp, mem, n, cap, marks, markCap);
    __syncthreads();
    ret = S.sp.ret; nseq = S.sp.nseq;
    __syncthreads();
}

__global__ void __launch_bounds__(kScanLanes) lz4_scan_par_kernel(lz4k_decode_args a, WsView w)
{
    extern __shared__ __align__(16) uint8_t smemRaw[];
    ScanParSmem& S = *reinterpret_cast<ScanParSmem*>(smemRaw);
    const int tid = threadIdx.x;
    uint32_t parity = 0;
    if (tid == 0) mbar_init(&S.mbar, 1);
    __syncthreads();
    for (int64_t b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
        const uint8_t* src = a.src + a.srcOff[b];
        const int n = a.srcSize[b];
        const int cap = a.dstCapArr ? a.dstCapArr[b] : a.dstCap;
        uint32_t* marks = block_marks(w, b, n, cap, w.wide ? kMarksWide : kMarksNarrow);
        int r = -1;
        uint32_t ns = 0;
        /* the lanes' walk over `mem`; in a wide batch the marks are two words per sequence (MemPtr<G, true>) */
        auto lanes = [&](auto mem) { scan_par_block(S, mem, n, cap, marks, mark_cap(w), r, ns); };
        if (n > 0 && n <= 65535 && cap > 0) {                     /* staged in shared memory */
            const int head = tma_stage(S.in, src, n, &S.mbar, tid == 0);
            while (!mbar_try_wait(&S.mbar, parity)) { }
            parity ^= 1;
            if (w.wide) lanes(MemPtr<false, true>{S.in + head});
            else lanes(MemPtr<false>{S.in + head});
        } else if (n > 65535 && cap >= 64) {                      /* walked in global memory */
            if (w.wide) lanes(MemPtr<true, true>{src});
            else lanes(MemPtr<true>{src});
        } else {                                                   /* degenerate arguments: the one-thread code decides (lz4.c:2036, :2064-2069) */
            if (tid == 0) { uint32_t q = 0; MemPtr<true> mem{src}; S.sp.ret = scan_block(mem, n, cap, &q, nullptr, 0u); S.sp.nseq = q; }
            __syncthreads();
            r = S.sp.ret; ns = S.sp.nseq;
            __syncthreads();
        }
        if (tid == 0) scan_result(a, w, b, n, cap, r, ns, w.wide && tiles_eligible(w, ns));
    }
}

/* ---- wide batches: per tile of kTile output bytes the first sequence whose match starts in or beyond it (tile_index_seq);
 * done flags cleared ---- */
__global__ void __launch_bounds__(256) lz4_tile_index_kernel(lz4k_decode_args a, WsView w)
{
    for (int64_t b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
        uint32_t* first = w.tileFirst + (size_t)b * (w.tilesMax + 1);
        uint32_t* flag = w.tileFlag + (size_t)b * (w.tilesMax + 1);
        for (uint32_t t = threadIdx.x; t <= w.tilesMax; t += blockDim.x) flag[t] = 0u;
        const int total = a.outSize[b];
        const uint32_t ns = w.nSeq[b];
        if (total <= 0 || ns == 0 || !tiles_eligible(w, ns)) continue;
        const uint32_t nT = tiles_of(total);
        const uint32_t* marks = w.marks + (size_t)b * w.markStride;
        for (uint32_t k = threadIdx.x; k < ns; k += blockDim.x) tile_index_seq(first, marks, k, ns, nT);
    }
}

/* =============================================================================================
 * expand (generic): one warp per accepted block, any block size, straight to global memory
 * ============================================================================================= */
/* PARTIAL: the partial call's blocks (route P2): the decode stops at the scan's return value, and the literal and match
 * runs that reach it are cut there (the scan's walk ended at the same place, lz4_scan_core.h: scan_tail) */
template <bool PARTIAL>
__device__ __forceinline__ void expand_generic(const lz4k_decode_args& a, const WsView& w)
{
    const int lane = threadIdx.x & 31;
    const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int64_t nWarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
    const int64_t count = w.hdr->slowCount;       // only blocks the scan accepted and left to this kernel
    for (int64_t idx = warp0; idx < count; idx += nWarps) {
    const int64_t b = w.slowList[idx];
    const uint8_t* __restrict__ src = a.src + a.srcOff[b];
    uint8_t* dst = a.dst + (a.dstOff ? a.dstOff[b] : b * a.dstStride);
    const int64_t n = a.srcSize[b];
    const int64_t total = PARTIAL ? a.outSize[b] : 0;
    int64_t ip = 0, op = 0;

    for (;;) {
        uint32_t token = ldb<true>(src + ip); ip++;
        int64_t ll = token >> 4;
        if (ll == 15) { uint32_t x; do { x = ldb<true>(src + ip); ip++; ll += x; } while (x == 255); }
        if (PARTIAL && ll > total - op) ll = total - op;
        for (int64_t k = lane; k < ll; k += 32) dst[op + k] = (uint8_t)ldb<true>(src + ip + k);
        ip += ll; op += ll;
        if (PARTIAL ? op >= total : ip >= n) break;
        uint32_t offset = ld16<true>(src + ip); ip += 2;
        int64_t ml = token & 15;
        if (ml == 15) { uint32_t x; do { x = ldb<true>(src + ip); ip++; ml += x; } while (x == 255); }
        ml += kMinMatch;
        if (PARTIAL && ml > total - op) ml = total - op;
        __syncwarp();                             // everything before `op` is now visible to all lanes
        if (offset == 0) {                        // reference zero-fills (lz4.c:2407, :500)
            for (int64_t k = lane; k < ml; k += 32) dst[op + k] = 0;
        } else if ((int64_t)offset >= ml) {
            const volatile uint8_t* from = dst + op - offset;
            for (int64_t k = lane; k < ml; k += 32) dst[op + k] = from[k];
        } else {                                  // self-overlapping match: period `offset`
            const volatile uint8_t* from = dst + op - offset;
            for (int64_t k = lane; k < ml; k += 32) dst[op + k] = from[k % offset];
        }
        op += ml;
        if (PARTIAL && op >= total) break;
    }
    __syncwarp();
    }
}

__global__ void __launch_bounds__(128) lz4_expand_generic_kernel(lz4k_decode_args a, WsView w) { expand_generic<false>(a, w); }
__global__ void __launch_bounds__(128) lz4_expand_generic_partial_kernel(lz4k_decode_args a, WsView w) { expand_generic<true>(a, w); }

/* =============================================================================================
 * expand (rows): one CTA per 64 KB block, one output BYTE per thread, waves + run table
 *
 * See lz4_rows_core.h for the formulation.  Per block:
 *   TMA bulk load  : compressed block HBM -> smem (`in`, placed below `out` in the window)
 *   runs, pass 1   : one lane per sequence re-reads its token (marks from the scan) and sets one bit
 *                    per run start (literal run, match run, pieces of self-overlapping matches)
 *   rank           : rows[r].y = (run starts before row r) - 1
 *   runs, pass 2   : the same lanes write delta(run) at the run's rank
 *   waves          : kWave bytes per CTA barrier; thread t handles bytes t, t+1024, ... of the wave:
 *                    rank -> delta -> (follow sources inside the wave) -> LDS.U8 -> STS.U8
 *   TMA bulk store : decoded block smem -> HBM
 * ============================================================================================= */
constexpr int kRowsThreads = 1024;
constexpr int kRowsRpt = 4;                  /* rows per thread per wave: wave = 1024 * kRowsRpt bytes */
constexpr int kWave = kRowsThreads * kRowsRpt;
constexpr int kRowsCache = 3;                /* sequences per thread whose parse is kept in registers between the passes */

struct RowsDesc {                            /* one block's arguments, fetched a block ahead */
    const uint8_t* src;
    uint8_t* dst;
    int n, total, nseq;
    int64_t b;
};

struct RowsSmem {
    alignas(16) uint8_t zero[16];            /* always-zero cell: source of offset-0 matches (lz4.c:2407) */
    alignas(16) uint8_t in[kInBytes];        /* staged compressed block; keeps the source's 16-byte phase */
    alignas(16) uint8_t out[65536];          /* output window; MUST lie above `zero` and `in` */
    alignas(16) uint32_t tab[kRowsMaxRuns];  /* delta per run */
    alignas(8) uint2 rows[2048];             /* {run-start bits of the row, run starts before the row - 1} */
    uint32_t warpSum[32];
    alignas(8) uint64_t mbar;                /* TMA load of `in` */
    alignas(8) uint64_t wbar;                /* wave barrier: one arrival per warp */
    RowsDesc desc[2];
    uint32_t nRuns;
};
static_assert(sizeof(RowsSmem) <= 232448, "RowsSmem exceeds the 227 KB of shared memory a CTA can opt in to");

__device__ __forceinline__ uint2 lds_u64(uint32_t a)
{
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds_u32(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds_u8(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u8(uint32_t a, uint32_t v)
{
    asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__device__ __forceinline__ uint32_t lanemask_le()
{
    uint32_t m;
    asm("mov.u32 %0, %%lanemask_le;" : "=r"(m));
    return m;
}

/* ---- the phases of a window shared by lz4_expand_rows_kernel and lz4_expand_tiles_kernel ---- */

/* runs pass 1 (PASS1: one bit per run start) or pass 2 (each run's delta at its rank) over the sequences [k0, k1):
 * thread t takes k0 + t, k0 + t + 1024, ...  Pass 1 keeps the parse of the thread's first kRowsCache sequences in sq for
 * pass 2.  parse(i, k) returns sequence k, the thread's i-th (i = kRowsCache for all past the cache); runs(s, f) calls
 * f(start, delta) for each run of s in the window, in increasing start order, and first(s) is the first one's start
 * (-1: none). */
template <bool PASS1, class Parse, class First, class Runs>
__device__ __forceinline__ void rows_runs_pass(RowsSmem& S, RwSeq (&sq)[kRowsCache], const int k0, const int k1,
                                               Parse&& parse, First&& first, Runs&& runs)
{
    auto body = [&](const RwSeq& s) {
        if constexpr (PASS1) runs(s, [&](int st, int) { atomicOr(&S.rows[st >> 5].x, 1u << (st & 31)); });
        else rw_put_deltas(S.rows, S.tab, first(s), [&](auto f) { runs(s, f); });
    };
    #pragma unroll
    for (int i = 0; i < kRowsCache; i++) {
        const int k = k0 + (int)threadIdx.x + i * kRowsThreads;
        if (k < k1) {
            if constexpr (PASS1) sq[i] = parse(i, k);
            body(sq[i]);
        }
    }
    for (int k = k0 + (int)threadIdx.x + kRowsCache * kRowsThreads; k < k1; k += kRowsThreads) body(parse(kRowsCache, k));
}

/* rank: rows[r].y = (number of run starts in rows [0, r)) - 1.  Returns the number of runs. */
__device__ __forceinline__ uint32_t rows_rank(RowsSmem& S)
{
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    constexpr int WPT = 2048 / kRowsThreads;
    uint32_t cnt[WPT], x = 0;
    #pragma unroll
    for (int j = 0; j < WPT; j++) { cnt[j] = __popc(S.rows[tid * WPT + j].x); x += cnt[j]; }
    uint32_t incl = x;
    #pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) { uint32_t y = __shfl_up_sync(kFull, incl, dd); if (lane >= dd) incl += y; }
    if (lane == 31) S.warpSum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t v = S.warpSum[lane];
        #pragma unroll
        for (int dd = 1; dd < 32; dd <<= 1) { uint32_t y = __shfl_up_sync(kFull, v, dd); if (lane >= dd) v += y; }
        S.warpSum[lane] = v;
        if (lane == 31) S.nRuns = v;
    }
    __syncthreads();
    uint32_t ex = incl - x + (warp ? S.warpSum[warp - 1] : 0);
    #pragma unroll
    for (int j = 0; j < WPT; j++) { S.rows[tid * WPT + j].y = ex - 1u; ex += cnt[j]; }
    return S.nRuns;
}

/* Source addresses of one thread's bytes of a wave: bytes p0 + r*1024 (r < kRowsRpt) of the window at shared address outS.
 * FULL: the whole wave lies inside the window (no bounds checks); otherwise bytes at or past `lim` get `pastEnd`, an
 * address the wave's fetch may read and that never tests as inside the wave.  A source x lies inside the wave being
 * resolved when key(x) >= keyFloor; those are followed through the run table again.  The test is written this way so
 * that "any row inside" is one maximum and one compare.  All addresses are 32-bit shared-window addresses.  Nothing here
 * reads the output window: the run table alone decides where a byte comes from, so a warp resolves wave w+1 while other
 * warps still copy wave w. */
template <bool FULL, class Key>
__device__ __forceinline__ void rows_resolve(uint32_t (&sa)[kRowsRpt], const uint32_t p0, const uint32_t lim,
                                             const uint32_t outS, const uint32_t rowsS, const uint32_t tabS,
                                             const uint32_t pastEnd, const uint32_t le, Key&& key, const uint32_t keyFloor)
{
    static_assert(kRowsThreads == 1024, "rows_resolve assumes 1024 threads (32 rows per wave slice)");
    const uint32_t rowAddr = rowsS + ((p0 >> 5) << 3);
    #pragma unroll
    for (int r = 0; r < kRowsRpt; r++) {
        sa[r] = pastEnd;
        if (FULL || p0 + (uint32_t)(r * 1024) < lim) {
            const uint2 row = lds_u64(rowAddr + (uint32_t)(r * 32 * 8));
            const uint32_t j = row.y + (uint32_t)__popc(row.x & le);
            sa[r] = outS + p0 + (uint32_t)(r * 1024) + lds_u32(tabS + (j << 2));
        }
    }
    uint32_t hi = key(sa[0]);
    #pragma unroll
    for (int r = 1; r < kRowsRpt; r++) hi = max(hi, key(sa[r]));
    while (hi >= keyFloor) {                                   /* sources inside this wave: follow them, all rows of the thread at once */
        hi = 0;
        #pragma unroll
        for (int r = 0; r < kRowsRpt; r++) {
            uint32_t x = sa[r];
            if (key(x) >= keyFloor) {
                const uint32_t q = x - outS;
                const uint2 row = lds_u64(rowsS + ((q >> 5) << 3));
                const uint32_t j = row.y + (uint32_t)__popc(row.x & (0xFFFFFFFFu >> (31u - (q & 31u))));
                x += lds_u32(tabS + (j << 2));
                sa[r] = x;
            }
            hi = max(hi, key(x));
        }
    }
}

/* The waves over the window's bytes [0, len) at shared address outS: thread t writes bytes t, t + 1024, ... of every
 * kWave-byte wave.  resolve(sa, wv) sets the source addresses of the thread's bytes of wave wv (rows_resolve); fetch(x)
 * reads the byte at source address x, also for bytes past the end (they are not stored).  A warp arrives on the wave
 * barrier once its bytes of a wave are written and then resolves the next wave while other warps still copy; `wpar` is
 * the wave barrier's phase parity, carried from window to window.  On return the window is written and visible to the
 * bulk store. */
template <class Resolve, class Fetch>
__device__ __forceinline__ void rows_waves(RowsSmem& S, const uint32_t outS, const int len, uint32_t& wpar,
                                           Resolve&& resolve, Fetch&& fetch)
{
    const int tid = threadIdx.x;
    const int nWaves = (len + kWave - 1) / kWave;
    uint32_t sa[kRowsRpt];
    auto copy = [&](int wv) {
        const uint32_t p0 = (uint32_t)(wv * kWave + tid);
        const uint32_t lim = ((wv + 1) * kWave <= len) ? 0xFFFFFFFFu : (uint32_t)len;
        uint32_t v[kRowsRpt];
        #pragma unroll
        for (int r = 0; r < kRowsRpt; r++) v[r] = fetch(sa[r]);
        #pragma unroll
        for (int r = 0; r < kRowsRpt; r++)
            if (p0 + (uint32_t)(r * kRowsThreads) < lim) sts_u8(outS + p0 + (uint32_t)(r * kRowsThreads), v[r]);
        if (wv == nWaves - 1) fence_proxy_async();         /* generic-proxy writes of `out` before the bulk store reads them */
    };
#ifdef LZ4K_WAVE_BARSYNC
    /* debug build: the same waves with a plain CTA barrier instead of the split mbarrier (no overlap of the resolve with
     * the wait).  compute-sanitizer's racecheck does not model mbarrier arrive / wait as synchronisation; this variant
     * shows that the wave structure itself is hazard free. */
    for (int wv = 0; wv < nWaves; wv++) {
        resolve(sa, wv);
        copy(wv);
        __syncthreads();
    }
#else
    resolve(sa, 0);
    for (int wv = 0; wv < nWaves; wv++) {
        if (wv > 0) { mbar_wait(&S.wbar, wpar); wpar ^= 1; }   /* every warp has copied wave wv-1 */
        copy(wv);
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(&S.wbar);         /* release: this warp's bytes of wave wv are written */
        if (wv + 1 < nWaves) resolve(sa, wv + 1);
    }
    mbar_wait(&S.wbar, wpar);
    wpar ^= 1;
#endif
}

/* the window's bytes [0, len) -> dst: if dst is 16-byte aligned, TMA bulk stores of the 16-byte multiple (thread 0, one
 * commit group) and plain stores of the tail; plain stores throughout otherwise.  FENCE: every thread's plain stores are
 * followed by __threadfence(). */
template <bool FENCE>
__device__ __forceinline__ void rows_store(uint8_t* dst, const uint8_t* out, const int len)
{
    const int tid = threadIdx.x;
    if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
        const uint32_t bulk = (uint32_t)len & ~15u;
        if (tid == 0 && bulk) {
            for (uint32_t o = 0; o < bulk; o += 16384u) tma_store_1d(dst + o, out + o, min(16384u, bulk - o));
            tma_commit();
        }
        if (tid < (len & 15)) { dst[bulk + tid] = out[bulk + tid]; if (FENCE) __threadfence(); }
    } else {
        for (int k = tid; k < len; k += kRowsThreads) dst[k] = out[k];
        if (FENCE) __threadfence();
    }
}

/* PARTIAL: the partial call's blocks (route P1).  The last sequence is rebuilt from its literal start and the return value
 * (rw_parse<true>), so no run starts at or past the return value; only the consumed input prefix is staged, and
 * eligibility is decided on (consumed, target) instead of (input size, capacity). */
template <bool PARTIAL>
__device__ __forceinline__ void expand_rows(const lz4k_decode_args& a, const WsView& w)
{
    extern __shared__ __align__(16) uint8_t smemRaw[];
    RowsSmem& S = *reinterpret_cast<RowsSmem*>(smemRaw);
    const int tid = threadIdx.x;
    const uint32_t le = lanemask_le();
    const uint32_t outA = (uint32_t)offsetof(RowsSmem, out);
    const int zeroDelta0 = (int)offsetof(RowsSmem, zero) - (int)outA;
    const uint32_t sBase = smem_u32(smemRaw);
    const uint32_t outS = sBase + outA, zeroS = sBase + (uint32_t)offsetof(RowsSmem, zero);
    const uint32_t rowsS = sBase + (uint32_t)offsetof(RowsSmem, rows), tabS = sBase + (uint32_t)offsetof(RowsSmem, tab);
    uint32_t parity = 0, wpar = 0;

    /* a block's arguments; n = 0 marks "nothing to do here" (past the end, rejected by the scan, or a block of the
     * generic kernel: input > 65535 bytes, capacity > 64 KB, more than kMaxSeqFast sequences).  The raw loads are
     * issued a block ahead (fetchRaw) and only looked at after the waves (finish), so nobody waits for them. */
    struct Raw { int64_t b, off, dOff; int n, total, cap; uint32_t ns; };
    auto fetchRaw = [&](int64_t b) {
        Raw r;
        r.b = b; r.off = 0; r.dOff = 0; r.n = 0; r.total = 0; r.cap = 0; r.ns = 0;
        if (b < a.nBlocks) {
            r.n = PARTIAL ? (w.used ? (int)w.used[b] : 0) : a.srcSize[b]; r.total = a.outSize[b]; r.ns = w.nSeq[b]; r.off = a.srcOff[b];
            r.cap = a.dstCapArr ? a.dstCapArr[b] : a.dstCap;
            r.dOff = a.dstOff ? a.dstOff[b] : b * a.dstStride;
        }
        return r;
    };
    auto finish = [&](const Raw& r) {
        RowsDesc d;
        d.b = r.b; d.src = nullptr; d.dst = nullptr; d.n = 0; d.total = 0; d.nseq = 0;
        if (r.b < a.nBlocks && r.total > 0 && rows_eligible(r.n, r.cap, r.ns, w.markStride)) {
            d.src = a.src + r.off; d.dst = a.dst + r.dOff;
            d.n = r.n; d.total = r.total; d.nseq = (int)r.ns;
        }
        return d;
    };
    auto issueLoad = [&](const RowsDesc& d) { tma_stage(S.in, d.src, d.n, &S.mbar); };   /* thread 0 */

    if (tid == 0) { mbar_init(&S.mbar, 1); mbar_init(&S.wbar, kRowsThreads / 32); }
    if (tid < 4) reinterpret_cast<uint32_t*>(S.zero)[tid] = 0;
    if (tid == 0) {
        S.desc[0] = finish(fetchRaw(blockIdx.x));
        if (S.desc[0].n > 0) issueLoad(S.desc[0]);
    }
    __syncthreads();
#ifdef LZ4K_PHASE_TIMING
    long long tPhase = clock64();
#endif

    /* static assignment: CTA c takes blocks c, c + grid, c + 2 grid, ... (blocks of a batch cost about the same) */
    for (uint32_t it = 0;; it++) {
        const int64_t b = (int64_t)blockIdx.x + (int64_t)it * gridDim.x;
        if (b >= a.nBlocks) break;
        const RowsDesc d = S.desc[it & 1];
        Raw rawNext;                                           /* the next block's arguments: loads issued now, used after the waves */
        if (tid == 0) rawNext = fetchRaw(b + gridDim.x);
        if (d.n == 0) {                                        /* not a block of this kernel */
            __syncthreads();
            if (tid == 0) { const RowsDesc dn = finish(rawNext); S.desc[(it + 1) & 1] = dn; if (dn.n > 0) issueLoad(dn); }
            __syncthreads();
            continue;
        }
        const int n = d.n, total = d.total, nseq = d.nseq;
        const int head = (int)(reinterpret_cast<uintptr_t>(d.src) & 15);

        for (int k = tid; k < 2048; k += kRowsThreads) S.rows[k] = make_uint2(0u, 0u);
        /* this thread's first marks, fetched while the TMA load is in flight */
        const uint32_t* marks = w.marks + d.b * w.markStride;
        uint32_t mk[kRowsCache];
        #pragma unroll
        for (int i = 0; i < kRowsCache; i++) {
            const int k = tid + i * kRowsThreads;
            mk[i] = (k < nseq) ? marks[k] : 0u;
        }
        __syncthreads();                                   /* rows are zero */
        PHASE_MARK(0);                                     // zeroing + marks
        mbar_wait(&S.mbar, parity);
        parity ^= 1;
        PHASE_MARK(1);                                     // TMA load wait

        /* ---- runs, pass 1: one bit per run start ---- */
        const uint8_t* in = S.in + head;
        const int litDelta = (int)((uint32_t)offsetof(RowsSmem, in) + (uint32_t)head - outA);
        auto parse = [&](int i, int k) { return rw_parse<PARTIAL>(in, i < kRowsCache ? mk[i] : marks[k], k, k + 1 == nseq, total); };
        auto firstRun = [](const RwSeq& s) { return rw_seq_first(s); };
        auto runs = [&](const RwSeq& s, auto f) { rw_seq_runs(s, litDelta, zeroDelta0, f); };
        RwSeq sq[kRowsCache];
        rows_runs_pass<true>(S, sq, 0, nseq, parse, firstRun, runs);
        __syncthreads();
        PHASE_MARK(2);                                     // pass 1

        const uint32_t nRuns = rows_rank(S);
        if (tid == 0) tma_wait_read0();                    /* the previous block's bulk store has finished reading S.out */
        __syncthreads();
        PHASE_MARK(3);                                     // rank
        const bool tooMany = nRuns > (uint32_t)kRowsMaxRuns;   /* (pathological) more runs than the table holds: generic kernel */
        if (tooMany && tid == 0) w.slowList[atomicAdd(&w.hdr->slowCount, 1u)] = (uint32_t)d.b;

        if (!tooMany) {
            /* ---- runs, pass 2: delta of every run at its rank ---- */
            rows_runs_pass<false>(S, sq, 0, nseq, parse, firstRun, runs);
            __syncthreads();
            PHASE_MARK(4);                                     // pass 2

            /* ---- waves: resolve (run table only) | wait for the previous wave | copy | arrive ---- */
            auto resolve = [&](uint32_t (&sa)[kRowsRpt], int wv) {
                const uint32_t p0 = (uint32_t)(wv * kWave + tid), waveS = outS + (uint32_t)(wv * kWave);
                auto key = [](uint32_t x) { return x; };           /* inside the wave: x >= waveS */
                if ((wv + 1) * kWave <= total) rows_resolve<true>(sa, p0, 0xFFFFFFFFu, outS, rowsS, tabS, zeroS, le, key, waveS);
                else rows_resolve<false>(sa, p0, (uint32_t)total, outS, rowsS, tabS, zeroS, le, key, waveS);
            };
            rows_waves(S, outS, total, wpar, resolve, [](uint32_t x) { return lds_u8(x); });
            PHASE_MARK(5);                                     // waves
        }

        /* `in`, `tab` and `rows` are dead: start the next block's load before anything else */
        if (tid == 0) {
            const RowsDesc dn = finish(rawNext);
            S.desc[(it + 1) & 1] = dn;
            if (dn.n > 0) issueLoad(dn);
        }
        /* ---- store: smem -> HBM ---- */
        if (!tooMany) rows_store<false>(d.dst, S.out, total);
        __syncthreads();                                   /* desc[(it+1)&1] is visible; `out` tail reads are done */
        PHASE_MARK(6);                                     // store issue
    }
    if (tid == 0) tma_wait_all0();
}

__global__ void __launch_bounds__(kRowsThreads, 1) lz4_expand_rows_kernel(lz4k_decode_args a, WsView w) { expand_rows<false>(a, w); }
__global__ void __launch_bounds__(kRowsThreads, 1) lz4_expand_rows_partial_kernel(lz4k_decode_args a, WsView w) { expand_rows<true>(a, w); }

/* =============================================================================================
 * expand (tiles): blocks ABOVE 64 KB (lz4frame's 256 KB .. 4 MB blocks), one CTA per 60 KB OUTPUT TILE
 *
 * The rows formulation applied to a window of a big block.  The scan (lz4_scan_par_kernel) leaves wide marks
 * {token position, match start} per sequence and lz4_tile_index_kernel the first sequence of every tile; a unit of work is
 * (block b, tile t) = output bytes [t * kTile, (t + 1) * kTile) of block b.  Differences to lz4_expand_rows_kernel:
 *   - the sequences that overlap the tile are parsed from GLOBAL memory (their tokens may lie megabytes apart from the
 *     tile's literals) and their runs are clipped to the tile (rw_tile_runs);
 *   - the compressed block is not staged: a literal run's delta maps into a virtual range [kLitBase, ...) that means
 *     "byte x - kLitBase of the compressed block", read from global memory through the read-only cache;
 *   - a match source below the tile start lies in an EARLIER tile of the same block: it is read from the destination
 *     in global memory (L2).  Tile t therefore waits, after its passes 1-2 and before its waves, for tile t - 1's flag,
 *     which that tile's CTA sets once its bulk store has completed.  Units are numbered tile-major (all blocks' tile 0,
 *     then tile 1, ...) and taken in ascending order by a grid of resident CTAs, so a tile's predecessor was started
 *     earlier: no deadlock; with at least one block per SM in the batch the wait is over before it begins.
 *   - a tile with more runs than the table holds hands its block to the generic kernel (which rewrites the whole block).
 * ============================================================================================= */
constexpr uint32_t kLitBase = 1u << 28;                   /* virtual window addresses >= kLitBase: compressed byte (address - kLitBase) */
constexpr uint32_t kZeroV = kLitBase + (1u << 27);         /* the always-zero cell (offset 0, lz4.c:2407) */

__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p)
{
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v)
{
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

__global__ void __launch_bounds__(kRowsThreads, 1) lz4_expand_tiles_kernel(lz4k_decode_args a, WsView w)
{
    extern __shared__ __align__(16) uint8_t smemRaw[];
    RowsSmem& S = *reinterpret_cast<RowsSmem*>(smemRaw);
    const int tid = threadIdx.x;
    const uint32_t le = lanemask_le();
    const uint32_t sBase = smem_u32(smemRaw);
    const uint32_t outS = sBase + (uint32_t)offsetof(RowsSmem, out);
    const uint32_t rowsS = sBase + (uint32_t)offsetof(RowsSmem, rows), tabS = sBase + (uint32_t)offsetof(RowsSmem, tab);
    const uint32_t tilesMax = w.tilesMax;
    uint32_t wpar = 0;
    uint32_t* pendFlag = nullptr;                               /* thread 0: flag of the unit whose bulk store is in flight */
    auto publishPending = [&]() {                               /* thread 0 */
        tma_wait_all0();                                        /* the store has completed (not only finished reading `out`) */
        if (pendFlag) { __threadfence(); st_release_gpu(pendFlag, 1u); pendFlag = nullptr; }
    };
    if (tid == 0) mbar_init(&S.wbar, kRowsThreads / 32);
    __syncthreads();

    const int64_t units = a.nBlocks * (int64_t)tilesMax;
    for (int64_t u = blockIdx.x; u < units; u += gridDim.x) {
        const int64_t b = u % a.nBlocks;
        const uint32_t t = (uint32_t)(u / a.nBlocks);
        const int total = a.outSize[b];
        const uint32_t nseq = w.nSeq[b];
        uint32_t* flags = w.tileFlag + (size_t)b * (tilesMax + 1);
        if (!(total > 0 && nseq > 0 && tiles_eligible(w, nseq) && t < tiles_of(total))) {     /* (the same for every thread) */
            if (tid == 0 && pendFlag) publishPending();
            continue;
        }
        const uint8_t* src = a.src + a.srcOff[b];
        uint8_t* dstB = a.dst + (a.dstOff ? a.dstOff[b] : b * a.dstStride);
        const uint32_t* marks = w.marks + (size_t)b * w.markStride;
        const uint32_t* first = w.tileFirst + (size_t)b * (tilesMax + 1);
        const int os = (int)(t * (uint32_t)kTile), oe = min(os + kTile, total), len = oe - os;
        const uint32_t f0 = first[t], f1 = first[t + 1];
        const int k0 = f0 ? (int)f0 - 1 : 0, k1 = (int)min(f1 + 1u, nseq);
        const uint32_t litBase = kLitBase - outS + (uint32_t)os;
        const int zeroDelta0 = (int)(kZeroV - outS + (uint32_t)os);
        auto parse = [&](int, int k) { return rw_parse_wide(src, marks[2 * (size_t)k], marks[2 * (size_t)k + 1], k + 1 == (int)nseq); };
        auto firstRun = [&](const RwSeq& s) { return rw_tile_first(s, os, oe); };
        auto runs = [&](const RwSeq& s, auto f) { rw_tile_runs(s, os, oe, litBase, zeroDelta0, f); };

        for (int k = tid; k < 2048; k += kRowsThreads) S.rows[k] = make_uint2(0u, 0u);
        __syncthreads();
        /* ---- runs, pass 1 (a thread's first sequences stay in registers for pass 2: parsing reads global memory) ---- */
        RwSeq sq[kRowsCache];
        rows_runs_pass<true>(S, sq, k0, k1, parse, firstRun, runs);
        __syncthreads();
        const uint32_t nRuns = rows_rank(S);
        if (tid == 0) publishPending();                       /* the previous unit's store is complete: its flag goes up, `out` is free */
        __syncthreads();
        if (nRuns > (uint32_t)kRowsMaxRuns) {                  /* (pathological) the generic kernel redoes the whole block */
            if (tid == 0) {
                if (atomicExch(&flags[tilesMax], 1u) == 0u) w.slowList[atomicAdd(&w.hdr->slowCount, 1u)] = (uint32_t)b;
                __threadfence();
                st_release_gpu(&flags[t], 1u);                 /* whoever waits for this tile may go on: its bytes will be rewritten */
            }
            __syncthreads();
            continue;
        }
        /* ---- runs, pass 2 ---- */
        rows_runs_pass<false>(S, sq, k0, k1, parse, firstRun, runs);
        __syncthreads();
        /* ---- the tile before this one must be in global memory ---- */
        if (t > 0) {
            if (tid == 0) { while (ld_acquire_gpu(&flags[t - 1]) == 0u) __nanosleep(200); }
            __syncthreads();
        }
        /* ---- waves: a source x is a compressed byte (x >= kLitBase), a byte of this tile, or one of an earlier tile ---- */
        auto resolve = [&](uint32_t (&sa)[kRowsRpt], int wv) {
            const uint32_t p0 = (uint32_t)(wv * kWave + tid), waveE = outS + (uint32_t)((wv + 1) * kWave);
            /* inside the wave: (x - waveS) < kWave, i.e. x - waveE >= -kWave; not x >= waveS, since the literal sources
             * lie above the window.  Bytes past the tile get outS + 65536: never inside a wave, and readable by the fetch. */
            auto key = [waveE](uint32_t x) { return x - waveE; };
            if ((wv + 1) * kWave <= len) rows_resolve<true>(sa, p0, 0xFFFFFFFFu, outS, rowsS, tabS, outS + 65536u, le, key, 0u - (uint32_t)kWave);
            else rows_resolve<false>(sa, p0, (uint32_t)len, outS, rowsS, tabS, outS + 65536u, le, key, 0u - (uint32_t)kWave);
        };
        rows_waves(S, outS, len, wpar, resolve, [&](uint32_t x) {
            if (x >= kLitBase) return (x == kZeroV) ? 0u : (uint32_t)__ldg(src + (x - kLitBase));
            if (x >= outS) return lds_u8(x);
            return (uint32_t)__ldcg(dstB + (os - (int)(outS - x)));
        });
        /* ---- store: smem -> HBM; the plain stores are fenced before the flag goes up ---- */
        rows_store<true>(dstB + os, S.out, len);
        if (tid == 0) pendFlag = &flags[t];
        __syncthreads();                                      /* `out` tail reads are done; direct stores are fenced */
    }
    if (tid == 0) publishPending();
}

/* ---- ceiling of the rows kernel's skeleton (developer tool; bench.py --ceiling) ----
 * Same persistent structure -- one CTA of 1024 threads per SM, TMA bulk load of the compressed block into `in`, TMA bulk
 * store of 64 KB from `out` -- with the decode replaced by
 *   mode 0: nothing (load b+1 and store b are both in flight): what HBM and the TMA path give this structure;
 *   mode 1: one LDS.U8 + STS.U8 per output byte, one byte per thread, 4096-byte waves with a CTA barrier each: the floor
 *           of moving every byte through shared memory at byte granularity, without any address resolution.
 * The bytes written are meaningless; the timing is the point. */
__global__ void __launch_bounds__(kRowsThreads, 1) lz4_ceiling_kernel(lz4k_decode_args a, int mode)
{
    extern __shared__ __align__(16) uint8_t smemRaw[];
    RowsSmem& S = *reinterpret_cast<RowsSmem*>(smemRaw);
    const int tid = threadIdx.x;
    const uint32_t sBase = smem_u32(smemRaw);
    const uint32_t outS = sBase + (uint32_t)offsetof(RowsSmem, out), inS = sBase + (uint32_t)offsetof(RowsSmem, in);
    uint32_t parity = 0;
    auto issueLoad = [&](int64_t b) { tma_stage(S.in, a.src + a.srcOff[b], a.srcSize[b], &S.mbar); };
    if (tid == 0) { mbar_init(&S.mbar, 1); }
    __syncthreads();
    if (tid == 0 && blockIdx.x < a.nBlocks) issueLoad(blockIdx.x);
    for (int64_t b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
        mbar_wait(&S.mbar, parity);
        parity ^= 1;
        if (mode >= 1) {
            if (tid == 0) tma_wait_read0();                    /* the previous store has finished reading `out` */
            __syncthreads();
            for (int wv = 0; wv < 65536 / kWave; wv++) {
                uint32_t v[kRowsRpt];
                #pragma unroll
                for (int r = 0; r < kRowsRpt; r++) v[r] = lds_u8(inS + (uint32_t)((wv * kWave + r * kRowsThreads + tid) & 0x7FFF));
                #pragma unroll
                for (int r = 0; r < kRowsRpt; r++) sts_u8(outS + (uint32_t)(wv * kWave + r * kRowsThreads + tid), v[r]);
                __syncthreads();
            }
            fence_proxy_async();
            __syncthreads();
        }
        if (tid == 0) {
            if (b + gridDim.x < a.nBlocks) issueLoad(b + gridDim.x);
            uint8_t* dst = a.dst + b * a.dstStride;
            for (uint32_t o = 0; o < 65536u; o += 16384u) tma_store_1d(dst + o, S.out + o, 16384u);
            tma_commit();
        }
        if (mode >= 1) __syncthreads();
    }
    if (tid == 0) tma_wait_all0();
}

/* =============================================================================================
 * encode: one warp per block, byte-identical replay of LZ4_compress_generic_validated
 * ============================================================================================= */

template <bool SMALL> struct Table;
template <> struct Table<true> {       // byU16, 13-bit 4-byte hash (lz4.c:779-780)
    uint16_t* t;
    __device__ __forceinline__ uint32_t hash(const uint8_t* p) const { return (ld32u<true>(p) * 2654435761u) >> 19; }
    __device__ __forceinline__ uint32_t hashv(const uint8_t* p, uint32_t& v32) const { v32 = ld32u<true>(p); return (v32 * 2654435761u) >> 19; }
    __device__ __forceinline__ uint32_t get(uint32_t h) const { return t[h]; }
    __device__ __forceinline__ void put(uint32_t h, uint32_t pos) const { t[h] = (uint16_t)pos; }
};
template <> struct Table<false> {      // byU32, 12-bit 5-byte hash (lz4.c:785-791,799)
    uint32_t* t;
    __device__ __forceinline__ static uint32_t h5(uint64_t v) { return (uint32_t)(((v << 24) * 889523592379ull) >> 52); }
    __device__ __forceinline__ uint32_t hash(const uint8_t* p) const { return h5(ld40u(p)); }
    __device__ __forceinline__ uint32_t hashv(const uint8_t* p, uint32_t& v32) const { uint64_t v = ld40u(p); v32 = (uint32_t)v; return h5(v); }
    __device__ __forceinline__ uint32_t get(uint32_t h) const { return t[h]; }
    __device__ __forceinline__ void put(uint32_t h, uint32_t pos) const { t[h] = pos; }
};

/* sum_{t<m} (accel + (t >> 6)): distance covered by m search steps after the first one,
 * from step = (searchMatchNb++ >> LZ4_skipTrigger) with searchMatchNb = accel << 6 (lz4.c:1044-1053) */
__device__ __forceinline__ uint32_t skip_distance(uint32_t m, uint32_t accel)
{
    uint32_t q = m >> kSkipTrigger, r = m & 63u;
    return accel * m + 32u * q * (q - 1u) + q * r;
}

/* run-length extension bytes: `len` -> 255,255,...,rem  (lz4.c:1123-1128) written by the warp */
__device__ __forceinline__ uint32_t emit_runlength(uint8_t* dst, uint32_t op, uint32_t len, int lane)
{
    uint32_t full = len / 255u;
    for (uint32_t k = lane; k < full; k += 32) dst[op + k] = 255;
    if (lane == 0) dst[op + full] = (uint8_t)(len - full * 255u);
    return op + full + 1;
}

/* The reference's output directive (lz4.c:930-1338) is FILL or not: without FILL, dstCap decides between notLimited and
 * limitedOutput at run time (LZ4_compress_fast_extState, lz4.c:1388); with FILL (fillOutput, LZ4_compress_destSize,
 * lz4.c:1489-1494) the parse stops where dstCap is reached and *consumed receives the input bytes the output holds. */
template <bool SMALL, bool FILL = false>
__device__ int encode_block(const uint8_t* __restrict__ src, const int n, uint8_t* __restrict__ dst,
                            const int dstCap, const uint32_t accel, void* tableMem, const int lane,
                            uint32_t* consumed = nullptr)
{
    Table<SMALL> T;
    T.t = reinterpret_cast<decltype(T.t)>(tableMem);
    if (FILL && dstCap < 1) return 0;                         // lz4.c:985
    const int bound = n + n / 255 + 16;
    const bool limited = !FILL && !(dstCap >= bound);
    const int64_t olimit = dstCap;
    const uint32_t mflimit1 = (uint32_t)n - kMfLimit + 1;     // lz4.c:963
    const uint32_t matchlimit = (uint32_t)n - kLastLiterals;  // lz4.c:964
    uint32_t ip = 0, anchor = 0, op = 0, cand = 0;

    {   // zeroed table, lz4.c:1558
        uint4* z = reinterpret_cast<uint4*>(tableMem);
        for (int k = lane; k < 1024; k += 32) z[k] = make_uint4(0, 0, 0, 0);
    }
    __syncwarp();

    if (n < kMinLength) goto tail;                            // lz4.c:1002

    if (lane == 0) T.put(T.hash(src), 0);                     // lz4.c:1005-1010
    __syncwarp();
    ip = 1;

    for (;;) {
        /* ---- search: lanes probe the next 32 positions of the reference's visiting order ---- */
        {
            uint32_t baseJ = 0;
            bool found = false;
            for (;;) {
                const uint32_t j = baseJ + lane;
                const uint32_t p = ip + (j ? 1u + skip_distance(j - 1, accel) : 0u);
                const uint32_t pnext = ip + 1u + skip_distance(j, accel);
                const bool term = pnext > mflimit1;           // lz4.c:1055 fires at this visit
                uint32_t v32 = 0, h = 0x80000000u | lane, old = 0;
                if (!term) { h = T.hashv(src + p, v32); old = T.get(h); }
                __syncwarp();                                 // every lane has read the table before any lane writes it (below)
                const unsigned peers = __match_any_sync(kFull, h);
                const unsigned lower = peers & ((1u << lane) - 1u);
                const int fromLane = lower ? (31 - __clz(lower)) : lane;
                const uint32_t pPrev = __shfl_sync(kFull, p, fromLane);
                const uint32_t c = lower ? pPrev : old;       // table value this visit would read
                bool hit = false;
                if (!term) {
                    if (SMALL || c + kMaxDistance >= p) hit = (ld32u<true>(src + c) == v32);   // lz4.c:1090-1096
                }
                const unsigned termMask = __ballot_sync(kFull, term);
                const unsigned hitMask = __ballot_sync(kFull, hit);
                const int firstTerm = termMask ? (__ffs(termMask) - 1) : 32;
                const int firstHit = hitMask ? (__ffs(hitMask) - 1) : 32;
                if (firstHit < firstTerm) {
                    /* visits 0..firstHit happened: each stored its position (lz4.c:1085); for equal
                     * hashes the latest visit wins */
                    const unsigned upto = (firstHit == 31) ? kFull : ((2u << firstHit) - 1u);
                    const unsigned mine = peers & upto;
                    if (lane <= firstHit && (mine >> lane) == 1u) T.put(h, p);
                    ip = __shfl_sync(kFull, p, firstHit);
                    cand = __shfl_sync(kFull, c, firstHit);
                    found = true;
                    __syncwarp();
                    break;
                }
                if (firstTerm < 32) break;                    // goto _last_literals
                if ((peers >> lane) == 1u) T.put(h, p);
                __syncwarp();
                baseJ += 32;
            }
            if (!found) goto tail;
        }

        /* ---- backward extension (lz4.c:1107-1109) ---- */
        for (;;) {
            const uint32_t room = min(ip - anchor, cand);
            const uint32_t k = lane + 1;
            const bool eq = (k <= room) && (ldb<true>(src + ip - k) == ldb<true>(src + cand - k));
            const unsigned m = __ballot_sync(kFull, eq);
            const uint32_t run = (m == kFull) ? 32u : (uint32_t)(__ffs(~m) - 1);
            ip -= run; cand -= run;
            if (run < 32) break;
        }

        {
            uint32_t lit = ip - anchor;
            bool haveLiterals = true;
            for (;;) {   /* the _next_match chain, lz4.c:1138-1294 */
                /* match length first (the token needs it): LZ4_count, lz4.c:1182 */
                uint32_t mcode = 0;
                {
                    const uint8_t* pa = src + ip + kMinMatch;
                    const uint8_t* pb = src + cand + kMinMatch;
                    const uint32_t lim = matchlimit - (ip + kMinMatch);    // bytes comparable
                    for (uint32_t base = 0;; base += 32) {
                        const uint32_t k = base + lane;
                        const bool eq = (k < lim) && (ldb<true>(pa + k) == ldb<true>(pb + k));
                        const unsigned m = __ballot_sync(kFull, eq);
                        if (m != kFull) { mcode = base + (uint32_t)(__ffs(~m) - 1); break; }
                    }
                }
                const uint32_t tokenPos = op;
                uint32_t o = op + 1;
                if (haveLiterals) {
                    /* lz4.c:1114-1117 */
                    if (limited && (int64_t)o + lit + (2 + 1 + kLastLiterals) + lit / 255 > olimit) return 0;
                    /* lz4.c:1118-1122: the token is dropped (op stays at tokenPos) */
                    if (FILL && (int64_t)o + (lit + 240) / 255 + lit + 2 + 1 + kMfLimit - kMinMatch > olimit) goto tail;
                    if (lit >= 15) o = emit_runlength(dst, o, lit - 15, lane);
                    for (uint32_t k = lane; k < lit; k += 32) dst[o + k] = (uint8_t)ldb<true>(src + anchor + k);
                    o += lit;
                }
                /* lz4.c:1147-1152: rewind to the token */
                if (FILL && (int64_t)o + 2 + 1 + kMfLimit - kMinMatch > olimit) goto tail;
                /* offset, lz4.c:1162 */
                const uint32_t off = ip - cand;
                if (lane == 0) { dst[o] = (uint8_t)off; dst[o + 1] = (uint8_t)(off >> 8); }
                o += 2;
                /* lz4.c:1187-1211 */
                if (limited && (int64_t)o + (1 + kLastLiterals) + (mcode + 240) / 255 > olimit) return 0;
                bool reduced = false;
                if (FILL && (int64_t)o + (1 + kLastLiterals) + (mcode + 240) / 255 > olimit) {
                    /* lz4.c:1190-1194: the match is cut to what fits before the last 1 + LASTLITERALS bytes */
                    mcode = 14u + ((uint32_t)(olimit - o) - 1u - kLastLiterals) * 255u;
                    reduced = true;
                }
                if (lane == 0) {
                    const uint32_t lt = haveLiterals ? min(lit, 15u) : 0u;
                    dst[tokenPos] = (uint8_t)((lt << 4) | min(mcode, 15u));
                }
                if (mcode >= 15) o = emit_runlength(dst, o, mcode - 15, lane);   // lz4.c:1213-1223
                op = o;

                ip += mcode + kMinMatch;
                anchor = ip;
                /* After a reduced match exactly 1 + LASTLITERALS bytes of room are left (op == olimit - 6), so every way on
                 * from here reaches _last_literals with this anchor and this op, writing nothing before it: the end test
                 * (lz4.c:1233) goes there directly, a re-test hit fails the _next_match check (op + 11 > olimit), and a
                 * match found by the search fails the literal check (op + 1 + 11 > olimit).  Which positions the table
                 * holds cannot change that, so the clearing of lz4.c:1195-1207 (it only matters to a later block that
                 * reuses the table; every block here starts from a zeroed one) is skipped and the parse ends now. */
                if (FILL && reduced) goto tail;
                if (ip >= mflimit1) goto tail;                         // lz4.c:1233

                if (lane == 0) T.put(T.hash(src + ip - 2), ip - 2);    // lz4.c:1236-1242
                __syncwarp();
                {   /* immediate re-test at ip, lz4.c:1255-1294 */
                    uint32_t v32;
                    const uint32_t h = T.hashv(src + ip, v32);
                    cand = T.get(h);
                    __syncwarp();
                    if (lane == 0) T.put(h, ip);
                    __syncwarp();
                    if ((SMALL || cand + kMaxDistance >= ip) && ld32u<true>(src + cand) == v32) {
                        haveLiterals = false; lit = 0;
                        continue;
                    }
                }
                break;
            }
        }
        ip++;                                                          // lz4.c:1298
    }

tail:   /* lz4.c:1302-1329 */
    {
        uint32_t last = (uint32_t)n - anchor;
        if (limited && (int64_t)op + last + 1 + (last + 255 - 15) / 255 > olimit) return 0;
        if (FILL && (int64_t)op + last + 1 + (last + 255 - 15) / 255 > olimit) {
            last = (uint32_t)(olimit - op) - 1u;              // lz4.c:1307-1311: as many literals as fit
            last -= (last + 256 - 15) / 256;
        }
        uint32_t o = op + 1;
        if (lane == 0) dst[op] = (uint8_t)(min(last, 15u) << 4);
        if (last >= 15) o = emit_runlength(dst, o, last - 15, lane);
        for (uint32_t k = lane; k < last; k += 32) dst[o + k] = (uint8_t)ldb<true>(src + anchor + k);
        if (FILL) *consumed = anchor + last;                   // lz4.c:1327, 1332
        return (int)(o + last);
    }
}

constexpr int kEncodeTableBytes = 16384;    // LZ4_HASHTABLESIZE, lz4.h:157-172 (LZ4_MEMORY_USAGE 14)

__global__ void __launch_bounds__(32) lz4_encode_kernel(lz4k_encode_args a)
{
    extern __shared__ uint4 tableMem[];
    const int lane = threadIdx.x;
    uint32_t accel = a.acceleration < 1 ? 1u : (a.acceleration > kAccelMax ? (uint32_t)kAccelMax : (uint32_t)a.acceleration);  // lz4.c:1386-1387
    for (int64_t b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
        const uint8_t* src = a.src + b * a.srcStride;
        uint8_t* dst = a.dst + b * a.dstStride;
        const int n = a.srcSizeArr ? a.srcSizeArr[b] : a.srcSize;
        if (n < a.minSize || n > a.maxSize) continue;                   // another launch's block
        int r;
        if ((uint32_t)n > kMaxInput) {                                  // lz4.c:1360
            r = 0;
        } else if (n == 0) {                                            // lz4.c:1361-1371
            const bool limited = !(a.dstCap >= 16);
            if (limited && a.dstCap <= 0) r = 0;
            else { if (lane == 0) dst[0] = 0; r = 1; }
        } else if (n < kSmallLimit) {                                   // lz4.c:1389
            r = encode_block<true>(src, n, dst, a.dstCap, accel, tableMem, lane);
        } else {
            r = encode_block<false>(src, n, dst, a.dstCap, accel, tableMem, lane);
        }
        if (lane == 0) a.outSize[b] = r;
        __syncwarp();
    }
}

/* the fill parse takes the acceleration unclamped (lz4.c:1490-1493); above this value `acceleration << 6` overflows int
 * (lz4.c:1044), and below 1 the reference asserts: both are brought into 1 .. kFillAccelMax */
constexpr int kFillAccelMax = (1 << 25) - 1;

/* LZ4_compress_destSize_extState per block (lz4.c:1481-1503), same warp, table and grid as lz4_encode_kernel: a target of
 * at least LZ4_compressBound(n) is LZ4_compress_fast_extState (clamped acceleration, notLimited); below it the fill parse.
 * srcConsumed[b] is what the reference leaves in *srcSizePtr: the consumed input, or n where it does not write it. */
__global__ void __launch_bounds__(32) lz4_encode_dest_kernel(lz4k_encode_args a, int32_t* srcConsumed)
{
    extern __shared__ uint4 tableMem[];
    const int lane = threadIdx.x;
    const int target = a.dstCap;
    const uint32_t accel = a.acceleration < 1 ? 1u : (a.acceleration > kAccelMax ? (uint32_t)kAccelMax : (uint32_t)a.acceleration);  // lz4.c:1386-1387
    const uint32_t accelFill = a.acceleration < 1 ? 1u : (a.acceleration > kFillAccelMax ? (uint32_t)kFillAccelMax : (uint32_t)a.acceleration);
    for (int64_t b = blockIdx.x; b < a.nBlocks; b += gridDim.x) {
        const uint8_t* src = a.src + b * a.srcStride;
        uint8_t* dst = a.dst + b * a.dstStride;
        const int n = a.srcSizeArr ? a.srcSizeArr[b] : a.srcSize;
        if (n < a.minSize || n > a.maxSize) continue;                   // another launch's block
        const int bound = (uint32_t)n > kMaxInput ? 0 : n + n / 255 + 16;   // LZ4_compressBound
        uint32_t consumed = (uint32_t)n;
        int r;
        if ((uint32_t)n > kMaxInput) {                                  // lz4.c:1360, on both routes
            r = 0;
        } else if (target >= bound) {                                   // lz4.c:1486-1487: notLimited, n > 0 (bound >= 16)
            if (n == 0) { if (lane == 0) dst[0] = 0; r = 1; }             // lz4.c:1361-1371
            else if (n < kSmallLimit) r = encode_block<true>(src, n, dst, target, accel, tableMem, lane);
            else r = encode_block<false>(src, n, dst, target, accel, tableMem, lane);
        } else if (n == 0) {                                            // lz4.c:1361-1371 with fillOutput
            if (target <= 0) r = 0;
            else { if (lane == 0) dst[0] = 0; r = 1; consumed = 0; }
        } else if (n < kSmallLimit) {                                   // lz4.c:1489-1490
            r = encode_block<true, true>(src, n, dst, target, accelFill, tableMem, lane, &consumed);
        } else {                                                        // lz4.c:1492-1493
            r = encode_block<false, true>(src, n, dst, target, accelFill, tableMem, lane, &consumed);
        }
        if (lane == 0) { a.outSize[b] = r; srcConsumed[b] = (int32_t)consumed; }
        __syncwarp();
    }
}

#include "lz4_encode_par.cuh"
#include "lz4_hc_core.h"
#include "lz4_encode_hc.cuh"

/* =============================================================================================
 * pack: exclusive scan of sizes (+ optional 4-byte headers) and gather into a contiguous stream
 * With a FrameRule the blocks become the body of an LZ4 frame (LZ4F_makeBlock, lz4frame.c:883-908): a block whose
 * compression did not gain (size 0 = did not fit size-1, or >= its source size) is stored raw -- payload = the
 * source bytes, bit 31 of the LE32 block header set.
 * ============================================================================================= */
struct FrameRule { const uint8_t* raw; int64_t rawStride; int32_t blockSize, lastSize; };     /* raw == nullptr: plain pack */

__device__ __forceinline__ int pack_payload(const FrameRule& fr, const int32_t* sizes, int64_t b, int64_t n, bool& isRaw)
{
    const int c = sizes[b];
    isRaw = false;
    if (!fr.raw) return c > 0 ? c : 0;
    const int sz = (b == n - 1 && fr.lastSize > 0) ? fr.lastSize : fr.blockSize;
    isRaw = (c <= 0 || c >= sz);                                /* lz4frame.c:896-899 */
    return isRaw ? sz : c;
}

__global__ void __launch_bounds__(1024) lz4_pack_scan_kernel(const int32_t* __restrict__ sizes, int64_t n,
                                                             int64_t* __restrict__ outOff, int headerBytes, FrameRule fr)
{
    __shared__ int64_t warpSums[32];
    __shared__ int64_t carry;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int64_t base = 0; base < n; base += 1024) {
        int64_t i = base + threadIdx.x;
        int64_t v = 0;
        if (i < n) { bool isRaw; v = pack_payload(fr, sizes, i, n, isRaw) + headerBytes; }
        int64_t x = v;
        for (int d = 1; d < 32; d <<= 1) { int64_t y = __shfl_up_sync(kFull, x, d); if (lane >= d) x += y; }
        if (lane == 31) warpSums[wid] = x;
        __syncthreads();
        if (wid == 0) {
            int64_t w = warpSums[lane];
            for (int d = 1; d < 32; d <<= 1) { int64_t y = __shfl_up_sync(kFull, w, d); if (lane >= d) w += y; }
            warpSums[lane] = w;
        }
        __syncthreads();
        int64_t prefix = carry + (wid ? warpSums[wid - 1] : 0) + x - v;
        if (i < n) outOff[i] = prefix;
        __syncthreads();
        if (threadIdx.x == 1023) carry = prefix + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) outOff[n] = carry;
}

__global__ void __launch_bounds__(256) lz4_pack_gather_kernel(const uint8_t* __restrict__ slots, int64_t slotStride,
                                                              const int32_t* __restrict__ sizes, int64_t n,
                                                              uint8_t* __restrict__ packed, const int64_t* __restrict__ outOff,
                                                              int headerBytes, FrameRule fr)
{
    for (int64_t b = blockIdx.x; b < n; b += gridDim.x) {
        bool isRaw;
        const int s = pack_payload(fr, sizes, b, n, isRaw);
        const uint8_t* from = isRaw ? fr.raw + b * fr.rawStride : slots + b * slotStride;
        uint8_t* to = packed + outOff[b];
        const uint32_t hw = (uint32_t)s | (isRaw ? 0x80000000u : 0u);
        if (headerBytes == 4 && threadIdx.x < 4) to[threadIdx.x] = (uint8_t)(hw >> (8 * threadIdx.x));   // lz4frame.c:896-907 LE32
        to += headerBytes;
        /* destination-aligned 16-byte stores, source read through aligned words */
        const uintptr_t ta = reinterpret_cast<uintptr_t>(to);
        int head = (int)((16 - (ta & 15)) & 15);
        if (head > s) head = s;
        for (int k = threadIdx.x; k < head; k += blockDim.x) to[k] = from[k];
        const int body = (s - head) >> 4;
        const uint8_t* fb = from + head;
        uint4* tb = reinterpret_cast<uint4*>(to + head);
        const uintptr_t fa = reinterpret_cast<uintptr_t>(fb);
        const uint32_t sh = (uint32_t)(fa & 3) * 8;
        const uint32_t* fw = reinterpret_cast<const uint32_t*>(fa & ~uintptr_t(3));
        for (int k = threadIdx.x; k < body; k += blockDim.x) {
            const uint32_t* w = fw + 4 * k;
            uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2), w3 = __ldg(w + 3);
            uint32_t w4 = sh ? __ldg(w + 4) : 0u;
            uint4 v;
            v.x = __funnelshift_r(w0, w1, sh); v.y = __funnelshift_r(w1, w2, sh);
            v.z = __funnelshift_r(w2, w3, sh); v.w = __funnelshift_r(w3, w4, sh);
            tb[k] = v;
        }
        for (int k = head + (body << 4) + threadIdx.x; k < s; k += blockDim.x) to[k] = from[k];
    }
}

}  // namespace

/* =============================================================================================
 * extern "C" launchers
 * ============================================================================================= */
static int device_sms()
{
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return sms;
}

static int launch_pack(const uint8_t* slots, int64_t slotStride, const int32_t* sizes, int64_t nBlocks, uint8_t* packed,
                       int64_t* outOff, int headerBytes, FrameRule fr, cudaStream_t s)
{
    lz4_pack_scan_kernel<<<1, 1024, 0, s>>>(sizes, nBlocks, outOff, headerBytes, fr);
    g_launches++;
    if (nBlocks > 0) {
        const int64_t cap = (int64_t)device_sms() * 16;
        int64_t grid = nBlocks < cap ? nBlocks : cap;
        lz4_pack_gather_kernel<<<(unsigned)grid, 256, 0, s>>>(slots, slotStride, sizes, nBlocks, packed, outOff, headerBytes, fr);
        g_launches++;
    }
    return (int)cudaGetLastError();
}

extern "C" {

uint64_t lz4k_launch_count(void) { return g_launches; }

/* debug: read and reset the phase-cycle counters (all zero unless built with -DLZ4K_PHASE_TIMING) */
int lz4k_debug_phase_cycles(unsigned long long* out8)   /* out8: 12 values (8 phase cycles + 4 loop statistics) */
{
    unsigned long long z[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    cudaError_t e = cudaMemcpyFromSymbol(out8, g_phaseCycles, sizeof(z));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_phaseCycles, z, sizeof(z));
    if (e == cudaSuccess) e = cudaMemcpyFromSymbol(out8 + 8, g_loopStats, 4 * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_loopStats, z, 4 * sizeof(unsigned long long));
    return (int)e;
}

size_t lz4k_decode_workspace_bytes(int64_t nBlocks, int perBlockCaps, int32_t dstCap, size_t workspaceBytes)
{
    return nBlocks < 0 ? 0 : plan_decode(nBlocks, perBlockCaps != 0, dstCap, workspaceBytes, kDecodeFull).bytes;
}

/* once per process (every device of a process runs the same kernels): the decode kernels' opt-in to the large dynamic
 * shared memory, the SMs the persistent kernels use, and the developer A/B switch of the scan */
static int g_decodeSms = 0, g_scanImpl = -1;
static cudaError_t decode_setup()
{
    if (g_decodeSms) return cudaSuccess;
    const int rowsSmem = (int)sizeof(RowsSmem);
    cudaError_t e = cudaFuncSetAttribute(lz4_expand_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, rowsSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(lz4_expand_rows_partial_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, rowsSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(lz4_expand_tiles_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, rowsSmem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(lz4_scan_par_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(ScanParSmem));
    if (e != cudaSuccess) return e;
    const char* env = getenv("LZ4K_SCAN_IMPL");                       /* "thread" | "par" | "split" */
    g_scanImpl = env ? (env[0] == 'p' ? kScanPar : env[0] == 's' ? kScanSplit : kScanThread) : -1;
    /* LZ4B200_RESERVE_SMS = k: the persistent expand kernels leave k SMs alone, for a communication kernel that runs
     * concurrently (N > 1: NCCL's send/recv of the previous chunk; bench.py --reserve-sms) */
    const int v = device_sms();
    const char* rs = getenv("LZ4B200_RESERVE_SMS");
    const int reserve = rs ? atoi(rs) : 0;
    g_decodeSms = (reserve > 0 && reserve < v) ? v - reserve : v;
    return cudaSuccess;
}

/* The full call: thread, split or parallel scan (plan_decode), then the rows or (wide batch) the tiles kernel, then the
 * generic kernel.  The partial call: one-thread partial scan, then route P1 (rows kernel, targets <= 64 KB whose consumed
 * prefix, sequences and runs fit it) and P2 (generic kernel, everything else); targets above 64 KB take the generic
 * kernel (correct, not tuned). */
int lz4k_launch_decode(const lz4k_decode_args* a, int phases, int partial, void* stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    if (a->nBlocks == 0) return 0;
    cudaError_t e = decode_setup();
    if (e != cudaSuccess) return (int)e;
    DecodePlan p = plan_decode(a->nBlocks, a->dstCapArr != nullptr, a->dstCap, a->workspaceBytes, partial ? kDecodePartial : kDecodeFull);
    /* the switch does not apply to a wide batch (only the parallel scan writes the wide marks) nor to the partial call */
    if (!partial && g_scanImpl >= 0 && !p.wide) p.scan = (DecodeScan)g_scanImpl;
    const WsView w = ws_view(p, a->workspace);
    const int64_t sms = g_decodeSms;
    if (phases & 1) {
        e = cudaMemsetAsync(a->workspace, 0, 256, s);                   // WsHeader: list counter
        if (e != cudaSuccess) return (int)e;
        if (p.scan == kScanSplit) {
            const int64_t grid = (a->nBlocks + kSplitBlocksPerCta - 1) / kSplitBlocksPerCta;
            lz4_scan_split_kernel<<<(unsigned)grid, kSplitThreads, 0, s>>>(*a, w);
        } else if (p.scan == kScanPar) {
            const int64_t want = sms * 12;                              // 3 resident CTAs per SM, 4 rounds for balance
            const int64_t grid = a->nBlocks < want ? a->nBlocks : want;
            lz4_scan_par_kernel<<<(unsigned)grid, kScanLanes, sizeof(ScanParSmem), s>>>(*a, w);
            if (p.wide) {                                               // tiles kernel: first sequence of every tile, flags cleared
                lz4_tile_index_kernel<<<(unsigned)(a->nBlocks < sms * 8 ? a->nBlocks : sms * 8), 256, 0, s>>>(*a, w);
                g_launches++;
            }
        } else {
            const unsigned grid = (unsigned)((a->nBlocks + 127) / 128);
            if (partial) lz4_scan_partial_kernel<<<grid, 128, 0, s>>>(*a, w);
            else lz4_scan_kernel<<<grid, 128, 0, s>>>(*a, w);
        }
        g_launches++;
    }
    if (phases & 2) {
        if (p.wide) {                                                   // blocks above 64 KB: one CTA per 60 KB output tile
            const int64_t units = a->nBlocks * (int64_t)p.tilesMax;
            const int64_t grid = units < sms ? units : sms;             // all CTAs resident: a tile may wait for its predecessor
            /* the tiles' done flags start at 0 for THIS expand (the index kernel clears them too; an expand repeated after one
             * scan must not see the last one's) */
            e = cudaMemsetAsync(w.tileFlag, 0, (size_t)a->nBlocks * (p.tilesMax + 1) * sizeof(uint32_t), s);
            if (e != cudaSuccess) return (int)e;
            lz4_expand_tiles_kernel<<<(unsigned)grid, kRowsThreads, sizeof(RowsSmem), s>>>(*a, w);
        } else {
            const unsigned grid = (unsigned)(a->nBlocks < sms ? a->nBlocks : sms);   // persistent: one CTA per SM
            if (partial) lz4_expand_rows_partial_kernel<<<grid, kRowsThreads, sizeof(RowsSmem), s>>>(*a, w);
            else lz4_expand_rows_kernel<<<grid, kRowsThreads, sizeof(RowsSmem), s>>>(*a, w);
        }
        int64_t grid2 = (a->nBlocks * 32 + 127) / 128;                 // 4 warps = 4 blocks per CTA, grid-stride over the slow list
        if (grid2 > sms * 16) grid2 = sms * 16;
        if (partial) lz4_expand_generic_partial_kernel<<<(unsigned)grid2, 128, 0, s>>>(*a, w);
        else lz4_expand_generic_kernel<<<(unsigned)grid2, 128, 0, s>>>(*a, w);
        g_launches += 2;
    }
    return (int)cudaGetLastError();
}

/* grid of the one-warp encoders (lz4_encode_kernel, lz4_encode_dest_kernel) */
static int64_t encode_grid(int64_t nBlocks)
{
    const int sms = device_sms();
    const int perSm = 13;    // 16 KB table per warp: 13 x 16 KB + reserved fits the 228 KB SM
    int64_t grid = (int64_t)sms * perSm;
    return grid > nBlocks ? nBlocks : grid;
}

int lz4k_launch_encode(const lz4k_encode_args* a, void* stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    if (a->nBlocks == 0) return 0;
    lz4_encode_kernel<<<(unsigned)encode_grid(a->nBlocks), 32, kEncodeTableBytes, s>>>(*a);
    g_launches++;
    return (int)cudaGetLastError();
}

int lz4k_launch_encode_dest(const lz4k_encode_args* a, int32_t* srcConsumed, void* stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    if (a->nBlocks == 0) return 0;
    lz4_encode_dest_kernel<<<(unsigned)encode_grid(a->nBlocks), 32, kEncodeTableBytes, s>>>(*a, srcConsumed);
    g_launches++;
    return (int)cudaGetLastError();
}

/* developer tool: fill bytes [lo, hi) of every CTA's dynamic shared memory (parallel compressor layout) with a pattern, so
 * that a later launch that read shared memory it never wrote would show it (tests/perf/enc_determinism.py) */
__global__ void __launch_bounds__(kEpThreads, 2) lz4_poison_smem_kernel(uint32_t pattern, int lo, int hi)
{
    extern __shared__ __align__(16) uint8_t smemRaw[];
    for (int i = lo + (int)threadIdx.x; i < hi; i += kEpThreads) smemRaw[i] = (uint8_t)(pattern >> ((i & 3) * 8));
    __syncthreads();
    if (smemRaw[lo] == 1 && pattern == 0x12345678u && hi == -1) smemRaw[0] = 0;   /* keep the stores */
}
int lz4k_debug_poison_smem(uint32_t pattern, int lo, int hi, void* stream)
{
    const int sms = device_sms();
    cudaError_t e = cudaFuncSetAttribute(lz4_poison_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(EncParSmem));
    if (e != cudaSuccess) return (int)e;
    if (hi > (int)sizeof(EncParSmem)) hi = (int)sizeof(EncParSmem);
    lz4_poison_smem_kernel<<<2 * sms, kEpThreads, sizeof(EncParSmem), (cudaStream_t)stream>>>(pattern, lo, hi);
    return (int)cudaGetLastError();
}

int lz4k_launch_ceiling(const lz4k_decode_args* a, int mode, void* stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    if (a->nBlocks == 0) return 0;
    const int sms = device_sms();
    cudaError_t e = cudaFuncSetAttribute(lz4_ceiling_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RowsSmem));
    if (e != cudaSuccess) return (int)e;
    const int64_t grid = a->nBlocks < sms ? a->nBlocks : sms;
    lz4_ceiling_kernel<<<(unsigned)grid, kRowsThreads, sizeof(RowsSmem), s>>>(*a, mode);
    return (int)cudaGetLastError();
}

int lz4k_launch_encode_par(const lz4k_encode_args* a, void* stream)
{
    cudaStream_t s = (cudaStream_t)stream;
    if (a->nBlocks == 0) return 0;
    static int sms = 0;
    if (sms == 0) {
        cudaError_t e = cudaFuncSetAttribute(lz4_encode_par_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(EncParSmem));
        if (e != cudaSuccess) return (int)e;
        sms = device_sms();
    }
    const int64_t grid = a->nBlocks < 2 * sms ? a->nBlocks : 2 * sms;        // persistent: two CTAs per SM, blocks c, c + grid, ...
    lz4_encode_par_kernel<<<(unsigned)grid, kEpThreads, sizeof(EncParSmem), s>>>(*a);
    g_launches++;
    return (int)cudaGetLastError();
}

/* The HC encoder's workspace slots: 16 384 x 256 KB = 4 GiB at most.  More slots in flight hide more of the chain
 * walk's load latency; a caller that passes a larger workspace gets up to one slot per block. */
constexpr int64_t kHcSlots = 16384;

size_t lz4k_encode_hc_workspace_bytes(int64_t nBlocks)
{
    return nBlocks <= 0 ? 0 : (size_t)(nBlocks < kHcSlots ? nBlocks : kHcSlots) * kHcSlotBytes;
}

int lz4k_launch_encode_hc(const lz4k_encode_args* a, int level, void* workspace, size_t workspaceBytes, void* stream)
{
    if (a->nBlocks == 0) return 0;
    const int64_t fit = (int64_t)(workspaceBytes / kHcSlotBytes);
    const int64_t slots = a->nBlocks < fit ? a->nBlocks : fit;
    const int64_t grid = (slots + kHcThreads - 1) / kHcThreads;
    lz4_encode_hc_kernel<<<(unsigned)grid, kHcThreads, 0, (cudaStream_t)stream>>>(*a, (uint8_t*)workspace, slots, level);
    g_launches++;
    return (int)cudaGetLastError();
}

int lz4k_launch_pack(const uint8_t* slots, int64_t slotStride, const int32_t* sizes, int64_t nBlocks,
                     uint8_t* packed, int64_t* outOff, int headerBytes, void* stream)
{
    FrameRule fr; fr.raw = nullptr; fr.rawStride = 0; fr.blockSize = 0; fr.lastSize = 0;
    return launch_pack(slots, slotStride, sizes, nBlocks, packed, outOff, headerBytes, fr, (cudaStream_t)stream);
}

/* frame body: [LE32 header][payload] per block, stored-raw rule applied on the device (src = the blocks' source bytes) */
int lz4k_launch_pack_frame(const uint8_t* slots, int64_t slotStride, const int32_t* sizes, const uint8_t* src, int64_t srcStride,
                           int32_t blockSize, int32_t lastSize, int64_t nBlocks, uint8_t* packed, int64_t* outOff, void* stream)
{
    FrameRule fr; fr.raw = src; fr.rawStride = srcStride; fr.blockSize = blockSize; fr.lastSize = lastSize;
    return launch_pack(slots, slotStride, sizes, nBlocks, packed, outOff, 4, fr, (cudaStream_t)stream);
}

}  // extern "C"
