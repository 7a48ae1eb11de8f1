/*
 * lz4_encode_hc.cuh -- LZ4_compress_HC at levels 1 .. 12 over a batch (included by lz4_kernels.cu).
 *
 * The HC parse is sequential within a block, so one THREAD compresses one block at a time with the parse of
 * lz4_hc_core.h, and the parallelism is across blocks.  A block's state is a 2^15 x u32 hash table and a 64 K x u16
 * chain table (256 KB), more than an SM's shared memory, so every thread owns one workspace slot in global memory and
 * takes blocks t, t + slots, t + 2 * slots, ...  The hash table is zeroed before every block; the chain table is not
 * (lz4_hc_core.h shows why no entry is read before it is written).  lz4_encode_hc_dest_kernel runs the fill parse of
 * LZ4_compress_HC_destSize on the same layout.  DESIGN.md section 3.7.
 * The optimal parser of levels 10 .. 12 (lz4_encode_hc_opt_kernel, lz4_encode_hc_opt_dest_kernel) runs in the same slot
 * loop on a larger slot: the tables, then its price table of kOptEntries x 16 bytes, which needs no initial value
 * either.  The price table stays in the workspace: as a local array it would make every resident thread reserve 64 KB
 * of local memory.  DESIGN.md section 3.8.
 */

#include <type_traits>

constexpr int kHcThreads = 32;
constexpr size_t kHcHashBytes = (size_t)hc::kHashEntries * sizeof(uint32_t);
constexpr size_t kHcSlotBytes = kHcHashBytes + (size_t)hc::kChainEntries * sizeof(uint16_t);
constexpr size_t kHcOptSlotBytes = kHcSlotBytes + (size_t)hc::kOptEntries * sizeof(hc::Opt);    /* 327 728 */
static_assert(kHcOptSlotBytes % 16 == 0, "every slot's hash table starts 16-byte aligned");

struct HcDevAcc {
    const uint8_t* src;
    uint8_t* dst;
    uint32_t* ht;
    uint16_t* ct;
    /* 4 input bytes from the two aligned words holding them: both words hold bytes of the block */
    __device__ __forceinline__ uint32_t in32(uint32_t p) const
    {
        const uintptr_t a = reinterpret_cast<uintptr_t>(src + p);
        const uint32_t lo = __ldg(reinterpret_cast<const uint32_t*>(a & ~uintptr_t(3)));
        const uint32_t hi = __ldg(reinterpret_cast<const uint32_t*>((a + 3) & ~uintptr_t(3)));
        return __funnelshift_r(lo, hi, (uint32_t)(a & 3) * 8);
    }
    __device__ __forceinline__ uint32_t in8(uint32_t p) const { return __ldg(src + p); }
    __device__ __forceinline__ uint64_t in64(uint32_t p) const { return (uint64_t)in32(p) | ((uint64_t)in32(p + 4) << 32); }
    __device__ __forceinline__ uint32_t hash(uint32_t h) const { return ht[h]; }
    __device__ __forceinline__ void set_hash(uint32_t h, uint32_t v) const { ht[h] = v; }
    __device__ __forceinline__ uint32_t chain(uint32_t i) const { return ct[i]; }
    __device__ __forceinline__ void set_chain(uint32_t i, uint32_t v) const { ct[i] = (uint16_t)v; }
    __device__ __forceinline__ void out(int64_t o, uint32_t v) const { dst[o] = (uint8_t)v; }
    __device__ __forceinline__ void copy(int64_t o, uint32_t p, uint32_t len) const
    {
        for (uint32_t k = 0; k < len; k++) dst[o + k] = __ldg(src + p + k);
    }
};

/* the optimal parser's accessor: the same, and its price table */
struct HcOptDevAcc : HcDevAcc {
    hc::Opt* op;
    __device__ __forceinline__ hc::Opt& opt(int r) const { return op[r]; }
};

/* One slot's blocks: t, t + slots, ...  FILL: LZ4_compress_HC_destSize with targetDstSize = the block's capacity, which also writes
 * srcConsumed[b].  OPT: the optimal parser (levels 10 and up) on slots of kHcOptSlotBytes. */
template <bool FILL, bool OPT = false>
__device__ __forceinline__ void hc_slot_blocks(const lz4k_encode_args& a, int32_t* srcConsumed, uint8_t* ws, int64_t t,
                                               int64_t slots, int level)
{
    constexpr size_t slotBytes = OPT ? kHcOptSlotBytes : kHcSlotBytes;
    typename std::conditional<OPT, HcOptDevAcc, HcDevAcc>::type acc;
    acc.ht = reinterpret_cast<uint32_t*>(ws + t * slotBytes);
    acc.ct = reinterpret_cast<uint16_t*>(ws + t * slotBytes + kHcHashBytes);
    if constexpr (OPT) acc.op = reinterpret_cast<hc::Opt*>(ws + t * slotBytes + kHcSlotBytes);
    for (int64_t b = t; b < a.nBlocks; b += slots) {
        const int n = a.srcSizeArr ? a.srcSizeArr[b] : a.srcSize;
        const int cap = enc_cap(a, b);
        acc.src = enc_src(a, b);
        acc.dst = enc_dst(a, b);
        if (n >= hc::kMinLength && (uint32_t)n <= hc::kMaxInput) {         // shorter blocks never touch the tables
            uint4* h = reinterpret_cast<uint4*>(acc.ht);
            for (int k = 0; k < (int)(kHcHashBytes / sizeof(uint4)); k++) h[k] = make_uint4(0, 0, 0, 0);
        }
        if constexpr (OPT) {    /* the level 1 .. 9 kernels never see the optimal parser's text */
            if (FILL) {
                int consumed;
                a.outSize[b] = hc::hc_compress_block_opt_dest(acc, n, cap, level, consumed);
                srcConsumed[b] = consumed;
            } else {
                a.outSize[b] = hc::hc_compress_block_opt(acc, n, cap, level);
            }
        } else if (FILL) {
            int consumed;
            a.outSize[b] = hc::hc_compress_block_dest(acc, n, cap, level, consumed);
            srcConsumed[b] = consumed;
        } else {
            a.outSize[b] = hc::hc_compress_block(acc, n, cap, level);
        }
    }
}

/* slots = the threads that run: min(nBlocks, workspace slots) */
__global__ void __launch_bounds__(kHcThreads) lz4_encode_hc_kernel(lz4k_encode_args a, uint8_t* ws, int64_t slots, int level)
{
    const int64_t t = (int64_t)blockIdx.x * kHcThreads + threadIdx.x;
    if (t >= slots) return;
    hc_slot_blocks<false>(a, nullptr, ws, t, slots, level);
}

/* the same slots and grid, LZ4_compress_HC_destSize per block: the parse stops at the target, so a block costs the input
 * it consumes */
__global__ void __launch_bounds__(kHcThreads) lz4_encode_hc_dest_kernel(lz4k_encode_args a, int32_t* srcConsumed, uint8_t* ws,
                                                                        int64_t slots, int level)
{
    const int64_t t = (int64_t)blockIdx.x * kHcThreads + threadIdx.x;
    if (t >= slots) return;
    hc_slot_blocks<true>(a, srcConsumed, ws, t, slots, level);
}

/* levels 10 and up, LZ4_compress_HC per block: the same grid on slots of kHcOptSlotBytes */
__global__ void __launch_bounds__(kHcThreads) lz4_encode_hc_opt_kernel(lz4k_encode_args a, uint8_t* ws, int64_t slots,
                                                                       int level)
{
    const int64_t t = (int64_t)blockIdx.x * kHcThreads + threadIdx.x;
    if (t >= slots) return;
    hc_slot_blocks<false, true>(a, nullptr, ws, t, slots, level);
}

/* levels 10 and up, LZ4_compress_HC_destSize per block */
__global__ void __launch_bounds__(kHcThreads) lz4_encode_hc_opt_dest_kernel(lz4k_encode_args a, int32_t* srcConsumed,
                                                                            uint8_t* ws, int64_t slots, int level)
{
    const int64_t t = (int64_t)blockIdx.x * kHcThreads + threadIdx.x;
    if (t >= slots) return;
    hc_slot_blocks<true, true>(a, srcConsumed, ws, t, slots, level);
}
