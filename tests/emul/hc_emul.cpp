// Host build of the HC parses the GPU kernels run (lz4_b200/csrc/lz4_hc_core.h): TEST INFRASTRUCTURE.
// The CPU checks (tests/test_hc*_emul.py) compare it with the reference's vectors; the GPU tests of the HC calls
// (tests/test_gpu_hc*.py) compare the kernels with it.
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../lz4_b200/csrc/lz4_hc_core.h"

namespace {

struct HostAcc {
    const uint8_t* src;
    uint8_t* dst;
    uint32_t* ht;
    uint16_t* ct;
    hc::Opt* op;
    uint32_t in8(uint32_t p) { return src[p]; }
    uint32_t in32(uint32_t p) { uint32_t v; memcpy(&v, src + p, 4); return v; }
    uint64_t in64(uint32_t p) { uint64_t v; memcpy(&v, src + p, 8); return v; }
    uint32_t hash(uint32_t h) { return ht[h]; }
    void set_hash(uint32_t h, uint32_t v) { ht[h] = v; }
    uint32_t chain(uint32_t i) { return ct[i]; }
    void set_chain(uint32_t i, uint32_t v) { ct[i] = (uint16_t)v; }
    void out(int64_t o, uint32_t v) { dst[o] = (uint8_t)v; }
    void copy(int64_t o, uint32_t p, uint32_t len) { memcpy(dst + o, src + p, len); }
    hc::Opt& opt(int r) { return op[r]; }
};

// The chain table starts filled with `chainFill` (the reference's 0xFFFF, or anything else) and every field of the
// optimal parser's table with `optFill`: the output must depend on neither.
struct State {
    std::vector<uint32_t> ht;
    std::vector<uint16_t> ct;
    std::vector<hc::Opt> op;
    State(uint32_t chainFill, uint32_t optFill)
        : ht(hc::kHashEntries, 0), ct(hc::kChainEntries, (uint16_t)chainFill),
          op(hc::kOptEntries, hc::Opt{(int)optFill, (int)optFill, (int)optFill, (int)optFill}) {}
    HostAcc acc(const uint8_t* src, uint8_t* dst) { return HostAcc{src, dst, ht.data(), ct.data(), op.data()}; }
};

}  // namespace

// LZ4_compress_HC(src, dst, n, cap, level) for level <= 9; -1 for levels above.
extern "C" int hc_emul_compress(const uint8_t* src, int n, uint8_t* dst, int cap, int level, uint32_t chainFill)
{
    State s(chainFill, 0);
    HostAcc a = s.acc(src, dst);
    return hc::hc_compress_block(a, n, cap, level);
}

// LZ4_compress_HC_destSize(state, src, dst, &n, target, level) for level <= 9; -1 for levels above.  *consumed is what
// the reference leaves in n.
extern "C" int hc_dest_emul_compress(const uint8_t* src, int n, uint8_t* dst, int target, int level, uint32_t chainFill,
                                     int* consumed)
{
    State s(chainFill, 0);
    HostAcc a = s.acc(src, dst);
    return hc::hc_compress_block_dest(a, n, target, level, *consumed);
}

// LZ4_compress_HC(src, dst, n, cap, level) for level >= 10; -1 for levels below.
extern "C" int hc_opt_emul_compress(const uint8_t* src, int n, uint8_t* dst, int cap, int level, uint32_t chainFill,
                                    uint32_t optFill)
{
    State s(chainFill, optFill);
    HostAcc a = s.acc(src, dst);
    return hc::hc_compress_block_opt(a, n, cap, level);
}

// LZ4_compress_HC_destSize(state, src, dst, &n, target, level) for level >= 10; -1 for levels below.  *consumed is
// what the reference leaves in n.
extern "C" int hc_opt_emul_compress_dest(const uint8_t* src, int n, uint8_t* dst, int target, int level,
                                         uint32_t chainFill, uint32_t optFill, int* consumed)
{
    State s(chainFill, optFill);
    HostAcc a = s.acc(src, dst);
    return hc::hc_compress_block_opt_dest(a, n, target, level, *consumed);
}
