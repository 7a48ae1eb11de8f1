// Host build of the HC fill parse the GPU kernel runs (lz4_b200/csrc/lz4_hc_core.h): TEST INFRASTRUCTURE.
// tests/test_hc_destsize_emul.py checks it against the reference's vectors; tests/test_gpu_hc_destsize.py checks the
// kernel against it.
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
    uint32_t in8(uint32_t p) { return src[p]; }
    uint32_t in32(uint32_t p) { uint32_t v; memcpy(&v, src + p, 4); return v; }
    uint64_t in64(uint32_t p) { uint64_t v; memcpy(&v, src + p, 8); return v; }
    uint32_t hash(uint32_t h) { return ht[h]; }
    void set_hash(uint32_t h, uint32_t v) { ht[h] = v; }
    uint32_t chain(uint32_t i) { return ct[i]; }
    void set_chain(uint32_t i, uint32_t v) { ct[i] = (uint16_t)v; }
    void out(int64_t o, uint32_t v) { dst[o] = (uint8_t)v; }
    void copy(int64_t o, uint32_t p, uint32_t len) { memcpy(dst + o, src + p, len); }
};

}  // namespace

// LZ4_compress_HC_destSize(state, src, dst, &n, target, level) for level <= 9; -1 for levels above.  *consumed is what
// the reference leaves in n.  The chain table starts filled with `chainFill`: the output must not depend on it.
extern "C" int hc_dest_emul_compress(const uint8_t* src, int n, uint8_t* dst, int target, int level, uint32_t chainFill,
                                     int* consumed)
{
    std::vector<uint32_t> ht(hc::kHashEntries, 0);
    std::vector<uint16_t> ct(hc::kChainEntries, (uint16_t)chainFill);
    HostAcc a{src, dst, ht.data(), ct.data()};
    return hc::hc_compress_block_dest(a, n, target, level, *consumed);
}
