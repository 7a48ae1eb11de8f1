// Host build of the carried XXH32 state of lz4_b200/csrc/lz4_frame_core.h (fc_xxh32_init / update / digest), which
// LZ4B200_decompress_files_host's carry kernel runs across the groups of a frame, and of the one-shot fc_xxh32.
#include "../../lz4_b200/csrc/lz4_frame_core.h"

extern "C" {

// XXH32(p[0 .. len), 0) fed in pieces that end at cuts[0] < cuts[1] < ... < cuts[nCuts - 1] (the last is len)
unsigned xxh32_state_pieces(const unsigned char* p, long long len, const long long* cuts, int nCuts)
{
    fc_xxh32_state s;
    long long at = 0;
    fc_xxh32_init(&s);
    for (int i = 0; i < nCuts; i++) { fc_xxh32_update(&s, p + at, (uint64_t)(cuts[i] - at)); at = cuts[i]; }
    if (at < len) fc_xxh32_update(&s, p + at, (uint64_t)(len - at));
    return fc_xxh32_digest(&s);
}

unsigned xxh32_state_oneshot(const unsigned char* p, long long len) { return fc_xxh32(p, (uint64_t)len, 0); }

}
