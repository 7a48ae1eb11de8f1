// Host build of LZ4B200_compress_frames_host's and LZ4B200_compress_legacy_host's plan and placement
// (lz4_b200/csrc/lz4_cfiles_plan.h): the verdicts, the headers, the cut of the blocks into groups of at most groupBytes
// source bytes and groupBlocks blocks, and per group what the device and the retire do -- each block encoded by a
// callback (the test's codec) at its capacity, the stored-raw rule, the 4-byte block header and the block checksum, the
// group's body laid out in file order and copied to each file's running position, the content hash carried across the
// cut in an fc_xxh32_state -- then the EndMark and the digest after a file's last block.
#include <vector>
#include "../../lz4_b200/csrc/lz4_cfiles_plan.h"

extern "C" {

// compressed size of block b (absolute source offset, size) at capacity cap into out (0: did not fit)
typedef int (*cfiles_encode_fn)(long long b, long long srcOff, int size, int cap, unsigned char* out);

static void put_le32(uint8_t* p, uint32_t v) { for (int i = 0; i < 4; i++) p[i] = (uint8_t)(v >> (8 * i)); }

// Returns the number of groups, -1 when memory runs out, -2 when a group breaks the cut's rules.
long long compress_files_host_emul(const unsigned char* src, const int64_t* srcOff, const int64_t* srcSize,
                                   unsigned char* dst, const int64_t* dstOff, const int64_t* dstCap, int64_t* result,
                                   long long nFiles, int legacy, int bsid, int contentSizeFlag, int sums,
                                   long long groupBytes, long long groupBlocks, cfiles_encode_fn encode)
{
    cp_plan p;
    if (!cp_build(srcOff, srcSize, dstCap, nFiles, legacy, bsid, contentSizeFlag, sums, &p)) { cp_free(&p); return -1; }
    std::vector<int64_t> pos((size_t)nFiles, 0);
    std::vector<fc_xxh32_state> st((size_t)nFiles);
    for (int64_t f = 0; f < nFiles; f++) {
        const fc_frame_rec* r = &p.files[f];
        if (r->status != LZ4B200_OK) { result[f] = r->status; continue; }
        pos[f] = cp_header(&p, f, dst + dstOff[f]);
        fc_xxh32_init(&st[f]);
        if (r->count == 0 && !legacy) {
            put_le32(dst + dstOff[f] + pos[f], 0);
            if (sums & FC_CONTENT_SUM) put_le32(dst + dstOff[f] + pos[f] + 4, fc_xxh32_digest(&st[f]));
            result[f] = pos[f] + 4 + ((sums & FC_CONTENT_SUM) ? 4 : 0);
        } else if (r->count == 0) {
            result[f] = pos[f];
        }
    }
    long long groups = 0;
    std::vector<uint8_t> slot, body;
    for (int64_t first = 0; first < p.nBlocks; groups++) {
        const int64_t end = cp_group_end(&p, first, groupBytes, groupBlocks);
        int64_t bytes = 0;
        if (end <= first || end > p.nBlocks || end - first > groupBlocks) { cp_free(&p); return -2; }
        body.clear();
        std::vector<int64_t> bodyOff;
        for (int64_t k = first; k < end; k++) {              // the encode, the stored-raw rule, the body in file order
            bytes += p.size[k];
            slot.assign((size_t)p.cap[k] + 16, 0);
            const int c = encode(k, p.srcOff[k], p.size[k], p.cap[k], slot.data());
            const bool raw = !legacy && (c <= 0 || c >= p.size[k]);
            const int s = raw ? p.size[k] : c;
            const uint8_t* payload = raw ? src + p.srcOff[k] : slot.data();
            uint8_t w[4];
            bodyOff.push_back((int64_t)body.size());
            put_le32(w, (uint32_t)s | (raw ? 0x80000000u : 0u));
            body.insert(body.end(), w, w + 4);
            body.insert(body.end(), payload, payload + s);
            if (!legacy && (sums & FC_BLOCK_SUM)) {
                put_le32(w, fc_xxh32(payload, (uint64_t)s, 0));
                body.insert(body.end(), w, w + 4);
            }
            // the content hash of the file's blocks in this group, from the state the group before left
            fc_xxh32_update(&st[p.file[k]], src + p.srcOff[k], (uint64_t)p.size[k]);
        }
        bodyOff.push_back((int64_t)body.size());
        if (end - first > 1 && bytes > groupBytes) { cp_free(&p); return -2; }
        for (int64_t k = first; k < end; k++) {              // the retire
            const int64_t f = p.file[k], len = bodyOff[k - first + 1] - bodyOff[k - first];
            const fc_frame_rec* r = &p.files[f];
            memcpy(dst + dstOff[f] + pos[f], body.data() + bodyOff[k - first], (size_t)len);
            pos[f] += len;
            if (k == r->base + r->count - 1) {
                if (legacy) { result[f] = pos[f]; continue; }
                put_le32(dst + dstOff[f] + pos[f], 0);
                if (sums & FC_CONTENT_SUM) put_le32(dst + dstOff[f] + pos[f] + 4, fc_xxh32_digest(&st[f]));
                result[f] = pos[f] + 4 + ((sums & FC_CONTENT_SUM) ? 4 : 0);
            }
        }
        first = end;
    }
    cp_free(&p);
    return groups;
}

}  // extern "C"
