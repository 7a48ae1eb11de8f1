"""Time LZ4B200_decompress_files against the frame and block calls on the same bytes, in the same run, alternating:
  (a) 65 536 one-frame files of 64 KB datagen P50 (a content checksum) against decompress_frames_checksummed;
  (b) one file of one frame of 1 GiB in 4 MB blocks with a content checksum (the `lz4` tool's default layout), verifying
      and skipping the checksums, against decompress_frames_checksummed;
  (c) one file of 256 concatenated 4 MB frames (content checksums) against decompress_frames_checksummed on the frames;
  (d) one 1 GiB `lz4 -l` legacy file against decompress_blocks on its 128 blocks with host-built tables;
  (e) the size-only pass on (a) and (b).
The frames are written on the GPU by compress_frames_checksummed (the reference's bytes), the legacy blocks by
compress_blocks.  CUDA events, median of 7 calls after 2 warm-up calls, the two calls of a pair alternating.  Prints the
card, its power limit and SM clocks, and one line per workload.
"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from lz4_b200 import batch  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402

MIB = 1 << 20


def timed_pair(f, g, reps=7, warmup=2):
    """medians (ms) of f and g, alternating"""
    for _ in range(warmup):
        f(); g()
    tf, tg = [], []
    for _ in range(reps):
        for fn, ts in ((f, tf), (g, tg)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(); fn(); b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
    return float(np.median(tf)), float(np.median(tg))


def source(orc, n, piece=64 * MIB):
    """n bytes of datagen P50 on the device, in 64 MiB segments of their own seeds"""
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    for k, at in enumerate(range(0, n, piece)):
        m = min(piece, n - at)
        out[at:at + m] = torch.from_numpy(orc.datagen(m, 0.5, k)).cuda()
    return out


def frames(src, n, size, bsid):
    """n checksummed frames of `size` bytes each from src, packed back to back: (buffer, offsets, lengths)"""
    offs = torch.arange(n, dtype=torch.int64, device="cuda") * size
    sizes = torch.full((n,), size, dtype=torch.int64, device="cuda")
    out, res = batch.compress_frames_checksummed(src, offs, sizes, block_size_id=bsid)
    torch.cuda.synchronize()
    lens = res.cpu().numpy()
    assert (lens > 0).all()
    bound = out.numel() // n
    pos = np.concatenate([[0], np.cumsum(lens)[:-1]]) + 16
    buf = torch.full((16 + int(lens.sum()) + 16,), 0xEE, dtype=torch.uint8, device="cuda")
    for f in range(n):                                  # the bound-spaced frames, closed up
        buf[int(pos[f]):int(pos[f]) + int(lens[f])] = out[f * bound:f * bound + int(lens[f])]
    return buf, torch.from_numpy(pos).cuda(), torch.from_numpy(lens.astype(np.int64)).cuda()


def files_call(comp, offs, sizes, caps, mu, mb, skip=False, size_only=False, out=None, ws=None):
    if size_only:
        return lambda: batch.decompressed_file_sizes(comp, offs, sizes, mu, mb, skip, workspace=ws)
    return lambda: batch.decompress_files(comp, offs, sizes, caps, mu, mb, skip, out=out, workspace=ws)


def main():
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip())
    orc = Oracle()
    rows = []

    # (a) 65 536 one-frame files of 64 KB
    n, sz = 65536, 65536
    src = source(orc, n * sz)
    comp, offs, lens = frames(src, n, sz, 4)
    caps = torch.full((n,), sz, dtype=torch.int64, device="cuda")
    out = torch.empty(n * sz, dtype=torch.uint8, device="cuda")
    mbf = [n, 0, 0, 0]
    f = files_call(comp, offs, lens, caps, n, mbf + [0], out=out)
    g = lambda: batch.decompress_frames_checksummed(comp, offs, lens, caps, mbf, out=out)  # noqa: E731
    rows.append(("a: 65536 x 64 KB one-frame files", *timed_pair(f, g), n * sz))
    s = files_call(comp, offs, lens, None, n, mbf + [0], size_only=True)
    rows.append(("e: sizes of (a)", *timed_pair(s, g), n * sz))
    del comp, out, src

    # (b) one file of one 1 GiB frame in 4 MB blocks; (c) the same bytes as 256 frames of 4 MB, concatenated
    total = 1 << 30
    src = source(orc, total)
    comp, offs, lens = frames(src, 1, total, 7)
    one = torch.tensor([total], dtype=torch.int64, device="cuda")
    out = torch.empty(total, dtype=torch.uint8, device="cuda")
    mb7 = [0, 0, 0, 256]
    for skip in (False, True):
        f = files_call(comp, offs, lens, one, 1, mb7 + [0], skip, out=out)
        g = lambda: batch.decompress_frames_checksummed(comp, offs, lens, one, mb7, skip, out=out)  # noqa: E731
        rows.append(("b: 1 GiB frame, 4 MB blocks, %s" % ("skip" if skip else "verify"), *timed_pair(f, g), total))
    s = files_call(comp, offs, lens, None, 1, mb7 + [0], size_only=True)
    g = lambda: batch.decompress_frames_checksummed(comp, offs, lens, one, mb7, out=out)  # noqa: E731
    rows.append(("e: sizes of (b)", *timed_pair(s, g), total))
    del comp
    comp, offs, lens = frames(src, 256, 4 * MIB, 7)
    whole = torch.tensor([16], dtype=torch.int64, device="cuda")
    wlen = torch.tensor([comp.numel() - 32], dtype=torch.int64, device="cuda")
    caps = torch.full((256,), 4 * MIB, dtype=torch.int64, device="cuda")
    f = files_call(comp, whole, wlen, one, 256, mb7 + [0], out=out)
    g = lambda: batch.decompress_frames_checksummed(comp, offs, lens, caps, mb7, out=out)  # noqa: E731
    rows.append(("c: 256 concatenated 4 MB frames", *timed_pair(f, g), total))
    del comp

    # (d) a 1 GiB legacy file against the block call on its blocks
    nb, bs = 128, 8 * MIB
    slots, sizes, stride = batch.compress_blocks(src, bs, 1)
    torch.cuda.synchronize()
    sz = sizes.cpu().numpy().astype(np.int64)
    pos = 16 + 4 + np.concatenate([[0], np.cumsum(sz + 4)[:-1]]) + 4        # each block after its size word
    leg = torch.full((16 + 4 + int((sz + 4).sum()) + 16,), 0xEE, dtype=torch.uint8, device="cuda")
    leg[16:20] = torch.tensor(list((0x184C2102).to_bytes(4, "little")), dtype=torch.uint8)
    for k in range(nb):
        p = int(pos[k])
        leg[p - 4:p] = torch.tensor(list(int(sz[k]).to_bytes(4, "little")), dtype=torch.uint8)
        leg[p:p + int(sz[k])] = slots[k * stride:k * stride + int(sz[k])]
    boffs = torch.from_numpy(pos).cuda()
    bsz = sizes.clone()
    loffs = torch.tensor([16], dtype=torch.int64, device="cuda")
    llen = torch.tensor([leg.numel() - 32], dtype=torch.int64, device="cuda")
    f = files_call(leg, loffs, llen, one, 1, [0, 0, 0, 0, nb], out=out)
    g = lambda: batch.decompress_blocks(leg, boffs, bsz, bs, out=out)  # noqa: E731
    _, res, _, _ = f()
    torch.cuda.synchronize()
    assert int(res[0]) == total and torch.equal(out, src)
    rows.append(("d: 1 GiB legacy file (128 x 8 MiB)", *timed_pair(f, g), total))

    print("%-40s %12s %12s %10s %10s" % ("workload", "files ms", "other ms", "files GB/s", "overhead"))
    for name, tf, tg, nbytes in rows:
        print("%-40s %12.3f %12.3f %10.1f %9.1f%%" % (name, tf, tg, nbytes / tf / 1e6, 100.0 * (tf - tg) / tg))


if __name__ == "__main__":
    main()
