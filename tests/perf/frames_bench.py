"""Time LZ4B200_decompress_frames on frames already in device memory, against LZ4B200_decompress_blocks on the same blocks
with tables built on the host, in the same run:
  (a) 65 536 one-block frames of 64 KB datagen P50,
  (b) one frame of 1 024 x 4 MB blocks,
  (c) a mixed batch: 8 192 one-block 64 KB frames, 1 024 two-block 256 KB frames, 256 two-block 1 MB frames and 32
      three-block 4 MB frames (one blocks call per block size for the comparison).
CUDA events, median of 10 calls after 2 warm-up calls; then one torch.profiler run per workload for the frame call's own
kernels (index, scan, fill, verdict, raw copy).  Prints the card, its power limit and SM clocks.
"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lz4_b200 import batch  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402
import frame_corpus as fc  # noqa: E402


def timed(fn, reps=10, warmup=2):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def build(orc, classes, seed=0):
    """frames of (bsid, frames, blocks per frame) groups on the device, 16 bytes of padding at both ends; returns the
    frame tables, the decoded size, and per class the block tables of the same blocks (absolute offsets, sizes)"""
    groups, total_src = [], 16
    for g, (bsid, nf, k) in enumerate(classes):
        bs = 1 << (8 + 2 * bsid)
        data = torch.from_numpy(orc.datagen_mt(bs * nf * k, 65536, 0.5, seed + g)).cuda()
        slots, sizes, stride = batch.compress_blocks(data, bs, 1)
        assert bool((sizes > 0).all()) and bool((sizes < bs).all())
        packed, offs = batch.pack_blocks(slots, stride, sizes, header_bytes=4)
        del slots, data
        offs_h = offs.cpu().numpy()
        flen = offs_h[k::k] - offs_h[:-1:k][:nf] + 11                   # header (7) + blocks + EndMark (4)
        fpos = total_src + np.concatenate([[0], np.cumsum(flen)[:-1]])
        total_src += int(flen.sum())
        groups.append((bsid, nf, k, bs, packed, offs_h, sizes, flen, fpos))
    src = torch.zeros(total_src + 16, dtype=torch.uint8, device="cuda")
    f_off, f_size, blk = [], [], {}
    for bsid, nf, k, bs, packed, offs_h, sizes, flen, fpos in groups:
        fh = torch.tensor(list(fc.header((1 << 6) | (1 << 5), bsid << 4)), dtype=torch.uint8, device="cuda")
        for f in range(nf):
            lo, hi, p = int(offs_h[f * k]), int(offs_h[(f + 1) * k]), int(fpos[f])
            src[p + 7:p + 7 + hi - lo] = packed[lo:hi]
        idx = torch.from_numpy(fpos).cuda()[:, None] + torch.arange(7, device="cuda")[None, :]
        src[idx.reshape(-1)] = fh.repeat(nf)
        j = np.arange(nf * k)
        b_off = fpos[j // k] + 7 + (offs_h[j] - offs_h[(j // k) * k]) + 4
        blk[bsid] = (torch.from_numpy(b_off.astype(np.int64)).cuda(), sizes.contiguous(), bs)
        f_off.append(fpos)
        f_size.append(flen)
    f_off = torch.from_numpy(np.concatenate(f_off).astype(np.int64)).cuda()
    f_size = torch.from_numpy(np.concatenate(f_size).astype(np.int64)).cuda()
    decoded = [nf * k * bs for bsid, nf, k, bs, *_ in groups]
    caps = torch.tensor(sum([[k * bs] * nf for bsid, nf, k, bs, *_ in groups], []), dtype=torch.int64, device="cuda")
    budget = [0, 0, 0, 0]
    for bsid, nf, k, *_ in groups:
        budget[bsid - 4] += nf * k
    return src, f_off, f_size, caps, budget, sum(decoded), blk


def run(name, orc, classes):
    src, f_off, f_size, caps, budget, total, blk = build(orc, classes)
    ws = torch.empty(batch.decompress_frames_workspace_bytes(f_off.numel(), budget), dtype=torch.uint8, device="cuda")
    out, res, cons = batch.decompress_frames(src, f_off, f_size, caps, budget, workspace=ws)
    torch.cuda.synchronize()
    assert torch.equal(res, caps) and torch.equal(cons, f_size), name
    ms = timed(lambda: batch.decompress_frames(src, f_off, f_size, caps, budget, out=out, results=res, consumed=cons,
                                               workspace=ws))
    # the same blocks through LZ4B200_decompress_blocks, one call per block size
    bouts = {}
    for bsid, (o, s, bs) in blk.items():
        bw = torch.empty(batch._lib.load().LZ4B200_decompress_workspace_bytes_for(s.numel(), 0, bs), dtype=torch.uint8,
                         device="cuda")
        bo, br = batch.decompress_blocks(src, o, s, bs, workspace=bw)
        torch.cuda.synchronize()
        assert bool((br == bs).all())
        bouts[bsid] = (o, s, bs, bo, br, bw)
    if len(blk) == 1:
        assert torch.equal(bouts[next(iter(blk))][3][:total], out[:total]), name
    bms = timed(lambda: [batch.decompress_blocks(src, o, s, bs, out=bo, out_sizes=br, workspace=bw)
                         for o, s, bs, bo, br, bw in bouts.values()])
    print("%-42s frames %9.3f ms %7.1f GB/s | blocks %9.3f ms %7.1f GB/s | frame call / blocks %.3f"
          % (name, ms, total / ms / 1e6, bms, total / bms / 1e6, ms / bms))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        batch.decompress_frames(src, f_off, f_size, caps, budget, out=out, results=res, consumed=cons, workspace=ws)
        torch.cuda.synchronize()
    own = {}
    for e in prof.key_averages():
        if "lz4_frames_" in e.key:
            k = e.key.split("lz4_frames_")[1].split("_kernel")[0]
            own[k] = own.get(k, 0.0) + e.device_time_total / 1e3
    print("    frame kernels (profiler, ms): " + ", ".join("%s %.3f" % kv for kv in sorted(own.items())))
    del src, out, ws, bouts
    torch.cuda.empty_cache()


def main():
    print("card:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                   "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    orc = Oracle()
    run("(a) 65536 one-block frames of 64 KB", orc, [(4, 65536, 1)])
    run("(b) one frame of 1024 x 4 MB", orc, [(7, 1, 1024)])
    run("(c) mixed 64 KB / 256 KB / 1 MB / 4 MB", orc, [(4, 8192, 1), (5, 1024, 2), (6, 256, 2), (7, 32, 3)])


if __name__ == "__main__":
    main()
