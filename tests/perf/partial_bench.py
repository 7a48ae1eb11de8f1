"""Time LZ4B200_decompress_blocks_partial: 65 536 x 64 KB datagen P50 blocks (bench.py's workload) at targets of 4 096,
16 384 and 65 536 against LZ4B200_decompress_blocks on the same batch, and 1 024 x 4 MB blocks at 61 440.  CUDA events,
median of 20 calls after 3 warm-up calls; prints the card, its power limit and SM clocks.
"""
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
from lz4_b200 import batch  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402


def timed(fn, reps=20, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def batch_of(orc, bs, n, seed):
    src = torch.from_numpy(orc.datagen_mt(bs * n, 65536, 0.5, seed)).cuda()
    slots, sizes, stride = batch.compress_blocks(src, bs, 1)
    packed, offs = batch.pack_blocks(slots, stride, sizes)
    return src, packed, offs[:-1].contiguous(), sizes


def main():
    print("card:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                   "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    orc = Oracle()
    n = 65536
    src, packed, offs, sizes = batch_of(orc, 65536, n, 0)
    out, rets = batch.decompress_blocks(packed, offs, sizes, 65536)
    ms = timed(lambda: batch.decompress_blocks(packed, offs, sizes, 65536, out=out, out_sizes=rets))
    print("full decode    %d x 64 KB: %8.3f ms" % (n, ms))
    for t in (4096, 16384, 65536):
        pout, prets = batch.decompress_blocks_partial(packed, offs, sizes, t)
        assert bool((prets == t).all())
        ms = timed(lambda: batch.decompress_blocks_partial(packed, offs, sizes, t, out=pout, out_sizes=prets))
        print("partial %5d  %d x 64 KB: %8.3f ms  %6.1f GB/s of prefix" % (t, n, ms, t * n / ms / 1e6))
    del src, packed, out, pout
    torch.cuda.empty_cache()
    n, t = 1024, 61440
    src, packed, offs, sizes = batch_of(orc, 4 << 20, n, 1)
    pout, prets = batch.decompress_blocks_partial(packed, offs, sizes, t)
    assert bool((prets == t).all()) and torch.equal(pout.view(n, t), src.view(n, 4 << 20)[:, :t])
    ms = timed(lambda: batch.decompress_blocks_partial(packed, offs, sizes, t, out=pout, out_sizes=prets))
    print("partial %5d  %d x 4 MB:   %8.3f ms" % (t, n, ms))


if __name__ == "__main__":
    main()
