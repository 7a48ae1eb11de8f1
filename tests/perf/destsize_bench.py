#!/usr/bin/env python
"""Time LZ4B200_compress_blocks_destSize on bench.py's workload: 65 536 blocks of 64 KB, datagen P50 (bench.py's
generator), one warp per block.  Targets 4096, 16384, 32768 and 65809 (= LZ4_compressBound(65536): the compress_fast
route); LZ4B200_compress_blocks is timed in the same run, as the yardstick of the bound target.  Warm-up and CUDA-event
timing as bench.py's compress leg.  Prints one JSON line.

    python tests/perf/destsize_bench.py [--steps 3] [--warmup 1]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from bench import BLOCK, SEG, ClockSampler  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--blocks", type=int, default=65536)
    args = ap.parse_args()

    import torch
    from lz4_b200 import _lib, batch
    from oracle.pyoracle import Oracle

    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "needs a CUDA device"
    device = torch.device("cuda", 0)
    gpu = {"name": torch.cuda.get_device_name(device)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.split(",")
        gpu.update(power_limit_w=float(q[0]), sm_max_mhz=float(q[1]))
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    total = args.blocks * BLOCK
    host = Oracle().datagen_mt(total, SEG, 0.5, 0, os.cpu_count() or 1)
    src = torch.from_numpy(host).to(device)
    bound = batch.compress_bound(BLOCK)

    sampler = ClockSampler(0)
    sampler.start()
    time.sleep(0.3)

    def timed(fn):
        for _ in range(max(args.warmup, 1)):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps, sampler.summary(t0, time.time())

    rows = []
    for target in (4096, 16384, 32768, bound):
        slots, sizes, consumed, stride = batch.compress_blocks_dest_size(src, BLOCK, target, 1)
        ms, clocks = timed(lambda: batch.compress_blocks_dest_size(src, BLOCK, target, 1, slots=slots, slot_stride=stride,
                                                                   out_sizes=sizes, consumed=consumed))
        used = int(consumed.sum().item())
        out = int(sizes.clamp(min=0).sum().item())
        rows.append({"target": target, "ms": round(ms, 3), "consumed_gbps": round(used / ms / 1e6, 2),
                     "output_gbps": round(out / ms / 1e6, 2), "mean_consumed": round(used / args.blocks, 1),
                     "sm_mhz": clocks["sm_mhz"]})
    slots, sizes, stride = batch.compress_blocks(src, BLOCK, 1)
    ms, clocks = timed(lambda: batch.compress_blocks(src, BLOCK, 1, slots=slots, out_sizes=sizes))
    fast = {"ms": round(ms, 3), "input_gbps": round(total / ms / 1e6, 2), "sm_mhz": clocks["sm_mhz"]}
    sampler.stop()
    print(json.dumps({"metric": "LZ4B200_compress_blocks_destSize, %d x 64 KB datagen P50, acceleration 1" % args.blocks,
                      "steps": args.steps, "warmup": max(args.warmup, 1), "gpu": gpu, "dest_size": rows,
                      "compress_blocks": fast}))


if __name__ == "__main__":
    main()
