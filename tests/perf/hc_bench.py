#!/usr/bin/env python
"""Time LZ4B200_compress_blocks_hc on bench.py's workload: 64 KB blocks of datagen P50 (bench.py's generator), levels 2,
3, 6 and 9, one thread per block.  A level whose 65 536 blocks would take longer than --budget-s per call runs on fewer
blocks (the first N of the same data); the JSON line says how many.  In the same run, per level:
  - ms per call (CUDA events, warm-up first) and input GB/s, and the ratio against LZ4B200_compress_blocks's output;
  - the reference's LZ4_compress_HC on every host thread over the same blocks (Oracle.time_compress), when
    oracle/_ref/libref_lz4.so exists;
  - LZ4B200_decompress_blocks GB/s on the HC output, next to the same blocks from LZ4B200_compress_blocks.
Card name, power limit and SM clock are read in the same run.  Prints one JSON line.

    python tests/perf/hc_bench.py [--steps 2] [--warmup 1] [--budget-s 4]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from bench import BLOCK, SEG, ClockSampler  # noqa: E402


class _RefHC:
    """A codec for Oracle.time_compress whose _compress is the reference's LZ4_compress_HC (LZ4_compress_fast's
    signature, the level in the acceleration slot)."""

    def __init__(self):
        from oracle.pyoracle import Reference
        self._compress = Reference().lib.LZ4_compress_HC
        self._compress.restype = C.c_int
        self._compress.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--budget-s", type=float, default=4.0)
    ap.add_argument("--levels", default="2,3,6,9")
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
    orc = Oracle()
    threads = os.cpu_count() or 1
    host = orc.datagen_mt(args.blocks * BLOCK, SEG, 0.5, 0, threads)
    src_all = torch.from_numpy(host).to(device)
    try:
        ref = _RefHC()
    except (FileNotFoundError, OSError, AttributeError):
        ref = None

    sampler = ClockSampler(0)
    sampler.start()
    time.sleep(0.3)

    def timed(fn, warmup, steps):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.time()
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / steps, sampler.summary(t0, time.time())

    def decode_gbps(slots, stride, sizes, nb):
        packed, offs = batch.pack_blocks(slots, stride, sizes)
        out, rets = batch.decompress_blocks(packed, offs[:-1].contiguous(), sizes, BLOCK)
        ms, _ = timed(lambda: batch.decompress_blocks(packed, offs[:-1].contiguous(), sizes, BLOCK, out=out, out_sizes=rets),
                      1, 5)
        assert bool((rets == BLOCK).all()) and torch.equal(out, src_all[:nb * BLOCK])
        return round(nb * BLOCK / ms / 1e6, 2)

    rows = []
    for lv in [int(x) for x in args.levels.split(",")]:
        probe = min(2048, args.blocks)
        t0 = time.time()
        batch.compress_blocks_hc(src_all[:probe * BLOCK], BLOCK, lv)
        torch.cuda.synchronize()
        probe_s = time.time() - t0
        # 2 048 blocks run side by side (one slot each), so a call's time grows with the rounds of 16 384 slots
        rounds = max(1, int(args.budget_s / max(probe_s, 1e-3)))
        nb = min(args.blocks, 16384 * rounds if probe_s > 0 else args.blocks)
        src = src_all[:nb * BLOCK]
        slots, sizes, stride = batch.compress_blocks_hc(src, BLOCK, lv)
        ms, clocks = timed(lambda: batch.compress_blocks_hc(src, BLOCK, lv, slots=slots, slot_stride=stride,
                                                            out_sizes=sizes), args.warmup, args.steps)
        hc_bytes = int(sizes.sum().item())
        fslots, fsizes, fstride = batch.compress_blocks(src, BLOCK, 1)
        fms, _ = timed(lambda: batch.compress_blocks(src, BLOCK, 1, slots=fslots, out_sizes=fsizes), 1, 3)
        fast_bytes = int(fsizes.sum().item())
        row = {"level": lv, "blocks": nb, "ms": round(ms, 2), "input_gbps": round(nb * BLOCK / ms / 1e6, 3),
               "ratio": round(nb * BLOCK / hc_bytes, 4), "fast_ratio": round(nb * BLOCK / fast_bytes, 4),
               "fast_compress_ms": round(fms, 2), "sm_mhz": clocks["sm_mhz"],
               "decode_gbps_hc_output": decode_gbps(slots, stride, sizes, nb),
               "decode_gbps_fast_output": decode_gbps(fslots, fstride, fsizes, nb)}
        if ref is not None:
            out = np.empty(nb * stride, dtype=np.uint8)
            orc.first_touch(out, stride, nb, threads)
            t, rets = orc.time_compress(ref, host[:nb * BLOCK], BLOCK, out, stride, lv, threads)
            assert int(rets.sum()) == hc_bytes, "the reference's sizes differ from the GPU's"
            row.update(cpu_ref_ms=round(t * 1e3, 1), cpu_ref_gbps=round(nb * BLOCK / t / 1e9, 3), cpu_threads=threads)
        rows.append(row)
        del slots, sizes, fslots, fsizes
    sampler.stop()
    print(json.dumps({"metric": "LZ4B200_compress_blocks_hc, 64 KB blocks of datagen P50", "steps": args.steps,
                      "warmup": args.warmup, "gpu": gpu, "levels": rows}))


if __name__ == "__main__":
    main()
