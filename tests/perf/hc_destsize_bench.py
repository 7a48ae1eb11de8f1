#!/usr/bin/env python
"""Time LZ4B200_compress_blocks_hc_destSize on bench.py's workload: 64 KB blocks of datagen P50 (bench.py's generator), at
levels 2, 3 and 9 and targets of 4 096, 16 384 and LZ4_compressBound(65 536) bytes, one thread per block.  A row whose
65 536 blocks would take longer than --budget-s per call runs on fewer blocks (the first N of the same data), as in
hc_bench.py; the JSON line says how many.  In the same run, per row:
  - ms per call (CUDA events, warm-up first), consumed input GB/s, output GB/s and the mean consumed bytes per block;
  - the mean consumed bytes of LZ4B200_compress_blocks_destSize (the fast parse) at the same target;
  - the reference's LZ4_compress_HC_destSize over the same blocks, called through ctypes from a pool of one Python thread
    per host CPU (ctypes releases the GIL during the call), when oracle/_ref/libref_lz4.so exists; its sums of output
    and consumed bytes must equal the GPU's.
Card name, power limit and SM clock are read in the same run.  Prints one JSON line.

    python tests/perf/hc_destsize_bench.py [--steps 2] [--warmup 1] [--budget-s 4]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from bench import BLOCK, SEG, ClockSampler  # noqa: E402


def reference_rows(host, nb, target, level, threads):
    """(seconds, total output bytes, total consumed bytes) of the reference's LZ4_compress_HC_destSize over the first nb
    blocks, one state per pool thread; None without oracle/_ref"""
    try:
        from oracle.pyoracle import Reference
        lib = Reference().lib
        fn = lib.LZ4_compress_HC_destSize
    except (FileNotFoundError, OSError, AttributeError):
        return None
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int]
    lib.LZ4_sizeofStateHC.restype = C.c_int
    state_words = int(lib.LZ4_sizeofStateHC()) // 8 + 8
    room = max(min(target, BLOCK + BLOCK // 255 + 16), 1)
    base = host.ctypes.data

    def part(k):
        state = np.zeros(state_words, dtype=np.uint64)
        dst = np.empty(room, dtype=np.uint8)
        out = used = 0
        for b in range(k, nb, threads):
            n = C.c_int(BLOCK)
            out += fn(state.ctypes.data, base + b * BLOCK, dst.ctypes.data, C.byref(n), target, level)
            used += n.value
        return out, used

    t0 = time.time()
    with ThreadPoolExecutor(threads) as pool:
        parts = list(pool.map(part, range(threads)))
    return time.time() - t0, sum(p[0] for p in parts), sum(p[1] for p in parts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--budget-s", type=float, default=4.0)
    ap.add_argument("--levels", default="2,3,9")
    ap.add_argument("--targets", default="4096,16384,bound")
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
    threads = os.cpu_count() or 1
    host = Oracle().datagen_mt(args.blocks * BLOCK, SEG, 0.5, 0, threads)
    src_all = torch.from_numpy(host).to(device)
    bound = batch.compress_bound(BLOCK)
    targets = [bound if t == "bound" else int(t) for t in args.targets.split(",")]

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

    rows = []
    for lv in [int(x) for x in args.levels.split(",")]:
        for target in targets:
            probe = min(2048, args.blocks)
            t0 = time.time()
            batch.compress_blocks_hc_dest_size(src_all[:probe * BLOCK], BLOCK, target, lv)
            torch.cuda.synchronize()
            probe_s = time.time() - t0
            # 2 048 blocks run side by side (one slot each), so a call's time grows with the rounds of 16 384 slots
            rounds = max(1, int(args.budget_s / max(probe_s, 1e-3)))
            nb = min(args.blocks, 16384 * rounds)
            src = src_all[:nb * BLOCK]
            slots, sizes, consumed, stride = batch.compress_blocks_hc_dest_size(src, BLOCK, target, lv)
            ms, clocks = timed(lambda: batch.compress_blocks_hc_dest_size(src, BLOCK, target, lv, slots=slots,
                                                                          slot_stride=stride, out_sizes=sizes,
                                                                          consumed=consumed),
                               args.warmup, args.steps)
            out_bytes, used = int(sizes.sum().item()), int(consumed.sum().item())
            _, _, fcons, _ = batch.compress_blocks_dest_size(src, BLOCK, target, 1)
            row = {"level": lv, "target": target, "blocks": nb, "ms": round(ms, 2),
                   "consumed_gbps": round(used / ms / 1e6, 3), "output_gbps": round(out_bytes / ms / 1e6, 3),
                   "mean_consumed": round(used / nb, 1), "fast_destsize_mean_consumed": round(int(fcons.sum().item()) / nb, 1),
                   "sm_mhz": clocks["sm_mhz"]}
            ref = reference_rows(host, nb, target, lv, threads)
            if ref is not None:
                t, ref_out, ref_used = ref
                assert (ref_out, ref_used) == (out_bytes, used), "the reference's sums differ from the GPU's"
                row.update(cpu_ref_ms=round(t * 1e3, 1), cpu_ref_consumed_gbps=round(used / t / 1e9, 3),
                           cpu_threads=threads, cpu_ref_via="ctypes from a thread pool")
            rows.append(row)
            del slots, sizes, consumed
    sampler.stop()
    print(json.dumps({"metric": "LZ4B200_compress_blocks_hc_destSize, 64 KB blocks of datagen P50", "steps": args.steps,
                      "warmup": args.warmup, "gpu": gpu, "rows": rows}))


if __name__ == "__main__":
    main()
