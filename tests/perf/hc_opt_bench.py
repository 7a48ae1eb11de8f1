#!/usr/bin/env python
"""Time LZ4B200_compress_blocks_hc_opt (LZ4HC levels 10 .. 12, the optimal parser) on bench.py's workload: 64 KB blocks
of datagen P50 (bench.py's generator), one thread per block, at the bound capacity for each level, plus one fill-mode row
(LZ4B200_compress_blocks_hc_opt_destSize) at a 16 384-byte target.  A row first times a probe of --probe blocks (one
round: every block has its own slot); a row then runs on as many rounds of 16 384 slots as fit --budget-s per call (at
least the probe's blocks; the first N blocks of the same data), and the JSON line says how many.  In the same run, per
row:
  - ms per call (CUDA events, warm-up first), input GB/s and output GB/s, the compression ratio (input / output bytes)
    or, in fill mode, the mean consumed bytes per block;
  - the decode rate of the output through LZ4B200_decompress_blocks (packed first; decoded bytes per second), checked
    equal to the input;
  - the reference's LZ4_compress_HC (or LZ4_compress_HC_destSize) over the same blocks, called through ctypes from a pool
    of one Python thread per host CPU (ctypes releases the GIL during the call), when oracle/_ref/libref_lz4.so exists;
    its output bytes must equal the GPU's.
Card name, power limit and SM clock are read in the same run.  Prints one JSON line.

    python tests/perf/hc_opt_bench.py [--steps 1] [--warmup 0] [--budget-s 20]
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


def reference_rows(host, nb, limit, level, fill, threads):
    """(seconds, total output bytes, total consumed bytes) of the reference over the first nb blocks, one state per pool
    thread; None without oracle/_ref"""
    try:
        from oracle.pyoracle import Reference
        lib = Reference().lib
        plain, dest = lib.LZ4_compress_HC, lib.LZ4_compress_HC_destSize
    except (FileNotFoundError, OSError, AttributeError):
        return None
    plain.restype = dest.restype = C.c_int
    plain.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    dest.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int]
    lib.LZ4_sizeofStateHC.restype = C.c_int
    state_words = int(lib.LZ4_sizeofStateHC()) // 8 + 8
    room = max(min(limit, BLOCK + BLOCK // 255 + 16), 1)
    base = host.ctypes.data

    def part(k):
        state = np.zeros(state_words, dtype=np.uint64)
        dst = np.empty(room, dtype=np.uint8)
        out = used = 0
        for b in range(k, nb, threads):
            if fill:
                n = C.c_int(BLOCK)
                out += dest(state.ctypes.data, base + b * BLOCK, dst.ctypes.data, C.byref(n), limit, level)
                used += n.value
            else:
                out += plain(base + b * BLOCK, dst.ctypes.data, BLOCK, limit, level)
                used += BLOCK
        return out, used

    t0 = time.time()
    with ThreadPoolExecutor(threads) as pool:
        parts = list(pool.map(part, range(threads)))
    return time.time() - t0, sum(p[0] for p in parts), sum(p[1] for p in parts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1)
    ap.add_argument("--warmup", type=int, default=0)
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--probe", type=int, default=256)
    ap.add_argument("--budget-s", type=float, default=20.0)
    ap.add_argument("--levels", default="10,11,12")
    ap.add_argument("--dest-target", type=int, default=16384)
    ap.add_argument("--dest-level", type=int, default=12)
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

    def call(src, limit, lv, fill, **kw):
        if fill:
            return batch.compress_blocks_hc_opt_dest_size(src, BLOCK, limit, lv, **kw)
        slots, sizes, stride = batch.compress_blocks_hc_opt(src, BLOCK, lv, **kw)
        return slots, sizes, None, stride

    rows = []
    for lv, limit, fill in [(int(x), bound, False) for x in args.levels.split(",")] + \
                           [(args.dest_level, args.dest_target, True)]:
        probe = min(args.probe, args.blocks)
        t0 = time.time()
        call(src_all[:probe * BLOCK], limit, lv, fill)
        torch.cuda.synchronize()
        probe_s = time.time() - t0
        rounds = int(args.budget_s / max(probe_s, 1e-3))
        nb = max(probe, min(args.blocks, 16384 * rounds))
        src = src_all[:nb * BLOCK]
        slots, sizes, consumed, stride = call(src, limit, lv, fill)
        kw = dict(slots=slots, slot_stride=stride, out_sizes=sizes)
        if fill:
            kw["consumed"] = consumed
        ms, clocks = timed(lambda: call(src, limit, lv, fill, **kw), args.warmup, args.steps)
        out_bytes = int(sizes.sum().item())
        used = int(consumed.sum().item()) if fill else nb * BLOCK
        packed, offs = batch.pack_blocks(slots, stride, sizes)
        cap = int(consumed.max().item()) if fill else BLOCK
        dec = lambda: batch.decompress_blocks(packed, offs[:-1].contiguous(), sizes, cap)
        out, rets = dec()
        if fill:
            assert torch.equal(rets, consumed)
        else:
            assert bool((rets == BLOCK).all()) and torch.equal(out[:nb * BLOCK], src)
        dms, _ = timed(dec, 1, 3)
        row = {"level": lv, "mode": "destSize" if fill else "plain", "limit": limit, "blocks": nb,
               "probe_blocks": probe, "probe_s": round(probe_s, 2), "ms": round(ms, 1),
               "input_gbps": round(used / ms / 1e6, 4), "output_gbps": round(out_bytes / ms / 1e6, 4),
               "decode_gbps": round(used / dms / 1e6, 1), "sm_mhz": clocks["sm_mhz"]}
        if fill:
            row["mean_consumed"] = round(used / nb, 1)
        else:
            row["ratio"] = round(used / out_bytes, 4)
        ref = reference_rows(host, nb, limit, lv, fill, threads)
        if ref is not None:
            t, ref_out, ref_used = ref
            assert (ref_out, ref_used) == (out_bytes, used), "the reference's sums differ from the GPU's"
            row.update(cpu_ref_ms=round(t * 1e3, 1), cpu_ref_input_gbps=round(used / t / 1e9, 4), cpu_threads=threads,
                       cpu_ref_via="ctypes from a thread pool")
        rows.append(row)
        del slots, sizes, consumed, packed, out
    sampler.stop()
    print(json.dumps({"metric": "LZ4B200_compress_blocks_hc_opt(_destSize), 64 KB blocks of datagen P50",
                      "steps": args.steps, "warmup": args.warmup, "gpu": gpu, "rows": rows}))


if __name__ == "__main__":
    main()
