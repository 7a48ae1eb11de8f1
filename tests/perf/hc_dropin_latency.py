#!/usr/bin/env python
"""Time one drop-in LZ4_compress_HC call (liblz4_b200.so, one block from host memory to host memory) against the
reference's LZ4_compress_HC on one host thread, in the same run.

Inputs are datagen P50 blocks (the oracle's generator) of each --sizes; levels are --levels.  A row is the median wall
time of N calls (N from --reps, per size), each call synchronous: host -> device copy, one kernel launch, device -> host
copy of the returned bytes.  Before the timed calls every level takes one 4 KB call and every size one call whose
capacity of 1 byte stops the parse at its first sequence, so that module loading and the growth of the library's device
buffers stay out of the window.  The reference (oracle/_ref/libref_lz4.so) is timed on the same bytes and buffers from
this thread, and its output must equal the GPU's.  Card name, power limit and SM clocks are read in the same run.
Prints one JSON line.

    python tests/perf/hc_dropin_latency.py [--sizes 4096,65536,1048576] [--levels 2,3,9,10,12]
                                           [--reps 4096:15,65536:5,1048576:3]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from bench import ClockSampler  # noqa: E402


def card():
    import torch
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.split(",")
        gpu.update(power_limit_w=float(q[0]), sm_max_mhz=float(q[1]))
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return gpu


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,65536,1048576")
    ap.add_argument("--levels", default="2,3,9,10,12")
    ap.add_argument("--reps", default="4096:15,65536:5,1048576:3")
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    sizes = [int(x) for x in args.sizes.split(",")]
    levels = [int(x) for x in args.levels.split(",")]
    reps = {int(k): int(v) for k, v in (x.split(":") for x in args.reps.split(","))}

    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle, Reference
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "needs a CUDA device"
    ref = Reference().lib
    ref.LZ4_compress_HC.restype = C.c_int
    ref.LZ4_compress_HC.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]

    data = Oracle().datagen(max(sizes), 0.5, args.seed)
    bound = int(lib.LZ4_compressBound(max(sizes)))
    gdst = np.empty(bound, dtype=np.uint8)
    rdst = np.empty(bound, dtype=np.uint8)
    src = data.ctypes.data

    for lv in levels:                                   # module load, first launch per level
        assert lib.LZ4_compress_HC(src, gdst.ctypes.data, 4096, bound, lv) > 0
    for n in sizes:                                     # the library's device buffers grow to the largest input
        lib.LZ4_compress_HC(src, gdst.ctypes.data, n, 1, 3)

    sampler = ClockSampler(0)
    sampler.start()
    time.sleep(0.3)
    rows = []
    t_all = time.time()
    for n in sizes:
        cap = int(lib.LZ4_compressBound(n))
        for lv in levels:
            k = reps.get(n, 3)
            g, r = [], []
            t0 = time.time()
            for _ in range(k):
                s = time.perf_counter()
                gr = lib.LZ4_compress_HC(src, gdst.ctypes.data, n, cap, lv)
                g.append(time.perf_counter() - s)
            clocks = sampler.summary(t0, time.time())
            for _ in range(max(k, 5)):
                s = time.perf_counter()
                rr = ref.LZ4_compress_HC(src, rdst.ctypes.data, n, cap, lv)
                r.append(time.perf_counter() - s)
            assert gr == rr > 0 and gdst[:gr].tobytes() == rdst[:rr].tobytes(), (n, lv)
            gms, rms = statistics.median(g) * 1e3, statistics.median(r) * 1e3
            rows.append({"size": n, "level": lv, "calls": k, "gpu_ms": round(gms, 3), "gpu_ms_min": round(min(g) * 1e3, 3),
                         "gpu_ms_max": round(max(g) * 1e3, 3), "ref_ms": round(rms, 3), "gpu_over_ref": round(gms / rms, 1),
                         "ratio": round(n / gr, 4), "sm_mhz": clocks["sm_mhz"]})
    sampler.stop()
    print(json.dumps({"metric": "LZ4_compress_HC wall ms per call (median), one block, datagen P50",
                      "gpu": card(), "ref": "reference LZ4_compress_HC on one host thread, gcc -O3",
                      "seconds": round(time.time() - t_all, 1), "rows": rows}))


if __name__ == "__main__":
    main()
