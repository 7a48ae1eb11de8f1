#!/usr/bin/env python
"""Time LZ4B200_compress_blocks_indexed against the strided compress calls.  Prints one JSON line.

(a) Same blocks, same addresses: bench.py's workload (65 536 x 64 KB blocks of datagen P50) through the strided call
    (LZ4B200_compress_blocks, LZ4B200_compress_blocks_parallel; the latter also with per-block sizes, which makes it
    launch both of its kernels as the indexed call does) and through the indexed call with offsets i * stride and one
    capacity, for PARSE_FAST and PARSE_PARALLEL; PARSE_HC at level 9 (LZ4B200_compress_blocks_hc) on the first
    --hc-blocks blocks.  With --baseline-lib (a liblz4_b200.so built from an earlier commit) the strided calls of that
    library are timed too.  The variants alternate within every round, so that they share the card's state; each
    reports the median and the min .. max of its rounds (CUDA events around one call).  Every variant's sizes and
    bytes are checked equal to the first one's.
(b) Buffers of mixed sizes: --buffers buffers of sizes log-uniform in 512 B .. 1 MB (datagen P50) at packed offsets,
    one indexed call (capacities LZ4_compressBound(n_i), outputs abutting) against one strided call over a copy padded
    to the largest size (slots of LZ4_compressBound(largest)).  Reports ms per call and the output bytes each needs;
    the strided call is skipped, and says so, when the card lacks the memory for its padded copy.
Card name, power limit and SM clock are read in the same run.

    python tests/perf/compress_indexed_bench.py [--rounds 7] [--baseline-lib PATH] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from bench import BLOCK, SEG  # noqa: E402

FAST, PARALLEL, HC = 0, 1, 2


def bound(n):
    return n + n // 255 + 16


def load_baseline(path):
    """an earlier build of the library, with the prototypes of the strided calls it shares with this one"""
    from lz4_b200 import _lib
    lib = C.CDLL(os.path.abspath(path))
    for name, res, args in _lib.PROTOTYPES:
        if name in ("LZ4B200_compress_blocks", "LZ4B200_compress_blocks_parallel", "LZ4B200_compress_blocks_hc",
                    "LZ4B200_compress_blocks_hc_workspace_bytes", "LZ4B200_device_count"):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib


def card():
    import torch
    gpu = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm,clocks.sm",
                            "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout.split(",")
        gpu.update(power_limit_w=float(q[0]), sm_max_mhz=float(q[1]), sm_now_mhz=float(q[2]))
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        pass
    return gpu


def event_ms(fn):
    import torch
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def summary(ms):
    ms = sorted(ms)
    return {"median_ms": round(float(np.median(ms)), 3), "min_ms": round(ms[0], 3), "max_ms": round(ms[-1], 3),
            "spread_pct": round(100.0 * (ms[-1] - ms[0]) / ms[0], 2)}


def same_addresses(lib, base, src, n, parse, level, rounds):
    """(a): {variant: timing} for the strided call(s) and the indexed call over the same n blocks"""
    import torch
    st = torch.cuda.current_stream().cuda_stream
    cap = bound(BLOCK)
    stride = (cap + 15) // 16 * 16
    i64 = torch.arange(n, dtype=torch.int64, device="cuda")
    soff, doff = i64 * BLOCK, i64 * stride
    ssz = torch.full((n,), BLOCK, dtype=torch.int32, device="cuda")
    caps = torch.full((n,), cap, dtype=torch.int32, device="cuda")
    ws = None
    if parse == HC:
        ws = torch.empty(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n)), dtype=torch.uint8, device="cuda")
    param = level if parse == HC else 1

    def strided(L, dst, out, sizes=None):
        if parse == HC:
            return lambda: L.LZ4B200_compress_blocks_hc(src.data_ptr(), BLOCK, None, BLOCK, dst.data_ptr(), stride,
                                                        cap, level, out.data_ptr(), n, ws.data_ptr(), ws.numel(), st)
        fn = L.LZ4B200_compress_blocks if parse == FAST else L.LZ4B200_compress_blocks_parallel
        return lambda: fn(src.data_ptr(), BLOCK, sizes, BLOCK, dst.data_ptr(), stride, cap, 1, out.data_ptr(), n, st)

    def indexed(dst, out):
        return lambda: lib.LZ4B200_compress_blocks_indexed(
            src.data_ptr(), soff.data_ptr(), ssz.data_ptr(), dst.data_ptr(), doff.data_ptr(), caps.data_ptr(),
            out.data_ptr(), n, parse, param, ws.data_ptr() if ws is not None else None,
            ws.numel() if ws is not None else 0, st)

    variants = {}
    names = (["baseline_strided"] if base is not None else []) + ["strided", "indexed"]
    if parse == PARALLEL:           # with per-block sizes the strided call launches both kernels, as the indexed call does
        names.append("strided_with_sizes")
    for name in names:
        dst = torch.empty(n * stride, dtype=torch.uint8, device="cuda")
        out = torch.empty(n, dtype=torch.int32, device="cuda")
        if name == "indexed":
            fn = indexed(dst, out)
        else:
            fn = strided(base if name == "baseline_strided" else lib, dst, out,
                         ssz.data_ptr() if name == "strided_with_sizes" else None)
        variants[name] = (fn, dst, out)
    for fn, _, _ in variants.values():                      # warm-up, and every variant's result against the first
        assert fn() == 0
    torch.cuda.synchronize()
    first = next(iter(variants.values()))
    for name, (_, dst, out) in variants.items():
        assert torch.equal(out, first[2]), name + ": sizes differ"
        for i in range(0, n, max(n // 64, 1)):
            r = int(out[i])
            assert torch.equal(dst[i * stride:i * stride + r], first[1][i * stride:i * stride + r]), name + ": bytes"
    times = {k: [] for k in variants}
    for r in range(rounds):
        order = list(variants) if r % 2 == 0 else list(reversed(list(variants)))
        for name in order:
            times[name].append(event_ms(variants[name][0]))
    res = {k: summary(v) for k, v in times.items()}
    res.update(blocks=n, input_gbps_indexed=round(n * BLOCK / res["indexed"]["median_ms"] / 1e6, 2),
               ratio=round(n * BLOCK / float(first[2].sum()), 4))
    if base is not None:
        res["strided_vs_baseline_pct"] = round(100.0 * (res["strided"]["median_ms"] / res["baseline_strided"]["median_ms"]
                                                        - 1.0), 2)
    for k in ("strided", "strided_with_sizes"):
        if k in res:
            res["indexed_vs_%s_pct" % k] = round(100.0 * (res["indexed"]["median_ms"] / res[k]["median_ms"] - 1.0), 2)
    return res


def mixed_buffers(lib, orc, n, parse, rounds):
    """(b): one indexed call over n buffers of log-uniform sizes against one strided call over a padded copy"""
    import torch
    st = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(16384)
    sizes = np.exp(rng.uniform(np.log(512), np.log(1 << 20), n)).astype(np.int64)
    total, largest = int(sizes.sum()), int(sizes.max())
    host = orc.datagen_mt(total, SEG, 0.5, 7, os.cpu_count() or 1)
    soff = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    caps = np.array([bound(int(s)) for s in sizes], np.int64)
    doff = np.concatenate([[0], np.cumsum(caps)[:-1]])
    src = torch.from_numpy(host).cuda()
    t = lambda a, d: torch.from_numpy(np.ascontiguousarray(a, dtype=d)).cuda()
    soff_t, ssz, doff_t, caps_t = t(soff, np.int64), t(sizes, np.int32), t(doff, np.int64), t(caps, np.int32)
    dst = torch.empty(int(caps.sum()), dtype=torch.uint8, device="cuda")
    out = torch.empty(n, dtype=torch.int32, device="cuda")
    call = lambda: lib.LZ4B200_compress_blocks_indexed(src.data_ptr(), soff_t.data_ptr(), ssz.data_ptr(), dst.data_ptr(),
                                                      doff_t.data_ptr(), caps_t.data_ptr(), out.data_ptr(), n, parse, 1,
                                                      None, 0, st)
    pad_slot = (bound(largest) + 15) // 16 * 16
    res = {"buffers": n, "input_bytes": total, "largest": largest, "indexed_out_bytes": int(caps.sum()),
           "strided_out_bytes": n * pad_slot, "strided_src_copy_bytes": n * largest}
    assert call() == 0
    times = {"indexed": []}
    free, _ = torch.cuda.mem_get_info()
    scall = None
    if free > n * largest + n * pad_slot + (2 << 30):
        padded = torch.zeros(n * largest, dtype=torch.uint8, device="cuda")
        for i in range(n):                                   # the copy a strided caller makes
            padded[i * largest:i * largest + int(sizes[i])] = src[int(soff[i]):int(soff[i]) + int(sizes[i])]
        sdst = torch.empty(n * pad_slot, dtype=torch.uint8, device="cuda")
        sout = torch.empty(n, dtype=torch.int32, device="cuda")
        fn = lib.LZ4B200_compress_blocks if parse == FAST else lib.LZ4B200_compress_blocks_parallel
        scall = lambda: fn(padded.data_ptr(), largest, ssz.data_ptr(), largest, sdst.data_ptr(), pad_slot,
                           bound(largest), 1, sout.data_ptr(), n, st)
        assert scall() == 0
        torch.cuda.synchronize()
        assert torch.equal(sout, out), "strided and indexed sizes differ"
        times["strided_padded"] = []
    else:
        res["strided_padded"] = "not run: %.1f GiB free" % (free / 2 ** 30)
    for r in range(rounds):
        times["indexed"].append(event_ms(call))
        if scall is not None:
            times["strided_padded"].append(event_ms(scall))
    res.update({k: summary(v) for k, v in times.items()})
    res["input_gbps_indexed"] = round(total / res["indexed"]["median_ms"] / 1e6, 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=65536)
    ap.add_argument("--hc-blocks", type=int, default=4096)
    ap.add_argument("--buffers", type=int, default=16384)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--baseline-lib", default=None, help="liblz4_b200.so of an earlier commit: its strided calls are timed too")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()

    import torch
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle

    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "needs a CUDA device"
    base = load_baseline(args.baseline_lib) if args.baseline_lib else None
    orc = Oracle()
    host = orc.datagen_mt(args.blocks * BLOCK, SEG, 0.5, 0, os.cpu_count() or 1)
    src = torch.from_numpy(host).cuda()
    result = {"card": card(), "rounds": args.rounds}
    result["fast"] = same_addresses(lib, base, src, args.blocks, FAST, 0, args.rounds)
    result["parallel"] = same_addresses(lib, base, src, args.blocks, PARALLEL, 0, args.rounds)
    result["hc9"] = same_addresses(lib, base, src, min(args.hc_blocks, args.blocks), HC, 9, max(args.rounds // 2, 3))
    del src
    torch.cuda.empty_cache()
    result["mixed_fast"] = mixed_buffers(lib, orc, args.buffers, FAST, args.rounds)
    torch.cuda.empty_cache()
    result["mixed_parallel"] = mixed_buffers(lib, orc, args.buffers, PARALLEL, args.rounds)
    result["card_after"] = card()
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
