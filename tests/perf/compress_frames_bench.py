#!/usr/bin/env python
"""Time LZ4B200_compress_frames against the block calls it is built from.  Prints one JSON line.

(1) 65 536 one-block frames of 64 KB datagen P50 (bench.py's data) at FAST and PARALLEL, against compress_buffers on
    the same blocks (capacity size - 1, as the frame call compresses them) + pack_blocks(slot_offsets=, header_bytes=4).
(2) One frame of 4 GiB at block size ID 7: the device call from device memory, against LZ4B200_compressFrame_host from
    pinned host memory (its PCIe pipeline included) and, where oracle/_ref exists, the reference's LZ4F_compressFrame on
    every host thread (one frame per thread over an equal share of the source).
(3) 4 096 one-block frames of 64 KB at HC level 9, against compress_blocks_hc on the same blocks.
The variants of a workload alternate within every round; each reports the median and min .. max of its rounds (CUDA
events around the device calls, a host clock around the host calls).  The frames are checked to decode to their
source.  Card name, power limit and SM clock are read in the same run.

    python tests/perf/compress_frames_bench.py [--rounds 5] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "perf")]

from compress_indexed_bench import card, event_ms, summary  # noqa: E402

BLOCK = 65536


def run(args):
    import torch
    from lz4_b200 import _lib, batch
    from oracle.pyoracle import Oracle, have_reference
    lib = _lib.load()
    orc = Oracle()
    dev = "cuda:0"
    res = {"gpu": card(), "rounds": args.rounds}

    # (1) 65 536 one-block frames
    n = args.frames
    host = orc.datagen_mt(n * BLOCK, 1 << 20, 0.5, 0)
    src = torch.from_numpy(host).to(dev)
    offs = torch.arange(n, dtype=torch.int64, device=dev) * BLOCK
    sz64 = torch.full((n,), BLOCK, dtype=torch.int64, device=dev)
    sz32 = sz64.to(torch.int32)
    budget = [n, 0, 0, 0]
    cap = lib.LZ4B200_compressFrameBound(BLOCK, 4)
    caps = torch.full((n,), cap, dtype=torch.int64, device=dev)
    doffs = torch.arange(n, dtype=torch.int64, device=dev) * cap + 16     # 16 readable bytes around every frame
    out = torch.empty(n * cap + 32, dtype=torch.uint8, device=dev)
    fres = torch.empty(n, dtype=torch.int64, device=dev)
    ws = torch.empty(batch.compress_frames_workspace_bytes(n, budget, 0), dtype=torch.uint8, device=dev)
    bcap = torch.full((n,), BLOCK - 1, dtype=torch.int32, device=dev)
    slot_off = torch.arange(n, dtype=torch.int64, device=dev) * BLOCK
    slots = torch.empty(n * BLOCK + 16, dtype=torch.uint8, device=dev)
    bsz = torch.empty(n, dtype=torch.int32, device=dev)
    packed = torch.empty(n * (BLOCK + 4) + 16, dtype=torch.uint8, device=dev)

    def frames(par):
        return lambda: batch.compress_frames(src, offs, sz64, max_blocks=budget, out=out, out_offsets=doffs,
                                             capacities=caps, results=fres, workspace=ws, parallel=par)

    def blocks(parse):
        def go():
            batch.compress_buffers(src, offs, sz32, parse=parse, out=slots, out_offsets=slot_off, capacities=bcap,
                                   out_sizes=bsz)
            batch.pack_blocks(slots, None, bsz, header_bytes=4, packed=packed, slot_offsets=slot_off)
        return go

    variants = {"frames_fast": frames(False), "blocks_pack_fast": blocks("fast"),
                "frames_parallel": frames(True), "blocks_pack_parallel": blocks("parallel")}
    ms = {k: [] for k in variants}
    for fn in variants.values():
        fn()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for k, fn in variants.items():
            ms[k].append(event_ms(fn))
    for par, parse in ((False, "fast"), (True, "parallel")):     # the frames hold what the block calls compute
        frames(par)()
        blocks(parse)()
        torch.cuda.synchronize()
        r = fres.cpu().numpy()
        assert (r > 0).all()
        dec, dres, _ = batch.decompress_frames(out, doffs, fres, torch.full((n,), BLOCK, dtype=torch.int64, device=dev),
                                               budget)
        assert bool((dres == BLOCK).all()) and torch.equal(dec, src)
    res["one_block_frames"] = {"frames": n, "bytes": n * BLOCK, **{k: summary(v) for k, v in ms.items()}}
    del out, slots, packed, ws

    # (3) HC level 9
    m = args.hc_frames
    hws = torch.empty(batch.compress_frames_workspace_bytes(m, [m, 0, 0, 0], 9), dtype=torch.uint8, device=dev)
    hout = torch.empty(m * cap + 32, dtype=torch.uint8, device=dev)
    hslots = torch.empty(m * BLOCK, dtype=torch.uint8, device=dev)
    hsz = torch.empty(m, dtype=torch.int32, device=dev)
    hbws = torch.empty(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(m)), dtype=torch.uint8, device=dev)
    hsrc = src[:m * BLOCK]
    hv = {"frames_hc9": lambda: batch.compress_frames(hsrc, offs[:m], sz64[:m], max_blocks=[m, 0, 0, 0], level=9,
                                                       out=hout, out_offsets=doffs[:m], capacities=caps[:m],
                                                       results=fres[:m], workspace=hws),
          "blocks_hc9": lambda: batch.compress_blocks_hc(hsrc, BLOCK, 9, slots=hslots, slot_stride=BLOCK,
                                                         slot_capacity=BLOCK - 1, out_sizes=hsz, workspace=hbws)}
    hms = {k: [] for k in hv}
    for fn in hv.values():
        fn()
    for _ in range(args.hc_rounds):
        for k, fn in hv.items():
            hms[k].append(event_ms(fn))
    res["hc9_frames"] = {"frames": m, **{k: summary(v) for k, v in hms.items()}}
    del hout, hslots, hws, hbws, src, host
    torch.cuda.empty_cache()

    # (2) one 4 GiB frame at block size ID 7
    big = 4 << 30
    bhost = torch.from_numpy(orc.datagen_mt(big, 1 << 20, 0.5, 3)).pin_memory()
    bsrc = bhost.to(dev)
    bcapv = int(lib.LZ4B200_compressFrameBound(big, 7))
    bbudget = [0, 0, 0, big >> 22]
    bout = torch.empty(bcapv, dtype=torch.uint8, device=dev)
    bws = torch.empty(batch.compress_frames_workspace_bytes(1, bbudget, 0), dtype=torch.uint8, device=dev)
    z = torch.zeros(1, dtype=torch.int64, device=dev)
    bsize = torch.tensor([big], dtype=torch.int64, device=dev)
    bcap = torch.tensor([bcapv], dtype=torch.int64, device=dev)
    bres = torch.empty(1, dtype=torch.int64, device=dev)
    hdst = torch.empty(bcapv, dtype=torch.uint8).pin_memory()

    def dev_frame():
        batch.compress_frames(bsrc, z, bsize, max_blocks=bbudget, block_size_id=7, out=bout, out_offsets=z,
                              capacities=bcap, results=bres, workspace=bws)

    def host_frame():
        t0 = time.perf_counter()
        r = lib.LZ4B200_compressFrame_host(bhost.data_ptr(), big, hdst.data_ptr(), bcapv, 7, 0, 0)
        assert r > 0
        return (time.perf_counter() - t0) * 1e3, r

    bms = {"device_frame": [], "host_frame_pinned": []}
    dev_frame()
    host_frame()
    for _ in range(args.big_rounds):
        bms["device_frame"].append(event_ms(dev_frame))
        bms["host_frame_pinned"].append(host_frame()[0])
    torch.cuda.synchronize()
    dlen = int(bres[0])
    hms_, hlen = host_frame()
    assert dlen == hlen and torch.equal(bout[:dlen].cpu(), hdst[:hlen]), "device and host frames differ"
    res["frame_4gib"] = {"bytes": big, "frame_bytes": dlen, **{k: summary(v) for k, v in bms.items()}}
    if have_reference():
        res["frame_4gib"]["reference_all_threads"] = reference_threads(bhost.numpy(), args.big_rounds)
    del bsrc, bout, bws
    return res


def reference_threads(src, rounds):
    """the reference's LZ4F_compressFrame on every host thread: thread k writes one frame of the k-th share"""
    from oracle.pyoracle import Reference
    lib = Reference().lib
    lib.LZ4F_compressFrame.restype = C.c_size_t
    lib.LZ4F_compressFrame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.LZ4F_compressFrameBound.restype = C.c_size_t
    lib.LZ4F_compressFrameBound.argtypes = [C.c_size_t, C.c_void_p]
    threads = os.cpu_count() or 1
    share = -(-len(src) // threads)
    prefs = (C.c_int * 16)()                            # LZ4F_preferences_t (lz4frame.h:192-198), 56 bytes: level 0
    prefs[0] = 7                                        # frameInfo.blockSizeID
    prefs[1] = 1                                        # frameInfo.blockMode = LZ4F_blockIndependent
    cap = int(lib.LZ4F_compressFrameBound(share, prefs))
    dsts = [np.empty(cap, dtype=np.uint8) for _ in range(threads)]
    base = src.ctypes.data

    def one(k):
        lo = k * share
        n = max(min(share, len(src) - lo), 0)
        lib.LZ4F_compressFrame(dsts[k].ctypes.data, cap, base + lo, n, prefs)

    ms = []
    for _ in range(rounds):
        ts = [threading.Thread(target=one, args=(k,)) for k in range(threads)]
        t0 = time.perf_counter()
        for th in ts:
            th.start()
        for th in ts:
            th.join()
        ms.append((time.perf_counter() - t0) * 1e3)
    return {"threads": threads, **summary(ms)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--hc-rounds", type=int, default=3)
    ap.add_argument("--big-rounds", type=int, default=3)
    ap.add_argument("--frames", type=int, default=65536)
    ap.add_argument("--hc-frames", type=int, default=4096)
    ap.add_argument("--out")
    args = ap.parse_args()
    res = run(args)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
