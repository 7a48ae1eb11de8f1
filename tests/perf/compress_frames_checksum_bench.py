#!/usr/bin/env python
"""Time LZ4B200_compress_frames_checksummed and the content hash it shares with LZ4B200_decompress_frames_checksummed.
Prints one JSON line.

Writer, the checksummed call against the checksum-free call on the same data (datagen P50), and the parent commit's
LZ4B200_compress_frames with --baseline-lib:
  (a) 65 536 one-block 64 KB frames with a content checksum,
  (b) one frame of 1 024 x 4 MB blocks at level 1 with a content checksum (the `lz4` tool's layout),
  (c) (a) with block checksums as well,
  (d) 1 024 frames of 4 MB each with a content checksum.
Decoder: LZ4B200_decompress_frames_checksummed verifying the frames of (a), (b) and (d), this library against
--baseline-lib.
Content hash threshold: the content-checksum kernel of the verifying decoder (torch.profiler) on 1 GiB of frames of
64 KB .. 4 MB, for every --variant library (label=path: builds of this tree with -DLZ4K_XXH_STAGED_MIN=0, every frame
by a warp, and a large value, every frame by one thread).
The variants of a workload alternate within every round; each reports the median and min .. max of its rounds (CUDA
events around one call).  Every frame's result is checked, and the checksummed frames decode and verify.  Card name,
power limit and SM clock are read in the same run.

    python tests/perf/compress_frames_checksum_bench.py [--rounds 5] [--baseline-lib PATH] [--variant L=PATH ...]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "perf")]

from compress_indexed_bench import card, event_ms, summary  # noqa: E402

NAMES = ("LZ4B200_compress_frames", "LZ4B200_compress_frames_checksummed", "LZ4B200_compress_frames_workspace_bytes",
         "LZ4B200_decompress_frames_checksummed", "LZ4B200_decompress_frames_workspace_bytes",
         "LZ4B200_compressFrameBound")


def load(path):
    from lz4_b200 import _lib
    lib = C.CDLL(os.path.abspath(path))
    for name, res, args in _lib.PROTOTYPES:
        if name in NAMES and hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
    return lib


def budget(v):
    return (C.c_int64 * 4)(*v)


class Frames:
    """nf frames of k blocks of block size ID bsid over one P50 source, written by `lib`; the buffers of every call"""

    def __init__(self, torch, orc, bsid, nf, k, dev):
        self.torch, self.bsid, self.nf = torch, bsid, nf
        bs = 1 << (8 + 2 * bsid)
        self.n = nf * k * bs
        self.src = torch.from_numpy(orc.datagen_mt(self.n, 1 << 20, 0.5, 0)).to(dev)
        self.offs = torch.arange(nf, dtype=torch.int64, device=dev) * (k * bs)
        self.sizes = torch.full((nf,), k * bs, dtype=torch.int64, device=dev)
        self.mb = [0, 0, 0, 0]
        self.mb[bsid - 4] = nf * k
        cap = 19 + 8 * k + k * bs + 8
        self.caps = torch.full((nf,), cap, dtype=torch.int64, device=dev)
        self.doffs = torch.arange(nf, dtype=torch.int64, device=dev) * cap + 16
        self.out = torch.empty(nf * cap + 32, dtype=torch.uint8, device=dev)
        self.res = torch.empty(nf, dtype=torch.int64, device=dev)
        self.ws = None

    def writer(self, lib, sums):
        """a call of lib's LZ4B200_compress_frames (sums None) or LZ4B200_compress_frames_checksummed"""
        t = self
        wb = int(lib.LZ4B200_compress_frames_workspace_bytes(t.nf, budget(t.mb), 1))
        if t.ws is None or t.ws.numel() < wb:
            t.ws = t.torch.empty(wb, dtype=t.torch.uint8, device=t.src.device)
        head = (t.src.data_ptr(), t.offs.data_ptr(), t.sizes.data_ptr(), t.out.data_ptr(), t.doffs.data_ptr(),
                t.caps.data_ptr(), t.res.data_ptr(), t.nf, t.bsid, 1, 0, 0)
        tail = (budget(t.mb), t.ws.data_ptr(), t.ws.numel(), t.torch.cuda.current_stream().cuda_stream)
        if sums is None:
            return lambda: lib.LZ4B200_compress_frames(*head, *tail)
        return lambda: lib.LZ4B200_compress_frames_checksummed(*head, *sums, *tail)

    def check_written(self, sums):
        r = self.res.cpu().numpy()
        assert (r > 0).all(), r[:8]
        if sums is not None and sums[1]:
            last = self.doffs.cpu().numpy() + r - 8
            end = self.out[self.torch.from_numpy(last).to(self.out.device)[:, None]
                           + self.torch.arange(4, device=self.out.device)].cpu().numpy()
            assert (end == 0).all()                             # the EndMark before the content checksum

    def decoder(self, lib):
        """a verifying LZ4B200_decompress_frames_checksummed of the frames last written (checked once)"""
        t, torch = self, self.torch
        dev = t.src.device
        if getattr(t, "dec", None) is None or not torch.equal(t.dec[1], t.res):     # buffers shared by every library
            wb = int(lib.LZ4B200_decompress_frames_workspace_bytes(t.nf, budget(t.mb)))
            t.dec = None
            t.dec = (t.out.clone(), t.res.clone(), torch.empty(t.n + 16, dtype=torch.uint8, device=dev),
                     torch.arange(t.nf, dtype=torch.int64, device=dev) * t.sizes[0],
                     torch.empty(t.nf, dtype=torch.int64, device=dev), torch.empty(t.nf, dtype=torch.int64, device=dev),
                     torch.empty(wb, dtype=torch.uint8, device=dev), wb)
        comp, dsizes, dout, doffs, res, cons, ws, wb = t.dec

        def go():
            rc = lib.LZ4B200_decompress_frames_checksummed(comp.data_ptr(), t.doffs.data_ptr(), dsizes.data_ptr(),
                                                           dout.data_ptr(), doffs.data_ptr(), t.sizes.data_ptr(),
                                                           res.data_ptr(), cons.data_ptr(), t.nf, budget(t.mb), 0,
                                                           ws.data_ptr(), wb, torch.cuda.current_stream().cuda_stream)
            assert rc == 0
        go()
        torch.cuda.synchronize()
        assert torch.equal(res, t.sizes) and torch.equal(cons, dsizes)
        assert torch.equal(dout[:t.n], t.src)
        return go


def rounds(torch, variants, n):
    ms = {k: [] for k in variants}
    for fn in variants.values():
        fn()
    torch.cuda.synchronize()
    for _ in range(n):
        for k, fn in variants.items():
            ms[k].append(event_ms(fn))
    return {k: summary(v) for k, v in ms.items()}


def content_kernel_ms(torch, fn, name):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return round(sum(e.device_time_total for e in prof.key_averages() if name in e.key) / 1e3, 3)


def run(args):
    import torch
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle
    orc = Oracle()
    dev = "cuda:0"
    new = load(_lib.LIB_PATH)
    base = load(args.baseline_lib) if args.baseline_lib else None
    out = {"gpu": card(), "rounds": args.rounds, "writer": {}, "decoder": {}, "threshold": {}}
    work = {"a": (4, 65536, 1, (0, 1)), "b": (7, 1, 1024, (0, 1)), "c": (4, 65536, 1, (1, 1)), "d": (7, 1024, 1, (0, 1))}
    for key in args.workloads:
        bsid, nf, k, sums = work[key]
        fr = Frames(torch, orc, bsid, nf, k, dev)
        fr.writer(new, sums)()
        torch.cuda.synchronize()
        fr.check_written(sums)
        variants = {"checksummed": fr.writer(new, sums), "checksum_free": fr.writer(new, None)}
        if base is not None:
            variants["parent_checksum_free"] = fr.writer(base, None)
        slow = key == "b"
        r = rounds(torch, variants, 3 if slow else args.rounds)
        for v in ("checksummed", "checksum_free"):
            r[v]["GBps"] = round(fr.n / r[v]["median_ms"] / 1e6, 2)
        r["content_sum_kernel_ms"] = content_kernel_ms(torch, variants["checksummed"], "lz4_cframes_content_sum")
        r["block_sum_kernel_ms"] = content_kernel_ms(torch, variants["checksummed"], "lz4_cframes_block_sum")
        out["writer"][key] = r
        print(key, "writer", json.dumps(r), flush=True)
        if key in ("a", "b", "d"):
            fr.writer(new, sums)()
            dv = {"this": fr.decoder(new)}
            if base is not None:
                dv["parent"] = fr.decoder(base)
            if slow and base is not None:               # the parent hashes 4 GiB on one thread: one call
                d = {"this": summary([event_ms(dv["this"]) for _ in range(3)]),
                     "parent": summary([event_ms(dv["parent"])])}
            else:
                d = rounds(torch, dv, 3 if slow else args.rounds)
            for v in dv:
                d[v]["content_sum_kernel_ms"] = content_kernel_ms(torch, dv[v], "lz4_frames_content_sum")
                d[v]["content_GBps"] = round(fr.n / d[v]["content_sum_kernel_ms"] / 1e6, 2)
            out["decoder"][key] = d
            print(key, "decoder", json.dumps(d), flush=True)
        del fr, variants
        torch.cuda.empty_cache()

    libs = {"this": new}
    for v in args.variant:
        label, path = v.split("=", 1)
        libs[label] = load(path)
    if len(libs) > 1:
        total = args.sweep_total
        for size in args.sweep_sizes:
            bsid = max(b for b in (4, 5, 6, 7) if 1 << (8 + 2 * b) <= min(size, 4 << 20))
            bs = 1 << (8 + 2 * bsid)
            fr = Frames(torch, orc, bsid, total // size, size // bs, dev)
            fr.writer(new, (0, 1))()
            torch.cuda.synchronize()
            row = {}
            calls = {label: fr.decoder(lib) for label, lib in libs.items()}
            for _ in range(args.rounds):
                for label, fn in calls.items():
                    row.setdefault(label, []).append(content_kernel_ms(torch, fn, "lz4_frames_content_sum"))
            out["threshold"][size] = {label: {"median_ms": float(np.median(v)), "min_ms": min(v), "max_ms": max(v)}
                                      for label, v in row.items()}
            print("threshold", size, json.dumps(out["threshold"][size]), flush=True)
            del fr, calls
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--baseline-lib")
    ap.add_argument("--variant", action="append", default=[])
    ap.add_argument("--workloads", default="abcd")
    ap.add_argument("--sweep-total", type=int, default=1 << 30, help="bytes of frames per size of the threshold sweep")
    ap.add_argument("--sweep-sizes", type=lambda v: [int(x) for x in v.split(",")],
                    default=[65536, 131072, 262144, 524288, 1 << 20, 2 << 20, 4 << 20])
    ap.add_argument("--out")
    args = ap.parse_args()
    res = run(args)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
