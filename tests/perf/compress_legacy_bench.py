#!/usr/bin/env python
"""Time LZ4B200_compress_legacy.  Prints one JSON line.

(1) One file of 1 GiB and one of 4 GiB of datagen P50 at level 1, against LZ4B200_compress_frames at block size ID 7 on
    the same bytes.
(2) 1 024 files of 1 MiB at levels 1 and 9, against compress_frames at block size ID 7 (1 MB blocks, one per frame).
(3) One 8 MiB P50 chunk at level 3: one thread parses it.
(4) Where oracle/_ref/lz4 exists, the reference tool's `lz4 -l -T0` on the host's threads: the 1 GiB file at -1 and the
    1 024 files, concatenated, at -9; and the 8 MiB chunk at -3.
The variants of a workload alternate within every round; each reports the median and min .. max of its rounds (CUDA
events around the device calls, a host clock around the tool).  Every legacy stream is checked to decode to its
source through decompress_files.  Card name, power limit and SM clock are read in the same run.

    python tests/perf/compress_legacy_bench.py [--rounds 5] [--hc-rounds 2] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "perf")]

from compress_indexed_bench import card, event_ms, summary  # noqa: E402

CHUNK = 8 << 20
LZ4 = os.path.join(ROOT, "oracle", "_ref", "lz4")


def legacy_bound(n):
    full, last = divmod(n, CHUNK)
    return 4 + full * (4 + CHUNK + CHUNK // 255 + 16) + (4 + last + last // 255 + 16 if last else 0)


class Case:
    """one workload's buffers: len(sizes) sources of src, written by the legacy call and by compress_frames"""

    def __init__(self, src, sizes, level):
        import torch
        from lz4_b200 import _lib, batch
        self.batch, self.level, self.src = batch, level, src
        dev = src.device
        n = len(sizes)
        self.n = n
        self.offs = torch.tensor(np.concatenate([[0], np.cumsum(sizes)[:-1]]), dtype=torch.int64, device=dev)
        self.sizes = torch.tensor(sizes, dtype=torch.int64, device=dev)
        caps = [legacy_bound(s) for s in sizes]
        self.caps = torch.tensor(caps, dtype=torch.int64, device=dev)
        self.doffs = torch.tensor(np.concatenate([[0], np.cumsum(caps)[:-1]]), dtype=torch.int64, device=dev)
        self.out = torch.empty(sum(caps) + 16, dtype=torch.uint8, device=dev)
        self.res = torch.empty(n, dtype=torch.int64, device=dev)
        self.budget = sum((s + CHUNK - 1) // CHUNK for s in sizes)
        self.ws = torch.empty(batch.compress_legacy_workspace_bytes(n, self.budget, level), dtype=torch.uint8,
                              device=dev)
        lib = _lib.load()
        fb = [0, 0, 0, 0]
        fcaps = []
        for s in sizes:
            b = 4
            while b < 7 and s > 1 << (8 + 2 * b):
                b += 1
            fb[b - 4] += (s + (1 << (8 + 2 * b)) - 1) >> (8 + 2 * b)
            fcaps.append(int(lib.LZ4B200_compressFrameBound(s, b)))
        self.fbudget = fb
        self.fcaps = torch.tensor(fcaps, dtype=torch.int64, device=dev)
        self.fdoffs = torch.tensor(np.concatenate([[0], np.cumsum(fcaps)[:-1]]), dtype=torch.int64, device=dev)
        self.fout = torch.empty(sum(fcaps) + 16, dtype=torch.uint8, device=dev)
        self.fres = torch.empty(n, dtype=torch.int64, device=dev)
        self.fws = torch.empty(batch.compress_frames_workspace_bytes(n, fb, level), dtype=torch.uint8, device=dev)

    def legacy(self):
        self.batch.compress_legacy(self.src, self.offs, self.sizes, max_blocks=self.budget, level=self.level,
                                   out=self.out, out_offsets=self.doffs, capacities=self.caps, results=self.res,
                                   workspace=self.ws)

    def frames(self):
        self.batch.compress_frames(self.src, self.offs, self.sizes, max_blocks=self.fbudget, block_size_id=7,
                                   level=self.level, out=self.fout, out_offsets=self.fdoffs, capacities=self.fcaps,
                                   results=self.fres, workspace=self.fws)

    def check(self):
        """every stream decodes to its source through decompress_files; returns the total stream bytes"""
        import torch
        r = self.res.cpu().numpy()
        assert (r > 0).all(), r[r <= 0][:4]
        dec, dres, _, _ = self.batch.decompress_files(self.out, self.doffs, self.res, self.sizes, max_units=self.n,
                                                      max_blocks=[0, 0, 0, 0, self.budget])
        torch.cuda.synchronize()
        assert torch.equal(dres, self.sizes)
        assert torch.equal(dec[:self.src.numel()], self.src[:int(self.sizes.sum())])
        del dec
        return int(r.sum())


def alternate(case, rounds, frames=True):
    legacy, fr = [], []
    for _ in range(rounds):
        legacy.append(event_ms(case.legacy))
        if frames:
            fr.append(event_ms(case.frames))
    out = {"legacy": summary(legacy), "stream_bytes": case.check()}
    if frames:
        out["compress_frames_bsid7"] = summary(fr)
    return out


def tool(args_, data, rounds):
    """the reference tool on `data` from a file, output discarded: {median, min .. max} of a host clock"""
    if not os.path.exists(LZ4):
        return None
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "in.bin")
        data.tofile(path)
        ms = []
        for _ in range(rounds):
            t0 = time.perf_counter()
            subprocess.run([LZ4, "-q", "-f", "-l", "-c"] + args_ + [path], stdout=subprocess.DEVNULL, check=True)
            ms.append(1000 * (time.perf_counter() - t0))
    return dict(summary(ms), args=args_, host_threads=os.cpu_count())


def run(args):
    import torch
    from oracle.pyoracle import Oracle
    orc = Oracle()
    dev = "cuda:0"
    res = {"gpu": card(), "rounds": args.rounds, "hc_rounds": args.hc_rounds}
    gib = 1 << 30
    host = orc.datagen_mt(gib, 1 << 20, 0.5, 0)
    src1 = torch.from_numpy(host).to(dev)

    case = Case(src1, [gib], 1)
    case.legacy(), case.frames()
    res["one_1GiB_file_level1"] = alternate(case, args.rounds)
    del case
    src4 = src1.repeat(4)
    case = Case(src4, [4 * gib], 1)
    case.legacy(), case.frames()
    res["one_4GiB_file_level1"] = alternate(case, max(args.rounds - 2, 1))
    del case, src4
    torch.cuda.empty_cache()

    for level, rounds in ((1, args.rounds), (9, args.hc_rounds)):
        case = Case(src1, [1 << 20] * 1024, level)
        if level == 1:
            case.legacy(), case.frames()
        res["1024_files_1MiB_level%d" % level] = alternate(case, rounds)
        del case
        torch.cuda.empty_cache()

    chunk = Case(src1[:CHUNK].clone(), [CHUNK], 3)
    res["one_8MiB_chunk_level3"] = alternate(chunk, 1, frames=False)
    del chunk

    res["tool"] = {"1GiB_-1": tool(["-1", "-T0"], host, args.rounds),
                   "1024x1MiB_concatenated_-9": tool(["-9", "-T0"], host, args.hc_rounds),
                   "8MiB_-3": tool(["-3", "-T0"], host[:CHUNK], args.rounds)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--hc-rounds", type=int, default=2)
    ap.add_argument("--out")
    args = ap.parse_args()
    res = run(args)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
