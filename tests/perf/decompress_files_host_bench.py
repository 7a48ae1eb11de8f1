#!/usr/bin/env python
"""Time LZ4B200_decompress_files_host.  Prints one JSON line.

(a) One file of one 4 GiB frame of 4 MB blocks (datagen P50, content checksum) with skipChecksums, against
    LZ4B200_decompress_blocks_host on the same blocks with tables built on the host: the same PCIe work.
(b) The same file, verified.
(c) 65 536 one-frame files of 64 KB, against doing it by hand: H2D, LZ4B200_decompress_files, D2H.
(d) One 1 GiB `lz4 -l` legacy file.
Each from pinned and from pageable host memory (source and destination alike), the variants of a workload alternating
within every round; medians and min .. max of a host clock around each synchronous call.  Every output is checked
against its source.  The files are written on the GPU by compress_frames_checksummed and compress_legacy.  Card name,
power limit and SM clock are read in the same run.

    python tests/perf/decompress_files_host_bench.py [--rounds 7] [--out FILE]
"""
import argparse
import json
import os
import struct
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "perf")]

from compress_indexed_bench import card, summary  # noqa: E402

GIB, MB4 = 1 << 30, 4 << 20


def host_buffers(nbytes, pinned):
    import torch
    t = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=pinned)
    return t, t.numpy()


def files_call(lib, src, offs, sizes, dst, doffs, caps, skip):
    n = len(offs)
    res, con, pre = (np.zeros(n, dtype=np.int64) for _ in range(3))
    t0 = time.perf_counter()
    rc = lib.LZ4B200_decompress_files_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, dst.ctypes.data,
                                           doffs.ctypes.data, caps.ctypes.data, res.ctypes.data, con.ctypes.data,
                                           pre.ctypes.data, n, skip, 0)
    ms = 1000 * (time.perf_counter() - t0)
    assert rc == 0, lib.LZ4B200_last_cuda_error()
    return ms, res


def frame_blocks(f):
    """(offsets, sizes) of the blocks of a frame without block checksums, walked on the host"""
    flg = f[4]
    ip = 7 + (8 if flg & 8 else 0)
    offs, sizes = [], []
    while True:
        w = struct.unpack_from("<I", f, ip)[0]
        ip += 4
        if w == 0:
            return np.array(offs, dtype=np.int64), np.array(sizes, dtype=np.int32)
        assert not w >> 31, "a stored-raw block: the blocks call would reject it"
        offs.append(ip)
        sizes.append(w)
        ip += w


def gpu_frames(src, sizes, bsid):
    """frames of consecutive pieces of the device tensor src, with content checksums, as one host array and offsets"""
    import torch
    from lz4_b200 import batch
    sz = torch.tensor(sizes, dtype=torch.int64, device="cuda")
    offs = torch.zeros_like(sz)
    offs[1:] = torch.cumsum(sz, 0)[:-1]
    out, res = batch.compress_frames_checksummed(src, offs, sz, block_size_id=bsid)[:2]
    torch.cuda.synchronize()
    r = res.cpu().numpy()
    assert (r > 0).all()
    o = out.cpu().numpy()
    caps = batch._frame_plan(sz, bsid, False, True)[1]
    starts = np.zeros(len(sizes), dtype=np.int64)
    starts[1:] = np.cumsum(caps)[:-1]
    parts = [o[s:s + n] for s, n in zip(starts, r)]
    return np.concatenate(parts), r.astype(np.int64)


def run(args):
    import torch
    from lz4_b200 import _lib, batch
    from oracle.pyoracle import Oracle
    lib = _lib.load()
    orc = Oracle()
    res = {"gpu": card(), "rounds": args.rounds}
    data = orc.datagen_mt(4 * GIB, 1 << 20, 0.5, 0)
    src = torch.from_numpy(data).cuda()

    # (a), (b): one 4 GiB frame of 4 MB blocks
    frame, flen = gpu_frames(src, [4 * GIB], 7)
    boffs, bsizes = frame_blocks(frame)
    nb = len(boffs)
    want = hash(data[::4093].tobytes())
    cases = {}
    for pinned in (True, False):
        t, s = host_buffers(len(frame) + 16, pinned)
        s[:len(frame)] = frame
        dt, d = host_buffers(4 * GIB, pinned)
        cases[pinned] = (t, s, dt, d)
    one = lambda a: np.array([a], dtype=np.int64)
    for skip, key in ((1, "a_4GiB_frame_4MB_blocks_skip"), (0, "b_4GiB_frame_4MB_blocks_verify")):
        out = {}
        for pinned in (True, False):
            _, s, _, d = cases[pinned]
            ms_files, ms_blocks = [], []
            rets = np.zeros(nb, dtype=np.int32)
            files_call(lib, s, one(0), one(len(frame)), d, one(0), one(4 * GIB), skip)       # warm-up
            lib.LZ4B200_decompress_blocks_host(s.ctypes.data, boffs.ctypes.data, bsizes.ctypes.data, d.ctypes.data, MB4,
                                               MB4, rets.ctypes.data, nb)
            for _ in range(args.rounds):
                ms, r = files_call(lib, s, one(0), one(len(frame)), d, one(0), one(4 * GIB), skip)
                assert r[0] == 4 * GIB
                ms_files.append(ms)
                if skip:
                    t0 = time.perf_counter()
                    rc = lib.LZ4B200_decompress_blocks_host(s.ctypes.data, boffs.ctypes.data, bsizes.ctypes.data,
                                                            d.ctypes.data, MB4, MB4, rets.ctypes.data, nb)
                    ms_blocks.append(1000 * (time.perf_counter() - t0))
                    assert rc == 0 and (rets == MB4).all()
            files_call(lib, s, one(0), one(len(frame)), d, one(0), one(4 * GIB), skip)
            assert hash(d[::4093].tobytes()) == want
            name = "pinned" if pinned else "pageable"
            out[name] = {"files_host": summary(ms_files), "GB_per_s": round(4 * GIB / np.median(ms_files) / 1e6, 2)}
            if skip:
                out[name]["decompress_blocks_host"] = summary(ms_blocks)
                out[name]["blocks_GB_per_s"] = round(4 * GIB / np.median(ms_blocks) / 1e6, 2)
        res[key] = out
    del cases, frame
    torch.cuda.empty_cache()

    # (c): 65 536 one-frame 64 KB files
    n = 65536
    files, flens = gpu_frames(src[:n * 65536], [65536] * n, 4)
    foffs = np.zeros(n, dtype=np.int64)
    foffs[1:] = np.cumsum(flens)[:-1]
    caps = np.full(n, 65536, dtype=np.int64)
    doffs = np.arange(n, dtype=np.int64) * 65536
    mu, mb = n, [n, 0, 0, 0, 0]
    out = {}
    for pinned in (True, False):
        _, s = host_buffers(len(files) + 16, pinned)
        s[:len(files)] = files
        _, d = host_buffers(n * 65536, pinned)
        dev_comp = torch.empty(len(files) + 32, dtype=torch.uint8, device="cuda")
        dev_out = torch.empty(n * 65536, dtype=torch.uint8, device="cuda")
        d_offs, d_sizes = torch.from_numpy(foffs + 16).cuda(), torch.from_numpy(flens).cuda()
        d_caps, d_doffs = torch.from_numpy(caps).cuda(), torch.from_numpy(doffs).cuda()
        ws = torch.empty(batch.decompress_files_workspace_bytes(n, mu, mb), dtype=torch.uint8, device="cuda")
        host_src = torch.from_numpy(s[:len(files)])
        host_dst = torch.from_numpy(d)

        def by_hand():
            t0 = time.perf_counter()
            dev_comp[16:16 + len(files)].copy_(host_src, non_blocking=pinned)
            _, r, _, _ = batch.decompress_files(dev_comp, d_offs, d_sizes, d_caps, mu, mb, out=dev_out,
                                                out_offsets=d_doffs, workspace=ws)
            host_dst.copy_(dev_out, non_blocking=pinned)
            torch.cuda.synchronize()
            return 1000 * (time.perf_counter() - t0), r
        ms_files, ms_hand = [], []
        for _ in range(args.rounds + 1):
            ms, r = files_call(lib, s, foffs, flens, d, doffs, caps, 0)
            assert (r == 65536).all()
            ms_files.append(ms)
            ms, r = by_hand()
            ms_hand.append(ms)
        assert hash(d[::4093].tobytes()) == hash(data[:n * 65536][::4093].tobytes())
        out["pinned" if pinned else "pageable"] = {"files_host": summary(ms_files[1:]), "by_hand": summary(ms_hand[1:])}
        del dev_comp, dev_out, ws
    res["c_65536_files_64KB"] = out
    torch.cuda.empty_cache()

    # (d): one 1 GiB legacy file
    sz = torch.tensor([GIB], dtype=torch.int64, device="cuda")
    lout, lres = batch.compress_legacy(src, torch.zeros(1, dtype=torch.int64, device="cuda"), sz)[:2]
    torch.cuda.synchronize()
    leg = lout[:int(lres[0])].cpu().numpy()
    out = {}
    for pinned in (True, False):
        _, s = host_buffers(len(leg) + 16, pinned)
        s[:len(leg)] = leg
        _, d = host_buffers(GIB, pinned)
        ms_l = []
        for _ in range(args.rounds + 1):
            ms, r = files_call(lib, s, one(0), one(len(leg)), d, one(0), one(GIB), 0)
            assert r[0] == GIB
            ms_l.append(ms)
        assert hash(d[::4093].tobytes()) == hash(data[:GIB][::4093].tobytes())
        out["pinned" if pinned else "pageable"] = {"files_host": summary(ms_l[1:]),
                                                   "GB_per_s": round(GIB / np.median(ms_l[1:]) / 1e6, 2)}
    res["d_1GiB_legacy"] = out
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
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
