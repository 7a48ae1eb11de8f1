#!/usr/bin/env python
"""Time LZ4B200_compress_frames_host and LZ4B200_compress_legacy_host.  Prints one JSON line.

(a) One 4 GiB datagen P50 file at level 1, block size ID 7, no checksums, against LZ4B200_compressFrame_host on the same
    bytes (whose frame must be the same bytes); and the sweep of the group size G over 64, 256, 512 and 1024 MiB, each
    in a child process (the size is read once per process).
(b) The same file with the content checksum, the `lz4` tool's default: one frame's content is hashed by one warp.
(c) 65 536 files of 64 KB with the defaults, against doing it by hand: H2D, compress_frames_checksummed, D2H.
(d) One 1 GiB legacy file, against doing it by hand with compress_legacy.
Pinned and pageable host memory (source and destination alike), the variants of a workload alternating within every
round; medians and min .. max of a host clock around each synchronous call.  Card name, power limit and SM clock are
read in the same run.

    python tests/perf/compress_files_host_bench.py [--rounds 5] [--out FILE] [--sweep 64,256,512,1024]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "perf")]

from compress_indexed_bench import card, summary  # noqa: E402

GIB = 1 << 30


def host_buffers(nbytes, pinned):
    import torch
    t = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=pinned)
    return t, t.numpy()


def frames_call(lib, src, offs, sizes, dst, doffs, caps, bsid=7, level=1, bsum=0, csum=0, legacy=False):
    n = len(offs)
    res = np.zeros(n, dtype=np.int64)
    t0 = time.perf_counter()
    if legacy:
        rc = lib.LZ4B200_compress_legacy_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, dst.ctypes.data,
                                              doffs.ctypes.data, caps.ctypes.data, res.ctypes.data, n, level)
    else:
        rc = lib.LZ4B200_compress_frames_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, dst.ctypes.data,
                                              doffs.ctypes.data, caps.ctypes.data, res.ctypes.data, n, bsid, level, 0,
                                              0, bsum, csum)
    ms = 1000 * (time.perf_counter() - t0)
    assert rc == 0 and (res > 0).all(), lib.LZ4B200_last_cuda_error()
    return ms, res


def one(a):
    return np.array([a], dtype=np.int64)


def big_file(lib, rounds, with_frame_host):
    """(a) or, with the content checksum, (b) on the 4 GiB file: {pinned, pageable}"""
    from oracle.pyoracle import Oracle
    data = Oracle().datagen_mt(4 * GIB, 1 << 20, 0.5, 0)
    out = {}
    bufs = {}
    for pinned in (True, False):
        t, s = host_buffers(4 * GIB, pinned)
        s[:] = data
        cap = max(int(lib.LZ4B200_compressFrameBound_checksummed(4 * GIB, 7, 0, 1)),
                  int(lib.LZ4B200_compressFrameBound(4 * GIB, 7)))          # (the latter is the one-shot call's own)
        dt, d = host_buffers(cap, pinned)
        bufs[pinned] = (t, s, dt, d, cap)
    del data
    for csum, key in ((0, "a"), (1, "b")):
        if csum and not with_frame_host:
            continue
        ms = {True: [], False: []}
        ms_fh = {True: [], False: []}
        for r in range(rounds + 1):
            for pinned in (True, False):
                _, s, _, d, cap = bufs[pinned]
                t, res = frames_call(lib, s, one(0), one(4 * GIB), d, one(0), one(cap), csum=csum)
                if r:
                    ms[pinned].append(t)
                if with_frame_host and not csum:
                    fh = np.empty(cap, dtype=np.uint8) if r == 0 and not pinned else None
                    t0 = time.perf_counter()
                    n = lib.LZ4B200_compressFrame_host(s.ctypes.data, 4 * GIB, (fh if fh is not None else d).ctypes.data,
                                                       cap, 7, 1, 0)
                    tt = 1000 * (time.perf_counter() - t0)
                    assert n == res[0], (n, res[0])
                    if fh is not None:
                        frames_call(lib, s, one(0), one(4 * GIB), d, one(0), one(cap))
                        assert np.array_equal(fh[:n], d[:n]), "compressFrame_host wrote other bytes"
                    if r:
                        ms_fh[pinned].append(tt)
        out[key] = {}
        for pinned in (True, False):
            e = {"files_host": summary(ms[pinned]), "GB_per_s": round(4 * GIB / np.median(ms[pinned]) / 1e6, 2)}
            if ms_fh[pinned]:
                e["compressFrame_host"] = summary(ms_fh[pinned])
                e["compressFrame_host_GB_per_s"] = round(4 * GIB / np.median(ms_fh[pinned]) / 1e6, 2)
            out[key]["pinned" if pinned else "pageable"] = e
    return out


def run(args):
    import torch
    from lz4_b200 import _lib, batch
    lib = _lib.load()
    res = {"gpu": card(), "rounds": args.rounds,
           "G_MiB": int(os.environ.get("LZ4B200_HOST_WRITE_MB", "0")) or "default"}
    if args.only_a:
        res.update(big_file(lib, args.rounds, False))
        return res
    res.update({k + "_4GiB_P50": v for k, v in big_file(lib, args.rounds, True).items()})
    torch.cuda.empty_cache()
    from oracle.pyoracle import Oracle
    print(json.dumps(res), file=sys.stderr, flush=True)
    data = Oracle().datagen_mt(4 * GIB, 1 << 20, 0.5, 1)

    # (c) 65 536 files of 64 KB with the defaults
    n = 65536
    sizes = np.full(n, 65536, dtype=np.int64)
    offs = np.arange(n, dtype=np.int64) * 65536
    cap1 = int(lib.LZ4B200_compressFrameBound_checksummed(65536, 7, 0, 1))
    caps = np.full(n, cap1, dtype=np.int64)
    doffs = np.arange(n, dtype=np.int64) * cap1
    out = {}
    d_src = torch.empty(n * 65536 + 32, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(n * cap1, dtype=torch.uint8, device="cuda")
    d_offs, d_sizes = torch.from_numpy(offs + 16).cuda(), torch.from_numpy(sizes).cuda()
    d_caps, d_doffs = torch.from_numpy(caps).cuda(), torch.from_numpy(doffs).cuda()
    budget = [n, 0, 0, 0]
    ws = torch.empty(batch.compress_frames_workspace_bytes(n, budget, 1), dtype=torch.uint8, device="cuda")
    bufs = {}
    for pinned in (True, False):
        _, s = host_buffers(n * 65536, pinned)
        s[:] = data[:n * 65536]
        _, d = host_buffers(n * cap1, pinned)
        bufs[pinned] = (s, d)
    ms = {(p, w): [] for p in (True, False) for w in ("files_host", "by_hand")}
    for r in range(args.rounds + 1):
        for pinned in (True, False):
            s, d = bufs[pinned]
            t, got = frames_call(lib, s, offs, sizes, d, doffs, caps, csum=1)
            if r:
                ms[(pinned, "files_host")].append(t)
            hs, hd = torch.from_numpy(s), torch.from_numpy(d)
            t0 = time.perf_counter()
            d_src[16:16 + n * 65536].copy_(hs, non_blocking=pinned)
            _, hres = batch.compress_frames_checksummed(d_src, d_offs, d_sizes, max_blocks=budget, block_size_id=7,
                                                        level=1, out=d_out, out_offsets=d_doffs, capacities=d_caps,
                                                        workspace=ws)
            hd.copy_(d_out, non_blocking=pinned)
            torch.cuda.synchronize()
            if r:
                ms[(pinned, "by_hand")].append(1000 * (time.perf_counter() - t0))
            if r == 0:
                assert (hres.cpu().numpy() == got).all()
    for pinned in (True, False):
        out["pinned" if pinned else "pageable"] = {w: summary(ms[(pinned, w)]) for w in ("files_host", "by_hand")}
    res["c_65536_files_64KB"] = out
    print(json.dumps(out), file=sys.stderr, flush=True)
    del d_src, d_out, ws, bufs
    torch.cuda.empty_cache()

    # (d) one 1 GiB legacy file
    lcap = int(lib.LZ4B200_compressLegacyBound(GIB))
    d_src = torch.empty(GIB + 32, dtype=torch.uint8, device="cuda")
    d_out = torch.empty(lcap, dtype=torch.uint8, device="cuda")
    z = torch.zeros(1, dtype=torch.int64, device="cuda")
    lsz, lcaps = z + GIB, z + lcap
    lws = torch.empty(batch.compress_legacy_workspace_bytes(1, 128, 1), dtype=torch.uint8, device="cuda")
    bufs = {}
    for pinned in (True, False):
        _, s = host_buffers(GIB, pinned)
        s[:] = data[:GIB]
        _, d = host_buffers(lcap, pinned)
        bufs[pinned] = (s, d)
    ms = {(p, w): [] for p in (True, False) for w in ("files_host", "by_hand")}
    for r in range(args.rounds + 1):
        for pinned in (True, False):
            s, d = bufs[pinned]
            t, got = frames_call(lib, s, one(0), one(GIB), d, one(0), one(lcap), legacy=True)
            if r:
                ms[(pinned, "files_host")].append(t)
            hs, hd = torch.from_numpy(s), torch.from_numpy(d)
            t0 = time.perf_counter()
            d_src[:GIB].copy_(hs, non_blocking=pinned)
            _, lres = batch.compress_legacy(d_src, z, lsz, max_blocks=128, level=1, out=d_out, out_offsets=z,
                                            capacities=lcaps, workspace=lws)
            hd.copy_(d_out, non_blocking=pinned)
            torch.cuda.synchronize()
            if r:
                ms[(pinned, "by_hand")].append(1000 * (time.perf_counter() - t0))
            if r == 0:
                assert int(lres[0]) == int(got[0])
    res["d_1GiB_legacy"] = {("pinned" if p else "pageable"): {w: summary(ms[(p, w)]) for w in ("files_host", "by_hand")}
                            for p in (True, False)}

    # the G sweep on (a), one child process per size
    sweep = {}
    for mb in [int(x) for x in args.sweep.split(",") if x]:
        env = dict(os.environ, LZ4B200_HOST_WRITE_MB=str(mb))
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--only-a", "--rounds", str(args.rounds)],
                           env=env, capture_output=True, text=True, timeout=3000)
        assert p.returncode == 0, p.stderr[-3000:]
        sweep[mb] = json.loads(p.stdout.strip().splitlines()[-1])["a"]
    res["a_sweep_G_MiB"] = sweep
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    ap.add_argument("--sweep", default="64,256,512,1024")
    ap.add_argument("--only-a", action="store_true", help="(a) alone, for the sweep's children")
    args = ap.parse_args()
    line = json.dumps(run(args))
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
