#!/usr/bin/env python
"""Time LZ4B200_decompress_files_to_device and LZ4B200_compress_frames_from_device.  Prints one JSON line.

Reader, from a .lz4 file in host memory to its content in device memory, against (1) LZ4B200_decompress_files_host into
host memory followed by an H2D copy of its output and (2) an H2D copy of the file followed by LZ4B200_decompress_files
with its budget and workspace:
(a) one 4 GiB frame of 4 MB blocks (datagen P50, content checksum), skipChecksums;
(b) the same file, verified;
(c) 65 536 one-frame files of 64 KB.
Writer, from device memory to .lz4 files in host memory, level 1, -B7, against (1) a D2H copy of the source followed by
LZ4B200_compress_frames_host and (2) LZ4B200_compress_frames_checksummed followed by a D2H copy of its output:
(d) one 4 GiB device tensor, with and without the content checksum;
(e) 65 536 device buffers of 64 KB, with the content checksum.
Each from pinned and pageable host memory, the variants alternating within every round; medians and min .. max of a
host clock around each synchronous call.  Every output is checked.  Device memory per variant: the growth of used
device memory (torch.cuda.mem_get_info) over its first call, in the order the variants first run, plus the tensors the
variant holds.  Card name, power limit and SM clock are read in the same run.

    python tests/perf/files_device_io_bench.py [--rounds 5] [--workloads abcde] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests", "perf")]

from compress_indexed_bench import card, summary               # noqa: E402
from decompress_files_host_bench import gpu_frames, host_buffers  # noqa: E402

GIB, MIB = 1 << 30, 1 << 20


def used():
    import torch
    torch.cuda.synchronize()
    f, t = torch.cuda.mem_get_info()
    return t - f


def timed(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    r = fn()
    torch.cuda.synchronize()
    return 1000 * (time.perf_counter() - t0), r


def rounds_of(variants, rounds):
    """{name: (timings, device bytes)}: each variant's first call measures its memory growth, then rounds alternate"""
    mem, ms = {}, {k: [] for k in variants}
    for name, (fn, held) in variants.items():
        u = used()
        fn()
        mem[name] = used() - u + held
    for _ in range(rounds):
        for name, (fn, _) in variants.items():
            ms[name].append(timed(fn)[0])
    return {k: dict(summary(ms[k]), device_bytes=int(mem[k])) for k in variants}


def reader(lib, files, flens, out_bytes, per_file, skip, mu, mb, pinned, rounds):
    """the three reader variants over host files (concatenated, lengths flens) into out_bytes of device memory, each
    file per_file bytes; returns (timings, the device output of the new call)"""
    import torch
    from lz4_b200 import batch
    n = len(flens)
    foffs = np.zeros(n, dtype=np.int64)
    foffs[1:] = np.cumsum(flens)[:-1]
    caps = np.full(n, per_file, dtype=np.int64)
    doffs = np.arange(n, dtype=np.int64) * per_file
    _, s = host_buffers(len(files) + 16, pinned)
    s[:len(files)] = files
    _, h = host_buffers(out_bytes, pinned)
    res, con, pre = (np.zeros(n, dtype=np.int64) for _ in range(3))
    dev_out = torch.empty(out_bytes, dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    hdst = torch.from_numpy(h)

    def new():
        rc = lib.LZ4B200_decompress_files_to_device(s.ctypes.data, foffs.ctypes.data, flens.ctypes.data, dev_out.data_ptr(),
                                                    doffs.ctypes.data, caps.ctypes.data, res.ctypes.data, con.ctypes.data,
                                                    pre.ctypes.data, n, skip, st)
        assert rc == 0 and (res == per_file).all(), lib.LZ4B200_last_cuda_error()

    def host_then_h2d():
        rc = lib.LZ4B200_decompress_files_host(s.ctypes.data, foffs.ctypes.data, flens.ctypes.data, h.ctypes.data,
                                               doffs.ctypes.data, caps.ctypes.data, res.ctypes.data, con.ctypes.data,
                                               pre.ctypes.data, n, skip, 0)
        assert rc == 0 and (res == per_file).all()
        dev_out.copy_(hdst, non_blocking=pinned)

    comp = torch.empty(len(files) + 32, dtype=torch.uint8, device="cuda")
    d_offs, d_sizes = torch.from_numpy(foffs + 16).cuda(), torch.from_numpy(flens).cuda()
    d_caps, d_doffs = torch.from_numpy(caps).cuda(), torch.from_numpy(doffs).cuda()
    ws = torch.empty(batch.decompress_files_workspace_bytes(n, mu, mb), dtype=torch.uint8, device="cuda")
    host_src = torch.from_numpy(s[:len(files)])

    def h2d_then_device():
        comp[16:16 + len(files)].copy_(host_src, non_blocking=pinned)
        _, r, _, _ = batch.decompress_files(comp, d_offs, d_sizes, d_caps, mu, mb, bool(skip), out=dev_out,
                                            out_offsets=d_doffs, workspace=ws)
        assert bool((r == per_file).all())

    out = rounds_of({"to_device": (new, out_bytes), "host_then_h2d": (host_then_h2d, out_bytes),
                     "h2d_then_decompress_files": (h2d_then_device, out_bytes + comp.numel() + ws.numel())}, rounds)
    new()
    return out, dev_out


def writer(lib, src, offs, sizes, csum, pinned, rounds):
    """the three writer variants over device sources at src + offs; returns (timings, the new call's files)"""
    import torch
    from lz4_b200 import batch
    n = len(sizes)
    caps = np.array([lib.LZ4B200_compressFrameBound_checksummed(int(k), 7, 0, csum) for k in sizes], dtype=np.int64)
    doffs = np.zeros(n, dtype=np.int64)
    doffs[1:] = np.cumsum(caps)[:-1]
    _, h = host_buffers(int(caps.sum()), pinned)
    total = int(sizes.sum())
    _, hs = host_buffers(total, pinned)
    hsrc = torch.from_numpy(hs)
    soffs = np.zeros(n, dtype=np.int64)
    soffs[1:] = np.cumsum(sizes)[:-1]
    res = np.zeros(n, dtype=np.int64)
    st = torch.cuda.current_stream().cuda_stream
    contiguous = bool((offs == soffs).all())

    def new():
        rc = lib.LZ4B200_compress_frames_from_device(src.data_ptr(), offs.ctypes.data, sizes.ctypes.data, h.ctypes.data,
                                                     doffs.ctypes.data, caps.ctypes.data, res.ctypes.data, n, 7, 1, 0,
                                                     0, 0, csum, st)
        assert rc == 0 and (res > 0).all(), lib.LZ4B200_last_cuda_error()

    def d2h_then_host():
        assert contiguous
        hsrc.copy_(src[:total], non_blocking=pinned)
        torch.cuda.synchronize()
        rc = lib.LZ4B200_compress_frames_host(hs.ctypes.data, soffs.ctypes.data, sizes.ctypes.data, h.ctypes.data,
                                              doffs.ctypes.data, caps.ctypes.data, res.ctypes.data, n, 7, 1, 0, 0, 0,
                                              csum)
        assert rc == 0 and (res > 0).all()

    d_offs, d_sizes = torch.from_numpy(offs).cuda(), torch.from_numpy(sizes).cuda()
    d_doffs, d_caps = torch.from_numpy(doffs).cuda(), torch.from_numpy(caps).cuda()
    dev_out = torch.empty(int(caps.sum()), dtype=torch.uint8, device="cuda")
    hout = torch.from_numpy(h)
    budget = batch._frame_plan(d_sizes, 7, False, bool(csum))[0]
    ws = torch.empty(batch.compress_frames_workspace_bytes(n, budget, 1), dtype=torch.uint8, device="cuda")

    def device_then_d2h():
        _, r = batch.compress_frames_checksummed(src, d_offs, d_sizes, max_blocks=budget, block_size_id=7, level=1,
                                                 content_checksum=bool(csum), out=dev_out, out_offsets=d_doffs,
                                                 capacities=d_caps, workspace=ws)[:2]
        hout.copy_(dev_out, non_blocking=pinned)
        torch.cuda.synchronize()
        assert bool((r > 0).all())

    out = rounds_of({"from_device": (new, 0), "d2h_then_host": (d2h_then_host, 0),
                     "compress_frames_checksummed_then_d2h": (device_then_d2h, dev_out.numel() + ws.numel())}, rounds)
    new()
    return out, [h[o:o + r].tobytes() for o, r in zip(doffs[:4], res[:4])], res.copy()


def run(args):
    import torch
    from lz4_b200 import _lib, frame
    from oracle.pyoracle import Oracle
    lib = _lib.load()
    orc = Oracle()
    res = {"gpu": card(), "rounds": args.rounds}
    data = orc.datagen_mt(4 * GIB, 1 << 20, 0.5, 0)
    src = torch.from_numpy(data).cuda()
    want = hash(data[::4093].tobytes())

    big, blen = gpu_frames(src, [4 * GIB], 7) if set("ab") & set(args.workloads) else (None, None)
    for skip, key in ((1, "a_4GiB_frame_4MB_blocks_skip"), (0, "b_4GiB_frame_4MB_blocks_verify")):
        if key[0] not in args.workloads:
            continue
        res[key] = {}
        for pinned in (True, False):
            r, out = reader(lib, big, blen, 4 * GIB, 4 * GIB, skip, 1, [0, 0, 0, 1024, 0], pinned, args.rounds)
            assert hash(out.cpu().numpy()[::4093].tobytes()) == want
            res[key]["pinned" if pinned else "pageable"] = r
            del out
            torch.cuda.empty_cache()
    del big

    n = 65536
    small, slen = gpu_frames(src[:n * 65536], [65536] * n, 4) if "c" in args.workloads else (None, None)
    for pinned in (True, False) if "c" in args.workloads else ():
        res.setdefault("c_65536_files_64KB", {})
        r, out = reader(lib, small, slen, n * 65536, 65536, 0, n, [n, 0, 0, 0, 0], pinned, args.rounds)
        assert hash(out.cpu().numpy()[::4093].tobytes()) == want
        res["c_65536_files_64KB"]["pinned" if pinned else "pageable"] = r
        del out
        torch.cuda.empty_cache()
    del small

    one = lambda v: np.array([v], dtype=np.int64)                 # noqa: E731
    for csum in (1, 0):
        key = "d_4GiB_tensor_level1_B7_" + ("content_checksum" if csum else "no_checksum")
        for pinned in (True, False) if "d" in args.workloads else ():
            res.setdefault(key, {})
            r, files, _ = writer(lib, src, one(0), one(4 * GIB), csum, pinned, args.rounds)
            if pinned and csum:
                assert frame.decompress_file(files[0], 4 * GIB)[::4093] == data[::4093].tobytes()
            res[key]["pinned" if pinned else "pageable"] = r
            torch.cuda.empty_cache()
    offs = np.arange(n, dtype=np.int64) * 65536
    sizes = np.full(n, 65536, dtype=np.int64)
    for pinned in (True, False) if "e" in args.workloads else ():
        res.setdefault("e_65536_buffers_64KB", {})
        r, files, lens = writer(lib, src, offs, sizes, 1, pinned, args.rounds)
        assert frame.decompress_file(files[3]) == data[3 * 65536:4 * 65536].tobytes()
        res["e_65536_buffers_64KB"]["pinned" if pinned else "pageable"] = r
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--workloads", default="abcde", help="the workloads to run, a subset of abcde")
    ap.add_argument("--out")
    args = ap.parse_args()
    line = json.dumps(run(args))
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
