"""Time LZ4B200_decompress_frames_checksummed on checksummed frames in device memory, verifying and skipping the checksums,
against LZ4B200_decompress_frames on checksum-free frames holding the same blocks, in the same run:
  (a) 65 536 one-block frames of 64 KB datagen P50 with a content checksum,
  (b) one frame of 1 024 x 4 MB blocks with a content checksum (the layout of the reference `lz4` tool),
  (c) (a) with block checksums as well.
CUDA events, median of 10 calls after 2 warm-up calls (for (b), whose content checksum runs on one thread, the
verifying call is timed over 2 calls after 1); then one torch.profiler run per workload for the two checksum kernels and
the call's other frame kernels.  The frames are assembled on the host, with checksums from the host build of
lz4_frame_core.h's fc_xxh32 (tests/host_build.py).  Prints the card, its power limit and SM clocks.
Arguments: the workloads to run (default: a b c).
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from lz4_b200 import batch  # noqa: E402
from oracle.pyoracle import Oracle  # noqa: E402
import frame_corpus as fc  # noqa: E402
import host_build  # noqa: E402


def timed(fn, reps=10, warmup=2):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def frames_of(xxh, data, packed, offs, bsid, nf, k, block_sum, content_sum):
    """nf frames of k blocks each from the packed blocks ([LE32 header][payload] per block, at offs): the frame bytes on
    the host with 16 bytes of padding at both ends, the frame offsets and sizes"""
    bs = 1 << (8 + 2 * bsid)
    flg = (1 << 6) | (1 << 5) | ((1 << 4) if block_sum else 0) | ((1 << 2) if content_sum else 0)
    hdr = np.frombuffer(fc.header(flg, bsid << 4), dtype=np.uint8)
    blen = np.diff(offs)
    flen = 7 + blen.reshape(nf, k).sum(1) + (4 * k if block_sum else 0) + 4 + (4 if content_sum else 0)
    fpos = 16 + np.concatenate([[0], np.cumsum(flen)[:-1]])
    buf = np.zeros(16 + int(flen.sum()) + 16, dtype=np.uint8)
    for f in range(nf):
        p = int(fpos[f])
        buf[p:p + 7] = hdr
        p += 7
        for j in range(f * k, (f + 1) * k):
            blk = packed[offs[j]:offs[j + 1]]
            buf[p:p + len(blk)] = blk
            p += len(blk)
            if block_sum:
                buf[p:p + 4] = np.frombuffer(np.uint32(xxh(blk[4:].ctypes.data, len(blk) - 4, 0)).tobytes(), np.uint8)
                p += 4
        p += 4                                                   # EndMark
        if content_sum:
            c = data[f * k * bs:(f + 1) * k * bs]
            buf[p:p + 4] = np.frombuffer(np.uint32(xxh(c.ctypes.data, len(c), 0)).tobytes(), np.uint8)
    return buf, fpos.astype(np.int64), flen.astype(np.int64)


def run(name, orc, xxh, bsid, nf, k, block_sum, verify_reps=(10, 2)):
    bs = 1 << (8 + 2 * bsid)
    data = orc.datagen_mt(bs * nf * k, 65536, 0.5, 0)
    dd = torch.from_numpy(data).cuda()
    slots, sizes, stride = batch.compress_blocks(dd, bs, 1)
    assert bool((sizes > 0).all()) and bool((sizes < bs).all())
    packed, offs = batch.pack_blocks(slots, stride, sizes, header_bytes=4)
    del slots, dd
    packed, offs = packed.cpu().numpy(), offs.cpu().numpy()
    budget = [0, 0, 0, 0]
    budget[bsid - 4] = nf * k
    caps = torch.full((nf,), k * bs, dtype=torch.int64, device="cuda")
    calls = {}
    for mode, sums in (("verify", (block_sum, True)), ("skip", (block_sum, True)), ("plain", (False, False))):
        buf, fpos, flen = frames_of(xxh, data, packed, offs, bsid, nf, k, *sums)
        src = torch.from_numpy(buf).cuda()
        off, size = torch.from_numpy(fpos).cuda(), torch.from_numpy(flen).cuda()
        ws = torch.empty(batch.decompress_frames_workspace_bytes(nf, budget), dtype=torch.uint8, device="cuda")
        out = torch.empty(nf * k * bs, dtype=torch.uint8, device="cuda")
        res = torch.empty(nf, dtype=torch.int64, device="cuda")
        cons = torch.empty(nf, dtype=torch.int64, device="cuda")
        if mode == "plain":
            fn = (lambda src=src, off=off, size=size, out=out, res=res, cons=cons, ws=ws:
                  batch.decompress_frames(src, off, size, caps, budget, out=out, results=res, consumed=cons, workspace=ws))
        else:
            fn = (lambda src=src, off=off, size=size, out=out, res=res, cons=cons, ws=ws, skip=(mode == "skip"):
                  batch.decompress_frames_checksummed(src, off, size, caps, budget, skip, out=out, results=res,
                                                      consumed=cons, workspace=ws))
        fn()
        torch.cuda.synchronize()
        assert torch.equal(res, caps) and torch.equal(cons, size), (name, mode)
        assert torch.equal(out[:1 << 20].cpu(), torch.from_numpy(data[:1 << 20])), (name, mode)
        calls[mode] = fn
        del buf
    del data, packed
    ms = {mode: timed(fn, *(verify_reps if mode == "verify" else (10, 2))) for mode, fn in calls.items()}
    total = nf * k * bs
    print("%-50s verify %9.3f ms | skip %9.3f ms | plain frames %9.3f ms | verify / plain %.3f  (%.1f GB/s verified)"
          % (name, ms["verify"], ms["skip"], ms["plain"], ms["verify"] / ms["plain"], total / ms["verify"] / 1e6))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        calls["verify"]()
        torch.cuda.synchronize()
    own = {}
    for e in prof.key_averages():
        if "lz4_frames_" in e.key:
            kk = e.key.split("lz4_frames_")[1].split("_kernel")[0]
            own[kk] = own.get(kk, 0.0) + e.device_time_total / 1e3
    print("    frame kernels of the verifying call (profiler, ms): " + ", ".join("%s %.3f" % kv for kv in sorted(own.items())))
    calls.clear()
    torch.cuda.empty_cache()


def main():
    print("card:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                                   "--format=csv,noheader"], capture_output=True, text=True).stdout.strip())
    h = host_build.load()
    assert h is not None, "needs g++ for the host build of fc_xxh32"
    xxh = h.frames_xxh32_host
    xxh.restype = C.c_uint
    xxh.argtypes = [C.c_void_p, C.c_ulonglong, C.c_uint]
    orc = Oracle()
    todo = sys.argv[1:] or ["a", "b", "c"]
    if "a" in todo:
        run("(a) 65536 one-block 64 KB frames, content checksums", orc, xxh, 4, 65536, 1, False)
    if "b" in todo:
        run("(b) one frame of 1024 x 4 MB, content checksum", orc, xxh, 7, 1, 1024, False, verify_reps=(2, 1))
    if "c" in todo:
        run("(c) (a) with block checksums", orc, xxh, 4, 65536, 1, True)


if __name__ == "__main__":
    main()
