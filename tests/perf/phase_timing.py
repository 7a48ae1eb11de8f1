"""Developer tool: per-phase cycle breakdown of the fast expand kernel.
Build with LZ4K_PHASE_TIMING=1 (python tests/perf/phase_timing.py --build), run under gpurun."""
import ctypes as C
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    import numpy as np
    import torch
    from lz4_b200 import _lib, batch
    from oracle.pyoracle import Oracle
    lib = _lib.load()
    raw = C.CDLL(_lib.LIB_PATH)
    orc = Oracle()
    n_blocks, bs = 8192, 65536
    proba = float(os.environ.get("PROBA", "0.5"))
    data = orc.datagen_mt(n_blocks * bs, 64 << 20, proba, 0)
    src = torch.from_numpy(data).cuda()
    slots, sizes, stride = batch.compress_blocks(src, bs, 1)
    packed, offs = batch.pack_blocks(slots, stride, sizes)
    offs = offs[:-1].contiguous()
    out = torch.empty_like(src)
    rets = torch.empty(n_blocks, dtype=torch.int32, device="cuda")
    ws = torch.empty(int(_lib.load().LZ4B200_decompress_workspace_bytes_for(n_blocks, 0, bs)), dtype=torch.uint8, device="cuda")
    for _ in range(3):
        batch.decompress_blocks(packed, offs, sizes, bs, out=out, out_sizes=rets)
    torch.cuda.synchronize()
    buf = (C.c_ulonglong * 12)()
    raw.LZ4B200_debug_phase_cycles(buf)
    reps = 5
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    batch.decompress_blocks(packed, offs, sizes, bs, out=out, out_sizes=rets, workspace=ws, phases=1)
    t0.record()
    for _ in range(reps):
        batch.decompress_blocks(packed, offs, sizes, bs, out=out, out_sizes=rets, workspace=ws, phases=2)
    t1.record()
    torch.cuda.synchronize()
    raw.LZ4B200_debug_phase_cycles(buf)
    names = ["fetch+zero", "tma load wait", "runs pass 1", "rank + prev store", "runs pass 2", "waves", "store issue", "-"]
    tot = sum(buf[:8])
    print("expand ms per launch %.3f, blocks %d" % (t0.elapsed_time(t1) / reps, n_blocks))
    for n, v in zip(names, buf[:8]):
        print("%-16s %8.0f cycles/block  %5.1f%%" % (n, v / (reps * n_blocks), 100.0 * v / max(tot, 1)))
    assert torch.equal(out, src)


if __name__ == "__main__":
    main()
