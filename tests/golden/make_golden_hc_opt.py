#!/usr/bin/env python
"""Generate tests/golden/kat_hc_opt.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

Run where the reference sources exist:
    make -C oracle ref && python tests/golden/make_golden_hc_opt.py
Every `ret`, `consumed` and digest below is a result of lib/lz4hc.c's LZ4_compress_HC and LZ4_compress_HC_destSize
(v1.10.0, gcc -O3, x86-64) at levels 10 .. 12, and 13 and 100 (read as 12) on a few inputs: the optimal parser.  The
inputs are rebuilt by the tests from the recipes of make_golden_hc.py (`make_input`, `KINDS`) and the ones stored here
(`inputs`, `random_cases`), without the reference.
"""
import ctypes as C
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from make_golden_hc import KINDS, capacities, compress_bound, digest, make_input  # noqa: E402
from make_golden_hc import run_digest as run_digest_hc  # noqa: E402
from make_golden_hc_destsize import run_digest, targets  # noqa: E402

OUT = os.path.join(HERE, "kat_hc_opt.json")

LEVELS = [10, 11, 12]
ABOVE = [13, 100]                       # read as 12, in ultra mode like it
SMALL_SIZES = list(range(41))
SMALL_KINDS = ["p50", "per1", "per2", "random"]
MID_SIZES = [4096, 65536, 256 << 10]
ABOVE_KINDS = ["p50", "per1", "random"]  # the mid inputs that also take ABOVE
BIG_SIZES = [1 << 20, 4 << 20]
BIG_KINDS = ["p50", "p90l60", "per1", "random"]
BIG_LEVELS = [10, 12]


def inputs():
    """[(id, size, kind, seed, levels)] of the known-answer vectors: below 41 bytes each size takes one of SMALL_KINDS in
    turn, and sizes 20 and 40 also take ABOVE."""
    out = []
    for size in SMALL_SIZES:
        kind = SMALL_KINDS[size % len(SMALL_KINDS)]
        out.append((len(out), size, kind, 7000 + len(out), LEVELS + (ABOVE if size in (20, 40) else [])))
    for size in MID_SIZES:
        for kind in KINDS:
            out.append((len(out), size, kind, 7000 + len(out),
                        LEVELS + (ABOVE if size == 65536 and kind in ABOVE_KINDS else [])))
    for size in BIG_SIZES:
        for kind in BIG_KINDS:
            out.append((len(out), size, kind, 7000 + len(out), BIG_LEVELS))
    return out


RUN_SIZES = [0, 14, 1000, 65536, 70000]
RUN_LEVELS = [10, 11, 12]
SHARED = [1000, 1 << 30]


def run_limits(n):
    """The capacities and targets a run case draws from: the size's bound and bound - 1, and the SHARED values (so a
    batch call per (limit, level) covers every case)"""
    b = compress_bound(n)
    return [b, b - 1] + SHARED


def random_cases(gen, count, seed):
    """The seeded random cases of a run digest: yields (data, capacity or target, level)."""
    rng = np.random.default_rng(seed)
    for k in range(count):
        n = int(rng.choice(RUN_SIZES))
        kind = KINDS[int(rng.integers(0, len(KINDS)))]
        d = make_input(gen, n, kind, seed * 100 + k)
        lims = run_limits(n)
        yield d, lims[int(rng.integers(0, len(lims)))], int(rng.choice(RUN_LEVELS))


RUN_CASES, RUN_CHUNK = 600, 100
PLAIN_SEED, DEST_SEED = 2029, 2030


def _source(data):
    """The input with a real address even when empty: the optimal parser computes iend - MFLIMIT before its loop, and
    from a NULL source that wraps around and the loop reads address 0."""
    src = np.zeros(max(len(data), 1), dtype=np.uint8)
    src[:len(data)] = np.asarray(data, dtype=np.uint8)
    return src


def reference_hc(ref, data, cap, level):
    """(ret, bytes) of the reference's LZ4_compress_HC; its bytes past dstCapacity are checked untouched."""
    fn = ref.lib.LZ4_compress_HC
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    src = _source(data)
    room = max(min(cap, compress_bound(len(data))), 0)
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    r = fn(src.ctypes.data, dst.ctypes.data, len(data), cap, level)
    assert (dst[room:] == 0xA5).all()
    return r, dst[:max(r, 0)].tobytes()


def reference_hc_dest(ref, data, target, level):
    """(ret, consumed, bytes) of the reference's LZ4_compress_HC_destSize from a fresh state; its bytes at and past
    min(target, bound) are checked untouched."""
    fn = ref.lib.LZ4_compress_HC_destSize
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int]
    ref.lib.LZ4_sizeofStateHC.restype = C.c_int
    state = np.zeros(int(ref.lib.LZ4_sizeofStateHC()) // 8 + 8, dtype=np.uint64)
    src = _source(data)
    room = max(min(target, compress_bound(len(data))), 0)
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    n = C.c_int(len(data))
    r = fn(state.ctypes.data, src.ctypes.data, dst.ctypes.data, C.byref(n), target, level)
    assert (dst[room:] == 0xA5).all()
    return r, n.value, dst[:max(r, 0)].tobytes()


def main():
    from oracle.pyoracle import Reference
    ref = Reference()
    ins, vecs, dvecs = [], [], []
    for (iid, size, kind, seed, levels) in inputs():
        d = make_input(ref, size, kind, seed)
        ins.append({"id": iid, "size": size, "kind": kind, "seed": seed, "levels": levels, "sha256": digest(d)})
        for lv in levels:
            rb, _ = reference_hc(ref, d, compress_bound(size), lv)
            res = [reference_hc(ref, d, cap, lv) for cap in capacities(size, rb)]
            vecs.append([iid, lv, rb, [r for r, _ in res], run_digest_hc(res)])
            rbd = reference_hc_dest(ref, d, compress_bound(size), lv)[0]
            dres = [reference_hc_dest(ref, d, t, lv) for t in targets(size, rbd)]
            dvecs.append([iid, lv, rbd, [r for r, _, _ in dres], [c for _, c, _ in dres], run_digest(dres)])
    runs, res = [], []
    for d, cap, lv in random_cases(ref, RUN_CASES, PLAIN_SEED):
        res.append(reference_hc(ref, d, cap, lv))
        if len(res) == RUN_CHUNK:
            runs.append(run_digest_hc(res))
            res = []
    druns = []
    for d, t, lv in random_cases(ref, RUN_CASES, DEST_SEED):
        res.append(reference_hc_dest(ref, d, t, lv))
        if len(res) == RUN_CHUNK:
            druns.append(run_digest(res))
            res = []
    assert not res
    doc = {"source": "lz4 v1.10.0 lib/lz4hc.c LZ4_compress_HC and LZ4_compress_HC_destSize, gcc -O3 x86-64",
           "fields": {"vectors": ["input", "level", "LZ4_compress_HC's ret at the bound",
                                  "ret at each of make_golden_hc.capacities(size, ret at the bound)",
                                  "make_golden_hc.run_digest of those (ret, output) results"],
                      "dest_vectors": ["input", "level", "LZ4_compress_HC_destSize's ret at the bound",
                                       "ret at each of make_golden_hc_destsize.targets(size, ret at the bound)",
                                       "consumed at each of those targets",
                                       "make_golden_hc_destsize.run_digest of those (ret, consumed, output) results"]},
           "inputs": ins, "vectors": vecs, "dest_vectors": dvecs, "run_cases": RUN_CASES, "run_chunk": RUN_CHUNK,
           "run_digests": runs, "dest_run_digests": druns}
    with open(OUT, "w") as f:
        json.dump(doc, f, separators=(",", ":"))
        f.write("\n")
    print("HC optimal-parser vectors %d + %d over %d inputs, %d + %d run digests"
          % (len(vecs), len(dvecs), len(ins), len(runs), len(druns)))


if __name__ == "__main__":
    main()
