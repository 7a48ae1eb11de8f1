#!/usr/bin/env python
"""Generate tests/golden/kat_hc_destsize.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

Run where the reference sources exist:
    make -C oracle ref && python tests/golden/make_golden_hc_destsize.py
Every `ret`, `consumed` and digest below is a result of lib/lz4hc.c's LZ4_compress_HC_destSize (v1.10.0, gcc -O3,
x86-64) at levels -1 .. 9.  The inputs are rebuilt by the tests from the recipes of make_golden_hc.py (`make_input`,
`KINDS`) and the ones stored here (`inputs`, `random_cases`), without the reference.
"""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

from make_golden_hc import KINDS, compress_bound, digest, make_input  # noqa: E402

OUT = os.path.join(HERE, "kat_hc_destsize.json")

LEVELS = [-1, 0, 1, 2, 3, 4, 6, 9]
SMALL_SIZES = list(range(41))
SMALL_KINDS = ["p50", "per1", "per2", "random"]
MID_SIZES = [4096, 65536, 256 << 10]
BIG_SIZES = [1 << 20, 4 << 20]
BIG_KINDS = ["p50", "p90l60", "per1", "random"]
BIG_LEVELS = [2, 3, 9]


def inputs():
    """[(id, size, kind, seed, levels)] of the known-answer vectors: below 41 bytes each size takes one of SMALL_KINDS in
    turn (a block under 13 bytes is all literals at every level)."""
    out = []
    for size in SMALL_SIZES:
        kind = SMALL_KINDS[size % len(SMALL_KINDS)]
        out.append((len(out), size, kind, 5000 + len(out), LEVELS if size >= 13 else [9]))
    for size in MID_SIZES:
        for kind in KINDS:
            out.append((len(out), size, kind, 5000 + len(out), LEVELS))
    for size in BIG_SIZES:
        for kind in BIG_KINDS:
            out.append((len(out), size, kind, 5000 + len(out), BIG_LEVELS))
    return out


def targets(n, ret_bound):
    """Fixed targets, the bound -1/0, 2^30, and the size of the output at the bound -0/1/2: those land inside its last
    sequences and force the clamped-match path."""
    b = compress_bound(n)
    t = [-1, 0] + list(range(1, 17)) + [20, 100, 1000, 4096, 16384, 65536, b - 1, b, 1 << 30,
                                        ret_bound, ret_bound - 1, ret_bound - 2]
    return sorted(set(t))


def random_cases(gen, count):
    """The seeded random cases of the run digest: yields (data, target, level)."""
    rng = np.random.default_rng(2028)
    for k in range(count):
        n = int(rng.choice([0, 1, 12, 13, 14, 40, 100, 300, 1000, 4096, 20000, 65536, 70000]))
        kind = KINDS[int(rng.integers(0, len(KINDS)))]
        d = make_input(gen, n, kind, 70000 + k)
        b = compress_bound(n)
        target = int(rng.choice([int(rng.integers(-2, 40)), int(rng.integers(1, max(b, 2))), b - 1, b, 1 << 30,
                                 int(rng.integers(1, max(b // 4, 2)))]))
        yield d, target, int(rng.choice(LEVELS))


def run_digest(results):
    """12 hex digits over (ret, consumed, bytes) results, in order."""
    h = hashlib.sha256()
    for r, c, b in results:
        h.update(b"%d:%d:%d:" % (r, c, len(b)))
        h.update(bytes(b))
    return h.hexdigest()[:12]


RUN_CASES, RUN_CHUNK = 3000, 250


def reference_hc_dest(ref, data, target, level):
    """(ret, consumed, bytes) of the reference's LZ4_compress_HC_destSize from a fresh state; its bytes at and past
    min(target, bound) are checked untouched."""
    fn = ref.lib.LZ4_compress_HC_destSize
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int]
    ref.lib.LZ4_sizeofStateHC.restype = C.c_int
    state = np.zeros(int(ref.lib.LZ4_sizeofStateHC()) // 8 + 8, dtype=np.uint64)
    src = np.ascontiguousarray(data, dtype=np.uint8)
    room = max(min(target, compress_bound(len(src))), 0)
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    n = C.c_int(len(src))
    r = fn(state.ctypes.data, src.ctypes.data if len(src) else None, dst.ctypes.data, C.byref(n), target, level)
    assert (dst[room:] == 0xA5).all()
    return r, n.value, dst[:max(r, 0)].tobytes()


def main():
    from oracle.pyoracle import Reference
    ref = Reference()
    ins, vecs = [], []
    for (iid, size, kind, seed, levels) in inputs():
        d = make_input(ref, size, kind, seed)
        ins.append({"id": iid, "size": size, "kind": kind, "seed": seed, "levels": levels, "sha256": digest(d)})
        for lv in levels:
            rb = reference_hc_dest(ref, d, compress_bound(size), lv)[0]
            res = [reference_hc_dest(ref, d, t, lv) for t in targets(size, rb)]
            vecs.append([iid, lv, rb, [r for r, _, _ in res], [c for _, c, _ in res], run_digest(res)])
    runs, res = [], []
    for d, t, lv in random_cases(ref, RUN_CASES):
        res.append(reference_hc_dest(ref, d, t, lv))
        if len(res) == RUN_CHUNK:
            runs.append(run_digest(res))
            res = []
    assert not res
    doc = {"source": "lz4 v1.10.0 lib/lz4hc.c LZ4_compress_HC_destSize, gcc -O3 x86-64",
           "fields": ["input", "level", "ret at the bound", "ret at each of targets(size, ret at the bound)",
                      "consumed at each of those targets", "run_digest of those (ret, consumed, output) results"],
           "inputs": ins, "vectors": vecs, "run_cases": RUN_CASES, "run_chunk": RUN_CHUNK, "run_digests": runs}
    with open(OUT, "w") as f:
        json.dump(doc, f, separators=(",", ":"))
        f.write("\n")
    print("HC destSize vectors %d over %d inputs, %d run digests" % (len(vecs), len(ins), len(runs)))


if __name__ == "__main__":
    main()
