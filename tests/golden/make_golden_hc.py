#!/usr/bin/env python
"""Generate tests/golden/kat_hc.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

Run where the reference sources exist:
    make -C oracle ref && python tests/golden/make_golden_hc.py
Every `ret` and digest below is a result of lib/lz4hc.c's LZ4_compress_HC (v1.10.0, gcc -O3, x86-64) at levels -1 .. 9.
The tests rebuild the inputs from the recipes stored here (`inputs`, `random_cases`), without the reference: datagen
buffers come from tests/datagen.c's generator, which the oracle reproduces byte for byte.
"""
import ctypes as C
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "kat_hc.json")

LEVELS = [-1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9]
# datagen match probabilities, two literal-probability variants, runs of short periods (1 and 2 reach the repeat-pattern
# search of level 9's chain walk, lz4hc.c:988-1059; the longer ones check that it stays shut) and random bytes
KINDS = ["p0", "p20", "p50", "p90", "p100", "p50l20", "p90l60", "per1", "per2", "per3", "per4", "per5", "per8", "random"]
BIG_KINDS = ["p50", "p90l60", "per1", "per3", "random"]
SMALL_KINDS = ["p0", "p50", "p100", "per1", "per2", "per3", "random"]
SMALL_LEVELS = [-1, 0, 1, 2, 3, 6, 9]
SMALL_SIZES = list(range(41))
MID_SIZES = [65536, 256 << 10]
BIG_SIZES = [1 << 20, 4 << 20]
BIG_LEVELS = [1, 2, 3, 9]


def digest(b):
    return hashlib.sha256(bytes(b)).hexdigest()[:16]


def compress_bound(n):
    return n + n // 255 + 16 if 0 <= n <= 0x7E000000 else 0


def make_input(gen, size, kind, seed):
    """Input bytes of one recipe; `gen` is anything with datagen(size, proba, seed, lit_proba) (Oracle or Reference)."""
    if kind[0] == "p" and kind[1].isdigit():
        proba, _, lit = kind[1:].partition("l")
        return np.asarray(gen.datagen(size, int(proba) / 100.0, seed, int(lit) / 100.0 if lit else 0.0), dtype=np.uint8)
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, size, dtype=np.uint8)
    assert kind.startswith("per")
    period = int(kind[3:])
    return np.tile(rng.integers(0, 256, period, dtype=np.uint8), size // period + 1)[:size].copy()


def inputs():
    """[(id, size, kind, seed, levels)] of the known-answer vectors."""
    out = []
    for size in SMALL_SIZES:
        for kind in SMALL_KINDS:
            out.append((len(out), size, kind, 3000 + len(out), SMALL_LEVELS))
    for size in MID_SIZES:
        for kind in KINDS:
            out.append((len(out), size, kind, 3000 + len(out), LEVELS))
    for size in BIG_SIZES:
        for kind in BIG_KINDS:
            out.append((len(out), size, kind, 3000 + len(out), BIG_LEVELS))
    return out


def capacities(n, ret_bound):
    """The bound, the exact size the bound gives, one byte less (must give 0) and a few small capacities."""
    return sorted({compress_bound(n), ret_bound, ret_bound - 1, 0, 1, 8, 20})


def random_cases(gen, count):
    """The seeded random cases of the run digest: yields (data, capacity, level)."""
    rng = np.random.default_rng(2027)
    for k in range(count):
        n = int(rng.choice([0, 1, 12, 13, 14, 40, 100, 300, 1000, 4096, 20000, 65536, 70000]))
        kind = KINDS[int(rng.integers(0, len(KINDS)))]
        d = make_input(gen, n, kind, 60000 + k)
        b = compress_bound(n)
        cap = int(rng.choice([b, b - 1, int(rng.integers(0, max(b, 2))), int(rng.integers(b // 3, max(b, 2))), 1 << 30]))
        yield d, cap, int(rng.choice(LEVELS))


def run_digest(results):
    """12 hex digits over (ret, bytes) results, in order."""
    h = hashlib.sha256()
    for r, b in results:
        h.update(b"%d:%d:" % (r, len(b)))
        h.update(bytes(b))
    return h.hexdigest()[:12]


RUN_CASES, RUN_CHUNK = 3000, 250


def reference_hc(ref, data, cap, level):
    """(ret, bytes) of the reference's LZ4_compress_HC; its bytes past dstCapacity are checked untouched."""
    fn = ref.lib.LZ4_compress_HC
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    src = np.ascontiguousarray(data, dtype=np.uint8)
    room = max(min(cap, compress_bound(len(src))), 0)           # a capacity of at least the bound writes below it
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    r = fn(src.ctypes.data if len(src) else None, dst.ctypes.data, len(src), cap, level)
    assert (dst[room:] == 0xA5).all()
    return r, dst[:max(r, 0)].tobytes()


def main():
    from oracle.pyoracle import Reference
    ref = Reference()
    ins, vecs = [], []
    for (iid, size, kind, seed, levels) in inputs():
        d = make_input(ref, size, kind, seed)
        ins.append({"id": iid, "size": size, "kind": kind, "seed": seed, "levels": levels, "sha256": digest(d)})
        for lv in levels:
            rb, _ = reference_hc(ref, d, compress_bound(size), lv)
            res = [reference_hc(ref, d, cap, lv) for cap in capacities(size, rb)]
            vecs.append([iid, lv, rb, [r for r, _ in res], run_digest(res)])
    runs, res = [], []
    for d, cap, lv in random_cases(ref, RUN_CASES):
        res.append(reference_hc(ref, d, cap, lv))
        if len(res) == RUN_CHUNK:
            runs.append(run_digest(res))
            res = []
    assert not res
    doc = {"source": "lz4 v1.10.0 lib/lz4hc.c LZ4_compress_HC, gcc -O3 x86-64",
           "fields": ["input", "level", "ret at the bound", "ret at each of capacities(size, ret at the bound)",
                      "run_digest of those (ret, output) results"],
           "inputs": ins, "vectors": vecs, "run_cases": RUN_CASES, "run_chunk": RUN_CHUNK, "run_digests": runs}
    with open(OUT, "w") as f:
        json.dump(doc, f, separators=(",", ":"))
        f.write("\n")
    print("HC vectors %d over %d inputs, %d run digests" % (len(vecs), len(ins), len(runs)))


if __name__ == "__main__":
    main()
