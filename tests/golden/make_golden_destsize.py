#!/usr/bin/env python
"""Generate tests/golden/kat_destsize.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

Run where the reference sources exist:
    make -C oracle ref && python tests/golden/make_golden_destsize.py
Every `ret`, `consumed`, output and digest below is a result of lib/lz4.c's LZ4_compress_destSize /
LZ4_compress_destSize_extState (v1.10.0, gcc -O3, x86-64).  The inputs are rebuilt by the tests from the recipes stored
here (`inputs`, `random_cases`), without the reference: datagen buffers come from tests/datagen.c's generator, which the
oracle reproduces byte for byte.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for _p in (ROOT, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "kat_destsize.json")

SIZES = [0, 1, 12, 13, 14, 100, 4096, 65535, 65546, 65547, 65548, 200000, 4 << 20]
KINDS = ["p0", "p50", "p90", "p99", "random", "zero", "period"]
# the fill parse's accelerations: the ends of lz4.c's clamp (65537, 65538), large values and the largest one it
# takes without `acceleration << 6` overflowing int
ACCELS = [1, 2, 8, 65537, 65538, 1 << 20, (1 << 25) - 1]
HEX_MAX = 64


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def compress_bound(n):
    return n + n // 255 + 16 if 0 <= n <= 0x7E000000 else 0


def make_input(gen, size, kind, seed):
    """Input bytes of one recipe; `gen` is anything with datagen(size, proba, seed) (Oracle or Reference)."""
    if kind[0] == "p" and kind[1:].isdigit():
        return np.asarray(gen.datagen(size, int(kind[1:]) / 100.0, seed), dtype=np.uint8)
    rng = np.random.default_rng(seed)
    if kind == "random":
        return rng.integers(0, 256, size, dtype=np.uint8)
    if kind == "zero":
        return np.zeros(size, dtype=np.uint8)
    assert kind == "period"                      # short period: long matches that the fill parse has to shorten
    period = 2 + seed % 6
    return np.tile(rng.integers(0, 256, period, dtype=np.uint8), size // period + 1)[:size].copy()


def inputs():
    """[(id, size, kind, seed)] of the known-answer vectors."""
    out = []
    for size in SIZES:
        for kind in KINDS:
            out.append((len(out), size, kind, 1000 + len(out)))
    return out


def targets(n, fast_size):
    """The target list of one input: fixed sizes, the LZ4_compress_fast size -1/0/+1 and the bound -1/0."""
    b = compress_bound(n)
    t = [-1, 0] + list(range(1, 21)) + [64, 100, 4096, 16384, 32768, fast_size - 1, fast_size, fast_size + 1, b - 1, b]
    return sorted(set(t))


def random_cases(gen, count):
    """The seeded random cases of the run digest: yields (data, target, acceleration or None)."""
    rng = np.random.default_rng(2026)
    for k in range(count):
        n = int(rng.choice([0, 1, 13, 14, 40, 100, 300, 1000, 4096, 20000, 65535, 65546, 65547, 65548, 100000]))
        kind = KINDS[int(rng.integers(0, len(KINDS)))]
        d = make_input(gen, n, kind, 50000 + k)
        b = compress_bound(n)
        target = int(rng.choice([int(rng.integers(-2, 40)), int(rng.integers(1, max(b, 2))), b - 1, b,
                                 int(rng.integers(1, max(b // 4, 2)))]))
        pick = int(rng.integers(0, len(ACCELS) + 1))
        yield d, target, (None if pick == len(ACCELS) else ACCELS[pick])


def run_digest(results):
    """12 hex digits over (ret, consumed, bytes) results, in order."""
    h = hashlib.sha256()
    for r, c, b in results:
        h.update(b"%d:%d:%d:" % (r, c, len(b)))
        h.update(bytes(b))
    return h.hexdigest()[:12]


RUN_CASES, RUN_CHUNK = 3000, 250


def main():
    from oracle.pyoracle import Reference
    from destsize_oracle import reference_dest_size
    ref = Reference()
    ins, vecs = [], []
    for (iid, size, kind, seed) in inputs():
        d = make_input(ref, size, kind, seed)
        fast, _ = ref.compress(d, 1)
        ins.append({"id": iid, "size": size, "kind": kind, "seed": seed, "sha256": sha(d)})
        for ti, t in enumerate(targets(size, fast)):
            # the plain entry point for every target, _extState with the accelerations in turn
            for acc in (None, ACCELS[(iid + ti) % len(ACCELS)]):
                r, c, out, _ = reference_dest_size(ref, d, t, acc)
                vecs.append([iid, t, acc, r, c, out.hex() if len(out) <= HEX_MAX else sha(out)])
    runs = []
    res = []
    for d, t, acc in random_cases(ref, RUN_CASES):
        r, c, out, _ = reference_dest_size(ref, d, t, acc)
        res.append((r, c, out))
        if len(res) == RUN_CHUNK:
            runs.append(run_digest(res))
            res = []
    assert not res
    doc = {"source": "lz4 v1.10.0 lib/lz4.c LZ4_compress_destSize / LZ4_compress_destSize_extState, gcc -O3 x86-64",
           "fields": ["input", "target", "acceleration (null: LZ4_compress_destSize)", "ret", "consumed",
                      "output hex (<= %d bytes) or its sha256" % HEX_MAX],
           "inputs": ins, "vectors": vecs, "run_cases": RUN_CASES, "run_chunk": RUN_CHUNK, "run_digests": runs}
    with open(OUT, "w") as f:
        json.dump(doc, f, separators=(",", ":"))
        f.write("\n")
    print("destSize vectors %d over %d inputs, %d run digests" % (len(vecs), len(ins), len(runs)))


if __name__ == "__main__":
    main()
