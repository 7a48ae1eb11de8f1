#!/usr/bin/env python
"""Generate tests/golden/kat_partial.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

Run where the reference sources exist:
    make -C oracle ref && python tests/golden/make_golden_partial.py
Every `ret` and output digest below is a result of lib/lz4.c's LZ4_decompress_safe_partial (v1.10.0, gcc -O3, x86-64),
decoding into a zeroed destination.  The cases are rebuilt by the tests from the recipes here (`groups`, `random_cases`)
without the reference: datagen buffers come from tests/datagen.c's generator and the blocks
from LZ4_compress_fast, which the oracle reproduces byte for byte; `sha256` pins every rebuilt input.
"""
import hashlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_destsize import KINDS, make_input  # noqa: E402  (the destSize vectors' input recipes)
OUT = os.path.join(HERE, "kat_partial.json")

SIZES = [0, 1, 13, 100, 4096, 65536, 200000, 4 << 20]
DELTAS = (0, 1, 4, 5, 11, 12, 13)
SWEEP = [("p50", 1000, 7), ("period", 700, 8), ("random", 300, 9)]
RUN_CASES, RUN_CHUNK = 2000, 250


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def make_block(codec, size, kind, seed):
    """(raw bytes, LZ4_compress_fast block) of one recipe; `codec` is an Oracle or a Reference"""
    raw = make_input(codec, size, kind, seed)
    r, comp = codec.compress(raw, 1)
    assert r > 0
    return raw.tobytes(), comp


def blocks():
    """[(id, size, kind, seed)]"""
    out = []
    for size in SIZES:
        for kind in KINDS:
            out.append((len(out), size, kind, 3000 + len(out)))
    return out


def variant(comp, v):
    """The source bytes of a variant recipe: ["exact"], ["trunc", k] (k bytes cut), ["ext", k, seed] (k bytes appended:
    seeded random, or zeros for seed < 0), ["flip", pos, xor]"""
    if v[0] == "exact":
        return comp
    if v[0] == "trunc":
        return comp[:max(len(comp) - v[1], 0)]
    if v[0] == "ext":
        tail = bytes(v[1]) if v[2] < 0 else np.random.default_rng(v[2]).integers(0, 256, v[1], dtype=np.uint8).tobytes()
        return comp + tail
    assert v[0] == "flip"
    b = bytearray(comp)
    b[v[1] % len(b)] ^= v[2]
    return bytes(b)


def variants(bid, comp):
    vs = [["exact"]]
    if len(comp) > 2:
        vs += [["trunc", 1], ["trunc", 5], ["trunc", len(comp) // 2]]
        vs += [["ext", k, 100 * bid + k] for k in range(1, 10)] + [["ext", k, -1] for k in (1, 5, 9)]
        vs += [["flip", 7 * bid + 3, 0x40], ["flip", len(comp) - 4, 0xFF]]
    return vs


def targets(dec, full):
    t = [-1, 0] + list(range(1, 21)) + [31, 32, 33, 63, 64, 65, 4096] + [dec + d for d in range(-13, 2)]
    if not full:
        t = [1, 17, 64, 65, 4096, dec - 13, dec - 5, dec - 1, dec, dec + 1]
    return sorted(set(x for x in t if x >= -1))


def sequences(comp):
    """[(literal start, match start, match end)] of a valid block, in decoded positions"""
    ip, op, out = 0, 0, []
    while True:
        tok = comp[ip]; ip += 1
        ll = tok >> 4
        if ll == 15:
            while True:
                x = comp[ip]; ip += 1; ll += x
                if x != 255:
                    break
        start = op
        ip += ll; op += ll
        if ip >= len(comp):
            return out
        ip += 2
        ml = tok & 15
        if ml == 15:
            while True:
                x = comp[ip]; ip += 1; ml += x
                if x != 255:
                    break
        out.append((start, op, op + ml + 4))
        op += ml + 4


def boundary_targets(comp):
    seqs = sequences(comp)
    pick = seqs[:30] + seqs[-30:]
    t = set()
    for (_, ms, me) in pick:
        for p in (ms, me):
            for d in DELTAS:
                t.update((p - d, p + d))
    return sorted(x for x in t if x >= 0)


def groups(codec):
    """yields (name, [(src bytes, target, capacity)]) of the known-answer vectors: every variant of every block at its
    targets, capacities below the target, match boundaries of a 64 KB P50 block, and the exhaustive sweeps"""
    for (bid, size, kind, seed) in blocks():
        comp = make_block(codec, size, kind, seed)[1]
        for v in variants(bid, comp):
            src = variant(comp, v)
            yield "%d/%s" % (bid, v), [(src, t, t) for t in targets(size, v == ["exact"] or size <= 4096)]
        yield "%d/cap" % bid, [(comp, t, c) for t, c in ((size, size - 1), (size + 5, size // 2), (100, 64), (4096, 17),
                                                         (size, 0))]
        if size == 65536 and kind == "p50":
            yield "%d/boundary" % bid, [(comp, t, t) for t in boundary_targets(comp)]
    for kind, size, seed in SWEEP:
        comp = make_block(codec, size, kind, seed)[1]
        yield "sweep/%s" % kind, [(comp, t, t) for t in range(0, size + 17)]


def random_cases(codec, count):
    """yields (src bytes, target, capacity) of the seeded random cases of the run digests"""
    rng = np.random.default_rng(2026)
    cache = {}
    for k in range(count):
        size = int(rng.choice([1, 13, 40, 100, 1000, 4096, 20000, 65536]))
        kind = KINDS[int(rng.integers(0, len(KINDS)))]
        key = (size, kind)
        if key not in cache:
            cache[key] = make_block(codec, size, kind, 90000 + len(cache))[1]
        comp = cache[key]
        m = int(rng.integers(0, 4))
        if m == 1:
            comp = comp[:int(rng.integers(1, len(comp) + 1))]
        elif m == 2:
            comp = comp + rng.integers(0, 256, int(rng.integers(1, 10)), dtype=np.uint8).tobytes()
        elif m == 3:
            b = bytearray(comp); b[int(rng.integers(0, len(b)))] ^= int(rng.integers(1, 256)); comp = bytes(b)
        target = int(rng.choice([int(rng.integers(-1, 80)), int(rng.integers(0, size + 20)), size]))
        cap = target if rng.integers(0, 3) else int(rng.integers(0, max(target, 1) + 1))
        yield comp, target, cap


def run_digest(results):
    """12 hex digits over (ret, bytes or None) results, in order"""
    h = hashlib.sha256()
    for r, b in results:
        if b is None:                            # bytes that depend on dst: the return value only
            h.update(b"%d:dst:" % r)
            continue
        h.update(b"%d:%d:" % (r, len(b)))
        h.update(bytes(b))
    return h.hexdigest()[:12]


def reference_partial_stable(ref, orc, data, target, capacity=None):
    """The reference's (ret, bytes), with None for bytes that depend on what dst held (the oracle tells which calls do)"""
    r, out = ref.decompress_partial(data, target, capacity)
    return (r, None) if orc.decompress_partial_traced(data, target, capacity)[3] else (r, out)


def golden():
    """kat_partial.json with its cases rebuilt by the oracle (no reference needed):
    (doc, [(group name, [(src, target, capacity)], [ret], digest)]).  Check a group with run_digest over
    (ret, bytes or None) pairs, None where Oracle.decompress_partial_traced reports dst_dependent."""
    from oracle.pyoracle import Oracle
    with open(OUT) as f:
        doc = json.load(f)
    orc = Oracle()
    for b in doc["blocks"]:
        comp = make_block(orc, b["size"], b["kind"], b["seed"])[1]
        assert sha(comp) == b["sha256"], "rebuilt block %d differs" % b["id"]
    out = []
    for (name, cases), (gname, rets, digest) in zip(groups(orc), doc["groups"]):
        assert name == gname and len(cases) == len(rets)
        out.append((name, cases, rets, digest))
    assert len(out) == len(doc["groups"])
    return doc, out


def main():
    from oracle.pyoracle import Oracle, Reference
    ref, orc = Reference(), Oracle()
    bl = []
    for (bid, size, kind, seed) in blocks():
        comp = make_block(ref, size, kind, seed)[1]
        bl.append({"id": bid, "size": size, "kind": kind, "seed": seed, "sha256": sha(comp)})
    gs = []
    for name, cases in groups(ref):
        res = [reference_partial_stable(ref, orc, src, t, c) for src, t, c in cases]
        gs.append([name, [r for r, _ in res], run_digest(res)])
    res = [reference_partial_stable(ref, orc, comp, t, c) for comp, t, c in random_cases(ref, RUN_CASES)]
    runs = [run_digest(res[k:k + RUN_CHUNK]) for k in range(0, RUN_CASES, RUN_CHUNK)]
    doc = {"source": "lz4 v1.10.0 lib/lz4.c LZ4_decompress_safe_partial, gcc -O3 x86-64, zeroed destination",
           "fields": ["group (see groups())", "ret of every case", "run_digest of the outputs (null where they depend on "
                      "what dst held: the return value only)"],
           "blocks": bl, "groups": gs, "run_cases": RUN_CASES, "run_chunk": RUN_CHUNK, "run_digests": runs}
    with open(OUT, "w") as f:
        json.dump(doc, f, separators=(",", ":"))
        f.write("\n")
    print("partial vectors %d in %d groups, %d run digests" % (sum(len(g[1]) for g in gs), len(gs), len(runs)))


if __name__ == "__main__":
    main()
