#!/usr/bin/env python
"""Generate tests/golden/kat_hc_dropin.json from the COMPILED REFERENCE (oracle/_ref/libref_lz4.so).

Run where the reference sources exist:
    make -C oracle ref && python tests/golden/make_golden_hc_dropin.py
Every value below is a result of lib/lz4hc.c (v1.10.0, gcc -O3, x86-64) through its one-shot API, the calls that
liblz4_b200.so's drop-in HC family replaces: LZ4_compress_HC at levels -3 .. 100 (every capacity class: the bound, the
exact output size, one byte less, 1 and 0), LZ4_compress_HC_destSize at the targets 1, 7, 8, 4 096, the bound and the
output at the bound minus 1 and 2, the verdicts of LZ4_compress_HC_extStateHC, _extStateHC_fastReset and _destSize on
NULL and misaligned states, LZ4_sizeofStateHC, and the image LZ4_initStreamHC leaves in a state.  kat_hc.json and
kat_hc_opt.json hold the same two calls at sizes 0 .. 40 and 4 KB .. 4 MB on datagen, periodic and random inputs, each
file at its own levels; this file puts every level (-3 .. 100) on the same inputs, and adds text, the sizes 65 537 and
300 000, the capacity 1 and the state rules.  Its inputs use the recipes of make_golden_hc.py plus text, with seeds of
their own.
The tests rebuild the inputs from the recipes stored here (`make_input`), without the reference.
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

import make_golden_hc as mg  # noqa: E402
from make_golden_hc import compress_bound, digest, run_digest  # noqa: E402
from make_golden_hc_destsize import run_digest as dest_run_digest  # noqa: E402

OUT = os.path.join(HERE, "kat_hc_dropin.json")

LEVELS = [-3, 0, 1, 2, 3, 4, 6, 9, 10, 11, 12, 13, 100]
KINDS = ["p50", "p90", "random", "text"]
SIZES = [0, 1, 12, 13, 4096, 65536, 65537, 300000]
STATE_BYTES = 262200                     # LZ4_STREAMHC_MINSIZE, lz4hc.h:252
STATE_FILL = 0xA5                        # what a state holds before LZ4_initStreamHC
STATE_OFFSETS = list(range(9))           # byte offsets of the state from a 64-byte aligned buffer

WORDS = ("the of and to in is that for it as was with be by on not he this are or his from at which but have an they "
         "you were her she there been one all we their has would when if so no will more can out up into do any time "
         "block input output level state parse match literal offset token stream frame buffer bytes length search "
         "chain table window value return call first last next each other about than them these some only new two "
         "over such our after most also made many before must through back years where much your way well down should "
         "because each just those people how too little state world very still own see men work long get here between "
         "both life being under never day same another know while last might us great old year off come since against "
         "go came right used take three").split()


def make_text(size, seed):
    """English-like text: seeded words from WORDS with spaces, commas, full stops and line breaks"""
    rng = np.random.default_rng(seed)
    out, n = [], 0
    while n < size:
        w = WORDS[int(rng.integers(0, len(WORDS)))]
        r = int(rng.integers(0, 20))
        sep = ".\n" if r == 0 else (", " if r < 3 else " ")
        out.append(w + sep)
        n += len(w) + len(sep)
    return np.frombuffer("".join(out).encode()[:size], dtype=np.uint8).copy()


def make_input(gen, size, kind, seed):
    """Input bytes of one recipe: make_golden_hc.make_input's kinds, and text"""
    return make_text(size, seed) if kind == "text" else mg.make_input(gen, size, kind, seed)


BIG_PLAIN_LEVELS = [-3, 0, 1, 2, 3, 4, 6, 9, 10, 12]
BIG_DEST_LEVELS = [2, 3, 9, 10]


def levels_of(size):
    """(LZ4_compress_HC levels, LZ4_compress_HC_destSize levels) of an input: every level up to 64 KB + 1; at 300 000
    bytes, where one GPU thread takes up to a second or two per call, levels 11, 13 and 100 are left to the smaller
    sizes (and 12 takes two capacities, see plain_caps)"""
    if size <= 65537:
        return LEVELS, LEVELS
    return BIG_PLAIN_LEVELS, BIG_DEST_LEVELS


def plain_caps(size, level, ret_bound):
    """The capacities of one LZ4_compress_HC vector: the bound, the exact size, one byte less (which must give 0), 1 and
    0; at 300 000 bytes level 12 takes the bound and the exact size only"""
    if size > 65537 and level >= 12:
        return sorted({compress_bound(size), ret_bound})
    return sorted({compress_bound(size), ret_bound, ret_bound - 1, 1, 0})


def dest_targets(size, ret_bound):
    """The targets of one LZ4_compress_HC_destSize vector: 1, 7, 8, 4 096, the output at the bound minus 1 and 2, and
    the bound"""
    return sorted({t for t in (1, 7, 8, 4096, ret_bound - 1, ret_bound - 2, compress_bound(size)) if t >= 1})


def inputs():
    """[(id, size, kind, seed)]: every kind at every size"""
    out = []
    for size in SIZES:
        for kind in KINDS:
            out.append((len(out), size, kind, 9000 + len(out)))
    return out


def _source(data):
    """The input with a real address even when empty (the optimal parser reads from it before its loop)"""
    src = np.zeros(max(len(data), 1), dtype=np.uint8)
    src[:len(data)] = np.asarray(data, dtype=np.uint8)
    return src


def _bind(lib):
    lib.LZ4_compress_HC.restype = C.c_int
    lib.LZ4_compress_HC.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    for name in ("LZ4_compress_HC_extStateHC", "LZ4_compress_HC_extStateHC_fastReset"):
        getattr(lib, name).restype = C.c_int
        getattr(lib, name).argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    lib.LZ4_compress_HC_destSize.restype = C.c_int
    lib.LZ4_compress_HC_destSize.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_int, C.c_int]
    lib.LZ4_sizeofStateHC.restype = C.c_int
    lib.LZ4_initStreamHC.restype = C.c_void_p
    lib.LZ4_initStreamHC.argtypes = [C.c_void_p, C.c_size_t]
    return lib


def reference_hc(lib, data, cap, level):
    """(ret, bytes) of LZ4_compress_HC; its bytes at and past min(cap, bound) are checked untouched"""
    src = _source(data)
    room = max(min(cap, compress_bound(len(data))), 0)
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    r = lib.LZ4_compress_HC(src.ctypes.data, dst.ctypes.data, len(data), cap, level)
    assert (dst[room:] == 0xA5).all()
    return r, dst[:max(r, 0)].tobytes()


def reference_hc_dest(lib, data, target, level):
    """(ret, consumed, bytes) of LZ4_compress_HC_destSize on a fresh aligned state; its bytes at and past
    min(target, bound) are checked untouched"""
    state = np.zeros(STATE_BYTES // 8, dtype=np.uint64)
    src = _source(data)
    room = max(min(target, compress_bound(len(data))), 0)
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    n = C.c_int(len(data))
    r = lib.LZ4_compress_HC_destSize(state.ctypes.data, src.ctypes.data, dst.ctypes.data, C.byref(n), target, level)
    assert (dst[room:] == 0xA5).all()
    return r, n.value, dst[:max(r, 0)].tobytes()


def state_buffer(offset):
    """A STATE_FILL-filled state at `offset` bytes from a 64-byte aligned address (the array that holds it comes
    second, to keep it alive)"""
    raw = np.full(STATE_BYTES + 128, STATE_FILL, dtype=np.uint8)
    base = (-raw.ctypes.data) % 64
    return raw.ctypes.data + base + offset, raw


VERDICT_LEVEL, VERDICT_SIZE = 9, 4096


def state_verdicts(lib, data):
    """{call: [[offset or None (NULL), ret, consumed or None]]} on one input of VERDICT_SIZE bytes at VERDICT_LEVEL, at
    the bound / a 4 096-byte target.  _extStateHC_fastReset is not run on NULL: the reference dereferences it."""
    src = _source(data)
    cap = compress_bound(len(data))
    out = {"LZ4_compress_HC_extStateHC": [], "LZ4_compress_HC_extStateHC_fastReset": [], "LZ4_compress_HC_destSize": []}
    for off in [None] + STATE_OFFSETS:
        for name in out:
            if off is None and name.endswith("fastReset"):
                continue
            p, keep = state_buffer(off) if off is not None else (None, None)
            if p is not None and name.endswith("fastReset"):
                C.memset(p, 0, STATE_BYTES)            # a state the reference may read: all zero is a valid one
            dst = np.zeros(cap, dtype=np.uint8)
            if name.endswith("destSize"):
                n = C.c_int(len(data))
                r = lib.LZ4_compress_HC_destSize(p, src.ctypes.data, dst.ctypes.data, C.byref(n), 4096, VERDICT_LEVEL)
                out[name].append([off, r, n.value])
            else:
                r = getattr(lib, name)(p, src.ctypes.data, dst.ctypes.data, len(data), cap, VERDICT_LEVEL)
                out[name].append([off, r, None])
            del keep
    return out


def state_image(lib):
    """sizeof, and the digest of a STATE_FILL-filled state after LZ4_initStreamHC"""
    p, keep = state_buffer(0)
    assert lib.LZ4_initStreamHC(p, STATE_BYTES) == p
    img = C.string_at(p, STATE_BYTES)
    return {"fill": STATE_FILL, "bytes": int(lib.LZ4_sizeofStateHC()), "sha256": hashlib.sha256(img).hexdigest(),
            "zero_bytes": sum(1 for b in img if b == 0), "fill_bytes": sum(1 for b in img if b == STATE_FILL)}


def main(out=OUT):
    from oracle.pyoracle import Reference
    ref = Reference()
    lib = _bind(ref.lib)
    ins, vecs, dvecs = [], [], []
    verdict_input = None
    for (iid, size, kind, seed) in inputs():
        d = make_input(ref, size, kind, seed)
        ins.append({"id": iid, "size": size, "kind": kind, "seed": seed, "sha256": digest(d)})
        if size == VERDICT_SIZE and kind == "p50":
            verdict_input = (iid, d)
        plain_levels, dest_levels = levels_of(size)
        for lv in plain_levels:
            rb, _ = reference_hc(lib, d, compress_bound(size), lv)
            caps = plain_caps(size, lv, rb)
            res = [reference_hc(lib, d, cap, lv) for cap in caps]
            vecs.append([iid, lv, caps, [r for r, _ in res], run_digest(res)])
        for lv in dest_levels:
            rbd = reference_hc_dest(lib, d, compress_bound(size), lv)[0]
            ts = dest_targets(size, rbd)
            res = [reference_hc_dest(lib, d, t, lv) for t in ts]
            dvecs.append([iid, lv, ts, [r for r, _, _ in res], [c for _, c, _ in res], dest_run_digest(res)])
    doc = {"source": "lz4 v1.10.0 lib/lz4hc.c one-shot API (LZ4_compress_HC, _extStateHC, _extStateHC_fastReset, "
                     "_destSize, LZ4_sizeofStateHC, LZ4_initStreamHC), gcc -O3 x86-64",
           "fields": {"vectors": ["input", "level", "capacities", "LZ4_compress_HC's ret at each",
                                  "make_golden_hc.run_digest of those (ret, output) results"],
                      "dest_vectors": ["input", "level", "targets", "LZ4_compress_HC_destSize's ret at each",
                                       "consumed at each",
                                       "make_golden_hc_destsize.run_digest of those (ret, consumed, output) results"],
                      "state_verdicts": ["state offset from a 64-byte aligned address (null: NULL)", "ret",
                                         "*srcSizePtr after the call (destSize)"]},
           "state": state_image(lib),
           "verdicts": {"input": verdict_input[0], "level": VERDICT_LEVEL, "target": 4096,
                        "calls": state_verdicts(lib, verdict_input[1])},
           "inputs": ins, "vectors": vecs, "dest_vectors": dvecs}
    with open(out, "w") as f:
        json.dump(doc, f, separators=(",", ":"))
        f.write("\n")
    print("HC drop-in vectors %d + %d over %d inputs" % (len(vecs), len(dvecs), len(ins)))


if __name__ == "__main__":
    main()
