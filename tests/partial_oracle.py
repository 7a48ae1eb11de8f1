"""LZ4_decompress_safe_partial on the CPU -- TEST INFRASTRUCTURE ONLY.

`PartialOracle()` builds tests/partial_oracle.c (gcc, into a temporary directory, once per process) and wraps
oracle_lz4_decompress_safe_partial.  `reference_partial` calls the reference's own LZ4_decompress_safe_partial in
oracle/_ref/libref_lz4.so (an `oracle.pyoracle.Reference`).  Both decode into a zeroed destination followed by guard
bytes and check that nothing at or past outputSize = min(target, capacity) was written.
"""
import atexit
import ctypes as C
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

_u8p = C.POINTER(C.c_uint8)
_lib = None


def _load():
    global _lib
    if _lib is None:
        gcc = shutil.which("gcc") or shutil.which("cc")
        if not gcc:
            raise RuntimeError("a C compiler (gcc) is needed to build the partial-decode oracle")
        tmp = tempfile.mkdtemp(prefix="partial_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libpartial_oracle.so")
        subprocess.run([gcc, "-O2", "-std=c99", "-Wall", "-shared", "-fPIC", "-o", so,
                        os.path.join(HERE, "partial_oracle.c")], check=True)
        lib = C.CDLL(so)
        lib.oracle_lz4_decompress_safe_partial.restype = C.c_int
        lib.oracle_lz4_decompress_safe_partial.argtypes = [_u8p, _u8p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
        _lib = lib
    return _lib


def _call(fn, data, target, capacity):
    """fn(src pointer, dst pointer) -> ret; returns (ret, bytes) after checking 64 guard bytes past outputSize"""
    src = np.frombuffer(bytes(data), dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
    room = max(min(int(target), int(capacity)), 0)
    dst = np.zeros(room + 64, dtype=np.uint8)
    dst[room:] = 0xA5
    r = fn(src.ctypes.data_as(_u8p), dst.ctypes.data_as(_u8p))
    assert (dst[room:] == 0xA5).all(), "partial decode wrote at or past outputSize"
    return r, dst[:max(r, 0)].tobytes()


class PartialOracle:
    """decompress_partial(data, target, capacity=None) -> (ret, bytes), capacity defaulting to target.  After a call,
    `last_path` says how it ended (1 after literals, 2 inside a match, 0 otherwise) and `dst_dependent` whether the
    reference's bytes depend on what dst held (an offset-0 match on its cut path, lz4.c:2392-2404)."""

    def __init__(self):
        self.lib = _load()
        self.last_path, self.dst_dependent = 0, False

    def decompress_partial(self, data, target, capacity=None):
        cap = int(target) if capacity is None else int(capacity)
        path = C.c_int(0)
        r = _call(lambda sp, dp: int(self.lib.oracle_lz4_decompress_safe_partial(sp, dp, len(data), int(target), cap,
                                                                                  C.byref(path))), data, target, cap)
        self.last_path, self.dst_dependent = path.value & 3, bool(path.value & 4)
        return r

    def result(self, data, target, capacity=None):
        """(ret, bytes), or (ret, None) where the reference's bytes depend on dst: what the golden digests hold"""
        r, out = self.decompress_partial(data, target, capacity)
        return (r, None) if self.dst_dependent else (r, out)


def reference_partial(ref, data, target, capacity=None):
    """The reference's LZ4_decompress_safe_partial(src, dst, len(data), target, capacity) -> (ret, bytes)."""
    lib = ref.lib
    lib.LZ4_decompress_safe_partial.restype = C.c_int
    lib.LZ4_decompress_safe_partial.argtypes = [_u8p, _u8p, C.c_int, C.c_int, C.c_int]
    cap = int(target) if capacity is None else int(capacity)
    return _call(lambda sp, dp: int(lib.LZ4_decompress_safe_partial(sp, dp, len(data), int(target), cap)), data, target, cap)


def reference_partial_stable(ref, data, target, capacity=None):
    """reference_partial, with None for bytes that depend on what dst held (the checker tells which calls do)"""
    r, out = reference_partial(ref, data, target, capacity)
    po = PartialOracle()
    po.decompress_partial(data, target, capacity)
    return (r, None) if po.dst_dependent else (r, out)


def golden():
    """tests/golden/kat_partial.json with its cases rebuilt by the oracle (no reference needed):
    (doc, [(group name, [(src, target, capacity)], [ret], digest)]).  Check a group with make_golden_partial.run_digest
    over PartialOracle.result-shaped (ret, bytes or None) pairs."""
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import make_golden_partial as mg
    from oracle.pyoracle import Oracle
    with open(os.path.join(HERE, "golden", "kat_partial.json")) as f:
        doc = json.load(f)
    orc = Oracle()
    for b in doc["blocks"]:
        comp = mg.make_block(orc, b["size"], b["kind"], b["seed"])[1]
        assert hashlib.sha256(comp).hexdigest() == b["sha256"], "rebuilt block %d differs" % b["id"]
    out = []
    for (name, cases), (gname, rets, digest) in zip(mg.groups(orc), doc["groups"]):
        assert name == gname and len(cases) == len(rets)
        out.append((name, cases, rets, digest))
    assert len(out) == len(doc["groups"])
    return doc, out
