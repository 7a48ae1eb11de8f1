"""The host build of the GPU's HC fill parse (tests/emul/hc_dest_emul.cpp over lz4_b200/csrc/lz4_hc_core.h) and the HC
destSize golden vectors: TEST INFRASTRUCTURE shared by tests/test_hc_destsize_emul.py and tests/test_gpu_hc_destsize.py."""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.dirname(HERE), os.path.join(HERE, "golden")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import make_golden_hc as mg  # noqa: E402
import make_golden_hc_destsize as mgd  # noqa: E402

_lib = None


def load():
    """Compile the host build into a temporary directory (once per process); None without g++."""
    global _lib
    if _lib is None:
        gxx = shutil.which("g++")
        if not gxx:
            return None
        so = os.path.join(tempfile.mkdtemp(prefix="hcdestemul"), "libhcdestemul.so")
        subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-shared", "-fPIC", "-o", so,
                        os.path.join(HERE, "emul", "hc_dest_emul.cpp")], check=True)
        lib = C.CDLL(so)
        lib.hc_dest_emul_compress.restype = C.c_int
        lib.hc_dest_emul_compress.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint32,
                                              C.POINTER(C.c_int)]
        _lib = lib
    return _lib


def room(n, target):
    """The bytes a call may write: min(target, LZ4_compressBound(n)), at least 0"""
    return max(min(target, mg.compress_bound(n)), 0)


def host_hc_dest(data, target, level, chain_fill=0xFFFF):
    """(ret, consumed, bytes) of the host build; the bytes at and past min(target, bound) are checked untouched."""
    src = np.frombuffer(bytes(data), dtype=np.uint8) if isinstance(data, bytes) else np.ascontiguousarray(data, np.uint8)
    lim = room(len(src), target)
    dst = np.full(lim + 64, 0xA5, dtype=np.uint8)
    consumed = C.c_int(-7)
    r = load().hc_dest_emul_compress(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, target, level,
                                     chain_fill, C.byref(consumed))
    assert (dst[lim:] == 0xA5).all(), "wrote at or past min(target, bound)"
    return r, consumed.value, dst[:max(r, 0)].tobytes()


def golden():
    """(doc, {input id: input record}) of kat_hc_destsize.json"""
    with open(os.path.join(HERE, "golden", "kat_hc_destsize.json")) as f:
        doc = json.load(f)
    return doc, {i["id"]: i for i in doc["inputs"]}
