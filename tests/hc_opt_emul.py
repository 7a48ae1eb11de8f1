"""The host build of the GPU's HC optimal parse (tests/emul/hc_opt_emul.cpp over lz4_b200/csrc/lz4_hc_core.h) and the
level 10 .. 12 golden vectors: TEST INFRASTRUCTURE shared by tests/test_hc_opt_emul.py and tests/test_gpu_hc_opt.py."""
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
import make_golden_hc_opt as mgo  # noqa: E402

_lib = None


def load():
    """Compile the host build into a temporary directory (once per process); None without g++."""
    global _lib
    if _lib is None:
        gxx = shutil.which("g++")
        if not gxx:
            return None
        so = os.path.join(tempfile.mkdtemp(prefix="hcoptemul"), "libhcoptemul.so")
        subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-shared", "-fPIC", "-o", so,
                        os.path.join(HERE, "emul", "hc_opt_emul.cpp")], check=True)
        lib = C.CDLL(so)
        lib.hc_opt_emul_compress.restype = C.c_int
        lib.hc_opt_emul_compress.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint32, C.c_uint32]
        lib.hc_opt_emul_compress_dest.restype = C.c_int
        lib.hc_opt_emul_compress_dest.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint32,
                                                  C.c_uint32, C.POINTER(C.c_int)]
        _lib = lib
    return _lib


def _src(data):
    return np.frombuffer(bytes(data), dtype=np.uint8) if isinstance(data, bytes) else np.ascontiguousarray(data, np.uint8)


def host_hc_opt(data, cap, level, chain_fill=0xFFFF, opt_fill=0):
    """(ret, bytes) of the host build's LZ4_compress_HC; the bytes past the capacity are checked untouched."""
    src = _src(data)
    room = max(min(cap, mg.compress_bound(len(src))), 0)
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    r = load().hc_opt_emul_compress(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, cap, level,
                                    chain_fill, opt_fill)
    assert (dst[room:] == 0xA5).all(), "wrote past the capacity"
    return r, dst[:max(r, 0)].tobytes()


def host_hc_opt_dest(data, target, level, chain_fill=0xFFFF, opt_fill=0):
    """(ret, consumed, bytes) of the host build's LZ4_compress_HC_destSize; the bytes at and past min(target, bound)
    are checked untouched."""
    src = _src(data)
    lim = max(min(target, mg.compress_bound(len(src))), 0)
    dst = np.full(lim + 64, 0xA5, dtype=np.uint8)
    consumed = C.c_int(-7)
    r = load().hc_opt_emul_compress_dest(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, target,
                                         level, chain_fill, opt_fill, C.byref(consumed))
    assert (dst[lim:] == 0xA5).all(), "wrote at or past min(target, bound)"
    return r, consumed.value, dst[:max(r, 0)].tobytes()


def golden():
    """(doc, {input id: input record}) of kat_hc_opt.json"""
    with open(os.path.join(HERE, "golden", "kat_hc_opt.json")) as f:
        doc = json.load(f)
    return doc, {i["id"]: i for i in doc["inputs"]}
