"""The host build of the GPU's HC parse (tests/emul/hc_emul.cpp over lz4_b200/csrc/lz4_hc_core.h) and the HC golden
vectors: TEST INFRASTRUCTURE shared by tests/test_hc_emul.py and tests/test_gpu_hc.py."""
import ctypes as C
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

_lib = None


def load():
    """Compile the host build into a temporary directory (once per process); None without g++."""
    global _lib
    if _lib is None:
        gxx = shutil.which("g++")
        if not gxx:
            return None
        so = os.path.join(tempfile.mkdtemp(prefix="hcemul"), "libhcemul.so")
        subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-Wextra", "-shared", "-fPIC", "-o", so,
                        os.path.join(HERE, "emul", "hc_emul.cpp")], check=True)
        lib = C.CDLL(so)
        lib.hc_emul_compress.restype = C.c_int
        lib.hc_emul_compress.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_uint32]
        _lib = lib
    return _lib


def host_hc(data, cap, level, chain_fill=0xFFFF):
    """(ret, bytes) of the host build; the bytes past the capacity are checked untouched."""
    src = np.frombuffer(bytes(data), dtype=np.uint8) if isinstance(data, bytes) else np.ascontiguousarray(data, np.uint8)
    room = max(min(cap, mg.compress_bound(len(src))), 0)        # a capacity of at least the bound writes below it
    dst = np.full(room + 64, 0xA5, dtype=np.uint8)
    r = load().hc_emul_compress(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, cap, level, chain_fill)
    assert (dst[room:] == 0xA5).all(), "wrote past the capacity"
    return r, dst[:max(r, 0)].tobytes()


def golden():
    """(doc, {input id: (size, kind, seed, levels, sha)}) of kat_hc.json"""
    import json
    with open(os.path.join(HERE, "golden", "kat_hc.json")) as f:
        doc = json.load(f)
    return doc, {i["id"]: i for i in doc["inputs"]}
