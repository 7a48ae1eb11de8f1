"""The host builds of the GPU's HC parses (tests/emul/hc_emul.cpp over lz4_b200/csrc/lz4_hc_core.h) and the HC golden
vectors: TEST INFRASTRUCTURE shared by the CPU checks of the parses (tests/test_hc*_emul.py) and the GPU tests of the
HC calls.  Every call skips the calling test without g++."""
import ctypes as C
import json
import os
import sys

import numpy as np

import host_build

HERE = os.path.dirname(os.path.abspath(__file__))
for _p in (os.path.dirname(HERE), os.path.join(HERE, "golden")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import make_golden_hc as mg  # noqa: E402
import make_golden_hc_destsize as mgd  # noqa: E402
import make_golden_hc_opt as mgo  # noqa: E402


def _src(data):
    return np.frombuffer(bytes(data), dtype=np.uint8) if isinstance(data, bytes) else np.ascontiguousarray(data, np.uint8)


def room(n, target):
    """The bytes a call may write: min(target, LZ4_compressBound(n)), at least 0"""
    return max(min(target, mg.compress_bound(n)), 0)


def _plain(fn, data, cap, *fills):
    """(ret, bytes) of LZ4_compress_HC; the bytes past the capacity are checked untouched."""
    src = _src(data)
    lim = room(len(src), cap)                   # a capacity of at least the bound writes below it
    dst = np.full(lim + 64, 0xA5, dtype=np.uint8)
    r = fn(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, cap, *fills)
    assert (dst[lim:] == 0xA5).all(), "wrote past the capacity"
    return r, dst[:max(r, 0)].tobytes()


def _dest(fn, data, target, *fills):
    """(ret, consumed, bytes) of LZ4_compress_HC_destSize; the bytes at and past min(target, bound) are checked
    untouched."""
    src = _src(data)
    lim = room(len(src), target)
    dst = np.full(lim + 64, 0xA5, dtype=np.uint8)
    consumed = C.c_int(-7)
    r = fn(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, target, *fills, C.byref(consumed))
    assert (dst[lim:] == 0xA5).all(), "wrote at or past min(target, bound)"
    return r, consumed.value, dst[:max(r, 0)].tobytes()


def host_hc(data, cap, level, chain_fill=0xFFFF):
    """(ret, bytes) of the level 1 .. 9 parse; ret -1 above 9"""
    return _plain(host_build.require().hc_emul_compress, data, cap, level, chain_fill)


def host_hc_dest(data, target, level, chain_fill=0xFFFF):
    """(ret, consumed, bytes) of the level 1 .. 9 fill parse; ret -1 above 9"""
    return _dest(host_build.require().hc_dest_emul_compress, data, target, level, chain_fill)


def host_hc_opt(data, cap, level, chain_fill=0xFFFF, opt_fill=0):
    """(ret, bytes) of the optimal parse (levels 10 and up); ret -1 below 10"""
    return _plain(host_build.require().hc_opt_emul_compress, data, cap, level, chain_fill, opt_fill)


def host_hc_opt_dest(data, target, level, chain_fill=0xFFFF, opt_fill=0):
    """(ret, consumed, bytes) of the optimal parse's fill mode (levels 10 and up); ret -1 below 10"""
    return _dest(host_build.require().hc_opt_emul_compress_dest, data, target, level, chain_fill, opt_fill)


def golden(name):
    """(doc, {input id: input record}) of tests/golden/<name>"""
    with open(os.path.join(HERE, "golden", name)) as f:
        doc = json.load(f)
    return doc, {i["id"]: i for i in doc["inputs"]}
