"""CPU check of the decode call's plan (lz4_b200/csrc/lz4_decode_plan.h): workspace layout, wide flag and scan choice.

tests/emul/plan_emul.cpp compiles the header with g++.  Over a grid of batch sizes, capacities (one for every block, or
per block), both call kinds (full and partial) and workspaces of the size that enables the tiles kernel ("sized-for"),
the size for any capacities and one byte less than sized-for, the plan must agree with
  - LZ4B200_decompress_workspace_bytes and _for (host functions of the library: no GPU needed), and with the sizes the
    layout had before it was gathered in the plan (SIZED_FOR / ANY below);
  - the offsets the Python readers of the GPU tests use (gpu_util.ws_lists, gpu_util.wide_workspace,
    test_gpu_scan_marks.narrow_workspace), read back from a workspace whose every word holds its own index;
  - gpu_util.route's R1 .. R6 for the wide flag and the scan kernel.
"""
import ctypes as C
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch

import gpu_util
from test_gpu_scan_marks import narrow_workspace

HERE = os.path.dirname(os.path.abspath(__file__))
SIZE_MAX = 2**64 - 1
THREAD, PAR, SPLIT = 0, 1, 2                                  # DecodeScan
FIELDS = ("wide", "markStride", "tilesMax", "scan", "nSeq", "slowList", "marks", "scratch", "used", "tileFirst",
          "tileFlag", "bytes")

N = [1, 7, 64, 65, 8192, 8193, 65536]
CAPS = [-1, 0, 1, 4, 100, 16383, 16384, 20000, 65535, 65536, 65537, 122880, 122881, 4 << 20, 64 << 20, (64 << 20) + 1,
        2**31 - 1]
# LZ4B200_decompress_workspace_bytes(n) and LZ4B200_decompress_workspace_bytes_for(n, 0, CAPS[i]) of the layout as it was
# before the plan existed (per-block capacities: _for(n, 1, any) = ANY[n])
ANY = {1: 99328, 7: 689152, 64: 6292480, 65: 6391296, 8192: 805372416, 8193: 805471232, 65536: 6442975744}
SIZED_FOR = {
    1: [1024, 1024, 1792, 1792, 1792, 50944, 50944, 61696, 99328, 99328, 132864, 247552, 247552, 8390912, 134228224, 1024,
        1024],
    7: [1024, 1024, 1792, 1792, 3328, 345856, 345856, 421888, 689152, 689152, 919296, 1722112, 1722112, 58725632,
        939586816, 1024, 1024],
    64: [1024, 1024, 2560, 3328, 21760, 3147520, 3148288, 3842560, 6292480, 6292480, 8392192, 15732224, 15732736,
         536908800, 8590496768, 1024, 1024],
    65: [1536, 1536, 3840, 4608, 23040, 3197952, 3198720, 3903744, 6391296, 6391296, 8524544, 15979264, 15979776,
         545299200, 8724724480, 1536, 1536],
    8192: [66048, 66048, 262656, 360960, 2720256, 402817536, 402915840, 491782656, 805372416, 805372416, 1074135552,
           2013659648, 2013725184, 68724261376, 1099583521280, 66048, 66048],
    8193: [66560, 66560, 263936, 362240, 2721536, 402867968, 402966272, 491843840, 805471232, 805471232, 1074267904,
           2013906688, 2013972224, 68732651776, 1099717748992, 66560, 66560],
    65536: [524800, 524800, 2097664, 2884096, 21758464, 3222536704, 3223323136, 3934257664, 6442975744, 6442975744,
            8593080832, 16109273600, 16109797888, 549794087424, 8796668166656, 524800, 524800],
}
ROUTE_PLAN = {"R1": (False, THREAD), "R2": (False, SPLIT), "R3": (False, THREAD), "R4": (False, THREAD),
              "R5": (True, PAR), "R6": (False, PAR)}
READ_BACK_MAX = 64 << 20                                      # workspaces the reader check materialises


@pytest.fixture(scope="module")
def plan(tmp_path_factory):
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    so = str(tmp_path_factory.mktemp("planemul") / "libplanemul.so")
    subprocess.run([gxx, "-O2", "-std=c++17", "-Wall", "-shared", "-fPIC", "-o", so,
                    os.path.join(HERE, "emul", "plan_emul.cpp")], check=True)
    lib = C.CDLL(so)
    lib.plan_host.restype = None
    lib.plan_host.argtypes = [C.c_int64, C.c_int, C.c_int32, C.c_uint64, C.c_int, C.POINTER(C.c_uint64)]

    def run(n, per_block, cap, ws_bytes, partial=False):
        out = (C.c_uint64 * len(FIELDS))()
        lib.plan_host(n, int(per_block), cap, ws_bytes, int(partial), out)
        return dict(zip(FIELDS, list(out)))
    return run


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    return _lib.load()


def index_workspace(nbytes, n):
    """a workspace whose word i holds i, except word 0 (the slow-list count), which holds n"""
    w = np.arange(nbytes // 4, dtype=np.uint32)
    w[0] = n
    return torch.from_numpy(w.view(np.uint8))


def check_readers(p, n, cap, per_block=False):
    """the GPU tests' readers find every region where the plan puts it"""
    ws = index_workspace(p["bytes"], n)
    nseq, slow = gpu_util.ws_lists(ws, n)
    assert nseq[0] * 4 == p["nSeq"] and slow[0] * 4 == p["slowList"]
    if p["wide"]:
        marks, tile_first = gpu_util.wide_workspace(types.SimpleNamespace(ws=ws), n, cap)
        b = n - 1
        assert marks(b, 1)[0] * 4 == p["marks"] + b * p["markStride"] * 4
        assert tile_first(b, 0)[0] * 4 == p["tileFirst"] + b * (p["tilesMax"] + 1) * 4
    elif p["markStride"]:
        stride = 8192 if per_block else min(cap // 4 + 2, 8192)   # test_gpu_scan_marks.decode_phases
        assert stride == p["markStride"]
        nseq, marks = narrow_workspace(ws, n, stride)
        assert nseq[0] * 4 == p["nSeq"]
        assert marks[n - 1, 0] * 4 == p["marks"] + (n - 1) * stride * 4


def check_layout(p, n):
    """the regions follow each other in the documented order, each on 256 bytes, none overlapping"""
    r = lambda x: (x + 255) // 256 * 256
    lst, mk = r(n * 4), r(n * p["markStride"] * 4)
    assert (p["nSeq"], p["slowList"], p["marks"]) == (256, 256 + lst, 256 + 2 * lst)
    end = p["marks"] + mk
    if p["wide"]:
        tl = r(n * (p["tilesMax"] + 1) * 4)
        assert (p["scratch"], p["used"], p["tileFirst"], p["tileFlag"]) == (0, 0, end, end + tl)
        assert p["bytes"] == end + 2 * tl + 256
    else:
        assert p["tileFirst"] == p["tileFlag"] == 0 and p["bytes"] == end + 2 * mk + 256


@pytest.mark.parametrize("n", N)
def test_uniform_capacities(plan, lib, n):
    for i, cap in enumerate(CAPS):
        sized = plan(n, False, cap, SIZE_MAX)
        assert sized["bytes"] == SIZED_FOR[n][i] == lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap), (n, cap)
        for ws_bytes in (sized["bytes"], ANY[n], sized["bytes"] - 1):
            p = plan(n, False, cap, ws_bytes)
            check_layout(p, n)
            rt = gpu_util.route(n, cap, ws_bytes=ws_bytes)
            assert (bool(p["wide"]), p["scan"]) == ROUTE_PLAN[rt], (n, cap, ws_bytes, rt)
            # a call is refused only for one byte short of a workspace that has no smaller (narrow) layout
            accepted = ws_bytes != sized["bytes"] - 1 or sized["wide"]
            assert (p["bytes"] <= ws_bytes) == accepted, (n, cap, ws_bytes)
            assert p["wide"] == (p["bytes"] == sized["bytes"] and sized["wide"])
            assert (p["scratch"] != 0) == (not p["wide"]) and p["used"] == 0
            if p["bytes"] <= READ_BACK_MAX and n <= 65:
                check_readers(p, n, cap)
            q = plan(n, False, cap, ws_bytes, partial=True)     # the partial call: the narrow layout, one-thread scan
            narrow = plan(n, False, cap, 0)
            check_layout(q, n)
            assert not q["wide"] and q["scan"] == THREAD and q["scratch"] == 0
            assert q["bytes"] == narrow["bytes"] and q["markStride"] == narrow["markStride"]
            assert q["used"] == (narrow["scratch"] if q["markStride"] else 0)


@pytest.mark.parametrize("n", N)
def test_per_block_capacities(plan, lib, n):
    assert lib.LZ4B200_decompress_workspace_bytes(n) == ANY[n]
    for cap in CAPS:
        assert lib.LZ4B200_decompress_workspace_bytes_for(n, 1, cap) == ANY[n]
        for ws_bytes in (ANY[n], SIZE_MAX, ANY[n] - 1, 0):
            p = plan(n, True, cap, ws_bytes)
            check_layout(p, n)
            assert p["bytes"] == ANY[n] and p["markStride"] == 8192
            assert (bool(p["wide"]), p["scan"]) == ROUTE_PLAN[gpu_util.route(n, per_block_caps=True)]
            q = plan(n, True, cap, ws_bytes, partial=True)
            assert q["bytes"] == ANY[n] and q["used"] == p["scratch"] and not q["wide"] and q["scan"] == THREAD
            if n <= 65:
                check_readers(p, n, cap, per_block=True)


def test_split_scan_crossover(plan):
    """the split scan is the default up to 8 192 blocks of 16..64 KB, the parallel scan above 64 KB"""
    assert plan(8192, False, 16384, SIZE_MAX)["scan"] == SPLIT and plan(8193, False, 16384, SIZE_MAX)["scan"] == THREAD
    assert plan(8192, False, 16383, SIZE_MAX)["scan"] == THREAD and plan(1, False, 65536, SIZE_MAX)["scan"] == SPLIT
    assert plan(65536, False, 65537, SIZE_MAX)["scan"] == PAR and plan(1, False, 2**31 - 1, SIZE_MAX)["scan"] == PAR
