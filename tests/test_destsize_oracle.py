"""LZ4_compress_destSize on the CPU: the fill parse of oracle/lz4_oracle.c (oracle_lz4_compress_destSize_extState)
against the reference's results in tests/golden/kat_destsize.json (tests/golden/make_golden_destsize.py), its
properties, a live differential against the compiled reference when it is present, and the drop-in's behaviour without
a device."""
import collections
import ctypes as C
import os

import numpy as np
import pytest

from conftest import load_golden
from oracle.pyoracle import PATHS as PATHS_BY_CODE
from golden.make_golden_destsize import ACCELS, inputs, make_input, random_cases, run_digest, sha, HEX_MAX

PATHS = ["fast", "empty", "no_room", "literals", "next_match", "reduced", "last_literals", "filled"]


@pytest.fixture(scope="module")
def kat():
    return load_golden("kat_destsize.json")


@pytest.fixture(scope="module")
def kat_inputs(kat, oracle):
    data = {}
    for (iid, size, kind, seed), row in zip(inputs(), kat["inputs"]):
        assert row["id"] == iid and row["size"] == size and row["kind"] == kind and row["seed"] == seed
        d = make_input(oracle, size, kind, seed)
        assert sha(d) == row["sha256"], (iid, size, kind)
        data[iid] = d
    return data


def _out_key(out):
    return out.hex() if len(out) <= HEX_MAX else sha(out)


def path_name(code):
    return PATHS_BY_CODE[code]


def test_oracle_reproduces_every_golden_vector(kat, kat_inputs, oracle):
    seen = collections.Counter()
    fill_accels = set()
    for iid, target, acc, ret, consumed, out in kat["vectors"]:
        d = kat_inputs[iid]
        r, c, o, path = oracle.compress_dest_size(d, target, acc)
        assert (r, c, _out_key(o)) == (ret, consumed, out), (iid, len(d), target, acc)
        seen[(path_name(path), len(d) < 65547)] += 1
        if path_name(path) in PATHS[3:]:
            fill_accels.add(acc)
    # every route and every exit of the fill parse, on both table types (an empty input has none)
    assert seen[("empty", True)] >= 5, seen
    for p in PATHS:
        if p != "empty":
            assert seen[(p, True)] >= 5 and seen[(p, False)] >= 5, (p, seen)
    assert fill_accels == set(ACCELS) | {None}


def test_oracle_reproduces_the_run_digest(kat, oracle):
    res, digests = [], []
    for d, t, acc in random_cases(oracle, kat["run_cases"]):
        r, c, o, _ = oracle.compress_dest_size(d, t, acc)
        res.append((r, c, o))
        if len(res) == kat["run_chunk"]:
            digests.append(run_digest(res))
            res = []
    assert digests == kat["run_digests"]


def test_properties_over_random_cases(oracle):
    rng = np.random.default_rng(7)
    for k in range(600):
        n = int(rng.choice([1, 13, 50, 500, 5000, 65546, 65547, 90000]))
        d = make_input(oracle, n, ["p0", "p50", "p90", "random", "zero", "period"][k % 6], 900 + k)
        b = oracle.compress_bound(n)
        t = int(rng.integers(1, b + 2))
        acc = int(rng.choice(ACCELS))
        r, c, o, path = oracle.compress_dest_size(d, t, acc)
        assert 0 < r <= t and 0 <= c <= n, (n, t, acc, r, c)
        # the v1.9.2 guarantee (lz4.h:261-270): the output decodes with a capacity of exactly `consumed`
        assert oracle.decompress(o, c) == (c, d[:c].tobytes()), (n, t, acc)
        if t >= b:
            assert path_name(path) == "fast" and c == n
            assert (r, o) == oracle.compress(d, acc, t)


def test_routes_in_front_of_the_parse(oracle):
    d = make_input(oracle, 1000, "p50", 1)
    assert oracle.compress_dest_size(d, 0, None)[:2] == (0, 1000)
    assert oracle.compress_dest_size(d, -5, 3)[:2] == (0, 1000)
    assert oracle.compress_dest_size(b"", 0, None)[:2] == (0, 0)
    assert oracle.compress_dest_size(b"", 1, None)[:3] == (1, 0, b"\x00")
    assert oracle.compress_dest_size(b"", 16, None)[:3] == (1, 0, b"\x00")
    # the ends of the acceleration range are brought into it (documented deviations)
    assert oracle.compress_dest_size(d, 300, 0)[:3] == oracle.compress_dest_size(d, 300, 1)[:3]
    assert oracle.compress_dest_size(d, 300, 1 << 30)[:3] == oracle.compress_dest_size(d, 300, (1 << 25) - 1)[:3]


def test_live_differential_against_the_reference(oracle, reference):
    for k, (d, t, acc) in enumerate(random_cases(oracle, 400)):
        assert oracle.compress_dest_size(d, t, acc)[:3] == reference.compress_dest_size(d, t, acc)[:3], (k, len(d), t, acc)


def test_drop_in_without_a_device_leaves_srcsize_alone():
    from lz4_b200 import _lib
    lib = _lib.load()
    if lib.LZ4B200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    src = np.frombuffer(os.urandom(1000), dtype=np.uint8)
    dst = np.full(600, 0xA5, dtype=np.uint8)
    for call in (lambda n: lib.LZ4_compress_destSize(src.ctypes.data, dst.ctypes.data, C.byref(n), 500),
                 lambda n: lib.LZ4_compress_destSize_extState(np.zeros(2052, dtype=np.uint64).ctypes.data, src.ctypes.data,
                                                              dst.ctypes.data, C.byref(n), 500, 4)):
        n = C.c_int(1000)
        assert call(n) == 0
        assert n.value == 1000
    assert (dst == 0xA5).all()
