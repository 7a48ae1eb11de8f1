"""The drop-in LZ4_compress_HC family on the host: LZ4_sizeofStateHC, the rules decided without a launch (state checks,
sizes, capacities and targets, the empty input) against the reference's values in tests/golden/kat_hc_dropin.json, the
state image LZ4_compress_HC_extStateHC and LZ4_compress_HC_destSize leave, and, on a machine without a CUDA device,
that every call that would launch returns 0 and writes nothing.  No row here reaches the device, so the launch counter
must not move.  The GPU results are tests/test_gpu_hc_dropin.py's."""
import ctypes as C
import hashlib
import os
import tempfile

import numpy as np
import pytest

import hc_emul as he
import make_golden_hc_dropin as mk

MAX_INPUT = 0x7E000000
NAMES = ("LZ4_compress_HC_extStateHC", "LZ4_compress_HC_extStateHC_fastReset", "LZ4_compress_HC_destSize")


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


@pytest.fixture(scope="module")
def golden():
    return he.golden("kat_hc_dropin.json")


_keep = np.zeros(1 << 16, dtype=np.uint8)
P = _keep.ctypes.data + (-_keep.ctypes.data) % 64      # a 64-byte aligned host pointer no row reads


def call(lib, name, state, src, dst, n, cap, level):
    """one call of a drop-in HC entry point; destSize returns (ret, *srcSizePtr after the call)"""
    if name == "LZ4_compress_HC":
        return lib.LZ4_compress_HC(src, dst, n, cap, level)
    if name == "LZ4_compress_HC_destSize":
        m = C.c_int(n)
        return lib.LZ4_compress_HC_destSize(state, src, dst, C.byref(m), cap, level), m.value
    return getattr(lib, name)(state, src, dst, n, cap, level)


def test_sizeof_state(lib, golden):
    doc, _ = golden
    assert lib.LZ4_sizeofStateHC() == 262200 == doc["state"]["bytes"]


def test_golden_inputs_rebuild_without_the_reference(golden, oracle):
    doc, ins = golden
    for iid, i in ins.items():
        assert mk.digest(mk.make_input(oracle, i["size"], i["kind"], i["seed"])) == i["sha256"], i


def test_state_verdicts(lib, golden):
    """NULL and misaligned states give the reference's 0 and are not written; *srcSizePtr is left alone.  A valid state
    is taken (the call goes on to the device, so its result is not checked here).  _extStateHC_fastReset on NULL is a
    deviation: 0, where the reference dereferences it."""
    doc, _ = golden
    dst = np.full(64, 0x5A, dtype=np.uint8)
    l0 = lib.LZ4B200_launch_count()
    for name, rows in doc["verdicts"]["calls"].items():
        offsets = [off for off, ret, _ in rows if ret == 0]
        assert offsets == ([None] if name != NAMES[1] else []) + list(range(1, 8)), name
        for off in offsets + ([None] if name == NAMES[1] else []):
            p, keep = mk.state_buffer(off) if off is not None else (None, None)
            got = call(lib, name, p, P, dst.ctypes.data, 4096, 8192, 9)
            assert got == ((0, 4096) if name.endswith("destSize") else 0), (name, off)
            if p is not None:
                assert (np.frombuffer(C.string_at(p, mk.STATE_BYTES), np.uint8) == mk.STATE_FILL).all(), (name, off)
            del keep
    assert (dst == 0x5A).all()
    assert lib.LZ4B200_launch_count() == l0


@pytest.mark.parametrize("name", ["LZ4_compress_HC_extStateHC", "LZ4_compress_HC_destSize"])
@pytest.mark.parametrize("offset", [0, 8])
def test_valid_state_is_left_as_init_stream_hc_leaves_it(lib, golden, name, offset):
    """The state image after the call is the reference's LZ4_initStreamHC image (the empty input: no launch)"""
    doc, _ = golden
    p, keep = mk.state_buffer(offset)
    dst = np.zeros(16, dtype=np.uint8)
    got = call(lib, name, p, P, dst.ctypes.data, 0, 16, 12)
    assert got == ((1, 0) if name.endswith("destSize") else 1)
    assert hashlib.sha256(C.string_at(p, mk.STATE_BYTES)).hexdigest() == doc["state"]["sha256"]
    del keep


def test_fast_reset_neither_reads_nor_writes_the_state(lib):
    p, keep = mk.state_buffer(0)
    dst = np.zeros(16, dtype=np.uint8)
    assert lib.LZ4_compress_HC_extStateHC_fastReset(p, P, dst.ctypes.data, 0, 16, 9) == 1
    assert (np.frombuffer(C.string_at(p, mk.STATE_BYTES), np.uint8) == mk.STATE_FILL).all()
    del keep


def golden_host_rows(doc, ins):
    """(name, size, capacity or target, level, ret, consumed) of every golden row the reference decides without
    parsing: the empty input, and a capacity below 1"""
    rows = []
    for iid, lv, caps, rets, dig in doc["vectors"]:
        for cap, r in zip(caps, rets):
            if ins[iid]["size"] == 0 or cap < 1:
                rows.append(("LZ4_compress_HC", ins[iid]["size"], cap, lv, r, None))
    for iid, lv, ts, rets, cons, dig in doc["dest_vectors"]:
        for t, r, c in zip(ts, rets, cons):
            if ins[iid]["size"] == 0:
                rows.append(("LZ4_compress_HC_destSize", 0, t, lv, r, c))
    return rows


def test_host_decided_golden_rows(lib, golden):
    """Every such golden row through each entry point: the reference's return value, the one 0x00 byte of an empty
    input and nothing else written, and no launch"""
    doc, ins = golden
    rows = golden_host_rows(doc, ins)
    assert len(rows) > 100
    p, keep = mk.state_buffer(0)
    l0 = lib.LZ4B200_launch_count()
    for name, n, cap, lv, r, c in rows:
        names = ["LZ4_compress_HC", NAMES[0], NAMES[1]] if name == "LZ4_compress_HC" else [name]
        for nm in names:
            dst = np.full(64, 0x5A, dtype=np.uint8)
            got = call(lib, nm, p, P, dst.ctypes.data, n, cap, lv)
            assert got == (r if c is None else (r, c)), (nm, n, cap, lv)
            assert dst[:r].tobytes() == b"\0" * r and (dst[r:] == 0x5A).all(), (nm, n, cap, lv)
    assert lib.LZ4B200_launch_count() == l0
    del keep


def test_size_and_capacity_rules(lib):
    """Sizes outside 0 .. LZ4_MAX_INPUT_SIZE, capacities and targets below 1, NULL pointers (NULL dst, NULL src with
    bytes to read, NULL srcSizePtr: deviations, the reference dereferences them): 0, nothing written, *srcSizePtr left
    alone, no launch"""
    dst = np.full(64, 0x5A, dtype=np.uint8)
    d = dst.ctypes.data
    p, keep = mk.state_buffer(0)
    l0 = lib.LZ4B200_launch_count()
    for lv in (-3, 0, 2, 9, 10, 12, 100):
        for name in ("LZ4_compress_HC",) + NAMES:
            dest = name.endswith("destSize")
            for n, cap in ((-1, 64), (MAX_INPUT + 1, 64), (-(1 << 31), 64), (100, 0), (100, -1), (0, 0), (0, -7)):
                assert call(lib, name, p, P, d, n, cap, lv) == ((0, n) if dest else 0), (name, n, cap, lv)
            assert call(lib, name, p, P, None, 100, 64, lv) == ((0, 100) if dest else 0), (name, lv)
            assert call(lib, name, p, None, d, 100, 64, lv) == ((0, 100) if dest else 0), (name, lv)
        assert lib.LZ4_compress_HC_destSize(p, P, d, None, 64, lv) == 0
    assert (dst == 0x5A).all()
    assert lib.LZ4B200_launch_count() == l0
    del keep


def test_no_device_every_call_fails_and_writes_nothing(lib):
    """Without a CUDA device each entry point that has a block to parse returns 0, leaves dst and *srcSizePtr alone and
    launches nothing: there is no CPU fallback"""
    if lib.LZ4B200_device_count() > 0:
        pytest.skip("a CUDA device is present")
    from lz4_b200 import block
    src = np.frombuffer(b"abcdabcdabcdabcdabcdabcd" * 40, dtype=np.uint8)
    p, keep = mk.state_buffer(0)
    l0 = lib.LZ4B200_launch_count()
    for lv in (-3, 1, 2, 3, 9, 10, 11, 12, 13):
        for name in ("LZ4_compress_HC",) + NAMES:
            for cap in (1, 7, 100, 4096):
                dst = np.full(4096 + 64, 0x5A, dtype=np.uint8)
                got = call(lib, name, p, src.ctypes.data, dst.ctypes.data, len(src), cap, lv)
                assert got == ((0, len(src)) if name.endswith("destSize") else 0), (name, lv, cap)
                assert (dst == 0x5A).all()
        assert block.LZ4_compress_HC(src, lv) == (0, b"")
        assert block.LZ4_compress_HC_destSize(src, 100, lv) == (0, len(src), b"")
    assert b"no CUDA device" in lib.LZ4B200_last_cuda_error()
    assert lib.LZ4B200_launch_count() == l0
    del keep


def test_golden_file_regenerates_byte_identically(reference):
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "kat_hc_dropin.json")
        mk.main(out)
        with open(out, "rb") as a, open(os.path.join(mk.HERE, "kat_hc_dropin.json"), "rb") as b:
            assert a.read() == b.read()
