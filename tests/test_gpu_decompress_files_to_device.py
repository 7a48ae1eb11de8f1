"""LZ4B200_decompress_files_to_device on the GPU against LZ4B200_decompress_files_host: every file of
tests/golden/decompress_files.json, verified and with skipChecksums, at exact capacity and one byte less, with the same
results and the same bytes in device memory as in host memory, and guard bytes intact around every region (regions at
odd offsets, so that the scatter's byte edges and its shifted words both run); the 1 MiB-group corpus in a child
process (frames, units and blocks across group edges, carried content hashes, files that fail in a later group than
their first bytes); a 1 GiB frame, 65 536 files of 64 KB and an output past 2^32 in one allocation; the launch count;
ordering after the caller's stream; the pointer checks; device memory over repeated calls; threads beside the host
calls; and the Python wrappers."""
import hashlib
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if __name__ == "__main__":
    sys.path[:0] = [os.path.dirname(HERE), HERE]

import decompress_files_model as dm                      # noqa: E402
import test_gpu_decompress_files_host as H               # noqa: E402
from lz4_b200 import frame                               # noqa: E402

pytestmark = pytest.mark.gpu

GUARD, GAP = H.GUARD, H.GAP
MIB = 1 << 20
ERR_ARG = -1


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


@pytest.fixture(scope="module")
def corpus(oracle):
    return H.golden_files(oracle)


def layout(caps):
    """H.host_call's output layout: regions GAP guard bytes apart, and the buffer's length"""
    oo = np.zeros(len(caps), dtype=np.int64)
    at = GAP
    for k, c in enumerate(caps):
        oo[k] = at
        at += max(c, 0) + GAP
    return oo, at


def dev_call(lib, files, caps, skip=False, stream=None, out=None, oo=None):
    """the call on files packed in one host buffer into a guard-filled device buffer laid out as H.host_call's:
    (rc, results, consumed, prefixes, device output, offsets)"""
    sizes = np.array([len(f) for f in files], dtype=np.int64)
    offs = np.zeros(len(files), dtype=np.int64)
    offs[1:] = np.cumsum(sizes)[:-1]
    src = np.frombuffer(b"".join(files) or b"\0", dtype=np.uint8)
    n = len(files)
    res, con, pre = (np.full(n, -99, dtype=np.int64) for _ in range(3))
    capa = np.array(caps, dtype=np.int64)
    if out is None:
        oo, total = layout(caps)
        out = torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
    s = stream.cuda_stream if stream is not None else torch.cuda.current_stream().cuda_stream
    rc = lib.LZ4B200_decompress_files_to_device(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, out.data_ptr(),
                                                oo.ctypes.data, capa.ctypes.data, res.ctypes.data, con.ctypes.data,
                                                pre.ctypes.data, n, 1 if skip else 0, s)
    return rc, res.tolist(), con.tolist(), pre.tolist(), out, oo


def check_against_host(lib, files, caps, skip):
    """the same results as the host call and the same whole buffer: every region's bytes, and the guards around them"""
    hres, hcon, hpre, hout, _ = H.host_call(lib, files, caps, skip)
    rc, res, con, pre, out, _ = dev_call(lib, files, caps, skip)
    assert rc == 0, lib.LZ4B200_last_cuda_error()
    assert (res, con, pre) == (hres, hcon, hpre)
    d = out.cpu().numpy()
    assert d.tobytes() == hout.tobytes()
    return res, pre


@pytest.mark.parametrize("mode", ["verify", "skip"])
def test_golden_files(lib, corpus, oracle, mode):
    g, files = corpus
    skip = mode == "skip"
    exact = H.sized_caps(files, skip)
    for caps in (exact, [e - 1 if e > 0 else 0 for e in exact]):
        check_against_host(lib, files, caps, skip)


def child_main(d):
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle
    lib = _lib.load()
    files = H.chunked_files(Oracle())
    with open(os.path.join(d, "ok.txt"), "w") as f:
        for skip in (False, True):
            caps = H.sized_caps(files, skip)
            res, pre = check_against_host(lib, files, caps, skip)
            f.write("%s %d %d\n" % (skip, sum(r < 0 for r in res), sum(p > 0 for r, p in zip(res, pre) if r < 0)))


def test_one_mib_groups_in_a_child(lib, oracle, tmp_path):
    env = dict(os.environ, LZ4B200_HOST_CHUNK_MB="1", LZ4B200_HOST_WRITE_MB="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, timeout=1200,
                       capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    lines = open(str(tmp_path / "ok.txt")).read().split("\n")
    # verified, files fail -- among them the late corruptions, which fail with bytes placed by earlier groups
    assert int(lines[0].split()[1]) > 0 and int(lines[0].split()[2]) > 0, lines


def test_one_gib_frame(lib, oracle):
    data = oracle.datagen_mt(1 << 30, 1 << 20, 0.5, 41)
    f = H.gpu_frame(data, 7)
    for skip in (False, True):
        rc, res, con, pre, out, oo = dev_call(lib, [f], [len(data)], skip)
        assert rc == 0 and res == [len(data)] and con == [len(f)]
        assert torch.equal(out[GAP:GAP + len(data)].cpu(), torch.from_numpy(data))
        assert (out[:GAP] == GUARD).all() and (out[GAP + len(data):] == GUARD).all()
        del out


def test_many_small_files(lib, oracle):
    """65 536 one-frame files of 64 KB; the host call's results and bytes"""
    pool = oracle.datagen(8 * MIB, 0.5, 9)
    rng = np.random.default_rng(5)
    datas = [pool[a:a + 65536] for a in rng.integers(0, len(pool) - 65536, 64)]
    frames = [frame.compress_file(d, block_size_id=4) for d in datas]
    files = [frames[k % 64] for k in range(65536)]
    caps = [65536] * len(files)
    check_against_host(lib, files, caps, False)


def test_output_past_4gib(lib, oracle):
    """one allocation of 4 GiB + 3 MiB: the second file's region starts past 2^32, at an odd offset"""
    d = oracle.datagen(3 * MIB - 5, 0.5, 13)
    f = frame.compress_file(d, block_size_id=4)
    out = torch.full(((1 << 32) + 3 * MIB + 64,), GUARD, dtype=torch.uint8, device="cuda")
    oo = np.array([0, (1 << 32) + 7], dtype=np.int64)
    rc, res, _, _, out, _ = dev_call(lib, [f, f], [len(d), len(d)], out=out, oo=oo)
    assert rc == 0 and res == [len(d)] * 2
    for o in oo:
        assert torch.equal(out[int(o):int(o) + len(d)].cpu(), torch.from_numpy(d))
    assert (out[(1 << 32):(1 << 32) + 7] == GUARD).all() and (out[(1 << 32) + 7 + len(d):] == GUARD).all()
    del out


def test_launches_are_the_host_calls_plus_one_scatter(lib, corpus):
    _, files = corpus
    files = files[:6]
    caps = H.sized_caps(files)
    before = lib.LZ4B200_launch_count()
    H.host_call(lib, files, caps)
    host = lib.LZ4B200_launch_count() - before
    before = lib.LZ4B200_launch_count()
    assert dev_call(lib, files, caps)[0] == 0
    assert lib.LZ4B200_launch_count() - before == host + 1


def test_ordered_after_the_callers_stream(lib, oracle):
    """a fill of the destination still pending on the caller's stream is overwritten by the decoded bytes"""
    d = oracle.datagen(5 * MIB + 3, 0.5, 7)
    f = frame.compress_file(d)
    oo, total = layout([len(d)])
    side = torch.cuda.Stream()
    out = torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        out.fill_(0x5A)
        rc, res = dev_call(lib, [f], [len(d)], stream=side, out=out, oo=oo)[:2]
    assert rc == 0 and res == [len(d)]
    torch.cuda.synchronize()
    assert torch.equal(out[GAP:GAP + len(d)].cpu(), torch.from_numpy(d))
    assert (out[:GAP] == 0x5A).all()


def test_pointer_checks(lib, oracle):
    f = frame.compress_file(oracle.datagen(1000, 0.5, 3))
    src = np.frombuffer(f, dtype=np.uint8)
    i64 = lambda *v: np.array(v, dtype=np.int64)              # noqa: E731
    off, size, cap, res = i64(0), i64(len(f)), i64(1000), i64(-99)
    host_dst = np.full(1000, GUARD, dtype=np.uint8)
    s = torch.cuda.current_stream().cuda_stream
    rc = lib.LZ4B200_decompress_files_to_device(src.ctypes.data, off.ctypes.data, size.ctypes.data, host_dst.ctypes.data,
                                                off.ctypes.data, cap.ctypes.data, res.ctypes.data, None, None, 1, 0, s)
    assert rc == ERR_ARG and b"d_dst" in lib.LZ4B200_last_cuda_error()
    assert (host_dst == GUARD).all() and res[0] == -99
    dsrc = torch.from_numpy(src.copy()).cuda()
    out = torch.full((1000,), GUARD, dtype=torch.uint8, device="cuda")
    rc = lib.LZ4B200_decompress_files_to_device(dsrc.data_ptr(), off.ctypes.data, size.ctypes.data, out.data_ptr(),
                                                off.ctypes.data, cap.ctypes.data, res.ctypes.data, None, None, 1, 0, s)
    assert rc == ERR_ARG and b"h_src" in lib.LZ4B200_last_cuda_error()
    assert (out == GUARD).all() and res[0] == -99


def test_device_memory_stays_under_the_ceiling(lib, corpus):
    """growth over the first calls is at most section 3.17's four slots (the default 64 MiB groups: the slots and the
    staged pieces, 2 x 64 MiB + 16; the decode workspace, at most 2 x 64 MiB; the packed output, 64 MiB + 16; the
    table; each buffer rounded up by at most 1 MiB) plus the run tables, and none after"""
    _, files = corpus
    caps = H.sized_caps(files)
    G = 64 * MIB
    ceiling = 4 * (2 * G + 2 * G + G + 8 * MIB + 6 * (MIB + 16)) + 5 * 40
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    out = torch.empty(layout(caps)[1], dtype=torch.uint8, device="cuda")
    oo = layout(caps)[0]
    dev_call(lib, files, caps, out=out, oo=oo)
    free1 = torch.cuda.mem_get_info()[0]
    for _ in range(4):
        dev_call(lib, files, caps, out=out, oo=oo)
        H.host_call(lib, files, caps)
    assert torch.cuda.mem_get_info()[0] >= free1
    assert free0 - free1 - out.numel() <= ceiling, (free0 - free1, ceiling)


def test_threads_beside_the_host_calls(lib, corpus, oracle):
    _, files = corpus
    caps = H.sized_caps(files)
    want = H.host_call(lib, files, caps)
    datas = [oracle.datagen(n, 0.5, n % 7).tobytes() for n in (100, 70000, 3 * MIB + 5)]
    written = frame.compress_files(datas)
    errors = []

    def to_device():
        for _ in range(3):
            rc, res, con, pre, out, _ = dev_call(lib, files, caps)
            if rc != 0 or (res, con, pre) != tuple(want[:3]) or out.cpu().numpy().tobytes() != want[3].tobytes():
                errors.append("to_device")

    def host():
        for _ in range(3):
            if H.host_call(lib, files, caps)[:3] != tuple(want[:3]) or frame.compress_files(datas) != written:
                errors.append("host")

    ts = [threading.Thread(target=to_device) for _ in range(2)] + [threading.Thread(target=host) for _ in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_python_wrappers(oracle):
    d = oracle.datagen(500000, 0.5, 8).tobytes()
    for t in (torch.arange(1000, dtype=torch.float32), torch.randn(3, 77777).to(torch.bfloat16),
              torch.randint(0, 1000, (5 * MIB + 3,), dtype=torch.int16), torch.zeros(0, dtype=torch.int64)):
        t = t.cuda()
        raw = t.view(-1).view(torch.uint8) if t.numel() else torch.zeros(0, dtype=torch.uint8, device="cuda")
        for kw in (dict(), dict(block_size_id=4, block_checksum=True), dict(legacy=True)):
            f = frame.compress_file_from_device(t, **kw)
            assert f == frame.compress_file(raw.cpu().numpy(), **kw)
            back = frame.decompress_file_to_device(f)
            assert back.is_cuda and back.dtype == torch.uint8 and torch.equal(back, raw)
    f = frame.compress_file(d)
    bad = bytearray(f)
    bad[-1] ^= 1
    cut = f + f[:-30]
    datas = [f, bytes(bad), cut, b"", f]
    for caps in (None, [len(d), len(d), 2 * len(d), 0, len(d) - 1]):
        for skip in (False, True):
            want = frame.decompress_files(datas, caps, skip)
            got = frame.decompress_files_to_device(datas, caps, skip)
            assert [g[:3] for g in got] == [w[:3] for w in want]
            assert [g[3].cpu().numpy().tobytes() for g in got] == [w[3] for w in want]
            base = got[0][3].untyped_storage().data_ptr()
            assert all(g[3].untyped_storage().data_ptr() == base for g in got)
    with pytest.raises(frame.Lz4FrameError) as e:
        frame.decompress_file_to_device(bytes(bad))
    assert e.value.code == -7
    assert frame.decompress_files_to_device([]) == []


if __name__ == "__main__":
    child_main(sys.argv[1])
