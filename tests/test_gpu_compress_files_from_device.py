"""LZ4B200_compress_frames_from_device and LZ4B200_compress_legacy_from_device on the GPU against the host writers:
every golden frame of tests/golden/compress_frames_checksum.json (three flag combinations) and every legacy stream of
tests/golden/compress_legacy.json written from device memory, byte-identical to the host writers and to the recorded
lengths and digests, LZ4B200_ERR_DSTSIZE one byte below the bound, guard bytes around every output; the host writers'
1 MiB-group runs in a child process; a 1 GiB frame, 65 536 sources of 64 KB and a source past 2^32 in one allocation;
the launch count; ordering after the caller's stream; the pointer checks; device memory against the stated ceiling;
threads beside the host calls; and the Python wrappers."""
import json
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

import compress_frames_checksum_model as M               # noqa: E402
import compress_legacy_model as LM                       # noqa: E402
import test_gpu_compress_files_host as W                 # noqa: E402
from lz4_b200 import frame                               # noqa: E402

pytestmark = pytest.mark.gpu

GUARD, GAP, sha, frame_bound = W.GUARD, W.GAP, W.sha, W.frame_bound
MIB = 1 << 20
ERR_ARG, ERR_DSTSIZE = -1, -5
FLAGS = W.FLAGS


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


def dev_call(lib, datas, caps, legacy=False, level=1, bsid=7, cs=0, parallel=0, bsum=0, csum=1, src=None, soff=None,
             stream=None):
    """one call over sources GAP bytes apart at an odd offset of one device buffer (or src at soff) into abutting
    outputs at an odd base between guards: (return code, results, the output of each file as bytes)"""
    n = len(datas)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    if src is None:
        soff = np.zeros(n, dtype=np.int64) + 3
        if n:
            soff[1:] += np.cumsum(sizes + GAP)[:-1]
        host = np.zeros(int((sizes + GAP).sum()) + 3 + 16, dtype=np.uint8)
        for d, o in zip(datas, soff):
            host[o:o + len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
        src = torch.from_numpy(host).cuda()
    caps = np.array(caps, dtype=np.int64)
    room = np.maximum(caps, 0)
    doff = 7 + np.concatenate([[0], np.cumsum(room)[:-1]]).astype(np.int64) if n else np.zeros(0, dtype=np.int64)
    out = np.full(int(room.sum()) + 7 + 64, GUARD, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int64)
    s = stream.cuda_stream if stream is not None else torch.cuda.current_stream().cuda_stream
    if legacy:
        rc = lib.LZ4B200_compress_legacy_from_device(src.data_ptr(), soff.ctypes.data, sizes.ctypes.data, out.ctypes.data,
                                                     doff.ctypes.data, caps.ctypes.data, res.ctypes.data, n, level, s)
    else:
        rc = lib.LZ4B200_compress_frames_from_device(src.data_ptr(), soff.ctypes.data, sizes.ctypes.data, out.ctypes.data,
                                                     doff.ctypes.data, caps.ctypes.data, res.ctypes.data, n, bsid, level,
                                                     cs, parallel, bsum, csum, s)
    mask = np.ones(len(out), dtype=bool)
    for o, r in zip(doff, res):
        if r > 0:
            mask[o:o + r] = False
    assert not (out[mask] != GUARD).any(), "a byte outside [dst_f, dst_f + result_f) was written"
    return rc, res.tolist(), [out[o:o + r].tobytes() if r > 0 else b"" for o, r in zip(doff, res)]


def both(lib, datas, caps, **kw):
    """the call and the host writer on the same arguments agree; the call's (results, outputs)"""
    rc, res, outs = dev_call(lib, datas, caps, **kw)
    hrc, hres, houts = W.host_call(lib, datas, caps, **kw)
    assert rc == hrc == 0, lib.LZ4B200_last_cuda_error()
    assert res == hres and outs == houts
    return res, outs


@pytest.fixture(scope="module")
def frames_fixture():
    with open(os.path.join(HERE, "golden", "compress_frames_checksum.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("flags", sorted(FLAGS))
def test_golden_frames(lib, oracle, frames_fixture, flags):
    bsum, csum = FLAGS[flags]
    calls = {}
    for c in frames_fixture["frames"]:
        calls.setdefault((c["level"], c["bsid"], c["content_size"]), []).append(c)
    for (level, bsid, cs), cases in sorted(calls.items()):
        datas = [M.corpus_data(oracle, c["kind"], c["size"], c["seed"]) for c in cases]
        bounds = [frame_bound(lib, len(d), bsid, bsum, csum) for d in datas]
        kw = dict(level=level, bsid=bsid, cs=int(cs), bsum=bsum, csum=csum)
        res, outs = both(lib, datas, bounds, **kw)
        for c, r, o in zip(cases, res, outs):
            g = c["sums"][flags]
            assert (r, sha(o)) == (g["length"], g["sha256"]), (c["id"], flags)
        short = list(bounds)
        short[len(short) // 2] -= 1
        res2, _ = both(lib, datas, short, **kw)
        assert res2[len(short) // 2] == ERR_DSTSIZE


def test_golden_legacy(lib, oracle):
    with open(os.path.join(HERE, "golden", "compress_legacy.json")) as f:
        streams = json.load(f)["streams"]
    calls = {}
    for c in streams:
        calls.setdefault(c["level"], []).append(c)
    for level, cases in sorted(calls.items()):
        datas = [LM.corpus_data(oracle, c["kind"], c["size"], c["seed"]) for c in cases]
        bounds = [LM.bound(len(d)) for d in datas]
        res, outs = both(lib, datas, bounds, legacy=True, level=level)
        for c, r, o in zip(cases, res, outs):
            assert (r, sha(o)) == (c["length"], c["sha256"]), c["id"]
        res2, _ = both(lib, datas, [b - 1 if b > 4 else b for b in bounds], legacy=True, level=level)
        assert all(r == ERR_DSTSIZE for r, b in zip(res2, bounds) if b > 4)


def child_main(out_dir):
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle
    lib, oracle = _lib.load(), Oracle()
    names = []
    for name, files, hargs, _ in W.child_runs(oracle):
        if hargs.get("level") not in (1, 9):
            continue
        if hargs.get("legacy"):
            caps = [LM.bound(len(d)) for d in files]
        else:
            caps = [frame_bound(lib, len(d), hargs["bsid"], hargs["bsum"], hargs["csum"]) for d in files]
        both(lib, files, caps, **hargs)
        names.append(name)
    with open(os.path.join(out_dir, "groups.json"), "w") as f:
        json.dump(names, f)


def test_one_mib_groups_in_a_child(lib, oracle, tmp_path):
    env = dict(os.environ, LZ4B200_HOST_CHUNK_MB="1", LZ4B200_HOST_WRITE_MB="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, timeout=3000,
                       capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    with open(str(tmp_path / "groups.json")) as f:
        assert len(json.load(f)) == 2 * 9


def test_one_gib_frame(lib, oracle):
    data = oracle.datagen_mt(1 << 30, 1 << 20, 0.5, 41)
    for csum in (1, 0):
        res, outs = both(lib, [data], [frame_bound(lib, len(data), 7, 0, csum)], csum=csum)
    assert frame.decompress_file(outs[0]) == data.tobytes()


def test_many_small_files(lib, oracle):
    pool = oracle.datagen(8 * MIB, 0.5, 9)
    rng = np.random.default_rng(3)
    datas = [pool[a:a + 65536] for a in rng.integers(0, len(pool) - 65536, 65536)]
    both(lib, datas, [frame_bound(lib, 65536, 7, 0, 1)] * len(datas))


def test_source_past_4gib(lib, oracle):
    a, b = oracle.datagen(100000, 0.5, 12), oracle.datagen(5 * MIB + 7, 0.5, 13)
    src = torch.zeros((1 << 32) + 6 * MIB, dtype=torch.uint8, device="cuda")
    soff = np.array([5, (1 << 32) + 9], dtype=np.int64)
    src[5:5 + len(a)] = torch.from_numpy(a).cuda()
    src[int(soff[1]):int(soff[1]) + len(b)] = torch.from_numpy(b).cuda()
    for legacy in (False, True):
        caps = [LM.bound(len(d)) if legacy else frame_bound(lib, len(d), 7, 1, 1) for d in (a, b)]
        kw = dict(legacy=True) if legacy else dict(bsum=1, csum=1)
        rc, res, outs = dev_call(lib, [a, b], caps, src=src, soff=soff, **kw)
        hrc, hres, houts = W.host_call(lib, [a, b], caps, **kw)
        assert rc == hrc == 0 and res == hres and outs == houts
    del src


def test_launches_are_the_host_writers(lib, oracle):
    datas = [oracle.datagen(n, 0.5, 3).tobytes() for n in (0, 1000, 5 * MIB)]
    for kw in (dict(bsum=1, csum=1), dict(legacy=True, level=9)):
        caps = [LM.bound(len(d)) if kw.get("legacy") else frame_bound(lib, len(d), 7, 1, 1) for d in datas]
        before = lib.LZ4B200_launch_count()
        W.host_call(lib, datas, caps, **kw)
        host = lib.LZ4B200_launch_count() - before
        before = lib.LZ4B200_launch_count()
        dev_call(lib, datas, caps, **kw)
        assert lib.LZ4B200_launch_count() - before == host


def test_ordered_after_the_callers_stream(lib, oracle):
    """a write of the source still pending on the caller's stream is what the call compresses"""
    d = oracle.datagen(5 * MIB + 3, 0.5, 7)
    src = torch.zeros(len(d) + 16, dtype=torch.uint8, device="cuda")
    staged = torch.from_numpy(d).cuda()
    side = torch.cuda.Stream()
    torch.cuda.synchronize()
    cap = [frame_bound(lib, len(d), 7, 0, 1)]
    with torch.cuda.stream(side):
        torch.cuda._sleep(200_000_000)
        src[:len(d)].copy_(staged)
        rc, res, outs = dev_call(lib, [d], cap, src=src, soff=np.zeros(1, dtype=np.int64), stream=side)
    assert rc == 0 and outs == W.host_call(lib, [d], cap)[2]


def test_pointer_checks(lib):
    i64 = lambda *v: np.array(v, dtype=np.int64)              # noqa: E731
    off, size, cap, res = i64(0), i64(100), i64(200), i64(-99)
    host_src = np.zeros(200, dtype=np.uint8)
    out = np.full(200, GUARD, dtype=np.uint8)
    s = torch.cuda.current_stream().cuda_stream
    for legacy in (False, True):
        tail = (1, 0) if legacy else (1, 7, 1, 0, 0, 0, 1)
        call = lib.LZ4B200_compress_legacy_from_device if legacy else lib.LZ4B200_compress_frames_from_device
        rc = call(host_src.ctypes.data, off.ctypes.data, size.ctypes.data, out.ctypes.data, off.ctypes.data,
                  cap.ctypes.data, res.ctypes.data, *tail, s)
        assert rc == ERR_ARG and b"d_src" in lib.LZ4B200_last_cuda_error()
        dsrc = torch.zeros(200, dtype=torch.uint8, device="cuda")
        dout = torch.full((200,), GUARD, dtype=torch.uint8, device="cuda")
        rc = call(dsrc.data_ptr(), off.ctypes.data, size.ctypes.data, dout.data_ptr(), off.ctypes.data,
                  cap.ctypes.data, res.ctypes.data, *tail, s)
        assert rc == ERR_ARG and b"h_dst" in lib.LZ4B200_last_cuda_error()
        assert (dout == GUARD).all() and (out == GUARD).all() and res[0] == -99


def test_device_memory_stays_under_the_ceiling(lib, oracle):
    """the host writers' ceiling at G = 512 MiB and the fast levels without the staged source: 4 slots x (G + G/255 +
    32 B + G + G/255 + 24 B + 56 B + 8, each buffer rounded up by 1 MiB + 16) + the ring; no growth after the first call"""
    G, B = 512 * MIB, 65536
    ceiling = 4 * (2 * (G + G // 255) + 128 * B + 8 + 5 * (MIB + 16)) + 5 * 40
    data = torch.from_numpy(oracle.datagen_mt(1 << 30, 1 << 20, 0.5, 43)).cuda()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    cap = [frame_bound(lib, data.numel(), 7, 1, 1)]
    zero = np.zeros(1, dtype=np.int64)
    sizes = [data.numel()]
    out = np.empty(cap[0], dtype=np.uint8)
    res = np.zeros(1, dtype=np.int64)
    args = (data.data_ptr(), zero.ctypes.data, np.array(sizes, dtype=np.int64).ctypes.data, out.ctypes.data,
            zero.ctypes.data, np.array(cap, dtype=np.int64).ctypes.data, res.ctypes.data, 1, 7, 1, 0, 0, 1, 1,
            torch.cuda.current_stream().cuda_stream)
    assert lib.LZ4B200_compress_frames_from_device(*args) == 0
    free1 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        assert lib.LZ4B200_compress_frames_from_device(*args) == 0
    assert torch.cuda.mem_get_info()[0] >= free1
    assert free0 - free1 <= ceiling, (free0 - free1, ceiling)


def test_threads_beside_the_host_calls(lib, oracle):
    datas = [oracle.datagen(n, 0.5, n % 7).tobytes() for n in (100, 70000, 3 * MIB + 5)]
    caps = [frame_bound(lib, len(d), 7, 1, 1) for d in datas]
    serial = W.host_call(lib, datas, caps, bsum=1)
    files = frame.compress_files(datas)
    errors = []

    def from_device():
        for _ in range(3):
            if dev_call(lib, datas, caps, bsum=1) != serial:
                errors.append("from_device")

    def host():
        for _ in range(3):
            if W.host_call(lib, datas, caps, bsum=1) != serial or [g[3] for g in frame.decompress_files(files)] != datas:
                errors.append("host")

    ts = [threading.Thread(target=from_device) for _ in range(2)] + [threading.Thread(target=host) for _ in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_python_wrappers(oracle):
    d = oracle.datagen(300000, 0.5, 4)
    ts = [torch.from_numpy(d).cuda(), torch.from_numpy(d[:1000].copy()).cuda().view(torch.int32).reshape(10, 25),
          torch.zeros(0, dtype=torch.float16, device="cuda")]
    raws = [d, d[:1000], np.zeros(0, dtype=np.uint8)]
    for kw in (dict(), dict(level=3, block_size_id=4, content_size=True, block_checksum=True), dict(legacy=True),
               dict(parallel=True)):
        assert frame.compress_files_from_device(ts, **kw) == frame.compress_files(raws, **kw), kw
    assert frame.compress_file_from_device(ts[1]) == frame.compress_file(raws[1])
    assert frame.compress_files_from_device([]) == []
    with pytest.raises(ValueError, match="contiguous"):
        frame.compress_file_from_device(ts[1].t())
    with pytest.raises(ValueError, match="CPU"):
        frame.compress_file_from_device(torch.from_numpy(d))
    if torch.cuda.device_count() > 1:
        with pytest.raises(ValueError, match="device"):
            frame.compress_file_from_device(ts[0].to("cuda:1"))


if __name__ == "__main__":
    child_main(sys.argv[1])
