"""LZ4B200_compress_frames_host and LZ4B200_compress_legacy_host on the GPU: every frame of
tests/golden/compress_frames_checksum.json in its three flag combinations, the `lz4` tool's own files of it and every
stream of tests/golden/compress_legacy.json, byte-identical to the reference at capacity == bound and
LZ4B200_ERR_DSTSIZE at bound - 1, with guard bytes around every output region; edge sizes, a 40 MiB checksummed frame of
64 KB blocks and a 20 MiB + 1 legacy stream in a child process with 1 MiB writer groups (every slot reused, frames
spanning hundreds of groups) against the device calls; at the default group size a 1 GiB level-1 frame against the
device call, 20 000 small files in one call and outputs past 2^32 in one buffer; pinned and pageable sources; round
trips through LZ4B200_decompress_files_host; four threads beside the other host calls; device memory over repeated
calls against the stated ceiling; and the Python wrappers."""
import hashlib
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
from lz4_b200 import batch, frame                        # noqa: E402

pytestmark = pytest.mark.gpu

GUARD, GAP = 0xA5, 40
MIB = 1 << 20
ERR_DSTSIZE = -5
FLAGS = {"B": (1, 0), "C": (0, 1), "BC": (1, 1)}


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    return lib


@pytest.fixture(scope="module")
def oracle():
    from oracle.pyoracle import Oracle
    return Oracle()


@pytest.fixture(autouse=True)
def release_workspaces():
    yield
    torch.cuda.synchronize()
    batch._workspaces.clear()
    torch.cuda.empty_cache()


def frame_bound(lib, n, bsid, bsum, csum):
    return int(lib.LZ4B200_compressFrameBound_checksummed(n, bsid, bsum, csum))


def host_call(lib, datas, caps, legacy=False, level=1, bsid=7, cs=0, parallel=0, bsum=0, csum=1, pinned=False,
              src_gap=GAP):
    """one host call over sources GAP bytes apart and abutting outputs at an odd base between guards: (return code,
    results, the output of each file as bytes)"""
    n = len(datas)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    soff = np.zeros(n, dtype=np.int64)
    if n:
        soff[1:] = np.cumsum(sizes + src_gap)[:-1]
    total = int((sizes + src_gap).sum()) + 1
    src = torch.empty(total, dtype=torch.uint8).pin_memory().numpy() if pinned else np.empty(total, dtype=np.uint8)
    for d, o in zip(datas, soff):
        src[o:o + len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
    caps = np.array(caps, dtype=np.int64)
    room = np.maximum(caps, 0)
    doff = 7 + np.concatenate([[0], np.cumsum(room)[:-1]]).astype(np.int64) if n else np.zeros(0, dtype=np.int64)
    out = np.full(int(room.sum()) + 7 + 64, GUARD, dtype=np.uint8)
    res = np.zeros(n, dtype=np.int64)
    if legacy:
        rc = lib.LZ4B200_compress_legacy_host(src.ctypes.data, soff.ctypes.data, sizes.ctypes.data, out.ctypes.data,
                                              doff.ctypes.data, caps.ctypes.data, res.ctypes.data, n, level)
    else:
        rc = lib.LZ4B200_compress_frames_host(src.ctypes.data, soff.ctypes.data, sizes.ctypes.data, out.ctypes.data,
                                              doff.ctypes.data, caps.ctypes.data, res.ctypes.data, n, bsid, level, cs,
                                              parallel, bsum, csum)
    mask = np.ones(len(out), dtype=bool)
    for o, r in zip(doff, res):
        if r > 0:
            mask[o:o + r] = False
    assert not (out[mask] != GUARD).any(), "a byte outside [dst_f, dst_f + result_f) was written"
    return rc, res.tolist(), [out[o:o + r].tobytes() if r > 0 else b"" for o, r in zip(doff, res)]


def device_call(datas, legacy=False, level=1, bsid=7, cs=False, parallel=False, bsum=False, csum=True):
    """the device call on the same files with a budget that covers them all: (results, bytes)"""
    n = len(datas)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    offs = np.zeros(n, dtype=np.int64)
    offs[1:] = np.cumsum(sizes)[:-1]
    src = torch.from_numpy(np.frombuffer(b"".join(bytes(d) for d in datas) + b"\0" * 64, dtype=np.uint8).copy()).cuda()
    t = lambda a: torch.from_numpy(a).cuda()
    if legacy:
        caps = np.array([LM.bound(len(d)) for d in datas], dtype=np.int64)
    else:
        caps = np.array([M.bound(len(d), bsid or 4, bsum, csum) for d in datas], dtype=np.int64)
    o = np.concatenate([[0], np.cumsum(caps)[:-1]]).astype(np.int64)
    kw = dict(out_offsets=t(o), capacities=t(caps))
    if legacy:
        out, res = batch.compress_legacy(src, t(offs), t(sizes), level=level, **kw)
    else:
        out, res = batch.compress_frames_checksummed(src, t(offs), t(sizes), block_size_id=bsid, level=level,
                                                     content_size=cs, parallel=parallel, block_checksum=bsum,
                                                     content_checksum=csum, **kw)
    torch.cuda.synchronize()
    res = res.cpu().tolist()
    h = out.cpu().numpy()
    del src, out
    return res, [h[a:a + r].tobytes() if r > 0 else b"" for a, r in zip(o, res)]


# ------------------------------------------------------------------------------------------
# the golden corpus
# ------------------------------------------------------------------------------------------
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
        assert bounds == [c["sums"][flags]["bound"] for c in cases]
        rc, res, outs = host_call(lib, datas, bounds, level=level, bsid=bsid, cs=int(cs), bsum=bsum, csum=csum)
        assert rc == 0
        for c, r, o in zip(cases, res, outs):
            g = c["sums"][flags]
            assert (r, sha(o)) == (g["length"], g["sha256"]), (c["id"], flags)
        # one byte below the bound: LZ4B200_ERR_DSTSIZE for that file alone
        short = list(bounds)
        short[len(short) // 2] -= 1
        rc, res2, outs2 = host_call(lib, datas, short, level=level, bsid=bsid, cs=int(cs), bsum=bsum, csum=csum)
        assert rc == 0 and res2[len(short) // 2] == ERR_DSTSIZE
        assert [r for k, r in enumerate(res2) if k != len(short) // 2] == [r for k, r in enumerate(res)
                                                                            if k != len(short) // 2]


def test_cli_frames(lib, oracle, frames_fixture):
    data = M.cli_data(oracle)
    for c in frames_fixture["cli"]:
        bsum, csum = int(c["block_sum"]), int(c["content_sum"])
        for pinned in (False, True):
            rc, res, outs = host_call(lib, [data], [frame_bound(lib, len(data), c["bsid"], bsum, csum)], level=c["level"],
                                      bsid=c["bsid"], bsum=bsum, csum=csum, pinned=pinned)
            assert rc == 0 and (res[0], sha(outs[0])) == (c["length"], c["sha256"]), c["args"]


def test_golden_legacy(lib, oracle):
    with open(os.path.join(HERE, "golden", "compress_legacy.json")) as f:
        streams = json.load(f)["streams"]
    calls = {}
    for c in streams:
        calls.setdefault(c["level"], []).append(c)
    for level, cases in sorted(calls.items()):
        datas = [LM.corpus_data(oracle, c["kind"], c["size"], c["seed"]) for c in cases]
        bounds = [LM.bound(len(d)) for d in datas]
        assert bounds == [c["bound"] for c in cases]
        rc, res, outs = host_call(lib, datas, bounds, legacy=True, level=level)
        assert rc == 0
        for c, r, o in zip(cases, res, outs):
            assert (r, sha(o)) == (c["length"], c["sha256"]), c["id"]
        short = [b - 1 if b > 4 else b for b in bounds]
        rc, res2, _ = host_call(lib, datas, short, legacy=True, level=level)
        assert rc == 0 and all(r == ERR_DSTSIZE for r, b in zip(res2, bounds) if b > 4)


# ------------------------------------------------------------------------------------------
# 1 MiB groups, in a child process (the group size is read once per process)
# ------------------------------------------------------------------------------------------
LEVELS = [-5, 1, 2, 9, 10]


def child_files(oracle, level):
    """edge sizes around the block size and, at the fast levels, the long frame and the long legacy stream"""
    small = [oracle.datagen(n, 0.5, n % 97).tobytes() for n in (0, 1, 65535, 65536, 65537)]
    if level >= 2:
        return small, small
    big = [oracle.datagen(n, 0.5, 5).tobytes() for n in (4 * MIB - 1, 4 * MIB, 4 * MIB + 1)]
    frames = small + big + [oracle.datagen(40 * MIB, 0.5, 6).tobytes()]
    legacy = small + [oracle.datagen(20 * MIB + 1, 0.5, 7).tobytes()]
    return frames, legacy


def child_runs(oracle):
    """every (name, files, host arguments, device arguments) the child runs"""
    for level in LEVELS:
        frames, legacy = child_files(oracle, level)
        for flags in ("", "B", "C", "BC"):
            bsum, csum = int("B" in flags), int("C" in flags)
            for bsid, cs in ((4, 0), (7, 1)):
                yield ("F%d_%s_b%d_cs%d" % (level, flags, bsid, cs), frames,
                       dict(level=level, bsid=bsid, cs=cs, bsum=bsum, csum=csum),
                       dict(level=level, bsid=bsid, cs=bool(cs), bsum=bool(bsum), csum=bool(csum)))
        yield ("L%d" % level, legacy, dict(legacy=True, level=level), dict(legacy=True, level=level))


def child_main(out_dir):
    from lz4_b200 import _lib
    from oracle.pyoracle import Oracle
    lib, oracle = _lib.load(), Oracle()
    got = {}
    for name, files, hargs, _ in child_runs(oracle):
        if hargs.get("legacy"):
            caps = [LM.bound(len(d)) for d in files]
        else:
            caps = [frame_bound(lib, len(d), hargs["bsid"], hargs["bsum"], hargs["csum"]) for d in files]
        rc, res, outs = host_call(lib, files, caps, **hargs)
        got[name] = [rc, res, [sha(o) for o in outs]]
    with open(os.path.join(out_dir, "groups.json"), "w") as f:
        json.dump(got, f)


def test_one_mib_groups_in_a_child(lib, oracle, tmp_path):
    env = dict(os.environ, LZ4B200_HOST_WRITE_MB="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, timeout=3000,
                       capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    with open(str(tmp_path / "groups.json")) as f:
        got = json.load(f)
    for name, files, _, dargs in child_runs(oracle):
        res, outs = device_call(files, **dargs)
        assert got[name] == [0, res, [sha(o) for o in outs]], name


# ------------------------------------------------------------------------------------------
# the default group size
# ------------------------------------------------------------------------------------------
def test_one_gib_frame(lib, oracle):
    data = oracle.datagen_mt(1 << 30, 1 << 20, 0.5, 41)
    res, outs = device_call([data.tobytes()])
    rc, hres, houts = host_call(lib, [data], [frame_bound(lib, len(data), 7, 0, 1)], pinned=True, src_gap=0)
    assert rc == 0 and hres == res and sha(houts[0]) == sha(outs[0])
    assert frame.decompress_file(houts[0]) == data.tobytes()


def test_many_small_files(lib, oracle):
    rng = np.random.default_rng(3)
    pool = oracle.datagen(8 * MIB, 0.5, 9).tobytes()
    datas = []
    for k in range(20000):
        n = int(rng.integers(0, 3000))
        a = int(rng.integers(0, len(pool) - n))
        datas.append(pool[a:a + n])
    for bsum, csum in ((0, 1), (1, 1)):
        res, outs = device_call(datas, bsum=bool(bsum), csum=bool(csum))
        rc, hres, houts = host_call(lib, datas, [frame_bound(lib, len(d), 7, bsum, csum) for d in datas], bsum=bsum,
                                    csum=csum)
        assert rc == 0 and hres == res and houts == outs
    # legacy streams: the device call holds an 8 MiB slot per chunk, so the model stands in for it past 500 files
    res, outs = device_call(datas[:500], legacy=True)
    rc, hres, houts = host_call(lib, datas, [LM.bound(len(d)) for d in datas], legacy=True)
    assert rc == 0 and hres[:500] == res and houts[:500] == outs
    codec = LM.block_codec(oracle, 1)
    assert houts == [LM.stream(d, codec) for d in datas] and hres == [len(h) for h in houts]


def test_outputs_past_4gib(lib, oracle):
    """a first file with 4 GiB of room: the second file's output starts past 2^32 in the same buffer"""
    a, b = oracle.datagen(100000, 0.5, 12).tobytes(), oracle.datagen(5 * MIB + 7, 0.5, 13).tobytes()
    caps = [(1 << 32) + 5, frame_bound(lib, len(b), 7, 1, 1)]
    rc, res, outs = host_call(lib, [a, b], caps, bsum=1, csum=1)
    dres, douts = device_call([a, b], bsum=True, csum=True)
    assert rc == 0 and res == dres and outs == douts


def test_round_trips(oracle):
    datas = [oracle.datagen(n, 0.5, n % 13).tobytes() for n in (0, 1, 70000, 5 * MIB + 3)]
    for kw in (dict(), dict(block_checksum=True, block_size_id=4, content_size=True), dict(content_checksum=False),
               dict(level=9, block_size_id=4), dict(legacy=True), dict(legacy=True, level=-3)):
        if kw.get("level") == 9:
            ds = datas[:3]
        else:
            ds = datas
        files = frame.compress_files(ds, **kw)
        got = frame.decompress_files(files)
        assert [g[3] for g in got] == ds, kw


def test_device_memory_stays_under_the_ceiling(lib, oracle):
    """device memory after repeated calls: the growth since before the first call is at most the stated ceiling for
    G = 512 MiB at the fast levels (4 slots x (2 G + 16 B + G + G/255 + 32 B + G + G/255 + 24 B + 56 B + 8, each
    buffer rounded up by 1 MiB + 16) + the ring), and does not grow from the second call on"""
    G, B = 512 * MIB, 65536
    slot = 2 * G + 2 * (G + G // 255) + 128 * B + 8 + 5 * (MIB + 16)
    ceiling = 4 * slot + 5 * 40
    data = oracle.datagen_mt(1 << 30, 1 << 20, 0.5, 43)
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    cap = [frame_bound(lib, len(data), 7, 1, 1)]
    host_call(lib, [data], cap, bsum=1, src_gap=0)
    free1 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        host_call(lib, [data], cap, bsum=1, src_gap=0)
    assert torch.cuda.mem_get_info()[0] >= free1
    assert free0 - free1 <= ceiling, (free0 - free1, ceiling)


def test_threads_beside_the_other_host_calls(lib, oracle):
    datas = [oracle.datagen(n, 0.5, n % 7).tobytes() for n in (100, 70000, 3 * MIB + 5)]
    caps = [frame_bound(lib, len(d), 7, 1, 1) for d in datas]
    serial = host_call(lib, datas, caps, bsum=1)
    files = frame.compress_files(datas)
    blk = oracle.datagen(64 * 65536, 0.5, 1)
    errors = []

    def writer():
        for _ in range(3):
            if host_call(lib, datas, caps, bsum=1) != serial:
                errors.append("compress_frames_host")

    def reader():
        for _ in range(3):
            if [g[3] for g in frame.decompress_files(files)] != datas:
                errors.append("decompress_files_host")

    def blocks():
        for _ in range(3):
            out = np.zeros(64 * 65792, dtype=np.uint8)
            sizes = np.zeros(64, dtype=np.int32)
            rc = lib.LZ4B200_compress_blocks_host(blk.ctypes.data, 65536, 65536, 65536, out.ctypes.data, 65792, 65792,
                                                  1, sizes.ctypes.data, 64)
            if rc != 0 or (sizes <= 0).any():
                errors.append("compress_blocks_host")

    ts = [threading.Thread(target=writer) for _ in range(4)] + [threading.Thread(target=reader),
                                                               threading.Thread(target=blocks)]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert errors == []


def test_python_wrappers(oracle):
    d = oracle.datagen(300000, 0.5, 4).tobytes()
    assert frame.compress_file(d) == frame.compress_files([d])[0]
    f = frame.compress_file(np.frombuffer(d, dtype=np.uint8).reshape(3, -1), level=3, block_size_id=4,
                            content_size=True, block_checksum=True)
    assert frame.decompress_file(f) == d
    assert frame.compress_file(d, parallel=True)[:4] == b"\x04\x22\x4d\x18"
    assert frame.compress_file(d, legacy=True)[:4] == b"\x02\x21\x4c\x18"
    assert frame.compress_files([]) == []


if __name__ == "__main__":
    child_main(sys.argv[1])
