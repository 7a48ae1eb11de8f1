"""A seeded fuzz of the container calls on the GPU, after the reference's tests/frametest.c (tests/container_fuzz.py
draws the cases and judges them).

Per seed, each case is one writer call -- compress_frames, compress_frames_checksummed or compress_legacy -- over
sources at shuffled offsets of every 16-byte phase, with outputs abutting at an odd base between guard bytes, each at
the bound, the bound - 1, a smaller capacity or -1.  The same sources then go through the host writer and the
device-to-host writer, which must return the device call's bytes; a frame of the parallel parse must be the host
model's (tests/encpar_model.py) and decode to its source.  The written frames, valid and mutated (a corrupted
header with its checksum right or stale, block words, payloads, checksums, cuts at unit edges, garbage, skippable
frames and legacy streams around them, blocks swapped between frames), go through decompress_frames_checksummed with
and without skipChecksums and decompress_frames where no checksum flag is set; the files go through decompress_files,
decompress_files_host and decompress_files_to_device, and the size-only pass of the first two.  Every call gives its
judge's result, consumed count, prefix and bytes, and writes nothing outside its outputs.  One generator case per seed
runs again in a child process with 1 MiB host groups, its files valid and mutated.  The judges are the
reference's LZ4F_compressFrame / LZ4F_decompress / block compressors where oracle/_ref is built, else the models.
"""
import collections
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import compress_frames_checksum_model as CM  # noqa: E402
import compress_frames_model as CFM  # noqa: E402
import compress_legacy_model as LM  # noqa: E402
import container_fuzz as F  # noqa: E402
import decompress_files_model as DM  # noqa: E402
import encpar_model as EP  # noqa: E402
import frame_corpus as FC  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
GUARD = 0xA5
SEEDS = [1, 2, 2026]
CASES = 14
STATS = collections.Counter()


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    if torch.cuda.mem_get_info()[0] < (8 << 30):
        pytest.skip("the fuzz needs 8 GiB of free device memory")
    yield lib
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def release_workspaces():
    yield
    from lz4_b200 import batch
    torch.cuda.synchronize()
    batch._workspaces.clear()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def judge(oracle):
    return F.Judge(oracle)


def t(a):
    return torch.from_numpy(np.array(a)).to(DEV)


def place(datas, seed, gap=64):
    """an arena holding every source at a shuffled offset of every 16-byte phase, 16 readable bytes around each"""
    rng = np.random.default_rng(seed)
    offs, at = [0] * len(datas), 16
    for k, i in enumerate(rng.permutation(len(datas))):
        at += k % 16
        offs[i] = at
        at += len(datas[i]) + gap
    arena = np.full(at + 16, 0x3C, dtype=np.uint8)
    for i, d in enumerate(datas):
        arena[offs[i]:offs[i] + len(d)] = np.frombuffer(bytes(d), dtype=np.uint8)
    return arena, np.array(offs, dtype=np.int64)


def outputs(caps):
    """out offsets abutting from an odd base, and a guard-filled device buffer around them"""
    room = np.maximum(np.array(caps, dtype=np.int64), 0)
    doff = 7 + np.concatenate([[0], np.cumsum(room)[:-1]]).astype(np.int64)
    return doff, torch.full((int(room.sum()) + 7 + 64,), GUARD, dtype=torch.uint8, device=DEV)


def check_guards(out, doff, limits, what):
    """every byte outside the [doff_f, doff_f + limit_f) is still a guard"""
    mask = np.ones(len(out), dtype=bool)
    for o, n in zip(doff, limits):
        if n > 0:
            mask[o:o + n] = False
    assert not (out[mask] != GUARD).any(), "%s wrote outside its outputs" % what


def note(verdicts):
    for r in verdicts:
        STATS["verdict " + F.verdict(int(r))] += 1


# ------------------------------------------------------------------------------------------
# writers
# ------------------------------------------------------------------------------------------
def device_write(c, datas, caps, seed, k):
    """one compress_frames / compress_frames_checksummed / compress_legacy call: (results, output bytes per item)"""
    from lz4_b200 import batch
    arena, soff = place(datas, seed * 7919 + k)
    sizes = np.array([len(d) for d in datas], dtype=np.int64)
    doff, out = outputs(caps)
    passing = [n if cap >= F.bound(c, n) else -1 for n, cap in zip(sizes, caps)]
    if c["legacy"]:
        need = sum(LM.n_chunks(n) for n in passing if n >= 0)
        _, res = batch.compress_legacy(t(arena), t(soff), t(sizes), max_blocks=need, level=c["level"], out=out,
                                       out_offsets=t(doff), capacities=t(caps))
    else:
        kw = dict(max_blocks=CM.budget(passing, c["bsid"]), block_size_id=c["bsid"], level=c["level"],
                  content_size=c["cs"], parallel=c["parallel"], out=out, out_offsets=t(doff), capacities=t(caps))
        if c["bsum"] or c["csum"] or k % 2:
            _, res = batch.compress_frames_checksummed(t(arena), t(soff), t(sizes), block_checksum=c["bsum"],
                                                       content_checksum=c["csum"], **kw)
        else:
            _, res = batch.compress_frames(t(arena), t(soff), t(sizes), **kw)
    torch.cuda.synchronize()
    res, host = res.cpu().numpy(), out.cpu().numpy()
    check_guards(host, doff, res, "the writer")
    return [int(r) for r in res], [host[o:o + max(r, 0)].tobytes() for o, r in zip(doff, res)]


def files_kwargs(c):
    if c["legacy"]:
        return dict(level=c["level"], legacy=True)
    return dict(level=c["level"], block_size_id=c["bsid"], content_size=c["cs"], block_checksum=c["bsum"],
                content_checksum=c["csum"], parallel=c["parallel"])


def parallel_frame(judge, d, c):
    """the frame of the parallel parse: compress_frames_checksum_model's frame around the payloads of the host model of
    the parse (tests/encpar_model.py) at the frame's acceleration, each block at capacity size - 1"""
    accel = CFM.acceleration(c["level"])

    def payload(i, blk):
        r = EP.compress(blk, accel, len(blk) - 1, judge.oracle)
        return r.ret, r.out
    xxh = judge.ref.xxh32 if judge.ref is not None else F.FM.xxh32
    return CM.frame(d, c["bsid"], c["cs"], None, payload=payload, block_sum=c["bsum"], content_sum=c["csum"], xxh=xxh)


def check_writer(judge, c, datas, seed, k):
    """the device call against the judge at every capacity, the host and device-to-host writers against the device
    call at the bound: the files at the bound"""
    from lz4_b200 import frame
    caps = [F.capacity(c, it, seed * 1000003 + k * 1009 + i) for i, it in enumerate(c["items"])]
    res, outs = device_write(c, datas, caps, seed, k)
    note(res)
    for i, (d, cap) in enumerate(zip(datas, caps)):
        want, wb = judge.write(d, c, cap)
        if c["parallel"] and want > 0:
            model = parallel_frame(judge, d, c)
            assert res[i] == len(model) and outs[i] == model, (seed, k, i, res[i], len(model))
            assert judge.read_frame(outs[i], len(d), False) == (len(d), bytes(d)), (seed, k, i)
        else:
            assert res[i] == want and outs[i] == wb, (seed, k, i, res[i], want)
    bounds = [F.bound(c, len(d)) for d in datas]
    res, outs = device_write(c, datas, bounds, seed, k + 1)
    assert all(r > 0 for r in res)
    assert frame.compress_files(datas, **files_kwargs(c)) == outs, (seed, k, "host writer")
    tens = [torch.from_numpy(np.frombuffer(bytes(d) + b"\0", dtype=np.uint8)[:len(d)].copy()).to(DEV) for d in datas]
    assert frame.compress_files_from_device(tens, **files_kwargs(c)) == outs, (seed, k, "device-to-host writer")
    return outs


# ------------------------------------------------------------------------------------------
# readers
# ------------------------------------------------------------------------------------------
def check_frame_readers(judge, frames, caps, seed):
    from lz4_b200 import batch
    arena, soff = place(frames, seed)
    sizes = np.array([len(f) for f in frames], dtype=np.int64)
    budget = [0, 0, 0, 0]
    for f in frames:
        if len(f) >= 7 and len(f) >= FC.header_len(f) and 4 <= (f[5] >> 4) & 7:
            budget[((f[5] >> 4) & 7) - 4] += F.chain_blocks(f) + 1
    plain = [i for i, f in enumerate(frames) if len(f) > 4 and not f[4] & 0x14]
    for entry, skip in (("sums", False), ("sums", True), ("plain", False)):
        idx = plain if entry == "plain" else range(len(frames))
        if not idx:
            continue
        fs, cs = [frames[i] for i in idx], [caps[i] for i in idx]
        doff, out = outputs([c + 16 for c in cs])
        if entry == "sums":
            _, res, _ = batch.decompress_frames_checksummed(t(arena), t(soff), t(sizes), t(cs), budget,
                                                            skip_checksums=skip, out=out, out_offsets=t(doff))
        else:
            _, res, _ = batch.decompress_frames(t(arena), t(soff[list(idx)]), t(sizes[list(idx)]), t(cs), budget,
                                                out=out, out_offsets=t(doff))
        torch.cuda.synchronize()
        res, host = res.cpu().numpy(), out.cpu().numpy()
        check_guards(host, doff, cs, "decompress_frames")
        note(res)
        for j, (f, cap) in enumerate(zip(fs, cs)):
            want, wb = judge.read_frame(f, cap, skip)
            assert res[j] == want, (seed, entry, skip, j, int(res[j]), want)
            if want >= 0:
                assert host[doff[j]:doff[j] + want].tobytes() == wb, (seed, entry, skip, j)


def check_file_readers(judge, files, seed, rng):
    """device, host and host-to-device file calls, and the size-only passes, against the judge and each other"""
    from lz4_b200 import batch, frame
    arena, soff = place(files, seed)
    sizes = np.array([len(f) for f in files], dtype=np.int64)
    for skip in (False, True):
        mu, mb = DM.budget_needed(files, skip)
        sized = judge.read_files(files, [1 << 40] * len(files), mu, mb, skip)
        caps = [r if r >= 0 else p for r, _, p, _ in sized]
        caps = [c - 1 if c > 0 and rng.random() < 0.15 else c for c in caps]
        want = judge.read_files(files, caps, mu, mb, skip)
        doff, out = outputs([c + 16 for c in caps])
        _, res, con, pre = batch.decompress_files(t(arena), t(soff), t(sizes), t(caps), mu, mb, skip_checksums=skip,
                                                  out=out, out_offsets=t(doff))
        torch.cuda.synchronize()
        got = list(zip(res.cpu().tolist(), con.cpu().tolist(), pre.cpu().tolist()))
        host = out.cpu().numpy()
        check_guards(host, doff, caps, "decompress_files")
        note(res.cpu().tolist())
        for j, (w, g) in enumerate(zip(want, got)):
            assert tuple(g) == w[:3], (seed, skip, j, g, w[:3])
            n = w[0] if w[0] >= 0 else w[2]
            assert host[doff[j]:doff[j] + n].tobytes() == w[3][:n], (seed, skip, j)
        hgot = frame.decompress_files(files, caps, skip)
        assert [h[:3] for h in hgot] == got, (seed, skip, "host")
        assert all(h[3] == w[3][:len(h[3])] and len(h[3]) == (w[0] if w[0] >= 0 else w[2]) for h, w in zip(hgot, want))
        dgot = frame.decompress_files_to_device(files, caps, skip)
        assert [tuple(x[:3]) for x in dgot] == got, (seed, skip, "to device")
        assert all(x[3].cpu().numpy().tobytes() == h[3] for x, h in zip(dgot, hgot))
        swant = [w[:3] for w in judge.read_files(files, caps, mu, mb, skip, size_only=True)]
        sres, scon, spre = batch.decompressed_file_sizes(t(arena), t(soff), t(sizes), mu, mb, skip_checksums=skip)
        torch.cuda.synchronize()
        assert list(zip(sres.cpu().tolist(), scon.cpu().tolist(), spre.cpu().tolist())) == swant, (seed, skip, "sizes")
        assert [h[:3] for h in frame.decompress_files(files, skip_checksums=skip, size_only=True)] == swant


# ------------------------------------------------------------------------------------------
# the loop
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", SEEDS)
def test_fuzz(lib, oracle, judge, seed):
    for k in range(CASES):
        c = F.case(seed, k)
        datas = F.case_data(oracle, c)
        STATS["level %d" % c["level"]] += 1
        STATS["legacy" if c["legacy"] else "bsid %d" % c["bsid"]] += 1
        if not c["legacy"]:
            STATS["flags cs=%d bsum=%d csum=%d" % (c["cs"], c["bsum"], c["csum"])] += 1
            STATS["parallel %d" % c["parallel"]] += 1
        outs = check_writer(judge, c, datas, seed, k)
        rng = np.random.default_rng([seed, k, 11])
        muts = F.mutated_files(oracle, c, outs, rng)
        for cls, _ in muts:
            STATS["mutation " + cls] += 1
        if not c["legacy"]:
            frames = [f for _, f in muts] + list(outs)
            caps = [F.room(f) for _, f in muts] + [max(len(d) - int(rng.random() < 0.2), 0) for d in datas]
            check_frame_readers(judge, frames, caps, seed * 31 + k)
        files = [f for _, f in muts] + [b"".join(outs[:3]) + DM.skippable(b"abc") + b"".join(outs[3:5])]
        check_file_readers(judge, files, seed * 37 + k, rng)
        STATS["cases"] += 1
    print("\nSTATS after seed %d (%s judges):" % (seed, judge.name), dict(sorted(STATS.items())))


def child_cases():
    """the one generator case per seed the child runs with 1 MiB groups: the first fast-level case with at least 2 MiB
    of sources, so that group edges fall inside its frames or legacy blocks"""
    out = []
    for seed in SEEDS:
        k = 0
        while True:
            c = F.case(seed, k)
            if c["level"] < 2 and sum(it["size"] for it in c["items"]) >= 2 * F.MIB:
                break
            k += 1
        out.append((seed, k, c))
    return out


def child_files(oracle, seed, k, c, outs):
    """the files the child reads: each written file valid or mutated, and the valid files concatenated"""
    muts = F.mutated_files(oracle, c, outs, np.random.default_rng([seed, k, 23]))
    return [f for _, f in muts] + [b"".join(outs)]


def test_one_mib_groups_in_a_child(lib, oracle, judge, tmp_path):
    """the host writers and readers with LZ4B200_HOST_WRITE_MB = LZ4B200_HOST_CHUNK_MB = 1, so that group edges fall
    inside frames, valid and mutated: the device writer's bytes and the judge's results, consumed counts, prefixes and
    bytes"""
    plan, want = {}, {}
    for seed, k, c in child_cases():
        datas = F.case_data(oracle, c)
        _, outs = device_write(c, datas, [F.bound(c, len(d)) for d in datas], seed, k)
        files = child_files(oracle, seed, k, c, outs)
        mu, mb = DM.budget_needed(files)
        sized = judge.read_files(files, [1 << 40] * len(files), mu, mb)
        caps = [r if r >= 0 else p for r, _, p, _ in sized]
        caps = [x - 1 if x > 0 and i % 3 == 1 else x for i, x in enumerate(caps)]
        plan[str(seed)] = dict(k=k, caps=caps)
        want[str(seed)] = dict(write=[F.sha(o) for o in outs],
                               read=[[w[0], w[1], w[2], F.sha(w[3])] for w in judge.read_files(files, caps, mu, mb)],
                               sizes=[list(w[:3]) for w in judge.read_files(files, caps, mu, mb, size_only=True)])
        STATS["child files"] += len(files)
    with open(str(tmp_path / "plan.json"), "w") as f:
        json.dump(plan, f)
    env = dict(os.environ, LZ4B200_HOST_WRITE_MB="1", LZ4B200_HOST_CHUNK_MB="1")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), str(tmp_path)], env=env, timeout=1200,
                       capture_output=True, text=True)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    with open(str(tmp_path / "child.json")) as f:
        got = json.load(f)
    for seed in want:
        for key in ("write", "read", "sizes"):
            assert got[seed][key] == want[seed][key], (seed, key)


def test_coverage():
    """every block size ID, level, flag combination, mutation class and verdict was reached"""
    if not STATS["cases"]:
        pytest.skip("the fuzz loop did not run")
    print("\nSTATS:", dict(sorted(STATS.items())), "peak device memory %.2f GiB" % (torch.cuda.max_memory_allocated() / 2 ** 30))
    missing = ["level %d" % v for v in F.LEVELS] + ["bsid %d" % b for b in F.BSIDS] + ["legacy"]
    missing += ["mutation " + m for m in F.MUTATIONS]
    missing += ["verdict " + v for v in ("OK", "FRAME", "UNSUPPORTED", "CHECKSUM", "DSTSIZE", "ARG")]
    missing += ["flags cs=%d bsum=%d csum=%d" % (a, b, c) for a in (0, 1) for b in (0, 1) for c in (0, 1)]
    missing += ["parallel 0", "parallel 1"]
    missing = [m for m in missing if not STATS[m]]
    assert not missing, missing


def _child(tmp):
    """run in a child process with 1 MiB groups: the host and device-to-host writers, and the host and host-to-device
    readers at the capacities of plan.json, on child_cases()"""
    from lz4_b200 import frame
    from oracle.pyoracle import Oracle
    oracle = Oracle()
    with open(os.path.join(tmp, "plan.json")) as f:
        plan = json.load(f)
    got = {}
    for seed, k, c in child_cases():
        caps = plan[str(seed)]["caps"]
        assert plan[str(seed)]["k"] == k
        datas = F.case_data(oracle, c)
        outs = frame.compress_files(datas, **files_kwargs(c))
        tens = [torch.from_numpy(np.frombuffer(bytes(d) + b"\0", dtype=np.uint8)[:len(d)].copy()).cuda() for d in datas]
        assert frame.compress_files_from_device(tens, **files_kwargs(c)) == outs
        files = child_files(oracle, seed, k, c, outs)
        read = frame.decompress_files(files, caps)
        dev = frame.decompress_files_to_device(files, caps)
        assert [tuple(x[:3]) for x in dev] == [r[:3] for r in read]
        assert all(x[3].cpu().numpy().tobytes() == r[3] for x, r in zip(dev, read))
        sizes = frame.decompress_files(files, size_only=True)
        got[str(seed)] = dict(write=[F.sha(o) for o in outs], read=[[r[0], r[1], r[2], F.sha(r[3])] for r in read],
                              sizes=[list(r[:3]) for r in sizes])
    with open(os.path.join(tmp, "child.json"), "w") as f:
        json.dump(got, f)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(HERE))
    _child(sys.argv[1])
