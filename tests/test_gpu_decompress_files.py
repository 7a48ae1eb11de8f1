"""LZ4B200_decompress_files on the GPU: every file of tests/golden/decompress_files.json against the Python model (which
tests/test_decompress_files_rules.py pins to the reference `lz4` tool) and the tool's output, in both checksum modes,
with guard bytes around every output region at exact capacity and one byte less; the size-only pass; a single-frame file
against LZ4B200_decompress_frames_checksummed; the unit and block budgets at their edges, LZ4B200_ERR_LIMIT on the 4 095th
and 4 096th of 16 389 files; a 64 MiB + 17 legacy file, a file of 30 000 skippable frames, offsets past 2^31 and 2^32;
launch counts, a side stream with graph capture and replay, and the wrapper's argument checks."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

import decompress_files_model as dm
from conftest import load_golden
from lz4_b200 import batch

pytestmark = pytest.mark.gpu

GUARD, FILL, GAP = 0xA5, 0xEE, 48
MIB = 1 << 20


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
    g = load_golden("decompress_files.json")["files"]
    return g, [dm.build_file(oracle, c) for c in g]


@pytest.fixture(autouse=True)
def release_workspaces():
    yield
    batch._workspaces.clear()
    torch.cuda.empty_cache()


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def dev(a, dtype=torch.int64):
    return torch.tensor(list(a), dtype=dtype, device="cuda")


class Layout:
    """files on the device at odd offsets with 16 bytes of padding; output regions GAP guard bytes apart"""

    def __init__(self, files, caps):
        buf, offs = bytearray(b"\xEE" * 16), []
        for f in files:
            buf += b"\xEE" * ((1 - len(buf)) % 16)
            offs.append(len(buf))
            buf += f
            buf += b"\xEE" * 16
        self.files, self.caps = files, caps
        self.comp = torch.frombuffer(buf, dtype=torch.uint8).cuda()
        self.offs, self.sizes = dev(offs), dev(len(f) for f in files)
        oo, at = [], GAP
        for c in caps:
            oo.append(at)
            at += max(c, 0) + GAP
        self.oo, self.out_bytes = oo, at
        self.out_offs, self.caps_d = dev(oo), dev(caps)

    def out(self):
        return torch.full((self.out_bytes,), GUARD, dtype=torch.uint8, device="cuda")


def run(lay, mu, mb, skip=False):
    out = lay.out()
    _, res, con, pre = batch.decompress_files(lay.comp, lay.offs, lay.sizes, lay.caps_d, mu,
                                              mb, skip, out=out, out_offsets=lay.out_offs)
    torch.cuda.synchronize()
    return out.cpu().numpy(), res.tolist(), con.tolist(), pre.tolist()


def check(oracle, lay, mu, mb, skip=False, want=None):
    """the call against the model: results, consumed, prefixes, the prefix bytes, and the guard bytes untouched"""
    out, res, con, pre = run(lay, mu, mb, skip)
    want = want or dm.decompress_files(oracle, lay.files, lay.caps, mu, mb, skip)
    for k, (r, at, p, b) in enumerate(want):
        assert (res[k], con[k], pre[k]) == (r, at, p), (k, (res[k], con[k], pre[k]), (r, at, p))
        o = lay.oo[k]
        assert out[o:o + p].tobytes() == b, k
        assert (out[o - GAP:o] == GUARD).all() and (out[o + max(lay.caps[k], 0):o + max(lay.caps[k], 0) + GAP] == GUARD).all(), k
    return want


@pytest.mark.parametrize("mode", ["verify", "skip"])
def test_golden_files(corpus, oracle, mode):
    g, files = corpus
    skip = mode == "skip"
    mu, mb = dm.budget_needed(files, skip)
    sized = dm.decompress_files(oracle, files, [1 << 40] * len(files), mu, mb, skip)
    exact = [r if r >= 0 else p + (1 << 16) for r, _, p, _ in sized]
    want = check(oracle, Layout(files, exact), mu, mb, skip)
    for c, (r, _, p, b) in zip(g, want):                 # the tool's bytes, where the model has no deviation from them
        if c[mode]["exit"] == 0 and r >= 0:
            assert sha(b) == c[mode]["sha256"], c["name"]
    short = [e - 1 if e > 0 else 0 for e in exact]
    check(oracle, Layout(files, short), mu, mb, skip)
    # the size-only pass gives the decoding call's results at unlimited room, and writes nothing
    lay = Layout(files, exact)
    res, con, pre = batch.decompressed_file_sizes(lay.comp, lay.offs, lay.sizes, mu, mb, skip)
    nocontent = dm.decompress_files(oracle, files, exact, mu, mb, skip, size_only=True)
    assert (res.tolist(), con.tolist(), pre.tolist()) == ([w[0] for w in nocontent], [w[1] for w in nocontent],
                                                          [w[2] for w in nocontent])
    if skip:                                              # no content checksum is compared either way
        assert [w[0] for w in nocontent] == [w[0] for w in sized]


def test_size_only_without_output(corpus, oracle):
    """sizeOnly takes no output pointers at all"""
    g, files = corpus
    lay = Layout(files[:30], [0] * 30)
    mu, mb = dm.budget_needed(lay.files)
    res, _, _ = batch.decompressed_file_sizes(lay.comp, lay.offs, lay.sizes, mu, mb)
    got = dm.decompress_files(oracle, lay.files, lay.caps, mu, mb, size_only=True)
    assert res.tolist() == [w[0] for w in got]
    lib = batch._lib.load()
    ws = torch.empty(batch.decompress_files_workspace_bytes(30, mu, mb), dtype=torch.uint8, device="cuda")
    r = torch.empty(30, dtype=torch.int64, device="cuda")
    rc = lib.LZ4B200_decompress_files(lay.comp.data_ptr(), lay.offs.data_ptr(), lay.sizes.data_ptr(), None, None, None,
                                      r.data_ptr(), None, None, 30, mu, (C.c_int64 * 5)(*mb), 0, 1, ws.data_ptr(),
                                      ws.numel(), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == 0 and r.tolist() == res.tolist()


def test_single_frame_matches_frames_call(corpus):
    g, files = corpus
    pick = [f for c, f in zip(g, files) if c["name"].startswith(("frame", "cli"))]
    for skip in (False, True):
        caps = [len(f) * 4 + 1000 for f in pick]
        lay = Layout(pick, caps)
        mu, mb = dm.budget_needed(pick, skip)
        out, res, con, pre = run(lay, mu, mb, skip)
        fout = lay.out()
        _, fres, fcon = batch.decompress_frames_checksummed(lay.comp, lay.offs, lay.sizes, lay.caps_d, mb[:4], skip,
                                                           out=fout, out_offsets=lay.out_offs)
        torch.cuda.synchronize()
        fout = fout.cpu().numpy()
        for k, (r, fr) in enumerate(zip(res, fres.tolist())):
            assert r == fr, k
            if r >= 0:
                o = lay.oo[k]
                assert (out[o:o + r] == fout[o:o + r]).all()


def test_budget_edges(corpus, oracle):
    g, files = corpus
    pick = [f for c, f in zip(g, files) if c["size"] < 2 * MIB and not c["name"].startswith("trunc")][:60]
    pick.append(dm.build_file(oracle, {"parts": [["legacy", [17 * MIB, 0.5, 7, 0]], ["skip", 1, 5, 1]]}))
    mu, mb = dm.budget_needed(pick)
    caps = [1 << 26] * len(pick)
    lay = Layout(pick, caps)
    edges = [(mu, mb), (mu - 1, mb), (0, mb), (1, mb)]
    for c in range(5):
        if mb[c]:
            edges.append((mu, mb[:c] + [mb[c] - 1] + mb[c + 1:]))
    for u, b in edges:
        check(oracle, lay, u, b)


def test_limit_at_scan_round_edges(oracle):
    """16 389 one-frame files: the unit budget runs out at file 4 095, then 4 096 (the files scan's rounds are 4 096
    files), and the 64 KB block budget likewise"""
    frame = dm.fm.compress_frame(oracle, oracle.datagen(3000, 0.5, 1).tobytes(), 4, False, 0, 1)
    n = 16389
    files = [frame] * n
    lay = Layout(files, [3000] * n)
    for mu, mb0 in [(4095, n), (4096, n), (n, 4095), (n, 4096), (n, n)]:
        _, res, con, _ = run(lay, mu, [mb0, 0, 0, 0, 0])
        lim = min(mu, mb0)
        assert res[:lim] == [3000] * lim and res[lim:] == [dm.ERR_LIMIT] * (n - lim), (mu, mb0)
        assert con[lim:] == [0] * (n - lim)


def test_big_legacy_and_many_skippable(oracle):
    data = oracle.datagen(64 * MIB + 17, 0.5, 9).tobytes()
    leg = dm.legacy(lambda b: oracle.compress(b, 1)[1], data)
    many = b"".join(dm.skippable(b"x" * (k % 3), k % 16) for k in range(30000)) + \
        dm.fm.compress_frame(oracle, data[:5000], 4, False, 0, 1)
    files = [leg, many]
    mu, mb = dm.budget_needed(files)
    assert mb[4] == 9 and mu == 30002
    lay = Layout(files, [len(data), 5000])
    out, res, con, pre = run(lay, mu, mb)
    assert res == [len(data), 5000] and con == [len(leg), len(many)]
    assert out[lay.oo[0]:lay.oo[0] + len(data)].tobytes() == data
    assert out[lay.oo[1]:lay.oo[1] + 5000].tobytes() == data[:5000]
    _, res, con, _ = run(lay, 30000, mb)                  # the skippable walk stops after maxUnits + 1 units
    assert res == [len(data), dm.ERR_LIMIT] and con[1] == 8 * 29999 + sum(k % 3 for k in range(29999))


def test_offsets_past_4gib(oracle):
    """files and outputs placed past 2^31 and 2^32 in one buffer"""
    d = oracle.datagen(300000, 0.5, 5).tobytes()
    files = [dm.fm.compress_frame(oracle, d, 5, True, 1, 1), dm.legacy(lambda b: oracle.compress(b, 1)[1], d),
             dm.skippable(b"abc") + dm.fm.compress_frame(oracle, d[:1000], 4, False, 0, 1)]
    total = (1 << 32) + (1 << 20)
    comp = torch.full((total,), FILL, dtype=torch.uint8, device="cuda")
    offs = [(1 << 31) - 5, (1 << 32) - 100, (1 << 32) + (1 << 19) + 4097]
    for o, f in zip(offs, files):
        comp[o:o + len(f)] = torch.frombuffer(bytearray(f), dtype=torch.uint8).cuda()
    out = torch.full((total,), GUARD, dtype=torch.uint8, device="cuda")
    oo = [(1 << 32) - 7, (1 << 31) + 3, (1 << 32) + 500000]
    caps = [300000, 300000, 1000]
    mu, mb = dm.budget_needed(files)
    _, res, con, pre = batch.decompress_files(comp, dev(offs), dev(len(f) for f in files), dev(caps), mu, mb,
                                              out=out, out_offsets=dev(oo))
    torch.cuda.synchronize()
    assert res.tolist() == [300000, 300000, 1000] and con.tolist() == [len(f) for f in files]
    for o, c, want in zip(oo, caps, [d, d, d[:1000]]):
        assert out[o:o + c].cpu().numpy().tobytes() == want
        assert int(out[o - 1]) == GUARD and int(out[o + c]) == GUARD
    del comp, out


def expected_launches(mu, mb, skip, size_only):
    n = 4
    if mu:
        n += 3 + (0 if skip else 1)
        for c in range(5):
            if mb[c]:
                n += (1 if c == 0 else 2) + (0 if size_only else 2)
        if not size_only:
            n += 3 + (0 if skip else 1)
    return n


def test_launch_counts(lib, corpus):
    g, files = corpus
    pick = files[:20]
    lay = Layout(pick, [1 << 22] * 20)
    mu, mb = dm.budget_needed(pick)
    for u, b in [(mu, mb), (0, mb), (mu, [mb[0], 0, 0, 0, 0]), (mu, [0, 0, 0, 0, 0]), (mu, [1, 1, 1, 1, 1])]:
        for skip in (False, True):
            for size_only in (False, True):
                n0 = lib.LZ4B200_launch_count()
                if size_only:
                    batch.decompressed_file_sizes(lay.comp, lay.offs, lay.sizes, u, b, skip)
                else:
                    batch.decompress_files(lay.comp, lay.offs, lay.sizes, lay.caps_d, u, b, skip, out=lay.out(),
                                           out_offsets=lay.out_offs)
                assert lib.LZ4B200_launch_count() - n0 == expected_launches(u, b, skip, size_only), (u, b, skip, size_only)
    n0 = lib.LZ4B200_launch_count()
    batch.decompress_files(lay.comp, lay.offs[:0], lay.sizes[:0], lay.caps_d[:0], mu, mb, out=lay.out())
    assert lib.LZ4B200_launch_count() == n0


def test_side_stream_and_graph(corpus, oracle):
    g, files = corpus
    pick = [f for c, f in zip(g, files) if c["size"] < MIB][:40]
    mu, mb = dm.budget_needed(pick)
    want = dm.decompress_files(oracle, pick, [1 << 21] * len(pick), mu, mb)
    lay = Layout(pick, [1 << 21] * len(pick))
    s = torch.cuda.Stream()
    ws = torch.empty(batch.decompress_files_workspace_bytes(len(pick), mu, mb), dtype=torch.uint8, device="cuda")
    out = lay.out()
    res, con, pre = (torch.empty(len(pick), dtype=torch.int64, device="cuda") for _ in range(3))
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        batch.decompress_files(lay.comp, lay.offs, lay.sizes, lay.caps_d, mu, mb, out=out, out_offsets=lay.out_offs,
                               results=res, consumed=con, prefix=pre, workspace=ws, stream=s)
    s.synchronize()
    assert res.tolist() == [w[0] for w in want]
    graph = torch.cuda.CUDAGraph()
    out.fill_(GUARD)
    res.fill_(0)
    torch.cuda.synchronize()
    with torch.cuda.graph(graph, stream=s):
        batch.decompress_files(lay.comp, lay.offs, lay.sizes, lay.caps_d, mu, mb, out=out, out_offsets=lay.out_offs,
                               results=res, consumed=con, prefix=pre, workspace=ws)
    for _ in range(2):
        out.fill_(GUARD)
        res.fill_(0)
        graph.replay()
        torch.cuda.synchronize()
        h = out.cpu().numpy()
        assert res.tolist() == [w[0] for w in want] and con.tolist() == [w[1] for w in want]
        for k, w in enumerate(want):
            assert h[lay.oo[k]:lay.oo[k] + w[2]].tobytes() == w[3]


def test_wrapper_checks(corpus):
    g, files = corpus
    lay = Layout(files[:3], [100, 100, 100])
    mb = [4, 4, 4, 4, 4]
    ok = dict(out=lay.out(), out_offsets=lay.out_offs)
    bad = [
        (dict(max_blocks=[1, 2, 3, 4]), "5 values"),
        (dict(max_units=-1), "max_units"),
        (dict(max_blocks=[1, 1, 1, 1, 1 << 31]), "budgets"),
        (dict(offsets=lay.offs.cpu()), "CUDA tensor"),
        (dict(offsets=lay.offs[:2]), "offsets has"),
        (dict(sizes=lay.sizes.to(torch.int32)), "sizes must be"),
        (dict(capacities=lay.caps_d[:2]), "capacities has"),
        (dict(capacities=lay.caps_d.repeat(2)[::2]), "contiguous"),
        (dict(results=torch.empty(2, dtype=torch.int64, device="cuda")), "results has"),
        (dict(prefix=torch.empty(3, dtype=torch.int32, device="cuda")), "prefix must be"),
        (dict(consumed=torch.empty(2, dtype=torch.int64, device="cuda")), "consumed has"),
        (dict(workspace=torch.empty(16, dtype=torch.uint8, device="cuda")), "workspace has"),
        (dict(out=lay.out().to(torch.int8)), "out must be"),
    ]
    for kw, msg in bad:
        args = dict(comp=lay.comp, offsets=lay.offs, sizes=lay.sizes, capacities=lay.caps_d, max_units=8, max_blocks=mb,
                    **ok)
        args.update(kw)
        with pytest.raises(ValueError, match=msg):
            batch.decompress_files(**args)
    with pytest.raises(ValueError, match="5 values"):
        batch.decompressed_file_sizes(lay.comp, lay.offs, lay.sizes, 8, [1, 1])
    with pytest.raises(ValueError, match="workspace has"):
        batch.decompressed_file_sizes(lay.comp, lay.offs, lay.sizes, 8, mb,
                                      workspace=torch.empty(16, dtype=torch.uint8, device="cuda"))
    with pytest.raises(ValueError, match="capacities"):
        batch.decompress_files(lay.comp, lay.offs, lay.sizes, None, 8, mb)
