"""LZ4B200_decompress_frames and LZ4B200_decompress_frames_checksummed at scale on the GPU:
  A. batches of 4 095 .. 16 389 frames, across every round of the frames scan (4 096 frames a round), with each class's
     first LZ4B200_ERR_LIMIT on the last frame of round 0, the first of round 1, item 2 or 3 of a later round's thread
     and the last frame;
  B. results that do not depend on the budget: a 64 KB class decoded by the split scan and by the one-thread scan, and
     a caller's workspace reused after a larger call;
  C. one frame of 30 000 tiny blocks with block and content checksums;
  D. one frame whose content passes 2^32 bytes, with the reference's content checksum (tests/golden/frames_scale.json);
  E. checksummed frames at source and destination offsets on and past 2^31 and 2^32, in the arena of
     tests/test_gpu_far_offsets.py.
Every frame's result, consumed length and decoded bytes are checked against LZ4B200_decompressFrame_host (checksum-free
call) or tests/frame_checksum_model.py (checksummed call), with guard bytes around every output region; bulk output is
compared on the device.  Each test skips without the device memory it needs and holds its peak to 11 GiB."""
import ctypes as C
import hashlib
import struct

import numpy as np
import pytest
import torch

import frame_checksum_model as fm
import frame_corpus as fc
import test_frames_scale_rules as S
from conftest import load_golden
from test_gpu_far_offsets import SRC_ORG, Arena
from test_gpu_frames import host_call

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MiB, GiB = 1 << 20, 1 << 30
L31, L32 = 1 << 31, 1 << 32
PEAK = 11 * GiB
GUARD = 0xA5
GAP = 48
SPLIT_MAX_BLOCKS = 8192                             # kSplitMaxBlocks (lz4_decode_plan.h)


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    assert lib.LZ4B200_device_count() > 0, "GPU tests need a CUDA device"
    yield lib
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture(autouse=True)
def memory_peak():
    """frees what the test left, and holds its peak to PEAK.  The workspaces lz4_b200.batch keeps for calls without one
    are dropped first: the far frame's call needs nearly all of the 11 GiB by itself."""
    from lz4_b200 import batch
    torch.cuda.synchronize()
    batch._workspaces.clear()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    yield
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    torch.cuda.empty_cache()
    print("peak device memory %.2f GiB" % (peak / GiB))
    assert peak <= PEAK, "peak device memory %.2f GiB" % (peak / GiB)


def need_memory(nbytes):
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + 256 * MiB:
        pytest.skip("needs %.1f GiB of free device memory, %.1f GiB free" % (nbytes / GiB, free / GiB))


def ws_bytes(n, mb):
    from lz4_b200 import batch
    return batch.decompress_frames_workspace_bytes(n, mb)


def launches_of(mb, mode):
    """the header's count: 5, 3 for a 64 KB budget, 4 per larger class with a budget, 2 more when verifying"""
    return 5 + (3 if mb[0] else 0) + 4 * sum(1 for c in (1, 2, 3) if mb[c]) + (2 if mode == "verify" else 0)


_expected = {}


def expected(lib, oracle, frame, cap, mode):
    """(result, bytes, consumed) of the frame alone: LZ4B200_decompressFrame_host for the checksum-free call, the model
    of the checksummed call otherwise; once per (frame, capacity, mode)"""
    key = (frame, cap, mode)
    if key not in _expected:
        _expected[key] = host_call(lib, frame, cap) if mode == "plain" else fm.decode(oracle, frame, cap, mode == "skip")
    return _expected[key]


class Batch:
    """frames at odd offsets with 16 bytes of padding (fc.layout); output regions with GAP guard bytes between them"""

    def __init__(self, frames, caps, seed=0):
        self.frames, self.caps = frames, caps
        buf, offs = fc.layout(frames, seed=seed)
        self.src = torch.from_numpy(np.frombuffer(buf, dtype=np.uint8).copy()).to(DEV)
        self.off = torch.tensor(offs, dtype=torch.int64, device=DEV)
        self.size = torch.tensor([len(f) for f in frames], dtype=torch.int64, device=DEV)
        doff, at = [], 3
        for c in caps:
            doff.append(at)
            at += max(c, 0) + GAP + 1
        self.dst_off = doff
        self.out = torch.full((at + GAP,), GUARD, dtype=torch.uint8, device=DEV)
        self.d_off = torch.tensor(doff, dtype=torch.int64, device=DEV)
        self.d_cap = torch.tensor(caps, dtype=torch.int64, device=DEV)

    def run(self, mb, mode, workspace=None):
        """one call ("plain": LZ4B200_decompress_frames, "skip" / "verify": the checksummed call) into a guard-filled
        output; (results, consumed) as lists"""
        from lz4_b200 import batch
        self.out.fill_(GUARD)
        if mode == "plain":
            _, r, c = batch.decompress_frames(self.src, self.off, self.size, self.d_cap, mb, out=self.out,
                                              out_offsets=self.d_off, workspace=workspace)
        else:
            _, r, c = batch.decompress_frames_checksummed(self.src, self.off, self.size, self.d_cap, mb, mode == "skip",
                                                          out=self.out, out_offsets=self.d_off, workspace=workspace)
        return r.cpu().tolist(), c.cpu().tolist()

    def check(self, lib, oracle, mode, res, cons, planned=None):
        """every frame against its expectation (LZ4B200_ERR_LIMIT and consumed 0 where planned), and the whole output on
        the device: the decoded bytes of every frame that passed, the guard bytes outside every region"""
        img = np.full(self.out.numel(), GUARD, dtype=np.uint8)
        mask = np.ones(self.out.numel(), dtype=bool)
        for f, (fr, cap) in enumerate(zip(self.frames, self.caps)):
            o = self.dst_off[f]
            if planned is not None and planned[f] == fc.ERR_LIMIT:
                assert (res[f], cons[f]) == (fc.ERR_LIMIT, 0), f
                mask[o:o + cap] = False
                continue
            r, data, used = expected(lib, oracle, fr, cap, mode)
            assert (res[f], cons[f]) == (r, used), (f, res[f], cons[f], r, used)
            if r >= 0:
                img[o:o + r] = np.frombuffer(data, dtype=np.uint8)
            mask[o + max(r, 0):o + cap] = False                  # inside the region: unspecified
        m = torch.from_numpy(mask).to(DEV)
        bad = int(((self.out != torch.from_numpy(img).to(DEV)) & m).sum())
        assert bad == 0, "%d output bytes differ from the expected bytes or the guard" % bad


def batch_of(entries, seed):
    return Batch([e.frame for e in entries], [e.cap for e in entries], seed=seed)


# ------------------------------------------------------------------------------------------
# A. many frames: the scan's rounds
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", S.BATCHES)
def test_many_frames_limit_in_every_scan_round(lib, oracle, n):
    seen = set()
    for rot in range(4):
        entries = S.many_batch(oracle, n, rot)
        b = batch_of(entries, seed=n + rot)
        for mode in ("plain", "verify", "skip") if rot == 0 else ("plain", "verify"):
            budget, want = S.limit_budget(entries, mode, rot)
            need_memory(ws_bytes(n, budget) + 2 * b.out.numel())
            planned = S.plan(entries, mode, budget)
            res, cons = b.run(budget, mode)
            b.check(lib, oracle, mode, res, cons, planned)
            assert S.first_limits(zip(res, [e.pass1(mode)[0] for e in entries])) == want
            seen |= {(mode, min(r, 0)) for r in res}
    for mode in ("plain", "verify"):
        assert {fc.OK, fc.ERR_FRAME, fc.ERR_DSTSIZE, fc.ERR_LIMIT} <= {r for m, r in seen if m == mode}
    assert ("verify", fm.ERR_CHECKSUM) in seen and ("plain", fc.ERR_UNSUPPORTED) in seen
    assert ("skip", fm.ERR_CHECKSUM) not in seen


# ------------------------------------------------------------------------------------------
# B. the budget: scan routes and a reused workspace
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["plain", "verify"])
def test_results_do_not_depend_on_the_budget(lib, oracle, mode):
    entries = S.many_batch(oracle, 4097)
    b = batch_of(entries, seed=1)
    full = S.need(entries, mode)
    big = [full[0] + 9000, full[1] + 3, full[2] + 2, full[3] + 1]
    assert 0 < full[0] <= SPLIT_MAX_BLOCKS < big[0] and all(full)     # the split scan, then the one-thread scan
    large = S.many_batch(oracle, S.BATCHES[-1], 2)
    lb = batch_of(large, seed=2)
    lbudget = [max(x, y) for x, y in zip(S.need(large, mode), big)]
    lbudget = [x + 5 for x in lbudget]
    nbytes = ws_bytes(len(large), lbudget)
    assert nbytes >= ws_bytes(len(entries), big)
    need_memory(2 * nbytes + lb.out.numel() + 4 * b.out.numel())
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    ws.fill_(0xC3)
    res, cons = lb.run(lbudget, mode, workspace=ws)              # a larger call leaves its tables and marks behind
    lb.check(lib, oracle, mode, res, cons)
    del lb

    n0 = lib.LZ4B200_launch_count()
    r1, c1 = b.run(full, mode, workspace=ws)
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() - n0 == launches_of(full, mode)
    b.check(lib, oracle, mode, r1, c1)
    out1 = b.out.clone()
    n0 = lib.LZ4B200_launch_count()
    r2, c2 = b.run(big, mode, workspace=ws)
    torch.cuda.synchronize()
    assert lib.LZ4B200_launch_count() - n0 == launches_of(big, mode)
    assert (r2, c2) == (r1, c1) and torch.equal(b.out, out1)
    fresh = torch.zeros(ws_bytes(len(entries), big), dtype=torch.uint8, device=DEV)
    r3, c3 = b.run(big, mode, workspace=fresh)
    assert (r3, c3) == (r1, c1) and torch.equal(b.out, out1)


# ------------------------------------------------------------------------------------------
# C. one frame of many blocks
# ------------------------------------------------------------------------------------------
C_BLOCKS = 30000


def many_block_frame(oracle):
    """a 64 KB-class frame of C_BLOCKS blocks: compressed blocks of 4 .. 8 bytes and one-byte stored-raw blocks, block and
    content checksums, the content size; (frame, content)"""
    pieces, raw = [], set()
    for i in range(C_BLOCKS):
        if i % 3 == 1:
            raw.add(i)
            pieces.append(bytes([i & 0xFF]))
        else:
            pieces.append(struct.pack("<I", i * 2654435761 & 0xFFFFFFFF)[:4] + b"xyzw"[:i % 5])
    content = b"".join(pieces)
    f = fm.frame_of_blocks(oracle, pieces, 4, raw=raw, block_sum=True, content_sum=True, content_size=len(content))
    return f, content


def test_one_frame_of_many_blocks(lib, oracle):
    f, content = many_block_frame(oracle)
    blocks, consumed = fm.walk(f)
    assert len(blocks) == C_BLOCKS and consumed == len(f)
    mb = [C_BLOCKS + 1, 0, 0, 0]
    nbytes = ws_bytes(1, mb)
    need_memory(nbytes + 2 * len(f))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    print("workspace %.2f GiB" % (nbytes / GiB))
    b = Batch([f], [len(content)])
    for k, mode in ((C_BLOCKS, "verify"), (C_BLOCKS + 1, "verify"), (C_BLOCKS, "skip"), (C_BLOCKS - 1, "verify")):
        res, cons = b.run([k, 0, 0, 0], mode, workspace=ws)
        planned = [fc.ERR_LIMIT] if k < C_BLOCKS else None
        b.check(lib, oracle, mode, res, cons, planned)
        assert res == ([fc.ERR_LIMIT] if planned else [len(content)])
    bad = []
    for k in (0, C_BLOCKS // 2 + 1, C_BLOCKS - 1):                  # a block checksum: first, a middle (raw), last
        o, sz, _ = blocks[k]
        w = bytearray(f)
        w[o + sz + 1] ^= 0x08
        bad.append(bytes(w))
    for w in bad:
        c = Batch([w], [len(content)])
        res, cons = c.run([C_BLOCKS, 0, 0, 0], "verify", workspace=ws)
        c.check(lib, oracle, "verify", res, cons)
        assert res == [fm.ERR_CHECKSUM] and cons == [len(f)]
    res, cons = c.run([C_BLOCKS, 0, 0, 0], "skip", workspace=ws)
    c.check(lib, oracle, "skip", res, cons)
    assert res == [len(content)]


# ------------------------------------------------------------------------------------------
# D. a frame whose content passes 2^32 bytes
# ------------------------------------------------------------------------------------------
def check_far_content(out, at):
    """out[at : at + S.FAR_SIZE] against the far content, rebuilt on the device 2 048 blocks at a time"""
    step = 2048
    for a in range(0, S.FAR_FULL, step):
        k = min(step, S.FAR_FULL - a)
        rows = out[at + a * S.BLOCK:at + (a + k) * S.BLOCK].view(k, S.BLOCK)
        idx = torch.arange(a, a + k, dtype=torch.int64, device=DEV)
        fill = ((idx * 37 + 11) & 0xFF).to(torch.uint8)
        assert torch.equal(rows[:, :8].contiguous().view(torch.int64).view(-1), idx), "block index at block %d.." % a
        assert bool((rows[:, 8:] == fill[:, None]).all()), "fill bytes in blocks %d.." % a
    tail = out[at + S.FAR_FULL * S.BLOCK:at + S.FAR_SIZE].cpu().numpy().tobytes()
    assert tail == struct.pack("<Q", S.FAR_FULL) + bytes([S.far_fill(S.FAR_FULL)]) * (S.FAR_TAIL - 8)


def test_frame_past_4_gib(lib):
    from lz4_b200 import batch
    g = load_golden("frames_scale.json")
    f = S.far_frame(g["xxh32"])
    assert hashlib.sha256(f).hexdigest() == g["frame_sha256"]
    mb = [S.FAR_BLOCKS, 0, 0, 0]
    nbytes = ws_bytes(1, mb)
    at = 3
    total = nbytes + S.FAR_SIZE + at + GAP + len(f) + 512 * MiB
    print("workspace %.2f GiB, output %.2f GiB, in all %.2f GiB" % (nbytes / GiB, S.FAR_SIZE / GiB, total / GiB))
    need_memory(total)
    src = torch.from_numpy(np.frombuffer(b"\0" * 16 + f + b"\0" * 16, dtype=np.uint8).copy()).to(DEV)
    wrong = [torch.from_numpy(np.frombuffer(b"\0" * 16 + S.far_frame(g["xxh32"], S.FAR_SIZE + d) + b"\0" * 16,
                                            dtype=np.uint8).copy()).to(DEV) for d in (-L32, L32)]   # the same low 32 bits
    out = torch.empty(at + S.FAR_SIZE + GAP, dtype=torch.uint8, device=DEV)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    off = torch.tensor([16], dtype=torch.int64, device=DEV)
    size = torch.tensor([len(f)], dtype=torch.int64, device=DEV)
    d_off = torch.tensor([at], dtype=torch.int64, device=DEV)

    def run(s, cap, skip):
        out.fill_(GUARD)
        _, r, c = batch.decompress_frames_checksummed(s, off, size, torch.tensor([cap], dtype=torch.int64, device=DEV),
                                                      mb, skip, out=out, out_offsets=d_off, workspace=ws)
        r, c = int(r[0]), int(c[0])
        assert bool((out[:at] == GUARD).all()) and bool((out[at + cap:] == GUARD).all()), "a guard byte was written"
        return r, c

    assert run(src, S.FAR_SIZE, True) == (g["lz4f"]["size"], g["lz4f"]["consumed"]) == (S.FAR_SIZE, len(f))
    check_far_content(out, at)
    assert run(src, S.FAR_SIZE - 1, True) == (fc.ERR_DSTSIZE, len(f))
    assert run(wrong[0], S.FAR_SIZE, True) == (fc.ERR_FRAME, len(f))        # a block passes the content size
    assert run(wrong[1], S.FAR_SIZE, True) == (fc.ERR_FRAME, len(f))        # the content falls short of it
    assert run(src, S.FAR_SIZE, False) == (S.FAR_SIZE, len(f))       # the content checksum: one thread, 4 GiB
    check_far_content(out, at)


# ------------------------------------------------------------------------------------------
# E. the checksummed call at far offsets
# ------------------------------------------------------------------------------------------
def far_frames(oracle):
    """two checksummed frames (block and content checksums, compressed and stored-raw blocks, content size) and, of each,
    a copy with a flipped payload byte and a copy with a flipped content checksum"""
    d = oracle.datagen(300000, 0.5, 41).tobytes()
    noise = np.random.default_rng(41).integers(0, 256, 5000, dtype=np.uint8).tobytes()
    out = []
    for bsid, pieces, raw in ((4, [d[:65536], noise[:3001], d[65536:90001]], (1,)),
                              (5, [noise[:777], d[100000:300000]], (0,))):
        content = b"".join(pieces)
        f = fm.frame_of_blocks(oracle, pieces, bsid, raw=raw, block_sum=True, content_sum=True, content_size=len(content))
        blocks, consumed = fm.walk(f)
        o, sz, _ = blocks[1]
        payload = bytearray(f)
        payload[o + sz // 2] ^= 0x04
        csum = bytearray(f)
        csum[consumed - 2] ^= 0x40
        out += [(f, len(content)), (bytes(payload), len(content)), (bytes(csum), len(content))]
    return out


FAR_LINES = {"2^31-1": L31 - 1, "2^31": L31, "2^32-3": L32 - 3, "2^32+17": L32 + 17, "across 2^32": None}


@pytest.mark.parametrize("line", sorted(FAR_LINES))
def test_checksummed_frames_at_far_offsets(lib, oracle, line):
    """the frames from a line on, 1 MiB + an odd number apart, in the source (SRC_ORG from the arena's base) and at the
    same offsets in the destination (the base); both checksum modes"""
    pairs = far_frames(oracle)
    first = FAR_LINES[line] if FAR_LINES[line] is not None else L32 - len(pairs[0][0]) // 2
    offs = [first + k * (MiB + 2 * k + 1) for k in range(len(pairs))]
    mb = [0, 0, 0, 0]
    for f, _ in pairs:
        mb[((f[5] >> 4) & 7) - 4] += len(fm.walk(f)[0])
    nbytes = ws_bytes(len(pairs), mb)
    need_memory(nbytes + 8 * GiB)
    ar = Arena()
    for (f, cap), o in zip(pairs, offs):
        ar.put(SRC_ORG + o, f)
        ar.far(SRC_ORG, o, len(f))
        ar.far(0, o, cap)
    t = lambda v: torch.tensor(v, dtype=torch.int64, device=DEV)      # noqa: E731
    d_off, d_size, d_cap = t(offs), t([len(f) for f, _ in pairs]), t([c for _, c in pairs])
    res, cons = t([0] * len(pairs)), t([0] * len(pairs))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    for skip in (0, 1):
        rc = lib.LZ4B200_decompress_frames_checksummed(ar.ptr(SRC_ORG), d_off.data_ptr(), d_size.data_ptr(), ar.ptr(0),
                                                       d_off.data_ptr(), d_cap.data_ptr(), res.data_ptr(),
                                                       cons.data_ptr(), len(pairs), (C.c_int64 * 4)(*mb), skip,
                                                       ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream)
        assert rc == fc.OK
        torch.cuda.synchronize()
        got_r, got_c = res.cpu().tolist(), cons.cpu().tolist()
        for k, ((f, cap), o) in enumerate(zip(pairs, offs)):
            r, data, used = fm.decode(oracle, f, cap, bool(skip))
            assert (got_r[k], got_c[k]) == (r, used), (skip, k, got_r[k], r)
            if r >= 0:
                assert ar.view(o, r).cpu().numpy().tobytes() == data, (skip, k)
        if not skip:
            assert got_r[1::3] == [fm.ERR_CHECKSUM] * 2 and got_r[2::3] == [fm.ERR_CHECKSUM] * 2
    dont_care = []
    for (f, cap), o in zip(pairs, offs):               # the skip call wrote last
        r, data, _ = fm.decode(oracle, f, cap, True)
        if r == cap:
            ar.expect(o, data)
        else:
            dont_care.append((o, cap))
    ar.check(dont_care)
