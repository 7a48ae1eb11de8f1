"""LZ4B200_decompress_frames_checksummed on the GPU, in both checksum modes: the reference's checksummed frames and a
frame of its `lz4` tool, the reference's outcome on every corrupted frame, LZ4B200_decompress_frames's results on frames
without checksums, XXH32's tail and alignment paths in both checksum kernels, mixed batches with a budget overrun and
guard bytes, and a side stream with graph capture.  Reads only tests/golden/frames_checksum.json."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch

import frame_checksum_model as fm
import frame_corpus as fc
from conftest import load_golden

pytestmark = pytest.mark.gpu

GUARD = 0xA5
GAP = 48


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    return _lib.load()


@pytest.fixture(scope="module")
def golden():
    return load_golden("frames_checksum.json")


def sha(b):
    return hashlib.sha256(bytes(b)).hexdigest()


def need(frames):
    """blocks per class of the frames whose header and chain (checksum fields included) are valid"""
    n = [0, 0, 0, 0]
    for f in frames:
        if len(f) >= 7 and f[:4] == fc.MAGIC.to_bytes(4, "little"):
            w = fm.walk(f)
            c = ((f[5] >> 4) & 7) - 4
            if w is not None and 0 <= c < 4:
                n[c] += len(w[0])
    return n


class Batch:
    """frames on the device at the given offsets mod 16 (default: odd ones), PAD bytes of padding; output regions with
    GAP guard bytes between them"""

    def __init__(self, frames, caps, src_mod=None, dst_mod=None, seed=0):
        rng = np.random.default_rng(seed)
        self.frames, self.caps = frames, caps
        buf, offs = bytearray(b"\xEE" * fc.PAD), []
        for k, f in enumerate(frames):
            want = src_mod[k] if src_mod else int(rng.integers(0, 16)) | 1
            buf += b"\xEE" * ((want - len(buf)) % 16)
            offs.append(len(buf))
            buf += f + b"\xEE" * fc.PAD
        self.src = torch.from_numpy(np.frombuffer(bytes(buf), dtype=np.uint8).copy()).cuda()
        self.off = torch.tensor(offs, dtype=torch.int64, device="cuda")
        self.size = torch.tensor([len(f) for f in frames], dtype=torch.int64, device="cuda")
        doff, at = [], 16
        for k, c in enumerate(caps):
            at += ((dst_mod[k] if dst_mod else int(rng.integers(0, 16))) - at) % 16
            doff.append(at)
            at += max(c, 0) + GAP
        self.dst_off = doff
        self.out = torch.full((at + GAP,), GUARD, dtype=torch.uint8, device="cuda")
        self.d_off = torch.tensor(doff, dtype=torch.int64, device="cuda")
        self.d_cap = torch.tensor(caps, dtype=torch.int64, device="cuda")

    def run(self, mb, skip=None, **kw):
        """the checksummed call (skip: 0 / 1), or LZ4B200_decompress_frames (skip None); (results, consumed, out)"""
        from lz4_b200 import batch
        self.out.fill_(GUARD)
        if skip is None:
            _, r, c = batch.decompress_frames(self.src, self.off, self.size, self.d_cap, mb, out=self.out,
                                              out_offsets=self.d_off, **kw)
        else:
            _, r, c = batch.decompress_frames_checksummed(self.src, self.off, self.size, self.d_cap, mb, bool(skip),
                                                          out=self.out, out_offsets=self.d_off, **kw)
        torch.cuda.synchronize()
        out = self.out.cpu().numpy()
        inside = np.zeros(len(out), dtype=bool)
        for o, cap in zip(self.dst_off, self.caps):
            inside[o:o + max(cap, 0)] = True
        assert (out[~inside] == GUARD).all(), "a byte outside every output region was written"
        return r.cpu().tolist(), c.cpu().tolist(), out

    def data(self, out, f, n):
        return out[self.dst_off[f]:self.dst_off[f] + n].tobytes()


_decoded = {}


def model(oracle, frame, cap, skip):
    """fm.decode, once per (frame, capacity, mode)"""
    key = (frame, cap, skip)
    if key not in _decoded:
        _decoded[key] = fm.decode(oracle, frame, cap, skip)
    return _decoded[key]


def check_model(b, oracle, res, cons, out, skip, skip_rows=()):
    """every frame's result, bytes and consumed length against the model"""
    for f, (fr, cap) in enumerate(zip(b.frames, b.caps)):
        if f in skip_rows:
            continue
        r, d, used = model(oracle, fr, cap, skip)
        assert res[f] == r, (f, res[f], r)
        assert cons[f] == used, (f, cons[f], used)
        if r >= 0:
            assert b.data(out, f, r) == d, f


def golden_frames(oracle, golden):
    out = []
    for row in golden["frames"]:
        data = fm.content(oracle.datagen, row["spec"])
        f = fm.compress_frame(oracle, data, row["bsid"], row["content_size"], row["block_sum"], row["content_sum"])
        assert sha(f) == row["frame_sha256"]
        out.append((f, data))
    cli = bytes.fromhex(golden["cli"]["frame_hex"])
    out.append((cli, fm.content(oracle.datagen, golden["cli"]["spec"])))
    return out


@pytest.mark.parametrize("skip", [0, 1])
def test_reference_and_cli_frames(lib, oracle, golden, skip):
    pairs = golden_frames(oracle, golden)
    frames = [f for f, _ in pairs]
    b = Batch(frames, [max(len(d), 1) for _, d in pairs])
    res, cons, out = b.run(need(frames), skip)
    assert res == [len(d) for _, d in pairs]
    assert cons == [len(f) for f in frames]
    for k, (_, d) in enumerate(pairs):
        assert b.data(out, k, len(d)) == d, k


@pytest.mark.parametrize("skip", [0, 1])
def test_corrupted_corpus_gets_the_references_outcome(lib, oracle, golden, skip):
    pairs = golden_frames(oracle, golden)
    frames, caps, rows = [], [], []
    good = pairs[2][0]
    for row in golden["corrupted"]:
        m = dict(fm.mutations(pairs[row["frame"]][0]))[row["mutation"]]
        frames += [m, good]
        caps += [row["cap"], len(pairs[2][1])]
        rows.append(row)
    b = Batch(frames, caps, seed=3)
    res, cons, out = b.run(need(frames), skip)
    assert res[1::2] == [len(pairs[2][1])] * len(rows)
    check_model(b, oracle, res, cons, out, skip)
    mode = "skip" if skip else "verify"
    for k, row in enumerate(rows):
        ref = row[mode]
        if skip and ref["error"] == "blockChecksum_invalid":     # compared by lz4frame.c even under skipChecksums
            continue
        assert res[2 * k] == fm.ref_class(ref), (row, res[2 * k])
        assert (res[2 * k] == fm.ERR_CHECKSUM) == (ref["error"] in ("blockChecksum_invalid", "contentChecksum_invalid"))
        if ref["error"] is None:
            assert sha(b.data(out, 2 * k, ref["size"])) == ref["sha"] and cons[2 * k] == ref["consumed"]
    if not skip:
        assert fm.ERR_CHECKSUM in res


@pytest.mark.parametrize("skip", [0, 1])
def test_frames_without_checksums_match_decompress_frames(lib, oracle, skip):
    pairs = fc.good_frames(oracle)
    frames = [f for f, _ in pairs]
    for g in (frames[4], frames[9], frames[-1]):
        frames += [m for _, m in fc.mutations(g) if len(m) < 5 or not m[4] & (fm.FLG_BLOCK_SUM | fm.FLG_CONTENT_SUM)]
    caps = [1 << 23 if k % 5 else 1000 for k in range(len(frames))]
    b = Batch(frames, caps, seed=7)
    mb = need(frames)
    r0, c0, o0 = b.run(mb)
    r1, c1, o1 = b.run(mb, skip)
    assert r1 == r0 and c1 == c0
    for f, r in enumerate(r0):
        if r >= 0:
            assert b.data(o1, f, r) == b.data(o0, f, r), f
    assert {fc.OK, fc.ERR_FRAME, fc.ERR_UNSUPPORTED} <= {min(r, 0) for r in r0}


EDGES = [0, 1, 2, 3, 15, 16, 17, 31, 32, 33, 47, 48, 49]


def edge_frames(oracle):
    """raw blocks (payload = the length) with block and content checksums at every edge length, 64 KB and 4 MB, each
    intact and with its last payload byte flipped; and compressed blocks of every source size mod 16"""
    rng = np.random.default_rng(5)
    frames = []
    for n in EDGES + [65536, 4 << 20]:
        d = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        bsid = 7 if n > 65536 else 4
        pieces = [d] if n else []
        f = fm.frame_of_blocks(oracle, pieces, bsid, raw=(0,), block_sum=True, content_sum=True)
        frames.append(f)
        if n:
            blocks, _ = fm.walk(f)
            o, sz, _ = blocks[0]
            bad = bytearray(f)
            bad[o + sz - 1] ^= 1
            frames.append(bytes(bad))                                    # the block checksum's tail path
            frames.append(fm.frame_of_blocks(oracle, [d[:n // 2], d[n // 2:]] if n > 1 else [d], bsid,
                                             raw=(0, 1), content_sum=True))
    d = oracle.datagen(70000, 0.5, 9).tobytes()
    for k in range(16):                                                  # compressed blocks of every length mod 16
        frames.append(fm.frame_of_blocks(oracle, [d[:3000 + k], d[3000 + k:9000]], 4, block_sum=True, content_sum=True))
    return frames


def test_xxh32_edges_at_every_alignment(lib, oracle):
    frames = edge_frames(oracle)
    caps = [(4 << 20) + 64] * len(frames)
    mb = need(frames)
    for shift in range(16):
        b = Batch(frames, caps, src_mod=[(k + shift) % 16 for k in range(len(frames))],
                  dst_mod=[(3 * k + shift) % 16 for k in range(len(frames))], seed=shift)
        res, cons, out = b.run(mb, 0)
        check_model(b, oracle, res, cons, out, 0)
        assert res.count(fm.ERR_CHECKSUM) == len(EDGES) + 1
    res, cons, out = b.run(mb, 1)
    check_model(b, oracle, res, cons, out, 1)
    assert fm.ERR_CHECKSUM not in res


def content_sum_flipped(frame):
    b = bytearray(frame)
    b[-1] ^= 0x80
    return bytes(b)


def mixed(oracle, golden):
    pairs = golden_frames(oracle, golden)
    plain = [f for f, _ in fc.good_frames(oracle, big=False)]
    frames = []
    for k in range(max(len(pairs), len(plain))):
        if k < len(pairs):
            frames.append(pairs[k][0])
        if k < len(plain):
            frames.append(plain[k])
    frames.append(content_sum_flipped(pairs[0][0]))
    return frames


def budget_status(frames, mb):
    run, out = [0, 0, 0, 0], []
    for f in frames:
        c = ((f[5] >> 4) & 7) - 4
        n = len(fm.walk(f)[0])
        out.append(fc.ERR_LIMIT if run[c] + n > mb[c] else fc.OK)
        run[c] += n
    return out


@pytest.mark.parametrize("skip", [0, 1])
def test_mixed_batches_with_a_budget_overrun(lib, oracle, golden, skip):
    frames = mixed(oracle, golden)
    order = np.random.default_rng(2).permutation(len(frames))
    frames = [frames[i] for i in order]
    caps = [(5 << 20) if k % 3 else (4 << 20) + 20000 for k in range(len(frames))]
    full = need(frames)
    b = Batch(frames, caps, seed=11)
    res, cons, out = b.run(full, skip)
    check_model(b, oracle, res, cons, out, skip)
    assert (fm.ERR_CHECKSUM in res) == (not skip)
    for c in range(4):
        mb = list(full)
        mb[c] -= 1
        want = budget_status(frames, mb)
        res, cons, out = b.run(mb, skip)
        limited = {f for f, s in enumerate(want) if s == fc.ERR_LIMIT}
        assert limited and all(res[f] == fc.ERR_LIMIT and cons[f] == 0 for f in limited)
        check_model(b, oracle, res, cons, out, skip, skip_rows=limited)


def test_side_stream_graph_capture_and_launch_count(lib, oracle, golden):
    from lz4_b200 import batch
    frames = mixed(oracle, golden)
    caps = [5 << 20] * len(frames)
    mb = need(frames)
    ref = Batch(frames, caps)
    r0, c0, _ = ref.run(mb, 0)
    want_out = ref.out.clone()
    launches = {}
    for skip in (None, 0, 1):
        n0 = lib.LZ4B200_launch_count()
        ref.run(mb, skip)
        launches[skip] = lib.LZ4B200_launch_count() - n0
    assert launches[1] == launches[None] and launches[0] == launches[None] + 2

    b = Batch(frames, caps)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ws = torch.empty(batch.decompress_frames_workspace_bytes(len(frames), mb), dtype=torch.uint8, device="cuda")
        res = torch.full((len(frames),), 7, dtype=torch.int64, device="cuda")
        cons = torch.full((len(frames),), 7, dtype=torch.int64, device="cuda")
    side.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
        batch.decompress_frames_checksummed(b.src, b.off, b.size, b.d_cap, mb, False, out=b.out, out_offsets=b.d_off,
                                            results=res, consumed=cons, workspace=ws)
    torch.cuda.synchronize()
    assert (res == 7).all().item()                  # captured: nothing ran
    for _ in range(2):
        b.out.fill_(GUARD)
        res.fill_(7)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert res.cpu().tolist() == r0 and cons.cpu().tolist() == c0 and torch.equal(b.out, want_out)
    rc = lib.LZ4B200_decompress_frames_checksummed(b.src.data_ptr(), b.off.data_ptr(), b.size.data_ptr(),
                                                   b.out.data_ptr(), b.d_off.data_ptr(), b.d_cap.data_ptr(),
                                                   res.data_ptr(), None, len(frames), (C.c_int64 * 4)(*mb), 0,
                                                   ws.data_ptr(), ws.numel() - 1, None)
    assert rc == fc.ERR_ARG


@pytest.mark.parametrize("skip", [False, True])
def test_content_size_field_past_2_63(lib, oracle, skip):
    """a content-size field with bit 63 set (its header checksum right) is a size no frame decodes to: LZ4F_decompress
    fails it with frameSize_wrong, so the frame calls and the file calls give LZ4B200_ERR_FRAME (the frame calls once
    read such a field as "no content size" and decoded the frame)"""
    import struct
    from lz4_b200 import batch
    data = oracle.datagen(13, 0.5, 9).tobytes()
    good = bytearray(fm.compress_frame(oracle, data, 4, True, True, True))
    bad = bytearray(good)
    struct.pack_into("<Q", bad, 6, (1 << 63) | len(data))
    hl = fc.header_len(bytes(bad))
    bad[hl - 1] = (fm.xxh32(bytes(bad[4:hl - 1])) >> 8) & 0xFF
    assert fm.decode(oracle, bytes(bad), 64, skip)[0] == fc.ERR_FRAME
    frames = [bytes(good), bytes(bad)]
    arena = np.zeros(16 + sum(len(f) + 16 for f in frames), dtype=np.uint8)
    offs = [16, 32 + len(frames[0])]
    for o, f in zip(offs, frames):
        arena[o:o + len(f)] = np.frombuffer(f, dtype=np.uint8)
    t = lambda a: torch.tensor(a, dtype=torch.int64, device="cuda")      # noqa: E731
    src = torch.from_numpy(arena).cuda()
    _, res, _ = batch.decompress_frames_checksummed(src, t(offs), t([len(f) for f in frames]), t([64, 64]), [2, 0, 0, 0],
                                                    skip_checksums=skip)
    _, fres, _, _ = batch.decompress_files(src, t(offs), t([len(f) for f in frames]), t([64, 64]), 2, [2, 0, 0, 0, 0],
                                           skip_checksums=skip)
    torch.cuda.synchronize()
    assert res.cpu().tolist() == [len(data), fc.ERR_FRAME]
    assert fres.cpu().tolist() == [len(data), fc.ERR_FRAME]
