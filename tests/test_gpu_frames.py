"""LZ4B200_decompress_frames on the GPU: every frame's result, decoded bytes and consumed length against
LZ4B200_decompressFrame_host on that frame alone, with guard bytes around every output region, for golden and reference
frames, mixed batches of every block size, malformed frames among good ones, budgets, streams and graphs, and offsets past
4 GiB."""
import ctypes as C
import struct

import numpy as np
import pytest
import torch

import frame_corpus as fc
import frame_oracle as fo
from conftest import load_golden

pytestmark = pytest.mark.gpu

GUARD = 0xA5
GAP = 48                                            # guard bytes between output regions


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    return _lib.load()


def host_call(lib, frame, cap):
    """LZ4B200_decompressFrame_host on one frame: (result, bytes written, consumed)"""
    src = np.frombuffer(bytes(frame) + b"\0" * 16, dtype=np.uint8)
    dst = np.zeros(max(cap, 1), dtype=np.uint8)
    used = C.c_int64(0)
    r = int(lib.LZ4B200_decompressFrame_host(src.ctypes.data, len(frame), dst.ctypes.data, cap, C.byref(used)))
    return r, dst[:max(r, 0)].tobytes(), used.value


def need(frames):
    """blocks per class of the frames whose header and chain are valid"""
    n = [0, 0, 0, 0]
    for f in frames:
        if len(f) >= 7 and struct.unpack_from("<I", f, 0)[0] == fc.MAGIC and fc.walk(f) is not None:
            c = ((f[5] >> 4) & 7) - 4
            if 0 <= c < 4:
                n[c] += len(fc.walk(f)[0])
    return n


class Batch:
    """frames laid out on the device (odd offsets, PAD bytes of padding), output regions with GAP guard bytes between
    them at odd offsets"""

    def __init__(self, frames, caps, seed=0, src_base=0, dst_base=0):
        self.frames, self.caps = frames, caps
        buf, offs = fc.layout(frames, seed=seed)
        self.src = torch.zeros(src_base + len(buf), dtype=torch.uint8, device="cuda")
        self.src[src_base:] = torch.from_numpy(np.frombuffer(buf, dtype=np.uint8).copy()).cuda()
        self.off = torch.tensor([src_base + o for o in offs], dtype=torch.int64, device="cuda")
        self.size = torch.tensor([len(f) for f in frames], dtype=torch.int64, device="cuda")
        doff, at = [], dst_base + 3
        for c in caps:
            doff.append(at)
            at += max(c, 0) + GAP + 1
        self.dst_off = doff
        self.out = torch.full((at + GAP,), GUARD, dtype=torch.uint8, device="cuda")
        self.d_off = torch.tensor(doff, dtype=torch.int64, device="cuda")
        self.d_cap = torch.tensor(caps, dtype=torch.int64, device="cuda")

    def run(self, mb, **kw):
        from lz4_b200 import batch
        return batch.decompress_frames(self.src, self.off, self.size, self.d_cap, mb, out=self.out,
                                       out_offsets=self.d_off, **kw)

    def check(self, lib, res, cons, want_status=None, sources=None):
        """results and consumed against the host call, decoded bytes of every good frame, untouched guards"""
        res, cons = res.cpu().tolist(), cons.cpu().tolist()
        out = self.out.cpu().numpy()
        inside = np.zeros(len(out), dtype=bool)
        for f, (fr, cap) in enumerate(zip(self.frames, self.caps)):
            o = self.dst_off[f]
            if cap > 0:
                inside[o:o + cap] = True
            if want_status is not None and want_status[f] == fc.ERR_LIMIT:
                assert res[f] == fc.ERR_LIMIT and cons[f] == 0, f
                continue
            r, data, used = host_call(lib, fr, cap)
            assert res[f] == r, (f, res[f], r)
            assert cons[f] == used, (f, cons[f], used)   # the host call sets it once the chain is valid, else leaves 0
            if r >= 0:
                assert out[o:o + r].tobytes() == data, f
                if sources is not None and sources[f] is not None:
                    assert data == sources[f]
        assert (out[~inside] == GUARD).all(), "a byte outside every output region was written"
        return res


def mixed(oracle):
    pairs = fc.good_frames(oracle)
    frames = [f for f, _ in pairs]
    srcs = [d for _, d in pairs]
    frames.append(pairs[9][0] + b"trailing garbage")                    # bytes after the frame: not consumed
    srcs.append(pairs[9][1])
    return frames, srcs


def test_golden_and_reference_frames_in_one_batch(lib, oracle):
    from oracle.pyoracle import Reference, have_reference
    frames, srcs = [], []
    for row in load_golden("frames.json")["frames"]:
        d = oracle.datagen(row["size"], row["proba"], row["seed"]).tobytes() if row["size"] else b""
        f = fo.compress_frame(oracle, d, row["bsid"], row["level"], row["content_size"])
        assert len(f) == row["frame_size"] and fc.walk(f) is not None
        frames.append(f)
        srcs.append(d)
        if have_reference() and Reference().have_frame():
            frames.append(Reference().compress_frame(d, row["bsid"], row["level"], row["content_size"]))
            srcs.append(d)
    caps = [max(len(d), 1) for d in srcs]
    b = Batch(frames, caps)
    _, res, cons = b.run(need(frames))
    got = b.check(lib, res, cons, sources=srcs)
    assert got == [len(d) for d in srcs]
    assert cons.cpu().tolist() == [len(f) for f in frames]


@pytest.mark.parametrize("seed", [0, 1])
def test_mixed_batches_of_every_block_size(lib, oracle, seed):
    frames, srcs = mixed(oracle)
    order = np.random.default_rng(seed).permutation(len(frames))
    frames, srcs = [frames[i] for i in order], [srcs[i] for i in order]
    caps = [len(d) + int(k % 3) * 1000 for k, d in enumerate(srcs)]
    b = Batch(frames, caps, seed=seed)
    _, res, cons = b.run(need(frames))
    assert b.check(lib, res, cons, sources=srcs) == [len(d) for d in srcs]


def errors(oracle):
    """good frames interleaved with every kind of failure"""
    d = oracle.datagen(300000, 0.5, 21).tobytes()
    good = fo.compress_frame(oracle, d, 4, 0, True)
    out = [(good, len(d))]
    # a malformed block in the middle of a frame (a lone token that promises more literal-length bytes)
    blocks, _ = fc.walk(good)
    hl = fc.header_len(good)
    o, sz, _ = blocks[2]
    bad = good[:o - 4] + struct.pack("<I", 1) + b"\xf0" + good[o + sz:]
    out.append((bad, len(d)))
    # content size +-1 (checksum fixed), dstCap one short and exact
    for delta in (1, -1):
        w = bytearray(good)
        struct.pack_into("<Q", w, 6, len(d) + delta)
        w[hl - 1] = (fo.xxh32_short(bytes(w[4:hl - 1])) >> 8) & 0xFF
        out.append((bytes(w), len(d) + 1))
    out.append((good, len(d) - 1))
    out.append((good, len(d)))
    big = fo.compress_frame(oracle, d, 5, 0, False)
    out.append((big, len(d) - 1))                                        # DSTSIZE on the last 256 KB block
    for g in (good, big, fc.good_frames(oracle, big=False)[-1][0]):
        out += [(m, len(d)) for _, m in fc.mutations(g)]
    out += [(good, -1)]                                                  # a negative capacity
    return out


def test_every_error_interleaved_with_good_frames(lib, oracle):
    errs = errors(oracle)
    good = errs[0][0]
    frames, caps = [], []
    for f, c in errs:
        frames += [f, good]
        caps += [c, 300000]
    b = Batch(frames, caps, seed=5)
    _, res, cons = b.run(need(frames))
    got = b.check(lib, res, cons)
    assert all(r == 300000 for r in got[1::2])
    assert {fc.ERR_FRAME, fc.ERR_DSTSIZE, fc.ERR_UNSUPPORTED, fc.ERR_ARG} <= set(got)


@pytest.mark.parametrize("which", ["need", "one_less", "zero"])
def test_budgets(lib, oracle, which):
    from lz4_b200 import batch
    frames, srcs = mixed(oracle)
    order = np.random.default_rng(4).permutation(len(frames))
    frames, srcs = [frames[i] for i in order], [srcs[i] for i in order]
    caps = [max(len(d), 1) for d in srcs]
    full = need(frames)
    cls = [((f[5] >> 4) & 7) - 4 for f in frames]
    for c in range(4):
        mb = list(full)
        mb[c] = {"need": full[c], "one_less": full[c] - 1, "zero": 0}[which]
        want = fc.budget_rule(frames, [fc.OK] * len(frames), cls, mb)
        b = Batch(frames, caps, seed=c)
        nbytes = batch.decompress_frames_workspace_bytes(len(frames), mb)
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        _, res, cons = b.run(mb, workspace=ws)
        b.check(lib, res, cons, want_status=want, sources=srcs)
        if which != "need":
            assert fc.ERR_LIMIT in res.cpu().tolist()
        # one byte less of workspace: refused
        rc = lib.LZ4B200_decompress_frames(b.src.data_ptr(), b.off.data_ptr(), b.size.data_ptr(), b.out.data_ptr(),
                                           b.d_off.data_ptr(), b.d_cap.data_ptr(), res.data_ptr(), None, len(frames),
                                           (C.c_int64 * 4)(*mb), ws.data_ptr(), nbytes - 1, None)
        assert rc == fc.ERR_ARG


def test_side_stream_graph_replay_and_launch_count(lib, oracle):
    from lz4_b200 import batch
    frames, srcs = mixed(oracle)
    caps = [max(len(d), 1) for d in srcs]
    mb = need(frames)
    ref = Batch(frames, caps)
    _, r0, c0 = ref.run(mb)
    want_out = ref.out.clone()
    ref.check(lib, r0, c0, sources=srcs)

    side = torch.cuda.Stream()
    b = Batch(frames, caps)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ws = torch.empty(batch.decompress_frames_workspace_bytes(len(frames), mb), dtype=torch.uint8, device="cuda")
        res = torch.empty(len(frames), dtype=torch.int64, device="cuda")
        cons = torch.empty(len(frames), dtype=torch.int64, device="cuda")
        n0 = lib.LZ4B200_launch_count()
        b.run(mb, results=res, consumed=cons, workspace=ws, stream=side)
        launches = lib.LZ4B200_launch_count() - n0
    side.synchronize()
    assert launches == 5 + sum((3 if c == 0 else 4) for c in range(4) if mb[c] > 0)
    assert torch.equal(res, r0) and torch.equal(cons, c0) and torch.equal(b.out, want_out)

    g = torch.cuda.CUDAGraph()
    b.out.fill_(GUARD)
    res.fill_(7)
    cons.fill_(7)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.graph(g, stream=s):
        b.run(mb, results=res, consumed=cons, workspace=ws)
    for _ in range(2):
        b.out.fill_(GUARD)
        res.fill_(7)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        assert torch.equal(res, r0) and torch.equal(cons, c0) and torch.equal(b.out, want_out)


def test_offsets_beyond_4_gib(lib, oracle):
    free, _ = torch.cuda.mem_get_info()
    if free < (11 << 30):
        pytest.skip("needs 11 GiB of free device memory")
    d = oracle.datagen(300000, 0.5, 31).tobytes()
    f1 = fo.compress_frame(oracle, d, 4, 0, True)
    f2 = fo.compress_frame(oracle, d[:100000], 5, 0, False)
    frames, caps = [f1, f2], [len(d), 100000]
    mb = need(frames)
    far = (1 << 32) + 12345
    b = Batch(frames, caps, src_base=far)                                # the frames past 4 GiB in d_src
    _, res, cons = b.run(mb)
    b.check(lib, res, cons, sources=[d, d[:100000]])
    del b
    torch.cuda.empty_cache()
    b = Batch(frames, caps, dst_base=far)                                # decoded past 4 GiB in d_dst
    _, res, cons = b.run(mb)
    assert res.cpu().tolist() == caps
    assert b.out[far + 3:far + 3 + len(d)].cpu().numpy().tobytes() == d
    lo = b.out[:far].eq(GUARD).all().item()
    assert lo, "a byte below the first region was written"
    del b
    torch.cuda.empty_cache()
