"""The drop-in LZ4_compress_HC family on the GPU: LZ4_compress_HC, LZ4_compress_HC_extStateHC(_fastReset) and
LZ4_compress_HC_destSize, and their Python faces in lz4_b200.block, against the reference's results
(tests/golden/kat_hc_dropin.json) with guard bytes past every capacity and target, in-place calls, the batch calls on
random inputs, eight host threads at once, and the state a later reference LZ4_compress_HC_continue takes over.

One GPU thread parses each call's block, so every golden row goes through one of the entry points in turn rather than
through all of them."""
import ctypes as C
import hashlib
import threading

import numpy as np
import pytest
import torch

import hc_emul as he
import make_golden_hc_dropin as mk
from make_golden_hc import compress_bound, run_digest
from make_golden_hc_destsize import run_digest as dest_run_digest

pytestmark = pytest.mark.gpu

SENTINEL = 0x5A
GUARD = 64
DEV = "cuda:0"
PLAIN = ("LZ4_compress_HC", "LZ4_compress_HC_extStateHC", "LZ4_compress_HC_extStateHC_fastReset", "block")
DEST = ("LZ4_compress_HC_destSize", "block")


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    lib = _lib.load()
    if lib.LZ4B200_device_count() <= 0:
        pytest.skip("no CUDA device")
    return lib


@pytest.fixture(scope="module")
def golden(oracle):
    doc, ins = he.golden("kat_hc_dropin.json")
    return doc, ins, {iid: mk.make_input(oracle, i["size"], i["kind"], i["seed"]) for iid, i in ins.items()}


def _src(data):
    """the input with a real address even when empty"""
    src = np.zeros(max(len(data), 1), dtype=np.uint8)
    src[:len(data)] = np.asarray(data, dtype=np.uint8)
    return src


def plain(lib, how, data, cap, level):
    """(ret, bytes) of one LZ4_compress_HC-type call through `how`; nothing at or past the returned size is written"""
    from lz4_b200 import block
    if how == "block":
        return block.LZ4_compress_HC(data, level, cap)
    src = _src(data)
    dst = np.full(max(min(cap, compress_bound(len(data))), 0) + GUARD, SENTINEL, dtype=np.uint8)
    state = np.zeros(mk.STATE_BYTES // 8, dtype=np.uint64)
    if how == "LZ4_compress_HC":
        r = lib.LZ4_compress_HC(src.ctypes.data, dst.ctypes.data, len(data), cap, level)
    else:
        r = getattr(lib, how)(state.ctypes.data, src.ctypes.data, dst.ctypes.data, len(data), cap, level)
    assert (dst[max(r, 0):] == SENTINEL).all(), ("write past the returned size", how, len(data), cap, level)
    return r, dst[:max(r, 0)].tobytes()


def dest(lib, how, data, target, level):
    """(ret, consumed, bytes) of one LZ4_compress_HC_destSize call through `how`; nothing past the returned size is
    written"""
    from lz4_b200 import block
    if how == "block":
        return block.LZ4_compress_HC_destSize(data, target, level)
    src = _src(data)
    dst = np.full(max(min(target, compress_bound(len(data))), 0) + GUARD, SENTINEL, dtype=np.uint8)
    state = np.zeros(mk.STATE_BYTES // 8, dtype=np.uint64)
    n = C.c_int(len(data))
    r = lib.LZ4_compress_HC_destSize(state.ctypes.data, src.ctypes.data, dst.ctypes.data, C.byref(n), target, level)
    assert (dst[max(r, 0):] == SENTINEL).all(), ("write past the returned size", len(data), target, level)
    return r, n.value, dst[:max(r, 0)].tobytes()


def launches_of(n, limit):
    return 1 if n > 0 and limit >= 1 else 0


def test_golden_plain_rows(lib, golden):
    """Every LZ4_compress_HC vector, each through one of the three C entry points or block.LZ4_compress_HC in turn: the
    reference's return values and bytes, and one launch per call that has a block to parse"""
    doc, ins, data = golden
    wrong, launches = [], 0
    l0 = lib.LZ4B200_launch_count()
    for k, (iid, lv, caps, rets, dig) in enumerate(doc["vectors"]):
        how = PLAIN[k % len(PLAIN)]
        res = [plain(lib, how, data[iid], cap, lv) for cap in caps]
        launches += sum(launches_of(ins[iid]["size"], cap) for cap in caps)
        if [r for r, _ in res] != rets or run_digest(res) != dig:
            wrong.append((how, ins[iid], lv, caps, [r for r, _ in res], rets))
    assert not wrong, wrong[:5]
    assert lib.LZ4B200_launch_count() - l0 == launches


def test_golden_dest_rows(lib, golden):
    """Every LZ4_compress_HC_destSize vector, through the C entry point and block.LZ4_compress_HC_destSize in turn"""
    doc, ins, data = golden
    wrong, launches = [], 0
    l0 = lib.LZ4B200_launch_count()
    for k, (iid, lv, ts, rets, cons, dig) in enumerate(doc["dest_vectors"]):
        how = DEST[k % len(DEST)]
        res = [dest(lib, how, data[iid], t, lv) for t in ts]
        launches += sum(launches_of(ins[iid]["size"], t) for t in ts)
        if [r for r, _, _ in res] != rets or [c for _, c, _ in res] != cons or dest_run_digest(res) != dig:
            wrong.append((how, ins[iid], lv, ts, [(r, c) for r, c, _ in res], list(zip(rets, cons))))
    assert not wrong, wrong[:5]
    assert lib.LZ4B200_launch_count() - l0 == launches


def test_valid_states_give_the_reference_results(lib, golden):
    """The verdict rows whose state the reference accepts (aligned at 0 and 8 bytes from a 64-byte boundary) give its
    results, and _extStateHC and _destSize leave the state image LZ4_initStreamHC leaves"""
    doc, ins, data = golden
    v = doc["verdicts"]
    d = _src(data[v["input"]])
    cap = compress_bound(len(data[v["input"]]))
    for name, rows in v["calls"].items():
        for off, ret, cons in rows:
            if ret == 0:
                continue
            p, keep = mk.state_buffer(off)
            dst = np.full(cap + GUARD, SENTINEL, dtype=np.uint8)
            if name.endswith("destSize"):
                n = C.c_int(len(data[v["input"]]))
                got = (lib.LZ4_compress_HC_destSize(p, d.ctypes.data, dst.ctypes.data, C.byref(n), v["target"],
                                                    v["level"]), n.value)
                assert got == (ret, cons)
            else:
                assert getattr(lib, name)(p, d.ctypes.data, dst.ctypes.data, len(data[v["input"]]), cap,
                                          v["level"]) == ret
            img = C.string_at(p, mk.STATE_BYTES)
            if name.endswith("fastReset"):
                assert img == bytes([mk.STATE_FILL]) * mk.STATE_BYTES
            else:
                assert hashlib.sha256(img).hexdigest() == doc["state"]["sha256"], (name, off)
            del keep


@pytest.mark.parametrize("level", [2, 9, 10])
def test_in_place_and_overlapping_buffers(lib, oracle, level):
    """src and dst in one buffer: dst at the start and the input at its end (lz4.h's in-place layout), the input and
    dst at the same address, and dst one byte after the input's start; the results are those of separate buffers"""
    for n in (4096, 20000):
        data = mk.make_input(oracle, n, "p50" if n == 4096 else "text", 31 + n + level)
        bound = compress_bound(n)
        want = plain(lib, "LZ4_compress_HC", data, bound, level)
        want_d = dest(lib, "LZ4_compress_HC_destSize", data, 1500, level)
        for src_off, dst_off in ((bound + GUARD - n, 0), (0, 0), (0, 1)):
            buf = np.full(bound + GUARD + 1, SENTINEL, dtype=np.uint8)
            buf[src_off:src_off + n] = data
            r = lib.LZ4_compress_HC(buf.ctypes.data + src_off, buf.ctypes.data + dst_off, n, bound, level)
            assert (r, buf[dst_off:dst_off + r].tobytes()) == want, (n, src_off, dst_off)
            buf[:] = SENTINEL
            buf[src_off:src_off + n] = data
            m = C.c_int(n)
            state = np.zeros(mk.STATE_BYTES // 8, dtype=np.uint64)
            r = lib.LZ4_compress_HC_destSize(state.ctypes.data, buf.ctypes.data + src_off, buf.ctypes.data + dst_off,
                                             C.byref(m), 1500, level)
            assert (r, m.value, buf[dst_off:dst_off + r].tobytes()) == want_d, (n, src_off, dst_off)


def batch_call(lib, blocks, limit, level, fill):
    """One batched call over `blocks` (per-block sizes): LZ4B200_compress_blocks_hc(_opt)(_destSize) by level.  Returns
    [(ret, bytes)] or [(ret, consumed, bytes)]."""
    nb = len(blocks)
    sizes = [len(b) for b in blocks]
    src_stride = max(sizes) + 16
    dst_stride = max(min(limit, compress_bound(n)) for n in sizes) + 16
    src_h = np.zeros(nb * src_stride + 16, dtype=np.uint8)
    for i, b in enumerate(blocks):
        src_h[i * src_stride:i * src_stride + len(b)] = b
    src = torch.from_numpy(src_h).to(DEV)
    dst = torch.zeros(nb * dst_stride + 16, dtype=torch.uint8, device=DEV)
    szs = torch.tensor(sizes, dtype=torch.int32, device=DEV)
    outs = torch.zeros(nb, dtype=torch.int32, device=DEV)
    cons = torch.zeros(nb, dtype=torch.int32, device=DEV)
    opt = level >= 10
    ws = torch.empty(int((lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes if opt else
                          lib.LZ4B200_compress_blocks_hc_workspace_bytes)(nb)), dtype=torch.uint8, device=DEV)
    s = torch.cuda.current_stream().cuda_stream
    if fill:
        fn = lib.LZ4B200_compress_blocks_hc_opt_destSize if opt else lib.LZ4B200_compress_blocks_hc_destSize
        rc = fn(src.data_ptr(), src_stride, szs.data_ptr(), 0, dst.data_ptr(), dst_stride, limit, level, outs.data_ptr(),
                cons.data_ptr(), nb, ws.data_ptr(), ws.numel(), s)
    else:
        fn = lib.LZ4B200_compress_blocks_hc_opt if opt else lib.LZ4B200_compress_blocks_hc
        rc = fn(src.data_ptr(), src_stride, szs.data_ptr(), 0, dst.data_ptr(), dst_stride, limit, level, outs.data_ptr(),
                nb, ws.data_ptr(), ws.numel(), s)
    assert rc == 0
    torch.cuda.synchronize()
    d, rets, cs = dst.cpu().numpy(), outs.cpu().tolist(), cons.cpu().tolist()
    out = [d[i * dst_stride:i * dst_stride + max(rets[i], 0)].tobytes() for i in range(nb)]
    return [(rets[i], cs[i], out[i]) if fill else (rets[i], out[i]) for i in range(nb)]


@pytest.mark.parametrize("level", [-3, 1, 2, 4, 9, 10, 11, 12, 100])
def test_random_inputs_agree_with_the_batch_calls(lib, oracle, level):
    rng = np.random.default_rng(4100 + level)
    kinds = mk.KINDS + ["per1", "per3", "p0"]
    blocks = [mk.make_input(oracle, int(rng.choice([1, 12, 13, 14, 100, 777, 3000, 9000, 20000])),
                            kinds[int(rng.integers(0, len(kinds)))], 5000 + 10 * level + k) for k in range(8)]
    for limit in (1 << 20, 900, 13):
        got = batch_call(lib, blocks, limit, level, False)
        assert [plain(lib, PLAIN[k % len(PLAIN)], b, limit, level) for k, b in enumerate(blocks)] == got, limit
    for target in (1 << 20, 1000, 9):
        got = batch_call(lib, blocks, target, level, True)
        assert [dest(lib, DEST[k % len(DEST)], b, target, level) for k, b in enumerate(blocks)] == got, target


def test_eight_host_threads(lib, golden):
    """Eight threads call the drop-in entry points at once, each on its own share of the golden rows up to 4 KB"""
    doc, ins, data = golden
    jobs = [("plain", iid, lv, caps, rets, dig) for iid, lv, caps, rets, dig in doc["vectors"]
            if 0 < ins[iid]["size"] <= 4096] + \
           [("dest", iid, lv, ts, (rets, cons), dig) for iid, lv, ts, rets, cons, dig in doc["dest_vectors"]
            if 0 < ins[iid]["size"] <= 4096]
    wrong = []

    def work(t):
        for k in range(t, len(jobs), 8):
            mode, iid, lv, limits, want, dig = jobs[k]
            if mode == "plain":
                res = [plain(lib, PLAIN[k % 3], data[iid], c, lv) for c in limits]
                ok = [r for r, _ in res] == want and run_digest(res) == dig
            else:
                res = [dest(lib, DEST[0], data[iid], t_, lv) for t_ in limits]
                ok = ([r for r, _, _ in res], [c for _, c, _ in res]) == want and dest_run_digest(res) == dig
            if not ok:
                wrong.append((mode, iid, lv))

    threads = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert len(jobs) > 200 and not wrong, wrong[:5]


@pytest.mark.parametrize("level", [3, 9, 12])
def test_reference_continues_from_the_state(lib, reference, oracle, level):
    """After this library's LZ4_compress_HC_extStateHC, the reference's LZ4_resetStreamHC_fast and two
    LZ4_compress_HC_continue calls (the second one uses the first block as its dictionary) give what they give on a state
    from the reference's LZ4_initStreamHC; the first call's result is the reference's LZ4_compress_HC_extStateHC's"""
    rl = reference.lib
    rl.LZ4_initStreamHC.restype = C.c_void_p
    rl.LZ4_initStreamHC.argtypes = [C.c_void_p, C.c_size_t]
    rl.LZ4_resetStreamHC_fast.restype = None
    rl.LZ4_resetStreamHC_fast.argtypes = [C.c_void_p, C.c_int]
    rl.LZ4_compress_HC_continue.restype = C.c_int
    rl.LZ4_compress_HC_continue.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    rl.LZ4_compress_HC_extStateHC.restype = C.c_int
    rl.LZ4_compress_HC_extStateHC.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int]
    first = mk.make_input(oracle, 20000, "text", 77 + level)
    blocks = [mk.make_input(oracle, 9000, "text", 78 + level), mk.make_input(oracle, 9000, "p50", 79 + level)]
    stream = np.concatenate(blocks)                     # contiguous, so the second block sees the first as a prefix
    cap = compress_bound(len(first))

    def continued(p):
        rl.LZ4_resetStreamHC_fast(p, level)
        out = []
        for k, n in ((0, 9000), (9000, 9000)):
            dst = np.zeros(compress_bound(n), dtype=np.uint8)
            r = rl.LZ4_compress_HC_continue(p, stream.ctypes.data + k, dst.ctypes.data, n, len(dst))
            out.append((r, dst[:max(r, 0)].tobytes()))
        return out

    ours, keep1 = mk.state_buffer(0)
    theirs, keep2 = mk.state_buffer(0)
    dst = np.zeros(cap, dtype=np.uint8)
    r = lib.LZ4_compress_HC_extStateHC(ours, first.ctypes.data, dst.ctypes.data, len(first), cap, level)
    rdst = np.zeros(cap, dtype=np.uint8)
    scratch, keep3 = mk.state_buffer(0)
    assert (r, dst[:r].tobytes()) == (rl.LZ4_compress_HC_extStateHC(scratch, first.ctypes.data, rdst.ctypes.data,
                                                                   len(first), cap, level), rdst[:r].tobytes())
    assert rl.LZ4_initStreamHC(theirs, mk.STATE_BYTES) == theirs
    assert C.string_at(ours, mk.STATE_BYTES) == C.string_at(theirs, mk.STATE_BYTES)
    got, want = continued(ours), continued(theirs)
    assert got == want and all(r > 0 for r, _ in got)
    del keep1, keep2, keep3
