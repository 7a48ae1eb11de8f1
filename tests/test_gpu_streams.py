"""The batch layer off the default stream: every device-pointer call on a side stream, a phased decode across two
streams, four streams at once, host threads, CUDA graph capture, and the launch counter under threads.

The rest of the GPU suite runs on the legacy default stream, which serialises against all other work, so it cannot
tell a launcher that ignores its `stream` from one that honours it.  Here a side stream first sleeps about 100 ms; then
the real payload is copied over a zeroed input and the outputs are filled with sentinels, all on that stream, and the
call is made with it.  A launch that ran early reads zeros, one that ran late leaves sentinels in the copies taken on
the stream after the call, and either gives wrong bytes.  Everything that decides an address (offset, size, capacity
and target tables, strides) is final before the sleep, so a wrong stream can only change bytes, never reach an address
out of range.

Every result is compared with a reference: the oracle for decodes, partial decodes, compress and destSize; the host
build of the HC parses (hc_emul); the parallel compressor's host model (encpar_model); the pack
restatement (gpu_util.pack_model); the frame restatement (frame_oracle).  Guard bytes are checked as the route tests
do: a rejected block's slot and the bytes past every returned size stay as they were.

The tiles kernel (route R5) assumes its whole grid is resident, so it runs here alone on a side stream and inside a
graph, never next to other kernels."""
import ctypes as C
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for _p in (ROOT, HERE):
    if _p not in sys.path:
        sys.path.insert(0, _p)

import encpar_model  # noqa: E402
import frame_oracle  # noqa: E402
from gpu_util import GUARD, hostile_corpus, odd_stride, pack_host_blocks, pack_model, route  # noqa: E402
from hc_emul import host_hc, host_hc_dest  # noqa: E402
from lz4_b200 import _lib, batch  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SLEEP_CYCLES = 200_000_000          # torch.cuda._sleep: about 100 ms at the H100 SXM's 1.98 GHz
RET = -123456789                    # sentinel of the return-value arrays
OFF = -1                            # sentinel of pack's offset table


def bound(n):
    return n + n // 255 + 16


def lib():
    return _lib.load()


def to_dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


_memo = {}


def memo(key, fn):
    if key not in _memo:
        _memo[key] = fn()
    return _memo[key]


class Case:
    """One call on static device tensors `t`.  var[k]: variant k of the inputs (host arrays) -- the tables decide
    addresses, `data` names the payload buffers; outs: {output name: sentinel}; launch(stream) makes the call and
    returns extra output tensors it allocated; want(k) / check(res, k): the reference of variant k and the comparison."""

    def __init__(self, name, t, var, data, outs, launch, check, launches, want=None):
        self.name, self.t, self.var, self.data, self.outs = name, t, var, data, outs
        self.launch, self._check, self.launches, self.want = launch, check, launches, want or (lambda k: None)
        self._dev = {}
        self.r = {k: torch.empty_like(t[k]) for k in outs}          # result copies, allocated before any delay

    def dev(self, k):
        if k not in self._dev:
            self._dev[k] = {n: to_dev(a) for n, a in self.var[k].items()}
        return self._dev[k]

    def load_tables(self, k):
        for n, a in self.dev(k).items():
            if n not in self.data:
                self.t[n].copy_(a)

    def zero_data(self):
        for n in self.data:
            self.t[n].zero_()

    def arm(self, k):
        """on the current stream: the payload of variant k into the inputs, sentinels into the outputs"""
        for n in self.data:
            self.t[n].copy_(self.dev(k)[n])
        for n, v in self.outs.items():
            self.t[n].fill_(v)

    def collect(self, extra):
        """on the current stream: the outputs into the result copies"""
        for n in self.outs:
            self.r[n].copy_(self.t[n])
        return dict(self.r, **{n: x.clone() for n, x in (extra or {}).items()})

    def check(self, res, k):
        self._check({n: x.cpu().numpy() for n, x in res.items()}, k)


def ok(rc, what):
    _lib.check(rc, what)
    return {}


# ------------------------------------------------------------------------------------------
# decode cases: routes R1 .. R6, phased, partial
# ------------------------------------------------------------------------------------------
PB_CAPS = [65536, 65600, 65535, 30000, 4096]            # R1's per-block capacities, by block index
PB_TARGETS = [1, 4096, 30000, 65536, 0, 777]            # per-block partial targets, by block index
DECODE = {  # id: (capacity, blocks, route)
    "R1": (None, 300, "R1"), "R2": (65536, 300, "R2"), "R3": (16384, 8200, "R3"), "R4": (4096, 300, "R4"),
    "R5": (131072, 40, "R5"), "R6": (131072, 40, "R6"),
}


def corpus(oracle, cap):
    return memo(("corpus", cap), lambda: [b for _, b in hostile_corpus(oracle, cap, seed=cap % 7, n_corrupt=2)])


def decode_case(oracle, cid, mode="full", py=False):
    """mode: full (LZ4B200_decompress_blocks), phased (phases 1 then 2), partial (uniform target 30 000),
    partial-pb (per-block targets)"""
    cap, n, rt = DECODE[cid] if mode in ("full", "phased") else (65536, 300, None)
    blocks = corpus(oracle, cap or 65536)
    order = np.resize(np.random.default_rng(n).permutation(len(blocks)), n)
    per_cap = cid == "R1"
    caps = np.array([PB_CAPS[i % len(PB_CAPS)] for i in range(n)], dtype=np.int32) if per_cap else None
    targets = np.array([PB_TARGETS[i % len(PB_TARGETS)] for i in range(n)], dtype=np.int32)
    if mode == "partial-pb":
        limit, ws_bytes = int(targets.max()), int(lib().LZ4B200_decompress_workspace_bytes_for(n, 1, 0))
    elif mode == "partial":
        limit, ws_bytes = 30000, int(lib().LZ4B200_decompress_workspace_bytes_for(n, 0, 30000))
    elif per_cap or cid == "R6":
        limit, ws_bytes = int(caps.max()) if per_cap else cap, int(lib().LZ4B200_decompress_workspace_bytes(n))
    else:
        limit, ws_bytes = cap, int(lib().LZ4B200_decompress_workspace_bytes_for(n, 0, cap))
    if rt:
        assert route(n, cap, per_block_caps=per_cap, ws_bytes=ws_bytes) == rt
    stride = (limit + 64 + 15) // 16 * 16
    var = []
    for k in range(3):                                  # variant k: the batch rotated by 7k blocks, same total size
        bl = [blocks[j] for j in np.roll(order, 7 * k)]
        buf, offs, sizes = pack_host_blocks(bl)
        var.append({"comp": np.concatenate([np.zeros(16, np.uint8), buf]), "offs": offs + 16, "sizes": sizes})
        if per_cap:
            var[-1]["caps"] = caps
        if mode == "partial-pb":
            var[-1]["targets"] = targets
    t = {nm: torch.zeros(a.shape, dtype=torch.from_numpy(a[:0]).dtype, device=DEV) for nm, a in var[0].items()}
    t["out"] = torch.empty(n * stride + 64, dtype=torch.uint8, device=DEV)
    t["ret"] = torch.empty(n, dtype=torch.int32, device=DEV)
    t["ws"] = torch.zeros(ws_bytes, dtype=torch.uint8, device=DEV)

    def args():
        return (t["comp"].data_ptr(), t["offs"].data_ptr(), t["sizes"].data_ptr(), t["out"].data_ptr(), None, stride)

    def tail():
        return (t["ret"].data_ptr(), n, t["ws"].data_ptr(), ws_bytes)

    def phase(p, s):
        h = s.cuda_stream
        cap_args = (t["caps"].data_ptr(), 0) if per_cap else (None, cap)
        return ok(lib().LZ4B200_decompress_blocks_phased(*args(), *cap_args, *tail(), p, h), "phased %d" % p)

    def launch(s):
        h = s.cuda_stream
        if mode.startswith("partial"):
            tg = t["targets"] if mode == "partial-pb" else 30000
            if py:
                batch.decompress_blocks_partial(t["comp"], t["offs"], t["sizes"], tg, out=t["out"], out_stride=stride,
                                                out_sizes=t["ret"], workspace=t["ws"], stream=s)
                return {}
            pb = mode == "partial-pb"
            return ok(lib().LZ4B200_decompress_blocks_partial(*args(), t["targets"].data_ptr() if pb else None,
                                                              0 if pb else 30000, *tail(), h), "partial")
        if py:
            batch.decompress_blocks(t["comp"], t["offs"], t["sizes"], cap, out=t["out"], out_stride=stride,
                                    out_sizes=t["ret"], workspace=t["ws"], stream=s, phases=3)
            return {}
        if mode == "phased":
            phase(1, s)
            return phase(2, s)
        cap_args = (t["caps"].data_ptr(), 0) if per_cap else (None, cap)
        return ok(lib().LZ4B200_decompress_blocks(*args(), *cap_args, *tail(), h), "decompress_blocks")

    def want(k):
        def one(b, i):
            if mode == "partial-pb":
                return memo(("part", b, int(targets[i])), lambda: oracle.decompress_partial(b, int(targets[i])))
            if mode == "partial":
                return memo(("part", b, 30000), lambda: oracle.decompress_partial(b, 30000))
            c = int(caps[i]) if per_cap else cap
            return memo(("dec", b, c), lambda: oracle.decompress(b, c))
        return [one(blocks[j], i) for i, j in enumerate(np.roll(order, 7 * k))]

    def check(res, k):
        out, ret = res["out"], res["ret"]
        for i, (er, eb) in enumerate(want(k)):
            r, o = int(ret[i]), i * stride
            assert r == er, (cid, mode, k, i, r, er)
            keep = max(r, 0)
            assert out[o:o + keep].tobytes() == eb, (cid, mode, k, i)
            assert (out[o + keep:o + stride] == GUARD).all(), ("wrote past its return value", cid, mode, k, i)
        assert (out[n * stride:] == GUARD).all()

    c = Case(cid if mode == "full" else mode, t, var, ("comp",), {"out": GUARD, "ret": RET}, launch, check,
             4 if rt == "R5" else 3, want)
    c.phase = phase
    return c


# ------------------------------------------------------------------------------------------
# compress cases
# ------------------------------------------------------------------------------------------
COMPRESS = {  # id: (block sizes, None: one scalar size)
    "compress": [0, 1, 13, 100, 4096, 30000, 65536, 65537, 70000, 200000, 65536, 65536],
    "parallel-scalar": [65536] * 8,
    "parallel-split": [100, 65536, 65537, 70000, 30000, 0, 13, 200000],
    "destSize": [0, 13, 100, 4096, 30000, 65536, 65536, 70000],
    "hc": [0, 13, 4096, 30000, 65536, 65536, 70000],
    "hc-destSize": [0, 13, 4096, 30000, 65536, 65536, 70000],
}
PY_COMPRESS = 8                      # the wrappers' cases: 8 blocks of 64 KB, back to back
TARGET, ACCEL, HC_LEVEL, HCD_LEVEL = 5000, 2, 9, 6


def block_data(oracle, n, k, i):
    kind = (i + k) % 4
    if kind == 3:
        return np.random.default_rng(1000 * k + i).integers(0, 256, n, dtype=np.uint8).tobytes()
    return oracle.datagen(n, (0.5, 0.9, 0.2)[kind], 100 * k + i).tobytes()


def compress_case(oracle, cid, py=False):
    sizes = [65536] * PY_COMPRESS if py else COMPRESS[cid]
    n = len(sizes)
    scalar = py or cid == "parallel-scalar"
    src_stride = 65536 if py else max(sizes) + 16
    cap = bound(max(sizes))
    dest = cid in ("destSize", "hc-destSize")
    room = [min(TARGET, bound(m)) if dest else (min(cap, bound(m)) if cid == "hc" else None) for m in sizes]
    dst_stride = odd_stride(TARGET if dest else cap)
    var = []
    for k in range(3):
        src = np.zeros(16 + n * src_stride + 16, dtype=np.uint8)
        for i, m in enumerate(sizes):
            src[16 + i * src_stride:16 + i * src_stride + m] = np.frombuffer(block_data(oracle, m, k, i), np.uint8)
        var.append({"src": src, "sizes": np.array(sizes, dtype=np.int32)})
    t = {"src": torch.zeros(len(var[0]["src"]), dtype=torch.uint8, device=DEV),
         "sizes": torch.zeros(n, dtype=torch.int32, device=DEV),
         "dst": torch.empty(n * dst_stride + 64, dtype=torch.uint8, device=DEV),
         "ret": torch.empty(n, dtype=torch.int32, device=DEV)}
    outs = {"dst": GUARD, "ret": RET}
    if dest:
        t["consumed"] = torch.empty(n, dtype=torch.int32, device=DEV)
        outs["consumed"] = RET
    hc = cid in ("hc", "hc-destSize")
    if hc:
        t["ws"] = torch.empty(int(lib().LZ4B200_compress_blocks_hc_workspace_bytes(n)), dtype=torch.uint8, device=DEV)

    def launch(s):
        h = s.cuda_stream
        src_p, sz_p = t["src"].data_ptr() + 16, None if scalar else t["sizes"].data_ptr()
        if py:
            src = t["src"][16:16 + n * 65536]
            kw = dict(slots=t["dst"], slot_stride=dst_stride, out_sizes=t["ret"], stream=s)
            if cid in ("compress", "parallel-scalar"):
                batch.compress_blocks(src, 65536, 1, slot_capacity=cap, mode="exact" if cid == "compress" else "parallel",
                                      **kw)
            elif cid == "destSize":
                batch.compress_blocks_dest_size(src, 65536, TARGET, ACCEL, consumed=t["consumed"], **kw)
            elif cid == "hc":
                batch.compress_blocks_hc(src, 65536, HC_LEVEL, slot_capacity=cap, workspace=t["ws"], **kw)
            else:
                batch.compress_blocks_hc_dest_size(src, 65536, TARGET, HCD_LEVEL, consumed=t["consumed"],
                                                   workspace=t["ws"], **kw)
            return {}
        dst_p, ret_p, sc = t["dst"].data_ptr(), t["ret"].data_ptr(), sizes[0] if scalar else 0
        if cid == "compress":
            return ok(lib().LZ4B200_compress_blocks(src_p, src_stride, sz_p, sc, dst_p, dst_stride, cap, 1, ret_p, n, h), cid)
        if cid.startswith("parallel"):
            return ok(lib().LZ4B200_compress_blocks_parallel(src_p, src_stride, sz_p, sc, dst_p, dst_stride, cap, 1, ret_p,
                                                             n, h), cid)
        if cid == "destSize":
            return ok(lib().LZ4B200_compress_blocks_destSize(src_p, src_stride, sz_p, sc, dst_p, dst_stride, TARGET,
                                                             ACCEL, ret_p, t["consumed"].data_ptr(), n, h), cid)
        ws = (t["ws"].data_ptr(), t["ws"].numel(), h)
        if cid == "hc":
            return ok(lib().LZ4B200_compress_blocks_hc(src_p, src_stride, sz_p, sc, dst_p, dst_stride, cap, HC_LEVEL,
                                                       ret_p, n, *ws), cid)
        return ok(lib().LZ4B200_compress_blocks_hc_destSize(src_p, src_stride, sz_p, sc, dst_p, dst_stride, TARGET,
                                                            HCD_LEVEL, ret_p, t["consumed"].data_ptr(), n, *ws), cid)

    def ref(b):
        if cid == "compress":
            return oracle.compress(b, 1, cap)
        if cid.startswith("parallel"):
            m = encpar_model.compress(b, 1, cap, oracle)
            return m.ret, m.out[:m.ret]
        if cid == "destSize":
            r, used, out, _ = oracle.compress_dest_size(b, TARGET, ACCEL)
            return r, out, used
        if cid == "hc":
            return host_hc(b, cap, HC_LEVEL)
        r, used, out = host_hc_dest(b, TARGET, HCD_LEVEL)
        return r, out, used

    def want(k):
        return [memo((cid, b), lambda: ref(b)) for b in (block_data(oracle, m, k, i) for i, m in enumerate(sizes))]

    def check(res, k):
        d, ret = res["dst"], res["ret"]
        for i, w in enumerate(want(k)):
            r, o = int(ret[i]), i * dst_stride
            assert r == w[0], (cid, k, i, sizes[i], r, w[0])
            assert d[o:o + r].tobytes() == w[1], (cid, k, i)
            if dest:
                assert int(res["consumed"][i]) == w[2], (cid, k, i)
            keep = room[i] if room[i] is not None else r
            assert (d[o + keep:o + dst_stride] == GUARD).all(), ("wrote past its slot's limit", cid, k, i)
        assert (d[n * dst_stride:] == GUARD).all()

    launches = 2 if cid == "parallel-split" and not py else 1
    return Case(("py-" if py else "") + cid, t, var, ("src",), outs, launch, check, launches, want)


# ------------------------------------------------------------------------------------------
# pack cases
# ------------------------------------------------------------------------------------------
PK_N, PK_STRIDE, PK_SRC_STRIDE, PK_BLOCK, PK_LAST = 40, 1001, 1003, 1000, 321


def pack_case(cid, py=False):
    """pack-0 / pack-4 (LZ4B200_pack_blocks with 0- and 4-byte headers), pack-frame (LZ4B200_pack_frame_blocks)"""
    frame = cid == "pack-frame"
    hdr = 4 if cid != "pack-0" else 0
    var = []
    for k in range(3):
        rng = np.random.default_rng(77 + k)
        sizes = rng.integers(0, PK_STRIDE + 1 if not frame else PK_BLOCK + 40, PK_N).astype(np.int32)
        sizes[::9] = 0
        v = {"slots": rng.integers(1, 256, PK_N * PK_STRIDE + 64, dtype=np.uint8), "sizes": sizes}
        if frame:
            v["fsrc"] = rng.integers(1, 256, PK_N * PK_SRC_STRIDE + 64, dtype=np.uint8)
        var.append(v)
    t = {nm: torch.zeros(a.shape, dtype=torch.from_numpy(a[:0]).dtype, device=DEV) for nm, a in var[0].items()}
    t["packed"] = torch.empty(PK_N * (PK_SRC_STRIDE + 4) + 64, dtype=torch.uint8, device=DEV)
    t["off"] = torch.empty(PK_N + 1, dtype=torch.int64, device=DEV)
    outs = {"packed": GUARD} if py else {"packed": GUARD, "off": OFF}

    def launch(s):
        if py:
            _, off = batch.pack_blocks(t["slots"], PK_STRIDE, t["sizes"], header_bytes=hdr, packed=t["packed"], stream=s)
            return {"off": off}
        if frame:
            return ok(lib().LZ4B200_pack_frame_blocks(t["slots"].data_ptr(), PK_STRIDE, t["sizes"].data_ptr(),
                                                      t["fsrc"].data_ptr(), PK_SRC_STRIDE, PK_BLOCK, PK_LAST, PK_N,
                                                      t["packed"].data_ptr(), t["off"].data_ptr(), s.cuda_stream), cid)
        return ok(lib().LZ4B200_pack_blocks(t["slots"].data_ptr(), PK_STRIDE, t["sizes"].data_ptr(), PK_N,
                                            t["packed"].data_ptr(), t["off"].data_ptr(), hdr, s.cuda_stream), cid)

    def check(res, k):
        v = var[k]
        fr = (v["fsrc"].tobytes(), PK_SRC_STRIDE, PK_BLOCK, PK_LAST) if frame else None
        want_off, want = pack_model(v["slots"].tobytes(), PK_STRIDE, v["sizes"], hdr, fr)
        assert (res["off"] == want_off).all(), (cid, k)
        assert res["packed"][:len(want)].tobytes() == want, (cid, k)
        assert (res["packed"][len(want):] == GUARD).all(), (cid, k, "wrote past the stream")

    data = ("slots", "fsrc") if frame else ("slots",)
    return Case(("py-" if py else "") + cid, t, var, data, outs, launch, check, 2)


def make_case(oracle, cid):
    py = cid.startswith("py-")
    base = cid[3:] if py else cid
    if base in DECODE:
        return decode_case(oracle, base, py=py)
    if base in ("phased", "partial", "partial-pb"):
        return decode_case(oracle, "R2", mode=base, py=py)
    if base in COMPRESS:
        return compress_case(oracle, base, py=py)
    return pack_case(base, py=py)


NATIVE = list(DECODE) + ["phased", "partial", "partial-pb"] + list(COMPRESS) + ["pack-0", "pack-4", "pack-frame"]
PY = ["py-R2", "py-partial", "py-partial-pb", "py-compress", "py-parallel-scalar", "py-destSize", "py-hc",
      "py-hc-destSize", "py-pack-4"]


# ------------------------------------------------------------------------------------------
# 1. ordering on a side stream
# ------------------------------------------------------------------------------------------
def warm(case):
    """one call on the current stream first: the first launch of a kernel loads its module, which can hold the host
    until the device is idle, and a delayed call would then run in order whatever stream it used"""
    case.load_tables(0)
    case.arm(0)
    case.launch(torch.cuda.current_stream())
    torch.cuda.synchronize()


def sleep_on(s):
    """about 100 ms of sleep on stream s; returns an event recorded behind it"""
    with torch.cuda.stream(s):
        torch.cuda._sleep(SLEEP_CYCLES)
        slept = torch.cuda.Event()
        slept.record(s)
    return slept


def still_asleep(slept):
    assert not slept.query(), "the sleep ended before the host had enqueued everything: the test proves nothing"


def run_after_sleep(case, k=0):
    """The call on a fresh non-blocking stream behind a ~100 ms sleep, payload and sentinels enqueued on that stream
    after the sleep; checks that the host had finished enqueueing before the stream got past the sleep.  Returns the
    results (device tensors)."""
    warm(case)
    s = torch.cuda.Stream()
    case.load_tables(k)
    case.zero_data()
    torch.cuda.synchronize()
    slept = sleep_on(s)
    with torch.cuda.stream(s):
        case.arm(k)
        res = case.collect(case.launch(s))
    still_asleep(slept)
    s.synchronize()
    case.check(res, k)
    return res


@pytest.mark.parametrize("cid", NATIVE + PY)
def test_call_is_ordered_on_its_stream(oracle, cid):
    run_after_sleep(make_case(oracle, cid))


# ------------------------------------------------------------------------------------------
# 2. a phased decode across streams
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", ["R1", "R2", "R3", "R4", "R6"])
def test_scan_on_one_stream_expand_on_another(oracle, cid):
    """scan on A (behind the sleep), an event, B waits on it and expands with the same workspace"""
    case = decode_case(oracle, cid)
    warm(case)
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    case.load_tables(0)
    case.zero_data()
    torch.cuda.synchronize()
    slept = sleep_on(sa)
    with torch.cuda.stream(sa):
        case.arm(0)
        case.phase(1, sa)
        scanned = torch.cuda.Event()
        scanned.record(sa)
    sb.wait_event(scanned)
    with torch.cuda.stream(sb):
        case.phase(2, sb)
        res = case.collect({})
    still_asleep(slept)
    sb.synchronize()
    case.check(res, 0)


def test_two_workspace_pipeline(oracle):
    """tests/perf/pipeline_probe.py's schedule: scan k + 1 on A while expand k runs on B, two workspaces, a 2 048-block
    batch per step, each step in a different block order into its own output, and every step checked"""
    nb, bs, steps = 2048, 65536, 8
    data = oracle.datagen_mt(nb * bs, 16 << 20, 0.5, 11)
    src = torch.from_numpy(data).to(DEV)
    slots, sizes, stride = batch.compress_blocks(src, bs, 1)
    packed, offs = batch.pack_blocks(slots, stride, sizes)
    offs = offs[:-1].contiguous()
    perms = [torch.roll(torch.arange(nb, device=DEV), 97 * k) for k in range(steps)]
    p_offs = [offs[p].contiguous() for p in perms]
    p_sizes = [sizes[p].contiguous() for p in perms]
    outs = [torch.zeros(nb * bs, dtype=torch.uint8, device=DEV) for _ in range(steps)]
    rets = [torch.full((nb,), RET, dtype=torch.int32, device=DEV) for _ in range(steps)]
    ws_bytes = int(lib().LZ4B200_decompress_workspace_bytes_for(nb, 0, bs))
    ws = [torch.empty(ws_bytes, dtype=torch.uint8, device=DEV) for _ in range(2)]
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    scanned = [torch.cuda.Event() for _ in range(steps)]
    expanded = [torch.cuda.Event() for _ in range(steps)]
    for k in range(steps):
        if k >= 2:
            sa.wait_event(expanded[k - 2])              # workspace k & 1 is free again
        batch.decompress_blocks(packed, p_offs[k], p_sizes[k], bs, out=outs[k], out_sizes=rets[k], workspace=ws[k & 1],
                                stream=sa, phases=1)
        scanned[k].record(sa)
        sb.wait_event(scanned[k])
        batch.decompress_blocks(packed, p_offs[k], p_sizes[k], bs, out=outs[k], out_sizes=rets[k], workspace=ws[k & 1],
                                stream=sb, phases=2)
        expanded[k].record(sb)
    torch.cuda.synchronize()
    for k in range(steps):
        assert bool((rets[k] == bs).all()), k
        assert torch.equal(outs[k].view(nb, bs), src.view(nb, bs)[perms[k]]), k


# ------------------------------------------------------------------------------------------
# 3. four streams at once
# ------------------------------------------------------------------------------------------
MIXES = [["R1", "R2", "partial", "compress"], ["R3", "R4", "parallel-split", "pack-4"],
         ["R6", "partial-pb", "destSize", "pack-frame"], ["hc", "hc-destSize", "parallel-scalar", "pack-0"]]


def test_four_streams_at_once(oracle):
    """Four streams, each with its own workspaces, inputs and outputs, wait on one gate event recorded after a sleep,
    so their kernels start together; every result equals the same call made alone and the reference."""
    cases = [[make_case(oracle, c) for c in mix] for mix in MIXES]
    alone = [[{n: x.cpu() for n, x in run_after_sleep(c).items()} for c in mix] for mix in cases]
    streams = [torch.cuda.Stream() for _ in MIXES]
    for mix in cases:
        for c in mix:
            c.load_tables(0)
            c.zero_data()
    torch.cuda.synchronize()
    gate = sleep_on(torch.cuda.Stream())
    results = []
    for s, mix in zip(streams, cases):
        s.wait_event(gate)
        with torch.cuda.stream(s):
            for c in mix:
                c.arm(0)
            results.append([c.collect(c.launch(s)) for c in mix])
    still_asleep(gate)
    torch.cuda.synchronize()
    for mix, got, ref in zip(cases, results, alone):
        for c, g, a in zip(mix, got, ref):
            c.check(g, 0)
            for n in a:
                assert torch.equal(g[n].cpu(), a[n]), (c.name, n, "differs from the call made alone")


# ------------------------------------------------------------------------------------------
# 4. host threads
# ------------------------------------------------------------------------------------------
def child(mode, env=None):
    p = subprocess.run([sys.executable, os.path.abspath(__file__), mode], env=dict(os.environ, **(env or {})),
                       timeout=900, capture_output=True, text=True, cwd=ROOT)
    assert p.returncode == 0 and p.stdout.strip().endswith("ok"), (p.stdout[-3000:], p.stderr[-5000:])


def test_drop_in_and_host_calls_from_threads():
    """8 threads loop over the drop-in calls while one runs the host-buffer batch calls over several 1 MiB chunks and
    one compresses and decodes frames of 64 KB blocks (a child process: the chunk size is read once per process)"""
    child("dropin-threads", {"LZ4B200_HOST_CHUNK_MB": "1"})


def test_device_calls_from_threads_first_calls_of_the_process():
    """4 threads, each on its own stream, make the first device-pointer calls of a process: they race through the decode
    setup and the parallel compressor's one-time attribute, then check every result"""
    child("device-threads")


def _dropin_threads():
    from oracle.pyoracle import Oracle
    L = lib()
    orc = Oracle()
    errors = []
    blocks = [orc.datagen(m, p, 40 + i).tobytes() for i, (m, p) in
              enumerate([(0, .5), (13, .5), (100, .5), (5000, .2), (65536, .5), (65536, .9), (70000, .5)])]
    comp = [orc.compress(b, 1)[1] for b in blocks]
    comp.append(comp[4][:len(comp[4]) // 2])                     # a truncated block: a negative return value
    decomp_want = [orc.decompress(c, 70000) for c in comp]
    partial_want = [orc.decompress_partial(c, 3000) for c in comp]

    def dropin(tid):
        try:
            st = np.zeros(16416 // 8, dtype=np.uint64)
            for it in range(6):
                for i, b in enumerate(blocks):
                    src = np.frombuffer(b, np.uint8) if b else np.zeros(1, np.uint8)
                    cap = bound(len(b))
                    dst = np.zeros(cap + 64, dtype=np.uint8)
                    for name, fn, accel in (("default", lambda: L.LZ4_compress_default(src.ctypes.data, dst.ctypes.data,
                                                                                       len(b), cap), 1),
                                            ("fast", lambda: L.LZ4_compress_fast(src.ctypes.data, dst.ctypes.data, len(b),
                                                                                 cap, 3), 3),
                                            ("extState", lambda: L.LZ4_compress_fast_extState(
                                                st.ctypes.data, src.ctypes.data, dst.ctypes.data, len(b), cap, 2), 2)):
                        r = fn()
                        w = memo(("c", b, accel), lambda: orc.compress(b, accel, cap))
                        if (r, dst[:max(r, 0)].tobytes()) != w:
                            errors.append((tid, name, i))
                    for accel in (None, 2):
                        n = C.c_int(len(b))
                        dst[:] = 0
                        r = (L.LZ4_compress_destSize(src.ctypes.data, dst.ctypes.data, C.byref(n), 3000) if accel is None
                             else L.LZ4_compress_destSize_extState(st.ctypes.data, src.ctypes.data, dst.ctypes.data,
                                                                   C.byref(n), 3000, accel))
                        w = memo(("d", b, accel), lambda: orc.compress_dest_size(b, 3000, accel))
                        if (r, n.value, dst[:max(r, 0)].tobytes()) != w[:3]:
                            errors.append((tid, "destSize", accel, i))
                for i, c in enumerate(comp):
                    src = np.frombuffer(c, np.uint8)
                    dst = np.zeros(70000, dtype=np.uint8)
                    r = L.LZ4_decompress_safe(src.ctypes.data, dst.ctypes.data, len(c), 70000)
                    if (r, dst[:max(r, 0)].tobytes()) != decomp_want[i]:
                        errors.append((tid, "decompress_safe", i))
                    r = L.LZ4_decompress_safe_usingDict(src.ctypes.data, dst.ctypes.data, len(c), 70000, None, 0)
                    if (r, dst[:max(r, 0)].tobytes()) != decomp_want[i]:
                        errors.append((tid, "usingDict", i))
                    r = L.LZ4_decompress_safe_partial(src.ctypes.data, dst.ctypes.data, len(c), 3000, 3000)
                    if (r, dst[:max(r, 0)].tobytes()) != partial_want[i]:
                        errors.append((tid, "partial", i))
        except Exception as e:                                   # noqa: BLE001 -- reported below
            errors.append((tid, repr(e)))

    def host_batch():
        try:
            nb, bs = 150, 65536
            data = orc.datagen_mt(nb * bs, 4 << 20, 0.5, 9)
            cap = bound(bs)
            stride = (cap + 15) // 16 * 16
            for it in range(2):
                slots = np.zeros(nb * stride, dtype=np.uint8)
                sizes = np.full(nb, -7, dtype=np.int32)
                rc = L.LZ4B200_compress_blocks_host(data.ctypes.data, bs, bs, bs, slots.ctypes.data, stride, cap, 1,
                                                    sizes.ctypes.data, nb)
                blocks = [slots[i * stride:i * stride + int(sizes[i])].tobytes() for i in range(nb)]
                for i in range(0, nb, 7):
                    if (int(sizes[i]), blocks[i]) != memo(("h", i), lambda: orc.compress(data[i * bs:(i + 1) * bs], 1)):
                        errors.append(("host compress", it, i))
                buf, offs, bsz = pack_host_blocks(blocks)
                out = np.zeros(nb * bs, dtype=np.uint8)
                rets = np.zeros(nb, dtype=np.int32)
                rc2 = L.LZ4B200_decompress_blocks_host(buf.ctypes.data, offs.ctypes.data, bsz.ctypes.data, out.ctypes.data,
                                                       bs, bs, rets.ctypes.data, nb)
                if rc or rc2 or not (rets == bs).all() or not np.array_equal(out, data):
                    errors.append(("host decompress", it, rc, rc2))
        except Exception as e:                                   # noqa: BLE001
            errors.append(("host", repr(e)))

    def frames():
        try:
            d = orc.datagen_mt(3 << 20, 1 << 20, 0.5, 21)
            want = frame_oracle.compress_frame(orc, d, 4, 0, True)
            cap = int(L.LZ4B200_compressFrameBound(len(d), 4))
            for it in range(3):
                dst = np.zeros(cap, dtype=np.uint8)
                r = int(L.LZ4B200_compressFrame_host(d.ctypes.data, len(d), dst.ctypes.data, cap, 4, 0, 1))
                if dst[:max(r, 0)].tobytes() != want:
                    errors.append(("frame compress", it, r))
                back = np.zeros(len(d), dtype=np.uint8)
                used = C.c_int64(0)
                r = int(L.LZ4B200_decompressFrame_host(dst.ctypes.data, len(want), back.ctypes.data, len(d), C.byref(used)))
                if r != len(d) or used.value != len(want) or not np.array_equal(back, d):
                    errors.append(("frame decompress", it, r))
        except Exception as e:                                   # noqa: BLE001
            errors.append(("frame", repr(e)))

    ths = [threading.Thread(target=dropin, args=(i,)) for i in range(8)]
    ths += [threading.Thread(target=host_batch), threading.Thread(target=frames)]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors, errors[:20]
    assert L.LZ4B200_last_cuda_error() == b"", L.LZ4B200_last_cuda_error()


THREAD_MIXES = [["parallel-scalar", "R2", "hc"], ["parallel-split", "R4", "pack-4"], ["R1", "destSize", "pack-0"],
                ["partial-pb", "compress", "hc-destSize", "pack-frame"]]


def _device_threads():
    from oracle.pyoracle import Oracle
    orc = Oracle()
    cases = [[make_case(orc, c) for c in mix] for mix in THREAD_MIXES]
    for mix in cases:                                       # the references first: the threads only call and compare
        for c in mix:
            for k in range(3):
                c.want(k)
                c.dev(k)
    torch.cuda.synchronize()
    errors = []
    go = threading.Barrier(len(cases))

    def run(mix):
        try:
            s = torch.cuda.Stream()
            go.wait()
            for k in (0, 1, 2):
                with torch.cuda.stream(s):
                    for c in mix:
                        c.load_tables(k)
                        c.arm(k)
                    res = [c.collect(c.launch(s)) for c in mix]
                s.synchronize()
                for c, r in zip(mix, res):
                    c.check(r, k)
        except Exception as e:                              # noqa: BLE001
            errors.append(repr(e)[:500])

    ths = [threading.Thread(target=run, args=(m,)) for m in cases]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors, errors


# ------------------------------------------------------------------------------------------
# 5. graph capture
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", NATIVE + PY)
def test_captured_call_replays_on_new_payloads(oracle, cid):
    """Warm up, capture the call on a side stream, then replay it three times with other payloads (and tables) copied
    into the static inputs.  LZ4B200_launch_count counts the launches the library issues: the capture counts as one
    call, a replay issues nothing through the library and leaves the counter alone."""
    case = make_case(oracle, cid)
    run_after_sleep(case)
    s = torch.cuda.Stream()
    case.load_tables(0)
    case.arm(0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    l0 = lib().LZ4B200_launch_count()
    with torch.cuda.graph(g, stream=s):
        extra = case.launch(s)
    assert lib().LZ4B200_launch_count() == l0 + case.launches
    l1 = lib().LZ4B200_launch_count()
    for k in (1, 2, 0):
        case.load_tables(k)
        case.arm(k)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        case.check(case.collect(extra), k)
    assert lib().LZ4B200_launch_count() == l1


def test_first_library_call_of_a_process_is_captured():
    """The one-time setup (the decode kernels' shared-memory opt-in, the parallel compressor's) runs inside a capture
    when the process's first calls are captured"""
    child("first-call-captured")


def _first_call_captured():
    from oracle.pyoracle import Oracle
    orc = Oracle()
    cases = [make_case(orc, c) for c in ("R2", "parallel-scalar", "hc", "R5")]
    for c in cases:
        c.load_tables(1)
        c.arm(1)
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        extras = [c.launch(s) for c in cases]
    for k in (1, 0):
        for c in cases:
            c.load_tables(k)
            c.arm(k)
        torch.cuda.synchronize()
        g.replay()
        torch.cuda.synchronize()
        for c, x in zip(cases, extras):
            c.check(c.collect(x), k)


# ------------------------------------------------------------------------------------------
# 6. the launch counter under threads
# ------------------------------------------------------------------------------------------
def test_launch_count_under_threads():
    """8 threads x 150 iterations of one compress (1 launch) and one pack (2 launches), each thread on its own stream
    and buffers: the counter moves by exactly 3 600.  A counter that loses increments fails this only when the race
    happens, so a pass does not prove the counter correct; a failure proves it wrong."""
    L = lib()
    threads, iters = 8, 150
    per = []
    for i in range(threads):
        src = torch.randint(0, 4, (16 + 4 * 1000 + 16,), dtype=torch.uint8, device=DEV)
        per.append({"src": src, "dst": torch.zeros(4 * 1040, dtype=torch.uint8, device=DEV),
                    "ret": torch.zeros(4, dtype=torch.int32, device=DEV),
                    "packed": torch.zeros(4 * 1044 + 16, dtype=torch.uint8, device=DEV),
                    "off": torch.zeros(5, dtype=torch.int64, device=DEV)})
    torch.cuda.synchronize()
    errors = []
    go = threading.Barrier(threads)

    def run(t):
        try:
            s = torch.cuda.Stream()
            go.wait()
            for _ in range(iters):
                rc = L.LZ4B200_compress_blocks(t["src"].data_ptr() + 16, 1000, None, 1000, t["dst"].data_ptr(), 1040,
                                               1040, 1, t["ret"].data_ptr(), 4, s.cuda_stream)
                rc |= L.LZ4B200_pack_blocks(t["dst"].data_ptr(), 1040, t["ret"].data_ptr(), 4, t["packed"].data_ptr(),
                                            t["off"].data_ptr(), 4, s.cuda_stream)
                if rc:
                    errors.append(rc)
            s.synchronize()
        except Exception as e:                              # noqa: BLE001
            errors.append(repr(e))

    l0 = L.LZ4B200_launch_count()
    ths = [threading.Thread(target=run, args=(t,)) for t in per]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors, errors[:5]
    assert L.LZ4B200_launch_count() - l0 == threads * iters * 3


if __name__ == "__main__":
    {"dropin-threads": _dropin_threads, "device-threads": _device_threads,
     "first-call-captured": _first_call_captured}[sys.argv[1]]()
    print("ok")
