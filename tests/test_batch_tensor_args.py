"""The tensor arguments of every lz4_b200.batch wrapper: what the kernels would misread or write past is refused before
anything runs, and every layout the wrappers accept gives the oracle's result.

The wrappers hand data_ptr() and numel() to the C calls.  A float32 source, a strided view, a CPU tensor, an output one
element short, slots closer than their capacity, or an int that ctypes would cut to 32 bits would make the kernels read
the wrong bytes or write past the tensor into whatever the caching allocator placed next to it.  So:
  - rejections: one table row per (wrapper, argument, defect), run against a stand-in of the library that records every
    call (gpu_util.Recorder).  Each row must raise ValueError with no call recorded: a deficient tensor never reaches
    the kernels, here or anywhere;
  - accepted layouts, through the real library: views at odd storage offsets, 2-D contiguous byte tensors, odd strides,
    n = 0, n = 1, a 1-byte last block, blocks above 64 KB, and every given output cut at exactly its minimum size from a
    larger arena of guard values whose remainder must stay intact;
  - two devices (skipped below two GPUs): tensors on cuda:1 with cuda:0 current run on cuda:1."""
import numpy as np
import pytest
import torch

import frame_oracle as fo
from gpu_util import GUARD, Recorder, compress_call, pack_model
from hc_emul import host_hc, host_hc_dest, host_hc_opt, host_hc_opt_dest
from lz4_b200 import _lib, batch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
N = 3                                   # blocks of every call in the rejection table
UNSET = -7                              # what an int output holds where the call must not write


@pytest.fixture
def rec(monkeypatch):
    r = Recorder(_lib.load())
    monkeypatch.setattr(_lib, "load", lambda: r)
    monkeypatch.setattr(batch, "_workspaces", {})
    return r


# ------------------------------------------------------------------------------------------
# the rejection table
# ------------------------------------------------------------------------------------------
def z(n, dtype=torch.uint8, dev=DEV):
    return torch.zeros(n, dtype=dtype, device=dev)


def good_call(name, dev=DEV):
    """(wrapper, keyword arguments): a call over N blocks that passes every check, with every output given at exactly
    the size the call needs"""
    lib = _lib.load()
    i32, i64 = torch.int32, torch.int64
    if name.startswith("decompress_blocks"):
        kw = dict(comp=z(64, dev=dev), offsets=z(N, i64, dev), sizes=torch.full((N,), 16, dtype=i32, device=dev),
                  out_sizes=z(N, i32, dev))
        if name == "decompress_blocks":
            kw.update(block_capacity=1000, out_stride=1001, out=z(2 * 1001 + 1000, dev=dev),
                      workspace=z(int(lib.LZ4B200_decompress_workspace_bytes_for(N, 0, 1000)), dev=dev))
            return batch.decompress_blocks, kw
        if name == "decompress_blocks_partial":
            kw.update(target=500, out_stride=501, out=z(2 * 501 + 500, dev=dev),
                      workspace=z(int(lib.LZ4B200_decompress_workspace_bytes_for(N, 0, 500)), dev=dev))
        else:                                                           # per-block targets: slots of out_stride bytes
            kw.update(target=torch.full((N,), 400, dtype=i32, device=dev), out_stride=600, out=z(N * 600, dev=dev),
                      workspace=z(int(lib.LZ4B200_decompress_workspace_bytes_for(N, 1, 0)), dev=dev))
        return batch.decompress_blocks_partial, kw
    if name.startswith("decompress_frames"):
        mb = [1, 1, 1, 1]
        kw = dict(comp=z(64, dev=dev), offsets=z(N, i64, dev), sizes=torch.full((N,), 16, dtype=i64, device=dev),
                  capacities=torch.full((N,), 10, dtype=i64, device=dev), max_blocks=mb, out=z(30, dev=dev),
                  out_offsets=z(N, i64, dev), results=z(N, i64, dev), consumed=z(N, i64, dev),
                  workspace=z(batch.decompress_frames_workspace_bytes(N, mb), dev=dev))
        return getattr(batch, name), kw
    if name == "pack_blocks":
        return batch.pack_blocks, dict(slots=z(N * 1001, dev=dev), slot_stride=1001, sizes=z(N, i32, dev),
                                       header_bytes=4, packed=z(N * 1005, dev=dev))
    # the compress calls: N blocks of 1 000 bytes, the last one 993
    kw = dict(src=z(N * 1000 - 7, dev=dev), block_size=1000, out_sizes=z(N, i32, dev))
    dest = name.endswith("dest_size")
    if dest:
        kw.update(target=700, slot_stride=701, slots=z(2 * 701 + 700, dev=dev), consumed=z(N, i32, dev),
                  src_sizes=torch.tensor([1000, 1000, 993], dtype=i32, device=dev))
    else:
        kw.update(slot_capacity=1100, slot_stride=1101, slots=z(2 * 1101 + 1100, dev=dev))
    if name.startswith("compress_blocks_hc_opt"):
        kw.update(level=12, workspace=z(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(N)), dev=dev))
    elif name.startswith("compress_blocks_hc"):
        kw.update(level=9, workspace=z(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(N)), dev=dev))
    else:
        kw.update(acceleration=1)
    if name in ("compress_blocks", "compress_blocks parallel"):
        kw.update(src_sizes=torch.tensor([1000, 1000, 993], dtype=i32, device=dev),
                  mode="exact" if name == "compress_blocks" else "parallel")
        return batch.compress_blocks, kw
    return getattr(batch, name), kw


WRAPPERS = ["decompress_blocks", "decompress_blocks_partial", "decompress_blocks_partial per-block", "decompress_frames",
            "decompress_frames_checksummed", "compress_blocks", "compress_blocks parallel", "compress_blocks_dest_size",
            "compress_blocks_hc", "compress_blocks_hc_dest_size", "compress_blocks_hc_opt",
            "compress_blocks_hc_opt_dest_size", "pack_blocks"]
ENTRY = {"decompress_blocks": "LZ4B200_decompress_blocks_phased",
         "decompress_blocks_partial": "LZ4B200_decompress_blocks_partial",
         "decompress_blocks_partial per-block": "LZ4B200_decompress_blocks_partial",
         "decompress_frames": "LZ4B200_decompress_frames",
         "decompress_frames_checksummed": "LZ4B200_decompress_frames_checksummed",
         "compress_blocks": "LZ4B200_compress_blocks", "compress_blocks parallel": "LZ4B200_compress_blocks_parallel",
         "compress_blocks_dest_size": "LZ4B200_compress_blocks_destSize",
         "compress_blocks_hc": "LZ4B200_compress_blocks_hc",
         "compress_blocks_hc_dest_size": "LZ4B200_compress_blocks_hc_destSize",
         "compress_blocks_hc_opt": "LZ4B200_compress_blocks_hc_opt",
         "compress_blocks_hc_opt_dest_size": "LZ4B200_compress_blocks_hc_opt_destSize",
         "pack_blocks": "LZ4B200_pack_blocks"}

# every tensor argument of good_call's calls
TENSORS = {"decompress_blocks": ["comp", "offsets", "sizes", "out_sizes", "out", "workspace"],
           "decompress_blocks_partial": ["comp", "offsets", "sizes", "out_sizes", "out", "workspace"],
           "decompress_blocks_partial per-block": ["comp", "offsets", "sizes", "out_sizes", "target", "out",
                                                   "workspace"],
           "compress_blocks": ["src", "out_sizes", "slots", "src_sizes"],
           "compress_blocks_dest_size": ["src", "out_sizes", "slots", "consumed", "src_sizes"],
           "compress_blocks_hc": ["src", "out_sizes", "slots", "workspace"],
           "pack_blocks": ["slots", "sizes", "packed"]}
TENSORS["compress_blocks parallel"] = TENSORS["compress_blocks"]
TENSORS["compress_blocks_hc_opt"] = TENSORS["compress_blocks_hc"]
TENSORS["compress_blocks_hc_dest_size"] = TENSORS["compress_blocks_hc_opt_dest_size"] = \
    TENSORS["compress_blocks_dest_size"][:-1] + ["src_sizes", "workspace"]
TENSORS["decompress_frames"] = TENSORS["decompress_frames_checksummed"] = [
    "comp", "offsets", "sizes", "capacities", "out", "out_offsets", "results", "consumed", "workspace"]

# the arguments whose element count the call reads or writes (the others only need the right dtype and layout), and
# those whose count must be exact
SIZED = {"offsets", "out", "out_sizes", "workspace", "capacities", "out_offsets", "results", "consumed", "src_sizes",
         "slots", "packed", "target"}
EXACT = {"capacities", "src_sizes", "target"}
UNSIZED = {("decompress_frames", "out"), ("decompress_frames_checksummed", "out"), ("pack_blocks", "slots")}
LAYOUT = {"out", "out_stride", "slots", "slot_stride", "packed", "workspace"}     # (pack_blocks needs its slots)
WRONG_DTYPE = {torch.uint8: torch.float32, torch.int32: torch.int64, torch.int64: torch.int32}


def stride_defect(name):
    """(stride argument, the value one below what its slots hold)"""
    if name.startswith("decompress_blocks_partial"):
        return ("out_stride", 499) if name == "decompress_blocks_partial" else None
    if name == "decompress_blocks":
        return "out_stride", 999
    if name.startswith("compress"):
        return "slot_stride", 699 if name.endswith("dest_size") else 1099
    return None


def int_defects(name):
    """(argument, value) pairs outside what the C call takes"""
    out = []
    if name.startswith("compress"):
        out += [("block_size", 0), ("block_size", -1), ("block_size", 2 ** 31), ("block_size", 2 ** 32 + 1000)]
        cap = "target" if name.endswith("dest_size") else "slot_capacity"
        out += [(cap, 2 ** 31), (cap, 2 ** 32 + 1100)]
        out += [("level" if "_hc" in name else "acceleration", 2 ** 32 + 1)]
    if name == "decompress_blocks":
        out += [("block_capacity", 2 ** 31), ("block_capacity", 2 ** 32 + 1000)]
    if name == "decompress_blocks_partial":
        out += [("target", 2 ** 31), ("target", 2 ** 32 + 500)]
    if name == "pack_blocks":
        out += [("header_bytes", 2 ** 32 + 4)]
    return out


def defects():
    """every (wrapper, argument, defect) row"""
    rows = []
    for name in WRAPPERS:
        for arg in TENSORS[name]:
            rows += [(name, arg, d) for d in ("dtype", "strided", "cpu")]
            if arg in SIZED and (name, arg) not in UNSIZED:
                rows.append((name, arg, "short"))
                if arg in EXACT:
                    rows.append((name, arg, "long"))
        if stride_defect(name):
            rows.append((name, stride_defect(name)[0], "stride"))
        rows += [(name, arg, "value %d" % v) for arg, v in int_defects(name)]
    return rows


@pytest.mark.parametrize("name", WRAPPERS)
def test_the_table_starts_from_calls_that_pass(rec, name):
    """every row changes one argument of a call that goes through: with nothing changed, it reaches the library once"""
    fn, kw = good_call(name)
    assert sorted(a for a, v in kw.items() if isinstance(v, torch.Tensor)) == sorted(TENSORS[name])
    fn(**kw)
    assert [c[0] for c in rec.calls] == [ENTRY[name]] and rec.devices == [0]


ROWS = defects()


@pytest.mark.parametrize("name,arg,defect", ROWS, ids=["%s-%s-%s" % r for r in ROWS])
def test_a_deficient_argument_raises_before_any_launch(rec, name, arg, defect):
    fn, kw = good_call(name)
    if defect == "stride":
        kw[arg] = stride_defect(name)[1]
    else:
        v = kw[arg]
        if defect == "dtype":
            kw[arg] = torch.zeros(v.shape, dtype=WRONG_DTYPE[v.dtype], device=v.device)
        elif defect == "strided":
            kw[arg] = torch.zeros(v.numel() * 2, dtype=v.dtype, device=v.device)[::2]
        elif defect == "cpu":
            kw[arg] = v.cpu()
        elif defect == "short":
            kw[arg] = v[:-1]
        elif defect == "long":
            kw[arg] = torch.zeros(v.numel() + 1, dtype=v.dtype, device=v.device)
        else:                                   # an int: without the outputs and strides it would also overrun
            kw = {a: v for a, v in kw.items() if a not in LAYOUT or name == "pack_blocks" and a != "packed"}
            kw[arg] = int(defect.split()[1])
    with pytest.raises(ValueError):
        fn(**kw)
    assert rec.calls == [], "%s reached the library with %s %s" % (name, arg, defect)


def test_a_2d_byte_tensor_counts_all_its_bytes(rec):
    """a contiguous (3, 1000) source is 3 000 bytes, 3 blocks: not 3 bytes, and a float32 one is refused"""
    src = z(3000).view(3, 1000)
    batch.compress_blocks(src, 1000)
    (name, args), = rec.calls
    assert args[0] == src.data_ptr() and args[9] == 3
    with pytest.raises(ValueError):
        batch.compress_blocks(z(750, torch.float32), 1000)
    assert len(rec.calls) == 1


def test_checks_make_no_host_sync(rec):
    """the checks read shapes, dtypes and devices only: every wrapper with its sizes given runs under sync debug mode
    "error", which raises on any synchronising torch op"""
    calls = [good_call(name) for name in WRAPPERS]
    for _, kw in calls:
        if "src" in kw:
            kw["src"] = z(N * 1000)             # whole blocks: the HC calls would build per-block sizes otherwise
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for fn, kw in calls:
            fn(**kw)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert len(rec.calls) == len(WRAPPERS)


# ------------------------------------------------------------------------------------------
# accepted layouts, through the real library
# ------------------------------------------------------------------------------------------
class Arena:
    """a tensor of `fill` values with a view of `count` elements at element `lead` (odd: an odd data_ptr for bytes);
    .intact() checks that nothing outside the view changed"""

    def __init__(self, count, dtype=torch.uint8, fill=GUARD, lead=3, tail=61):
        self.base = torch.full((lead + count + tail,), fill, dtype=dtype, device=DEV)
        self.view, self.lead, self.count, self.fill = self.base[lead:lead + count], lead, count, fill

    def intact(self):
        b = self.base.cpu().numpy()
        return (b[:self.lead] == self.fill).all() and (b[self.lead + self.count:] == self.fill).all()


def device_bytes(data, lead=5, cols=None):
    """data as a byte view at an odd offset of a larger tensor; cols: as a contiguous 2-D (-1, cols) view"""
    a = Arena(len(data), lead=lead, fill=0)
    if len(data):
        a.view.copy_(torch.from_numpy(np.frombuffer(bytes(data), dtype=np.uint8).copy()).to(DEV))
    return a.view.view(-1, cols) if cols else a.view


def device_ints(values, dtype, lead=1):
    a = Arena(len(values), dtype=dtype, lead=lead, fill=0)
    if len(values):
        a.view.copy_(torch.tensor(list(values), dtype=dtype))
    return a.view


def cols_of(nbytes):
    """a row length for a contiguous 2-D view of nbytes: its largest divisor up to 64 (1 when it has none)"""
    return max([d for d in range(1, 65) if nbytes % d == 0], default=1) if nbytes else None


def blocks_of(data, bs):
    return [data[i:i + bs] for i in range(0, len(data), bs)]


# (n, block size, last block's size): none, one, a 1-byte last block of odd blocks, and blocks above 64 KB
SHAPES = [(0, 4099, 0), (1, 4099, 4099), (5, 4099, 1), (4, 1027, 514), (3, 70001, 70001), (2, 200003, 17)]


def source(oracle, n, bs, last, seed=0):
    return oracle.datagen((n - 1) * bs + last, 0.5, seed).tobytes() if n else b""


def compressed(oracle, data, bs):
    """(comp bytes, offsets, sizes) of data's blocks, compressed by the oracle, with 16 readable bytes after the last"""
    blocks = [oracle.compress(b, 1)[1] for b in blocks_of(data, bs)]
    offs = np.cumsum([0] + [len(b) for b in blocks])[:-1].tolist()
    return b"".join(blocks) + b"\0" * 16, offs, [len(b) for b in blocks]


@pytest.mark.parametrize("n,bs,last", SHAPES)
def test_decode_at_odd_offsets_and_exact_sizes(oracle, n, bs, last):
    data = source(oracle, n, bs, last, seed=n)
    comp, offs, sizes = compressed(oracle, data, bs)
    blocks = blocks_of(data, bs)
    stride = bs + (2 if bs % 2 else 3)                          # odd
    out = Arena((n - 1) * stride + bs if n else 0)
    rets = Arena(n, torch.int32, fill=UNSET)
    c2d = device_bytes(comp, cols=cols_of(len(comp)))                # 2-D, contiguous
    got_out, got_rets = batch.decompress_blocks(c2d, device_ints(offs, torch.int64), device_ints(sizes, torch.int32),
                                                bs, out=out.view, out_stride=stride, out_sizes=rets.view)
    torch.cuda.synchronize()
    assert got_out.data_ptr() == out.view.data_ptr() and got_rets.data_ptr() == rets.view.data_ptr()
    assert out.intact() and rets.intact()
    o, r = out.view.cpu().numpy(), rets.view.cpu().tolist()
    for i, b in enumerate(blocks):
        c = comp[offs[i]:offs[i] + sizes[i]]
        want = oracle.decompress(c, bs)
        assert (r[i], o[i * stride:i * stride + r[i]].tobytes()) == want == (len(b), bytes(b)), i
        end = (i + 1) * stride if i < n - 1 else len(o)
        assert (o[i * stride + r[i]:end] == GUARD).all(), "block %d wrote past its %d bytes" % (i, r[i])


@pytest.mark.parametrize("n,bs,last", SHAPES[:4])
@pytest.mark.parametrize("per_block", [False, True])
def test_partial_decode_at_odd_offsets_and_exact_sizes(oracle, n, bs, last, per_block):
    data = source(oracle, n, bs, last, seed=10 + n)
    comp, offs, sizes = compressed(oracle, data, bs)
    rng = np.random.default_rng(n)
    targets = [int(t) for t in rng.integers(0, bs + 1, n)] if per_block else [bs // 2 + 1] * n
    stride = (max(targets, default=bs // 2 + 1) + 1) | 1
    need = n * stride if per_block else ((n - 1) * stride + bs // 2 + 1 if n else 0)
    out = Arena(need)
    rets = Arena(n, torch.int32, fill=UNSET)
    target = device_ints(targets, torch.int32) if per_block else bs // 2 + 1
    batch.decompress_blocks_partial(device_bytes(comp), device_ints(offs, torch.int64), device_ints(sizes, torch.int32),
                                    target, out=out.view, out_stride=stride, out_sizes=rets.view)
    torch.cuda.synchronize()
    assert out.intact() and rets.intact()
    o, r = out.view.cpu().numpy(), rets.view.cpu().tolist()
    for i in range(n):
        want = oracle.decompress_partial(comp[offs[i]:offs[i] + sizes[i]], targets[i])
        assert (r[i], o[i * stride:i * stride + max(r[i], 0)].tobytes()) == want, i
        assert (o[i * stride + max(r[i], 0):min((i + 1) * stride, len(o))] == GUARD).all(), i


@pytest.mark.parametrize("checksummed", [False, True])
@pytest.mark.parametrize("n", [0, 1, 4])
def test_frames_at_odd_offsets_and_exact_sizes(oracle, checksummed, n):
    """frames of 1 byte to 300 KB (several block sizes), every output given at exactly the size the call needs"""
    lens = [1, 300001, 65536, 4099][:n]
    contents = [oracle.datagen(k, 0.5, 20 + i).tobytes() for i, k in enumerate(lens)]
    frames = [fo.compress_frame(oracle, d, 4 + i % 4) for i, d in enumerate(contents)]
    buf, offs = b"\0" * 16, []
    for f in frames:
        offs.append(len(buf))
        buf += f + b"\0" * 3
    buf += b"\0" * 16
    caps = [len(d) for d in contents]
    out = Arena(sum(caps))
    out_offs = np.cumsum([0] + caps)[:-1].tolist()
    results = Arena(n, torch.int64, fill=UNSET)
    consumed = Arena(n, torch.int64, fill=UNSET)
    fn = batch.decompress_frames_checksummed if checksummed else batch.decompress_frames
    fn(device_bytes(buf, lead=7), device_ints(offs, torch.int64), device_ints([len(f) for f in frames], torch.int64),
       device_ints(caps, torch.int64), [4, 4, 4, 4], out=out.view, out_offsets=device_ints(out_offs, torch.int64),
       results=results.view, consumed=consumed.view)
    torch.cuda.synchronize()
    assert out.intact() and results.intact() and consumed.intact()
    o = out.view.cpu().numpy()
    for i, f in enumerate(frames):
        back, used = fo.decompress_frame(oracle, f)
        assert back == contents[i]
        assert results.view[i].item() == len(back) and consumed.view[i].item() == used, i
        assert o[out_offs[i]:out_offs[i] + caps[i]].tobytes() == back, i


COMPRESS = ["exact", "dest_size", "hc", "hc_dest_size", "hc_opt", "hc_opt_dest_size"]


def expected(oracle, kind, block, cap, target, level):
    """(ret, consumed or None, bytes) of one block from the oracle (exact, destSize) or the host build (HC)"""
    if kind == "dest_size":
        r, k, c, _ = oracle.compress_dest_size(block, target, 1)
        return r, k, c
    if kind.endswith("dest_size"):
        return (host_hc_dest if kind == "hc_dest_size" else host_hc_opt_dest)(block, target, level)
    r, c = oracle.compress(block, 1, cap) if kind == "exact" else (host_hc if kind == "hc" else host_hc_opt)(block, cap,
                                                                                                           level)
    return r, None, c


@pytest.mark.parametrize("n,bs,last", SHAPES[:4] + [(2, 70001, 3)])
@pytest.mark.parametrize("kind", COMPRESS)
def test_compress_at_odd_offsets_and_exact_sizes(oracle, kind, n, bs, last):
    """every given output at exactly its minimum size; with n = 0 the outputs are the wrapper's (the C calls refuse
    the null pointer of an empty tensor)"""
    if kind.startswith("hc_opt") and bs > 5000:
        pytest.skip("one thread parses a block at level 12: the large blocks are the hash-chain calls' cases")
    data = source(oracle, n, bs, last, seed=30 + n)
    blocks = blocks_of(data, bs)
    dest = kind.endswith("dest_size")
    level = 12 if kind.startswith("hc_opt") else 9
    target = bs // 3 + 1
    cap = batch.compress_bound(bs)
    room = max(min(target, cap), 1) if dest else cap
    stride = room + (1 if room % 2 == 0 else 2)                 # odd
    slots = Arena(n and (n - 1) * stride + room)
    sizes = Arena(n, torch.int32, fill=UNSET)
    cons = Arena(n, torch.int32, fill=UNSET)
    src = device_bytes(data, cols=cols_of(len(data)))
    kw = dict(slots=slots.view, slot_stride=stride, out_sizes=sizes.view) if n else dict(slot_stride=stride)
    if dest and n:
        kw["consumed"] = cons.view
    if kind == "exact":
        res = batch.compress_blocks(src, bs, 1, slot_capacity=cap, **kw)
    elif kind == "dest_size":
        res = batch.compress_blocks_dest_size(src, bs, target, 1, **kw)
    elif kind in ("hc", "hc_opt"):
        res = getattr(batch, "compress_blocks_" + kind)(src, bs, level, slot_capacity=cap, **kw)
    else:
        res = getattr(batch, "compress_blocks_" + kind)(src, bs, target, level, **kw)
    torch.cuda.synchronize()
    assert res[-1] == stride and res[1].numel() == n and (res[0].data_ptr() == slots.view.data_ptr() or not n)
    assert slots.intact() and sizes.intact() and cons.intact()
    s, r, k = slots.view.cpu().numpy(), sizes.view.cpu().tolist(), cons.view.cpu().tolist()
    for i, b in enumerate(blocks):
        want = expected(oracle, kind, b, cap, target, level)
        assert (r[i], k[i] if dest else None, s[i * stride:i * stride + r[i]].tobytes()) == want, (i, len(b))


@pytest.mark.parametrize("n,bs,last", SHAPES[:4])
def test_parallel_compress_at_odd_offsets_and_exact_sizes(oracle, n, bs, last):
    """the parallel parse: every block decodes to its input, and equals the C call's output on the same blocks"""
    data = source(oracle, n, bs, last, seed=40 + n)
    blocks = blocks_of(data, bs)
    cap = batch.compress_bound(bs)
    stride = cap + (1 if cap % 2 == 0 else 2)
    slots = Arena(n and (n - 1) * stride + cap)
    sizes = Arena(n, torch.int32, fill=UNSET)
    batch.compress_blocks(device_bytes(data, cols=cols_of(len(data))), bs, 1, slots=slots.view,
                          slot_stride=stride, slot_capacity=cap, out_sizes=sizes.view, mode="parallel")
    torch.cuda.synchronize()
    assert slots.intact() and sizes.intact()
    s, r = slots.view.cpu().numpy(), sizes.view.cpu().tolist()
    got = [s[i * stride:i * stride + r[i]].tobytes() for i in range(n)]
    for i, b in enumerate(blocks):
        assert oracle.decompress(got[i], len(b)) == (len(b), bytes(b)), i
    if n:
        rets, direct = compress_call(True, [bytes(b) for b in blocks], cap, 1)
        assert rets.tolist() == r and direct == got


@pytest.mark.parametrize("hdr", [0, 4])
@pytest.mark.parametrize("n", [0, 1, 7])
def test_pack_at_odd_offsets_and_exact_sizes(n, hdr):
    """the gather into a stream of exactly n * (slot_stride + header_bytes) bytes, one slot at a time full"""
    stride = 1001
    rng = np.random.default_rng(n + hdr)
    host_slots = rng.integers(1, 256, n * stride, dtype=np.uint8).tobytes()
    sizes = [int(x) for x in rng.integers(0, stride + 1, n)]
    if n:
        sizes[n // 2] = stride
    packed = Arena(n * (stride + hdr))
    _, offs = batch.pack_blocks(device_bytes(host_slots, cols=stride if n else None), stride,
                                device_ints(sizes, torch.int32), header_bytes=hdr, packed=packed.view)
    torch.cuda.synchronize()
    want_off, want = pack_model(host_slots, stride, sizes, hdr)
    assert offs.cpu().tolist() == want_off.tolist() and packed.intact()
    p = packed.view.cpu().numpy()
    assert p[:len(want)].tobytes() == want and (p[len(want):] == GUARD).all()


# ------------------------------------------------------------------------------------------
# two devices
# ------------------------------------------------------------------------------------------
two_gpus = pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two CUDA devices")


@two_gpus
def test_tensors_on_the_second_device_run_there(oracle):
    """with cuda:0 current, a decode and a compress of tensors on cuda:1 give the oracle's result"""
    data = oracle.datagen(5 * 4099 + 1, 0.5, 50).tobytes()
    comp, offs, sizes = compressed(oracle, data, 4099)
    d1 = "cuda:1"
    with torch.cuda.device(0):
        out, rets = batch.decompress_blocks(torch.from_numpy(np.frombuffer(comp, np.uint8).copy()).to(d1),
                                            torch.tensor(offs, device=d1), torch.tensor(sizes, dtype=torch.int32,
                                                                                        device=d1), 4099)
        slots, csz, stride = batch.compress_blocks(torch.from_numpy(np.frombuffer(data, np.uint8).copy()).to(d1), 4099)
        torch.cuda.synchronize(1)
    assert out.device == slots.device == torch.device(d1)
    o, r = out.cpu().numpy(), rets.cpu().tolist()
    s, c = slots.cpu().numpy(), csz.cpu().tolist()
    for i, b in enumerate(blocks_of(data, 4099)):
        assert (r[i], o[i * 4099:i * 4099 + r[i]].tobytes()) == (len(b), bytes(b))
        assert (c[i], s[i * stride:i * stride + c[i]].tobytes()) == oracle.compress(b, 1)


@two_gpus
def test_calls_run_with_their_tensors_device_current(rec):
    """every wrapper, given cuda:1 tensors while cuda:0 is current, calls the library with cuda:1 current and on
    cuda:1's current stream"""
    with torch.cuda.device(0):
        for name in WRAPPERS:
            fn, kw = good_call(name, dev="cuda:1")
            fn(**kw)
    assert rec.devices == [1] * len(WRAPPERS)
    st1 = torch.cuda.current_stream(1).cuda_stream
    assert all(args[-1] == st1 for _, args in rec.calls)


@two_gpus
@pytest.mark.parametrize("name", WRAPPERS)
def test_mixed_devices_and_a_foreign_stream_raise(rec, name):
    fn, kw = good_call(name, dev="cuda:1")
    first = next(a for a, v in kw.items() if isinstance(v, torch.Tensor))
    mixed = dict(kw, **{first: kw[first].to("cuda:0")})
    with pytest.raises(ValueError):
        fn(**mixed)
    with pytest.raises(ValueError):
        fn(**kw, stream=torch.cuda.Stream(device=0))
    assert rec.calls == []
