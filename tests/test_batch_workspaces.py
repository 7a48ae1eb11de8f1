"""The workspace rule of lz4_b200.batch, pinned with a stand-in of the library that records every call and launches
nothing: the wrappers' choice of workspace, stream and host synchronisation is host logic, and a wrong choice on the
GPU (two overlapping calls on one HC hash table or one mark table) would be a fault rather than a wrong byte.

The rule (batch.py's docstring): a caller's `workspace=` is used as given and must be large enough; a workspace the
module owns is used only on the stream it was allocated on; a phased decode and any call under stream capture bring
their own; no wrapper synchronises with the host when its sizes are given.  The tests allocate device tensors (the
wrappers allocate outputs with torch), so they run with the GPU suite."""
import pytest
import torch

from gpu_util import Recorder
from lz4_b200 import _lib, batch

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
BLOCK = 65536


# where each recorded call keeps its workspace pointer, its size and its stream (positions in the C prototypes)
WS_ARGS = {"LZ4B200_decompress_blocks_phased": (10, 11, 13), "LZ4B200_decompress_blocks_partial": (10, 11, 12),
           "LZ4B200_compress_blocks_hc": (10, 11, 12), "LZ4B200_compress_blocks_hc_destSize": (11, 12, 13)}


def ws_of(call):
    """(range [ptr, ptr + bytes), stream handle) of a recorded call"""
    name, args = call
    p, b, s = WS_ARGS[name]
    return (args[p], args[p] + args[b]), args[s]


@pytest.fixture
def rec(monkeypatch):
    real = _lib.load()
    r = Recorder(real)
    monkeypatch.setattr(_lib, "load", lambda: r)
    monkeypatch.setattr(batch, "_workspaces", {})        # start from an empty cache, leave the real one alone
    return r


def decode_inputs(n):
    comp = torch.zeros(n * 16 + 32, dtype=torch.uint8, device=DEV)
    offs = torch.arange(n, dtype=torch.int64, device=DEV) * 16 + 16
    sizes = torch.full((n,), 16, dtype=torch.int32, device=DEV)
    return comp, offs, sizes


def hc_input(n):
    return torch.zeros(n * BLOCK, dtype=torch.uint8, device=DEV)


# every wrapper that needs a workspace, as f(workspace=..., stream=...) over n blocks
def wrappers(n):
    comp, offs, sizes = decode_inputs(n)
    src = hc_input(n)
    targets = torch.full((n,), 4096, dtype=torch.int32, device=DEV)
    lib = _lib.load()
    return {
        "decompress_blocks": (lambda **k: batch.decompress_blocks(comp, offs, sizes, BLOCK, **k),
                              int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, BLOCK))),
        "decompress_blocks_partial": (lambda **k: batch.decompress_blocks_partial(comp, offs, sizes, 4096, **k),
                                      int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, 4096))),
        "decompress_blocks_partial per-block": (
            lambda **k: batch.decompress_blocks_partial(comp, offs, sizes, targets, out_stride=4096, **k),
            int(lib.LZ4B200_decompress_workspace_bytes_for(n, 1, 0))),
        "compress_blocks_hc": (lambda **k: batch.compress_blocks_hc(src, BLOCK, 9, **k),
                               int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n))),
        "compress_blocks_hc_dest_size": (lambda **k: batch.compress_blocks_hc_dest_size(src, BLOCK, 4096, 9, **k),
                                         int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n))),
    }


NAMES = ["decompress_blocks", "decompress_blocks_partial", "decompress_blocks_partial per-block", "compress_blocks_hc",
         "compress_blocks_hc_dest_size"]


@pytest.mark.parametrize("name", NAMES)
def test_every_wrapper_takes_the_callers_workspace(rec, name):
    fn, need = wrappers(3)[name]
    s = torch.cuda.Stream()
    ws = torch.empty(need + 1000, dtype=torch.uint8, device=DEV)
    fn(workspace=ws, stream=s)
    (rng, st), = [ws_of(c) for c in rec.calls]
    assert rng == (ws.data_ptr(), ws.data_ptr() + ws.numel()) and st == s.cuda_stream
    with pytest.raises(ValueError):                      # too small: never swapped for a workspace of the module's
        fn(workspace=ws[:need - 1], stream=s)
    assert len(rec.calls) == 1


def overlap(a, b):
    return a[0] < b[1] and b[0] < a[1]


def test_owned_workspaces_are_never_shared_across_streams(rec):
    """A decode on A, an HC compress on B, a partial decode on C, then all three again with more blocks (the cache
    grows) and once more as the first time: no range the module hands to a call on one stream overlaps one it handed to a
    call on another, at any point of the sequence.  (A module that kept one workspace per device fails on the first B;
    one that grew it on B and went on using it on A, without A's stream owning it, fails on the second A.)"""
    sa, sb, sc = torch.cuda.Stream(), torch.cuda.Stream(), torch.cuda.Stream()
    for n in (4, 2, 40, 4):
        f = wrappers(n)
        f["decompress_blocks"][0](stream=sa)
        f["compress_blocks_hc"][0](stream=sb)
        f["decompress_blocks_partial"][0](stream=sc)
    seen = [ws_of(c) for c in rec.calls]
    assert len(seen) == 12
    for i, (ri, si) in enumerate(seen):
        for rj, sj in seen[:i]:
            assert si == sj or not overlap(ri, rj), ("stream %#x got [%#x, %#x), stream %#x [%#x, %#x)" %
                                                     (si, ri[0], ri[1], sj, rj[0], rj[1]))


def test_hc_wrappers_keep_their_stream_own_workspace(rec):
    """Two HC calls that overlap in time on different streams get different memory (the compressor keeps a 256 KB hash
    table per block in it)."""
    sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
    f = wrappers(2)
    f["compress_blocks_hc"][0](stream=sa)
    f["compress_blocks_hc_dest_size"][0](stream=sb)
    (ra, a), (rb, b) = [ws_of(c) for c in rec.calls]
    assert a != b and not overlap(ra, rb)


@pytest.mark.parametrize("phases", [1, 2])
def test_phased_decode_needs_its_own_workspace(rec, phases):
    """The expand reads the marks its scan left: through the module's cache any call in between (an HC compress, a
    larger decode that grows it) could overwrite them."""
    comp, offs, sizes = decode_inputs(3)
    with pytest.raises(ValueError):
        batch.decompress_blocks(comp, offs, sizes, BLOCK, phases=phases)
    ws = torch.empty(int(_lib.load().LZ4B200_decompress_workspace_bytes_for(3, 0, BLOCK)), dtype=torch.uint8, device=DEV)
    batch.decompress_blocks(comp, offs, sizes, BLOCK, phases=phases, workspace=ws)
    (rng, _), = [ws_of(c) for c in rec.calls]
    assert rng[0] == ws.data_ptr() and rec.calls[0][1][12] == phases


@pytest.mark.parametrize("name", NAMES)
def test_capture_needs_an_explicit_workspace(rec, name):
    """A graph keeps the address of the workspace it was captured with; the module's cache frees that memory when it
    grows.  So under capture a wrapper without `workspace=` raises, and one with it captures that workspace."""
    fn, need = wrappers(3)[name]
    ws = torch.empty(need, dtype=torch.uint8, device=DEV)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    raised = False
    with torch.cuda.graph(g, stream=s):
        try:
            fn(stream=s)
        except ValueError:
            raised = True
        fn(workspace=ws, stream=s)
    assert raised, "%s under capture used a workspace of the module's" % name
    (rng, st), = [ws_of(c) for c in rec.calls]
    assert rng[0] == ws.data_ptr() and st == s.cuda_stream


def test_partial_with_per_block_targets_makes_no_host_sync(rec):
    """With per-block targets and out_stride given, nothing needs the targets on the host: the call is captured (and
    any synchronising torch op in it would raise under sync debug mode "error")."""
    n = 5
    comp, offs, sizes = decode_inputs(n)
    targets = torch.tensor([1, 70000, 3, 4096, 0], dtype=torch.int32, device=DEV)
    ws = torch.empty(int(_lib.load().LZ4B200_decompress_workspace_bytes_for(n, 1, 0)), dtype=torch.uint8, device=DEV)
    out = torch.empty(n * 70000, dtype=torch.uint8, device=DEV)
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        torch.cuda.set_sync_debug_mode("error")
        try:
            batch.decompress_blocks_partial(comp, offs, sizes, targets, out=out, out_stride=70000, workspace=ws, stream=s)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    (name, args), = rec.calls
    assert name == "LZ4B200_decompress_blocks_partial" and args[5] == 70000 and args[6] == targets.data_ptr()
    # without out_stride the stride is the largest target, read on the host: refused under capture
    with torch.cuda.graph(torch.cuda.CUDAGraph(), stream=s):
        with pytest.raises(ValueError):
            batch.decompress_blocks_partial(comp, offs, sizes, targets, out=out, workspace=ws, stream=s)
