"""Batched block codec on device-resident torch tensors (the measured path).

torch is plumbing here: it owns the device memory and the stream; all work is done by
LZ4B200_* in liblz4_b200.so on raw pointers.

Every call is enqueued on `stream` (default: the current stream) and does no host synchronisation, so it can be
captured into a CUDA graph.  The workspace rule of the calls that need one (the decoders and the HC compressors):
  - `workspace=` is the caller's: it must hold what the call needs (ValueError otherwise), and calls that overlap in
    time must use different ones;
  - without it the call draws on a workspace the module owns, one per (device, stream): it is only ever used on the
    stream it was allocated on, so calls on different streams never share one, and calls on one stream are ordered by
    that stream;
  - a phased decode (phases 1 or 2) and any call under stream capture need their own: the expand consumes what its
    scan left in the workspace, which a call in between would overwrite, and a graph keeps the workspace's address,
    which the module's cache may free when it grows.
"""
import ctypes as C

import torch

from . import _lib


def _stream(stream=None):
    return stream if stream is not None else torch.cuda.current_stream()


_workspaces = {}        # (device index, stream handle) -> workspace owned by this module (grown on demand)


def _workspace(device, nbytes, stream, given, what):
    """The workspace of one call: `given` if the caller passed one (ValueError when it is smaller than nbytes), else the
    one this module keeps for (device, stream), allocated on that stream and used on no other.  A call that has to keep
    its workspace past its return -- under stream capture, or a scan whose expand comes later -- must bring its own."""
    if given is not None:
        _need_cuda(given)
        if given.numel() < nbytes:
            raise ValueError("%s: workspace of %d bytes, the call needs %d" % (what, given.numel(), nbytes))
        return given
    if torch.cuda.is_current_stream_capturing():
        raise ValueError("%s under stream capture needs its own workspace= (the graph would keep a cached one's "
                         "address)" % what)
    key = (device.index, stream.cuda_stream)
    ws = _workspaces.get(key)
    if ws is None or ws.numel() < nbytes:
        with torch.cuda.stream(stream):
            ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
        _workspaces[key] = ws
    return ws


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise ValueError("device tensors required (got a CPU tensor)")


def compress_bound(n):
    return int(_lib.load().LZ4_compressBound(int(n)))


def _decode_outputs(lib, comp, offsets, sizes, out_bytes, per_block, cap, out, out_sizes, workspace, st, what):
    """out, out_sizes and the workspace of a decode call: the ones given, else new ones on the launch stream (the
    workspace is sized by LZ4B200_decompress_workspace_bytes_for(n, per_block, cap); see _workspace)"""
    n = int(sizes.numel())
    ws_bytes = int(lib.LZ4B200_decompress_workspace_bytes_for(n, int(per_block), int(cap)))
    workspace = _workspace(comp.device, ws_bytes, st, workspace, what)
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if out is None:
            out = torch.empty(out_bytes, dtype=torch.uint8, device=comp.device)
        if out_sizes is None:
            out_sizes = torch.empty(n, dtype=torch.int32, device=comp.device)
    assert offsets.dtype == torch.int64 and sizes.dtype == torch.int32 and comp.dtype == torch.uint8
    return out, out_sizes, workspace


def _compress_layout(src, block_size, room, slots, slot_stride, out_sizes, src_sizes, st):
    """The blocks of a compress call: ceil(len(src) / block_size) of them, in slots of slot_stride bytes (default: room
    rounded up to 16).  slots, out_sizes and, for a short last block, the per-block src_sizes are allocated on the launch
    stream unless given.  Returns (n, stride, slots, out_sizes, src_sizes)."""
    total = int(src.numel())
    n = (total + block_size - 1) // block_size if total else 0
    stride = int(slot_stride if slot_stride is not None else ((room + 15) // 16) * 16)
    with torch.cuda.stream(st):
        if slots is None:
            slots = torch.empty(max(n, 1) * stride, dtype=torch.uint8, device=src.device)
        if out_sizes is None:
            out_sizes = torch.empty(max(n, 1), dtype=torch.int32, device=src.device)
        if src_sizes is None and n and total != n * block_size:
            src_sizes = torch.full((n,), block_size, dtype=torch.int32, device=src.device)
            src_sizes[-1] = total - (n - 1) * block_size
    return n, stride, slots, out_sizes, src_sizes


def decompress_blocks(comp, offsets, sizes, block_capacity, out=None, out_stride=None, out_sizes=None,
                      workspace=None, stream=None, phases=3):
    """Decode len(sizes) independent blocks.

    comp: u8[*] device buffer; block i = comp[offsets[i] : offsets[i]+sizes[i]] (int64 / int32 device
    tensors).  Block i is written to out[i*out_stride : ...] with capacity block_capacity.
    phases: 3 decodes; 1 only scans (out_sizes gets the sizes), 2 expands what the scan with the same arguments left
    in `workspace`, which both phases must be given (ValueError otherwise).
    Returns (out, out_sizes) -- out_sizes[i] is LZ4_decompress_safe's return value.
    """
    lib = _lib.load()
    _need_cuda(comp, offsets, sizes, out)
    if int(phases) in (1, 2) and workspace is None:
        raise ValueError("decompress_blocks: phases %d needs workspace= (the expand reads what the scan left there)"
                         % int(phases))
    n = int(sizes.numel())
    stride = int(out_stride if out_stride is not None else block_capacity)
    st = _stream(stream)
    out, out_sizes, workspace = _decode_outputs(lib, comp, offsets, sizes, n * stride, 0, block_capacity, out, out_sizes,
                                                workspace, st, "decompress_blocks")
    rc = lib.LZ4B200_decompress_blocks_phased(comp.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(),
                                              None, stride, None, int(block_capacity), out_sizes.data_ptr(), n,
                                              workspace.data_ptr(), workspace.numel(), int(phases),
                                              st.cuda_stream)
    _lib.check(rc, "LZ4B200_decompress_blocks")
    return out, out_sizes


def decompress_blocks_partial(comp, offsets, sizes, target, out=None, out_stride=None, out_sizes=None,
                              workspace=None, stream=None):
    """Decode a prefix of len(sizes) independent blocks (LZ4B200_decompress_blocks_partial: block i is
    LZ4_decompress_safe_partial(block_i, slot_i, sizes[i], t_i, t_i)).

    target: one int for every block, or an int32 device tensor of per-block targets.  Block i is written to
    out[i*out_stride : i*out_stride + out_sizes[i]] (out_stride defaults to the largest target: with per-block targets
    that reads target.max() on the host, so a captured call passes out_stride).
    Returns (out, out_sizes) -- out_sizes[i] is LZ4_decompress_safe_partial's return value.
    """
    lib = _lib.load()
    per_block = isinstance(target, torch.Tensor)
    _need_cuda(comp, offsets, sizes, out, target if per_block else None)
    n = int(sizes.numel())
    if per_block:
        assert target.dtype == torch.int32 and target.numel() == n
        uniform = 0
        if out_stride is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("decompress_blocks_partial under stream capture with per-block targets needs out_stride")
            biggest = int(target.max()) if n else 0
    else:
        uniform = biggest = int(target)
    stride = int(out_stride if out_stride is not None else max(biggest, 0))
    st = _stream(stream)
    out, out_sizes, workspace = _decode_outputs(lib, comp, offsets, sizes, max(n * stride, 1), per_block, uniform, out,
                                                out_sizes, workspace, st, "decompress_blocks_partial")
    rc = lib.LZ4B200_decompress_blocks_partial(comp.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(),
                                               None, stride, target.data_ptr() if per_block else None, uniform,
                                               out_sizes.data_ptr(), n, workspace.data_ptr(), workspace.numel(),
                                               st.cuda_stream)
    _lib.check(rc, "LZ4B200_decompress_blocks_partial")
    return out, out_sizes


def _budget(max_blocks):
    """the per-class budget (64 KB, 256 KB, 1 MB, 4 MB blocks) as the C array the frame calls take"""
    mb = [int(x) for x in max_blocks]
    if len(mb) != 4:
        raise ValueError("max_blocks: one budget per block size ID 4 .. 7 (4 values)")
    return (C.c_int64 * 4)(*mb)


def decompress_frames_workspace_bytes(n_frames, max_blocks):
    """LZ4B200_decompress_frames_workspace_bytes: the workspace decompress_frames needs (0: arguments it rejects)"""
    return int(_lib.load().LZ4B200_decompress_frames_workspace_bytes(int(n_frames), _budget(max_blocks)))


def decompress_frames(comp, offsets, sizes, capacities, max_blocks, out=None, out_offsets=None, results=None,
                      consumed=None, workspace=None, stream=None):
    """Decode len(sizes) LZ4 frames held in device memory (LZ4B200_decompress_frames).

    comp: u8[*] device buffer; frame f = comp[offsets[f] : offsets[f]+sizes[f]] (int64 device tensors), with 16
    readable bytes before and after it.  Frame f decodes to out[out_offsets[f] : out_offsets[f]+capacities[f]]
    (int64 device tensors).  out_offsets defaults to the exclusive sum of capacities, and out to their total (read on
    the host: a captured call passes out).  max_blocks: the blocks the call decodes at most from frames of each block
    size ID 4 .. 7 (4 host ints); a frame past its class's budget gets LZ4B200_ERR_LIMIT (-6).
    Returns (out, results, consumed): results[f] is LZ4B200_decompressFrame_host's return value for frame f (decoded
    bytes or a negative error code), consumed[f] the frame's length when its header and chain are valid, else 0.
    """
    return _decompress_frames("LZ4B200_decompress_frames", (), comp, offsets, sizes, capacities, max_blocks, out,
                              out_offsets, results, consumed, workspace, stream)


def decompress_frames_checksummed(comp, offsets, sizes, capacities, max_blocks, skip_checksums=False, out=None,
                                  out_offsets=None, results=None, consumed=None, workspace=None, stream=None):
    """decompress_frames for frames that may carry XXH32 block and content checksums
    (LZ4B200_decompress_frames_checksummed): same arguments, workspace and results, and a mismatching checksum gives
    LZ4B200_ERR_CHECKSUM (-7).  skip_checksums: parse the checksum fields without comparing them.  One thread hashes a
    frame's whole content, so the content check of a single large frame runs at one thread's speed."""
    return _decompress_frames("LZ4B200_decompress_frames_checksummed", (1 if skip_checksums else 0,), comp, offsets,
                              sizes, capacities, max_blocks, out, out_offsets, results, consumed, workspace, stream)


def _decompress_frames(entry, mode_args, comp, offsets, sizes, capacities, max_blocks, out, out_offsets, results,
                       consumed, workspace, stream):
    """the body of both frame calls: entry is the C function, mode_args what it takes after maxBlocks"""
    lib = _lib.load()
    _need_cuda(comp, offsets, sizes, capacities, out, out_offsets, results, consumed)
    assert comp.dtype == torch.uint8 and offsets.dtype == torch.int64 and sizes.dtype == torch.int64
    assert capacities.dtype == torch.int64
    n = int(sizes.numel())
    budget = _budget(max_blocks)
    st = _stream(stream)
    ws_bytes = int(lib.LZ4B200_decompress_frames_workspace_bytes(n, budget))
    if ws_bytes == 0:
        raise ValueError("decompress_frames: budgets must be 0 .. 2^31 - 1")
    workspace = _workspace(comp.device, ws_bytes, st, workspace, "decompress_frames")
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if out_offsets is None:
            out_offsets = torch.cumsum(capacities, 0) - capacities
        if out is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("decompress_frames under stream capture needs out=")
            out = torch.empty(max(int(capacities.sum()) if n else 0, 1), dtype=torch.uint8, device=comp.device)
        if results is None:
            results = torch.empty(n, dtype=torch.int64, device=comp.device)
        if consumed is None:
            consumed = torch.empty(n, dtype=torch.int64, device=comp.device)
    rc = getattr(lib, entry)(comp.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(),
                             out_offsets.data_ptr(), capacities.data_ptr(), results.data_ptr(), consumed.data_ptr(), n,
                             budget, *mode_args, workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    _lib.check(rc, entry)
    return out, results, consumed


def compress_blocks(src, block_size, acceleration=1, slots=None, slot_stride=None, slot_capacity=None,
                    out_sizes=None, src_sizes=None, stream=None, mode="exact"):
    """Compress src (u8 device tensor) as ceil(len/block_size) independent blocks.

    mode "exact": byte-identical to LZ4_compress_fast (LZ4B200_compress_blocks); mode "parallel": the
    parallel-parse encoder (LZ4B200_compress_blocks_parallel: valid, deterministic, ratio within 2 %, much faster).

    Returns (slots, out_sizes, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]].
    """
    lib = _lib.load()
    _need_cuda(src, slots)
    cap = int(slot_capacity if slot_capacity is not None else compress_bound(block_size))
    st = _stream(stream)
    n, stride, slots, out_sizes, src_sizes = _compress_layout(src, block_size, cap, slots, slot_stride, out_sizes,
                                                              src_sizes, st)
    if mode not in ("exact", "parallel"):
        raise ValueError("mode must be 'exact' or 'parallel'")
    fn = lib.LZ4B200_compress_blocks if mode == "exact" else lib.LZ4B200_compress_blocks_parallel
    rc = fn(src.data_ptr(), int(block_size), src_sizes.data_ptr() if src_sizes is not None else None,
            int(block_size), slots.data_ptr(), stride, cap, int(acceleration), out_sizes.data_ptr(), n, st.cuda_stream)
    _lib.check(rc, "LZ4B200_compress_blocks")
    return slots, out_sizes[:n], stride


def compress_blocks_hc(src, block_size, level=9, slots=None, slot_stride=None, slot_capacity=None, out_sizes=None,
                       workspace=None, stream=None):
    """Compress src (u8 device tensor) as ceil(len/block_size) independent blocks at an HC level
    (LZ4B200_compress_blocks_hc: block i is LZ4_compress_HC(block_i, slot_i, n_i, slot_capacity, level), byte for byte).

    Levels 1 .. 9 (below 1 means 9); 10 .. 12 raise, their optimal parser is not built.  workspace: at least
    LZ4B200_compress_blocks_hc_workspace_bytes(n) bytes (the module's rule above).
    Returns (slots, out_sizes, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]].
    """
    lib = _lib.load()
    _need_cuda(src, slots)
    cap = int(slot_capacity if slot_capacity is not None else compress_bound(block_size))
    st = _stream(stream)
    n, stride, slots, out_sizes, src_sizes = _compress_layout(src, block_size, cap, slots, slot_stride, out_sizes, None, st)
    workspace = _workspace(src.device, max(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n)), 1), st, workspace,
                           "compress_blocks_hc")
    rc = lib.LZ4B200_compress_blocks_hc(src.data_ptr(), int(block_size),
                                        src_sizes.data_ptr() if src_sizes is not None else None, int(block_size),
                                        slots.data_ptr(), stride, cap, int(level), out_sizes.data_ptr(), n,
                                        workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    _lib.check(rc, "LZ4B200_compress_blocks_hc")
    return slots, out_sizes[:n], stride


def compress_blocks_dest_size(src, block_size, target, acceleration=1, slots=None, slot_stride=None, out_sizes=None,
                              consumed=None, src_sizes=None, stream=None):
    """Compress as much of each block of src as fits into `target` bytes (LZ4B200_compress_blocks_destSize: block i is
    LZ4_compress_destSize_extState(state, block_i, slot_i, &n_i, target, acceleration)).

    Returns (slots, out_sizes, consumed, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]]
    and hold its first consumed[i] input bytes.
    """
    lib = _lib.load()
    _need_cuda(src, slots, src_sizes)
    room = max(min(int(target), compress_bound(block_size)), 1)
    st = _stream(stream)
    n, stride, slots, out_sizes, src_sizes = _compress_layout(src, block_size, room, slots, slot_stride, out_sizes,
                                                              src_sizes, st)
    if consumed is None:
        with torch.cuda.stream(st):
            consumed = torch.empty(max(n, 1), dtype=torch.int32, device=src.device)
    rc = lib.LZ4B200_compress_blocks_destSize(src.data_ptr(), int(block_size),
                                              src_sizes.data_ptr() if src_sizes is not None else None, int(block_size),
                                              slots.data_ptr(), stride, int(target), int(acceleration),
                                              out_sizes.data_ptr(), consumed.data_ptr(), n, st.cuda_stream)
    _lib.check(rc, "LZ4B200_compress_blocks_destSize")
    return slots, out_sizes[:n], consumed[:n], stride


def compress_blocks_hc_dest_size(src, block_size, target, level=9, slots=None, slot_stride=None, out_sizes=None,
                                 consumed=None, src_sizes=None, workspace=None, stream=None):
    """Compress as much of each block of src as fits into `target` bytes at an HC level
    (LZ4B200_compress_blocks_hc_destSize: block i is LZ4_compress_HC_destSize(state, block_i, slot_i, &n_i, target, level)).

    Levels 1 .. 9 (below 1 means 9); 10 .. 12 raise, their optimal parser is not built.  workspace: as for
    compress_blocks_hc.
    Returns (slots, out_sizes, consumed, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]]
    and hold its first consumed[i] input bytes.
    """
    lib = _lib.load()
    _need_cuda(src, slots, src_sizes)
    room = max(min(int(target), compress_bound(block_size)), 1)
    st = _stream(stream)
    n, stride, slots, out_sizes, src_sizes = _compress_layout(src, block_size, room, slots, slot_stride, out_sizes,
                                                              src_sizes, st)
    if consumed is None:
        with torch.cuda.stream(st):
            consumed = torch.empty(max(n, 1), dtype=torch.int32, device=src.device)
    workspace = _workspace(src.device, max(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n)), 1), st, workspace,
                           "compress_blocks_hc_dest_size")
    rc = lib.LZ4B200_compress_blocks_hc_destSize(src.data_ptr(), int(block_size),
                                                 src_sizes.data_ptr() if src_sizes is not None else None,
                                                 int(block_size), slots.data_ptr(), stride, int(target), int(level),
                                                 out_sizes.data_ptr(), consumed.data_ptr(), n, workspace.data_ptr(),
                                                 workspace.numel(), st.cuda_stream)
    _lib.check(rc, "LZ4B200_compress_blocks_hc_destSize")
    return slots, out_sizes[:n], consumed[:n], stride


def compress_blocks_hc_opt(src, block_size, level=12, slots=None, slot_stride=None, slot_capacity=None, out_sizes=None,
                           workspace=None, stream=None):
    """compress_blocks_hc at levels 10 .. 12, the optimal parser (LZ4B200_compress_blocks_hc_opt: block i is
    LZ4_compress_HC(block_i, slot_i, n_i, slot_capacity, level), byte for byte).

    Levels above 12 read as 12; levels below 10 raise (they are compress_blocks_hc's).  workspace: at least
    LZ4B200_compress_blocks_hc_opt_workspace_bytes(n) bytes (the module's rule above).  One thread parses a block, so
    large blocks at levels 11 and 12 take a long time.
    Returns (slots, out_sizes, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]].
    """
    lib = _lib.load()
    _need_cuda(src, slots)
    cap = int(slot_capacity if slot_capacity is not None else compress_bound(block_size))
    st = _stream(stream)
    n, stride, slots, out_sizes, src_sizes = _compress_layout(src, block_size, cap, slots, slot_stride, out_sizes, None, st)
    workspace = _workspace(src.device, max(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n)), 1), st, workspace,
                           "compress_blocks_hc_opt")
    rc = lib.LZ4B200_compress_blocks_hc_opt(src.data_ptr(), int(block_size),
                                            src_sizes.data_ptr() if src_sizes is not None else None, int(block_size),
                                            slots.data_ptr(), stride, cap, int(level), out_sizes.data_ptr(), n,
                                            workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    _lib.check(rc, "LZ4B200_compress_blocks_hc_opt")
    return slots, out_sizes[:n], stride


def compress_blocks_hc_opt_dest_size(src, block_size, target, level=12, slots=None, slot_stride=None, out_sizes=None,
                                     consumed=None, src_sizes=None, workspace=None, stream=None):
    """compress_blocks_hc_dest_size at levels 10 .. 12, the optimal parser (LZ4B200_compress_blocks_hc_opt_destSize:
    block i is LZ4_compress_HC_destSize(state, block_i, slot_i, &n_i, target, level)).

    Levels as for compress_blocks_hc_opt; workspace: as for compress_blocks_hc_opt.
    Returns (slots, out_sizes, consumed, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]]
    and hold its first consumed[i] input bytes.
    """
    lib = _lib.load()
    _need_cuda(src, slots, src_sizes)
    room = max(min(int(target), compress_bound(block_size)), 1)
    st = _stream(stream)
    n, stride, slots, out_sizes, src_sizes = _compress_layout(src, block_size, room, slots, slot_stride, out_sizes,
                                                              src_sizes, st)
    if consumed is None:
        with torch.cuda.stream(st):
            consumed = torch.empty(max(n, 1), dtype=torch.int32, device=src.device)
    workspace = _workspace(src.device, max(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n)), 1), st, workspace,
                           "compress_blocks_hc_opt_dest_size")
    rc = lib.LZ4B200_compress_blocks_hc_opt_destSize(src.data_ptr(), int(block_size),
                                                     src_sizes.data_ptr() if src_sizes is not None else None,
                                                     int(block_size), slots.data_ptr(), stride, int(target), int(level),
                                                     out_sizes.data_ptr(), consumed.data_ptr(), n, workspace.data_ptr(),
                                                     workspace.numel(), st.cuda_stream)
    _lib.check(rc, "LZ4B200_compress_blocks_hc_opt_destSize")
    return slots, out_sizes[:n], consumed[:n], stride


def pack_blocks(slots, slot_stride, sizes, header_bytes=0, packed=None, stream=None):
    """Gather variable-size blocks into one contiguous stream.  Returns (packed, offsets[n+1])."""
    lib = _lib.load()
    _need_cuda(slots, sizes)
    n = int(sizes.numel())
    st = _stream(stream)
    with torch.cuda.stream(st):
        offsets = torch.empty(n + 1, dtype=torch.int64, device=slots.device)
        if packed is None:
            packed = torch.empty(n * (int(slot_stride) + header_bytes) + 16, dtype=torch.uint8, device=slots.device)
    rc = lib.LZ4B200_pack_blocks(slots.data_ptr(), int(slot_stride), sizes.data_ptr(), n, packed.data_ptr(),
                                 offsets.data_ptr(), int(header_bytes), st.cuda_stream)
    _lib.check(rc, "LZ4B200_pack_blocks")
    return packed, offsets
