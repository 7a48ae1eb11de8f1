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

Every wrapper checks its arguments before it allocates or launches anything (_checked) and raises ValueError when one
fails: tensors are contiguous CUDA tensors on one device, of the dtype their argument takes, with the elements the call
reads or writes; strides hold a slot's capacity; ints the C call takes as 32-bit ints fit one.  The launch runs with
that device current, on `stream` (default: that device's current stream).  What would need a read of device memory is
not checked, so no wrapper synchronises for it: the values of offsets, sizes, per-block targets and src_sizes (a block
read or written past its buffer), and whether a frames call's `out` holds what out_offsets and capacities place in it.
Those are the caller's responsibility.
"""
import ctypes as C

import torch

from . import _lib


U8, I32, I64 = torch.uint8, torch.int32, torch.int64
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
ANY = (0, None)                 # an element count _checked accepts: at least 0, no upper limit


def _checked(what, stream, tensors, ints=(), strides=()):
    """The argument check of every wrapper: what the kernels would misread or write past, as far as it shows without
    reading device memory.  Raises ValueError when a check fails.
      tensors: (name, tensor or None, dtype, (least, most)): a contiguous CUDA tensor of that dtype with least .. most
               elements (most None: no limit); a byte buffer's elements are its bytes, whatever its shape.  All given
               tensors are on one device.
      ints:    (name, value, lo, hi): a host int the C call takes as a 32-bit int, within lo .. hi
      strides: (name, stride, capacity): slots `stride` bytes apart, each of `capacity` bytes, do not overlap
    Returns (device, stream): the tensors' device and the stream to launch on -- `stream` if given (it must be on that
    device), else the device's current stream."""
    device = None
    for name, t, dtype, (least, most) in tensors:
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise ValueError("%s: %s must be a CUDA tensor (got %s)" % (
                what, name, "one on %s" % t.device if isinstance(t, torch.Tensor) else type(t).__name__))
        if device is None:
            device = t.device
        elif t.device != device:
            raise ValueError("%s: %s is on %s, the other tensors on %s" % (what, name, t.device, device))
        if t.dtype != dtype:
            raise ValueError("%s: %s must be %s (got %s)" % (what, name, dtype, t.dtype))
        if not t.is_contiguous():
            raise ValueError("%s: %s must be contiguous" % (what, name))
        if t.numel() < least or (most is not None and t.numel() > most):
            raise ValueError("%s: %s has %d elements, the call needs %s" % (
                what, name, t.numel(), "at least %d" % least if most is None else "%d .. %d" % (least, most)))
    for name, v, lo, hi in ints:
        if not lo <= int(v) <= hi:
            raise ValueError("%s: %s = %d is outside %d .. %d" % (what, name, int(v), lo, hi))
    for name, stride, cap in strides:
        if int(stride) < max(int(cap), 0):
            raise ValueError("%s: %s = %d is below the %d bytes of a slot" % (what, name, int(stride), int(cap)))
    if stream is None:
        return device, torch.cuda.current_stream(device)
    if device is not None and stream.device != device:
        raise ValueError("%s: the stream is on %s, the tensors on %s" % (what, stream.device, device))
    return device, stream


def _int32(name, v):
    """an int the C call takes as a 32-bit int, as _checked takes it"""
    return (name, v, INT32_MIN, INT32_MAX)


def _extent(n, stride, cap):
    """the bytes n slots of `cap` bytes, `stride` apart, span"""
    return (n - 1) * int(stride) + max(int(cap), 0) if n else 0


def _launch(device, what, fn, *args):
    """one C call with `device` current (the library launches on the current device)"""
    with torch.cuda.device(device):
        rc = fn(*args)
    _lib.check(rc, what)


_workspaces = {}        # (device index, stream handle) -> workspace owned by this module (grown on demand)


def _workspace(device, nbytes, stream, given, what):
    """The workspace of one call: `given` if the caller passed one (_checked made sure it holds nbytes), else the one
    this module keeps for (device, stream), allocated on that stream and used on no other.  A call that has to keep its
    workspace past its return -- under stream capture, or a scan whose expand comes later -- must bring its own."""
    if given is not None:
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


def compress_bound(n):
    return int(_lib.load().LZ4_compressBound(int(n)))


def _decode_outputs(device, n, out_bytes, ws_bytes, out, out_sizes, workspace, st, what):
    """out, out_sizes and the workspace of a decode call: the ones given, else new ones on the launch stream (see
    _workspace)"""
    workspace = _workspace(device, ws_bytes, st, workspace, what)
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if out is None:
            out = torch.empty(out_bytes, dtype=torch.uint8, device=device)
        if out_sizes is None:
            out_sizes = torch.empty(n, dtype=torch.int32, device=device)
    return out, out_sizes, workspace


def _decode_tensors(comp, offsets, sizes, n, out, out_bytes, out_sizes, workspace, ws_bytes):
    """the tensors of a decode call as _checked takes them"""
    return [("comp", comp, U8, ANY), ("offsets", offsets, I64, (n, None)), ("sizes", sizes, I32, ANY),
            ("out", out, U8, (out_bytes, None)), ("out_sizes", out_sizes, I32, (n, None)),
            ("workspace", workspace, U8, (ws_bytes, None))]


def _block_count(src, block_size):
    """ceil(len(src) / block_size): the blocks of a compress call (0 for a block_size _checked rejects)"""
    total, bs = int(src.numel()) if isinstance(src, torch.Tensor) else 0, int(block_size)
    return (total + bs - 1) // bs if total and bs > 0 else 0


def _compress_layout(what, src, block_size, n, room, slots, slot_stride, out_sizes, src_sizes, stream, tensors=(),
                     ints=()):
    """The n blocks of a compress call, in slots of slot_stride bytes (default: room rounded up to 16) of which the
    kernels write at most `room`.  Checks the call's arguments (_checked; tensors and ints: the call's own besides
    these), then allocates slots, out_sizes and, for a short last block, the per-block src_sizes on the launch stream
    unless given.  Returns (device, stream, stride, slots, out_sizes, src_sizes)."""
    bs = int(block_size)
    stride = int(slot_stride if slot_stride is not None else ((room + 15) // 16) * 16)
    device, st = _checked(what, stream,
                          [("src", src, U8, ANY), ("slots", slots, U8, (_extent(n, stride, room), None)),
                           ("out_sizes", out_sizes, I32, (n, None)), ("src_sizes", src_sizes, I32, (n, n))]
                          + list(tensors), [("block_size", bs, 1, INT32_MAX)] + list(ints),
                          [("slot_stride", stride, room)])
    total = int(src.numel())
    with torch.cuda.stream(st):
        if slots is None:
            slots = torch.empty(max(n, 1) * stride, dtype=torch.uint8, device=device)
        if out_sizes is None:
            out_sizes = torch.empty(max(n, 1), dtype=torch.int32, device=device)
        if src_sizes is None and n and total != n * bs:
            src_sizes = torch.full((n,), bs, dtype=torch.int32, device=device)
            src_sizes[-1] = total - (n - 1) * bs
    return device, st, stride, slots, out_sizes, src_sizes


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
    if int(phases) in (1, 2) and workspace is None:
        raise ValueError("decompress_blocks: phases %d needs workspace= (the expand reads what the scan left there)"
                         % int(phases))
    n = int(sizes.numel())
    cap = int(block_capacity)
    stride = int(out_stride if out_stride is not None else cap)
    ws_bytes = int(lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap))
    device, st = _checked("decompress_blocks", stream,
                          _decode_tensors(comp, offsets, sizes, n, out, _extent(n, stride, cap), out_sizes, workspace,
                                          ws_bytes),
                          [_int32("block_capacity", cap)], [("out_stride", stride, cap)])
    out, out_sizes, workspace = _decode_outputs(device, n, n * stride, ws_bytes, out, out_sizes, workspace, st,
                                                "decompress_blocks")
    _launch(device, "LZ4B200_decompress_blocks", lib.LZ4B200_decompress_blocks_phased, comp.data_ptr(),
            offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(), None, stride, None, cap, out_sizes.data_ptr(), n,
            workspace.data_ptr(), workspace.numel(), int(phases), st.cuda_stream)
    return out, out_sizes


def decompress_blocks_partial(comp, offsets, sizes, target, out=None, out_stride=None, out_sizes=None,
                              workspace=None, stream=None):
    """Decode a prefix of len(sizes) independent blocks (LZ4B200_decompress_blocks_partial: block i is
    LZ4_decompress_safe_partial(block_i, slot_i, sizes[i], t_i, t_i)).

    target: one int for every block, or an int32 device tensor of per-block targets.  Block i is written to
    out[i*out_stride : i*out_stride + out_sizes[i]] (out_stride defaults to the largest target: with per-block targets
    that reads target.max() on the host, so a captured call passes out_stride).  With per-block targets each block's
    slot is out_stride bytes, so a given out holds len(sizes) * out_stride bytes and no target may exceed out_stride.
    Returns (out, out_sizes) -- out_sizes[i] is LZ4_decompress_safe_partial's return value.
    """
    lib = _lib.load()
    per_block = isinstance(target, torch.Tensor)
    n = int(sizes.numel())
    if per_block:
        uniform = 0
        if out_stride is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("decompress_blocks_partial under stream capture with per-block targets needs out_stride")
            biggest = int(target.max()) if target.numel() else 0
    else:
        uniform = biggest = int(target)
    stride = int(out_stride if out_stride is not None else max(biggest, 0))
    ws_bytes = int(lib.LZ4B200_decompress_workspace_bytes_for(n, int(per_block), uniform))
    tensors = _decode_tensors(comp, offsets, sizes, n, out, n * stride if per_block else _extent(n, stride, uniform),
                              out_sizes, workspace, ws_bytes)
    if per_block:
        tensors.append(("target", target, I32, (n, n)))
    device, st = _checked("decompress_blocks_partial", stream, tensors, [_int32("target", uniform)],
                          [("out_stride", stride, uniform)])
    out, out_sizes, workspace = _decode_outputs(device, n, max(n * stride, 1), ws_bytes, out, out_sizes, workspace, st,
                                                "decompress_blocks_partial")
    _launch(device, "LZ4B200_decompress_blocks_partial", lib.LZ4B200_decompress_blocks_partial, comp.data_ptr(),
            offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(), None, stride,
            target.data_ptr() if per_block else None, uniform, out_sizes.data_ptr(), n, workspace.data_ptr(),
            workspace.numel(), st.cuda_stream)
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
    LZ4B200_ERR_CHECKSUM (-7).  skip_checksums: parse the checksum fields without comparing them.  A frame's content
    checksum is hashed by one thread below 256 KiB of content and by a warp that stages the content through shared
    memory from 256 KiB on."""
    return _decompress_frames("LZ4B200_decompress_frames_checksummed", (1 if skip_checksums else 0,), comp, offsets,
                              sizes, capacities, max_blocks, out, out_offsets, results, consumed, workspace, stream)


def _decompress_frames(entry, mode_args, comp, offsets, sizes, capacities, max_blocks, out, out_offsets, results,
                       consumed, workspace, stream):
    """the body of both frame calls: entry is the C function, mode_args what it takes after maxBlocks"""
    lib = _lib.load()
    n = int(sizes.numel())
    budget = _budget(max_blocks)
    ws_bytes = int(lib.LZ4B200_decompress_frames_workspace_bytes(n, budget))
    if ws_bytes == 0:
        raise ValueError("decompress_frames: budgets must be 0 .. 2^31 - 1")
    at_least_n = (n, None)
    device, st = _checked("decompress_frames", stream,
                          [("comp", comp, U8, ANY), ("offsets", offsets, I64, at_least_n), ("sizes", sizes, I64, ANY),
                           ("capacities", capacities, I64, (n, n)), ("out", out, U8, ANY),
                           ("out_offsets", out_offsets, I64, at_least_n), ("results", results, I64, at_least_n),
                           ("consumed", consumed, I64, at_least_n), ("workspace", workspace, U8, (ws_bytes, None))])
    workspace = _workspace(device, ws_bytes, st, workspace, "decompress_frames")
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if out_offsets is None:
            out_offsets = torch.cumsum(capacities, 0) - capacities
        if out is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("decompress_frames under stream capture needs out=")
            out = torch.empty(max(int(capacities.sum()) if n else 0, 1), dtype=torch.uint8, device=device)
        if results is None:
            results = torch.empty(n, dtype=torch.int64, device=device)
        if consumed is None:
            consumed = torch.empty(n, dtype=torch.int64, device=device)
    _launch(device, entry, getattr(lib, entry), comp.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(),
            out_offsets.data_ptr(), capacities.data_ptr(), results.data_ptr(), consumed.data_ptr(), n, budget,
            *mode_args, workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    return out, results, consumed


def _file_budget(max_blocks):
    """the per-class budget of the file calls (64 KB, 256 KB, 1 MB, 4 MB frame blocks, 8 MiB legacy blocks)"""
    mb = [int(x) for x in max_blocks]
    if len(mb) != 5:
        raise ValueError("max_blocks: one budget per block size ID 4 .. 7 and one for legacy blocks (5 values)")
    return (C.c_int64 * 5)(*mb)


def decompress_files_workspace_bytes(n_files, max_units, max_blocks):
    """LZ4B200_decompress_files_workspace_bytes: the workspace decompress_files and decompressed_file_sizes need (0:
    arguments they reject)"""
    return int(_lib.load().LZ4B200_decompress_files_workspace_bytes(int(n_files), int(max_units),
                                                                     _file_budget(max_blocks)))


def decompress_files(comp, offsets, sizes, capacities, max_units, max_blocks, skip_checksums=False, out=None,
                     out_offsets=None, results=None, consumed=None, prefix=None, workspace=None, stream=None):
    """Decode len(sizes) whole .lz4 files held in device memory as `lz4 -d` decodes them (LZ4B200_decompress_files):
    LZ4 frames one after another, skippable frames and `lz4 -l` legacy streams.

    comp: u8[*] device buffer; file f = comp[offsets[f] : offsets[f]+sizes[f]] (int64 device tensors), with 16 readable
    bytes before and after it.  File f decodes to out[out_offsets[f] : out_offsets[f]+capacities[f]] (int64 device
    tensors); out_offsets defaults to the exclusive sum of capacities, and out to their total (read on the host: a
    captured call passes out).  max_units: the units (frames, skippable frames, legacy streams) the call takes over all
    files; max_blocks: its blocks per class (5 host ints: frame blocks of block size ID 4 .. 7, legacy blocks).
    skip_checksums: `lz4 -d --no-frame-crc`.
    Returns (out, results, consumed, prefix): results[f] the decoded size or the code of the file's first failing unit,
    consumed[f] sizes[f] or that unit's offset, prefix[f] the decoded bytes of the units before it."""
    return _decompress_files(False, comp, offsets, sizes, capacities, max_units, max_blocks, skip_checksums, out,
                             out_offsets, results, consumed, prefix, workspace, stream)


def decompressed_file_sizes(comp, offsets, sizes, max_units, max_blocks, skip_checksums=False, results=None,
                            consumed=None, prefix=None, workspace=None, stream=None):
    """The size-only pass of decompress_files (sizeOnly): the same results with unlimited room and no byte written --
    the decoded size of every file, block checksums verified unless skipped, content checksums not compared.
    Returns (results, consumed, prefix)."""
    return _decompress_files(True, comp, offsets, sizes, None, max_units, max_blocks, skip_checksums, None, None,
                             results, consumed, prefix, workspace, stream)[1:]


def _decompress_files(size_only, comp, offsets, sizes, capacities, max_units, max_blocks, skip_checksums, out,
                      out_offsets, results, consumed, prefix, workspace, stream):
    lib = _lib.load()
    what = "decompressed_file_sizes" if size_only else "decompress_files"
    n = int(sizes.numel()) if isinstance(sizes, torch.Tensor) else 0
    budget = _file_budget(max_blocks)
    ws_bytes = int(lib.LZ4B200_decompress_files_workspace_bytes(n, int(max_units), budget))
    if ws_bytes == 0:
        raise ValueError("%s: max_units and the budgets must be 0 .. 2^31 - 1" % what)
    at_least_n = (n, None)
    device, st = _checked(what, stream,
                          [("comp", comp, U8, ANY), ("offsets", offsets, I64, at_least_n), ("sizes", sizes, I64, ANY),
                           ("capacities", capacities, I64, (n, n)), ("out", out, U8, ANY),
                           ("out_offsets", out_offsets, I64, at_least_n), ("results", results, I64, at_least_n),
                           ("consumed", consumed, I64, at_least_n), ("prefix", prefix, I64, at_least_n),
                           ("workspace", workspace, U8, (ws_bytes, None))])
    if not size_only and capacities is None:
        raise ValueError("%s: capacities must be a CUDA tensor" % what)
    workspace = _workspace(device, ws_bytes, st, workspace, what)
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if not size_only:
            if out_offsets is None:
                out_offsets = torch.cumsum(capacities, 0) - capacities
            if out is None:
                if torch.cuda.is_current_stream_capturing():
                    raise ValueError("%s under stream capture needs out=" % what)
                out = torch.empty(max(int(capacities.sum()) if n else 0, 1), dtype=torch.uint8, device=device)
        if results is None:
            results = torch.empty(n, dtype=torch.int64, device=device)
        if consumed is None:
            consumed = torch.empty(n, dtype=torch.int64, device=device)
        if prefix is None:
            prefix = torch.empty(n, dtype=torch.int64, device=device)
    ptr = (lambda t: t.data_ptr() if t is not None else None)
    _launch(device, "LZ4B200_decompress_files", lib.LZ4B200_decompress_files, comp.data_ptr(), offsets.data_ptr(),
            sizes.data_ptr(), ptr(out), ptr(out_offsets), ptr(capacities), results.data_ptr(), consumed.data_ptr(),
            prefix.data_ptr(), n, int(max_units), budget, 1 if skip_checksums else 0, 1 if size_only else 0,
            workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    return out, results, consumed, prefix


def compress_frames_workspace_bytes(n_frames, max_blocks, level=0):
    """LZ4B200_compress_frames_workspace_bytes: the workspace compress_frames needs (0: arguments it rejects)"""
    return int(_lib.load().LZ4B200_compress_frames_workspace_bytes(int(n_frames), _budget(max_blocks), int(level)))


def _frame_plan(sizes, block_size_id, block_checksum=False, content_checksum=False):
    """(budget, capacities) for frames of these sizes: the blocks of each class, and LZ4B200_compressFrameBound per
    frame at its optimal block size ID (which is at least the reference's bound), plus 4 bytes per block with block
    checksums and 4 per frame with a content checksum.  Reads sizes on the host."""
    bsid = int(block_size_id) or 4
    budget, caps = [0, 0, 0, 0], []
    for n in sizes.tolist():
        b = 4
        while b < bsid and n > 1 << (8 + 2 * b):
            b += 1
        bs = 1 << (8 + 2 * b)
        k = (max(n, 0) + bs - 1) // bs
        if n >= 0:
            budget[b - 4] += k
        caps.append(max(int(_lib.load().LZ4B200_compressFrameBound(max(n, 0), b)), 0)
                    + (4 * k if block_checksum else 0) + (4 if content_checksum else 0))
    return budget, caps


def compress_frames(src, offsets, sizes, max_blocks=None, block_size_id=4, level=0, content_size=False, parallel=False,
                    out=None, out_offsets=None, capacities=None, results=None, workspace=None, stream=None):
    """Write len(sizes) LZ4 frames from buffers in device memory (LZ4B200_compress_frames): frame f is, byte for byte,
    LZ4F_compressFrame of src[offsets[f] : offsets[f]+sizes[f]] with independent blocks, no checksums, the block size
    ID block_size_id (0 or 4 .. 7, shrunk per frame as LZ4F_optimalBSID does), the content size when content_size, and
    the compression level `level` (levels 2 and up through the HC encoders).  parallel: the parallel parse (levels
    below 2 only): valid frames, not the reference's bytes.

    offsets, sizes: int64 device tensors.  Frame f is written at out[out_offsets[f]:] with capacities[f] bytes of room
    (int64 device tensors).  max_blocks: the blocks the call compresses at most from frames of each block size ID 4 .. 7
    (4 host ints); a frame past its class's budget gets LZ4B200_ERR_LIMIT (-6).  Left as None, max_blocks and
    capacities are computed from sizes read on the host (capacities: LZ4B200_compressFrameBound per frame), which is a
    host sync: under stream capture max_blocks, out and capacities must be given.  out_offsets defaults to the
    exclusive sum of the capacities and out to their total.
    Returns (out, results): results[f] is the frame's length, or LZ4B200_ERR_ARG (a negative size or capacity),
    LZ4B200_ERR_DSTSIZE (a capacity below the reference's bound) or LZ4B200_ERR_LIMIT.
    """
    return _compress_frames("compress_frames", None, src, offsets, sizes, max_blocks, block_size_id, level,
                            content_size, parallel, out, out_offsets, capacities, results, workspace, stream)


def compress_frames_checksummed(src, offsets, sizes, max_blocks=None, block_size_id=4, level=0, content_size=False,
                                parallel=False, block_checksum=False, content_checksum=True, out=None, out_offsets=None,
                                capacities=None, results=None, workspace=None, stream=None):
    """compress_frames with XXH32 checksums (LZ4B200_compress_frames_checksummed): block_checksum puts the LE32
    XXH32(payload, 0) after every block, content_checksum the LE32 XXH32(source, 0) after the EndMark, as
    LZ4F_compressFrame does with blockChecksumFlag and contentChecksumFlag.  The defaults are the `lz4` tool's: a content
    checksum, no block checksums.  Same arguments, capture rules and results as compress_frames; the default capacities
    are its bound plus 4 bytes per block with block checksums and 4 per frame with a content checksum, the reference's
    LZ4F_compressFrameBound for those flags."""
    return _compress_frames("compress_frames_checksummed", (1 if block_checksum else 0, 1 if content_checksum else 0),
                            src, offsets, sizes, max_blocks, block_size_id, level, content_size, parallel, out,
                            out_offsets, capacities, results, workspace, stream)


def _compress_frames(name, sums, src, offsets, sizes, max_blocks, block_size_id, level, content_size, parallel, out,
                     out_offsets, capacities, results, workspace, stream):
    """the body of compress_frames (sums None) and compress_frames_checksummed (sums: the two flags)"""
    lib = _lib.load()
    n = int(sizes.numel()) if isinstance(sizes, torch.Tensor) else 0
    capturing = torch.cuda.is_current_stream_capturing()
    if capturing and (max_blocks is None or out is None or capacities is None):
        raise ValueError("%s under stream capture needs max_blocks=, out= and capacities= (computing them "
                         "reads sizes on the host)" % name)
    at_least_n = (n, None)
    device, st = _checked(name, stream,
                          [("src", src, U8, ANY), ("offsets", offsets, I64, at_least_n), ("sizes", sizes, I64, ANY),
                           ("out", out, U8, ANY), ("out_offsets", out_offsets, I64, at_least_n),
                           ("capacities", capacities, I64, (n, n)), ("results", results, I64, at_least_n),
                           ("workspace", workspace, U8, ANY)],
                          [_int32("block_size_id", block_size_id), _int32("level", level)])
    if int(block_size_id) not in (0, 4, 5, 6, 7):
        raise ValueError("%s: block_size_id must be 0 or 4 .. 7 (got %d)" % (name, int(block_size_id)))
    if parallel and int(level) >= 2:
        raise ValueError("%s: parallel takes levels below 2 (got %d)" % (name, int(level)))
    plan = (_frame_plan(sizes, block_size_id, *(bool(x) for x in (sums or (0, 0))))
            if max_blocks is None or capacities is None else None)
    budget = _budget(max_blocks if max_blocks is not None else plan[0])
    ws_bytes = int(lib.LZ4B200_compress_frames_workspace_bytes(n, budget, int(level)))
    if ws_bytes == 0:
        raise ValueError("%s: budgets must be 0 .. 2^31 - 1" % name)
    if workspace is not None and workspace.numel() < ws_bytes:
        raise ValueError("%s: workspace has %d elements, the call needs at least %d"
                         % (name, workspace.numel(), ws_bytes))
    workspace = _workspace(device, ws_bytes, st, workspace, name)
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if capacities is None:
            capacities = torch.tensor(plan[1], dtype=I64, device=device)
        if out_offsets is None:
            out_offsets = torch.cumsum(capacities.clamp(min=0), 0) - capacities.clamp(min=0)
        if out is None:
            out = torch.empty(max(int(capacities.clamp(min=0).sum()) if n else 0, 1), dtype=torch.uint8, device=device)
        if results is None:
            results = torch.empty(max(n, 1), dtype=torch.int64, device=device)
    entry = "LZ4B200_" + name
    _launch(device, entry, getattr(lib, entry), src.data_ptr(), offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(),
            out_offsets.data_ptr(), capacities.data_ptr(), results.data_ptr(), n, int(block_size_id), int(level),
            1 if content_size else 0, 1 if parallel else 0, *(sums or ()), budget, workspace.data_ptr(),
            workspace.numel(), st.cuda_stream)
    return out, results[:n]


LEGACY_BLOCK = 8 << 20          # the chunk an `lz4 -l` stream compresses at a time


def legacy_bound(n):
    """LZ4B200_compressLegacyBound: the longest `lz4 -l` stream of n bytes, 4 + the sum over its 8 MiB chunks of 4 +
    LZ4_compressBound(chunk) (LZ4B200_ERR_ARG for n < 0)"""
    return int(_lib.load().LZ4B200_compressLegacyBound(int(n)))


def compress_legacy_workspace_bytes(n_files, max_blocks, level=1):
    """LZ4B200_compress_legacy_workspace_bytes: the workspace compress_legacy needs (0: arguments it rejects)"""
    return int(_lib.load().LZ4B200_compress_legacy_workspace_bytes(int(n_files), int(max_blocks), int(level)))


def compress_legacy(src, offsets, sizes, max_blocks=None, level=1, out=None, out_offsets=None, capacities=None,
                    results=None, workspace=None, stream=None):
    """Write len(sizes) `lz4 -l` legacy streams from buffers in device memory (LZ4B200_compress_legacy): stream f is,
    byte for byte, what `lz4 -l -c -<level>` (`--fast=N` for level -N) writes for src[offsets[f] : offsets[f]+sizes[f]]
    piped to its standard input -- the magic, then per 8 MiB chunk its LE32 compressed size and block.  The level
    mapping is the tool's: below 3 the fast parse (acceleration -level for negative levels), 3 and up LZ4_compress_HC.

    offsets, sizes: int64 device tensors.  Stream f is written at out[out_offsets[f]:] with capacities[f] bytes of room
    (int64 device tensors).  max_blocks: the 8 MiB chunks the call compresses at most (a host int); a file past it gets
    LZ4B200_ERR_LIMIT (-6).  Left as None, max_blocks and capacities are computed from sizes read on the host
    (capacities: legacy_bound per file), which is a host sync: under stream capture max_blocks, out and capacities must
    be given.  out_offsets defaults to the exclusive sum of the capacities and out to their total.
    Returns (out, results): results[f] is the stream's length, or LZ4B200_ERR_ARG (a negative size or capacity),
    LZ4B200_ERR_DSTSIZE (a capacity below legacy_bound) or LZ4B200_ERR_LIMIT.
    """
    name = "compress_legacy"
    lib = _lib.load()
    n = int(sizes.numel()) if isinstance(sizes, torch.Tensor) else 0
    if torch.cuda.is_current_stream_capturing() and (max_blocks is None or out is None or capacities is None):
        raise ValueError("%s under stream capture needs max_blocks=, out= and capacities= (computing them "
                         "reads sizes on the host)" % name)
    at_least_n = (n, None)
    device, st = _checked(name, stream,
                          [("src", src, U8, ANY), ("offsets", offsets, I64, at_least_n), ("sizes", sizes, I64, ANY),
                           ("out", out, U8, ANY), ("out_offsets", out_offsets, I64, at_least_n),
                           ("capacities", capacities, I64, (n, n)), ("results", results, I64, at_least_n),
                           ("workspace", workspace, U8, ANY)],
                          [_int32("level", level)])
    if max_blocks is None or capacities is None:
        host_sizes = sizes.tolist()
        need = sum((s + LEGACY_BLOCK - 1) // LEGACY_BLOCK for s in host_sizes if s >= 0)
        caps = [max(legacy_bound(max(s, 0)), 0) for s in host_sizes]
    budget = int(max_blocks) if max_blocks is not None else need
    ws_bytes = compress_legacy_workspace_bytes(n, budget, level)
    if ws_bytes == 0:
        raise ValueError("%s: max_blocks must be 0 .. 2^31 - 1 (got %d)" % (name, budget))
    if workspace is not None and workspace.numel() < ws_bytes:
        raise ValueError("%s: workspace has %d elements, the call needs at least %d"
                         % (name, workspace.numel(), ws_bytes))
    workspace = _workspace(device, ws_bytes, st, workspace, name)
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if capacities is None:
            capacities = torch.tensor(caps, dtype=I64, device=device)
        if out_offsets is None:
            out_offsets = torch.cumsum(capacities.clamp(min=0), 0) - capacities.clamp(min=0)
        if out is None:
            out = torch.empty(max(int(capacities.clamp(min=0).sum()) if n else 0, 1), dtype=torch.uint8, device=device)
        if results is None:
            results = torch.empty(max(n, 1), dtype=torch.int64, device=device)
    _launch(device, "LZ4B200_" + name, lib.LZ4B200_compress_legacy, src.data_ptr(), offsets.data_ptr(),
            sizes.data_ptr(), out.data_ptr(), out_offsets.data_ptr(), capacities.data_ptr(), results.data_ptr(), n,
            int(level), budget, workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    return out, results[:n]


def compress_blocks(src, block_size, acceleration=1, slots=None, slot_stride=None, slot_capacity=None,
                    out_sizes=None, src_sizes=None, stream=None, mode="exact"):
    """Compress src (u8 device tensor) as ceil(len/block_size) independent blocks.

    mode "exact": byte-identical to LZ4_compress_fast (LZ4B200_compress_blocks); mode "parallel": the
    parallel-parse encoder (LZ4B200_compress_blocks_parallel: valid, deterministic, ratio within 2 %, much faster).

    Returns (slots, out_sizes, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]].
    """
    lib = _lib.load()
    if mode not in ("exact", "parallel"):
        raise ValueError("mode must be 'exact' or 'parallel'")
    cap = int(slot_capacity if slot_capacity is not None else compress_bound(block_size))
    n = _block_count(src, block_size)
    device, st, stride, slots, out_sizes, src_sizes = _compress_layout(
        "compress_blocks", src, block_size, n, cap, slots, slot_stride, out_sizes, src_sizes, stream,
        ints=[_int32("slot_capacity", cap), _int32("acceleration", acceleration)])
    fn = lib.LZ4B200_compress_blocks if mode == "exact" else lib.LZ4B200_compress_blocks_parallel
    _launch(device, "LZ4B200_compress_blocks", fn, src.data_ptr(), int(block_size),
            src_sizes.data_ptr() if src_sizes is not None else None, int(block_size), slots.data_ptr(), stride, cap,
            int(acceleration), out_sizes.data_ptr(), n, st.cuda_stream)
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
    cap = int(slot_capacity if slot_capacity is not None else compress_bound(block_size))
    n = _block_count(src, block_size)
    ws_bytes = max(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n)), 1)
    device, st, stride, slots, out_sizes, src_sizes = _compress_layout(
        "compress_blocks_hc", src, block_size, n, cap, slots, slot_stride, out_sizes, None, stream,
        [("workspace", workspace, U8, (ws_bytes, None))], [_int32("slot_capacity", cap), _int32("level", level)])
    workspace = _workspace(device, ws_bytes, st, workspace, "compress_blocks_hc")
    _launch(device, "LZ4B200_compress_blocks_hc", lib.LZ4B200_compress_blocks_hc, src.data_ptr(), int(block_size),
            src_sizes.data_ptr() if src_sizes is not None else None, int(block_size), slots.data_ptr(), stride, cap,
            int(level), out_sizes.data_ptr(), n, workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    return slots, out_sizes[:n], stride


def _consumed(consumed, n, device, st):
    """the consumed counts of a destSize call: the given ones, else new ones on the launch stream"""
    if consumed is None:
        with torch.cuda.stream(st):
            consumed = torch.empty(max(n, 1), dtype=torch.int32, device=device)
    return consumed


def compress_blocks_dest_size(src, block_size, target, acceleration=1, slots=None, slot_stride=None, out_sizes=None,
                              consumed=None, src_sizes=None, stream=None):
    """Compress as much of each block of src as fits into `target` bytes (LZ4B200_compress_blocks_destSize: block i is
    LZ4_compress_destSize_extState(state, block_i, slot_i, &n_i, target, acceleration)).

    Returns (slots, out_sizes, consumed, slot_stride): block i's bytes are slots[i*slot_stride : i*slot_stride+out_sizes[i]]
    and hold its first consumed[i] input bytes.
    """
    lib = _lib.load()
    room = max(min(int(target), compress_bound(block_size)), 1)
    n = _block_count(src, block_size)
    device, st, stride, slots, out_sizes, src_sizes = _compress_layout(
        "compress_blocks_dest_size", src, block_size, n, room, slots, slot_stride, out_sizes, src_sizes, stream,
        [("consumed", consumed, I32, (n, None))], [_int32("target", target), _int32("acceleration", acceleration)])
    consumed = _consumed(consumed, n, device, st)
    _launch(device, "LZ4B200_compress_blocks_destSize", lib.LZ4B200_compress_blocks_destSize, src.data_ptr(),
            int(block_size), src_sizes.data_ptr() if src_sizes is not None else None, int(block_size),
            slots.data_ptr(), stride, int(target), int(acceleration), out_sizes.data_ptr(), consumed.data_ptr(), n,
            st.cuda_stream)
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
    room = max(min(int(target), compress_bound(block_size)), 1)
    n = _block_count(src, block_size)
    ws_bytes = max(int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n)), 1)
    device, st, stride, slots, out_sizes, src_sizes = _compress_layout(
        "compress_blocks_hc_dest_size", src, block_size, n, room, slots, slot_stride, out_sizes, src_sizes, stream,
        [("consumed", consumed, I32, (n, None)), ("workspace", workspace, U8, (ws_bytes, None))],
        [_int32("target", target), _int32("level", level)])
    consumed = _consumed(consumed, n, device, st)
    workspace = _workspace(device, ws_bytes, st, workspace, "compress_blocks_hc_dest_size")
    _launch(device, "LZ4B200_compress_blocks_hc_destSize", lib.LZ4B200_compress_blocks_hc_destSize, src.data_ptr(),
            int(block_size), src_sizes.data_ptr() if src_sizes is not None else None, int(block_size),
            slots.data_ptr(), stride, int(target), int(level), out_sizes.data_ptr(), consumed.data_ptr(), n,
            workspace.data_ptr(), workspace.numel(), st.cuda_stream)
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
    cap = int(slot_capacity if slot_capacity is not None else compress_bound(block_size))
    n = _block_count(src, block_size)
    ws_bytes = max(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n)), 1)
    device, st, stride, slots, out_sizes, src_sizes = _compress_layout(
        "compress_blocks_hc_opt", src, block_size, n, cap, slots, slot_stride, out_sizes, None, stream,
        [("workspace", workspace, U8, (ws_bytes, None))], [_int32("slot_capacity", cap), _int32("level", level)])
    workspace = _workspace(device, ws_bytes, st, workspace, "compress_blocks_hc_opt")
    _launch(device, "LZ4B200_compress_blocks_hc_opt", lib.LZ4B200_compress_blocks_hc_opt, src.data_ptr(),
            int(block_size), src_sizes.data_ptr() if src_sizes is not None else None, int(block_size),
            slots.data_ptr(), stride, cap, int(level), out_sizes.data_ptr(), n, workspace.data_ptr(), workspace.numel(),
            st.cuda_stream)
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
    room = max(min(int(target), compress_bound(block_size)), 1)
    n = _block_count(src, block_size)
    ws_bytes = max(int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n)), 1)
    device, st, stride, slots, out_sizes, src_sizes = _compress_layout(
        "compress_blocks_hc_opt_dest_size", src, block_size, n, room, slots, slot_stride, out_sizes, src_sizes, stream,
        [("consumed", consumed, I32, (n, None)), ("workspace", workspace, U8, (ws_bytes, None))],
        [_int32("target", target), _int32("level", level)])
    consumed = _consumed(consumed, n, device, st)
    workspace = _workspace(device, ws_bytes, st, workspace, "compress_blocks_hc_opt_dest_size")
    _launch(device, "LZ4B200_compress_blocks_hc_opt_destSize", lib.LZ4B200_compress_blocks_hc_opt_destSize,
            src.data_ptr(), int(block_size), src_sizes.data_ptr() if src_sizes is not None else None, int(block_size),
            slots.data_ptr(), stride, int(target), int(level), out_sizes.data_ptr(), consumed.data_ptr(), n,
            workspace.data_ptr(), workspace.numel(), st.cuda_stream)
    return slots, out_sizes[:n], consumed[:n], stride


_PARSES = {"fast": 0, "parallel": 1, "hc": 2}     # LZ4B200_PARSE_FAST, _PARALLEL, _HC


def compress_buffers(src, offsets, sizes, parse="fast", acceleration=1, level=9, out=None, out_offsets=None,
                     capacities=None, out_sizes=None, workspace=None, stream=None):
    """Compress len(sizes) buffers of any sizes at any offsets of src in one call (LZ4B200_compress_blocks_indexed).

    src: u8 device buffer; buffer i = src[offsets[i] : offsets[i]+sizes[i]] (int64 / int32 device tensors).  Buffer i
    is compressed to out[out_offsets[i] : out_offsets[i]+capacities[i]] (int64 / int32 device tensors), and
    out_sizes[i] is what the one-block call returns for it:
      parse "fast":     LZ4_compress_fast(buf_i, out_i, sizes[i], capacities[i], acceleration), byte for byte;
      parse "parallel": the parallel parse of compress_blocks(mode="parallel") for buffers of up to 64 KB, "fast" above;
      parse "hc":       LZ4_compress_HC(buf_i, out_i, sizes[i], capacities[i], level) at levels 1 .. 12, byte for byte.
    capacities defaults to LZ4_compressBound(sizes), computed on the device; out_offsets to the exclusive sum of the
    capacities (those below 0 count as 0), so the outputs abut; out to their total, which is read on the host, so a
    captured call passes out.  Whether a given out holds what out_offsets and capacities place in it is the caller's
    responsibility.  workspace: "hc" only, at least LZ4B200_compress_blocks_indexed_workspace_bytes(n, 2, level) bytes
    (the module's rule above).  "parallel" reads the 16-byte granules around every buffer, "hc" the aligned 4-byte
    words around it: that memory must be readable.
    Returns (out, out_sizes, out_offsets, capacities).
    """
    lib = _lib.load()
    if parse not in _PARSES:
        raise ValueError("compress_buffers: parse must be 'fast', 'parallel' or 'hc' (got %r)" % (parse,))
    hc = parse == "hc"
    param = int(level) if hc else int(acceleration)
    n = int(sizes.numel())
    ws_bytes = max(int(lib.LZ4B200_compress_blocks_indexed_workspace_bytes(n, _PARSES[parse], param)), 1) if hc else 0
    at_least_n = (n, None)
    device, st = _checked("compress_buffers", stream,
                          [("src", src, U8, ANY), ("offsets", offsets, I64, at_least_n), ("sizes", sizes, I32, ANY),
                           ("out", out, U8, ANY), ("out_offsets", out_offsets, I64, at_least_n),
                           ("capacities", capacities, I32, (n, n)), ("out_sizes", out_sizes, I32, at_least_n),
                           ("workspace", workspace, U8, (ws_bytes, None))],
                          [_int32("acceleration", acceleration), _int32("level", level)])
    if hc:
        workspace = _workspace(device, ws_bytes, st, workspace, "compress_buffers")
    with torch.cuda.stream(st):                     # temporaries belong to the stream the kernels run on
        if capacities is None:                      # LZ4_compressBound: 0 outside 0 .. LZ4_MAX_INPUT_SIZE
            capacities = torch.where((sizes >= 0) & (sizes <= 0x7E000000), sizes + sizes // 255 + 16,
                                     torch.zeros_like(sizes))
        room = capacities.clamp(min=0).to(I64)
        if out_offsets is None:
            out_offsets = torch.cumsum(room, 0) - room
        if out is None:
            if torch.cuda.is_current_stream_capturing():
                raise ValueError("compress_buffers under stream capture needs out=")
            out = torch.empty(max(int(room.sum()) if n else 0, 1), dtype=torch.uint8, device=device)
        if out_sizes is None:
            out_sizes = torch.empty(max(n, 1), dtype=torch.int32, device=device)
    _launch(device, "LZ4B200_compress_blocks_indexed", lib.LZ4B200_compress_blocks_indexed, src.data_ptr(),
            offsets.data_ptr(), sizes.data_ptr(), out.data_ptr(), out_offsets.data_ptr(), capacities.data_ptr(),
            out_sizes.data_ptr(), n, _PARSES[parse], param, workspace.data_ptr() if workspace is not None else None,
            workspace.numel() if workspace is not None else 0, st.cuda_stream)
    return out, out_sizes[:n], out_offsets, capacities


def pack_blocks(slots, slot_stride, sizes, header_bytes=0, packed=None, stream=None, slot_offsets=None):
    """Gather variable-size blocks into one contiguous stream.  Returns (packed, offsets[n+1]).

    A given `packed` holds len(sizes) * (slot_stride + header_bytes) bytes: what the gather writes when every size fits
    its slot (a larger size is the caller's responsibility).
    slot_offsets: an int64 device tensor: block i's slot is slots[slot_offsets[i]:] (LZ4B200_pack_blocks_indexed), as
    compress_buffers leaves its outputs at out_offsets.  slot_stride may then be None: a given packed is not checked
    against it, and a new one is sized by the exact total of the sizes, which is read on the host (a captured call
    passes packed or slot_stride).  With slot_stride given, it bounds every block's size and sizes packed as above."""
    lib = _lib.load()
    n = int(sizes.numel())
    indexed = slot_offsets is not None
    room = n * (int(slot_stride) + int(header_bytes)) if slot_stride is not None or not indexed else None
    device, st = _checked("pack_blocks", stream,
                          [("slots", slots, U8, ANY), ("sizes", sizes, I32, ANY),
                           ("packed", packed, U8, (room or 0, None)), ("slot_offsets", slot_offsets, I64, (n, None))],
                          [_int32("header_bytes", header_bytes)],
                          [("slot_stride", slot_stride, 0)] if slot_stride is not None else [])
    with torch.cuda.stream(st):
        offsets = torch.empty(n + 1, dtype=torch.int64, device=device)
        if packed is None:
            if room is None:
                if torch.cuda.is_current_stream_capturing():
                    raise ValueError("pack_blocks under stream capture with slot_offsets needs packed= or slot_stride")
                room = (int(sizes.clamp(min=0).sum(dtype=I64)) if n else 0) + n * int(header_bytes)
            packed = torch.empty(room + 16, dtype=torch.uint8, device=device)
    if indexed:
        _launch(device, "LZ4B200_pack_blocks_indexed", lib.LZ4B200_pack_blocks_indexed, slots.data_ptr(),
                slot_offsets.data_ptr(), sizes.data_ptr(), n, packed.data_ptr(), offsets.data_ptr(), int(header_bytes),
                st.cuda_stream)
    else:
        _launch(device, "LZ4B200_pack_blocks", lib.LZ4B200_pack_blocks, slots.data_ptr(), int(slot_stride),
                sizes.data_ptr(), n, packed.data_ptr(), offsets.data_ptr(), int(header_bytes), st.cuda_stream)
    return packed, offsets
