"""One-shot LZ4 frames of independent blocks (SURVEY.md section 8 f-1): the Python face of
LZ4B200_compressFrame_host / LZ4B200_decompressFrame_host (the roles of LZ4F_compressFrame,
lz4frame.h:224, and of a one-shot LZ4F_decompress, lz4frame.h:470), of LZ4B200_decompress_files_host:
whole .lz4 files in host memory decoded as `lz4 -d` decodes them, of LZ4B200_compress_frames_host and
LZ4B200_compress_legacy_host: whole .lz4 files written from host memory as the `lz4` tool writes them, and of their
device-resident ends: LZ4B200_decompress_files_to_device (files in host memory decoded into CUDA tensors) and
LZ4B200_compress_frames_from_device / LZ4B200_compress_legacy_from_device (CUDA tensors written as .lz4 files in host
memory)."""
import ctypes as C

import numpy as np

from . import _lib
from .block import _c_int, _u8


class Lz4FrameError(RuntimeError):
    def __init__(self, code, what):
        names = {-1: "bad argument", -2: "CUDA error", -3: "malformed frame", -4: "unsupported frame feature",
                 -5: "destination too small", -6: "over the call's budget", -7: "checksum mismatch"}
        super().__init__("%s: %s (%d)" % (what, names.get(int(code), "error"), int(code)))
        self.code = int(code)


def compress_frame(data, block_size_id=4, level=0, content_size=False):
    lib = _lib.load()
    src = _u8(data)
    cap = int(lib.LZ4B200_compressFrameBound(len(src), int(block_size_id)))
    if cap < 0:
        raise Lz4FrameError(cap, "LZ4B200_compressFrameBound")
    dst = np.empty(cap, dtype=np.uint8)
    r = int(lib.LZ4B200_compressFrame_host(src.ctypes.data if len(src) else None, len(src), dst.ctypes.data, cap,
                                           int(block_size_id), int(level), 1 if content_size else 0))
    if r < 0:
        raise Lz4FrameError(r, "LZ4B200_compressFrame_host")
    return dst[:r].tobytes()


def decompress_frame(frame, capacity):
    lib = _lib.load()
    src = _u8(frame)
    dst = np.empty(max(int(capacity), 1), dtype=np.uint8)
    consumed = C.c_int64(0)
    r = int(lib.LZ4B200_decompressFrame_host(src.ctypes.data, len(src), dst.ctypes.data, int(capacity), C.byref(consumed)))
    if r < 0:
        raise Lz4FrameError(r, "LZ4B200_decompressFrame_host")
    return dst[:r].tobytes()


def _i64(name, v):
    v = int(v)
    if not -2 ** 63 <= v < 2 ** 63:
        raise ValueError("%s = %d does not fit an int64" % (name, v))
    return v


def _files_call(src, offs, sizes, caps, skip_checksums, size_only):
    """one LZ4B200_decompress_files_host call: (results, consumed, prefixes, output or None)"""
    lib = _lib.load()
    n = len(offs)
    i64 = lambda a: np.ascontiguousarray(a, dtype=np.int64)
    offs, sizes = i64(offs), i64(sizes)
    res, con, pre = (np.zeros(n, dtype=np.int64) for _ in range(3))
    out = dst_offs = caps_a = None
    if not size_only:
        caps_a = i64(caps)
        dst_offs = np.zeros(n, dtype=np.int64)
        room = np.maximum(caps_a, 0)
        dst_offs[1:] = np.cumsum(room)[:-1]
        out = np.empty(max(int(room.sum()), 1), dtype=np.uint8)
    ptr = lambda a: a.ctypes.data if a is not None else None
    rc = int(lib.LZ4B200_decompress_files_host(src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, ptr(out),
                                               ptr(dst_offs), ptr(caps_a), res.ctypes.data, con.ctypes.data,
                                               pre.ctypes.data, n, 1 if skip_checksums else 0, 1 if size_only else 0))
    if rc < 0:
        raise Lz4FrameError(rc, "LZ4B200_decompress_files_host")
    return res.tolist(), con.tolist(), pre.tolist(), (out, dst_offs)


def _files_input(datas, capacities):
    """the files back to back in one host buffer: (src, offs, sizes, capacities checked or None)"""
    parts = [_u8(d) for d in datas]
    n = len(parts)
    sizes = [len(p) for p in parts]
    offs = np.zeros(n, dtype=np.int64)
    if n:
        offs[1:] = np.cumsum(sizes)[:-1]
    src = np.concatenate(parts) if n and sum(sizes) else np.zeros(1, dtype=np.uint8)
    if capacities is not None:
        capacities = [_i64("capacity", c) for c in capacities]
        if len(capacities) != n:
            raise ValueError("capacities has %d values for %d files" % (len(capacities), n))
    return src, offs, sizes, capacities


def _sized_capacities(src, offs, sizes, skip_checksums):
    """the size-only pass at unlimited room and the room it gives each file: a file that fails there is given its
    prefix as room, so that the decoding pass finds the content checksums of the units before the failing one"""
    sized = _files_call(src, offs, sizes, None, skip_checksums, True)
    return sized, [r if r >= 0 else p for r, p in zip(sized[0], sized[2])]


def _verdict(sized, k, r, c, p):
    """file k's (result, consumed, prefix), keeping the size-only pass's answer when the file fails there and, with the
    room that pass gave it, at that same unit"""
    if sized is not None and sized[0][k] < 0 and r < 0 and c == sized[1][k]:
        return sized[0][k], sized[1][k], sized[2][k]
    return r, c, p


def decompress_files(datas, capacities=None, skip_checksums=False, size_only=False):
    """Decode whole .lz4 files (concatenated frames, skippable frames, `lz4 -l` legacy streams) from host memory, as
    LZ4B200_decompress_files_host does.  Per file: (result, consumed, prefix, data) -- result the decoded size or the
    file's error code, consumed the failing unit's offset (the file's size on success), prefix the bytes decoded before
    it, and data the decoded bytes (the prefix's bytes on failure; None with size_only).  capacities: each file's room;
    None runs the size-only pass first and gives each file its decoded size, so that every result is the one at
    unlimited room."""
    src, offs, sizes, capacities = _files_input(datas, capacities)
    n = len(sizes)
    if size_only:
        res, con, pre, _ = _files_call(src, offs, sizes, None, skip_checksums, True)
        return [(r, c, p, None) for r, c, p in zip(res, con, pre)]
    sized = None
    if capacities is None:
        sized, capacities = _sized_capacities(src, offs, sizes, skip_checksums)
    res, con, pre, (out, dst_offs) = _files_call(src, offs, sizes, capacities, skip_checksums, False)
    got = []
    for k in range(n):
        r, c, p = _verdict(sized, k, res[k], con[k], pre[k])
        o = int(dst_offs[k])
        got.append((r, c, p, out[o:o + (r if r >= 0 else p)].tobytes()))
    return got


def decompress_file(data, capacity=None, skip_checksums=False):
    """One whole .lz4 file from host memory: its decoded bytes, or Lz4FrameError with the file's code.  capacity=None
    sizes the output with the size-only pass first."""
    (r, _, _, b), = decompress_files([data], None if capacity is None else [capacity], skip_checksums)
    if r < 0:
        raise Lz4FrameError(r, "LZ4B200_decompress_files_host")
    return b


def decompress_files_to_device(datas, capacities=None, skip_checksums=False):
    """Decode whole .lz4 files from host memory into device memory (LZ4B200_decompress_files_to_device): per file
    (result, consumed, prefix, tensor), what decompress_files returns for the same arguments, with the decoded bytes (the
    prefix's on failure) as a CUDA uint8 tensor on the current device.  The tensors are views of one allocation, each
    starting 16-byte aligned.  The call runs after the work on torch.cuda.current_stream() and its bytes are written
    when it returns.  capacities=None sizes the files with the host call's size-only pass first."""
    import torch
    src, offs, sizes, capacities = _files_input(datas, capacities)
    n = len(sizes)
    if n == 0:
        return []
    sized = None
    if capacities is None:
        sized, capacities = _sized_capacities(src, offs, sizes, skip_checksums)
    caps = np.array(capacities, dtype=np.int64)
    sizes = np.array(sizes, dtype=np.int64)
    room = (np.maximum(caps, 0) + 15) // 16 * 16
    dst_offs = np.zeros(n, dtype=np.int64)
    dst_offs[1:] = np.cumsum(room)[:-1]
    out = torch.empty(max(int(room.sum()), 1), dtype=torch.uint8, device="cuda")
    res, con, pre = (np.zeros(n, dtype=np.int64) for _ in range(3))
    rc = int(_lib.load().LZ4B200_decompress_files_to_device(
        src.ctypes.data, offs.ctypes.data, sizes.ctypes.data, out.data_ptr(), dst_offs.ctypes.data, caps.ctypes.data,
        res.ctypes.data, con.ctypes.data, pre.ctypes.data, n, 1 if skip_checksums else 0,
        torch.cuda.current_stream().cuda_stream))
    if rc < 0:
        raise Lz4FrameError(rc, "LZ4B200_decompress_files_to_device")
    got = []
    for k in range(n):
        r, c, p = _verdict(sized, k, int(res[k]), int(con[k]), int(pre[k]))
        o = int(dst_offs[k])
        got.append((r, c, p, out[o:o + (r if r >= 0 else p)]))
    return got


def decompress_file_to_device(data, capacity=None, skip_checksums=False):
    """One whole .lz4 file from host memory into a CUDA uint8 tensor, or Lz4FrameError with the file's code.
    capacity=None sizes the output with the size-only pass first."""
    (r, _, _, t), = decompress_files_to_device([data], None if capacity is None else [capacity], skip_checksums)
    if r < 0:
        raise Lz4FrameError(r, "LZ4B200_decompress_files_to_device")
    return t


# the `lz4` tool's defaults for a frame: -1, 4 MB blocks (-B7), a content checksum, no block checksums, no content size
_FRAME_DEFAULTS = dict(block_size_id=7, content_size=False, block_checksum=False, content_checksum=True, parallel=False)


def _check_legacy(legacy, block_size_id, content_size, block_checksum, content_checksum, parallel):
    """ValueError for legacy=True with a frame-only argument away from its default"""
    frame_args = dict(block_size_id=block_size_id, content_size=content_size, block_checksum=block_checksum,
                      content_checksum=content_checksum, parallel=parallel)
    if legacy and any(frame_args[k] != v for k, v in _FRAME_DEFAULTS.items()):
        raise ValueError("legacy streams take no %s" % ", ".join(k for k, v in _FRAME_DEFAULTS.items()
                                                                  if frame_args[k] != v))


def _write_files(src, offs, sizes, stream, level, block_size_id, content_size, block_checksum, content_checksum,
                 parallel, legacy):
    """one writer call over the sources at src + offs[k], sizes[k] bytes: src a host address, or with stream (a CUDA
    stream handle) not None a device address.  Every output is sized at its bound; one bytes per source."""
    lib = _lib.load()
    level = _c_int("level", level)
    bsid = _c_int("block_size_id", block_size_id)
    n = len(sizes)
    sizes = np.array(sizes, dtype=np.int64)
    if legacy:
        caps = [int(lib.LZ4B200_compressLegacyBound(int(k))) for k in sizes]
    else:
        caps = [int(lib.LZ4B200_compressFrameBound_checksummed(int(k), bsid, int(bool(block_checksum)),
                                                               int(bool(content_checksum)))) for k in sizes]
        if any(c < 0 for c in caps):
            raise Lz4FrameError(min(caps), "LZ4B200_compressFrameBound_checksummed")
    caps = np.array(caps, dtype=np.int64)
    dst_offs = np.zeros(n, dtype=np.int64)
    if n:
        dst_offs[1:] = np.cumsum(caps)[:-1]
    out = np.empty(max(int(caps.sum()), 1), dtype=np.uint8)
    res = np.zeros(n, dtype=np.int64)
    args = [src, offs.ctypes.data, sizes.ctypes.data, out.ctypes.data, dst_offs.ctypes.data, caps.ctypes.data,
            res.ctypes.data, n]
    if legacy:
        args.append(level)
    else:
        args += [bsid, level, int(bool(content_size)), int(bool(parallel)), int(bool(block_checksum)),
                 int(bool(content_checksum))]
    name = "LZ4B200_compress_%s_%s" % ("legacy" if legacy else "frames", "host" if stream is None else "from_device")
    rc = int(getattr(lib, name)(*(args if stream is None else args + [stream])))
    if rc < 0:
        raise Lz4FrameError(rc, name)
    for r in res:
        if r < 0:
            raise Lz4FrameError(int(r), name)
    return [out[int(o):int(o) + int(r)].tobytes() for o, r in zip(dst_offs, res)]


def compress_files(datas, level=1, block_size_id=7, content_size=False, block_checksum=False, content_checksum=True,
                   parallel=False, legacy=False):
    """Write whole .lz4 files from host memory (LZ4B200_compress_frames_host, or LZ4B200_compress_legacy_host with
    legacy=True): one bytes per input, what `lz4 -c -<level> [-B<id>] [--BX] [--no-frame-crc] [--content-size]` (or
    `lz4 -l -c -<level>`) writes for it.  The defaults are the tool's, not compress_frame's.  Every output is sized at
    its bound, so valid input gives no per-file error.  legacy=True with a frame-only argument away from its default
    raises ValueError."""
    _check_legacy(legacy, block_size_id, content_size, block_checksum, content_checksum, parallel)
    _c_int("level", level)
    parts = [_u8(d) for d in datas]
    n = len(parts)
    sizes = np.array([len(p) for p in parts], dtype=np.int64)
    offs = np.zeros(n, dtype=np.int64)
    if n:
        offs[1:] = np.cumsum(sizes)[:-1]
    src = np.concatenate(parts) if n and int(sizes.sum()) else np.zeros(1, dtype=np.uint8)
    return _write_files(src.ctypes.data, offs, sizes, None, level, block_size_id, content_size, block_checksum,
                        content_checksum, parallel, legacy)


def compress_file(data, **kwargs):
    """One whole .lz4 file from host memory: compress_files([data], **kwargs)[0]"""
    return compress_files([data], **kwargs)[0]


def compress_files_from_device(tensors, level=1, block_size_id=7, content_size=False, block_checksum=False,
                               content_checksum=True, parallel=False, legacy=False):
    """Write whole .lz4 files from CUDA tensors into host memory (LZ4B200_compress_frames_from_device, or
    LZ4B200_compress_legacy_from_device with legacy=True): one bytes per tensor, what compress_files writes for the
    tensor's contiguous bytes, whatever its dtype.  The arguments, defaults and legacy checks are compress_files'.  The
    tensors are read where they lie, after the work on torch.cuda.current_stream().  ValueError for a CPU tensor, a
    non-contiguous tensor or a tensor on another device than the current one."""
    _check_legacy(legacy, block_size_id, content_size, block_checksum, content_checksum, parallel)
    import torch
    tensors = list(tensors)
    for k, t in enumerate(tensors):
        if not isinstance(t, torch.Tensor):
            raise ValueError("source %d is not a tensor" % k)
        if not t.is_cuda:
            raise ValueError("source %d is a CPU tensor: compress_files takes host memory" % k)
        if not t.is_contiguous():
            raise ValueError("source %d is not contiguous" % k)
    if tensors:
        dev = torch.cuda.current_device()
        for k, t in enumerate(tensors):
            if t.device.index != dev:
                raise ValueError("source %d is on cuda:%d, not the current device cuda:%d" % (k, t.device.index, dev))
    sizes = [t.numel() * t.element_size() for t in tensors]
    # one base address with each source at its offset from it (device addresses are one flat space); an empty call or
    # one of empty sources still passes device memory as the base
    base = torch.empty(16, dtype=torch.uint8, device="cuda")
    ptrs = [t.data_ptr() for t, n in zip(tensors, sizes) if n] or [base.data_ptr()]
    lo = min(ptrs)
    offs = np.array([t.data_ptr() - lo if n else 0 for t, n in zip(tensors, sizes)], dtype=np.int64)
    return _write_files(lo, offs, sizes, torch.cuda.current_stream().cuda_stream, level, block_size_id, content_size,
                        block_checksum, content_checksum, parallel, legacy)


def compress_file_from_device(tensor, **kwargs):
    """One whole .lz4 file from a CUDA tensor: compress_files_from_device([tensor], **kwargs)[0]"""
    return compress_files_from_device([tensor], **kwargs)[0]
