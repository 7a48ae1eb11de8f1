"""ctypes loader for the CPU oracle -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference) may import
this.  `Oracle()` wraps oracle/liboracle.so (the plain-C restatement); `Reference()` wraps
oracle/_ref/libref_lz4.so (the unmodified reference lib/lz4.c + tests/datagen.c compiled by
oracle/Makefile) and raises FileNotFoundError when it has not been built.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "liboracle.so")
REF_SO = os.path.join(HERE, "_ref", "libref_lz4.so")

_u8p = C.POINTER(C.c_uint8)
_ip = C.POINTER(C.c_int)

# path codes of oracle_lz4_compress_destSize_extState (enum oracle_ds_path, lz4_oracle.h)
PATHS = {0: "fast", 1: "empty", 2: "no_room", 3: "literals", 4: "next_match", 5: "reduced", 6: "last_literals",
         7: "filled", 8: "bad_size"}


def build(quiet=True):
    """Compile liboracle.so (and _ref when /root/reference exists)."""
    out = subprocess.run(["make", "-C", HERE], capture_output=True, text=True)
    if out.returncode != 0:
        raise RuntimeError("oracle build failed:\n" + out.stdout + out.stderr)
    if not quiet:
        print(out.stdout)


def _ptr(a):
    return a.ctypes.data_as(_u8p)


def _as_u8(data):
    if isinstance(data, np.ndarray):
        assert data.dtype == np.uint8
        return np.ascontiguousarray(data)
    return np.frombuffer(bytes(data), dtype=np.uint8)


class _Codec:
    """Common python surface over (compress_fast, decompress_safe, compress_bound, compress_destSize,
    decompress_safe_partial)."""

    def compress_bound(self, n):
        return int(self._bound(int(n)))

    def compress(self, data, acceleration=1, capacity=None):
        """Returns (ret, bytes).  ret == 0 means failure (lz4.h:182-189)."""
        src = _as_u8(data)
        cap = self.compress_bound(len(src)) if capacity is None else int(capacity)
        dst = np.zeros(max(cap, 1) + 64, dtype=np.uint8)
        dst[cap:] = 0xA5  # guard
        r = int(self._compress(_ptr(src) if len(src) else None, _ptr(dst), len(src), cap, int(acceleration)))
        assert (dst[max(cap, 0):max(cap, 0) + 64] == 0xA5).all() or cap < 0, "compressor wrote past dstCapacity"
        return r, dst[:max(r, 0)].tobytes()

    def decompress(self, data, capacity):
        """Returns (ret, bytes) with bytes = dst[0:ret] when ret >= 0 (lz4.h:192-208)."""
        src = _as_u8(data)
        cap = int(capacity)
        dst = np.zeros(max(cap, 0) + 64, dtype=np.uint8)
        dst[max(cap, 0):] = 0xA5
        srcp = _ptr(src) if len(src) else _ptr(np.zeros(1, dtype=np.uint8))
        r = int(self._decompress(srcp, _ptr(dst), len(src), cap))
        assert (dst[max(cap, 0):] == 0xA5).all(), "decoder wrote past dstCapacity"
        return r, dst[:max(r, 0)].tobytes()

    def compress_dest_size(self, data, target, acceleration=None):
        """LZ4_compress_destSize (acceleration None) or LZ4_compress_destSize_extState (lz4.h:248-272, :613-617).  Returns
        (ret, consumed, bytes, path): consumed is what the call leaves in *srcSizePtr, path the oracle's route code
        (PATHS) or None for the reference."""
        src = _as_u8(data)
        room = max(int(target), 0)
        dst = np.full(room + 64, 0xA5, dtype=np.uint8)
        n = C.c_int(len(src))
        r, path = self._dest_size(_ptr(src) if len(src) else None, _ptr(dst), n, int(target), acceleration)
        assert (dst[room:] == 0xA5).all(), "destSize wrote at or past targetDstSize"
        return r, n.value, dst[:max(r, 0)].tobytes(), path

    def decompress_partial(self, data, target, capacity=None):
        """LZ4_decompress_safe_partial(src, dst, len(data), target, capacity) (lz4.h:274-308), capacity defaulting to
        target, into a zeroed dst.  Returns (ret, bytes)."""
        return self._decompress_partial(data, target, capacity)[:2]

    def _decompress_partial(self, data, target, capacity):
        """(ret, bytes, lastPath) after checking that nothing at or past outputSize = min(target, capacity) was written"""
        cap = int(target) if capacity is None else int(capacity)
        src = _as_u8(data) if len(data) else np.zeros(1, dtype=np.uint8)
        room = max(min(int(target), cap), 0)
        dst = np.zeros(room + 64, dtype=np.uint8)
        dst[room:] = 0xA5
        r, last = self._partial(_ptr(src), _ptr(dst), len(data), int(target), cap)
        assert (dst[room:] == 0xA5).all(), "partial decode wrote at or past outputSize"
        return r, dst[:max(r, 0)].tobytes(), last


class Oracle(_Codec):
    name = "port"

    def __init__(self):
        if not os.path.exists(ORACLE_SO):
            build()
        self.lib = lib = C.CDLL(ORACLE_SO)
        lib.oracle_lz4_compress_bound.restype = C.c_int
        lib.oracle_lz4_compress_bound.argtypes = [C.c_int]
        lib.oracle_lz4_compress_fast.restype = C.c_int
        lib.oracle_lz4_compress_fast.argtypes = [_u8p, _u8p, C.c_int, C.c_int, C.c_int]
        lib.oracle_lz4_decompress_safe.restype = C.c_int
        lib.oracle_lz4_decompress_safe.argtypes = [_u8p, _u8p, C.c_int, C.c_int]
        lib.oracle_lz4_compress_destSize_extState.restype = C.c_int
        lib.oracle_lz4_compress_destSize_extState.argtypes = [_u8p, _u8p, _ip, C.c_int, C.c_int, _ip]
        lib.oracle_lz4_decompress_safe_partial.restype = C.c_int
        lib.oracle_lz4_decompress_safe_partial.argtypes = [_u8p, _u8p, C.c_int, C.c_int, C.c_int, _ip]
        lib.oracle_datagen.restype = None
        lib.oracle_datagen.argtypes = [_u8p, C.c_size_t, C.c_double, C.c_double, C.c_uint]
        lib.oracle_datagen_mt.restype = None
        lib.oracle_datagen_mt.argtypes = [_u8p, C.c_size_t, C.c_size_t, C.c_double, C.c_uint, C.c_int]
        lib.oracle_lz4_block_stats.restype = C.c_int
        lib.oracle_lz4_block_stats.argtypes = [_u8p, C.c_int, C.c_void_p]
        lib.oracle_time_decompress.restype = C.c_double
        lib.oracle_time_decompress.argtypes = [C.c_void_p, _u8p, C.c_void_p, C.c_void_p, _u8p, C.c_int64,
                                               C.c_int32, C.c_void_p, C.c_int64, C.c_int]
        lib.oracle_time_compress.restype = C.c_double
        lib.oracle_time_compress.argtypes = [C.c_void_p, _u8p, C.c_int64, C.c_int32, C.c_int64, _u8p, C.c_int64,
                                             C.c_int32, C.c_int, C.c_void_p, C.c_int64, C.c_int]
        lib.oracle_first_touch.restype = None
        lib.oracle_first_touch.argtypes = [_u8p, C.c_int64, C.c_int64, C.c_int]
        lib.oracle_pack.restype = None
        lib.oracle_pack.argtypes = [_u8p, C.c_int64, C.c_void_p, C.c_void_p, _u8p, C.c_int64, C.c_int]
        self._bound = lib.oracle_lz4_compress_bound
        self._compress = lib.oracle_lz4_compress_fast
        self._decompress = lib.oracle_lz4_decompress_safe

    def _dest_size(self, sp, dp, n, target, acceleration):
        path = C.c_int(-1)
        acc = 1 if acceleration is None else int(acceleration)
        r = self.lib.oracle_lz4_compress_destSize_extState(sp, dp, C.byref(n), target, acc, C.byref(path))
        return int(r), path.value

    def _partial(self, sp, dp, size, target, cap):
        last = C.c_int(0)
        r = self.lib.oracle_lz4_decompress_safe_partial(sp, dp, size, target, cap, C.byref(last))
        return int(r), last.value

    def decompress_partial_traced(self, data, target, capacity=None):
        """decompress_partial plus how the decode ended: (ret, bytes, last_path, dst_dependent).  last_path is 1 after
        literals, 2 inside a match, 0 otherwise; dst_dependent says whether the reference's bytes depend on what dst
        held (an offset-0 match on its cut path, lz4.c:2392-2404), where the oracle writes zeros."""
        r, out, last = self._decompress_partial(data, target, capacity)
        return r, out, last & 3, bool(last & 4)

    # --- data generator (tests/datagen.c RDG_genBuffer) ---
    def datagen(self, size, proba=0.5, seed=0, lit_proba=0.0):
        buf = np.empty(int(size), dtype=np.uint8)
        if size:
            self.lib.oracle_datagen(_ptr(buf), int(size), float(proba), float(lit_proba), int(seed))
        return buf

    def datagen_mt(self, size, seg_bytes, proba=0.5, seed0=0, threads=None, out=None):
        """Segment k (seg_bytes each) = RDG_genBuffer(seg, proba, 0.0, seed0 + k) (SURVEY 8(d) C2)."""
        threads = threads or os.cpu_count() or 1
        buf = np.empty(int(size), dtype=np.uint8) if out is None else out
        self.lib.oracle_datagen_mt(_ptr(buf), int(size), int(seg_bytes), float(proba), int(seed0), int(threads))
        return buf

    def block_stats(self, data):
        class S(C.Structure):
            _fields_ = [("n_sequences", C.c_uint32), ("literal_bytes", C.c_uint32),
                        ("match_bytes", C.c_uint32), ("overlap_matches", C.c_uint32)]
        src = _as_u8(data)
        s = S()
        r = self.lib.oracle_lz4_block_stats(_ptr(src), len(src), C.byref(s))
        if r != 0:
            raise ValueError("not a valid block")
        return dict(n_sequences=s.n_sequences, literal_bytes=s.literal_bytes,
                    match_bytes=s.match_bytes, overlap_matches=s.overlap_matches)

    # --- timing harness: `codec` is an Oracle or Reference whose function pointers are timed ---
    def time_decompress(self, codec, comp, offsets, sizes, out, block_size, threads):
        """comp: u8 array; offsets int64[n]; sizes int32[n]; out: u8 array n*block_size."""
        n = len(sizes)
        rets = np.zeros(n, dtype=np.int32)
        fn = C.cast(codec._decompress, C.c_void_p)
        t = self.lib.oracle_time_decompress(fn, _ptr(comp), offsets.ctypes.data, sizes.ctypes.data, _ptr(out),
                                            int(block_size), int(block_size), rets.ctypes.data, n, int(threads))
        return t, rets

    def first_touch(self, buf, stride, n, threads):
        """zero-fill buf (n x stride bytes) with the worker partition / CPU pinning of the timed passes"""
        self.lib.oracle_first_touch(_ptr(buf), int(stride), int(n), int(threads))

    def pack(self, slots, stride, sizes, offsets, packed, threads):
        self.lib.oracle_pack(_ptr(slots), int(stride), sizes.ctypes.data, offsets.ctypes.data, _ptr(packed),
                             len(sizes), int(threads))

    def time_compress(self, codec, src, block_size, out, out_stride, accel, threads):
        n = (len(src) + block_size - 1) // block_size
        last = len(src) - (n - 1) * block_size
        rets = np.zeros(n, dtype=np.int32)
        fn = C.cast(codec._compress, C.c_void_p)
        t = self.lib.oracle_time_compress(fn, _ptr(src), int(block_size), int(block_size), int(last), _ptr(out),
                                          int(out_stride), int(out_stride), int(accel), rets.ctypes.data, n,
                                          int(threads))
        return t, rets


class Reference(_Codec):
    name = "reference"

    def __init__(self):
        if not os.path.exists(REF_SO):
            raise FileNotFoundError(REF_SO + " (run `make -C oracle ref` where /root/reference exists)")
        self.lib = lib = C.CDLL(REF_SO)
        lib.LZ4_compressBound.restype = C.c_int
        lib.LZ4_compressBound.argtypes = [C.c_int]
        lib.LZ4_compress_fast.restype = C.c_int
        lib.LZ4_compress_fast.argtypes = [_u8p, _u8p, C.c_int, C.c_int, C.c_int]
        lib.LZ4_decompress_safe.restype = C.c_int
        lib.LZ4_decompress_safe.argtypes = [_u8p, _u8p, C.c_int, C.c_int]
        lib.LZ4_compress_destSize.restype = C.c_int
        lib.LZ4_compress_destSize.argtypes = [_u8p, _u8p, _ip, C.c_int]
        lib.LZ4_compress_destSize_extState.restype = C.c_int
        lib.LZ4_compress_destSize_extState.argtypes = [C.c_void_p, _u8p, _u8p, _ip, C.c_int, C.c_int]
        lib.LZ4_decompress_safe_partial.restype = C.c_int
        lib.LZ4_decompress_safe_partial.argtypes = [_u8p, _u8p, C.c_int, C.c_int, C.c_int]
        lib.RDG_genBuffer.restype = None
        lib.RDG_genBuffer.argtypes = [_u8p, C.c_size_t, C.c_double, C.c_double, C.c_uint]
        self._bound = lib.LZ4_compressBound
        self._compress = lib.LZ4_compress_fast
        self._decompress = lib.LZ4_decompress_safe
        self.ext_state = np.zeros(16416 // 8, dtype=np.uint64)     # sizeof(LZ4_stream_t), lz4.h:729-733

    def _dest_size(self, sp, dp, n, target, acceleration):
        if acceleration is None:
            return int(self.lib.LZ4_compress_destSize(sp, dp, C.byref(n), target)), None
        return int(self.lib.LZ4_compress_destSize_extState(self.ext_state.ctypes.data, sp, dp, C.byref(n), target,
                                                           int(acceleration))), None

    def _partial(self, sp, dp, size, target, cap):
        return int(self.lib.LZ4_decompress_safe_partial(sp, dp, size, target, cap)), 0

    def datagen(self, size, proba=0.5, seed=0, lit_proba=0.0):
        buf = np.empty(int(size), dtype=np.uint8)
        if size:
            self.lib.RDG_genBuffer(_ptr(buf), int(size), float(proba), float(lit_proba), int(seed))
        return buf

    # --- frame layer (lib/lz4frame.c), used to pin LZ4B200_compressFrame_host / decompressFrame_host ---
    class _FrameInfo(C.Structure):          # LZ4F_frameInfo_t, lz4frame.h:175-183
        _fields_ = [("blockSizeID", C.c_int), ("blockMode", C.c_int), ("contentChecksumFlag", C.c_int),
                    ("frameType", C.c_int), ("contentSize", C.c_ulonglong), ("dictID", C.c_uint),
                    ("blockChecksumFlag", C.c_int)]

    def have_frame(self):
        return hasattr(self.lib, "LZ4F_compressFrame")

    def compress_frame(self, data, block_size_id=4, level=0, content_size=False, block_mode=1,
                       content_checksum=0, block_checksum=0, capacity=None):
        """LZ4F_compressFrame (lz4frame.c:484) with the given preferences into capacity bytes (default: its
        LZ4F_compressFrameBound); returns the frame bytes, RuntimeError when the call fails."""
        lib = self.lib
        class Prefs(C.Structure):              # LZ4F_preferences_t, lz4frame.h:192-198
            _fields_ = [("frameInfo", Reference._FrameInfo), ("compressionLevel", C.c_int), ("autoFlush", C.c_uint),
                        ("favorDecSpeed", C.c_uint), ("reserved", C.c_uint * 3)]
        p = Prefs()
        p.frameInfo.blockSizeID = block_size_id
        p.frameInfo.blockMode = block_mode                 # 1 = LZ4F_blockIndependent
        p.frameInfo.contentChecksumFlag = content_checksum
        p.frameInfo.blockChecksumFlag = block_checksum
        p.frameInfo.contentSize = 1 if content_size else 0   # any non-zero value: replaced by srcSize (lz4frame.c:445)
        p.compressionLevel = level
        src = _as_u8(data)
        lib.LZ4F_compressFrameBound.restype = C.c_size_t
        lib.LZ4F_compressFrameBound.argtypes = [C.c_size_t, C.c_void_p]
        lib.LZ4F_compressFrame.restype = C.c_size_t
        lib.LZ4F_compressFrame.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
        lib.LZ4F_isError.restype = C.c_uint
        lib.LZ4F_isError.argtypes = [C.c_size_t]
        cap = lib.LZ4F_compressFrameBound(len(src), C.byref(p)) if capacity is None else int(capacity)
        dst = np.empty(max(cap, 1), dtype=np.uint8)
        r = lib.LZ4F_compressFrame(dst.ctypes.data, cap, src.ctypes.data if len(src) else None, len(src), C.byref(p))
        if lib.LZ4F_isError(r):
            raise RuntimeError("LZ4F_compressFrame failed")
        return dst[:r].tobytes()

    def decompress_frame(self, frame, capacity):
        """LZ4F_decompress (lz4frame.c:1613) of one whole frame; returns the decoded bytes."""
        lib = self.lib
        lib.LZ4F_createDecompressionContext.restype = C.c_size_t
        lib.LZ4F_createDecompressionContext.argtypes = [C.POINTER(C.c_void_p), C.c_uint]
        lib.LZ4F_freeDecompressionContext.argtypes = [C.c_void_p]
        lib.LZ4F_decompress.restype = C.c_size_t
        lib.LZ4F_decompress.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t), C.c_void_p,
                                        C.POINTER(C.c_size_t), C.c_void_p]
        lib.LZ4F_isError.restype = C.c_uint
        lib.LZ4F_isError.argtypes = [C.c_size_t]
        ctx = C.c_void_p()
        assert not lib.LZ4F_isError(lib.LZ4F_createDecompressionContext(C.byref(ctx), 100))
        src = _as_u8(frame)
        dst = np.empty(max(int(capacity), 1), dtype=np.uint8)
        sp, dp = 0, 0
        try:
            while sp < len(src):
                ssz = C.c_size_t(len(src) - sp)
                dsz = C.c_size_t(int(capacity) - dp)
                r = lib.LZ4F_decompress(ctx, dst.ctypes.data + dp, C.byref(dsz), src.ctypes.data + sp, C.byref(ssz), None)
                if lib.LZ4F_isError(r):
                    raise RuntimeError("LZ4F_decompress failed")
                sp += ssz.value
                dp += dsz.value
                if r == 0:
                    break
                if ssz.value == 0 and dsz.value == 0:
                    raise RuntimeError("LZ4F_decompress made no progress (dst too small?)")
        finally:
            lib.LZ4F_freeDecompressionContext(ctx)
        return dst[:dp].tobytes()


def have_reference():
    return os.path.exists(REF_SO)
