"""ctypes binding of liblz4_b200.so (the C ABI declared in include/lz4_b200.h).

The library is built in-tree by lz4_b200.build (nvcc, sm_90a).  There is no fallback: if the
shared object is missing this module raises, and every codec call fails on a machine without a
CUDA device.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# LZ4_B200_LIBRARY=<path> loads a developer variant built with `python -m lz4_b200.build --out <path> -D...`
LIB_PATH = os.environ.get("LZ4_B200_LIBRARY") or os.path.join(_HERE, "liblz4_b200.so")

# every symbol include/lz4_b200.h declares: (name, restype, argtypes)
_vp, _i32, _i64, _sz = C.c_void_p, C.c_int32, C.c_int64, C.c_size_t
PROTOTYPES = [
    ("LZ4_versionNumber", C.c_int, []),
    ("LZ4_versionString", C.c_char_p, []),
    ("LZ4_compressBound", C.c_int, [C.c_int]),
    ("LZ4_sizeofState", C.c_int, []),
    ("LZ4_compress_default", C.c_int, [_vp, _vp, C.c_int, C.c_int]),
    ("LZ4_compress_fast", C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int]),
    ("LZ4_compress_fast_extState", C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int]),
    ("LZ4_compress_fast_extState_fastReset", C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int]),
    ("LZ4_compress_destSize", C.c_int, [_vp, _vp, C.POINTER(C.c_int), C.c_int]),
    ("LZ4_compress_destSize_extState", C.c_int, [_vp, _vp, _vp, C.POINTER(C.c_int), C.c_int, C.c_int]),
    ("LZ4_sizeofStateHC", C.c_int, []),
    ("LZ4_compress_HC", C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int]),
    ("LZ4_compress_HC_extStateHC", C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int]),
    ("LZ4_compress_HC_extStateHC_fastReset", C.c_int, [_vp, _vp, _vp, C.c_int, C.c_int, C.c_int]),
    ("LZ4_compress_HC_destSize", C.c_int, [_vp, _vp, _vp, C.POINTER(C.c_int), C.c_int, C.c_int]),
    ("LZ4_decompress_safe", C.c_int, [_vp, _vp, C.c_int, C.c_int]),
    ("LZ4_decompress_safe_partial", C.c_int, [_vp, _vp, C.c_int, C.c_int, C.c_int]),
    ("LZ4_decompress_safe_usingDict", C.c_int, [_vp, _vp, C.c_int, C.c_int, _vp, C.c_int]),
    ("LZ4B200_device_count", C.c_int, []),
    ("LZ4B200_last_cuda_error", C.c_char_p, []),
    ("LZ4B200_launch_count", C.c_uint64, []),
    ("LZ4B200_decompress_workspace_bytes", _sz, [_i64]),
    ("LZ4B200_decompress_workspace_bytes_for", _sz, [_i64, C.c_int, _i32]),
    ("LZ4B200_decompress_blocks", C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _vp, _i64, _vp, _sz, _vp]),
    ("LZ4B200_decompress_blocks_phased", C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _vp, _i64, _vp, _sz, C.c_int, _vp]),
    ("LZ4B200_decompress_blocks_partial", C.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _vp, _i64, _vp, _sz, _vp]),
    ("LZ4B200_decompress_frames_workspace_bytes", _sz, [_i64, C.POINTER(_i64)]),
    ("LZ4B200_decompress_frames", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.POINTER(_i64), _vp, _sz, _vp]),
    ("LZ4B200_decompress_frames_checksummed", C.c_int,
     [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.POINTER(_i64), C.c_int, _vp, _sz, _vp]),
    ("LZ4B200_decompress_files_workspace_bytes", _sz, [_i64, _i64, C.POINTER(_i64)]),
    ("LZ4B200_decompress_files", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, C.POINTER(_i64),
                                           C.c_int, C.c_int, _vp, _sz, _vp]),
    ("LZ4B200_compress_frames_workspace_bytes", _sz, [_i64, C.POINTER(_i64), C.c_int]),
    ("LZ4B200_compress_frames", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, C.c_int, C.c_int, C.c_int,
                                          C.POINTER(_i64), _vp, _sz, _vp]),
    ("LZ4B200_compress_frames_checksummed", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, C.c_int, C.c_int,
                                                      C.c_int, C.c_int, C.c_int, C.POINTER(_i64), _vp, _sz, _vp]),
    ("LZ4B200_compressLegacyBound", _i64, [_i64]),
    ("LZ4B200_compress_legacy_workspace_bytes", _sz, [_i64, _i64, C.c_int]),
    ("LZ4B200_compress_legacy", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, _i64, _vp, _sz, _vp]),
    ("LZ4B200_compress_blocks", C.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _i32, C.c_int, _vp, _i64, _vp]),
    ("LZ4B200_compress_blocks_destSize", C.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _i32, C.c_int, _vp, _vp, _i64, _vp]),
    ("LZ4B200_compress_blocks_hc_workspace_bytes", _sz, [_i64]),
    ("LZ4B200_compress_blocks_hc", C.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _i32, C.c_int, _vp, _i64, _vp, _sz, _vp]),
    ("LZ4B200_compress_blocks_hc_destSize", C.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _i32, C.c_int, _vp, _vp, _i64, _vp,
                                                      _sz, _vp]),
    ("LZ4B200_compress_blocks_hc_opt_workspace_bytes", _sz, [_i64]),
    ("LZ4B200_compress_blocks_hc_opt", C.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _i32, C.c_int, _vp, _i64, _vp, _sz,
                                                 _vp]),
    ("LZ4B200_compress_blocks_hc_opt_destSize", C.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _i32, C.c_int, _vp, _vp, _i64,
                                                          _vp, _sz, _vp]),
    ("LZ4B200_compress_blocks_parallel",C.c_int, [_vp, _i64, _vp, _i32, _vp, _i64, _i32, C.c_int, _vp, _i64, _vp]),
    ("LZ4B200_pack_blocks", C.c_int, [_vp, _i64, _vp, _i64, _vp, _vp, C.c_int, _vp]),
    ("LZ4B200_compress_blocks_indexed_workspace_bytes", _sz, [_i64, C.c_int, C.c_int]),
    ("LZ4B200_compress_blocks_indexed", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, C.c_int, _vp, _sz,
                                                  _vp]),
    ("LZ4B200_pack_blocks_indexed", C.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, C.c_int, _vp]),
    ("LZ4B200_pack_frame_blocks", C.c_int, [_vp, _i64, _vp, _vp, _i64, _i32, _i32, _i64, _vp, _vp, _vp]),
    ("LZ4B200_peer_copy_async", C.c_int, [_vp, C.c_int, _vp, C.c_size_t, _vp]),
    ("LZ4B200_decompress_blocks_host", C.c_int, [_vp, _vp, _vp, _vp, _i64, _i32, _vp, _i64]),
    ("LZ4B200_compress_blocks_host", C.c_int, [_vp, _i64, _i32, _i64, _vp, _i64, _i32, C.c_int, _vp, _i64]),
    ("LZ4B200_decompress_files_host", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, C.c_int]),
    ("LZ4B200_compress_frames_host", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, C.c_int, C.c_int,
                                              C.c_int, C.c_int, C.c_int]),
    ("LZ4B200_compress_legacy_host", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int]),
    ("LZ4B200_decompress_files_to_device", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, _vp]),
    ("LZ4B200_compress_frames_from_device", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, C.c_int, C.c_int,
                                                      C.c_int, C.c_int, C.c_int, _vp]),
    ("LZ4B200_compress_legacy_from_device", C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, C.c_int, _vp]),
    ("LZ4B200_compressFrameBound_checksummed", _i64, [_i64, C.c_int, C.c_int, C.c_int]),
    ("LZ4B200_compressFrameBound", _i64, [_i64, C.c_int]),
    ("LZ4B200_compressFrame_host", _i64, [_vp, _i64, _vp, _i64, C.c_int, C.c_int, C.c_int]),
    ("LZ4B200_decompressFrame_host", _i64, [_vp, _i64, _vp, _i64, _vp]),
]

_lib = None


def load():
    """Load liblz4_b200.so (once) and attach prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "%s is missing: build it with `python -m lz4_b200.build` (nvcc, sm_90a). "
            "lz4_b200 has no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, res, args in PROTOTYPES:
        fn = getattr(lib, name)          # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class Lz4CudaError(RuntimeError):
    pass


def check(rc, what):
    if rc != 0:
        err = load().LZ4B200_last_cuda_error().decode()
        raise Lz4CudaError("%s failed (rc=%d): %s" % (what, rc, err))
