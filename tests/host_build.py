"""The host build of tests/emul/: TEST INFRASTRUCTURE.

Every tests/emul/*.cpp compiles device headers of lz4_b200/csrc/ with g++, so that the CPU suite can check the kernels'
logic without a GPU.  They are linked into one shared library, once per process, in a temporary directory removed at
exit.  PROTOTYPES holds every function the shims export; a missing one fails the load."""
import atexit
import ctypes as C
import glob
import os
import shutil
import subprocess
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
# -Wno-unknown-pragmas: the device's `#pragma unroll`
FLAGS = ["-O2", "-std=c++17", "-Wall", "-Wextra", "-Wno-unknown-pragmas", "-shared", "-fPIC"]

_vp, _i, _u32, _u64, _ll = C.c_void_p, C.c_int, C.c_uint32, C.c_uint64, C.c_longlong
_u32p, _ip, _llp, _cp = C.POINTER(C.c_uint32), C.POINTER(C.c_int), C.POINTER(C.c_longlong), C.c_char_p
# (name, restype, argtypes)
PROTOTYPES = [
    # scan_emul.cpp
    ("scan_host", _i, [_vp, _i, _i, _u32p, _vp]),
    ("scan_host_cap", _i, [_vp, _i, _i, _u32p, _vp, _u32]),
    ("scan_host_max_seq", _i, []),
    # scan_split_emul.cpp
    ("scan_split_host", _i, [_vp, _i, _i, _u32p, _vp, _u32, _ip]),
    ("scan_split_fuzz", _ll, [_cp, _i, _i, _i, _u64, _llp, _llp]),
    # scan_par_emul.cpp: the last argument is the lane count
    ("scan_par_host", _i, [_vp, _i, _i, _u32p, _vp, _ip, _i]),
    ("scan_par_host_wide", _i, [_vp, _i, _i, _u32p, _vp, _u32, _ip, _i]),
    ("scan_thread_host_wide", _i, [_vp, _i, _i, _u32p, _vp, _u32]),
    ("scan_par_fuzz", _ll, [_cp, _i, _i, _i, _u64, _llp, _i]),
    # rows_emul.cpp, tiles_emul.cpp, partial_emul.cpp
    ("rows_emulate", _i, [_cp, _i, _i, _cp, _i, _i, _llp]),
    ("tiles_emulate", _i, [_cp, _i, _i, _cp, _i, _llp]),
    ("partial_emulate", _i, [_cp, _i, _i, _u32p, _u32p, _u32p, _u32, _cp]),
    # plan_emul.cpp
    ("plan_host", None, [C.c_int64, _i, C.c_int32, _u64, _i, C.POINTER(C.c_uint64)]),
    # hc_emul.cpp
    ("hc_emul_compress", _i, [_vp, _i, _vp, _i, _i, _u32]),
    ("hc_dest_emul_compress", _i, [_vp, _i, _vp, _i, _i, _u32, _ip]),
    ("hc_opt_emul_compress", _i, [_vp, _i, _vp, _i, _i, _u32, _u32]),
    ("hc_opt_emul_compress_dest", _i, [_vp, _i, _vp, _i, _i, _u32, _u32, _ip]),
]

_lib = None


def load():
    """The library with PROTOTYPES attached, built on the first call; None without g++."""
    global _lib
    if _lib is None:
        gxx = shutil.which("g++")
        if not gxx:
            return None
        tmp = tempfile.mkdtemp(prefix="lz4emul")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, "libemul.so")
        subprocess.run([gxx, *FLAGS, "-o", so, *sorted(glob.glob(os.path.join(HERE, "emul", "*.cpp")))], check=True)
        lib = C.CDLL(so)
        for name, res, args in PROTOTYPES:
            fn = getattr(lib, name)          # AttributeError if the symbol is not exported
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def require():
    """load(), skipping the calling test without g++"""
    lib = load()
    if lib is None:
        import pytest
        pytest.skip("g++ not available")
    return lib
