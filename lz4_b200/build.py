"""Build liblz4_b200.so in-tree: nvcc (sm_90a, H100) for the kernels, gcc for the C host layer.

    python -m lz4_b200.build            # rebuild if sources are newer than the library
    python -m lz4_b200.build --force
"""
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "liblz4_b200.so")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")

SOURCES = ["lz4_kernels.cu", "lz4_api.c"]
HEADERS = [os.path.join(CSRC, "lz4_kernels.h"), os.path.join(CSRC, "lz4_rows_core.h"),
           os.path.join(CSRC, "lz4_scan_core.h"), os.path.join(CSRC, "lz4_scan_par.h"),
           os.path.join(CSRC, "lz4_scan_split.h"), os.path.join(CSRC, "lz4_encode_par.cuh"),
           os.path.join(CSRC, "lz4_decode_plan.h"), os.path.join(CSRC, "lz4_hc_core.h"),
           os.path.join(CSRC, "lz4_encode_hc.cuh"), os.path.join(CSRC, "lz4_frame_core.h"),
           os.path.join(CSRC, "lz4_files_plan.h"), os.path.join(CSRC, "lz4_cfiles_plan.h"),
           os.path.join(ROOT, "include", "lz4_b200.h")]

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC,-fvisibility=hidden", "--use_fast_math", "-diag-suppress", "177"]
if os.environ.get("LZ4K_PHASE_TIMING"):          # developer build: per-phase clock64 counters
    NVCC_FLAGS.append("-DLZ4K_PHASE_TIMING")
CC_FLAGS = ["-O2", "-fPIC", "-std=c99", "-Wall", "-Wextra", "-fvisibility=hidden",
            "-I" + os.path.join(CUDA_HOME, "include")]


def _stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, s) for s in SOURCES] + HEADERS + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("build failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
    return r.stdout + r.stderr


def build(force=False, verbose=False, out=None, extra_defines=()):
    """Build the library.  `out` / `extra_defines` are for developer variants (experimental kernels built
    next to the default library, e.g. out=build/liblz4_b200_barsync.so, extra_defines=["LZ4K_WAVE_BARSYNC"]);
    load one with LZ4_B200_LIBRARY=<path> (lz4_b200/_lib.py)."""
    lib = out or LIB
    if out is None and not extra_defines and not force and not _stale():
        return LIB
    if not os.path.exists(NVCC):
        raise RuntimeError("nvcc not found at %s" % NVCC)
    gcc = shutil.which("gcc") or "gcc"
    objdir = os.path.join(PKG, "build")
    os.makedirs(objdir, exist_ok=True)
    tag = "" if out is None else "_" + os.path.splitext(os.path.basename(out))[0]
    ko = os.path.join(objdir, "lz4_kernels%s.o" % tag)
    ao = os.path.join(objdir, "lz4_api%s.o" % tag)
    defs = ["-D" + d for d in extra_defines]
    log = _run([NVCC] + NVCC_FLAGS + defs + (["-Xptxas", "-v"] if verbose else []) +
               ["-c", os.path.join(CSRC, "lz4_kernels.cu"), "-o", ko])
    log += _run([gcc] + CC_FLAGS + ["-c", os.path.join(CSRC, "lz4_api.c"), "-o", ao])
    log += _run([NVCC, "-shared"] + ARCH + ["-o", lib, ko, ao,
                 "-Xlinker", "-Bsymbolic", "-lpthread"])
    if verbose:
        print(log)
    return lib


if __name__ == "__main__":
    # python -m lz4_b200.build [--force] [--out PATH] [-DNAME ...]
    argv = sys.argv[1:]
    out_path = argv[argv.index("--out") + 1] if "--out" in argv else None
    defines = [a[2:] for a in argv if a.startswith("-D")]
    print("built", build(force="--force" in argv, verbose=True, out=out_path, extra_defines=defines))
