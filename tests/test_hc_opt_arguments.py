"""The argument rules of LZ4B200_compress_blocks_hc_opt and LZ4B200_compress_blocks_hc_opt_destSize that
liblz4_b200.so decides on the host before any CUDA call, as one table.

Each row calls one entry point with arguments it must turn away (or accept with nothing to do) and states the return
value.  None of these rows reaches the device, so the table runs without a GPU, and the launch counter must not move.
Non-NULL pointers point at host memory that no row reads.  The level is checked first: the levels below 10 belong to
the hash-chain calls.
"""
import numpy as np
import pytest

OK, ARG = 0, -1
SLOT = 262144 + 4099 * 16


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


_keep = np.zeros(1 << 16, dtype=np.uint8)
P = _keep.ctypes.data


def rows(lib):
    ws = lambda n: int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n))

    def opt(level=12, src=P, dst=P, out=P, n=3, w=P, wb=None):
        wb = ws(max(n, 0)) if wb is None else wb
        return lib.LZ4B200_compress_blocks_hc_opt(src, 65536, None, 65536, dst, 65552, 65552, level, out, n, w, wb, None)

    def dest(level=12, src=P, dst=P, out=P, used=P, n=3, w=P, wb=None):
        wb = ws(max(n, 0)) if wb is None else wb
        return lib.LZ4B200_compress_blocks_hc_opt_destSize(src, 65536, None, 65536, dst, 4096, 4096, level, out, used,
                                                           n, w, wb, None)

    out = []
    for name, call in (("opt", opt), ("opt destSize", dest)):
        out += [
            ("%s level 9" % name, lambda call=call: call(level=9), ARG),
            ("%s level 1" % name, lambda call=call: call(level=1), ARG),
            ("%s level 0" % name, lambda call=call: call(level=0), ARG),
            ("%s level -1" % name, lambda call=call: call(level=-1), ARG),
            ("%s level 9 with no blocks" % name, lambda call=call: call(level=9, n=0, wb=0), ARG),
            ("%s level 9 before nBlocks < 0" % name, lambda call=call: call(level=9, n=-1), ARG),
            ("%s level 10 with no blocks" % name, lambda call=call: call(level=10, src=None, n=0, wb=0), OK),
            ("%s level 13 with no blocks" % name, lambda call=call: call(level=13, src=None, n=0, wb=0), OK),
            ("%s level 100 with no blocks" % name, lambda call=call: call(level=100, src=None, n=0, wb=0), OK),
            ("%s nBlocks < 0" % name, lambda call=call: call(n=-1), ARG),
            ("%s NULL d_dst with no blocks" % name, lambda call=call: call(dst=None, n=0), ARG),
            ("%s NULL d_outSize with no blocks" % name, lambda call=call: call(out=None, n=0), ARG),
            ("%s NULL d_workspace with no blocks" % name, lambda call=call: call(w=None, n=0), ARG),
            ("%s NULL d_src" % name, lambda call=call: call(src=None), ARG),
            ("%s workspace one byte short" % name, lambda call=call: call(wb=ws(3) - 1), ARG),
            ("%s hash-chain workspace" % name,
             lambda call=call: call(wb=int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(3))), ARG),
        ]
    out.append(("opt destSize NULL d_srcConsumed with no blocks", lambda: dest(used=None, n=0), ARG))
    return out


def test_argument_rules_are_decided_on_the_host(lib):
    launches = lib.LZ4B200_launch_count()
    wrong = []
    for name, call, want in rows(lib):
        got = call()
        if got != want:
            wrong.append((name, got, want))
    assert not wrong, wrong
    assert lib.LZ4B200_launch_count() == launches


def test_workspace_size():
    """327 728 bytes per slot for min(nBlocks, 16 384) slots; the hash-chain calls keep 256 KB per slot."""
    from lz4_b200 import build, _lib
    build.build()
    lib = _lib.load()
    ws = lambda n: int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n))
    assert [ws(n) for n in (-1, 0, 1, 3, 16384, 16385, 1 << 30)] == \
        [0, 0, SLOT, 3 * SLOT, 16384 * SLOT, 16384 * SLOT, 16384 * SLOT]
    assert int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(3)) == 3 * 262144
