"""The argument rules of LZ4B200_compress_blocks_indexed and LZ4B200_pack_blocks_indexed, and the indexed compress's
workspace size function, as decided on the host before any CUDA call.

No row reaches the device, so the table runs without a GPU and the launch counter must not move.  Non-NULL pointers
point at host memory that no row reads.
"""
import numpy as np
import pytest

OK, ARG = 0, -1
FAST, PARALLEL, HC = 0, 1, 2


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


_keep = np.zeros(1 << 16, dtype=np.uint8)
P = _keep.ctypes.data


def _rows(lib):
    hc_ws = lambda n: int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n))
    opt_ws = lambda n: int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n))

    def enc(parse=FAST, param=1, src=P, soff=P, ssz=P, dst=P, doff=P, cap=P, out=P, n=3, ws=P, wb=None):
        if wb is None:
            wb = int(lib.LZ4B200_compress_blocks_indexed_workspace_bytes(max(n, 0), parse, param))
        return lib.LZ4B200_compress_blocks_indexed(src, soff, ssz, dst, doff, cap, out, n, parse, param, ws, wb, None)

    def pack(slots=P, soff=P, sizes=P, packed=P, off=P, hdr=4, n=3):
        return lib.LZ4B200_pack_blocks_indexed(slots, soff, sizes, n, packed, off, hdr, None)

    rows = []
    for name, parse, param in (("fast", FAST, 1), ("parallel", PARALLEL, 1), ("hc", HC, 9), ("hc opt", HC, 12)):
        e = lambda parse=parse, param=param, **kw: enc(parse, param, **kw)
        rows += [
            ("%s nBlocks < 0" % name, lambda e=e: e(n=-1), ARG),
            ("%s nBlocks == 0, NULL d_src and d_dst" % name, lambda e=e: e(src=None, dst=None, n=0), OK),
            ("%s NULL d_srcOff" % name, lambda e=e: e(soff=None), ARG),
            ("%s NULL d_srcSize" % name, lambda e=e: e(ssz=None), ARG),
            ("%s NULL d_dstOff" % name, lambda e=e: e(doff=None), ARG),
            ("%s NULL d_dstCap" % name, lambda e=e: e(cap=None), ARG),
            ("%s NULL d_outSize" % name, lambda e=e: e(out=None), ARG),
            ("%s NULL d_srcOff with no blocks" % name, lambda e=e: e(soff=None, n=0), ARG),
            ("%s NULL d_outSize with no blocks" % name, lambda e=e: e(out=None, n=0), ARG),
            ("%s NULL d_src" % name, lambda e=e: e(src=None), ARG),
            ("%s NULL d_dst" % name, lambda e=e: e(dst=None), ARG),
        ]
    rows += [("unknown parse %d" % p, (lambda p=p: enc(parse=p)), ARG) for p in (-1, 3, 7)]
    rows += [("unknown parse %d with no blocks" % p, (lambda p=p: enc(parse=p, n=0, wb=0)), ARG) for p in (-1, 3)]
    rows += [
        ("parallel NULL workspace, no blocks", lambda: enc(PARALLEL, ws=None, wb=0, n=0), OK),
        ("hc NULL workspace", lambda: enc(HC, 9, ws=None), ARG),
        ("hc NULL workspace with no blocks", lambda: enc(HC, 9, ws=None, n=0), ARG),
        ("hc workspace one byte short", lambda: enc(HC, 9, wb=hc_ws(3) - 1), ARG),
        ("hc level 0 workspace one byte short", lambda: enc(HC, 0, wb=hc_ws(3) - 1), ARG),
        ("hc level 12 workspace one byte short", lambda: enc(HC, 12, wb=opt_ws(3) - 1), ARG),
        ("hc level 10 with a level-9 workspace", lambda: enc(HC, 10, wb=hc_ws(3)), ARG),
        ("hc level 13 workspace one byte short", lambda: enc(HC, 13, wb=opt_ws(3) - 1), ARG),
        ("hc nBlocks == 0, no workspace bytes", lambda: enc(HC, 9, src=None, dst=None, n=0, wb=0), OK),
        # pack: as LZ4B200_pack_blocks, no early return for nBlocks == 0 (d_outOff[0] is written on the device)
        ("pack nBlocks < 0", lambda: pack(n=-1), ARG),
        ("pack NULL d_outOff", lambda: pack(off=None), ARG),
        ("pack NULL d_outOff with no blocks", lambda: pack(off=None, n=0), ARG),
        ("pack NULL d_slots", lambda: pack(slots=None), ARG),
        ("pack NULL d_slotOff", lambda: pack(soff=None), ARG),
        ("pack NULL d_sizes", lambda: pack(sizes=None), ARG),
        ("pack NULL d_packed", lambda: pack(packed=None), ARG),
    ]
    rows += [("pack headerBytes %d" % h, (lambda h=h: pack(hdr=h)), ARG) for h in (-1, 1, 2, 3, 5, 8)]
    rows += [("pack headerBytes %d with no blocks" % h, (lambda h=h: pack(hdr=h, n=0)), ARG) for h in (-1, 3)]
    return rows


def test_argument_rules(lib):
    launches = lib.LZ4B200_launch_count()
    bad = []
    for name, call, want in _rows(lib):
        got = call()
        if got != want:
            bad.append("%s: %d, expected %d" % (name, got, want))
    assert not bad, "\n".join(bad)
    assert lib.LZ4B200_launch_count() == launches


def test_workspace_size_per_parse(lib):
    ws = lambda n, parse, param: int(lib.LZ4B200_compress_blocks_indexed_workspace_bytes(n, parse, param))
    hc = lambda n: int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n))
    opt = lambda n: int(lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n))
    for n in (0, 1, 3, 16383, 16384, 16385, 40000, 1 << 40, -1, -(1 << 40)):
        for param in (-5, 0, 1, 9, 65537, 2 ** 31 - 1, -2 ** 31):
            assert ws(n, FAST, param) == 0 and ws(n, PARALLEL, param) == 0, (n, param)
        for lv in (-2 ** 31, -1, 0, 1, 2, 3, 9):
            assert ws(n, HC, lv) == hc(n), (n, lv)
        for lv in (10, 11, 12, 13, 2 ** 31 - 1):
            assert ws(n, HC, lv) == opt(n), (n, lv)
        for p in (-1, 3, 100):
            assert ws(n, p, 9) == 0, (n, p)
    assert ws(1, HC, 9) == 256 * 1024 and ws(1, HC, 10) == 327728
    assert ws(40000, HC, 9) == 16384 * 256 * 1024 and ws(40000, HC, 12) == 16384 * 327728
