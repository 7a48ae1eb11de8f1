"""Every argument rule liblz4_b200.so decides on the host before any CUDA call, as one table.

Each row calls one entry point with arguments it must turn away (or accept with nothing to do) and states the return
value.  None of these rows reaches the device, so the table runs without a GPU, and the launch counter must not move.
Non-NULL pointers point at host memory that no row reads.  The rules differ from call to call on purpose (a NULL d_src,
or a NULL d_dst with no blocks); the table pins each call's own rules.
"""
import ctypes as C

import numpy as np
import pytest

OK, ARG, UNSUPPORTED, DSTSIZE = 0, -1, -4, -5


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import build, _lib
    build.build()
    return _lib.load()


_keep = np.zeros(1 << 16, dtype=np.uint8)
P = _keep.ctypes.data                 # a valid, aligned non-NULL pointer (8-byte aligned: a valid extState)
MIS = P + 1                           # misaligned state


def device_rows(lib):
    ws_bytes = lambda n, per, cap: int(lib.LZ4B200_decompress_workspace_bytes_for(n, per, cap))
    hc_ws = lambda n: int(lib.LZ4B200_compress_blocks_hc_workspace_bytes(n))

    def dec(src=P, off=P, size=P, dst=P, cap_arr=None, cap=65536, out=P, n=3, ws=P, ws_bytes_=None, phases=3):
        wb = ws_bytes(max(n, 0), cap_arr is not None, cap) if ws_bytes_ is None else ws_bytes_
        return lib.LZ4B200_decompress_blocks_phased(src, off, size, dst, None, cap, cap_arr, cap, out, n, ws, wb, phases, None)

    def full(src=P, off=P, size=P, dst=P, out=P, n=3, ws=P, wb=None):
        wb = ws_bytes(max(n, 0), 0, 65536) if wb is None else wb
        return lib.LZ4B200_decompress_blocks(src, off, size, dst, None, 65536, None, 65536, out, n, ws, wb, None)

    def part(src=P, off=P, size=P, dst=P, tgt=None, t=1000, out=P, n=3, ws=P, wb=None):
        wb = ws_bytes(max(n, 0), tgt is not None, t) if wb is None else wb
        return lib.LZ4B200_decompress_blocks_partial(src, off, size, dst, None, 4096, tgt, t, out, n, ws, wb, None)

    def enc(fn, src=P, sizes=None, dst=P, out=P, n=3):
        return fn(src, 65536, sizes, 65536, dst, 65552, 65552, 1, out, n, None)

    def hc(level=9, src=P, dst=P, out=P, n=3, ws=P, wb=None):
        wb = hc_ws(max(n, 0)) if wb is None else wb
        return lib.LZ4B200_compress_blocks_hc(src, 65536, None, 65536, dst, 65552, 65552, level, out, n, ws, wb, None)

    def dsz(src=P, dst=P, out=P, used=P, n=3):
        return lib.LZ4B200_compress_blocks_destSize(src, 65536, None, 65536, dst, 4096, 4096, 1, out, used, n, None)

    def pack(slots=P, sizes=P, packed=P, off=P, hdr=4, n=3):
        return lib.LZ4B200_pack_blocks(slots, 65552, sizes, n, packed, off, hdr, None)

    def pframe(slots=P, sizes=P, src=P, body=P, off=P, bs=65536, last=0, n=3):
        return lib.LZ4B200_pack_frame_blocks(slots, 65552, sizes, src, 65536, bs, last, n, body, off, None)

    fast = lib.LZ4B200_compress_blocks
    par = lib.LZ4B200_compress_blocks_parallel
    rows = [
        # decode: the phased call (the full call is phases = 3 of it), the full call and the partial call
        ("phased nBlocks < 0", lambda: dec(n=-1), ARG),
        ("phased nBlocks == 0 with NULL pointers", lambda: dec(src=None, off=None, size=None, dst=None, out=None, n=0,
                                                                ws=None, ws_bytes_=0), OK),
        ("phased NULL d_src", lambda: dec(src=None), ARG),
        ("phased NULL d_srcOff", lambda: dec(off=None), ARG),
        ("phased NULL d_srcSize", lambda: dec(size=None), ARG),
        ("phased NULL d_dst", lambda: dec(dst=None), ARG),
        ("phased NULL d_outSize", lambda: dec(out=None), ARG),
        ("phased NULL d_workspace", lambda: dec(ws=None), ARG),
        ("phased phases 0", lambda: dec(phases=0), ARG),
        ("phased phases 4", lambda: dec(phases=4), ARG),
        ("phased phases -1", lambda: dec(phases=-1), ARG),
        ("phased workspace one byte short", lambda: dec(ws_bytes_=ws_bytes(3, 0, 65536) - 1), ARG),
        ("phased per-block caps, workspace one byte short", lambda: dec(cap_arr=P, ws_bytes_=ws_bytes(3, 1, 0) - 1), ARG),
        ("full nBlocks < 0", lambda: full(n=-1), ARG),
        ("full nBlocks == 0", lambda: full(src=None, off=None, size=None, dst=None, out=None, n=0, ws=None, wb=0), OK),
        ("full NULL d_src", lambda: full(src=None), ARG),
        ("full NULL d_outSize", lambda: full(out=None), ARG),
        ("full NULL d_workspace", lambda: full(ws=None), ARG),
        ("full workspace one byte short", lambda: full(wb=ws_bytes(3, 0, 65536) - 1), ARG),
        ("partial nBlocks < 0", lambda: part(n=-1), ARG),
        ("partial nBlocks == 0", lambda: part(src=None, off=None, size=None, dst=None, out=None, n=0, ws=None, wb=0), OK),
        ("partial NULL d_src", lambda: part(src=None), ARG),
        ("partial NULL d_srcOff", lambda: part(off=None), ARG),
        ("partial NULL d_srcSize", lambda: part(size=None), ARG),
        ("partial NULL d_dst", lambda: part(dst=None), ARG),
        ("partial NULL d_outSize", lambda: part(out=None), ARG),
        ("partial NULL d_workspace", lambda: part(ws=None), ARG),
        ("partial workspace one byte short", lambda: part(wb=ws_bytes(3, 0, 1000) - 1), ARG),
        ("partial per-block targets, workspace one byte short", lambda: part(tgt=P, t=0, wb=ws_bytes(3, 1, 0) - 1), ARG),
        # compress, exact and parallel parse: nBlocks == 0 returns before the pointers are looked at
        ("compress nBlocks < 0", lambda: enc(fast, n=-1), ARG),
        ("compress nBlocks == 0 with NULL pointers", lambda: enc(fast, src=None, dst=None, out=None, n=0), OK),
        ("compress NULL d_dst", lambda: enc(fast, dst=None), ARG),
        ("compress NULL d_outSize", lambda: enc(fast, out=None), ARG),
        ("parallel nBlocks < 0", lambda: enc(par, n=-1), ARG),
        ("parallel nBlocks == 0 with NULL pointers", lambda: enc(par, src=None, dst=None, out=None, n=0), OK),
        ("parallel NULL d_dst", lambda: enc(par, dst=None), ARG),
        ("parallel NULL d_outSize", lambda: enc(par, out=None), ARG),
        # HC: the level first, then the output pointers even without blocks, then d_src and the workspace
        ("hc level 10", lambda: hc(level=10), ARG),
        ("hc level 12 with no blocks", lambda: hc(level=12, n=0), ARG),
        ("hc nBlocks < 0", lambda: hc(n=-1), ARG),
        ("hc nBlocks == 0", lambda: hc(src=None, n=0, wb=0), OK),
        ("hc NULL d_dst with no blocks", lambda: hc(dst=None, n=0), ARG),
        ("hc NULL d_outSize with no blocks", lambda: hc(out=None, n=0), ARG),
        ("hc NULL d_workspace with no blocks", lambda: hc(ws=None, n=0), ARG),
        ("hc NULL d_src", lambda: hc(src=None), ARG),
        ("hc workspace one byte short", lambda: hc(wb=hc_ws(3) - 1), ARG),
        # destSize: the output pointers even without blocks, then d_src
        ("destSize nBlocks < 0", lambda: dsz(n=-1), ARG),
        ("destSize nBlocks == 0", lambda: dsz(src=None, n=0), OK),
        ("destSize NULL d_dst with no blocks", lambda: dsz(dst=None, n=0), ARG),
        ("destSize NULL d_outSize with no blocks", lambda: dsz(out=None, n=0), ARG),
        ("destSize NULL d_srcConsumed with no blocks", lambda: dsz(used=None, n=0), ARG),
        ("destSize NULL d_src", lambda: dsz(src=None), ARG),
        # pack: no early return for nBlocks == 0 (d_outOff[0] is written on the device)
        ("pack nBlocks < 0", lambda: pack(n=-1), ARG),
        ("pack NULL d_outOff", lambda: pack(off=None), ARG),
        ("pack NULL d_outOff with no blocks", lambda: pack(off=None, n=0), ARG),
        ("pack NULL d_slots", lambda: pack(slots=None), ARG),
        ("pack NULL d_sizes", lambda: pack(sizes=None), ARG),
        ("pack NULL d_packed", lambda: pack(packed=None), ARG),
    ] + [("pack headerBytes %d" % h, (lambda h=h: pack(hdr=h)), ARG) for h in (-1, 1, 2, 3, 5, 8)] + [
        ("pack frame nBlocks < 0", lambda: pframe(n=-1), ARG),
        ("pack frame NULL d_outOff", lambda: pframe(off=None), ARG),
        ("pack frame NULL d_slots", lambda: pframe(slots=None), ARG),
        ("pack frame NULL d_sizes", lambda: pframe(sizes=None), ARG),
        ("pack frame NULL d_src", lambda: pframe(src=None), ARG),
        ("pack frame NULL d_body", lambda: pframe(body=None), ARG),
        ("pack frame blockSize 0", lambda: pframe(bs=0), ARG),
        ("pack frame blockSize < 0", lambda: pframe(bs=-65536), ARG),
        ("pack frame lastSize < 0", lambda: pframe(last=-1), ARG),
        ("pack frame lastSize > blockSize", lambda: pframe(last=65537), ARG),
    ]
    return rows


def host_rows(lib):
    def dec(src=P, off=P, size=P, dst=P, stride=65536, cap=65536, out=P, n=3):
        return lib.LZ4B200_decompress_blocks_host(src, off, size, dst, stride, cap, out, n)

    def enc(src=P, stride=65536, size=65536, last=65536, dst=P, out=P, n=3):
        return lib.LZ4B200_compress_blocks_host(src, stride, size, last, dst, 65552, 65552, 1, out, n)

    return [
        ("host decode nBlocks < 0", lambda: dec(n=-1), ARG),
        ("host decode dstCap < 0", lambda: dec(cap=-1, stride=0), ARG),
        ("host decode dstStride < dstCap", lambda: dec(stride=65535), ARG),
        ("host decode nBlocks == 0 with NULL pointers", lambda: dec(src=None, off=None, size=None, dst=None, out=None, n=0), OK),
        ("host decode NULL h_src", lambda: dec(src=None), ARG),
        ("host decode NULL h_srcOff", lambda: dec(off=None), ARG),
        ("host decode NULL h_srcSize", lambda: dec(size=None), ARG),
        ("host decode NULL h_dst", lambda: dec(dst=None), ARG),
        ("host decode NULL h_outSize", lambda: dec(out=None), ARG),
        ("host compress nBlocks < 0", lambda: enc(n=-1), ARG),
        ("host compress srcSize < 0", lambda: enc(size=-1, last=0), ARG),
        ("host compress lastSize < 0", lambda: enc(last=-1), ARG),
        ("host compress lastSize > srcSize", lambda: enc(last=65537), ARG),
        ("host compress srcStride < srcSize", lambda: enc(stride=65535), ARG),
        ("host compress nBlocks == 0 with NULL pointers", lambda: enc(src=None, dst=None, out=None, n=0), OK),
        ("host compress NULL h_dst", lambda: enc(dst=None), ARG),
        ("host compress NULL h_outSize", lambda: enc(out=None), ARG),
        ("host compress NULL h_src", lambda: enc(src=None), ARG),
    ]


def frame_rows(lib):
    src = P
    buf = np.zeros(4096, dtype=np.uint8)
    bound = int(lib.LZ4B200_compressFrameBound(1000, 4))

    def fr(src=src, n=1000, dst=True, cap=4096, bsid=4, level=0, csf=1):
        return lib.LZ4B200_compressFrame_host(src, n, buf.ctypes.data if dst else None, cap, bsid, level, csf)

    return [("frame block size id %d" % b, (lambda b=b: fr(bsid=b)), ARG) for b in (-1, 1, 2, 3, 8, 9)] + [
        ("frame level %d" % lv, (lambda lv=lv: fr(level=lv)), UNSUPPORTED) for lv in (2, 3, 9, 12)] + [
        ("frame dstCapacity one below the bound", lambda: fr(cap=bound - 1), DSTSIZE),
        ("frame srcSize < 0", lambda: fr(n=-1), ARG),
        ("frame NULL h_src", lambda: fr(src=None), ARG),
        ("frame NULL h_dst", lambda: fr(dst=False), ARG),
        ("frame empty input, default block size", lambda: fr(src=None, n=0, bsid=0), 11),
        ("frame empty input", lambda: fr(n=0, bsid=7, csf=0), 11),
    ]


def one_shot_rows(lib):
    buf = np.zeros(64, dtype=np.uint8)
    zero = np.zeros(4, dtype=np.uint8)
    one = np.ones(4, dtype=np.uint8)
    n = C.c_int(100)
    ds, dsp = lib.LZ4_decompress_safe, lib.LZ4_decompress_safe_partial
    return [
        ("decompress_safe dstCapacity 0, src {0x00}", lambda: ds(zero.ctypes.data, buf.ctypes.data, 1, 0), 0),
        ("decompress_safe dstCapacity 0, src {0x00}, NULL dst", lambda: ds(zero.ctypes.data, None, 1, 0), 0),
        ("decompress_safe dstCapacity 0, src {0x01}", lambda: ds(one.ctypes.data, buf.ctypes.data, 1, 0), -1),
        ("decompress_safe dstCapacity 0, src {0x00 0x00}", lambda: ds(zero.ctypes.data, buf.ctypes.data, 2, 0), -1),
        ("decompress_safe dstCapacity < 0", lambda: ds(zero.ctypes.data, buf.ctypes.data, 1, -1), -1),
        ("decompress_safe NULL src", lambda: ds(None, buf.ctypes.data, 1, 64), -1),
        ("decompress_safe compressedSize 0", lambda: ds(zero.ctypes.data, buf.ctypes.data, 0, 64), -1),
        ("decompress_safe compressedSize < 0", lambda: ds(zero.ctypes.data, buf.ctypes.data, -5, 64), -1),
        ("decompress_safe NULL dst", lambda: ds(zero.ctypes.data, None, 1, 64), -1),
        ("usingDict dictionary present", lambda: lib.LZ4_decompress_safe_usingDict(zero.ctypes.data, buf.ctypes.data, 1,
                                                                                   64, one.ctypes.data, 4), -1),
        ("usingDict no dictionary, dstCapacity 0", lambda: lib.LZ4_decompress_safe_usingDict(zero.ctypes.data,
                                                                                             buf.ctypes.data, 1, 0, None, 0), 0),
        ("partial target 0", lambda: dsp(one.ctypes.data, buf.ctypes.data, 4, 0, 64), 0),
        ("partial dstCapacity 0", lambda: dsp(one.ctypes.data, buf.ctypes.data, 4, 64, 0), 0),
        ("partial output size 0, srcSize 0, NULL dst", lambda: dsp(one.ctypes.data, None, 0, 0, 0), 0),
        ("partial output size < 0", lambda: dsp(one.ctypes.data, buf.ctypes.data, 4, -1, 64), -1),
        ("partial NULL src", lambda: dsp(None, buf.ctypes.data, 4, 0, 64), -1),
        ("partial srcSize 0", lambda: dsp(one.ctypes.data, buf.ctypes.data, 0, 64, 64), -1),
        ("partial srcSize < 0", lambda: dsp(one.ctypes.data, buf.ctypes.data, -1, 64, 64), -1),
        ("partial NULL dst", lambda: dsp(one.ctypes.data, None, 4, 64, 64), -1),
        ("compress_default dstCapacity 0", lambda: lib.LZ4_compress_default(P, buf.ctypes.data, 100, 0), 0),
        ("compress_default dstCapacity < 0", lambda: lib.LZ4_compress_default(P, buf.ctypes.data, 100, -1), 0),
        ("compress_default srcSize < 0", lambda: lib.LZ4_compress_default(P, buf.ctypes.data, -1, 64), 0),
        ("compress_default srcSize above the maximum",
         lambda: lib.LZ4_compress_default(P, buf.ctypes.data, 0x7E000001, 64), 0),
        ("compress_default NULL dst", lambda: lib.LZ4_compress_default(P, None, 100, 64), 0),
        ("compress_default NULL src", lambda: lib.LZ4_compress_default(None, buf.ctypes.data, 100, 64), 0),
        ("compress_fast dstCapacity 0", lambda: lib.LZ4_compress_fast(P, buf.ctypes.data, 100, 0, 1), 0),
        ("fast_extState dstCapacity 0", lambda: lib.LZ4_compress_fast_extState(P, P, buf.ctypes.data, 100, 0, 1), 0),
        ("fast_extState NULL state", lambda: lib.LZ4_compress_fast_extState(None, P, buf.ctypes.data, 100, 64, 1), 0),
        ("fast_extState misaligned state", lambda: lib.LZ4_compress_fast_extState(MIS, P, buf.ctypes.data, 100, 64, 1), 0),
        ("fastReset NULL state",
         lambda: lib.LZ4_compress_fast_extState_fastReset(None, P, buf.ctypes.data, 100, 64, 1), 0),
        ("fastReset misaligned state",
         lambda: lib.LZ4_compress_fast_extState_fastReset(MIS, P, buf.ctypes.data, 100, 64, 1), 0),
        ("destSize NULL srcSizePtr", lambda: lib.LZ4_compress_destSize(P, buf.ctypes.data, None, 64), 0),
        ("destSize targetDstSize 0", lambda: lib.LZ4_compress_destSize(P, buf.ctypes.data, C.byref(n), 0), 0),
        ("destSize_extState NULL srcSizePtr",
         lambda: lib.LZ4_compress_destSize_extState(P, P, buf.ctypes.data, None, 64, 1), 0),
        ("destSize_extState NULL state",
         lambda: lib.LZ4_compress_destSize_extState(None, P, buf.ctypes.data, C.byref(n), 64, 1), 0),
        ("destSize_extState misaligned state",
         lambda: lib.LZ4_compress_destSize_extState(MIS, P, buf.ctypes.data, C.byref(n), 64, 1), 0),
        ("destSize_extState targetDstSize < 0",
         lambda: lib.LZ4_compress_destSize_extState(P, P, buf.ctypes.data, C.byref(n), -1, 1), 0),
        ("destSize srcSizePtr untouched", lambda: n.value, 100),
    ]


@pytest.mark.parametrize("table", [device_rows, host_rows, frame_rows, one_shot_rows])
def test_argument_rules_are_decided_on_the_host(lib, table):
    launches = lib.LZ4B200_launch_count()
    wrong = []
    for name, call, want in table(lib):
        got = call()
        if got != want:
            wrong.append((name, got, want))
    assert not wrong, wrong
    assert lib.LZ4B200_launch_count() == launches


def test_empty_frame_is_header_and_end_mark(lib):
    dst = np.full(64, 0xAA, dtype=np.uint8)
    assert lib.LZ4B200_compressFrame_host(None, 0, dst.ctypes.data, 64, 7, 0, 1) == 11
    # the block size ID shrinks to 4 for an empty input and the content-size flag is dropped (lz4frame.c:445)
    assert dst[:11].tobytes().hex() == "04224d1860408200000000" and (dst[11:] == 0xAA).all()
