"""The numbers tests/test_gpu_far_offsets.py relies on, pinned on the CPU, so that a change to a layout cannot quietly move
a far case back below 2^31 or 2^32: the HC workspaces of a full call, the wide decode plan at 520 x 4 MiB and the narrow
plan at 8 200 x 64 KB (from the library's size functions and the host build of the plan), the bench-shaped batch, and
the GPU file's arena layouts: every block of them where it claims to be, and every alias window inside the arena and
clear of every block."""
import ctypes as C

import pytest

import host_build
import test_gpu_far_offsets as far

L31, L32, MiB = far.L31, far.L32, far.MiB
FIELDS = ["wide", "markStride", "tilesMax", "scan", "nSeq", "slowList", "marks", "scratch", "used", "tileFirst",
          "tileFlag", "bytes"]
HC_SLOT, HC_OPT_SLOT = 262144, 262144 + 4099 * 16


@pytest.fixture(scope="module")
def lib():
    from lz4_b200 import _lib
    return _lib.load()


def plan(n, cap, ws_bytes):
    out = (C.c_uint64 * len(FIELDS))()
    host_build.require().plan_host(n, 0, cap, ws_bytes, 0, out)
    return dict(zip(FIELDS, list(out)))


def test_hc_workspaces_of_a_full_call(lib):
    n = 16384 + 37
    assert lib.LZ4B200_compress_blocks_hc_workspace_bytes(n) == 16384 * HC_SLOT == L32
    assert lib.LZ4B200_compress_blocks_hc_opt_workspace_bytes(n) == 16384 * HC_OPT_SLOT == 5369495552
    first = lambda slot, line: -(-line // slot)
    assert first(HC_SLOT, L31) == 8192                             # slots 8 192 .. 16 383 start past 2^31
    assert first(HC_OPT_SLOT, L31) == 6553 and first(HC_OPT_SLOT, L32) == 13106
    assert 13105 * HC_OPT_SLOT < L32 < 13106 * HC_OPT_SLOT         # slot 13 105 straddles 2^32


def test_wide_plan_at_520_blocks_of_4_mib(lib):
    n, cap = 520, 4 << 20
    nbytes = lib.LZ4B200_decompress_workspace_bytes_for(n, 0, cap)
    p = plan(n, cap, nbytes)
    assert p["wide"] == 1 and p["bytes"] == nbytes == 4362381056
    stride = p["markStride"] * 4
    assert stride == 8388624
    marks = lambda b: p["marks"] + b * stride
    assert marks(511) < L32 < marks(511) + stride and marks(512) >= L32   # blocks 512 and up: their marks past 2^32
    assert p["tileFirst"] >= L32 and p["tileFlag"] > p["tileFirst"]
    assert p["tileFirst"] == 4362089472 and p["tileFlag"] == 4362235136
    assert p["tilesMax"] == 69 and nbytes + 2 * far.GiB <= far.PEAK


def test_narrow_plan_at_8200_blocks_of_64_kb(lib):
    nbytes = lib.LZ4B200_decompress_workspace_bytes_for(8200, 0, 65536)
    p = plan(8200, 65536, nbytes)
    assert p["wide"] == 0 and p["markStride"] == 8192 and p["bytes"] == nbytes == 806159360
    assert plan(8192, 65536, nbytes)["scan"] == 2 and p["scan"] == 0      # R2 (split scan) and R3 (one thread)


def test_bench_shaped_batch(lib):
    """blocks 8 129 and up of the 64 KB batch at stride 2^19 + 4 096 lie past 2^32; output and workspace fit the peak"""
    stride = (1 << 19) + 4096
    assert 8128 * stride + 65536 < L32 < 8129 * stride
    assert 8200 * stride + lib.LZ4B200_decompress_workspace_bytes_for(8200, 0, 65536) + far.GiB <= far.PEAK


def check_layout(ranges, blocks):
    """ranges: (origin, offset from it, bytes) a call addresses; blocks: (start, bytes) from the base.  Every range and
    every alias window inside the arena, no alias window over a block."""
    for o, n in blocks:
        assert -far.LOW <= o and o + n <= far.ABOVE
    for origin, off, n in ranges:
        for a in far.aliases(off, n):
            lo, hi = max(origin + a - far.W, -far.LOW), origin + a + n + far.W
            assert hi <= far.ABOVE and hi > -far.LOW
            assert not any(b < hi and lo < b + m for b, m in blocks), (origin, off, n, a)


@pytest.mark.parametrize("route", list(far.ROUTES))
def test_decode_layouts(route):
    cap = far.ROUTES[route][0]
    every = [s for sets in far.FAR_DST for s in sets(cap)]
    for line in (L31, L32):                                        # on, one byte short of, past and across each line
        assert line in every and any(s < line < s + cap for s in every) and any(s > line for s in every)
    assert any(s % 16 == 0 for s in every) and any(s % 2 == 1 for s in every)
    for sets in far.FAR_DST:
        starts = sorted(sets(cap))
        assert all(b - a >= cap for a, b in zip(starts, starts[1:]))
        ranges = [(0, s, cap) for s in starts]
        blocks = [(s, cap) for s in starts]
        # the hostile blocks' zones, the sources' runs (up to 64 MB each) and the fillers' slots
        blocks += [(L31 + 8 * MiB, 64 * MiB), (L32 + 8 * MiB, 64 * MiB), (160 * MiB, far.FILLERS * 65536)]
        ranges += [(0, L31 + 8 * MiB, 64 * MiB), (0, L32 + 8 * MiB, 64 * MiB)]
        for line in (L31, L32):
            blocks.append((far.SRC_ORG + line - MiB, 65 * MiB))
            ranges.append((far.SRC_ORG, line - MiB, 65 * MiB))
        check_layout(ranges, blocks)
    for stride in far.STRIDES:
        assert stride > L31 and 2 * stride > L32
        for origin in (0, 3):
            check_layout([(origin, i * stride, cap) for i in range(3)], [(origin + i * stride, cap) for i in range(3)])
    assert far.FILLERS > 8192 and 160 * MiB + far.FILLERS * 65536 < far.SRC_ORG


def test_compress_and_pack_layouts():
    for s in (far.SRC_STRIDE, far.DST_STRIDE, far.PACK_STRIDE):
        assert L31 < s < L31 + 8 * MiB and s % 2 == 1 and L32 < 2 * s
    room = 65536 + 65536 // 255 + 16
    for src_stride, dst_stride in ((far.SRC_STRIDE, far.DST_STRIDE), (far.PACK_STRIDE, far.PACK_STRIDE)):
        ranges = [(far.SRC_ORG, i * src_stride, 100000) for i in range(3)]
        ranges += [(far.DST_ORG, i * dst_stride, room) for i in range(3)]
        check_layout(ranges, [(o + off, n) for o, off, n in ranges])


def test_aliases():
    assert far.aliases(L31 - 1 - far.W, 100) == []
    assert far.aliases(L31, 16) == [L31 - L32]
    assert far.aliases(L32 + 17, 16) == [17]
    assert far.aliases(L32 - 3, 16) == [L32 - 3 - L32]
