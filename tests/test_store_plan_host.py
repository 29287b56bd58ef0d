"""How the pair kernel's store warp cuts a 128-row output slab of a packed (uniform crop stride) output into TMA boxes, restated in
Python and checked on the CPU for every scale factor the segmented stores serve and every slab start that can occur.

The restatement follows ``tp_gemm2_kernel``'s store warp (tokenpacker_b200/csrc/tp_gemm.cuh:1076-1105): the slab's rows are walked
segment (crop) by segment; a run of up to kWholeLevels = 3 WHOLE segments inside the slab leaves as one box of k segments per
destination; a partial segment piece of L = n * unit rows (unit = gcd(M, 128)) leaves as one box per set bit of n, largest first,
with box heights unit << level for level < kBoxLevels = 4; the lanes then issue their jobs (tp_gemm.cuh:1107-1116).  The host side
it has to agree with is ``launch_gemm_pair_group`` (tokenpacker_b200/csrc/tp_api.cu:321-331 for the local maps, 379-433 for the
destination maps and the worst-piece bound): it builds one map per level with box height unit << level (unit when that exceeds
min(M, 128): such a level is never used), the k-segment maps for k <= 3 when M <= 128, and rejects a shape whose worst slab needs
more than 96 jobs (pieces x destinations, three per store-warp lane: kJobsPerLane in tp_gemm.cuh:1042).

A box taller than its piece would write into the next crop's rows or into the separator row after it (and, at a segment's far end,
stick out of the tensor, which DESIGN.md §3.1 records as faulting), a box too short would leave rows unwritten: both show up here as
a coverage failure without running a GPU.  tests/test_store_paths_gpu.py relies on this model (through the host's worst-piece
loop, restated there) to claim that its eight-destination cases fill the second and third job slot of every lane.
"""
import math

import pytest

SLAB = 128                 # kBlockM: rows of one output slab
BOX_LEVELS = 4             # kBoxLevels
WHOLE_LEVELS = 3           # kWholeLevels
JOB_SLOTS = 96             # 32 lanes x kJobsPerLane
MAX_PEERS = 8              # kMaxPeers
SCALES = [1, 2, 3, 4, 6, 8, 12, 24]


def unit_of(m):
    """gcd(M, 128), as the host computes it (seg_store_unit)"""
    u = SLAB
    while m % u:
        u >>= 1
    return u


def served(m):
    return unit_of(m) >= 4


def slab_pieces(m, n_segs, row0):
    """the store warp's pieces of the slab starting at GEMM row ``row0`` of an output of n_segs segments of m rows:
    (slab row, height, segment, row in segment, segments in the box (whole-segment box) or 0 (level box), level or None)"""
    unit = unit_of(m)
    whole_ok = m <= SLAB                    # peers.whole: the local packed output goes through the destination maps as well
    out = []
    seg = row0 // m
    a = seg * m - row0
    while a < SLAB and seg < n_segs:
        if whole_ok and a >= 0 and a + m <= SLAB:
            k = 1
            while k < WHOLE_LEVELS and a + (k + 1) * m <= SLAB and seg + k < n_segs:
                k += 1
            out.append((a, k * m, seg, 0, k, None))
            a += k * m
            seg += k
            continue
        lo, hi = max(a, 0), min(a + m, SLAB)
        for lvl in range(BOX_LEVELS - 1, -1, -1):
            rows = unit << lvl
            while hi - lo >= rows:
                out.append((lo, rows, seg, lo - a, 0, lvl))
                lo += rows
        a += m
        seg += 1
    return out


def host_level_rows(m, lvl):
    """box height of the host's level-``lvl`` map"""
    rows = unit_of(m) << lvl
    return unit_of(m) if rows > SLAB or rows > m else rows


def host_worst_pieces(m):
    """launch_gemm_pair_group's bound: the most pieces any slab start (a multiple of unit inside a segment) is cut into"""
    unit, whole = unit_of(m), m <= SLAB
    worst = 0
    for a0 in range(0, -m, -unit):
        pieces, a = 0, a0
        while a < SLAB:
            if whole and a >= 0 and a + m <= SLAB:
                k = 1
                while k < WHOLE_LEVELS and a + (k + 1) * m <= SLAB:
                    k += 1
                pieces += 1
                a += k * m
                continue
            length = min(a + m, SLAB) - max(a, 0)
            for lvl in range(BOX_LEVELS - 1, -1, -1):
                while length >= unit << lvl:
                    pieces += 1
                    length -= unit << lvl
            a += m
        worst = max(worst, pieces)
    return worst


def _problems(m):
    """crop counts whose slabs start at every residue a multiple of 128 can have modulo m, each with every end-of-output case"""
    period = math.lcm(SLAB, m) // m         # crops after which the slab starts repeat modulo m
    return range(1, period + 4)


@pytest.mark.parametrize("s", [s for s in SCALES if served((24 // s) ** 2)])
def test_pieces_cover_each_slab_exactly(s):
    """Every slab of every output: the boxes cover exactly the slab rows that exist (all of them belong to a segment), without
    overlap; every box lies inside one segment (level box) or is k whole segments (whole-segment box); each box's slab row is the
    GEMM row it stores; every box height is one the host built a map for; the slab's jobs stay within the host's worst-piece bound."""
    m = (24 // s) ** 2
    unit = unit_of(m)
    bound = host_worst_pieces(m)
    assert bound * MAX_PEERS <= JOB_SLOTS, (s, bound)
    whole_heights = {k * m for k in range(1, WHOLE_LEVELS + 1)} if m <= SLAB else set()
    level_heights = {unit << lvl for lvl in range(BOX_LEVELS) if unit << lvl <= min(m, SLAB)}
    seen_worst = 0
    residues = set()
    for n in _problems(m):
        q = n * m
        for row0 in range(0, q, SLAB):
            residues.add(row0 % m)
            pieces = slab_pieces(m, n, row0)
            covered = [0] * SLAB
            for lo, h, seg, r, k, lvl in pieces:
                assert h > 0 and 0 <= lo and lo + h <= SLAB, (s, n, row0, lo, h)
                assert row0 + lo == seg * m + r, (s, n, row0, lo, seg, r)
                if k:
                    assert r == 0 and h == k * m <= SLAB and seg + k <= n and h in whole_heights, (s, n, row0, lo, h, k)
                else:
                    assert 0 <= r and r + h <= m and seg < n, (s, n, row0, lo, h, r)
                    assert h == host_level_rows(m, lvl) and h in level_heights, (s, n, row0, h, lvl)
                for i in range(lo, lo + h):
                    covered[i] += 1
            rows = min(SLAB, q - row0)
            assert covered == [1] * rows + [0] * (SLAB - rows), (s, n, row0)
            assert len(pieces) <= bound, (s, n, row0, len(pieces), bound)
            seen_worst = max(seen_worst, len(pieces))
    assert residues == set(range(0, m, unit))              # every slab start the host's bound considers occurred
    assert seen_worst == bound, (s, seen_worst, bound)     # the bound is reached, not just respected


def test_unserved_scale_factors():
    """M = 9 (s = 8) and M = 1 (s = 24) are not a multiple of 4 rows: the pair kernel has no boxes for them (the host sends their
    packed output to the one-CTA kernels' row stores and rejects a fused all-gather of it)."""
    assert [s for s in SCALES if not served((24 // s) ** 2)] == [8, 24]


def test_worst_pieces_table():
    """The worst pieces per slab quoted for the eight-destination store tests: s = 4 (M = 36) needs 7 pieces, 56 jobs at eight
    destinations (lanes use their second job slot); s = 12 (M = 4) needs 11, 88 jobs (their third)."""
    worst = {s: host_worst_pieces((24 // s) ** 2) for s in SCALES if served((24 // s) ** 2)}
    assert worst == {1: 2, 2: 4, 3: 1, 4: 7, 6: 3, 12: 11}
    assert worst[4] * MAX_PEERS > 32 and worst[12] * MAX_PEERS > 64
