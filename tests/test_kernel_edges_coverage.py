"""CPU: the case table of tests/kernel_edge_cases.py reaches every launch threshold of the segment, row and instance
kernels that tests/test_gpu_kernel_edges.py is there to exercise. No GPU compute."""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kernel_edge_cases as kc  # noqa: E402
from softgroup_b200.ops import _lib  # noqa: E402


def test_launch_constants_match_the_library():
    L = _lib.lib()
    for N in (0, 1, 31, 32, 33, 4095, 4096, 1500000):
        assert L.sgb_bitmap_words(N) == kc.bitmap_words(N)
    assert [kc.pow2_cw(C) for C in (1, 2, 3, 4, 5, 8, 9, 16, 17, 32, 33, 96)] == [1, 2, 4, 4, 8, 8, 16, 16, 32, 32, 32, 32]


def test_minmax_cases_reach_every_path():
    cases = kc.MINMAX_CASES
    for c in cases:
        off = c.offsets
        assert off.dtype == np.int32 and (np.diff(off) >= 0).all() and len(off) >= 2
    S = [int(c.offsets[-1]) for c in cases]
    assert max(S) > kc.SEG_GRID * kc.SEG_CHUNK, 'grid-stride loop of seg_minmax_kernel'
    # every pow2_cw width, and channel counts above 32 (the c0 loop), one of them not a multiple of 32
    assert {kc.pow2_cw(c.C) for c in cases} == {1, 2, 4, 8, 16, 32}
    assert any(c.C > 64 for c in cases) and any(c.C > 32 and c.C % 32 for c in cases)
    # >= 2000 proposals that each span a chunk boundary, in one launch
    span = max(int(((c.offsets[1:] - 1) // kc.SEG_CHUNK > c.offsets[:-1] // kc.SEG_CHUNK).sum()) for c in cases)
    assert span >= 2000
    # proposal boundaries exactly on chunk starts, runs of empty proposals at a chunk start, empty first / last
    aligned = [c for c in cases if ((c.offsets[1:-1] % kc.SEG_CHUNK == 0) & (c.offsets[1:-1] > 0)).any()]
    assert any((np.diff(c.offsets) == 0).sum() >= 2 and c.offsets[0] == c.offsets[1] and c.offsets[-2] == c.offsets[-1]
               for c in aligned)
    assert any(c.offsets[0] > kc.SEG_CHUNK for c in cases), 'rows below offsets[0] outside every proposal'
    # an all -0.0 proposal over 3 chunks; one- and two-row special values
    assert any(c.kind == 'negzero' and np.diff(c.offsets).max() > 2 * kc.SEG_CHUNK for c in cases)
    assert any(c.kind == 'specials' and c.C == 1 for c in cases)
    c2 = [c for c in cases if c.name == 'c2_proposals'][0]
    assert len(c2.offsets) - 1 == 40 and c2.offsets[-1] == 131761 and c2.C == 3


def test_mean_cases_reach_every_path():
    cases = kc.MEAN_CASES
    assert max(len(c.offsets) - 1 for c in cases) > kc.MEAN_GRID, 'grid-stride loop of seg_reduce_kernel'
    assert max(int(np.diff(c.offsets).max()) for c in cases) >= 200000
    assert all(c.offsets[0] == 0 for c in cases)  # the float64 reference sums segments back to back
    assert any((np.diff(c.offsets) == 0).any() for c in cases), 'empty proposals'
    assert {c.data for c in cases} == {'relu', 'offset', 'cancel'}
    assert {kc.pow2_cw(c.C) for c in cases} == {1, 2, 4, 8, 16, 32}
    assert any(c.C > 32 for c in cases)
    # global_avg_pool_bp runs the non-relu cases and relu C in {3, 8}: long segments and nP > 65535 among them
    bp = [c for c in cases if c.data != 'relu' or c.C in (3, 8)]
    assert max(len(c.offsets) - 1 for c in bp) > kc.MEAN_GRID and max(int(np.diff(c.offsets).max()) for c in bp) >= 200000


def test_row_kernel_cases_reach_every_path():
    g = kc.GATHER_CASES
    vec = [c for c in g if c.C % 4 == 0 and c.in_off % 4 == 0 and c.out_off % 4 == 0]
    assert vec and any(c.C % 4 for c in g), 'float4 and scalar paths of gather_rows'
    assert any(c.C % 4 == 0 and c.in_off % 4 for c in g) and any(c.C % 4 == 0 and c.out_off % 4 for c in g)
    assert any(c.N >= 1500000 and c.C == 32 for c in g) and any(c.N == 1 for c in g)
    assert kc.LONG_VOXEL >= 2000 and set(kc.VOXEL_CHANNELS) == {3, 32, 35}


def test_instance_cases_reach_every_path():
    Ns = {c.N for c in kc.RLE_CASES}
    assert {1, 31, 32, 33, 63, 64, 65, 4096, 150000, 1500000} <= Ns
    words = {c.name: c.n_inst * kc.bitmap_words(c.N) for c in kc.RLE_CASES}
    tile = kc.SCAN_TILE
    assert any(tile - 200 < w < tile for w in words.values()) and tile in words.values()
    assert any(tile < w < tile + 200 for w in words.values())
    assert max(words.values()) > tile * tile, 'three-level exclusive_scan_i32'
    assert max(c.n_inst * kc.bitmap_words(c.N) * 4 for c in kc.RLE_CASES) < 2**30
    for c in kc.RLE_CASES:
        pats = kc.rle_patterns(c)
        assert c.n_inst >= len(pats) and ('alternate' in pats) == (c.N <= 150000)
    ic = kc.INST_CASES
    assert all(c.S % 32 for c in ic) and {c.nI for c in ic} == {1, 18}
    assert any(c.ms_stride > c.nI for c in ic)
    assert {c.layout for c in ic} == {'contiguous', 'single', 'interleaved'}
    # a proposal holds distinct points: no proposal longer than N
    assert all(c.layout == 'single' or kc._lengths(c.nP, c.S, seed=c.S).max() <= c.N for c in ic)
    assert kc.bitmap_words(kc.PANOPTIC_N) > kc.PAN_THREADS and kc.PANOPTIC_INST == 720
