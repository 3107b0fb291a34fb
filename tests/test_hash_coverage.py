"""CPU: the case table of tests/hash_cases.py reaches every edge of the voxel hash and the rulebook hash that
tests/test_gpu_hash_edges.py is there to exercise, the constants it mirrors still match the .cu sources, and the host
voxelize path (sgb_voxelize_idx_cpu_begin / _finish) equals the oracle on every case. No GPU compute."""
import ctypes
import os
import re
import sys

import numpy as np
import pytest
import torch

import oracle
from softgroup_b200 import ops
from softgroup_b200.ops import _lib

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_cases as hc  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _src(name):
    with open(os.path.join(ROOT, 'softgroup_b200', 'csrc', name)) as f:
        return f.read()


def _kernel(src, name):
    """Body of __global__ `name` up to the next __global__."""
    m = re.search(r'__global__ void %s\(.*?(?=__global__|\Z)' % name, src, re.S)
    assert m, name
    return m.group(0)


# ---- constants against the sources ------------------------------------------------------------------------------------
def test_hash_and_table_constants():
    common = _src('common.cuh')
    m = re.search(r'constexpr unsigned long long kEmptyKey = 0x([0-9A-Fa-f]+)ull;', common)
    assert m and int(m.group(1), 16) == hc.EMPTY_KEY
    body = re.search(r'uint32_t hash64\(unsigned long long k\) \{(.*?)\}', common, re.S).group(1)
    assert tuple(int(s) for s in re.findall(r'k \^= k >> (\d+);', body)) == hc.HASH_SHIFTS
    assert tuple(int(s, 16) for s in re.findall(r'k \*= 0x([0-9a-f]+)ull;', body)) == hc.HASH_MULS
    assert 'return (uint32_t)k;' in body
    assert 'uint32_t s = hash64(key) & cap_mask;' in common  # home slot, both for insert and find
    assert 's = (s + 1) & cap_mask;' in common  # linear probing that wraps
    # capacity rules
    assert 'static size_t vox_cap(int N) { return pow2_at_least((size_t)std::max(N, 1) * 2); }' in _src('voxelize.cu')
    assert 'static size_t rb_cap(int M) { return pow2_at_least((size_t)std::max(M, 1) * 2); }' in _src('spconv.cu')
    assert [hc.vox_cap(n) for n in (0, 1, 2, 3, 4096, 4097)] == [2, 2, 4, 8, 8192, 16384]
    # the scan tile
    core = _src('core.cu')
    t, i = (int(re.search(r'constexpr int %s = (\d+);' % k, core).group(1)) for k in ('kScanThreads', 'kScanItems'))
    assert t * i == hc.SCAN_TILE and 'constexpr int kScanTile = kScanThreads * kScanItems;' in core


def test_key_layouts_and_bounds():
    vox = _src('voxelize.cu')
    assert ('bool ok = (b >= 0 && b < %d) && (x >= %d && x < %d) && (y >= %d && y < %d) &&\n'
            '            (z >= %d && z < %d);' % ((hc.VOX_B[1] + 1, ) + (hc.VOX_XYZ[0], hc.VOX_XYZ[1] + 1) * 3)) in vox
    for field, shift in (('(b & 0xFFFF)', 48), ('((x + %d) & 0xFFFF)' % hc.VOX_XYZ_BIAS, 32),
                         ('((y + %d) & 0xFFFF)' % hc.VOX_XYZ_BIAS, 16)):
        assert '(unsigned long long)%s << %d' % (field, shift) in vox, field
    assert '(unsigned long long)((z + %d) & 0xFFFF);' % hc.VOX_XYZ_BIAS in vox
    sp = _src('spconv.cu')
    assert ('return b >= 0 && b < %d && x >= 0 && x < %d && y >= 0 && y < %d && z >= 0 && z < %d;' %
            ((hc.RB_B[1] + 1, ) + (hc.RB_XYZ[1] + 1, ) * 3)) in sp
    assert hc.RB_XYZ[0] == 0
    for field, shift in (('(b & 0xFFFF)', 48), ('((x + 1) & 0xFFFF)', 32), ('((y + 1) & 0xFFFF)', 16)):
        assert '(unsigned long long)(unsigned)%s << %d' % (field, shift) in sp, field
    assert '(unsigned long long)(unsigned)((z + 1) & 0xFFFF);' in sp
    # the restatements agree with the layouts on the corners
    k, ok = hc.pack_key([[0, -32768, -32768, -32768], list(hc.SENTINEL_POINT)])
    assert ok.all() and k.tolist() == [0, hc.EMPTY_KEY]
    assert np.array_equal(hc.unpack_key(k), [[0, -32768, -32768, -32768], list(hc.SENTINEL_POINT)])
    assert hc.vkey([[1, -1, 0, 32766]]).tolist() == [(1 << 48) | (1 << 16) | 32767]


def test_sort_limits():
    body = _kernel(_src('voxelize.cu'), 'vox_sort_rows_kernel')
    assert 'bool long_row = c > %d;' % hc.SORT_INSERTION_MAX in body
    assert 'int nchunk = (cc + 31) >> 5;' in body and 'if (nchunk <= %d) {' % (hc.SORT_WARP_MAX // 32) in body


def test_sentinel_key_has_its_own_slot():
    """The key equal to kEmptyKey bypasses the table; the per-slot arrays have the extra slot `cap` for it."""
    vox = _src('voxelize.cu')
    assert 'uint32_t s = (key == kEmptyKey) ? w.cap : hash_insert(w.keys, w.cap - 1, key);' in vox
    for a in ('first', 'last', 'cnt', 'vid'):
        assert 'w.%s = a.take<int32_t>((size_t)w.cap + 1);' % a in vox, a
    for a in ('first', 'last', 'cnt'):
        assert re.search(r'cudaMemsetAsync\(w\.%s, 0x[0-9A-F]+|cudaMemsetAsync\(w\.%s, 0' % (a, a), vox)
        assert re.search(r'cudaMemsetAsync\(w\.%s, [^,]+, \(\(size_t\)w\.cap \+ 1\) \* 4, st\)' % a, vox), a
    assert 'b += 4 * align_up((cap + 1) * 4);' in vox  # sgb_voxelize_idx_workspace_bytes


def test_range_error_path_never_uses_a_stale_slot():
    """A point outside the key range gets slot -1, and every consumer of slot_of between the insert and the host's
    range check skips it (outputs cannot show a stale slot, so this is checked on the source)."""
    vox = _src('voxelize.cu')
    ins = _kernel(vox, 'vox_insert_kernel')
    assert '{ w.scalars[2] = 1; w.slot_of[i] = -1; return; }' in ins
    assert 'w.rank[i] = (s >= 0 && w.first[s] == i) ? 1 : 0;' in _kernel(vox, 'vox_flag_kernel')
    assert 'if (s >= 0 && w.first[s] == i) {' in _kernel(vox, 'vox_assign_kernel')
    assert 'input_map[i] = (s >= 0) ? w.vid[s] : -1;' in _kernel(vox, 'vox_inputmap_kernel')
    for k in ('vox_flag_kernel', 'vox_assign_kernel', 'vox_inputmap_kernel'):
        assert 'w.slot_of[i]]' not in _kernel(vox, k), k  # no direct index through slot_of


def test_subm3_never_looks_up_a_rejected_row():
    body = _kernel(_src('spconv.cu'), 'rb_subm3_kernel')
    assert re.search(r'else if \(idx_ok\(c\.x, c\.y, c\.z, c\.w\)\) \{.*hash_find', body, re.S)
    assert body.count('hash_find') == 1


# ---- the rulebook keys cannot reach the empty marker ------------------------------------------------------------------
def test_rulebook_keys_never_pack_to_the_empty_marker():
    """Every accepted row, every neighbour lookup from one and every down2 parent has x + 1 <= 32768 < 0xFFFF in its
    coordinate fields, so no vkey of theirs is kEmptyKey."""
    lo, hi = hc.RB_XYZ
    for v in (lo - 1, lo, hi, hi + 1):  # lookups reach one past each end of the accepted range
        assert 0 <= v + hc.RB_XYZ_BIAS < 0xFFFF
    extremes = np.array([[b, x, y, z] for b in hc.RB_B for x in (lo - 1, hi + 1) for y in (lo - 1, hi + 1)
                         for z in (lo - 1, hi + 1)])
    keys = hc.vkey(extremes)
    assert (keys != np.uint64(hc.EMPTY_KEY)).all()
    assert ((keys & np.uint64(0xFFFF)) <= np.uint64(hi + 1 + hc.RB_XYZ_BIAS)).all()
    # and the rejected row of the table does reach it: its (+1, +1, +1) lookup
    bad = np.array(hc.RB_OUT_OF_RANGE[-1])
    assert not hc.idx_ok(bad).any() and hc.vkey(bad + [0, 1, 1, 1]).tolist() == [hc.EMPTY_KEY]


# ---- the table reaches every edge -------------------------------------------------------------------------------------
def test_sentinel_cases_share_a_home_slot():
    for name, n_partners in (('sentinel_merge', 1), ('sentinel_crowd', 64)):
        pts = hc.vox_case(name).make()
        cap = hc.vox_cap(len(pts))
        keys = np.unique(hc.pack_key(pts)[0])
        assert hc.EMPTY_KEY in keys.tolist(), name
        h = hc.home(keys, cap)
        h_sent = hc.home([hc.EMPTY_KEY], cap)[0]
        assert (h[keys != np.uint64(hc.EMPTY_KEY)] == h_sent).sum() >= n_partners, name
    assert hc.vox_cap(2) == 4 and hc.home(hc.pack_key([hc.SENTINEL_PARTNER])[0], 4)[0] == 1 == hc.home([hc.EMPTY_KEY], 4)[0]
    # the sentinel point of sentinel_crowd lands in different 256-point blocks
    pts = hc.vox_case('sentinel_crowd').make()
    at = np.nonzero((pts == hc.SENTINEL_POINT).all(1))[0]
    assert len(np.unique(at // 256)) >= 8
    # corners holds the sentinel too; with 3 columns the same coordinates cannot reach the marker
    assert hc.EMPTY_KEY in hc.pack_key(hc.vox_case('corners').make())[0].tolist()
    k3, ok3 = hc.pack_key(hc.vox_case('sentinel_ncol3').make(), 3)
    assert ok3.all() and hc.EMPTY_KEY not in k3.tolist() and (k3 == np.uint64(0xFFFFFFFFFFFF)).any()


def test_wrap_probe_chains_pass_the_last_slot():
    for keys, cap in ((np.unique(hc.pack_key(hc.vox_case('wrap_probe').make())[0]),
                       hc.vox_cap(len(hc.vox_case('wrap_probe').make()))),
                      (hc.vkey(hc.rb_case('wrap_probe').make()), hc.rb_cap(len(hc.rb_case('wrap_probe').make())))):
        assert len(keys) == hc.WRAP_DISTINCT
        h = hc.home(keys, cap)
        assert (h >= cap - 8).all()
        # every chain runs through slot cap - 1 and on from slot 0
        assert (h + hc.chain_lengths(h, cap) > cap).all()
    pts = hc.vox_case('wrap_probe').make()
    _, cnt = np.unique(pts, axis=0, return_counts=True)
    assert sorted(np.bincount(cnt)[1:].tolist()) == [hc.WRAP_DISTINCT // 2] * 2


def _voxel_order(pts):
    """(point count per voxel in voxel-id order) -- voxel id = rank of the first point."""
    _, first, inv, cnt = np.unique(pts, axis=0, return_index=True, return_inverse=True, return_counts=True)
    order = np.argsort(first)
    return cnt[order]


def test_row_lengths_reach_both_sides_of_every_sort_limit():
    cnt = _voxel_order(hc.vox_case('row_lengths').make())
    for lim in (hc.SORT_INSERTION_MAX, 32, hc.SORT_WARP_MAX):
        assert lim in cnt and lim + 1 in cnt, lim
    assert {1, 2, 3000} <= set(cnt.tolist())
    warps = [cnt[w:w + 32] for w in range(0, len(cnt), 32)]
    assert any((w > hc.SORT_INSERTION_MAX).sum() >= 2 and (w <= hc.SORT_INSERTION_MAX).any() for w in warps)
    assert any(((w > hc.SORT_WARP_MAX).any() and ((w > 24) & (w <= hc.SORT_WARP_MAX)).any()) for w in warps)


def test_scan_levels_and_capacity_steps():
    ns = {c.name: len(c.make()) for c in hc.VOX_CASES if c.name not in hc.LARGE_VOX}
    ns['three_level_scan'] = hc.THREE_LEVEL_N
    assert {hc.scan_levels(n) for n in ns.values()} == {1, 2, 3}
    assert {1, 2, hc.SCAN_TILE, hc.SCAN_TILE + 1, 65536, 65537, hc.SCAN_TILE ** 2 + 1} <= set(ns.values())
    assert hc.scan_levels(hc.SCAN_TILE) == 1 and hc.scan_levels(hc.SCAN_TILE + 1) == 2
    assert hc.scan_levels(hc.SCAN_TILE ** 2) == 2 and hc.scan_levels(hc.SCAN_TILE ** 2 + 1) == 3
    # the capacity doubles between 2^k and 2^k + 1 points
    for n in (hc.SCAN_TILE, 65536):
        assert hc.vox_cap(n + 1) == 2 * hc.vox_cap(n)
    ms = {c.name: (None if c.name == 'three_level_scan' else len(c.make())) for c in hc.RB_CASES}
    assert {1, hc.SCAN_TILE, hc.SCAN_TILE + 1} <= set(ms.values())
    assert hc.scan_levels(hc.RB_THREE_LEVEL_M) == 3 and not hc.rb_case('three_level_scan').subm
    # the unique cases are unique (mode 0 runs on them), the others are not
    for c in hc.VOX_CASES:
        if c.name not in hc.LARGE_VOX:
            pts = c.make()
            assert (len(np.unique(pts, axis=0)) == len(pts)) == c.unique, c.name


def test_vox_field_boundaries_on_both_sides():
    inside = np.concatenate([hc.vox_case(n).make() for n in ('corners', 'batch_isolation')])
    assert set(inside[:, 0].tolist()) >= set(hc.VOX_B)
    for j in (1, 2, 3):
        assert {hc.VOX_XYZ[0], -1, 0, hc.VOX_XYZ[1]} <= set(inside[:, j].tolist())
    rows = np.array([list(r) for r in hc.vox_case('corners').make()])
    assert len(np.unique(rows, axis=0)) == 2 * 4 ** 3
    outside = {(f, v) for f, v in hc.VOX_OUT_OF_RANGE}
    for f in hc.VOX_FIELDS:
        lo, hi = hc.VOX_B if f == 'b' else hc.VOX_XYZ
        assert {(f, lo - 1), (f, hi + 1), (f, (1 << 32) + 3)} <= outside
    for f, v in hc.VOX_OUT_OF_RANGE:
        pts = hc.vox_out_of_range(f, v)
        ok = hc.pack_key(pts)[1]
        assert np.nonzero(~ok)[0].tolist() == [123]
    # batch isolation: the same coordinates in batches 0, 1 and 65535
    p = hc.vox_case('batch_isolation').make()
    xyz_b = {b: {tuple(r) for r in p[p[:, 0] == b, 1:]} for b in (0, 1, hc.VOX_B[1])}
    assert xyz_b[0] == xyz_b[1] == xyz_b[hc.VOX_B[1]]


def test_rulebook_cases_reach_every_edge():
    c = hc.rb_case('corners').make()
    assert set(c[:, 0].tolist()) == set(hc.RB_B)
    for j in (1, 2, 3):
        assert {0, 1, 2, hc.RB_MAX_LO, hc.RB_XYZ[1]} <= set(c[:, j].tolist())
    # all 27 offsets hit at the block centres; lookups at -1 and 32767 stay inside the key layout and miss
    from oracle import spconv_oracle as so
    mp = so.subm_map(c)
    assert ((mp >= 0).sum(0) == 27).sum() == 16
    for case in hc.RB_CASES:
        if case.name != 'three_level_scan':
            rows = case.make()
            assert rows.dtype == np.int32 and rows.shape[1] == 4 and hc.idx_ok(rows).all(), case.name
            assert len(np.unique(rows, axis=0)) == len(rows), case.name
    # down2: one odd axis at a time, the max plane of it occupied; D = 1 (no parent) and D = 2; 32766 dropped
    for name, axis in (('odd_x', 0), ('odd_y', 1), ('odd_z', 2)):
        case = hc.rb_case(name)
        assert [s % 2 for s in case.shape] == [int(a == axis) for a in range(3)]
        assert (case.make()[:, 1 + axis] == case.shape[axis] - 1).any()
    assert so.down_map(hc.rb_case('d1_axis').make(), hc.rb_case('d1_axis').shape)[0].shape[0] == 0
    assert 2 in hc.rb_case('d2_axis').shape
    assert hc.rb_case('corners').shape[0] // 2 == 16383 and (c[:, 1:] == hc.RB_XYZ[1]).any()
    # children: parents with 8 children, with 1, and parents whose first child is among the last rows
    rows = hc.rb_case('children').make()
    par = rows[:, 1:] >> 1
    _, first, inv, cnt = np.unique(par, axis=0, return_index=True, return_inverse=True, return_counts=True)
    assert {1, 8} <= set(cnt.tolist()) and (first >= len(rows) - 240).sum() >= 50
    # batch isolation under vkey
    b = hc.rb_case('batch_isolation').make()
    xyz_b = {v: {tuple(r) for r in b[b[:, 0] == v, 1:]} for v in (0, 1, hc.RB_B[1])}
    assert xyz_b[0] == xyz_b[1] == xyz_b[hc.RB_B[1]]
    # out of range: each field just outside on both sides, and the row whose lookup packs to the marker
    bad = np.array(hc.RB_OUT_OF_RANGE)
    assert {-1, hc.RB_B[1] + 1} <= set(bad[:, 0].tolist())
    for j in (1, 2, 3):
        assert {hc.RB_XYZ[0] - 1, hc.RB_XYZ[1] + 1} <= set(bad[:, j].tolist())
    for r in hc.RB_OUT_OF_RANGE:
        rows, at = hc.rb_out_of_range(r)
        assert np.nonzero(~hc.idx_ok(rows))[0].tolist() == [at]
    # the 16-bit alias of b = 65536 is a batch-0 row of the set
    rows, at = hc.rb_out_of_range((hc.RB_B[1] + 1, 5, 5, 5))
    assert ((rows[:, 0] == 0) & (np.abs(rows[:, 1:] - 5) <= 1).all(1)).sum() == 27


# ---- the host voxelize path against the oracle -------------------------------------------------------------------------
HOST_CASES = [(c.name, m) for c in hc.VOX_CASES if c.name not in hc.LARGE_VOX for m in hc.vox_modes(c)]


def _host_abi(pts, ncol, mode):
    L = _lib.lib()
    pts = np.ascontiguousarray(pts, np.int64)
    n = len(pts)
    im = np.zeros(n, np.int32)
    M, mx = ctypes.c_int(), ctypes.c_int()
    h = L.sgb_voxelize_idx_cpu_begin(pts.ctypes.data, n, ncol, mode, im.ctypes.data, ctypes.byref(M), ctypes.byref(mx))
    _lib.check(h, 'sgb_voxelize_idx_cpu_begin')
    oc = np.zeros((M.value, ncol), np.int64)
    om = np.zeros((M.value, mx.value + 1), np.int32)
    _lib.check(L.sgb_voxelize_idx_cpu_finish(ctypes.c_void_p(h), pts.ctypes.data, oc.ctypes.data, om.ctypes.data),
               'sgb_voxelize_idx_cpu_finish')
    return oc, im, om


def _check_host(pts, ncol, mode):
    want = oracle.voxelization_idx(pts, 1, mode)
    got_abi = _host_abi(pts, ncol, mode)
    got_op = [t.numpy() for t in ops.voxelization_idx(torch.from_numpy(np.ascontiguousarray(pts)), 1, mode)]
    for what, got in (('C ABI', got_abi), ('ops', got_op)):
        for name, g, w in zip(('output_coords', 'input_map', 'output_map'), got, want):
            assert g.dtype == w.dtype and np.array_equal(g, w), (what, name)


@pytest.mark.parametrize('name,mode', HOST_CASES, ids=['%s-m%d' % x for x in HOST_CASES])
def test_host_voxelize_matches_oracle(name, mode):
    c = hc.vox_case(name)
    _check_host(c.make(), c.ncol, mode)


@pytest.mark.parametrize('field,value', hc.VOX_OUT_OF_RANGE, ids=['%s=%d' % x for x in hc.VOX_OUT_OF_RANGE])
def test_host_voxelize_out_of_range_matches_oracle(field, value):
    """The host path has no key-range limit: it narrows to int32 like the reference (and the oracle)."""
    _check_host(hc.vox_out_of_range(field, value), 4, 4)
