"""GPU: point-to-voxel hashing (sgb_voxelize_idx_count / _fill) and the sparse-convolution rulebooks (sgb_rulebook_subm3,
sgb_rulebook_down2_count / _fill) over their whole key range, against the oracles bit for bit: the C restatement of
the reference's voxelize_idx and oracle/spconv_oracle.py. The cases are listed in tests/hash_cases.py;
tests/test_hash_coverage.py checks that they reach every edge (the key corners, the empty-marker key, probe chains that
wrap, the sort limits, the 1-, 2- and 3-level scans)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from oracle import spconv_oracle as so
from softgroup_b200 import harness, ops, spconv
from softgroup_b200.ops import _lib
from softgroup_b200.ops._lib import SgbError, check, ptr

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import hash_cases as hc  # noqa: E402

pytestmark = pytest.mark.gpu
SGB_ERR_RANGE = -4
VOX_RANGE_MSG = 'voxelize_idx: coordinate outside the packed key range'
RB_RANGE_MSG = 'rulebook: index outside the packed key range'


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _assert_vox(got, want, what):
    for name, g, w in zip(('output_coords', 'input_map', 'output_map'), got, want):
        g = g.cpu().numpy()
        assert g.dtype == w.dtype and g.shape == w.shape, (what, name, g.shape, w.shape)
        if not np.array_equal(g, w):
            bad = np.nonzero((g != w).reshape(len(g), -1).any(1))[0]
            raise AssertionError('%s: %s differs in %d rows, first %s' % (what, name, len(bad), bad[:5]))


# ================================================================== voxelize_idx
VOX = [(c.name, m) for c in hc.VOX_CASES if c.name not in hc.LARGE_VOX for m in hc.vox_modes(c)]


@pytest.mark.parametrize('name,mode', VOX, ids=['%s-m%d' % x for x in VOX])
def test_voxelize_matches_oracle(name, mode):
    c = hc.vox_case(name)
    pts = c.make()
    _assert_vox(ops.voxelization_idx(_cuda(pts), 1, mode), oracle.voxelization_idx(pts, 1, mode), (name, mode))


def test_voxelize_three_level_scan():
    """16,777,217 distinct voxels: the rank scan over the points takes three levels. Without duplicates every mode has
    the same output (row v = [1, first point of v]), so the oracle runs once."""
    c = hc.vox_case('three_level_scan')
    pts = c.make()
    want = oracle.voxelization_idx(pts, 1, 4)
    assert want[2].shape == (hc.THREE_LEVEL_N, 2)
    d = _cuda(pts)
    for mode in hc.vox_modes(c):
        _assert_vox(ops.voxelization_idx(d, 1, mode), want, ('three_level_scan', mode))


def _raw_count(pts, mode, ws):
    L = _lib.lib()
    d = _cuda(pts)
    im = torch.empty(len(pts), dtype=torch.int32, device='cuda')
    M, mx = ctypes.c_int(), ctypes.c_int()
    rc = L.sgb_voxelize_idx_count(ptr(d), len(pts), 4, mode, ptr(im), ptr(ws), ws.numel(), ctypes.byref(M),
                                  ctypes.byref(mx), _stream())
    return rc, d, im, M.value, mx.value


@pytest.mark.parametrize('field,value', hc.VOX_OUT_OF_RANGE, ids=['%s=%d' % x for x in hc.VOX_OUT_OF_RANGE])
def test_voxelize_out_of_range(field, value):
    L = _lib.lib()
    pts = hc.vox_out_of_range(field, value)
    with pytest.raises(SgbError, match=VOX_RANGE_MSG):
        ops.voxelization_idx(_cuda(pts), 1, 4)
    # the raw C ABI, on a workspace of zeros; the next valid call on the same workspace is unaffected
    ws = torch.zeros(L.sgb_voxelize_idx_workspace_bytes(len(pts)), dtype=torch.uint8, device='cuda')
    rc, *_ = _raw_count(pts, 4, ws)
    assert rc == SGB_ERR_RANGE and VOX_RANGE_MSG in L.sgb_last_error().decode()
    good = pts.copy()
    good[123] = good[124]
    rc, d, im, M, mx = _raw_count(good, 4, ws)
    check(rc, 'sgb_voxelize_idx_count')
    oc = torch.empty((M, 4), dtype=torch.int64, device='cuda')
    om = torch.empty((M, mx + 1), dtype=torch.int32, device='cuda')
    check(L.sgb_voxelize_idx_fill(ptr(d), len(good), 4, 4, M, mx, ptr(oc), ptr(om), ptr(ws), ws.numel(), _stream()),
          'sgb_voxelize_idx_fill')
    _assert_vox((oc, im, om), oracle.voxelization_idx(good, 1, 4), (field, value))


# ================================================================== rulebooks
def _check_rulebooks(rows, shape, subm=True, what=''):
    d = _cuda(rows)
    if subm:
        assert np.array_equal(spconv.build_subm_map(d).cpu().numpy(), so.subm_map(rows)), (what, 'subm3')
    out_idx, mp, inv, oshape = spconv.build_down_map(d, shape)
    o_idx, o_mp, o_inv, o_shape = so.down_map(rows, shape)
    assert oshape == o_shape == [int(s) // 2 for s in shape], what
    assert np.array_equal(out_idx.cpu().numpy(), o_idx), (what, 'out_indices')
    assert np.array_equal(mp.cpu().numpy(), o_mp), (what, 'map')
    assert np.array_equal(inv.cpu().numpy(), o_inv), (what, 'inv_map')
    return o_idx, o_shape


@pytest.mark.parametrize('name', [c.name for c in hc.RB_CASES])
def test_rulebooks_match_oracle(name):
    c = hc.rb_case(name)
    _check_rulebooks(c.make(), c.shape, c.subm, name)


def _instance_indices():
    """The indices clusters_voxelization hands the tiny U-Net in a seeded c2_scannet forward (one batch id per
    cluster, spatial shape 20). The point-wise predictions are injected with the load of a real checkpoint: objects
    cut into fragments, a share of the points under a second class -- hundreds of proposals."""
    from softgroup_b200 import synth
    from softgroup_b200.configs import model_cfg
    from softgroup_b200.model import SoftGroup
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet')).cuda().eval()
    scan = synth.make_scan('c2_scannet', seed=0)
    got = []
    orig = model.clusters_voxelization

    def capture(*a, **kw):
        out = orig(*a, **kw)
        got.append((out[0].indices.cpu().numpy(), list(out[0].spatial_shape)))
        return out

    model.clusters_voxelization = capture
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=0, fragments=8, confusion=0.3)
    with torch.no_grad():
        harness.run_scan(model, harness.to_host_batch(scan, pin=False), device_only=True, inject_pointwise=inj)
    assert len(got) == 1
    return got[0]


def test_rulebooks_instance_branch():
    rows, shape = _instance_indices()
    nb = len(np.unique(rows[:, 0]))
    print('instance branch: %d rows, %d batch ids' % (len(rows), nb))
    assert shape == [20, 20, 20] and rows.dtype == np.int32 and nb >= 100
    # both tiny U-Net levels: subm of level 0, the down map 0 -> 1, subm of level 1
    o_idx, o_shape = _check_rulebooks(rows, shape, True, 'instance level 0')
    _check_rulebooks(o_idx, o_shape, True, 'instance level 1')


@pytest.mark.parametrize('bad', hc.RB_OUT_OF_RANGE, ids=['%d,%d,%d,%d' % b for b in hc.RB_OUT_OF_RANGE])
def test_rulebooks_out_of_range(bad):
    rows, at = hc.rb_out_of_range(bad)
    with pytest.raises(SgbError, match=RB_RANGE_MSG):
        spconv.build_down_map(_cuda(rows), (16, 16, 16))
    # subm3 reports nothing: the accepted rows get the rulebook of the accepted rows alone, the rejected row its centre
    ok = hc.idx_ok(rows)
    keep = np.nonzero(ok)[0]
    sub = so.subm_map(rows[ok])
    want = np.full((27, len(rows)), -1, np.int32)
    want[:, keep] = np.where(sub >= 0, keep[np.maximum(sub, 0)], -1)
    want[13, at] = at
    got = spconv.build_subm_map(_cuda(rows)).cpu().numpy()
    bad_rows = keep[(got[:, keep] != want[:, keep]).any(0)]
    assert len(bad_rows) == 0, ('accepted rows differ', bad_rows[:5], got[:, bad_rows[:1]].ravel().tolist())
    assert got[:, at].tolist() == want[:, at].tolist(), 'rejected row'
