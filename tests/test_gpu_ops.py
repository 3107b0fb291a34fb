"""GPU parity: every softgroup_b200.ops kernel (through the C ABI) against the CPU oracle on the same
seeded inputs, plus the golden vectors from the compiled reference. Integer/index outputs are bit-exact;
floats within the tolerance stated in each test (north star: 1e-4 relative)."""
import numpy as np
import pytest
import torch

import oracle
from softgroup_b200 import ops, synth

pytestmark = pytest.mark.gpu
MEAN = [-1., -1., 3917., 12056., 2303., 8331., 3948., 3166., 5629., 11719., 1003., 3317., 4912., 10221., 3889., 4136.,
        2120., 945., 3967., 2589.]


def _cuda(a, dt=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dt is not None:
        t = t.to(dt)
    return t.cuda()


def _lists(idx, sl):
    idx = idx.cpu().numpy() if torch.is_tensor(idx) else idx
    sl = sl.cpu().numpy() if torch.is_tensor(sl) else sl
    return [idx[s:s + l] for s, l in sl]


def _assert_lists_equal(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), 'point %d: %s vs %s' % (i, x[:8], y[:8])


# ------------------------------------------------------------------ voxelize_idx
def test_voxelize_idx_golden(golden):
    oc, im, om = ops.voxelization_idx(_cuda(golden['vox_c1_coords']), 1, 4)
    assert oc.is_cuda
    assert np.array_equal(oc.cpu().numpy(), golden['vox_c1_out_coords'])
    assert np.array_equal(im.cpu().numpy(), golden['vox_c1_input_map'])
    assert np.array_equal(om.cpu().numpy(), golden['vox_c1_output_map'])


@pytest.mark.parametrize('mode', [1, 2, 3, 4])
def test_voxelize_idx_ragged_negative(golden, mode):
    oc, im, om = ops.voxelization_idx(_cuda(golden['vox_rag_coords']), 2, mode)
    assert np.array_equal(oc.cpu().numpy(), golden['vox_rag_m%d_out_coords' % mode])
    assert np.array_equal(im.cpu().numpy(), golden['vox_rag_m%d_input_map' % mode])
    assert np.array_equal(om.cpu().numpy(), golden['vox_rag_m%d_output_map' % mode])


@pytest.mark.parametrize('shape,n', [('c2_scannet', 150000), ('c3_s3dis', 800000)])
def test_voxelize_idx_full_size(shape, n):
    scan = synth.make_scan(shape, seed=1, n_points=n)
    oc, im, om = ops.voxelization_idx(_cuda(scan['coords']), 1, 4)
    a, b, d = oracle.voxelization_idx(scan['coords'], 1, 4)
    assert np.array_equal(oc.cpu().numpy(), a)
    assert np.array_equal(im.cpu().numpy(), b)
    assert np.array_equal(om.cpu().numpy(), d)


def test_voxelize_idx_long_rows():
    # cluster re-voxelisation shape: few voxels, many points each (rows > 24 and > 1024 entries)
    rng = np.random.RandomState(3)
    c = np.concatenate([rng.randint(0, 3, (20000, 1)), rng.randint(0, 3, (20000, 3))], 1).astype(np.int64)
    c[:3000, 1:] = 0
    c[:3000, 0] = 0
    oc, im, om = ops.voxelization_idx(_cuda(c), 3, 4)
    a, b, d = oracle.voxelization_idx(c, 3, 4)
    assert np.array_equal(oc.cpu().numpy(), a) and np.array_equal(im.cpu().numpy(), b)
    assert np.array_equal(om.cpu().numpy(), d)


def test_voxelize_idx_empty():
    # out-of-range coordinates: tests/test_gpu_hash_edges.py
    oc, im, om = ops.voxelization_idx(torch.zeros((0, 4), dtype=torch.int64, device='cuda'), 1, 4)
    assert oc.shape == (0, 4) and im.shape == (0, ) and om.shape == (0, 2)


# ------------------------------------------------------------------ voxelize fp/bp
@pytest.mark.parametrize('C', [3, 6, 32])
def test_voxelization_fp_bp(C):
    scan = synth.make_scan('c1_plumbing', seed=2, n_points=20000)
    _, _, om = oracle.voxelization_idx(scan['coords'], 1, 4)
    rng = np.random.RandomState(0)
    feats = rng.randn(20000, C).astype(np.float32)
    f = _cuda(feats).requires_grad_(True)
    out = ops.voxelization(f, _cuda(om), 4)
    ref = oracle.voxelization(feats, om, 4)
    assert np.array_equal(out.detach().cpu().numpy(), ref)  # same sequential order -> bit-exact
    g = rng.randn(*ref.shape).astype(np.float32)
    out.backward(_cuda(g))
    assert np.allclose(f.grad.cpu().numpy(), oracle.voxelization_bp(g, om, 20000, 4), rtol=1e-6, atol=1e-7)


# ------------------------------------------------------------------ ball query
def _bq_case(n, B, r, sigma, seed):
    rng = np.random.RandomState(seed)
    centers = rng.rand(12, 3) * 2
    xyz = (centers[rng.randint(0, 12, n)] + rng.randn(n, 3) * sigma).astype(np.float32)
    cuts = np.sort(rng.choice(np.arange(1, n), B - 1, replace=False)) if B > 1 else np.array([], np.int64)
    bo = np.concatenate([[0], cuts, [n]]).astype(np.int32)
    bi = np.repeat(np.arange(B), np.diff(bo)).astype(np.int32)
    return xyz, bi, bo


@pytest.mark.parametrize('n,B,r,sigma', [(2000, 1, 0.04, 0.03), (5000, 3, 0.04, 0.05), (3000, 2, 0.1, 0.01),
                                         (1, 1, 0.04, 0.03), (4000, 4, 0.02, 0.2)])
def test_ballquery_vs_oracle(n, B, r, sigma):
    xyz, bi, bo = _bq_case(n, B, r, sigma, seed=n)
    idx, sl = ops.ballquery_batch_p(_cuda(xyz), _cuda(bi), _cuda(bo), r, 50)
    oidx, osl = oracle.ballquery_batch_p(xyz, bi, bo, r)
    assert idx.numel() == oidx.size
    assert np.array_equal(sl.cpu().numpy()[:, 1], osl[:, 1])
    _assert_lists_equal(_lists(idx, sl), _lists(oidx, osl))
    # layout: lists tile [0, nActive) without overlap
    s = sl.cpu().numpy()
    order = np.argsort(s[:, 0], kind='stable')
    assert np.array_equal(np.cumsum(s[order, 1]) - s[order, 1], s[order, 0])


def test_ballquery_cap_and_oversize_cell():
    # 5000 candidates in one stencil (pass 0's staged path, just under its 5120 records; the exact scan and the other
    # paths are in test_gpu_neighbour_edges.py) and > 1000 neighbours (cap = first 1000 by index)
    rng = np.random.RandomState(1)
    xyz = (rng.randn(6000, 3) * 0.004).astype(np.float32)
    xyz[5000:] += 1.0
    bi = np.zeros(6000, np.int32)
    bo = np.array([0, 6000], np.int32)
    idx, sl = ops.ballquery_batch_p(_cuda(xyz), _cuda(bi), _cuda(bo), 0.04, 300)
    oidx, osl = oracle.ballquery_batch_p(xyz, bi, bo, 0.04)
    assert osl[:, 1].max() == 1000
    _assert_lists_equal(_lists(idx, sl), _lists(oidx, osl))


def test_ballquery_staged_cap():
    # cap hit inside the staged (shared-memory) path: ~3000 points in one stencil
    rng = np.random.RandomState(2)
    xyz = (rng.randn(3000, 3) * 0.006).astype(np.float32)
    bi = np.zeros(3000, np.int32)
    bo = np.array([0, 3000], np.int32)
    idx, sl = ops.ballquery_batch_p(_cuda(xyz), _cuda(bi), _cuda(bo), 0.04, 300)
    oidx, osl = oracle.ballquery_batch_p(xyz, bi, bo, 0.04)
    assert osl[:, 1].max() == 1000
    _assert_lists_equal(_lists(idx, sl), _lists(oidx, osl))


def test_ballquery_boundary_pairs():
    # pairs placed exactly around d = r: the fp32 contraction order decides; must match the oracle bit for bit
    rng = np.random.RandomState(4)
    r = np.float32(0.04)
    base = (rng.rand(2000, 3) * 0.3).astype(np.float32)
    d = rng.randn(2000, 3)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    eps = (rng.randint(-3, 4, (2000, 1)) * 2e-9)
    other = (base.astype(np.float64) + d * (float(r) + eps)).astype(np.float32)
    xyz = np.concatenate([base, other], 0)
    bi = np.zeros(4000, np.int32)
    bo = np.array([0, 4000], np.int32)
    idx, sl = ops.ballquery_batch_p(_cuda(xyz), _cuda(bi), _cuda(bo), float(r), 20)
    oidx, osl = oracle.ballquery_batch_p(xyz, bi, bo, float(r))
    _assert_lists_equal(_lists(idx, sl), _lists(oidx, osl))


def test_ballquery_full_size_scan():
    scan = synth.make_scan('c2_scannet', seed=0)
    scores, off = synth.grouping_inputs(scan, sigma=0.03, seed=0)
    sem = scan['semantic_labels']
    sel = np.where(sem >= 2)[0]
    order = np.argsort(sem[sel], kind='stable')
    sel = sel[order]
    xyz = (scan['coords_float'][sel] + off[sel]).astype(np.float32)
    cls, counts = np.unique(sem[sel], return_counts=True)
    bo = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    bi = np.repeat(np.arange(len(cls)), counts).astype(np.int32)
    idx, sl = ops.ballquery_batch_p(_cuda(xyz), _cuda(bi), _cuda(bo), 0.04, 300)
    # size-independent properties at full size + exact check on a sample of points
    s = sl.cpu().numpy()
    idn = idx.cpu().numpy()
    assert s[:, 1].min() >= 1 and s[:, 1].max() <= 1000
    rng = np.random.RandomState(0)
    for i in rng.choice(len(sel), 300, replace=False):
        lst = idn[s[i, 0]:s[i, 0] + s[i, 1]]
        b = bi[i]
        seg = np.arange(bo[b], bo[b + 1])
        o = xyz[i]
        p = xyz[seg]
        dx, dy, dz = (o[0] - p[:, 0]), (o[1] - p[:, 1]), (o[2] - p[:, 2])
        d2 = (dy * dy).astype(np.float32)
        d2 = (dx.astype(np.float64) * dx + d2).astype(np.float32)  # fma: exact product + single rounding
        d2 = (dz.astype(np.float64) * dz + d2).astype(np.float32)
        want = seg[d2 < np.float32(0.04) * np.float32(0.04)][:1000]
        assert np.array_equal(lst, want)


# ------------------------------------------------------------------ bfs_cluster
def test_bfs_cluster_golden(golden):
    mean = torch.tensor(golden['class_numpoint_mean'])
    for k in range(int(golden['bfs_count'])):
        ci, co = ops.bfs_cluster(mean, _cuda(golden['bfs%d_idx' % k]), _cuda(golden['bfs%d_sl' % k]),
                                 float(golden['bfs%d_thr' % k]), int(golden['bfs%d_cls' % k]))
        assert np.array_equal(ci.cpu().numpy(), golden['bfs%d_cidx' % k]), k
        assert np.array_equal(co.cpu().numpy(), golden['bfs%d_coff' % k]), k


def test_bfs_cluster_cpu_tensors_roundtrip(golden):
    # the reference passes CPU tensors (softgroup.py:458) and gets CPU tensors back
    mean = torch.tensor(golden['class_numpoint_mean'])
    ci, co = ops.bfs_cluster(mean, torch.from_numpy(golden['bfs0_idx']), torch.from_numpy(golden['bfs0_sl']),
                             float(golden['bfs0_thr']), int(golden['bfs0_cls']))
    assert not ci.is_cuda and not co.is_cuda
    assert np.array_equal(ci.numpy(), golden['bfs0_cidx']) and np.array_equal(co.numpy(), golden['bfs0_coff'])


def test_bfs_cluster_random_directed():
    rng = np.random.RandomState(11)
    mean = np.full(20, -1, np.float32)
    for t in range(25):
        n = rng.randint(1, 400)
        lens = rng.randint(0, 8, n)
        idx = rng.randint(0, n, int(lens.sum()) + 1).astype(np.int32)  # duplicates inside lists allowed
        sl = np.stack([np.concatenate([[0], np.cumsum(lens)[:-1]]), lens], 1).astype(np.int32)
        thr = float(rng.randint(1, 6))
        ci, co = ops.bfs_cluster(torch.from_numpy(mean), _cuda(idx), _cuda(sl), thr, 0)
        oi, oo = oracle.bfs_cluster(mean, idx, sl, thr, 0)
        assert np.array_equal(ci.cpu().numpy(), oi), t
        assert np.array_equal(co.cpu().numpy(), oo), t


def test_bfs_cluster_capped_lists_and_chain():
    # dense blob whose lists hit the 1000 cap (asymmetric graph) + a long chain (deep BFS, many levels)
    rng = np.random.RandomState(5)
    blob = (rng.randn(2500, 3) * 0.008).astype(np.float32)
    chain = np.stack([np.arange(3000) * 0.03 + 5, np.zeros(3000), np.zeros(3000)], 1).astype(np.float32)
    xyz = np.concatenate([blob, chain], 0)
    perm = rng.permutation(len(xyz))
    xyz = xyz[perm]
    n = len(xyz)
    oidx, osl = oracle.ballquery_batch_p(xyz, np.zeros(n, np.int32), np.array([0, n], np.int32), 0.04)
    assert osl[:, 1].max() == 1000
    mean = np.full(20, -1, np.float32)
    ci, co = ops.bfs_cluster(torch.from_numpy(mean), _cuda(oidx), _cuda(osl), 50.0, 3)
    oi, oo = oracle.bfs_cluster(mean, oidx, osl, 50.0, 3)
    assert len(oo) >= 3
    assert np.array_equal(co.cpu().numpy(), oo)
    assert np.array_equal(ci.cpu().numpy(), oi)


def test_bfs_cluster_edges_into_other_components():
    """Directed edges INTO other components (a node of a later component lists nodes of earlier ones: what lists cut by the
    1000 cap produce where objects touch). The listed node belongs to the component with the smaller seed and must not be
    claimed by the later one, whichever of the two the GPU happens to emit first: many components in flight at once,
    repeated to give the race a chance (it corrupted the BFS order on the 1.5M-point STPLS3D-shape tile before the fix)."""
    rng = np.random.RandomState(17)
    mean = np.full(20, -1, np.float32)
    sizes = rng.randint(40, 400, 300)
    starts = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    n = int(sizes.sum())
    lists = []
    for g, (s0, sz) in enumerate(zip(starts, sizes)):
        for i in range(sz):
            u = s0 + i
            nb = [s0 + (i + 1) % sz, s0 + (i * 7 + 3) % sz]               # a cycle + a chord: the group is strongly connected
            nb += list(s0 + rng.randint(0, sz, rng.randint(0, 6)))
            if g > 0:                                                    # edges into EARLIER groups only (labels stay apart)
                k = rng.randint(0, 12)
                h = rng.randint(0, g, k)
                nb += list(starts[h] + (rng.rand(k) * sizes[h]).astype(np.int64))
            rng.shuffle(nb)
            lists.append(np.asarray(nb, np.int32))
    lens = np.array([len(x) for x in lists], np.int32)
    idx = np.concatenate(lists).astype(np.int32)
    sl = np.stack([np.concatenate([[0], np.cumsum(lens)[:-1]]), lens], 1).astype(np.int32)
    oi, oo = oracle.bfs_cluster(mean, idx, sl, 10.0, 0)
    assert len(oo) - 1 == len(sizes) and oi.shape[0] == n
    d_idx, d_sl = _cuda(idx), _cuda(sl)
    for rep in range(10):
        ci, co = ops.bfs_cluster(torch.from_numpy(mean), d_idx, d_sl, 10.0, 0)
        assert np.array_equal(co.cpu().numpy(), oo), rep
        assert np.array_equal(ci.cpu().numpy(), oi), rep


def test_bfs_cluster_full_size_pipeline():
    # full-size scan, one class at a time like the reference loop; GPU lists -> GPU bfs vs oracle bfs on same lists
    scan = synth.make_scan('c2_scannet', seed=1)
    scores, off = synth.grouping_inputs(scan, sigma=0.03, seed=1)
    sem = scan['semantic_labels']
    mean = np.array(MEAN, np.float32)
    cls_ids, cnts = np.unique(sem, return_counts=True)
    tested = 0
    for cls in cls_ids[np.argsort(-cnts)]:
        if cls < 2:
            continue
        sel = np.where(sem == cls)[0]
        xyz = (scan['coords_float'][sel] + off[sel]).astype(np.float32)
        bi = torch.zeros(len(sel), dtype=torch.int32, device='cuda')
        bo = torch.tensor([0, len(sel)], dtype=torch.int32, device='cuda')
        idx, sl = ops.ballquery_batch_p(_cuda(xyz), bi, bo, 0.04, 300)
        ci, co = ops.bfs_cluster(torch.from_numpy(mean), idx, sl, 0.05, int(cls))
        oi, oo = oracle.bfs_cluster(mean, idx.cpu().numpy(), sl.cpu().numpy(), 0.05, int(cls))
        assert np.array_equal(co.cpu().numpy(), oo)
        assert np.array_equal(ci.cpu().numpy(), oi)
        tested += 1
        if tested == 3:
            break


# ------------------------------------------------------------------ segment ops
def _segments(rng, nP, maxlen, allow_empty=True):
    lens = rng.randint(0 if allow_empty else 1, maxlen, nP)
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)


@pytest.mark.parametrize('C', [3, 32, 40])
def test_sec_ops_and_avg_pool(C):
    rng = np.random.RandomState(C)
    off = _segments(rng, 57, 900, allow_empty=False)
    x = rng.randn(off[-1], C).astype(np.float32)
    xc, oc = _cuda(x), _cuda(off)
    assert np.array_equal(ops.sec_min(xc, oc).cpu().numpy(), oracle.sec_min(x, off))
    assert np.array_equal(ops.sec_max(xc, oc).cpu().numpy(), oracle.sec_max(x, off))
    # tree-order sums: within 1e-5 relative of the sequential reference order (bar: 1e-4)
    np.testing.assert_allclose(ops.sec_mean(xc, oc).cpu().numpy(), oracle.sec_mean(x, off), rtol=1e-5, atol=1e-6)
    xg = xc.clone().requires_grad_(True)
    y = ops.global_avg_pool(xg, oc)
    np.testing.assert_allclose(y.detach().cpu().numpy(), oracle.global_avg_pool(x, off), rtol=1e-5, atol=1e-6)
    g = rng.randn(57, C).astype(np.float32)
    y.backward(_cuda(g))
    np.testing.assert_allclose(xg.grad.cpu().numpy(), oracle.global_avg_pool_bp(g, off, off[-1]), rtol=1e-6, atol=1e-7)


def test_sec_ops_empty_segment():
    off = np.array([0, 3, 3, 5], np.int32)
    x = np.arange(15, dtype=np.float32).reshape(5, 3)
    assert np.array_equal(ops.sec_min(_cuda(x), _cuda(off)).cpu().numpy(), oracle.sec_min(x, off))  # +inf row
    assert np.array_equal(ops.sec_max(_cuda(x), _cuda(off)).cpu().numpy(), oracle.sec_max(x, off))
    assert np.array_equal(ops.sec_mean(_cuda(x), _cuda(off)).cpu().numpy(), oracle.sec_mean(x, off))


# ------------------------------------------------------------------ mask IoU / labels
def test_mask_iou_and_label():
    rng = np.random.RandomState(9)
    N, nI, nP = 5000, 23, 31
    labels = rng.randint(-1, nI, N).astype(np.int64)
    labels[labels < 0] = -100
    pointnum = np.bincount(labels[labels >= 0], minlength=nI).astype(np.int32)
    cls = rng.randint(0, 18, nI).astype(np.int64)
    cls[[2, 7]] = -100
    off = _segments(rng, nP, 400, allow_empty=False)
    pidx = rng.randint(0, N, off[-1]).astype(np.int32)
    sig = rng.rand(off[-1]).astype(np.float32)
    a = ops.get_mask_iou_on_cluster(_cuda(pidx), _cuda(off), _cuda(labels), _cuda(pointnum))
    assert np.array_equal(a.cpu().numpy(), oracle.get_mask_iou_on_cluster(pidx, off, labels, pointnum))
    b = ops.get_mask_iou_on_pred(_cuda(pidx), _cuda(off), _cuda(labels), _cuda(pointnum), _cuda(sig))
    assert np.array_equal(b.cpu().numpy(), oracle.get_mask_iou_on_pred(pidx, off, labels, pointnum, sig))
    iou = a.cpu().numpy()
    m = ops.get_mask_label(_cuda(pidx), _cuda(off), _cuda(labels), _cuda(cls), _cuda(pointnum), a, 0.02)
    assert np.array_equal(m.cpu().numpy(), oracle.get_mask_label(pidx, off, labels, cls, pointnum, iou, 0.02))


# ------------------------------------------------------------------ octree ball query (SoftGroup++)
def test_octree_build_golden(golden):
    boxes, pt_inds, psl = ops.build_octree(_cuda(golden['oct_pts']))
    assert np.array_equal(boxes.cpu().numpy(), golden['oct_boxes'])
    assert np.array_equal(pt_inds.cpu().numpy(), golden['oct_pt_inds'])
    assert np.array_equal(psl.cpu().numpy(), golden['oct_psl'])


@pytest.mark.parametrize('n,r,scale', [(3000, 0.15, (3., 2., 1.)), (20000, 0.05, (2., 2., 0.5)), (1, 0.1, (1., 1., 1.)),
                                       (6000, 0.6, (1., 1., 1.))])
def test_octree_ball_query_vs_oracle(n, r, scale):
    rng = np.random.RandomState(n)
    pts = (rng.rand(n, 3) * np.array(scale)).astype(np.float32)
    boxes, pt_inds, psl = ops.build_octree(_cuda(pts))
    ob, oi, op = oracle.build_octree(pts)
    assert np.array_equal(boxes.cpu().numpy(), ob) and np.array_equal(pt_inds.cpu().numpy(), oi)
    assert np.array_equal(psl.cpu().numpy(), op)
    idx, sl = ops.octree_ball_query(_cuda(pts), 20, r)
    oidx, osl = oracle.octree_ball_query(pts, 20, r)
    assert idx.numel() == oidx.size
    _assert_lists_equal(_lists(idx, sl), _lists(oidx, osl))  # leaf-major order, cap 1000 (n=6000, r=0.6 hits it)


def test_ballquery_wide_index_range_uses_sort_fallback():
    # two far-apart index blocks in one dense stencil: index range > 262144 -> bitonic fallback path
    rng = np.random.RandomState(8)
    n = 300000
    xyz = (rng.rand(n, 3) * 40).astype(np.float32)      # sparse background
    xyz[:300] = (rng.randn(300, 3) * 0.01 + 5).astype(np.float32)    # dense blob, low indices
    xyz[-300:] = (rng.randn(300, 3) * 0.01 + 5).astype(np.float32)   # same blob, high indices
    bi = np.zeros(n, np.int32)
    bo = np.array([0, n], np.int32)
    idx, sl = ops.ballquery_batch_p(_cuda(xyz), _cuda(bi), _cuda(bo), 0.04, 5)
    s = sl.cpu().numpy()
    g = idx.cpu().numpy()
    for i in list(range(0, 300, 7)) + list(range(n - 300, n, 7)):
        o = xyz[i]
        d = xyz - o
        d2 = (d[:, 1] * d[:, 1]).astype(np.float32)
        d2 = (d[:, 0].astype(np.float64) * d[:, 0] + d2).astype(np.float32)
        d2 = (d[:, 2].astype(np.float64) * d[:, 2] + d2).astype(np.float32)
        want = np.where(d2 < np.float32(0.04) * np.float32(0.04))[0][:1000]
        assert np.array_equal(g[s[i, 0]:s[i, 0] + s[i, 1]], want), i


@pytest.mark.parametrize('n,batch,min_npoint', [(5000, 1, 0), (40000, 3, 60), (150000, 1, 100), (1, 1, 0)])
def test_group_entries_equals_reference_loop(n, batch, min_npoint):
    """csrc/grouping.cu vs the reference's per-class loop (softgroup.py:430-446): entries, segments, shifted coordinates,
    segment offsets and per-class counts, bit-exact (random scores around the threshold, classes dropped by min_npoint)."""
    from softgroup_b200.ops import group_entries
    from test_host_grouping import _fake_group_entries
    g = torch.Generator().manual_seed(n + batch)
    C = 20
    logits = torch.randn(n, C, generator=g) * 2
    logits[:, 5] -= 6  # a rare class: falls below min_npoint
    scores = logits.softmax(-1)
    classes = [c for c in range(C) if c not in (0, 1)]
    bsz = torch.sort(torch.randint(0, batch, (n, ), generator=g))[0].int()
    coords, offs = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g) * 0.1
    want = _fake_group_entries(scores, classes, 0.2, min_npoint, bsz, batch, coords, offs)
    got = group_entries(scores.cuda(), classes, 0.2, min_npoint, bsz.cuda(), batch, coords.cuda(), offs.cuda())
    tot = got[4].cpu()
    assert torch.equal(tot, want[4])
    m = int(tot[0])
    assert torch.equal(got[0][:m].cpu(), want[0]) and torch.equal(got[1][:m].cpu(), want[1])
    assert torch.equal(got[2][:m].cpu(), want[2])
    assert torch.equal(got[3].cpu(), want[3])
