"""GPU: the ball query, the clustering and the octree ball query on every internal path, against the C oracle (the
reference's algorithms, pinned on its compiled kernels) index for index. The cases are listed in
tests/neighbour_cases.py; tests/test_neighbour_coverage.py checks that they reach every path.

Where a segment is too large for the brute-force oracle (the 327k-point wide-index-range case), a fixed sample of
queries -- every query of a structure and 2000 others, covering every path the case reaches -- is checked against a
numpy restatement of the reference: same-segment points in ascending index order whose float32 distance, in the
reference's contraction order fma(dz, dz, fma(dx, dx, dy * dy)), is below radius^2, first 1000 kept."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from softgroup_b200 import ops
from softgroup_b200.ops import _lib, ballquery_batch_p_nosync, bfs_cluster_segments
from softgroup_b200.ops._lib import check, ptr

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import neighbour_cases as nc  # noqa: E402

pytestmark = pytest.mark.gpu
SENTINEL = 0x5A5A5A5A
GUARD = 4096  # sentinel words behind the capacity


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _lists(idx, sl):
    return [idx[s:s + l] for s, l in sl]


def _assert_tiles(sl, total):
    """start_len lists tile [0, total) without gaps or overlap (in the order the atomic cursor handed them out)."""
    nz = sl[sl[:, 1] > 0]
    nz = nz[np.argsort(nz[:, 0], kind='stable')]
    assert int(sl[:, 1].sum()) == total
    assert np.array_equal(np.cumsum(nz[:, 1]) - nz[:, 1], nz[:, 0])


def _assert_lists(got_idx, got_sl, want, queries, what):
    for i in queries:
        s, l = got_sl[i]
        assert np.array_equal(got_idx[s:s + l], want[i]), '%s: point %d: %s vs %s' % (what, i, got_idx[s:s + l][:8],
                                                                                          want[i][:8])


# ================================================================== ball query
def _numpy_ballquery(xyz, bi, bo, radius, queries):
    """{query: list} by the reference's rule, for the given queries (see the module docstring)."""
    r2 = np.float32(radius) * np.float32(radius)
    out = {}
    queries = np.asarray(queries)
    for b in np.unique(bi[queries]):
        seg = np.arange(bo[b], bo[b + 1])
        by_x = seg[np.argsort(xyz[seg, 0], kind='stable')]
        xs = xyz[by_x, 0].astype(np.float64)
        qs = queries[bi[queries] == b]
        coarse = np.floor(xyz[qs].astype(np.float64) / (8 * radius)).astype(np.int64)
        _, group = np.unique(coarse, axis=0, return_inverse=True)
        for g in range(group.max() + 1):
            G = qs[group.reshape(-1) == g]
            lo = xyz[G].astype(np.float64).min(0) - 1.01 * radius
            hi = xyz[G].astype(np.float64).max(0) + 1.01 * radius
            a, e = np.searchsorted(xs, lo[0]), np.searchsorted(xs, hi[0], side='right')
            cand = by_x[a:e]
            p = xyz[cand].astype(np.float64)
            cand = np.sort(cand[((p[:, 1:] >= lo[1:]) & (p[:, 1:] <= hi[1:])).all(1)])
            P = xyz[cand]
            for c0 in range(0, len(G), 128):
                Q = xyz[G[c0:c0 + 128]]
                dx, dy, dz = (Q[:, None, k] - P[None, :, k] for k in range(3))  # float32 differences
                d2 = dy * dy
                d2 = (dx.astype(np.float64) * dx + d2).astype(np.float32)  # fma: exact product, one rounding
                d2 = (dz.astype(np.float64) * dz + d2).astype(np.float32)
                hit = d2 < r2
                for k, q in enumerate(G[c0:c0 + 128]):
                    out[int(q)] = cand[hit[k]][:nc.MAX_NEIGHBORS]
    return out


@pytest.fixture(scope='module')
def bq_cases():
    cache = {}

    def get(name):
        if name not in cache:
            c = nc.bq_case(name)
            xyz, bi, bo = c.make()
            cache[name] = (c, xyz, bi, bo, nc.bq_route(xyz, bi, c.radius))
        return cache[name]
    return get


@pytest.mark.parametrize('name', [c.name for c in nc.BQ_CASES])
def test_ballquery_case(bq_cases, name):
    """Blocking (relaunching) and asynchronous entry points, every list against the oracle (or the sample)."""
    c, xyz, bi, bo, route = bq_cases(name)
    n = len(xyz)
    d_xyz, d_bi, d_bo = _cuda(xyz), _cuda(bi), _cuda(bo)
    idx, sl = ops.ballquery_batch_p(d_xyz, d_bi, d_bo, c.radius, 50)
    aidx, asl, atot = ballquery_batch_p_nosync(d_xyz, d_bi, d_bo, c.radius)
    torch.cuda.synchronize()
    idx, sl, asl, atot = idx.cpu().numpy(), sl.cpu().numpy(), asl.cpu().numpy(), atot.cpu().numpy()
    aidx = aidx[:int(atot[0])].cpu().numpy()
    assert atot[1] == 0
    _assert_tiles(sl, len(idx))
    _assert_tiles(asl, int(atot[0]))
    path_of = np.where(route.cell_of >= 0, route.cell_path[np.maximum(route.cell_of, 0)], 'none')
    if c.full_oracle:
        oidx, osl = oracle.ballquery_batch_p(xyz, bi, bo, c.radius)
        assert len(idx) == len(oidx) and np.array_equal(sl[:, 1], osl[:, 1])
        want = _lists(oidx, osl)
        queries = np.arange(n)
    else:
        rng = np.random.RandomState(0)
        structure = np.nonzero(path_of != 'p0_bitmap')[0]
        queries = np.union1d(structure, rng.choice(n, 2000, replace=False))
        want = _numpy_ballquery(xyz, bi, bo, c.radius, queries)
        assert set(path_of[queries]) == set(path_of), 'the sample misses a path'
    _assert_lists(idx, sl, want, queries, 'blocking')
    _assert_lists(aidx, asl, want, queries, 'async')
    counts = {p: int((path_of[queries] == p).sum()) for p in nc.BQ_PATHS}
    print('%s: %d points, %d checked per path %s' % (name, n, len(queries), counts))


def _assert_truncated(buf, sl, cap, want_lists):
    """Reference truncation (bfs_cluster.cu:55-61): lists below the capacity exact, the list across it a prefix, nothing
    written at or beyond it."""
    straddle = 0
    for (s, l), w in zip(sl, want_lists):
        assert l == len(w)
        if s + l <= cap:
            assert np.array_equal(buf[s:s + l], w)
        elif s < cap:
            assert np.array_equal(buf[s:cap], w[:cap - s])
            straddle += 1
    assert straddle == 1
    assert (buf[cap:] == SENTINEL).all(), 'words written beyond the capacity'


@pytest.mark.parametrize('name,mean_active', nc.BQ_TRUNCATION)
def test_ballquery_truncation_at_the_c_abi(bq_cases, name, mean_active):
    """The C entry points with a capacity that ends inside a list (every list is capped at 1000 entries and n = 1 mod
    1000): the blocking one at n * meanActive, the asynchronous one at an arbitrary capacity."""
    c, xyz, bi, bo, route = bq_cases(name)
    n, B = len(xyz), len(bo) - 1
    oidx, osl = oracle.ballquery_batch_p(xyz, bi, bo, c.radius)
    want = _lists(oidx, osl)
    L = _lib.lib()
    d_xyz, d_bi, d_bo = _cuda(xyz), _cuda(bi), _cuda(bo)
    ws = torch.empty(L.sgb_ballquery_workspace_bytes(n), dtype=torch.uint8, device='cuda')
    for cap in (n * mean_active, len(oidx) // 2 + 517):
        buf = torch.full((cap + GUARD, ), SENTINEL, dtype=torch.int32, device='cuda')
        sl = torch.full((n, 2), -1, dtype=torch.int32, device='cuda')
        if cap == n * mean_active:
            total = check(L.sgb_ballquery_batch_p(n, mean_active, float(c.radius), ptr(d_xyz), ptr(d_bi), ptr(d_bo), B,
                                                  ptr(buf), ptr(sl), ptr(ws), ws.numel(), _stream()), 'ballquery')
        else:
            tot = torch.full((2, ), -1, dtype=torch.int32, device='cuda')
            check(L.sgb_ballquery_batch_p_async(n, cap, float(c.radius), ptr(d_xyz), ptr(d_bi), ptr(d_bo), B, ptr(buf),
                                                ptr(sl), ptr(tot), ptr(ws), ws.numel(), _stream()), 'ballquery_async')
            t = tot.cpu().numpy()
            assert t[1] == 0
            total = int(t[0])
        torch.cuda.synchronize()
        assert total == len(oidx) > cap
        s = sl.cpu().numpy()
        _assert_tiles(s, total)
        _assert_truncated(buf.cpu().numpy(), s, cap, want)


# ================================================================== bfs_cluster
_MEAN = np.full(1, -1, np.float32)  # class mean -1: the threshold is absolute (bfs_cluster.cpp:70-77)


@pytest.mark.parametrize('name', [c.name for c in nc.BFS_CASES])
def test_bfs_case(name):
    c = nc.bfs_case(name)
    idx, sl = c.make()
    ci, co = ops.bfs_cluster(torch.from_numpy(_MEAN), _cuda(idx), _cuda(sl), c.thr, 0)
    oi, oo = oracle.bfs_cluster(_MEAN, idx, sl, c.thr, 0)
    assert np.array_equal(co.cpu().numpy(), oo)
    assert np.array_equal(ci.cpu().numpy(), oi)
    print('%s: N=%d maxLen=%d clusters=%d' % (name, len(sl), sl[:, 1].max(), len(oo) - 1))


def _count_launches(idx, sl, thr):
    """Launches of sgb_bfs_cluster_count alone (label propagation, sizes, threshold, scan)."""
    L = _lib.lib()
    n = len(sl)
    d_idx, d_sl = _cuda(idx), _cuda(sl)
    ws = torch.empty(L.sgb_bfs_cluster_workspace_bytes(n), dtype=torch.uint8, device='cuda')
    s, mx = ctypes.c_int(0), ctypes.c_int(0)
    l0 = L.sgb_launch_count()
    nc_ = check(L.sgb_bfs_cluster_count(ptr(d_idx), ptr(d_sl), n, float(thr), None, None, None, ptr(ws), ws.numel(),
                                        ctypes.byref(s), ctypes.byref(mx), _stream()), 'bfs_cluster_count')
    return L.sgb_launch_count() - l0, nc_, s.value


def test_bfs_label_propagation_takes_several_batches():
    """Descending chains need one propagation pass per hop: the count must run several batches of 12 passes (each
    batch re-runs size, pack and scan) and still give the oracle's clusters."""
    c = nc.bfs_case('descending_chains')
    idx, sl = c.make()
    n = len(sl)
    self_loops = np.arange(n, dtype=np.int32)  # converges in the first batch
    one, _, _ = _count_launches(self_loops, np.stack([np.arange(n), np.ones(n)], 1).astype(np.int32), c.thr)
    many, ncl, s = _count_launches(idx, sl, c.thr)
    oi, oo = oracle.bfs_cluster(_MEAN, idx, sl, c.thr, 0)
    assert (ncl, s) == (len(oo) - 1, len(oi))
    assert (many - 1) % (one - 1) == 0, (many, one)  # init + batches * (2 * 12 + size + pack + scan)
    batches = (many - 1) // (one - 1)
    assert batches >= 3, batches
    print('descending chains: %d batches of %d passes' % (batches, nc.BFS_BATCH))


def _segment_threshold_oracle(idx, sl, node_seg, seg_thr):
    """Every component of the oracle's BFS, kept iff (float)size >= seg_thr[node_seg[seed]], renumbered."""
    oi, oo = oracle.bfs_cluster(_MEAN, idx, sl, 0.0, 0)
    rows, offs = [], [0]
    for k in range(len(oo) - 1):
        comp = oi[oo[k]:oo[k + 1], 1]
        if np.float32(len(comp)) >= seg_thr[node_seg[comp[0]]]:
            rows.append(np.stack([np.full(len(comp), len(offs) - 1), comp], 1))
            offs.append(offs[-1] + len(comp))
    return (np.concatenate(rows).astype(np.int32) if rows else np.zeros((0, 2), np.int32)), np.array(offs, np.int32)


def test_bfs_segment_thresholds():
    idx, sl, node_seg = nc.threshold_graph()
    n = len(sl)
    for seg_thr in (nc.threshold_values(n), np.full(len(nc.threshold_values(n)), n + 1.0, np.float32)):
        ci, co = bfs_cluster_segments(_cuda(idx), _cuda(sl), 0.0, node_seg=_cuda(node_seg), seg_thr=_cuda(seg_thr))
        wi, wo = _segment_threshold_oracle(idx, sl, node_seg, seg_thr)
        assert np.array_equal(co.cpu().numpy(), wo)
        assert np.array_equal(ci.cpu().numpy().reshape(-1, 2), wi)
    assert len(wo) == 1  # the second set keeps nothing: nCluster = 0


# ================================================================== octree ball query
@pytest.mark.parametrize('name', [c.name for c in nc.OC_CASES])
def test_octree_case(name, ref_ops):
    c = nc.oc_case(name)
    pts = c.make()
    boxes, pt_inds, psl = ops.build_octree(_cuda(pts))
    ob, oi, op = oracle.build_octree(pts)
    assert np.array_equal(boxes.cpu().numpy(), ob) and np.array_equal(pt_inds.cpu().numpy(), oi)
    assert np.array_equal(psl.cpu().numpy(), op)
    idx, sl = ops.octree_ball_query(_cuda(pts), 20, c.radius)
    idx, sl = idx.cpu().numpy(), sl.cpu().numpy()
    oidx, osl = oracle.octree_ball_query(pts, 20, c.radius)
    assert len(idx) == len(oidx) and np.array_equal(sl[:, 1], osl[:, 1])
    _assert_tiles(sl, len(idx))
    want = _lists(oidx, osl)
    _assert_lists(idx, sl, want, range(len(pts)), name)
    if name in nc.DEGENERATE_OC and ref_ops is not None:
        # the oracle's restatement was pinned on regular clouds: pin it on the degenerate boxes as well
        n = len(pts)
        rb, rp, rs = torch.zeros(585, 6), torch.zeros(n, dtype=torch.int32), torch.zeros(512, 2, dtype=torch.int32)
        mx, mn = pts.max(0), pts.min(0)
        xyzwhl = torch.from_numpy(np.concatenate([(mx + mn) / np.float32(2), mx - mn]).astype(np.float32))
        ref_ops.build_and_export_octree(torch.from_numpy(pts), xyzwhl, rb, rp, rs, 3)
        assert np.array_equal(rb.numpy(), ob) and np.array_equal(rp.numpy(), oi) and np.array_equal(rs.numpy(), op)
        mean_active = nc.MAX_NEIGHBORS
        out_inds = torch.zeros(n * mean_active, dtype=torch.int32, device='cuda')
        out_sl = torch.zeros((n, 2), dtype=torch.int32, device='cuda')
        tot = ref_ops.octree_ball_query(_cuda(pts), _cuda(ob), _cuda(oi), _cuda(op), out_inds, out_sl, mean_active,
                                        c.radius)
        assert tot == len(oidx)
        _assert_lists(out_inds.cpu().numpy(), out_sl.cpu().numpy(), want, range(n), name + ' (reference kernel)')
        print('%s: oracle == compiled reference (build and query)' % name)


@pytest.mark.parametrize('name,mean_active', nc.OC_TRUNCATION)
def test_octree_truncation_at_the_c_abi(name, mean_active):
    c = nc.oc_case(name)
    pts = c.make()
    n = len(pts)
    oidx, osl = oracle.octree_ball_query(pts, 20, c.radius)
    L = _lib.lib()
    d_pts = _cuda(pts)
    boxes, pt_inds, psl = ops.build_octree(d_pts)
    cap = n * mean_active
    buf = torch.full((cap + GUARD, ), SENTINEL, dtype=torch.int32, device='cuda')
    sl = torch.full((n, 2), -1, dtype=torch.int32, device='cuda')
    total = torch.zeros(1, dtype=torch.int32, device='cuda')
    got = check(L.sgb_octree_ball_query(ptr(d_pts), ptr(boxes), ptr(pt_inds), ptr(psl), n, mean_active, float(c.radius),
                                        ptr(buf), ptr(sl), ptr(total), _stream()), 'octree_ball_query')
    assert got == len(oidx) > cap
    s = sl.cpu().numpy()
    _assert_tiles(s, got)
    _assert_truncated(buf.cpu().numpy(), s, cap, _lists(oidx, osl))
