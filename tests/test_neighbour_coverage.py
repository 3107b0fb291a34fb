"""CPU: the case table of tests/neighbour_cases.py reaches every internal path of the ball query, the clustering and the
octree query that tests/test_gpu_neighbour_edges.py is there to exercise, and the launch constants it mirrors still
match the .cu sources. No GPU compute."""
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import neighbour_cases as nc  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _src(name):
    with open(os.path.join(ROOT, 'softgroup_b200', 'csrc', name)) as f:
        return f.read()


def _const(src, pattern):
    m = re.search(pattern, src)
    assert m, pattern
    return int(m.group(1))


def test_constants_match_the_sources():
    bq = _src('ballquery.cu')
    for p, c in nc.BQ_CFG.items():
        m = re.search(r'struct BqCfg<%d> \{ static constexpr int kThreads = (\d+), kSMax = (\d+), kSortMax = (\d+), '
                      r'kBmWords = (\d+)' % p, bq)
        assert m, p
        assert tuple(int(x) for x in m.groups()) == (c['threads'], c['smax'], c['sort_max'], c['bm_words'])
        assert 'sizeof(float4) * BqCfg<%d>::kSMax + 6 * BqCfg<%d>::kBmWords' % (p, p) in bq  # bq_smem_bytes
    assert _const(bq, r'constexpr int kBqChunk = (\d+);') == nc.BQ_CHUNK
    assert _const(bq, r'constexpr int kMaxSeg = (\d+);') == nc.BQ_MAX_SEG
    assert _const(bq, r'constexpr int kCellBias = (\d+);') == nc.BQ_CELL_BIAS
    assert 'const double lim = (double)(kCellBias - 2);' in bq
    assert 'double h = (double)radius * (1.0 + 1e-4);' in bq
    # the routing bq_path restates
    assert 'const bool use_bitmap = nwords <= kBmWords;' in bq
    assert 'const bool staged = total_s <= (use_bitmap ? kBqSMax : BqCfg<PASS>::kSortMax);' in bq
    bfs = _src('bfs_cluster.cu')
    assert 'if (W > %d) return 0;' % nc.BFS_EMIT2_MAX_W in bfs and 'if (W <= %d) {' % nc.BFS_EMIT2_MAX_W in bfs
    assert _const(bfs, r'constexpr int kBatch = (\d+);') == nc.BFS_BATCH
    assert _const(bfs, r'constexpr int kCl = (\d+);') == nc.BFS_CL
    assert _const(bfs, r'constexpr int kClThreads = (\d+);') == nc.BFS_CL_THREADS
    assert _const(_src('octree.cu'), r'constexpr int OC_BLK = (\d+);') == nc.OC_BLK
    with open(os.path.join(ROOT, 'include', 'sgb200.h')) as f:
        assert _const(f.read(), r'#define SGB_MAX_NEIGHBORS (\d+)') == nc.MAX_NEIGHBORS


def test_routing_table():
    assert nc.bq_path(5120, 4096) == 'p0_bitmap' and nc.bq_path(5121, 4096) == 'p1_bitmap'
    assert nc.bq_path(4096, 4097) == 'p0_bitonic' and nc.bq_path(4097, 4097) == 'p1_bitmap'
    assert nc.bq_path(4097, 8193) == 'p1_bitonic' and nc.bq_path(8192, 8193) == 'p1_bitonic'
    assert nc.bq_path(8193, 8193) == 'exact' and nc.bq_path(10240, 8192) == 'p1_bitmap'
    assert nc.bq_path(10241, 1) == 'exact'
    # every staged stencil fits its configuration's staging area, bitonic padding included
    for t in range(1, 12001, 7):
        for w in (1, 4096, 4097, 8192, 8193):
            path = nc.bq_path(t, w)
            if path != 'exact':
                c = nc.BQ_CFG[int(path[1])]
                assert t <= c['smax'] and ('bitmap' in path or nc.bitonic_p(t) <= c['smax']), (t, w)


@pytest.fixture(scope='module')
def bq_routes():
    out = {}
    for c in nc.BQ_CASES:
        xyz, bi, bo = c.make()
        r = nc.bq_route(xyz, bi, c.radius)
        cnt = nc.neighbour_counts(xyz, bi, c.radius)
        cell_max = np.zeros(len(r.cell_cnt), np.int64)
        hashed = r.cell_of >= 0
        np.maximum.at(cell_max, r.cell_of[hashed], cnt[hashed])
        out[c.name] = (xyz, bi, bo, r, cell_max)
    return out


def test_ballquery_cases_reach_every_path(bq_routes):
    capped, uncapped = set(), set()
    for xyz, bi, bo, r, cell_max in bq_routes.values():
        capped |= set(r.cell_path[cell_max >= nc.MAX_NEIGHBORS + 100])
        uncapped |= set(r.cell_path[cell_max <= nc.MAX_NEIGHBORS - 100])
    assert capped == set(nc.BQ_PATHS), 'a path without a case whose lists hit the 1000 cap'
    assert uncapped == set(nc.BQ_PATHS), 'a path without a case below the cap'


def test_ballquery_bitonic_bands(bq_routes):
    """The stencils whose bitonic padding used to overrun the staging area are in the table, capped and not, and now go
    on to the next configuration: (4096, 5120] from pass 0 to pass 1, (8192, 10240] from pass 1 to the exact scan."""
    for p, lo, hi, now in ((0, 4096, 5120, {'p1_bitmap', 'p1_bitonic'}), (1, 8192, 10240, {'exact'})):
        c = nc.BQ_CFG[p]
        seen = set()
        for xyz, bi, bo, r, cell_max in bq_routes.values():
            band = (r.total_s > lo) & (r.total_s <= hi) & (r.nwords > c['bm_words'])
            for t, w, path, m in zip(r.total_s[band], r.nwords[band], r.cell_path[band], cell_max[band]):
                assert nc.bq_path_before_fix(t, w) == 'p%d_bitonic' % p
                assert 16 * nc.bitonic_p(t) > nc.bq_smem_bytes(p)  # what the old routing staged
                assert path in now
                seen.add(m >= nc.MAX_NEIGHBORS + 100)
        assert seen == {True, False}, (p, seen)
    # and the wide case reaches pass 1's bitonic sort outside the band as well
    r = bq_routes['wide_index_range'][3]
    assert ((r.cell_path == 'p1_bitonic') & (r.total_s > nc.BQ_CFG[0]['smax'])).any()


def test_ballquery_cases_reach_the_edges(bq_routes):
    q = np.concatenate([r.cell_cnt for _, _, _, r, _ in bq_routes.values()])
    assert {128, 129} <= set(q.tolist()) and (q > 2 * nc.BQ_CHUNK).any(), 'work items per cell: 1, 2 and 3+'
    xyz, bi, bo, r, _ = bq_routes['segments_1023']
    lens = np.diff(bo)
    assert len(lens) == nc.BQ_MAX_SEG and (lens == 0).sum() >= 2 and lens[-1] == 0 and (lens == 1).sum() >= 2
    # the same coordinates in different segments
    _, first, counts = np.unique(xyz, axis=0, return_index=True, return_counts=True)
    dup = first[counts > 1]
    assert len(dup) >= 40 and all(len(np.unique(bi[(xyz == xyz[i]).all(1)])) > 1 for i in dup[:5])
    # the outermost addressable cells, on every axis and both sides
    xyz, bi, bo, r, _ = bq_routes['cell_range_edges']
    f = np.floor(xyz.astype(np.float64) * (1.0 / (1.0 * (1 + 1e-4))))
    lim = nc.BQ_CELL_BIAS - 3
    assert (f.max(0) == lim).all() and (f.min(0) == -lim).all()
    assert ((f == lim - 1).any(0)).all() and ((f == 1 - lim).any(0)).all() and ((f == -1).any(0)).all()


def test_bfs_cases_reach_every_path():
    import oracle
    maxlen, wide, comps = {}, 0, 0
    for c in nc.BFS_CASES:
        idx, sl = c.make()
        n = len(sl)
        assert idx.dtype == np.int32 and sl.dtype == np.int32 and (idx >= 0).all() and (idx < n).all()
        assert np.array_equal(np.cumsum(sl[:, 1]) - sl[:, 1], sl[:, 0])
        m = int(sl[:, 1].max())
        maxlen[c.name] = m
        seeds, widest = nc.bfs_levels(idx, sl)
        wide = max(wide, widest)
        comps = max(comps, len(seeds))
        if c.name not in ('wide_frontier', 'many_components', 'descending_chains'):
            # self-loops and duplicate entries inside lists, on both emit paths
            lists = [idx[s:s + l] for s, l in sl]
            assert any(u in lst for u, lst in enumerate(lists)) and any(len(np.unique(x)) < len(x) for x in lists)
        ci, co = oracle.bfs_cluster(np.full(1, -1, np.float32), idx, sl, c.thr, 0)
        assert len(co) >= 2, 'every case keeps a cluster'
    w = {k: (v + 31) // 32 for k, v in maxlen.items()}
    assert {32, 33, 2048, 2049} <= set(maxlen.values()) and any(4500 <= v <= 6000 for v in maxlen.values())
    assert {1, 2, nc.BFS_EMIT2_MAX_W, nc.BFS_EMIT2_MAX_W + 1} <= set(w.values())
    assert wide > nc.BFS_CL_THREADS, 'a BFS level wider than one emit2 scan tile'
    assert comps >= 20000 > 132 * 4 // nc.BFS_CL, 'more components than resident emit2 clusters'
    # label propagation: one pass per hop of a descending chain, several batches of kBatch passes
    idx, sl = nc.bfs_case('descending_chains').make()
    s = 0
    hops = 0
    u = s
    while True:
        nxt = [v for v in idx[sl[u, 0]:sl[u, 0] + sl[u, 1]] if v != u]
        if not nxt:
            break
        u = nxt[0]
        hops += 1
    assert hops >= 3 * nc.BFS_BATCH


def test_threshold_cases():
    idx, sl, node_seg = nc.threshold_graph()
    n = len(sl)
    thr = nc.threshold_values(n)
    sizes = set(nc.THR_COMPONENT_SIZES)
    assert 0.0 in thr and (thr > n).any() and len(sizes & set(thr.tolist())) >= 2
    assert any(np.float32(t) > s and np.nextafter(np.float32(t), np.float32(0)) <= s for t in thr for s in sizes)
    assert node_seg.max() + 1 == len(thr)


def _octree_splits(pts):
    """Per level, the number of points lying exactly on a split plane of the node they pass through."""
    import oracle
    boxes = oracle.build_octree(pts)[0]
    node = np.zeros(len(pts), np.int64)
    ties = []
    for lvl in range(3):
        b = boxes[node]
        ties.append(int((pts == b[:, :3]).any(1).sum()))
        o = (pts >= b[:, :3]).astype(np.int64)
        node = 8 * node + (o[:, 2] << 2) + (o[:, 1] << 1) + o[:, 0] + 1
    return ties


def test_octree_cases_reach_every_path():
    import oracle
    ns = {c.name: len(c.make()) for c in nc.OC_CASES}
    assert {1, nc.OC_BLK - 1, nc.OC_BLK, nc.OC_BLK + 1} <= set(ns.values()) and max(ns.values()) >= 300000
    assert all(t > 0 for t in _octree_splits(nc.oc_case('ties_grid').make()))
    for name, zero_axes in (('all_equal', 3), ('all_equal_capped', 3), ('flat_z', 1)):
        p = nc.oc_case(name).make()
        assert ((p.max(0) - p.min(0)) == 0).sum() == zero_axes
    assert len(nc.oc_case('all_equal_capped').make()) > nc.MAX_NEIGHBORS
    # the cap: every query lists every point (radius beyond the cloud's diagonal); the 1000th entry ends a leaf in one
    # case and falls inside a leaf in the other
    for name, on_boundary in (('cap_on_leaf_boundary', True), ('cap_inside_leaf', False)):
        c = nc.oc_case(name)
        p = c.make()
        assert c.radius > np.linalg.norm(p.max(0) - p.min(0)) and len(p) > nc.MAX_NEIGHBORS
        psl = oracle.build_octree(p)[2]
        assert (nc.MAX_NEIGHBORS in set(np.cumsum(psl[:, 1]).tolist())) == on_boundary
    for name, mean_active in nc.OC_TRUNCATION:
        c = nc.oc_case(name)
        p = c.make()
        cnt = nc.neighbour_counts(p, np.zeros(len(p), np.int32), c.radius)
        assert cnt.min() >= nc.MAX_NEIGHBORS + 100 and (len(p) * mean_active) % nc.MAX_NEIGHBORS
    for name, mean_active in nc.BQ_TRUNCATION:
        xyz, bi, bo = nc.bq_case(name).make()
        cnt = nc.neighbour_counts(xyz, bi, nc.bq_case(name).radius)
        assert cnt.min() >= nc.MAX_NEIGHBORS + 100 and (len(xyz) * mean_active) % nc.MAX_NEIGHBORS
