"""The cases tests/test_gpu_neighbour_edges.py runs for the neighbour-graph kernels -- the ball query (ballquery.cu),
the clustering (bfs_cluster.cu) and the octree ball query (octree.cu) -- next to the launch constants those cases must
reach and a CPU restatement of the ball query's routing. tests/test_neighbour_coverage.py checks on the CPU that the
table reaches every internal path, and that the constants below still match the .cu sources."""
import collections

import numpy as np

# ---- launch constants of softgroup_b200/csrc -------------------------------------------------------------------------
MAX_NEIGHBORS = 1000  # SGB_MAX_NEIGHBORS: the reference keeps the first 1000 neighbours
# ballquery.cu BqCfg<PASS>: staging area kSMax records, bitonic limit kSortMax, bitmap kBmWords words
BQ_CFG = {0: dict(threads=512, smax=5120, sort_max=4096, bm_words=4096),
          1: dict(threads=1024, smax=10240, sort_max=8192, bm_words=8192)}
BQ_CHUNK = 128  # kBqChunk: queries per work item
BQ_MAX_SEG = 1023  # kMaxSeg
BQ_CELL_BIAS = 131072  # kCellBias; a point is hashed iff |floor(x / h)| < kCellBias - 2 on every axis
BFS_EMIT2_MAX_W = 64  # bfs_emit2_kernel takes bitmap rows of W <= 64 words (lists <= 2048); longer: bfs_emit_kernel
BFS_BATCH = 12  # kBatch: label-propagation passes per host round trip
BFS_CL, BFS_CL_THREADS = 8, 512  # kCl CTAs of kClThreads threads per emit2 cluster (one scan tile = 512 parents)
OC_BLK = 512  # octree.cu OC_BLK: points per block of the leaf histogram / stable scatter

BQ_PATHS = ('p0_bitmap', 'p0_bitonic', 'p1_bitmap', 'p1_bitonic', 'exact')


def bq_smem_bytes(p):
    """Dynamic shared memory of bq_query_kernel<p>: S[kSMax] float4 records, the bitmap and the prefix words."""
    c = BQ_CFG[p]
    return 16 * c['smax'] + 6 * c['bm_words']


def bitonic_p(total_s):
    """Records the bitonic fallback pads a stencil of total_s points to."""
    P = 32
    while P < total_s:
        P <<= 1
    return P


def bq_path(total_s, nwords):
    """Path of a work item with total_s stencil points whose id range spans nwords 32-bit words (see ballquery.cu)."""
    for p in (0, 1):
        c = BQ_CFG[p]
        if nwords <= c['bm_words'] and total_s <= c['smax']:
            return 'p%d_bitmap' % p
        if nwords > c['bm_words'] and total_s <= c['sort_max']:
            return 'p%d_bitonic' % p
    return 'exact'


def bq_path_before_fix(total_s, nwords):
    """The routing before the bitonic limit: every stencil of <= kSMax points was staged, whatever its P."""
    for p in (0, 1):
        c = BQ_CFG[p]
        if total_s <= c['smax']:
            return 'p%d_%s' % (p, 'bitmap' if nwords <= c['bm_words'] else 'bitonic')
    return 'exact'


BqRouting = collections.namedtuple('BqRouting', 'cell_of cell_cnt cell_path total_s nwords item_cell item_q0')


def bq_route(xyz, batch_idxs, radius):
    """numpy restatement of bq_insert_kernel / bq_cellstart_kernel / the stencil set-up of bq_query_kernel.
    cell_of[i]: cell of point i (-1: not hashed); per cell: queries, path, stencil points and id range in words; per
    work item: its cell and first query."""
    xyz = np.asarray(xyz, np.float32)
    seg = np.asarray(batch_idxs, np.int64)
    h = float(np.float32(radius)) * (1.0 + 1e-4)
    f = np.floor(xyz.astype(np.float64) * (1.0 / h))
    lim = BQ_CELL_BIAS - 2
    with np.errstate(invalid='ignore'):
        ok = (np.abs(f) < lim).all(1) & (seg >= 0) & (seg <= BQ_MAX_SEG)
    if (~ok & np.isfinite(xyz).all(1)).any():
        raise ValueError('finite point outside the addressable cell range or segment id outside [0, 1023]')
    idx = np.nonzero(ok)[0]
    fc = (f[idx].astype(np.int64) + BQ_CELL_BIAS).astype(np.uint64)
    key = ((seg[idx].astype(np.uint64) << np.uint64(54)) | (fc[:, 0] << np.uint64(36)) | (fc[:, 1] << np.uint64(18)) |
           fc[:, 2])
    cells, inv = np.unique(key, return_inverse=True)
    cell_of = np.full(len(xyz), -1, np.int64)
    cell_of[idx] = inv
    cnt = np.bincount(inv, minlength=len(cells))
    order = np.argsort(inv, kind='stable')  # ascending point index inside each cell
    ends = np.cumsum(cnt)
    lo = idx[order][ends - cnt]
    hi = idx[order][ends - 1]
    total = np.zeros(len(cells), np.int64)
    s_lo = np.full(len(cells), np.iinfo(np.int64).max)
    s_hi = np.full(len(cells), -1)
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                nk = cells.astype(np.int64) + (dx << 36) + (dy << 18) + dz  # fields stay inside [3, 2^18 - 3]
                pos = np.minimum(np.searchsorted(cells, nk.astype(np.uint64)), len(cells) - 1)
                hit = cells[pos] == nk.astype(np.uint64)
                total += np.where(hit, cnt[pos], 0)
                s_lo = np.minimum(s_lo, np.where(hit, lo[pos], s_lo))
                s_hi = np.maximum(s_hi, np.where(hit, hi[pos], s_hi))
    nwords = (s_hi - s_lo + 32) >> 5
    path = np.array([bq_path(t, w) for t, w in zip(total, nwords)])
    nch = (cnt + BQ_CHUNK - 1) // BQ_CHUNK
    item_cell = np.repeat(np.arange(len(cells)), nch)
    item_q0 = (np.arange(nch.sum()) - np.repeat(np.cumsum(nch) - nch, nch)) * BQ_CHUNK
    return BqRouting(cell_of, cnt, path, total, nwords, item_cell, item_q0)


def neighbour_counts(xyz, batch_idxs, radius):
    """Same-segment points within `radius` of every point (float64 distances, the query point included). Close to the
    list length before the 1000 cap; the cases keep clear of the cap where it matters (see test_neighbour_coverage)."""
    from scipy.spatial import cKDTree
    xyz = np.asarray(xyz, np.float64)
    out = np.zeros(len(xyz), np.int64)
    fin = np.isfinite(xyz).all(1)
    for b in np.unique(batch_idxs):
        sel = np.nonzero((batch_idxs == b) & fin)[0]
        if len(sel):
            out[sel] = cKDTree(xyz[sel]).query_ball_point(xyz[sel], radius, return_length=True)
    return out


# ---- ball query cases ------------------------------------------------------------------------------------------------
# Every case is (xyz float32 [n,3], batch_idxs int32 [n], batch_offsets int32 [B+1]) from a seeded generator, at radius
# R = 0.04 unless the case says otherwise. Structures are laid out on the cell grid of h = R (1 + 1e-4):
#  cube(n)     : n points uniform in a cube of side 0.99 h inside one cell, so its stencil holds all n points. The ball
#                around a cube corner holds ~pi/6 of the cube: every list is capped once n >= ~2000.
#  shell(q, c) : q queries within 0.1 h of one cell's centre and, in each of the 26 neighbouring cells, a clump of c
#                points at the far side (> 1.25 h from every query). The queries' stencil holds q + 26 c points, but
#                their lists only the q queries.
R = 0.04
H = R * (1 + 1e-4)


def _uniform_ball(rng, n, rad):
    d = rng.randn(n, 3)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return d * (rad * rng.rand(n, 1) ** (1.0 / 3))


def _cube(rng, n, cell):
    """n points of a cube structure whose lowest cell is `cell` (integer triple)."""
    return (np.asarray(cell) + 0.005) * H + rng.rand(n, 3) * 0.99 * H


def _shell(rng, q, c, cell):
    """(queries, clumps) of a shell structure centred in cell `cell`."""
    centre = (np.asarray(cell) + 0.5) * H
    queries = centre + _uniform_ball(rng, q, 0.1 * H)
    far = {-1: -1.4, 0: 0.0, 1: 1.4}
    clumps = [centre + np.array([far[dx], far[dy], far[dz]]) * H + _uniform_ball(rng, c, 0.05 * H)
              for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dx, dy, dz) != (0, 0, 0)]
    return queries, np.concatenate(clumps)


def _segments(parts):
    """Concatenate per-segment point arrays into (xyz, batch_idxs, batch_offsets)."""
    lens = [len(p) for p in parts]
    xyz = np.concatenate([np.asarray(p, np.float64).reshape(-1, 3) for p in parts]).astype(np.float32)
    bo = np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)
    return xyz, np.repeat(np.arange(len(parts)), lens).astype(np.int32), bo


def _clusters(seed=0):
    """Gaussian blobs over 3 segments: ordinary stencils, nothing capped."""
    rng = np.random.RandomState(seed)
    centres = rng.rand(12, 3) * 2
    return _segments([centres[rng.randint(0, 12, n)] + rng.randn(n, 3) * 0.03 for n in (7000, 5000, 8000)])


def _cube_case(n, seed):
    rng = np.random.RandomState(seed)
    return _segments([_cube(rng, n, (10, 10, 10))])


def _shells(seed=1):
    """One segment per shell: queries of 128, 129 and 300 points (1, 2 and 3 work items) with stencils of 5121..10240
    points; 4096 < total_s <= 5120 on the bitmap; stencils beyond 10240 points."""
    rng = np.random.RandomState(seed)
    parts = []
    for q, c in ((128, 230), (129, 230), (300, 180), (100, 170), (100, 420), (300, 420)):
        a, b = _shell(rng, q, c, (5, 5, 5))
        parts.append(np.concatenate([a, b]))
    return _segments(parts)


def _segments_1023(seed=2):
    """1023 segments (the most one call takes): empty and one-point segments, and the same coordinates in many
    segments -- lists must never cross a segment."""
    rng = np.random.RandomState(seed)
    shared = rng.rand(40, 3) * 0.2  # appears in every segment b % 7 == 3
    parts = []
    for b in range(BQ_MAX_SEG):
        k = b % 7
        if k == 0:
            parts.append(np.zeros((0, 3)))
        elif k == 1:
            parts.append(rng.rand(1, 3) * 0.2)
        elif k == 3:
            parts.append(shared)
        else:
            parts.append(rng.rand(rng.randint(2, 60), 3) * 0.2)
    parts[-1] = np.zeros((0, 3))  # the last segment is empty as well
    parts[-2] = shared[:1]  # and a one-point segment that duplicates a point of other segments
    return _segments(parts)


def _cell_range_edges(seed=3):
    """Coordinates in the last addressable cells, +-131069 (|floor(x / h)| < 131070), on every axis and on both sides
    of zero, plus points around 0 itself. Radius 1 keeps the float32 spacing at 1.3e5 (2^-7) far below the radius."""
    rng = np.random.RandomState(seed)
    h = 1.0 * (1 + 1e-4)
    parts = []
    for sgn in (1, -1):
        for axis in range(3):
            p = (rng.rand(300, 3) * 1.4 + 4.3 * sgn) * h
            # the outermost valid cell and the one inside it: cells 131068..131069 resp. -131069..-131068
            p[:, axis] = (rng.rand(300) * 1.96 + (131068.02 if sgn > 0 else -131068.98)) * h
            parts.append(p)
    parts.append(rng.randn(400, 3) * 0.8)  # cells -1 / 0 on every axis
    return _segments([np.concatenate(parts)])


# The wide case: one segment of ~327k points. Every structure puts its first part (queries, or the first half of a cube)
# at the lowest indices and the rest at the highest, with FILLER sparse points in between, so every structure stencil
# spans more than 8192 bitmap words and has to be ordered by the bitonic sort -- or, where P would not fit, goes on to
# the next configuration. The (4096, 5120] and (8192, 10240] structures are the stencils whose padded sort used to
# overrun the staging area (P = 8192 records of 16 B in 106,496 B; P = 16384 in 212,992 B).
WIDE_FILLER = 280000
WIDE_STRUCTURES = (('shell', 100, 100), ('cube', 3000), ('shell', 100, 170), ('cube', 4600), ('shell', 100, 230),
                   ('cube', 7000), ('shell', 100, 350), ('cube', 9500))


def _wide_index_range(seed=4):
    rng = np.random.RandomState(seed)
    low, high = [], []
    for k, s in enumerate(WIDE_STRUCTURES):
        cell = (2000 + 10 * k, 5, 5)  # x = 80 m + 0.4 m per structure: far from the filler and from each other
        if s[0] == 'shell':
            a, b = _shell(rng, s[1], s[2], cell)
        else:
            p = _cube(rng, s[1], cell)
            a, b = p[:s[1] // 2], p[s[1] // 2:]
        low.append(a)
        high.append(b)
    filler = rng.rand(WIDE_FILLER, 3) * np.array([60.0, 60.0, 20.0])
    return _segments([np.concatenate(low + [filler] + high)])


BqCase = collections.namedtuple('BqCase', 'name radius make full_oracle')
BQ_CASES = [
    BqCase('clusters_b3', R, _clusters, True),
    BqCase('cube_p0_cap', R, lambda: _cube_case(4501, 5), True),
    BqCase('cube_p1_cap', R, lambda: _cube_case(8001, 6), True),
    BqCase('cube_exact_cap', R, lambda: _cube_case(12001, 7), True),
    BqCase('shells', R, _shells, True),
    BqCase('segments_1023', R, _segments_1023, True),
    BqCase('cell_range_edges', 1.0, _cell_range_edges, True),
    # too large for the brute-force oracle: a fixed sample of queries against the numpy restatement
    BqCase('wide_index_range', R, _wide_index_range, False),
]
# truncation at the C ABI: (case, meanActive) with every list capped at 1000, so the lists start at multiples of 1000
# and the capacity n * meanActive (n = 1 mod 1000) ends inside one
BQ_TRUNCATION = (('cube_p0_cap', 333), ('cube_p1_cap', 333), ('cube_exact_cap', 333))


def bq_case(name):
    return [c for c in BQ_CASES if c.name == name][0]


# ---- bfs_cluster cases -----------------------------------------------------------------------------------------------
# Each case is (idx int32 [nnz], start_len int32 [N,2], threshold): directed lists, compared with the sequential BFS of
# the oracle. Random lists hold duplicates and self-loops.
def _lists_to_graph(lists):
    lens = np.array([len(x) for x in lists], np.int64)
    idx = np.concatenate([np.asarray(x, np.int64) for x in lists] + [np.zeros(0, np.int64)]).astype(np.int32)
    sl = np.stack([np.cumsum(lens) - lens, lens], 1).astype(np.int32)
    return idx, sl


def _random_lists(seed, n, max_len, long_len=None, comp=50):
    """n nodes in groups of `comp` (lists stay mostly inside a group, a few edges leave it), list lengths < max_len,
    self-loops and duplicates included; node 0 of a middle group gets one list of exactly `long_len` entries."""
    rng = np.random.RandomState(seed)
    lists = []
    for u in range(n):
        g0 = (u // comp) * comp
        k = rng.randint(0, max_len)
        nb = g0 + rng.randint(0, min(comp, n - g0), k)
        nb[rng.rand(k) < 0.02] = rng.randint(0, n)  # edges into other groups
        if k > 2:
            nb[0] = u  # self-loop
            nb[1] = nb[2]  # duplicate
        lists.append(nb)
    if long_len is not None:
        u = (n // comp // 2) * comp
        nb = rng.randint(0, n, long_len)
        nb[:3] = [u, nb[5], nb[5]]
        lists[u] = nb
    return _lists_to_graph(lists)


def _wide_frontier(seed=5):
    """Node 0 lists 900 nodes (a level of 900 parents: two 512-parent scan tiles), each of which lists 3 more."""
    rng = np.random.RandomState(seed)
    n = 1 + 900 + 2700
    lists = [np.arange(1, 901)] + [901 + 3 * (u - 1) + np.arange(3) for u in range(1, 901)] + \
        [rng.randint(0, n, rng.randint(0, 3)) for _ in range(2700)]
    return _lists_to_graph(lists)


def _many_components(seed=6):
    """20,000 components of 2-5 nodes (cudaOccupancyMaxActiveClusters of the 8-CTA emit2 kernel allows at most
    132 * 4 / 8 = 66 in flight on an H100), each a directed cycle plus a duplicate entry."""
    rng = np.random.RandomState(seed)
    sizes = rng.randint(2, 6, 20000)
    lists, base = [], 0
    for s in sizes:
        for i in range(s):
            lists.append([base + (i + 1) % s, base + (i + 1) % s, base + i])
        base += s
    return _lists_to_graph(lists)


def _descending_chains(seed=7, chains=20, length=40):
    """Chains s -> s+L -> s+L-1 -> ... -> s+1: every hop lowers a node that only pushes once its own label fell, so the
    label of s needs one propagation pass per hop (pointer jumping cannot help) -- more than one batch of 12 passes."""
    lists = []
    n = chains * (length + 1)
    out = [[] for _ in range(n)]
    for c in range(chains):
        s = c * (length + 1)
        seq = [s] + list(range(s + length, s, -1))
        for a, b in zip(seq[:-1], seq[1:]):
            out[a].append(b)
    for u in range(n):
        lists.append(out[u] + [u])
    return _lists_to_graph(lists)


BfsCase = collections.namedtuple('BfsCase', 'name make thr')
BFS_CASES = [
    BfsCase('maxlen_32', lambda: _random_lists(10, 4000, 33, long_len=32), 3.0),
    BfsCase('maxlen_33', lambda: _random_lists(11, 4000, 20, long_len=33), 3.0),
    BfsCase('maxlen_2048', lambda: _random_lists(12, 6000, 12, long_len=2048), 5.0),
    BfsCase('maxlen_2049', lambda: _random_lists(13, 6000, 12, long_len=2049), 5.0),
    BfsCase('list_5000', lambda: _random_lists(14, 9000, 30, long_len=5000, comp=300), 2.0),
    BfsCase('wide_frontier', _wide_frontier, 1.0),
    BfsCase('many_components', _many_components, 1.0),
    BfsCase('descending_chains', _descending_chains, 2.0),
]


def bfs_case(name):
    return [c for c in BFS_CASES if c.name == name][0]


def bfs_levels(idx, sl):
    """Sequential BFS of bfs_cluster.cpp: (seed of every component, widest BFS level of any component)."""
    n = len(sl)
    seen = np.zeros(n, bool)
    seeds, widest = [], 0
    for i in range(n):
        if seen[i]:
            continue
        seeds.append(i)
        seen[i] = True
        level = [i]
        while level:
            widest = max(widest, len(level))
            nxt = []
            for u in level:
                for v in idx[sl[u, 0]:sl[u, 0] + sl[u, 1]]:
                    if not seen[v]:
                        seen[v] = True
                        nxt.append(int(v))
            level = nxt
    return np.array(seeds), widest


# Per-node segment thresholds (bfs_cluster_segments(node_seg, seg_thr)): components of known sizes in 6 segments,
# thresholds relative to those sizes. seg_thr[k] applies to the components whose seed lies in segment k.
THR_COMPONENT_SIZES = (1, 2, 7, 7, 30, 64, 150)


def threshold_graph(seed=8):
    """(idx, start_len, node_seg): every segment holds one component of each size in THR_COMPONENT_SIZES (a cycle plus
    random chords), in shuffled order."""
    rng = np.random.RandomState(seed)
    lists, node_seg, base = [], [], 0
    for s in range(6):
        for size in rng.permutation(THR_COMPONENT_SIZES):
            for i in range(size):
                lists.append([base + (i + 1) % size] + list(base + rng.randint(0, size, rng.randint(0, 4))))
                node_seg.append(s)
            base += size
    idx, sl = _lists_to_graph(lists)
    return idx, sl, np.array(node_seg, np.int32)


def threshold_values(n):
    """seg_thr of the 6 segments: 0, a component size exactly (7 and 30: equal is kept), half below one, one float32
    ulp above the largest component, and above every component (n + 1)."""
    above_150 = np.nextafter(np.float32(150), np.float32(np.inf))
    return np.array([0.0, 7.0, 30.0, 6.5, above_150, n + 1.0], np.float32)


# ---- octree cases ----------------------------------------------------------------------------------------------------
def _oc_uniform(n, seed, scale=(1.0, 1.0, 1.0)):
    return (np.random.RandomState(seed).rand(n, 3) * np.array(scale)).astype(np.float32)


def _oc_ties():
    """A 9^3 grid of k/8: the box centre and every split plane of the three levels (0.5, 0.25, 0.125, ...) is a grid
    value, so many points sit exactly on a split (`<` goes low, equal goes high)."""
    g = np.arange(9, dtype=np.float32) / 8
    return np.stack(np.meshgrid(g, g, g, indexing='ij'), -1).reshape(-1, 3).astype(np.float32)


def _oc_flat(seed=20):
    p = _oc_uniform(6000, seed, (2.0, 1.5, 1.0))
    p[:, 2] = 0.75  # zero z extent: every box has l = 0
    return p


def _oc_leaf_clusters(sizes, seed=21):
    """Clusters in leaves of increasing index (leaf-major order = cluster order), all within the radius of each other:
    every query lists the first 1000 points of the concatenation."""
    rng = np.random.RandomState(seed)
    corners = np.array([[0.05, 0.05, 0.05], [0.95, 0.05, 0.05], [0.05, 0.95, 0.95]])  # top-level octants 0, 1, 6
    parts = [corners[k] + rng.rand(s, 3) * 0.03 for k, s in enumerate(sizes)]
    perm = rng.permutation(sum(sizes))  # indices not in leaf order
    return np.concatenate(parts)[perm].astype(np.float32)


OcCase = collections.namedtuple('OcCase', 'name radius make')
OC_CASES = [
    OcCase('n1', 0.1, lambda: _oc_uniform(1, 30)),
    OcCase('n511', 0.15, lambda: _oc_uniform(511, 31)),
    OcCase('n512', 0.15, lambda: _oc_uniform(512, 32)),
    OcCase('n513', 0.15, lambda: _oc_uniform(513, 33)),
    OcCase('n300k', 0.03, lambda: _oc_uniform(300000, 34, (4.0, 4.0, 1.0))),
    OcCase('ties_grid', 0.2, _oc_ties),
    OcCase('all_equal', 0.1, lambda: np.tile(np.array([[1.5, -2.0, 3.0]], np.float32), (100, 1))),
    OcCase('all_equal_capped', 0.1, lambda: np.tile(np.array([[-0.25, 0.0, 7.0]], np.float32), (1300, 1))),
    OcCase('flat_z', 0.05, _oc_flat),
    OcCase('cap_on_leaf_boundary', 2.0, lambda: _oc_leaf_clusters((600, 400, 300))),
    OcCase('cap_inside_leaf', 2.0, lambda: _oc_leaf_clusters((700, 400, 300))),
    OcCase('cube_capped', 0.9, lambda: _oc_uniform(4001, 35)),
]
# truncation at the C ABI: every list of cube_capped is capped at 1000, the capacity 4001 * 333 ends inside one
OC_TRUNCATION = (('cube_capped', 333), )
DEGENERATE_OC = ('all_equal', 'all_equal_capped', 'flat_z', 'ties_grid')


def oc_case(name):
    return [c for c in OC_CASES if c.name == name][0]
