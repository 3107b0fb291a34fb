"""Synthetic scans shaped like the reference's datasets (no dataset files exist offline).

Follows SURVEY.md section 8(d): float32 xyz in metres centred by the mean
(dataset/scannetv2/prepare_data_inst.py:55), rgb in [-1,1] (:56), then the reference test
transform: rotate 0.35*pi about z, * scale, - min, .long() (softgroup/data/custom.py:103-107,
162-166, 180) and the collate layout of custom.py:191-256 (coords int64 [N,4] with the batch
index in column 0, coords_float f32 [N,3], feats f32 [N,3], labels, spatial_shape).

numpy only; no CUDA, no oracle.
"""
import math

import numpy as np

# name -> (n_points, room size m, n_objects, semantic classes, stuff classes, voxel scale)
SHAPES = {
    'c1_plumbing': dict(n=2000, room=(2.0, 2.0, 1.0), n_obj=4, sem=20, stuff=(0, 1), scale=50, walls=False),
    'c2_scannet': dict(n=150000, room=(7.0, 5.0, 2.6), n_obj=40, sem=20, stuff=(0, 1), scale=50, walls=True),
    'c3_s3dis': dict(n=800000, room=(15.0, 12.0, 3.0), n_obj=120, sem=13, stuff=(0, 1), scale=50, walls=True),
    'c4_kitti': dict(n=120000, room=(60.0, 60.0, 3.0), n_obj=30, sem=19, stuff=tuple(range(0, 11)), scale=20,
                     walls=False),
    'c5_stpls3d': dict(n=1500000, room=(250.0, 250.0, 30.0), n_obj=400, sem=15, stuff=(0, ), scale=3, walls=False),
    # ScanNet200-shape: a larger room with one object of every one of the 198 grouped classes (spread: object k has thing
    # class k instead of a random one)
    'c6_scannet200': dict(n=150000, room=(16.0, 14.0, 3.0), n_obj=198, sem=200, stuff=(0, 1), scale=50, walls=True,
                          spread=True),
}


def _box_faces(lo, hi, with_bottom=False):
    """Faces of an axis-aligned box as (origin, edge_u, edge_v) triples."""
    lo = np.asarray(lo, np.float64)
    hi = np.asarray(hi, np.float64)
    d = hi - lo
    faces = []
    for ax in range(3):
        u, v = [a for a in range(3) if a != ax]
        for side in (0, 1):
            if ax == 2 and side == 0 and not with_bottom:
                continue
            o = lo.copy()
            if side:
                o[ax] = hi[ax]
            eu = np.zeros(3)
            ev = np.zeros(3)
            eu[u] = d[u]
            ev[v] = d[v]
            faces.append((o, eu, ev))
    return faces


def make_scan(shape='c2_scannet', seed=0, n_points=None, batch_id=0):
    """One synthetic scan. Returns a dict of numpy arrays in the reference collate layout (one item)."""
    cfg = dict(SHAPES[shape])
    if n_points is not None:
        cfg['n'] = int(n_points)
    rng = np.random.RandomState(seed)
    n = cfg['n']
    rx, ry, rz = cfg['room']
    thing_classes = [c for c in range(cfg['sem']) if c not in cfg['stuff']]

    surfaces = []  # (origin, eu, ev, sem, inst)
    surfaces.append((np.zeros(3), np.array([rx, 0, 0.]), np.array([0, ry, 0.]), cfg['stuff'][-1], -100))  # floor
    if cfg['walls']:
        w = cfg['stuff'][0]
        surfaces.append((np.zeros(3), np.array([rx, 0, 0.]), np.array([0, 0, rz]), w, -100))
        surfaces.append((np.array([0, ry, 0.]), np.array([rx, 0, 0.]), np.array([0, 0, rz]), w, -100))
        surfaces.append((np.zeros(3), np.array([0, ry, 0.]), np.array([0, 0, rz]), w, -100))
        surfaces.append((np.array([rx, 0, 0.]), np.array([0, ry, 0.]), np.array([0, 0, rz]), w, -100))
    smax = min(1.8, 0.45 * min(rx, ry)) if rx < 100 else 12.0
    smin = 0.3 if rx < 100 else 3.0
    for k in range(cfg['n_obj']):
        size = rng.uniform(smin, smax, 3)
        size[2] = min(size[2], 0.9 * rz)
        lo = np.array([rng.uniform(0, rx - size[0]), rng.uniform(0, ry - size[1]), 0.0])
        cls = thing_classes[k % len(thing_classes)] if cfg.get('spread') else thing_classes[rng.randint(len(thing_classes))]
        for (o, eu, ev) in _box_faces(lo, lo + size):
            surfaces.append((o, eu, ev, cls, k))

    areas = np.array([np.linalg.norm(np.cross(s[1], s[2])) for s in surfaces])
    # keep floor/walls from swallowing the budget so that objects carry a realistic share of points
    weight = areas.copy()
    n_stuff = 5 if cfg['walls'] else 1
    weight[:n_stuff] *= 0.35
    counts = np.floor(weight / weight.sum() * n).astype(np.int64)
    counts[0] += n - counts.sum()
    xyz = np.empty((n, 3), np.float64)
    sem = np.empty(n, np.int64)
    inst = np.empty(n, np.int64)
    pos = 0
    for (o, eu, ev, c, k), m in zip(surfaces, counts):
        uv = rng.rand(m, 2)
        strips = max(1, int(np.sqrt(m) / 4))
        uv = uv[np.lexsort((uv[:, 1], np.floor(uv[:, 0] * strips)))]
        xyz[pos:pos + m] = o + uv[:, :1] * eu + uv[:, 1:] * ev
        sem[pos:pos + m] = c
        inst[pos:pos + m] = k
        pos += m
    xyz += rng.randn(n, 3) * 0.003
    # Point order: ScanNet vertex order is spatially coherent (mesh chunks) but not grouped by object. Emulate it:
    # every surface is rastered in strips, then the cloud is cut into blocks of 64 consecutive points and the
    # blocks are shuffled.
    blk = 64
    nb = (n + blk - 1) // blk
    perm = np.concatenate([np.arange(b * blk, min((b + 1) * blk, n)) for b in rng.permutation(nb)])
    xyz, sem, inst = xyz[perm], sem[perm], inst[perm]

    palette = rng.uniform(-0.8, 0.8, (cfg['sem'], 3))
    rgb = np.clip(palette[sem] + rng.randn(n, 3) * 0.1, -1, 1).astype(np.float32)
    xyz = (xyz - xyz.mean(0)).astype(np.float32)

    # reference test transform (custom.py:103-107 with aug off, :162-166)
    theta = 0.35 * math.pi
    m = np.eye(3)
    m = np.matmul(m, [[math.cos(theta), math.sin(theta), 0], [-math.sin(theta), math.cos(theta), 0], [0, 0, 1]])
    xyz_middle = np.matmul(xyz, m)  # float64, like the reference (numpy promotes)
    xyz_scaled = xyz_middle * cfg['scale']
    xyz_scaled -= xyz_scaled.min(0)
    coord = xyz_scaled.astype(np.int64)  # torch.from_numpy(xyz).long() truncates toward zero (values >= 0)
    coords_float = xyz_middle.astype(np.float32)

    # instance info (custom.py:61-84): centroid offsets, per-instance point counts and classes
    inst_ids = np.unique(inst[inst >= 0])
    remap = -100 * np.ones(int(inst.max()) + 2, np.int64)
    remap[inst_ids] = np.arange(len(inst_ids))
    inst = np.where(inst >= 0, remap[np.clip(inst, 0, None)], -100)
    pt_offset = np.zeros((n, 3), np.float32)
    pointnum, cls = [], []
    centroids = np.zeros((len(inst_ids), 3), np.float32)
    for k in range(len(inst_ids)):
        sel = inst == k
        centroids[k] = coords_float[sel].mean(0)
        pt_offset[sel] = centroids[k] - coords_float[sel]
        pointnum.append(int(sel.sum()))
        cls.append(int(sem[np.argmax(sel)]))

    coords = np.concatenate([np.full((n, 1), batch_id, np.int64), coord], 1)
    spatial_shape = np.clip(coord.max(0) + 1, 128, None)
    return dict(
        scan_ids=['synth_%s_seed%d' % (shape, seed)],
        coords=coords,
        batch_idxs=coords[:, 0].astype(np.int32),
        coords_float=coords_float,
        feats=rgb,
        semantic_labels=sem,
        instance_labels=inst,
        instance_pointnum=np.asarray(pointnum, np.int32),
        instance_cls=np.asarray(cls, np.int64),
        pt_offset_labels=pt_offset,
        spatial_shape=spatial_shape,
        batch_size=1,
        n_semantic=cfg['sem'],
        stuff=cfg['stuff'],
        scale=cfg['scale'],
    )


def grouping_inputs(scan, sigma=0.03, seed=0, logit=8.0, fragments=1, confusion=0.0):
    """Stage inputs for forward_grouping (SURVEY.md 8(d) fallback): semantic scores = one-hot*logit + N(0,1),
    pt_offsets = (centroid - xyz) + N(0, sigma).

    fragments > 1 / confusion > 0 give the load of a REAL checkpoint on a real scan (hundreds of proposals with
    fragments, not one clean proposal per object): every object is cut into up to `fragments` spatial parts (k-means-like
    split along its longest axes) whose points shift to the PART's centroid, and a share `confusion` of the instance points
    carries a second plausible class (logit - 1 instead of noise), so the same points are clustered under two classes."""
    rng = np.random.RandomState(seed + 1000)
    n = scan['coords_float'].shape[0]
    scores = rng.randn(n, scan['n_semantic']).astype(np.float32)
    scores[np.arange(n), scan['semantic_labels']] += logit
    target = scan['pt_offset_labels'].astype(np.float32).copy()
    inst = scan['instance_labels']
    if fragments > 1:
        xyz = scan['coords_float']
        order = np.argsort(inst, kind='stable')
        bounds = np.flatnonzero(np.diff(inst[order])) + 1
        for seg in np.split(order, bounds):
            if inst[seg[0]] < 0 or seg.size < 200:
                continue
            k = int(rng.randint(2, fragments + 1))
            p = xyz[seg]
            axis = int(np.argmax(p.max(0) - p.min(0)))
            cuts = np.quantile(p[:, axis], np.sort(rng.uniform(0.1, 0.9, k - 1)))
            part = np.searchsorted(cuts, p[:, axis])
            for q in range(k):
                sel = seg[part == q]
                if sel.size:
                    target[sel] = xyz[sel].mean(0) - xyz[sel]
    if confusion > 0:
        cand = np.flatnonzero(inst >= 0)
        pick = cand[rng.rand(cand.size) < confusion]
        alt = rng.randint(2, scan['n_semantic'], pick.size)
        scores[pick, alt] += logit - 1.0
    off = target + (rng.randn(n, 3) * sigma).astype(np.float32)
    off[inst < 0] = 0
    return scores, off.astype(np.float32)


def to_x4_split(scan):
    """S3DIS test-time layout (softgroup/data/s3dis.py:46-115): the cloud is cut into 4 interleaved pieces
    (inds[k::4]) that go through the backbone one after another; per-point arrays are stored piece after piece,
    coords carry the piece id in column 0 (each piece shifted to its own origin), batch_idxs stay 0, batch_size 4."""
    n = scan['coords'].shape[0]
    pieces = [np.arange(n)[k::4] for k in range(4)]
    order = np.concatenate(pieces)
    out = dict(scan)
    for k in ('coords_float', 'feats', 'semantic_labels', 'instance_labels', 'pt_offset_labels'):
        out[k] = scan[k][order]
    coords = []
    for b, piece in enumerate(pieces):
        xyz = scan['coords_float'][piece].astype(np.float64) * scan['scale']
        xyz -= xyz.min(0)
        coords.append(np.concatenate([np.full((len(piece), 1), b, np.int64), xyz.astype(np.int64)], 1))
    out['coords'] = np.concatenate(coords, 0)
    out['batch_idxs'] = np.zeros(n, np.int32)
    out['spatial_shape'] = np.clip(out['coords'][:, 1:].max(0) + 1, 128, None)
    out['batch_size'] = 4
    out['x4_order'] = order
    return out
