"""The cases tests/test_gpu_forward_stages.py runs the whole forward on, stage by stage against tests/forward_oracle.py.

  * one case per bench.py workload (c2, c2frag, c3, c4, c5), read from bench.WORKLOADS and built the way bench.main
    builds it: the same scan (seed 0, full size, x4 split / intensity only), the same injected point-wise predictions
    (sigma, fragments, confusion) and the same model (torch.manual_seed(0), random init);
  * c2_bn: c2 with random BatchNorm statistics and affine parameters, so that no folded scale / shift is the identity;
  * a constructed instance-branch case (`instance_case`) for the edges the workloads need not reach: more than 1000
    proposals (tiny U-Net batch items), single-point clusters and clusters flat in one or all axes (the cluster scale is
    inf, then clamped), clusters whose extent puts the scale at the clamp while their coordinates are far from the
    origin, so that voxel coordinates land just below spatial_shape, and points shared by several proposals."""
import collections
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import bench  # noqa: E402
from softgroup_b200 import synth  # noqa: E402
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402

WorkloadCase = collections.namedtuple('WorkloadCase', 'name key bn_seed')
WORKLOAD_CASES = [WorkloadCase(k, k, None) for k in sorted(bench.WORKLOADS)] + [WorkloadCase('c2_bn', 'c2', 1)]


def workload_case(name):
    return [c for c in WORKLOAD_CASES if c.name == name][0]


def randomize_bn(model, seed):
    """Every BatchNorm1d gets random running statistics and affine parameters (eval-mode scale / shift away from 1 / 0)."""
    g = torch.Generator().manual_seed(seed)
    for m in model.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            with torch.no_grad():
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g) * 0.4 + 0.8)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)


def build_workload(case, seed=0):
    """bench.main's scan, injection and model for case.key (rank 0, --seed `seed`). Returns dict(cfg, wl, scan: the host
    scan the forward gets (x4 layout for c3), base: the scan in point order, inj: (scores, offsets) numpy, model: CPU)."""
    wl = bench.WORKLOADS[case.key]
    cfg = model_cfg(wl['cfg'])
    torch.manual_seed(0)
    model = SoftGroup(**cfg).eval()
    if case.bn_seed is not None:
        randomize_bn(model, case.bn_seed)
    sc = synth.make_scan(wl['shape'], seed=seed, n_points=wl['n'])
    if wl.get('intensity_only'):
        sc['feats'] = sc['feats'][:, :1].copy()
    base = sc
    if wl.get('x4'):
        sc = synth.to_x4_split(sc)
    inj = synth.grouping_inputs(base, sigma=wl['sigma'], seed=seed, fragments=wl.get('fragments', 1),
                                confusion=wl.get('confusion', 0.0))
    return dict(cfg=cfg, wl=wl, scan=sc, base=base, inj=inj, model=model)


# ---------------------------------------------------------------------------------------------------------------------
# the constructed instance-branch case
# ---------------------------------------------------------------------------------------------------------------------
INSTANCE_CFG = 'scannet'  # instance_voxel_cfg scale 50, spatial_shape 20
N_BLOBS = 340  # three proposals per blob: the whole blob, a random half, the half below its median x
N_SINGLE, N_FLAT1, N_FLATALL, N_EDGE = 24, 12, 6, 4


def _edge_cluster(rng, x0, scale, spatial_shape):
    """Points of one cluster far from the origin whose x extent e gives the scale 1 / (e / S) - 0.01 at the clamp
    (e ~ S / (scale + 0.01)) and whose largest voxel coordinate, in float32 as the forward computes it, is in
    [S - 0.02, S): the first such e of a fixed sweep of relative steps of 1e-7 around the boundary."""
    base = np.float32(spatial_shape / (scale + 0.01))
    for j in range(400):
        e = np.float32(base * (1 + (j // 2) * 1e-7 * (1 if j % 2 else -1)))
        x = np.float32(x0) + np.concatenate([[0, e], rng.rand(30) * e]).astype(np.float32)
        xyz = np.stack([x, np.float32(x0 * 0.5) + (rng.rand(32) * 0.1).astype(np.float32),
                        (rng.rand(32) * 0.2).astype(np.float32)], 1).astype(np.float32)
        t = torch.from_numpy(xyz)
        mn, mx = t.min(0)[0], t.max(0)[0]
        inv = torch.tensor(1.0) / torch.tensor(float(spatial_shape))  # the forward's `/ spatial_shape` on the GPU
        s = torch.clamp(1 / ((mx - mn) * inv).max() - 0.01, max=scale)
        top = float((t * s - mn * s).max())
        if spatial_shape - 0.02 <= top < spatial_shape:
            return xyz
    raise AssertionError('no cluster of the sweep lands in [S - 0.02, S)')


def instance_case(seed=0):
    """Inputs of the instance branch (clusters_voxelization onwards) and the model. Returns dict(cfg, model: CPU,
    coords_float float32 [N,3], feats float32 [N,C] (the backbone output the branch gathers), proposals_idx int32
    [S,2], proposals_offset int32 [nP+1], semantic_scores float32 [N, classes], kinds: proposal ids of every edge)."""
    cfg = model_cfg(INSTANCE_CFG)
    vc = cfg['instance_voxel_cfg']
    rng = np.random.RandomState(seed)
    xyz, props, kinds = [], [], collections.defaultdict(list)
    n = [0]

    def points(p):
        ids = np.arange(n[0], n[0] + len(p))
        xyz.append(np.asarray(p, np.float32))
        n[0] += len(p)
        return ids

    def proposal(ids, kind):
        kinds[kind].append(len(props))
        props.append(np.sort(np.asarray(ids)))

    for _ in range(N_BLOBS):
        c, r = rng.uniform(0, 12, 3), rng.uniform(0.05, 0.8)
        ids = points(c + rng.randn(rng.randint(40, 400), 3) * r / 3)
        proposal(ids, 'blob')
        proposal(ids[rng.rand(ids.size) < 0.5], 'shared')
        x = xyz[-1][:, 0]
        proposal(ids[x < np.median(x)], 'shared')
    for _ in range(N_SINGLE):
        proposal(points(rng.uniform(0, 12, (1, 3))), 'single_point')
    for _ in range(N_FLAT1):
        p = rng.uniform(0, 12, 3) + rng.randn(rng.randint(20, 200), 3) * 0.1
        p[:, rng.randint(3)] = p[0, 0]
        proposal(points(p), 'flat_one_axis')
    for _ in range(N_FLATALL):
        proposal(points(np.repeat(rng.uniform(0, 12, (1, 3)), rng.randint(2, 150), 0)), 'flat_all_axes')
    for k in range(N_EDGE):
        # (beyond ~4000 the float32 rounding of coords * scale can reach spatial_shape itself, which the reference
        # asserts against, softgroup.py:699)
        proposal(points(_edge_cluster(rng, 1000.37 + 250 * k, vc['scale'], vc['spatial_shape'])), 'scale_clamp_edge')
    coords = np.concatenate(xyz).astype(np.float32)
    perm = rng.permutation(len(coords))  # proposals' points are spread over the whole index range
    inv = np.argsort(perm)
    coords = coords[perm]
    pidx = np.concatenate([np.stack([np.full(len(p), i), np.sort(inv[p])], 1) for i, p in enumerate(props)]).astype(np.int32)
    poff = np.concatenate([[0], np.cumsum([len(p) for p in props])]).astype(np.int32)
    torch.manual_seed(seed)
    model = SoftGroup(**cfg).eval()
    randomize_bn(model, seed + 1)
    g = torch.Generator().manual_seed(seed + 2)
    with torch.no_grad():  # heads whose decisions are not all alike: ~ half the mask scores below mask_score_thr
        model.mask_linear[-1].weight.copy_(torch.randn(model.mask_linear[-1].weight.shape, generator=g) * 0.3)
        model.mask_linear[-1].bias.fill_(-0.5)
        model.cls_linear.weight.copy_(torch.randn(model.cls_linear.weight.shape, generator=g) * 2.0)
        model.iou_score_linear.weight.copy_(torch.randn(model.iou_score_linear.weight.shape, generator=g) * 2.0)
    feats = (rng.randn(len(coords), cfg['channels']) * rng.uniform(0.2, 3, cfg['channels'])).astype(np.float32)
    sem = rng.randn(len(coords), cfg['semantic_classes']).astype(np.float32)
    return dict(cfg=cfg, model=model, coords_float=coords, feats=feats, proposals_idx=pidx, proposals_offset=poff,
                semantic_scores=sem, kinds=dict(kinds))
