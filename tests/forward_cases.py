"""The cases tests/test_gpu_forward_stages.py runs the whole forward on, stage by stage against tests/forward_oracle.py.

  * one case per bench.py workload (c2, c2frag, c3, c4, c5), read from bench.WORKLOADS and built the way bench.main
    builds it: the same scan (seed 0, full size, x4 split / intensity only), the same injected point-wise predictions
    (sigma, fragments, confusion) and the same model (torch.manual_seed(0), random init);
  * c2_bn: c2 with random BatchNorm statistics and affine parameters, so that no folded scale / shift is the identity;
  * a constructed instance-branch case (`instance_case`) for the edges the workloads need not reach: more than 1000
    proposals (tiny U-Net batch items), single-point clusters and clusters flat in one or all axes (the cluster scale is
    inf, then clamped), clusters whose extent puts the scale at the clamp while their coordinates are far from the
    origin, so that voxel coordinates land just below spatial_shape, and points shared by several proposals;
  * the config cases (`CONFIG_CASES`, tests/test_gpu_forward_stages_configs.py) for the paths no bench workload takes:
    lvl_fusion (scannet++) with every class at pyramid level 1 and with one class at level 2 from voxel rows, ScanNet200,
    pyramid level 3 (c5 with every thing point in one class), SoftGroup++ S3DIS (lvl_fusion with sem2ins classes on the
    whole 800k-point room, one merged class at level 2) and the plain SoftGroup STPLS3D config (the c5 tile through a
    one-pass ball query of 1.24e9 neighbours). On one H100 the two last took 1.14 s and 0.59 s of GPU forward and
    192 s and 134 s of CPU oracle."""
import collections
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
import forward_oracle as fo  # noqa: E402
import oracle  # noqa: E402
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
# the config cases
# ---------------------------------------------------------------------------------------------------------------------
# n_points: the scan's size (shape at seed 0), or None for the c5 workload's scan, injection parameters and weights.
# relabel: every thing point (instance label >= 0) carries this semantic class when the injection is drawn, so that one
# class holds all of them (its instances stay apart: their offsets still point to their own centroids); a pair (a, b):
# the thing points of class a carry class b, so b holds the things of both. level: the pyramid level that class must
# take (every other class at level 1), or 1 for every class at level 1; None without a pyramid. min_classes: the
# classes with proposals, at least. from_grouping: the backbone is not checked (the c5 workload case checks it on the
# same scan and weights).
ConfigCase = collections.namedtuple('ConfigCase', 'name cfg shape n_points relabel level min_classes from_grouping')
CONFIG_CASES = [ConfigCase('pp_lvlfusion', 'scannet++', 'c2_scannet', 150000, None, 1, 1, False),
                ConfigCase('pp_lvlfusion_l2', 'scannet++', 'c2_scannet', 150000, 17, 2, 1, False),
                ConfigCase('scannet200', 'scannet200', 'c6_scannet200', 150000, None, None, 20, False),
                ConfigCase('c5_level3', 'stpls3d++', 'c5_stpls3d', None, 9, 3, 1, True),
                ConfigCase('s3dis_pp', 's3dis++', 'c3_s3dis', 800000, (7, 5), 2, 9, False),
                ConfigCase('stpls3d', 'stpls3d', 'c5_stpls3d', None, None, None, 10, True)]


def config_case(name):
    return [c for c in CONFIG_CASES if c.name == name][0]


def relabel_target(case):
    """The class that holds the relabelled thing points, or None."""
    return case.relabel[1] if isinstance(case.relabel, tuple) else case.relabel


def _relabelled(scan, relabel):
    sc = dict(scan)
    sem = scan['semantic_labels'].copy()
    if isinstance(relabel, tuple):
        sem[(scan['instance_labels'] >= 0) & (sem == relabel[0])] = relabel[1]
    else:
        sem[scan['instance_labels'] >= 0] = relabel
    sc['semantic_labels'] = sem
    return sc


def voxel_mean(a, v2p, num_voxels):
    """The mean of every voxel's rows of a, summed in float64, as float32."""
    v2p = np.asarray(v2p, np.int64)
    cnt = np.bincount(v2p, minlength=num_voxels).astype(np.float64)
    s = np.stack([np.bincount(v2p, weights=np.asarray(a, np.float64)[:, j], minlength=num_voxels)
                  for j in range(a.shape[1])], 1)
    return (s / cnt[:, None]).astype(np.float32)


def class_counts(prob, cfg):
    """Rows above score_thr of every class the grouping takes (not ignored, at least min_npoint rows)."""
    g = cfg['grouping_cfg']
    n = (np.asarray(prob) > np.float32(g['score_thr'])).sum(0)
    return {c: int(n[c]) for c in range(cfg['semantic_classes'])
            if c not in g['ignore_classes'] and n[c] >= cfg['test_cfg']['min_npoint']}


def build_config_case(case, seed=0):
    """Scan, injected point-wise predictions and model of a config case. Returns dict(cfg, scan: the host scan the
    forward gets, model: CPU, inj: (scores, offsets) numpy on the rows the grouping takes, voxel rows under lvl_fusion,
    v2p: the scan's v2p_map under lvl_fusion else None, counts: class_counts of the injection's float32 softmax).
    Under lvl_fusion the heads' outputs are replaced by the injection averaged per voxel (the synthetic predictions
    are per point); c5_level3 and stpls3d use the c5 workload's scan and injection parameters, and its weights."""
    if case.n_points is None:
        w = build_workload(workload_case('c5'), seed=seed)
        cfg, scan, model, wl = w['cfg'], w['scan'], w['model'], w['wl']
        if case.cfg != 'stpls3d++':  # the same module tree, hence the same weights: the c5 case checks its backbone
            cfg = model_cfg(case.cfg)
            torch.manual_seed(0)
            model = SoftGroup(**cfg).eval()
            sd, sd5 = model.state_dict(), w['model'].state_dict()
            assert list(sd) == list(sd5) and all(torch.equal(v, sd5[k]) for k, v in sd.items()), case.name
        src = w['base'] if case.relabel is None else _relabelled(w['base'], case.relabel)
        inj = synth.grouping_inputs(src, sigma=wl['sigma'], seed=seed)
    else:
        cfg = model_cfg(case.cfg)
        torch.manual_seed(0)
        model = SoftGroup(**cfg).eval()
        scan = synth.make_scan(case.shape, seed=seed, n_points=case.n_points)
        src = scan if case.relabel is None else _relabelled(scan, case.relabel)
        inj = synth.grouping_inputs(src, sigma=0.03, seed=seed)
    v2p = None
    if cfg['test_cfg'].get('lvl_fusion'):
        vc, v2p, _ = oracle.voxelization_idx(scan['coords'], 1, 4)
        inj = tuple(voxel_mean(a, v2p, vc.shape[0]) for a in inj)
    prob = torch.from_numpy(inj[0]).softmax(-1).numpy()
    return dict(cfg=cfg, scan=scan, model=model, inj=inj, v2p=v2p, counts=class_counts(prob, cfg))


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
