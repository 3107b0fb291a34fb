"""The host restatement of the forward (tests/forward_oracle.py) and its cases (tests/forward_cases.py), checked before
tests/test_gpu_forward_stages.py trusts them:
  * on tests/golden/ref_forward_c1.npz (the reference's own forward_test) it reproduces every stage: voxel data,
    proposals, instance voxel data and the instances' RLE strings exactly, floats within the fixture's 2e-4;
  * the grid ball query (oracle.ballquery_batch_p_grid) returns the brute-force oracle's lists on the neighbour cases
    and on random ones (the 1000 cap, several batches, NaN / Inf points, pairs at exactly the radius);
  * the case table follows bench.WORKLOADS, and the constructed instance case reaches every edge it is there for;
  * the config cases reach the paths they are there for (lvl_fusion at pyramid levels 1 and 2, ScanNet200, level 3),
    and the lvl_fusion paths of the restatement (grouping_pp on voxel rows, get_instances through v2p_map) equal the
    dense restatements of tests/test_host_grouping.py and tests/test_host_instances.py."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, 'golden'))
import bench  # noqa: E402
import forward_cases as fc  # noqa: E402
import forward_oracle as fo  # noqa: E402
import neighbour_cases as nc  # noqa: E402
import oracle  # noqa: E402
from seeded_weights import CFG_OVERRIDES, SCAN, WEIGHT_SEED, fill_seeded, load_calibrated  # noqa: E402
from softgroup_b200 import synth  # noqa: E402
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402
from softgroup_b200.ops.functions import BALLQUERY_MAX_CAPACITY  # noqa: E402

REL = 2e-4  # the fixture's float bar (tests/test_gpu_forward_golden.py), relative to the largest golden magnitude


def _close(got, want, rel=REL):
    want = np.asarray(want, np.float64)
    return np.abs(np.asarray(got, np.float64) - want).max() <= rel * max(1e-6, np.abs(want).max())


@pytest.fixture(scope='module')
def c1():
    gold = np.load(os.path.join(HERE, 'golden', 'ref_forward_c1.npz'))
    cfg = model_cfg('scannet', **CFG_OVERRIDES)
    m = SoftGroup(**cfg).eval()
    fill_seeded(m, WEIGHT_SEED)
    load_calibrated(m, gold['calibrated'])
    sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
    return gold, cfg, sd, synth.make_scan(SCAN['shape'], seed=SCAN['seed'])


def test_voxelize_and_backbone_reproduce_reference_fixture(c1):
    gold, cfg, sd, scan = c1
    vc, v2p, p2v, vf = fo.voxelize(scan['coords'], scan['feats'], scan['coords_float'], True, 1)
    assert np.array_equal(vc, gold['voxel_coords']) and np.array_equal(v2p, gold['v2p_map'])
    assert np.array_equal(vf, gold['voxel_feats'])
    out = fo.backbone(gold['voxel_feats'], gold['voxel_coords'], gold['v2p_map'], scan['spatial_shape'], sd,
                      cfg['channels'], cfg['num_blocks'])
    assert _close(out, gold['output_feats'])
    sem, off = fo.pointwise_heads(gold['output_feats'], sd)
    assert _close(sem, gold['semantic_scores']) and _close(off, gold['pt_offsets'])


def test_grouping_reproduces_reference_fixture(c1):
    gold, cfg, sd, scan = c1
    prob = torch.from_numpy(gold['semantic_scores']).softmax(-1).numpy()  # the fixture's softmax: torch on the CPU
    n = prob.shape[0]
    pidx, poff = fo.grouping(prob, gold['pt_offsets'], np.zeros(n, np.int32), scan['coords_float'], cfg, 1)
    assert np.array_equal(pidx, gold['proposals_idx']) and np.array_equal(poff, gold['proposals_offset'])


def test_instance_branch_reproduces_reference_fixture(c1):
    gold, cfg, sd, scan = c1
    ivc = cfg['instance_voxel_cfg']
    coords, inp_map, feats, nb = fo.clusters_voxelization(gold['proposals_idx'], gold['proposals_offset'],
                                                          gold['output_feats'], scan['coords_float'], ivc['scale'],
                                                          ivc['spatial_shape'])
    assert np.array_equal(coords, gold['inst_voxel_coords']) and np.array_equal(inp_map, gold['inst_map'])
    assert np.array_equal(feats, gold['inst_voxel_feats'])
    t = fo.tiny_unet(gold['inst_voxel_feats'], gold['inst_voxel_coords'], sd, cfg['channels'], ivc['spatial_shape'])
    cls, iou, mask = fo.instance_heads(t, gold['inst_voxel_coords'], gold['inst_map'], sd, nb)
    assert _close(cls, gold['cls_scores']) and _close(iou, gold['iou_scores']) and _close(mask, gold['mask_scores'])
    r = fo.get_instances(gold['proposals_idx'], gold['semantic_scores'], gold['cls_scores'], gold['iou_scores'],
                         gold['mask_scores'], cfg)
    inst = r['instances']
    assert len(inst) == gold['inst_conf'].size > 0
    assert [x[0] for x in inst] == gold['inst_label_id'].tolist()
    assert np.allclose([x[1] for x in inst], gold['inst_conf'], rtol=1e-6, atol=0)
    assert [x[2] for x in inst] == gold['inst_rle'].tolist()


def test_rle_and_panoptic_restatements():
    """rle_from_ids equals the dense encoding (rle.py:5-19) and rle_decode inverts it; the paste loop on a case with a
    skipped (covered) instance and a stuff class."""
    from softgroup_b200.util import rle_encode
    rng = np.random.RandomState(0)
    for n in (1, 7, 500):
        for p in (0.0, 0.3, 0.9, 1.0):
            m = (rng.rand(n) < p).astype(np.int64)
            assert fo.rle_from_ids(np.flatnonzero(m), n) == rle_encode(m)['counts']
            assert np.array_equal(fo.rle_decode(rle_encode(m)['counts'], n), m)
    cfg = model_cfg('kitti')
    sem = np.array([0, 12, 12, 12, 12, 3, 15, 15])
    inst = [(2, 0.9, '2 3'), (4, 0.5, '3 2'), (5, 0.4, '7 2')]  # the second is 100 % covered by the first: skipped
    got = fo.panoptic_fusion(sem, inst, cfg)
    cls = np.array([0, 12, 12, 12, 12, 3, 15, 15])
    cls[1:4] = 2 + 10
    cls[6:8] = 5 + 10
    ids = np.array([0, 1, 1, 1, 0, 0, 2, 2])
    want = (cls | (ids << 16)).astype(np.uint32)
    want[4] = 19  # thing class without an id
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------------------------
# the grid ball query
# ---------------------------------------------------------------------------------------------------------------------
def _assert_same_lists(xyz, bi, bo, radius):
    want = oracle.ballquery_batch_p(xyz, bi, bo, radius)
    got = oracle.ballquery_batch_p_grid(xyz, bi, bo, radius)
    assert np.array_equal(got[1], want[1]) and np.array_equal(got[0], want[0])
    return want


@pytest.mark.parametrize('case', [c for c in nc.BQ_CASES if c.full_oracle], ids=lambda c: c.name)
def test_grid_ball_query_equals_brute_force_on_neighbour_cases(case):
    xyz, bi, bo = case.make()
    _assert_same_lists(xyz, bi, bo, case.radius)


def _random_case(seed):
    """Three segments (one empty) of clustered points, a dense clump capped at 1000, NaN / Inf coordinates, and pairs at
    exactly the radius along an axis and one float step inside it."""
    rng = np.random.RandomState(seed)
    r = np.float32(0.04)
    parts = []
    for n in (3000, 0, 2500):
        p = rng.rand(n, 3).astype(np.float32) * 0.6
        if n:
            p[:1500] = p[:1500] * 0.05 + 0.3  # ~1500 points within one radius: lists capped at 1000
            p[rng.randint(0, n, 20), rng.randint(0, 3, 20)] = np.float32(np.nan)
            p[rng.randint(0, n, 10), rng.randint(0, 3, 10)] = np.float32(np.inf)
            p[rng.randint(0, n, 10), rng.randint(0, 3, 10)] = -np.float32(np.inf)
            base = rng.rand(40, 3).astype(np.float32) + 2
            p[-80:-40] = base
            p[-40:] = base
            p[-40:-20, 0] += r  # exactly r apart (d2 == r*r or just off by rounding): the test decides either way
            p[-20:, 1] = np.nextafter(p[-20:, 1] + r, np.float32(0))
        parts.append(p)
    return nc._segments(parts)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_grid_ball_query_equals_brute_force_on_random_cases(seed):
    xyz, bi, bo = _random_case(seed)
    idx, sl = _assert_same_lists(xyz, bi, bo, 0.04)
    assert sl[:, 1].max() == nc.MAX_NEIGHBORS and (sl[:, 1] == 0).any()


def test_grid_ball_query_degenerate_radius_and_far_coordinates():
    rng = np.random.RandomState(5)
    xyz = (rng.rand(2000, 3) * 0.1).astype(np.float32)
    xyz[:500] += np.float32(3e7)  # far from the rest: float32 spacing 2 there, cells bounded by the extent
    bi, bo = np.zeros(2000, np.int32), np.array([0, 2000], np.int32)
    for radius in (0.0, -0.04, 0.04, 5.0, 1e30, float('nan')):
        _assert_same_lists(xyz, bi, bo, radius)


# ---------------------------------------------------------------------------------------------------------------------
# the case table
# ---------------------------------------------------------------------------------------------------------------------
def test_workload_cases_follow_bench():
    assert sorted({c.key for c in fc.WORKLOAD_CASES}) == sorted(bench.WORKLOADS)
    assert sorted(c.name for c in fc.WORKLOAD_CASES if c.bn_seed is None) == sorted(bench.WORKLOADS)
    assert any(c.bn_seed is not None for c in fc.WORKLOAD_CASES)
    w = fc.build_workload(fc.workload_case('c4'))
    wl = bench.WORKLOADS['c4']
    assert w['scan']['coords'].shape[0] == wl['n'] and w['scan']['feats'].shape[1] == 1
    assert w['cfg'] == model_cfg(wl['cfg'])
    scores, offs = synth.grouping_inputs(w['base'], sigma=wl['sigma'], seed=0)
    assert np.array_equal(w['inj'][0], scores) and np.array_equal(w['inj'][1], offs)
    torch.manual_seed(0)
    ref = SoftGroup(**model_cfg(wl['cfg'])).eval().state_dict()
    assert all(torch.equal(v, ref[k]) for k, v in w['model'].state_dict().items())


def test_config_cases_reach_their_paths():
    """The table of forward_cases.CONFIG_CASES, from the injection alone (its float32 softmax on the CPU): pp_lvlfusion
    groups every class at pyramid level 1 from voxel rows, pp_lvlfusion_l2 one class holding every thing voxel at level
    2, scannet200 at least 20 classes, c5_level3 one class of 1.25M points at level 3, s3dis_pp the whole S3DIS room as
    voxel rows with one merged class at level 2 and nine at level 1, stpls3d the 1.5M-point tile through one ball query
    whose lists hold more than 1e9 neighbours (4.95 GB, past 4 GiB of byte offset) yet fit one int32 cursor. The
    stpls3d neighbour total is counted with the grid ball query of the restatement (about a minute)."""
    for case in fc.CONFIG_CASES:
        w = fc.build_config_case(case)
        cfg, scan, counts = w['cfg'], w['scan'], w['counts']
        levels = {c: fo.get_level(n) for c, n in counts.items()}
        inst, sem = scan['instance_labels'], scan['semantic_labels']
        assert len(counts) >= case.min_classes, case.name
        assert (w['v2p'] is not None) == bool(cfg['test_cfg'].get('lvl_fusion')), case.name
        if w['v2p'] is not None:  # voxel rows, the injection their mean
            vc, v2p, _ = oracle.voxelization_idx(scan['coords'], 1, 4)
            assert np.array_equal(w['v2p'], v2p) and w['inj'][0].shape[0] == vc.shape[0] < scan['coords'].shape[0]
            thing_voxels = np.unique(v2p[inst >= 0]).size
        if case.name == 'pp_lvlfusion':
            assert set(levels.values()) == {1} and len(levels) >= 10
            assert np.unique(inst[np.isin(sem, list(counts)) & (inst >= 0)]).size >= 10
        elif case.name == 'pp_lvlfusion_l2':
            assert levels == {17: 2} and thing_voxels == 119638 and counts[17] > 100000
        elif case.name == 'scannet200':
            assert not cfg['grouping_cfg'].get('with_pyramid') and cfg['semantic_classes'] == 200
            assert cfg['instance_classes'] == 198 and np.unique(sem[inst >= 0]).size >= 20
        elif case.name == 'c5_level3':
            assert levels == {9: 3}
            assert (inst >= 0).sum() == counts[9] == 1250073
        elif case.name == 's3dis_pp':  # thing points of class 7 merged into class 5
            assert not cfg['test_cfg']['x4_split'] and cfg['sem2ins_classes'] == [0, 1]
            assert scan['coords'].shape[0] == 800000 and w['inj'][0].shape[0] == 687804 and thing_voxels == 576809
            assert 7 not in counts and counts[5] == 181026 and sum(counts.values()) == 579163
            assert levels[5] == 2 and sorted(c for c, lv in levels.items() if lv == 1) == [2, 3, 4, 6, 8, 9, 10, 11, 12]
        else:
            assert case.name == 'stpls3d' and not cfg['grouping_cfg'].get('with_pyramid') and case.relabel is None
            assert scan['coords'].shape[0] == 1500000 and len(counts) == 14
            n_sel = sum(counts.values())
            assert n_sel == 1250088 and n_sel * 1000 <= BALLQUERY_MAX_CAPACITY
            prob = torch.from_numpy(w['inj'][0]).softmax(-1).numpy()
            g = cfg['grouping_cfg']
            total = 0
            for c in counts:
                obj = np.flatnonzero(prob[:, c] > np.float32(g['score_thr']))
                xyz = (scan['coords_float'][obj] + w['inj'][1][obj]).astype(np.float32)
                total += oracle.ballquery_total_grid(xyz, np.zeros(obj.size, np.int32), np.array([0, obj.size], np.int32),
                                                     g['radius'])
            assert total == 1237543570 and total * 4 > 4 << 30


@pytest.mark.parametrize('lvl_fusion', [False, True])
def test_grouping_pp_equals_dense_reference_loop(monkeypatch, lvl_fusion):
    """grouping_pp against test_host_grouping's restatement with the dense [nCluster, n] inverse map, on a small scan
    with classes at pyramid levels 1 and 2 (get_level scaled down on both sides). Under lvl_fusion both are fed voxel
    rows: the scan's voxel-mean coordinates and the injection averaged per voxel."""
    import test_host_grouping as thg
    cfg = model_cfg('scannet++', channels=16, num_blocks=2, test_cfg=dict(min_npoint=30))
    cfg['grouping_cfg'].update(class_numpoint_mean=[-1.] * 20, npoint_thr=10)  # components of >= 10 rows
    model = SoftGroup(**cfg).eval()
    sc = synth.make_scan('c2_scannet', seed=5, n_points=20000)
    scores, offs = synth.grouping_inputs(sc, sigma=0.03, seed=5)
    coords = sc['coords_float']
    if lvl_fusion:
        vc, v2p, p2v = oracle.voxelization_idx(sc['coords'], 1, 4)
        scores, offs = (fc.voxel_mean(a, v2p, vc.shape[0]) for a in (scores, offs))
        coords = oracle.voxelization(coords, p2v, 4)
    prob = torch.from_numpy(scores).softmax(-1).numpy()
    split = np.median(list(fc.class_counts(prob, cfg).values()))  # the larger classes at level 2
    get_level = lambda n: 2 if n > split else 1  # noqa: E731
    monkeypatch.setattr(fo, 'get_level', get_level)
    model.get_level = get_level
    bidx = np.zeros(scores.shape[0], np.int32)
    want_idx, want_off = thg.reference_forward_grouping_pp(model, scores, offs, bidx, coords, lvl_fusion)
    info = {}
    got_idx, got_off = fo.grouping_pp(prob, offs, coords, cfg, lvl_fusion=lvl_fusion, info=info)
    assert set(info['levels'].values()) == {1, 2} and want_off.size > 10
    assert len(info['classes']) == got_off.size - 1 and info['classes'] == sorted(info['classes'])
    assert np.array_equal(got_idx, want_idx) and np.array_equal(got_off, want_off)


@pytest.mark.parametrize('name,seed', [('scannet', 3), ('s3dis', 4)])
def test_get_instances_v2p_equals_dense_procedure(name, seed):
    """get_instances(v2p_map=...) against test_host_instances' dense procedure under lvl_fusion: (proposal, voxel)
    entries, masks taken to points, min_npoint counted in points (at a min_npoint where counting voxels would keep fewer
    instances), sem2ins classes (s3dis) from the per-point semantic prediction."""
    import test_host_instances as thi
    thr = dict(min_npoint=40, cls_score_thr=0.02, mask_score_thr=-0.5)
    cfg = model_cfg(name, test_cfg=thr)
    nI, sem2ins = cfg['instance_classes'], cfg['sem2ins_classes']
    n_vox, n_pts = 300, 1000
    rng = np.random.RandomState(100 + seed)
    v2p = rng.randint(0, n_vox, n_pts).astype(np.int32)  # some voxels hold several points, some none
    pidx, sem, cls, iou, msk = thi._case(seed, n_vox, 12, cfg['semantic_classes'], nI)
    want = thi.reference_get_instances('s', pidx, sem, cls, iou, msk, nI, sem2ins, thr['cls_score_thr'],
                                       thr['mask_score_thr'], thr['min_npoint'], v2p_map=v2p.astype(np.int64),
                                       lvl_fusion=True)
    r = fo.get_instances(pidx, sem, cls, iou, msk, cfg, v2p_map=v2p)
    got = r['instances']
    assert len(got) == len(want) > len(sem2ins)
    assert [x[0] for x in got] == [int(x['label_id']) for x in want]
    assert [x[2] for x in got] == [x['pred_mask']['counts'] for x in want]
    assert all(x['pred_mask']['length'] == n_pts for x in want)
    conf_w = np.array([x['conf'] for x in want], np.float64)
    assert np.all(np.abs(np.array([x[1] for x in got]) - conf_w) <= 1e-6 * np.abs(conf_w))
    assert np.array_equal(r['semantic_preds'], sem.argmax(1)[v2p])
    on = msk[:, :nI] > np.float32(thr['mask_score_thr'])
    voxels = np.stack([np.bincount(pidx[:, 0], weights=on[:, i], minlength=cls.shape[0]) for i in range(nI)], 1)
    cls_ok = fo.softmax64(cls)[:, :nI] > thr['cls_score_thr']
    assert np.any(r['keep'] & (voxels < thr['min_npoint']))  # kept only because points are counted
    assert np.array_equal(r['keep'], cls_ok & (r['npoint'] >= thr['min_npoint']) & ~np.isin(np.arange(nI), sem2ins))


def test_instance_case_reaches_its_edges():
    c = fc.instance_case()
    cfg, pidx, poff = c['cfg'], c['proposals_idx'], c['proposals_offset']
    ivc = cfg['instance_voxel_cfg']
    S, scale = ivc['spatial_shape'], ivc['scale']
    nP = len(poff) - 1
    assert nP >= 1000 and np.array_equal(np.diff(poff), np.bincount(pidx[:, 0], minlength=nP))
    pts = c['coords_float'][pidx[:, 1]]
    ext = oracle.sec_max(pts, poff) - oracle.sec_min(pts, poff)
    k = c['kinds']
    assert np.all(np.diff(poff)[k['single_point']] == 1)
    assert np.all(ext[k['flat_all_axes']] == 0) and np.all(np.diff(poff)[k['flat_all_axes']] > 1)
    assert np.all((ext[k['flat_one_axis']] == 0).sum(1) == 1)
    with np.errstate(divide='ignore'):
        raw = 1 / (ext / np.float32(S)).max(1).astype(np.float32) - np.float32(0.01)
    assert np.all(np.isinf(raw[k['single_point'] + k['flat_all_axes']]))
    assert np.all(np.abs(raw[k['scale_clamp_edge']] - scale) < 0.05)
    assert np.all(np.abs(pts[np.isin(pidx[:, 0], k['scale_clamp_edge'])]).max() > 1000)
    coords, inp_map, feats, nb = fo.clusters_voxelization(pidx, poff, c['feats'], c['coords_float'], scale, S)
    assert nb == nP and coords[:, 1:].max() == S - 1 and coords[:, 1:].min() == 0
    edge_rows = np.isin(coords[:, 0], k['scale_clamp_edge'])
    assert coords[edge_rows, 1].max() == S - 1
    shared = np.bincount(pidx[:, 1])
    assert shared.max() >= 3
