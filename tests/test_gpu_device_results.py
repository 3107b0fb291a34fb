"""forward_test(device_results=True): the scan's results as CUDA tensors -- point-wise predictions, instances as point-id
lists, panoptic labels -- against the host results of the same forward.

  * ops: bitmap rows -> ascending point ids and class bitmaps against numpy, over more than 65,535 rows, 1.5M points,
    N a multiple of 32 and not, one word per row, empty and full rows, and set bits at N and beyond (ignored); launch
    counts through sgb_launch_count;
  * whole forward, as a user calls it (harness.run_scan), once with host results and once with device_results, on every
    bench workload (c2, c2frag, c3 x4 + sem2ins, c4 panoptic, c5 SoftGroup++), scannet++ (lvl_fusion) and scannet200:
    instance k's label and confidence bit for bit, its point ids equal to its decoded RLE mask, point-wise predictions
    and panoptic labels exactly;
  * edges: no proposals, proposals without a kept instance, a sem2ins class without points, instances covering every point;
  * host reads: one more synchronisation than the device_only forward, two under 'panoptic';
  * several scans in flight (harness.ScanPipeline) equal sequential calls."""
import os
import sys
import warnings

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import forward_cases as fc  # noqa: E402
from softgroup_b200 import harness, synth  # noqa: E402
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402
from softgroup_b200.ops import _lib  # noqa: E402
from softgroup_b200.ops import instances as inst_ops  # noqa: E402
from softgroup_b200.util import rle_decode  # noqa: E402

pytestmark = pytest.mark.gpu
ALL_TASKS = ['semantic', 'instance', 'panoptic']
SKIP_IOU = 0.5  # panoptic_skip_iou of the one reference config with a panoptic task (kitti), for the configs without one


# ---------------------------------------------------------------------------------------------------------------------
# ops
# ---------------------------------------------------------------------------------------------------------------------
def _scan_launches(n):
    """Launches of the library's device-wide exclusive scan over n > 0 elements (tiles of 512 x 8)."""
    nb = -(-n // 4096)
    return 1 if nb == 1 else 2 + _scan_launches(nb)


def _random_bitmaps(rng, n_rows, n_points):
    """Rows of mixed density (empty, full, sparse, dense) with random bits also at N and beyond."""
    W = inst_ops.bitmap_words(n_points)
    dens = rng.choice([0.0, 1.0, 0.002, 0.05, 0.5], size=n_rows)
    dens[:2] = [0.0, 1.0][:n_rows]
    bits = rng.rand(n_rows, W * 32) < dens[:, None]
    words = np.packbits(bits.reshape(n_rows, W, 32)[:, :, ::-1], axis=2).view('>u4').reshape(n_rows, W)
    return words.astype(np.uint32).view(np.int32), bits[:, :n_points]


@pytest.mark.parametrize('n_rows,n_points', [(70000, 31), (66000, 64), (3, 1500000), (40, 32 * 4096), (17, 4096 + 17),
                                             (1, 1), (0, 100)])
def test_bitmap_point_ids_vs_numpy(n_rows, n_points):
    rng = np.random.RandomState(n_rows + n_points)
    words, bits = _random_bitmaps(rng, n_rows, n_points)
    bm = torch.from_numpy(words).cuda()
    L = _lib.lib()
    before = L.sgb_launch_count()
    off, ids = inst_ops.bitmap_point_ids(bm, n_points)
    torch.cuda.synchronize()
    n_seg = n_rows * -(-inst_ops.bitmap_words(n_points) // 1024)
    assert L.sgb_launch_count() - before == (3 + _scan_launches(n_seg) if n_rows else 0)
    assert off.dtype == torch.int64 and ids.dtype == torch.int32
    off, ids = off.cpu().numpy(), ids.cpu().numpy()
    counts = bits.sum(1)
    assert np.array_equal(off, np.concatenate([[0], np.cumsum(counts)]))
    rows, cols = np.nonzero(bits)  # row-major: ascending ids inside each row
    assert np.array_equal(ids, cols.astype(np.int32))
    # the caller-sized form (no read between the passes) gives the same ids
    off2, ids2 = inst_ops.bitmap_point_ids(bm, n_points, total=int(counts.sum()))
    assert np.array_equal(off2.cpu().numpy(), off) and np.array_equal(ids2.cpu().numpy(), ids)


@pytest.mark.parametrize('n_points,classes', [(1500000, [3, 0, 17]), (64, [1]), (33, [2, 5]), (4096, list(range(40))),
                                              (100, [])])
def test_class_bitmaps_vs_numpy(n_points, classes):
    rng = np.random.RandomState(n_points)
    labels = rng.randint(-2, 22, size=n_points).astype(np.int64)
    L = _lib.lib()
    before = L.sgb_launch_count()
    bm, cnt = inst_ops.class_bitmaps(torch.from_numpy(labels).cuda(), classes, n_points)
    torch.cuda.synchronize()
    assert L.sgb_launch_count() - before == (1 if classes else 0)
    W = inst_ops.bitmap_words(n_points)
    assert bm.shape == (len(classes), W)
    got = np.unpackbits(bm.cpu().numpy().view(np.uint32).astype('>u4').view(np.uint8).reshape(len(classes), W, 4), axis=2,
                        bitorder='big').reshape(len(classes), W, 32)[:, :, ::-1].reshape(len(classes), W * 32)
    for k, c in enumerate(classes):
        want = np.zeros(W * 32, bool)
        want[:n_points] = labels == c
        assert np.array_equal(got[k].astype(bool), want), c
    assert np.array_equal(cnt.cpu().numpy(), [(labels == c).sum() for c in classes])


# ---------------------------------------------------------------------------------------------------------------------
# whole forward
# ---------------------------------------------------------------------------------------------------------------------
def _rle_ids(rle):
    """np.flatnonzero(rle_decode(rle)) without the dense mask."""
    s = np.asarray(rle['counts'].split(), dtype=np.int64)
    starts, nums = s[0::2] - 1, s[1::2]
    return (np.arange(nums.sum()) + np.repeat(starts - (np.cumsum(nums) - nums), nums)).astype(np.int32)


def _run_both(model, hb, inj=None, host_tasks=None):
    """The host-results forward (eval_tasks = host_tasks) and the device_results forward (every task) of the same inputs."""
    tc = model.test_cfg
    tc.setdefault('panoptic_skip_iou', SKIP_IOU)
    keep = tc['eval_tasks']
    try:
        tc['eval_tasks'] = host_tasks or ALL_TASKS
        with torch.no_grad():
            host = harness.run_scan(model, hb, inject_pointwise=inj)
        tc['eval_tasks'] = ALL_TASKS
        with torch.no_grad():
            dev = harness.run_scan(model, hb, inject_pointwise=inj, device_results=True)
        torch.cuda.synchronize()
    finally:
        tc['eval_tasks'] = keep
    return host, dev


def _same(model, host, dev, n_points, min_instances=1):
    assert set(dev) == {'scan_id', 'semantic_preds', 'offset_preds', 'instances', 'panoptic_preds'}
    assert dev['scan_id'] == host['scan_id']
    inst = dev['instances']
    for k, dt in (('label_id', torch.int32), ('conf', torch.float32), ('point_offsets', torch.int64), ('point_ids', torch.int32)):
        assert inst[k].is_cuda and inst[k].dtype == dt, k
    label, conf, off, ids = (inst[k].cpu().numpy() for k in ('label_id', 'conf', 'point_offsets', 'point_ids'))
    pred = host['pred_instances']
    assert len(pred) == label.size >= min_instances
    assert off.size == label.size + 1 and off[0] == 0 and off[-1] == ids.size and np.all(np.diff(off) >= 0)
    for k, x in enumerate(pred):
        assert int(x['label_id']) == int(label[k]), k
        assert np.float32(x['conf']).tobytes() == conf[k].tobytes(), k
        assert x['pred_mask']['length'] == n_points
        assert np.array_equal(ids[off[k]:off[k + 1]], _rle_ids(x['pred_mask'])), k
    for k in {0, len(pred) // 2, len(pred) - 1} if pred else ():
        assert np.array_equal(_rle_ids(pred[k]['pred_mask']), np.flatnonzero(rle_decode(pred[k]['pred_mask'])))
    sem = dev['semantic_preds'].cpu().numpy()
    assert sem.dtype == np.int64 and sem.shape == (n_points, )
    assert np.array_equal(sem, host['semantic_preds'])
    assert np.array_equal(dev['offset_preds'].cpu().numpy(), host['offset_preds'])
    pan = dev['panoptic_preds'].cpu().numpy()
    assert np.array_equal(pan, model.panoptic_fusion(host['semantic_preds'], pred))
    if 'panoptic_preds' in host:
        assert np.array_equal(pan, host['panoptic_preds'])
    return len(pred)


@pytest.mark.parametrize('name', sorted(fc.bench.WORKLOADS))
def test_bench_workload_device_results_equal_host(name):
    w = fc.build_workload(fc.workload_case(name))
    model = w['model'].cuda()
    hb = harness.to_host_batch(w['scan'])
    inj = tuple(torch.from_numpy(a).cuda() for a in w['inj'])
    host, dev = _run_both(model, hb, inj)
    n = _same(model, host, dev, w['base']['coords'].shape[0], min_instances=10)
    print('\n[device results] %s: %d instances, %d point ids' % (name, n, dev['instances']['point_ids'].numel()))


def test_scannet_pp_lvl_fusion_device_results_equal_host():
    """lvl_fusion: heads, grouping and masks on voxels, results per point through v2p_map. The heads' outputs are replaced
    by the c2 workload's synthetic predictions averaged per voxel (computed once, so both forwards group the same input).
    The host forward's panoptic path takes voxel-level semantic predictions under lvl_fusion, so the host side here is
    panoptic_fusion on its point-level results."""
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet++')).cuda().eval()
    scan = synth.make_scan('c2_scannet', seed=0)
    scores, offs = (torch.from_numpy(a).cuda().double() for a in synth.grouping_inputs(scan, sigma=0.03, seed=0))
    orig, cache = model.forward_backbone, {}

    def voxel_heads(input, input_map, **kw):
        sem, off, feats = orig(input, input_map, **kw)
        if 'sem' not in cache:
            v = input_map.long()
            cnt = torch.zeros(sem.size(0), dtype=torch.float64, device=v.device).index_add_(0, v, torch.ones_like(v, dtype=torch.float64))
            cache['sem'] = (torch.zeros_like(sem, dtype=torch.float64).index_add_(0, v, scores) / cnt[:, None]).float()
            cache['off'] = (torch.zeros_like(off, dtype=torch.float64).index_add_(0, v, offs) / cnt[:, None]).float()
        return cache['sem'], cache['off'], feats

    model.forward_backbone = voxel_heads
    host, dev = _run_both(model, harness.to_host_batch(scan), host_tasks=['semantic', 'instance'])
    n = _same(model, host, dev, scan['coords'].shape[0], min_instances=10)
    print('\n[device results] scannet++: %d instances, %d point ids' % (n, dev['instances']['point_ids'].numel()))


def test_scannet200_device_results_equal_host():
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet200')).cuda().eval()
    scan = synth.make_scan('c6_scannet200', seed=0)
    hb = harness.to_host_batch(scan)
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=0)
    host, dev = _run_both(model, hb, inj)
    n = _same(model, host, dev, scan['coords'].shape[0], min_instances=10)
    print('\n[device results] scannet200: %d instances, %d point ids' % (n, dev['instances']['point_ids'].numel()))


# ---------------------------------------------------------------------------------------------------------------------
# edges
# ---------------------------------------------------------------------------------------------------------------------
def _small_model(**over):
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet', channels=16, num_blocks=4, **over)).cuda().eval()
    model.test_cfg.setdefault('panoptic_skip_iou', SKIP_IOU)
    return model


def test_no_proposals():
    model = _small_model(grouping_cfg=dict(score_thr=1.5))  # no softmax value passes: nothing is grouped
    scan = synth.make_scan('c2_scannet', seed=1, n_points=20000)
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=1)
    host, dev = _run_both(model, harness.to_host_batch(scan), inj)
    assert _same(model, host, dev, 20000, min_instances=0) == 0
    assert dev['instances']['point_offsets'].cpu().tolist() == [0]


def test_proposals_without_kept_instance():
    model = _small_model(test_cfg=dict(cls_score_thr=1.0))  # no softmax value is above 1
    scan = synth.make_scan('c2_scannet', seed=2, n_points=20000)
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=2)
    calls = []
    orig = model.clusters_voxelization

    def spy(pidx, poff, *a, **kw):
        calls.append(poff.numel() - 1)
        return orig(pidx, poff, *a, **kw)

    model.clusters_voxelization = spy
    host, dev = _run_both(model, harness.to_host_batch(scan), inj)
    assert min(calls) > 0  # both forwards had proposals
    assert _same(model, host, dev, 20000, min_instances=0) == 0


def test_sem2ins_class_without_points():
    """sem2ins classes 3 and 7; class 7 is nobody's prediction: its instance is there, at its class's position, empty."""
    model = _small_model(sem2ins_classes=[3, 7])
    scan = synth.make_scan('c2_scannet', seed=3, n_points=30000)
    scores, off = harness.pointwise_injection(scan, sigma=0.03, seed=3)
    scores[:, 7] = -1e4
    host, dev = _run_both(model, harness.to_host_batch(scan), (scores, off))
    _same(model, host, dev, 30000, min_instances=3)
    label = dev['instances']['label_id'].cpu().numpy()
    off_ = dev['instances']['point_offsets'].cpu().numpy()
    k7 = int(np.flatnonzero(label == 8)[0])
    assert off_[k7] == off_[k7 + 1] and dev['instances']['conf'][k7].item() == 1.0
    k3 = int(np.flatnonzero(label == 4)[0])
    assert off_[k3 + 1] - off_[k3] == int((scores.argmax(1) == 3).sum())


def test_instances_covering_every_point():
    """900 points all predicted as one class and shifted onto one spot: one proposal of every point, kept for every class
    with every mask score above the threshold -- rows with every bit below N set."""
    n = 900
    model = _small_model(test_cfg=dict(mask_score_thr=-1e9, min_npoint=10))
    scan = synth.make_scan('c2_scannet', seed=4, n_points=n)
    n = scan['coords'].shape[0]
    scores = torch.full((n, 20), -8.0)
    scores[:, 5] = 8.0
    cf = torch.from_numpy(scan['coords_float'])
    off = cf[0:1] - cf
    host, dev = _run_both(model, harness.to_host_batch(scan), (scores.cuda(), off.contiguous().cuda()))
    k = _same(model, host, dev, n)
    offs = dev['instances']['point_offsets'].cpu().numpy()
    assert np.all(np.diff(offs) == n)
    assert k == model.instance_classes


# ---------------------------------------------------------------------------------------------------------------------
# host reads, scans in flight
# ---------------------------------------------------------------------------------------------------------------------
def _syncs(fn):
    prev = torch.cuda.get_sync_debug_mode()
    try:
        with warnings.catch_warnings(record=True) as seen, torch.no_grad():
            warnings.simplefilter('always')
            torch.cuda.set_sync_debug_mode('warn')
            fn()
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    return sum('synchronizing CUDA operation' in str(w.message) for w in seen)


@pytest.mark.parametrize('sem2ins', [[], [3]])
def test_host_reads(sem2ins):
    model = _small_model(sem2ins_classes=sem2ins)
    scan = synth.make_scan('c2_scannet', seed=5, n_points=40000)
    hb = harness.to_host_batch(scan)
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=5)
    tc = model.test_cfg
    counts = {}
    for tasks in (['semantic', 'instance'], ALL_TASKS):
        tc['eval_tasks'] = tasks
        for mode in ('device_only', 'device_results'):
            def run():
                return harness.run_scan(model, hb, inject_pointwise=inj, **{mode: True})
            with torch.no_grad():
                run()  # warm-up: plans, pinned blocks, first launches
                torch.cuda.synchronize()
            counts[(tuple(tasks), mode)] = _syncs(run)
            torch.cuda.synchronize()
    with torch.no_grad():
        ret = harness.run_scan(model, hb, inject_pointwise=inj, device_results=True)
    assert ret['instances']['label_id'].numel() > 0
    for tasks, extra in ((('semantic', 'instance'), 1), (tuple(ALL_TASKS), 2)):
        assert counts[(tasks, 'device_results')] - counts[(tasks, 'device_only')] == extra, counts
    with pytest.raises(ValueError):
        harness.run_scan(model, hb, inject_pointwise=inj, device_only=True, device_results=True)


def test_scans_in_flight_equal_sequential_calls():
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet', test_cfg=dict(eval_tasks=ALL_TASKS, panoptic_skip_iou=SKIP_IOU))).cuda().eval()
    scans = [synth.make_scan('c2_scannet', seed=s, n_points=n) for s, n in ((1, 40000), (2, 61000), (3, 52000))] * 2
    hbs = [harness.to_host_batch(sc) for sc in scans]
    injs = [harness.pointwise_injection(sc, sigma=0.03, seed=7) for sc in scans]
    with torch.no_grad():
        seq = [harness.run_scan(model, hb, inject_pointwise=inj, device_results=True) for hb, inj in zip(hbs, injs)]
    torch.cuda.synchronize()
    seq = [_to_host(r) for r in seq]
    pipe = harness.ScanPipeline(model, workers=3)
    try:
        par = [_to_host(r) for r in pipe.run_scans(hbs, inject_pointwise=injs, device_results=True)]
    finally:
        pipe.close()
    assert len(par) == len(seq)
    for a, b in zip(seq, par):
        assert a.keys() == b.keys() and a['instances.label_id'].size > 0
        for k in a:
            assert np.array_equal(a[k], b[k]), k


def _to_host(ret):
    out = {}
    for k, v in ret.items():
        if isinstance(v, dict):
            out.update({k + '.' + kk: vv.cpu().numpy() for kk, vv in v.items()})
        elif torch.is_tensor(v):
            out[k] = v.cpu().numpy()
    return out
