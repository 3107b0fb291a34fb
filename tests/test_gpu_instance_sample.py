"""instance_farthest_point_sample (sgb_id_lists_fps) against the C restatement of its contract (tests/fps_oracle.c),
bit for bit:

  * the worked example of include/sgb200.h, lists of length 1;
  * random lists: more than 65,535 of them; lengths at +-1 around every granularity threshold the header defines;
    K in {1, 2, 31, 32, 33, 1024, 4096} (K > len and K >> len included); empty lists, all-invalid lists, an invalid first
    position, repeated ids, duplicate coordinates, exact lattice ties, NaN and +-inf coordinates, strided coords;
  * one list of all 1.5M points (streaming cluster path), and more than 2^31 ids in all;
  * the device results of every bench workload, scannet++ (lvl_fusion) and scannet200, K = 256;
  * the same bytes twice, the launch count of the header, no host wait, scans in flight equal sequential calls."""
import os
import re
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import forward_cases as fc  # noqa: E402
import fps_oracle  # noqa: E402
from softgroup_b200 import harness, synth  # noqa: E402
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402
from softgroup_b200.ops import _lib  # noqa: E402
from softgroup_b200.ops import instances as inst_ops  # noqa: E402
from test_gpu_instance_reduce import _device_results  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = dict((m, int(v)) for m, v in re.findall(r'#define (SGB_FPS_\w+) (\d+)', open(os.path.join(ROOT, 'include', 'sgb200.h')).read()))
THRESHOLDS = [HDR['SGB_FPS_WARP_MAX'], HDR['SGB_FPS_CTA_MAX'], HDR['SGB_FPS_CLUSTER_MAX']]


def granularity(lens):
    """lists per path: warp, CTA, cluster (on chip), cluster (streaming)"""
    w, c, cl = THRESHOLDS
    return dict(warp=int(np.sum(lens <= w)), cta=int(np.sum((lens > w) & (lens <= c))),
                cluster=int(np.sum((lens > c) & (lens <= cl))), streaming=int(np.sum(lens > cl)))


def _instances(off, ids):
    return dict(point_offsets=torch.from_numpy(off).cuda(), point_ids=torch.from_numpy(ids).cuda())


def _fps(inst, coords, K):
    return inst_ops.instance_farthest_point_sample(inst, coords, K).cpu().numpy()


def test_worked_example_and_lists_of_one():
    ex = fps_oracle.WORKED_EXAMPLE
    got = _fps(_instances(ex['off'], ex['ids']), torch.from_numpy(ex['xyz']).cuda(), ex['K'])
    assert got.dtype == np.int32 and got.tolist() == ex['want']
    xyz = np.float32([[0, 0, 0], [np.nan, 1, 2], [np.inf, 0, 0]])
    off, ids = np.arange(5, dtype=np.int64), np.int32([0, 1, 2, 3])
    for K in (1, 4, 33):
        assert _fps(_instances(off, ids), torch.from_numpy(xyz).cuda(), K).tolist() == [[0] * K, [1] * K, [2] * K, [-1] * K]


def _threshold_lens():
    lens = [0, 1, 2, 31, 32, 33]
    for t in THRESHOLDS:
        lens += [t - 1, t, t + 1]
    return np.array(lens * 2, np.int64)


CASES = {
    # name: (lengths(rng), N, row padding of coords, K values)
    'many_lists': (lambda rng: rng.randint(0, 40, size=70000), 100003, 0, (1, 33, 1024)),
    'thresholds': (lambda rng: _threshold_lens(), 200003, 0, (1, 2, 31, 32, 33, 1024, 4096)),
    'thresholds_strided': (lambda rng: _threshold_lens()[::-1].copy(), 70001, 5, (32, 1024)),
    'mixed_lengths': (lambda rng: rng.choice([0, 3, 200, 600, 3000, 9000, 70000], size=300), 500000, 2, (2, 256)),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_random_lists_vs_oracle(name):
    make, N, pad, Ks = CASES[name]
    rng = np.random.RandomState(len(name))
    lens = make(rng)
    xyz = fps_oracle.edge_points(rng, N)
    off, ids = fps_oracle.edge_lists(rng, lens, N)
    full = torch.from_numpy(np.concatenate([xyz, rng.randn(N, pad).astype(np.float32)], 1)).cuda()
    coords = full[:, :3]
    assert coords.stride(0) == 3 + pad
    inst = _instances(off, ids)
    print('\n[fps] %s: %d lists, %s' % (name, lens.size, granularity(lens)))
    for K in Ks:
        got = _fps(inst, coords, K)
        want = fps_oracle.id_lists_fps(off, ids, xyz, K)
        assert got.shape == (lens.size, K) and np.array_equal(got, want), (K, np.argwhere(got != want)[:5])
        again = _fps(inst, coords, K)
        assert got.tobytes() == again.tobytes()


def test_one_list_of_all_points():
    """1.5M points in one list (with empty lists around it): the streaming cluster path, K = 64."""
    N = 1500000
    rng = np.random.RandomState(15)
    xyz = fps_oracle.edge_points(rng, N)
    off = np.array([0, 0, N, N], np.int64)
    ids = rng.permutation(N).astype(np.int32)
    assert N > HDR['SGB_FPS_CLUSTER_MAX']
    got = _fps(_instances(off, ids), torch.from_numpy(xyz).cuda(), 64)
    assert np.array_equal(got, fps_oracle.id_lists_fps(off, ids, xyz, 64))


def test_beyond_int32_ids():
    """Copies of one 1.5M-point list until the ids pass 2^31 (8.6 GB of int32 ids), then three short lists whose offsets
    are beyond 2^31; K = 4. The oracle runs once for the copied list."""
    N = 1500000
    rng = np.random.RandomState(31)
    xyz = fps_oracle.edge_points(rng, N)
    one = rng.permutation(N).astype(np.int32)
    copies = (1 << 31) // N + 1
    short = [rng.randint(0, N, size=s).astype(np.int32) for s in (5, 700, 9000)]
    lens = np.array([N] * copies + [s.size for s in short], np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    assert off[copies] > (1 << 31)
    ids = torch.from_numpy(one).cuda().repeat(copies)
    ids = torch.cat([ids] + [torch.from_numpy(s).cuda() for s in short])
    inst = dict(point_offsets=torch.from_numpy(off).cuda(), point_ids=ids)
    got = inst_ops.instance_farthest_point_sample(inst, torch.from_numpy(xyz).cuda(), 4)
    del ids, inst
    want_one = fps_oracle.id_lists_fps(np.array([0, N], np.int64), one, xyz, 4)[0]
    got = got.cpu().numpy()
    assert np.array_equal(got[:copies], np.broadcast_to(want_one, (copies, 4)))
    soff = np.concatenate([[0], np.cumsum([s.size for s in short])]).astype(np.int64)
    assert np.array_equal(got[copies:], fps_oracle.id_lists_fps(soff, np.concatenate(short), xyz, 4))


# ---------------------------------------------------------------------------------------------------------------------
# device results of real forwards
# ---------------------------------------------------------------------------------------------------------------------
def _check_device_results(dev, coords_float, name, K=256):
    inst = dev['instances']
    off = inst['point_offsets'].cpu().numpy()
    ids = inst['point_ids'].cpu().numpy()
    assert off.size - 1 >= 10
    got = _fps(inst, torch.from_numpy(np.ascontiguousarray(coords_float)).cuda(), K)
    assert np.array_equal(got, fps_oracle.id_lists_fps(off, ids, coords_float, K))
    g = granularity(np.diff(off))
    print('\n[fps] %s: %d instances, %d point ids, K = %d, lists per path %s' % (name, off.size - 1, ids.size, K, g))
    return np.diff(off), inst['label_id'].cpu().numpy()


@pytest.mark.parametrize('name', sorted(fc.bench.WORKLOADS))
def test_bench_workload_instances(name):
    w = fc.build_workload(fc.workload_case(name))
    model = w['model'].cuda()
    inj = tuple(torch.from_numpy(a).cuda() for a in w['inj'])
    dev = _device_results(model, harness.to_host_batch(w['scan']), inj)
    lens, label = _check_device_results(dev, w['base']['coords_float'], name)
    if name == 'c3':  # sem2ins instances (label_id = class + 1) hold every point of their class: the cluster path
        sem2ins = np.isin(label - 1, w['cfg']['sem2ins_classes'])
        assert sem2ins.any() and np.all(lens[sem2ins] > HDR['SGB_FPS_CTA_MAX'])


def test_scannet_pp_lvl_fusion_instances():
    """lvl_fusion: the lists hold point ids, so coords are per point (the heads as in test_gpu_instance_reduce)."""
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
    dev = _device_results(model, harness.to_host_batch(scan))
    _check_device_results(dev, scan['coords_float'], 'scannet++')


def test_scannet200_instances():
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet200')).cuda().eval()
    scan = synth.make_scan('c6_scannet200', seed=0)
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=0)
    dev = _device_results(model, harness.to_host_batch(scan), inj)
    _check_device_results(dev, scan['coords_float'], 'scannet200')


# ---------------------------------------------------------------------------------------------------------------------
# launches, no host wait, scans in flight
# ---------------------------------------------------------------------------------------------------------------------
def test_launch_count():
    rng = np.random.RandomState(3)
    xyz = torch.from_numpy(rng.randn(1000, 3).astype(np.float32)).cuda()
    L = _lib.lib()
    for lens in ([5, 0, 7], [9000], [0, 0]):
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
        inst = _instances(off, rng.randint(0, 1000, size=int(off[-1])).astype(np.int32))
        before = L.sgb_launch_count()
        inst_ops.instance_farthest_point_sample(inst, xyz, 8)
        assert L.sgb_launch_count() - before == HDR['SGB_FPS_LAUNCHES'] == 4
    before = L.sgb_launch_count()
    out = inst_ops.instance_farthest_point_sample(_instances(np.zeros(1, np.int64), np.zeros(0, np.int32)), xyz, 8)
    assert L.sgb_launch_count() == before and out.shape == (0, 8)


def test_call_enqueues_without_waiting():
    """The call returns while its stream is still busy with work enqueued before it (a ~0.2 s spin); its result then
    equals that of a call on an idle stream."""
    rng = np.random.RandomState(9)
    off, ids = fps_oracle.edge_lists(rng, rng.choice([10, 600, 9000, 70000], size=40), 200000)
    xyz = torch.from_numpy(fps_oracle.edge_points(rng, 200000)).cuda()
    inst = _instances(off, ids)
    want = inst_ops.instance_farthest_point_sample(inst, xyz, 64)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    prev = torch.cuda.get_sync_debug_mode()
    with torch.cuda.stream(side):
        torch.cuda._sleep(400_000_000)
        try:
            torch.cuda.set_sync_debug_mode('error')
            got = inst_ops.instance_farthest_point_sample(inst, xyz, 64)
        finally:
            torch.cuda.set_sync_debug_mode(prev)
        busy = not side.query()
    side.synchronize()
    assert busy and torch.equal(got, want)


def test_scans_in_flight_equal_sequential_calls():
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet')).cuda().eval()
    scans = [synth.make_scan('c2_scannet', seed=s, n_points=n) for s, n in ((1, 40000), (2, 61000), (3, 52000))] * 2
    hbs = [harness.to_host_batch(sc) for sc in scans]
    injs = [harness.pointwise_injection(sc, sigma=0.03, seed=7) for sc in scans]
    cfs = [torch.from_numpy(sc['coords_float']).cuda() for sc in scans]

    def one(a):
        hb, inj, cf = a
        dev = harness.run_scan(model, hb, inject_pointwise=inj, device_results=True)
        return inst_ops.instance_farthest_point_sample(dev['instances'], cf, 256)

    with torch.no_grad():
        seq = [one(a).cpu().numpy() for a in zip(hbs, injs, cfs)]
    pipe = harness.ScanPipeline(model, workers=3)
    try:
        res, evs = pipe.map(one, list(zip(hbs, injs, cfs)))
        for e in evs:
            e.synchronize()
        par = [r.cpu().numpy() for r in res]
    finally:
        pipe.close()
    for a, b in zip(seq, par):
        assert a.shape[0] > 0 and a.tobytes() == b.tobytes()
