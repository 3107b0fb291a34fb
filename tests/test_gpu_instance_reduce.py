"""instance_point_reduce / instance_point_map (sgb_id_lists_reduce / sgb_id_lists_point_map) against numpy.

  * synthetic lists: more than 65,535 lists, one list of all 1.5M points, empty lists, ids shared by several lists, N a
    multiple of 32 and not, C in {1, 3, 32, 33}, strided values, values holding NaN, +-inf and -0.0; min, max, counts
    and the point map exactly, mean within the bound of include/sgb200.h and with the same bits twice; confidence ties,
    -0.0 against +0.0, NaN and +-inf confidences, points in no list;
  * more than 2^31 ids in all (8.6 GB of int32 ids), int64 offsets end to end;
  * the device results of every bench workload, scannet++ (lvl_fusion) and scannet200: coords_float and offset_preds
    reduced over every instance, and the point map, against numpy over point_ids;
  * launch counts, no host wait (the calls return while their stream is still busy), scans in flight equal sequential
    calls."""
import os
import sys

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

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------------
# numpy restatements
# ---------------------------------------------------------------------------------------------------------------------
def np_reduce(off, ids, values):
    """float64 restatement: min / max with NaN never winning (empty: +inf / -inf), float64 mean (empty: NaN), sum|x|
    and counts."""
    n, C = off.size - 1, values.shape[1]
    lens = np.diff(off)
    g = values[ids].astype(np.float64)
    mn = np.full((n, C), np.inf)
    mx = np.full((n, C), -np.inf)
    sm = np.zeros((n, C))
    ab = np.zeros((n, C))
    ne = np.flatnonzero(lens > 0)
    with np.errstate(invalid='ignore', divide='ignore'):  # inf - inf and 0 / 0 are NaN, as on the device
        if ne.size:
            st = off[ne]
            mn[ne] = np.minimum.reduceat(np.where(np.isnan(g), np.inf, g), st, axis=0)
            mx[ne] = np.maximum.reduceat(np.where(np.isnan(g), -np.inf, g), st, axis=0)
            sm[ne] = np.add.reduceat(g, st, axis=0)
            ab[ne] = np.add.reduceat(np.abs(g), st, axis=0)
        mean = sm / lens[:, None]
    return mn, mx, mean, ab, lens


def np_point_map(off, ids, conf, n_points):
    """A loop over the lists in k order: a list takes a point when it holds no list yet, when its confidence is strictly
    higher, or when the holder's confidence is NaN and its own is not."""
    best = np.full(n_points, -1, np.int64)
    bc = np.zeros(n_points, np.float32)
    for k in range(off.size - 1):
        p = ids[off[k]:off[k + 1]]
        if p.size == 0:
            continue
        c, cur = conf[k], bc[p]
        take = (best[p] < 0) | (c > cur) | (np.isnan(cur) & ~np.isnan(c))
        best[p[take]] = k
        bc[p[take]] = c
    return best


def mean_bound(want, ab, lens):
    """The bound of include/sgb200.h (sgb_id_lists_reduce), plus the error of numpy's own float64 pairwise sum."""
    L = np.maximum(lens, 1).astype(np.float64)[:, None]
    return 2.0 ** -24 * np.abs(want) + ((L / 256 + 300) * 2.0 ** -52 + (np.log2(L) + 2) * 2.0 ** -53) * ab / L


def check_reduce(out, off, ids, values):
    mn, mx, mean, ab, lens = np_reduce(off, ids, values)
    assert out['counts'].dtype == torch.int64 and np.array_equal(out['counts'].cpu().numpy(), lens)
    got_mn, got_mx, got_mean = (out[k].cpu().numpy() for k in ('min', 'max', 'mean'))
    assert np.array_equal(got_mn, mn) and np.array_equal(got_mx, mx)  # -0.0 == 0.0: the sign of a zero is unspecified
    fin = np.isfinite(mean)
    assert np.array_equal(np.isnan(got_mean), np.isnan(mean))
    assert np.array_equal(got_mean[~fin & ~np.isnan(mean)], mean[~fin & ~np.isnan(mean)])
    err = np.abs(got_mean[fin].astype(np.float64) - mean[fin])
    assert np.all(err <= mean_bound(mean, ab, lens)[fin]), err.max()


def _special_values(rng, N, C, stride_pad=0):
    """float32 [N, C] CUDA, a view with row stride C + stride_pad: normal values with NaN, +-inf, -0.0 and 0.0 mixed in."""
    v = (rng.randn(N, C + stride_pad) * rng.uniform(0.1, 100, C + stride_pad)).astype(np.float32)
    for val, share in ((np.nan, 0.002), (np.inf, 0.001), (-np.inf, 0.001), (-0.0, 0.003), (0.0, 0.003)):
        v[rng.rand(N, C + stride_pad) < share] = val
    t = torch.from_numpy(v).cuda()[:, :C]
    return t, v[:, :C]


def _random_lists(rng, n, n_points, max_len):
    """n lists of 0..max_len ids (a quarter of them empty), random ids: a point is in several lists, ids repeat."""
    lens = rng.randint(0, max_len + 1, size=n)
    lens[rng.rand(n) < 0.25] = 0
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return off, rng.randint(0, n_points, size=int(off[-1])).astype(np.int32)


def _instances(off, ids, conf=None):
    d = dict(point_offsets=torch.from_numpy(off).cuda(), point_ids=torch.from_numpy(ids).cuda())
    if conf is not None:
        d['conf'] = torch.from_numpy(conf).cuda()
    return d


def _confs(rng, n):
    """Confidences with ties, -0.0 / +0.0, NaN and +-inf."""
    c = rng.choice(np.float32([0.1, 0.25, 0.5, 0.9, 0.0, -0.0, np.nan, np.inf, -np.inf, 0.5]), size=n)
    c[rng.rand(n) < 0.3] = np.float32(0.625)  # a large group of equal confidences
    return c.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# synthetic lists
# ---------------------------------------------------------------------------------------------------------------------
def _chunk_crossing_lists(rng, n_points):
    """Lengths around the 256-id chunk: lists inside one chunk, ending on a boundary, spanning several chunks."""
    lens = np.array([0, 1, 255, 256, 257, 0, 511, 1000, 5000, 3, 0, 70000, 2, 256, 0], np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    return off, rng.randint(0, n_points, size=int(off[-1])).astype(np.int32)


CASES = {
    # name: (lists(rng) -> (off, ids), N, C, row padding)
    'many_lists_C1': (lambda rng: _random_lists(rng, 70000, 100003, 8), 100003, 1, 0),
    'many_lists_C33_strided': (lambda rng: _random_lists(rng, 66000, 4096, 12), 4096, 33, 7),
    'all_points_C3': (lambda rng: (np.array([0, 0, 1500000, 1500000], np.int64), np.arange(1500000, dtype=np.int32)),
                      1500000, 3, 0),
    'chunk_crossing_C32_strided': (lambda rng: _chunk_crossing_lists(rng, 4099), 4099, 32, 5),
    'chunk_crossing_C3': (lambda rng: _chunk_crossing_lists(rng, 64), 64, 3, 0),
}


@pytest.mark.parametrize('name', sorted(CASES))
def test_reduce_and_point_map_vs_numpy(name):
    make, N, C, pad = CASES[name]
    rng = np.random.RandomState(len(name))
    off, ids = make(rng)
    values, v_np = _special_values(rng, N, C, pad)
    assert values.stride(0) == C + pad
    conf = _confs(rng, off.size - 1)
    inst = _instances(off, ids, conf)
    L = _lib.lib()
    before = L.sgb_launch_count()
    out = inst_ops.instance_point_reduce(inst, values)
    pmap = inst_ops.instance_point_map(inst, N)
    torch.cuda.synchronize()
    assert L.sgb_launch_count() - before == 4
    check_reduce(out, off, ids, v_np)
    assert pmap.dtype == torch.int32 and np.array_equal(pmap.cpu().numpy(), np_point_map(off, ids, conf, N))
    # the same bits on a second run, and for every subset of the ops
    again = inst_ops.instance_point_reduce(inst, values)
    for k in ('min', 'max', 'mean', 'counts'):
        assert out[k].cpu().numpy().tobytes() == again[k].cpu().numpy().tobytes(), k
    only = inst_ops.instance_point_reduce(inst, values, ops=('mean', ))
    assert set(only) == {'mean', 'counts'} and only['mean'].cpu().numpy().tobytes() == out['mean'].cpu().numpy().tobytes()


def test_point_map_ties_nan_and_uncovered_points():
    """Lists 0..6 over 10 points: equal confidences (the smaller k wins), -0.0 against +0.0 (a tie), NaN (below every
    number, -inf included, but still a holder when nothing else holds the point), points 8 and 9 in no list."""
    lists = [[0, 1], [1, 2], [2, 3], [3, 4], [4, 5, 6], [5, 7], [6, 7]]
    conf = np.float32([0.5, 0.5, -0.0, 0.0, np.nan, -np.inf, np.nan])
    off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
    ids = np.concatenate(lists).astype(np.int32)
    got = inst_ops.instance_point_map(_instances(off, ids, conf), 10).cpu().numpy()
    assert got.tolist() == [0, 0, 1, 2, 3, 5, 4, 5, -1, -1]
    assert np.array_equal(got, np_point_map(off, ids, conf, 10))


def test_no_lists_and_empty_lists():
    values = torch.randn(100, 3, device='cuda')
    L = _lib.lib()
    before = L.sgb_launch_count()
    out = inst_ops.instance_point_reduce(_instances(np.zeros(1, np.int64), np.zeros(0, np.int32)), values)
    assert L.sgb_launch_count() == before and out['mean'].shape == (0, 3) and out['counts'].shape == (0, )
    inst = _instances(np.zeros(4, np.int64), np.zeros(0, np.int32), np.float32([0.1, 0.2, 0.3]))
    out = inst_ops.instance_point_reduce(inst, values)
    pmap = inst_ops.instance_point_map(inst, 100)
    torch.cuda.synchronize()
    assert L.sgb_launch_count() - before == 2  # the list pass of the reduction, the decode pass of the map
    assert torch.all(out['min'] == float('inf')) and torch.all(out['max'] == -float('inf'))
    assert torch.all(torch.isnan(out['mean'])) and torch.all(out['counts'] == 0) and torch.all(pmap == -1)


def test_beyond_int32_ids():
    """One list of 2^31 + 1000 ids cycling over 1,000,003 points, with short lists before and after it (their offsets
    beyond 2^31) and an empty one: counts, offsets int64 end to end, the long list's min / max exactly and its mean within
    the bound, the short lists exactly, and the point map."""
    N, C = 1000003, 3
    rng = np.random.RandomState(31)
    v = rng.randn(N, C).astype(np.float32)
    v[5] = [np.nan, -np.inf, 7.0]
    big = (1 << 31) + 1000
    lens = np.array([17, big, 0, 300, 5, 1], np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    total = int(off[-1])
    ids = torch.empty(total, dtype=torch.int32, device='cuda')
    step = 1 << 28
    for a in range(int(off[1]), int(off[2]), step):  # the long list: global index i holds point i % N
        b = min(a + step, int(off[2]))
        ids[a:b] = (torch.arange(a, b, device='cuda') % N).int()
    small = {k: rng.randint(0, N, size=int(lens[k])).astype(np.int32) for k in (0, 3, 4, 5)}
    for k, s in small.items():
        ids[int(off[k]):int(off[k + 1])] = torch.from_numpy(s).cuda()
    conf = np.float32([0.2, 0.5, 0.9, 0.9, 0.1, 0.7])
    inst = dict(point_offsets=torch.from_numpy(off).cuda(), point_ids=ids, conf=torch.from_numpy(conf).cuda())
    values = torch.from_numpy(v).cuda()
    out = inst_ops.instance_point_reduce(inst, values)
    pmap = inst_ops.instance_point_map(inst, N).cpu().numpy()
    assert inst['point_offsets'].dtype == torch.int64 and int(inst['point_offsets'][-1]) == total == ids.numel()
    assert out['counts'].cpu().numpy().tolist() == lens.tolist()
    got = {k: out[k].cpu().numpy() for k in ('min', 'max', 'mean')}
    # the long list: point p appears q or q + 1 times
    a, b = int(off[1]), int(off[2])
    times = np.full(N, (b - a) // N, np.int64)
    first = a % N
    extra = (np.arange(N) - first) % N < (b - a) % N
    times += extra
    vd = v.astype(np.float64)
    assert np.array_equal(got['min'][1], np.where(np.isnan(vd), np.inf, vd).min(0))
    assert np.array_equal(got['max'][1], np.where(np.isnan(vd), -np.inf, vd).max(0))
    with np.errstate(invalid='ignore'):
        m = (times[:, None] * vd).sum(0) / big
    assert np.isnan(got['mean'][1, 0]) and got['mean'][1, 1] == -np.inf
    ab = (times * np.abs(vd[:, 2])).sum()
    assert abs(float(got['mean'][1, 2]) - m[2]) <= mean_bound(np.array([[m[2]]]), np.array([[ab]]), np.array([big]))[0, 0]
    for k, s in small.items():
        mn, mx, mean, ab_k, _ = np_reduce(np.array([0, s.size], np.int64), s, v)
        assert np.array_equal(got['min'][k], mn[0]) and np.array_equal(got['max'][k], mx[0]), k
        fin = np.isfinite(mean[0])
        assert np.all(np.abs(got['mean'][k][fin] - mean[0][fin]) <= mean_bound(mean, ab_k, np.array([s.size]))[0][fin]), k
    want = np.ones(N, np.int64)  # every point is in the long list (conf 0.5); the short lists above 0.5 take theirs
    want[small[5]] = 5  # conf 0.7
    want[small[3]] = 3  # conf 0.9 wins where both hold a point
    assert np.array_equal(pmap, want)


# ---------------------------------------------------------------------------------------------------------------------
# device results of real forwards
# ---------------------------------------------------------------------------------------------------------------------
def _check_device_results(dev, coords_float, n_points, min_instances=10):
    inst = dev['instances']
    off = inst['point_offsets'].cpu().numpy()
    ids = inst['point_ids'].cpu().numpy()
    assert off.size - 1 >= min_instances
    for values in (torch.from_numpy(np.ascontiguousarray(coords_float)).cuda(), dev['offset_preds']):
        out = inst_ops.instance_point_reduce(inst, values)
        check_reduce(out, off, ids, values.cpu().numpy())
    pmap = inst_ops.instance_point_map(inst, n_points).cpu().numpy()
    assert np.array_equal(pmap, np_point_map(off, ids, inst['conf'].cpu().numpy(), n_points))
    return off.size - 1


def _device_results(model, hb, inj=None):
    tc = model.test_cfg
    keep = tc['eval_tasks']
    tc['eval_tasks'] = ['semantic', 'instance']
    try:
        with torch.no_grad():
            dev = harness.run_scan(model, hb, inject_pointwise=inj, device_results=True)
        torch.cuda.synchronize()
    finally:
        tc['eval_tasks'] = keep
    return dev


@pytest.mark.parametrize('name', sorted(fc.bench.WORKLOADS))
def test_bench_workload_instances(name):
    w = fc.build_workload(fc.workload_case(name))
    model = w['model'].cuda()
    inj = tuple(torch.from_numpy(a).cuda() for a in w['inj'])
    dev = _device_results(model, harness.to_host_batch(w['scan']), inj)
    n = _check_device_results(dev, w['base']['coords_float'], w['base']['coords'].shape[0])
    print('\n[instance reduce] %s: %d instances, %d point ids' % (name, n, dev['instances']['point_ids'].numel()))


def test_scannet_pp_lvl_fusion_instances():
    """lvl_fusion: the lists hold point ids, so the values are per point. The heads' outputs are the c2 workload's
    synthetic predictions averaged per voxel, so that the random-init model groups instances."""
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
    assert dev['offset_preds'].shape[0] == scan['coords'].shape[0]
    _check_device_results(dev, scan['coords_float'], scan['coords'].shape[0])


def test_scannet200_instances():
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg('scannet200')).cuda().eval()
    scan = synth.make_scan('c6_scannet200', seed=0)
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=0)
    dev = _device_results(model, harness.to_host_batch(scan), inj)
    _check_device_results(dev, scan['coords_float'], scan['coords'].shape[0])


# ---------------------------------------------------------------------------------------------------------------------
# no host wait, scans in flight
# ---------------------------------------------------------------------------------------------------------------------
def test_calls_enqueue_without_waiting():
    """Both calls return while their stream is still busy with work enqueued before them (a ~0.2 s spin): neither waits
    for the device. Their results then equal those of calls on an idle stream."""
    rng = np.random.RandomState(9)
    off, ids = _random_lists(rng, 5000, 20000, 300)
    values = torch.from_numpy(rng.randn(20000, 32).astype(np.float32)).cuda()
    inst = _instances(off, ids, rng.rand(5000).astype(np.float32))
    want = inst_ops.instance_point_reduce(inst, values), inst_ops.instance_point_map(inst, 20000)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    prev = torch.cuda.get_sync_debug_mode()
    with torch.cuda.stream(side):
        torch.cuda._sleep(400_000_000)
        try:
            torch.cuda.set_sync_debug_mode('error')
            got = inst_ops.instance_point_reduce(inst, values), inst_ops.instance_point_map(inst, 20000)
        finally:
            torch.cuda.set_sync_debug_mode(prev)
        busy = not side.query()
    side.synchronize()
    assert busy
    for k in ('min', 'max', 'mean', 'counts'):
        assert got[0][k].cpu().numpy().tobytes() == want[0][k].cpu().numpy().tobytes(), k
    assert torch.equal(got[1], want[1])


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
        r = inst_ops.instance_point_reduce(dev['instances'], cf)
        r['map'] = inst_ops.instance_point_map(dev['instances'], cf.size(0))
        return r

    with torch.no_grad():
        seq = [one(a) for a in zip(hbs, injs, cfs)]
    torch.cuda.synchronize()
    seq = [{k: v.cpu().numpy() for k, v in r.items()} for r in seq]
    pipe = harness.ScanPipeline(model, workers=3)
    try:
        res, evs = pipe.map(one, list(zip(hbs, injs, cfs)))
        for e in evs:
            e.synchronize()
        par = [{k: v.cpu().numpy() for k, v in r.items()} for r in res]
    finally:
        pipe.close()
    for a, b in zip(seq, par):
        assert a['counts'].size > 0 and a.keys() == b.keys()
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), k
