"""Chunked one-pass grouping on the GPU. When the selected (class, point) entries are more than one ball query's int32
list cursor addresses (2^31 - 1 / 1000 = 2,147,483 entries), forward_grouping cuts the segments into chunks. Here:
  * forced chunks (the bound lowered) on a ScanNet-shape and a ScanNet200-shape scan: proposals and forward_test
    instances bit-identical to the single call;
  * a full-size S3DIS-shape room beyond the bound: proposals equal the reference-order per-class loop (ballquery_batch_p
    with its relaunch + bfs_cluster_segments per class);
  * one segment alone beyond the bound: it runs when its neighbour total fits int32 and raises SgbError, without
    clustering, when it does not."""
import itertools
import warnings

import numpy as np
import pytest
import torch

from softgroup_b200 import harness, ops, synth
from softgroup_b200.configs import model_cfg
from softgroup_b200.model import SoftGroup
from softgroup_b200.model import softgroup as sg_module
from softgroup_b200.ops import functions
from softgroup_b200.ops._lib import SgbError

pytestmark = pytest.mark.gpu

LIMIT = functions.BALLQUERY_MAX_CAPACITY // 1000  # 2,147,483 entries


def _model(cfg):
    torch.manual_seed(0)
    return SoftGroup(**cfg).cuda().eval()


def _segment_counts(monkeypatch, model, *args):
    """forward_grouping once, unpatched; returns its proposals and the entry count of every segment."""
    seen = []
    real = functions.group_entries

    def spy(*a, **k):
        out = real(*a, **k)
        seen.append(out[3])
        return out
    with monkeypatch.context() as m:
        m.setattr(sg_module, 'group_entries', spy)
        with torch.no_grad():
            idx, off = model.forward_grouping(*args)
    return idx.cpu().numpy(), off.cpu().numpy(), np.diff(seen[0].cpu().numpy().astype(np.int64))


def _one_per_segment(counts, max_capacity=None):
    return [(s, s + 1) for s in range(len(counts))]


def _forced(counts):
    """(bound, planner) pairs that cut the selection into 2 and 3 chunks, and one segment per chunk."""
    n = int(counts.sum())
    out = []
    for parts in (2, 3):
        bound = -(-n // parts) * 1000
        assert len([c for c in functions.plan_ballquery_chunks(counts, bound) if counts[c[0]:c[1]].sum()]) >= parts
        out.append((bound, None))
    out.append((n * 1000 - 1, _one_per_segment))
    return out


def _patched(m, bound, planner):
    m.setattr(functions, 'BALLQUERY_MAX_CAPACITY', bound)
    if planner is not None:
        m.setattr(functions, 'plan_ballquery_chunks', planner)


def _host_reads(model, *args):
    """Synchronising CUDA operations torch sees in one forward_grouping, with batch_size given as forward_test gives it
    (without it, forward_grouping reads the batch size back from the device)."""
    prev = torch.cuda.get_sync_debug_mode()
    try:
        with warnings.catch_warnings(record=True) as seen, torch.no_grad():
            warnings.simplefilter('always')
            torch.cuda.set_sync_debug_mode('warn')
            model.forward_grouping(*args, batch_size=1)
    finally:
        torch.cuda.set_sync_debug_mode(prev)
    return sum('synchronizing CUDA operation' in str(w.message) for w in seen)


def _same_instances(a, b):
    assert len(a) == len(b) and len(a) > 0
    for x, y in zip(a, b):
        assert x['label_id'] == y['label_id'] and x['pred_mask'] == y['pred_mask']
        assert float(x['conf']) == float(y['conf'])


CASES = {
    'scannet': (dict(name='scannet'), 'c2_scannet', 60000, 2),
    'scannet200': (dict(name='scannet200', grouping_cfg=dict(radius=0.15, class_numpoint_mean=[-1.] * 200, npoint_thr=50,
                                                             score_thr=0.1), test_cfg=dict(min_npoint=50)),
                   'c6_scannet200', 100000, 5),
}


@pytest.mark.parametrize('case', sorted(CASES))
def test_forced_chunks_bit_identical(monkeypatch, case):
    kw, shape, n_points, seed = CASES[case]
    kw = dict(kw)
    cfg = model_cfg(kw.pop('name'), **kw)
    model = _model(cfg)
    scan = synth.make_scan(shape, seed=seed, n_points=n_points)
    scores, offs = harness.pointwise_injection(scan, sigma=0.03, seed=seed)
    args = (scores, offs, torch.zeros(n_points, dtype=torch.int32, device='cuda'),
            torch.from_numpy(scan['coords_float']).cuda())
    want_idx, want_off, counts = _segment_counts(monkeypatch, model, *args)
    assert (counts > 0).sum() >= 3 and want_off.size > 10
    hb = harness.to_host_batch(scan)
    with torch.no_grad():
        want_inst = harness.run_scan(model, hb, inject_pointwise=(scores, offs))['pred_instances']
    # host reads after warm-up: below the bound only the entry count
    assert _host_reads(model, *args) == 1
    for bound, planner in _forced(counts):
        with monkeypatch.context() as m:
            _patched(m, bound, planner)
            with torch.no_grad():
                idx, off = model.forward_grouping(*args)
                inst = harness.run_scan(model, hb, inject_pointwise=(scores, offs))['pred_instances']
            reads = _host_reads(model, *args)
        assert np.array_equal(off.cpu().numpy(), want_off), (bound, planner)
        assert np.array_equal(idx.cpu().numpy(), want_idx), (bound, planner)
        _same_instances(inst, want_inst)
        # beyond it also the segment offsets, and the flags of every range whose entries x 1000 exceed the bound
        ranges = (planner or functions.plan_ballquery_chunks)(counts, bound)
        oversize = sum(1 for s0, s1 in ranges if counts[s0:s1].sum() * 1000 > bound)
        assert reads == 2 + oversize, (bound, planner, reads, oversize)


# ---- beyond the bound, unpatched -------------------------------------------------------------------------------------
def _per_class_loop(model, scores, offs, coords):
    """softgroup.py:430-473 of the reference on this repo's ops: one ballquery_batch_p (relaunched when the lists overflow
    mean_active) and one bfs_cluster_segments per class, proposals concatenated in class order."""
    g, get = model.grouping_cfg, model._cfg
    probs = scores.softmax(-1)
    cnm = get(g, 'class_numpoint_mean')
    npoint_thr = float(get(g, 'npoint_thr'))
    idx_list, off_list, n_prop, n_pts = [], [], 0, 0
    for c in range(model.semantic_classes):
        if c in get(g, 'ignore_classes'):
            continue
        obj = (probs[:, c] > get(g, 'score_thr')).nonzero().view(-1)
        if obj.size(0) < get(model.test_cfg, 'min_npoint'):
            continue
        xyz = (coords[obj] + offs[obj]).contiguous()
        bi = torch.zeros(obj.size(0), dtype=torch.int32, device='cuda')
        bo = torch.tensor([0, obj.size(0)], dtype=torch.int32, device='cuda')
        nb, sl = ops.ballquery_batch_p(xyz, bi, bo, get(g, 'radius'), get(g, 'mean_active'))
        thr = npoint_thr if cnm[c] == -1 else float(np.float32(npoint_thr) * np.float32(cnm[c]))
        pidx, poff = ops.bfs_cluster_segments(nb if nb.numel() else torch.zeros(1, dtype=torch.int32, device='cuda'), sl,
                                              thr)
        if pidx.size(0) == 0:
            continue
        pidx[:, 1] = obj[pidx[:, 1].long()].int()
        pidx[:, 0] += n_prop
        idx_list.append(pidx)
        off_list.append(poff[1:] + n_pts if off_list else poff)
        n_prop += poff.numel() - 1
        n_pts += pidx.size(0)
    return torch.cat(idx_list).cpu().numpy(), torch.cat(off_list).cpu().numpy()


def test_full_size_room_beyond_the_bound(monkeypatch):
    """S3DIS-shape room of 3,000,000 points with injected predictions (sigma 0.1): 2,556,688 entries of 11 grouped
    classes in two chunks, neighbour total 408,582,360 and 118 proposals (measured on an H100; the counts are printed).
    sigma 0.1 keeps the neighbour total below 2^31 over the whole room, not just per chunk."""
    n_points = 3000000
    model = _model(model_cfg('s3dis'))
    scan = synth.make_scan('c3_s3dis', seed=0, n_points=n_points)
    scores, offs = harness.pointwise_injection(scan, sigma=0.1, seed=0)
    coords = torch.from_numpy(scan['coords_float']).cuda()
    args = (scores, offs, torch.zeros(n_points, dtype=torch.int32, device='cuda'), coords)
    plans, totals = [], []
    real_plan, real_bq = functions.plan_ballquery_chunks, sg_module.ballquery_batch_p_nosync

    def bq(*a, **k):
        out = real_bq(*a, **k)
        totals.append(out[2])
        return out
    with monkeypatch.context() as m:
        m.setattr(functions, 'plan_ballquery_chunks', lambda c, cap=None: plans.append(real_plan(c, cap)) or plans[-1])
        m.setattr(sg_module, 'ballquery_batch_p_nosync', bq)
        idx, off, counts = _segment_counts(monkeypatch, model, *args)
    n = int(counts.sum())
    nbr = sum(int(t[0]) for t in totals)
    print('points %d entries %d chunks %d neighbour total %d proposals %d' % (n_points, n, len(plans[0]), nbr, off.size - 1))
    assert n > LIMIT
    assert len(plans) == 1 and len(plans[0]) == 2 and len(totals) == 2
    assert nbr < 2**31
    with torch.no_grad():
        want_idx, want_off = _per_class_loop(model, scores, offs, coords)
    assert want_off.size > 100
    assert np.array_equal(off, want_off)
    assert np.array_equal(idx, want_idx)


def _lattice(nx, ny, nz, drop_every=0):
    """Integer lattice points (spacing 1, x-major point order); drop_every > 0 leaves out every such x-plane."""
    xs = np.arange(nx)
    if drop_every:
        xs = xs[xs % drop_every != drop_every - 1]
    g = np.stack(np.meshgrid(xs, np.arange(ny), np.arange(nz), indexing='ij'), -1).reshape(-1, 3)
    return g.astype(np.float32)


def _lattice_total(shape, r2max):
    """Exact capped neighbour total of the full lattice at integer d^2 <= r2max (self included, lists cut at 1000):
    points are grouped by their distance to the faces, per axis clipped at the offset radius."""
    R = int(np.floor(np.sqrt(r2max)))
    off = np.array([d for d in itertools.product(range(-R, R + 1), repeat=3) if d[0]**2 + d[1]**2 + d[2]**2 <= r2max])
    classes = []
    for L in shape:  # per axis: representative coordinate and multiplicity
        reps = {}
        for x in range(L):
            key = (min(x, R), min(L - 1 - x, R))
            reps.setdefault(key, [x, 0])[1] += 1
        classes.append(list(reps.values()))
    total = 0
    for (x, mx), (y, my), (z, mz) in itertools.product(*classes):
        p = off + np.array([x, y, z])
        inside = np.all((p >= 0) & (p < np.array(shape)), 1).sum()
        total += min(int(inside), 1000) * mx * my * mz
    return total


def _one_class_scores(n, C, cls):
    logits = torch.zeros((n, C), device='cuda')
    logits[:, cls] = 20.0
    return logits


def test_oversize_segment_fits():
    """One class of 2,722,500 lattice points (one segment beyond the bound) at radius 1.5: it runs with capacity 2^31 - 1
    and gives the per-class loop's proposals (every tenth x-plane left out: 25 slab components)."""
    model = _model(model_cfg('s3dis', grouping_cfg=dict(radius=1.5)))
    xyz = torch.from_numpy(_lattice(250, 110, 110, drop_every=10)).cuda()
    n = xyz.size(0)
    assert n == 2722500 and n > LIMIT
    scores, offs = _one_class_scores(n, 13, 5), torch.zeros((n, 3), device='cuda')
    with torch.no_grad():
        idx, off = model.forward_grouping(scores, offs, torch.zeros(n, dtype=torch.int32, device='cuda'), xyz)
        want_idx, want_off = _per_class_loop(model, scores, offs, xyz)
    assert off.numel() == 26
    assert np.array_equal(off.cpu().numpy(), want_off) and np.array_equal(idx.cpu().numpy(), want_idx)


def test_oversize_segment_beyond_int32_raises(monkeypatch):
    """One class of 3,025,000 lattice points at radius 6.9 (1376 lattice points in an interior ball, lists cut at 1000):
    its neighbour total, computed exactly on the host, is beyond 2^31 - 1. The ball query's cursor cannot count it, the
    forward raises SgbError naming the limit, and nothing is clustered."""
    shape = (250, 110, 110)
    truth = _lattice_total(shape, 47)  # d^2 < 6.9^2 = 47.61 on integer offsets
    assert truth > 2**31 - 1
    model = _model(model_cfg('s3dis', grouping_cfg=dict(radius=6.9)))
    xyz = torch.from_numpy(_lattice(*shape)).cuda()
    n = xyz.size(0)
    scores, offs = _one_class_scores(n, 13, 5), torch.zeros((n, 3), device='cuda')
    clustered = []
    with monkeypatch.context() as m:
        m.setattr(sg_module, 'bfs_cluster_segments', lambda *a, **k: clustered.append(1))
        with pytest.raises(SgbError, match=r'2\^31 - 1'), torch.no_grad():
            model.forward_grouping(scores, offs, torch.zeros(n, dtype=torch.int32, device='cuda'), xyz)
    assert not clustered
    print('lattice %s: %d points, neighbour total %d' % (shape, n, truth))
