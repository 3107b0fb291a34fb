"""Chunked one-pass grouping on CPU: plan_ballquery_chunks, and forward_grouping cut into chunks of segments (the
selection's worst-case neighbour buffer beyond the ball query's int32 cursor) against the same forward in one call.
The device ops are the oracle stand-ins of test_host_grouping.py; the bound is lowered so that small scans chunk."""
import numpy as np
import pytest
import torch

from softgroup_b200 import synth
from softgroup_b200.configs import model_cfg
from softgroup_b200.model import SoftGroup
from softgroup_b200.model import softgroup as sg_module
from softgroup_b200.ops import functions
from softgroup_b200.ops._lib import SgbError
from test_host_grouping import _fake_ballquery_nosync, _fake_bfs_segments, _fake_group_entries

LIMIT = (2**31 - 1) // 1000  # most entries one chunk takes at the real bound: 2,147,483


# ---- the planner ------------------------------------------------------------------------------------------------
def test_plan_empty_segments():
    assert functions.plan_ballquery_chunks([]) == []
    assert functions.plan_ballquery_chunks([0, 0, 0]) == [(0, 3)]


def test_plan_one_chunk():
    assert functions.plan_ballquery_chunks([10, 0, 20, 30]) == [(0, 4)]
    assert functions.plan_ballquery_chunks([LIMIT]) == [(0, 1)]


def test_plan_exact_boundary():
    # sum * 1000 = 2,147,483,000 <= 2^31 - 1: one chunk; one entry more (+1000 in the buffer) is beyond the cursor
    assert functions.plan_ballquery_chunks([1000000, LIMIT - 1000000]) == [(0, 2)]
    assert functions.plan_ballquery_chunks([1000000, LIMIT - 1000000 + 1]) == [(0, 1), (1, 2)]
    assert functions.plan_ballquery_chunks([1000000, LIMIT - 1000000, 0, 0]) == [(0, 4)]
    assert functions.plan_ballquery_chunks([1000000, LIMIT - 1000000, 0, 1]) == [(0, 3), (3, 4)]


def test_plan_oversize_segment_alone():
    assert functions.plan_ballquery_chunks([5, LIMIT + 1, 7]) == [(0, 1), (1, 2), (2, 3)]
    assert functions.plan_ballquery_chunks([LIMIT + 1]) == [(0, 1)]
    assert functions.plan_ballquery_chunks([0, 0, 3 * LIMIT, 0, 2, LIMIT + 1]) == [(0, 2), (2, 3), (3, 5), (5, 6)]


def test_plan_preserves_segment_order():
    rng = np.random.RandomState(0)
    for trial in range(200):
        counts = rng.randint(0, 60, rng.randint(1, 80)) * (rng.rand() < 0.8)
        counts[rng.rand(counts.size) < 0.1] = 0
        cap = int(rng.randint(30, 300)) * 1000 + int(rng.randint(0, 1000))
        lim = cap // 1000
        chunks = functions.plan_ballquery_chunks(counts, cap)
        assert chunks[0][0] == 0 and chunks[-1][1] == counts.size
        for (a0, a1), (b0, b1) in zip(chunks, chunks[1:]):
            assert a1 == b0
        for k, (s0, s1) in enumerate(chunks):
            assert s1 > s0
            tot = int(counts[s0:s1].sum())
            if tot > lim:  # only an oversize segment, alone
                assert s1 - s0 == 1
            # greedy: the next segment would not have fit
            if k + 1 < len(chunks) and tot <= lim:
                assert tot + int(counts[s1]) > lim


def test_plan_reads_the_module_bound(monkeypatch):
    monkeypatch.setattr(functions, 'BALLQUERY_MAX_CAPACITY', 25999)
    assert functions.plan_ballquery_chunks([10, 15, 1, 30, 2]) == [(0, 2), (2, 3), (3, 4), (4, 5)]


# ---- forward_grouping chunked against one call ------------------------------------------------------------------
def _fake_ballquery_capacity(calls):
    def run(coords, batch_idxs, batch_offsets, radius, capacity=None):
        calls.append(capacity)
        return _fake_ballquery_nosync(coords, batch_idxs, batch_offsets, radius)
    return run


def _case(seed, batch):
    """test_host_grouping.py's many-segment scan: several classes, some under min_npoint, points in two classes."""
    model = SoftGroup(**model_cfg('scannet', channels=16, num_blocks=2, test_cfg=dict(min_npoint=30))).eval()
    parts = [synth.make_scan('c1_plumbing', seed=seed * 10 + b, n_points=1500) for b in range(batch)]
    scores, offs, coords, bidx = [], [], [], []
    for b, sc in enumerate(parts):
        s, o = synth.grouping_inputs(sc, sigma=0.03, seed=seed)
        rng = np.random.RandomState(seed)
        flip = rng.choice(s.shape[0], 60, replace=False)
        s[flip, rng.randint(2, 20, 60)] += 9.0
        scores.append(s)
        offs.append(o)
        coords.append(sc['coords_float'])
        bidx.append(np.full(s.shape[0], b, np.int32))
    args = [torch.from_numpy(np.concatenate(a)) for a in (scores, offs, bidx, coords)]
    return model, args


def _segments(model, args, batch):
    """Entry count and neighbour total of every segment (stand-in ops, as the forward computes them)."""
    g, get = model.grouping_cfg, model._cfg
    classes = model._grouped_classes(batch)
    pts, seg, shifted, seg_off, _ = _fake_group_entries(args[0].softmax(-1), classes, get(g, 'score_thr'),
                                                        get(model.test_cfg, 'min_npoint', 0), args[2], batch, args[3],
                                                        args[1])
    _, sl, _ = _fake_ballquery_nosync(shifted, seg, seg_off, get(g, 'radius'))
    counts = np.diff(seg_off.numpy())
    nbr = np.bincount(seg.numpy(), weights=sl[:, 1].numpy(), minlength=counts.size).astype(np.int64)
    return counts, nbr


def _run(monkeypatch, model, args, bound=None, planner=None):
    calls = []
    with monkeypatch.context() as m:
        m.setattr(sg_module, 'ballquery_batch_p_nosync', _fake_ballquery_capacity(calls))
        m.setattr(sg_module, 'bfs_cluster_segments', _fake_bfs_segments)
        m.setattr(sg_module, 'group_entries', _fake_group_entries)
        if bound is not None:
            m.setattr(functions, 'BALLQUERY_MAX_CAPACITY', bound)
        if planner is not None:
            m.setattr(functions, 'plan_ballquery_chunks', planner)
        idx, off = model.forward_grouping(*[a.clone() for a in args])
    return idx.numpy(), off.numpy(), calls


@pytest.mark.parametrize('seed,batch', [(0, 1), (1, 1), (2, 2)])
def test_chunked_equals_one_call(monkeypatch, seed, batch):
    model, args = _case(seed, batch)
    want_idx, want_off, calls = _run(monkeypatch, model, args)
    assert calls == [None], 'below the bound: one ball query, sized as before'
    assert want_off.size > 2
    counts, _ = _segments(model, args, batch)
    n = int(counts.sum())
    nonempty = int((counts > 0).sum())
    assert nonempty >= 3
    for parts in (2, 3):
        bound = -(-n // parts) * 1000
        chunks = functions.plan_ballquery_chunks(counts, bound)
        got_idx, got_off, calls = _run(monkeypatch, model, args, bound=bound)
        assert len([c for c in chunks if counts[c[0]:c[1]].sum() > 0]) == len(calls) >= parts
        assert np.array_equal(got_idx, want_idx) and np.array_equal(got_off, want_off)
    # one segment per chunk
    one = lambda c, cap=None: [(s, s + 1) for s in range(len(c))]  # noqa: E731
    got_idx, got_off, calls = _run(monkeypatch, model, args, bound=n * 1000 - 1, planner=one)
    assert len(calls) == nonempty
    assert np.array_equal(got_idx, want_idx) and np.array_equal(got_off, want_off)


def test_oversize_segment(monkeypatch):
    """Segments alone beyond the bound run with the bound as capacity: identical results when their neighbour totals
    fit, SgbError before that segment is clustered when one does not."""
    model, args = _case(0, 1)
    want_idx, want_off, _ = _run(monkeypatch, model, args)
    counts, nbr = _segments(model, args, 1)
    big = int(np.argmax(nbr))
    bound = int(nbr[big])
    assert (nbr == bound).sum() == 1 and counts[big] * 1000 > bound
    got_idx, got_off, calls = _run(monkeypatch, model, args, bound=bound)
    assert bound in calls  # the oversize segment ran with the largest buffer the bound allows
    assert np.array_equal(got_idx, want_idx) and np.array_equal(got_off, want_off)

    clustered = []

    def spy(*a, **k):
        clustered.append(a[1].shape[0])
        return _fake_bfs_segments(*a, **k)
    with monkeypatch.context() as m:
        m.setattr(sg_module, 'ballquery_batch_p_nosync', _fake_ballquery_capacity([]))
        m.setattr(sg_module, 'group_entries', _fake_group_entries)
        m.setattr(sg_module, 'bfs_cluster_segments', spy)
        m.setattr(functions, 'BALLQUERY_MAX_CAPACITY', bound - 1)
        with pytest.raises(SgbError, match='2\\^31 - 1'):
            model.forward_grouping(*[a.clone() for a in args])
    # the chunks before the oversize one were clustered, it and the ones after were not
    before = [(s0, s1) for s0, s1 in functions.plan_ballquery_chunks(counts, bound - 1) if s1 <= big]
    assert clustered == [int(counts[s0:s1].sum()) for s0, s1 in before if counts[s0:s1].sum() > 0]
