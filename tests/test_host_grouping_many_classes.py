"""forward_grouping with ScanNet200's class count (198 grouped classes) on CPU, against the reference's per-class loop
(softgroup/model/softgroup.py:411-480), with the device ops replaced by the oracle stand-ins of test_host_grouping.py;
and the batch-size limit of the one-pass grouping (every (class, batch item) pair is one ball-query segment)."""
import numpy as np
import pytest
import torch

from softgroup_b200 import synth
from softgroup_b200.configs import model_cfg
from softgroup_b200.model import SoftGroup
from softgroup_b200.model import softgroup as sg_module
from softgroup_b200.ops import BALLQUERY_MAX_SEGMENTS
from test_host_grouping import _fake_ballquery_nosync, _fake_bfs_segments, _fake_group_entries, reference_forward_grouping


def _scannet200(**test_cfg):
    return SoftGroup(**model_cfg('scannet200', channels=16, num_blocks=2, test_cfg=test_cfg)).eval()


def test_scannet200_config():
    cfg = model_cfg('scannet200')
    g = cfg['grouping_cfg']
    assert cfg['semantic_classes'] == 200 and cfg['instance_classes'] == 198
    assert g['ignore_classes'] == [0, 1] and len(g['class_numpoint_mean']) == 200
    assert cfg['channels'] == 32 and cfg['num_blocks'] == 7
    sc = synth.make_scan('c6_scannet200', seed=0, n_points=20000)
    # one object of every grouped class
    assert sorted(set(sc['instance_cls'].tolist())) == list(range(2, 200))


@pytest.mark.parametrize('seed,batch,confusion', [(0, 1, 0.0), (1, 1, 0.3), (2, 2, 0.3)])
def test_forward_grouping_200_classes_equals_reference_loop(monkeypatch, seed, batch, confusion):
    monkeypatch.setattr(sg_module, 'ballquery_batch_p_nosync', _fake_ballquery_nosync)
    monkeypatch.setattr(sg_module, 'bfs_cluster_segments', _fake_bfs_segments)
    monkeypatch.setattr(sg_module, 'group_entries', _fake_group_entries)
    model = _scannet200(min_npoint=30)
    scores, offs, coords, bidx = [], [], [], []
    for b in range(batch):
        sc = synth.make_scan('c6_scannet200', seed=seed * 10 + b, n_points=40000)
        s, o = synth.grouping_inputs(sc, sigma=0.01, seed=seed, confusion=confusion)
        scores.append(s)
        offs.append(o)
        coords.append(sc['coords_float'])
        bidx.append(np.full(s.shape[0], b, np.int32))
    scores, offs, coords, bidx = map(np.concatenate, (scores, offs, coords, bidx))
    got_idx, got_off = model.forward_grouping(torch.from_numpy(scores), torch.from_numpy(offs), torch.from_numpy(bidx),
                                              torch.from_numpy(coords))
    want_idx, want_off = reference_forward_grouping(model, scores, offs, bidx, coords)
    # proposals of more than 32 classes: the case the one-pass grouping could not take before
    sem = scores.argmax(1)
    assert len(set(sem[want_idx[want_off[1:] - 1, 1]].tolist())) > 32
    assert got_idx.dtype == torch.int32 and got_off.dtype == torch.int32
    assert np.array_equal(got_idx.numpy(), want_idx)
    assert np.array_equal(got_off.numpy(), want_off)


def _no_device_op(*a, **k):
    raise AssertionError('the grouping must not start')


@pytest.mark.parametrize('batch', [5, 6])
def test_segment_limit_raises_before_grouping(monkeypatch, batch):
    """198 classes: 5 scans per batch give 990 segments (accepted), 6 give 1188 (a ValueError before any device op)."""
    model = _scannet200(min_npoint=30)
    n = 64
    scores = torch.zeros(n, 200)
    args = (scores, torch.zeros(n, 3), torch.arange(n, dtype=torch.int32) % batch, torch.zeros(n, 3))
    if batch * 198 <= BALLQUERY_MAX_SEGMENTS:
        assert model._grouped_classes(batch) == list(range(2, 200))
        monkeypatch.setattr(sg_module, 'group_entries', _fake_group_entries)
        idx, off = model.forward_grouping(*args, batch_size=batch)  # scores 0.005 < score_thr: nothing is grouped
        assert idx.shape == (0, 2) and off.numel() == 0
        return
    monkeypatch.setattr(sg_module, 'group_entries', _no_device_op)
    monkeypatch.setattr(sg_module, 'ballquery_batch_p_nosync', _no_device_op)
    with pytest.raises(ValueError, match='1188 ball-query segments'):
        model.forward_grouping(*args, batch_size=batch)
    # forward_test checks it before the backbone runs
    monkeypatch.setattr(model, 'forward_backbone', _no_device_op)
    with pytest.raises(ValueError, match='run at most 5 scans per batch'):
        model.forward_test(batch_idxs=None, voxel_coords=None, p2v_map=None, v2p_map=None, coords_float=None, feats=None,
                           batch_size=batch, device_only=True)


def test_segment_limit_leaves_pyramid_grouping_alone():
    """SoftGroup++ groups class by class (one ball query per class): no segment limit from the class count."""
    cfg = model_cfg('scannet200', channels=16, num_blocks=2)
    cfg['grouping_cfg'].update(with_pyramid=True, with_octree=True)
    model = SoftGroup(**cfg).eval()
    assert len(model._grouped_classes(8)) == 198
