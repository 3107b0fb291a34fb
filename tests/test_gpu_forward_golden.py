"""The CUDA forward against the reference-generated fixture tests/golden/ref_forward_c1.npz (the reference's own
`forward_test`, softgroup/model/softgroup.py:300-361, run on CPU stand-ins by tests/golden/make_forward_golden.py):
backbone + heads, then grouping / clusters_voxelization / tiny U-Net / instance heads from the fixture's
intermediates."""
import os
import sys

import numpy as np
import pytest
import torch

from softgroup_b200 import spconv, synth
from softgroup_b200.configs import model_cfg
from softgroup_b200.model import SoftGroup
from softgroup_b200.ops import voxelization, voxelization_idx

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
from seeded_weights import CFG_OVERRIDES, SCAN, WEIGHT_SEED, fill_seeded, load_calibrated, weights_digest  # noqa: E402

pytestmark = pytest.mark.gpu
REL = 2e-4  # float outputs, relative to the largest magnitude of the golden array (north star: 1e-4 per feature scale)


def _close(got, want, rel=REL):
    want = np.asarray(want)
    return np.abs(got - want).max() <= rel * max(1e-6, np.abs(want).max())


@pytest.fixture(scope='module')
def gold():
    return np.load(os.path.join(HERE, 'golden', 'ref_forward_c1.npz'))


@pytest.fixture(scope='module')
def model(gold):
    m = SoftGroup(**model_cfg('scannet', **CFG_OVERRIDES)).eval()
    fill_seeded(m, WEIGHT_SEED)
    load_calibrated(m, gold['calibrated'])
    assert weights_digest(m) == int(gold['weights_digest'])
    return m.cuda()


def test_backbone_and_heads(gold, model):
    scan = synth.make_scan(SCAN['shape'], seed=SCAN['seed'])
    coords = torch.from_numpy(scan['coords']).cuda()
    vc, v2p, p2v = voxelization_idx(coords, 1)
    assert np.array_equal(vc.cpu().numpy(), gold['voxel_coords']) and np.array_equal(v2p.cpu().numpy(), gold['v2p_map'])
    feats = torch.cat((torch.from_numpy(scan['feats']), torch.from_numpy(scan['coords_float'])), 1).cuda()
    vf = voxelization(feats.contiguous(), p2v.contiguous())
    assert np.array_equal(vf.cpu().numpy(), gold['voxel_feats'])
    x = spconv.SparseConvTensor(vf, vc.int(), scan['spatial_shape'], 1)
    with torch.no_grad():
        sem, off, ofeat = model.forward_backbone(x, v2p)
    assert _close(ofeat.cpu().numpy(), gold['output_feats'])
    assert _close(sem.cpu().numpy(), gold['semantic_scores'])
    assert _close(off.cpu().numpy(), gold['pt_offsets'])


def test_grouping_and_instance_branch_from_golden_intermediates(gold, model):
    scan = synth.make_scan(SCAN['shape'], seed=SCAN['seed'])
    n = gold['semantic_scores'].shape[0]
    cf = torch.from_numpy(scan['coords_float']).cuda()
    with torch.no_grad():
        pidx, poff = model.forward_grouping(torch.from_numpy(gold['semantic_scores']).cuda(),
                                            torch.from_numpy(gold['pt_offsets']).cuda(),
                                            torch.zeros(n, dtype=torch.int32, device='cuda'), cf)
        assert np.array_equal(pidx.cpu().numpy(), gold['proposals_idx'])
        assert np.array_equal(poff.cpu().numpy(), gold['proposals_offset'])
        inst_feats, inst_map = model.clusters_voxelization(pidx, poff, torch.from_numpy(gold['output_feats']).cuda(), cf,
                                                           **model._voxel_cfg())
        assert np.array_equal(inst_feats.indices.cpu().numpy(), gold['inst_voxel_coords'])
        assert np.array_equal(inst_map.cpu().numpy(), gold['inst_map'])
        assert np.array_equal(inst_feats.features.cpu().numpy(), gold['inst_voxel_feats'])
        _, cls_s, iou_s, mask_s = model.forward_instance(inst_feats, inst_map)
    assert _close(cls_s.cpu().numpy(), gold['cls_scores'])
    assert _close(iou_s.cpu().numpy(), gold['iou_scores'])
    assert _close(mask_s.cpu().numpy(), gold['mask_scores'])
