"""Host-side methods of the model against the REFERENCE'S OWN methods: what the unmodified reference SoftGroup class
(instantiated on this repo's shims, CPU) returns for the inputs below is stored in tests/golden/ref_host_methods.npz
(tests/golden/make_reference_golden.py) -- panoptic_fusion (softgroup.py:606-639), get_gt_instances (:641-653),
merge_4_parts (:397-409), pyramid_inverse_map (:500-507, dense matrix), get_level (:482-489)."""
import os
import types

import numpy as np
import pytest
import torch

from softgroup_b200.configs import model_cfg
from softgroup_b200.model import SoftGroup
from softgroup_b200.util import rle_encode

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_host_methods.npz')
LEVEL_SIZES = (5, 100000, 100001, 1000000, 1000001)


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLDEN)


def _cfg(name):
    return model_cfg(name, channels=16, num_blocks=2)


def reference_instance(ref_model_module, name):
    """The reference class as the fixture generator instantiates it."""
    cfg = _cfg(name)
    ref = ref_model_module.SoftGroup(**cfg)
    ref.eval()  # the reference's train() override does not return self
    ref.test_cfg = types.SimpleNamespace(**cfg['test_cfg'])  # the reference reads attributes (Munch in tools/test.py)
    ref.grouping_cfg = types.SimpleNamespace(**cfg['grouping_cfg'])
    return ref


def _ours(name):
    return SoftGroup(**_cfg(name)).eval()


def panoptic_case(seed):
    rng = np.random.RandomState(seed)
    n = 800
    sem = rng.randint(0, 19, n)
    insts = []
    for _ in range(15):
        lo = rng.randint(0, n - 60)
        m = np.zeros(n, np.int64)
        m[lo:lo + rng.randint(5, 60)] = rng.rand() < 0.9  # overlapping runs -> the skip rule triggers
        insts.append(dict(scan_id='s', label_id=int(rng.randint(1, 9)), conf=float(rng.rand()), pred_mask=rle_encode(m)))
    return sem, insts


def gt_instances_case():
    rng = np.random.RandomState(0)
    sem = torch.from_numpy(rng.randint(-1, 20, 500)).long()
    sem[sem == -1] = -100
    inst = torch.from_numpy(rng.randint(-1, 12, 500)).long()
    inst[inst == -1] = -100
    return sem, inst


def merge_case():
    return torch.arange(4 * 7 * 3, dtype=torch.float32).view(28, 3)


def pyramid_case():
    rng = np.random.RandomState(1)
    n_vox, n_pts = 60, 400
    l2p = torch.from_numpy(rng.randint(0, n_vox, n_pts).astype(np.int32))
    members = rng.permutation(n_vox)[:45]  # a voxel belongs to at most one cluster
    cut = [0, 10, 11, 30, 45]
    pidx = torch.tensor([[c, int(v)] for c in range(4) for v in members[cut[c]:cut[c + 1]]], dtype=torch.int32)
    poff = torch.tensor(cut, dtype=torch.int32)
    return pidx, poff, n_vox, l2p


@pytest.mark.parametrize('seed', range(3))
def test_panoptic_fusion(gold, seed):
    sem, insts = panoptic_case(seed)
    want = gold['panoptic_fusion_%d' % seed]
    got = _ours('kitti').panoptic_fusion(sem.copy(), insts)
    assert got.dtype == want.dtype and np.array_equal(got, want)


def test_get_gt_instances(gold):
    sem, inst = gt_instances_case()
    got = _ours('scannet').get_gt_instances(sem.clone(), inst.clone())
    assert np.array_equal(got, gold['get_gt_instances'])


def test_merge_4_parts(gold):
    assert torch.equal(_ours('s3dis').merge_4_parts(merge_case()), torch.from_numpy(gold['merge_4_parts']))


def test_pyramid_inverse_map_and_level(gold):
    ours = _ours('stpls3d++')
    assert [ours.get_level(n) for n in LEVEL_SIZES] == gold['get_level'].tolist()
    got_idx, got_off = ours.pyramid_inverse_map(*pyramid_case())
    assert np.array_equal(got_idx.numpy(), gold['pyramid_inverse_map_idx'].astype(np.int32))
    assert np.array_equal(got_off.numpy(), gold['pyramid_inverse_map_offset'])
