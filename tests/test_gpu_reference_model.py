"""Drop-in proof on hardware (SURVEY.md 8b, VERDICT round 1 row g1): the UNMODIFIED reference `SoftGroup` class
(softgroup/model/softgroup.py + blocks.py, staged verbatim into the git-ignored oracle/_ref/pyref by
oracle/build_ref.py) is instantiated on `softgroup_b200.install_as_reference_backends()` -- this repo's `spconv.pytorch`
and `softgroup.ops` -- moved to the GPU and called exactly like tools/test.py:145-152 does (`model(batch)` on the
dataloader's collated batch). Its result dict is compared with

  * this repo's restructured `softgroup_b200.model.SoftGroup` with the same weights on the same scan: proposals / masks
    (RLE strings) / labels identical, scores within 1e-4, point-wise outputs within 1e-4 relative;
  * for the plain config also with the reference-generated fixture tests/golden/ref_forward_c1.npz (the reference's
    own forward_test on CPU stand-ins).

The `scannet++` case runs the reference's own lvl_fusion / pyramid / octree code path (softgroup.py:309-312, 332-334,
427-463, 560-561) on the GPU ops -- the reference-order procedure for this repo's sparse lvl_fusion implementation.
`s3dis++` runs it with sem2ins classes: their instances are the per-point class masks taken through v2p_map
(:556-561). `stpls3d` runs the plain one-pass grouping with mean_active 3, so the reference's ball query regrows its
buffer (functions.py:258-265) on the shim's ballquery_batch_p."""
import os
import sys

import numpy as np
import pytest
import torch

from softgroup_b200 import harness, synth
from softgroup_b200.configs import SHAPE_OF, model_cfg
from softgroup_b200.model import SoftGroup

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, 'golden'))
from seeded_weights import CFG_OVERRIDES, SCAN, WEIGHT_SEED, fill_seeded, load_calibrated  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def ref_module():
    from oracle import build_ref
    from softgroup_b200.ops import functions as F
    m = build_ref.import_reference_model()
    if m is None:
        pytest.skip('neither /root/reference nor oracle/_ref/pyref is present (run __graft_entry__.build() first)')
    # install_as_reference_backends(torch2_compat=True): softgroup.py:570 indexes a CPU tensor with a CUDA mask, which the
    # PyTorch 1.x of the reference accepted and PyTorch >= 2 does not
    F.TORCH2_COMPAT = True
    yield m
    F.TORCH2_COMPAT = False


class _Cfg(dict):
    """Attribute access on nested config dicts (the reference reads `self.test_cfg.x4_split`, `self.grouping_cfg.radius`:
    tools/test.py builds its configs with Munch)."""
    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError:
            raise AttributeError(name)

    @classmethod
    def wrap(cls, d):
        return cls({k: (cls.wrap(v) if isinstance(v, dict) else v) for k, v in d.items()})


def _pair(ref_module, cfg, calibrated=None, scan=None):
    ours = SoftGroup(**cfg).eval()
    fill_seeded(ours, WEIGHT_SEED)
    if calibrated is not None:
        load_calibrated(ours, calibrated)
    ours = ours.cuda()
    if calibrated is None:
        harness.calibrate_heads(ours, harness.to_host_batch(scan))
    ref = ref_module.SoftGroup(**_Cfg.wrap(cfg))
    ref.eval()  # the reference overrides train() without returning self (softgroup.py:98-104): no chaining
    ref.load_state_dict(ours.state_dict(), strict=True)  # identical names and shapes: checkpoints load unchanged
    return ours, ref.cuda()


def _compare(a, b, n_points, rel=1e-4):
    """a: reference class result, b: this repo's result."""
    assert set(a.keys()) == set(b.keys())
    assert a['scan_id'] == b['scan_id']
    for k in ('semantic_labels', 'instance_labels', 'coords_float', 'color_feats', 'offset_labels', 'gt_instances'):
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k
    off_a, off_b = np.asarray(a['offset_preds']), np.asarray(b['offset_preds'])
    assert np.abs(off_a - off_b).max() <= rel * max(np.abs(off_a).max(), 1e-6)
    sp_a, sp_b = np.asarray(a['semantic_preds']), np.asarray(b['semantic_preds'])
    assert (sp_a != sp_b).mean() <= 1e-3  # argmax of scores that agree to 1e-4: ties may flip on a handful of points
    ia, ib = a['pred_instances'], b['pred_instances']
    assert len(ia) == len(ib) and len(ia) > 0
    for x, y in zip(ia, ib):
        assert x['scan_id'] == y['scan_id'] and x['label_id'] == y['label_id']
        assert x['pred_mask']['length'] == n_points == y['pred_mask']['length']
        assert x['pred_mask']['counts'] == y['pred_mask']['counts']
        assert abs(float(x['conf']) - float(y['conf'])) <= rel * max(1.0, abs(float(y['conf'])))
    return len(ia)


def test_reference_class_runs_on_b200_and_matches(ref_module):
    gold = np.load(os.path.join(HERE, 'golden', 'ref_forward_c1.npz'), allow_pickle=True)
    cfg = model_cfg('scannet', **CFG_OVERRIDES)
    ours, ref = _pair(ref_module, cfg, calibrated=gold['calibrated'])
    scan = synth.make_scan(SCAN['shape'], seed=SCAN['seed'])
    batch = harness.collate_like_reference(scan)  # the reference dataloader's output (CPU hashing, custom.py:239)
    with torch.no_grad():
        r_ref = ref(dict(batch))  # tools/test.py:148 `result = model(batch)`
        r_our = ours(dict(batch))
    n = _compare(r_ref, r_our, scan['coords'].shape[0])
    # and both equal the reference's own CPU run (fixture): same number of instances, same masks
    assert n == len(gold['inst_rle'])
    assert [x['pred_mask']['counts'] for x in r_ref['pred_instances']] == [str(x) for x in gold['inst_rle']]
    assert [int(x['label_id']) for x in r_ref['pred_instances']] == [int(x) for x in gold['inst_label_id']]
    conf = np.array([float(x['conf']) for x in r_ref['pred_instances']])
    assert np.abs(conf - gold['inst_conf']).max() <= 2e-4 * max(1.0, np.abs(gold['inst_conf']).max())


# grouping thresholds that give proposals on a random-weight (calibrated-head) model: the yaml values (thresholds relative
# to the real datasets' class sizes) select nothing there -- both models returned 0 instances
GROUPING_OVERRIDES = {
    'scannet': (dict(radius=0.15, class_numpoint_mean=[-1.] * 20, npoint_thr=100), dict(min_npoint=50)),
    'scannet++': (dict(radius=0.15, class_numpoint_mean=[-1.] * 20, npoint_thr=100), dict(min_npoint=50)),
    's3dis++': (dict(radius=0.15, class_numpoint_mean=[-1.] * 13, npoint_thr=20), dict(min_npoint=20)),
    'stpls3d': (dict(radius=1.5, class_numpoint_mean=[-1.] * 15, npoint_thr=5), dict(min_npoint=5)),
}


@pytest.mark.parametrize('name,n_points', [('scannet', 30000), ('scannet++', 20000), ('s3dis++', 20000),
                                           ('stpls3d', 20000)])
def test_reference_class_vs_restructured_forward(ref_module, name, n_points):
    """Full-size model (7 levels) on a scan of the config's own shape; 'scannet++' and 's3dis++' = pyramid + octree +
    lvl_fusion at test time, 's3dis++' with sem2ins classes, 'stpls3d' = one-pass grouping at mean_active 3."""
    grouping, test = GROUPING_OVERRIDES[name]
    cfg = model_cfg(name, grouping_cfg=grouping, test_cfg=test)
    scan = synth.make_scan(SHAPE_OF[name], seed=5, n_points=n_points)
    ours, ref = _pair(ref_module, cfg, scan=scan)
    batch = harness.collate_like_reference(scan)
    with torch.no_grad():
        r_ref = ref(dict(batch))
        r_our = ours(dict(batch))
    _compare(r_ref, r_our, n_points)
    if cfg['sem2ins_classes']:
        labels = [int(x['label_id']) for x in r_ref['pred_instances']]
        assert set(labels) & {i + 1 for i in cfg['sem2ins_classes']}, labels
        assert set(labels) - {i + 1 for i in cfg['sem2ins_classes']}, labels
