"""csrc/grouping.cu at any class count, on the GPU: group_entries against the reference's per-class loop
(softgroup.py:430-446, the CPU stand-in of test_host_grouping.py) element by element, and the unmodified reference
`SoftGroup` class against this repo's forward on a ScanNet200-shape scan (200 semantic classes, 198 grouped)."""
import numpy as np
import pytest
import torch

from softgroup_b200 import harness, synth
from softgroup_b200.configs import model_cfg
from softgroup_b200.ops import _lib, group_entries
from test_gpu_reference_model import _compare, _pair, ref_module  # noqa: F401 (ref_module: fixture)
from test_host_grouping import _fake_group_entries

pytestmark = pytest.mark.gpu


def _case(n, C, batch, seed, thr_scale=2.0):
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(n, C, generator=g) * thr_scale
    logits[:, C - 2] -= 6  # a rare class: falls below min_npoint
    scores = logits.softmax(-1)
    bsz = torch.sort(torch.randint(0, batch, (n, ), generator=g))[0].int()
    coords, offs = torch.randn(n, 3, generator=g), torch.randn(n, 3, generator=g) * 0.1
    return scores, bsz, coords, offs


def _check(scores, classes, thr, min_npoint, bsz, batch, coords, offs):
    want = _fake_group_entries(scores, classes, thr, min_npoint, bsz, batch, coords, offs)
    got = group_entries(scores.cuda(), classes, thr, min_npoint, bsz.cuda(), batch, coords.cuda(), offs.cuda())
    tot = got[4].cpu()
    assert torch.equal(tot, want[4])
    m = int(tot[0])
    assert torch.equal(got[0][:m].cpu(), want[0]) and torch.equal(got[1][:m].cpu(), want[1])
    assert torch.equal(got[2][:m].cpu(), want[2])
    assert torch.equal(got[3].cpu(), want[3])
    return want


@pytest.mark.parametrize('nc', [1, 31, 32, 33, 64, 198, 200])
@pytest.mark.parametrize('batch', [1, 2])
def test_group_entries_any_class_count(nc, batch):
    """C = 200 score columns, the last nc of them grouped; N = 30001 (not a multiple of 256); one class dropped by
    min_npoint; softmax over 200 logits of scale 3 with score_thr 0.02, so that points pass several classes at once."""
    n, C = 30001, 200
    scores, bsz, coords, offs = _case(n, C, batch, seed=nc * 10 + batch, thr_scale=3.0)
    classes = list(range(C - nc, C))
    want = _check(scores, classes, 0.02, 40, bsz, batch, coords, offs)
    per_class = want[4][1:]
    if nc > 1:
        assert int((per_class == 0).sum()) >= 1  # the rare class is dropped
    if nc > 2:
        multi = (scores[:, classes] > 0.02).sum(1)
        assert int(multi.max()) >= 3  # some points pass three classes or more


@pytest.mark.parametrize('n', [1, 255, 257, 150000])
def test_group_entries_200_classes_sizes(n):
    """ScanNet200's 198 grouped classes at the edges of the 256-point blocks and at the 150k-point scan size."""
    scores, bsz, coords, offs = _case(n, 200, 1, seed=n)
    _check(scores, list(range(2, 200)), 0.02, 0, bsz, 1, coords, offs)


def test_group_entries_class_order_and_slices():
    """Classes in any order and any count: 300 of 320 columns, shuffled and with a repeated column, take two class-id
    slices (256 per count launch); ranks follow the list, not the column."""
    n, C = 20000, 320
    scores, bsz, coords, offs = _case(n, C, 2, seed=7, thr_scale=3.0)
    rng = np.random.RandomState(0)
    classes = [int(c) for c in rng.permutation(C)[:299]] + [5]
    _check(scores, classes, 0.01, 10, bsz, 2, coords, offs)


def test_group_entries_launches():
    """4 launches for up to 256 classes (the 20-class configs included), one more per further 256 class ids."""
    scores, bsz, coords, offs = [t.cuda() for t in _case(5000, 520, 1, seed=1)]
    L = _lib.lib()
    for nc, launches in ((18, 4), (198, 4), (256, 4), (257, 5), (520, 6)):
        l0 = L.sgb_launch_count()
        group_entries(scores, list(range(nc)), 0.2, 0, bsz, 1, coords, offs)
        assert L.sgb_launch_count() - l0 == launches, nc
    torch.cuda.synchronize()


def test_reference_class_vs_restructured_forward_200_classes(ref_module):  # noqa: F811
    """The reference's own per-class loop (softgroup.py:427-446) runs 198 times; this repo's forward groups them in one
    pass. Full-size model (32 channels x 7 levels), ScanNet200-shape scan with one object of every grouped class."""
    cfg = model_cfg('scannet200', grouping_cfg=dict(radius=0.15, class_numpoint_mean=[-1.] * 200, npoint_thr=50,
                                                    score_thr=0.1),
                    test_cfg=dict(min_npoint=50))
    n_points = 100000
    scan = synth.make_scan('c6_scannet200', seed=5, n_points=n_points)
    ours, ref = _pair(ref_module, cfg, scan=scan)
    # the heads' fit with the default target logit (6) leaves the softmax over 200 classes too flat for score_thr: fit
    # to a larger one (the same fit scaled, same argmax) and hand the weights to the reference class again
    harness.calibrate_heads(ours, harness.to_host_batch(scan), logit=30.0)
    ref.load_state_dict(ours.state_dict(), strict=True)
    batch = harness.collate_like_reference(scan)
    with torch.no_grad():
        r_ref = ref(dict(batch))
        r_our = ours(dict(batch))
    n = _compare(r_ref, r_our, n_points)
    labels = {int(x['label_id']) for x in r_our['pred_instances']}
    print('instances %d of %d classes' % (n, len(labels)))
