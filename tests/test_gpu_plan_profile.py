"""The compiled U-Net plan run one launch per call (SoftGroup.use_plan = False, the per-op instrumented pass of bench.py):
one profiler record per plan op, named like the module path's launch and carrying the same algorithmic bytes."""
from collections import Counter

import numpy as np
import pytest
import torch

from oracle import spconv_oracle as so
from softgroup_b200 import profiler, spconv, synth
from softgroup_b200.configs import model_cfg
from softgroup_b200.model import SoftGroup
from softgroup_b200.model.unet_plan import ACT_PACK, BN_RELU, CONV

pytestmark = pytest.mark.gpu


def test_per_launch_plan_records_one_event_per_op():
    import oracle
    torch.manual_seed(0)
    scan = synth.make_scan('c2_scannet', seed=1, n_points=30000)
    vc, _, p2v = oracle.voxelization_idx(scan['coords'], 1, 4)
    feats = np.concatenate([scan['feats'], scan['coords_float']], 1).astype(np.float32)
    vfeats = oracle.voxelization(feats, p2v, 4)
    idx = vc.astype(np.int32)
    model = SoftGroup(**model_cfg('scannet', channels=32, num_blocks=7)).cuda().eval()
    model.use_plan = False
    x = spconv.SparseConvTensor(torch.from_numpy(vfeats).cuda(), torch.from_numpy(idx).cuda(), scan['spatial_shape'], 1)
    profiler.reset()
    profiler.enable()
    try:
        with torch.no_grad():
            model._run_stack('backbone', model.input_conv, model.unet, model.output_layer, x)
        torch.cuda.synchronize()
    finally:
        profiler.disable()
        recs = [(name, nbytes) for name, nbytes, _, _ in profiler._records]
        profiler.reset()
    plan = model._plans['backbone'][1]

    # row count of every U-Net level, from the numpy restatement of the strided rulebook
    M, shape = [len(idx)], scan['spatial_shape']
    for _ in range(6):
        idx, _, _, shape = so.down_map(idx, shape)
        M.append(len(idx))

    want = []
    for d in plan.ops:
        Min, Mout = M[d['level_in']], M[d['level_out']]
        if d['kind'] == CONV:
            has_map = d['map_kind'] != 0
            want.append(('spconv_tc_kernel' if has_map else 'spconv_tc_kernel(1x1/linear)',
                         spconv.core.conv_bytes(Min, Mout, d['K'], d['Cin'], d['Cout'], has_map, d['res_buf'] >= 0)))
        else:
            assert d['kind'] in (ACT_PACK, BN_RELU)
            want.append(('act_pack' if d['kind'] == ACT_PACK else 'bn_relu', 8 * Min * d['Cin']))
    got = [r for r in recs if not r[0].startswith('rulebook_')]
    assert got == want
    # 53 SubM + 6 strided + 6 inverse, six 1x1 skips, 13 packs (input, 1x1 skip inputs, encoder halves of the concat
    # buffers), the output BatchNorm+ReLU; seven subm and six strided rulebooks; no whole-segment record
    assert Counter(r[0] for r in recs) == {'spconv_tc_kernel': 65, 'spconv_tc_kernel(1x1/linear)': 6, 'act_pack': 13,
                                           'bn_relu': 1, 'rulebook_subm3': 7, 'rulebook_down2': 6}
