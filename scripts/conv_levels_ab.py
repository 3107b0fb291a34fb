"""Per-level timing of one SubM 3x3x3 convolution (C_l -> C_l) on the rulebooks of the 150k-point bench scan (tensor-core
kernel; --morton puts the rows in Z-order first). L2 is flushed before every timed launch; the packed
input is prepared outside the timed region so the number is the conv kernel alone.
Usage: python scripts/conv_levels_ab.py [impl ...]"""
import sys

import numpy as np
import torch

sys.path.insert(0, '.')
from softgroup_b200 import ops, synth  # noqa: E402
from softgroup_b200.spconv import core  # noqa: E402
from softgroup_b200.ops import _lib  # noqa: E402
from softgroup_b200.ops._lib import check, ptr  # noqa: E402

impls = ['tc']
ORDER = 'morton' if '--morton' in sys.argv else 'orig'


def part1by2(v):
    v = v & 0x1fffff
    v = (v | (v << 32)) & 0x1f00000000ffff
    v = (v | (v << 16)) & 0x1f0000ff0000ff
    v = (v | (v << 8)) & 0x100f00f00f00f00f
    v = (v | (v << 4)) & 0x10c30c30c30c30c3
    v = (v | (v << 2)) & 0x1249249249249249
    return v
scan = synth.make_scan('c2_scannet', seed=0)
coords = torch.from_numpy(scan['coords']).cuda()
vc, v2p, p2v = ops.voxelization_idx(coords, 1)
idx = vc.int().contiguous()
if ORDER == 'morton':  # rows in Z-order: a 128-row tile is a compact blob, its 27-neighbourhoods overlap
    c = idx.long()
    key = (c[:, 0] << 60) | part1by2(c[:, 1]) | (part1by2(c[:, 2]) << 1) | (part1by2(c[:, 3]) << 2)
    idx = idx[torch.argsort(key)].contiguous()
print('row order:', ORDER, flush=True)
shape = [int(s) for s in scan['spatial_shape']]
flush = torch.empty(512 << 20, dtype=torch.uint8, device='cuda')
L = _lib.lib()
levels = []
for lvl in range(7):
    C = 32 * (lvl + 1)
    mp = core.build_subm_map(idx)
    levels.append((lvl, C, idx.size(0), mp))
    if lvl < 6:
        idx, _, _, shape = core.build_down_map(idx, shape)

torch.manual_seed(0)
for lvl, C, M, mp in levels:
    x = torch.randn(M, C, device='cuda')
    W = core.WeightPack((torch.randn(27, C, C, device='cuda') / (27 * C) ** 0.5).contiguous())
    nnz = int((mp >= 0).sum())
    line = 'level %d  M %6d  C %3d  pairs/row %.1f |' % (lvl, M, C, nnz / M)
    outs = {}
    for impl in impls:
        out = torch.empty(M, C, device='cuda')
        pk = core.act_pack(x, C, 0, C)

        def run():
            check(L.sgb_spconv_forward_tc(ptr(pk), C, M, ptr(mp), 27, M, ptr(W.tc()), C, C, None, 0, 0, None, ptr(out), C, 0,
                                          None, 0, 0, None, None, 0, 0, core._stream()))
        for _ in range(2):
            run()
        ts = []
        for _ in range(5):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            run()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1) * 1e3)
        outs[impl] = out.clone()
        gathered = nnz * C * 4 / 1e9
        line += ' %s %.1f us (%.2f TB/s gathered)' % (impl, float(np.median(ts)), gathered / (np.median(ts) * 1e-6) / 1e3)
    if len(impls) == 2:
        a, b = outs[impls[0]], outs[impls[1]]
        line += ' | max rel diff %.2e' % float((a - b).abs().max() / a.abs().max())
    print(line, flush=True)
