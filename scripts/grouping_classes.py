"""Grouping cost against the class count on the 150k-point scan: ScanNet (20 semantic classes, 18 grouped, c2_scannet)
and ScanNet200 (200 / 198, c6_scannet200), the bench protocol (random-init model, synthetic point-wise predictions
injected after the backbone).

Per config it reports
  * `grouping_stage_ms`: the `grouping` stage of SoftGroup.profile_stages (CUDA events from the end of the backbone to the
    end of forward_grouping: selection, ball query, clustering and the host reads in between), one forward per step;
  * `group_entries_kernel_us`: the summed device time of the group_entries kernels per call (torch.profiler, CUDA
    activity, a separate run of `--steps` calls on the scores the forward groups), per kernel and in all;
  * `algorithmic_bytes` = 4*N*C + 28*N (scores once; batch index, coordinates and offsets once) and that over the kernel
    time. The GPU's name, power limit and max SM clock are read in the same run.

    python scripts/grouping_classes.py [--steps 30] [--configs scannet scannet200] [--out result.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
from softgroup_b200 import harness, synth  # noqa: E402
from softgroup_b200.configs import SHAPE_OF, model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402
from softgroup_b200.ops import group_entries  # noqa: E402

N_POINTS = 150000


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    lines = q.stdout.strip().splitlines()
    return lines[torch.cuda.current_device()] if q.returncode == 0 and lines else torch.cuda.get_device_name()


def stats(xs):
    xs = np.asarray(xs, np.float64)
    return dict(median=round(float(np.median(xs)), 4), min=round(float(xs.min()), 4), max=round(float(xs.max()), 4))


@torch.no_grad()
def measure(name, steps):
    cfg = model_cfg(name)
    g = cfg['grouping_cfg']
    classes = [c for c in range(cfg['semantic_classes']) if c not in g['ignore_classes']]
    torch.manual_seed(0)
    model = SoftGroup(**cfg).cuda().eval()
    scan = synth.make_scan(SHAPE_OF[name], seed=0, n_points=N_POINTS)
    inj = harness.pointwise_injection(scan, sigma=0.03, seed=0)
    dev = harness.device_batch(harness.to_host_batch(scan))
    dev.pop('coords')

    def step():
        return model.forward_test(device_only=True, inject_pointwise=inj, **dev)

    for _ in range(3):
        ret = step()
    torch.cuda.synchronize()
    model.profile_stages = True
    stage = []
    for _ in range(steps):
        step()  # synchronises at its end under profile_stages
        stage.append(model.stage_ms['grouping'])
    model.profile_stages = False

    # the call forward_grouping makes, on the same inputs
    scores = inj[0].softmax(dim=-1)
    N, C = scores.shape
    args = (scores, classes, g['score_thr'], cfg['test_cfg']['min_npoint'], dev['batch_idxs'], 1, dev['coords_float'],
            inj[1])
    for _ in range(5):
        total = group_entries(*args)[4]
    entries = int(total[0])
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            group_entries(*args)
        torch.cuda.synchronize()
    kernels = {}
    for e in prof.key_averages():
        if 'ge_' in e.key and e.device_time_total > 0:
            kernels[e.key.split('(')[0]] = dict(us_per_call=round(e.device_time_total / steps, 2), launches=e.count // steps)
    kern_us = sum(k['us_per_call'] for k in kernels.values())
    nbytes = 4 * N * C + 28 * N
    po = ret['proposals_offset']
    return dict(config=name, shape=SHAPE_OF[name], N=N, C=C, grouped_classes=len(classes), entries=entries,
                classes_with_entries=int((total[1:] > 0).sum()), proposals=int(po.numel() - 1) if po.numel() else 0,
                grouping_stage_ms=stats(stage), group_entries_kernel_us=round(kern_us, 2), kernels=kernels,
                algorithmic_bytes=nbytes, gbs=round(nbytes / (kern_us * 1e-6) / 1e9, 1) if kern_us > 0 else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--configs', nargs='+', default=['scannet', 'scannet200'])
    ap.add_argument('--out', default=None, help='also write the result as JSON here')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'grouping_classes.py measures on the GPU (no CPU fallback)'
    res = dict(gpu=card(), steps=a.steps, results=[measure(n, a.steps) for n in a.configs])
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
