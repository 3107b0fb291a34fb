"""Time of instance_point_reduce and instance_point_map on the device results of bench workloads.

For each workload the device_results forward runs once; then each call is timed with CUDA events over --reps calls after
a warm-up: the reduction (min, max, mean) of coords_float (C = 3) and of a random [N, 32] tensor, and the point map.
Achieved bandwidth counts the algorithmic bytes of DESIGN.md section 3 (8(n+1) + 4 total + 4 C total + 4 C n ops for the
reduction; offsets, confidences, ids, the 8-byte key per point zeroed, updated and decoded, and the map for the point
map: the atomics on the keys land in L2) and is
given as a share of the H100 SXM data-sheet 3.35 TB/s. The card's name and power limit are read in the same run.
Usage: python scripts/instance_reduce.py [--workloads c2,c5] [--reps 50] [--out FILE.json]"""
import argparse
import json
import subprocess
import sys

import torch

sys.path.insert(0, '.')
import bench  # noqa: E402
from softgroup_b200 import harness, synth  # noqa: E402
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402
from softgroup_b200.ops import instances as inst_ops  # noqa: E402

PEAK_BPS = 3.35e12


def card():
    q = 'name,power.limit,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(','), [s.strip() for s in out.split(',')]))


def device_results(key):
    """bench.main's scan, injected predictions and model for workload `key` (seed 0) -> (device results, coords_float)."""
    wl = bench.WORKLOADS[key]
    torch.manual_seed(0)
    model = SoftGroup(**model_cfg(wl['cfg'])).cuda().eval()
    sc = synth.make_scan(wl['shape'], seed=0, n_points=wl['n'])
    if wl.get('intensity_only'):
        sc['feats'] = sc['feats'][:, :1].copy()
    base = sc
    if wl.get('x4'):
        sc = synth.to_x4_split(sc)
    s, o = synth.grouping_inputs(base, sigma=wl['sigma'], seed=0, fragments=wl.get('fragments', 1),
                                 confusion=wl.get('confusion', 0.0))
    with torch.no_grad():
        dev = harness.run_scan(model, harness.to_host_batch(sc), inject_pointwise=(torch.from_numpy(s).cuda(),
                                                                                    torch.from_numpy(o).cuda()),
                               device_results=True)
    torch.cuda.synchronize()
    return dev, torch.from_numpy(base['coords_float']).cuda()


def timed_ms(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='c2,c5')
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'instance_reduce.py measures on a GPU (no CPU fallback)'
    res = dict(card=card(), reps=args.reps, peak_bytes_per_s=PEAK_BPS, workloads={})
    for key in args.workloads.split(','):
        dev, cf = device_results(key)
        inst = dev['instances']
        n, total, N = inst['label_id'].numel(), inst['point_ids'].numel(), cf.size(0)
        feats = torch.randn(N, 32, device='cuda')
        r = dict(points=N, instances=n, point_ids=total)
        for name, values in (('reduce_coords_C3', cf), ('reduce_feats_C32', feats)):
            C = values.size(1)
            nbytes = 8 * (n + 1) + 4 * total + 4 * C * total + 4 * C * n * 3
            ms = timed_ms(lambda: inst_ops.instance_point_reduce(inst, values), args.reps)
            r[name] = dict(ms=ms, bytes=nbytes, gb_per_s=nbytes / ms / 1e6, share_of_peak=nbytes / ms / 1e-3 / PEAK_BPS)
        nbytes = 8 * (n + 1) + 4 * n + 4 * total + 20 * N
        ms = timed_ms(lambda: inst_ops.instance_point_map(inst, N), args.reps)
        r['point_map'] = dict(ms=ms, bytes=nbytes, gb_per_s=nbytes / ms / 1e6, share_of_peak=nbytes / ms / 1e-3 / PEAK_BPS)
        res['workloads'][key] = r
        del dev, inst, feats
        torch.cuda.empty_cache()
    res['card_after'] = card()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
