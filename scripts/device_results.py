"""Per-scan time of the three result forms of forward_test on bench workloads: device_only (what bench.py times),
device_results (instances as point-id lists, panoptic labels, all on the GPU) and host results (the reference's RLE dicts
and numpy arrays). Each form runs one scan at a time and with 3 scans in flight (harness.ScanPipeline); the forms
alternate round by round. The card's name, power limit and max SM clock are read in the same run.
Usage: python scripts/device_results.py [--workloads c2,c5] [--scans 24] [--rounds 3] [--out FILE.json]"""
import argparse
import json
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, '.')
import bench  # noqa: E402
from softgroup_b200 import harness, synth  # noqa: E402
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402

FORMS = {'device_only': dict(device_only=True), 'device_results': dict(device_results=True), 'host': dict()}


def card():
    q = 'name,power.limit,clocks.max.sm'
    out = subprocess.run(['nvidia-smi', '--query-gpu=' + q, '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                         capture_output=True, text=True, check=True).stdout.strip()
    return dict(zip(q.split(','), [s.strip() for s in out.split(',')]))


def workload(key):
    """bench.main's scan, injected predictions and model for workload `key` (seed 0)."""
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
    return model, harness.to_host_batch(sc), (torch.from_numpy(s).cuda(), torch.from_numpy(o).cuda())


def per_scan_ms(pipe, model, hb, inj, form, n_scans, inflight):
    def call(_):
        harness.run_scan(model, hb, inject_pointwise=inj, **FORMS[form])  # the result is dropped at once
        return None

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if inflight == 1:
        with torch.no_grad():
            for _ in range(n_scans):
                call(None)
    else:
        pipe.map(call, range(n_scans))
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n_scans


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='c2,c5')
    ap.add_argument('--scans', type=int, default=24, help='scans per timed window')
    ap.add_argument('--rounds', type=int, default=3, help='timed windows per form and in-flight count (alternating)')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'device_results.py measures on a GPU (no CPU fallback)'
    res = dict(card=card(), scans_per_window=args.scans, rounds=args.rounds, workloads={})
    for key in args.workloads.split(','):
        model, hb, inj = workload(key)
        pipe = harness.ScanPipeline(model, workers=3)
        n = max(3, args.scans // (4 if bench.WORKLOADS[key]['n'] > 500000 else 1))
        for form in FORMS:  # warm-up of every form, sequential and in flight
            per_scan_ms(pipe, model, hb, inj, form, 3, 1)
            per_scan_ms(pipe, model, hb, inj, form, 6, 3)
        times = {(f, k): [] for f in FORMS for k in (1, 3)}
        for _ in range(args.rounds):
            for inflight in (1, 3):
                for form in FORMS:
                    times[(form, inflight)].append(per_scan_ms(pipe, model, hb, inj, form, n, inflight))
        pipe.close()
        r = {}
        for (form, inflight), ts in times.items():
            r['%s/inflight%d' % (form, inflight)] = dict(ms_per_scan_median=float(np.median(ts)), ms_per_scan=ts,
                                                         scans_per_s=1e3 / float(np.median(ts)))
        res['workloads'][key] = dict(points=int(hb['coords'].shape[0]), scans_per_window=n, **r)
        del model
        torch.cuda.empty_cache()
    res['card_after'] = card()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
