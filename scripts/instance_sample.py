"""Time of instance_farthest_point_sample on the device results of bench workloads, against a torch restatement.

For each workload the device_results forward runs once; then, for each K, the call is timed with CUDA events over --reps
calls after a warm-up. A workload key ending in `all` (c5all) is one list holding every point of that scan. FPS is a
chain of K dependent argmax steps per list, bound by issue and step latency rather than HBM, so the rate reported is
distance updates per second: sum over the lists of len * K. The torch restatement is what a
caller writes without this call: the lists padded to the next power of two per size bucket (the bucket sizes come from
the host copy of the offsets, outside the timing), then K steps of torch ops per bucket; it is timed the same way and
checked to pick the same ids where no NaN or tie is involved (it breaks ties and orders NaN as torch.argmax does, so it
is a timing reference, not an oracle). The card's name, power limit and max SM clock are read in the same run.
Usage: python scripts/instance_sample.py [--workloads c2,c3,c5,c5all] [--ks 256,1024] [--reps 50] [--out FILE.json]"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from instance_reduce import card, device_results, timed_ms  # noqa: E402
from softgroup_b200.ops import instances as inst_ops  # noqa: E402

FPS_THRESHOLDS = (512, 8192, 65536)  # SGB_FPS_WARP_MAX, SGB_FPS_CTA_MAX, SGB_FPS_CLUSTER_MAX of include/sgb200.h


def torch_buckets(off_h, dev):
    """Lists grouped by the power of two at or above their length (empty lists left out)."""
    lens = np.diff(off_h)
    out = []
    nz = np.flatnonzero(lens > 0)
    b = np.ceil(np.log2(lens[nz])).astype(np.int64)
    for e in np.unique(b):
        ks = nz[b == e]
        out.append((torch.from_numpy(ks).to(dev), torch.from_numpy(off_h[ks]).to(dev), torch.from_numpy(lens[ks]).to(dev),
                    1 << int(e)))
    return out


def torch_fps(buckets, ids, coords, n, K):
    out = torch.full((n, K), -1, dtype=torch.int32, device=coords.device)
    for ks, st, ln, Lmax in buckets:
        ar = torch.arange(Lmax, device=coords.device)
        mask = ar[None] < ln[:, None]
        pid = ids[(st[:, None] + ar[None]).clamp(max=ids.numel() - 1)]
        P = coords[pid.long()]
        rows = torch.arange(ks.numel(), device=coords.device)
        d = torch.where(mask, float('inf'), -1.0)  # padding is never chosen
        s = torch.zeros(ks.numel(), dtype=torch.int64, device=coords.device)
        out[ks, 0] = pid[rows, s]
        for j in range(1, K):
            t = ((P - P[rows, s][:, None]) ** 2).sum(-1)
            d = torch.where(mask, torch.minimum(d, t), d)
            s = d.argmax(1)
            out[ks, j] = pid[rows, s]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workloads', default='c2,c3,c5,c5all')
    ap.add_argument('--ks', default='256,1024')
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'instance_sample.py measures on a GPU (no CPU fallback)'
    res = dict(card=card(), reps=args.reps, workloads={})
    for key in args.workloads.split(','):
        dev, cf = device_results(key[:-3] if key.endswith('all') else key)
        inst = dev['instances']
        if key.endswith('all'):  # one list of every point of the scan: the streaming cluster path
            N = cf.size(0)
            inst = dict(point_offsets=torch.tensor([0, N], dtype=torch.int64, device=cf.device),
                        point_ids=torch.arange(N, dtype=torch.int32, device=cf.device))
        off_h = inst['point_offsets'].cpu().numpy()
        lens = np.diff(off_h)
        n, total = lens.size, int(off_h[-1])
        w, c, cl = FPS_THRESHOLDS
        r = dict(points=cf.size(0), instances=n, point_ids=total, max_len=int(lens.max(initial=0)),
                 lists_per_path=dict(warp=int(np.sum(lens <= w)), cta=int(np.sum((lens > w) & (lens <= c))),
                                     cluster=int(np.sum((lens > c) & (lens <= cl))), streaming=int(np.sum(lens > cl))))
        buckets = torch_buckets(off_h, cf.device)
        for K in (int(k) for k in args.ks.split(',')):
            updates = int(lens.sum()) * K
            ms = timed_ms(lambda: inst_ops.instance_farthest_point_sample(inst, cf, K), args.reps)
            ms_t = timed_ms(lambda: torch_fps(buckets, inst['point_ids'], cf, n, K), args.reps)
            a = inst_ops.instance_farthest_point_sample(inst, cf, K)
            b = torch_fps(buckets, inst['point_ids'], cf, n, K)
            r['K=%d' % K] = dict(ms=ms, distance_updates=updates, updates_per_s=updates / ms * 1e3, torch_ms=ms_t,
                                 torch_updates_per_s=updates / ms_t * 1e3, speedup=ms_t / ms,
                                 rows_equal_to_torch=float((a == b).all(1).float().mean()))
            print(key, K, r['K=%d' % K], flush=True)
        res['workloads'][key] = r
        del dev, inst, buckets
        torch.cuda.empty_cache()
    res['card_after'] = card()
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        with open(args.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
