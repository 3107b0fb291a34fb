"""A room beyond one ball query's int32 list cursor, end to end: the S3DIS config (x4_split backbone) on a synthetic
3,000,000-point S3DIS-shape room with injected point-wise predictions (sigma 0.1), whose 2.5 M selected (class, point)
entries are more than the 2,147,483 one ball query addresses, so forward_grouping runs in chunks. The 150k-point ScanNet
scan of bench.py (below the bound, one ball query) is measured in the same run, alternating with the room.

Per scan it reports
  * `forward_ms`: forward_test (device_only) per call, CUDA events after warm-up;
  * `grouping_ms`: the `grouping` stage of SoftGroup.profile_stages in separate calls;
  * `launches`: the library's launch counter per forward;
  * `entries`, `chunks` (the ball queries forward_grouping made), `proposals`, `max_memory_allocated_gb`.
The GPU's name, power limit and max SM clock are read in the same run.

    python scripts/large_scan.py [--rounds 5] [--out result.json]
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
from softgroup_b200.configs import model_cfg  # noqa: E402
from softgroup_b200.model import SoftGroup  # noqa: E402
from softgroup_b200.model import softgroup as sg_module  # noqa: E402
from softgroup_b200.ops import _lib  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    lines = q.stdout.strip().splitlines()
    return lines[torch.cuda.current_device()] if q.returncode == 0 and lines else torch.cuda.get_device_name()


def stats(xs):
    xs = np.asarray(xs, np.float64)
    return dict(median=round(float(np.median(xs)), 3), min=round(float(xs.min()), 3), max=round(float(xs.max()), 3))


class Scan(object):

    def __init__(self, cfg, shape, n_points, sigma, x4):
        torch.manual_seed(0)
        self.model = SoftGroup(**model_cfg(cfg)).cuda().eval()
        scan = synth.make_scan(shape, seed=0, n_points=n_points)
        self.inj = harness.pointwise_injection(scan, sigma=sigma, seed=0)  # point order = merged x4 output order
        self.dev = harness.device_batch(harness.to_host_batch(synth.to_x4_split(scan) if x4 else scan))
        self.dev.pop('coords')
        self.n_points = n_points
        self.times, self.stage, self.launches = [], [], []

    def step(self):
        return self.model.forward_test(device_only=True, inject_pointwise=self.inj, **self.dev)

    def timed(self):
        L = _lib.lib()
        torch.cuda.synchronize()
        l0 = L.sgb_launch_count()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ret = self.step()
        b.record()
        torch.cuda.synchronize()
        self.launches.append(L.sgb_launch_count() - l0)
        self.times.append(a.elapsed_time(b))
        return ret

    def staged(self):
        self.model.profile_stages = True
        self.step()
        self.model.profile_stages = False
        self.stage.append(self.model.stage_ms['grouping'])


@torch.no_grad()
def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--out', default=None, help='also write the result as JSON here')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'large_scan.py measures on the GPU (no CPU fallback)'
    scans = {'s3dis_3M': Scan('s3dis', 'c3_s3dis', 3000000, 0.1, True),
             'scannet_150k': Scan('scannet', 'c2_scannet', 150000, 0.03, False)}
    chunks = []
    real_bq = sg_module.ballquery_batch_p_nosync

    def counting_bq(*args, **kw):
        chunks[-1] += 1
        return real_bq(*args, **kw)
    sg_module.ballquery_batch_p_nosync = counting_bq
    info = {}
    for name, s in scans.items():
        torch.cuda.reset_peak_memory_stats()
        chunks.append(0)
        ret = s.step()  # warm-up (module load, plan, caches)
        s.step()
        torch.cuda.synchronize()
        po = ret['proposals_offset']
        info[name] = dict(points=s.n_points, ball_queries=chunks[-1] // 2, proposals=int(po.numel() - 1),
                          max_memory_allocated_gb=round(torch.cuda.max_memory_allocated() / 2**30, 2))
    sg_module.ballquery_batch_p_nosync = real_bq
    for _ in range(a.rounds):  # alternating
        for s in scans.values():
            s.timed()
            s.staged()
    res = dict(gpu=card(), rounds=a.rounds, results={})
    for name, s in scans.items():
        res['results'][name] = dict(info[name], forward_ms=stats(s.times), grouping_ms=stats(s.stage),
                                    launches=sorted(set(s.launches)))
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
