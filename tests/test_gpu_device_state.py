"""GPU: the library's per-device launch state -- the device record of csrc/core.cu (SM count, fp16-overflow flag) and the
modules' one-time set-up per device (kernel attributes, occupancy) -- under concurrent first calls and on a second
device. That state lives as long as the process and only a process's first calls build it, so each case runs once in a
fresh interpreter."""
import os
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

# Inputs and the calls under test. Nothing here calls the library before the case does: the rulebook is built on the
# host, and packing the weights only asks the library for a constant.
PRELUDE = r'''
import sys
import threading
import numpy as np
import torch
sys.path.insert(0, %r)
import oracle
from softgroup_b200 import spconv
from softgroup_b200.ops import _lib, ballquery_batch_p_nosync, bfs_cluster_segments
from softgroup_b200.spconv import core

G, CIN, COUT = 40, 32, 64  # 64000 rows of a dense grid: the persistent tensor-core launch
RADIUS, THR = 0.04, 50.0


def subm_map(g):
    """[27, g^3] rulebook of a 3x3x3 submanifold conv on a dense g^3 grid: the row of each neighbour, or -1."""
    x, y, z = np.meshgrid(np.arange(g), np.arange(g), np.arange(g), indexing='ij')
    mp = np.full((27, g ** 3), -1, np.int32)
    for k, (dx, dy, dz) in enumerate(np.ndindex(3, 3, 3)):
        nx, ny, nz = x + dx - 1, y + dy - 1, z + dz - 1
        ok = (nx >= 0) & (nx < g) & (ny >= 0) & (ny < g) & (nz >= 0) & (nz < g)
        mp[k][ok.ravel()] = (nx * g * g + ny * g + nz)[ok]
    return mp


rng = np.random.default_rng(0)
FEATS = rng.standard_normal((G ** 3, CIN)).astype(np.float32)
W = (rng.standard_normal((27, CIN, COUT)) / (27 * CIN) ** 0.5).astype(np.float32)
MAP = subm_map(G)
centres = rng.random((20, 3))
XYZ = (centres.repeat(300, 0) + 0.02 * rng.standard_normal((6000, 3))).astype(np.float32)


def inputs(dev):
    return dict(x=torch.from_numpy(FEATS).to(dev), mp=torch.from_numpy(MAP).to(dev),
                w=core.WeightPack(torch.from_numpy(W).to(dev)), xyz=torch.from_numpy(XYZ).to(dev),
                bi=torch.zeros(len(XYZ), dtype=torch.int32, device=dev),
                bo=torch.tensor([0, len(XYZ)], dtype=torch.int32, device=dev))


def conv(a):
    """act_pack of the input rows, then the tensor-core conv."""
    return core.conv_forward(a['x'], CIN, 0, a['mp'], 27, G ** 3, a['w'], CIN, COUT)


def group(a):
    """Async ball query, then the clustering -> (per-point neighbour lists, cluster_idxs, cluster_offsets) on the host."""
    idx, sl, tot = ballquery_batch_p_nosync(a['xyz'], a['bi'], a['bo'], RADIUS)
    ci, co = bfs_cluster_segments(idx, sl, THR, upstream_err=tot[1:])
    idx, sl = idx.cpu().numpy(), sl.cpu().numpy()
    return [idx[s:s + n] for s, n in sl], ci.cpu().numpy(), co.cpu().numpy()


def group_oracle():
    idx, sl = oracle.ballquery_batch_p(XYZ, np.zeros(len(XYZ), np.int32), np.array([0, len(XYZ)], np.int32), RADIUS)
    ci, co = oracle.bfs_cluster(np.full(1, -1, np.float32), idx, sl, THR, 0)
    return [idx[s:s + n] for s, n in sl], ci, co


def same_groups(a, b):
    return len(a[0]) == len(b[0]) and all(np.array_equal(p, q) for p, q in zip(a[0], b[0])) and \
        np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
''' % ROOT

CONCURRENT = r'''
a = inputs('cuda:0')
torch.cuda.synchronize()
n_threads = 8
start = threading.Barrier(n_threads)
got, errors = [None] * n_threads, []


def worker(t):
    try:
        st = torch.cuda.Stream()
        with torch.cuda.stream(st), torch.no_grad():
            start.wait()
            if t % 2:  # half the threads enter through the grouping, half through the convolution
                g = group(a)
                y = conv(a)
            else:
                y = conv(a)
                g = group(a)
        st.synchronize()
        got[t] = (y, g)
    except BaseException as e:
        errors.append('thread %d: %r' % (t, e))


threads = [threading.Thread(target=worker, args=(t,)) for t in range(n_threads)]
for th in threads:
    th.start()
for th in threads:
    th.join()
assert not errors, errors
want_y, want_g = conv(a), group_oracle()
for t, (y, g) in enumerate(got):
    assert torch.equal(y, want_y), 'thread %d: conv differs from the same call made alone' % t
    assert same_groups(g, want_g), 'thread %d: grouping differs from the oracle' % t
assert want_g[2].size > 2, 'the scene must form clusters'
spconv.check_overflow()  # nothing above left the fp16 range

packer = threading.Thread(target=lambda: core.act_pack(torch.full((4, CIN), 1e5, device='cuda:0'), CIN, 0, CIN))
packer.start()
packer.join()
torch.cuda.synchronize()
try:
    spconv.check_overflow()
    raise AssertionError('the packed 1e5 was not reported')
except _lib.SgbError:
    pass
spconv.check_overflow()  # reading the flag cleared it
print('ok')
'''

TWO_DEVICES = r'''
want = group_oracle()
res = []
for dev in ('cuda:0', 'cuda:1'):
    torch.cuda.set_device(dev)
    a = inputs(dev)
    with torch.no_grad():
        res.append((conv(a).cpu(), group(a)))
assert torch.equal(res[0][0], res[1][0]), 'conv differs between the devices'
for d, (_, g) in enumerate(res):
    assert same_groups(g, want), 'device %d: grouping differs from the oracle' % d
print('ok')
'''


def _run(body):
    out = subprocess.run([sys.executable, '-c', PRELUDE + body], cwd=ROOT, capture_output=True, text=True, timeout=900)
    assert out.returncode == 0 and out.stdout.strip().endswith('ok'), (out.stdout[-3000:], out.stderr[-6000:])


def test_concurrent_first_calls_share_one_device_record():
    """Eight threads, each on its own stream, make the process's first library calls at the same moment: every result
    equals the call made alone (conv) or the oracle (ball query + clustering), and a value packed afterwards is reported
    once by check_overflow."""
    _run(CONCURRENT)


def test_second_device_gets_its_own_set_up():
    """The ball query, the clustering and a tensor-core conv on device 0, then on device 1, in one process: the kernel
    attributes and occupancy are set up per device, and the results are identical on both and equal the oracle."""
    if torch.cuda.device_count() < 2:
        pytest.skip('needs two visible GPUs')
    _run(TWO_DEVICES)
