"""Farthest-point sampling per id list on the CPU: fps_oracle.c (the C restatement the GPU tests compare against, fast
enough for every instance of a 1.5M-point tile) and np_fps (the same steps as a literal numpy float32 loop, which checks
the C code on small lists). The shared library is compiled on first use into a temporary directory, with
-ffp-contract=off, so that the tree stays read-only."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        d = tempfile.mkdtemp(prefix='fps_oracle_')
        atexit.register(shutil.rmtree, d, True)
        so = os.path.join(d, 'libfps_oracle.so')
        subprocess.check_call([os.environ.get('CC', 'gcc'), '-O2', '-ffp-contract=off', '-fPIC', '-shared', '-Wall', '-o', so,
                               os.path.join(_HERE, 'fps_oracle.c'), '-lm'])
        _LIB = ctypes.CDLL(so)
        _LIB.orc_id_lists_fps.restype = None
        _LIB.orc_id_lists_fps.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                                          ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]
    return _LIB


def id_lists_fps(off, ids, xyz, K):
    """off int64 [n + 1], ids int32, xyz float32 [N, 3] -> int32 [n, K] (sgb_id_lists_fps of include/sgb200.h)."""
    off = np.ascontiguousarray(off, dtype=np.int64)
    ids = np.ascontiguousarray(ids, dtype=np.int32)
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    assert xyz.ndim == 2 and xyz.shape[1] == 3
    n = off.size - 1
    out = np.empty((n, K), np.int32)
    # ranges of lists of about equal id counts on a thread pool (ctypes releases the GIL during the call)
    cuts = np.unique(np.concatenate([[0, n], np.searchsorted(off, np.linspace(off[0], off[-1], 65)[1:-1])])).clip(0, n)
    cuts = np.unique(cuts)
    fn, ip = lib().orc_id_lists_fps, ids.ctypes.data if ids.size else None
    xp = xyz.ctypes.data if xyz.size else None

    def run(a, b):
        a, b = int(a), int(b)
        fn(off.ctypes.data + 8 * a, ip, b - a, xyz.shape[0], xp, 3, int(K), out.ctypes.data + 4 * a * int(K))

    with ThreadPoolExecutor(os.cpu_count() or 1) as ex:
        list(ex.map(run, cuts[:-1], cuts[1:]))
    return out


WORKED_EXAMPLE = dict(  # lists [5, 6, 7, 8] (x = 0, 1, 3, 10), [42, 7] with N = 9, and an empty list; K = 6
    off=np.array([0, 4, 6, 6], np.int64), ids=np.array([5, 6, 7, 8, 42, 7], np.int32),
    xyz=np.array([[0, 0, 0]] * 5 + [[0, 0, 0], [1, 0, 0], [3, 0, 0], [10, 0, 0]], np.float32), K=6,
    want=[[5, 8, 7, 6, 5, 5], [7] * 6, [-1] * 6])


def edge_points(rng, N):
    """float32 [N, 3]: random points, with a share on a coarse integer lattice (exact ties), exact copies of other rows
    (duplicate coordinates), and NaN, +inf and -inf coordinates."""
    xyz = (rng.randn(N, 3) * 3).astype(np.float32)
    lat = rng.rand(N) < 0.3
    xyz[lat] = rng.randint(-3, 4, size=(int(lat.sum()), 3)).astype(np.float32)
    dup = rng.rand(N) < 0.1
    xyz[dup] = xyz[rng.randint(0, N, size=int(dup.sum()))]
    for val, share in ((np.nan, 0.01), (np.inf, 0.005), (-np.inf, 0.005)):
        m = rng.rand(N, 3) < share
        xyz[m] = val
    return xyz


def edge_lists(rng, lens, N):
    """(off int64, ids int32) with the given lengths: random ids with repeats inside a list, a share of invalid ids
    (negative, N and beyond), every 7th list all invalid and every 5th with an invalid first position."""
    lens = np.asarray(lens, np.int64)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    ids = rng.randint(0, N, size=int(off[-1])).astype(np.int32)
    bad = rng.rand(ids.size) < 0.05
    ids[bad] = rng.choice(np.int32([-1, -7, N, N + 3, np.iinfo(np.int32).min, np.iinfo(np.int32).max]), size=int(bad.sum()))
    for k in range(lens.size):
        a, b = int(off[k]), int(off[k + 1])
        if b == a:
            continue
        if k % 7 == 3:
            ids[a:b] = -1
        elif k % 5 == 1:
            ids[a] = N
        if k % 3 == 0 and b - a > 2:
            ids[a + 1:b:3] = ids[a + 1]  # the same id at several positions
    return off, ids


def _key(d, pos):
    hi = d.view(np.uint32).astype(np.uint64) + np.uint64(1)
    hi[np.isnan(d)] = 0
    return (hi << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - pos.astype(np.uint64))


def np_fps(off, ids, xyz, K):
    """The header's steps as a numpy float32 loop over the lists."""
    n, N = off.size - 1, xyz.shape[0]
    out = np.full((n, K), -1, np.int32)
    for k in range(n):
        p = ids[off[k]:off[k + 1]]
        pos = np.flatnonzero((p >= 0) & (p < N))
        if pos.size == 0:
            continue
        P = xyz[p[pos]].astype(np.float32)
        d = np.full(pos.size, np.inf, np.float32)
        s = 0
        out[k, 0] = p[pos[s]]
        for j in range(1, K):
            with np.errstate(invalid='ignore', over='ignore'):  # inf - inf is NaN, as on the device
                t = P - P[s]
                t = t[:, 0] * t[:, 0] + t[:, 1] * t[:, 1] + t[:, 2] * t[:, 2]
            d = np.minimum(d, t)
            s = int(np.argmax(_key(d, pos)))
            out[k, j] = p[pos[s]]
    return out
