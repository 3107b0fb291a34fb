"""CPU: the C restatement of sgb_id_lists_fps (tests/fps_oracle.c), which the GPU tests compare against bit for bit,
equals the literal numpy float32 loop of the header's steps: the worked example of include/sgb200.h's contract, and
small random lists with every edge (empty lists, all-invalid lists, an invalid first position, repeated ids, duplicate
coordinates, exact lattice ties, NaN and +-inf coordinates) for K below, at and far beyond the list lengths."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fps_oracle  # noqa: E402


def test_worked_example():
    ex = fps_oracle.WORKED_EXAMPLE
    for fn in (fps_oracle.np_fps, fps_oracle.id_lists_fps):
        assert fn(ex['off'], ex['ids'], ex['xyz'], ex['K']).tolist() == ex['want']


def test_lists_of_one_and_no_lists():
    xyz = np.float32([[0, 0, 0], [np.nan, 1, 2], [np.inf, 0, 0]])
    off = np.arange(5, dtype=np.int64)
    ids = np.int32([0, 1, 2, 3])
    want = [[0] * 4, [1] * 4, [2] * 4, [-1] * 4]
    assert fps_oracle.np_fps(off, ids, xyz, 4).tolist() == want
    assert fps_oracle.id_lists_fps(off, ids, xyz, 4).tolist() == want
    assert fps_oracle.id_lists_fps(np.zeros(1, np.int64), np.zeros(0, np.int32), xyz, 3).shape == (0, 3)


@pytest.mark.parametrize('K', [1, 2, 5, 33, 200])
def test_c_oracle_equals_numpy(K):
    rng = np.random.RandomState(K)
    N = 300
    xyz = fps_oracle.edge_points(rng, N)
    lens = rng.randint(0, 60, size=150)
    lens[::11] = 0
    lens[::13] = 1
    off, ids = fps_oracle.edge_lists(rng, lens, N)
    want = fps_oracle.np_fps(off, ids, xyz, K)
    got = fps_oracle.id_lists_fps(off, ids, xyz, K)
    assert np.array_equal(got, want)
    # the edges are there: rows of -1, rows whose tail repeats, NaN and inf points chosen
    assert np.any(np.all(want == -1, axis=1)) and np.any(lens[np.all(want == -1, axis=1)] > 0)
    if K > 60:
        assert np.all(want[:, -1] == want[:, -2])
