"""GPU: the segment reductions, the row kernels and the instance-mask kernels at full-size shapes and at the edges where
they go wrong, against plain references: the C oracle (pinned on the reference kernels), float64 numpy, or dense numpy
restatements of the reference code. The cases are listed in tests/kernel_edge_cases.py;
tests/test_kernel_edges_coverage.py checks that they reach every launch threshold of the kernels.

Segment min / max must equal the reference value for value (the sign of a zero result is not part of the contract, see
include/sgb200.h). Segment mean / global_avg_pool are held per element to |got - mean64| <= c * 2^-24 * sum|x| / n with
c = ceil(n / rows_par) + log2(rows_par) + 2, from the kernel's summation order (n / rows_par sequential terms per
thread, a log2(rows_par) tree, one division); the largest c each test measures is printed. Measured on an H100 80GB
HBM3 at 700 W: at most 3.3 on the segments of up to 9000 rows; on the 200k-row segment 26.5 for global_avg_pool (C = 32)
and 167 for sec_mean on 1e4 + N(0, 1) data (C = 5, bound 6257), where every term is divided by n before the sum."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from softgroup_b200 import ops
from softgroup_b200.ops import _lib
from softgroup_b200.ops import instances as inst_ops
from softgroup_b200.ops._lib import check
from softgroup_b200.util.rle import rle_encode

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import kernel_edge_cases as kc  # noqa: E402

pytestmark = pytest.mark.gpu
FLT_MAX = float(np.finfo(np.float32).max)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _addr(t, floats=0):
    return ctypes.c_void_p(t.data_ptr() + 4 * floats)


def _assert_same_values(got, want, what):
    """Value-exact, NaN where the reference has NaN; -0.0 == +0.0."""
    bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
    if bad.any():
        idx = np.argwhere(bad)[:8]
        raise AssertionError('%s: %d mismatches, first (proposal, channel) got / want: %s' %
                             (what, bad.sum(), [(tuple(i), got[tuple(i)], want[tuple(i)]) for i in idx]))


# ================================================================== segment min / max
def _specials(C):
    one = [-0.0, 0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1.17e-39, FLT_MAX, -FLT_MAX, -1.0]
    two = [-0.0, -1.0, -1.0, -0.0, np.nan, -0.0, 0.0, -0.0, -0.0, 0.0, np.nan, np.nan]
    col = np.array(one + two, np.float32)
    return np.stack([np.roll(col, 3 * c) if c else col for c in range(C)], 1)


def _minmax_values(case, rng):
    """(rows for sec_min, rows for sec_max) of a MinMaxCase."""
    off = case.offsets
    S, C = int(off[-1]), case.C
    if case.kind == 'specials':
        x = _specials(C)
        return x, x
    if case.kind == 'negzero':
        x = -(np.abs(rng.randn(S, C)) + 0.1).astype(np.float32)
        x[off[0]:off[1]] = -0.0
        x[8000:8006] = -0.0  # second proposal: its maximum only in chunk 3 of rows 5000..11199
        return x, x
    if case.kind == 'straddle':
        # proposal p >= 1: half A = rows [s, s + 1024) in one chunk, half B the rest in the next; the extreme sits in A
        # for odd p and in B for even p, so both chunk orders occur in one launch
        xmin = (rng.rand(S, C) + 0.5).astype(np.float32)
        xmax = -(rng.rand(S, C) + 0.5).astype(np.float32)
        for p in range(1, len(off) - 1):
            s = int(off[p])
            ext, zero = (slice(s, s + 1024), slice(s + 1024, s + 2048))[::1 if p % 2 else -1]
            xmin[ext] = -(rng.rand(1024, C) + 1.0)  # negative extreme; the other half only {+0, -0, positives}
            xmax[ext] = -(rng.rand(1024, C) + 1.0)  # the other half's maximum is -0.0
            zrows = zero.start + rng.choice(1024, 12, replace=False)
            xmin[zrows[:6]] = -0.0
            xmax[zrows[:6]] = -0.0
            if p % 4 >= 2:
                xmin[zrows[6:]] = 0.0
        return xmin, xmax
    x = (rng.randn(S, C) * 3 - 1).astype(np.float32)
    z = rng.rand(S) < 0.01
    x[z] = -0.0
    x[rng.rand(S) < 0.01] = 0.0
    if case.kind == 'lead':
        x[:off[0]:2] = -1e30  # rows outside every proposal
        x[1:off[0]:2] = 1e30
    if S > kc.SEG_GRID * kc.SEG_CHUNK:  # extremes in the chunks only the grid-stride loop reaches
        for c in range(C):
            x[S - 7 - c, c] = -1e6 - c
            x[S - 3 - c, c] = 1e6 + c
    return x, x


@pytest.mark.parametrize('case', kc.MINMAX_CASES, ids=lambda c: c.name)
def test_sec_min_max_value_exact(case):
    xmin, xmax = _minmax_values(case, np.random.RandomState(len(case.name)))
    oc = _cuda(case.offsets)
    got = ops.sec_min(_cuda(xmin), oc).cpu().numpy()
    _assert_same_values(got, oracle.sec_min(xmin, case.offsets), 'sec_min')
    got = ops.sec_max(_cuda(xmax), oc).cpu().numpy()
    _assert_same_values(got, oracle.sec_max(xmax, case.offsets), 'sec_max')


def test_sec_max_single_negative_zero():
    x = np.array([[-0.0], [-0.0], [-3.0]], np.float32)
    off = np.array([0, 1, 3], np.int32)
    got = ops.sec_max(_cuda(x), _cuda(off)).cpu().numpy()
    assert got[0, 0] == 0.0 and got[1, 0] == 0.0, got.ravel()  # -0.0 (or +0.0), not -inf / -3
    got = ops.sec_min(_cuda(x), _cuda(off)).cpu().numpy()
    assert got[0, 0] == 0.0 and got[1, 0] == -3.0, got.ravel()


# ================================================================== segment mean / global_avg_pool
def _mean_values(case, rng):
    S, C = int(case.offsets[-1]), case.C
    if case.data == 'relu':
        return np.maximum(rng.randn(S, C), 0).astype(np.float32)
    if case.data == 'offset':
        return (1e4 + rng.randn(S, C)).astype(np.float32)
    sign = np.where(np.arange(S) % 2 == 0, 1.0, -1.0)[:, None]
    return (1e3 * sign + 1e-2 * rng.randn(S, C)).astype(np.float32)


def _mean_bound_c(got, x, off, C):
    """Largest measured c, asserting c <= the summation-order bound on every element of every non-empty proposal."""
    rp = kc.rows_par(C)
    n = np.diff(off).astype(np.int64)
    ne = n > 0
    x64 = x.astype(np.float64)
    starts = off[:-1][ne]  # rows start at offsets[0] == 0, so each non-empty segment ends where the next one starts
    nn = n[ne][:, None]
    unit = 2.0**-24 * np.add.reduceat(np.abs(x64), starts, axis=0) / nn
    err = np.abs(got[ne].astype(np.float64) - np.add.reduceat(x64, starts, axis=0) / nn)
    bound = (np.ceil(nn / rp) + math.log2(rp) + 2) * unit
    bad = err > bound
    assert not bad.any(), 'n=%s: err %s > bound %s' % (nn[bad.any(1)][:4, 0], err[bad][:4], bound[bad][:4])
    nz = unit > 0
    return float((err[nz] / unit[nz]).max()) if nz.any() else 0.0


@pytest.mark.parametrize('case', kc.MEAN_CASES, ids=lambda c: c.name)
def test_sec_mean_and_avg_pool_error_bound(case):
    x = _mean_values(case, np.random.RandomState(7))
    off = case.offsets
    xc, oc = _cuda(x), _cuda(off)
    empty = off[1:] == off[:-1]
    for name, fn, ref in (('sec_mean', ops.sec_mean, oracle.sec_mean),
                          ('global_avg_pool', ops.global_avg_pool, oracle.global_avg_pool)):
        got = fn(xc, oc).cpu().numpy()
        if name == 'sec_mean':
            assert (got[empty] == 0).all()
        else:
            assert np.isnan(got[empty]).all()  # 0 / 0, like the reference
        c = _mean_bound_c(got, x, off, case.C)
        print('\n%s %s: measured c = %.2f (units of 2^-24 * sum|x| / n)' % (case.name, name, c))
        if case.data == 'relu':
            # against the reference's own sequential float sum: only up to ORACLE_REL_ROWS rows, beyond which that
            # sum itself drifts from the float64 mean by more than 1e-5 (1.5e-5 at 200k rows)
            n = off[1:] - off[:-1]
            rows = (n > 0) & (n <= kc.ORACLE_REL_ROWS)
            np.testing.assert_allclose(got[rows], ref(x, off)[rows], rtol=1e-5, atol=0)


@pytest.mark.parametrize('case', [c for c in kc.MEAN_CASES if c.data != 'relu' or c.C in (3, 8)],
                         ids=lambda c: c.name)
def test_global_avg_pool_bp_accumulates_bit_exact(case):
    rng = np.random.RandomState(11)
    off = case.offsets
    S, nP = int(off[-1]), len(off) - 1
    d_out = rng.randn(nP, case.C).astype(np.float32)
    pre = rng.randn(S, case.C).astype(np.float32)  # d_feats is accumulated into, not overwritten
    d_feats, oc, dc = _cuda(pre), _cuda(off), _cuda(d_out)  # held: a freed tensor's memory can be handed out again
    check(_lib.lib().sgb_global_avg_pool_bp(_addr(d_feats), _addr(oc), _addr(dc), nP, case.C, _stream()),
          'sgb_global_avg_pool_bp')
    want = pre.copy()
    oracle.lib().orc_global_avg_pool_bp(want.ctypes.data_as(oracle._f32p), off.ctypes.data_as(oracle._i32p),
                                        d_out.ctypes.data_as(oracle._f32p), nP, case.C)
    assert np.array_equal(d_feats.cpu().numpy(), want)


# ================================================================== voxelize_fp / voxelize_bp with long rows
@pytest.mark.parametrize('mode', [3, 4])
@pytest.mark.parametrize('C', kc.VOXEL_CHANNELS)
def test_voxelize_fp_bp_long_rows_bit_exact(C, mode):
    rng = np.random.RandomState(C + mode)
    n = 20000
    coords = np.concatenate([rng.randint(0, 2, (n, 1)), rng.randint(0, 30, (n, 3))], 1).astype(np.int64)
    coords[rng.choice(n, kc.LONG_VOXEL, replace=False)] = (1, 7, 7, 7)  # one voxel of 3000 points, spread over the scan
    _, _, om = oracle.voxelization_idx(coords, 2, mode)
    assert om.shape[1] - 1 >= kc.LONG_VOXEL
    feats = (rng.randn(n, C) * np.exp2(rng.randint(-8, 8, (1, C)))).astype(np.float32)
    f = _cuda(feats).requires_grad_(True)
    out = ops.voxelization(f, _cuda(om), mode)
    assert np.array_equal(out.detach().cpu().numpy(), oracle.voxelization(feats, om, mode))
    g = rng.randn(om.shape[0], C).astype(np.float32)
    out.backward(_cuda(g))
    assert np.array_equal(f.grad.cpu().numpy(), oracle.voxelization_bp(g, om, n, mode))


# ================================================================== row kernels
SENTINEL = np.float32(-7.75e33)


@pytest.mark.parametrize('case', kc.GATHER_CASES, ids=lambda c: c.name)
def test_gather_rows_bit_exact(case):
    rng = np.random.RandomState(case.N % 1000)
    src = rng.randn(case.n_src, case.C).astype(np.float32)
    src.ravel()[rng.choice(src.size, min(src.size, 5), replace=False)] = [-0.0, np.nan, np.inf, 1e-45, -FLT_MAX][:min(src.size, 5)]
    idx = rng.randint(0, case.n_src, case.N).astype(np.int32)  # repeated, unsorted
    want = np.take(src, idx, axis=0)
    if case.in_off == 0 and case.out_off == 0:
        got = ops.gather_rows(_cuda(src), _cuda(idx)).cpu().numpy()
        assert np.array_equal(got.view(np.int32), want.view(np.int32))
        if case.N > 200000:
            return
    # through the C ABI with the input / output one float past a 16-byte boundary (the scalar path)
    ib = torch.full((case.in_off + src.size + 8,), float(SENTINEL), device='cuda')
    ib[case.in_off:case.in_off + src.size] = _cuda(src.ravel())
    ob = torch.full((case.out_off + want.size + 8,), float(SENTINEL), device='cuda')
    ic = _cuda(idx)
    check(_lib.lib().sgb_gather_rows(_addr(ib, case.in_off), _addr(ic), _addr(ob, case.out_off), case.N, case.C,
                                     _stream()), 'sgb_gather_rows')
    o = ob.cpu().numpy()
    assert np.array_equal(o[case.out_off:case.out_off + want.size].view(np.int32), want.ravel().view(np.int32))
    assert (o[:case.out_off] == SENTINEL).all() and (o[case.out_off + want.size:] == SENTINEL).all()


@pytest.mark.parametrize('relu', [0, 1])
@pytest.mark.parametrize('C,xs,ys', [(3, 8, 5), (32, 37, 40), (37, 64, 38)])
def test_bn_relu_strided_single_rounding(C, xs, ys, relu):
    rng = np.random.RandomState(C * 2 + relu)
    M = 5003
    x = (rng.randn(M, xs) * np.exp2(rng.randint(-20, 20, (M, xs)))).astype(np.float32)
    scale = (rng.randn(C) * np.exp2(rng.randint(-6, 6, C))).astype(np.float32)
    shift = (rng.randn(C) * np.exp2(rng.randint(-6, 6, C))).astype(np.float32)
    y = torch.full((M, ys), float(SENTINEL), device='cuda')
    xc, sc, tc = _cuda(x), _cuda(scale), _cuda(shift)
    check(_lib.lib().sgb_bn_relu(_addr(xc), xs, _addr(sc), _addr(tc), relu, _addr(y), ys, M, C,
                                 _stream()), 'sgb_bn_relu')
    y = y.cpu().numpy()
    ref = x[:, :C].astype(np.float64) * scale.astype(np.float64) + shift.astype(np.float64)  # x*s exact in float64
    if relu:
        ref = np.maximum(ref, 0.0)
    half_ulp = 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    err = np.abs(y[:, :C].astype(np.float64) - ref)
    assert (err <= half_ulp + 2.0**-52 * np.abs(ref)).all(), 'worst %s ulp' % (err / (2 * half_ulp)).max()
    assert (y[:, C:] == SENTINEL).all()


# ================================================================== instances: RLE of bitmaps
def _pack(mask, W):
    bits = np.zeros(W * 32, np.uint8)
    bits[:mask.size] = mask
    return np.packbits(bits, bitorder='little').view('<u4')


@pytest.mark.parametrize('case', kc.RLE_CASES, ids=lambda c: c.name)
def test_bitmaps_to_rle_matches_rle_encode(case):
    N, W = case.N, kc.bitmap_words(case.N)
    pats = kc.rle_patterns(case)
    words = np.zeros((case.n_inst, W), np.uint32)
    want = []
    pairs = []
    for k in range(case.n_inst):
        m = kc.mask_of(pats[k % len(pats)], N, seed=k)
        words[k] = _pack(m, W)
        want.append(rle_encode(m.astype(np.uint8)))
        if N <= 150000:
            pairs.append(np.stack([np.full(m.sum(), k), np.flatnonzero(m)], 1))
    bm = _cuda(words.view(np.int32))
    got = inst_ops.bitmaps_to_rle(bm, N)
    assert len(got) == len(want)
    for k, (g, w) in enumerate(zip(got, want)):
        assert g == w, 'mask %d (%s): %s... vs %s...' % (k, pats[k % len(pats)], g['counts'][:60], w['counts'][:60])
    if pairs:  # the same bitmaps from (row, point) pairs
        pr = np.concatenate(pairs).astype(np.int32)
        got = inst_ops.bitmaps_from_pairs(_cuda(pr[:, 0]), _cuda(pr[:, 1]), case.n_inst, N).cpu().numpy()
        assert np.array_equal(got.view(np.uint32), words)


# ================================================================== instances: count / scatter of mask scores
def _inst_inputs(case, rng, thr):
    if case.layout == 'single':
        lengths = np.ones(case.nP, np.int64)
    else:
        lengths = np.diff(kc._offsets(kc._lengths(case.nP, case.S, seed=case.S)))
    pid = np.repeat(np.arange(case.nP), lengths)
    pts = np.concatenate([rng.permutation(case.N)[:n] for n in lengths])  # distinct points inside a proposal
    pidx = np.stack([pid, pts], 1).astype(np.int32)
    if case.layout == 'interleaved':  # shuffle inside each warp of entries
        for w in range(0, case.S, 32):
            pidx[w:w + 32] = pidx[w + rng.permutation(min(32, case.S - w))]
    scores = rng.rand(case.S, case.ms_stride).astype(np.float32)
    scores[rng.rand(case.S, case.ms_stride) < 0.1] = thr  # exactly the threshold: not counted (`> thr`)
    return pidx, scores


@pytest.mark.parametrize('case', kc.INST_CASES, ids=lambda c: c.name)
def test_inst_count_and_scatter_against_dense(case):
    rng = np.random.RandomState(case.S)
    thr = np.float32(0.5)
    pidx, scores = _inst_inputs(case, rng, thr)
    on = scores[:, :case.nI] > thr
    want = np.zeros((case.nP, case.nI), np.int64)
    np.add.at(want, pidx[:, 0], on.astype(np.int64))
    sc = _cuda(scores)[:, :case.nI]  # row stride ms_stride >= nI
    assert sc.stride(0) == case.ms_stride
    pc = _cuda(pidx)
    got = inst_ops.instance_point_counts(pc, sc, case.nI, float(thr), case.nP).cpu().numpy()
    assert np.array_equal(got, want)

    keep = rng.rand(case.nP, case.nI) < 0.6  # -1 holes in slot
    bm, kcls, kprop = inst_ops.instance_bitmaps(pc, sc, case.nI, float(thr), _cuda(keep), case.N)
    wc, wp = np.nonzero(keep.T)  # class-major, like the reference's instance order
    assert np.array_equal(kcls.cpu().numpy(), wc) and np.array_equal(kprop.cpu().numpy(), wp)
    row = np.full((case.nI, case.nP), -1, np.int64)
    row[wc, wp] = np.arange(wc.size)
    W = kc.bitmap_words(case.N)
    words = np.zeros(wc.size * W, np.uint32)
    e, i = np.nonzero(on)
    r = row[i, pidx[e, 0]]
    sel = r >= 0
    pt = pidx[e[sel], 1].astype(np.int64)
    np.bitwise_or.at(words, r[sel] * W + (pt >> 5), (np.uint32(1) << (pt & 31).astype(np.uint32)))
    assert np.array_equal(bm.cpu().numpy().view(np.uint32).ravel(), words)


# ================================================================== instances: evaluation intersections
@pytest.mark.parametrize('N,nG', [(33, 3), (150000, 7), (4096, 0)])
def test_bitmap_intersections_against_dense(N, nG):
    rng = np.random.RandomState(N + nG)
    n_rows = 40
    pats = [p for p in kc.PATTERNS]
    masks = np.stack([kc.mask_of(pats[k % len(pats)], N, seed=k) for k in range(n_rows)])
    gslot = rng.choice(np.arange(-2, nG), N).astype(np.int32)
    W = kc.bitmap_words(N)
    bm = _cuda(np.stack([_pack(m, W) for m in masks]).view(np.int32))
    inter, vert, void = inst_ops.bitmap_intersections(bm, _cuda(gslot), nG, N)
    want = np.stack([(masks & (gslot == g)[None]).sum(1) for g in range(nG)], 1) if nG else np.zeros((n_rows, 0))
    assert np.array_equal(inter.cpu().numpy(), want)
    assert np.array_equal(vert.cpu().numpy(), masks.sum(1))
    assert np.array_equal(void.cpu().numpy(), (masks & (gslot == -2)[None]).sum(1))


# ================================================================== instances: panoptic paste
def _panoptic_dense(masks, order, cls_values, semantic, skip_iou):
    """softgroup.py:606-632 of the reference on dense masks (instances visited in `order`)."""
    pan_cls = semantic.astype(np.uint32)
    pan_ids = np.zeros(semantic.size, np.uint32)
    prev = np.zeros(semantic.size, bool)
    pid = 1
    for r in order:
        mask = masks[r]
        if (mask * prev).sum() / (mask.sum() + 1e-5) > skip_iou:
            continue
        paste = mask * (~prev)
        pan_cls[paste] = cls_values[r]
        pan_ids[paste] = pid
        prev[paste] = 1
        pid += 1
    return pan_cls, pan_ids


def test_panoptic_paste_bench_size():
    N, n = kc.PANOPTIC_N, kc.PANOPTIC_INST
    rng = np.random.RandomState(3)
    masks = np.zeros((n, N), bool)
    for r in range(n):
        for _ in range(rng.randint(1, 4)):
            a = rng.randint(0, N)
            masks[r, a:a + rng.randint(1, 3000)] = True
    # the first two instances visited: [500, 1500) then [0, 1000), whose overlap ratio 500 / (1000 + 1e-5) is made the
    # threshold itself -- equal is not greater, so it is pasted; the third ([999, 2000), 501 of its 1001 points already
    # pasted) is skipped
    masks[:3] = False
    masks[0, 500:1500] = masks[1, 0:1000] = True
    masks[2, 999:2000] = True
    skip_iou = 500 / (1000 + 1e-5)
    order = np.concatenate([[0, 1, 2], 3 + rng.permutation(n - 3)]).astype(np.int32)
    cls_values = rng.randint(11, 40, n).astype(np.int32)
    semantic = rng.randint(0, 20, N).astype(np.int64)
    W = kc.bitmap_words(N)
    assert W > kc.PAN_THREADS
    bm = _cuda(np.stack([_pack(m, W) for m in masks]).view(np.int32))
    pan_cls, pan_ids = inst_ops.panoptic_paste(bm, _cuda(order), _cuda(cls_values), _cuda(semantic), skip_iou, N)
    want_cls, want_ids = _panoptic_dense(masks, order, cls_values, semantic, skip_iou)
    got_ids = pan_ids.cpu().numpy().view(np.uint32)
    assert got_ids[0] == 2 and (got_ids[500:1500] == 1).all()  # instance 1 pasted at equality
    assert np.array_equal(pan_cls.cpu().numpy().view(np.uint32), want_cls)
    assert np.array_equal(got_ids, want_ids)
