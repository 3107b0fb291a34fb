"""oracle -- CPU restatement of the reference algorithms. TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this package. The product (softgroup_b200) never does; it fails loudly when its CUDA
library is missing instead of falling back to anything in here.

numpy in / numpy out, function names follow softgroup/ops/functions.py of the reference.

Files: sg_oracle.c (the ops, plain C), spconv_oracle.py (sparse convolution restatement, numpy), build_ref.py (compiles
the unmodified reference ops into oracle/_ref), spconv_cpu.py + ops_cpu.py (module / function plumbing that lets the
unmodified reference MODEL code run on the CPU to generate whole-model golden vectors, tests/golden/).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

_i32p = ctypes.POINTER(ctypes.c_int32)
_i64p = ctypes.POINTER(ctypes.c_int64)
_f32p = ctypes.POINTER(ctypes.c_float)


def build():
    """Compile liboracle.so with gcc (idempotent)."""
    so = os.path.join(_HERE, 'liboracle.so')
    src = os.path.join(_HERE, 'sg_oracle.c')
    if not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(['make', '-C', _HERE, 'liboracle.so'], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
        _LIB.orc_voxelize_idx_begin.restype = ctypes.c_void_p
        _LIB.orc_bfs_cluster_begin.restype = ctypes.c_void_p
        _LIB.orc_ballquery_batch_p.restype = ctypes.c_longlong
        _LIB.orc_ballquery_batch_p_grid.restype = ctypes.c_longlong
        _LIB.orc_octree_ball_query.restype = ctypes.c_longlong
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(t)


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def voxelization_idx(coords, batchsize=1, mode=4):
    """functions.py:168-197 -> (output_coords i64 [M,ncol], input_map i32 [N], output_map i32 [M,maxActive+1])."""
    coords = _c(coords, np.int64)
    N, ncol = coords.shape
    input_map = np.zeros(N, np.int32)
    M = ctypes.c_int()
    mx = ctypes.c_int()
    h = lib().orc_voxelize_idx_begin(_p(coords, _i64p), N, ncol, mode, _p(input_map, _i32p), ctypes.byref(M),
                                     ctypes.byref(mx))
    out_coords = np.zeros((M.value, ncol), np.int64)
    out_map = np.zeros((M.value, mx.value + 1), np.int32)
    lib().orc_voxelize_idx_finish(ctypes.c_void_p(h), _p(coords, _i64p), _p(out_coords, _i64p), _p(out_map, _i32p))
    return out_coords, input_map, out_map


def voxelization(feats, map_rule, mode=4):
    feats = _c(feats, np.float32)
    map_rule = _c(map_rule, np.int32)
    M, W = map_rule.shape
    C = feats.shape[1]
    out = np.zeros((M, C), np.float32)
    lib().orc_voxelize_fp(_p(feats, _f32p), _p(out, _f32p), _p(map_rule, _i32p), M, W - 1, C, int(mode == 4))
    return out


def voxelization_bp(d_out, map_rule, N, mode=4):
    d_out = _c(d_out, np.float32)
    map_rule = _c(map_rule, np.int32)
    M, W = map_rule.shape
    C = d_out.shape[1]
    d_feats = np.zeros((N, C), np.float32)
    lib().orc_voxelize_bp(_p(d_out, _f32p), _p(d_feats, _f32p), _p(map_rule, _i32p), M, W - 1, C, int(mode == 4))
    return d_feats


def ballquery_batch_p(coords, batch_idxs, batch_offsets, radius, meanActive=None):
    """functions.py:237-275. Returns (idx i32 [nActive], start_len i32 [n,2]); deterministic layout."""
    coords = _c(coords, np.float32)
    batch_idxs = _c(batch_idxs, np.int32)
    batch_offsets = _c(batch_offsets, np.int32)
    n = coords.shape[0]
    start_len = np.zeros((n, 2), np.int32)
    tot = lib().orc_ballquery_batch_p(_p(coords, _f32p), _p(batch_idxs, _i32p), _p(batch_offsets, _i32p), n,
                                      ctypes.c_float(radius), None, ctypes.c_longlong(0), _p(start_len, _i32p))
    idx = np.zeros(max(tot, 1), np.int32)
    lib().orc_ballquery_batch_p(_p(coords, _f32p), _p(batch_idxs, _i32p), _p(batch_offsets, _i32p), n,
                                ctypes.c_float(radius), _p(idx, _i32p), ctypes.c_longlong(tot), _p(start_len, _i32p))
    return idx[:tot], start_len


def ballquery_batch_p_grid(coords, batch_idxs, batch_offsets, radius):
    """ballquery_batch_p's result (same lists, same layout) from a uniform grid of cell edge ~radius: O(n * neighbours)
    instead of O(n * segment size), for segments of hundreds of thousands of points."""
    coords = _c(coords, np.float32)
    batch_idxs = _c(batch_idxs, np.int32)
    batch_offsets = _c(batch_offsets, np.int32)
    n = coords.shape[0]
    nb = batch_offsets.shape[0] - 1
    start_len = np.zeros((n, 2), np.int32)
    args = (_p(coords, _f32p), _p(batch_idxs, _i32p), _p(batch_offsets, _i32p), nb, n, ctypes.c_float(radius))
    tot = lib().orc_ballquery_batch_p_grid(*args, None, ctypes.c_longlong(0), _p(start_len, _i32p))
    idx = np.zeros(max(tot, 1), np.int32)
    lib().orc_ballquery_batch_p_grid(*args, _p(idx, _i32p), ctypes.c_longlong(tot), _p(start_len, _i32p))
    return idx[:tot], start_len


def bfs_cluster(cluster_numpoint_mean, ball_query_idxs, start_len, threshold, class_id):
    """functions.py:278-308 -> (cluster_idxs i32 [sumNPoint,2], cluster_offsets i32 [nCluster+1])."""
    mean = _c(cluster_numpoint_mean, np.float32)
    idxs = _c(ball_query_idxs, np.int32)
    if idxs.size == 0:
        idxs = np.zeros(1, np.int32)
    sl = _c(start_len, np.int32)
    N = sl.shape[0]
    s = ctypes.c_int()
    c = ctypes.c_int()
    h = lib().orc_bfs_cluster_begin(_p(mean, _f32p), _p(idxs, _i32p), _p(sl, _i32p), N, ctypes.c_float(threshold),
                                    int(class_id), ctypes.byref(s), ctypes.byref(c))
    cidx = np.zeros((s.value, 2), np.int32)
    coff = np.zeros(c.value + 1, np.int32)
    lib().orc_bfs_cluster_finish(ctypes.c_void_p(h), _p(cidx, _i32p), _p(coff, _i32p))
    return cidx, coff


def _seg(fn, inp, offsets):
    inp = _c(inp, np.float32)
    offsets = _c(offsets, np.int32)
    nP = offsets.shape[0] - 1
    C = inp.shape[1]
    out = np.zeros((nP, C), np.float32)
    fn(_p(inp, _f32p), _p(offsets, _i32p), _p(out, _f32p), nP, C)
    return out


def sec_mean(inp, offsets):
    return _seg(lib().orc_sec_mean, inp, offsets)


def sec_min(inp, offsets):
    return _seg(lib().orc_sec_min, inp, offsets)


def sec_max(inp, offsets):
    return _seg(lib().orc_sec_max, inp, offsets)


def global_avg_pool(feats, proposals_offset):
    return _seg(lib().orc_global_avg_pool_fp, feats, proposals_offset)


def global_avg_pool_bp(d_out, proposals_offset, sumNPoint):
    d_out = _c(d_out, np.float32)
    off = _c(proposals_offset, np.int32)
    nP, C = d_out.shape
    d_feats = np.zeros((sumNPoint, C), np.float32)
    lib().orc_global_avg_pool_bp(_p(d_feats, _f32p), _p(off, _i32p), _p(d_out, _f32p), nP, C)
    return d_feats


def get_mask_iou_on_cluster(proposals_idx, proposals_offset, instance_labels, instance_pointnum):
    pidx = _c(proposals_idx, np.int32)
    poff = _c(proposals_offset, np.int32)
    lab = _c(instance_labels, np.int64)
    pn = _c(instance_pointnum, np.int32)
    nI, nP = pn.shape[0], poff.shape[0] - 1
    iou = np.zeros((nP, nI), np.float32)
    lib().orc_get_mask_iou_on_cluster(_p(pidx, _i32p), _p(poff, _i32p), _p(lab, _i64p), _p(pn, _i32p), _p(iou, _f32p),
                                      nI, nP)
    return iou


def get_mask_iou_on_pred(proposals_idx, proposals_offset, instance_labels, instance_pointnum, mask_scores_sigmoid):
    pidx = _c(proposals_idx, np.int32)
    poff = _c(proposals_offset, np.int32)
    lab = _c(instance_labels, np.int64)
    pn = _c(instance_pointnum, np.int32)
    ms = _c(mask_scores_sigmoid, np.float32)
    nI, nP = pn.shape[0], poff.shape[0] - 1
    iou = np.zeros((nP, nI), np.float32)
    lib().orc_get_mask_iou_on_pred(_p(pidx, _i32p), _p(poff, _i32p), _p(lab, _i64p), _p(pn, _i32p), _p(iou, _f32p), nI,
                                   nP, _p(ms, _f32p))
    return iou


def get_mask_label(proposals_idx, proposals_offset, instance_labels, instance_cls, instance_pointnum, proposals_iou,
                   iou_thr):
    pidx = _c(proposals_idx, np.int32)
    poff = _c(proposals_offset, np.int32)
    lab = _c(instance_labels, np.int64)
    cls = _c(instance_cls, np.int64)
    iou = _c(proposals_iou, np.float32)
    nP, nI = iou.shape
    ml = np.full(pidx.shape[0], -1.0, np.float32)
    lib().orc_get_mask_label(_p(pidx, _i32p), _p(poff, _i32p), _p(lab, _i64p), _p(cls, _i64p), _p(iou, _f32p), nI, nP,
                             ctypes.c_float(iou_thr), _p(ml, _f32p))
    return ml


def build_octree(coords):
    """functions.py:14-29 + octree_ball_query.cpp:150-165 -> (boxes [585,6], pt_inds [n], pt_start_len [512,2])."""
    coords = _c(coords, np.float32)
    n = coords.shape[0]
    mx, mn = coords.max(0), coords.min(0)
    xyzwhl = np.concatenate([(mx + mn) / np.float32(2), mx - mn]).astype(np.float32)
    boxes = np.zeros((585, 6), np.float32)
    pt_inds = np.zeros(n, np.int32)
    psl = np.zeros((512, 2), np.int32)
    lib().orc_build_octree(_p(coords, _f32p), _p(xyzwhl, _f32p), n, _p(boxes, _f32p), _p(pt_inds, _i32p),
                           _p(psl, _i32p))
    return boxes, pt_inds, psl


def octree_ball_query(coords, mean_active, radius):
    """functions.py:14-44 (leaf-major order, cap 1000)."""
    coords = _c(coords, np.float32)
    n = coords.shape[0]
    boxes, pt_inds, psl = build_octree(coords)
    sl = np.zeros((n, 2), np.int32)
    args = (_p(coords, _f32p), _p(boxes, _f32p), _p(pt_inds, _i32p), _p(psl, _i32p), n, ctypes.c_float(radius))
    tot = lib().orc_octree_ball_query(*args, None, ctypes.c_longlong(0), _p(sl, _i32p))
    idx = np.zeros(max(tot, 1), np.int32)
    lib().orc_octree_ball_query(*args, _p(idx, _i32p), ctypes.c_longlong(tot), _p(sl, _i32p))
    return idx[:tot], sl
