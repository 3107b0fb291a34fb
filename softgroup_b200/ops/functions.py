"""softgroup_b200.ops.functions -- the reference's `softgroup.ops` binding surface on libsgb200.so.

Same names, argument meaning and return layout as softgroup/ops/functions.py of the reference
(thangvubk/SoftGroup): ball_query, ballquery_batch_p, bfs_cluster, voxelization_idx, voxelization,
global_avg_pool, sec_mean/min/max, get_mask_iou_on_cluster, get_mask_iou_on_pred, get_mask_label.
Every op runs in hand-written sm_90a CUDA behind the C ABI of include/sgb200.h; nothing here computes
on the CPU except `voxelization_idx` on CPU tensors (the reference runs it inside DataLoader workers,
softgroup/data/custom.py:239) which calls the library's C++ host path.

Differences that are extensions, not changes:
  * voxelization_idx and bfs_cluster also accept CUDA tensors and then return CUDA tensors
    (the reference only takes CPU tensors there); CPU inputs to bfs_cluster are computed on the GPU and
    returned on the CPU, like `.new()` on the inputs did in the reference (functions.py:295-296).
  * ballquery_batch_p lays the per-point lists out through an atomic cursor exactly like the reference,
    so only `idx[start:start+len]` per point is meaningful (it always was).
"""
import ctypes

import numpy as np
import torch
from torch.autograd import Function

from .. import profiler
from . import _lib
from ._lib import check, ptr, stream as _stream, workspace as _ws


def _cuda(t):
    return t if t.is_cuda else t.cuda()


# ----------------------------------------------------------------------------------------------
# ball query
# ----------------------------------------------------------------------------------------------
def ball_query(coords, batch_idxs, batch_offsets, radius, mean_active, with_octree=False):
    """functions.py:7-11 of the reference."""
    if with_octree:
        return octree_ball_query(coords, mean_active, radius)
    return ballquery_batch_p(coords, batch_idxs, batch_offsets, radius, mean_active)


def build_octree(coords):
    """functions.py:14-29 of the reference, on the GPU: (boxes f32 [585,6], pt_inds i32 [n], pt_start_len i32 [512,2])."""
    L = _lib.lib()
    coords = _cuda(coords).contiguous()
    dev = coords.device
    n = coords.size(0)
    xyz_max = coords.max(0)[0]
    xyz_min = coords.min(0)[0]
    xyzwhl = torch.cat([(xyz_max + xyz_min) / 2, xyz_max - xyz_min]).contiguous()
    boxes = torch.empty((585, 6), dtype=torch.float32, device=dev)
    pt_inds = torch.empty(n, dtype=torch.int32, device=dev)
    pt_start_len = torch.empty((512, 2), dtype=torch.int32, device=dev)
    ws = _ws(L.sgb_octree_workspace_bytes(n), dev)
    with profiler.record('octree_build', 12 * n + 4 * n + 585 * 24 + 4096):
        check(L.sgb_octree_build(ptr(coords), n, ptr(xyzwhl), ptr(boxes), ptr(pt_inds), ptr(pt_start_len), ptr(ws),
                                 ws.numel(), _stream()), 'sgb_octree_build')
    return boxes, pt_inds, pt_start_len


def octree_ball_query(coords, mean_active, radius):
    """functions.py:14-44 of the reference (SoftGroup++): leaf-major neighbour order, first 1000 kept."""
    L = _lib.lib()
    coords = _cuda(coords).contiguous()
    assert coords.is_contiguous()
    dev = coords.device
    n = coords.size(0)
    boxes, pt_inds, pt_start_len = build_octree(coords)
    total = torch.zeros(1, dtype=torch.int32, device=dev)
    mean_active = int(mean_active)
    while True:
        out_inds = torch.empty(max(n * mean_active, 1), dtype=torch.int32, device=dev)
        out_start_len = torch.empty((n, 2), dtype=torch.int32, device=dev)
        rec = profiler.record('octree_ball_query')
        with rec:
            n_totals = check(
                L.sgb_octree_ball_query(ptr(coords), ptr(boxes), ptr(pt_inds), ptr(pt_start_len), n, mean_active,
                                        float(radius), ptr(out_inds), ptr(out_start_len), ptr(total), _stream()),
                'sgb_octree_ball_query')
            rec.nbytes = 24 * n + 585 * 24 + 4 * n + 4096 + 4 * min(n_totals, n * mean_active)
        if n_totals <= n * mean_active:
            break
        mean_active = int(n_totals // n + 1)
    return out_inds[:n_totals], out_start_len


class BallQueryBatchP(Function):
    """functions.py:237-275."""

    @staticmethod
    def forward(ctx, coords, batch_idxs, batch_offsets, radius, meanActive):
        n = coords.size(0)
        assert coords.is_contiguous() and coords.is_cuda
        assert batch_idxs.is_contiguous() and batch_idxs.is_cuda
        assert batch_offsets.is_contiguous() and batch_offsets.is_cuda
        L = _lib.lib()
        dev = coords.device
        B = batch_offsets.numel() - 1
        start_len = torch.empty((n, 2), dtype=torch.int32, device=dev)
        if n == 0:
            return torch.empty(0, dtype=torch.int32, device=dev), start_len
        ws = _ws(L.sgb_ballquery_workspace_bytes(n), dev)
        meanActive = int(meanActive)
        while True:
            idx = torch.empty(max(n * meanActive, 1), dtype=torch.int32, device=dev)
            rec = profiler.record('ballquery_batch_p')
            with rec:
                nActive = check(
                    L.sgb_ballquery_batch_p(n, meanActive, float(radius), ptr(coords), ptr(batch_idxs),
                                            ptr(batch_offsets), B, ptr(idx), ptr(start_len), ptr(ws), ws.numel(),
                                            _stream()), 'sgb_ballquery_batch_p')
                rec.nbytes = 24 * n + 4 * (B + 1) + 4 * min(nActive, n * meanActive)
            if nActive <= n * meanActive:
                break
            meanActive = int(nActive // n + 1)
        return idx[:nActive], start_len

    @staticmethod
    def backward(ctx, a=None, b=None):
        return None, None, None, None, None


ballquery_batch_p = BallQueryBatchP.apply

# most segments (batch_offsets.numel() - 1) one ballquery_batch_p call takes (csrc/ballquery.cu kMaxSeg)
BALLQUERY_MAX_SEGMENTS = 1023
# largest neighbour-index buffer one ball query addresses: its list cursor and start_len are int32
BALLQUERY_MAX_CAPACITY = 2**31 - 1
# flag bit in total[1] of ballquery_batch_p_nosync: the neighbour total passed 2^31 - 1 (csrc/ballquery.cu)
BALLQUERY_ERR_CURSOR = 2


def plan_ballquery_chunks(seg_counts, max_capacity=None):
    """Cut segments into contiguous ranges [s0, s1) for one ball query each, greedily in segment order, so that every
    range's worst-case index buffer (1000 entries per point) fits: sum(seg_counts[s0:s1]) * 1000 <= max_capacity
    (default BALLQUERY_MAX_CAPACITY). A segment that alone exceeds it gets a range of its own. The ranges tile
    [0, len(seg_counts)); a range may hold no entries (empty segments next to an oversize one)."""
    if max_capacity is None:
        max_capacity = BALLQUERY_MAX_CAPACITY
    limit = max_capacity // 1000  # most entries a chunk takes
    chunks, s0, acc = [], 0, 0
    for s, c in enumerate(int(c) for c in seg_counts):
        if c > limit:  # oversize: close the open range, then a range of its own
            if s > s0:
                chunks.append((s0, s))
            chunks.append((s, s + 1))
            s0, acc = s + 1, 0
        elif acc + c > limit:
            chunks.append((s0, s))
            s0, acc = s, c
        else:
            acc += c
    if s0 < len(seg_counts):
        chunks.append((s0, len(seg_counts)))
    return chunks


def ballquery_batch_p_nosync(coords, batch_idxs, batch_offsets, radius, capacity=None):
    """Device-resident variant for the fused forward: the index buffer is sized for the cap (n * 1000 entries, only
    the used prefix is ever touched), so there is no overflow relaunch (functions.py:258-266 of the reference) and
    no host synchronisation. Returns (idx buffer int32 [n*1000], start_len int32 [n,2], total int32 [2] on device:
    [sum of list lengths, error flags]); only idx[start:start+len] per point is meaningful. The error flags are
    reported by the next bfs_cluster_segments(..., upstream_err=total[1:]) at its own synchronisation. The buffer is
    4 KB per entry (0.5 GB at 131k entries, 3.2 GB at 800k); the int32 list cursor limits it to n < 2^31/1000 entries
    (plan_ballquery_chunks cuts larger selections).
    capacity: a smaller buffer (at most BALLQUERY_MAX_CAPACITY) for a segment whose n * 1000 exceeds that; lists beyond
    it are truncated, which total[0] > capacity shows, and a neighbour total beyond 2^31 - 1 sets
    BALLQUERY_ERR_CURSOR in total[1]. The caller has to check both before clustering."""
    n = coords.size(0)
    assert coords.is_contiguous() and coords.is_cuda
    L = _lib.lib()
    dev = coords.device
    B = batch_offsets.numel() - 1
    start_len = torch.empty((n, 2), dtype=torch.int32, device=dev)
    total = torch.zeros(2, dtype=torch.int32, device=dev)
    if capacity is None:
        assert n * 1000 < 2**31, 'ballquery_batch_p_nosync: %d entries need an index buffer beyond the int32 cursor' % n
        cap = max(n, 1) * 1000
    else:
        cap = int(capacity)
        assert 1 <= cap <= BALLQUERY_MAX_CAPACITY, 'ballquery_batch_p_nosync: capacity %d outside [1, 2^31 - 1]' % cap
    idx = torch.empty(cap, dtype=torch.int32, device=dev)
    if n == 0:
        return idx, start_len, total
    ws = _ws(L.sgb_ballquery_workspace_bytes(n), dev)
    # algorithmic bytes need nActive, which stays on the device: resolved lazily when the profiler is summarised
    with profiler.record('ballquery_batch_p', lambda: 24 * n + 4 * (B + 1) + 4 * int(total[0].item())):
        check(
            L.sgb_ballquery_batch_p_async(n, cap, float(radius), ptr(coords), ptr(batch_idxs), ptr(batch_offsets), B,
                                          ptr(idx), ptr(start_len), ptr(total), ptr(ws), ws.numel(), _stream()),
            'sgb_ballquery_batch_p_async')
    return idx, start_len, total


def gather_rows(feats, idx):
    """out[i] = feats[idx[i]] for float32 rows (`x[idx.long()]` of the reference at softgroup.py:374 and :672): float4 rows at
    ~3 TB/s instead of torch's generic int64 gather (0.5 TB/s on 131k x 32 rows)."""
    L = _lib.lib()
    feats = feats.contiguous()
    assert feats.dtype == torch.float32 and feats.dim() == 2 and feats.is_cuda
    idx = idx.int().contiguous()
    n, C = idx.numel(), feats.size(1)
    out = torch.empty((n, C), dtype=torch.float32, device=feats.device)
    if n == 0:
        return out
    with profiler.record('gather_rows', 4 * n + 4 * C * (feats.size(0) + n)):
        check(L.sgb_gather_rows(ptr(feats), ptr(idx), ptr(out), n, C, _stream()), 'sgb_gather_rows')
    return out


def group_entries(scores, classes, score_thr, min_npoint, batch_idxs, batch_size, coords_float, pt_offsets):
    """All classes of the grouping loop (softgroup/model/softgroup.py:430-446) in one pass on the device: entries in
    class-major, ascending point order. scores: softmax scores [N, C]; classes: list of class ids (any number).
    Returns (pts int32 [cap], seg int32 [cap], shifted float32 [cap, 3], seg_offsets int32 [nc*B+1], total int32 [1+nc]) with
    cap = N * len(classes); only the first total[0] entries are meaningful. No host synchronisation."""
    L = _lib.lib()
    dev = scores.device
    N, C = scores.shape
    nc = len(classes)
    cap = max(N * nc, 1)
    pts = torch.empty(cap, dtype=torch.int32, device=dev)
    seg = torch.empty(cap, dtype=torch.int32, device=dev)
    shifted = torch.empty((cap, 3), dtype=torch.float32, device=dev)
    seg_offsets = torch.empty(nc * batch_size + 1, dtype=torch.int32, device=dev)
    total = torch.empty(1 + nc, dtype=torch.int32, device=dev)
    ws = _ws(L.sgb_group_entries_workspace_bytes(N, nc, batch_size), dev)
    cls = (ctypes.c_int * nc)(*[int(c) for c in classes])
    scores = scores.contiguous()
    batch_idxs = batch_idxs.int().contiguous()
    coords_float = coords_float.float().contiguous()
    pt_offsets = pt_offsets.float().contiguous()
    with profiler.record('group_entries', 4 * N * C + 28 * N):
        check(
            L.sgb_group_entries(ptr(scores), N, C, cls, nc, float(score_thr), int(min_npoint), ptr(batch_idxs), int(batch_size),
                                ptr(coords_float), ptr(pt_offsets), ptr(pts), ptr(seg), ptr(shifted), ptr(seg_offsets), ptr(total),
                                ptr(ws), ws.numel(), _stream()), 'sgb_group_entries')
    return pts, seg, shifted, seg_offsets, total


# ----------------------------------------------------------------------------------------------
# clustering
# ----------------------------------------------------------------------------------------------
def cluster_threshold(npoint_thr, class_numpoint_mean):
    """Smallest component size kept for one class (bfs_cluster.cpp:70-77 of the reference): npoint_thr * class mean
    in float32 arithmetic like the C++ (`thr = threshold * _class_numpoint_mean`, both float), or npoint_thr itself
    when the class mean is -1."""
    if class_numpoint_mean == -1:
        return float(npoint_thr)
    return float(np.float32(npoint_thr) * np.float32(class_numpoint_mean))


def bfs_cluster_segments(ball_query_idxs, start_len, thr, node_seg=None, seg_thr=None, nactive=None,
                         upstream_err=None):
    """GPU clustering on device tensors. thr: float threshold on the component size (cluster_threshold of the class).
    Optional per-node segment thresholds. Returns CUDA tensors
    (cluster_idxs int32 [sumNPoint,2], cluster_offsets int32 [nCluster+1])."""
    L = _lib.lib()
    dev = start_len.device
    N = start_len.size(0)
    if ball_query_idxs.numel() == 0:  # no neighbours at all: a one-word buffer, never read, in place of an empty one
        ball_query_idxs = torch.zeros(1, dtype=torch.int32, device=dev)
    ws = _ws(L.sgb_bfs_cluster_workspace_bytes(N), dev)
    s = ctypes.c_int(0)
    mx = ctypes.c_int(0)
    nact = ball_query_idxs.numel() if nactive is None else nactive
    nb = (lambda: int(nact.item())) if torch.is_tensor(nact) else (lambda: int(nact))
    with profiler.record('bfs_cluster(label)', lambda: 8 * N + 4 * nb()):
        nC = check(
            L.sgb_bfs_cluster_count(ptr(ball_query_idxs), ptr(start_len), N, float(thr), ptr(node_seg), ptr(seg_thr),
                                    ptr(upstream_err), ptr(ws), ws.numel(), ctypes.byref(s), ctypes.byref(mx),
                                    _stream()),
            'sgb_bfs_cluster_count')
    cluster_idxs = torch.empty((s.value, 2), dtype=torch.int32, device=dev)
    cluster_offsets = torch.empty(nC + 1, dtype=torch.int32, device=dev)
    scratch = _ws(L.sgb_bfs_cluster_scratch_bytes(s.value, mx.value), dev)
    with profiler.record('bfs_cluster(emit)', lambda: 8 * N + 4 * nb() + 8 * s.value + 4 * (nC + 1)):
        check(
            L.sgb_bfs_cluster_fill(ptr(ball_query_idxs), ptr(start_len), N, nC, s.value, mx.value, ptr(cluster_idxs),
                                   ptr(cluster_offsets), ptr(ws), ws.numel(), ptr(scratch), scratch.numel(),
                                   _stream()), 'sgb_bfs_cluster_fill')
    return cluster_idxs, cluster_offsets


# PyTorch >= 2 compatibility of the UNMODIFIED reference model: its bfs_cluster wrapper returns CPU tensors
# (functions.py:295-301: `.new()` on the CPU inputs of softgroup.py:458) and get_instances later indexes that CPU tensor
# with a CUDA boolean mask (softgroup.py:570) -- accepted by the PyTorch 1.x the reference was written for, an error today.
# install_as_reference_backends(torch2_compat=True) makes this wrapper return the same CPU data as a tensor subclass whose
# indexing moves CUDA index tensors to the host first (what PyTorch 1.x did implicitly). Off by default.
TORCH2_COMPAT = False


class HostIndexTensor(torch.Tensor):
    """CPU tensor that accepts CUDA index / mask tensors in `t[idx]` by copying them to the host."""

    @staticmethod
    def __new__(cls, t):
        return torch.Tensor._make_subclass(cls, t)

    def __getitem__(self, idx):
        if torch.is_tensor(idx) and idx.is_cuda:
            idx = idx.cpu()
        elif isinstance(idx, tuple):
            idx = tuple(i.cpu() if (torch.is_tensor(i) and i.is_cuda) else i for i in idx)
        return super().__getitem__(idx)


class BFSCluster(Function):
    """functions.py:278-308. threshold semantics of bfs_cluster.cpp:70-82."""

    @staticmethod
    def forward(ctx, cluster_numpoint_mean, ball_query_idxs, start_len, threshold, class_id):
        assert cluster_numpoint_mean.is_contiguous()
        assert ball_query_idxs.is_contiguous()
        assert start_len.is_contiguous()
        thr = cluster_threshold(threshold, float(cluster_numpoint_mean[class_id]))
        on_cpu = not ball_query_idxs.is_cuda
        cidx, coff = bfs_cluster_segments(_cuda(ball_query_idxs), _cuda(start_len), thr)
        if on_cpu:
            cidx, coff = cidx.cpu(), coff.cpu()
            if TORCH2_COMPAT:
                cidx = HostIndexTensor(cidx)
        return cidx, coff

    @staticmethod
    def backward(ctx, a=None, b=None):
        return None, None, None, None, None


bfs_cluster = BFSCluster.apply


# ----------------------------------------------------------------------------------------------
# voxelisation
# ----------------------------------------------------------------------------------------------
class Voxelization_Idx(Function):
    """functions.py:168-197 -> (output_coords, input_map, output_map)."""

    @staticmethod
    def forward(ctx, coords, batchsize, mode=4):
        assert coords.is_contiguous() and coords.dtype == torch.int64
        L = _lib.lib()
        N, ncol = coords.size(0), coords.size(1)
        M = ctypes.c_int(0)
        mx = ctypes.c_int(0)
        if coords.is_cuda:
            dev = coords.device
            input_map = torch.empty(N, dtype=torch.int32, device=dev)
            ws = _ws(L.sgb_voxelize_idx_workspace_bytes(N), dev)
            rec = profiler.record('voxelize_idx')
            with rec:
                check(
                    L.sgb_voxelize_idx_count(ptr(coords), N, ncol, int(mode), ptr(input_map), ptr(ws), ws.numel(),
                                             ctypes.byref(M), ctypes.byref(mx), _stream()), 'sgb_voxelize_idx_count')
                output_coords = torch.empty((M.value, ncol), dtype=torch.int64, device=dev)
                output_map = torch.empty((M.value, mx.value + 1), dtype=torch.int32, device=dev)
                check(
                    L.sgb_voxelize_idx_fill(ptr(coords), N, ncol, int(mode), M.value, mx.value, ptr(output_coords),
                                            ptr(output_map), ptr(ws), ws.numel(), _stream()), 'sgb_voxelize_idx_fill')
                rec.nbytes = 8 * ncol * N + 4 * N + 8 * ncol * M.value + 4 * M.value * (mx.value + 1)
            return output_coords, input_map, output_map
        input_map = torch.zeros(N, dtype=torch.int32)
        h = L.sgb_voxelize_idx_cpu_begin(ptr(coords), N, ncol, int(mode), ptr(input_map), ctypes.byref(M),
                                         ctypes.byref(mx))
        check(h, 'sgb_voxelize_idx_cpu_begin')
        output_coords = torch.zeros((M.value, ncol), dtype=torch.int64)
        output_map = torch.zeros((M.value, mx.value + 1), dtype=torch.int32)
        check(L.sgb_voxelize_idx_cpu_finish(ctypes.c_void_p(h), ptr(coords), ptr(output_coords), ptr(output_map)),
              'sgb_voxelize_idx_cpu_finish')
        return output_coords, input_map, output_map

    @staticmethod
    def backward(ctx, a=None, b=None, c=None):
        return None, None, None


voxelization_idx = Voxelization_Idx.apply


class Voxelization(Function):
    """functions.py:200-234."""

    @staticmethod
    def forward(ctx, feats, map_rule, mode=4):
        assert map_rule.is_contiguous()
        assert feats.is_contiguous()
        assert feats.is_cuda and map_rule.is_cuda and feats.dtype == torch.float32
        N, C = feats.size()
        M = map_rule.size(0)
        maxActive = map_rule.size(1) - 1
        output_feats = torch.empty((M, C), dtype=torch.float32, device=feats.device)
        ctx.for_backwards = (map_rule, mode, maxActive, N)
        with profiler.record('voxelize_fp', 4 * M * (maxActive + 1) + 4 * C * (N + M)):
            check(
                _lib.lib().sgb_voxelize_fp(ptr(feats), ptr(output_feats), ptr(map_rule), int(mode), M, maxActive, C,
                                           _stream()), 'sgb_voxelize_fp')
        return output_feats

    @staticmethod
    def backward(ctx, d_output_feats):
        map_rule, mode, maxActive, N = ctx.for_backwards
        M, C = d_output_feats.size()
        d_feats = torch.zeros((N, C), dtype=torch.float32, device=d_output_feats.device)
        d_out = d_output_feats.contiguous()
        check(
            _lib.lib().sgb_voxelize_bp(ptr(d_out), ptr(d_feats), ptr(map_rule), int(mode), M, maxActive, C, _stream()),
            'sgb_voxelize_bp')
        return d_feats, None, None


voxelization = Voxelization.apply


# ----------------------------------------------------------------------------------------------
# pooling / segment reductions
# ----------------------------------------------------------------------------------------------
class GlobalAvgPool(Function):
    """functions.py:311-348."""

    @staticmethod
    def forward(ctx, feats, proposals_offset):
        nProposal = proposals_offset.size(0) - 1
        sumNPoint, C = feats.size()
        assert feats.is_contiguous() and feats.is_cuda
        assert proposals_offset.is_contiguous() and proposals_offset.is_cuda
        output_feats = torch.empty((nProposal, C), dtype=torch.float32, device=feats.device)
        with profiler.record('global_avg_pool', 4 * C * sumNPoint + 4 * (nProposal + 1) + 4 * C * nProposal):
            check(
                _lib.lib().sgb_global_avg_pool_fp(ptr(feats), ptr(proposals_offset), ptr(output_feats), nProposal, C,
                                                  _stream()), 'sgb_global_avg_pool_fp')
        ctx.for_backwards = (proposals_offset, sumNPoint)
        return output_feats

    @staticmethod
    def backward(ctx, d_output_feats):
        nProposal, C = d_output_feats.size()
        proposals_offset, sumNPoint = ctx.for_backwards
        d_feats = torch.zeros((sumNPoint, C), dtype=torch.float32, device=d_output_feats.device)
        d_out = d_output_feats.contiguous()
        check(
            _lib.lib().sgb_global_avg_pool_bp(ptr(d_feats), ptr(proposals_offset), ptr(d_out), nProposal, C, _stream()),
            'sgb_global_avg_pool_bp')
        return d_feats, None


global_avg_pool = GlobalAvgPool.apply


def _sec(name):

    class _Sec(Function):
        """functions.py:351-438 (SecMean / SecMin / SecMax)."""

        @staticmethod
        def forward(ctx, inp, offsets):
            nProposal = offsets.size(0) - 1
            C = inp.size(1)
            assert inp.is_contiguous() and inp.is_cuda
            assert offsets.is_contiguous() and offsets.is_cuda
            out = torch.empty((nProposal, C), dtype=torch.float32, device=inp.device)
            with profiler.record(name[4:], 4 * C * inp.size(0) + 4 * (nProposal + 1) + 4 * C * nProposal):
                check(getattr(_lib.lib(), name)(ptr(inp), ptr(offsets), ptr(out), nProposal, C, _stream()), name)
            return out

        @staticmethod
        def backward(ctx, a=None):
            return None, None

    _Sec.__name__ = name
    return _Sec.apply


sec_mean = _sec('sgb_sec_mean')
sec_min = _sec('sgb_sec_min')
sec_max = _sec('sgb_sec_max')


# ----------------------------------------------------------------------------------------------
# mask IoU / labels (training-side members of the binding surface)
# ----------------------------------------------------------------------------------------------
def _pidx_col(proposals_idx):
    # the reference passes proposals_idx[:, 1].contiguous() (softgroup/model/softgroup.py:189-191)
    assert proposals_idx.dim() == 1
    return proposals_idx


class GetMaskIoUOnCluster(Function):
    """functions.py:47-83."""

    @staticmethod
    def forward(ctx, proposals_idx, proposals_offset, instance_labels, instance_pointnum):
        nInstance = instance_pointnum.size(0)
        nProposal = proposals_offset.size(0) - 1
        assert proposals_idx.is_contiguous() and proposals_idx.is_cuda
        assert proposals_offset.is_contiguous() and proposals_offset.is_cuda
        assert instance_labels.is_contiguous() and instance_labels.is_cuda
        assert instance_pointnum.is_contiguous() and instance_pointnum.is_cuda
        proposals_iou = torch.zeros((nProposal, nInstance), dtype=torch.float32, device=proposals_idx.device)
        check(
            _lib.lib().sgb_get_mask_iou(ptr(_pidx_col(proposals_idx)), ptr(proposals_offset), ptr(instance_labels),
                                        ptr(instance_pointnum), None, ptr(proposals_iou), nInstance, nProposal,
                                        _stream()), 'sgb_get_mask_iou')
        return proposals_iou

    @staticmethod
    def backward(ctx, a=None):
        return None, None, None, None


get_mask_iou_on_cluster = GetMaskIoUOnCluster.apply


class GetMaskIoUOnPred(Function):
    """functions.py:86-125."""

    @staticmethod
    def forward(ctx, proposals_idx, proposals_offset, instance_labels, instance_pointnum, mask_scores_sigmoid):
        nInstance = instance_pointnum.size(0)
        nProposal = proposals_offset.size(0) - 1
        assert proposals_idx.is_contiguous() and proposals_idx.is_cuda
        assert proposals_offset.is_contiguous() and proposals_offset.is_cuda
        assert instance_labels.is_contiguous() and instance_labels.is_cuda
        assert instance_pointnum.is_contiguous() and instance_pointnum.is_cuda
        assert mask_scores_sigmoid.is_contiguous() and mask_scores_sigmoid.is_cuda
        proposals_iou = torch.zeros((nProposal, nInstance), dtype=torch.float32, device=proposals_idx.device)
        check(
            _lib.lib().sgb_get_mask_iou(ptr(_pidx_col(proposals_idx)), ptr(proposals_offset), ptr(instance_labels),
                                        ptr(instance_pointnum), ptr(mask_scores_sigmoid), ptr(proposals_iou), nInstance,
                                        nProposal, _stream()), 'sgb_get_mask_iou')
        return proposals_iou

    @staticmethod
    def backward(ctx, a=None):
        return None, None, None, None, None


get_mask_iou_on_pred = GetMaskIoUOnPred.apply


class GetMaskLabel(Function):
    """functions.py:128-165."""

    @staticmethod
    def forward(ctx, proposals_idx, proposals_offset, instance_labels, instance_cls, instance_pointnum, proposals_iou,
                iou_thr):
        nInstance = instance_pointnum.size(0)
        nProposal = proposals_offset.size(0) - 1
        assert proposals_iou.is_contiguous() and proposals_iou.is_cuda
        assert proposals_idx.is_contiguous() and proposals_idx.is_cuda
        assert proposals_offset.is_contiguous() and proposals_offset.is_cuda
        assert instance_labels.is_contiguous() and instance_labels.is_cuda
        assert instance_cls.is_contiguous() and instance_cls.is_cuda
        mask_label = torch.full(proposals_idx.shape, -1.0, dtype=torch.float32, device=proposals_idx.device)
        check(
            _lib.lib().sgb_get_mask_label(ptr(_pidx_col(proposals_idx)), ptr(proposals_offset), ptr(instance_labels),
                                          ptr(instance_cls), ptr(proposals_iou), nInstance, nProposal, float(iou_thr),
                                          ptr(mask_label), _stream()), 'sgb_get_mask_label')
        return mask_label

    @staticmethod
    def backward(ctx, a=None):
        return None, None, None, None, None, None, None


get_mask_label = GetMaskLabel.apply
