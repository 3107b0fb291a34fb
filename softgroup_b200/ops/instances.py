"""Instance masks / RLE / panoptic paste / evaluation intersections on the GPU (csrc/instances.cu through the C ABI).

Python mirror of the pieces of softgroup/model/softgroup.py:537-639 and softgroup/evaluation/instance_eval.py:228-309
that the reference runs as dense [nProposal, N] tensors + numpy loops. CUDA tensors only: there is no CPU fallback."""
import ctypes

import numpy as np
import torch

from .. import profiler
from . import _lib
from ._lib import check, ptr, stream as _stream, workspace as _ws


def bitmap_words(n_points):
    return (int(n_points) + 1 + 31) // 32


def instance_point_counts(proposals_idx, mask_scores, n_classes, thr, n_proposals):
    """npoint int32 [nP, nI]: #entries of proposal p with mask_scores[e, i] > thr (softgroup.py:553,563 `mask_pred.sum(1)`)."""
    assert proposals_idx.is_cuda and mask_scores.is_cuda and proposals_idx.dtype == torch.int32
    assert proposals_idx.is_contiguous() and mask_scores.stride(1) == 1 and mask_scores.dtype == torch.float32
    S = proposals_idx.size(0)
    npoint = torch.empty((n_proposals, n_classes), dtype=torch.int32, device=proposals_idx.device)
    with profiler.record('inst_count', 8 * S + 4 * S * n_classes):
        check(_lib.lib().sgb_inst_count(ptr(proposals_idx), ptr(mask_scores), mask_scores.stride(0), S, n_classes, float(thr),
                                        ptr(npoint), n_proposals, _stream()), 'sgb_inst_count')
    return npoint


def instance_bitmaps(proposals_idx, mask_scores, n_classes, thr, keep, n_points):
    """keep bool [nP, nI] -> (bitmaps int32 [n_inst, W], kept class int64 [n_inst], kept proposal int64 [n_inst]) in the
    reference's instance order (class-major, proposal order; softgroup.py:551-603)."""
    dev = proposals_idx.device
    nP = keep.size(0)
    kflat = keep.t().contiguous().view(-1)  # class-major
    slot = (torch.cumsum(kflat.int(), 0) - 1).int()
    slot = torch.where(kflat, slot, torch.full_like(slot, -1)).contiguous()
    kc, kp = keep.t().nonzero(as_tuple=True)
    n_inst = int(kc.numel())  # one small read-back: the bitmap allocation needs it
    W = bitmap_words(n_points)
    bm = torch.empty((n_inst, W), dtype=torch.int32, device=dev)
    with profiler.record('inst_scatter', 8 * proposals_idx.size(0) + 4 * n_inst * W):
        check(_lib.lib().sgb_inst_scatter(ptr(proposals_idx), ptr(mask_scores), mask_scores.stride(0), proposals_idx.size(0),
                                          n_classes, nP, float(thr), ptr(slot), ptr(bm), n_inst, int(n_points), _stream()),
              'sgb_inst_scatter')
    return bm, kc, kp


def scatter_instance_bitmaps(proposals_idx, mask_scores, n_classes, thr, slot, n_rows, n_points):
    """slot int32 [nI, nP] (class-major: bitmap row of (class i, proposal p), or -1) -> bitmaps int32 [n_rows, W], zeroed,
    with the mask of every slotted pair set (rows without a pair stay zero). No host wait."""
    assert slot.dtype == torch.int32 and slot.is_contiguous() and slot.size(0) == n_classes
    bm = torch.empty((n_rows, bitmap_words(n_points)), dtype=torch.int32, device=proposals_idx.device)
    with profiler.record('inst_scatter', 8 * proposals_idx.size(0) + 4 * bm.numel()):
        check(_lib.lib().sgb_inst_scatter(ptr(proposals_idx), ptr(mask_scores), mask_scores.stride(0), proposals_idx.size(0),
                                          n_classes, slot.size(1), float(thr), ptr(slot), ptr(bm), n_rows, int(n_points),
                                          _stream()), 'sgb_inst_scatter')
    return bm


def bitmaps_from_pairs(rows, points, n_rows, n_points):
    """(row, point) int32 pairs -> bitmaps int32 [n_rows, W] (rows < 0 are skipped)."""
    assert rows.is_cuda and rows.dtype == torch.int32 and points.dtype == torch.int32
    W = bitmap_words(n_points)
    bm = torch.empty((n_rows, W), dtype=torch.int32, device=rows.device)
    check(_lib.lib().sgb_bitmap_set(ptr(rows.contiguous()), ptr(points.contiguous()), rows.numel(), ptr(bm), n_rows, int(n_points), 1,
                                    _stream()), 'sgb_bitmap_set')
    return bm


def bitmaps_to_rle(bitmaps, n_points):
    """bitmaps int32 [n_inst, W] (CUDA) -> list of the reference's RLE dicts (rle.py:5-19). Run boundaries are found on
    the GPU; only the transition positions (2 ints per run) cross PCIe; the strings are formatted by the host routine."""
    n_inst = bitmaps.size(0)
    if n_inst == 0:
        return []
    L = _lib.lib()
    dev = bitmaps.device
    ws = _ws(L.sgb_rle_workspace_bytes(n_inst, int(n_points)), dev)
    with profiler.record('rle_runs', 8 * bitmaps.numel()):
        total = check(L.sgb_rle_count(ptr(bitmaps), n_inst, int(n_points), ptr(ws), ws.numel(), _stream()), 'sgb_rle_count')
        trans = torch.empty(max(total, 1), dtype=torch.int32, device=dev)
        inst_off = torch.empty(n_inst + 1, dtype=torch.int32, device=dev)
        check(L.sgb_rle_fill(ptr(bitmaps), n_inst, int(n_points), total, ptr(trans), ptr(inst_off), ptr(ws), ws.numel(), _stream()),
              'sgb_rle_fill')
    h_trans = torch.empty(max(total, 1), dtype=torch.int32, pin_memory=True)
    h_off = torch.empty(n_inst + 1, dtype=torch.int32, pin_memory=True)
    h_trans.copy_(trans, non_blocking=True)
    h_off.copy_(inst_off, non_blocking=True)
    torch.cuda.current_stream().synchronize()
    return format_runs(h_trans.numpy(), h_off.numpy(), n_points)


def format_runs(trans, offs, length):
    """Host: transition positions (1-based, ascending per mask) + offsets int32 [n+1] -> list of rle dicts."""
    trans = np.ascontiguousarray(trans, dtype=np.int32)
    offs = np.ascontiguousarray(offs, dtype=np.int32)
    n = offs.size - 1
    if n <= 0:
        return []
    cap = int(offs[-1]) * 12 + 64 * n + 64
    out = np.empty(cap, dtype=np.uint8)
    out_offs = np.empty(n + 1, dtype=np.int64)
    written = check(
        _lib.lib().sgb_rle_format_runs(trans.ctypes.data_as(ctypes.c_void_p), offs.ctypes.data_as(ctypes.c_void_p), n,
                                       out.ctypes.data_as(ctypes.c_void_p), cap, out_offs.ctypes.data_as(ctypes.c_void_p)),
        'sgb_rle_format_runs')
    buf = out[:written].tobytes()
    o = out_offs.tolist()
    return [dict(length=int(length), counts=buf[o[k]:o[k + 1]].decode('ascii')) for k in range(n)]


def bitmap_intersections(bitmaps, gslot, n_gt, n_points):
    """-> (inter int32 [n_rows, n_gt], vert int32 [n_rows], void int32 [n_rows]); gslot int32 [N]: gt column, -2 void, -1 other."""
    n_rows = bitmaps.size(0)
    dev = bitmaps.device
    inter = torch.empty((n_rows, max(n_gt, 1)), dtype=torch.int32, device=dev)
    vert = torch.empty(n_rows, dtype=torch.int32, device=dev)
    void = torch.empty(n_rows, dtype=torch.int32, device=dev)
    check(_lib.lib().sgb_bitmap_intersections(ptr(bitmaps), n_rows, int(n_points), ptr(gslot.contiguous()), int(n_gt), ptr(inter),
                                              ptr(vert), ptr(void), _stream()), 'sgb_bitmap_intersections')
    return inter[:, :n_gt], vert, void


def to_device_async(a, dtype, device):
    """Small host array -> CUDA tensor without a host wait: staged in pinned memory, copied on the current stream (torch's
    caching host allocator keeps the pinned block until the copy has run)."""
    h = torch.from_numpy(np.ascontiguousarray(a)).to(dtype).pin_memory()
    return h.to(device, non_blocking=True)


def bitmap_point_ids(bitmaps, n_points, total=None):
    """bitmaps int32 [n_rows, W] (CUDA) -> (offsets int64 [n_rows + 1], ids int32 [total]): the ids of row r, ascending, are
    ids[offsets[r]:offsets[r + 1]]; bits at n_points and beyond are ignored. `total` sizes `ids` when the caller knows the
    number of set bits; otherwise it is read back (one host wait between the count and the fill pass)."""
    assert bitmaps.is_cuda and bitmaps.dtype == torch.int32 and bitmaps.is_contiguous()
    n_rows = bitmaps.size(0)
    assert bitmaps.size(1) == bitmap_words(n_points) or n_rows == 0
    L = _lib.lib()
    dev = bitmaps.device
    offsets = torch.empty(n_rows + 1, dtype=torch.int64, device=dev)
    ws = _ws(L.sgb_bitmap_ids_workspace_bytes(n_rows, int(n_points)), dev)
    with profiler.record('bitmap_ids_count', 4 * bitmaps.numel()):
        check(L.sgb_bitmap_ids_count(ptr(bitmaps), n_rows, int(n_points), ptr(offsets), ptr(ws), ws.numel(), _stream()),
              'sgb_bitmap_ids_count')
    if total is None:
        total = int(offsets[-1].item())
    ids = torch.empty(max(int(total), 1), dtype=torch.int32, device=dev)
    with profiler.record('bitmap_ids_fill', 4 * bitmaps.numel() + 4 * int(total)):
        check(L.sgb_bitmap_ids_fill(ptr(bitmaps), n_rows, int(n_points), ptr(ids), ptr(ws), ws.numel(), _stream()),
              'sgb_bitmap_ids_fill')
    return offsets, ids[:int(total)]


def class_bitmaps(labels, classes, n_points):
    """labels int64 [N] (CUDA), classes: distinct non-negative ints (host) -> (bitmaps int32 [len(classes), W] with row k
    marking the points labelled classes[k], counts int64 [len(classes)] of their set bits). No host wait."""
    assert labels.is_cuda and labels.dtype == torch.int64 and labels.is_contiguous() and labels.numel() == int(n_points)
    classes = [int(c) for c in classes]
    assert len(set(classes)) == len(classes) and all(c >= 0 for c in classes)
    dev = labels.device
    n_rows = len(classes)
    row_of = np.full(max(classes) + 1 if classes else 0, -1, np.int32)
    row_of[classes] = np.arange(n_rows, dtype=np.int32)
    row_of_d = to_device_async(row_of, torch.int32, dev)
    bm = torch.empty((n_rows, bitmap_words(n_points)), dtype=torch.int32, device=dev)
    counts = torch.empty(n_rows, dtype=torch.int64, device=dev)
    with profiler.record('class_bitmaps', 8 * int(n_points) + 4 * bm.numel()):
        check(_lib.lib().sgb_class_bitmaps(ptr(labels), int(n_points), ptr(row_of_d), row_of.size, ptr(bm), n_rows, ptr(counts),
                                           _stream()), 'sgb_class_bitmaps')
    return bm, counts


REDUCE_OPS = {'min': 1, 'max': 2, 'mean': 4}  # SGB_REDUCE_* of include/sgb200.h


def _id_lists(instances):
    off, ids = instances['point_offsets'], instances['point_ids']
    assert off.is_cuda and off.dtype == torch.int64 and off.is_contiguous() and off.dim() == 1 and off.numel() >= 1
    assert ids.is_cuda and ids.dtype == torch.int32 and ids.is_contiguous() and ids.device == off.device
    return off, ids, off.numel() - 1, ids.numel()


def instance_point_reduce(instances, values, ops=('min', 'max', 'mean')):
    """Per instance and channel, min / max / mean of `values` over the instance's points, without gathering them.

    instances: the `instances` dict of forward_test(device_results=True) (or any int64 `point_offsets` [n + 1] and int32
    `point_ids` [point_offsets[n]] on the GPU); values: float32 CUDA [N, C] indexed by point id, rows may be strided
    (stride(1) == 1). Under lvl_fusion the lists already hold point ids (not voxel rows), so `values` are per point, like
    the dict's `offset_preds`. Returns dict(op -> float32 [n, C] for each op asked for, counts -> int64 [n]). min / max are
    exact (NaN never wins; an empty instance gives +inf / -inf); mean has the same bits on every run, within the bound
    stated in include/sgb200.h (sgb_id_lists_reduce), NaN for an empty instance. Enqueued on the current stream, no host
    wait. Example, boxes and centroids: r = instance_point_reduce(inst, coords_float); r['min'], r['max'], r['mean']."""
    off, ids, n, total = _id_lists(instances)
    assert values.is_cuda and values.dtype == torch.float32 and values.dim() == 2 and values.device == off.device
    assert values.size(1) >= 1 and (values.stride(1) == 1 or values.size(1) == 1)
    ops = tuple(ops)
    assert ops and all(o in REDUCE_OPS for o in ops) and len(set(ops)) == len(ops), ops
    N, C = values.shape
    ld = values.stride(0) if N > 1 else C
    dev = off.device
    out = {o: torch.empty((n, C), dtype=torch.float32, device=dev) for o in ops}
    out['counts'] = torch.empty(n, dtype=torch.int64, device=dev)
    L = _lib.lib()
    ws = _ws(L.sgb_id_lists_reduce_workspace_bytes(total, C), dev)
    with profiler.record('id_lists_reduce', 8 * (n + 1) + 4 * total + 4 * C * total + 4 * C * n * len(ops)):
        check(L.sgb_id_lists_reduce(ptr(off), ptr(ids), n, total, N, ptr(values), ld, C, sum(REDUCE_OPS[o] for o in ops),
                                    ptr(out.get('min')), ptr(out.get('max')), ptr(out.get('mean')), ptr(out['counts']), ptr(ws),
                                    ws.numel(), _stream()), 'sgb_id_lists_reduce')
    return out


def instance_farthest_point_sample(instances, coords, num_samples):
    """A fixed number of points per instance by farthest-point sampling: int32 CUDA [n, num_samples] of point ids.

    instances: the `instances` dict of forward_test(device_results=True) (or any int64 `point_offsets` [n + 1] and int32
    `point_ids` on the GPU); coords: float32 CUDA [N, 3] indexed by point id, rows may be strided (stride(1) == 1); under
    lvl_fusion the lists hold point ids, so coords are per point (coords_float). num_samples (K): any int >= 1.

    Semantics (include/sgb200.h, sgb_id_lists_fps): ids outside [0, N) are never read nor chosen; a list with no such id
    gives a row of -1. The first sample is the list's first valid id. Every later one is the valid position farthest from
    those chosen so far (min over them of the float32 squared distance, computed as (dx*dx + dy*dy) + dz*dz, rounded to
    nearest with no contraction, NaN propagating); a NaN distance ranks below every number, and ties go to the smaller
    position. A list with fewer distinct points than K repeats one id in its tail, as PointNet++ pads. The result does not
    depend on execution order. Enqueued on the current stream, no host wait.
    Example: ids = instance_farthest_point_sample(ret['instances'], coords_float, 1024); coords_float[ids.long()] is
    [n, 1024, 3]."""
    off, ids, n, total = _id_lists(instances)
    assert coords.is_cuda and coords.dtype == torch.float32 and coords.dim() == 2 and coords.size(1) == 3
    assert coords.stride(1) == 1 and coords.device == off.device
    K = int(num_samples)
    assert K >= 1, num_samples
    N = coords.size(0)
    ld = coords.stride(0) if N > 1 else 3
    out = torch.empty((n, K), dtype=torch.int32, device=off.device)
    L = _lib.lib()
    ws = _ws(L.sgb_id_lists_fps_workspace_bytes(n, total), off.device)
    with profiler.record('id_lists_fps', 8 * (n + 1) + 16 * total + 4 * n * K):
        check(L.sgb_id_lists_fps(ptr(off), ptr(ids), n, total, N, ptr(coords), ld, K, ptr(out), ptr(ws), ws.numel(), _stream()),
              'sgb_id_lists_fps')
    return out


def instance_point_map(instances, num_points):
    """One instance per point: int32 CUDA [num_points], the k of the highest-confidence instance (instances['conf']) that
    holds the point; ties go to the smaller k, a NaN confidence ranks below every number, a point in no instance gets -1.
    Takes the `instances` dict of forward_test(device_results=True) (point ids, also under lvl_fusion). Enqueued on the
    current stream, no host wait; the result does not depend on execution order."""
    off, ids, n, total = _id_lists(instances)
    conf = instances['conf']
    assert conf.is_cuda and conf.dtype == torch.float32 and conf.is_contiguous() and conf.numel() == n
    N = int(num_points)
    dev = off.device
    out = torch.empty(N, dtype=torch.int32, device=dev)
    L = _lib.lib()
    ws = _ws(L.sgb_id_lists_point_map_workspace_bytes(N), dev)
    with profiler.record('id_lists_point_map', 8 * (n + 1) + 4 * n + 4 * total + 20 * N):
        check(L.sgb_id_lists_point_map(ptr(off), ptr(ids), n, total, N, ptr(conf), ptr(out), ptr(ws), ws.numel(), _stream()),
              'sgb_id_lists_point_map')
    return out


def panoptic_paste(bitmaps, order, cls_values, semantic_preds, skip_iou, n_points):
    """softgroup.py:606-632 on bitmaps: -> (panoptic_cls uint32-valued int64 [N], panoptic_ids int64 [N]) CUDA tensors."""
    dev = bitmaps.device
    W = bitmap_words(n_points)
    pan_cls = semantic_preds.to(torch.int32).contiguous().clone()
    pan_ids = torch.zeros(int(n_points), dtype=torch.int32, device=dev)
    prev = torch.empty(W, dtype=torch.int32, device=dev)
    check(_lib.lib().sgb_panoptic_paste(ptr(bitmaps), int(n_points), ptr(order.int().contiguous()), ptr(cls_values.int().contiguous()),
                                        int(order.numel()), float(skip_iou), ptr(prev), ptr(pan_cls), ptr(pan_ids), _stream()),
          'sgb_panoptic_paste')
    return pan_cls, pan_ids
