"""Host restatement of the reference's SoftGroup.forward_test (softgroup/model/softgroup.py:300-361), one function per
stage, for comparing the CUDA forward stage by stage (tests/test_gpu_forward_stages.py).

Independent of softgroup_b200: numpy (float64 wherever the reference computes in floating point), the C oracle
(oracle/sg_oracle.c, oracle/spconv_oracle.py) and torch CPU ops only. Every function takes numpy arrays and the
model's state_dict as {name: numpy array}; each cites the reference lines it restates. No stage builds a dense
[proposals, points] array: at 1.5M points those do not fit, so proposals, masks and the pyramid's inverse map are
carried as (proposal, point) pairs throughout."""
import numpy as np
import torch

import oracle
from oracle import spconv_oracle as so


# ---------------------------------------------------------------------------------------------------------------------
# voxelization and backbone
# ---------------------------------------------------------------------------------------------------------------------
def voxelize(coords, feats, coords_float, with_coords, batch_size):
    """Dataloader voxelization_idx (custom.py:239, functions.py:168-197, mode 4) and the voxel features of
    softgroup.py:304-307 (`voxelization(feats, p2v_map)`, the mean over a voxel's points).
    Returns (voxel_coords int64 [M,4], v2p_map int32 [N], p2v_map int32 [M,maxActive+1], voxel_feats float32 [M,C])."""
    vc, v2p, p2v = oracle.voxelization_idx(coords, batch_size, 4)
    f = np.concatenate([feats, coords_float], 1) if with_coords else feats
    return vc, v2p, p2v, oracle.voxelization(np.asarray(f, np.float32), p2v, 4)


def merge_4_parts(x):
    """softgroup.py:397-409: rows of piece k (stored piece after piece) go back to positions k, k+4, k+8, ..."""
    n = x.shape[0]
    order = np.concatenate([np.arange(n)[k::4] for k in range(4)])
    out = np.zeros_like(x)
    out[order] = x
    return out


def backbone(voxel_feats, voxel_coords, v2p_map, spatial_shape, sd, channels, num_blocks, x4_split=False):
    """softgroup.py:363-378 up to output_feats (point rows, float64 accumulation). With x4_split (:380-395) every piece
    (batch column k) runs through the U-Net as a batch of one, its rows go back to the voxel rows of that piece, and the
    point rows are merged with merge_4_parts."""
    vc = np.asarray(voxel_coords).astype(np.int32)
    if not x4_split:
        out = so.backbone(voxel_feats, vc, spatial_shape, sd, channels, num_blocks, acc64=True)
        return out[v2p_map]
    out = np.zeros((vc.shape[0], channels), np.float32)
    for k in range(4):
        sel = np.flatnonzero(vc[:, 0] == k)
        idx = vc[sel].copy()
        idx[:, 0] = 0
        out[sel] = so.backbone(voxel_feats[sel], idx, spatial_shape, sd, channels, num_blocks, acc64=True)
    return merge_4_parts(out[v2p_map])


def _bn64(x, sd, p, eps=1e-4):
    """BatchNorm1d in eval mode (norm_fn of softgroup.py:48, eps 1e-4) in float64."""
    d = lambda k: sd[p + '.' + k].astype(np.float64)  # noqa: E731
    return (x - d('running_mean')) / np.sqrt(d('running_var') + eps) * d('weight') + d('bias')


def mlp(x, sd, prefix, norm):
    """blocks.py:9-19 MLP with num_layers 2 in float64: Linear, [BatchNorm1d,] ReLU, Linear."""
    d = lambda k: sd[prefix + '.' + k].astype(np.float64)  # noqa: E731
    h = np.asarray(x, np.float64) @ d('0.weight').T + d('0.bias')
    if norm:
        h = _bn64(h, sd, prefix + '.1')
    last = '3' if norm else '2'
    return np.maximum(h, 0) @ d(last + '.weight').T + d(last + '.bias')


def pointwise_heads(output_feats, sd):
    """softgroup.py:376-377: semantic_linear, offset_linear (float64)."""
    return mlp(output_feats, sd, 'semantic_linear', True), mlp(output_feats, sd, 'offset_linear', True)


def softmax64(x):
    x = np.asarray(x, np.float64)
    e = np.exp(x - x.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


# ---------------------------------------------------------------------------------------------------------------------
# grouping
# ---------------------------------------------------------------------------------------------------------------------
def _inv32(s):
    """The float32 reciprocal torch multiplies by when a CUDA float32 tensor is divided by the Python scalar s."""
    return torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(s), dtype=torch.float32)


def _append(idx_list, off_list, pidx, poff):
    """The merge of softgroup.py:466-473."""
    pidx = pidx.copy()
    if off_list:
        pidx[:, 0] += sum(len(x) for x in off_list) - 1
        poff = (poff + off_list[-1][-1])[1:]
    if pidx.shape[0] > 0:
        idx_list.append(pidx)
        off_list.append(poff)


def _concat(idx_list, off_list):
    if not idx_list:  # :477-479
        return np.zeros((0, 2), np.int32), np.zeros((0, ), np.int32)
    return np.concatenate(idx_list).astype(np.int32), np.concatenate(off_list).astype(np.int32)


def _batch_offsets(batch_idxs, batch_size):
    """softgroup.py:711-716."""
    return np.concatenate([[0], np.cumsum(np.bincount(batch_idxs, minlength=batch_size))]).astype(np.int32)


def grouping(prob, pt_offsets, batch_idxs, coords_float, cfg, batch_size):
    """softgroup.py:412-480 without the pyramid: the per-class loop, ball query (bfs_cluster.cu:15-66, restated on a grid:
    oracle.ballquery_batch_p_grid) over the class's points of every batch item, then bfs_cluster (bfs_cluster.cpp:60-86).
    prob: the softmax of the semantic scores (:422) as float32 [N, C]."""
    g, tc = cfg['grouping_cfg'], cfg['test_cfg']
    mean = np.asarray(g['class_numpoint_mean'], np.float32)
    batch_idxs = np.asarray(batch_idxs, np.int32)
    idx_list, off_list = [], []
    for c in range(cfg['semantic_classes']):
        if c in g['ignore_classes']:
            continue
        obj = np.flatnonzero(prob[:, c] > np.float32(g['score_thr']))  # :436-437
        if obj.size < tc['min_npoint']:  # :438-439
            continue
        b = batch_idxs[obj]
        xyz = (coords_float[obj] + pt_offsets[obj]).astype(np.float32)  # :452, float32 like the tensors
        nidx, sl = oracle.ballquery_batch_p_grid(xyz, b, _batch_offsets(b, batch_size), g['radius'])
        pidx, poff = oracle.bfs_cluster(mean, nidx, sl, g['npoint_thr'], c)
        pidx[:, 1] = obj[pidx[:, 1]]  # :464
        _append(idx_list, off_list, pidx, poff)
    return _concat(idx_list, off_list)


def get_level(n):
    """softgroup.py:482-489."""
    return 3 if n > 1000000 else 2 if n > 100000 else 1


def grouping_pp(prob, pt_offsets, coords_float, cfg):
    """SoftGroup++ grouping, batch size 1 (softgroup.py:412-507 with_pyramid + with_octree): per class the points are
    voxelised at base_size * level (pyramid_map :491-498, `.long()` truncation, mean of coords and offsets), the octree
    ball query (functions.py:14-44) runs at radius * level, bfs_cluster, and every point inherits the cluster of its
    level voxel (pyramid_inverse_map :500-507). The inverse map is built from the pairs: a level voxel is in at most one
    cluster, and `nonzero()` of the dense matrix lists (cluster, point) pairs sorted by cluster, then point."""
    g, tc = cfg['grouping_cfg'], cfg['test_cfg']
    mean = np.asarray(g['class_numpoint_mean'], np.float32)
    idx_list, off_list = [], []
    for c in range(cfg['semantic_classes']):
        if c in g['ignore_classes']:
            continue
        obj = np.flatnonzero(prob[:, c] > np.float32(g['score_thr']))
        if obj.size < tc['min_npoint']:
            continue
        cf, po = coords_float[obj], pt_offsets[obj]
        level = get_level(obj.size)
        # :492, a CUDA float32 tensor divided by a Python float: times the float32 reciprocal (see clusters_voxelization)
        q = cf * _inv32(g['pyramid_base_size'] * level).numpy()
        lc = np.concatenate([np.zeros((obj.size, 1), np.int64), np.trunc(q).astype(np.int64)], 1)
        _, l2p, p2l = oracle.voxelization_idx(lc, 1, 4)
        vcf, vpo = oracle.voxelization(cf, p2l, 4), oracle.voxelization(po, p2l, 4)
        nidx, sl = oracle.octree_ball_query((vcf + vpo).astype(np.float32), g['mean_active'], g['radius'] * level)
        pidx, poff = oracle.bfs_cluster(mean, nidx, sl, g['npoint_thr'], c)
        n_cluster = len(poff) - 1
        vox_cluster = np.full(vcf.shape[0], -1, np.int64)
        vox_cluster[pidx[:, 1]] = pidx[:, 0]
        c_of_point = vox_cluster[l2p]
        pts = np.flatnonzero(c_of_point >= 0)
        order = np.argsort(c_of_point[pts], kind='stable')
        pidx = np.stack([c_of_point[pts][order], pts[order]], 1).astype(np.int32)
        poff = np.concatenate([[0], np.cumsum(np.bincount(c_of_point[pts], minlength=n_cluster))]).astype(np.int32)
        pidx[:, 1] = obj[pidx[:, 1]]
        _append(idx_list, off_list, pidx, poff)
    return _concat(idx_list, off_list)


# ---------------------------------------------------------------------------------------------------------------------
# instance branch
# ---------------------------------------------------------------------------------------------------------------------
def clusters_voxelization(proposals_idx, proposals_offset, feats, coords, scale, spatial_shape):
    """softgroup.py:656-709 line for line in torch CPU float32 (the same IEEE-rounded single operations as the device),
    sec_min / sec_max from the oracle, the hash and the mean from oracle.voxelization_idx / voxelization (mode 4).
    Returns (voxel coords int32 [M,4], inp_map int64 [S], voxel feats float32 [M,C], batch size)."""
    if proposals_idx.shape[0] == 0:  # :664-673
        c = np.array([[0, 0, 0, 0], [0] + [spatial_shape - 1] * 3], np.int32)
        return c, np.zeros(1, np.int64), np.asarray(feats[0:2], np.float32), 1
    clusters_idx = torch.from_numpy(np.asarray(proposals_idx, np.int32))
    batch_idx = clusters_idx[:, 0].long()
    c_idxs = clusters_idx[:, 1].long()
    feats = torch.from_numpy(np.asarray(feats, np.float32))[c_idxs]
    coords = torch.from_numpy(np.asarray(coords, np.float32))[c_idxs]
    coords_min = torch.from_numpy(oracle.sec_min(coords.numpy(), proposals_offset))
    coords_max = torch.from_numpy(oracle.sec_max(coords.numpy(), proposals_offset))
    # :684 runs on the GPU in the reference, where torch divides by a Python scalar as a multiplication by its float32
    # reciprocal (div_true_kernel_cuda); on the CPU torch would divide
    clusters_scale = 1 / ((coords_max - coords_min) * _inv32(spatial_shape)).max(1)[0] - 0.01
    clusters_scale = torch.clamp(clusters_scale, min=None, max=scale)
    coords_min = coords_min * clusters_scale[:, None]
    clusters_scale = clusters_scale[batch_idx]
    coords = coords * clusters_scale[:, None]
    coords_min = coords_min[batch_idx]
    coords -= coords_min
    assert coords.shape.numel() == ((coords >= 0) * (coords < spatial_shape)).sum()  # :699
    coords = torch.cat([batch_idx.view(-1, 1), coords.long()], 1).numpy()
    n_clusters = int(proposals_idx[-1, 0]) + 1  # :703
    out_coords, inp_map, out_map = oracle.voxelization_idx(coords, n_clusters, 4)
    out_feats = oracle.voxelization(feats.numpy(), out_map, 4)
    return out_coords.astype(np.int32), inp_map.astype(np.int64), out_feats, n_clusters


def tiny_unet(inst_feats, inst_coords, sd, channels, spatial_shape):
    """softgroup.py:510-511: tiny_unet ([C, 2C], blocks.py:82-143) and its output BatchNorm+ReLU, float64 accumulation."""
    x = so.ublock(inst_feats, np.asarray(inst_coords, np.int32), [spatial_shape] * 3, sd, 'tiny_unet',
                  [channels, 2 * channels], acc64=True)
    return so._bn_relu(x, sd, 'tiny_unet_outputlayer.0', acc64=True)


def instance_heads(feats, inst_coords, inst_map, sd, batch_size):
    """softgroup.py:513-522 in float64: mask_linear on the voxel rows gathered by inst_map, global_pool (:719-731: the
    mean of every batch item's rows -- taken here by batch index, whatever the row order) into cls_linear and
    iou_score_linear. Returns (cls_scores, iou_scores, mask_scores)."""
    mask = mlp(feats, sd, 'mask_linear', False)[np.asarray(inst_map, np.int64)]
    b = np.asarray(inst_coords)[:, 0].astype(np.int64)
    cnt = np.bincount(b, minlength=batch_size).astype(np.float64)
    pooled = np.zeros((batch_size, feats.shape[1]))
    np.add.at(pooled, b, np.asarray(feats, np.float64))
    pooled /= cnt[:, None]
    lin = lambda p: pooled @ sd[p + '.weight'].astype(np.float64).T + sd[p + '.bias'].astype(np.float64)  # noqa: E731
    return lin('cls_linear'), lin('iou_score_linear'), mask


def rle_from_ids(ids, length):
    """rle.py:5-19 (`rle_encode` of the dense mask) from the mask's set positions: 1-based run starts and lengths."""
    ids = np.unique(np.asarray(ids, np.int64))
    if ids.size == 0:
        return ''
    brk = np.flatnonzero(np.diff(ids) != 1)
    starts = np.concatenate([[ids[0]], ids[brk + 1]])
    ends = np.concatenate([ids[brk], [ids[-1]]])
    runs = np.empty(2 * starts.size, np.int64)
    runs[0::2] = starts + 1
    runs[1::2] = ends - starts + 1
    return ' '.join(map(str, runs.tolist()))


def get_instances(proposals_idx, semantic_scores, cls_scores, iou_scores, mask_scores, cfg):
    """softgroup.py:538-604 from (proposal, point) pairs. Per instance class i (class-major, proposal order): a
    sem2ins class gives one instance of the points whose semantic argmax is i (conf 1); otherwise proposal p is kept iff
    softmax(cls)[p, i] > cls_score_thr and #{its points with mask_score[:, i] > mask_score_thr} >= min_npoint, its mask
    being those points. Returns dict(keep bool [nP, nI], npoint int64 [nP, nI], score float64 [nP, nI],
    cls_softmax float64 [nP, nI+1], instances = [(label_id, conf, rle counts)])."""
    tc, nI, sem2ins = cfg['test_cfg'], cfg['instance_classes'], list(cfg['sem2ins_classes'])
    N = semantic_scores.shape[0]
    nP = cls_scores.shape[0]
    pidx = np.asarray(proposals_idx, np.int64)
    cls_sm = softmax64(cls_scores)
    on = np.asarray(mask_scores)[:, :nI] > np.float32(tc['mask_score_thr'])  # :569 (float32 scores, float32 threshold)
    npoint = np.stack([np.bincount(pidx[:, 0], weights=on[:, i], minlength=nP) for i in range(nI)], 1).astype(np.int64)
    score = cls_sm[:, :nI] * np.clip(np.asarray(iou_scores, np.float64)[:, :nI], 0, 1)  # :567
    keep = (cls_sm[:, :nI] > tc['cls_score_thr']) & (npoint >= tc['min_npoint'])  # :574, :583-584
    keep[:, sem2ins] = False
    order = np.argsort(pidx[:, 0], kind='stable')
    start = np.concatenate([[0], np.cumsum(np.bincount(pidx[:, 0], minlength=nP))])
    sem_pred = None
    instances = []
    for i in range(nI):
        if i in sem2ins:  # :556-561
            if sem_pred is None:
                sem_pred = np.asarray(semantic_scores).argmax(1)
            instances.append((i + 1, 1.0, rle_from_ids(np.flatnonzero(sem_pred == i), N)))
            continue
        for p in np.flatnonzero(keep[:, i]):
            rows = order[start[p]:start[p + 1]]
            instances.append((i + 1, score[p, i], rle_from_ids(pidx[rows[on[rows, i]], 1], N)))
    return dict(keep=keep, npoint=npoint, score=score, cls_softmax=cls_sm, instances=instances)


def rle_decode(counts, length):
    """rle.py:22-30."""
    s = counts.split()
    mask = np.zeros(length, np.uint8)
    for lo, n in zip(np.asarray(s[0::2], np.int64) - 1, np.asarray(s[1::2], np.int64)):
        mask[lo:lo + n] = 1
    return mask


def panoptic_fusion(semantic_preds, instances, cfg):
    """softgroup.py:606-639, the numpy paste loop; instances = [(label_id, conf, rle counts)]."""
    cls_offset = cfg['semantic_classes'] - cfg['instance_classes'] - 1
    N = semantic_preds.shape[0]
    panoptic_cls = semantic_preds.copy().astype(np.uint32)
    panoptic_ids = np.zeros_like(semantic_preds).astype(np.uint32)
    score_inds = np.argsort([x[1] for x in instances])[::-1]
    prev_paste = np.zeros_like(semantic_preds, dtype=bool)
    panoptic_id = 1
    for i in score_inds:
        cls, _, counts = instances[i]
        mask = rle_decode(counts, N).astype(bool)
        intersect = (mask * prev_paste).sum()
        if intersect / (mask.sum() + 1e-5) > cfg['test_cfg']['panoptic_skip_iou']:
            continue
        paste = mask * (~prev_paste)
        panoptic_cls[paste] = cls + cls_offset
        panoptic_ids[paste] = panoptic_id
        prev_paste[paste] = 1
        panoptic_id += 1
    ignore_inds = (panoptic_cls >= 11) & (panoptic_ids == 0)
    panoptic_preds = (panoptic_cls & 0xFFFF) | (panoptic_ids << 16)
    panoptic_preds[ignore_inds] = cfg['semantic_classes']
    return panoptic_preds.astype(np.uint32)
