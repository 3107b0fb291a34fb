"""SoftGroup nn.Module -- inference forward of the reference's softgroup/model/softgroup.py on libsgb200.

Same constructor arguments, same module tree / state_dict names (checkpoints load unchanged), same
`forward(batch, return_loss=False)` entry and the same result dict as forward_test (softgroup.py:299-361).
Only the inference path is built (training losses are out of scope, SURVEY.md 2 #3).

What is restructured underneath (same outputs):
  * forward_grouping (softgroup.py:411-480): the 18-iteration per-class Python loop with >=6 host syncs per
    class becomes ONE segmented ball query + ONE clustering call -- class c of batch item b is segment
    (rank(c), b); segments are contiguous because entries are taken class-major in ascending point order,
    which is exactly the order in which the reference concatenates its per-class results. Neighbour lists
    never leave the GPU (the reference copies them to the CPU for BFS, :458). The call runs once per range of
    segments: one range holding every segment, or, for a selection beyond the ball query's int32 list cursor,
    the ranges of plan_ballquery_chunks, concatenated in order.
  * clusters_voxelization (:655-709): the hash runs on the GPU (the reference moves coords to the CPU, :701-703).
  * get_instances (:537-604): no dense [nProposal, N] int masks; per (proposal, class) point counts come from a
    segmented sum, kept masks are encoded to the reference's RLE wire format from sorted point ids.
"""
import functools
import threading

import numpy as np
import torch
import torch.nn as nn

from .. import spconv
from ..ops import (BALLQUERY_MAX_SEGMENTS, ball_query, ballquery_batch_p_nosync, bfs_cluster_segments, gather_rows, global_avg_pool,
                   group_entries, sec_max, sec_min,
                   voxelization,
                   voxelization_idx)
from ..ops import functions
from ..ops import instances as inst_ops
from ..ops._lib import SgbError
from ..util import cuda_cast, force_fp32, rle_encode_ids
from .blocks import MLP, ResidualBlock, UBlock


def expand_voxel_entries(proposals_idx, v2p_map, num_voxels):
    """(proposal, voxel) entries -> (proposal, point) entries for every point of the voxel (lvl_fusion, the sparse
    counterpart of `mask_pred[:, v2p_map.long()]`, softgroup.py:560-561). v2p_map: int [N] voxel of every point.
    Returns (int32 [S, 2] entries in entry order, points of one voxel ascending; int64 [S] source entry of each row)."""
    dev = proposals_idx.device
    v2p = v2p_map.long()
    cnt = torch.bincount(v2p, minlength=num_voxels)  # points per voxel
    start = torch.cumsum(cnt, 0) - cnt
    pts_by_voxel = torch.argsort(v2p, stable=True)  # points grouped by voxel, ascending inside a voxel
    vox = proposals_idx[:, 1].long()
    rep = cnt[vox]
    row_of = torch.repeat_interleave(torch.arange(vox.numel(), device=dev), rep)
    first = torch.cumsum(rep, 0) - rep  # first output row of every entry
    within = torch.arange(row_of.numel(), device=dev) - first[row_of]
    pts = pts_by_voxel[start[vox[row_of]] + within]
    out = torch.stack([proposals_idx[row_of, 0].long(), pts], 1).int().contiguous()
    return out, row_of


def _concat_proposals(parts, device):
    """Non-empty (cluster_idxs int32 [S, 2], cluster_offsets int32 [nCluster+1]) parts with global point ids -> one
    (proposals_idx, proposals_offset): cluster ids shifted by the clusters of the parts before, offsets by their
    entries. One part is returned as it is; no part gives the empty pair int32 [0, 2], [0]."""
    if len(parts) == 1:
        return parts[0]
    if not parts:
        return (torch.zeros((0, 2), dtype=torch.int32, device=device),
                torch.zeros((0, ), dtype=torch.int32, device=device))
    idx_list, off_list = [], []
    n_prop, n_pts = 0, 0
    for cidx, coff in parts:
        cidx[:, 0] += n_prop
        idx_list.append(cidx)
        off_list.append(coff[1:] + n_pts if off_list else coff)
        n_prop += coff.numel() - 1
        n_pts += cidx.size(0)
    return torch.cat(idx_list, 0), torch.cat(off_list)


class _HostFetcher(object):
    """Device -> host reads of result arrays without stalling the forward: every tensor is copied into pinned memory
    on a side stream as soon as it is final; `finish()` waits once and hands out numpy arrays that own their pinned
    block (torch's caching host allocator recycles it when the array dies)."""
    _streams = {}

    def __init__(self, device):
        dev = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
        key = (dev, threading.get_ident())  # one side stream per device and calling thread (scans in flight do not share it)
        if key not in _HostFetcher._streams:
            _HostFetcher._streams[key] = torch.cuda.Stream(device=dev)
        self.stream = _HostFetcher._streams[key]
        self.items = []

    def add(self, name, t):
        if t is None:
            self.items.append((name, None))
            return
        if not t.is_cuda:
            self.items.append((name, t))
            return
        t = t.contiguous()
        ready = torch.cuda.Event()
        ready.record()
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(ready)
            h = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
            h.copy_(t, non_blocking=True)
        t.record_stream(self.stream)
        self.items.append((name, h))

    def finish(self):
        self.stream.synchronize()
        return {k: (h.numpy() if h is not None else None) for k, h in self.items}


class SoftGroup(nn.Module):

    def __init__(self,
                 in_channels=3,
                 channels=32,
                 num_blocks=7,
                 semantic_only=False,
                 semantic_classes=20,
                 instance_classes=18,
                 semantic_weight=None,
                 sem2ins_classes=[],
                 ignore_label=-100,
                 with_coords=True,
                 grouping_cfg=None,
                 instance_voxel_cfg=None,
                 train_cfg=None,
                 test_cfg=None,
                 fixed_modules=[]):
        super().__init__()
        self.in_channels = in_channels
        self.channels = channels
        self.num_blocks = num_blocks
        self.semantic_only = semantic_only
        self.semantic_classes = semantic_classes
        self.instance_classes = instance_classes
        self.semantic_weight = semantic_weight
        self.sem2ins_classes = sem2ins_classes
        self.ignore_label = ignore_label
        self.with_coords = with_coords
        self.grouping_cfg = grouping_cfg
        self.instance_voxel_cfg = instance_voxel_cfg
        self.train_cfg = train_cfg
        self.test_cfg = test_cfg
        self.fixed_modules = fixed_modules

        block = ResidualBlock
        norm_fn = functools.partial(nn.BatchNorm1d, eps=1e-4, momentum=0.1)

        # backbone (softgroup.py:56-65)
        if with_coords:
            in_channels += 3
            self.in_channels += 3
        self.input_conv = spconv.SparseSequential(
            spconv.SubMConv3d(in_channels, channels, kernel_size=3, padding=1, bias=False, indice_key='subm1'))
        block_channels = [channels * (i + 1) for i in range(num_blocks)]
        self.unet = UBlock(block_channels, norm_fn, 2, block, indice_key_id=1)
        self.output_layer = spconv.SparseSequential(norm_fn(channels), nn.ReLU())

        # point-wise prediction (:68-69)
        self.semantic_linear = MLP(channels, semantic_classes, norm_fn=norm_fn, num_layers=2)
        self.offset_linear = MLP(channels, 3, norm_fn=norm_fn, num_layers=2)

        # top-down refinement path (:72-77)
        if not semantic_only:
            self.tiny_unet = UBlock([channels, 2 * channels], norm_fn, 2, block, indice_key_id=11)
            self.tiny_unet_outputlayer = spconv.SparseSequential(norm_fn(channels), nn.ReLU())
            self.cls_linear = nn.Linear(channels, instance_classes + 1)
            self.mask_linear = MLP(channels, instance_classes + 1, norm_fn=None, num_layers=2)
            self.iou_score_linear = nn.Linear(channels, instance_classes + 1)

        self.init_weights()
        for mod in fixed_modules:
            mod = getattr(self, mod)
            for param in mod.parameters():
                param.requires_grad = False
        # the backbone and the tiny U-Net run as compiled launch plans, one C call per U-Net level (model/unet_plan.py);
        # False = the same plan one launch per call, each in its own profiler record (per-kernel instrumentation)
        self.use_plan = True
        self._plans = {}
        self.stage_ms = None  # filled when profile_stages is set
        self._tls = threading.local()  # per-thread scratch of a forward (several scans may be in flight: harness.ScanPipeline)
        self.profile_stages = False

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.BatchNorm1d):
                nn.init.constant_(m.weight, 1)
                nn.init.constant_(m.bias, 0)
            elif isinstance(m, MLP):
                m.init_weights()
        if not self.semantic_only:
            for m in [self.cls_linear, self.iou_score_linear]:
                nn.init.normal_(m.weight, 0, 0.01)
                nn.init.constant_(m.bias, 0)

    def forward(self, batch, return_loss=False):
        if return_loss:
            raise NotImplementedError('softgroup_b200 builds the inference forward only (training is out of scope)')
        return self.forward_test(**batch)

    # ------------------------------------------------------------------------------------------------------
    def _cfg(self, cfg, name, default=None):
        if isinstance(cfg, dict):
            return cfg.get(name, default)
        return getattr(cfg, name, default)

    def _mark(self, name):
        if self.profile_stages:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._events.append((name, ev))

    @cuda_cast
    def forward_test(self, batch_idxs, voxel_coords, p2v_map, v2p_map, coords_float, feats, semantic_labels=None,
                     instance_labels=None, pt_offset_labels=None, spatial_shape=None, batch_size=1, scan_ids=None,
                     **kwargs):
        self._events = []
        self._mark('start')
        device_only = kwargs.get('device_only', False)  # bench: keep results on the GPU (no numpy / RLE)
        # the scan's results as CUDA tensors: point-wise predictions, instances as point-id lists, panoptic labels
        device_results = kwargs.get('device_results', False)
        if device_only and device_results:
            raise ValueError('forward_test: device_only and device_results are two different result forms; pass one')
        host_results = not (device_only or device_results)
        # The reference returns the caller's own inputs (labels, coords_float, feats) as numpy arrays, reading them back from
        # the GPU (softgroup.py:317-331). When the caller still holds them on the host (harness.run_scan), `host_inputs`
        # hands those tensors over and the result dict carries views of them: 7.8 of the 12.3 MB read back per 150k-point
        # scan were these copies.
        host_inputs = kwargs.get('host_inputs', None)
        tc = self.test_cfg
        eval_tasks = self._cfg(tc, 'eval_tasks', ['semantic', 'instance'])
        x4_split = self._cfg(tc, 'x4_split', False)
        if not self.semantic_only and ('instance' in eval_tasks or 'panoptic' in eval_tasks):
            self._grouped_classes(int(batch_size))  # a batch the grouping cannot take fails before the backbone runs
        color_feats = feats
        if self.with_coords:
            feats = torch.cat((feats, coords_float), 1)
        voxel_feats = voxelization(feats.contiguous(), p2v_map.contiguous())
        input = spconv.SparseConvTensor(voxel_feats, voxel_coords.int(), spatial_shape, batch_size)
        self._mark('voxelize')
        # lvl_fusion (softgroup.py:309-312): the voxels themselves are level 1 of the pyramid -- heads, grouping and the
        # instance branch run on voxel rows; results return to points through v2p_map
        lvl_fusion = bool(self._cfg(tc, 'lvl_fusion', False))
        semantic_scores, pt_offsets, output_feats = self.forward_backbone(input, v2p_map, x4_split=x4_split,
                                                                          lvl_fusion=lvl_fusion)
        self._mark('backbone')
        inject = kwargs.get('inject_pointwise', None)
        if inject is not None:
            # bench/test hook (SURVEY.md 8d fallback, DESIGN.md "Synthetic workload"): a random-init backbone cannot
            # produce trained-quality point-wise predictions, so the heads' outputs -- already computed above at full
            # cost -- are overwritten by synthetic ones (one-hot*logit + N(0,1), centroid offsets + N(0,sigma)) to
            # give the grouping stage the load a trained checkpoint would. Never used by the drop-in forward.
            assert not lvl_fusion, 'inject_pointwise carries point-level predictions'
            semantic_scores, pt_offsets = inject
        if x4_split:
            coords_float = self.merge_4_parts(coords_float)
            color_feats = color_feats  # the reference returns color_feats un-merged as well (softgroup.py:312-316)
            if semantic_labels is not None:
                semantic_labels = self.merge_4_parts(semantic_labels)
            if instance_labels is not None:
                instance_labels = self.merge_4_parts(instance_labels)
            if pt_offset_labels is not None:
                pt_offset_labels = self.merge_4_parts(pt_offset_labels)
        semantic_preds = semantic_scores.max(1)[1]
        ret = dict(scan_id=scan_ids[0] if scan_ids else None)
        # the reference reads these back with blocking .cpu() calls in the middle of the forward (softgroup.py:317-331);
        # here the copies go to pinned memory on a side stream and are awaited once, after the instance branch
        fetch = _HostFetcher(semantic_scores.device) if host_results else None

        def passthrough(name, dev_tensor, host_key):
            h = host_inputs.get(host_key) if (host_inputs is not None and not x4_split) else None
            if h is not None and torch.is_tensor(h) and not h.is_cuda and dev_tensor is not None and h.shape == dev_tensor.shape:
                fetch.add(name, h)  # CPU tensors pass through the fetcher untouched (numpy view of the caller's buffer)
            else:
                fetch.add(name, dev_tensor)

        if host_results:
            if 'semantic' in eval_tasks or 'panoptic' in eval_tasks:
                passthrough('semantic_labels', semantic_labels, 'semantic_labels')
                passthrough('instance_labels', instance_labels, 'instance_labels')
            if 'semantic' in eval_tasks:
                passthrough('coords_float', coords_float, 'coords_float')
                passthrough('color_feats', color_feats, 'feats')
                # get_point_wise_results (softgroup.py:524-536): voxel predictions go back to points under lvl_fusion
                fetch.add('semantic_preds', semantic_preds[v2p_map.long()] if lvl_fusion else semantic_preds)
                fetch.add('offset_preds', pt_offsets[v2p_map.long()] if lvl_fusion else pt_offsets)
                passthrough('offset_labels', pt_offset_labels, 'pt_offset_labels')
        if not self.semantic_only and ('instance' in eval_tasks or 'panoptic' in eval_tasks):
            if lvl_fusion:  # softgroup.py:332-334
                batch_idxs = input.indices[:, 0].int().contiguous()
                coords_float = voxelization(coords_float.contiguous(), p2v_map.contiguous())
            proposals_idx, proposals_offset = self.forward_grouping(semantic_scores, pt_offsets, batch_idxs,
                                                                    coords_float, self.grouping_cfg,
                                                                    lvl_fusion=lvl_fusion, batch_size=int(batch_size))
            self._mark('grouping')
            inst_feats, inst_map = self.clusters_voxelization(proposals_idx, proposals_offset, output_feats,
                                                              coords_float, **self._voxel_cfg())
            self._mark('clusters_voxelization')
            _, cls_scores, iou_scores, mask_scores = self.forward_instance(inst_feats, inst_map)
            self._mark('instance_head')
            inst = self.get_instances(scan_ids[0] if scan_ids else None, proposals_idx, semantic_scores, cls_scores,
                                      iou_scores, mask_scores, v2p_map=v2p_map, lvl_fusion=lvl_fusion,
                                      device_only=device_only, device_results=device_results)
            self._mark('get_instances')
            if device_only:
                ret.update(device_instances=inst, proposals_idx=proposals_idx, proposals_offset=proposals_offset)
            elif device_results:
                ret.update(instances=inst)
                if 'panoptic' in eval_tasks:
                    bm, npts = self._tls.instance_bitmaps
                    ret.update(panoptic_preds=self.panoptic_fusion_device(
                        semantic_preds[v2p_map.long()] if lvl_fusion else semantic_preds, inst, bm, npts))
            else:
                if 'instance' in eval_tasks:
                    ret.update(dict(pred_instances=inst))
                    # softgroup.py:353: computed on the device, read back with the other arrays (no blocking .cpu() here)
                    fetch.add('gt_instances', self._gt_instances_tensor(semantic_labels, instance_labels))
                if 'panoptic' in eval_tasks:
                    if self.sem2ins_classes or not inst or lvl_fusion:
                        pan = self.panoptic_fusion(semantic_preds.cpu().numpy(), inst)
                    else:  # every instance has its bitmap on the device: paste there (softgroup.py:606-639)
                        bm, npts = self._tls.instance_bitmaps
                        pan = self.panoptic_fusion_gpu(semantic_preds, inst, bm, npts)
                    ret.update(panoptic_preds=pan)
        if device_only:
            ret.update(semantic_preds=semantic_preds, pt_offsets=pt_offsets)
        elif device_results:  # per point, as get_point_wise_results returns them (softgroup.py:524-536)
            ret.update(semantic_preds=semantic_preds[v2p_map.long()] if lvl_fusion else semantic_preds,
                       offset_preds=pt_offsets[v2p_map.long()] if lvl_fusion else pt_offsets)
        else:
            ret.update(fetch.finish())
        if semantic_scores.is_cuda and host_results:
            # an activation beyond the fp16 hi/lo range raises here instead of saturating silently (the host has just waited
            # for the results anyway). device_only / device_results callers keep the forward free of this host wait and
            # call spconv.check_overflow() themselves where they synchronise.
            spconv.check_overflow()
        if self.profile_stages:
            torch.cuda.synchronize()
            self.stage_ms = {b[0]: a[1].elapsed_time(b[1]) for a, b in zip(self._events[:-1], self._events[1:])}
        return ret

    def _voxel_cfg(self):
        c = self.instance_voxel_cfg
        return dict(c) if isinstance(c, dict) else {k: getattr(c, k) for k in ('scale', 'spatial_shape') if hasattr(c, k)}

    # ------------------------------------------------------------------------------------------------------
    def _weights_version(self):
        """Changes whenever a parameter or buffer is written in place (load_state_dict, init, optimizer) or replaced (.cuda(),
        .to(), .float() go through _apply and drop the cached tensor list). Walking the module tree costs ~1 ms per call on
        this model (two calls per scan: backbone and tiny U-Net); the tensor list is therefore cached and only the in-place
        version counters and storage addresses are read per call."""
        ts = self.__dict__.get('_plan_tensors')
        if ts is None:
            ts = [t for t in list(self.parameters()) + list(self.buffers())]
            self.__dict__['_plan_tensors'] = ts
        v = 0
        for t in ts:
            v += t._version
        return (v, ts[0].data_ptr() if ts else 0, len(ts))

    def __getstate__(self):
        # copy.deepcopy / pickling of the module: per-thread scratch, compiled plans (ctypes arrays, raw device pointers) and
        # the cached tensor list are rebuilt on demand
        d = self.__dict__.copy()
        for k in ('_tls', '_plan_tensors', '_seg_thr_cache'):
            d.pop(k, None)
        d['_plans'] = {}
        return d

    def __setstate__(self, d):
        super().__setstate__(d)
        self._tls = threading.local()

    def _apply(self, fn, *args, **kwargs):
        self.__dict__.pop('_plan_tensors', None)
        self._plans = {}
        return super()._apply(fn, *args, **kwargs)

    def load_state_dict(self, *args, **kwargs):
        self.__dict__.pop('_plan_tensors', None)
        self._plans = {}
        return super().load_state_dict(*args, **kwargs)

    def _run_stack(self, name, input_conv, unet, output_layer, x):
        """input_conv -> unet -> output_layer on SparseConvTensor x -> fp32 feature rows. The compiled plan wherever the
        tensor path applies (one C call per U-Net level, or one per launch when use_plan is False), else the module path."""
        from ..spconv import core
        if core.CONV_IMPL == 'tc' and x.features.is_cuda and not self.training and max(unet.nPlanes) <= 256:
            ver = self._weights_version()
            hit = self._plans.get(name)
            if hit is None or hit[0] != ver:
                from .unet_plan import compile_backbone
                hit = (ver, compile_backbone(input_conv, unet, output_layer))
                self._plans[name] = hit
            return hit[1].run(x, per_launch=not self.use_plan)
        out = x
        if input_conv is not None:
            out = input_conv(out)
        out = unet(out)
        if output_layer is not None:
            out = output_layer(out)
        return out.features

    def forward_backbone(self, input, input_map, x4_split=False, lvl_fusion=False):
        """softgroup.py:363-378."""
        if x4_split:
            assert not lvl_fusion, 'x4_split not support lvl_fusion'  # softgroup.py:365
            output_feats = self.forward_4_parts(input, input_map)
            output_feats = self.merge_4_parts(output_feats)
        elif lvl_fusion:
            output_feats = self._run_stack('backbone', self.input_conv, self.unet, self.output_layer, input)  # voxel rows (:373-374)
        else:
            from ..ops import _lib
            from ..ops._lib import check, ptr
            vf = self._run_stack('backbone', self.input_conv, self.unet, self.output_layer, input)
            if vf.stride(0) != vf.size(1):
                vf = vf.contiguous()
            N = input_map.size(0)
            output_feats = torch.empty((N, vf.size(1)), dtype=vf.dtype, device=vf.device)
            # output_feats[input_map.long()] (:374) -- the "devoxelize" gather
            from .. import profiler
            with profiler.record('gather_rows(devoxelize)', 4 * N + 4 * vf.size(1) * (vf.size(0) + N)):
                check(_lib.lib().sgb_gather_rows(ptr(vf), ptr(input_map.contiguous()), ptr(output_feats), N, vf.size(1),
                                                 _lib.stream()), 'sgb_gather_rows')
        semantic_scores = self.semantic_linear(output_feats)
        pt_offsets = self.offset_linear(output_feats)
        return semantic_scores, pt_offsets, output_feats

    def forward_4_parts(self, x, input_map):
        """softgroup.py:380-395 (S3DIS): four interleaved quarter clouds through the backbone one after another."""
        outs = []
        for i in range(4):
            inds = x.indices[:, 0] == i
            feats = x.features[inds]
            coords = x.indices[inds].clone()
            coords[:, 0] = 0
            x_new = spconv.SparseConvTensor(indices=coords, features=feats, spatial_shape=x.spatial_shape,
                                            batch_size=1)
            outs.append(self._run_stack('backbone', self.input_conv, self.unet, self.output_layer, x_new))
        outs = torch.cat(outs, dim=0)
        return outs[input_map.long()]

    def merge_4_parts(self, x):
        """softgroup.py:397-409."""
        inds = torch.arange(x.size(0), device=x.device)
        ps = [inds[0::4], inds[1::4], inds[2::4], inds[3::4]]
        x_split = torch.split(x, [p.size(0) for p in ps])
        x_new = torch.zeros_like(x)
        for i, p in enumerate(ps):
            x_new[p] = x_split[i]
        return x_new

    # ------------------------------------------------------------------------------------------------------
    def _grouped_classes(self, batch_size):
        """The classes forward_grouping groups. The one-pass grouping hands every (class, batch item) pair to one ball query
        as a segment; a batch with more segments than it takes raises here, before any launch of the forward."""
        g = self.grouping_cfg
        ignore = set(self._cfg(g, 'ignore_classes', []))
        classes = [c for c in range(self.semantic_classes) if c not in ignore]
        one_pass = not (self._cfg(g, 'with_pyramid', False) or self._cfg(g, 'with_octree', False))
        if one_pass and len(classes) * batch_size > BALLQUERY_MAX_SEGMENTS:
            raise ValueError('forward_grouping: %d grouped classes x batch size %d = %d ball-query segments, more than the %d '
                             'one ball query takes; run at most %d scans per batch with this config' %
                             (len(classes), batch_size, len(classes) * batch_size, BALLQUERY_MAX_SEGMENTS,
                              BALLQUERY_MAX_SEGMENTS // len(classes)))
        return classes

    @force_fp32(apply_to=('semantic_scores, pt_offsets'))
    def forward_grouping(self, semantic_scores, pt_offsets, batch_idxs, coords_float, grouping_cfg=None,
                         lvl_fusion=False, batch_size=None):
        """softgroup.py:411-480, all classes in one segmented launch. Returns CUDA int32 tensors
        proposals_idx [sumNPoint,2] (proposal id, point idx), proposals_offset [nProposal+1]."""
        g = self.grouping_cfg
        dev = semantic_scores.device
        if batch_size is None:  # softgroup.py:415 reads it back from the device; forward_test knows it from the collated batch
            batch_size = int(batch_idxs.max().item()) + 1
        classes = self._grouped_classes(batch_size)
        scores = semantic_scores.softmax(dim=-1)
        radius = float(self._cfg(g, 'radius'))
        npoint_thr = float(self._cfg(g, 'npoint_thr'))
        score_thr = float(self._cfg(g, 'score_thr'))
        cnm = self._cfg(g, 'class_numpoint_mean')
        min_npoint = int(self._cfg(self.test_cfg, 'min_npoint', 0))
        if self._cfg(g, 'with_pyramid', False) or self._cfg(g, 'with_octree', False):
            return self._forward_grouping_pp(scores, pt_offsets, batch_idxs, coords_float, batch_size, classes, radius,
                                             npoint_thr, score_thr, cnm, min_npoint, lvl_fusion=lvl_fusion)
        assert len(cnm) == self.semantic_classes
        if not classes:
            return _concat_proposals([], dev)
        # every class of the loop :430-446 in one pass (csrc/grouping.cu): entries (class rank, point) in class-major,
        # ascending point order, their ball-query segments rank(c) * B + b and shifted coordinates; classes below min_npoint
        # are dropped like `object_idxs.size(0) < min_npoint -> continue` (:437-439)
        pts, seg, shifted, seg_offsets, total = group_entries(scores, classes, score_thr, min_npoint, batch_idxs,
                                                              batch_size, coords_float, pt_offsets)
        n = int(total[0].item())  # the one host synchronisation of the selection (the list buffers are sized from it)
        if n == 0:
            return _concat_proposals([], dev)
        seg_thr = self._seg_thr(classes, batch_size, npoint_thr, cnm, dev)
        # one ball query and clustering per range (s0, s1) of segments, entries [e0, e1). A selection whose list buffer
        # (1000 per entry) is beyond the int32 list cursor is cut into ranges that fit, at one more host read. No
        # neighbour list leaves its segment and components are numbered in node order: the concatenation is one call's.
        ranges = [(0, len(classes) * batch_size, 0, n)]
        if n * 1000 > functions.BALLQUERY_MAX_CAPACITY:
            seg_off = seg_offsets.cpu().numpy().astype(np.int64)
            ranges = [(s0, s1, int(seg_off[s0]), int(seg_off[s1]))
                      for s0, s1 in functions.plan_ballquery_chunks(np.diff(seg_off))]
        parts = []
        for s0, s1, e0, e1 in ranges:
            m = e1 - e0
            if m == 0:
                continue
            r_seg, r_off = seg[e0:e1], seg_offsets[s0:s1 + 1]
            if s0 > 0:  # rebased to the range
                r_seg, r_off = r_seg - s0, r_off - e0
            if m * 1000 <= functions.BALLQUERY_MAX_CAPACITY:  # the worst-case buffer fits: m * 1000 entries
                neighbor_inds, start_len, n_active = ballquery_batch_p_nosync(shifted[e0:e1], r_seg, r_off, radius)
            else:  # a segment alone beyond the bound: the largest buffer, and SgbError before clustering if it overflows
                capacity = functions.BALLQUERY_MAX_CAPACITY
                neighbor_inds, start_len, n_active = ballquery_batch_p_nosync(shifted[e0:e1], r_seg, r_off, radius,
                                                                              capacity=capacity)
                t, flags = (int(v) for v in n_active.cpu())
                if flags & functions.BALLQUERY_ERR_CURSOR or t > capacity:
                    raise SgbError('forward_grouping: segment %d (%d entries) has more neighbours than one ball query '
                                   'holds (%d; its int32 list cursor addresses at most 2^31 - 1)' % (s0, m, capacity))
            # lists that hit the 1000 cap make the graph asymmetric: the labelling is the exact directed one
            cidx, coff = bfs_cluster_segments(neighbor_inds, start_len, 0.0, node_seg=r_seg, seg_thr=seg_thr[s0:s1],
                                              nactive=n_active[0:1], upstream_err=n_active[1:2])
            if cidx.size(0) == 0:
                continue
            # proposals_idx[:, 1] = object_idxs[proposals_idx[:, 1]] (:464)
            cidx[:, 1] = pts[e0:e1][cidx[:, 1].long()].int()
            parts.append((cidx, coff))
        return _concat_proposals(parts, dev)

    def _seg_thr(self, classes, batch_size, npoint_thr, cnm, dev):
        """Per-segment thresholds on the device: functions.cluster_threshold of every class, once per batch item."""
        key = (tuple(classes), batch_size, npoint_thr, str(dev))
        hit = self.__dict__.get('_seg_thr_cache')
        if hit is None or hit[0] != key:
            thr_c = [functions.cluster_threshold(npoint_thr, cnm[c]) for c in classes]
            seg_thr = torch.tensor(np.repeat(np.asarray(thr_c, np.float32), batch_size), dtype=torch.float32, device=dev)
            hit = (key, seg_thr)
            self.__dict__['_seg_thr_cache'] = hit
        return hit[1]

    # ------------------------------------------------------------------------------------------------------
    def _forward_grouping_pp(self, scores, pt_offsets, batch_idxs, coords_float, batch_size, classes, base_radius,
                             npoint_thr, score_thr, cnm, min_npoint, lvl_fusion=False):
        """SoftGroup++ grouping (softgroup.py:427-463, 482-507): per class, optional pyramid re-voxelisation at
        base_size*level, octree ball query, clustering, inverse pyramid map -- every step on the GPU (the reference
        hashes on the CPU at :494 and builds a dense [nCluster, n] CPU matrix at :500-507). The radius and the level
        depend on the class size, so classes stay separate launches here."""
        g = self.grouping_cfg
        mean_active = int(self._cfg(g, 'mean_active'))
        with_pyramid = self._cfg(g, 'with_pyramid', False)
        with_octree = self._cfg(g, 'with_octree', False)
        base_size = self._cfg(g, 'pyramid_base_size', 0.02)
        radius = base_radius
        parts = []
        for class_id in classes:
            object_idxs = (scores[:, class_id] > score_thr).nonzero().view(-1)
            if object_idxs.size(0) < min_npoint:
                continue
            batch_idxs_ = batch_idxs[object_idxs].int()
            coords_ = coords_float[object_idxs]
            pt_offsets_ = pt_offsets[object_idxs]
            l2p_map = None
            if with_pyramid:
                level = self.get_level(coords_.size(0))
                radius = base_radius * level
                if level > 1 or not lvl_fusion:  # under lvl_fusion the rows already are level-1 voxels (:447)
                    coords_, pt_offsets_, batch_idxs_, l2p_map = self.pyramid_map(coords_, pt_offsets_, batch_idxs_,
                                                                                  level, base_size)
            batch_offsets_ = self.get_batch_offsets(batch_idxs_, batch_size)
            neighbor_inds, start_len = ball_query((coords_ + pt_offsets_).contiguous(), batch_idxs_.contiguous(),
                                                  batch_offsets_, radius, mean_active, with_octree=with_octree)
            thr = functions.cluster_threshold(npoint_thr, cnm[class_id])
            pidx, poff = bfs_cluster_segments(neighbor_inds.contiguous(), start_len, thr)
            if l2p_map is not None:
                pidx, poff = self.pyramid_inverse_map(pidx, poff, coords_.size(0), l2p_map)
            if pidx.size(0) == 0:
                continue
            pidx = pidx.clone()
            pidx[:, 1] = object_idxs[pidx[:, 1].long()].int()
            parts.append((pidx, poff))
        return _concat_proposals(parts, scores.device)

    def get_level(self, num_points):
        """softgroup.py:482-489."""
        if num_points > 1000000:
            return 3
        if num_points > 100000:
            return 2
        return 1

    def get_batch_offsets(self, batch_idxs, bs):
        """softgroup.py:711-716 without the per-batch host sync loop."""
        counts = torch.bincount(batch_idxs.long(), minlength=bs)
        off = torch.zeros(bs + 1, dtype=torch.int32, device=batch_idxs.device)
        off[1:] = counts.cumsum(0).int()
        return off

    def pyramid_map(self, coords_float, pt_offsets, batch_idxs, level=1, base_size=0.02):
        """softgroup.py:491-498, hash on the GPU. Returns level-voxel coords/offsets (means), their batch index and
        the point->level-voxel map."""
        coords = (coords_float / (base_size * level)).long()
        coords = torch.cat([batch_idxs[:, None].long(), coords], dim=1).contiguous()
        n_batch = int(batch_idxs[-1].item()) + 1
        vcoords, l2p_map, p2l_map = voxelization_idx(coords, n_batch)
        coords_float = voxelization(coords_float.contiguous(), p2l_map)
        pt_offsets = voxelization(pt_offsets.contiguous(), p2l_map)
        return coords_float, pt_offsets, vcoords[:, 0].int().contiguous(), l2p_map

    def pyramid_inverse_map(self, proposals_idx, proposals_offset, num_points, l2p_map):
        """softgroup.py:500-507 without the dense [nCluster, n] matrix: every level-voxel belongs to at most one
        cluster, so each point inherits the cluster of its voxel; pairs come out sorted by (cluster, point) exactly like
        `nonzero()` of the dense matrix."""
        dev = l2p_map.device
        n_cluster = proposals_offset.numel() - 1
        vox_cluster = torch.full((num_points, ), -1, dtype=torch.int64, device=dev)
        vox_cluster[proposals_idx[:, 1].long()] = proposals_idx[:, 0].long()
        c_of_point = vox_cluster[l2p_map.long()]
        pts = (c_of_point >= 0).nonzero().view(-1)
        c_sel = c_of_point[pts]
        order = torch.argsort(c_sel, stable=True)
        out_idx = torch.stack([c_sel[order], pts[order]], 1).int().contiguous()
        counts = torch.bincount(c_sel, minlength=n_cluster)
        out_off = torch.zeros(n_cluster + 1, dtype=torch.int32, device=dev)
        out_off[1:] = counts.cumsum(0).int()
        return out_idx, out_off

    # ------------------------------------------------------------------------------------------------------
    @force_fp32(apply_to='feats')
    def clusters_voxelization(self, clusters_idx, clusters_offset, feats, coords, scale, spatial_shape,
                              rand_quantize=False):
        """softgroup.py:655-709 with the hash on the GPU."""
        dev = feats.device
        if clusters_idx.size(0) == 0:
            coords = torch.tensor([[0, 0, 0, 0], [0, spatial_shape - 1, spatial_shape - 1, spatial_shape - 1]],
                                  dtype=torch.int, device=dev)
            feats = feats[0:2]
            voxelization_feats = spconv.SparseConvTensor(feats, coords, [spatial_shape] * 3, 1)
            inp_map = feats.new_zeros((1, ), dtype=torch.long)
            return voxelization_feats, inp_map
        clusters_idx = clusters_idx.to(dev)
        clusters_offset = clusters_offset.to(dev).contiguous()
        batch_idx = clusters_idx[:, 0].long()
        c_idxs = clusters_idx[:, 1].long()
        feats = gather_rows(feats, clusters_idx[:, 1]) if (feats.is_cuda and feats.dtype == torch.float32 and feats.size(1) % 4 == 0) \
            else feats[c_idxs]
        coords = coords[c_idxs].contiguous()
        coords_min = sec_min(coords, clusters_offset)
        coords_max = sec_max(coords, clusters_offset)
        # 0.01 to ensure voxel_coords < spatial_shape (:682-683)
        clusters_scale = 1 / ((coords_max - coords_min) / spatial_shape).max(1)[0] - 0.01
        clusters_scale = torch.clamp(clusters_scale, min=None, max=scale)
        coords_min = coords_min * clusters_scale[:, None]
        coords_max = coords_max * clusters_scale[:, None]
        clusters_scale = clusters_scale[batch_idx]
        coords = coords * clusters_scale[:, None]
        assert not rand_quantize, 'rand_quantize is a training-time augmentation'
        coords_min = coords_min[batch_idx]
        coords -= coords_min
        coords = coords.long()
        coords = torch.cat([batch_idx.view(-1, 1), coords], 1).contiguous()
        n_clusters = clusters_offset.numel() - 1
        out_coords, inp_map, out_map = voxelization_idx(coords, n_clusters)
        out_feats = voxelization(feats.contiguous(), out_map)
        voxelization_feats = spconv.SparseConvTensor(out_feats, out_coords.int(), [spatial_shape] * 3, n_clusters)
        return voxelization_feats, inp_map

    def forward_instance(self, inst_feats, inst_map):
        """softgroup.py:509-522."""
        f = self._run_stack('tiny', None, self.tiny_unet, self.tiny_unet_outputlayer, inst_feats)
        feats = inst_feats.replace_feature(f)
        mask_scores = self.mask_linear(feats.features)
        mask_scores = mask_scores[inst_map.long()]
        instance_batch_idxs = feats.indices[:, 0][inst_map.long()]
        feats = self.global_pool(feats)
        cls_scores = self.cls_linear(feats)
        iou_scores = self.iou_score_linear(feats)
        return instance_batch_idxs, cls_scores, iou_scores, mask_scores

    @force_fp32(apply_to=('x'))
    def global_pool(self, x, expand=False):
        """softgroup.py:718-731."""
        indices = x.indices[:, 0]
        batch_counts = torch.bincount(indices.long(), minlength=int(x.batch_size))
        batch_offset = torch.zeros(batch_counts.numel() + 1, dtype=torch.int32, device=indices.device)
        batch_offset[1:] = torch.cumsum(batch_counts, dim=0).int()
        x_pool = global_avg_pool(x.features.contiguous(), batch_offset)
        if not expand:
            return x_pool
        x_pool_expand = x_pool[indices.long()]
        x.features = torch.cat((x.features, x_pool_expand), dim=1)
        return x

    # ------------------------------------------------------------------------------------------------------
    @force_fp32(apply_to=('semantic_scores', 'cls_scores', 'iou_scores', 'mask_scores'))
    def get_instances(self, scan_id, proposals_idx, semantic_scores, cls_scores, iou_scores, mask_scores,
                      v2p_map=None, lvl_fusion=False, device_only=False, device_results=False):
        """softgroup.py:537-604 without dense masks.

        For every instance class i and proposal p (class-major, proposal order -- the order in which the reference
        concatenates its lists): kept iff cls_score[p,i] > cls_score_thr and
        #{points of p with mask_score[:, i] > mask_score_thr} >= min_npoint.
        device_results: the same instances as CUDA tensors, dict(label_id int32 [n], conf f32 [n], point_offsets int64
        [n + 1], point_ids int32 [total]) -- instance k's points, ascending, are point_ids[point_offsets[k]:point_offsets[k + 1]]."""
        if proposals_idx.size(0) == 0:
            if device_results:
                return self._no_device_instances(semantic_scores.device, v2p_map.numel() if lvl_fusion else semantic_scores.size(0))
            return []
        semantic_pred_rows = None
        if lvl_fusion:
            # the reference expands dense voxel masks with mask_pred[:, v2p_map.long()] (:560-561, :579-580) and counts
            # POINTS for min_npoint; here the (proposal, voxel) entries themselves are expanded to (proposal, point)
            proposals_idx, row_of = expand_voxel_entries(proposals_idx, v2p_map, semantic_scores.size(0))
            mask_scores = mask_scores[row_of]
            semantic_pred_rows = semantic_scores.max(1)[1][v2p_map.long()]
        tc = self.test_cfg
        mask_thr = float(self._cfg(tc, 'mask_score_thr'))
        cls_thr = float(self._cfg(tc, 'cls_score_thr'))
        min_npoint = int(self._cfg(tc, 'min_npoint'))
        num_instances = cls_scores.size(0)
        num_points = v2p_map.numel() if lvl_fusion else semantic_scores.size(0)  # length of the output masks
        nI = self.instance_classes
        cls_sm = cls_scores.softmax(1)
        mask_scores = mask_scores.contiguous()
        # points per (proposal, class) with mask_score > thr: `mask_pred.sum(1)` of the dense procedure (:563-565)
        npoint = inst_ops.instance_point_counts(proposals_idx.contiguous(), mask_scores, nI, mask_thr, num_instances)
        score = cls_sm[:, :nI] * iou_scores[:, :nI].clamp(0, 1)
        keep = (cls_sm[:, :nI] > cls_thr) & (npoint >= min_npoint)  # [nProp, nI]
        for i in self.sem2ins_classes:
            keep[:, i] = False
        if device_only:
            return dict(keep=keep, score=score, npoint=npoint)
        if device_results:
            sem_pts = None
            if self.sem2ins_classes:
                sem_pts = semantic_pred_rows if lvl_fusion else semantic_scores.max(1)[1]
            bm, label_id, conf, total = self._instance_bitmaps_in_order(proposals_idx.contiguous(), mask_scores, mask_thr,
                                                                       keep, score, npoint, sem_pts, num_points)
            self._tls.instance_bitmaps = (bm, num_points)  # reused by panoptic_fusion_device in the same forward (same thread)
            point_offsets, point_ids = inst_ops.bitmap_point_ids(bm, num_points, total=total)
            return dict(label_id=label_id, conf=conf, point_offsets=point_offsets, point_ids=point_ids)
        # kept (class, proposal) pairs in the reference's order (class-major, proposal order) -> one bitmap each; run
        # boundaries are found on the GPU and only (start, end) pairs are read back (rle.py:5-19 on the host before)
        bitmaps, kc, kp = inst_ops.instance_bitmaps(proposals_idx.contiguous(), mask_scores, nI, mask_thr, keep, num_points)
        conf = score.t()[kc, kp]
        rles = inst_ops.bitmaps_to_rle(bitmaps, num_points)
        kc_np, conf_np = kc.cpu().numpy(), conf.cpu().numpy()
        self._tls.instance_bitmaps = (bitmaps, num_points)  # reused by panoptic_fusion in the same forward (same thread)
        if not self.sem2ins_classes:
            # the common case in one comprehension (the loop below interleaves the semantic-only classes): the scan threads of
            # several scans in flight share the interpreter lock, so Python per instance is what bounds the end-to-end rate
            labels = (kc_np + 1).tolist()
            return [dict(scan_id=scan_id, label_id=l, conf=c, pred_mask=r) for l, c, r in zip(labels, conf_np, rles)]
        instances = []
        semantic_pred = None
        k = 0
        for i in range(nI):
            if i in self.sem2ins_classes:
                if semantic_pred is None:
                    semantic_pred = semantic_pred_rows if lvl_fusion else semantic_scores.max(1)[1]
                ids_i = (semantic_pred == i).nonzero().view(-1).cpu().numpy()
                instances.append(dict(scan_id=scan_id, label_id=i + 1, conf=np.float32(1.),
                                      pred_mask=rle_encode_ids(ids_i, num_points)))
                continue
            while k < kc_np.size and kc_np[k] == i:
                instances.append(dict(scan_id=scan_id, label_id=i + 1, conf=conf_np[k], pred_mask=rles[k]))
                k += 1
        return instances

    def _no_device_instances(self, dev, num_points):
        self._tls.instance_bitmaps = (torch.zeros((0, inst_ops.bitmap_words(num_points)), dtype=torch.int32, device=dev),
                                      num_points)
        return dict(label_id=torch.zeros(0, dtype=torch.int32, device=dev), conf=torch.zeros(0, dtype=torch.float32, device=dev),
                    point_offsets=torch.zeros(1, dtype=torch.int64, device=dev),
                    point_ids=torch.zeros(0, dtype=torch.int32, device=dev))

    def _instance_bitmaps_in_order(self, proposals_idx, mask_scores, mask_thr, keep, score, npoint, sem_pts, num_points):
        """Bitmaps of every instance get_instances returns, in its order: class-major, the kept proposals of a class in
        proposal order, a sem2ins class as one instance (its points: semantic prediction == class, conf 1.0) at its
        class's position. One host read: the instance count and the point total together (sizes of the bitmaps and of the
        point-id list). A proposal holds a point at most once, so its bitmap row has npoint[p, i] bits.
        Returns (bitmaps int32 [n, W], label_id int32 [n], conf f32 [n], total points)."""
        dev = keep.device
        nP, nI = keep.shape
        # (class, proposal) cells class-major, plus a last column per class for its sem2ins instance: instance k is the
        # k-th true cell
        cells = torch.zeros((nI, nP + 1), dtype=torch.bool, device=dev)
        cells[:, :nP] = keep.t()
        size = torch.zeros((nI, nP + 1), dtype=torch.int64, device=dev)
        size[:, :nP] = npoint.t()
        conf = torch.ones((nI, nP + 1), dtype=torch.float32, device=dev)
        conf[:, :nP] = score.t()
        sem2ins = [i for i in range(nI) if i in self.sem2ins_classes]
        if sem2ins:
            cls_bm, cls_cnt = inst_ops.class_bitmaps(sem_pts.contiguous(), sem2ins, num_points)
            rows = inst_ops.to_device_async(np.asarray(sem2ins), torch.int64, dev)
            cells[:, nP] = inst_ops.to_device_async(np.isin(np.arange(nI), sem2ins), torch.bool, dev)
            size[:, nP] = torch.zeros(nI, dtype=torch.int64, device=dev).index_copy_(0, rows, cls_cnt)
        flat = cells.view(-1)
        slot = torch.cumsum(flat, 0) - 1
        n_inst, total = (int(v) for v in torch.stack([flat.sum(), torch.where(flat, size.view(-1), 0).sum()]).cpu())
        slot = torch.where(flat, slot, torch.full_like(slot, -1)).view(nI, nP + 1)
        bm = inst_ops.scatter_instance_bitmaps(proposals_idx, mask_scores, nI, mask_thr, slot[:, :nP].int().contiguous(),
                                               n_inst, num_points)
        if sem2ins and n_inst:
            bm.index_copy_(0, slot[:, nP].index_select(0, rows), cls_bm)
        dst = torch.where(flat, slot.view(-1), n_inst)  # cells that are no instance land in a spare last entry
        label_id = torch.empty(n_inst + 1, dtype=torch.int32, device=dev)
        label_id.scatter_(0, dst, torch.arange(1, nI + 1, dtype=torch.int32, device=dev).repeat_interleave(nP + 1))
        conf_out = torch.empty(n_inst + 1, dtype=torch.float32, device=dev)
        conf_out.scatter_(0, dst, conf.view(-1))
        return bm, label_id[:n_inst], conf_out[:n_inst], total

    def panoptic_fusion_device(self, semantic_preds, instances, bitmaps, num_points):
        """panoptic_fusion on the device results: semantic_preds int64 [N] per point, `instances` get_instances'
        device_results dict, bitmaps row k the mask of its instance k. The visiting order is numpy's argsort of the
        confidences (one host read); returns int64 [N] CUDA holding the uint32 values panoptic_fusion returns."""
        dev = semantic_preds.device
        n_inst = bitmaps.size(0)
        order = torch.zeros(0, dtype=torch.int32, device=dev)
        if n_inst:
            scores = instances['conf'].cpu().numpy()
            order = inst_ops.to_device_async(np.argsort(scores)[::-1].astype(np.int32), torch.int32, dev)
        cls_offset = self.semantic_classes - self.instance_classes - 1
        pan_cls, pan_ids = inst_ops.panoptic_paste(bitmaps, order, instances['label_id'] + cls_offset, semantic_preds,
                                                   float(self._cfg(self.test_cfg, 'panoptic_skip_iou')), num_points)
        pan_cls, pan_ids = pan_cls.long() & 0xFFFFFFFF, pan_ids.long()
        ignore = (pan_cls >= 11) & (pan_ids == 0)
        preds = ((pan_cls & 0xFFFF) | (pan_ids << 16)) & 0xFFFFFFFF
        return torch.where(ignore, torch.full_like(preds, self.semantic_classes), preds)

    def panoptic_fusion_gpu(self, semantic_preds, instance_preds, bitmaps, num_points):
        """softgroup.py:606-639 on the GPU: `bitmaps` row k is the mask of instance_preds[k]. The visiting order is the
        reference's own `np.argsort(scores)[::-1]` (computed here with numpy on the confidences, a few hundred floats);
        the paste loop runs in one kernel (sgb_panoptic_paste). semantic_preds: CUDA int tensor [N]."""
        cls_offset = self.semantic_classes - self.instance_classes - 1
        scores = [x['conf'] for x in instance_preds]
        order = torch.from_numpy(np.ascontiguousarray(np.argsort(scores)[::-1]).astype(np.int32)).to(semantic_preds.device)
        cls_vals = torch.tensor([int(x['label_id']) + cls_offset for x in instance_preds], dtype=torch.int32,
                                device=semantic_preds.device)
        pan_cls, pan_ids = inst_ops.panoptic_paste(bitmaps, order, cls_vals, semantic_preds,
                                                   float(self._cfg(self.test_cfg, 'panoptic_skip_iou')), num_points)
        pan_cls, pan_ids = pan_cls.long(), pan_ids.long()
        ignore = (pan_cls >= 11) & (pan_ids == 0)
        preds = (pan_cls & 0xFFFF) | (pan_ids << 16)
        preds[ignore] = self.semantic_classes
        return preds.cpu().numpy().astype(np.uint32)

    def panoptic_fusion(self, semantic_preds, instance_preds):
        """softgroup.py:606-639, the reference's CPU numpy paste loop on RLE-decoded masks: kept for callers that hold host
        results only (and as the yardstick of panoptic_fusion_gpu in the tests); the forward uses panoptic_fusion_gpu."""
        from ..util import rle_decode
        cls_offset = self.semantic_classes - self.instance_classes - 1
        panoptic_cls = semantic_preds.copy().astype(np.uint32)
        panoptic_ids = np.zeros_like(semantic_preds).astype(np.uint32)
        scores = [x['conf'] for x in instance_preds]
        score_inds = np.argsort(scores)[::-1]
        prev_paste = np.zeros_like(semantic_preds, dtype=bool)
        panoptic_id = 1
        for i in score_inds:
            instance = instance_preds[i]
            cls = instance['label_id']
            mask = rle_decode(instance['pred_mask']).astype(bool)
            intersect = (mask * prev_paste).sum()
            if intersect / (mask.sum() + 1e-5) > self._cfg(self.test_cfg, 'panoptic_skip_iou'):
                continue
            paste = mask * (~prev_paste)
            panoptic_cls[paste] = cls + cls_offset
            panoptic_ids[paste] = panoptic_id
            prev_paste[paste] = 1
            panoptic_id += 1
        ignore_inds = (panoptic_cls >= 11) & (panoptic_ids == 0)
        panoptic_preds = (panoptic_cls & 0xFFFF) | (panoptic_ids << 16)
        panoptic_preds[ignore_inds] = self.semantic_classes
        return panoptic_preds.astype(np.uint32)

    def _gt_instances_tensor(self, semantic_labels, instance_labels):
        label_shift = self.semantic_classes - self.instance_classes
        semantic_labels = semantic_labels - label_shift + 1
        semantic_labels[semantic_labels < 0] = 0
        instance_labels = instance_labels + 1
        ignore_inds = instance_labels < 0
        gt_ins = semantic_labels * 1000 + instance_labels
        gt_ins[ignore_inds] = 0
        return gt_ins

    def get_gt_instances(self, semantic_labels, instance_labels):
        """softgroup.py:641-653."""
        return self._gt_instances_tensor(semantic_labels, instance_labels).cpu().numpy()
