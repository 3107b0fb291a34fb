"""Harness around the model: host batches in the reference's collate layout, the end-to-end call
(host buffers -> H2D -> GPU point->voxel hashing -> forward -> host results) and the closed-form calibration of
the point-wise heads that gives a synthetic checkpoint a realistic grouping load (SURVEY.md H5 / 8d)."""
import numpy as np
import torch

from . import ops

_KEYS = ('coords', 'batch_idxs', 'coords_float', 'feats', 'semantic_labels', 'instance_labels', 'pt_offset_labels')


def to_host_batch(scan, pin=True):
    """numpy scan (softgroup_b200.synth.make_scan) -> dict of CPU tensors, like custom.py:191-256 minus the
    voxel maps (those are produced on the GPU by `run_scan`, or on the CPU by `collate_like_reference`)."""
    b = {}
    for k in _KEYS:
        t = torch.from_numpy(np.ascontiguousarray(scan[k]))
        if k in ('semantic_labels', 'instance_labels'):
            t = t.long()
        if pin and torch.cuda.is_available():
            t = t.pin_memory()
        b[k] = t
    b['spatial_shape'] = np.asarray(scan['spatial_shape'])
    b['batch_size'] = int(scan['batch_size'])
    b['scan_ids'] = list(scan['scan_ids'])
    return b


def collate_like_reference(scan):
    """Exactly the reference's dataloader output: voxelization_idx on the CPU (custom.py:239)."""
    b = to_host_batch(scan, pin=False)
    voxel_coords, v2p_map, p2v_map = ops.voxelization_idx(b['coords'], b['batch_size'])
    b.update(voxel_coords=voxel_coords, v2p_map=v2p_map, p2v_map=p2v_map)
    return b


def h2d_bytes(batch):
    return int(sum(v.numel() * v.element_size() for v in batch.values() if isinstance(v, torch.Tensor)))


def pointwise_injection(scan, sigma=0.03, seed=0, logit=8.0, fragments=1, confusion=0.0):
    """Device-resident synthetic point-wise predictions (see SoftGroup.forward_test `inject_pointwise`)."""
    from . import synth
    scores, off = synth.grouping_inputs(scan, sigma=sigma, seed=seed, logit=logit, fragments=fragments, confusion=confusion)
    return torch.from_numpy(scores).cuda(), torch.from_numpy(off).cuda()


def run_scan(model, host_batch, device_only=False, inject_pointwise=None, device_results=False):
    """End-to-end call a user makes: pinned host tensors in, result dict out. Point->voxel hashing runs on the GPU
    (voxelization_idx with CUDA tensors), then SoftGroup.forward_test. device_results: the results stay CUDA tensors on
    the current stream (forward_test's device_results form)."""
    dev = {k: (v.cuda(non_blocking=True) if isinstance(v, torch.Tensor) else v) for k, v in host_batch.items()}
    voxel_coords, v2p_map, p2v_map = ops.voxelization_idx(dev['coords'], dev['batch_size'])
    dev.update(voxel_coords=voxel_coords, v2p_map=v2p_map, p2v_map=p2v_map)
    dev.pop('coords')
    return model.forward_test(device_only=device_only, device_results=device_results, inject_pointwise=inject_pointwise,
                              host_inputs=host_batch, **dev)


class ScanPipeline(object):
    """Several scans in flight on one GPU: `workers` host threads, each with its own CUDA stream, run `run_scan` on consecutive
    scans. One scan's forward has ~25 points where the host waits for a size from the device (voxel count, rulebook counts per
    U-Net level, entry / cluster / instance counts) and the GPU then idles until the next launch arrives -- about 15 % of a
    150k-point scan's wall time -- plus the H2D copy in front and the RLE / result-dict work behind it. With two scans in
    flight those holes are filled by the other scan's kernels (scans are independent: softgroup/data/__init__.py:45-54 hands
    them out one per rank and step). Results come back in input order and are identical to sequential calls: every kernel
    and every buffer of a scan lives on that scan's stream.
    The model must have been run once (plans compiled, weights packed) before the first concurrent call."""

    def __init__(self, model, workers=2, freeze_gc=False):
        """freeze_gc: move everything alive now (model, compiled plans, cached tensors) to the permanent generation of Python's
        cyclic GC (gc.collect(); gc.freeze()). The scan threads share the interpreter lock, so a full collection stalls ALL
        scans in flight; with the long-lived objects frozen the collections stay cheap. Off by default: it is a process-wide policy."""
        import concurrent.futures
        import threading
        if freeze_gc:
            import gc
            gc.collect()
            gc.freeze()
        self.model = model
        self.workers = int(workers)
        self.device = next(model.parameters()).device
        self._tls = threading.local()
        self._pool = concurrent.futures.ThreadPoolExecutor(max_workers=self.workers, thread_name_prefix='sgb-scan')

    def _stream(self):
        st = getattr(self._tls, 'stream', None)
        if st is None:
            torch.cuda.set_device(self.device)  # new threads start on device 0
            st = torch.cuda.Stream(device=self.device)
            self._tls.stream = st
        return st

    def _one(self, fn, arg, start_event, before):
        st = self._stream()
        with torch.cuda.stream(st), torch.no_grad():
            if start_event is not None:
                st.wait_event(start_event)
            if before is not None:
                before()
            ret = fn(arg)
            done = torch.cuda.Event(enable_timing=False)
            done.record(st)
        return ret, done

    def map(self, fn, items, start_event=None, before=None):
        """fn(item) on every item, up to `workers` at a time, each call on its worker's stream under no_grad. Returns
        ([results in order], [CUDA events recorded after each call on its stream])."""
        futs = [self._pool.submit(self._one, fn, it, start_event, before) for it in items]
        out = [f.result() for f in futs]
        return [o[0] for o in out], [o[1] for o in out]

    def run_scans(self, host_batches, inject_pointwise=None, device_only=False, device_results=False):
        """The end-to-end call for a sequence of scans: pinned host batches in, result dicts out (input order). With
        device_results the dicts hold CUDA tensors written on the workers' streams; they are complete when this returns."""
        inj = inject_pointwise if isinstance(inject_pointwise, (list, tuple)) and inject_pointwise and \
            isinstance(inject_pointwise[0], (list, tuple)) else [inject_pointwise] * len(host_batches)
        res, evs = self.map(lambda a: run_scan(self.model, a[0], device_only=device_only, inject_pointwise=a[1],
                                               device_results=device_results),
                            list(zip(host_batches, inj)))
        for e in evs:
            e.synchronize()
        return res

    def close(self):
        self._pool.shutdown(wait=True)


def device_batch(host_batch):
    """Inputs resident in HBM (for the `value` leg of bench.py): everything uploaded and hashed once."""
    dev = {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in host_batch.items()}
    voxel_coords, v2p_map, p2v_map = ops.voxelization_idx(dev['coords'], dev['batch_size'])
    dev.update(voxel_coords=voxel_coords, v2p_map=v2p_map, p2v_map=p2v_map)
    return dev


@torch.no_grad()
def calibrate_heads(model, host_batch, logit=6.0, ridge=1e-3):
    """Closed-form fit of the LAST Linear of semantic_linear / offset_linear on the (random) backbone features of
    one scan against its synthetic labels (ridge least squares), so that a realistic share of points passes
    score_thr and shifted coordinates collapse towards instance centroids. Returns fit statistics."""
    dev = device_batch(host_batch)
    feats = dev['feats']
    if model.with_coords:
        feats = torch.cat((feats, dev['coords_float']), 1)
    from . import spconv
    vf = ops.voxelization(feats.contiguous(), dev['p2v_map'])
    x = spconv.SparseConvTensor(vf, dev['voxel_coords'].int(), dev['spatial_shape'], dev['batch_size'])
    out = model.output_layer(model.unet(model.input_conv(x))).features
    pf = out[dev['v2p_map'].long()]

    def hidden(mlp):
        h = pf
        for m in list(mlp)[:-1]:
            h = m(h)
        return h

    def fit(mlp, target):
        h = hidden(mlp).double()
        A = torch.cat([h, torch.ones(h.size(0), 1, device=h.device, dtype=h.dtype)], 1)
        G = A.t() @ A + ridge * h.size(0) * torch.eye(A.size(1), device=h.device, dtype=h.dtype)
        sol = torch.linalg.solve(G, A.t() @ target.double())
        mlp[-1].weight.copy_(sol[:-1].t().float())
        mlp[-1].bias.copy_(sol[-1].float())

    sem = dev['semantic_labels']
    C = model.semantic_classes
    onehot = torch.zeros((sem.numel(), C), device=sem.device)
    valid = sem >= 0
    onehot[valid, sem[valid]] = logit
    fit(model.semantic_linear, onehot)
    inst = dev['instance_labels'] >= 0
    off_t = dev['pt_offset_labels'].clone()
    off_t[~inst] = 0
    fit(model.offset_linear, off_t)
    scores = model.semantic_linear(pf)
    offs = model.offset_linear(pf)
    acc = (scores.argmax(1) == sem).float().mean().item()
    res = (offs - off_t)[inst]
    return dict(sem_acc=acc, offset_residual_sigma=res.std().item(), offset_label_sigma=off_t[inst].std().item())


# ---------------------------------------------------------------------------------------------------------------------
# Test-time data preparation on the GPU (SURVEY.md 8f N2): CustomDataset.transform_test + collate_fn
# (softgroup/data/custom.py:162-168, 191-256) and the S3DIS x4 split (softgroup/data/s3dis.py:46-115) from RAW points.
# ---------------------------------------------------------------------------------------------------------------------
def _test_rotation():
    """dataAugment with every augmentation off (custom.py:87-107): m = eye(3) @ rot_z(0.35 pi), float64 like numpy."""
    import math
    m = np.eye(3)
    theta = 0.35 * math.pi
    return np.matmul(m, [[math.cos(theta), math.sin(theta), 0], [-math.sin(theta), math.cos(theta), 0], [0, 0, 1]])


def transform_test_gpu(xyz, scale, x4_split=False):
    """xyz float32 [N,3] CUDA (already centred like prepare_data_inst.py:55) -> (coords int64 [N,4] with the batch column,
    coords_float float32 [N,3], order int64 [N] or None). Same arithmetic as the reference: float64 rotation, `* scale`,
    `- min`, `.long()` truncation; with x4_split the four interleaved pieces (inds[k::4]) are shifted by their OWN minimum
    and concatenated piece-major (s3dis.py:53-75) -- `order` is that permutation of the input points."""
    import ctypes
    from .ops import _lib
    from .ops._lib import check, ptr
    assert xyz.is_cuda and xyz.dtype == torch.float32 and xyz.is_contiguous()
    N = xyz.size(0)
    m = np.ascontiguousarray(_test_rotation(), dtype=np.float64)
    mid = torch.empty((N, 3), dtype=torch.float64, device=xyz.device)
    check(_lib.lib().sgb_affine3_f64(ptr(xyz), m.ctypes.data_as(ctypes.c_void_p), ptr(mid), N, _lib.stream()), 'sgb_affine3_f64')
    if not x4_split:
        s = mid * float(scale)
        s = s - s.min(0)[0]
        coords = torch.cat([torch.zeros((N, 1), dtype=torch.int64, device=xyz.device), s.long()], 1)
        return coords, mid.float(), None
    order = torch.cat([torch.arange(k, N, 4, device=xyz.device) for k in range(4)])
    pieces, pos = [], 0
    for k in range(4):
        n_k = (N - k + 3) // 4
        s = mid[order[pos:pos + n_k]] * float(scale)
        s = s - s.min(0)[0]
        pieces.append(torch.cat([torch.full((n_k, 1), k, dtype=torch.int64, device=xyz.device), s.long()], 1))
        pos += n_k
    return torch.cat(pieces, 0), mid[order].float(), order


def prepare_test_batch_gpu(xyz, rgb, semantic_label=None, instance_label=None, scale=50, min_spatial_shape=128,
                           x4_split=False, scan_id='scan'):
    """Raw per-point arrays (numpy or tensors; xyz float32 [N,3], rgb float32 [N,C]) -> the reference collate dict
    (custom.py:240-256 / s3dis.py:99-115) with every tensor on the GPU and the point->voxel hash done there. Labels are
    passed through (their instance re-labelling and offset labels are evaluation inputs, not part of the forward)."""
    dev = torch.device('cuda')
    as_t = (lambda a, dt: (a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))).to(dev, non_blocking=True).to(dt))
    xyz_t = as_t(xyz, torch.float32).contiguous()
    coords, coords_float, order = transform_test_gpu(xyz_t, scale, x4_split=x4_split)
    feats = as_t(rgb, torch.float32)
    sem = as_t(semantic_label, torch.int64) if semantic_label is not None else None
    ins = as_t(instance_label, torch.int64) if instance_label is not None else None
    if order is not None:
        feats = feats[order]
        sem = sem[order] if sem is not None else None
        ins = ins[order] if ins is not None else None
    n_batch = 4 if x4_split else 1
    spatial_shape = np.clip(coords.max(0)[0][1:].cpu().numpy() + 1, min_spatial_shape, None)
    voxel_coords, v2p_map, p2v_map = ops.voxelization_idx(coords.contiguous(), n_batch)
    return dict(scan_ids=[scan_id], coords=coords, batch_idxs=(torch.zeros_like(coords[:, 0].int()) if x4_split else coords[:, 0].int()),
                voxel_coords=voxel_coords, p2v_map=p2v_map, v2p_map=v2p_map, coords_float=coords_float, feats=feats.contiguous(),
                semantic_labels=sem, instance_labels=ins, spatial_shape=spatial_shape, batch_size=n_batch)


def run_scan_raw(model, xyz, rgb, semantic_label=None, instance_label=None, scale=50, min_spatial_shape=128, x4_split=False,
                 scan_id='scan', **kw):
    """End to end from RAW points: GPU test transform + GPU hashing + forward (the call N2 adds in front of run_scan)."""
    b = prepare_test_batch_gpu(xyz, rgb, semantic_label, instance_label, scale, min_spatial_shape, x4_split, scan_id)
    b.pop('coords')
    return model.forward_test(**b, **kw)
