"""The whole CUDA forward of every bench workload (tests/forward_cases.py: c2, c2frag, c3, c4, c5 at full size, c2 with
random BatchNorm statistics) and of a constructed instance-branch case, stage by stage against the host restatement
tests/forward_oracle.py.

The forward runs as a user calls it (harness.run_scan); the stage methods are wrapped to record what each stage got
and returned, and each stage's oracle is fed the GPU's OWN inputs to that stage, so that a last-bit difference upstream
cannot move a threshold decision downstream and hide which stage is wrong.

Bars: voxel coords, maps and features, proposals, instance voxel coords / map / features, keep / npoint, labels, RLE
strings and panoptic labels bit for bit; float outputs (backbone, point-wise heads, tiny U-Net, cls / iou / mask scores)
per element at the north-star bar (_north_star <= 1e-4, tests/test_gpu_spconv_configs.py); confidences within 1e-6
relative. Decisions that would flip if the float64 values were used instead of the GPU's (mask_score > thr, keep) are
counted, and every such flip must have its float64 value within that stage's measured error of the threshold. Run with
-s for the per-stage error and time table.

Every stage is compared in full; no subset is taken. Measured on an H100 SXM (700 W power limit) with a 16-core host, the
CPU oracle took 16-52 s per case for c2, c2frag, c2_bn and c4, 127 s for c5 and 359 s for c3. The c3 oracle time is
split between the float64 backbone (four 200k-point pieces) and the grid ball query of its 800k points. The GPU forward
took 0.1-0.7 s per case."""
import hashlib
import os
import sys
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import forward_cases as fc  # noqa: E402
import forward_oracle as fo  # noqa: E402
from test_gpu_spconv_configs import _north_star  # noqa: E402
from softgroup_b200 import harness, spconv  # noqa: E402

pytestmark = pytest.mark.gpu
NS_BAR = 1e-4
CONF_REL = 1e-6
STAGES = ('forward_test', 'forward_backbone', 'forward_grouping', 'clusters_voxelization', 'forward_instance',
          'get_instances', 'panoptic_fusion_gpu', '_run_stack')


def _host(x):
    if torch.is_tensor(x):
        return x.detach().cpu().numpy()
    if isinstance(x, spconv.SparseConvTensor):
        return dict(features=_host(x.features), indices=_host(x.indices), batch_size=int(x.batch_size))
    if isinstance(x, dict):
        return {k: _host(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_host(v) for v in x)
    return x


def _record(monkeypatch, model):
    """Wrap the stage methods of `model`: rec[name] = (args, kwargs, output) of the last call, on the host. Of
    _run_stack only the tiny U-Net is kept (rec['tiny'])."""
    rec = {}
    for name in STAGES:
        orig = getattr(model, name)

        def wrap(*a, _orig=orig, _name=name, **kw):
            out = _orig(*a, **kw)
            if _name == '_run_stack':
                if a[0] == 'tiny':
                    rec['tiny'] = (_host(a[4]), out.detach().cpu().numpy())
            elif _name == 'forward_test':
                rec[_name] = ({k: _host(v) for k, v in kw.items() if k != 'host_inputs'}, None)
            else:
                rec[_name] = (_host(a), _host(kw), _host(out))
            return out

        monkeypatch.setattr(model, name, wrap)
    return rec


class Report(object):
    def __init__(self, tag):
        self.tag, self.rows, self.t_oracle = tag, [], 0.0

    def floats(self, stage, got, want, bar=NS_BAR):
        got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
        ns = _north_star(got, want)
        err = float(np.abs(got - want).max())
        self.rows.append('%-22s north-star %.3e, max |err| %.3e = %.3e of max |want|' %
                         (stage, ns, err, err / max(np.abs(want).max(), 1e-300)))
        assert ns <= bar, '%s %s: north-star %.3e' % (self.tag, stage, ns)
        return err

    def exact(self, stage, pairs):
        for k, (got, want) in pairs.items():
            assert np.array_equal(np.asarray(got), np.asarray(want)), '%s %s: %s differs' % (self.tag, stage, k)
        self.rows.append('%-22s exact (%s)' % (stage, ', '.join(pairs)))

    def oracle(self, fn, *a, **kw):
        t = time.perf_counter()
        r = fn(*a, **kw)
        self.t_oracle += time.perf_counter() - t
        return r

    def note(self, s):
        self.rows.append(s)

    def show(self, t_gpu):
        print('\n[forward stages] %s: GPU forward %.2f s, CPU oracle %.1f s' % (self.tag, t_gpu, self.t_oracle))
        for r in self.rows:
            print('    ' + r)


def _sd(model):
    return {k: v.detach().cpu().numpy() for k, v in model.state_dict().items()}


def _flips(gpu_on, want64, thr, err, what, rep):
    """Decisions `value > thr` that differ between the GPU's values and the float64 ones: each must sit within err."""
    flip = gpu_on != (want64 > thr)
    far = flip & (np.abs(want64 - thr) > err)
    rep.note('%-22s %d flips of %d decisions (all within %.2e of the threshold)' % (what, int(flip.sum()), flip.size, err))
    assert not far.any(), '%s: %d flips farther than %.2e from %g' % (what, int(far.sum()), err, thr)
    return flip


def _check_instance_branch(rep, cfg, sd, rec, pidx, poff, feats, coords_float, sem_scores, v2p_map=None):
    """clusters_voxelization -> tiny U-Net -> instance heads -> get_instances, each fed the GPU's input. v2p_map
    (lvl_fusion): the branch runs on voxel rows and get_instances takes its masks to points through it."""
    ivc = cfg['instance_voxel_cfg']
    a, kw, (inst_x, inst_map) = rec['clusters_voxelization']
    assert np.array_equal(a[0], pidx) and np.array_equal(a[1], poff)
    assert np.array_equal(a[2], feats) and np.array_equal(a[3], coords_float)
    assert np.array_equal(rec['get_instances'][0][2], sem_scores)
    vc, imap, vfeat, nb = rep.oracle(fo.clusters_voxelization, a[0], a[1], a[2], a[3], kw['scale'], kw['spatial_shape'])
    rep.exact('clusters_voxelization', dict(coords=(inst_x['indices'], vc), inst_map=(inst_map, imap),
                                            feats=(inst_x['features'], vfeat), batch_size=(inst_x['batch_size'], nb)))
    tin, tout = rec['tiny']
    t64 = rep.oracle(fo.tiny_unet, tin['features'], tin['indices'], sd, cfg['channels'], ivc['spatial_shape'])
    rep.floats('tiny U-Net', tout, t64)
    (ix, im), _, (_, cls, iou, mask) = rec['forward_instance']
    cls64, iou64, mask64 = rep.oracle(fo.instance_heads, tout, ix['indices'], im, sd, ix['batch_size'])
    err_cls = rep.floats('cls_scores', cls, cls64)
    rep.floats('iou_scores', iou, iou64)
    err_mask = rep.floats('mask_scores', mask, mask64)
    # get_instances on the GPU's scores
    ga, gkw, inst = rec['get_instances']
    _, p_idx, g_sem, g_cls, g_iou, g_mask = ga
    r = rep.oracle(fo.get_instances, p_idx, g_sem, g_cls, g_iou, g_mask, cfg, v2p_map=v2p_map)
    got = [(int(x['label_id']), float(x['conf']), x['pred_mask']['counts']) for x in inst]
    rep.exact('instances', dict(labels=([x[0] for x in got], [x[0] for x in r['instances']]),
                                rle=([x[2] for x in got], [x[2] for x in r['instances']])))
    conf_g, conf_w = np.array([x[1] for x in got]), np.array([x[1] for x in r['instances']], np.float64)
    assert np.all(np.abs(conf_g - conf_w) <= CONF_REL * np.abs(conf_w)), rep.tag + ': confidences'
    assert all(x['pred_mask']['length'] == r['semantic_preds'].shape[0] for x in inst)
    # decisions the float64 scores would take differently
    nI, tc = cfg['instance_classes'], cfg['test_cfg']
    on_gpu = g_mask[:, :nI] > np.float32(tc['mask_score_thr'])
    mflip = _flips(on_gpu, mask64[:, :nI], tc['mask_score_thr'], err_mask, 'mask_score > thr', rep)
    r64 = fo.get_instances(p_idx, g_sem, cls64, iou64, mask64, cfg, v2p_map=v2p_map)
    sm_err = float(np.abs(r64['cls_softmax'] - r['cls_softmax']).max()) + err_cls
    kflip = r['keep'] != r64['keep']
    by_cls = np.abs(r64['cls_softmax'][:, :nI] - tc['cls_score_thr']) <= sm_err
    nflip = np.zeros_like(r['npoint'])
    # a flipped (proposal, voxel) decision moves npoint by the voxel's points under lvl_fusion
    pts = 1 if v2p_map is None else np.bincount(v2p_map, minlength=g_sem.shape[0])[p_idx[:, 1]]
    for i in range(nI):
        nflip[:, i] = np.bincount(p_idx[:, 0], weights=mflip[:, i] * pts, minlength=nflip.shape[0])
    by_mask = np.abs(r['npoint'] - r64['npoint']) <= nflip
    rep.note('%-22s %d flips of %d decisions' % ('keep', int(kflip.sum()), kflip.size))
    assert np.all(~kflip | by_cls | (by_mask & (nflip > 0))), rep.tag + ': keep flips away from the thresholds'
    return r


def _check_device_only(rep, cfg, rec, v2p_map=None):
    ga, _, dev = rec['get_instances']
    _, p_idx, g_sem, g_cls, g_iou, g_mask = ga
    r = rep.oracle(fo.get_instances, p_idx, g_sem, g_cls, g_iou, g_mask, cfg, v2p_map=v2p_map)
    rep.exact('device_only keep/npoint', dict(keep=(dev['keep'], r['keep']), npoint=(dev['npoint'], r['npoint'])))
    # Scores of kept pairs (the confidences) within 1e-6. The others can be tiny: a float32 softmax value exp(x - max)
    # carries the rounding of x - max, a relative error ~2^-24 |x - max| (~1e-6 at probabilities ~1e-8), and values
    # below the normal float32 range carry fewer bits still.
    rel = np.where(r['keep'], CONF_REL, 10 * CONF_REL)
    bad = np.abs(dev['score'] - r['score']) > rel * np.abs(r['score']) + 1e-30
    assert not bad.any(), '%s: device_only score %s vs %s' % (rep.tag, dev['score'][bad][:5], r['score'][bad][:5])


_BACKBONE_CACHE = {}


@pytest.mark.parametrize('name', [c.name for c in fc.WORKLOAD_CASES])
def test_workload_forward_stages_vs_oracle(name, monkeypatch):
    case = fc.workload_case(name)
    w = fc.build_workload(case)
    cfg, scan, wl = w['cfg'], w['scan'], w['wl']
    model = w['model'].cuda()
    sd = _sd(model)
    hb = harness.to_host_batch(scan, pin=False)
    inj = tuple(torch.from_numpy(a).cuda() for a in w['inj'])
    rec = _record(monkeypatch, model)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        ret = harness.run_scan(model, hb, inject_pointwise=inj)
    torch.cuda.synchronize()
    t_gpu = time.perf_counter() - t0
    rep = Report(name)
    x4 = bool(wl.get('x4'))
    bs = int(scan['batch_size'])

    # voxelization (inputs of the forward: the GPU hash of run_scan, the voxel features of forward_test)
    fkw = rec['forward_test'][0]
    vc, v2p, p2v, vf = rep.oracle(fo.voxelize, scan['coords'], scan['feats'], scan['coords_float'], model.with_coords, bs)
    (bx, bmap), bkw, (sem, off, ofeat) = rec['forward_backbone']
    rep.exact('voxelize', dict(voxel_coords=(fkw['voxel_coords'], vc), v2p=(fkw['v2p_map'], v2p), p2v=(fkw['p2v_map'], p2v),
                               voxel_feats=(bx['features'], vf), indices=(bx['indices'], vc)))
    # backbone and point-wise heads
    key = hashlib.sha1(bx['features'].tobytes() + bx['indices'].tobytes() + b''.join(v.tobytes() for v in sd.values())).hexdigest()
    if key not in _BACKBONE_CACHE:  # c2 and c2frag run the same scan through the same model
        _BACKBONE_CACHE[key] = rep.oracle(fo.backbone, bx['features'], bx['indices'], bmap, scan['spatial_shape'], sd,
                                          cfg['channels'], cfg['num_blocks'], x4_split=x4)
    rep.floats('backbone', ofeat, _BACKBONE_CACHE[key])
    sem64, off64 = rep.oracle(fo.pointwise_heads, ofeat, sd)
    rep.floats('semantic_linear', sem, sem64)
    rep.floats('offset_linear', off, off64)

    # grouping, fed its GPU inputs; the softmax is torch's (softgroup.py:422), checked against float64
    ga, gkw, (pidx, poff) = rec['forward_grouping']
    g_sem, g_off, g_bidx, g_cf = ga[:4]
    assert np.array_equal(g_sem, w['inj'][0]) and np.array_equal(g_off, w['inj'][1])
    assert np.array_equal(g_cf, fo.merge_4_parts(scan['coords_float']) if x4 else scan['coords_float'])
    with torch.no_grad():
        prob = torch.from_numpy(g_sem).cuda().softmax(-1).cpu().numpy()
    p64 = fo.softmax64(g_sem)
    rep.floats('softmax', prob, p64, bar=CONF_REL)
    _flips(prob > np.float32(cfg['grouping_cfg']['score_thr']), p64, cfg['grouping_cfg']['score_thr'],
           float(np.abs(prob - p64).max()), 'score > score_thr', rep)
    if cfg['grouping_cfg'].get('with_pyramid'):
        want = rep.oracle(fo.grouping_pp, prob, g_off, g_cf, cfg)
    else:
        want = rep.oracle(fo.grouping, prob, g_off, g_bidx, g_cf, cfg, gkw['batch_size'])
    rep.exact('grouping', dict(proposals_idx=(pidx, want[0]), proposals_offset=(poff, want[1])))
    rep.note('%-22s %d proposals, %d (proposal, point) pairs' % ('', len(poff) - 1, len(pidx)))
    assert len(poff) - 1 > 10

    # instance branch
    _check_instance_branch(rep, cfg, sd, rec, pidx, poff, ofeat, g_cf, g_sem)
    if 'panoptic' in cfg['test_cfg']['eval_tasks']:
        (sp, inst, _, _), _, pan = rec['panoptic_fusion_gpu']
        assert np.array_equal(sp, g_sem.argmax(1))
        want_pan = rep.oracle(fo.panoptic_fusion, g_sem.argmax(1),
                              [(int(x['label_id']), x['conf'], x['pred_mask']['counts']) for x in inst], cfg)
        rep.exact('panoptic', dict(panoptic_preds=(pan, want_pan), returned=(ret['panoptic_preds'], want_pan)))
    # the bench path: results stay on the device
    with torch.no_grad():
        harness.run_scan(model, hb, inject_pointwise=inj, device_only=True)
    spconv.check_overflow()
    _check_device_only(rep, cfg, rec)
    rep.show(t_gpu)


def test_constructed_instance_branch_vs_oracle(monkeypatch):
    """clusters_voxelization -> tiny U-Net -> heads -> get_instances on > 1000 proposals with single-point and flat
    clusters, clusters at the scale clamp far from the origin and shared points (forward_cases.instance_case)."""
    c = fc.instance_case()
    cfg = c['cfg']
    model = c['model'].cuda()
    sd = _sd(model)
    rec = _record(monkeypatch, model)
    cu = lambda k: torch.from_numpy(c[k]).cuda()  # noqa: E731
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        x, imap = model.clusters_voxelization(cu('proposals_idx'), cu('proposals_offset'), cu('feats'), cu('coords_float'),
                                              **model._voxel_cfg())
        _, cls, iou, mask = model.forward_instance(x, imap)
        model.get_instances(None, cu('proposals_idx'), cu('semantic_scores'), cls, iou, mask)
    torch.cuda.synchronize()
    t_gpu = time.perf_counter() - t0
    spconv.check_overflow()
    rep = Report('instance_case')
    r = _check_instance_branch(rep, cfg, sd, rec, c['proposals_idx'], c['proposals_offset'], c['feats'],
                               c['coords_float'], c['semantic_scores'])
    assert rec['forward_instance'][0][0]['batch_size'] >= 1000
    assert 0 < r['keep'].sum() < r['keep'].size  # decisions go both ways
    with torch.no_grad():
        model.get_instances(None, cu('proposals_idx'), cu('semantic_scores'), cls, iou, mask, device_only=True)
    _check_device_only(rep, cfg, rec)
    rep.show(t_gpu)
