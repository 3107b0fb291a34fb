"""Generate the fixtures that pin this repo's host-side model logic on the UNMODIFIED reference SoftGroup code:

  * tests/golden/ref_model_meta.json -- the `model` sections of the reference configs this repo restates (`configs`,
    by configs.CONFIGS name), the `model` section of every configs/**/*.yaml the reference ships (`yamls`, by path) and
    the reference SoftGroup(scannet) state_dict names and shapes (in order);
  * tests/golden/ref_host_methods.npz -- what the reference's own CUDA-free methods return on the inputs of
    tests/test_host_vs_reference_methods.py and tests/test_host_grouping.py (panoptic_fusion, get_gt_instances,
    merge_4_parts, get_level, pyramid_inverse_map, forward_grouping with oracle stand-ins for its device ops).

Needs a checkout of the reference (thangvubk/SoftGroup) and runs on the CPU:

    python tests/golden/make_reference_golden.py /path/to/SoftGroup [--check]

The tests read only the fixtures; --check regenerates them in memory and compares with the stored files.
"""
import glob
import importlib
import json
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

YAMLS = {'scannet': 'configs/softgroup/softgroup_scannet.yaml',
         's3dis': 'configs/softgroup/softgroup_s3dis_fold5.yaml',
         'kitti': 'configs/softgroup/softgroup_kitti.yaml',
         'stpls3d++': 'configs/softgroup++/softgroup++_stpls3d.yaml',
         'scannet++': 'configs/softgroup++/softgroup++_scannet.yaml',
         's3dis++': 'configs/softgroup++/softgroup++_s3dis_fold5.yaml',
         'stpls3d': 'configs/softgroup/softgroup_stpls3d.yaml'}


def import_reference_model(ref_root):
    """The reference's `softgroup.model.softgroup` on this repo's spconv / ops shims (no softgroup/__init__ side effects)."""
    import softgroup_b200
    from softgroup_b200 import util as our_util
    softgroup_b200.install_as_reference_backends()
    pkg = types.ModuleType('softgroup')
    pkg.__path__ = [os.path.join(ref_root, 'softgroup')]
    sys.modules.setdefault('softgroup', pkg)
    util = types.ModuleType('softgroup.util')
    for n in ('cuda_cast', 'force_fp32', 'rle_decode', 'rle_encode'):
        setattr(util, n, getattr(our_util, n))
    sys.modules.setdefault('softgroup.util', util)
    return importlib.import_module('softgroup.model.softgroup')


def make(ref_root):
    import yaml
    import test_host_vs_reference_methods as hm
    import test_host_grouping as hg
    from softgroup_b200.configs import model_cfg

    ref_module = import_reference_model(ref_root)
    meta = dict(configs={k: yaml.safe_load(open(os.path.join(ref_root, p)))['model'] for k, p in YAMLS.items()})
    paths = sorted(os.path.relpath(p, ref_root) for p in glob.glob(os.path.join(ref_root, 'configs', '**', '*.yaml'),
                                                                   recursive=True))
    meta['yamls'] = {p: yaml.safe_load(open(os.path.join(ref_root, p)))['model'] for p in paths}
    sd = ref_module.SoftGroup(**model_cfg('scannet')).state_dict()
    meta['state_dict_scannet'] = [[k, list(v.shape)] for k, v in sd.items()]

    out = {}
    for seed in range(3):
        sem, insts = hm.panoptic_case(seed)
        out['panoptic_fusion_%d' % seed] = hm.reference_instance(ref_module, 'kitti').panoptic_fusion(sem.copy(), insts)
    sem, inst = hm.gt_instances_case()
    out['get_gt_instances'] = np.asarray(hm.reference_instance(ref_module, 'scannet').get_gt_instances(sem.clone(), inst.clone()))
    out['merge_4_parts'] = hm.reference_instance(ref_module, 's3dis').merge_4_parts(hm.merge_case()).numpy()
    ref = hm.reference_instance(ref_module, 'stpls3d++')
    out['get_level'] = np.array([ref.get_level(n) for n in hm.LEVEL_SIZES], np.int64)
    want_idx, want_off = ref.pyramid_inverse_map(*hm.pyramid_case())
    out['pyramid_inverse_map_idx'], out['pyramid_inverse_map_offset'] = want_idx.numpy(), want_off.numpy()

    # forward_grouping (softgroup.py:411-480) on CPU with its CUDA touch points replaced by oracle stand-ins
    cfg, args = hg.grouping_case()
    ours = hg.SoftGroup(**cfg).eval()
    ref = ref_module.SoftGroup(**cfg)
    ref.eval()
    ref.test_cfg = types.SimpleNamespace(**cfg['test_cfg'])
    ref.grouping_cfg = types.SimpleNamespace(**cfg['grouping_cfg'])
    ref.get_batch_offsets = ours.get_batch_offsets
    ref_module.ball_query = hg._fake_ball_query
    ref_module.bfs_cluster = hg.oracle_bfs_cluster
    want_idx, want_off = ref.forward_grouping(*[a.clone() for a in args], ref.grouping_cfg)
    out['forward_grouping_idx'], out['forward_grouping_offset'] = want_idx.numpy(), want_off.numpy()
    return meta, out


def main():
    ref_root = sys.argv[1]
    meta, out = make(ref_root)
    meta_path, npz_path = os.path.join(HERE, 'ref_model_meta.json'), os.path.join(HERE, 'ref_host_methods.npz')
    if '--check' in sys.argv:
        assert json.load(open(meta_path)) == json.loads(json.dumps(meta)), 'ref_model_meta.json differs'
        gold = np.load(npz_path)
        assert sorted(gold.files) == sorted(out), 'ref_host_methods.npz keys differ'
        for k, v in out.items():
            assert gold[k].dtype == v.dtype and np.array_equal(gold[k], v), k
        print('fixtures reproduced')
        return
    with open(meta_path, 'w') as f:
        json.dump(meta, f, sort_keys=True)
        f.write('\n')
    np.savez_compressed(npz_path, **out)
    print('wrote', meta_path, npz_path)


if __name__ == '__main__':
    main()
