"""Model hyper-parameters of the reference configs that BASELINE.json's workloads are quoted on
(values restated from /root/reference/configs/softgroup/*.yaml; data, not code).
`model_cfg(name)` returns kwargs for softgroup_b200.model.SoftGroup."""
import copy

_SCANNET = dict(  # configs/softgroup/softgroup_scannet.yaml:1-29
    channels=32, num_blocks=7, semantic_classes=20, instance_classes=18, sem2ins_classes=[], semantic_only=False,
    ignore_label=-100,
    grouping_cfg=dict(score_thr=0.2, radius=0.04, mean_active=300,
                      class_numpoint_mean=[-1., -1., 3917., 12056., 2303., 8331., 3948., 3166., 5629., 11719., 1003.,
                                           3317., 4912., 10221., 3889., 4136., 2120., 945., 3967., 2589.],
                      npoint_thr=0.05, ignore_classes=[0, 1]),
    instance_voxel_cfg=dict(scale=50, spatial_shape=20),
    train_cfg=dict(max_proposal_num=200, pos_iou_thr=0.5),
    test_cfg=dict(x4_split=False, cls_score_thr=0.001, mask_score_thr=-0.5, min_npoint=100,
                  eval_tasks=['semantic', 'instance']),
    fixed_modules=[])

_S3DIS = dict(  # configs/softgroup/softgroup_s3dis_fold5.yaml:1-28
    channels=32, num_blocks=7, semantic_classes=13, instance_classes=13, sem2ins_classes=[0, 1], semantic_only=False,
    ignore_label=-100,
    grouping_cfg=dict(score_thr=0.2, radius=0.04, mean_active=300,
                      class_numpoint_mean=[34229, 39796, 12210, 7457, 5439, 10225, 6016, 1724, 5092, 7424, 5279, 6189,
                                           1823],
                      npoint_thr=0.05, ignore_classes=[0, 1]),
    instance_voxel_cfg=dict(scale=50, spatial_shape=20),
    train_cfg=dict(max_proposal_num=200, pos_iou_thr=0.5),
    test_cfg=dict(x4_split=True, cls_score_thr=0.001, mask_score_thr=-0.5, min_npoint=100,
                  eval_tasks=['semantic', 'instance']),
    fixed_modules=[])

_KITTI = dict(  # configs/softgroup/softgroup_kitti.yaml:1-31
    in_channels=1, channels=32, num_blocks=7, semantic_classes=19, instance_classes=8, sem2ins_classes=[],
    semantic_only=False, ignore_label=-100, with_coords=False,
    grouping_cfg=dict(score_thr=0.2, radius=0.1, mean_active=300, class_numpoint_mean=[-1.] * 19, npoint_thr=5,
                      ignore_classes=list(range(11))),
    instance_voxel_cfg=dict(scale=20, spatial_shape=20),
    train_cfg=dict(max_proposal_num=200, pos_iou_thr=0.5),
    test_cfg=dict(x4_split=False, cls_score_thr=0.1, mask_score_thr=-0.5, min_npoint=25, eval_tasks=['panoptic'],
                  panoptic_skip_iou=0.5),
    fixed_modules=[])

_STPLS3D_PP = dict(  # configs/softgroup++/softgroup++_stpls3d.yaml:1-37 (lvl_fusion sits under train_cfg there: unused at test)
    channels=16, num_blocks=7, semantic_classes=15, instance_classes=14, sem2ins_classes=[], semantic_only=False,
    ignore_label=-100, with_coords=False,
    grouping_cfg=dict(score_thr=0.2, radius=0.9, mean_active=3,
                      class_numpoint_mean=[-1., 10408., 58., 124., 1351., 162., 430., 1090., 451., 26., 43., 61., 39., 109.,
                                           1239],
                      npoint_thr=0.01, ignore_classes=[0], with_pyramid=True, pyramid_base_size=0.3333, with_octree=True),
    instance_voxel_cfg=dict(scale=3, spatial_shape=20),
    train_cfg=dict(max_proposal_num=200, pos_iou_thr=0.5),
    test_cfg=dict(x4_split=False, cls_score_thr=0.001, mask_score_thr=-0.5, min_npoint=10,
                  eval_tasks=['semantic', 'instance']),
    fixed_modules=[])

_SCANNET_PP = dict(  # configs/softgroup++/softgroup++_scannet.yaml:1-36 (the one config that tests with lvl_fusion)
    channels=32, num_blocks=7, semantic_classes=20, instance_classes=18, sem2ins_classes=[], semantic_only=False,
    ignore_label=-100,
    grouping_cfg=dict(with_pyramid=True, pyramid_base_size=0.02, with_octree=True, score_thr=0.2, radius=0.04,
                      mean_active=300,
                      class_numpoint_mean=[-1., -1., 3917., 12056., 2303., 8331., 3948., 3166., 5629., 11719., 1003.,
                                           3317., 4912., 10221., 3889., 4136., 2120., 945., 3967., 2589.],
                      npoint_thr=0.05, ignore_classes=[0, 1]),
    instance_voxel_cfg=dict(scale=50, spatial_shape=20),
    train_cfg=dict(max_proposal_num=200, pos_iou_thr=0.5),
    test_cfg=dict(lvl_fusion=True, x4_split=False, cls_score_thr=0.001, mask_score_thr=-0.5, min_npoint=100,
                  eval_tasks=['semantic', 'instance']),
    fixed_modules=[])

_S3DIS_PP = dict(  # configs/softgroup++/softgroup++_s3dis_fold5.yaml:1-36 (the same model section in folds 1-6): lvl_fusion
    # with sem2ins classes, the backbone on the whole room
    channels=32, num_blocks=7, semantic_classes=13, instance_classes=13, sem2ins_classes=[0, 1], semantic_only=False,
    ignore_label=-100,
    grouping_cfg=dict(with_pyramid=True, pyramid_base_size=0.02, with_octree=True, score_thr=0.2, radius=0.04,
                      mean_active=300,
                      class_numpoint_mean=[34229, 39796, 12210, 7457, 5439, 10225, 6016, 1724, 5092, 7424, 5279, 6189,
                                           1823],
                      npoint_thr=0.05, ignore_classes=[0, 1]),
    instance_voxel_cfg=dict(scale=50, spatial_shape=20),
    train_cfg=dict(max_proposal_num=200, pos_iou_thr=0.5),
    test_cfg=dict(lvl_fusion=True, x4_split=False, cls_score_thr=0.001, mask_score_thr=-0.5, min_npoint=100,
                  eval_tasks=['semantic', 'instance']),
    fixed_modules=[])

_STPLS3D = dict(  # configs/softgroup/softgroup_stpls3d.yaml:1-36: the plain SoftGroup (one-pass grouping) on STPLS3D
    channels=16, num_blocks=7, semantic_classes=15, instance_classes=14, sem2ins_classes=[], semantic_only=False,
    ignore_label=-100, with_coords=False,
    grouping_cfg=dict(score_thr=0.2, radius=0.9, mean_active=3,
                      class_numpoint_mean=[-1., 10408., 58., 124., 1351., 162., 430., 1090., 451., 26., 43., 61., 39., 109.,
                                           1239],
                      npoint_thr=0.05, ignore_classes=[0]),
    instance_voxel_cfg=dict(scale=3, spatial_shape=20),
    train_cfg=dict(max_proposal_num=300, pos_iou_thr=0.5, match_low_quality=True, min_pos_thr=0.1),
    test_cfg=dict(x4_split=False, cls_score_thr=0.001, mask_score_thr=-0.5, min_npoint=15,
                  eval_tasks=['semantic', 'instance']),
    fixed_modules=[])

_SCANNET200 = dict(  # a custom dataset as docs/custom_dataset.md describes it: ScanNet200's 200 semantic classes (198 grouped)
    # on the ScanNet model. The reference ships no such config: class_numpoint_mean is SYNTHETIC (log-spaced 500..10000
    # points per instance), not measured on ScanNet200.
    channels=32, num_blocks=7, semantic_classes=200, instance_classes=198, sem2ins_classes=[], semantic_only=False,
    ignore_label=-100,
    grouping_cfg=dict(score_thr=0.2, radius=0.04, mean_active=300,
                      class_numpoint_mean=[-1., -1.] + [float(round(500 * 20 ** (k / 197))) for k in range(198)],
                      npoint_thr=0.05, ignore_classes=[0, 1]),
    instance_voxel_cfg=dict(scale=50, spatial_shape=20),
    train_cfg=dict(max_proposal_num=200, pos_iou_thr=0.5),
    test_cfg=dict(x4_split=False, cls_score_thr=0.001, mask_score_thr=-0.5, min_npoint=100,
                  eval_tasks=['semantic', 'instance']),
    fixed_modules=[])

CONFIGS = {'scannet': _SCANNET, 's3dis': _S3DIS, 'kitti': _KITTI, 'stpls3d++': _STPLS3D_PP, 'scannet++': _SCANNET_PP,
           'scannet200': _SCANNET200, 's3dis++': _S3DIS_PP, 'stpls3d': _STPLS3D}
# which synthetic shape (softgroup_b200.synth.SHAPES) goes with which config
SHAPE_OF = {'scannet': 'c2_scannet', 's3dis': 'c3_s3dis', 'kitti': 'c4_kitti', 'stpls3d++': 'c5_stpls3d',
            'scannet++': 'c2_scannet', 'scannet200': 'c6_scannet200', 's3dis++': 'c3_s3dis', 'stpls3d': 'c5_stpls3d'}


def model_cfg(name='scannet', **overrides):
    cfg = copy.deepcopy(CONFIGS[name])
    for k, v in overrides.items():
        if isinstance(v, dict) and isinstance(cfg.get(k), dict):
            cfg[k].update(v)
        else:
            cfg[k] = v
    return cfg
