# Model / test settings of the reference's configs/dota/orientedrepoints_r101_demo.py:1-73 (the inference-relevant part:
# model dict, test_cfg, img_norm_cfg), restated so that `build_detector(model, test_cfg=test_cfg)` of this repository is
# driven by the same dictionaries.  Loss entries are accepted and ignored (training is out of scope).
norm_cfg = dict(type='GN', num_groups=32, requires_grad=True)
_losses = dict(
    loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
    loss_rbox_init=dict(type='GIoULoss', loss_weight=0.375), loss_rbox_refine=dict(type='GIoULoss', loss_weight=1.0),
    loss_spatial_init=dict(type='SpatialBorderLoss', loss_weight=0.05),
    loss_spatial_refine=dict(type='SpatialBorderLoss', loss_weight=0.1))
model = dict(
    type='OrientedRepPointsDetector', pretrained='torchvision://resnet101',
    backbone=dict(type='ResNet', depth=101, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1,
                  norm_cfg=dict(type='BN', requires_grad=True), style='pytorch'),
    neck=dict(type='FPN', in_channels=[256, 512, 1024, 2048], out_channels=256, start_level=1, add_extra_convs=True,
              num_outs=5, norm_cfg=norm_cfg),
    bbox_head=dict(type='OrientedRepPointsHead', num_classes=16, in_channels=256, feat_channels=256, point_feat_channels=256,
                   stacked_convs=3, num_points=9, gradient_mul=0.3, point_strides=[8, 16, 32, 64, 128], point_base_scale=2,
                   norm_cfg=norm_cfg, top_ratio=0.4, **_losses))
test_cfg = dict(nms_pre=2000, min_bbox_size=0, score_thr=0.05, nms=dict(type='rnms', iou_thr=0.4), max_per_img=2000)
img_norm_cfg = dict(mean=[123.675, 116.28, 103.53], std=[58.395, 57.12, 57.375], to_rgb=True)
# test-time pipeline of the reference config (test_pipeline / data.test.pipeline): run on the device by
# orientedreppoints_b200.datasets.pipelines (Normalize and Pad are fused into the stem / patch-embed input transform)
test_pipeline = [
    dict(type='LoadImageFromFile'),
    dict(
        type='MultiScaleFlipAug',
        img_scale=(1333, 960),
        flip=False,
        transforms=[
            dict(type='RotateResize', keep_ratio=True),
            dict(type='RotateRandomFlip'),
            dict(type='Normalize', **img_norm_cfg),
            dict(type='Pad', size_divisor=32),
            dict(type='ImageToTensor', keys=['img']),
            dict(type='Collect', keys=['img']),
        ])
]
data = dict(test=dict(pipeline=test_pipeline))
