# Single-class (Car) SA-SSD inference config in the reference's config dialect
# (same keys/values as the reference's configs/car_cfg.py for model, test_cfg and the
# data-side voxel/anchor generators; of the training data section only the augmentor).  The
# reference's own file also loads unchanged through sassd_b200.Config.fromfile.
model = dict(
    type='SingleStageDetector',
    backbone=dict(type='SimpleVoxel', num_input_features=4, use_norm=True, num_filters=[32, 64],
                  with_distance=False),
    neck=dict(type='SpMiddleFHD', output_shape=[40, 1600, 1408], num_input_features=4,
              num_hidden_features=64 * 5),
    bbox_head=dict(type='SSDRotateHead', num_class=1, num_output_filters=256, num_anchor_per_loc=2,
                   use_sigmoid_cls=True, encode_rad_error_by_sin=True, use_direction_classifier=True,
                   box_code_size=7),
    extra_head=dict(type='PSWarpHead', grid_offsets=(0., 40.), featmap_stride=.4, in_channels=256,
                    num_class=1, num_parts=28),
)
# Target assignment of the losses (SingleStageDetector.forward_train / loss_points); inference reads none of it.
train_cfg = dict(
    rpn=dict(
        assigner=dict(
            Car=dict(pos_iou_thr=0.6, neg_iou_thr=0.45, min_pos_iou=0.45),
            ignore_iof_thr=-1, similarity_fn='NearestIouSimilarity'),
        anchor_thr=0.1),
    extra=dict(
        assigner=dict(pos_iou_thr=0.7, neg_iou_thr=0.7, min_pos_iou=0.7, ignore_iof_thr=-1,
                      similarity_fn='RotateIou3dSimilarity')),
)
test_cfg = dict(
    rpn=dict(nms_across_levels=False, nms_pre=2000, nms_post=100, nms_thr=0.7, min_bbox_size=0),
    extra=dict(score_thr=0.3, nms=dict(type='nms', iou_thr=0.1), max_per_img=100),
)
_generator = dict(type='VoxelGenerator', voxel_size=[0.05, 0.05, 0.1],
                  point_cloud_range=[0., -40., -3., 70.4, 40., 1.], max_num_points=5, max_voxels=20000)
_anchor = dict(type='AnchorGeneratorStride', anchor_strides=[0.4, 0.4, 1.0],
               anchor_offsets=[0.2, -39.8, -1.78], rotations=[0, 1.57])
data = dict(
    # Training-time augmentation (sassd_b200.augment): the reference's data.train.augmentor; `--data-root` replaces
    # root_path and info_path with paths under that root.
    train=dict(class_names=['Car'], generator=_generator,
               augmentor=dict(type='PointAugmentor', root_path='data/kitti/',
                              info_path='data/kitti/kitti_dbinfos_train.pkl', sample_classes=['Car'],
                              min_num_points=[5], sample_max_num=[15], removed_difficulties=[-1],
                              global_rot_range=[-0.78539816, 0.78539816], gt_rot_range=[-0.78539816, 0.78539816],
                              center_noise_std=[1., 1., .5], scale_range=[0.95, 1.05])),
    val=dict(class_names=['Car'], generator=_generator,
             anchor_generator=dict(Car=dict(_anchor, sizes=[1.6, 3.9, 1.56])),
             anchor_area_threshold=1, out_size_factor=8, test_mode=True),
)
