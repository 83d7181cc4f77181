"""Detections -> KITTI result annotations (SURVEY.md §8 row f3, host side).

Mirrors the reference's result formatter so a `tools/test.py`-style loop can
hand detections from `SingleStageDetector.forward_test` straight to the KITTI
evaluation code:

* `kitti_bbox2results`  <- mmdet/core/bbox/transforms.py:225-279
* `Calibration`         <- mmdet/datasets/kitti_utils.py:49-107 (the fields the
  formatter reads: P2, V2C, R0), `read_calib_file` :109-125,
  `Calibration.from_video` <- `read_calib_from_video` :128-144
* `empty_result_anno`   <- tools/kitti_common.py:632-646
* `kitti_result_line`, `annos_to_kitti_label` <- tools/kitti_common.py:413-471 (label / result file lines)

This is float64 numpy on a few dozen boxes per frame; it stays on the host in
the reference and here (DESIGN.md §8: not on the device path).
"""
import os

import numpy as np

from .lib import KITTI_META, KITTI_ROW      # the header's SASSD_KITTI_META / SASSD_KITTI_ROW

_RESULT_KEYS = ('name', 'truncated', 'occluded', 'alpha', 'bbox',
                'dimensions', 'location', 'rotation_y', 'score')


class Calibration:
    """KITTI calibration: P2 (3x4), V2C = Tr_velo_to_cam (3x4), R0 (3x3).

    Accepts a calib .txt path (reference constructor) or a dict with the keys
    'P2', 'Tr_velo_to_cam', 'R0_rect' (flat or shaped arrays).
    """

    def __init__(self, calib):
        if not isinstance(calib, dict):
            calib = self.read_calib_file(calib)
        self.P2 = np.asarray(calib['P2'], dtype=np.float64).reshape(3, 4)
        if 'P3' in calib:
            self.P3 = np.asarray(calib['P3'], dtype=np.float64).reshape(3, 4)
        self.V2C = np.asarray(calib['Tr_velo_to_cam'],
                              dtype=np.float64).reshape(3, 4)
        rot = self.V2C[:, :3]
        self.C2V = np.concatenate([rot.T, (-rot.T @ self.V2C[:, 3])[:, None]],
                                  axis=1)
        self.R0 = np.asarray(calib['R0_rect'], dtype=np.float64).reshape(3, 3)
        self.c_u, self.c_v = self.P2[0, 2], self.P2[1, 2]
        self.f_u, self.f_v = self.P2[0, 0], self.P2[1, 1]
        self.b_x = self.P2[0, 3] / (-self.f_u)
        self.b_y = self.P2[1, 3] / (-self.f_v)

    @classmethod
    def from_video(cls, calib_dir):
        """The calibration of a raw KITTI drive (the reference's ``Calibration(calib_dir, from_video=True)``):
        ``calib_cam_to_cam.txt`` gives P2 = P_rect_02 and R0 = R_rect_00, ``calib_velo_to_cam.txt`` gives
        Tr_velo_to_cam = [R | T].  Date lines are skipped."""
        cam = cls.read_calib_file(os.path.join(calib_dir, 'calib_cam_to_cam.txt'))
        velo = cls.read_calib_file(os.path.join(calib_dir, 'calib_velo_to_cam.txt'))
        tr = np.zeros((3, 4))
        tr[:, :3] = np.reshape(velo['R'], (3, 3))
        tr[:, 3] = velo['T']
        calib = {'P2': cam['P_rect_02'], 'Tr_velo_to_cam': tr, 'R0_rect': cam['R_rect_00']}
        if 'P_rect_03' in cam:
            calib['P3'] = cam['P_rect_03']
        return cls(calib)

    @staticmethod
    def read_calib_file(path):
        out = {}
        with open(path, 'r') as fh:
            for line in fh:
                line = line.rstrip()
                if not line:
                    continue
                key, value = line.split(':', 1)
                try:
                    out[key] = np.array([float(v) for v in value.split()])
                except ValueError:
                    pass  # date stamps in raw-data calib files
        return out


def _homogeneous(pts):
    return np.concatenate([pts, np.ones(list(pts.shape[:-1]) + [1])], axis=-1)


def project_velo_to_rect(pts_velo, calib):
    """kitti_utils.py:165-181 (velo -> ref -> rect)."""
    return (_homogeneous(pts_velo) @ calib.V2C.T) @ calib.R0.T


def project_rect_to_velo(pts_rect, calib):
    """kitti_utils.py:173-191 (rect -> ref through inv(R0), ref -> velo through C2V), float64."""
    return _homogeneous(pts_rect @ np.linalg.inv(calib.R0).T) @ calib.C2V.T


def project_rect_to_image(pts_rect, calib):
    """kitti_utils.py:194-202."""
    uvw = _homogeneous(pts_rect) @ calib.P2.T
    uvw[..., 0] /= uvw[..., 2]
    uvw[..., 1] /= uvw[..., 2]
    return uvw[..., 0:2]


def limit_period(val, offset=0.5, period=np.pi):
    """geometry.py:404-405."""
    return val - np.floor(val / period + offset) * period


# corner order of the reference's corners_nd for ndim=3 (geometry.py:303-316):
# unravel_index order permuted by [0, 1, 3, 2, 4, 5, 7, 6]
_UNIT_CORNERS = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0],
                          [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]],
                         dtype=np.float64)


def camera_box_corners(boxes_cam, origin=(0.5, 1.0, 0.5)):
    """Corners of camera-frame boxes (x, y, z, l, h, w, ry), rotated about the
    camera y axis.  geometry.py:380-402 with axis=1, :340-360 for the matrix.
    Returns [N, 8, 3]."""
    boxes_cam = np.asarray(boxes_cam)
    unit = (_UNIT_CORNERS - np.asarray(origin)).astype(boxes_cam.dtype)
    corners = boxes_cam[:, None, 3:6] * unit[None]
    s, c = np.sin(boxes_cam[:, 6]), np.cos(boxes_cam[:, 6])
    o, z = np.ones_like(c), np.zeros_like(c)
    rot_t = np.stack([[c, z, -s], [z, o, z], [s, z, c]])      # [3, 3, N]
    corners = np.einsum('aij,jka->aik', corners, rot_t)
    return corners + boxes_cam[:, None, :3]


def empty_result_anno():
    return {
        'name': np.array([]), 'truncated': np.array([]),
        'occluded': np.array([]), 'alpha': np.array([]),
        'bbox': np.zeros([0, 4]), 'dimensions': np.zeros([0, 3]),
        'location': np.zeros([0, 3]), 'rotation_y': np.array([]),
        'score': np.array([]),
    }


def kitti_bbox2results(boxes_lidar, scores, labels, meta, class_names=None):
    """LiDAR-frame detections of one frame -> KITTI annotation dict.

    `meta` carries 'calib' (Calibration), 'sample_idx' and 'img_shape'.
    As in the reference, `boxes_lidar[:, 6]` is wrapped in place, boxes whose
    image projection lies wholly outside the image are dropped, and the 2-D
    box is clipped to the image.
    """
    calib = meta['calib']
    sample_id = meta['sample_idx']
    img_h, img_w = meta['img_shape'][:2]
    if scores is None or len(scores) == 0 \
            or boxes_lidar is None or len(boxes_lidar) == 0:
        return empty_result_anno()

    boxes_lidar[:, -1] = limit_period(boxes_lidar[:, -1], offset=0.5,
                                      period=np.pi * 2)
    boxes_cam = np.zeros_like(boxes_lidar)
    boxes_cam[:, :3] = project_velo_to_rect(boxes_lidar[:, :3], calib)
    boxes_cam[:, 3:] = boxes_lidar[:, [4, 5, 3, 6]]      # (l, h, w, ry)
    corners_img = project_rect_to_image(camera_box_corners(boxes_cam), calib)
    box2d = np.concatenate([corners_img.min(axis=1), corners_img.max(axis=1)],
                           axis=1)
    alphas = -np.arctan2(-boxes_lidar[:, 1], boxes_lidar[:, 0]) \
        + boxes_lidar[:, 6]

    # one mask instead of the reference's per-box loop (transforms.py:252-271): drop boxes whose projection lies
    # wholly outside the image, clip the rest to it
    labels = np.asarray(labels)
    keep = ~((box2d[:, 0] > img_w) | (box2d[:, 1] > img_h) | (box2d[:, 2] < 0) | (box2d[:, 3] < 0))
    n = int(keep.sum())
    if n == 0:
        return empty_result_anno()
    rect = box2d[keep]
    rect[:, 2:] = np.minimum(rect[:, 2:], [img_w, img_h])
    rect[:, :2] = np.maximum(rect[:, :2], [0, 0])
    cam = boxes_cam[keep]
    names = np.asarray(class_names)[labels[keep]]
    names = names.astype('<U%d' % int(np.char.str_len(names).max()))     # dtype np.stack gives a list of str
    return {
        'name': names, 'truncated': np.zeros(n), 'occluded': np.zeros(n, np.int64), 'alpha': alphas[keep],
        'bbox': rect, 'dimensions': cam[:, 3:6], 'location': cam[:, :3], 'rotation_y': cam[:, 6],
        'score': np.asarray(scores)[keep], 'image_idx': np.full(n, int(sample_id), np.int64),
    }


def kitti_bbox2results_batch(boxes_lidar, scores, labels, metas, class_names=None):
    """All frames of a batch (the loop of single_stage.py:127-131 over ``kitti_bbox2results``)."""
    return [kitti_bbox2results(b, s, l, m, class_names) for b, s, l, m in zip(boxes_lidar, scores, labels, metas)]


def meta_block(calib, img_shape):
    """Calibration + image (h, w, ...) -> the float64 [36] block the device formatter reads per frame
    (ops.kitti_format): P2, Tr_velo_to_cam, R0_rect row-major, then img_h, img_w and one pad value."""
    out = np.zeros(KITTI_META, np.float64)
    out[0:12] = calib.P2.ravel()
    out[12:24] = calib.V2C.ravel()
    out[24:33] = calib.R0.ravel()
    out[33], out[34] = float(img_shape[0]), float(img_shape[1])
    return out


def annos_from_rows(rows, n_out, class_names, sample_ids):
    """Device formatter output (rows [B,cap,14] f64 = alpha, bbox (4), dimensions l h w, location (3), rotation_y,
    score, label; n_out [B]) -> one annotation dict per frame, with the keys and dtypes of ``kitti_bbox2results``; a
    frame without rows gets ``empty_result_anno()``."""
    names_all = np.asarray(class_names)
    out = []
    for b in range(len(sample_ids)):
        n = int(n_out[b])
        if n == 0:
            out.append(empty_result_anno())
            continue
        r = rows[b, :n]
        names = names_all[r[:, 13].astype(np.int64)]
        names = names.astype('<U%d' % int(np.char.str_len(names).max()))
        out.append({
            'name': names, 'truncated': np.zeros(n), 'occluded': np.zeros(n, np.int64),
            'alpha': r[:, 0].astype(np.float32), 'bbox': r[:, 1:5].copy(),
            'dimensions': r[:, 5:8].astype(np.float32), 'location': r[:, 8:11].astype(np.float32),
            'rotation_y': r[:, 11].astype(np.float32), 'score': r[:, 12].astype(np.float32),
            'image_idx': np.full(n, int(sample_ids[b]), np.int64),
        })
    return out


def rows_from_annos(annos, class_names, cap):
    """Inverse of ``annos_from_rows`` (exact: every field widens to float64): annotation dicts -> (rows [B,cap,14]
    f64, n_out [B] int32), e.g. for one fixed-size exchange of a rank's results (dist.DetectionGather)."""
    index = {n: i for i, n in enumerate(class_names)}
    rows = np.zeros((len(annos), cap, KITTI_ROW), np.float64)
    n_out = np.zeros(len(annos), np.int32)
    for b, a in enumerate(annos):
        n = len(a['name'])
        if n > cap:
            raise ValueError("frame %d: %d rows exceed the capacity %d" % (b, n, cap))
        n_out[b] = n
        if n:
            rows[b, :n] = np.concatenate([a['alpha'][:, None], a['bbox'], a['dimensions'], a['location'],
                                          a['rotation_y'][:, None], a['score'][:, None],
                                          np.array([index[str(x)] for x in a['name']], np.float64)[:, None]], axis=1)
    return rows, n_out


_LINE_DEFAULTS = (('name', None), ('truncated', -1), ('occluded', -1), ('alpha', -10), ('bbox', None),
                  ('dimensions', [-1, -1, -1]), ('location', [-1000, -1000, -1000]), ('rotation_y', -10),
                  ('score', 0.0))


def kitti_result_line(result_dict, precision=4):
    """One line of a KITTI label/result file from a dict of fields (tools/kitti_common.py:413-453): fields in the
    official order, floats with ``precision`` decimals, missing optional fields as their defaults."""
    fmt = "{:.%df}" % precision
    defaults = dict(_LINE_DEFAULTS)
    for key in result_dict:
        if key not in defaults:
            raise ValueError("unknown key. supported key:{}".format([k for k, _ in _LINE_DEFAULTS]))
    parts = []
    for key, default in _LINE_DEFAULTS:
        val = result_dict.get(key)
        if val is None and default is None and key in result_dict:
            raise ValueError("you must specify a value for {}".format(key))
        if key == 'name':
            parts.append(val)
        elif key in ('truncated', 'alpha', 'rotation_y', 'score'):
            parts.append(str(default) if val is None else fmt.format(val))
        elif key == 'occluded':
            parts.append(str(default) if val is None else '{}'.format(val))
        else:
            parts += [str(v) for v in default] if val is None else [fmt.format(v) for v in val]
    return ' '.join(parts)


def annos_to_kitti_label(annos, with_score=False):
    """Lines of one frame's annotation dict (tools/kitti_common.py:455-471; the reference leaves the score out,
    ``with_score`` appends it for result files)."""
    keys = ['name', 'truncated', 'occluded', 'alpha', 'bbox', 'dimensions', 'location', 'rotation_y']
    if with_score:
        keys.append('score')
    return [kitti_result_line({k: annos[k][i] for k in keys}) for i in range(len(annos['name']))]
