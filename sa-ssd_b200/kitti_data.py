"""Reading KITTI data from disk for detection and evaluation (host side of ``python -m sassd_b200.test``).

Object splits (KittiSplit; the reference's ``data/kitti``): ``ImageSets/<split>.txt`` lists the frame ids; every
frame's files are under ``training/``, or ``testing/`` for the split ``test`` (which has no labels):
  * ``velodyne/%06d.bin`` full sweeps (cropped to the camera frustum on the device) or ``velodyne_reduced/%06d.bin``
    (cropped offline), float32 (x, y, z, reflectance) rows;
  * ``calib/%06d.txt`` (results.Calibration);
  * ``image_2/%06d.png``, of which only the IHDR chunk is read: the reference decodes the whole image for its shape
    alone (mmdet/datasets/kitti.py:270-272), and KITTI image sizes vary (375x1242, 370x1224, 376x1241, ...);
  * ``label_2/%06d.txt``, read into ground-truth annotations with the semantics of the reference's
    get_label_anno / get_label_annos (tools/kitti_common.py:560-601, 648-666).

Raw drives (KittiDrive; the reference's KittiVideo, mmdet/datasets/kitti.py:356-399): a ``*_sync`` directory with
``image_02/data/%010d.png`` and ``velodyne_points/data/%010d.bin`` per frame, and one calibration for the drive from
``calib_cam_to_cam.txt`` and ``calib_velo_to_cam.txt`` in the recording day's directory (results.Calibration.from_video).
No labels.
"""
import os
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from .frustum import camera_frustum_planes
from .results import Calibration, project_rect_to_velo

PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
_PNG_CHANNELS = {0: 1, 2: 3, 3: 3, 4: 2, 6: 4}      # IHDR colour type -> channels of the decoded image


def read_split(root, split):
    """Frame ids of ``ImageSets/<split>.txt`` (one integer per line), in file order."""
    with open(os.path.join(root, "ImageSets", split + ".txt")) as fh:
        return [int(line) for line in fh.read().split()]


def png_shape(path):
    """(height, width, channels) from a PNG's IHDR chunk; anything that is not a PNG is refused."""
    with open(path, "rb") as fh:
        head = fh.read(33)          # signature (8) + IHDR length (4), type (4), data (13) ...
    if len(head) < 8 or head[:8] != PNG_SIGNATURE:
        raise ValueError("%s: not a PNG file" % path)
    if len(head) < 29:
        raise ValueError("%s: truncated PNG header" % path)
    length, ctype = struct.unpack(">I4s", head[8:16])
    if ctype != b"IHDR" or length != 13:
        raise ValueError("%s: PNG does not start with an IHDR chunk" % path)
    width, height, _depth, colour = struct.unpack(">IIBB", head[16:26])
    if width == 0 or height == 0 or colour not in _PNG_CHANNELS:
        raise ValueError("%s: invalid PNG header" % path)
    return int(height), int(width), _PNG_CHANNELS[colour]


def read_points(path):
    """float32 [N, 4] point cloud; a file whose size is not a multiple of 16 bytes is refused."""
    size = os.path.getsize(path)
    if size % 16:
        raise ValueError("%s: %d bytes is not a whole number of (x, y, z, r) float32 rows" % (path, size))
    return np.fromfile(path, dtype=np.float32).reshape(-1, 4)


def read_plane(path):
    """One ``planes/%06d.txt`` road plane (the format AVOD ships for KITTI: three header lines, then ``a b c d`` of
    a x + b y + c z + d = 0 in the rectified camera frame) -> float64 [4], as the reference's get_road_plane
    (kitti.py:96-108): the normal turned up (negated when b > 0), then the whole vector divided by the normal's
    length."""
    if not os.path.isfile(path):
        raise FileNotFoundError("road plane file %s not found" % path)
    with open(path) as fh:
        lines = fh.readlines()
    if len(lines) < 4:
        raise ValueError("%s: a road plane file has its coefficients on line 4" % path)
    plane = np.asarray([float(v) for v in lines[3].split()])
    if plane[1] > 0:
        plane = -plane
    return plane / np.linalg.norm(plane[0:3])


def read_label(path):
    """One ``label_2`` file -> ground-truth annotation dict (get_label_anno's semantics).

    Every line's name is kept, DontCare included; ``index`` numbers the objects that are not DontCare, which KITTI
    lists first, and gives -1 to the rest; ``group_ids`` numbers every line.  The file's h, w, l dimensions become
    l, h, w.  ``score`` is the 16th field when the first line has one, zeros otherwise."""
    with open(path) as fh:
        fields = [line.strip().split(" ") for line in fh.readlines()]
    n = len(fields)
    n_obj = sum(1 for f in fields if f[0] != "DontCare")
    floats = lambda lo, hi: np.array([[float(v) for v in f[lo:hi]] for f in fields])    # noqa: E731
    anno = {
        "name": np.array([f[0] for f in fields]),
        "truncated": np.array([float(f[1]) for f in fields]),
        "occluded": np.array([int(float(f[2])) for f in fields]),
        "alpha": np.array([float(f[3]) for f in fields]),
        "bbox": floats(4, 8).reshape(-1, 4),
        "dimensions": floats(8, 11).reshape(-1, 3)[:, [2, 0, 1]],
        "location": floats(11, 14).reshape(-1, 3),
        "rotation_y": np.array([float(f[14]) for f in fields]).reshape(-1),
    }
    if n and len(fields[0]) == 16:
        anno["score"] = np.array([float(f[15]) for f in fields])
    else:
        anno["score"] = np.zeros((anno["bbox"].shape[0],))
    anno["index"] = np.array(list(range(n_obj)) + [-1] * (n - n_obj), dtype=np.int32)
    anno["group_ids"] = np.arange(n, dtype=np.int32)
    return anno


def labelled_boxes(anno, calib):
    """One frame's read_label annotation -> (boxes [G,7] float32, names [G]) of its non-DontCare objects in file order,
    as the reference's prepare_train_img reads them (kitti.py:147-154): box3d built in float32 (kitti_utils.py:36-37),
    its centre through project_rect_to_velo in float64 and stored back into float32; the raw names, Van included."""
    names = np.asarray(anno["name"]).reshape(-1)
    keep = names != "DontCare"
    box3d = np.concatenate([np.asarray(anno["location"]).reshape(-1, 3),
                            np.asarray(anno["dimensions"]).reshape(-1, 3)[:, [2, 0, 1]],     # l, h, w -> w, l, h
                            np.asarray(anno["rotation_y"]).reshape(-1, 1)], 1)[keep].astype(np.float32)
    if len(box3d):
        box3d[:, :3] = project_rect_to_velo(box3d[:, :3], calib)
    return box3d.reshape(-1, 7), [str(n) for n in names[keep]]


def gt_from_anno(anno, calib, class_names):
    """One frame's read_label annotation -> the ground truth of the reference's labelled test path
    (prepare_test_img(with_label=True), kitti.py:276-293): (boxes [G,7] float32 as (x, y, z_bottom, w, l, h, ry) in the
    lidar frame, labels [G] int64, 1-based over ``class_names``).  The boxes are labelled_boxes', Van counts as Car,
    and only ``class_names`` are kept, in file order.  A frame with no box left gives [0,7] and [0] (the reference's
    empty array there is 1-D and fails to index)."""
    box3d, names = labelled_boxes(anno, calib)
    types = ["Car" if n == "Van" else n for n in names]
    selected = [i for i, n in enumerate(types) if n in class_names]
    labels = np.array([list(class_names).index(types[i]) + 1 for i in selected], dtype=np.int64)
    return box3d[selected].reshape(-1, 7), labels


_NO_GT = (np.zeros((0, 7), np.float32), np.zeros((0,), np.int64))


def read_labels(label_dir, ids):
    """``label_dir/%06d.txt`` of every id -> annotation dicts with ``image_idx`` (get_label_annos)."""
    annos = []
    for idx in ids:
        anno = read_label(os.path.join(label_dir, "%06d.txt" % idx))
        anno["image_idx"] = np.array([idx] * anno["name"].shape[0], dtype=np.int64)
        annos.append(anno)
    return annos


class PlaneCache:
    """camera_frustum_planes per (calibration values, image height and width): a KITTI split has few distinct
    calibrations (one per recording day), so the plane sets are computed once each."""

    def __init__(self):
        self._planes = {}

    def __call__(self, calib, img_shape):
        key = (calib.P2.tobytes(), calib.V2C.tobytes(), calib.R0.tobytes(), int(img_shape[0]), int(img_shape[1]))
        p = self._planes.get(key)
        if p is None:
            p = self._planes[key] = camera_frustum_planes(calib, img_shape)
        return p

    def __len__(self):
        return len(self._planes)


def padded_batches(ids, batch):
    """Frame ids -> lists of ``batch`` entries; the last list is padded with None (empty frames whose results the
    caller drops)."""
    out = [list(ids[i:i + batch]) for i in range(0, len(ids), batch)]
    if out and len(out[-1]) < batch:
        out[-1] += [None] * (batch - len(out[-1]))
    return out


class _Frames:
    """What Prefetcher reads: ``ids``, ``frame(idx)`` -> (points [N,4] f32, img_meta dict with calib, img_shape,
    sample_idx) and ``pad_frame()``.  ``result_name`` formats a frame id as its result file's name."""
    result_name = "%06d.txt"
    labelled = True
    gt_classes = None

    def pad_frame(self):
        """A padding frame: no points, the calibration and image shape of the first frame, sample_idx -1 (and no GT
        when the frames carry it).
        It does not depend on the batch it pads, which may hold no real frame at all (a rank's last batch under
        torchrun, or every batch of a rank when there are fewer frames than ranks)."""
        if self._pad_meta is None:
            self._pad_meta = dict(self.meta(self.ids[0]), sample_idx=-1)
        return (np.zeros((0, 4), np.float32), self._pad_meta) + ((_NO_GT,) if self.gt_classes is not None else ())


class KittiSplit(_Frames):
    """Frames of one object split (``test`` reads ``testing/``, every other split ``training/``).  With ``gt_classes``
    (a labelled split only) every frame also carries its ground truth, gt_from_anno's (boxes, labels) over those
    classes, and Prefetcher yields the batches' GT lists after their metas."""

    def __init__(self, root, split="val", lidar="velodyne", gt_classes=None):
        if lidar not in ("velodyne", "velodyne_reduced"):
            raise ValueError("lidar must be velodyne or velodyne_reduced, not %r" % lidar)
        self.root, self.split, self.lidar = root, split, lidar
        self.ids = read_split(root, split)
        self.labelled = split != "test"
        if gt_classes is not None and not self.labelled:
            raise ValueError("the test split has no labels to give as ground truth")
        self.gt_classes = None if gt_classes is None else list(gt_classes)
        self.dir = os.path.join(root, "training" if self.labelled else "testing")
        self.planes = PlaneCache()
        self._pad_meta = None

    def path(self, sub, idx, ext):
        return os.path.join(self.dir, sub, "%06d.%s" % (idx, ext))

    def meta(self, idx):
        """img_meta-style dict of one frame: calib, img_shape (from the PNG header), sample_idx."""
        return dict(calib=Calibration(self.path("calib", idx, "txt")),
                    img_shape=png_shape(self.path("image_2", idx, "png")), sample_idx=idx)

    def frame(self, idx):
        meta = self.meta(idx)
        if self.gt_classes is None:
            return read_points(self.path(self.lidar, idx, "bin")), meta
        gt = gt_from_anno(read_label(self.path("label_2", idx, "txt")), meta["calib"], self.gt_classes)
        return read_points(self.path(self.lidar, idx, "bin")), meta, gt

    def gt_annos(self, ids=None):
        if not self.labelled:
            raise ValueError("the test split has no labels")
        return read_labels(os.path.join(self.dir, "label_2"), self.ids if ids is None else ids)


def _stems(path, ext):
    """The frame ids of the ``%010d<ext>`` files of a raw-drive data directory; any other name is refused."""
    ids = []
    for name in os.listdir(path):
        stem, e = os.path.splitext(name)
        if e != ext:
            continue
        if not (len(stem) == 10 and stem.isdigit()):
            raise ValueError("%s: %s is not a %%010d%s frame file" % (path, name, ext))
        ids.append(int(stem))
    return sorted(ids)


class KittiDrive(_Frames):
    """Frames of one raw KITTI drive (``.../2011_09_26/2011_09_26_drive_0001_sync``), for detection with the image-FOV
    crop.  ``calib_dir`` holds the day's calib_cam_to_cam.txt and calib_velo_to_cam.txt (default: the drive's parent
    directory, the raw data's layout).  The frames are the images' stems; the sweeps must have the same stems (the
    reference pairs the two sorted listings by position and would silently misalign a drive with a missing file)."""
    result_name = "%010d.txt"
    labelled = False

    def __init__(self, drive_dir, calib_dir=None):
        self.root = drive_dir
        if calib_dir is None:
            calib_dir = os.path.dirname(os.path.abspath(drive_dir).rstrip(os.sep))
        for name in ("calib_cam_to_cam.txt", "calib_velo_to_cam.txt"):
            if not os.path.isfile(os.path.join(calib_dir, name)):
                raise FileNotFoundError("raw-drive calibration %s not found in %s (pass calib_dir)" % (name, calib_dir))
        self.calib = Calibration.from_video(calib_dir)
        self.img_dir = os.path.join(drive_dir, "image_02", "data")
        self.lidar_dir = os.path.join(drive_dir, "velodyne_points", "data")
        self.ids = _stems(self.img_dir, ".png")
        sweeps = _stems(self.lidar_dir, ".bin")
        if sweeps != self.ids:
            only_img, only_lidar = sorted(set(self.ids) - set(sweeps)), sorted(set(sweeps) - set(self.ids))
            raise ValueError("%s: image_02 and velodyne_points frames differ (images only: %s; sweeps only: %s)" % (
                drive_dir, only_img[:5], only_lidar[:5]))
        self._pad_meta = None

    def meta(self, idx):
        return dict(calib=self.calib, img_shape=png_shape(os.path.join(self.img_dir, "%010d.png" % idx)),
                    sample_idx=idx)

    def frame(self, idx):
        return read_points(os.path.join(self.lidar_dir, "%010d.bin" % idx)), self.meta(idx)


class Prefetcher:
    """Reads batches of frames ``depth`` batches ahead on a thread pool (np.fromfile releases the GIL) and yields
    (ids, points_list, metas) in order, or (ids, points_list, metas, gts) when the split's frames carry their ground
    truth (KittiSplit's ``gt_classes``).  ``wait`` accumulates the seconds the consumer spent blocked on reads."""

    def __init__(self, split, batches, depth=4, workers=4):
        self.split, self.batches, self.depth = split, batches, max(1, int(depth))
        self.pool = ThreadPoolExecutor(max_workers=max(1, int(workers)))
        self.wait = 0.0

    def _submit(self, ids):
        return [self.pool.submit(self.split.frame, i) if i is not None else None for i in ids]

    def __iter__(self):
        import time
        try:
            pending = [(ids, self._submit(ids)) for ids in self.batches[:self.depth]]
            nxt = len(pending)
            while pending:
                ids, futs = pending.pop(0)
                t0 = time.perf_counter()
                frames = [f.result() if f is not None else None for f in futs]
                self.wait += time.perf_counter() - t0
                if nxt < len(self.batches):
                    pending.append((self.batches[nxt], self._submit(self.batches[nxt])))
                    nxt += 1
                frames = [fr if fr is not None else self.split.pad_frame() for fr in frames]
                yield (ids,) + tuple(list(parts) for parts in zip(*frames))
        finally:
            self.pool.shutdown(wait=True, cancel_futures=True)
