"""A small synthetic KITTI root for the create_data tests: full sweeps from synth_cloud(seed, fov_deg=180), two
calibration rigs, two image sizes, minimal valid PNGs and label files with the cases the ground-truth database must
handle (every class, DontCare rows, overlapping boxes, a box across a frustum face and one outside it, rotations near
+-pi, a zero-height box, a frame of DontCare rows only and an empty label file).

tests/golden/make_golden_create_data.py runs the reference on this tree; the GPU tests rebuild the same tree and run
the product on it.  ``flatten`` / ``unflatten`` store the info and dbinfo structures as plain arrays (with their
Python types) in an npz."""
import hashlib
import os
import struct
import zlib

import numpy as np

CALIB_TXT = """P0: 7.215377e+02 0.0 6.095593e+02 0.0 0.0 7.215377e+02 1.728540e+02 0.0 0.0 0.0 1.0 0.0
P1: 7.215377e+02 0.0 6.095593e+02 -3.875744e+02 0.0 7.215377e+02 1.728540e+02 0.0 0.0 0.0 1.0 0.0
P2: 7.215377e+02 0.0 6.095593e+02 4.485728e+01 0.0 7.215377e+02 1.728540e+02 2.163791e-01 0.0 0.0 1.0 2.745884e-03
P3: 7.215377e+02 0.0 6.095593e+02 -3.395242e+02 0.0 7.215377e+02 1.728540e+02 2.199936e+00 0.0 0.0 1.0 2.729905e-03
R0_rect: 9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 7.402527e-03 4.351614e-03 9.999631e-01
Tr_velo_to_cam: 7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 -7.631618e-02 9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01
Tr_imu_to_velo: 9.999976e-01 7.553071e-04 -2.035826e-03 -8.086759e-01 -7.854027e-04 9.998898e-01 -1.482298e-02 3.195559e-01 2.024406e-03 1.482454e-02 9.998881e-01 -7.997231e-01
"""
SHAPES = ((375, 1242), (370, 1224))
TRAIN, VAL, TEST = [0, 1, 2, 3, 4, 6], [5, 7], [0, 1]


def _parse(txt):
    out = {}
    for line in txt.strip().splitlines():
        key, value = line.split(":", 1)
        out[key] = np.array([float(v) for v in value.split()])
    return out


def _rig(r):
    """Rig 0 is CALIB_TXT; rig 1 has a 1.3 % longer focal length, a moved principal point and a LiDAR yawed by 0.8
    degrees and shifted."""
    c = _parse(CALIB_TXT)
    if r == 1:
        P2 = c["P2"].reshape(3, 4).copy()
        P2[0, 0] *= 1.013; P2[1, 1] *= 1.013
        P2[0, 2] += 3.7; P2[1, 2] -= 2.1
        a = np.deg2rad(0.8)
        yaw = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
        Tr = c["Tr_velo_to_cam"].reshape(3, 4).copy()
        Tr[:, :3] = Tr[:, :3] @ yaw
        Tr[:, 3] += [0.02, -0.015, 0.03]
        c["P2"], c["Tr_velo_to_cam"] = P2.reshape(-1), Tr.reshape(-1)
    return c


def calib_text(r):
    return "".join("%s: %s\n" % (k, " ".join(repr(float(v)) for v in vals)) for k, vals in _rig(r).items())


def png_bytes(h, w):
    """An 8-bit RGB PNG of h x w black pixels."""
    def chunk(kind, data):
        return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)
    raw = b"".join(b"\x00" + b"\x00" * (3 * w) for _ in range(h))
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0))
            + chunk(b"IDAT", zlib.compress(raw, 9)) + chunk(b"IEND", b""))


def _velo_to_cam(xyz, c):
    Tr = c["Tr_velo_to_cam"].reshape(3, 4)
    R0 = c["R0_rect"].reshape(3, 3)
    return (R0 @ (Tr[:, :3] @ np.asarray(xyz, np.float64) + Tr[:, 3]))


def _line(name, c, xyz, wlh, ry, rng, trunc=None, occ=None, bbox_h=None):
    """A label row for a box with its bottom centre at LiDAR xyz and size (w, l, h)."""
    w, l, h = wlh
    loc = _velo_to_cam(xyz, c)
    trunc = rng.choice([0.0, 0.1, 0.2, 0.4, 0.7]) if trunc is None else trunc
    occ = int(rng.integers(0, 4)) if occ is None else occ
    top = float(rng.uniform(100, 200))
    bh = float(rng.choice([20.0, 30.0, 45.0, 60.0])) if bbox_h is None else bbox_h
    left = float(rng.uniform(0, 1000))
    return "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
        name, trunc, occ, -1.5, left, top, left + 80.0, top + bh, h, w, l, loc[0], loc[1], loc[2], ry)


_SIZES = {"Car": (1.6, 3.9, 1.56), "Van": (1.9, 5.0, 2.1), "Pedestrian": (0.6, 0.8, 1.7),
          "Cyclist": (0.6, 1.8, 1.7), "Truck": (2.5, 9.0, 3.2), "Misc": (1.0, 1.5, 1.2)}
_DONTCARE = "DontCare -1 -1 -10 500.00 170.00 540.00 190.00 -1 -1 -1 -1000 -1000 -1000 -10"
GROUND_Z = -1.73


def label_lines(idx, c, rng):
    """The label rows of training frame idx (rig c)."""
    g = GROUND_Z - 0.05
    if idx == 0:        # every class of the default database, overlapping Car and Van, DontCare rows last
        return [_line("Car", c, (15.0, 2.0, g), _SIZES["Car"], 0.3, rng, 0.0, 0, 50.0),
                _line("Van", c, (16.0, 2.5, g), _SIZES["Van"], -0.2, rng, 0.2, 1, 30.0),
                _line("Pedestrian", c, (9.0, -3.0, g), _SIZES["Pedestrian"], 1.2, rng),
                _line("Cyclist", c, (20.0, -6.0, g), _SIZES["Cyclist"], -1.4, rng),
                _DONTCARE, _DONTCARE]
    if idx == 1:        # a box across the frustum's side face, and one behind the camera
        return [_line("Car", c, (10.0, 8.4, g), _SIZES["Car"], 1.0, rng),
                _line("Truck", c, (-12.0, 0.0, g), _SIZES["Truck"], 0.0, rng),
                _line("Pedestrian", c, (6.0, 1.0, g), _SIZES["Pedestrian"], 0.0, rng), _DONTCARE]
    if idx == 2:        # rotations near +-pi and a zero-height box
        return [_line("Car", c, (12.0, -2.0, g), _SIZES["Car"], 3.14, rng),
                _line("Car", c, (25.0, 4.0, g), _SIZES["Car"], -3.14, rng),
                _line("Cyclist", c, (18.0, 0.0, g), (0.6, 1.8, 0.0), 3.1415926, rng),
                _line("Misc", c, (30.0, -5.0, g), _SIZES["Misc"], -3.1415926, rng)]
    if idx == 3:
        return [_DONTCARE, _DONTCARE, _DONTCARE]
    if idx == 4:
        return []
    names = ["Car", "Car", "Car", "Van", "Pedestrian", "Cyclist", "Truck", "Misc"]
    rows = []
    for _ in range(15):
        n = names[int(rng.integers(0, len(names)))]
        xyz = (float(rng.uniform(4, 45)), float(rng.uniform(-15, 15)), g)
        rows.append(_line(n, c, xyz, _SIZES[n], float(rng.uniform(-np.pi, np.pi)), rng))
    return rows + [_DONTCARE]


def frame_seed(training, idx):
    return (100 if training else 200) + idx


def write_tree(root):
    """Write the synthetic KITTI root under ``root``: ImageSets and training/, testing/ with velodyne, calib, image_2
    (and label_2 for training).  Returns {(training, idx): seed} of the sweeps."""
    from sassd_b200.synth import synth_cloud
    os.makedirs(os.path.join(root, "ImageSets"), exist_ok=True)
    for name, ids in (("train", TRAIN), ("val", VAL), ("trainval", TRAIN + VAL), ("test", TEST)):
        with open(os.path.join(root, "ImageSets", name + ".txt"), "w") as fh:
            fh.write("".join("%06d\n" % i for i in ids))
    seeds = {}
    for training, ids in ((True, sorted(TRAIN + VAL)), (False, TEST)):
        sub = os.path.join(root, "training" if training else "testing")
        for d in ("velodyne", "calib", "image_2") + (("label_2",) if training else ()):
            os.makedirs(os.path.join(sub, d), exist_ok=True)
        for idx in ids:
            seed = frame_seed(training, idx)
            seeds[(training, idx)] = seed
            synth_cloud(seed, fov_deg=180.0).tofile(os.path.join(sub, "velodyne", "%06d.bin" % idx))
            rig = idx % 2
            with open(os.path.join(sub, "calib", "%06d.txt" % idx), "w") as fh:
                fh.write(calib_text(rig))
            h, w = SHAPES[(idx // 2) % 2]
            with open(os.path.join(sub, "image_2", "%06d.png" % idx), "wb") as fh:
                fh.write(png_bytes(h, w))
            if training:
                rows = label_lines(idx, _rig(rig), np.random.default_rng(seed))
                with open(os.path.join(sub, "label_2", "%06d.txt" % idx), "w") as fh:
                    fh.write("".join(r + "\n" for r in rows))
    return seeds


def file_digest(path):
    with open(path, "rb") as fh:
        return hashlib.sha256(fh.read()).hexdigest()


def output_files(root):
    """Relative paths of the files create_data writes besides the pickles: reduced clouds and database files."""
    out = []
    for sub in ("training/velodyne_reduced", "testing/velodyne_reduced", "gt_database"):
        d = os.path.join(root, sub)
        if os.path.isdir(d):
            out += [sub + "/" + f for f in sorted(os.listdir(d))]
    return out


# -------------------------------------------------------------------------------------------- structures <-> arrays
def flatten(obj, prefix, out):
    """dicts, lists and leaves (numpy arrays and scalars, Python scalars and strings) -> npz entries under prefix."""
    if isinstance(obj, dict):
        out[prefix + "|keys"] = np.array([str(k) for k in obj], dtype=str)
        for k, v in obj.items():
            flatten(v, prefix + "|" + str(k), out)
    elif isinstance(obj, list):
        out[prefix + "|len"] = np.array(len(obj))
        for i, v in enumerate(obj):
            flatten(v, "%s|%d" % (prefix, i), out)
    else:
        out[prefix] = np.asarray(obj)
        out[prefix + "|type"] = np.array(type(obj).__name__)
    return out


def unflatten(z, prefix):
    """The inverse of flatten: (structure, with each leaf as (type name, array))."""
    if prefix + "|keys" in z:
        return {str(k): unflatten(z, prefix + "|" + str(k)) for k in z[prefix + "|keys"]}
    if prefix + "|len" in z:
        return [unflatten(z, "%s|%d" % (prefix, i)) for i in range(int(z[prefix + "|len"]))]
    return (str(z[prefix + "|type"]), z[prefix])


def leaves(obj):
    """A structure with its leaves as (type name, array), for comparing against unflatten's output."""
    if isinstance(obj, dict):
        return {str(k): leaves(v) for k, v in obj.items()}
    if isinstance(obj, list):
        return [leaves(v) for v in obj]
    return (type(obj).__name__, np.asarray(obj))


def assert_same(got, exp, where="root"):
    """Equal structures: same keys in the same order, same lengths, leaves of the same type, dtype, shape and bits."""
    if isinstance(exp, dict):
        assert isinstance(got, dict) and list(got) == list(exp), (where, list(got), list(exp))
        for k in exp:
            assert_same(got[k], exp[k], where + "." + k)
    elif isinstance(exp, list):
        assert isinstance(got, list) and len(got) == len(exp), (where, len(got), len(exp))
        for i, (g, e) in enumerate(zip(got, exp)):
            assert_same(g, e, "%s[%d]" % (where, i))
    else:
        (gt, ga), (et, ea) = got, exp
        assert gt == et, (where, gt, et)
        assert ga.dtype == ea.dtype and ga.shape == ea.shape, (where, ga.dtype, ea.dtype, ga.shape, ea.shape)
        assert np.ascontiguousarray(ga).tobytes() == np.ascontiguousarray(ea).tobytes(), (where, ga, ea)
