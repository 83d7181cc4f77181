"""Evaluate a checkpoint on a KITTI split end to end (the reference's tools/test.py), or detect on unlabelled data:

    python -m sassd_b200.test CONFIG CHECKPOINT --data-root DIR [--split val] [--batch 16]
                              [--lidar velodyne|velodyne_reduced] [--out DIR] [--workers N] [--json FILE]
                              [--losses] [--r40] [--coco]
    python -m sassd_b200.test CONFIG CHECKPOINT --data-root DIR --split test --out DIR [...]
    python -m sassd_b200.test CONFIG CHECKPOINT --drive DRIVE_DIR [--calib-dir DIR] --out DIR [...]
    python -m sassd_b200.test CONFIG CHECKPOINT --model CONFIG2 CHECKPOINT2 [--model ...] --data-root DIR [...]
    python -m sassd_b200.test CONFIG CHECKPOINT --checkpoints CHECKPOINT2 [...] --data-root DIR [--losses] [--r40] [--coco] [...]

Frames are read from disk a few batches ahead (kitti_data.Prefetcher) and streamed through the captured step
(SingleStageDetector.detect_stream): full sweeps (``--lidar velodyne``) are cropped to the camera frustum on the
device, and every step ends with the KITTI result formatter on the device (ops.kitti_format).  The last batch is
padded with empty frames whose results are dropped.  Prints the official AP table (kitti_eval), the frame rate (wall
clock of the streamed detection, the evaluation excluded) and the time spent waiting on reads.  ``--r40`` also prints
the table at 40 recall positions (kitti_eval.official_eval(recall_positions=40)), and ``--coco`` the reference's
COCO-style table, AP averaged over ten IoU thresholds per class (kitti_eval.coco_eval), after the official one(s).
All tables come from one evaluation (kitti_eval.eval_many), which runs on the device, against the split's labels as
kitti_eval.read_block parses them on the device.

``--losses`` (labelled splits): every frame also carries its ground truth (kitti_data.gt_from_anno) and the captured
step computes SA-SSD's six losses beside the detections (detect_stream(losses=True)); the result files and AP tables
are those of a run without it.  The driver prints each loss's mean over the batches that hold a real frame.  A
batch's losses are normalised per batch (by its frame count and positives), so the values depend on ``--batch``, as
the reference's depend on imgs_per_gpu; the last batch's padding frames count as frames without GT.

The test split (``testing/``) and raw drives (kitti_data.KittiDrive) have no labels: the driver writes the result
files (``--out`` is required) and prints the frame rate and read wait only.  A raw drive's full sweeps are cropped on
the device to the points that project into image 2 (ops.image_fov_crop, the reference's KittiVideo), and its result
files are named by the frames' stems, ``%010d.txt``.

``--model CONFIG CHECKPOINT`` (repeatable) adds a model after the positional one: the models run as one
detectors.DetectorSet, one model per class as the reference's single-class checkpoints are used.  Every step
voxelizes and builds the rulebooks once for all of them, each frame's result file holds every model's rows in model
order, and the AP table covers the models' classes in that order.  The models must share the voxel grid and may not
share a class; ``--losses`` takes one model.

``--checkpoints CHECKPOINT2 [...]`` validates several checkpoints of one config (e.g. those a training run saved) in
one pass over a labelled split: the models run as one detectors.CheckpointSweep, so every frame is read, cropped and
voxelized once, the rulebooks and anchor mask are built once and, with ``--losses``, the targets are assigned once, while
each checkpoint runs its own network.  The driver prints each checkpoint's AP table(s) and loss means under its file
name, then one summary line per checkpoint (moderate 3D AP per class, with ``--coco`` also its COCO-style AP,
rpn_cls_loss and loss_cls means); every checkpoint's tables come from one evaluation.  ``--out DIR``
writes each checkpoint's result files to DIR/<checkpoint stem>/.  Each checkpoint's output equals that of a run of its
own.

Under torchrun, frame i of the split goes to rank i mod W; at the end every rank contributes one fixed-size block of
KITTI rows and counts to a single all_gather_into_tensor (dist.DetectionGather) and rank 0 re-interleaves, writes and
evaluates; with ``--losses`` one more all_gather brings every rank's per-batch loss vectors to rank 0.  A checkpoint
sweep exchanges all checkpoints' rows in the one all_gather and all their loss vectors in the other.
"""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

DEFAULT_MAX_POINTS = {"velodyne": 131072, "velodyne_reduced": 32768}


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m sassd_b200.test", description=__doc__.split("\n\n")[0])
    p.add_argument("config")
    p.add_argument("checkpoint")
    src = p.add_mutually_exclusive_group(required=True)
    src.add_argument("--data-root", help="KITTI root holding ImageSets/ and training/ (testing/ for --split test)")
    src.add_argument("--drive", help="a raw KITTI drive directory (*_sync) holding image_02/ and velodyne_points/")
    p.add_argument("--calib-dir", default=None,
                   help="with --drive: the directory of calib_cam_to_cam.txt / calib_velo_to_cam.txt "
                        "(default: the drive's parent)")
    p.add_argument("--split", default="val")
    p.add_argument("--batch", type=int, default=16)
    p.add_argument("--lidar", default=None, choices=("velodyne", "velodyne_reduced"),
                   help="full sweeps (cropped on the device) or the offline-cropped reduced clouds (default velodyne)")
    p.add_argument("--max-points", type=int, default=None,
                   help="points per frame the captured step holds (default 131072 full, 32768 reduced)")
    p.add_argument("--out", default=None, help="write one KITTI result file %%06d.txt (drives: %%010d.txt) per frame "
                                               "here; required without labels (--split test, --drive)")
    p.add_argument("--workers", type=int, default=4, help="reader threads")
    p.add_argument("--depth", type=int, default=4, help="batches read ahead")
    p.add_argument("--json", default=None, help="write the AP arrays and rates here")
    p.add_argument("--losses", action="store_true",
                   help="also compute SA-SSD's losses against the split's labels in the detection step and print "
                        "their means over the batches")
    p.add_argument("--r40", action="store_true", help="also print the AP table at 40 recall positions")
    p.add_argument("--coco", action="store_true",
                   help="also print the COCO-style AP table (AP averaged over ten IoU thresholds per class)")
    p.add_argument("--model", nargs=2, action="append", default=[], metavar=("CONFIG", "CHECKPOINT"),
                   help="one more single-class model, run with the first as one set (repeatable)")
    p.add_argument("--checkpoints", nargs="+", default=[], metavar="CHECKPOINT",
                   help="more checkpoints of CONFIG, validated with CHECKPOINT in one pass over a labelled split")
    args = p.parse_args(argv)
    if args.batch < 1:
        p.error("--batch must be positive")
    if args.checkpoints:
        if args.model:
            p.error("--checkpoints sweeps checkpoints of one config: it does not combine with --model")
        if args.drive or args.split == "test":
            p.error("--checkpoints needs a labelled split: %s has no labels" % (
                "--drive" if args.drive else "--split test"))
        paths = [os.path.realpath(c) for c in [args.checkpoint] + args.checkpoints]
        if len(set(paths)) != len(paths):
            p.error("--checkpoints: a checkpoint is given twice")
        stems = [checkpoint_stem(c) for c in [args.checkpoint] + args.checkpoints]
        if args.out and len(set(stems)) != len(stems):
            p.error("--checkpoints with --out: two checkpoints have the same file stem, so their result directories "
                    "under %s would clash" % args.out)
    if args.losses and args.model:
        p.error("--losses computes one model's losses: it does not combine with --model")
    if args.losses and (args.drive or args.split == "test"):
        p.error("--losses needs a labelled split: %s has no labels" % ("--drive" if args.drive else "--split test"))
    if args.r40 and (args.drive or args.split == "test"):
        p.error("--r40 needs a labelled split: %s has no labels" % ("--drive" if args.drive else "--split test"))
    if args.coco and (args.drive or args.split == "test"):
        p.error("--coco needs a labelled split: %s has no labels" % ("--drive" if args.drive else "--split test"))
    if args.drive:
        if args.lidar == "velodyne_reduced":
            p.error("--drive reads full sweeps: --lidar velodyne_reduced does not apply")
    elif args.calib_dir is not None:
        p.error("--calib-dir goes with --drive")
    args.lidar = args.lidar or "velodyne"
    if (args.drive or args.split == "test") and not args.out:
        p.error("%s has no labels to evaluate against: --out is required" % ("--drive" if args.drive else "--split test"))
    if args.max_points is None:
        args.max_points = DEFAULT_MAX_POINTS[args.lidar]
    return args


def checkpoint_stem(path):
    """A checkpoint's file name without its extension: its result directory under --out."""
    return os.path.splitext(os.path.basename(path))[0]


def rank_batches(ids, rank, world, batch):
    """This rank's frames (ids[rank::world]) as padded batches; every rank gets the same number of batches so that the
    result blocks of the final exchange have one size."""
    from .kitti_data import padded_batches
    per_rank = math.ceil(len(ids) / world)
    n_batches = max(1, math.ceil(per_rank / batch))
    mine = list(ids[rank::world])
    return padded_batches(mine + [None] * (n_batches * batch - len(mine)), batch)


def gather_annos(annos_local, ids, class_names, cap, device):
    """Every rank's per-frame annotation dicts (its frames j*W + rank, padding included) -> the annotations of the
    split's frames ``ids``, in order, on every rank, through one all_gather of [rows | n_out]."""
    return gather_annos_many([annos_local], ids, class_names, cap, device)[0]


def gather_annos_many(annos_sets, ids, class_names, cap, device):
    """gather_annos for K sets of annotations of the same frames (one per checkpoint), in one all_gather: each local
    frame's K row blocks go one after another."""
    import torch
    from . import dist as D
    from .results import annos_from_rows, rows_from_annos
    K, F = len(annos_sets), len(annos_sets[0])
    rows, n_out = rows_from_annos([a[j] for j in range(F) for a in annos_sets], class_names, cap)
    g = D.DetectionGather(F * K, cap, device, width=2 * rows.shape[2])
    rows_all, n_all = g(torch.from_numpy(rows).to(device).view(torch.float32),
                        torch.from_numpy(n_out).to(device))
    W = rows_all.shape[0]          # [W, F*K, ...] -> global frame order (frame j*W + r), then the K blocks
    rows_all = rows_all.reshape(W, F, K, cap, -1).permute(1, 0, 2, 3, 4).reshape(W * F, K, cap, -1)
    n_all = n_all.reshape(W, F, K).permute(1, 0, 2).reshape(W * F, K)
    rows_all = rows_all.contiguous().view(torch.float64)[:len(ids)].cpu().numpy()
    n_all = n_all[:len(ids)].cpu().numpy()
    return [annos_from_rows(rows_all[:, k], n_all[:, k], class_names, ids) for k in range(K)]


def gather_losses(losses_local, n_real, device):
    """Every rank's per-batch loss vectors (ops.LOSS_KEYS order; a checkpoint sweep's K vectors one after another)
    and real-frame counts -> the vectors of the batches that hold a real frame, on every rank, in (batch, rank) order,
    through one all_gather (dist.DetectionGather)."""
    import torch
    from . import dist as D
    width = len(losses_local[0])
    g = D.DetectionGather(len(n_real), 1, device, width=width)
    vec = torch.tensor(losses_local, dtype=torch.float32).reshape(len(n_real), 1, width)
    vec_all, n_all = D.interleave(*g(vec.to(device), torch.tensor(n_real, dtype=torch.int32).to(device)))
    return [v[0].tolist() for v, n in zip(vec_all.cpu(), n_all.cpu().tolist()) if n > 0]


def write_results(out_dir, ids, annos, name="%06d.txt"):
    """One file per frame (``name`` % id), annos_to_kitti_label(with_score=True); a frame without detections gets an
    empty file.  The annotations hold dimensions as l, h, w; KITTI files hold h, w, l (what kitti_data.read_label and the
    official devkit read)."""
    from .results import annos_to_kitti_label
    os.makedirs(out_dir, exist_ok=True)
    for idx, anno in zip(ids, annos):
        lines = annos_to_kitti_label(dict(anno, dimensions=anno["dimensions"][:, [1, 2, 0]]), with_score=True)
        with open(os.path.join(out_dir, name % idx), "w") as fh:
            fh.write("".join(l + "\n" for l in lines))


def run(args, log=print):
    """Returns the result dict (AP arrays as nested lists and rates; rates only without labels) on rank 0, None on the
    other ranks."""
    import torch
    import sassd_b200 as S
    from . import dist as D
    from . import ops
    from .checkpoint import load_params_from_file
    from .kitti_data import KittiDrive, KittiSplit, Prefetcher

    if args.drive:
        split = KittiDrive(args.drive, args.calib_dir)
        if not split.ids:
            raise ValueError("drive %s has no frames" % args.drive)
    else:
        split = KittiSplit(args.data_root, args.split, args.lidar)
        if not split.ids:
            raise ValueError("split %s of %s lists no frames" % (args.split, args.data_root))
    cfg = S.Config.fromfile(args.config)
    rank, world, local = D.init_from_env()
    batches = rank_batches(split.ids, rank, world, args.batch)
    ops.require_cuda()                  # first device use below
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    model, _, _ = S.build_from_config(cfg, device=device)
    load_params_from_file(model, args.checkpoint)
    det_cap = model.extra_head.det_cap
    if args.model:                      # the positional model and every --model, run as one set
        members = [model]
        for cfg_m, ckpt_m in args.model:
            m, _, _ = S.build_from_config(S.Config.fromfile(cfg_m), device=device)
            load_params_from_file(m, ckpt_m)
            members.append(m)
        model = S.DetectorSet(members)
        det_cap = model.det_cap
    elif args.checkpoints:              # the positional checkpoint and every --checkpoints one, run as one sweep
        members = [model]
        for ckpt in args.checkpoints:
            m, _, _ = S.build_from_config(cfg, device=device)
            load_params_from_file(m, ckpt)
            members.append(m)
        model = S.CheckpointSweep(members)
    sweep = bool(args.checkpoints)
    K = len(args.checkpoints) + 1 if sweep else 1
    fov = bool(args.drive)
    crop = args.lidar == "velodyne" and not fov
    class_names = model.class_names
    if args.losses:                     # from here on every frame carries its GT over the model's classes
        split = KittiSplit(args.data_root, args.split, args.lidar, gt_classes=class_names)

    def items(reader):
        for ids, points, metas, *gts in reader:
            item = (points, [split.planes(m["calib"], m["img_shape"]) for m in metas], metas) if crop else (points, metas)
            if args.losses:
                item += (([b for b, _ in gts[0]], [l for _, l in gts[0]]),)
            yield item

    loss_kw = dict(losses=True) if args.losses else {}
    stream = lambda src: model.detect_stream(src, args.batch, args.max_points, depth=4, crop=crop,  # noqa: E731
                                             kitti=True, image_fov=fov, **loss_kw)
    for _ in stream([]):                # capture the slots' graphs before the clock starts
        pass
    torch.cuda.synchronize(device)
    reader = Prefetcher(split, batches, depth=args.depth, workers=args.workers)
    t0 = time.perf_counter()
    annos_local, losses_local = [[] for _ in range(K)], []      # per checkpoint; per batch (all checkpoints')
    for out in stream(items(reader)):
        outs = out if sweep else [out]
        if args.losses:
            losses_local.append([losses[k] for _, losses in outs for k in ops.LOSS_KEYS])
            outs = [o for o, _ in outs]
        for a, o in zip(annos_local, outs):
            a += o
    torch.cuda.synchronize(device)
    wall = time.perf_counter() - t0
    n_local = sum(i is not None for ids in batches for i in ids)
    wall = D.max_over_ranks(wall, device)

    if world > 1:
        dt_sets = gather_annos_many(annos_local, split.ids, class_names, det_cap, device)
    else:
        order = [i for ids in batches for i in ids]
        dt_sets = [[a for i, a in zip(order, local) if i is not None] for local in annos_local]
    per_batch = None
    if args.losses:
        per_batch = gather_losses(losses_local, [sum(i is not None for i in ids) for ids in batches], device)
    if rank != 0:
        D.barrier()
        return None
    dt_annos = dt_sets[0]
    if args.out and sweep:
        for path, dts in zip([args.checkpoint] + args.checkpoints, dt_sets):
            write_results(os.path.join(args.out, checkpoint_stem(path)), split.ids, dts, split.result_name)
    elif args.out:
        write_results(args.out, split.ids, dt_annos, split.result_name)
    fps = len(split.ids) / wall
    rate = "frames: %d (%d rank%s), %.1f frames/s, read wait %.3f s on rank 0 (%d of %d frames on rank 0)" % (
        len(split.ids), world, "s" if world > 1 else "", fps, reader.wait, n_local, len(split.ids))
    result = dict(frames=len(split.ids), world=world, batch=args.batch, lidar=args.lidar, frames_per_s=fps,
                  wall_s=wall, read_wait_s=reader.wait)
    if not split.labelled:
        log(rate)
        _write_json(args.json, result)
        D.barrier()
        return result
    from .kitti_eval import ap_lists, eval_many, read_block
    gt = read_block(os.path.join(split.dir, "label_2"), split.ids)
    if sweep:
        result["checkpoints"] = _report_sweep(args, gt, dt_sets, class_names, per_batch, log)
        log(rate)
        _write_json(args.json, result)
        D.barrier()
        return result
    ev = eval_many(gt, [dt_annos], class_names, _tables(args))[0]
    text, ap = ev[11]
    log(text, end="")
    result.update(text=text, ap=ap_lists(ap))
    if args.r40:
        log(ev[40][0], end="")
        result.update(text_r40=ev[40][0], ap_r40=ap_lists(ev[40][1]))
    if args.coco:
        log(ev["coco"][0], end="")
        result.update(text_coco=ev["coco"][0], ap_coco=ap_lists(ev["coco"][1]))
    if args.losses:
        result.update(_loss_means(per_batch, args.batch, log))
    log(rate)
    _write_json(args.json, result)
    D.barrier()
    return result


def _tables(args):
    """The kitti_eval.eval_many tables the arguments ask for."""
    return (11,) + ((40,) if args.r40 else ()) + (("coco",) if args.coco else ())


def _loss_means(per_batch, batch, log):
    """Print the mean of each loss over the per-batch vectors; returns the result dict's losses entries."""
    from . import ops
    means = np.mean(np.asarray(per_batch, np.float64), axis=0)
    log("losses: mean over %d batches of %d frames (per-batch values depend on --batch): %s" % (
        len(per_batch), batch, ", ".join("%s %.6f" % (k, v) for k, v in zip(ops.LOSS_KEYS, means))))
    return dict(losses=dict(zip(ops.LOSS_KEYS, means.tolist())),
                losses_per_batch=[dict(zip(ops.LOSS_KEYS, v)) for v in per_batch])


def _report_sweep(args, gt, dt_sets, class_names, per_batch, log):
    """Evaluate and print each checkpoint of a sweep (one kitti_eval.eval_many for all of them), then one summary line
    per checkpoint: moderate 3D AP per class at the class's strict overlap (R11, and R40 with --r40), the moderate 3D
    COCO-style AP with --coco, and the rpn_cls_loss / loss_cls means.  Returns the result dict's ``checkpoints``
    list."""
    from . import ops
    from .kitti_eval import eval_many, report_sets
    paths = [args.checkpoint] + args.checkpoints
    n = len(ops.LOSS_KEYS)

    def losses(k, entry):
        if per_batch is None:
            return []
        entry.update(_loss_means([v[k * n:(k + 1) * n] for v in per_batch], args.batch, log))
        return ["rpn_cls_loss %.6f loss_cls %.6f" % (entry["losses"]["rpn_cls_loss"], entry["losses"]["loss_cls"])]
    return report_sets([dict(path=p) for p in paths], [os.path.basename(p) for p in paths],
                       eval_many(gt, dt_sets, class_names, _tables(args)), class_names, "checkpoints", log, losses)


def _write_json(path, result):
    if path:
        with open(path, "w") as fh:
            json.dump(result, fh, indent=1)


def main(argv=None):
    return run(parse_args(argv))


if __name__ == "__main__":
    main(sys.argv[1:])
    sys.exit(0)
