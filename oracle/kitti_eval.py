"""CPU restatement of the reference's KITTI evaluation (SURVEY.md §8 row f4) — TEST INFRASTRUCTURE ONLY.

Only tests/ may import this module (it is the checker for sassd_b200.kitti_eval, never the thing shipped).
Pinned against the reference itself: tests/golden/eval.npz holds overlaps, AP tables and the printed result of
mmdet/core/evaluation/kitti_eval.py run in the build container with numba's CUDA simulator
(tests/golden/make_golden_eval.py).

Follows, function by function:
  rotated overlap      mmdet/core/post_processing/rotate_nms_gpu.py:153-381 (corners, quadrilateral
                       intersection, vertex sort, fan area), :536-548 (criterion), :592-627 (float32 I/O)
  image_box_overlap    mmdet/core/evaluation/kitti_eval.py:95-122
  d3 overlap           :130-161
  clean_data           :39-92
  get_thresholds       :17-36
  compute_statistics   :164-283
  eval / mAP           :549-657 (eval_class_v3), :683-688 (get_mAP_v2), :690-710 (do_eval_v2),
                       :791-851 (get_official_eval_result)
Plain Python loops: use on small cases only.
"""
import math

import numpy as np

F = np.float32


# ------------------------------------------------------------------ rotated overlap (float32)
def _corners(box):
    """rotate_nms_gpu.py:340-363: clockwise corners, rotated clockwise by the angle."""
    cx, cy, dx, dy, ang = (F(v) for v in box)
    c, s = F(math.cos(ang)), F(math.sin(ang))
    xs = [-dx / F(2), -dx / F(2), dx / F(2), dx / F(2)]
    ys = [-dy / F(2), dy / F(2), dy / F(2), -dy / F(2)]
    out = []
    for x, y in zip(xs, ys):
        out.append((F(c * x + s * y + cx), F(-s * x + c * y + cy)))
    return out


def _inside(px, py, q):
    """:297-313 point_in_quadrilateral (projections on the edges a->b and a->d)."""
    ab0, ab1 = q[1][0] - q[0][0], q[1][1] - q[0][1]
    ad0, ad1 = q[3][0] - q[0][0], q[3][1] - q[0][1]
    ap0, ap1 = px - q[0][0], py - q[0][1]
    abab = ab0 * ab0 + ab1 * ab1
    abap = ab0 * ap0 + ab1 * ap1
    adad = ad0 * ad0 + ad1 * ad1
    adap = ad0 * ap0 + ad1 * ap1
    return abab >= abap and abap >= 0 and adad >= adap and adap >= 0


def _segment_hit(p1, p2, i, j):
    """:209-252 line_segment_intersection of edge i of p1 with edge j of p2."""
    a, b = p1[i], p1[(i + 1) % 4]
    c, d = p2[j], p2[(j + 1) % 4]
    ba0, ba1 = b[0] - a[0], b[1] - a[1]
    da0, ca0 = d[0] - a[0], c[0] - a[0]
    da1, ca1 = d[1] - a[1], c[1] - a[1]
    acd = da1 * ca0 > ca1 * da0
    bcd = (d[1] - b[1]) * (c[0] - b[0]) > (c[1] - b[1]) * (d[0] - b[0])
    if acd != bcd:
        abc = ca1 * ba0 > ba1 * ca0
        abd = da1 * ba0 > ba1 * da0
        if abc != abd:
            dc0, dc1 = d[0] - c[0], d[1] - c[1]
            abba = a[0] * b[1] - b[0] * a[1]
            cddc = c[0] * d[1] - d[0] * c[1]
            dh = ba1 * dc0 - ba0 * dc1
            return (F((abba * dc0 - ba0 * cddc) / dh), F((abba * dc1 - ba1 * cddc) / dh))
    return None


def _clipped_area(p1, p2, amin):
    """csrc/kitti_eval.cu clipped_area: Sutherland-Hodgman clipping of p1 against p2's edges in float64 (Python float
    operations in the kernel's order), rounded to float32 and clamped to [0, amin]."""
    sx, sy = [float(x) for x, _ in p1], [float(y) for _, y in p1]
    s2 = 0.0
    for i in range(4):
        k = (i + 1) % 4
        s2 += float(p2[i][0]) * float(p2[k][1]) - float(p2[k][0]) * float(p2[i][1])
    if not s2 != 0.0:
        return F(0)
    sg = 1.0 if s2 > 0.0 else -1.0
    for e in range(4):
        if not sx:
            break
        ax, ay = float(p2[e][0]), float(p2[e][1])
        ex, ey = float(p2[(e + 1) % 4][0]) - ax, float(p2[(e + 1) % 4][1]) - ay
        d = [sg * (ex * (y - ay) - ey * (x - ax)) for x, y in zip(sx, sy)]
        n, tx, ty = len(sx), [], []
        for i in range(n):
            k = 0 if i + 1 == n else i + 1
            if d[i] >= 0.0 and len(tx) < 16:
                tx.append(sx[i]); ty.append(sy[i])
            if (d[i] >= 0.0) != (d[k] >= 0.0) and len(tx) < 16:
                t = d[i] / (d[i] - d[k])
                tx.append(sx[i] + t * (sx[k] - sx[i])); ty.append(sy[i] + t * (sy[k] - sy[i]))
        sx, sy = tx, ty
    a = 0.0
    for i in range(len(sx)):
        k = 0 if i + 1 == len(sx) else i + 1
        a += sx[i] * sy[k] - sx[k] * sy[i]
    r = F(abs(a) * 0.5)
    return r if r < amin else amin


def collected_points(box1, box2):
    """The points quadrilateral_intersection (:317-337) collects: corners inside the other box, then edge hits."""
    p1, p2 = _corners(box1), _corners(box2)
    pts = []
    for i in range(4):
        if _inside(p1[i][0], p1[i][1], p2):
            pts.append(p1[i])
        if _inside(p2[i][0], p2[i][1], p1):
            pts.append(p2[i])
    for i in range(4):
        for j in range(4):
            hit = _segment_hit(p1, p2, i, j)
            if hit is not None:
                pts.append(hit)
    return p1, p2, pts


def rotated_intersection(box1, box2):
    """Area of the intersection polygon of two rotated boxes (x, y, dx, dy, angle) — `inter`, :366-380.  Past 8
    collected points, where the reference overruns its 8-point buffer and is undefined, the kernel's fp64 clipping
    (csrc/kitti_eval.cu, the comment at pts[24])."""
    p1, p2, pts = collected_points(box1, box2)
    if len(pts) > 8:
        return _clipped_area(p1, p2, min(abs(F(box1[2]) * F(box1[3])), abs(F(box2[2]) * F(box2[3]))))
    n = len(pts)
    if n > 0:                                            # :169-206 sort by a monotone key of the polar angle
        cx = F(sum(p[0] for p in pts) / F(n))
        cy = F(sum(p[1] for p in pts) / F(n))
        keys = []
        for p in pts:
            vx, vy = p[0] - cx, p[1] - cy
            d = F(math.sqrt(vx * vx + vy * vy))
            vx, vy = vx / d, vy / d
            keys.append(F(-2) - vx if vy < 0 else vx)
        for i in range(1, n):                            # insertion sort, same comparison sequence
            if keys[i - 1] > keys[i]:
                tk, tp, j = keys[i], pts[i], i
                while j > 0 and keys[j - 1] > tk:
                    keys[j], pts[j] = keys[j - 1], pts[j - 1]
                    j -= 1
                keys[j], pts[j] = tk, tp
    area = 0.0                                           # :153-166 triangle fan about the first vertex
    for i in range(n - 2):
        a, b, c = pts[0], pts[i + 1], pts[i + 2]
        area += abs(((a[0] - c[0]) * (b[1] - c[1]) - (a[1] - c[1]) * (b[0] - c[0])) / 2.0)
    return area


def rotate_iou_eval(boxes, query_boxes, criterion=-1):
    """[N,5] x [K,5] -> [N,K]; criterion -1 IoU, 0 / area(query), 1 / area(box), 2 raw intersection (:536-548;
    the kernel passes the QUERY box first, :586-588)."""
    boxes = np.asarray(boxes, np.float32)
    query_boxes = np.asarray(query_boxes, np.float32)
    out = np.zeros((boxes.shape[0], query_boxes.shape[0]), np.float32)
    for n in range(boxes.shape[0]):
        for k in range(query_boxes.shape[0]):
            q, b = query_boxes[k], boxes[n]
            a1, a2 = q[2] * q[3], b[2] * b[3]
            it = rotated_intersection(q, b)
            if criterion == -1:
                v = it / (a1 + a2 - it)
            elif criterion == 0:
                v = it / a1
            elif criterion == 1:
                v = it / a2
            else:
                v = it
            out[n, k] = v
    return out


def image_box_overlap(boxes, query_boxes, criterion=-1):
    """kitti_eval.py:95-122."""
    N, K = boxes.shape[0], query_boxes.shape[0]
    out = np.zeros((N, K), dtype=boxes.dtype)
    for k in range(K):
        qa = (query_boxes[k, 2] - query_boxes[k, 0]) * (query_boxes[k, 3] - query_boxes[k, 1])
        for n in range(N):
            iw = min(boxes[n, 2], query_boxes[k, 2]) - max(boxes[n, 0], query_boxes[k, 0])
            if iw > 0:
                ih = min(boxes[n, 3], query_boxes[k, 3]) - max(boxes[n, 1], query_boxes[k, 1])
                if ih > 0:
                    if criterion == -1:
                        ua = (boxes[n, 2] - boxes[n, 0]) * (boxes[n, 3] - boxes[n, 1]) + qa - iw * ih
                    elif criterion == 0:
                        ua = (boxes[n, 2] - boxes[n, 0]) * (boxes[n, 3] - boxes[n, 1])
                    elif criterion == 1:
                        ua = qa
                    else:
                        ua = 1.0
                    out[n, k] = iw * ih / ua
    return out


def d3_box_overlap(boxes, qboxes, criterion=-1):
    """Camera-frame boxes (x, y, z, l, h, w, ry): BEV intersection x height overlap, :130-161."""
    rinc = rotate_iou_eval(boxes[:, [0, 2, 3, 5, 6]], qboxes[:, [0, 2, 3, 5, 6]], 2)
    for i in range(boxes.shape[0]):
        for j in range(qboxes.shape[0]):
            if rinc[i, j] > 0:
                iw = min(boxes[i, 1], qboxes[j, 1]) - max(boxes[i, 1] - boxes[i, 4], qboxes[j, 1] - qboxes[j, 4])
                if iw > 0:
                    a1 = boxes[i, 3] * boxes[i, 4] * boxes[i, 5]
                    a2 = qboxes[j, 3] * qboxes[j, 4] * qboxes[j, 5]
                    inc = iw * rinc[i, j]
                    ua = {-1: a1 + a2 - inc, 0: a1, 1: a2}.get(criterion, 1.0)
                    rinc[i, j] = inc / ua
                else:
                    rinc[i, j] = 0.0
    return rinc


def frame_overlaps(gt, dt, metric):
    """overlaps[dt, gt] of one frame (calculate_iou_partly is called with (dt, gt), :584)."""
    if metric == 0:
        return image_box_overlap(dt["bbox"], gt["bbox"])
    if metric == 1:
        def bev(a):
            return np.concatenate([a["location"][:, [0, 2]], a["dimensions"][:, [0, 2]], a["rotation_y"][:, None]], 1)
        return rotate_iou_eval(bev(dt), bev(gt)).astype(np.float64)

    def cam(a):
        return np.concatenate([a["location"], a["dimensions"], a["rotation_y"][:, None]], 1)
    return d3_box_overlap(cam(dt), cam(gt)).astype(np.float64)


# ------------------------------------------------------------------ matching
CLASS_NAMES = ['car', 'pedestrian', 'cyclist', 'van', 'person_sitting', 'car', 'tractor', 'trailer']
MIN_HEIGHT, MAX_OCCLUSION, MAX_TRUNCATION = [40, 25, 25], [0, 1, 2], [0.15, 0.3, 0.5]


def clean_data(gt, dt, current_class, difficulty):
    """:39-92 -> (num_valid_gt, ignored_gt, ignored_dt, dontcare boxes)."""
    cls = CLASS_NAMES[current_class].lower()
    ign_gt, ign_dt, dc, valid = [], [], [], 0
    for i in range(len(gt["name"])):
        name = gt["name"][i].lower()
        height = gt["bbox"][i][3] - gt["bbox"][i][1]
        if name == cls:
            vc = 1
        elif (cls == "pedestrian" and name == "person_sitting") or (cls == "car" and name == "van"):
            vc = 0
        else:
            vc = -1
        ignore = (gt["occluded"][i] > MAX_OCCLUSION[difficulty] or gt["truncated"][i] > MAX_TRUNCATION[difficulty]
                  or height <= MIN_HEIGHT[difficulty])
        if vc == 1 and not ignore:
            ign_gt.append(0); valid += 1
        elif vc == 0 or (ignore and vc == 1):
            ign_gt.append(1)
        else:
            ign_gt.append(-1)
        if gt["name"][i] == "DontCare":
            dc.append(gt["bbox"][i])
    for i in range(len(dt["name"])):
        vc = 1 if dt["name"][i].lower() == cls else -1
        height = abs(dt["bbox"][i, 3] - dt["bbox"][i, 1])
        ign_dt.append(1 if height < MIN_HEIGHT[difficulty] else (0 if vc == 1 else -1))
    return valid, ign_gt, ign_dt, dc


def get_thresholds(scores, num_gt, num_sample_pts=41):
    """:17-36."""
    scores = np.sort(np.asarray(scores, np.float64))[::-1]
    cur, out = 0.0, []
    for i, s in enumerate(scores):
        l = (i + 1) / num_gt
        r = (i + 2) / num_gt if i < len(scores) - 1 else l
        if (r - cur) < (cur - l) and i < len(scores) - 1:
            continue
        out.append(s)
        cur += 1 / (num_sample_pts - 1.0)
    return out


def compute_statistics(overlaps, gt_alpha, dt_bbox, dt_alpha, dt_score, ign_gt, ign_dt, dc, metric, min_overlap,
                       thresh=0.0, compute_fp=False, compute_aos=False):
    """:164-283 -> tp, fp, fn, similarity, scores of the true positives."""
    nd, ng = len(dt_score), len(ign_gt)
    assigned = [False] * nd
    below = [compute_fp and dt_score[j] < thresh for j in range(nd)]
    NO = -10000000
    tp = fp = fn = 0
    similarity = 0
    tp_scores, delta = [], []
    for i in range(ng):
        if ign_gt[i] == -1:
            continue
        det, valid, max_ov, assigned_ign = -1, NO, 0, False
        for j in range(nd):
            if ign_dt[j] == -1 or assigned[j] or below[j]:
                continue
            ov = overlaps[j, i]
            if not compute_fp and ov > min_overlap and dt_score[j] > valid:
                det, valid = j, dt_score[j]
            elif compute_fp and ov > min_overlap and (ov > max_ov or assigned_ign) and ign_dt[j] == 0:
                max_ov, det, valid, assigned_ign = ov, j, 1, False
            elif compute_fp and ov > min_overlap and valid == NO and ign_dt[j] == 1:
                det, valid, assigned_ign = j, 1, True
        if valid == NO and ign_gt[i] == 0:
            fn += 1
        elif valid != NO and (ign_gt[i] == 1 or ign_dt[det] == 1):
            assigned[det] = True
        elif valid != NO:
            tp += 1
            tp_scores.append(dt_score[det])
            if compute_aos:
                delta.append(gt_alpha[i] - dt_alpha[det])
            assigned[det] = True
    if compute_fp:
        for j in range(nd):
            if not (assigned[j] or ign_dt[j] == -1 or ign_dt[j] == 1 or below[j]):
                fp += 1
        nstuff = 0
        if metric == 0 and len(dc):
            ov_dc = image_box_overlap(np.asarray(dt_bbox, np.float64), np.asarray(dc, np.float64), 0)
            for i in range(len(dc)):
                for j in range(nd):
                    if assigned[j] or ign_dt[j] in (-1, 1) or below[j]:
                        continue
                    if ov_dc[j, i] > min_overlap:
                        assigned[j] = True
                        nstuff += 1
        fp -= nstuff
        if compute_aos:
            if tp > 0 or fp > 0:      # :271-279: np.sum over [zeros(fp), (1 + cos(delta)) / 2 ...]
                tmp = np.zeros((fp + len(delta),))
                for i, d in enumerate(delta):
                    tmp[i + fp] = (1.0 + np.cos(d)) / 2.0
                similarity = np.sum(tmp)
            else:
                similarity = -1
    return tp, fp, fn, similarity, tp_scores


def eval_classes(gt_annos, dt_annos, classes, difficulties, metric, min_overlaps, compute_aos=False):
    """eval_class_v3, :549-657.  min_overlaps [num_minoverlap, metric, class] -> precision / recall / aos
    [class, difficulty, minoverlap, 41]."""
    nfr = len(gt_annos)
    overlaps = [frame_overlaps(gt_annos[i], dt_annos[i], metric) for i in range(nfr)]
    shape = (len(classes), len(difficulties), len(min_overlaps), 41)
    precision, recall, aos = np.zeros(shape), np.zeros(shape), np.zeros(shape)
    for m, cls in enumerate(classes):
        for l, diff in enumerate(difficulties):
            prep = [clean_data(gt_annos[i], dt_annos[i], cls, diff) for i in range(nfr)]
            total_valid = sum(p[0] for p in prep)
            for k, mo in enumerate(min_overlaps[:, metric, m]):
                def run(i, thresh, fp):
                    g, d = gt_annos[i], dt_annos[i]
                    return compute_statistics(overlaps[i], g["alpha"], d["bbox"], d["alpha"], d["score"], prep[i][1],
                                              prep[i][2], prep[i][3], metric, mo, thresh, fp, compute_aos and fp)
                scores = []
                for i in range(nfr):
                    scores += run(i, 0.0, False)[4]
                ths = get_thresholds(np.array(scores), total_valid)
                pr = np.zeros((len(ths), 4))
                for i in range(nfr):
                    for t, th in enumerate(ths):
                        tp, fp, fn, sim, _ = run(i, th, True)
                        pr[t, 0] += tp; pr[t, 1] += fp; pr[t, 2] += fn
                        if sim != -1:
                            pr[t, 3] += sim
                for t in range(len(ths)):
                    recall[m, l, k, t] = pr[t, 0] / (pr[t, 0] + pr[t, 2])
                    precision[m, l, k, t] = pr[t, 0] / (pr[t, 0] + pr[t, 1])
                    if compute_aos:
                        aos[m, l, k, t] = pr[t, 3] / (pr[t, 0] + pr[t, 1])
                for t in range(len(ths)):
                    precision[m, l, k, t] = np.max(precision[m, l, k, t:])
                    recall[m, l, k, t] = np.max(recall[m, l, k, t:])
                    if compute_aos:
                        aos[m, l, k, t] = np.max(aos[m, l, k, t:])
    return dict(recall=recall, precision=precision, orientation=aos)


def get_map(prec):
    """:683-688: 11-point interpolation over the 41 sampled recalls."""
    return sum(prec[..., i] for i in range(0, prec.shape[-1], 4)) / 11 * 100


OVERLAP_0_7 = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7]] * 3)
OVERLAP_0_5 = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5],
                        [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5]])
CLASS_TO_NAME = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist', 3: 'Van', 4: 'Person_sitting', 5: 'car', 6: 'tractor',
                 7: 'trailer'}


def official_eval(gt_annos, dt_annos, current_classes, difficulties=(0, 1, 2)):
    """get_official_eval_result, :791-851 -> (text, dict of AP arrays [class, difficulty, minoverlap])."""
    if not isinstance(current_classes, (list, tuple)):
        current_classes = [current_classes]
    name_to_class = {v: k for k, v in CLASS_TO_NAME.items()}
    classes = [name_to_class[c] if isinstance(c, str) else c for c in current_classes]
    min_overlaps = np.stack([OVERLAP_0_7, OVERLAP_0_5], 0)[:, :, classes]
    compute_aos = False
    for anno in dt_annos:
        if anno['alpha'].shape[0] != 0:
            compute_aos = anno['alpha'][0] != -10
            break
    diffs = list(difficulties)
    r0 = eval_classes(gt_annos, dt_annos, classes, diffs, 0, min_overlaps, compute_aos)
    ap = dict(bbox=get_map(r0["precision"]), aos=get_map(r0["orientation"]) if compute_aos else None,
              bev=get_map(eval_classes(gt_annos, dt_annos, classes, diffs, 1, min_overlaps)["precision"]),
              d3=get_map(eval_classes(gt_annos, dt_annos, classes, diffs, 2, min_overlaps)["precision"]))
    text = ''
    for j, c in enumerate(classes):
        for i in range(min_overlaps.shape[0]):
            text += "%s AP@%.2f, %.2f, %.2f:\n" % ((CLASS_TO_NAME[c],) + tuple(min_overlaps[i, :, j]))
            for key, label in (("bbox", "bbox AP"), ("bev", "bev  AP"), ("d3", "3d   AP")):
                text += "%s:%.2f, %.2f, %.2f\n" % (label, ap[key][j, 0, i], ap[key][j, 1, i], ap[key][j, 2, i])
            if compute_aos:
                text += "aos  AP:%.2f, %.2f, %.2f\n" % (ap["aos"][j, 0, i], ap["aos"][j, 1, i], ap["aos"][j, 2, i])
    return text, ap
