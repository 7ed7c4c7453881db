"""NumPy restatement of the reference's KITTI evaluator (kitti_native_evaluation/src/evaluate_object_3d_offline.cpp).

TEST INFRASTRUCTURE ONLY.  It computes what ``pg_kitti_eval`` computes - tp / fp / fn per threshold, the number of
thresholds and the precision / AOS / AHS curves of every (metric, class, difficulty) - and is checked against the
goldens of the compiled reference evaluator (tests/golden/kitti_eval_*.json, made by tools/make_golden.py).  It is
the comparison target on trees too large to commit.

The computation follows eval_class (:639-739) frame by frame and GT row by GT row in the reference's order; the
PR pass runs all thresholds of a curve at once as rows of NumPy arrays.  Footprint intersections use the Sutherland-
Hodgman clipper of oracle/postprocess.py.
"""
import numpy as np

from oracle.postprocess import clip_convex, polygon_area
from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev

MIN_HEIGHT = [40, 25, 25]
MAX_OCCLUSION = [0, 1, 2]
MAX_TRUNCATION = [0.15, 0.3, 0.5]
NO_DETECTION = -10000000.0
DONTCARE = 5


def _footprints(v):
    """toPolygon (:265-288) of every row of v: [n, 4, 2] (x, z) corners."""
    l, w, t1, t3, ry = v[:, 9], v[:, 8], v[:, 10], v[:, 12], v[:, 13]
    c, s = np.cos(ry), np.sin(ry)
    lx = np.stack([l / 2, l / 2, -l / 2, -l / 2], 1)
    lz = np.stack([w / 2, -w / 2, -w / 2, w / 2], 1)
    x = c[:, None] * lx + s[:, None] * lz + t1[:, None]
    z = -s[:, None] * lx + c[:, None] * lz + t3[:, None]
    return np.stack([x, z], 2)


def overlaps(gt, gt_codes, det):
    """[3, D, G] overlaps of a frame: image / ground / 3D, criterion -1 against ordinary rows and 0 against DontCare."""
    ng, nd = len(gt), len(det)
    out = np.zeros((3, nd, ng))
    if ng == 0 or nd == 0:
        return out
    dc = (np.asarray(gt_codes) == DONTCARE)[None, :]
    d, g = det[:, None, :], gt[None, :, :]
    with np.errstate(divide='ignore', invalid='ignore'):
        w = np.minimum(d[..., 5], g[..., 5]) - np.maximum(d[..., 3], g[..., 3])
        h = np.minimum(d[..., 6], g[..., 6]) - np.maximum(d[..., 4], g[..., 4])
        inter = w * h
        a_area = (d[..., 5] - d[..., 3]) * (d[..., 6] - d[..., 4])
        b_area = (g[..., 5] - g[..., 3]) * (g[..., 6] - g[..., 4])
        img = np.where(dc, inter / a_area, inter / (a_area + b_area - inter))
        out[0] = np.where((w <= 0) | (h <= 0), 0.0, img)
        gp, dp = _footprints(gt), _footprints(det)
        g_area = np.array([polygon_area(p) for p in gp])
        d_area = np.array([polygon_area(p) for p in dp])
        inter_area = np.zeros((nd, ng))
        gc, dcn = gp.mean(1), dp.mean(1)
        gr = np.sqrt(((gp - gc[:, None]) ** 2).sum(-1)).max(1)
        dr = np.sqrt(((dp - dcn[:, None]) ** 2).sum(-1)).max(1)
        for j in range(nd):
            near = np.sqrt(((gc - dcn[j]) ** 2).sum(-1)) <= gr + dr[j] + 1e-9
            for i in np.nonzero(near)[0]:
                inter_area[j, i] = polygon_area(clip_convex(gp[i], dp[j]))
        out[1] = np.where(dc, inter_area / d_area[:, None], inter_area / (g_area[None, :] + d_area[:, None] - inter_area))
        ymax = np.minimum(d[..., 11], g[..., 11])
        ymin = np.maximum(d[..., 11] - d[..., 7], g[..., 11] - g[..., 7])
        inter_vol = inter_area * np.maximum(0.0, ymax - ymin)
        det_vol = d[..., 7] * d[..., 9] * d[..., 8]
        gt_vol = g[..., 7] * g[..., 9] * g[..., 8]
        out[2] = np.where(dc, inter_vol / det_vol, inter_vol / (det_vol + gt_vol - inter_vol))
    return out


def clean_data(cls, diff, gt, gt_codes, det, det_codes):
    """cleanData (:378-451) -> (ignored_gt [G], ignored_det [D], n_gt)."""
    ig_gt = np.full(len(gt), -1, np.int64)
    for i in range(len(gt)):
        code = gt_codes[i]
        valid = 1 if code == cls else (0 if (cls == 1 and code == 4) or (cls == 0 and code == 3) else -1)
        height = gt[i, 6] - gt[i, 4]
        ignore = gt[i, 1] > MAX_OCCLUSION[diff] or gt[i, 0] > MAX_TRUNCATION[diff] or height <= MIN_HEIGHT[diff]
        if valid == 1 and not ignore:
            ig_gt[i] = 0
        elif valid == 0 or (ignore and valid == 1):
            ig_gt[i] = 1
    height = np.abs(det[:, 4] - det[:, 6]).astype(np.int32) if len(det) else np.zeros(0, np.int32)
    ig_det = np.where(height < MIN_HEIGHT[diff], 1, np.where(np.asarray(det_codes) == cls, 0, -1)).astype(np.int64)
    return ig_gt, ig_det, int((ig_gt == 0).sum())


def compute_statistics(ov, gt, gt_codes, det, ig_gt, ig_det, min_ov, thresh, compute_aos, compute_aos_ground):
    """computeStatistics (:453-633) of one frame.  thresh None: the recall pass (-> list of TP scores); else an array
    of T thresholds, all run at once (-> tp, fp, fn, similarity, similarity_ground, each [T])."""
    fp_mode = thresh is not None
    nd = len(det)
    t = len(thresh) if fp_mode else 1
    scores = det[:, 14] if nd else np.zeros(0)
    assigned = np.zeros((t, nd), bool)
    below = scores[None, :] < np.asarray(thresh)[:, None] if fp_mode else np.zeros((1, nd), bool)
    tp, fn = np.zeros(t, np.int64), np.zeros(t, np.int64)
    sim, sim_g = np.zeros(t), np.zeros(t)
    tp_scores = []
    rows = np.arange(t)
    for i in range(len(gt)):
        if ig_gt[i] == -1:
            continue
        o = ov[:, i]
        elig = (ig_det != -1)[None, :] & ~assigned & ~below & (o > min_ov)[None, :]
        if not fp_mode:
            cand = elig[0] & (scores > NO_DETECTION)
            valid = np.array([cand.any()])
            idx = np.array([int(np.argmax(np.where(cand, scores, -np.inf)))]) if valid[0] else np.zeros(1, np.int64)
        else:
            e0 = elig & (ig_det == 0)[None, :]
            e1 = elig & (ig_det == 1)[None, :]
            has0, has1 = e0.any(1), e1.any(1)
            j0 = np.argmax(np.where(e0, o[None, :], -np.inf), axis=1) if nd else np.zeros(t, np.int64)
            j1 = np.argmax(e1, axis=1) if nd else np.zeros(t, np.int64)
            valid = has0 | has1
            idx = np.where(has0, j0, j1)
        fn += (~valid) & (ig_gt[i] == 0)
        ign = valid & ((ig_gt[i] == 1) | (ig_det[idx] == 1)) if nd else valid
        is_tp = valid & ~ign
        if nd:
            assigned[rows[valid], idx[valid]] = True
        tp += is_tp
        if not fp_mode and is_tp[0]:
            tp_scores.append(scores[idx[0]])
        if compute_aos:
            sim = np.where(is_tp, sim + (1.0 + np.cos(gt[i, 2] - det[idx, 2] if nd else 0.0)) / 2.0, sim)
        if compute_aos_ground:
            sim_g = np.where(is_tp, sim_g + (1.0 + np.cos(np.abs(gt[i, 13] - det[idx, 13]) if nd else 0.0)) / 2.0, sim_g)
    if not fp_mode:
        return tp_scores
    fp = (~(assigned | (ig_det == -1)[None, :] | (ig_det == 1)[None, :] | below)).sum(1)
    for i in range(len(gt)):
        if gt_codes[i] != DONTCARE:
            continue
        cand = ~assigned & (ig_det == 0)[None, :] & ~below & (ov[:, i] > min_ov)[None, :]
        assigned |= cand
        fp = fp - cand.sum(1)
    empty = ~((tp > 0) | (fp > 0))
    if compute_aos:
        sim = np.where(empty, -1.0, sim)
    if compute_aos_ground:
        sim_g = np.where(empty, -1.0, sim_g)
    return tp, fp, fn, sim, sim_g


def get_thresholds(v, n_groundtruth):
    """getThresholds (:343-376), keeping at most 41 (pg_kitti_eval's defined behaviour)."""
    v = sorted(v, reverse=True)
    t = []
    current_recall = 0.0
    for i in range(len(v)):
        l_recall = (i + 1) / float(n_groundtruth)
        r_recall = (i + 2) / float(n_groundtruth) if i < len(v) - 1 else l_recall
        if (r_recall - current_recall) < (current_recall - l_recall) and i < len(v) - 1:
            continue
        t.append(v[i])
        current_recall += 1.0 / (41 - 1.0)
    return t[:41]


def _max_element(v, i):
    largest = i
    for j in range(i + 1, len(v)):
        if v[largest] < v[j]:
            largest = j
    return v[largest]


def evaluate_arrays(groundtruth, detections):
    """The raw arrays pg_kitti_eval returns, for per-frame (types, values) lists."""
    compute_aos, _ = ev.eval_flags(detections)
    frames = []
    for (gn, gv), (dn, dv) in zip(groundtruth, detections):
        gv = np.asarray(gv, np.float64).reshape(-1, ev.GT_FIELDS)
        dv = np.asarray(dv, np.float64).reshape(-1, ev.DET_FIELDS)
        gc = np.array([ev.class_code(n) for n in gn], np.int64)
        dc = np.array([ev.class_code(n) for n in dn], np.int64)
        frames.append((gv, gc, dv, dc, overlaps(gv, gc, dv)))
    out = {k: np.zeros((3, 3, 3, 41)) for k in ('precision', 'aos', 'ahs')}
    out.update({k: np.zeros((3, 3, 3, 41), np.int32) for k in ('tp', 'fp', 'fn')})
    out['num_thresholds'] = np.zeros((3, 3, 3), np.int32)
    with np.errstate(divide='ignore', invalid='ignore'):
        for c in range(3):
            min_ov = 0.7 if c == 0 else 0.5
            for d in range(3):
                cleaned = [clean_data(c, d, gv, gc, dv, dc) for gv, gc, dv, dc, _ in frames]
                n_gt = sum(x[2] for x in cleaned)
                for m in range(3):
                    do_aos, do_ahs = m == 0 and compute_aos, m != 0
                    v = []
                    for (gv, gc, dv, dc, ov), (ig, idt, _) in zip(frames, cleaned):
                        v += compute_statistics(ov[m], gv, gc, dv, ig, idt, min_ov, None, False, False)
                    thr = np.array(get_thresholds(v, n_gt))
                    n = len(thr)
                    out['num_thresholds'][m, c, d] = n
                    if n == 0:
                        continue
                    tp, fp, fn = np.zeros(n, np.int64), np.zeros(n, np.int64), np.zeros(n, np.int64)
                    sim, sim_g = np.zeros(n), np.zeros(n)
                    for (gv, gc, dv, dc, ov), (ig, idt, _) in zip(frames, cleaned):
                        a, b, e, s, sg = compute_statistics(ov[m], gv, gc, dv, ig, idt, min_ov, thr, do_aos, do_ahs)
                        tp += a
                        fp += b
                        fn += e
                        sim = np.where(s != -1, sim + s, sim)
                        sim_g = np.where(sg != -1, sim_g + sg, sim_g)
                    out['tp'][m, c, d, :n], out['fp'][m, c, d, :n], out['fn'][m, c, d, :n] = tp, fp, fn
                    den = (tp + fp).astype(np.float64)
                    curves = [tp / den, sim / den if do_aos else None, sim_g / den if do_ahs else None]
                    for key, cur in zip(('precision', 'aos', 'ahs'), curves):
                        if cur is None:
                            continue
                        full = np.zeros(41)
                        full[:n] = cur
                        for i in range(n):
                            full[i] = _max_element(full, i)
                        out[key][m, c, d] = full
    return out


def evaluate_frames(groundtruth, detections):
    """Same result as evaluate_object_3d_offline.evaluate_frames, computed on the CPU."""
    compute_aos, evaluated = ev.eval_flags(detections)
    return ev.report(evaluate_arrays(groundtruth, detections), compute_aos, evaluated)


def evaluate_tree(gt_dir, result_dir):
    """evaluate_frames on a result tree (frames in ascending index order); files are not written."""
    _, groundtruth, detections = ev.load_tree(gt_dir, result_dir)
    return evaluate_frames(groundtruth, detections)


# ---------------------------------------------------------------------------------------------
# seeded synthetic trees
# ---------------------------------------------------------------------------------------------
_GT_TYPES = ['Car', 'car', 'CAR', 'Van', 'Pedestrian', 'pedestrian', 'Person_sitting', 'Cyclist', 'cYcList',
             'DontCare', 'Misc', 'Truck']
_GT_WEIGHTS = [0.3, 0.05, 0.03, 0.07, 0.14, 0.03, 0.04, 0.1, 0.02, 0.1, 0.06, 0.06]
_SIZE = {0: (1.5, 1.6, 3.9), 1: (1.75, 0.6, 0.8), 2: (1.7, 0.6, 1.8), 3: (2.2, 1.9, 5.0), 4: (1.2, 0.6, 0.8)}
_DET_NAME = {0: ['Car', 'car'], 1: ['Pedestrian', 'PEDESTRIAN'], 2: ['Cyclist', 'cyclist'], 3: ['Car', 'Van'],
             4: ['Pedestrian', 'Person_sitting']}
_HEIGHT_CUTS = [24.5, 25.0, 25.5, 39.5, 40.0, 40.5]
_DET_HEIGHT_CUTS = [24.6, 25.0, 25.3, 39.7, 40.0, 40.2]


def _fmt(values, digits):
    return ['%.*f' % (digits, v) for v in values]


def _gt_row(rng, name):
    code = ev.class_code(name)
    if code == DONTCARE:
        x1, y1 = rng.uniform(0, 1000), rng.uniform(100, 300)
        x2, y2 = x1 + rng.uniform(20, 200), y1 + rng.uniform(15, 80)
        return [name] + _fmt([-1], 2) + ['-1'] + _fmt([-10, x1, y1, x2, y2, -1, -1, -1, -1000, -1000, -1000, -10], 2)
    h0, w0, l0 = _SIZE.get(code, (1.6, 1.0, 2.0))
    height = rng.choice(_HEIGHT_CUTS) if rng.random() < 0.35 else rng.uniform(15, 150)
    x1, y1 = rng.uniform(0, 1100), rng.uniform(100, 300)
    x2, y2 = x1 + height * rng.uniform(0.5, 2.0), y1 + height
    trunc = rng.choice([0.0, 0.1, 0.15, 0.2, 0.3, 0.4, 0.5, 0.6])
    occ = int(rng.integers(0, 4))
    vals = [rng.uniform(-np.pi, np.pi), x1, y1, x2, y2, h0 * rng.uniform(0.85, 1.15), w0 * rng.uniform(0.85, 1.15),
            l0 * rng.uniform(0.85, 1.15), rng.uniform(-15, 15), rng.uniform(1.0, 2.2), rng.uniform(5, 45),
            rng.uniform(-np.pi, np.pi)]
    return [name] + _fmt([trunc], 2) + [str(occ)] + _fmt(vals, 2)


def _det_row(rng, name, like=None, score_digits=2, frac_height=True):
    if like is None:     # a false positive somewhere
        code = ev.class_code(name)
        h0, w0, l0 = _SIZE.get(code, (1.6, 1.0, 2.0))
        x1, y1, hgt = rng.uniform(-5, 1100), rng.uniform(100, 300), rng.uniform(15, 150)
        box = [x1, y1, x1 + hgt * rng.uniform(0.5, 2), y1 + hgt]
        geo = [h0, w0, l0, rng.uniform(-15, 15), rng.uniform(1.0, 2.2), rng.uniform(5, 45), rng.uniform(-np.pi, np.pi)]
        alpha = rng.uniform(-np.pi, np.pi)
    else:
        g = [float(v) for v in like[1:]]
        bw, bh = g[5] - g[3], g[6] - g[4]
        box = [g[3] + rng.normal(0, 0.07 * bw), g[4] + rng.normal(0, 0.07 * bh), g[5] + rng.normal(0, 0.07 * bw),
               g[6] + rng.normal(0, 0.07 * bh)]
        if frac_height and rng.random() < 0.25:
            box[3] = box[1] + rng.choice(_DET_HEIGHT_CUTS)
        geo = [g[7] * rng.uniform(0.85, 1.15), g[8] * rng.uniform(0.85, 1.15), g[9] * rng.uniform(0.85, 1.15),
               g[10] + rng.normal(0, 0.3), g[11] + rng.normal(0, 0.25), g[12] + rng.normal(0, 0.3),
               g[13] + rng.normal(0, 0.3)]
        alpha = g[2] + rng.normal(0, 0.4)
    if rng.random() < 0.03:
        geo[3] = -1000
    score = rng.uniform(0, 1)
    return [name, '-1', '-1'] + _fmt([alpha] + box + geo, 2) + _fmt([score], score_digits)


def _parse_rows(rows, width):
    return [r[0] for r in rows], np.array([[float(v) for v in r[1:]] for r in rows], np.float64).reshape(len(rows), width)


def _near_cut(gt_rows, det_rows):
    gn, gv = _parse_rows(gt_rows, ev.GT_FIELDS)
    dn, dv = _parse_rows(det_rows, ev.DET_FIELDS)
    ov = overlaps(gv, [ev.class_code(n) for n in gn], dv)
    return bool(np.any((np.abs(ov - 0.5) < 1e-9) | (np.abs(ov - 0.7) < 1e-9)))


def synthetic_tree(seed, num_frames, big_frames=(), alpha_invalid=False, never_detected=(), score_digits=2):
    """Seeded KITTI label and result texts -> (gt_texts, det_texts), lists of file contents per frame.

    The frames mix every class the evaluator distinguishes (in mixed case), heights / occlusion / truncation on both
    sides of each difficulty cut, fractional detection heights, detections on DontCare regions, tied scores (scores
    rounded to `score_digits`), t1 = -1000 detections, empty ground-truth and empty result files.  big_frames: indices
    of frames with >= 200 detections.  never_detected: class codes that get no detection.  Any frame with an overlap
    within 1e-9 of 0.5 or 0.7 is drawn again, so that results do not depend on the clipper's last bits."""
    rng = np.random.default_rng(seed)
    gt_texts, det_texts = [], []
    for f in range(num_frames):
        while True:
            ng = 0 if f % 17 == 5 else int(rng.integers(1, 13))     # some empty label files
            gts = [_gt_row(rng, rng.choice(_GT_TYPES, p=_GT_WEIGHTS)) for _ in range(ng)]
            dets = []
            if f % 13 != 4:                                             # some empty result files
                for g in gts:
                    code = ev.class_code(g[0])
                    if code == DONTCARE:
                        if rng.random() < 0.7:     # a detection inside the DontCare region
                            x1, y1, x2, y2 = [float(v) for v in g[4:8]]
                            like = ['x', '0', '0', '0', '%f' % x1, '%f' % y1, '%f' % x2, '%f' % y2, '1.5', '1.6', '3.9',
                                    '%f' % rng.uniform(-10, 10), '1.6', '%f' % rng.uniform(5, 40), '0']
                            dets.append(_det_row(rng, rng.choice(['Car', 'Pedestrian', 'Cyclist']), like, score_digits,
                                                 False))
                        continue
                    if code > 4:
                        if rng.random() < 0.3:
                            dets.append(_det_row(rng, g[0], g, score_digits))
                        continue
                    for _ in range(int(rng.choice([0, 1, 1, 1, 2]))):
                        dets.append(_det_row(rng, rng.choice(_DET_NAME[code]), g, score_digits))
                nfp = int(rng.integers(0, 5)) + (int(rng.integers(200, 240)) if f in big_frames else 0)
                for _ in range(nfp):
                    dets.append(_det_row(rng, rng.choice(['Car', 'pedestrian', 'Cyclist', 'Misc', 'Van']), None,
                                         score_digits))
                if nfp and f in big_frames:       # big frames also get many true-ish detections of their objects
                    for g in gts:
                        if ev.class_code(g[0]) <= 4:
                            for _ in range(8):
                                dets.append(_det_row(rng, rng.choice(_DET_NAME[ev.class_code(g[0])]), g, score_digits))
                dets = [d for d in dets if ev.class_code(d[0]) not in never_detected]
                if rng.random() < 0.3 and len(dets) > 1:     # an exact score tie inside the frame
                    dets[-1][-1] = dets[0][-1]
            if not _near_cut(gts, dets):
                break
        if alpha_invalid and f == num_frames // 2 and dets:
            dets[0][3] = '-10'
        gt_texts.append(''.join(' '.join(r) + '\n' for r in gts))
        det_texts.append(''.join(' '.join(r) + ' \n' for r in dets) + '\n')
    return gt_texts, det_texts


def write_tree(gt_dir, result_dir, gt_texts, det_texts, names=None):
    """Write label files into gt_dir and result files into result_dir/data/ (names: file names, default NNNNNN.txt)."""
    import os
    names = names or ['%06d.txt' % i for i in range(len(gt_texts))]
    os.makedirs(gt_dir, exist_ok=True)
    os.makedirs(os.path.join(result_dir, 'data'), exist_ok=True)
    for name, g, d in zip(names, gt_texts, det_texts):
        with open(os.path.join(gt_dir, name), 'w') as f:
            f.write(g)
        with open(os.path.join(result_dir, 'data', name), 'w') as f:
            f.write(d)
