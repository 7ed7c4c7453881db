"""NMS and KITTI-evaluator decisions at the overlap thresholds, against exact rational arithmetic
(oracle/exact_overlap.py) on the boundary families of tests/test_overlap_exact_cpu.py.

A decision is asserted only where the perturbation interval of the exact overlap (cos / sin moved by a few ulp, plus
the fp64 rounding of the clipper) lies on one side of the threshold; with yaw 0 and dyadic boxes one inside the other
every value is exact and exact ties are asserted too.  Inside an interval the reference's own float result may differ
from exact math; that is not asserted."""
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import exact_overlap as ex
from oracle import kitti_eval as ke
from test_overlap_exact_cpu import DEGENERATE, FAMILIES, kitti_families, nms_families

pytestmark = pytest.mark.gpu


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _nms(pairs, thres, merge=False, rescore=False, labels=(1, 1), scores=(0.5, 0.25), int_corners=False):
    """One two-box frame per pair (a scored above b) in one batched pg_nms_boxes_3d call -> (kept count per frame,
    kept scores, kept boxes, det frame_ptr)."""
    from pointgnn_b200 import _lib
    n = len(pairs)
    boxes = np.stack([np.stack([a, b]) for a, b in pairs]).reshape(-1, 7).astype(np.float32)
    lab = np.tile(np.array(labels, np.int32), n)
    sc = np.tile(np.array(scores, np.float32), n)
    fp = np.arange(0, 2 * n + 1, 2, dtype=np.int32)
    _, box, score, index, dfp = _lib.nms_boxes_3d(_cuda(lab), _cuda(boxes), _cuda(sc), _cuda(fp), thres, merge, rescore,
                                                  appr_factor=100.0 if int_corners else 0.0, int_corners=int_corners)
    dfp = dfp.cpu().numpy()
    return np.diff(dfp), score.cpu().numpy(), box.cpu().numpy(), dfp, index.cpu().numpy()


def _exact_ties():
    """Yaw 0, dyadic boxes, the single box inside the other: IoU exactly 0.5 and 0.01 (as the double quotient), and
    their float32 neighbours in size."""
    out = []
    for t, lb in ((0.5, 8.0), (0.01, 400.0)):
        a = np.array([1.0, 1.0, 10.0, 4.0, 1.0, 2.0, 0.0], np.float32)          # 4 x 2 x 1
        b = np.array([1.0, 1.0, 10.0, lb, 1.0, 2.0, 0.0], np.float32)           # lb x 2 x 1, around a
        for l in (lb, np.nextafter(np.float32(lb), np.float32(0)), np.nextafter(np.float32(lb), np.float32(1e9))):
            bb = b.copy()
            bb[3] = l
            out.append(dict(family='tie', t=t, a=a, b=bb, exact=True))
    return out


_PAIRS = {}


def _pairs():
    if not _PAIRS:
        fams = nms_families(variants=4, seed=11)
        for p in fams:
            p['exact'] = False
        _PAIRS['all'] = fams + _exact_ties()
    return _PAIRS['all']


def _certified(pairs, thres, appr=None):
    """-> (asserted indices, expected removed flags) for the pairs whose interval excludes thres."""
    idx, removed = [], []
    for i, p in enumerate(pairs):
        if p['t'] != thres:
            continue
        interval = ex.nms_iou_interval(p['a'], p['b'], appr=appr, exact_fp=p['exact'])
        d = ex.decide(interval, thres)
        if d is not None:
            idx.append(i)
            removed.append(d)
    return np.array(idx), np.array(removed)


@pytest.mark.parametrize('thres', [0.01, 0.5])
def test_nms_decisions_match_exact(thres):
    """The second box is kept iff its exact IoU with the first is <= thres; with different labels both are kept."""
    pairs = _pairs()
    idx, removed = _certified(pairs, thres)
    sel = [(pairs[i]['a'], pairs[i]['b']) for i in idx]
    kept, *_ = _nms(sel, thres)
    assert np.array_equal(kept == 1, removed)
    for fam in FAMILIES:                    # no family may be swallowed by its intervals
        assert any(pairs[i]['family'] == fam for i in idx), fam
    ties = [k for k, i in enumerate(idx) if pairs[i]['family'] == 'tie']
    assert len(ties) == 3 and not removed[ties[0]]          # the exact tie is kept: IoU > thres is false
    kept, *_ = _nms(sel, thres, labels=(1, 3))
    assert np.all(kept == 2)
    print('thres %g: %d of %d pairs asserted, %s' % (thres, len(idx), sum(p['t'] == thres for p in pairs),
                                                      {f: sum(pairs[i]['family'] == f for i in idx) for f in FAMILIES}))


@pytest.mark.parametrize('merge', [False, True])
def test_nms_rescore_iou_matches_exact(merge):
    """merge=False, rescore=True, thres 0.01: the kept score is s1 + s2 * IoU; with merge the IoU is the merged
    (median) box's with the second box.  The IoU backed out of the float32 score must lie in the exact interval."""
    pairs = [p for p in _pairs() if p['t'] == 0.5]
    s1, s2 = 0.5, 0.25
    kept, score, box, dfp, _ = _nms([(p['a'], p['b']) for p in pairs], 0.01, merge=merge, rescore=True,
                                    scores=(s1, s2))
    checked = 0
    for f, p in enumerate(pairs):
        if kept[f] != 1:
            continue
        single = p['a']
        if merge:
            single = np.median(np.stack([p['b'], p['a']]), axis=0).astype(np.float32)
            assert np.array_equal(box[dfp[f]], single)
        lo, hi = ex.nms_iou_interval(single, p['b'], exact_fp=p['exact'])
        got = (float(score[dfp[f]]) - s1) / s2
        tol = float(np.spacing(np.float32(score[dfp[f]]))) / s2
        assert lo - tol <= got <= hi + tol, (p['family'], got, lo, hi)
        checked += 1
    assert checked > 0.8 * len(pairs)


def test_nms_int_corners_decisions_match_exact():
    """int_corners (appr_factor 100): the truncated corners are enumerated where the trig can flip a truncation;
    with yaw 0 every decision is asserted, exact ties included (bboxes_nms keeps iff ov <= thres)."""
    pairs = _pairs()
    for thres in (0.01, 0.5):
        idx, removed = _certified(pairs, thres, appr=100.0)
        kept, *_ = _nms([(pairs[i]['a'], pairs[i]['b']) for i in idx], thres, int_corners=True)
        assert np.array_equal(kept == 1, removed), thres
        yaw0 = [i for i, p in enumerate(pairs) if p['t'] == thres and p['family'] in ('yaw0', 'shared_edge', 'tie')]
        assert set(yaw0) <= set(idx.tolist())
        assert len(idx) > 0.5 * sum(p['t'] == thres for p in pairs)


@pytest.mark.parametrize('int_corners', [False, True])
@pytest.mark.parametrize('merge, rescore', [(False, False), (True, True)])
def test_nms_degenerate_boxes(int_corners, merge, rescore):
    """Zero length / width / height and thres 0 with touching boxes: the rules of DEGENERATE (checked against the
    reference's nms.py in test_overlap_exact_cpu.py).  A NaN overlap (0 / 0) never removes a box under the merge /
    rescore variants' `overlap > thres` and always removes it under bboxes_nms's `keep iff overlap <= thres`."""
    if int_corners and merge:
        pytest.skip('the int_corners path is bboxes_nms: no merge / rescore')
    for name, thres, boxes, keep_unc, keep_plain, _ in DEGENERATE:
        a, b = np.array(boxes, np.float32)
        kept, score, _, _, index = _nms([(a, b)], thres, merge=merge, rescore=rescore, scores=(0.9, 0.5),
                                        int_corners=int_corners)
        want = keep_plain if int_corners else keep_unc
        assert list(index) == want, name
        if rescore:
            assert np.all(np.isfinite(score)), name


def test_nms_intersection_is_rounded_to_float32():
    """nms.py's IoU is np.float32(intersection) / (union - intersection).  With a (l = w = 1 + 2^-20) inside the
    4 x 2 x 1 box b every value is exact: the intersection (1 + 2^-20)^2 rounds to 1 + 2^-19 in float32, so at
    thres = (1 + 2^-19) / 8 the IoU ties the threshold and the second box is kept; without the rounding it would
    exceed it."""
    e = np.float32(1 + 2.0 ** -20)
    a = np.array([1.0, 1.0, 10.0, e, 1.0, e, 0.0], np.float32)
    b = np.array([1.0, 1.0, 10.0, 4.0, 1.0, 2.0, 0.0], np.float32)
    tie = (1 + 2.0 ** -19) / 8
    assert ex.nms_iou(ex.nms_corners(a), ex.nms_corners(b)) == tie
    assert ex.decide(ex.nms_iou_interval(a, b, exact_fp=True), tie) is False
    for thres, kept in ((tie, 2), (np.nextafter(tie, 0), 1)):
        assert _nms([(a, b)], thres)[0][0] == kept, thres


# ---------------------------------------------------------------------------------------------
# the KITTI evaluator
# ---------------------------------------------------------------------------------------------
_CLASS = {0.7: ('Car', 0), 0.5: ('Pedestrian', 1)}


def _fmt(row):
    return ' '.join(repr(float(v)) for v in row)


def _frames(items):
    """-> (gt_texts, det_texts): one ground-truth row and one detection per item (item: name, gt, det)."""
    gts, dets = [], []
    for name, gt_name, g, d in items:
        gts.append('%s %r %d %s\n' % (gt_name, float(g[0]), int(g[1]), _fmt(g[2:])))     # the occlusion is an int
        dets.append('%s %s\n' % (name, _fmt(d)))
    return gts, dets


def _eval_items(metric, criterion, variants, seed):
    """Certified frames of one metric: (items, decisions, classes) where a decision is exact overlap > min_overlap."""
    items, dec, codes = [], [], []
    for fam in kitti_families(variants=variants, seed=seed, metric=metric, criterion=criterion):
        name, code = _CLASS[fam['t']]
        if fam['t'] == 0.5 and len(items) % 2:
            name, code = 'Cyclist', 2
        interval = ex.eval_overlap_interval(fam['gt'], fam['det'], metric, criterion)
        d = ex.decide(interval, fam['t'])
        if d is None:
            continue
        g, det = fam['gt'].copy(), fam['det'].copy()
        det[14] = 0.001 * (len(items) + 1)
        items.append((name, 'DontCare' if criterion == 0 else name, g, det))
        dec.append(d)
        codes.append(code)
    return items, np.array(dec), np.array(codes)


def _parse(gt_texts, det_texts, tmp_path):
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    gt_dir, res_dir = str(tmp_path / 'gt'), str(tmp_path / 'res')
    ke.write_tree(gt_dir, res_dir, gt_texts, det_texts)
    return gt_dir, res_dir, ev.load_tree(gt_dir, res_dir)


@pytest.mark.parametrize('metric, criterion', [(1, -1), (2, -1), (1, 0), (2, 0)])
def test_evaluator_decisions_match_exact(metric, criterion, tmp_path, monkeypatch):
    """One ground-truth row and one detection per frame, aimed at 0.7 (car) and 0.5 (pedestrian, cyclist); criterion
    0 puts the detection on a DontCare region.  tp / fp / fn follow from the exact decisions under `overlap >
    min_overlap`: the NumPy restatement run with those decisions in place of its overlaps gives the expected counts."""
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    items, dec, codes = _eval_items(metric, criterion, variants=1, seed=21 + metric + criterion)
    assert len(items) > 60 and dec.any() and (~dec).any()
    if criterion == 0:     # DontCare frames alone have no TP and so no thresholds: add exact matches of each class
        for name, code in (('Car', 0), ('Pedestrian', 1), ('Cyclist', 2)):
            for k in range(3):
                g, d = items[0][2].copy(), items[0][2].copy()
                d = np.r_[-1.0, -1.0, d[2:], 0.9 - 0.01 * k - 0.001 * code]
                items.append((name, name, g, d))
                dec = np.r_[dec, True]
    _, _, (_, groundtruth, detections) = _parse(*_frames(items), tmp_path)
    got = ev.evaluate_frames(groundtruth, detections)
    table = {(g.tobytes(), d.tobytes()): (1.0 if x else 0.0) for (_, _, g, d), x in zip(items, dec)}
    real = ke.overlaps

    def overlaps(gt, gcodes, det):
        out = real(gt, gcodes, det)
        out[metric, 0, 0] = table[(gt[0].tobytes(), det[0].tobytes())]
        return out
    monkeypatch.setattr(ke, 'overlaps', overlaps)
    want = ke.evaluate_arrays(groundtruth, detections)
    for k in ('num_thresholds', 'tp', 'fp', 'fn'):
        assert np.array_equal(got[k][metric], want[k][metric]), k
    assert want['num_thresholds'][metric].sum() > 0


def test_evaluator_image_ties(tmp_path):
    """Dyadic image boxes at exact overlaps 0.7 / 0.5 and a quarter pixel either side; a tie is not a match
    (`overlap > min_overlap`), also for criterion 0 on a DontCare region."""
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    geo = [1.5, 1.6, 3.9, 0.0, 1.6, 20.0, 0.0]
    items, want = [], []
    k = 0
    for name, t in (('Car', 0.7), ('Pedestrian', 0.5), ('Cyclist', 0.5)):
        for dc in (False, True):
            for dw in (0.0, 0.25, -0.25):
                width = 100.0 * t + dw
                if not dc:   # detection [100, 100 + width] inside [100, 200]: overlap width / 100
                    g = np.array([0.0, 0, 0, 100, 100, 200, 200] + geo)
                    d = np.array([-1.0, -1, 0, 100, 100, 100 + width, 200] + geo + [0.5 + 0.001 * k])
                else:        # detection [100, 200] on a DontCare region [100, 100 + width]: criterion 0, width / 100
                    g = np.array([-1.0, -1, -10, 100, 100, 100 + width, 200] + geo)
                    d = np.array([-1.0, -1, 0, 100, 100, 200, 200] + geo + [0.5 + 0.001 * k])
                o = ex.image_overlap(d, g, 0 if dc else -1)
                assert (o == t) == (dw == 0)
                items.append((name, 'DontCare' if dc else name, g, d))
                want.append(o > t)
                k += 1
    _, _, (_, groundtruth, detections) = _parse(*_frames(items), tmp_path)
    got = ev.evaluate_frames(groundtruth, detections)
    for i, (name, gname, g, d) in enumerate(items):
        o = ke.overlaps(g[None], [ev.class_code(gname)], d[None])[0, 0, 0]
        assert (o > (0.7 if name == 'Car' else 0.5)) == want[i], (name, gname, o)
    want_arr = ke.evaluate_arrays(groundtruth, detections)
    for key in ('num_thresholds', 'tp', 'fp', 'fn'):
        assert np.array_equal(got[key][0], want_arr[key][0]), key
    # the ties: no TP from them, so each class has exactly its one above-threshold ordinary frame as a TP
    assert np.array_equal(got['tp'][0, :, :, 0], np.ones((3, 3)))


def test_boundary_tree_matches_compiled_reference(tmp_path):
    """The reference evaluator binary on a tree of certified boundary frames (no redraw near the cuts): its files
    equal the GPU's."""
    from oracle import kitti_eval_build
    binary = kitti_eval_build.binary()
    if binary is None:
        pytest.skip('oracle/_ref/evaluate_object_3d_offline was not built (no reference tree)')
    from pointgnn_b200.kitti_native_evaluation import evaluate_object_3d_offline as ev
    items = []
    for metric in (1, 2):
        items += _eval_items(metric, -1, variants=1, seed=31 + metric)[0]
    texts = _frames(items)
    gt_a, res_a, _ = _parse(*texts, tmp_path / 'a')
    gt_b, res_b, _ = _parse(*texts, tmp_path / 'b')
    subprocess.run([binary, gt_b, res_b], capture_output=True, text=True, check=True)
    r = ev.evaluate(gt_a, res_a)
    assert r['files']
    for rel, text in r['files'].items():
        with open(os.path.join(res_b, rel)) as f:
            want = f.read()
        if 'orientation' in rel:
            a, b = text.split(), want.split()
            assert len(a) == len(b) and all(x == y or abs(float(x) - float(y)) <= 5.01e-7 for x, y in zip(a, b)), rel
        else:
            assert text == want, rel
