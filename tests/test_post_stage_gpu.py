"""pg_nms_boxes_3d on multi-frame batches, the one decode rule behind pg_decode_boxes and pg_postprocess, the detection
buffer retry of _lib.postprocess and the per-frame candidate limit of both NMS entry points.

Tolerance as in test_postprocess_gpu.py: kept sets, labels and indices identical; boxes and scores within 1e-4."""
import numpy as np
import pytest
import torch

from oracle import postprocess as pp

pytestmark = pytest.mark.gpu


def _cuda(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _table(c):
    from pointgnn_b200.models import box_encoding
    return box_encoding.class_table(pp.LABEL_MAPS['Car'], c)


def _candidates(seed, num_objects, per_object):
    """(labels, boxes [B,7] float32, scores float32) of one synthetic frame, as run.py selects them."""
    pts, enc, probs = pp.synthetic_outputs(seed, num_objects, per_object, 4)
    dec = pp.decode_boxes(enc, pts, pp.LABEL_MAPS['Car'])
    lab, boxes, scores, _ = pp.select_candidates(probs, dec, 4)
    return lab, boxes, scores


def _nms_batch():
    """Frames of different sizes, one of them a single box."""
    frames = [_candidates(41, 10, 20), _candidates(42, 3, 8), _candidates(43, 20, 25)]
    lab, boxes, scores = frames[1]
    frames.insert(2, (lab[:1], boxes[:1], scores[:1]))
    fp = np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)
    return frames, fp


@pytest.mark.parametrize('merge', [False, True])
@pytest.mark.parametrize('rescore', [False, True])
def test_nms_boxes_3d_multi_frame_vs_oracle(merge, rescore):
    from pointgnn_b200 import _lib
    frames, fp = _nms_batch()
    assert len(frames[2][0]) == 1
    lab = np.concatenate([f[0] for f in frames])
    boxes = np.vstack([f[1] for f in frames])
    scores = np.concatenate([f[2] for f in frames])
    out_l, out_b, out_s, out_i, dfp = _lib.nms_boxes_3d(_cuda(lab, torch.int32), _cuda(boxes), _cuda(scores), _cuda(fp),
                                                        0.01, merge, rescore)
    out_l, out_b, out_s, out_i = (t.cpu().numpy() for t in (out_l, out_b, out_s, out_i))
    dfp = dfp.cpu().numpy()
    assert dfp[0] == 0 and dfp[-1] == len(out_l) and np.all(np.diff(dfp) >= 0)
    for f, (fl, fb, fs) in enumerate(frames):
        want_l, want_b, want_s, order = pp.nms_boxes_3d_uncertainty(fl, fb, fs, 0.01, merge, rescore)
        sl = slice(dfp[f], dfp[f + 1])
        assert np.array_equal(out_i[sl] - fp[f], order)
        assert np.array_equal(out_l[sl], want_l)
        assert np.abs(out_b[sl] - want_b).max() < 1e-4
        assert np.abs(out_s[sl] - want_s).max() < 1e-4


def _int_corner_nms(labels, boxes, scores, thres, appr):
    """nms.py:109-131 (bboxes_nms, models.nms.nms_boxes_3d): plain greedy NMS on np.int32(corners * appr) with the
    fast_poly IoU.  -> order indices of the kept boxes into the input."""
    order = np.argsort(-scores)
    labels = np.asarray(labels)[order]
    corners = np.int32(pp.boxes_3d_to_corners(np.asarray(boxes)[order]) * appr)
    keep = np.ones(len(order), dtype=bool)
    for i in range(len(order) - 1):
        if keep[i]:
            ov = pp.overlapped_boxes_3d_fast_poly(corners[i], corners[i + 1:])
            keep[i + 1:] &= (ov <= thres) | (labels[i + 1:] != labels[i])
    return order[keep]


def test_nms_boxes_3d_int_corners_multi_frame():
    """PG_NMS_INT_CORNERS (appr_factor 100, as run.py's plain NMS) on the multi-frame batch, frame by frame."""
    from pointgnn_b200 import _lib
    frames, fp = _nms_batch()
    lab = np.concatenate([f[0] for f in frames])
    boxes = np.vstack([f[1] for f in frames])
    scores = np.concatenate([f[2] for f in frames])
    out_l, out_b, out_s, out_i, dfp = _lib.nms_boxes_3d(_cuda(lab, torch.int32), _cuda(boxes), _cuda(scores), _cuda(fp),
                                                        0.01, False, False, appr_factor=100.0, int_corners=True)
    out_l, out_b, out_s, out_i = (t.cpu().numpy() for t in (out_l, out_b, out_s, out_i))
    dfp = dfp.cpu().numpy()
    assert dfp[0] == 0 and dfp[-1] == len(out_l) and np.all(np.diff(dfp) >= 0)
    for f, (fl, fb, fs) in enumerate(frames):
        order = _int_corner_nms(fl, fb, fs, 0.01, 100.0)
        sl = slice(dfp[f], dfp[f + 1])
        assert np.array_equal(out_i[sl] - fp[f], order)
        assert np.array_equal(out_l[sl], fl[order])
        assert np.array_equal(out_b[sl], fb[order]) and np.array_equal(out_s[sl], fs[order])


def test_postprocess_boxes_are_decode_boxes():
    """Without merge every kept box is the pg_decode_boxes box of its (vertex, class), bit for bit."""
    from pointgnn_b200 import _lib
    frames = [pp.synthetic_outputs(51, 12, 20, 4), pp.synthetic_outputs(52, 5, 10, 4)]
    pts, enc, probs = (np.vstack([f[i] for f in frames]) for i in range(3))
    fp = np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)
    table = _table(4)
    det = _lib.postprocess(_cuda(probs), _cuda(enc), _cuda(pts), _cuda(fp), table, 0.01, merge=False, rescore=False)
    dec = _lib.decode_boxes(_cuda(enc), _cuda(pts), table).cpu().numpy().reshape(-1, 7)
    index = det['index'].cpu().numpy()
    assert len(index) > 0
    assert np.array_equal(det['box'].cpu().numpy().view(np.uint32), dec[index].view(np.uint32))


def test_postprocess_detection_buffer_retry():
    """More kept boxes than the first buffer guess max(1024, K): two perpendicular boxes per far-apart vertex (class 2
    decodes at yaw + pi/2; car-sized footprints overlap with IoU ~0.27 < 0.5), so all 2K candidates are kept."""
    from pointgnn_b200 import _lib
    k, c = 600, 4
    i = np.arange(k)
    pts = np.c_[(i % 25) * 20.0, np.ones(k), (i // 25) * 20.0].astype(np.float32)
    enc = np.zeros((k, c, 7), np.float32)
    enc[:, 1] = enc[:, 2] = np.random.default_rng(61).normal(0, 0.1, (k, 7)).astype(np.float32)
    enc[:, 1:3, 3:6] = 0.0                        # the median car size: IoU of the perpendicular pair 0.27
    probs = np.zeros((k, c), np.float32)
    probs[:, 1] = 0.3 + i * 1e-4                  # distinct scores: the order of the kept boxes is defined
    probs[:, 2] = 0.3 + (i + 0.5) * 1e-4
    probs[:, 0] = probs[:, 3] = (1.0 - probs[:, 1] - probs[:, 2]) / 2
    fp = np.array([0, k], np.int32)
    det = _lib.postprocess(_cuda(probs), _cuda(enc), _cuda(pts), _cuda(fp), _table(c), 0.5)
    assert len(det['label']) == 2 * k > max(1024, k)
    dec = pp.decode_boxes(enc, pts, pp.LABEL_MAPS['Car'])
    lab, boxes, scores, idx = pp.select_candidates(probs, dec, c)
    want_l, want_b, want_s, order = pp.nms_boxes_3d_uncertainty(lab, boxes, scores, 0.5)
    assert np.array_equal(det['index'].cpu().numpy(), idx[order])
    assert np.array_equal(det['label'].cpu().numpy(), want_l)
    assert np.abs(det['box'].cpu().numpy() - want_b).max() < 1e-4
    assert np.abs(det['score'].cpu().numpy() - want_s).max() < 1e-4
    assert np.array_equal(det['frame_ptr'].cpu().numpy(), [0, 2 * k])


def test_max_candidates_per_frame(monkeypatch):
    """A frame with more candidates than MAX_CANDIDATES_PER_FRAME raises PG_ERR_CAPACITY on both entry points; the
    next call within the limit succeeds."""
    from pointgnn_b200 import _lib
    monkeypatch.setattr(_lib, 'MAX_CANDIDATES_PER_FRAME', 32)
    table = _table(4)
    big = pp.synthetic_outputs(71, 10, 20, 4)        # ~100 candidates
    small = pp.synthetic_outputs(72, 2, 5, 4)        # <= 20 candidates
    for frames, ok in (([small, big], False), ([small, small], True)):
        pts, enc, probs = (np.vstack([f[i] for f in frames]) for i in range(3))
        fp = np.cumsum([0] + [len(f[0]) for f in frames]).astype(np.int32)
        args = (_cuda(probs), _cuda(enc), _cuda(pts), _cuda(fp), table, 0.01)
        dec = pp.decode_boxes(enc, pts, pp.LABEL_MAPS['Car'])
        lab, boxes, scores, idx = pp.select_candidates(probs, dec, 4)
        cfp = np.searchsorted(idx, fp * 4).astype(np.int32)      # candidate frame_ptr
        nms_args = (_cuda(lab, torch.int32), _cuda(boxes), _cuda(scores), _cuda(cfp), 0.01, True, True)
        if ok:
            assert np.diff(cfp).max() <= 32
            assert len(_lib.postprocess(*args)['label']) > 0
            assert len(_lib.nms_boxes_3d(*nms_args)[0]) > 0
            continue
        assert np.diff(cfp).max() > 32
        for call in (lambda: _lib.postprocess(*args), lambda: _lib.nms_boxes_3d(*nms_args)):
            with pytest.raises(_lib.PointGNNError) as e:
                call()
            assert e.value.code == _lib.PG_ERR_CAPACITY
