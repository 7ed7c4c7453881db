"""pg_kitti_rows (models.postprocess.kitti_rows) against run.kitti_labels, the NumPy form pinned to the reference's
result text in test_kitti_cpu.py, frame by frame: the same surviving rows in the same order, the float32 fields
(h, w, l, x, y, z, yaw) bit-identical, the float64 fields (clipped 2-D box, rescored score) within 1e-9 relative, and
every field of the type kitti_labels gives it, so that write_kitti_file prints the same text.

Inputs: the detections behind the reference's own kitti_result_car.txt (post_car.npz with kitti_calib.txt), and
seeded random batches of 1 to 9 frames with frames without detections, frames without candidates, boxes across
each image edge (truncation on both sides of 0.4), boxes behind other boxes with many candidates inside, and three
calibrations.  A frame whose truncation rate lies within 1e-9 of 0.4, or with a candidate within 1e-9 of a box face,
is drawn again, so that the comparison pins decisions and not rounding."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu
CALIB_FILE = os.path.join(GOLDEN, 'kitti_calib.txt')
NUM_CLASSES = 4
MARGIN = 1e-9


def _calibs():
    from pointgnn_b200.dataset import kitti_dataset
    base = kitti_dataset.parse_calib(CALIB_FILE)
    out = []
    for scale, shift in ((1.0, 0.0), (0.93, 11.5), (1.08, -7.25)):
        p2 = base['P2'].copy()
        p2[0, 0] *= np.float32(scale)
        p2[1, 1] *= np.float32(scale)
        p2[0, 2] += np.float32(shift)
        out.append({'cam_to_image': np.hstack([p2[:, 0:3], [[0], [0], [0]]])})
    return out


def _points_in_box(rng, box, n):
    x, y, z, l, h, w, yaw = [float(v) for v in box]
    local = np.c_[rng.uniform(-l / 2, l / 2, n), rng.uniform(-h, 0, n), rng.uniform(-w / 2, w / 2, n)]
    c, s = np.cos(yaw), np.sin(yaw)
    rot = np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]])
    return local.dot(rot.T) + [x, y, z]


def _margins_ok(boxes, cand_xyz, calib, stats):
    """False when a truncation rate is within MARGIN of 0.4 or a candidate within MARGIN of a kept box's face."""
    from pointgnn_b200.dataset import kitti_dataset
    from pointgnn_b200.models import nms
    if len(boxes) == 0:
        return True
    for corners, box in zip(nms.boxes_3d_to_corners(boxes), boxes):
        img = np.matmul(np.hstack([corners, np.ones([8, 1])]), np.transpose(calib['cam_to_image']))
        xy = (img / img[:, [2]])[:, :2]
        (xmin, ymin), (xmax, ymax) = np.amin(xy, axis=0), np.amax(xy, axis=0)
        cx0, cy0, cx1, cy1 = max(xmin, 0.0), max(ymin, 0.0), min(xmax, 1242.0), min(ymax, 375.0)
        trunc = 1.0 - (cy1 - cy0) * (cx1 - cx0) / ((ymax - ymin) * (xmax - xmin))
        if abs(trunc - 0.4) < MARGIN:
            return False
        stats['dropped' if trunc > 0.4 else ('cut' if trunc > 0 else 'whole')] += 1
        if trunc > 0.4 or len(cand_xyz) == 0:
            continue
        lab = dict(zip(('x3d', 'y3d', 'z3d', 'length', 'height', 'width', 'yaw'), box))
        normals, lower, upper = kitti_dataset.box3d_to_normals(lab)
        proj = np.matmul(cand_xyz, np.transpose(normals))
        scale = np.maximum(1.0, np.abs(np.concatenate([lower, upper])))
        if np.any(np.abs(proj - lower) < MARGIN * scale[:3]) or np.any(np.abs(proj - upper) < MARGIN * scale[3:]):
            return False
        stats['inside'] += int(kitti_dataset.sel_xyz_in_box3d(lab, cand_xyz).sum())
    return True


def _random_frame(rng, calib, stats):
    """-> (labels [D], boxes [D,7], scores [D], vertices [K,3], cand (v, c) pairs [B,2]) of one frame."""
    while True:
        num_boxes = int(rng.choice([0, 1, 3, 8, 20]))
        fx, cx = float(calib['cam_to_image'][0, 0]), float(calib['cam_to_image'][0, 2])
        boxes = []
        for _ in range(num_boxes):
            kind = int(rng.integers(0, 5))
            z = rng.uniform(6, 45)
            x = rng.uniform(-0.6, 0.6) * z * cx / fx
            if kind == 1:      # across the left edge
                x = (0 - cx) / fx * z + rng.uniform(-3, 3)
            elif kind == 2:    # across the right edge
                x = (1242 - cx) / fx * z + rng.uniform(-3, 3)
            elif kind == 3:    # near: across the bottom edge
                z = rng.uniform(3, 8)
                x = rng.uniform(-2, 2)
            box = [x, rng.uniform(1.2, 2.0), z, rng.uniform(3, 5), rng.uniform(1.3, 2.0), rng.uniform(1.4, 2.0),
                   rng.uniform(-np.pi, np.pi)]
            boxes.append(box)
            if kind == 4:      # a second box behind this one, overlapping it
                boxes.append([box[0] + rng.uniform(-0.5, 0.5), box[1], box[2] + rng.uniform(1, 2.5)] + box[3:6]
                             + [rng.uniform(-np.pi, np.pi)])
        boxes = np.array(boxes, np.float32).reshape(-1, 7)
        parts = [np.c_[rng.uniform(-20, 20, 60), rng.uniform(-1, 2.5, 60), rng.uniform(3, 50, 60)]]
        for box in boxes:
            if rng.uniform() < 0.6:
                parts.append(_points_in_box(rng, box, int(rng.integers(20, 200))))
        vertices = np.concatenate(parts).astype(np.float32)
        num_cand = 0 if (len(boxes) and rng.uniform() < 0.15) else int(rng.integers(1, 2 * len(vertices)))
        flat = np.sort(rng.choice(len(vertices) * 2, size=min(num_cand, 2 * len(vertices)), replace=False))
        cand = np.c_[flat // 2, 1 + flat % 2]          # classes 1 and 2: a vertex may appear twice
        if _margins_ok(boxes, vertices[cand[:, 0]], calib, stats):
            labels = np.ones(len(boxes), np.int32)
            scores = rng.uniform(0.3, 1.0, len(boxes)).astype(np.float32)
            return labels, boxes, scores, vertices, cand


def _run_kernel(frames, use_box_score):
    """frames: list of (labels, boxes, scores, vertices, cand pairs, calib) -> kitti_labels_from_rows per frame."""
    from pointgnn_b200 import run
    from pointgnn_b200.models import postprocess
    dev = torch.device('cuda')
    det_fp, cand_fp, cand_index, offset = [0], [0], [], 0
    for _, boxes, _, vertices, cand, _ in frames:
        det_fp.append(det_fp[-1] + len(boxes))
        cand_fp.append(cand_fp[-1] + len(cand))
        cand_index.append((cand[:, 0] + offset) * NUM_CLASSES + cand[:, 1])
        offset += len(vertices)

    def cat(i, dtype, width=None):
        a = np.concatenate([np.asarray(f[i], dtype).reshape((-1,) + (() if width is None else (width,)))
                            for f in frames])
        return torch.from_numpy(a).to(dev)
    det = {'label': cat(0, np.int32), 'box': cat(1, np.float32, 7), 'score': cat(2, np.float32),
           'frame_ptr': torch.tensor(det_fp, dtype=torch.int32, device=dev),
           'cand_index': torch.from_numpy(np.concatenate(cand_index).astype(np.int32)).to(dev),
           'cand_frame_ptr': torch.tensor(cand_fp, dtype=torch.int32, device=dev)}
    xyz = cat(3, np.float32, 3)
    cti = np.stack([f[5]['cam_to_image'] for f in frames])
    rows, row_fp = postprocess.kitti_rows(det, xyz, cti, NUM_CLASSES, use_box_score)
    rows = rows.cpu().numpy()
    per_frame = run.kitti_labels_from_rows(rows, len(frames), 'Car')
    assert row_fp.cpu().tolist() == list(np.cumsum([0] + [len(p) for p in per_frame]))
    return per_frame


def _compare(frames, use_box_score):
    from pointgnn_b200 import run
    got = _run_kernel(frames, use_box_score)
    rows = 0
    for f, (labels, boxes, scores, vertices, cand, calib) in enumerate(frames):
        want = run.kitti_labels(labels, boxes, scores, vertices[cand[:, 0]], calib, 'Car', use_box_score)
        assert len(got[f]) == len(want), (f, len(got[f]), len(want))
        for g, w in zip(got[f], want):
            assert g[:4] == w[:4]
            for a, b in zip(g[4:8], w[4:8]):          # clipped 2-D box: float64 (np.amin's, or Python's 0.0 / 1242.0)
                assert isinstance(a, float) and isinstance(b, float)
                assert abs(a - b) <= 1e-9 * abs(b), (f, g, w)
            for a, b in zip(g[8:15], w[8:15]):        # h, w, l, x, y, z, yaw: the float32 box values
                assert type(a) is np.float32 and type(b) is np.float32
                assert a.tobytes() == b.tobytes(), (f, g, w)
            assert type(g[15]) is type(w[15]), (type(g[15]), type(w[15]))
            assert abs(g[15] - w[15]) <= 1e-9 * abs(w[15]), (f, g[15], w[15])
        rows += len(want)
    return rows


def test_reference_detections_match_numpy_writer():
    from pointgnn_b200.dataset import kitti_dataset
    g = dict(np.load(os.path.join(GOLDEN, 'post_car.npz')))
    calib = kitti_dataset.parse_calib(CALIB_FILE)
    cand_index = g['cand_index'].astype(np.int64)
    cand = np.c_[cand_index // NUM_CLASSES, cand_index % NUM_CLASSES]
    frame = (g['uncertainty_label'].astype(np.int32), g['uncertainty_box'].astype(np.float32),
             g['uncertainty_score'].astype(np.float32), g['points_xyz'].astype(np.float32), cand, calib)
    for use_box_score in (True, False):
        assert _compare([frame], use_box_score) > 0
    # several copies of the frame in one batch, with an empty frame between them
    empty = (np.zeros(0, np.int32), np.zeros((0, 7), np.float32), np.zeros(0, np.float32), frame[3][:5],
             cand[:0], calib)
    assert _compare([frame, empty, frame], True) > 0


@pytest.mark.parametrize('seed', range(3))
def test_random_batches_match_numpy_writer(seed):
    rng = np.random.default_rng(seed)
    calibs = _calibs()
    stats = {'dropped': 0, 'cut': 0, 'whole': 0, 'inside': 0}
    for num_frames in range(1, 10):
        frames = []
        for _ in range(num_frames):
            calib = calibs[int(rng.integers(0, len(calibs)))]
            frames.append(_random_frame(rng, calib, stats) + (calib,))
        rows = _compare(frames, True)
        assert _compare(frames, False) == rows
    # the 45 frames exercise both sides of the filter, boxes cut by an edge, and the rescoring
    assert stats['dropped'] > 0 and stats['cut'] > 0 and stats['inside'] > 0, stats


def test_all_frames_empty():
    calib = _calibs()[0]
    empty = (np.zeros(0, np.int32), np.zeros((0, 7), np.float32), np.zeros(0, np.float32),
             np.zeros((3, 3), np.float32), np.zeros((0, 2), np.int64), calib)
    assert _run_kernel([empty, empty], True) == [[], []]


def test_surviving_box_with_nonpositive_length_is_an_error():
    from pointgnn_b200 import _lib, run
    calib = _calibs()[0]
    vertices = np.array([[0.0, 1.0, 20.0]], np.float32)
    cand = np.array([[0, 1]])
    visible = np.array([[0.0, 1.6, 20.0, -3.9, 1.5, 1.6, 0.3]], np.float32)
    with pytest.raises(AssertionError):
        run.kitti_labels(np.ones(1, np.int32), visible, np.ones(1, np.float32), vertices, calib, 'Car', True)
    with pytest.raises(_lib.PointGNNError, match='length'):
        _run_kernel([(np.ones(1, np.int32), visible, np.ones(1, np.float32), vertices, cand, calib)], True)
    # a box the truncation filter drops never reaches the assert
    hidden = np.array([[-40.0, 1.6, 10.0, -3.9, 1.5, 1.6, 0.3]], np.float32)
    assert run.kitti_labels(np.ones(1, np.int32), hidden, np.ones(1, np.float32), vertices, calib, 'Car', True) == []
    assert _run_kernel([(np.ones(1, np.int32), hidden, np.ones(1, np.float32), vertices, cand, calib)], True) == [[]]
